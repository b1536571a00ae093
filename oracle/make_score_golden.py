"""Generate tests/golden/score_reference.npz: MaiMod's per-token scores on the logits of the UNMODIFIED reference
`server.model_forward` (the teacher-forced pass `Processor.ai_mod` makes, processor.py:421-579).

TEST INFRASTRUCTURE.  Usage:  MAPPERATORINATOR_REFERENCE=<checkout of the original project> python -m oracle.make_score_golden
A recipe of its own, so regenerating this fixture leaves the other fixtures byte-identical.  Tiny model, torchaudio front end,
weights `init_model_state_dict(cfg, 0)`, PCM `cases.model_pcm(cfg, 3, 6)`, ids / mask `score.score_case(cfg)` (3 windows, 40 / 300 /
700 real tokens left-padded to 700).  Stores ids, mask, the four [B, L] arrays and the top-2 logit gap of each scored row.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mapperatorinator_b200 import tiny_model_config  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402
from oracle import cases, ref_build, score  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
PCM_SEED = 6


def make_score_golden():
    import transformers
    torch.set_grad_enabled(False)
    meta = dict(torch=torch.__version__, transformers=transformers.__version__)
    tok = ref_build.reference_tokenizer()
    from osuT5.osuT5.inference.server import model_forward
    melc = cases.MODEL_FLAVOURS["torchaudio"]
    cfg = tiny_model_config(mel=melc)
    model, _, _ = ref_build.reference_model(cfg, tok=tok, mel_impl=melc.implementation)
    ref_build.load_state_dict_into_reference(model, init_model_state_dict(cfg, 0))
    ids, mask = score.score_case(cfg)
    mk = dict(inputs=cases.model_pcm(cfg, ids.shape[0], PCM_SEED), decoder_input_ids=ids, decoder_attention_mask=mask)
    logits = model_forward(model, dict(mk), dict(precision="fp32", cfg_scale=1.0))
    out = score.score_from_logits(logits, ids)
    print(f"logits {tuple(logits.shape)}; targets >= V: {int((ids[:, 1:] >= cfg.vocab_size_out).sum())}; "
          f"min top-2 gap {float(np.nanmin(out['top2_gap'].numpy())):.2e}")
    np.savez_compressed(os.path.join(OUT, "score_reference.npz"), ids=ids.numpy(), mask=mask.numpy(),
                        **{k: v.numpy() for k, v in out.items()}, **{f"meta_{k}": v for k, v in meta.items()})


if __name__ == "__main__":
    make_score_golden()
