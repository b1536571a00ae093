"""Generate tests/golden/beam_reference.npz from the UNMODIFIED reference `server.model_generate` with `num_beams > 1`.

TEST INFRASTRUCTURE.  Usage:  MAPPERATORINATOR_REFERENCE=<checkout of the original project> python -m oracle.make_beam_golden
A recipe of its own, so regenerating the beam fixture leaves the other fixtures byte-identical.  Tiny model, torchaudio
front end, weights `init_model_state_dict(cfg, 0)`.  Per case it stores the reference ids and generated-token counts, the
reference's `sequences_scores` (captured from the same `generate` call) and the oracle's smallest decisive score gap.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mapperatorinator_b200 import TokenLayout, tiny_model_config  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402
from oracle import beam, cases, ref_build  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
MIN_GAP = 1e-4


def make_beam_golden():
    import transformers
    torch.set_grad_enabled(False)
    meta = dict(torch=torch.__version__, transformers=transformers.__version__)
    tok = ref_build.reference_tokenizer()
    layout = TokenLayout.from_json(os.path.join(OUT, "tokenizer_v29.json"))
    from osuT5.osuT5.inference.server import model_generate
    melc = cases.MODEL_FLAVOURS["torchaudio"]
    cfg = tiny_model_config(mel=melc)
    model, tok2, _ = ref_build.reference_model(cfg, tok=tok, mel_impl=melc.implementation)
    sd = init_model_state_dict(cfg, 0)
    ref_build.load_state_dict_into_reference(model, sd)
    captured = {}
    plain_generate = model.generate

    def generate_with_scores(*a, **k):        # the same call, asked for its sequences_scores as well
        r = plain_generate(*a, **k, return_dict_in_generate=True, output_scores=True)
        captured["scores"] = r.sequences_scores
        return r.sequences

    model.generate = generate_with_scores
    out = {}
    for name, (prompt, neg, gk, seed) in beam.beam_cases().items():
        B = prompt.shape[0]
        mk = dict(inputs=cases.model_pcm(cfg, B, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0),
                  negative_prompt=neg, negative_prompt_attention_mask=None if neg is None else neg.ne(0))
        ids, stats = model_generate(model, tok2, dict(mk), dict(gk))
        o_ids, o_stats, o_scores, gap = beam.beam_generate(sd, cfg, layout, dict(mk), dict(gk))
        ok = np.array_equal(o_ids.numpy(), ids.numpy())
        print(f"{name}: L={ids.shape[1]} counts={stats['generated_tokens_per_sample']} oracle_match={ok} gap={gap:.3g} "
              f"score_diff={float((o_scores - captured['scores'].float()).abs().max()):.3g}")
        if gap < MIN_GAP:
            raise SystemExit(f"{name}: smallest decisive gap {gap} < {MIN_GAP}; pick another seed")
        out[f"{name}/ids"] = ids.numpy()
        out[f"{name}/counts"] = np.array(stats["generated_tokens_per_sample"])
        out[f"{name}/scores"] = captured["scores"].float().numpy()
        out[f"{name}/min_gap"] = np.array(gap)
    np.savez_compressed(os.path.join(OUT, "beam_reference.npz"), **out, **{f"meta_{k}": v for k, v in meta.items()})


if __name__ == "__main__":
    make_beam_golden()
