"""Generate tests/golden/ragged_reference.npz: the UNMODIFIED reference `server.model_generate` called with batch size 1 for
every request of every case of oracle/ragged.py (what `Processor.generate_sequential` does, one window at a time).

TEST INFRASTRUCTURE.  Usage:  MAPPERATORINATOR_REFERENCE=<checkout of the original project> python -m oracle.make_ragged_golden
A recipe of its own, so regenerating this fixture leaves the other fixtures byte-identical.  Tiny model, torchaudio front end,
weights `init_model_state_dict(cfg, 0)`.  Per request it stores the reference ids and the generated-token count.
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
from oracle import cases, generate, ragged, ref_build  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def make_ragged_golden():
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
    out = {}
    for name, reqs in ragged.ragged_cases().items():
        for r, req in enumerate(reqs):
            mk = ragged.model_kwargs(cfg, req)
            ids, stats = model_generate(model, tok2, dict(mk), dict(req["gk"]))
            o_ids, _ = generate.model_generate(sd, cfg, layout, dict(mk), dict(req["gk"]))
            P, L = req["prompt"].shape[1], ids.shape[1]
            eos = layout.eos_token_ids(req["gk"]["lookback_time"], req["gk"]["lookahead_time"], req["gk"]["context_type"])
            how = "eos" if int(ids[0, -1]) in eos else "max_length"
            print(f"{name}[{r}]: P={P} L={L} new={L - P} stop={how} oracle_match={torch.equal(o_ids, ids)} tail={ids[0, P:P + 8].tolist()}")
            out[f"{name}/{r}/ids"] = ids.numpy()
            out[f"{name}/{r}/counts"] = np.array(stats["generated_tokens_per_sample"])
    np.savez_compressed(os.path.join(OUT, "ragged_reference.npz"), **out, **{f"meta_{k}": v for k, v in meta.items()})


if __name__ == "__main__":
    make_ragged_golden()
