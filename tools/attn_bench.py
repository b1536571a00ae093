#!/usr/bin/env python
"""Decode-attention roofline at batch: B songs decode one token each (BASELINE config[3]: 8 songs per GPU; swept to 64 rows).
The split-KV decode attention kernel reads every row's cross K|V (512 keys) and self K|V (ctx keys) of all 12 layers once per
token: bytes = B * 12 * 2 * (512 + ctx) * 768 * 4.  Prints achieved GB/s of the attention launches alone (CUDA events around each
launch, `mb200_model_profile_step`) against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), plus the GEMV and sample totals of the same token step."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from mapperatorinator_b200 import TokenLayout, _lib, v29_model_config  # noqa: E402
from mapperatorinator_b200.modeling import B200Mapperatorinator  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

batches = [int(a) for a in sys.argv[1:]] or [1, 8, 32, 64]
BMAX = max(batches)
cfg = v29_model_config()
layout = TokenLayout.from_json(os.path.join(ROOT, "tests", "golden", "tokenizer_v29.json"))
model = B200Mapperatorinator(cfg, init_model_state_dict(cfg, 0), max_windows=BMAX, max_batch=BMAX)
windows, _, _ = bench.segment(bench.synth_song(0, 90.0), cfg)
for i in range(0, BMAX, 16):
    model.engine.encode(windows[i:i + 16].cuda(), i)
lib = _lib.load()
peak = 3350.0
P = 50
for B in batches:
    prompt = torch.tensor([bench.prompt_for(1, [list(range(100 + r, 164 + r))]) for r in range(B)])
    gk = bench.gen_kwargs(1, 211, P)
    gk["max_length"] = P + 2
    gk["min_new_tokens"] = 2
    model.engine.generate(list(range(B)), prompt, prompt.ne(0), layout, gk)        # sets up the decode state for B rows
    out = np.zeros(4, dtype=np.float32)
    iters = 20
    _lib.check(lib.mb200_model_profile_step(model.engine.handle, B, B, P + bench.NEW_TOKENS, iters, out.ctypes.data, torch.cuda.current_stream().cuda_stream))
    ctx = P + 1 + (iters - 1) / 2
    nbytes = B * cfg.decoder_layers * 2 * (cfg.max_source_positions + ctx) * cfg.d_model * 4
    n_attn = (int(out[3]) // 1000) % 1000
    gbs = nbytes / (out[1] * 1e-6) / 1e9
    print(f"B={B:3d}: attention {out[1]:8.1f} us/token over {n_attn} launches ({nbytes / 1e6:8.1f} MB) -> {gbs:7.1f} GB/s = {gbs / peak:5.3f} of {peak:.0f} GB/s;"
          f"  gemv {out[0]:8.1f} us  sample {out[2]:6.1f} us")
