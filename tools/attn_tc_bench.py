#!/usr/bin/env python
"""Dense attention, tensor-core (wgmma 3xTF32, attention_tc.cu) vs fp32 SIMT (attention.cu), CUDA-event timed through the C ABI.
Shapes: Whisper encoder self-attention of a 16-window chunk (B = 16, H = 12, T = 512) and the DiT block (B = 2, H = 12, T = 1024, +-128 band)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mapperatorinator_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
for name, B, H, T, mode, band in (("encoder 16 windows", 16, 12, 512, "none", 0), ("DiT chunk (CFG pair)", 2, 12, 1024, "band", 128),
                                  ("encoder 1 window", 1, 12, 512, "none", 0)):
    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(B, T, H * 64, generator=g).cuda() for _ in range(3))
    flops = 4.0 * B * H * T * T * 64 * (1.0 if mode == "none" else min(1.0, 2.0 * band / T))
    res = {}
    for tc in (0, 1):
        _lib.check(lib.mb200_set_attention_tc(tc, 64))
        for _ in range(3):
            out = ops.attention(q, k, v, H, 1.0, mode, 0, band=band)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            out = ops.attention(q, k, v, H, 1.0, mode, 0, band=band)
        e1.record()
        torch.cuda.synchronize()
        res[tc] = (e0.elapsed_time(e1) / 20.0, out)
    _lib.check(lib.mb200_set_attention_tc(1, 256))
    err = (res[0][1] - res[1][1]).abs().max().item()
    print(f"{name:24s} SIMT {res[0][0] * 1e3:8.1f} us   wgmma (prep + kernel) {res[1][0] * 1e3:8.1f} us   "
          f"{flops / res[1][0] / 1e9:6.1f} TFLOP/s algorithmic   max |diff| {err:.2e}")
