#!/usr/bin/env python
"""Time of one decoder prefill (+ first token) at the bench's prompt lengths, v29 dimensions, set against the FMA and byte floors.

A `generate` call with max_length = P + 1 runs the prefill, the final LayerNorm + vocabulary projection of the last row and the first
selection, and nothing else.  Two numbers per prompt length:
  * call time: CUDA events around the whole call (it ends in a device sync, so this includes its host staging and read-back);
  * device time: from a torch.profiler run of its own, the span from the start of the prefill's embedding kernel to the end of the
    first-token selection kernel of each call (the launches of the prefill graph and the gaps between them), and the summed kernel
    time inside that span.  The floor fractions are taken against the device span.
Usage: python tools/prefill_bench.py [--out tools/prefill_bench_result.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from mapperatorinator_b200 import TokenLayout, v29_model_config  # noqa: E402
from mapperatorinator_b200.modeling import B200Mapperatorinator  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

FP32_FMA_PER_S = 67e12 / 2          # H100 SXM data sheet, FP32 non-tensor (not a measured peak)
HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet, HBM3 (not a measured peak)


def floors(cfg, P: int) -> dict:
    """FMAs the prefill needs at M = P rows (no padding) and the bytes it must read at least once (layer weights + cross K/V)."""
    d, f, L, T, V = cfg.d_model, cfg.ffn_dim, cfg.decoder_layers, cfg.src_seq_len // 2, cfg.vocab_size_out
    gemm = P * L * (3 * d * d + d * d + d * d + d * d + 2 * d * f)
    attn = 2 * L * (P * P + P * T) * d          # QK^T and PV over all heads; causal self-attention counted in full
    fma = gemm + attn + V * d
    wbytes = 4 * (L * (6 * d * d + 2 * d * f + 13 * d + f) + V * d)      # weights + biases + LayerNorms the prefill reads
    kvbytes = 4 * L * T * 2 * d
    return {"fma": fma, "bytes": wbytes + kvbytes, "fma_floor_us": fma / FP32_FMA_PER_S * 1e6, "byte_floor_us": (wbytes + kvbytes) / HBM_BYTES_PER_S * 1e6}


def device_time(call, n: int):
    """Median over n calls of (embedding-kernel start -> selection-kernel end, summed kernel time in between), in us."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("Mem")),
                key=lambda e: e.time_range.start)
    spans, busy, t0, acc = [], [], None, 0.0
    for e in ev:
        if "embed_kernel" in e.name:
            t0, acc = e.time_range.start, 0.0
        if t0 is None:
            continue
        acc += e.time_range.end - e.time_range.start
        if "sample_kernel" in e.name:
            spans.append(e.time_range.end - t0)
            busy.append(acc)
            t0 = None
    assert len(spans) == n, f"found {len(spans)} prefills in the trace, expected {n}"
    spans.sort(); busy.sort()
    return spans[n // 2], busy[n // 2]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "prefill_bench_result.json"))
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    cfg = v29_model_config()
    layout = TokenLayout.from_json(os.path.join(ROOT, "tests", "golden", "tokenizer_v29.json"))
    model = B200Mapperatorinator(cfg, init_model_state_dict(cfg, 0), max_windows=4, max_batch=2)
    windows, _, _ = bench.segment(bench.synth_song(0, 30.0), cfg)
    model.engine.encode(windows[:2].cuda(), 0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "config": "v29 (whisper-small decoder: d 768, 12 layers, 12 heads, ffn 3072), 1 row, greedy", "results": []}
    for P in (18, 50):
        base = bench.COND_IDS + [1, 9]
        prompt = torch.tensor([(base + list(range(100, 100 + P)))[:P]])
        gk = bench.gen_kwargs(1, 211, P)
        gk["max_length"] = P + 1
        gk["min_new_tokens"] = 1
        for _ in range(5):
            model.engine.generate([1], prompt, prompt.ne(0), layout, gk)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model.engine.generate([1], prompt, prompt.ne(0), layout, gk)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) * 1000)
        times.sort()
        us = times[len(times) // 2]
        span, busy = device_time(lambda: model.engine.generate([1], prompt, prompt.ne(0), layout, gk), 20)
        fl = floors(cfg, P)
        res["results"].append({"P": P, "call_us_median": us, "call_us_min": times[0], "device_span_us_median": span,
                               "device_kernel_us_median": busy, **fl,
                               "frac_of_fma_floor": fl["fma_floor_us"] / span, "frac_of_byte_floor": fl["byte_floor_us"] / span})
    print(json.dumps(res, indent=1))
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
