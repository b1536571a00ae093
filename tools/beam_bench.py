"""Beam-search token-loop timing at whisper-small dimensions (v29 config, `init_model_state_dict` weights) in the shape of the
timing pre-pass (`SuperTimingGenerator`: num_beams 2, top_k 50 passed and ignored): B = 8 items x K = 2 beams = 16 decoder rows,
a 100-token prompt, 64 new tokens.

Reports, from one run on the GPU it executes on:
  * ms per token step of the beam path and of the greedy CUDA-graph path at the same row count (16 greedy rows), each as
    (time of a 64-token call - time of an 8-token call) / 56, so the prefill and the call set-up cancel;
  * the share of the beam kernels (scores; selection + reorder gather) in the device time of the beam call's kernels, from
    torch.profiler CUDA activity in a separate run;
  * the card name and power limit, read in the same run.
Usage: python tools/beam_bench.py [--out results/beam_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from mapperatorinator_b200 import TokenLayout, v29_model_config  # noqa: E402
from mapperatorinator_b200.engine import ModelEngine  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

B, K, P, NEW = 8, 2, 100, 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    layout = TokenLayout.from_json(os.path.join(ROOT, "tests", "golden", "tokenizer_v29.json"))
    cfg = v29_model_config()
    eng = ModelEngine(cfg, init_model_state_dict(cfg, 0), max_windows=16, max_batch=16)
    g = torch.Generator().manual_seed(0)
    eng.encode((torch.randn(16, cfg.samples_per_window, generator=g) * 0.1).cuda(), 0)
    prompt = torch.randint(17, 3600, (16, P), generator=g)
    prompt[:, :4] = torch.tensor([3700, 3705, 1, 5])

    def gk(new, beams):
        return dict(do_sample=False, num_beams=beams, top_k=50, top_p=0.9, types_first=True, temperature=0.9, timing_temperature=0.3,
                    mania_column_temperature=0.9, taiko_hit_temperature=0.9, max_length=P + new, min_new_tokens=new,
                    lookback_time=0.0, lookahead_time=0.0, context_type="timing")

    def beam_call(new):
        return eng.generate_beams(list(range(B)), prompt[:B], None, layout, gk(new, K))

    def greedy_call(new):
        return eng.generate(list(range(16)), prompt, None, layout, gk(new, 1))

    eng.set_option("mega", 0)            # the greedy CUDA-graph path (16 rows never take the megakernels anyway)

    def per_step(fn):
        for new in (8, NEW):             # warm up: graphs captured, kernels loaded
            fn(new); fn(new)
        t = {}
        for new in (8, NEW):
            best = float("inf")
            for _ in range(args.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(new)
                torch.cuda.synchronize()
                best = min(best, time.perf_counter() - t0)
            t[new] = best
        return 1000.0 * (t[NEW] - t[8]) / (NEW - 8)

    res = {"shape": {"items": B, "num_beams": K, "decoder_rows": B * K, "prompt": P, "new_tokens": NEW, "d_model": cfg.d_model,
                     "decoder_layers": cfg.decoder_layers, "vocab_out": cfg.vocab_size_out}}
    res["beam_ms_per_token_step"] = per_step(beam_call)
    res["greedy_graph_ms_per_token_step_16_rows"] = per_step(greedy_call)
    ids, scores = beam_call(NEW)
    res["beam_generated_tokens"] = int(ids.shape[1] - P)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        beam_call(NEW)
        torch.cuda.synchronize()
    tot, parts = 0.0, {"beam_scores_kernel": 0.0, "beam_select_kernel": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
        if t <= 0 or "Memcpy" in e.key or "Memset" in e.key:
            continue
        tot += t
        for k in parts:
            if k in e.key:
                parts[k] += t
    res["kernel_time_us_total"] = tot
    res["share_scores"] = parts["beam_scores_kernel"] / tot
    res["share_selection_and_gather"] = parts["beam_select_kernel"] / tot
    res["share_beam_kernels"] = (parts["beam_scores_kernel"] + parts["beam_select_kernel"]) / tot
    res["beam_kernel_us_per_step"] = {k: v / NEW for k, v in parts.items()}
    res.update(card())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
