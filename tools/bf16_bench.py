"""Token-loop step time of a bf16-loaded model (bf16 token-loop weight store) against the same values served from fp32, at whisper-small
dimensions (v29 config, `init_model_state_dict(cfg, 0)` weights): sd16 = {k: v.bfloat16()}, sd32 = {k: v.float() for sd16}.

The sd16 engine streams its bf16 store on every driver, the sd32 engine its fp32 weights.  Per case, the two engines alternate inside one process after every shape has been warmed; --reps pairs, best and
median of each side, and the ids of every pair asserted equal.  Step time = (time of a call with NEW new tokens - time of one with 8)
/ (NEW - 8), each call timed by CUDA events recorded on the engine's stream before and after it (the call ends in a device
synchronise), so prefill, staging and hand-back cancel out.  Cases:
  * dataflow megakernel at rows 1 and 2, the grid-barrier megakernel at rows 1, the CUDA-graph driver at rows 1, 8 and 16 (greedy,
    the bench's window kind);
  * beam search 8 items x 2 beams (16 decoder rows, graph driver);
  * the decode stream of tools/continuous_bench.py (32 requests through 8 rows): device ms per replayed step from CUDA events
    around each burst.
Achieved weight bytes per second = the GEMV weight bytes one token step streams (q|k|v, out, cross q, cross out, fc1, fc2 of every
layer + proj_out, at 2 or 4 bytes per element; K/V cache and activation bytes are not counted) over the step time.  The card's name and
power limit are read in the same run.  Needs a GPU; queries the card, changes nothing.
Usage: python tools/bf16_bench.py [--out tools/bf16_bench_result.json] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from collections import deque

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mapperatorinator_b200 import TokenLayout, v29_model_config  # noqa: E402
from mapperatorinator_b200.engine import ModelEngine  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

NEW, SHORT, P = 72, 8, 50
N_REQ, STREAM_ROWS = 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power}


def weight_elems(cfg):
    d, f, L = cfg.d_model, cfg.ffn_dim, cfg.decoder_layers
    return L * (3 * d * d + d * d + d * d + d * d + f * d + d * f) + cfg.vocab_size_out * d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bf16_bench needs a CUDA device: there is nothing to time without one")
    layout = TokenLayout.from_json(os.path.join(ROOT, "tests", "golden", "tokenizer_v29.json"))
    cfg = v29_model_config()
    sd = init_model_state_dict(cfg, 0)
    sd16 = {k: (v.bfloat16() if v.is_floating_point() else v) for k, v in sd.items()}
    sd32 = {k: (v.float() if v.is_floating_point() else v) for k, v in sd16.items()}
    engines = {"bf16": ModelEngine(cfg, sd16, max_windows=N_REQ, max_batch=16), "fp32": ModelEngine(cfg, sd32, max_windows=N_REQ, max_batch=16)}
    assert engines["bf16"].token_weight_dtype == torch.bfloat16 and engines["fp32"].token_weight_dtype == torch.float32
    g = torch.Generator().manual_seed(0)
    pcm = (torch.randn(N_REQ, cfg.samples_per_window, generator=g) * 0.1).cuda()
    for e in engines.values():
        e.encode(pcm, 0)
    prompt = torch.randint(17, 3600, (16, P), generator=g)
    prompt[:, :4] = torch.tensor([3700, 3705, 1, 9])

    def gk(new, beams=1):
        return dict(do_sample=False, num_beams=beams, top_k=0, top_p=0.9, types_first=True, temperature=0.9, timing_temperature=0.1,
                    mania_column_temperature=0.5, taiko_hit_temperature=0.5, max_length=P + new, min_new_tokens=new,
                    lookback_time=4092.0, lookahead_time=3273.6, context_type="map")

    def greedy(mega, rows):
        def call(eng, new):
            eng.set_option("mega", mega)
            try:
                return eng.generate(list(range(rows)), prompt[:rows], None, layout, gk(new))
            finally:
                eng.set_option("mega", 2)
        return call

    def beam_call(eng, new):
        eng.set_option("mega", 0)
        try:
            return eng.generate_beams(list(range(8)), prompt[:8], None, layout, gk(new, 2))[0]
        finally:
            eng.set_option("mega", 2)


    cases = {"dataflow_rows1": (greedy(2, 1), 1), "dataflow_rows2": (greedy(2, 2), 2), "megakernel_rows1": (greedy(1, 1), 1),
             "graph_rows1": (greedy(0, 1), 1), "graph_rows8": (greedy(0, 8), 8), "graph_rows16": (greedy(0, 16), 16),
             "beam_8x2": (beam_call, 16)}

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1000.0, out

    # ---- the decode stream workload of tools/continuous_bench.py ----
    lens = torch.randint(40, 401, (N_REQ,), generator=torch.Generator().manual_seed(0)).tolist()
    gs = torch.Generator().manual_seed(2)
    sprompts = []
    for n in lens:
        p = torch.randint(17, 3600, (n,), generator=gs)
        p[:4] = torch.tensor([3700, 3705, 1, 9])
        sprompts.append(p)
    budgets = torch.randint(16, 129, (N_REQ,), generator=torch.Generator().manual_seed(1)).tolist()

    def sgk(r):
        return dict(gk(budgets[r]), max_length=lens[r] + budgets[r])

    def stream_run(eng):
        out, rows, queue, run_ms = [None] * N_REQ, {}, deque(range(N_REQ)), 0.0
        with eng.open_stream(layout, STREAM_ROWS) as st:
            while queue or st.live_rows:
                while queue and st.free_rows:
                    r = queue.popleft()
                    rows[st.admit(r, sprompts[r], sgk(r))] = r
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                finished = st.run(waiting=len(queue))
                e1.record()
                torch.cuda.synchronize()
                run_ms += e0.elapsed_time(e1)
                for row, ids in finished:
                    out[rows.pop(row)] = ids
            steps = st.steps
        return run_ms / steps, out

    res = {"shape": {"d_model": cfg.d_model, "decoder_layers": cfg.decoder_layers, "ffn_dim": cfg.ffn_dim, "vocab_out": cfg.vocab_size_out,
                     "prompt": P, "new_tokens": [SHORT, NEW], "stream": {"requests": N_REQ, "rows": STREAM_ROWS}},
           "reps": args.reps, "weight_bytes_per_step": {"bf16": 2 * weight_elems(cfg), "fp32": 4 * weight_elems(cfg)}, "cases": {}}
    for name, (call, rows) in cases.items():
        for eng in engines.values():     # warm-up: kernels loaded, graphs captured, phase tables built
            for new in (SHORT, NEW):
                call(eng, new); call(eng, new)
        us = {k: [] for k in engines}
        equal = True
        for _ in range(args.reps):
            outs = {}
            for k, eng in engines.items():
                t_short, _ = timed(lambda: call(eng, SHORT))
                t_new, outs[k] = timed(lambda: call(eng, NEW))
                us[k].append(1e6 * (t_new - t_short) / (NEW - SHORT))
            equal = equal and torch.equal(torch.as_tensor(outs["bf16"]), torch.as_tensor(outs["fp32"]))
        assert equal, f"{name}: ids differ between the bf16 and fp32 stores"
        res["cases"][name] = {"rows": rows, "ids_equal": equal}
        for k in engines:
            res["cases"][name][k] = {"us_per_step_best": min(us[k]), "us_per_step_median": float(np.median(us[k])), "us_all": us[k],
                                     "weight_GB_per_s_best": res["weight_bytes_per_step"][k] / min(us[k]) / 1e3}
        print(name, {k: round(min(us[k]), 1) for k in engines}, flush=True)
    for eng in engines.values():
        stream_run(eng)
    us = {k: [] for k in engines}
    for _ in range(args.reps):
        outs = {}
        for k, eng in engines.items():
            ms, outs[k] = stream_run(eng)
            us[k].append(1000.0 * ms)
        assert all(torch.equal(a, b) for a, b in zip(outs["bf16"], outs["fp32"])), "stream: ids differ between the bf16 and fp32 stores"
    res["cases"]["stream_8_rows"] = {"rows": STREAM_ROWS, "ids_equal": True}
    for k in engines:
        res["cases"]["stream_8_rows"][k] = {"us_per_step_best": min(us[k]), "us_per_step_median": float(np.median(us[k])), "us_all": us[k],
                                            "weight_GB_per_s_best": res["weight_bytes_per_step"][k] / min(us[k]) / 1e3}
    print("stream_8_rows", {k: round(min(us[k]), 1) for k in engines}, flush=True)
    res.update(card())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
