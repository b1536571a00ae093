"""Continuous batching (the decode stream) against static batching at whisper-small dimensions (v29 config, `init_model_state_dict`
weights): 32 requests, one resident encoder slot each, seeded prompt lengths in 40..400 as in tools/ragged_bench.py, and per-request
budgets drawn once from a fixed seed over 16..128 new tokens, enforced with min_new_tokens = budget and max_length = P + budget, so
every arm does the same work.  Greedy decoding.  The requests arrive all at once, in index order.

Three arms, alternated inside one process after every shape has been warmed, best and all of --reps:
  (a) one decode stream of 8 rows: requests admitted in order as rows free up, handed back as they finish;
  (b) static batching: waves of 8 requests in arrival order through `generate_ragged` (a wave ends with its longest request);
  (c) the 32 batch-1 `generate()` calls one after another on the default driver.
Reports per arm the wall ms (host clock around work that ends in a device synchronise) and tokens/s, p50 / p90 request latency from
the start of the arm; for the stream the mean rows holding a request per replayed token step (counted at each burst's start), the
device ms per step (CUDA events around each burst, its row-status read included) and the time per admission outside the token steps
(arm wall time minus the bursts' device time, over the 32 admissions: staging, the eager prefill, hand-back); whether all three
arms' ids are equal; the card's name and power limit read in the same run.  Needs a GPU; queries the card, changes nothing.
Usage: python tools/continuous_bench.py [--out tools/continuous_bench_result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from collections import deque

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mapperatorinator_b200 import TokenLayout, v29_model_config  # noqa: E402
from mapperatorinator_b200.engine import ModelEngine  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

N_REQ, ROWS = 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("continuous_bench needs a CUDA device: there is nothing to time without one")
    layout = TokenLayout.from_json(os.path.join(ROOT, "tests", "golden", "tokenizer_v29.json"))
    cfg = v29_model_config()
    eng = ModelEngine(cfg, init_model_state_dict(cfg, 0), max_windows=N_REQ, max_batch=ROWS)
    g = torch.Generator().manual_seed(0)
    eng.encode((torch.randn(N_REQ, cfg.samples_per_window, generator=g) * 0.1).cuda(), 0)
    lens = torch.randint(40, 401, (N_REQ,), generator=g).tolist()
    prompts = []
    for P in lens:
        p = torch.randint(17, 3600, (P,), generator=g)
        p[:4] = torch.tensor([3700, 3705, 1, 9])
        prompts.append(p)
    budgets = torch.randint(16, 129, (N_REQ,), generator=torch.Generator().manual_seed(1)).tolist()

    def gk(r):
        return dict(do_sample=False, num_beams=1, top_k=0, top_p=0.9, types_first=True, temperature=0.9, timing_temperature=0.1,
                    mania_column_temperature=0.5, taiko_hit_temperature=0.5, max_length=lens[r] + budgets[r], min_new_tokens=budgets[r],
                    lookback_time=4092.0, lookahead_time=3273.6, context_type="map")

    stats = {}

    def arm_stream():
        t0 = time.perf_counter()
        out, done_at, rows = [None] * N_REQ, [0.0] * N_REQ, {}
        queue = deque(range(N_REQ))
        run_ms = 0.0
        live_steps = 0
        with eng.open_stream(layout, ROWS) as st:
            while queue or st.live_rows:
                while queue and st.free_rows:
                    r = queue.popleft()
                    rows[st.admit(r, prompts[r], gk(r))] = r
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                live, before = st.live_rows, st.steps
                e0.record()
                finished = st.run(waiting=len(queue))
                e1.record()
                torch.cuda.synchronize()
                run_ms += e0.elapsed_time(e1)
                live_steps += live * (st.steps - before)
                for row, ids in finished:
                    r = rows.pop(row)
                    out[r], done_at[r] = ids, (time.perf_counter() - t0) * 1000.0
            steps = st.steps
        stats["stream"] = dict(steps=steps, run_ms=run_ms, live_row_steps=live_steps)
        return out, done_at

    def arm_waves():
        t0 = time.perf_counter()
        out, done_at = [], []
        for w in range(0, N_REQ, ROWS):
            out += eng.generate_ragged([(r, prompts[r], gk(r), None) for r in range(w, w + ROWS)], layout)
            done_at += [(time.perf_counter() - t0) * 1000.0] * ROWS
        return out, done_at

    def arm_single():
        t0 = time.perf_counter()
        out, done_at = [], []
        for r in range(N_REQ):
            out.append(eng.generate([r], prompts[r][None], None, layout, gk(r)))
            done_at.append((time.perf_counter() - t0) * 1000.0)
        return out, done_at

    arms = {"stream_8_rows": arm_stream, "waves_of_8_ragged": arm_waves, "batch1_calls": arm_single}
    for fn in arms.values():             # warm every shape: kernels loaded, prefill and token-step graphs captured
        fn(); fn()
    ids = {k: fn()[0] for k, fn in arms.items()}
    equal = all(ids[k][r].shape[1] == lens[r] + budgets[r] and torch.equal(ids[k][r], ids["batch1_calls"][r]) for k in ids for r in range(N_REQ))
    ms = {k: [] for k in arms}
    lat = {k: [] for k in arms}
    stream_stats = []
    for _ in range(args.reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, done_at = fn()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1000.0)
            lat[k].append(done_at)
            if k == "stream_8_rows":
                stream_stats.append(dict(stats["stream"]))
    tokens = sum(budgets)
    res = {"shape": {"requests": N_REQ, "rows": ROWS, "prompt_lengths": lens, "new_tokens": budgets, "total_new_tokens": tokens,
                     "d_model": cfg.d_model, "decoder_layers": cfg.decoder_layers, "vocab_out": cfg.vocab_size_out},
           "reps": args.reps, "ids_equal_across_arms": bool(equal)}
    for k in arms:
        b = int(np.argmin(ms[k]))
        res[k] = {"ms_best": ms[k][b], "ms_all": ms[k], "tokens_per_s": tokens / (ms[k][b] / 1000.0),
                  "latency_ms_p50": float(np.percentile(lat[k][b], 50)), "latency_ms_p90": float(np.percentile(lat[k][b], 90))}
        if k == "stream_8_rows":
            s = stream_stats[b]
            res[k].update({"replayed_steps": s["steps"], "mean_live_rows_per_step": s["live_row_steps"] / max(1, s["steps"]),
                           "device_ms_per_step": s["run_ms"] / max(1, s["steps"]),
                           "host_ms_per_admission": (ms[k][b] - s["run_ms"]) / N_REQ})
    res["speedup_stream_vs_waves"] = res["waves_of_8_ragged"]["ms_best"] / res["stream_8_rows"]["ms_best"]
    res.update(card())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
