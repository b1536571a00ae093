"""Ragged batched generate against its alternatives at whisper-small dimensions (v29 config, `init_model_state_dict` weights):
8 requests with seeded prompt lengths in 40..400, 64 new tokens each (fixed with min_new_tokens), encoder states resident.

Three arms, alternated inside one process after every shape has been warmed, timed with CUDA events around the whole arm
(prefills included — they are part of what a caller waits for):
  (i)   the 8 batch-1 `generate()` calls one after another on the default driver (the dataflow megakernel);
  (ii)  one `generate_ragged()` call;
  (iii) one uniform `generate()` call with the prompts left-padded to the longest — the only batched option without the ragged
        call; its ids differ from the batch-1 calls (padding consumes positions), it is here for its time only.
Reports tokens/s and ms per token step (arm time / 64; arm (i): per step of one request, i.e. arm time / (8 * 64)) per arm, the
card's name and power limit read in the same run, and asserts that arm (ii) produced the ids of arm (i).  Needs a GPU; queries the
card, changes nothing.
Usage: python tools/ragged_bench.py [--out tools/ragged_bench_result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from mapperatorinator_b200 import TokenLayout, v29_model_config  # noqa: E402
from mapperatorinator_b200.engine import ModelEngine  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

N, NEW = 8, 64


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
        raise SystemExit("ragged_bench needs a CUDA device: there is nothing to time without one")
    layout = TokenLayout.from_json(os.path.join(ROOT, "tests", "golden", "tokenizer_v29.json"))
    cfg = v29_model_config()
    eng = ModelEngine(cfg, init_model_state_dict(cfg, 0), max_windows=N, max_batch=N)
    g = torch.Generator().manual_seed(0)
    eng.encode((torch.randn(N, cfg.samples_per_window, generator=g) * 0.1).cuda(), 0)
    lens = torch.randint(40, 401, (N,), generator=g).tolist()
    prompts = []
    for P in lens:
        p = torch.randint(17, 3600, (1, P), generator=g)
        p[0, :4] = torch.tensor([3700, 3705, 1, 9])
        prompts.append(p)

    def gk(P):
        return dict(do_sample=False, num_beams=1, top_k=0, top_p=0.9, types_first=True, temperature=0.9, timing_temperature=0.1,
                    mania_column_temperature=0.5, taiko_hit_temperature=0.5, max_length=P + NEW, min_new_tokens=NEW,
                    lookback_time=4092.0, lookahead_time=3273.6, context_type="map")
    Pmax = max(lens)
    padded = torch.zeros(N, Pmax, dtype=torch.long)
    for r, p in enumerate(prompts):
        padded[r, Pmax - p.shape[1]:] = p[0]

    def arm_single():
        return [eng.generate([r], prompts[r], None, layout, gk(lens[r])) for r in range(N)]

    def arm_ragged():
        return eng.generate_ragged([(r, prompts[r][0], gk(lens[r]), None) for r in range(N)], layout)

    def arm_padded():
        return eng.generate(list(range(N)), padded, padded.ne(0), layout, gk(Pmax))

    arms = {"batch1_calls": arm_single, "ragged_call": arm_ragged, "padded_uniform_call": arm_padded}
    for fn in arms.values():             # warm every shape: kernels loaded, prefill and token-step graphs captured
        fn(); fn(); fn()
    single, rag = arm_single(), arm_ragged()
    for r in range(N):
        assert single[r].shape[1] == lens[r] + NEW and torch.equal(single[r], rag[r]), f"request {r}: ragged ids differ from its batch-1 call"
    ms = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    res = {"shape": {"requests": N, "prompt_lengths": lens, "new_tokens": NEW, "d_model": cfg.d_model, "decoder_layers": cfg.decoder_layers,
                     "vocab_out": cfg.vocab_size_out}, "reps": args.reps, "ragged_ids_equal_batch1_calls": True}
    for k, v in ms.items():
        best = min(v)
        steps = N * NEW if k == "batch1_calls" else NEW
        res[k] = {"ms_best": best, "ms_all": v, "tokens_per_s": N * NEW / (best / 1000.0), "ms_per_token_step": best / steps}
    res.update(card())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
