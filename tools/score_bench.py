#!/usr/bin/env python
"""MaiMod's scoring of given tokens, two ways, at v29 (whisper-small) dimensions with seeded weights, B = 8 windows per call:
  (a) today's path: `server.model_forward` (the [B, L, V] fp32 logits copied to the host), then processor.py:519-525 in CPU torch;
  (b) `server.model_score`: the same teacher-forced pass, projection in row chunks, statistics on the device, four [B, L] arrays back.
Per prompt length L it reports:
  * wall time of each arm (host clock around the whole call, which ends in a device-to-host copy), median and min over --reps,
    the arms alternating;
  * device span of each arm (first to last GPU activity of one call, kernels and copies, from a torch.profiler run of its own), and
    the split of arm (b)'s kernel time into encoder / decoder prefill (to the final LayerNorm) / vocabulary projection / statistics;
  * bytes copied to the host by each arm;
  * the statistics kernel's time per call and the fraction of the HBM byte floor it reaches: it reads every projected row once,
    rows x V x 4 bytes over the data-sheet 3.35 TB/s (rows include the overlap of the last chunk).
Usage: python tools/score_bench.py [--out tools/score_bench_result.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mapperatorinator_b200 import v29_model_config  # noqa: E402
from mapperatorinator_b200.modeling import B200Mapperatorinator  # noqa: E402
from mapperatorinator_b200.server import model_forward, model_score  # noqa: E402
from mapperatorinator_b200.weights import init_model_state_dict  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet, HBM3 (not a measured peak)
CHUNK_ROWS = 3072                   # SCORE_CHUNK_ROWS of engine_model.cu
GEMM_KERNELS = ("gemm_tf32x3_kernel", "tf32_split_kernel", "gemm_f32_kernel", "gemm_splitk_reduce_kernel")


def host_scores(logits: torch.Tensor, ids: torch.Tensor) -> dict:
    """processor.py:519-525 on every row of the call (MaiMod runs it slice by slice over the same rows)."""
    z, y = logits[:, :-1], ids[:, 1:]
    probs = z.softmax(dim=-1)
    entropy = -torch.sum(probs * torch.log2(probs + 1e-10), dim=-1)
    surprisal = -torch.log2(probs.gather(-1, y.clamp(max=z.shape[-1] - 1)[..., None])[..., 0] + 1e-10)
    relative = torch.where(entropy > 0, surprisal / entropy, torch.zeros_like(entropy))
    return dict(entropy=entropy, surprisal=surprisal, relative=relative, suggested=z.argmax(dim=-1))


def case(cfg, B: int, L: int):
    g = torch.Generator().manual_seed(L)
    ids = torch.randint(17, cfg.vocab_size_in, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.bool)
    for b in range(B):
        npad = (b * L) // (2 * B)                 # MaiMod left-pads every window to the song's longest prompt
        ids[b, :npad] = 0
        mask[b, :npad] = False
    return ids, mask


def profile_call(call):
    """One call under torch.profiler -> (device span us, {kernel name: summed us}, ordered kernel list)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    span = ev[-1].time_range.end - ev[0].time_range.start
    return span, ev


def split_b(ev) -> dict:
    """Kernel time of a model_score call: encoder (before the decoder embedding), prefill (embedding .. final LayerNorm),
    projection (GEMM kernels after it), statistics (score_rows_kernel)."""
    k = [e for e in ev if not e.name.startswith("Memcpy") and not e.name.startswith("Memset")]
    i_emb = next(i for i, e in enumerate(k) if "embed_kernel" in e.name)
    first_stats = next(i for i, e in enumerate(k) if "score_rows_kernel" in e.name)
    i_ln = max(i for i in range(first_stats) if "layernorm_kernel" in k[i].name)
    dur = lambda es: sum(e.time_range.end - e.time_range.start for e in es)
    tail = k[i_ln + 1:]
    return {"encoder_us": dur(k[:i_emb]), "prefill_us": dur(k[i_emb:i_ln + 1]),
            "projection_us": dur([e for e in tail if any(n in e.name for n in GEMM_KERNELS)]),
            "stats_us": dur([e for e in tail if "score_rows_kernel" in e.name]),
            "stats_launches": sum("score_rows_kernel" in e.name for e in tail)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "score_bench_result.json"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lengths", default="256,512,1024,2048")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs the GPU"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cfg = v29_model_config()
    B, V = 8, cfg.vocab_size_out
    model = B200Mapperatorinator(cfg, init_model_state_dict(cfg, 0), max_windows=B, max_batch=B)
    pcm = torch.randn(B, cfg.samples_per_window, generator=torch.Generator().manual_seed(0)) * 0.1
    res = {"gpu": gpu, "torch_threads": torch.get_num_threads(),
           "config": f"v29 (whisper-small: d 768, 12+12 layers, 12 heads, ffn 3072, V {V}), seeded weights, B = {B}, fp32",
           "arm_a": "server.model_forward, then processor.py:519-525 in CPU torch on its output",
           "arm_b": "server.model_score", "results": []}
    for L in [int(x) for x in args.lengths.split(",")]:
        ids, mask = case(cfg, B, L)
        mk = dict(inputs=pcm, decoder_input_ids=ids, decoder_attention_mask=mask)
        arm_a = lambda: host_scores(model_forward(model, mk, dict(precision="fp32")), ids)
        arm_b = lambda: model_score(model, mk, dict(precision="fp32"))
        for _ in range(args.warmup):
            arm_a(); arm_b()
        ta, tb = [], []
        for _ in range(args.reps):
            for arm, ts in ((arm_a, ta), (arm_b, tb)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                arm()
                ts.append((time.perf_counter() - t0) * 1e3)
        ta.sort(); tb.sort()
        span_a, _ = profile_call(lambda: model_forward(model, mk, dict(precision="fp32")))
        span_b, ev_b = profile_call(arm_b)
        sp = split_b(ev_b)
        R = B * L
        rows = R if R <= CHUNK_ROWS else -(-R // CHUNK_ROWS) * CHUNK_ROWS
        floor_us = rows * V * 4 / HBM_BYTES_PER_S * 1e6
        r = {"L": L, "rows": R, "chunks": sp["stats_launches"],
             "a_wall_ms_median": ta[len(ta) // 2], "a_wall_ms_min": ta[0], "b_wall_ms_median": tb[len(tb) // 2], "b_wall_ms_min": tb[0],
             "speedup_median": ta[len(ta) // 2] / tb[len(tb) // 2],
             "a_device_span_ms": span_a / 1e3, "b_device_span_ms": span_b / 1e3,
             "a_bytes_to_host": R * V * 4, "b_bytes_to_host": R * (3 * 4 + 8),
             "b_split_us": {k: v for k, v in sp.items() if k != "stats_launches"},
             "stats_rows_read": rows, "stats_byte_floor_us": floor_us, "stats_frac_of_byte_floor": floor_us / sp["stats_us"]}
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
