"""Parity and self-consistency at FULL whisper-small (v29) dimensions, where the tensor-core GEMM, its split-K rules and the
megakernel's row partition are the production ones (the tiny config of test_gpu_model.py picks different tiles and splits).

  * batch invariance: a window's encoder states / a row's GEMM result must be bit-identical whether it is computed alone or
    inside a larger batch (round-1 bug: split-K was chosen from grid fill, so `encode_song` and per-window `model_generate`
    disagreed in the last bit and greedy argmax flipped on 5 of 8 songs);
  * `SongDecoder` (encoder once per song, resident cross-K/V) == one `server.model_generate` call per window, on 3 song seeds;
  * greedy ids vs the CPU oracle through a teacher-forced pass with the first-divergence / top-2-gap report.
"""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _song(seed, seconds, sr=16000):
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    t = np.arange(n) / sr
    x = sum(np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi)) for f in np.geomspace(55, 7000, 8)) / 8
    x = x + rng.normal(0, 0.01, n)
    return (x / np.abs(x).max()).astype(np.float32)


@pytest.fixture(scope="module")
def full():
    from mapperatorinator_b200 import v29_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = v29_model_config()
    sd = init_model_state_dict(cfg, 0)
    return cfg, sd, B200Mapperatorinator(cfg, sd, max_windows=24, max_batch=2)


@pytest.mark.parametrize("M_small,M_big,N,K", [(512, 8192, 768, 768), (512, 2048, 768, 3072), (1024, 4096, 768, 2304), (512, 1536, 2304, 768),
                                               (512, 8192, 3072, 768)])
def test_tc_gemm_rows_do_not_depend_on_batch(M_small, M_big, N, K):
    """Grid split (under-filled grid), in-tile split (large M) and the unsplit shape give the same bits for the same rows."""
    from mapperatorinator_b200 import ops
    g = torch.Generator().manual_seed(N + K)
    a, w = torch.randn(M_big, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K)
    bias, res = torch.randn(N, generator=g), torch.randn(M_big, N, generator=g)
    big = ops.gemm_tc(a.cuda(), w.cuda(), bias.cuda(), "gelu", 1.0, res.cuda()).cpu()
    small = ops.gemm_tc(a[:M_small].cuda().contiguous(), w.cuda(), bias.cuda(), "gelu", 1.0, res[:M_small].cuda().contiguous()).cpu()
    assert torch.equal(big[:M_small], small)


@pytest.mark.parametrize("M_small,M_big,N,K", [(50, 100, 768, 768), (18, 300, 3072, 768), (50, 2200, 768, 3072), (7, 64, 3667, 768)])
def test_simt_gemm_rows_do_not_depend_on_batch(M_small, M_big, N, K):
    from mapperatorinator_b200 import ops
    g = torch.Generator().manual_seed(N + K + 1)
    a, w = torch.randn(M_big, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K)
    bias = torch.randn(N, generator=g)
    big = ops.gemm(a.cuda(), w.cuda(), bias.cuda(), "none", 1.0, None, None, 1).cpu()
    small = ops.gemm(a[:M_small].cuda().contiguous(), w.cuda(), bias.cuda(), "none", 1.0, None, None, 1).cpu()
    assert torch.equal(big[:M_small], small)
    ref = torch.nn.functional.linear(a, w, bias)
    assert torch.allclose(big, ref, rtol=2e-5, atol=2e-5)


def test_encoder_window_alone_equals_window_in_chunk(full):
    """encode(w_i) alone == encode(w_i) inside a 16-chunk == inside the 3-window tail chunk (torch.equal), tensor cores on."""
    from mapperatorinator_b200.pipeline import segment
    cfg, sd, model = full
    windows, _, _ = segment(_song(3, 19 * 0.82 + 8.3), cfg)
    windows = windows[:19].cuda()
    assert windows.shape[0] == 19
    all_states = model.engine.encode(windows, 0, return_states=True)
    for i in (0, 7, 15, 16, 18):
        alone = model.engine.encode(windows[i:i + 1], 20, return_states=True)
        assert torch.equal(alone[0], all_states[i]), f"window {i}: max diff {(alone[0] - all_states[i]).abs().max().item():.3e}"
    pair = model.engine.encode(windows[4:6], 20, return_states=True)
    assert torch.equal(pair, all_states[4:6])


def _bench_like(cfg, layout, n_windows, new_tokens):
    cond = [3667, 3680, 3700, 3710, 3730, 3798, 3810, 3870, 3965, 3975, 3992, 4006, 4100, 3862, 3863, 3864]
    prompt_fn = lambda i, streams: (cond + [1, 9]) if i == 0 else (cond + [1, 9] + streams[i - 1][-32:])
    ms = 8184.0

    def gk_fn(i, P):
        return dict(do_sample=False, num_beams=1, top_p=0.9, top_k=0, cfg_scale=1.0, timeshift_bias=0, types_first=True, temperature=0.9,
                    timing_temperature=0.1, mania_column_temperature=0.5, taiko_hit_temperature=0.5, max_length=P + new_tokens,
                    min_new_tokens=new_tokens, lookback_time=0.5 * ms if i > 0 else 0.0, lookahead_time=0.4 * ms if i < n_windows - 1 else 0.0,
                    context_type="map")
    return prompt_fn, gk_fn


@pytest.mark.parametrize("seed", [2, 3, 5])
def test_song_decoder_equals_per_window_calls_full_dims(full, layout, seed):
    """The bench's two arms on three of the songs that diverged in round 1 (ranks 2, 3, 5 of the 8-GPU run), 20 windows each:
    16-chunk + 4-window tail through `encode_song` vs one window per call."""
    from mapperatorinator_b200.pipeline import SongDecoder, segment
    from mapperatorinator_b200.server import model_generate
    cfg, sd, model = full
    n, new = 20, 32                      # 32 new tokens: window i > 0 then has the bench's 50-token prompt (18 + the last 32 ids)
    windows, _, _ = segment(_song(seed, 25.0), cfg)
    windows = windows[:n]
    prompt_fn, gk_fn = _bench_like(cfg, layout, n, new)
    song = SongDecoder(model, layout)
    song.encode_song(windows.cuda())
    a = song.decode_windows(n, prompt_fn, lambda i: gk_fn(i, 18 if i == 0 else 50))
    b = []
    for i in range(n):
        p = torch.tensor([prompt_fn(i, b)])
        ids, _ = model_generate(model, layout, dict(inputs=windows[i:i + 1], decoder_input_ids=p, decoder_attention_mask=p.ne(0)), gk_fn(i, p.shape[1]))
        b.append(ids[0, p.shape[1]:].tolist())
    for i in range(n):
        assert len(a[i]) == len(b[i]) == new
        assert a[i] == b[i], f"song {seed} window {i}: first differing token {next(j for j in range(new) if a[i][j] != b[i][j])}"


def test_greedy_ids_vs_oracle_teacher_forced_full_dims(full, layout):
    """GPU greedy ids of 3 sequential windows vs the CPU oracle: one teacher-forced oracle pass per window replays the processor
    chain on the GPU's ids and must pick the same token everywhere (min top-2 gap reported on failure)."""
    from mapperatorinator_b200.pipeline import SongDecoder, segment
    from oracle import generate as go
    cfg, sd, model = full
    n, new = 3, 32
    windows, _, _ = segment(_song(11, 12.0), cfg)
    windows = windows[:n]
    prompt_fn, gk_fn = _bench_like(cfg, layout, n, new)
    song = SongDecoder(model, layout)
    song.encode_song(windows.cuda())
    streams = song.decode_windows(n, prompt_fn, lambda i: gk_fn(i, 18 if i == 0 else 50))
    torch.set_num_threads(min(os.cpu_count() or 1, 16))
    with torch.no_grad():
        for i in range(n):
            prompt = prompt_fn(i, streams)
            full_ids = torch.tensor([prompt + streams[i]])
            rep = go.teacher_forced_check(sd, cfg, layout, windows[i:i + 1], full_ids, len(prompt), gk_fn(i, len(prompt)))
            assert rep["match"], f"window {i}: {rep}"


# ---- the token loop at the model's own max_length (2 048): every self-attention split plan, every driver -------------------------
# max_length -> S = max_length <= 128 ? 1 : ceil(max_length / 64).  S = 11 is 132 attention units per row (one per SM of an H100), 12 is
# the first plan with more units than CTAs, 17 the first past the dataflow merge's 16 in-flight splits, 32 the plan of every drop-in call.
PLAN_LENGTHS = [128, 192, 640, 704, 705, 1024, 1025, 1408, 2048]
DRIVERS = {"dataflow": 2, "megakernel": 1, "graph": 0}
TOP2_GAP = 1e-4


def _plan_case(max_length, rows):
    """P = max_length - 17 random ids (built like cases.long_context_cases), min_new_tokens fixes the length: 16 tokens decode inside
    the token loop at nearly full context.  rows == 2: the CFG pair (negative prompt of the same length)."""
    from oracle import cases
    P = max_length - 17
    g = torch.Generator().manual_seed(max_length)
    prompt = torch.randint(17, 3600, (1, P), generator=g)
    prompt[0, :4] = torch.tensor([3700, 3705, 1, 9])
    neg = None
    if rows == 2:
        neg = torch.randint(17, 3600, (1, P), generator=g)
        neg[0, :4] = torch.tensor([3700, 3705, 1, 9])
    gk = dict(cases.GK, max_length=max_length, min_new_tokens=max_length - P, lookback_time=0.0, lookahead_time=0.0, context_type="map",
              cfg_scale=1.5 if rows == 2 else 1.0)
    return prompt, neg, gk


def _generate(model, layout, slot, prompt, neg, gk, driver):
    model.engine.set_option("mega", DRIVERS[driver])
    try:
        return model.engine.generate([slot], prompt, None, layout, dict(gk), negative_prompt=neg)
    finally:
        model.engine.set_option("mega", 2)


def _oracle_check(sd, cfg, layout, pcm, ids, P, gk, what):
    """Teacher-forced CPU oracle on the GPU ids: every position whose top-2 gap exceeds TOP2_GAP must be the oracle's argmax.
    Returns (positions under the gap, smallest gap) for the report."""
    from oracle import generate as go
    torch.set_num_threads(min(os.cpu_count() or 1, 16))
    with torch.no_grad():
        rep = go.teacher_forced_check(sd, cfg, layout, pcm, ids, P, gk)
    gaps = np.asarray(rep["gaps"])
    bad = [P + i for i, (g, m) in enumerate(zip(rep["gaps"], rep["mismatch"])) if m and g > TOP2_GAP]
    near = int((gaps <= TOP2_GAP).sum())
    print(f"{what}: {rep['n_checked']} positions checked, {near} with a top-2 gap <= {TOP2_GAP}, smallest gap {rep['min_gap']:.3e}")
    assert not bad, f"{what}: mismatches at positions {bad[:10]} with top-2 gap > {TOP2_GAP} ({rep['first_divergence']})"
    return near, rep["min_gap"]


@pytest.mark.parametrize("max_length", PLAN_LENGTHS, ids=[f"ml{m}" for m in PLAN_LENGTHS])
def test_split_plans_all_drivers_full_dims(full, layout, max_length):
    """Every driver decodes every plan, and their ids are equal bit for bit: B = 1, and for S in {11, 22, 32} also the CFG pair
    (264, 528, 768 attention units).  S in {11, 17, 32}: the dataflow ids also pass the teacher-forced oracle."""
    from oracle import cases
    cfg, sd, model = full
    S = 1 if max_length <= 128 else (max_length + 63) // 64
    pcm = cases.model_pcm(cfg, 1, 40 + max_length)
    model.engine.encode(pcm.cuda(), slot_begin=0)
    for rows in ((1, 2) if S in (11, 22, 32) else (1,)):
        prompt, neg, gk = _plan_case(max_length, rows)
        got = {drv: _generate(model, layout, 0, prompt, neg, gk, drv) for drv in DRIVERS}
        for drv, ids in got.items():
            assert ids.shape == (1, max_length), f"S {S} rows {rows} {drv}: shape {tuple(ids.shape)}"
            assert torch.equal(ids[:, :prompt.shape[1]], prompt)
            assert torch.equal(ids, got["graph"]), f"S {S} rows {rows}: {drv} differs from graph at {(ids != got['graph']).nonzero()[:4].tolist()}"
        if rows == 1 and S in (11, 17, 32):
            _oracle_check(sd, cfg, layout, pcm, got["dataflow"].cpu(), prompt.shape[1], gk, f"max_length {max_length} (S {S})")


@pytest.mark.parametrize("P", [18, 50])
def test_reference_call_shape_max_length_2048_full_dims(full, layout, P):
    """The reference's own call: a bench-like prompt and max_length = tgt_seq_len = 2048, ~2 000 tokens through 32 splits.  Dataflow ids
    equal graph ids; the P = 18 run also passes the teacher-forced oracle."""
    from oracle import cases
    cfg, sd, model = full
    pcm = cases.model_pcm(cfg, 1, 70 + P)
    model.engine.encode(pcm.cuda(), slot_begin=0)
    cond = [3667, 3680, 3700, 3710, 3730, 3798, 3810, 3870, 3965, 3975, 3992, 4006, 4100, 3862, 3863, 3864, 1, 9]
    g = torch.Generator().manual_seed(P)
    prompt = torch.tensor([(cond + torch.randint(17, 3600, (P - len(cond),), generator=g).tolist())[:P]])
    gk = dict(cases.GK, max_length=2048, min_new_tokens=2048 - P, lookback_time=0.0, lookahead_time=0.0, context_type="map")
    a = _generate(model, layout, 0, prompt, None, gk, "dataflow")
    b = _generate(model, layout, 0, prompt, None, gk, "graph")
    assert a.shape == b.shape == (1, 2048)
    assert torch.equal(a, b), f"dataflow differs from graph at {(a != b).nonzero()[:4].tolist()}"
    if P == 18:
        _oracle_check(sd, cfg, layout, pcm, a.cpu(), P, gk, f"P {P}, max_length 2048")
