"""bf16 token-loop weight store: a model whose decoder GEMV matrices and proj_out arrive as bf16 is served with the token loop's per-step
GEMVs reading a bf16 copy of those matrices (half the bytes per token), and every result equals the same model served from fp32.

The claim is bitwise, not a tolerance: widening bf16 to fp32 is exact, and the bf16 GEMV widens each weight and runs the fp32 kernel's
FMAs in the fp32 kernel's order.  So every comparison below is between

  * sd16 = {k: v.bfloat16()} of the seeded state dict (the engine selects the bf16 store), and
  * sd32 = {k: v.float() for k, v in sd16.items()} (the same values in fp32: the engine keeps today's fp32-only behaviour),

first one GEMV phase at a time through `ops.gemv` (bf16 `w` against `w.float()`), then through every token-loop entry point."""
import math

import numpy as np
import pytest
import torch

from oracle import beam, cases, ragged

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FA5A5A5                 # a NaN bit pattern no kernel output can have
WHISPER = dict(d=768, f=3072, V=3667)
TINY = dict(d=128, f=256, V=3667)
DRIVERS = {"dataflow": 2, "megakernel": 1, "graph": 0, "graph_pdl": 0}


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_bits(a, b, what):
    a, b = _bits(a), _bits(b)
    if not torch.equal(a, b):
        idx = (a != b).nonzero()[0].tolist()
        pytest.fail(f"{what}: first differing element {idx}")


def _sentinel(*shape):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _w16(g, N, K, ld=None):
    """bf16 weights [N, K] (row stride ld) and their exact fp32 widening."""
    ld = K if ld is None else ld
    w = (torch.randn(N, ld, device="cuda", generator=g) / math.sqrt(K)).bfloat16()[:, :K]
    return w, w.float()


def _both(x, w16, w32, make=None, **kw):
    """ops.gemv with the bf16 weights and with their fp32 widening; make() gives each run fresh output buffers (segments / out /
    residual).  Returns the two runs' output buffers."""
    from mapperatorinator_b200 import ops
    outs = []
    for w in (w16, w32):
        k = dict(kw)
        bufs = make() if make else {}
        k.update({n: v for n, v in bufs.items() if n != "_buffers"})
        r = ops.gemv(x, w, **k)
        outs.append(bufs.get("_buffers", [r]))
    return outs


def _cache_segments(B, T, d):
    """q [B, d] and a sentinel-filled cache [B, T, 2d] whose k | v halves take segments 1 and 2 at the cache position."""
    from mapperatorinator_b200 import ops
    q, cache = _sentinel(B, d), _sentinel(B, T, 2 * d)
    segs = [ops.GemvSegment(q, 0, d, d), ops.GemvSegment(cache, d, 2 * d, T * 2 * d, 2 * d),
            ops.GemvSegment(cache[:, :, d:], 2 * d, 3 * d, T * 2 * d, 2 * d)]
    return dict(segments=segs, _buffers=[q, cache])


# ---- op level -------------------------------------------------------------------------------------------------------------------------
def _phase(name, dims, B, cur_len, g):
    """One production GEMV phase of the token step: (x, w16, w32, kwargs)."""
    from mapperatorinator_b200 import ops
    d, f, V = dims["d"], dims["f"], dims["V"]
    K, N = {"qkv": (d, 3 * d), "out": (d, d), "cross_q": (d, d), "cross_out": (d, d), "fc1": (d, f), "fc2": (f, d), "proj_out": (d, V)}[name]
    x = torch.randn(B, K, device="cuda", generator=g)
    w16, w32 = _w16(g, N, K)
    bias = None if name == "proj_out" else torch.randn(N, device="cuda", generator=g)
    kw = dict(bias=bias)
    if name in ("qkv", "cross_q", "fc1", "proj_out"):
        kw["ln_weight"] = torch.randn(K, device="cuda", generator=g) * 0.3 + 1
        kw["ln_bias"] = torch.randn(K, device="cuda", generator=g) * 0.3
    if name == "qkv":
        kw["cur_len"] = cur_len
        kw["make"] = lambda: _cache_segments(B, cur_len + 1, d)
    elif name in ("out", "cross_out", "fc2"):
        r = torch.randn(B, N, device="cuda", generator=g)

        def make():                          # in place, as the token step adds into the residual stream
            o = r.clone()
            return dict(out=o, residual=o, _buffers=[o])
        kw["make"] = make
    else:
        if name == "fc1":
            kw["act"] = "gelu"
        kw["make"] = lambda: (lambda o: dict(out=o, _buffers=[o]))(_sentinel(B, N))
    return x, w16, w32, kw


PHASES = ["qkv", "out", "cross_q", "cross_out", "fc1", "fc2", "proj_out"]


@pytest.mark.parametrize("dims", ["whisper", "tiny"])
@pytest.mark.parametrize("name", PHASES)
def test_op_production_shapes_every_batch_tile(dims, name):
    """Every production phase at B = 1 .. 16 (per-phase kernel) and B = 1, 2 (megakernel body): bf16 == fp32 bit for bit."""
    D = WHISPER if dims == "whisper" else TINY
    for B in range(1, 17):
        g = _gen(1000 * B + PHASES.index(name))
        x, w16, w32, kw = _phase(name, D, B, 5, g)
        for form in (("kernel", "mega") if B <= 2 else ("kernel",)):
            a, b = _both(x, w16, w32, form=form, **kw)
            for i, (u, v) in enumerate(zip(a, b)):
                _assert_bits(u, v, f"{dims} {name} B {B} {form} output {i}")


@pytest.mark.parametrize("cur_len", [1, 2, 2048])
@pytest.mark.parametrize("form", ["kernel", "mega"])
def test_op_cache_position_segments(cur_len, form):
    """q | k | v with k / v written at the cache position: the whole cache buffer (sentinels elsewhere) equals the fp32 run's."""
    for B in (1, 2):
        x, w16, w32, kw = _phase("qkv", WHISPER, B, cur_len, _gen(cur_len + B))
        a, b = _both(x, w16, w32, form=form, **kw)
        for i, (u, v) in enumerate(zip(a, b)):
            _assert_bits(u, v, f"cur_len {cur_len} B {B} {form} segment {i}")


def test_op_ragged_rows_finished_untouched():
    """Ragged qkv with per-row cache positions and finished rows (rows r and r + n_req share request r): equal buffers, and a finished
    row's cache keeps its sentinels."""
    d = WHISPER["d"]
    g = _gen(7)
    n_req, B, T = 5, 10, 64
    cur = [3, 1, 60, 17, 2]
    fin = [0, 1, 0, 0, 1]
    x = torch.randn(B, d, device="cuda", generator=g)
    w16, w32 = _w16(g, 3 * d, d)
    lw, lb = torch.randn(d, device="cuda", generator=g) * 0.3 + 1, torch.randn(d, device="cuda", generator=g) * 0.3
    bias = torch.randn(3 * d, device="cuda", generator=g)
    a, b = _both(x, w16, w32, make=lambda: _cache_segments(B, T, d), bias=bias, ln_weight=lw, ln_bias=lb, ragged_cur_len=cur,
                 ragged_finished=fin, n_req=n_req)
    for i, (u, v) in enumerate(zip(a, b)):
        _assert_bits(u, v, f"ragged segment {i}")
    kc = a[1]
    for r in range(B):
        if fin[r % n_req]:
            assert bool((_bits(kc[r]) == SENTINEL).all()), f"finished row {r} was written"


@pytest.mark.parametrize("K", [8, 128, 136, 1024, 3072, 4096])
def test_op_k_edges(K):
    """Plain inputs at K from one bf16 group per row up to 4096, N not a multiple of the warp count, a strided weight."""
    for B in (1, 2, 3, 9):
        g = _gen(K + B)
        x = torch.randn(B, K, device="cuda", generator=g)
        w16, w32 = _w16(g, 37, K, ld=K + 8)
        for form in (("kernel", "mega") if B <= 2 else ("kernel",)):
            a, b = _both(x, w16, w32, bias=torch.randn(37, device="cuda", generator=g), form=form)
            _assert_bits(a[0], b[0], f"K {K} B {B} {form}")


def test_op_rejections_launch_nothing():
    from mapperatorinator_b200 import _lib, ops
    g = _gen(3)
    x = torch.randn(1, 132, device="cuda", generator=g)
    w = torch.randn(4, 132, device="cuda", generator=g).bfloat16()
    n0 = _lib.load().mb200_launch_count()
    with pytest.raises(RuntimeError, match="multiples of 8"):
        ops.gemv(x, w)
    x = torch.randn(1, 128, device="cuda", generator=g)
    flat = torch.randn(4 * 128 + 8, device="cuda", generator=g).bfloat16()
    with pytest.raises(RuntimeError, match="float4"):
        ops.gemv(x, flat[1:1 + 4 * 128].view(4, 128))          # 2 bytes past a 16-byte boundary
    assert _lib.load().mb200_launch_count() == n0


# ---- engines --------------------------------------------------------------------------------------------------------------------------
def _dicts(cfg):
    from mapperatorinator_b200.weights import init_model_state_dict
    sd = init_model_state_dict(cfg, 0)
    sd16 = {k: (v.bfloat16() if v.is_floating_point() else v) for k, v in sd.items()}
    sd32 = {k: (v.float() if v.is_floating_point() else v) for k, v in sd16.items()}
    return sd16, sd32


def _model(cfg, sd, **kw):
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    return B200Mapperatorinator(cfg, sd, **kw)


@pytest.fixture(scope="module")
def tiny_pair():
    from mapperatorinator_b200 import tiny_model_config
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd16, sd32 = _dicts(cfg)
    m16, m32 = _model(cfg, sd16, max_windows=24, max_batch=16), _model(cfg, sd32, max_windows=24, max_batch=16)
    assert m16.engine.token_weight_dtype == torch.bfloat16
    assert m32.engine.token_weight_dtype == torch.float32
    return cfg, sd16, sd32, m16, m32


def _with_driver(model, driver, fn):
    model.engine.set_option("mega", DRIVERS[driver])
    model.engine.set_option("pdl", 1 if driver == "graph_pdl" else 0)
    try:
        return fn()
    finally:
        model.engine.set_option("mega", 2)
        model.engine.set_option("pdl", 0)


def _same_ids(a, b, what):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    assert a.shape == b.shape, f"{what}: shapes {tuple(a.shape)} vs {tuple(b.shape)}"
    if not torch.equal(a, b):
        r = (a != b).nonzero()[0].tolist()
        pytest.fail(f"{what}: first divergence at {r}")


def test_selection_falls_back_to_fp32(tiny_pair, layout):
    """The store stays fp32 when one packed q element is not a bf16 value (2^-133 * 0.125 = 2^-136 is below bf16's subnormals), and
    when one token-loop matrix arrives as fp32; both engines then decode like the sd32 engine."""
    from mapperatorinator_b200.server import model_generate
    cfg, sd16, sd32, _, m32 = tiny_pair
    odd = dict(sd16)
    q = odd["transformer.model.decoder.layers.0.encoder_attn.q_proj.weight"].clone()
    q.view(-1)[5] = 2.0 ** -133
    odd["transformer.model.decoder.layers.0.encoder_attn.q_proj.weight"] = q
    odd32 = dict(sd32)
    odd32["transformer.model.decoder.layers.0.encoder_attn.q_proj.weight"] = q.float()
    mixed = dict(sd16)
    mixed["transformer.model.decoder.layers.1.fc1.weight"] = sd16["transformer.model.decoder.layers.1.fc1.weight"].float()
    prompt, neg, gk, seed = cases.generate_cases()[next(iter(cases.generate_cases()))]
    B = prompt.shape[0]
    mk = dict(inputs=cases.model_pcm(cfg, B, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0), negative_prompt=neg,
              negative_prompt_attention_mask=None if neg is None else neg.ne(0))
    for what, sd, ref_sd in (("subnormal q", odd, odd32), ("one fp32 matrix", mixed, sd32)):
        m = _model(cfg, sd, max_windows=4, max_batch=4)
        assert m.engine.token_weight_dtype == torch.float32, what
        ref = m32 if ref_sd is sd32 else _model(cfg, ref_sd, max_windows=4, max_batch=4)
        for drv in ("graph", "dataflow"):
            a, _ = _with_driver(m, drv, lambda: model_generate(m, layout, dict(mk), dict(gk)))
            b, _ = _with_driver(ref, drv, lambda: model_generate(ref, layout, dict(mk), dict(gk)))
            _same_ids(a, b, f"{what} {drv}")


def _wbf16_launches():
    from mapperatorinator_b200 import _lib
    return _lib.load().mb200_wbf16_launch_count()


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("case", list(cases.generate_cases()))
def test_generate_cases_every_driver(tiny_pair, layout, case, driver):
    """Ids equal on every driver.  The bf16-launch count shows which store ran: the sd32 engine never launches a bf16-weight kernel, the
    sd16 engine does on every driver."""
    from mapperatorinator_b200.server import model_generate
    cfg, _, _, m16, m32 = tiny_pair
    prompt, neg, gk, seed = cases.generate_cases()[case]
    B = prompt.shape[0]
    mk = dict(inputs=cases.model_pcm(cfg, B, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0), negative_prompt=neg,
              negative_prompt_attention_mask=None if neg is None else neg.ne(0))
    n0 = _wbf16_launches()
    a, sa = _with_driver(m16, driver, lambda: model_generate(m16, layout, dict(mk), dict(gk)))
    n1 = _wbf16_launches()
    b, sb = _with_driver(m32, driver, lambda: model_generate(m32, layout, dict(mk), dict(gk)))
    assert _wbf16_launches() == n1, "the fp32 engine launched a bf16-weight kernel"
    _same_ids(a, b, f"{case} {driver}")
    assert sa["generated_tokens_per_sample"] == sb["generated_tokens_per_sample"]
    assert n1 > n0, f"{case} {driver}: no bf16-weight kernel ran"


@pytest.mark.parametrize("driver", ["dataflow", "megakernel", "graph"])
@pytest.mark.parametrize("case", list(cases.long_context_cases()))
def test_long_context(tiny_pair, layout, case, driver):
    from mapperatorinator_b200.server import model_generate
    cfg, _, _, m16, m32 = tiny_pair
    prompt, gk, seed = cases.long_context_cases()[case]
    mk = dict(inputs=cases.model_pcm(cfg, 2, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
    a, _ = _with_driver(m16, driver, lambda: model_generate(m16, layout, dict(mk), dict(gk)))
    b, _ = _with_driver(m32, driver, lambda: model_generate(m32, layout, dict(mk), dict(gk)))
    _same_ids(a, b, f"{case} {driver}")


@pytest.mark.parametrize("driver", ["dataflow", "graph"])
def test_sampling_fixed_seeds(tiny_pair, layout, driver):
    cfg, _, _, m16, m32 = tiny_pair
    prompt = torch.tensor([[3700, 3705, 1, 9, 3645, 30], [3700, 3705, 1, 9, 3646, 31]])
    gk = dict(cases.GK, do_sample=True, top_k=0, top_p=0.9, temperature=1.0, max_length=70, min_new_tokens=10)
    for m in (m16, m32):
        m.engine.encode(cases.model_pcm(cfg, 2, 5).cuda(), slot_begin=0)
    for seed in (1, 2, 3):
        g = dict(gk, seed=seed)
        a = _with_driver(m16, driver, lambda: m16.engine.generate([0, 1], prompt, None, layout, dict(g)))
        b = _with_driver(m32, driver, lambda: m32.engine.generate([0, 1], prompt, None, layout, dict(g)))
        _same_ids(a, b, f"sampling seed {seed} {driver}")


def _beam_search(tiny_pair, layout, case):
    """Beam search (K = 2 and 4 in the reference's cases): ids and best-hypothesis scores bitwise equal."""
    cfg, _, _, m16, m32 = tiny_pair
    prompt, neg, gk, seed = beam.beam_cases()[case]
    B = prompt.shape[0]
    res = []
    for m in (m16, m32):
        m.engine.encode(cases.model_pcm(cfg, B, seed).cuda(), slot_begin=0)
        res.append(m.engine.generate_beams(list(range(B)), prompt, prompt.ne(0), layout, dict(gk), negative_prompt=neg,
                                           negative_mask=None if neg is None else neg.ne(0)))
    _same_ids(res[0][0], res[1][0], f"{case} ids")
    _assert_bits(torch.as_tensor(res[0][1]), torch.as_tensor(res[1][1]), f"{case} scores")


@pytest.mark.parametrize("case", list(beam.beam_cases()))
def test_beam_search(tiny_pair, layout, case):
    """Beam search on both engines: the sd16 engine's bf16-weight kernels run, ids equal."""
    n0 = _wbf16_launches()
    _beam_search(tiny_pair, layout, case)
    assert _wbf16_launches() > n0, "no bf16-weight kernel ran"


def _ragged_reference_sets(tiny_pair, layout, case):
    cfg, _, _, m16, m32 = tiny_pair
    reqs = ragged.ragged_cases()[case]
    pcm = torch.cat([cases.model_pcm(cfg, 1, q["seed"]) for q in reqs]).cuda()
    rq = [(r, q["prompt"][0], dict(q["gk"]), None if q["neg"] is None else q["neg"][0]) for r, q in enumerate(reqs)]
    out = []
    for m in (m16, m32):
        m.engine.encode(pcm, slot_begin=0)
        out.append(m.engine.generate_ragged(rq, layout))
    for r, (a, b) in enumerate(zip(*out)):
        _same_ids(a, b, f"{case}[{r}]")


@pytest.mark.parametrize("case", list(ragged.ragged_cases()))
def test_ragged_reference_sets(tiny_pair, layout, case):
    """The ragged reference sets on both engines: the sd16 engine's bf16-weight kernels run, ids equal."""
    n0 = _wbf16_launches()
    _ragged_reference_sets(tiny_pair, layout, case)
    assert _wbf16_launches() > n0, "no bf16-weight kernel ran"


def _stream_with_admissions(tiny_pair, layout):
    """A decode stream of 3 rows fed 8 requests of different lengths, admitted as rows free up: ids equal per request."""
    cfg, _, _, m16, m32 = tiny_pair
    reqs = [dict(prompt=ragged._prompt(P, s), gk=dict(cases.GK, max_length=P + new, min_new_tokens=new // 2))
            for s, (P, new) in enumerate([(6, 40), (20, 12), (9, 90), (33, 20), (7, 17), (12, 60), (40, 30), (5, 25)])]
    pcm = torch.cat([cases.model_pcm(cfg, 1, 100 + i) for i in range(len(reqs))]).cuda()
    got = []
    for m in (m16, m32):
        m.engine.encode(pcm, slot_begin=0)
        stream = m.engine.open_stream(layout, 3)
        done, rows, nxt = {}, {}, 0
        try:
            while len(done) < len(reqs):
                while nxt < len(reqs) and stream.free_rows:
                    rows[stream.admit(nxt, reqs[nxt]["prompt"][0], dict(reqs[nxt]["gk"]))] = nxt
                    nxt += 1
                for row, ids in stream.run(waiting=len(reqs) - nxt):
                    done[rows.pop(row)] = ids
        finally:
            stream.close()
        got.append(done)
    for i in range(len(reqs)):
        _same_ids(got[0][i], got[1][i], f"stream request {i}")


def test_stream_with_admissions(tiny_pair, layout):
    """A decode stream on both engines: the sd16 engine's bf16-weight kernels run, ids equal."""
    n0 = _wbf16_launches()
    _stream_with_admissions(tiny_pair, layout)
    assert _wbf16_launches() > n0, "no bf16-weight kernel ran"


def test_teacher_forcing(tiny_pair):
    """forward_logits and score_tokens read the fp32 weights in both engines: bitwise equal."""
    cfg, _, _, m16, m32 = tiny_pair
    ids, mask = cases.teacher_forcing_case(cfg)
    B = ids.shape[0]
    res = []
    for m in (m16, m32):
        m.engine.encode(cases.model_pcm(cfg, B, 2).cuda(), slot_begin=0)
        res.append((m.engine.forward_logits(list(range(B)), ids, mask), m.engine.score_tokens(list(range(B)), ids, mask)))
    _assert_bits(res[0][0], res[1][0], "forward_logits")
    for k in res[0][1]:
        a, b = res[0][1][k], res[1][1][k]
        if a.dtype == torch.int64:
            _same_ids(a.cpu(), b.cpu(), f"score_tokens {k}")
        else:
            _assert_bits(a, b, f"score_tokens {k}")


# ---- whisper-small dimensions ---------------------------------------------------------------------------------------------------------
PLAN_LENGTHS = [128, 192, 640, 704, 705, 1024, 1025, 1408, 2048]


@pytest.fixture(scope="module")
def full_pair():
    from mapperatorinator_b200 import v29_model_config
    cfg = v29_model_config()
    sd16, sd32 = _dicts(cfg)
    m16, m32 = _model(cfg, sd16, max_windows=24, max_batch=2), _model(cfg, sd32, max_windows=24, max_batch=2)
    assert m16.engine.token_weight_dtype == torch.bfloat16
    assert m32.engine.token_weight_dtype == torch.float32
    return cfg, sd16, sd32, m16, m32


def _plan_case(max_length):
    P = max_length - 17
    g = torch.Generator().manual_seed(max_length)
    prompt = torch.randint(17, 3600, (1, P), generator=g)
    prompt[0, :4] = torch.tensor([3700, 3705, 1, 9])
    gk = dict(cases.GK, max_length=max_length, min_new_tokens=max_length - P, lookback_time=0.0, lookahead_time=0.0, context_type="map")
    return prompt, gk


@pytest.mark.parametrize("max_length", PLAN_LENGTHS, ids=[f"ml{m}" for m in PLAN_LENGTHS])
def test_split_plans_full_dims(full_pair, layout, max_length):
    cfg, sd16, sd32, m16, m32 = full_pair
    pcm = cases.model_pcm(cfg, 1, 40 + max_length).cuda()
    prompt, gk = _plan_case(max_length)
    for m in (m16, m32):
        m.engine.encode(pcm, slot_begin=0)
    for drv in ("dataflow", "megakernel", "graph"):
        n0 = _wbf16_launches()
        a = _with_driver(m16, drv, lambda: m16.engine.generate([0], prompt, None, layout, dict(gk)))
        assert _wbf16_launches() > n0, f"max_length {max_length} {drv}: the token loop did not read the bf16 store"
        b = _with_driver(m32, drv, lambda: m32.engine.generate([0], prompt, None, layout, dict(gk)))
        assert a.shape == (1, max_length)
        _same_ids(a, b, f"max_length {max_length} {drv}")
    if max_length == 704:
        from oracle import generate as go
        import os
        torch.set_num_threads(min(os.cpu_count() or 1, 16))
        with torch.no_grad():
            rep = go.teacher_forced_check(sd32, cfg, layout, pcm.cpu(), b.cpu(), prompt.shape[1], gk)
        bad = [i for i, (gap, mm) in enumerate(zip(rep["gaps"], rep["mismatch"])) if mm and gap > 1e-4]
        assert not bad, f"teacher-forced oracle: mismatches at {bad[:10]} ({rep['first_divergence']})"


def test_song_decoder_full_dims(full_pair, layout):
    """A bench-like song (20 windows, 32 new tokens each) through the resident SongDecoder: ids equal."""
    from mapperatorinator_b200.pipeline import SongDecoder, segment
    cfg, _, _, m16, m32 = full_pair
    rng = np.random.default_rng(3)
    sr, n_s = 16000, 25.0
    t = np.arange(int(n_s * sr)) / sr
    x = sum(np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi)) for f in np.geomspace(55, 7000, 8)) / 8 + rng.normal(0, 0.01, t.size)
    windows, _, _ = segment((x / np.abs(x).max()).astype(np.float32), cfg)
    n, new = min(20, windows.shape[0]), 32
    cond = [3667, 3680, 3700, 3710, 3730, 3798, 3810, 3870, 3965, 3975, 3992, 4006, 4100, 3862, 3863, 3864, 1, 9]

    def prompt_fn(i, streams):
        return cond if i == 0 else cond + streams[i - 1][-32:]

    def gk_fn(i, P):
        return dict(cases.GK, max_length=P + new, min_new_tokens=new, lookback_time=0.0, lookahead_time=0.0, context_type="map")

    out = []
    for m in (m16, m32):
        song = SongDecoder(m, layout)
        song.encode_song(windows[:n].cuda())
        out.append(song.decode_windows(n, prompt_fn, lambda i: gk_fn(i, 18 if i == 0 else 50)))
    for i in range(n):
        assert out[0][i] == out[1][i], f"window {i}"
