"""Weight-streaming GEMV family of the token loop (decode.cu: `gemv_kernel<NB[, RAGGED]>` built from `gemv_stage_x` / `gemv_dot` /
`gemv_row` of decode_device.cuh) against a plain fp64 act(W . LN(x) + b) * alpha + R from the same fp32 operands, one phase at a time
through `mb200_op_gemv`, which fills GemvParams the way the token step does and calls the engine's own `launch_gemv`.

Tolerance, derived from the kernel's summation order (u = 2^-24, first-order bounds; nothing here is fitted to a measurement):
  * dot product: lane l of the row's warp runs 4 sequential fma chains (the x / y / z / w components of float4 columns l, l + 32, ...),
    about K / 128 terms each; then (x + y) + (z + w) is 2 adds and the warp shuffle tree 5 more.  Every rounding is at most u times a
    partial sum of |w_k x_k|, so |err| <= (ceil(K / 128) + 8) u sum_k |w_k x_k|, the 8th u for the bias add.
  * epilogue: u |pre-activation| for the bias add, the activation's input error times its slope (<= 1.2 for GELU / SiLU) plus 4 u
    (|v| + |act(v)|) for erff / tanhf / expf (2 ulp each) and their few roundings, u for alpha and u for the residual add.
  * fused LayerNorm prologue: the mean and the variance are summed over a tree of depth D (4 floats of a lane: 2, warp shuffle: 5,
    8 chunk partials: 3, so D = 10; norm.cu's one-warp rows: K / 128 sequential + 2 + 5).  The fp32 mean is off by <= (D + 2) u mean|x|,
    which shifts every normalised value by that times rstd -- the term that grows with |mean| / sigma; rstd (variance sum, eps add,
    rsqrtf's 2 ulp) is off by <= (D / 2 + 5) u relative.  Per element
        |LN_fp32 - LN| <= u ((D + 4) |ln_w| rstd (|x - mean| + mean|x|) + 2 |LN|),
    and that error reaches the output through sum_k |w_k| |LN error_k|.
`test_tolerance_is_not_vacuous` shows that leaving one k term out of the reference moves it by more than 10x this bound.

Bitwise claims checked here: a row's output does not depend on the batch tile it shares (B = 1 .. 16, NB = 1 / 2 / 4 / 8 and the b0
loop past 8), a ragged row equals its uniform launch, an in-place residual equals the out-of-place one, and the barrier megakernel's
phase body (512 threads, weights in shared memory; `form="mega"`) equals the per-phase kernel (128 threads, weights from global memory).

Out of scope: the dataflow megakernel's fc2 K-split (`m3_rows` in decode_mega2.cu) sums its K slices in its own order, and its LayerNorm
poll path; both keep their end-to-end coverage (ids equal across drivers, the teacher-forced oracle)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LN_DEPTH = 10                         # the GEMV prologue's reduction tree: 2 + 5 + 3
SENTINEL = 0x7FA5A5A5                 # a NaN bit pattern no kernel output can have
WHISPER = dict(d=768, f=3072, V=3667)
TINY = dict(d=128, f=256, V=3667)
RATIOS = {}                           # largest |err| / bound per case group, printed after the module (pytest -s)


@pytest.fixture(scope="module", autouse=True)
def _ratio_summary():
    yield
    if RATIOS:
        print("\nlargest |err| / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(RATIOS.items())))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape, scale=1.0, offset=0.0):
    return torch.randn(*shape, device="cuda", generator=g) * scale + offset


def _weights(g, N, K, bias=True):
    return _randn(g, N, K, scale=1 / math.sqrt(K)), (_randn(g, N) if bias else None)


def _ln_params(g, K):
    return _randn(g, K, scale=0.3, offset=1.0), _randn(g, K, scale=0.3)


def _sentinel(*shape):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def _is_sentinel(t):
    return t.contiguous().view(torch.int32).eq(SENTINEL)


def _ln64(x, lw, lb, eps=1e-5, depth=LN_DEPTH):
    """fp64 LayerNorm of the fp32 rows and the per-element bound on the fp32 kernel's error."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    r = 1 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    y = (x - mu) * r * lw.double() + lb.double()
    e = U * ((depth + 4) * lw.double().abs() * r * ((x - mu).abs() + x.abs().mean(-1, keepdim=True)) + 2 * y.abs())
    return y, e


def _act64(v, act):
    if act == "gelu":
        return 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
    if act == "gelu_tanh":
        return 0.5 * v * (1 + torch.tanh(math.sqrt(2 / math.pi) * (v + 0.044715 * v ** 3)))
    if act == "silu":
        return v * torch.sigmoid(v)
    return v


def _reference(x, w, bias=None, ln=None, act="none", alpha=1.0, residual=None, drop_col=None):
    """fp64 act(w . X(x) + bias) * alpha + residual and its error bound, both (B, N); drop_col leaves that k term out."""
    K = x.shape[1]
    w64 = w.double()
    y, e_y = _ln64(x, *ln) if ln is not None else (x.double(), None)
    if drop_col is not None:
        y = y.clone()
        y[:, drop_col] = 0
    pre = y @ w64.T + (bias.double() if bias is not None else 0)
    e = (math.ceil(K / 128) + 8) * U * (y.abs() @ w64.abs().T) + U * pre.abs()
    if e_y is not None:
        e = e + e_y @ w64.abs().T
    a = _act64(pre, act)
    if act != "none":
        e = 1.2 * e + 4 * U * (pre.abs() + a.abs())
    out = a * alpha
    e = abs(alpha) * e + U * out.abs()
    if residual is not None:
        out = out + residual.double()
        e = e + U * out.abs()
    return out, e


def _check(group, got, want, bound, what=""):
    ratio = ((got.double() - want).abs() / bound).max().item()
    RATIOS[group] = max(RATIOS.get(group, 0.0), ratio)
    assert ratio <= 1.0, f"{group} {what}: max |err| / bound = {ratio:.3f}"


def _gemv(*args, **kw):
    from mapperatorinator_b200 import ops
    return ops.gemv(*args, **kw)


def _qkv(q, cache, d):
    """The token step's LN1 -> q | k | v segments: q rows, then k and v at the token's position of the [rows, T, 2d] self cache."""
    from mapperatorinator_b200.ops import GemvSegment
    T = cache.shape[1]
    return [GemvSegment(q, 0, d, q.stride(0)), GemvSegment(cache, d, 2 * d, T * 2 * d, 2 * d),
            GemvSegment(cache[..., d:], 2 * d, 3 * d, T * 2 * d, 2 * d)]


def _check_qkv(group, q, cache, want, bound, d, cur_len, written=None):
    """q within the bound; the cache holds K | V at cur_len - 1 of every written row and the sentinel everywhere else."""
    B = q.shape[0]
    cur = [cur_len] * B if isinstance(cur_len, int) else cur_len
    written = [True] * B if written is None else written
    _check(group, q, want[:, :d], bound[:, :d], "q")
    untouched = torch.ones(cache.shape[:2], dtype=torch.bool, device="cuda")
    for b in range(B):
        if written[b]:
            _check(group, cache[b, cur[b] - 1], want[b, d:], bound[b, d:], f"row {b} k|v")
            untouched[b, cur[b] - 1] = False
    assert _is_sentinel(cache[untouched]).all(), f"{group}: a cache element off the token's position was written"


# ---- every production shape ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B", [2, 9])
@pytest.mark.parametrize("dims", [WHISPER, TINY], ids=["whisper_small", "tiny"])
def test_production_shapes_vs_fp64(dims, B):
    """Every GEMV of a decoder layer and the vocabulary projection with the token step's segment layout and epilogue, plus the
    prefill logits of a ragged request (rows P * d apart in, written N * V apart)."""
    d, f, V = dims["d"], dims["f"], dims["V"]
    g = _gen(d + B)
    x = _randn(g, B, d, scale=2.0, offset=0.5)
    # LN1 -> q | k | v, k and v into the self cache at position cur_len - 1
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, 3 * d, d)
    q, cache = _sentinel(B, d), _sentinel(B, 40, 2 * d)
    _gemv(x, w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q, cache, d), cur_len=37)
    _check_qkv("production", q, cache, *_reference(x, w, b, ln=(lw, lb)), d, 37)
    # out_proj + residual and the cross-attention out_proj + residual: the residual stream is updated in place
    for _ in range(2):
        attn = _randn(g, B, d)
        w, b = _weights(g, d, d)
        want, bound = _reference(attn, w, b, residual=x)
        _gemv(attn, w, b, residual=x, out=x)
        _check("production", x, want, bound, "out_proj + residual")
    # LN2 -> cross q
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, d, d)
    _check("production", _gemv(x, w, b, ln_weight=lw, ln_bias=lb), *_reference(x, w, b, ln=(lw, lb)), "cross q")
    # LN3 -> fc1 + GELU, then fc2 + residual in place
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, f, d)
    h = _gemv(x, w, b, ln_weight=lw, ln_bias=lb, act="gelu")
    _check("production", h, *_reference(x, w, b, ln=(lw, lb), act="gelu"), "fc1")
    w, b = _weights(g, d, f)
    want, bound = _reference(h, w, b, residual=x)
    _gemv(h, w, b, residual=x, out=x)
    _check("production", x, want, bound, "fc2 + residual")
    # final LN -> vocabulary projection, no bias
    lw, lb = _ln_params(g, d)
    w, _ = _weights(g, V, d, bias=False)
    _check("production", _gemv(x, w, ln_weight=lw, ln_bias=lb), *_reference(x, w, ln=(lw, lb)), "logits")
    # prefill logits of request r of a ragged call: the last prompt position of each of its rows (x_ld = P * d) into logits rows r and
    # n_req + r (out_bs = n_req * V)
    from mapperatorinator_b200.ops import GemvSegment
    P, n_req, r = 11, 3, 1
    px = _randn(g, B, P, d, offset=0.3)
    xs = px[:, P - 1]
    logits = _sentinel(B * n_req, V)
    _gemv(xs, w, ln_weight=lw, ln_bias=lb, segments=[GemvSegment(logits[r], 0, V, n_req * V)])
    want, bound = _reference(xs, w, ln=(lw, lb))
    rows = [r + b * n_req for b in range(B)]
    _check("production", logits[rows], want, bound, "strided prefill logits")
    others = [i for i in range(B * n_req) if i not in rows]
    assert _is_sentinel(logits[others]).all(), "prefill logits landed in another request's rows"


# ---- edges of gemv_dot and of the staging --------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [4, 128, 132, 1024, 1536, 1540, 3072, 4096])
def test_dot_and_staging_edges_vs_fp64(K):
    """K at and past one 128-float lane pass and one 1 536-float `gemv_dot` pass, N leaving the last 4-warp block partial; three rows
    (a partial NB = 4 tile).  Plain rows with bias and residual, and the LayerNorm prologue wherever it applies (K <= 1024: at 1024
    all 8 chunks are full, at 132 the second chunk holds one float4)."""
    for N in (1, 3, 5, 3667):
        g = _gen(K * 7 + N)
        x, R = _randn(g, 3, K), _randn(g, 3, N)
        w, b = _weights(g, N, K)
        _check("dot edges", _gemv(x, w, b, residual=R), *_reference(x, w, b, residual=R), f"K {K} N {N} plain")
        if K <= 1024:
            lw, lb = _ln_params(g, K)
            got = _gemv(x, w, b, ln_weight=lw, ln_bias=lb)
            _check("dot edges", got, *_reference(x, w, b, ln=(lw, lb)), f"K {K} N {N} layernorm")


@pytest.mark.parametrize("K,ln,cols", [(3072, False, (0, 127, 128, 1535, 1536, 3071)), (1024, True, (0, 127, 128, 1023))])
def test_tolerance_is_not_vacuous(K, ln, cols):
    """Leaving the k term out of the reference at the first and last column and at the 128-float lane-pass / 1 536-float
    `gemv_dot`-pass boundaries moves some output by more than 10x its bound, so a kernel that dropped or doubled such a term fails."""
    g = _gen(K)
    x = _randn(g, 2, K)
    w, b = _weights(g, 768, K)
    lnp = _ln_params(g, K) if ln else None
    kw = dict(ln_weight=lnp[0], ln_bias=lnp[1]) if ln else {}
    want, bound = _reference(x, w, b, ln=lnp)
    _check("not vacuous", _gemv(x, w, b, **kw), want, bound)
    for c in cols:
        moved = ((want - _reference(x, w, b, ln=lnp, drop_col=c)[0]).abs() / bound).max().item()
        assert moved > 10, f"dropping column {c} moves the reference by only {moved:.2f}x the bound"


def test_layernorm_beyond_1024_and_bad_arguments_are_rejected():
    """Every rejection names its reason and launches nothing: the output keeps its sentinel."""
    from mapperatorinator_b200.ops import GemvSegment
    g = _gen(1)
    B, K, N = 2, 768, 64
    x = _randn(g, B, K)
    w, b = _weights(g, N, K)
    lw, lb = _ln_params(g, K)
    out = _sentinel(B, N)

    def rejected(match, *args, **kw):
        with pytest.raises(RuntimeError, match=match):
            _gemv(*args, **kw)
        assert _is_sentinel(out).all(), f"a rejected call ({match}) wrote its output"

    seg = lambda n0, n1, pos=0: GemvSegment(out, n0, n1, N, pos)
    for segs in ([seg(0, 30), seg(31, N)], [seg(0, 30), seg(20, N)], [seg(30, N), seg(0, 30)], [seg(0, 30)], [seg(1, N)],
                 [seg(0, 0), seg(0, N)]):
        rejected("tile", x, w, b, segments=segs)
    rejected("cur_len", x, w, b, segments=[seg(0, N, pos=N)], cur_len=0)
    rejected("LayerNorm input", x, w, b, xmode="layernorm", ln_weight=None, ln_bias=lb, out=out)
    rejected("multiples of 4", torch.empty(B, K + 2, device="cuda")[:, :K], w, b, out=out)                 # x_ld
    rejected("multiples of 4", x, torch.empty(N, K + 2, device="cuda")[:, :K], b, out=out)                 # ldw
    rejected("multiples of 4", torch.empty(B, 8, device="cuda")[:, :6], torch.empty(N, 8, device="cuda")[:, :6], b, out=out)   # K
    x5, w5 = _randn(g, B, 1028), _randn(g, N, 1028)
    l5w, l5b = _ln_params(g, 1028)
    rejected("K <= 1024", x5, w5, b, ln_weight=l5w, ln_bias=l5b, out=out)
    rejected("1 or 2 rows", _randn(g, 3, K), w, b, out=_sentinel(3, N), form="mega")
    assert _is_sentinel(out).all()


# ---- every batch tile --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 7, 8, 9, 15, 16])
def test_every_batch_tile_row_equals_its_own_launch(B):
    """B rows of distinct data (NB = 1 / 2 / 4 / 8, partial tiles, the b0 loop past 8) within the bound, and every row -- its q and its
    cache row, its fc2 output -- equal bit for bit to the row launched alone: the per-row arithmetic does not depend on NB."""
    d, f, T, cur = 768, 3072, 6, 4
    g = _gen(100 + B)
    x = _randn(g, B, d) + torch.arange(B, device="cuda").view(B, 1)      # row b centred near b: a row mix-up changes every value
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, 3 * d, d)
    q, cache = _sentinel(B, d), _sentinel(B, T, 2 * d)
    _gemv(x, w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q, cache, d), cur_len=cur)
    _check_qkv("batch tiles", q, cache, *_reference(x, w, b, ln=(lw, lb)), d, cur)
    h, R = _randn(g, B, f, scale=0.5), _randn(g, B, d)
    w2, b2 = _weights(g, d, f)
    y = _gemv(h, w2, b2, residual=R)
    _check("batch tiles", y, *_reference(h, w2, b2, residual=R))
    for r in range(B):
        q1, c1 = _sentinel(1, d), _sentinel(1, T, 2 * d)
        _gemv(x[r:r + 1], w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q1, c1, d), cur_len=cur)
        assert torch.equal(q1[0], q[r]) and torch.equal(c1[0, cur - 1], cache[r, cur - 1]), f"B {B}: row {r} LN -> q|k|v"
        assert torch.equal(_gemv(h[r:r + 1], w2, b2, residual=R[r:r + 1])[0], y[r]), f"B {B}: row {r} fc2 + residual"


# ---- LayerNorm prologue ------------------------------------------------------------------------------------------------------

def _ln_rows(g, K):
    """unit-scale, offset (mean ~ 30, sigma ~ 0.5), near-constant (variance ~ 1e-8, eps dominates), a scaled, shifted row, and one whose
    128-float chunks each have their own scale and sign."""
    return torch.stack([_randn(g, K), _randn(g, K, scale=0.5, offset=30.0), _randn(g, K, scale=1e-4, offset=5.0),
                        _randn(g, K, scale=8.0, offset=-3.0), _chunk_scaled_rows(K, 1)[0]])


@pytest.mark.parametrize("K", [768, 1024])
def test_layernorm_prologue_and_norm_cu_vs_fp64(K):
    """The fused prologue, with identity and non-trivial ln_w / ln_b, on rows whose fp32 mean rounding matters; and norm.cu's
    `layernorm` on the same rows against the same fp64 LayerNorm (its reduction depth is K / 128 + 7)."""
    from mapperatorinator_b200 import ops
    g = _gen(K + 5)
    x = _ln_rows(g, K)
    w, b = _weights(g, 768, K)
    for lw, lb in ((torch.ones(K, device="cuda"), torch.zeros(K, device="cuda")), _ln_params(g, K),
                   (_randn(g, K, scale=2.0), _randn(g, K, scale=2.0))):
        want, bound = _reference(x, w, b, ln=(lw, lb))
        got = _gemv(x, w, b, ln_weight=lw, ln_bias=lb)
        for r, name in enumerate(("unit", "offset", "near-constant", "scaled", "chunk-scaled")):
            _check("layernorm prologue", got[r], want[r], bound[r], name)
        y, e = _ln64(x, lw, lb, depth=K // 128 + 7)
        _check("norm.cu layernorm", ops.layernorm(x, lw, lb, eps=1e-5), y, e)


# ---- activations, alpha, in-place residual -------------------------------------------------------------------------------------

@pytest.mark.parametrize("act", ["none", "gelu", "gelu_tanh", "silu"])
def test_activations_alpha_and_in_place_residual(act):
    """Every epilogue activation with alpha != 1 on the fc1 shape (pre-activations ~ N(0, 2^2): both tails of GELU / SiLU), and the
    residual added in place (R is the output, as out_proj and fc2 run) giving the out-of-place bits."""
    g = _gen(len(act))
    d, f = 768, 3072
    x, R = _randn(g, 3, d), _randn(g, 3, f)
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, f, d)
    w = w * 2
    for alpha in (0.5, -1.75):
        got = _gemv(x, w, b, ln_weight=lw, ln_bias=lb, act=act, alpha=alpha, residual=R)
        _check("activations", got, *_reference(x, w, b, ln=(lw, lb), act=act, alpha=alpha, residual=R), f"alpha {alpha}")
        inplace = R.clone()
        _gemv(x, w, b, ln_weight=lw, ln_bias=lb, act=act, alpha=alpha, residual=inplace, out=inplace)
        assert torch.equal(inplace, got), f"in-place residual, alpha {alpha}"


# ---- cache-position segments ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cur_len", [1, 2, 2048])
def test_cache_position_segments(cur_len):
    """The qkv GEMV into a sentinel-filled [rows, 2048, 2d] cache: K | V land at position cur_len - 1 of every row within the bound,
    and every other element keeps the sentinel bit for bit."""
    d, T, B = 768, 2048, 3
    g = _gen(cur_len)
    x = _randn(g, B, d)
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, 3 * d, d)
    q, cache = _sentinel(B, d), _sentinel(B, T, 2 * d)
    _gemv(x, w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q, cache, d), cur_len=cur_len)
    _check_qkv("cache position", q, cache, *_reference(x, w, b, ln=(lw, lb)), d, cur_len)


# ---- ragged ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rows,n_req", [(3, 3), (6, 3), (10, 5)])
def test_ragged_rows_write_their_own_position(rows, n_req):
    """Requests at cur_len 1 / 700 / 2048 / ..., one of them finished; rows r and r + n_req share request r (CFG when n_req = rows / 2).
    Each row writes K | V at its own position, a finished row leaves its cache untouched but still writes q, and every row equals its
    uniform launch at its own cur_len bit for bit."""
    d, T = 768, 2048
    cur = [1, 700, 2048, 129, 64][:n_req]
    fin = [0, 1, 0, 0, 1][:n_req]
    g = _gen(rows * 10 + n_req)
    x = _randn(g, rows, d)
    lw, lb = _ln_params(g, d)
    w, b = _weights(g, 3 * d, d)
    q, cache = _sentinel(rows, d), _sentinel(rows, T, 2 * d)
    _gemv(x, w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q, cache, d), ragged_cur_len=cur, ragged_finished=fin, n_req=n_req)
    row_cur = [cur[r % n_req] for r in range(rows)]
    written = [not fin[r % n_req] for r in range(rows)]
    _check_qkv("ragged", q, cache, *_reference(x, w, b, ln=(lw, lb)), d, row_cur, written)
    for r in range(rows):
        q1, c1 = _sentinel(1, d), _sentinel(1, T, 2 * d)
        _gemv(x[r:r + 1], w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q1, c1, d), cur_len=row_cur[r])
        assert torch.equal(q1[0], q[r]), f"row {r}: q"
        if written[r]:
            assert torch.equal(c1[0, row_cur[r] - 1], cache[r, row_cur[r] - 1]), f"row {r}: k|v at {row_cur[r] - 1}"


# ---- the barrier megakernel's phase body ---------------------------------------------------------------------------------------

def _chunk_scaled_rows(K, n=64):
    """n rows whose 128-float chunks each have their own scale (1e-2 .. 1e2) and sign, like a residual stream with outlier channels.
    Reassociating the 8 chunk partials of the LayerNorm mean changes the fp32 mean of about one row in five of these (of few plain
    randn rows), so a prologue that summed them in another order would show up in the bits."""
    g = torch.Generator().manual_seed(K)
    c = max(K // 128, 1)
    sc = 10 ** (torch.rand(n, c, 1, generator=g) * 4 - 2) * torch.randn(n, c, 1, generator=g).sign()
    return ((torch.randn(n, c, K // c, generator=g) + 3) * sc).reshape(n, K).cuda()


@pytest.mark.parametrize("K", [768, 128, 1024])
@pytest.mark.parametrize("B", [1, 2])
def test_megakernel_body_equals_per_phase_kernel(B, K):
    """`gemv_stage_x<NB, 512>` + `gemv_row<NB, false>` on shared-memory weight rows (form "mega") give the bits of the 128-thread
    kernel reading weights from global memory -- the claim in `gemv_stage_x` that the LayerNorm reduction does not depend on the warp
    count: LayerNorm -> q|k|v into the cache for 64 chunk-scaled rows, and plain rows with and without a residual over a
    vocabulary-sized N (several rows per warp)."""
    g = _gen(B * 1000 + K)
    lw, lb = _ln_params(g, K)
    w, b = _weights(g, 3 * K, K)
    rows = _chunk_scaled_rows(K)
    for i in range(0, rows.shape[0], B):
        x = rows[i:i + B]
        outs = []
        for form in ("kernel", "mega"):
            q, cache = _sentinel(B, K), _sentinel(B, 8, 2 * K)
            _gemv(x, w, b, ln_weight=lw, ln_bias=lb, segments=_qkv(q, cache, K), cur_len=5, form=form)
            outs.append((q, cache))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1].view(torch.int32), outs[1][1].view(torch.int32)), \
            f"LN -> q|k|v, rows {i}..{i + B - 1}"
        _check_qkv("megakernel body", *outs[1], *_reference(x, w, b, ln=(lw, lb)), K, 5)
    x = _randn(g, B, K)
    wv, bv = _weights(g, 3667, K)
    R = _randn(g, B, 3667)
    for res in (None, R):
        a = _gemv(x, wv, bv, residual=res, form="kernel")
        m = _gemv(x, wv, bv, residual=res, form="mega")
        assert torch.equal(a, m), f"plain rows, residual {res is not None}"
        _check("megakernel body", m, *_reference(x, wv, bv, residual=res))
