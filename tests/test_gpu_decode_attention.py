"""Split-KV decode attention (decode.cu: `decode_attention_kernel<64|128[, TABLE]>`, `decode_attention_warp_kernel`,
`decode_attention_ragged_kernel` and the ticket merge) against a plain fp64 softmax(q K^T) V, one phase at a time through
`mb200_op_decode_attention`, which launches the engine's own functions with the engine's own split plan.

Every self-attention plan edge up to the model's 2 048 positions (one 128-key split; 3 .. 32 splits of 64 keys, so both merge branches
run: every load in flight for <= 8 splits, two rolled passes beyond), every 64-key boundary a plan reaches (most splits empty at small
L), prompt masks that empty a whole split or straddle a split edge, a peaked case whose merge weights underflow, cross attention
through `row_slot`, and the bitwise equalities the kernels claim between their forms."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

H, D = 12, 64                # whisper-small heads
TOL = 1e-5                   # q, K, V ~ N(0, 1), q / 8: ~10x the fp32 error of a 64-term dot plus one exp
PLANS = [1, 2, 63, 64, 65, 127, 128, 129, 192, 193, 640, 641, 704, 705, 1024, 1025, 1409, 2047, 2048]


def _splits(max_length):
    return 1 if max_length <= 128 else (max_length + 63) // 64


def _lengths(max_length):
    """1, max_length, and k*64 - 1, k*64, k*64 + 1 for every boundary the plan reaches."""
    out = {1, max_length}
    for k in range(1, max_length // 64 + 2):
        out.update(x for x in (k * 64 - 1, k * 64, k * 64 + 1) if 1 <= x <= max_length)
    return sorted(out)


def _data(rows, slots, t_max, seed, q_scale=1.0 / 8):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(rows, H * D, generator=g) * q_scale).cuda()
    kv = torch.randn(slots, t_max, 2 * H * D, generator=g).cuda()
    return q, kv


def _reference(q, kv, row_slot, L, P=0, key_valid=None, kv_src=None, drop_key=None):
    """fp64 softmax(q K^T) V of every row over keys [0, L); prompt keys t < P with key_valid 0 are masked."""
    rows = q.shape[0]
    d = H * D
    out = torch.empty(rows, d, dtype=torch.float64, device=q.device)
    t = torch.arange(L, device=q.device)
    for r in range(rows):
        keys = kv[kv_src[r, :L].long(), t] if kv_src is not None else kv[int(row_slot[r]), :L]
        K = keys[:, :d].double().view(L, H, D)
        V = keys[:, d:].double().view(L, H, D)
        s = torch.einsum("hd,lhd->hl", q[r].double().view(H, D), K)
        if key_valid is not None and P > 0:
            s[:, :P] = s[:, :P].masked_fill(key_valid[r, :min(P, L)].eq(0), -math.inf)
        if drop_key is not None:
            s[:, drop_key] = -math.inf
        out[r] = torch.einsum("hl,lhd->hd", torch.softmax(s, dim=-1), V).reshape(d)
    return out


def _err(got, want):
    return (got.double() - want).abs().max().item()


def _run(q, kv, **kw):
    from mapperatorinator_b200 import ops
    return ops.decode_attention(q, kv, H, **kw)


@pytest.mark.parametrize("max_length", PLANS, ids=[f"ml{m}_S{_splits(m)}" for m in PLANS])
def test_self_attention_every_boundary_vs_fp64(max_length):
    """Two rows on shuffled cache rows, row 0 left-padded, at every key count L the plan reaches; flat (score std 1) and peaked
    (q x 16: most splits' merge weights exp(m_s - max m) underflow to zero)."""
    q, kv = _data(2, 3, max_length, max_length)
    row_slot = torch.tensor([2, 0], dtype=torch.int32, device="cuda")
    for L in _lengths(max_length):
        P = L // 2
        kvld = torch.ones(2, max_length, dtype=torch.uint8, device="cuda")
        kvld[0, :P // 3] = 0
        for scale in (1, 16):
            qs = (q * scale).contiguous()
            got = _run(qs, kv, row_slot=row_slot, cur_len=L, prompt_len=P, key_valid=kvld, max_length=max_length)
            want = _reference(qs, kv, row_slot.tolist(), L, P, kvld)
            err = _err(got, want)
            assert err <= TOL * scale, f"max_length {max_length} L {L} P {P} q x {scale}: max |err| {err:.3e}"


@pytest.mark.parametrize("max_length", [128, 704, 2048])
def test_masks_that_empty_a_split_or_straddle_an_edge(max_length):
    """Prompt masks: a left pad covering all of split 0 and part of split 1 (split 0's partial is m = -inf, l = 0), a pad run across
    the 64-key edge in the middle of the prompt, and a whole middle split masked."""
    L = max_length
    q, kv = _data(3, 3, max_length, 7 + max_length)
    row_slot = torch.tensor([1, 2, 0], dtype=torch.int32, device="cuda")
    P = min(L - 1, 200)
    kvld = torch.ones(3, max_length, dtype=torch.uint8, device="cuda")
    kvld[0, :70] = 0
    kvld[1, 60:68] = 0
    kvld[2, 64:128] = 0
    got = _run(q, kv, row_slot=row_slot, cur_len=L, prompt_len=P, key_valid=kvld, max_length=max_length)
    want = _reference(q, kv, row_slot.tolist(), L, P, kvld)
    assert _err(got, want) <= TOL
    # the masks change the answer by far more than the tolerance
    assert _err(got, _reference(q, kv, row_slot.tolist(), L)) > 10 * TOL


@pytest.mark.parametrize("max_length", [192, 1025, 2048])
def test_tolerance_is_not_vacuous(max_length):
    """Dropping the one key at a split boundary from the fp64 reference moves it by more than 10x the tolerance, so a kernel that
    lost or double-counted a boundary key fails."""
    q, kv = _data(2, 2, max_length, 3 + max_length)
    row_slot = torch.tensor([1, 0], dtype=torch.int32, device="cuda")
    L = max_length
    got = _run(q, kv, row_slot=row_slot, cur_len=L, max_length=max_length)
    want = _reference(q, kv, row_slot.tolist(), L)
    assert _err(got, want) <= TOL
    for key in (63, 64, L - 1):
        moved = (want - _reference(q, kv, row_slot.tolist(), L, drop_key=key)).abs().max().item()
        assert moved > 10 * TOL, f"dropping key {key} moves the reference by only {moved:.3e}"


@pytest.mark.parametrize("fixed_len", [512, 500])
def test_cross_attention_through_row_slot(fixed_len):
    """Cross attention over the encoder slots (64-key splits, 8 of them at 512) for two rows and for 16 rows on shuffled slots."""
    for rows in (2, 16):
        q, kv = _data(rows, 16, 512, fixed_len + rows)
        perm = torch.randperm(16, generator=torch.Generator().manual_seed(rows))[:rows]
        row_slot = perm.to(torch.int32).cuda()
        got = _run(q, kv, row_slot=row_slot, fixed_len=fixed_len)
        assert _err(got, _reference(q, kv, perm.tolist(), fixed_len)) <= TOL


@pytest.mark.parametrize("max_length", [192, 704, 1025, 2048])
def test_kmax64_equals_kmax128_and_warp_form_equals_cta_form(max_length):
    """On 64-key chunks the KMAX 64 body gives the KMAX 128 body's bits; the one-warp batch form gives the CTA body's bits (16 rows,
    the shape it is meant for, and 2)."""
    for rows in (2, 16):
        q, kv = _data(rows, rows, max_length, 11 + max_length + rows)
        row_slot = torch.randperm(rows, generator=torch.Generator().manual_seed(rows)).to(torch.int32).cuda()
        kvld = torch.ones(rows, max_length, dtype=torch.uint8, device="cuda")
        kvld[0, 30:90] = 0                  # row 0 keeps keys 0..29, so even L = 1 has a key to attend to
        for L in (1, 64, 65, max_length // 2 + 3, max_length):
            kw = dict(row_slot=row_slot, cur_len=L, prompt_len=min(L, 100), key_valid=kvld, max_length=max_length)
            a = _run(q, kv, form="cta128", **kw)
            b = _run(q, kv, form="cta64", **kw)
            c = _run(q, kv, form="warp", **kw)
            assert torch.equal(a, b), f"KMAX 64 vs 128, L {L}"
            assert torch.equal(a, c), f"warp vs CTA form, L {L}"
            assert torch.equal(a, _run(q, kv, **kw)), f"default form, L {L}"
            assert _err(a, _reference(q, kv, row_slot.tolist(), L, min(L, 100), kvld)) <= TOL


def test_form_that_cannot_hold_the_chunk_is_rejected():
    q, kv = _data(1, 1, 128, 0)
    with pytest.raises(RuntimeError, match="KMAX 64"):
        _run(q, kv, cur_len=100, max_length=128, form="cta64")
    with pytest.raises(RuntimeError, match="cur_len"):
        _run(q, kv, cur_len=129, max_length=128)


@pytest.mark.parametrize("max_length", [128, 705, 2048])
def test_table_identity_and_permuted_cache(max_length):
    """`TABLE` with the identity table (every key of row r in row r's cache row) gives the no-table bits; a table that scatters every
    key position over the cache rows gives the bits of the cache rows physically permuted that way."""
    rows, slots = 2, 4
    q, kv = _data(rows, slots, max_length, 5 + max_length)
    row_slot = torch.tensor([3, 1], dtype=torch.int32, device="cuda")
    g = torch.Generator().manual_seed(max_length)
    for L in (1, 64, 65, max_length):
        kw = dict(cur_len=L, max_length=max_length)
        plain = _run(q, kv, row_slot=row_slot, **kw)
        ident = row_slot.view(rows, 1).expand(rows, max_length).contiguous()
        for form in ("cta128", "cta64") if max_length > 128 else ("cta128",):
            assert torch.equal(_run(q, kv, row_slot=row_slot, kv_src=ident, form=form, **kw), _run(q, kv, row_slot=row_slot, form=form, **kw))
        assert torch.equal(_run(q, kv, row_slot=row_slot, kv_src=ident, **kw), plain)
        # key t of row r moves to cache row perm_t[r]
        src = torch.stack([torch.randperm(slots, generator=g)[:rows] for _ in range(max_length)], dim=1).to(torch.int32).cuda()
        moved = torch.randn(slots, max_length, 2 * H * D, generator=g).cuda()
        t = torch.arange(max_length, device="cuda")
        for r in range(rows):
            moved[src[r].long(), t] = kv[int(row_slot[r]), t]
        assert torch.equal(_run(q, moved, kv_src=src, **kw), plain), f"L {L}"
        assert _err(plain, _reference(q, kv, row_slot.tolist(), L)) <= TOL


@pytest.mark.parametrize("max_length", [128, 641, 2048])
def test_row_alone_equals_row_among_16(max_length):
    rows = 16
    q, kv = _data(rows, rows, max_length, 13 + max_length)
    row_slot = torch.randperm(rows, generator=torch.Generator().manual_seed(5)).to(torch.int32).cuda()
    kvld = (torch.rand(rows, max_length, generator=torch.Generator().manual_seed(6)) > 0.1).to(torch.uint8).cuda()
    L, P = max_length - 1, max_length // 3
    kw = dict(cur_len=L, prompt_len=P, max_length=max_length)
    many = _run(q, kv, row_slot=row_slot, key_valid=kvld, **kw)
    assert _err(many, _reference(q, kv, row_slot.tolist(), L, P, kvld)) <= TOL
    for r in (0, 7, 15):
        one = _run(q[r:r + 1].contiguous(), kv, row_slot=row_slot[r:r + 1].contiguous(), key_valid=kvld[r:r + 1].contiguous(), **kw)
        assert torch.equal(one[0], many[r]), f"row {r}"


def test_ragged_rows_equal_their_uniform_launches():
    """One ragged launch holding rows of different plans (1, 2, 3, 11, 17 and 32 splits; a row with an empty split; a row at one key)
    gives each row the bits of the uniform launch of that row with its own max_length."""
    plans = [(1, 64), (128, 128), (150, 193), (640, 704), (700, 1025), (2048, 2048), (600, 2048), (129, 129)]
    rows, t_max = len(plans), 2048
    q, kv = _data(rows, rows, t_max, 17)
    cur, mls = [p[0] for p in plans], [p[1] for p in plans]
    got = _run(q, kv, ragged_cur_len=cur, ragged_max_length=mls)
    for r, (L, ml) in enumerate(plans):
        alone = _run(q[r:r + 1].contiguous(), kv, row_slot=torch.tensor([r], dtype=torch.int32, device="cuda"), cur_len=L, max_length=ml)
        assert torch.equal(got[r], alone[0]), f"row {r}: cur_len {L}, max_length {ml}"
        assert _err(alone, _reference(q[r:r + 1], kv, [r], L)) <= TOL
