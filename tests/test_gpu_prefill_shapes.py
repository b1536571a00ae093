"""Decoder-prefill shapes take their own kernel instantiations: the SIMT GEMM with 64-row tiles when M fits one 128-row tile, and the
SIMT attention with 16 queries per CTA when 64-query CTAs would leave most SMs idle.  Both must give every output bit for bit what
the larger instantiation gives it, so the same rows are compared against a launch big enough to take the other one."""
import pytest
import torch

from mapperatorinator_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N,K", [(768, 768), (1536, 768), (3072, 768), (768, 3072), (384, 512)])
@pytest.mark.parametrize("M", [1, 17, 18, 50, 64, 100, 128])
def test_small_m_gemm_bitwise(M, N, K):
    g = torch.Generator().manual_seed(M * 7 + N + K)
    big = 300                                                  # > 128 rows: 128-row tiles; < 512: stays on the SIMT path
    a = (torch.randn(big, K, generator=g) * 0.5).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(big, N, generator=g).cuda()
    for act, r in (("none", None), ("gelu", None), ("none", res)):
        small = ops.gemm(a[:M].contiguous(), w, bias, act=act, residual=None if r is None else r[:M].contiguous())
        ref = ops.gemm(a, w, bias, act=act, residual=r)
        assert torch.equal(small, ref[:M]), (M, N, K, act)


@pytest.mark.parametrize("Tq", [1, 17, 18, 50, 64, 128])
@pytest.mark.parametrize("kind", ["causal_leftpad", "causal_offset", "cross"])
def test_short_query_attention_bitwise(Tq, kind):
    H, Bbig = 12, 12                                          # 12 x 12 (batch, head) CTAs >= 132 SMs: the 64-query kernel
    g = torch.Generator().manual_seed(Tq)
    q_pos0 = 37 if kind == "causal_offset" else 0             # queries after 37 cached keys (a ragged request's later rows)
    Tk = {"causal_leftpad": Tq, "causal_offset": Tq + q_pos0, "cross": 512}[kind]
    q = torch.randn(Bbig, Tq, H * 64, generator=g).cuda()
    k = torch.randn(Bbig, Tk, H * 64, generator=g).cuda()
    v = torch.randn(Bbig, Tk, H * 64, generator=g).cuda()
    kv = None
    mask = "none"
    if kind != "cross":
        mask = "causal"
        kv = torch.ones(Bbig, Tk, dtype=torch.uint8)
        for b in range(Bbig):
            kv[b, :min(b, Tk - 1)] = 0                        # left padding of b tokens (row 0 unpadded)
        kv = kv.cuda()
    ref = ops.attention(q, k, v, H, 1.0, mask, q_pos0, key_valid=kv)
    for b0, n in ((0, 1), (Bbig // 2, 1), (Bbig - 1, 1), (4, 2)):          # single rows and a CFG-shaped pair
        sl = slice(b0, b0 + n)
        got = ops.attention(q[sl].contiguous(), k[sl].contiguous(), v[sl].contiguous(), H, 1.0, mask, q_pos0,
                            key_valid=None if kv is None else kv[sl].contiguous())
        assert torch.equal(got, ref[sl]), (Tq, kind, b0, n)


@pytest.fixture(scope="module")
def wide():
    """whisper-small dimensions with room for 12 decoder rows over 2 resident encoder slots."""
    from mapperatorinator_b200 import v29_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = v29_model_config()
    model = B200Mapperatorinator(cfg, init_model_state_dict(cfg, 0), max_windows=2, max_batch=12)
    pcm = torch.randn(2, cfg.samples_per_window, generator=torch.Generator().manual_seed(3)) * 0.1
    model.engine.encode(pcm.cuda(), 0)
    return cfg, model


@pytest.mark.parametrize("P", [17, 40])
def test_prefill_rows_bitwise_alone_and_in_twelve(wide, P):
    """The whole decoder prefill through the engine (cross-attention through the row -> encoder slot table, left-padded causal
    self-attention, every projection): a row alone or in a CFG-sized pair runs the 16-query attention and 64-row GEMM tiles, the
    same row among 12 (12 x 12 CTAs; 12 * P < 512 rows keeps the SIMT GEMM) runs the 64-query attention and 128-row tiles.
    All-position logits must agree bit for bit."""
    cfg, model = wide
    g = torch.Generator().manual_seed(P)
    ids = torch.randint(4, 3000, (12, P), generator=g)
    mask = torch.ones(12, P, dtype=torch.bool)
    for r in range(12):
        mask[r, :r % 4] = False                               # 0..3 left-pad tokens
        ids[r, :r % 4] = 0
    slots = [r % 2 for r in range(12)]
    big = model.engine.forward_logits(slots, ids, mask).cpu()
    for b0, n in ((0, 1), (3, 1), (7, 1), (2, 2)):
        got = model.engine.forward_logits(slots[b0:b0 + n], ids[b0:b0 + n], mask[b0:b0 + n]).cpu()
        assert torch.equal(got, big[b0:b0 + n]), (P, b0, n)
