"""Kernel-level parity: each CUDA kernel, called through the C ABI, against plain torch fp32 on the CPU."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("M,N,K", [(1, 4, 128), (77, 130, 388), (300, 768, 768), (257, 3667, 128), (513, 256, 600),
                                   (50, 768, 768), (64, 3667, 128), (33, 130, 388), (18, 768, 3072)])   # M <= 64: skinny kernel
@pytest.mark.parametrize("act", ["none", "gelu", "gelu_tanh", "silu"])
def test_gemm_epilogues(M, N, K, act):
    from mapperatorinator_b200 import ops
    g = _g(M * 31 + N)
    a, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K)
    bias, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    rpb = 7
    gate = torch.randn((M + rpb - 1) // rpb, N, generator=g)
    ref = F.linear(a, w, bias)
    ref = {"none": lambda x: x, "gelu": F.gelu, "gelu_tanh": lambda x: F.gelu(x, approximate="tanh"), "silu": F.silu}[act](ref) * 0.5
    ref = res + gate.repeat_interleave(rpb, 0)[:M] * ref
    out = ops.gemm(a.cuda(), w.cuda(), bias.cuda(), act, 0.5, res.cuda(), gate.cuda(), rpb).cpu()
    assert torch.allclose(out, ref, rtol=2e-5, atol=2e-5), (out - ref).abs().max()


@pytest.mark.parametrize("M,N,K", [(1024, 768, 768), (640, 3072, 388), (512, 130, 3072), (2048, 2304, 768), (1500, 768, 2304)])
def test_gemm_tcgen05_3xtf32_matches_fp64(M, N, K):
    """The tensor-core path must be fp32-grade (3xTF32 split, fp32 accumulation): error vs an fp64 product far below plain
    TF32 (~1e-3).  The operand split is exact to ~2^-22 but the tensor core's fp32 accumulator truncates (not rounds) each
    partial sum, so the error grows with K (to ~8e-6 relative at K = 3072; SIMT FMA kernel: ~1e-6).  The bound below leaves
    head-room over that envelope; token-level parity with tensor cores on is covered in test_gpu_model."""
    from mapperatorinator_b200 import ops
    g = _g(M + N + K)
    a, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K)
    bias, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    ref = F.gelu(a.double() @ w.double().T + bias.double()) * 0.5 + res.double()
    tc = ops.gemm_tc(a.cuda(), w.cuda(), bias.cuda(), "gelu", 0.5, res.cuda()).cpu().double()
    simt = ops.gemm(a.cuda(), w.cuda(), bias.cuda(), "gelu", 0.5, res.cuda()).cpu().double()
    scale = ref.abs().max().item()
    e_tc, e_simt = (tc - ref).abs().max().item() / scale, (simt - ref).abs().max().item() / scale
    assert e_tc <= max(2e-5, 3 * e_simt), (e_tc, e_simt)       # fp32-grade (plain TF32 would be ~1e-3)


@pytest.mark.parametrize("dim", [128, 768, 1024])
def test_layernorm_affine_and_modulate(dim):
    from mapperatorinator_b200 import ops
    g = _g(dim)
    x = torch.randn(37, dim, generator=g) * 3 + 1
    w, b = torch.randn(dim, generator=g), torch.randn(dim, generator=g)
    ref = F.layer_norm(x, (dim,), w, b, 1e-5)
    out = ops.layernorm(x.cuda(), w.cuda(), b.cuda(), eps=1e-5).cpu()
    assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5)
    rpb = 10
    sh, sc = torch.randn(4, dim, generator=g), torch.randn(4, dim, generator=g)
    ref = F.layer_norm(x, (dim,), eps=1e-6) * (1 + sc.repeat_interleave(rpb, 0)[:37]) + sh.repeat_interleave(rpb, 0)[:37]
    out = ops.layernorm(x.cuda(), shift=sh.cuda(), scale=sc.cuda(), rows_per_batch=rpb, eps=1e-6).cpu()
    assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5)


def _ref_attn(q, k, v, H, allowed):
    B, Tq, D = q.shape
    sp = lambda z: z.view(B, -1, H, 64).transpose(1, 2)
    s = sp(q) @ sp(k).transpose(2, 3)
    s = s.masked_fill(~allowed[:, None], float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    return (p @ sp(v)).transpose(1, 2).reshape(B, Tq, D)


@pytest.mark.parametrize("Tq,Tk", [(64, 64), (70, 70), (512, 512), (33, 512), (300, 300)])
@pytest.mark.parametrize("mode", ["none", "causal", "band", "dense"])
def test_attention_masks(Tq, Tk, mode):
    from mapperatorinator_b200 import ops
    if mode in ("causal", "band", "dense") and Tq != Tk:
        pytest.skip("square only")
    B, H = 2, 3
    g = _g(Tq * 7 + Tk)
    q, k, v = (torch.randn(B, t, H * 64, generator=g) * 0.5 for t in (Tq, Tk, Tk))
    r, c = torch.arange(Tq)[:, None], torch.arange(Tk)[None, :]
    allowed = torch.ones(B, Tq, Tk, dtype=torch.bool)
    kw = {}
    if mode == "causal":
        kvalid = torch.ones(B, Tk, dtype=torch.uint8)
        kvalid[1, :5] = 0                                    # left padding on row 1 (fully masked pad queries -> 0)
        allowed = (c <= r)[None] & kvalid.bool()[:, None, :]
        kw = dict(key_valid=kvalid.cuda())
    elif mode == "band":
        w = 128 if Tq > 200 else 17
        allowed = ((r >= c - w) & (r < c + w))[None].expand(B, -1, -1)
        kw = dict(band=w)
    elif mode == "dense":
        dm = torch.rand(Tq, Tk, generator=g) < 0.3
        dm[torch.arange(Tq), torch.arange(Tq)] = False
        allowed = (~dm)[None].expand(B, -1, -1)
        kw = dict(dense_mask=dm.to(torch.uint8).cuda())
    ref = _ref_attn(q, k, v, H, allowed)
    out = ops.attention(q.cuda(), k.cuda(), v.cuda(), H, 1.0, mode, 0, **kw).cpu()
    assert torch.allclose(out, ref, rtol=2e-5, atol=2e-5), (out - ref).abs().max()


@pytest.mark.parametrize("Tq,Tk,mode,scale", [(1024, 1024, "band", 0.125), (512, 512, "none", 1.0), (130, 700, "none", 0.3),
                                              (333, 333, "causal", 1.0), (260, 260, "band", 1.0)])
def test_attention_tensor_cores(Tq, Tk, mode, scale):
    """wgmma flash attention (3xTF32 for Q.K^T and P.V, online softmax in registers) vs an fp64 reference, and against the
    fp32 SIMT kernel it replaces: DiT shape (T = 1024, +-128 band), encoder shape (T = 512), ragged tiles, causal with left padding."""
    from mapperatorinator_b200 import _lib, ops
    lib = _lib.load()
    B, H = 2, 3
    g = _g(Tq * 3 + Tk)
    q, k, v = (torch.randn(B, t, H * 64, generator=g) for t in (Tq, Tk, Tk))
    r, c = torch.arange(Tq)[:, None], torch.arange(Tk)[None, :]
    allowed = torch.ones(B, Tq, Tk, dtype=torch.bool)
    kw = {}
    if mode == "causal":
        kvalid = torch.ones(B, Tk, dtype=torch.uint8)
        kvalid[1, :9] = 0
        allowed = (c <= r)[None] & kvalid.bool()[:, None, :]
        kw = dict(key_valid=kvalid.cuda())
    elif mode == "band":
        allowed = ((r >= c - 128) & (r < c + 128))[None].expand(B, -1, -1)
        kw = dict(band=128)
    ref = _ref_attn((q * scale).double(), k.double(), v.double(), H, allowed).float()
    try:
        _lib.check(lib.mb200_set_attention_tc(1, 64))
        out_tc = ops.attention(q.cuda(), k.cuda(), v.cuda(), H, scale, mode, 0, **kw).cpu()
        _lib.check(lib.mb200_set_attention_tc(0, 256))
        out_simt = ops.attention(q.cuda(), k.cuda(), v.cuda(), H, scale, mode, 0, **kw).cpu()
    finally:
        _lib.check(lib.mb200_set_attention_tc(1, 256))
    assert torch.allclose(out_tc, ref, rtol=2e-5, atol=2e-5), (out_tc - ref).abs().max()
    assert torch.allclose(out_tc, out_simt, rtol=2e-5, atol=2e-5), (out_tc - out_simt).abs().max()


@pytest.mark.parametrize("flavour", ["nnAudio", "torchaudio", "torchaudio_log_reflect"])
@pytest.mark.parametrize("n_samples", [130944, 128 * 37])
def test_mel_vs_oracle(flavour, n_samples):
    from mapperatorinator_b200 import MelConfig
    from mapperatorinator_b200.engine import MelEngine
    from oracle import mel as mo
    cfg = {"nnAudio": MelConfig(), "torchaudio": MelConfig("torchaudio", n_mels=80),
           "torchaudio_log_reflect": MelConfig("torchaudio", True, n_mels=128, f_min=20, pad_mode="reflect")}[flavour]
    g = _g(n_samples)
    t = torch.arange(n_samples) / 16000.0
    pcm = 0.3 * torch.sin(2 * math.pi * 440 * t)[None] + 0.05 * torch.randn(3, n_samples, generator=g)
    ref = mo.mel_forward(pcm, cfg)
    out = MelEngine(cfg).forward(pcm.cuda()).cpu()
    assert out.shape == ref.shape
    scale = ref.abs().max()
    assert (out - ref).abs().max() <= 2e-5 * scale + 1e-6, ((out - ref).abs().max(), scale)
