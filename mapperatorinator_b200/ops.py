"""Kernel-level wrappers over the C ABI (`mb200_op_*`) for parity tests; operands are CUDA torch tensors."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib

ACT = {"none": 0, "gelu": 1, "gelu_tanh": 2, "silu": 3}
MASK = {"none": 0, "causal": 1, "band": 2, "dense": 3}


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f32c(t: torch.Tensor) -> torch.Tensor:
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    return t


GEMM_PATHS = {"engine": 0, "simt": 1, "tc": 2}


def _rowmap(t: torch.Tensor, what: str):
    """RowMap of a float32 CUDA view: 2-D (rows, cols) -> rows at stride(0); 3-D (batches, rpb, cols) -> ld = stride(1), bstride =
    stride(0), so `as_strided` views with overlapping rows and `expand`ed tables (stride(0) == 0) map directly.  Returns (map, rows)."""
    assert t.is_cuda and t.dtype == torch.float32 and t.stride(-1) == 1, f"{what}: float32 CUDA view with unit column stride"
    if t.dim() == 2:
        return _lib.RowMapC(t.data_ptr(), t.stride(0), 0, 0), t.shape[0]
    assert t.dim() == 3, f"{what}: 2-D (rows, cols) or 3-D (batches, rows per batch, cols)"
    return _lib.RowMapC(t.data_ptr(), t.stride(1), t.shape[1], t.stride(0)), t.shape[0] * t.shape[1]


def gemm_mapped(a, w, c, bias=None, act="none", alpha=1.0, residual=None, gate=None, gate_rows_per_batch=1, path="engine"):
    """c = act(a @ w.T + bias) * alpha [* gate[row // gate_rows_per_batch]] [+ residual], written through the views' row maps
    (`mb200_op_gemm_mapped`).  a (rows, K) or (batches, rpb, K); c and residual (rows, N) or (batches, rpb, N), the same row count
    (residual may be c itself); w (N, K) and gate (groups, N) with unit column stride.  path "engine" dispatches as the engine does for a
    registered weight, "simt" forces the fp32 kernel, "tc" the wgmma 3xTF32 kernel (an error if the problem is not eligible).  Returns c."""
    lib = _lib.load()
    am, M = _rowmap(a, "a")
    cm, Mc = _rowmap(c, "c")
    assert w.is_cuda and w.dtype == torch.float32 and w.dim() == 2 and w.stride(1) == 1
    N, K = w.shape
    assert a.shape[-1] == K and c.shape[-1] == N and Mc == M, "shapes do not chain"
    rm = None
    if residual is not None:
        rm, Mr = _rowmap(residual, "residual")
        assert residual.shape[-1] == N and Mr == M
    if gate is not None:
        assert gate.is_cuda and gate.dtype == torch.float32 and gate.dim() == 2 and gate.stride(1) == 1 and gate.shape[1] == N
    if bias is not None:
        assert bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == N
    _lib.check(lib.mb200_op_gemm_mapped(am, _ptr(w), w.stride(0), cm, _ptr(bias), ACT[act], float(alpha), rm, _ptr(gate),
                                        gate.stride(0) if gate is not None else 0, int(gate_rows_per_batch), M, N, K, GEMM_PATHS[path],
                                        _stream()))
    return c


def gemm(a, w, bias=None, act="none", alpha=1.0, residual=None, gate=None, gate_rows_per_batch=1):
    """act(a @ w.T + bias) * alpha [* gate[row // rpb]] [+ residual], on the fp32 SIMT kernel."""
    a, w = _f32c(a), _f32c(w)
    out = torch.empty(a.shape[0], w.shape[0], device=a.device, dtype=torch.float32)
    return gemm_mapped(a, w, out, bias, act, alpha, residual, gate, gate_rows_per_batch, path="simt")


def gemm_tc(a, w, bias=None, act="none", alpha=1.0, residual=None):
    """Same contract as `gemm`, forced through the wgmma 3xTF32 kernel."""
    a, w = _f32c(a), _f32c(w)
    out = torch.empty(a.shape[0], w.shape[0], device=a.device, dtype=torch.float32)
    return gemm_mapped(a, w, out, bias, act, alpha, residual, path="tc")


def layernorm(x, weight=None, bias=None, shift=None, scale=None, rows_per_batch=1, eps=1e-5):
    """LayerNorm of the rows of x: affine (weight / bias), or modulate by shift / scale (batches, dim) rows, which may be views into a
    wider buffer (their common row stride is the modulation stride)."""
    lib = _lib.load()
    x = _f32c(x)
    rows, dim = x.shape
    y = torch.empty_like(x)
    mod_ld = 0
    if shift is not None:
        assert shift.stride() == scale.stride() and shift.stride(1) == 1, "shift and scale rows at one stride"
        mod_ld = shift.stride(0)
    _lib.check(lib.mb200_op_layernorm(_ptr(x), _ptr(y), _ptr(weight), _ptr(bias), _ptr(shift), _ptr(scale), mod_ld, int(rows_per_batch), rows,
                                      dim, float(eps), _stream()))
    return y


def attention(q, k, v, heads, scale=1.0, mask="none", q_pos0=0, key_valid=None, band=0, dense_mask=None, kv_slot=None, out=None):
    """q (B, Tq, >= H*64), k / v (B or slots, Tk, >= H*64) token-major views with unit column stride (column slices of one qkv buffer,
    the K | V cache) -> out (B, Tq, H*64), allocated when not given.  key_valid (B, >= Tk) uint8 view; kv_slot int32 (B,): batch row b
    reads K / V of batch index kv_slot[b]."""
    lib = _lib.load()
    for t in (q, k, v):
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 3 and t.stride(2) == 1
    B, Tq, _ = q.shape
    Tk = k.shape[1]
    if out is None:
        out = torch.empty(B, Tq, heads * 64, device=q.device, dtype=torch.float32)
    assert out.is_cuda and out.dtype == torch.float32 and out.dim() == 3 and out.stride(2) == 1
    if key_valid is not None:
        assert key_valid.is_cuda and key_valid.dtype == torch.uint8 and key_valid.stride(1) == 1
    if kv_slot is not None:
        assert kv_slot.is_cuda and kv_slot.dtype == torch.int32 and kv_slot.is_contiguous() and kv_slot.numel() == B
    _lib.check(lib.mb200_op_attention(_ptr(q), q.stride(1), q.stride(0), _ptr(k), k.stride(1), k.stride(0), _ptr(v), v.stride(1), v.stride(0),
                                      _ptr(out), out.stride(1), out.stride(0), B, heads, Tq, Tk, float(scale), MASK[mask], int(q_pos0),
                                      _ptr(key_valid), key_valid.stride(0) if key_valid is not None else 0, int(band), _ptr(dense_mask),
                                      _ptr(kv_slot), _stream()))
    return out


DECODE_ATTENTION_FORMS = {"default": 0, "cta128": 1, "cta64": 2, "warp": 3}


def decode_attention(q, kv, heads, *, row_slot=None, cur_len=0, prompt_len=0, key_valid=None, max_length=0, fixed_len=0, kv_src=None,
                     ragged_cur_len=None, ragged_max_length=None, form="default"):
    """One split-KV decode-attention phase of the token loop (`mb200_op_decode_attention`).

    q (rows, H*64) already scaled; kv the engine's K|V cache (slots, T_max, 2*H*64); row_slot int32 (rows,) cache row per decoder row;
    key_valid uint8 (rows, ld) prompt mask; kv_src int32 (rows, ld) source-row table.  Self attention over keys [0, cur_len) with the
    split plan of `max_length`, cross attention over [0, fixed_len) when fixed_len > 0, or a ragged launch when the per-row lists
    `ragged_cur_len` / `ragged_max_length` are given.  Returns the merged heads (rows, H*64)."""
    import ctypes as C
    lib = _lib.load()
    q, kv = _f32c(q), _f32c(kv)
    rows = q.shape[0]
    slots, t_max, _ = kv.shape
    for t, dt in ((row_slot, torch.int32), (key_valid, torch.uint8), (kv_src, torch.int32)):
        assert t is None or (t.is_cuda and t.dtype == dt and t.is_contiguous())
    out = torch.empty_like(q)
    rc = rm = None
    if ragged_cur_len is not None:
        rc = (C.c_int32 * rows)(*[int(x) for x in ragged_cur_len])
        rm = (C.c_int32 * rows)(*[int(x) for x in ragged_max_length])
    _lib.check(lib.mb200_op_decode_attention(_ptr(q), _ptr(kv), slots, t_max, int(heads), rows, _ptr(row_slot), int(cur_len), int(prompt_len),
                                             _ptr(key_valid), key_valid.shape[1] if key_valid is not None else 0, int(max_length),
                                             int(fixed_len), _ptr(kv_src), kv_src.shape[1] if kv_src is not None else 0,
                                             None if rc is None else C.cast(rc, C.c_void_p), None if rm is None else C.cast(rm, C.c_void_p),
                                             DECODE_ATTENTION_FORMS[form], _ptr(out), _stream()))
    return out


@dataclass
class GemvSegment:
    """Columns [n_begin, n_end) of a GEMV's stacked weight, written from the data pointer of `out` (any float32 CUDA view): row b at
    b * out_bs + (cur_len - 1) * pos_stride + (n - n_begin), the middle term only for a segment that writes at the cache position."""
    out: torch.Tensor
    n_begin: int
    n_end: int
    out_bs: int
    pos_stride: int = 0
    act: str = "none"
    alpha: float = 1.0


GEMV_FORMS = {"kernel": 0, "mega": 1}


def gemv(x, w, bias=None, *, ln_weight=None, ln_bias=None, eps=1e-5, xmode=None, residual=None, act="none", alpha=1.0, out=None,
         segments=None, cur_len=0, ragged_cur_len=None, ragged_finished=None, n_req=None, form="kernel"):
    """One weight-streaming GEMV phase of the token loop (`mb200_op_gemv`): act(w @ X(x[b]) + bias) * alpha + residual[b].

    x (B, K) and w (N, K) may be row-strided views (unit column stride); X is the fused LayerNorm when ln_weight / ln_bias are given
    (xmode "layernorm", or force either mode by name).  Without `segments` the output is one segment over [0, N) into `out` (allocated
    (B, N) when not given; it may be `residual` itself) and is returned.  `segments` (GemvSegment, 1 to 3) route the columns instead,
    positional ones at `cur_len` (or per request: ragged_cur_len / ragged_finished with rows r and r + n_req sharing request r).
    form "kernel" is the per-phase kernel, "mega" the barrier megakernel's phase body.  A bfloat16 `w` runs the bf16-weight GEMV of
    the token loop's bf16 store (`mb200_op_gemv_bf16`: K and w's row stride multiples of 8, rows 16-byte aligned)."""
    import ctypes as C
    lib = _lib.load()
    w_bf16 = w.dtype == torch.bfloat16
    assert w.is_cuda and w.stride(-1) == 1 and w.dtype in (torch.float32, torch.bfloat16)
    for t in (x, bias, ln_weight, ln_bias, residual, out):
        assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.stride(-1) == 1)
    B, K = x.shape
    N = w.shape[0]
    if xmode is None:
        xmode = "layernorm" if ln_weight is not None else "plain"
    if segments is None:
        if out is None:
            out = torch.empty(B, N, device=x.device, dtype=torch.float32)
        segments = [GemvSegment(out, 0, N, out.stride(0), 0, act, alpha)]
    segs = (_lib.GemvSegC * len(segments))(*[_lib.GemvSegC(s.out.data_ptr(), int(s.out_bs), int(s.pos_stride), int(s.n_begin), int(s.n_end),
                                                             float(s.alpha), ACT[s.act]) for s in segments])
    rc = rf = None
    if ragged_cur_len is not None:
        n_req = len(ragged_cur_len) if n_req is None else n_req
        rc = (C.c_int32 * n_req)(*[int(v) for v in ragged_cur_len])
        rf = (C.c_int32 * n_req)(*[int(v) for v in ragged_finished])
    _lib.check((lib.mb200_op_gemv_bf16 if w_bf16 else lib.mb200_op_gemv)(_ptr(x), x.stride(0), B, K, {"plain": 0, "layernorm": 1}[xmode], _ptr(ln_weight), _ptr(ln_bias), float(eps),
                                 _ptr(w), w.stride(0), N, _ptr(bias), _ptr(residual), residual.stride(0) if residual is not None else 0,
                                 segs, len(segments), int(cur_len), None if rc is None else C.cast(rc, C.c_void_p),
                                 None if rf is None else C.cast(rf, C.c_void_p), int(n_req or 0), GEMV_FORMS[form], _stream()))
    return out
