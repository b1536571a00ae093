// Device-side bodies of the decode path, shared by the per-kernel launches (decode.cu) and the persistent token-loop
// megakernel (decode_mega.cu).  Everything that one CTA reads and ANOTHER CTA may have written during the same launch
// (residual stream, q, split-KV partials, logits, ids, K/V cache rows, GenState) is loaded with ld.global.cg (L2) so the
// same code is coherent inside a persistent kernel, where L1 is not invalidated between phases.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace mb200 {

__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float2 ldcg2(const float* p) { return __ldcg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ int ld_state(const int* p) { return __ldcg(p); }

// ---- tagged pairs of the dataflow megakernel (decode_mega2.cu): one 64-bit word = fp32 bits | tag << 32, written by ONE 64-bit
// store, so a reader that sees the expected tag also sees the value (NCCL's "LL" protocol).  Scalar 64-bit accesses: single-copy atomic.
typedef unsigned long long ll_t;
__device__ __forceinline__ void ll_store(ll_t* p, float v, unsigned tag) {
    asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(((ll_t)tag << 32) | (ll_t)__float_as_uint(v)) : "memory");
}
__device__ __forceinline__ void ll_store2(ll_t* p, float a, float b, unsigned tag) {      // p 16-byte aligned
    asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"(((ll_t)tag << 32) | (ll_t)__float_as_uint(a)),
                 "l"(((ll_t)tag << 32) | (ll_t)__float_as_uint(b)) : "memory");
}
__device__ __forceinline__ void ll_load2(const ll_t* p, ll_t& a, ll_t& b) {                // p 16-byte aligned
    asm volatile("ld.relaxed.gpu.global.v2.b64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
static __constant__ int c_ll_sleep_ns = 0;      // tuning knob (engine option "ll_sleep"): back off this long after a failed poll (0 = spin)
constexpr long long LL_SPIN_LIMIT = 1ll << 24;      // ~ seconds; a dataflow wait that long is a bug, never a slow producer
// Wait for one / two / four consecutive pairs carrying `tag`.  Bounded: on a timeout (or when another CTA raised `err`) the error flag is
// set and zeros are returned, so a logic error ends the launch instead of hanging the GPU.
// diagnostics only (engine option "ll_debug", tools/mega2_trace.py): bit 0 = no weight copies, bit 1 = polls never wait (whatever is in the
// exchange buffer is taken), bit 2 = GEMV phases skip their multiply-reduce.  Any bit set -> the tokens are garbage, the TIMING tells
// which part of a phase the time goes to.
static __constant__ int c_ll_debug = 0;
// The wait that times out first also records where it was: err[1] = CTA, err[2] = thread, err[3] = the tag it expected, i.e. the step
// (tag / 128 - 1) and the phase (tag % 128 - 1) whose output never arrived.  Waits that give up because the flag is already raised
// record nothing.
__device__ __forceinline__ bool ll_spin_check(long long& spin, int* err, unsigned tag) {
    if (c_ll_debug & 2) return false;
    if (c_ll_sleep_ns > 0) __nanosleep((unsigned)c_ll_sleep_ns);
    if ((++spin & 0x3FF) == 0 && (spin > LL_SPIN_LIMIT || *reinterpret_cast<volatile int*>(err) != 0)) {
        if (spin > LL_SPIN_LIMIT && atomicCAS(err, 0, 4) == 0) {
            err[1] = (int)blockIdx.x; err[2] = (int)threadIdx.x; err[3] = (int)tag;
            __threadfence();
        }
        return false;
    }
    return true;
}
__device__ __forceinline__ float ll_wait1(const ll_t* p, unsigned tag, int* err) {
    ll_t v;
    long long spin = 0;
    while (true) {
        asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
        if ((unsigned)(v >> 32) == tag) return __uint_as_float((unsigned)v);
        if (!ll_spin_check(spin, err, tag)) return 0.f;
    }
}
__device__ __forceinline__ float2 ll_wait2(const ll_t* p, unsigned tag, int* err) {
    ll_t a, b;
    long long spin = 0;
    while (true) {
        ll_load2(p, a, b);
        if ((unsigned)(a >> 32) == tag && (unsigned)(b >> 32) == tag) return make_float2(__uint_as_float((unsigned)a), __uint_as_float((unsigned)b));
        if (!ll_spin_check(spin, err, tag)) return make_float2(0.f, 0.f);
    }
}
__device__ __forceinline__ float4 ll_wait4(const ll_t* p, unsigned tag, int* err) {        // p 32-byte aligned
    ll_t a, b, c, d;
    long long spin = 0;
    while (true) {
        ll_load2(p, a, b);
        ll_load2(p + 2, c, d);
        if ((unsigned)(a >> 32) == tag && (unsigned)(b >> 32) == tag && (unsigned)(c >> 32) == tag && (unsigned)(d >> 32) == tag)
            return make_float4(__uint_as_float((unsigned)a), __uint_as_float((unsigned)b), __uint_as_float((unsigned)c), __uint_as_float((unsigned)d));
        if (!ll_spin_check(spin, err, tag)) return make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// activation staging for the GEMV family: xs[NB][K] <- LayerNorm(x) | x
// ---------------------------------------------------------------------------------------------------------------------
template <int NB, int NT>
__device__ __forceinline__ void gemv_stage_x(const GemvParams& p, int b0, float* xs, float* scratch /* >= 32 floats */,
                                             int tid, unsigned long long* dbg = nullptr /* trace: loads-landed stamp */) {
    constexpr int nthreads = NT;
    const int lane = tid & 31, warp = tid >> 5;
    const int K = p.K, K4 = K >> 2;
    if (p.xmode == X_LAYERNORM) {
        // All warps share the row(s): float4 index idx = c*32 + lane belongs to chunk c in [0, 8) (K <= 1024).  Each chunk is reduced
        // by one warp, the 8 chunk partials by a fixed tree, so the arithmetic does not depend on the caller's warp count (the
        // per-kernel path with 4 warps and the megakernel with 16 stay bit-identical).  Per lane only 1-2 float4 triples are live:
        // the old one-warp-per-row form held 24 float4 in flight, which (a) serialised ~3000 cycles on one warp and (b) under the
        // megakernel's 128-register cap spilled freshly loaded values to local memory, i.e. waited for them.
        constexpr int NW = NT / 32;
        static_assert(NW == 1 || NW == 2 || NW == 4 || NW == 8 || NW == 16 || NW == 32, "warp count must be a power of two");
        constexpr int CPW = NW >= 8 ? 1 : 8 / NW;          // chunks per warp inside a row
        constexpr int RG = NW >= 8 ? NW / 8 : 1;           // rows staged per round
        float* red = scratch;                              // [2][RG][8]
        const float inv = 1.0f / (float)K;
        for (int g0 = 0; g0 < NB; g0 += RG) {
            const int rl = (warp * CPW) >> 3, bb = g0 + rl, c0 = (warp * CPW) & 7;
            const bool row_ok = rl < RG && bb < NB && b0 + bb < p.B;
            const float* src = p.x + (long long)(b0 + bb) * p.x_ld;
            float4 v[CPW], lw[CPW], lb[CPW];
#pragma unroll
            for (int i = 0; i < CPW; ++i) {
                const int idx = (c0 + i) * 32 + lane;
                const bool ok = row_ok && idx < K4;
                v[i] = ok ? ldcg4(src + idx * 4) : make_float4(0, 0, 0, 0);
                lw[i] = ok ? __ldg(reinterpret_cast<const float4*>(p.ln_w) + idx) : make_float4(0, 0, 0, 0);
                lb[i] = ok ? __ldg(reinterpret_cast<const float4*>(p.ln_b) + idx) : make_float4(0, 0, 0, 0);
            }
#pragma unroll
            for (int i = 0; i < CPW; ++i) {
                const float sc = warp_sum((v[i].x + v[i].y) + (v[i].z + v[i].w));
                if (lane == 0 && rl < RG) red[rl * 8 + c0 + i] = sc;
            }
            if (dbg && tid == 0) *dbg = (unsigned long long)clock64();
            __syncthreads();
            float mean = 0.f;
            if (rl < RG) {
                const float* r = red + rl * 8;
                mean = (((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))) * inv;
            }
#pragma unroll
            for (int i = 0; i < CPW; ++i) {
                const bool ok = row_ok && (c0 + i) * 32 + lane < K4;
                float q = 0.f;
                if (ok) {
                    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
                    q = (a * a + b * b) + (c * c + d * d);
                }
                q = warp_sum(q);
                if (lane == 0 && rl < RG) red[RG * 8 + rl * 8 + c0 + i] = q;
            }
            __syncthreads();
            if (rl < RG && bb < NB) {
                const float* r = red + RG * 8 + rl * 8;
                const float rstd = rsqrtf((((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))) * inv + p.eps);
                float* dst = xs + bb * K;
#pragma unroll
                for (int i = 0; i < CPW; ++i) {
                    const int idx = (c0 + i) * 32 + lane;
                    if (idx < K4) {
                        float4 o = make_float4(0, 0, 0, 0);
                        if (row_ok) {
                            o.x = (v[i].x - mean) * rstd * lw[i].x + lb[i].x; o.y = (v[i].y - mean) * rstd * lw[i].y + lb[i].y;
                            o.z = (v[i].z - mean) * rstd * lw[i].z + lb[i].z; o.w = (v[i].w - mean) * rstd * lw[i].w + lb[i].w;
                        }
                        reinterpret_cast<float4*>(dst)[idx] = o;
                    }
                }
            }
            // no barrier between rounds: the next round's first write to either half of `red` is ordered behind this round's reads
            // of that half by the barrier in between
        }
    } else {
        // plain rows: a thread's loads are all issued before its first store (one L2 round trip for up to 4*NT float4)
        for (int e0 = tid; e0 < NB * K4; e0 += 4 * nthreads) {
            float4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int e = e0 + u * nthreads, bb = e / K4, c = e - bb * K4;
                v[u] = (e < NB * K4 && b0 + bb < p.B) ? ldcg4(p.x + (long long)(b0 + bb) * p.x_ld + c * 4) : make_float4(0, 0, 0, 0);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int e = e0 + u * nthreads;
                if (e < NB * K4) reinterpret_cast<float4*>(xs)[e] = v[u];
            }
        }
    }
}

// one output row n for NB batch rows: dot(W[n, :], xs[b, :]) with the weight row at `wrow` (global or shared memory)
template <int NB>
__device__ __forceinline__ void gemv_row_operands(const GemvParams& p, int n, int b0, int lane, float& bias_v, float& r_v) {
    // epilogue operands (bias of output n, residual of (row lane, n)); fetched early so their latency hides under the dot product
    bias_v = 0.f; r_v = 0.f;
    if (lane < NB && b0 + lane < p.B) {
        if (p.bias) bias_v = __ldg(p.bias + n);
        if (p.R) r_v = __ldcg(p.R + (long long)(b0 + lane) * p.r_ld + n);
    }
}

// dot(W[n, :], xs[b, :]) for NB batch rows; lane b < NB ends up holding row b's sum in `mine`.  Four independent accumulation chains
// per batch row (the x / y / z / w components of the float4 stream), merged as (x + y) + (z + w) before the shuffle tree.  Shared by
// every decode driver (per-kernel GEMV, barrier megakernel, dataflow megakernel): same order, same bits.
// WBF16: the row holds bf16 bits (wrow_f is reinterpreted).  A lane loads the 4 weights of group idx as 8 bytes instead of 16, widens
// them (exact) and runs the same FMAs in the same order, so the result is the bits of the fp32 kernel on the widened row.
__device__ __forceinline__ float4 bf16x4_to_float4(uint2 v) {
    return make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xffff0000u));
}
template <int NB, bool W_GLOBAL, bool WBF16 = false>
__device__ __forceinline__ float gemv_dot(int K, const float* wrow_f, const float* xs, int lane, unsigned long long* dbg = nullptr) {
    const int K4 = K >> 2;
    float4 acc[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) acc[b] = make_float4(0.f, 0.f, 0.f, 0.f);
    constexpr int U = W_GLOBAL ? 12 : 6;     // loads in flight per lane (same j-major summation order either way)
    for (int base = 0; base < K4; base += 32 * U) {
        float4 w[U];
        if constexpr (WBF16) {
            const uint2* wrow = reinterpret_cast<const uint2*>(wrow_f);
            uint2 raw[U];
#pragma unroll
            for (int j = 0; j < U; ++j) {
                int idx = base + j * 32 + lane;
                if (W_GLOBAL) raw[j] = idx < K4 ? __ldg(wrow + idx) : make_uint2(0, 0);
                else          raw[j] = idx < K4 ? wrow[idx] : make_uint2(0, 0);
            }
#pragma unroll
            for (int j = 0; j < U; ++j) w[j] = bf16x4_to_float4(raw[j]);
        } else {
            const float4* wrow = reinterpret_cast<const float4*>(wrow_f);
#pragma unroll
            for (int j = 0; j < U; ++j) {
                int idx = base + j * 32 + lane;
                if (W_GLOBAL) w[j] = idx < K4 ? __ldg(wrow + idx) : make_float4(0, 0, 0, 0);
                else          w[j] = idx < K4 ? wrow[idx] : make_float4(0, 0, 0, 0);
            }
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
            int idx = base + j * 32 + lane;
            if (idx < K4) {
#pragma unroll
                for (int b = 0; b < NB; ++b) {
                    float4 xv = reinterpret_cast<const float4*>(xs + b * K)[idx];
                    acc[b].x = fmaf(w[j].x, xv.x, acc[b].x); acc[b].y = fmaf(w[j].y, xv.y, acc[b].y);
                    acc[b].z = fmaf(w[j].z, xv.z, acc[b].z); acc[b].w = fmaf(w[j].w, xv.w, acc[b].w);
                }
            }
        }
    }
    if (dbg && lane == 0) dbg[0] = (unsigned long long)clock64();
    float mine = 0.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
        float s = warp_sum((acc[b].x + acc[b].y) + (acc[b].z + acc[b].w));
        if (lane == b) mine = s;
    }
    if (dbg && lane == 0) dbg[1] = (unsigned long long)clock64();
    return mine;
}
// weight row n of a [N, ldw] matrix of fp32 (WBF16 = false) or bf16 elements, as the pointer gemv_dot takes
template <bool WBF16>
__device__ __forceinline__ const float* gemv_wrow(const float* W, long long row_elems) {
    if (WBF16) return reinterpret_cast<const float*>(reinterpret_cast<const unsigned short*>(W) + row_elems);
    return W + row_elems;
}

// RAGGED (p.st heads a ragged state, `cur_pos` unused): a segment with pos_stride writes row b at the row's own cache position, and
// leaves the cache of a finished row alone.
template <int NB, bool W_GLOBAL, bool RAGGED = false, bool WBF16 = false>
__device__ __forceinline__ void gemv_row(const GemvParams& p, int n, const float* wrow_f, const float* xs, int b0, int lane, int cur_pos,
                                         bool have_operands = false, float bias_v = 0.f, float r_v = 0.f, unsigned long long* dbg = nullptr) {
    if (!have_operands) gemv_row_operands<NB>(p, n, b0, lane, bias_v, r_v);
    // Everything the epilogue needs besides the dot product is derived NOW, branch-free and for every lane (batch index clamped), so
    // its shared-memory lookups overlap the dot product instead of forming a ~0.25 us dependent chain behind the shuffle tree.
    const int bl = min(b0 + (lane < NB ? lane : 0), p.B - 1);
    const int si = (int)(p.nseg > 1 && n >= p.seg[1].n_begin) + (int)(p.nseg > 2 && n >= p.seg[2].n_begin);
    const GemvSeg& sg = p.seg[si];
    bool live = true;
    if (RAGGED) {
        const RowState* rs = ragged_rows(p.st) + bl % ld_state(&p.st->n_req);
        cur_pos = ld_state(&rs->cur_len) - 1;
        live = sg.pos_stride == 0 || ld_state(&rs->finished) == 0;
    }
    float* const outp = sg.out + ((long long)bl * sg.out_bs + (long long)cur_pos * sg.pos_stride + (n - sg.n_begin));
    const int act = sg.act;
    const float alpha = sg.alpha;
    const bool has_bias = p.bias != nullptr, has_res = p.R != nullptr;
    const float mine = gemv_dot<NB, W_GLOBAL, WBF16>(p.K, wrow_f, xs, lane, dbg);
    if (lane < NB && b0 + lane < p.B) {
        float v = mine;
        if (has_bias) v += bias_v;
        v = apply_act(v, act) * alpha;
        if (has_res) v += r_v;
        if (!RAGGED || live) *outp = v;
    }
}

// Merge of the split-KV partials, done ONCE per (row, head) by whichever split arrives last (threadfence-reduction pattern):
// out[r, h*64+d] = sum_s w_s o_s[d] / sum_s w_s l_s, w_s = exp(m_s - max m), splits visited in index order, so the result does not
// depend on which CTA happens to be last.  (It used to be a prologue of the following GEMV, i.e. every CTA re-did it, each
// pulling every partial out of L2: 2-6 us per layer on the token's critical path.)
__device__ __forceinline__ void decode_attention_merge(const DecAttnParams& p, int h, int r, float* stat, int tid) {
    // Arrival = ONE acq_rel atomic by thread 0 behind a CTA barrier (the same release/acquire shape as the grid barrier): the
    // barrier orders every thread's partial stores before the release, and the last arriver's loads after the acquire.  No
    // per-thread __threadfence (each one waits for the whole SM's outstanding stores).
    __syncthreads();
    int* ticket = p.ticket + r * p.H + h;
    if (tid == 0) {
        int t;
        asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;" : "=r"(t) : "l"(ticket) : "memory");
        stat[0] = (t == p.n_splits - 1) ? 1.f : 0.f;
    }
    __syncthreads();
    if (stat[0] == 0.f) return;                        // uniform across the CTA
    if (tid < 64) {
        const int S = p.n_splits;
        const long long base = ((long long)r * p.H + h) * S;
        const float* ml = p.part_ml + base * 2;
        const float* po = p.part_o + base * 64 + tid;
        float num = 0.f, den = 0.f;
        if (S <= 8) {                                  // every load in flight at once
            float2 mv[8]; float ov[8];
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                mv[s] = s < S ? ldcg2(ml + s * 2) : make_float2(-INFINITY, 0.f);
                ov[s] = s < S ? __ldcg(po + s * 64) : 0.f;
            }
            float mmax = -INFINITY;
#pragma unroll
            for (int s = 0; s < 8; ++s) if (s < S) mmax = fmaxf(mmax, mv[s].x);
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                if (s < S && mv[s].y > 0.f) {
                    const float w = expf(mv[s].x - mmax);
                    num = fmaf(w, ov[s], num);
                    den = fmaf(w, mv[s].y, den);
                }
            }
        } else {                                       // contexts beyond 512 tokens: two rolled passes
            float mmax = -INFINITY;
#pragma unroll 1
            for (int s = 0; s < S; ++s) mmax = fmaxf(mmax, __ldcg(ml + s * 2));
#pragma unroll 1
            for (int s = 0; s < S; ++s) {
                const float2 mv = ldcg2(ml + s * 2);
                const float ov = __ldcg(po + s * 64);
                if (mv.y > 0.f) {
                    const float w = expf(mv.x - mmax);
                    num = fmaf(w, ov, num);
                    den = fmaf(w, mv.y, den);
                }
            }
        }
        p.out[(long long)r * p.out_ld + h * 64 + tid] = den > 0.f ? num / den : 0.f;
    }
    if (tid == 0) *ticket = 0;                         // ready for the next phase that uses this (row, head)
}

// ---------------------------------------------------------------------------------------------------------------------
// split-KV decode attention for one (split s, head h, row r); NW warps cooperate; smem: sc[128], red[NW][64], stat[2]
// ---------------------------------------------------------------------------------------------------------------------
// cache address of key position t of decoder row r, head h, through the source-row table
__device__ __forceinline__ const float* table_row(const DecAttnParams& p, int r, int t, int h, const float* base) {
    return base + (long long)__ldcg(p.kv_src + (long long)r * p.kv_src_ld + t) * p.row_stride + h * 64 + (long long)t * p.tok_stride;
}

// K / validity / V operands of one (split, head, row) unit, held in registers between the load and the compute half so that the load
// can be issued EARLY: cross-attention K/V are constants of the call, the megakernel requests them before the preceding grid barrier.
// KMAX = keys a unit may hold: 128 (default), or 64 for launches whose chunks are 64 keys (the batched per-phase kernel: half the K
// registers -> 6 instead of 4 resident CTAs per SM, i.e. more K/V bytes in flight; the arithmetic of the keys that exist is unchanged).
template <int NW, int KMAX = 128>
struct AttnRegs {
    static constexpr int SC_ITERS = KMAX / (4 * NW), PV_PRE = 16;
    float4 ka[SC_ITERS], kb4[SC_ITERS];
    unsigned char kvalid[SC_ITERS];                      // prompt-padding validity, fetched in the same batch as K
    float2 vpre[PV_PRE];
};

// TABLE: self-attention keys are read through the per-position source-row table p.kv_src (beam search: key t of row r lives in
// cache row kv_src[r][t]); the arithmetic is unchanged.
template <int NW, int KMAX = 128, bool TABLE = false>
__device__ __forceinline__ void decode_attention_load(const DecAttnParams& p, int s, int h, int r, int slot, int L, int P, int tid, AttnRegs<NW, KMAX>& R) {
    constexpr int SC_ITERS = AttnRegs<NW, KMAX>::SC_ITERS, PV_PRE = AttnRegs<NW, KMAX>::PV_PRE;
    const int lane = tid & 31, warp = tid >> 5;
    const int k_begin = s * p.chunk, k_end = min(L, k_begin + p.chunk);
    // one 64-bit base per operand, 32-bit offsets from there (token strides and chunk offsets are small)
    const int tok = (int)p.tok_stride;
    const float* kb = p.kc + (long long)slot * p.row_stride + h * 64 + (long long)k_begin * tok;
    const float* vb = p.vc + (long long)slot * p.row_stride + h * 64 + (long long)k_begin * tok;
    const unsigned char* kv = p.key_valid ? p.key_valid + (long long)r * p.key_valid_ld + k_begin : nullptr;
    const int nk = k_end - k_begin, n_prompt = P - k_begin;      // keys [0, n_prompt) of this split are prompt positions (nk <= 0: empty split)
    const int sub = lane & 7, kq = lane >> 3;                   // scores: 8 lanes per key, each lane owns 8 of the 64 dims
    // fixed trip count (chunk <= 128) so every K load of the chunk is in flight before the first shuffle
#pragma unroll
    for (int it = 0; it < SC_ITERS; ++it) {
        const int kk = it * 4 * NW + warp * 4 + kq;
        R.kvalid[it] = 1;
        if (kk < nk) {
            const float* kr = (TABLE ? table_row(p, r, k_begin + kk, h, p.kc) : kb + kk * tok) + sub * 8;
            R.ka[it] = ldcg4(kr); R.kb4[it] = ldcg4(kr + 4);
            if (kv && kk < n_prompt) R.kvalid[it] = kv[kk];
        } else {
            R.ka[it] = make_float4(0, 0, 0, 0); R.kb4[it] = make_float4(0, 0, 0, 0);
        }
    }
    // V rows do not depend on the scores: fetched in the same batch (warps 0..3, 16 keys each cover a 64-key chunk) so the whole
    // phase costs one memory round trip instead of two
    if (warp < 4) {
#pragma unroll
        for (int i = 0; i < PV_PRE; ++i) {
            const int kk = warp + 4 * i;
            R.vpre[i] = kk < nk ? ldcg2((TABLE ? table_row(p, r, k_begin + kk, h, p.vc) : vb + kk * tok) + lane * 2) : make_float2(0.f, 0.f);
        }
    }
}

template <int NW, int KMAX = 128, bool TABLE = false>
__device__ __forceinline__ void decode_attention_body(const DecAttnParams& p, int s, int h, int r, int slot, int L, int P, float* sc,
                                                      float (*red)[64], float* stat, int tid, const AttnRegs<NW, KMAX>& R,
                                                      unsigned long long* dbg = nullptr) {
#define ATTN_STAMP(i) do { if (dbg && tid == 0) dbg[i] = (unsigned long long)clock64(); } while (0)
    constexpr int SC_ITERS = AttnRegs<NW, KMAX>::SC_ITERS, PV_PRE = AttnRegs<NW, KMAX>::PV_PRE;
    const int lane = tid & 31, warp = tid >> 5;
    const int k_begin = s * p.chunk, k_end = min(L, k_begin + p.chunk);
    const long long out_idx = ((long long)r * p.H + h) * p.n_splits + s;
    if (k_begin >= k_end) {                               // empty split (uniform across the CTA): it still takes its ticket below
        if (p.n_splits == 1) { if (tid < 64) p.out[(long long)r * p.out_ld + h * 64 + tid] = 0.f; return; }
        if (tid == 0) { p.part_ml[out_idx * 2] = -INFINITY; p.part_ml[out_idx * 2 + 1] = 0.f; }
    } else {
    const int tok = (int)p.tok_stride;
    const float* vb = p.vc + (long long)slot * p.row_stride + h * 64 + (long long)k_begin * tok;
    const int nk = k_end - k_begin;
    const int sub = lane & 7, kq = lane >> 3;
    const float* qp = p.q + (long long)r * p.q_ld + h * 64 + sub * 8;
    const float4 q0 = ldcg4(qp), q1 = ldcg4(qp + 4);      // the only operand another CTA produced in the previous phase
    const auto& ka = R.ka; const auto& kb4 = R.kb4; const auto& kvalid = R.kvalid; const auto& vpre = R.vpre;
#pragma unroll
    for (int it = 0; it < SC_ITERS; ++it) {
        const int kk = it * 4 * NW + warp * 4 + kq;
        const float4 a = ka[it], b = kb4[it];
        float d = q0.x * a.x;
        d = fmaf(q0.y, a.y, d); d = fmaf(q0.z, a.z, d); d = fmaf(q0.w, a.w, d);
        d = fmaf(q1.x, b.x, d); d = fmaf(q1.y, b.y, d); d = fmaf(q1.z, b.z, d); d = fmaf(q1.w, b.w, d);
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        d += __shfl_xor_sync(0xffffffffu, d, 4);
        if (kk < nk && sub == 0) sc[kk] = kvalid[it] ? d : -INFINITY;
    }
    ATTN_STAMP(0);
    __syncthreads();
    // Softmax statistics + o = sum_k p_k V_k in the four PV warps.  Every PV warp derives (m, l, p) itself — the same per-lane order
    // (keys lane, lane+32, ...) and the same shuffle tree a single warp would use, so the bits do not depend on who computes them —
    // instead of one warp computing them for everybody behind two CTA barriers.  Warp w owns keys w, w+4, ...; lane owns dims
    // 2*lane, 2*lane+1: always four accumulation chains, whatever NW is (per-kernel path and megakernel stay bit-identical).
    if (warp < 4) {
        float pv[4];                                     // p of keys lane, lane+32, lane+64, lane+96
        float m = -INFINITY;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = lane + 32 * t;
            pv[t] = i < nk ? sc[i] : -INFINITY;
            m = fmaxf(m, pv[t]);
        }
        m = warp_max(m);
        float l = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = lane + 32 * t;
            pv[t] = (i < nk && pv[t] != -INFINITY) ? expf(pv[t] - m) : 0.f;
            if (i < nk) l += pv[t];
        }
        l = warp_sum(l);
        if (tid == 0) { stat[0] = m; stat[1] = l; }
        ATTN_STAMP(1);
        float2 o = make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < PV_PRE; ++i) {
            const int kk = warp + 4 * i;                 // < 32 for i < 8, in [32, 64) otherwise (warp <= 3)
            const float pk = __shfl_sync(0xffffffffu, pv[i >> 3], kk & 31);
            if (kk < nk) {
                o.x = fmaf(pk, vpre[i].x, o.x);
                o.y = fmaf(pk, vpre[i].y, o.y);
            }
        }
        if (KMAX > 64 && nk > 64) {                      // chunks longer than 64 keys (uniform): loads issued first, then consumed
#pragma unroll
            for (int t = 2; t < 4; ++t) {
                float2 vv[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int kk = 32 * t + warp + 4 * i;
                    vv[i] = kk < nk ? ldcg2((TABLE ? table_row(p, r, k_begin + kk, h, p.vc) : vb + kk * tok) + lane * 2) : make_float2(0.f, 0.f);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int kk = 32 * t + warp + 4 * i;
                    const float pk = __shfl_sync(0xffffffffu, pv[t], kk & 31);
                    if (kk < nk) {
                        o.x = fmaf(pk, vv[i].x, o.x);
                        o.y = fmaf(pk, vv[i].y, o.y);
                    }
                }
            }
        }
        red[warp][lane * 2] = o.x;
        red[warp][lane * 2 + 1] = o.y;
    }
    __syncthreads();
    if (p.n_splits == 1) {
        // one split holds the whole context: the merge degenerates to o / l (w = exp(m - m) = 1: the same bits as the general path)
        if (tid < 64) {
            const float v = (red[0][tid] + red[1][tid]) + (red[2][tid] + red[3][tid]);
            const float num = fmaf(1.f, v, 0.f), den = fmaf(1.f, stat[1], 0.f);
            p.out[(long long)r * p.out_ld + h * 64 + tid] = (stat[1] > 0.f && den > 0.f) ? num / den : 0.f;
        }
        return;
    }
    if (tid < 64) {
        float v = (red[0][tid] + red[1][tid]) + (red[2][tid] + red[3][tid]);
        p.part_o[out_idx * 64 + tid] = v;
        if (tid == 0) { p.part_ml[out_idx * 2] = stat[0]; p.part_ml[out_idx * 2 + 1] = stat[1]; }
    }
    }
    ATTN_STAMP(2);
    decode_attention_merge(p, h, r, stat, tid);
    ATTN_STAMP(3);
#undef ATTN_STAMP
}

// ---------------------------------------------------------------------------------------------------------------------
// The same unit computed by ONE warp (batch throughput form: no CTA barriers, no shared-memory reductions; many independent warps
// per SM hide the memory latency instead of one CTA prefetching everything).  Arithmetic is the 4-warp body's, value for value:
// a score = 8-lane FMA chain + xor-shuffles 1, 2, 4; (m, l, p) with per-lane key order lane, lane+32, ... and the full shuffle tree;
// o = four accumulation chains over keys = c mod 4 in ascending order, merged as (c0 + c1) + (c2 + c3).  A row therefore decodes
// to the same bits whether it runs alone through the megakernel or inside a batch through this kernel.
// sc: 128 floats of shared memory private to the warp.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void decode_attention_warp_body(const DecAttnParams& p, int s, int h, int r, int slot, int L, int P, float* sc, int lane) {
    const int k_begin = s * p.chunk, k_end = min(L, k_begin + p.chunk), nk = k_end - k_begin;
    const long long out_idx = ((long long)r * p.H + h) * p.n_splits + s;
    float* outp = p.out + (long long)r * p.out_ld + h * 64 + 2 * lane;
    if (nk <= 0) {
        if (p.n_splits == 1) { outp[0] = 0.f; outp[1] = 0.f; return; }
        if (lane == 0) { p.part_ml[out_idx * 2] = -INFINITY; p.part_ml[out_idx * 2 + 1] = 0.f; }
    } else {
        const int tok = (int)p.tok_stride;
        const float* kb = p.kc + (long long)slot * p.row_stride + h * 64 + (long long)k_begin * tok;
        const float* vb = p.vc + (long long)slot * p.row_stride + h * 64 + (long long)k_begin * tok;
        const unsigned char* kv = p.key_valid ? p.key_valid + (long long)r * p.key_valid_ld + k_begin : nullptr;
        const int n_prompt = P - k_begin;
        const int sub = lane & 7, kq = lane >> 3;
        const float* qp = p.q + (long long)r * p.q_ld + h * 64 + sub * 8;
        const float4 q0 = ldcg4(qp), q1 = ldcg4(qp + 4);
        // scores, 16 keys per batch (4 instructions x 4 keys): loads of a batch are all in flight before its first use
        for (int k0 = 0; k0 < nk; k0 += 16) {
            float4 ka[4], kb4[4];
            unsigned char valid[4];
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const int kk = k0 + it * 4 + kq;
                valid[it] = 1;
                if (kk < nk) {
                    const float* kr = kb + kk * tok + sub * 8;
                    ka[it] = ldcg4(kr); kb4[it] = ldcg4(kr + 4);
                    if (kv && kk < n_prompt) valid[it] = kv[kk];
                } else {
                    ka[it] = make_float4(0, 0, 0, 0); kb4[it] = make_float4(0, 0, 0, 0);
                }
            }
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const int kk = k0 + it * 4 + kq;
                const float4 a = ka[it], b = kb4[it];
                float d = q0.x * a.x;
                d = fmaf(q0.y, a.y, d); d = fmaf(q0.z, a.z, d); d = fmaf(q0.w, a.w, d);
                d = fmaf(q1.x, b.x, d); d = fmaf(q1.y, b.y, d); d = fmaf(q1.z, b.z, d); d = fmaf(q1.w, b.w, d);
                d += __shfl_xor_sync(0xffffffffu, d, 1);
                d += __shfl_xor_sync(0xffffffffu, d, 2);
                d += __shfl_xor_sync(0xffffffffu, d, 4);
                if (kk < nk && sub == 0) sc[kk] = valid[it] ? d : -INFINITY;
            }
        }
        __syncwarp();
        float pv[4];                                     // p of keys lane, lane+32, lane+64, lane+96
        float m = -INFINITY;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = lane + 32 * t;
            pv[t] = i < nk ? sc[i] : -INFINITY;
            m = fmaxf(m, pv[t]);
        }
        m = warp_max(m);
        float l = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = lane + 32 * t;
            pv[t] = (i < nk && pv[t] != -INFINITY) ? expf(pv[t] - m) : 0.f;
            if (i < nk) l += pv[t];
        }
        l = warp_sum(l);
        float2 o[4] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
        for (int t = 0; t < 4; ++t) {                    // 32 keys per pass, 16 V rows in flight at a time
            if (32 * t < nk) {                           // uniform
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    float2 vv[16];
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int kk = 32 * t + 16 * half + i;
                        vv[i] = kk < nk ? ldcg2(vb + kk * tok + lane * 2) : make_float2(0.f, 0.f);
                    }
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int kk = 32 * t + 16 * half + i;
                        const float pk = __shfl_sync(0xffffffffu, pv[t], kk & 31);
                        if (kk < nk) {
                            o[i & 3].x = fmaf(pk, vv[i].x, o[i & 3].x);
                            o[i & 3].y = fmaf(pk, vv[i].y, o[i & 3].y);
                        }
                    }
                }
            }
        }
        const float vx = (o[0].x + o[1].x) + (o[2].x + o[3].x), vy = (o[0].y + o[1].y) + (o[2].y + o[3].y);
        if (p.n_splits == 1) {
            const float den = fmaf(1.f, l, 0.f);
            const bool okd = l > 0.f && den > 0.f;
            outp[0] = okd ? fmaf(1.f, vx, 0.f) / den : 0.f;
            outp[1] = okd ? fmaf(1.f, vy, 0.f) / den : 0.f;
            return;
        }
        p.part_o[out_idx * 64 + 2 * lane] = vx;
        p.part_o[out_idx * 64 + 2 * lane + 1] = vy;
        if (lane == 0) { p.part_ml[out_idx * 2] = m; p.part_ml[out_idx * 2 + 1] = l; }
    }
    // ticket + merge by the last split to arrive (warp-scope version of decode_attention_merge: bar.warp.sync orders the lanes'
    // partial stores before lane 0's release, and the others' loads after its acquire)
    __syncwarp();
    int* ticket = p.ticket + r * p.H + h;
    int t = 0;
    if (lane == 0) asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;" : "=r"(t) : "l"(ticket) : "memory");
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t != p.n_splits - 1) return;
    const int S = p.n_splits;
    const long long base = ((long long)r * p.H + h) * S;
    const float* ml = p.part_ml + base * 2;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const float* po = p.part_o + base * 64 + 2 * lane + e;
        float mmax = -INFINITY, num = 0.f, den = 0.f;
#pragma unroll 1
        for (int q = 0; q < S; ++q) mmax = fmaxf(mmax, __ldcg(ml + q * 2));
#pragma unroll 1
        for (int q = 0; q < S; ++q) {
            const float2 mv = ldcg2(ml + q * 2);
            const float ov = __ldcg(po + q * 64);
            if (mv.y > 0.f) {
                const float w = expf(mv.x - mmax);
                num = fmaf(w, ov, num);
                den = fmaf(w, mv.y, den);
            }
        }
        outp[e] = den > 0.f ? num / den : 0.f;
    }
    if (lane == 0) *ticket = 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// fused logits-processor chain + token selection
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SAMPLE_THREADS = 512;
constexpr int VMAX = 4096;

template <int NT>
static __device__ __forceinline__ float block_reduce(float v, bool is_max, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = lane < NT / 32 ? scratch[lane] : (is_max ? -INFINITY : 0.f);
        t = is_max ? warp_max(t) : warp_sum(t);
        if (lane == 0) scratch[32] = t;
    }
    __syncthreads();
    return scratch[32];
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

struct SampleSmem {
    float s[VMAX];
    int sidx[VMAX];
    float scratch[34];
    int chosen_sh;
    float wb[SAMPLE_THREADS / 32];
    int wi[SAMPLE_THREADS / 32];
};


// ---- register-resident greedy chain (dataflow megakernel) ------------------------------------------------------------------------------
// sample_body walks the vocabulary through shared memory once per processor (rolled loops, three CTA barriers per reduction): 15 us
// per token on ONE CTA while 147 wait for the next token's embedding.  For greedy selection every stage is elementwise or a reduction,
// so the thread's V / NT scores can stay in registers from the poll to the argmax: one pass, three fused reductions (two maxima; four
// sums; the argmax), each one warp shuffle tree + one barrier + one shuffle tree in EVERY warp (no broadcast barrier).  The per-thread
// visiting order (v = tid, tid + NT, ...) and the two-level shuffle trees are those of sample_body / block_reduce, so the scores carry
// the same bits as the shared-memory chain with the same NT.
template <int NT, int N>
static __device__ __forceinline__ void block_reduce_fused(float (&v)[N], bool is_max, float* region /* >= N * 32 floats, alternate between calls */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = is_max ? warp_max(v[k]) : warp_sum(v[k]);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) region[k * 32 + warp] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        float t = lane < NT / 32 ? region[k * 32 + lane] : (is_max ? -INFINITY : 0.f);
        v[k] = is_max ? warp_max(t) : warp_sum(t);
    }
}

// (0)+(1) of the chain for the dataflow megakernel: tagged logits -> CFG mix -> min_new_tokens EOS suppression -> s[v] (per-thread slots
// v = tid + j * NT).
template <int NT>
static __device__ __forceinline__ void sample_poll_ll(const SampleParams& p, int b, float* s, bool suppress_eos) {
    constexpr int PER = VMAX / NT;
    const int tid = threadIdx.x;
    const SampleConfig& c = *p.cfg;
    const int V = c.V, B = c.B;
    const unsigned in_tag = p.ll_in_tag;
    const unsigned char* __restrict__ vfl = p.vflags;
    const bool use_cfg = c.use_cfg != 0;
    const float cfg_scale = c.cfg_scale;
    // Polled in rounds of 8 pairs per thread (all 8 in flight before the first tag check); the conditional half of a CFG pair waits in
    // s[] itself for the unconditional one.
    {
        constexpr int CH = 8;
        for (int half = 0; half < (use_cfg ? 2 : 1); ++half) {
            const ll_t* src = p.ll_logits + (long long)(half * B + b) * V;
#pragma unroll 1
            for (int j0 = 0; j0 < PER; j0 += CH) {
                ll_t w[CH];
                long long spin = 0;
                while (true) {
                    bool ok = true;
#pragma unroll
                    for (int j = 0; j < CH; ++j) {
                        const int v = tid + (j0 + j) * NT;
                        if (v < V) asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w[j]) : "l"(src + v) : "memory");
                    }
#pragma unroll
                    for (int j = 0; j < CH; ++j) {
                        const int v = tid + (j0 + j) * NT;
                        if (v < V) ok = ok && (unsigned)(w[j] >> 32) == in_tag;
                    }
                    if (ok || !ll_spin_check(spin, p.ll_err, in_tag)) break;
                    __nanosleep(96);      // one CTA spinning on 29 KB of lines that 147 CTAs are storing into: back off so the stores get through
                }
                // (flags first, all at once: a load behind a conditional cannot be moved above the previous element's store by the compiler,
                //  and eight dependent L2 round trips cost 3 us here)
                unsigned char fl[CH];
#pragma unroll
                for (int j = 0; j < CH; ++j) {
                    const int v = tid + (j0 + j) * NT;
                    fl[j] = (suppress_eos && v < V) ? __ldg(vfl + v) : (unsigned char)0;
                }
#pragma unroll
                for (int j = 0; j < CH; ++j) {
                    const int v = tid + (j0 + j) * NT;
                    if (v < V) {
                        const float xv = __uint_as_float((unsigned)w[j]);
                        if (use_cfg && half == 0) s[v] = xv;                   // first half = "conditional" in HF's processor
                        else {
                            const float y = use_cfg ? xv + (s[v] - xv) * cfg_scale : xv;
                            s[v] = (fl[j] & VF_EOS) ? -INFINITY : y;
                        }
                    }
                }
                if (p.trace && tid == 0 && j0 == 0) { p.trace[7] = (unsigned long long)clock64(); p.trace[10] = (unsigned long long)spin; }
            }
        }
    }
}

template <int NT>
static __device__ __forceinline__ int sample_greedy_regs(const SampleParams& p, int b, SampleSmem& sm, int L, int st_step, int st_has_last, bool suppress_eos) {
    constexpr int PER = VMAX / NT;
    const int tid = threadIdx.x;
    const SampleConfig& c = *p.cfg;
    const int V = c.V, B = c.B;
    float* regions = reinterpret_cast<float*>(sm.sidx);            // the sort's index array is idle on the greedy path: 2 x 4 x 32 floats of scratch
    // Every thread only ever touches ITS OWN scores (v = tid + j * NT): s[] is per-thread scratch here, so no barrier is needed between
    // the passes — only inside the reductions.  (Registers instead of s[] made this function so register-hungry that the calling
    // megakernel spilled in its per-layer phases: +10 % per token.)
    float* s = sm.s;
    sample_poll_ll<NT>(p, b, s, suppress_eos);
    if (p.trace && tid == 0) p.trace[1] = (unsigned long long)clock64();
    // (2) MonotonicTimeShift, (3) TimeshiftBias, (4) temperature (decided on batch row 0)
    const int lts = p.last_ts[b];
    float temp = c.temperature;
    if (c.types_first) {
        for (int i = 0; i < c.n_cond; ++i) {
            const int off = c.cond_offset[i];
            if (L >= off) {
                long long t0 = __ldcg(p.ids + (L - off));   // row 0
                if (t0 >= 0 && (p.vflags[t0] & c.cond_flag[i])) { temp = c.cond_temp[i]; break; }
            }
        }
    }
    const bool lb_plain = c.lookback_on && !c.types_first;
    const bool lb_scores = c.lookback_on && c.types_first;
    float* ls_cur = p.last_scores + ((long long)(st_step & 1) * B + b) * V;
    const float* ls_prev = p.last_scores + ((long long)((st_step + 1) & 1) * B + b) * V;
    bool lb_apply = false;
    if (lb_scores) {
        const long long last_tok = L > 0 ? __ldcg(p.ids + (long long)b * c.ids_ld + (L - 1)) : -1;
        lb_apply = st_has_last && last_tok >= 0 && (p.vflags[last_tok] & VF_TIMED);
    }
    // The passes below run in batches of 4 elements with every load of a batch issued before its first store: the compiler must assume
    // that s[], the two score buffers and the flags alias, so a load written after a store stays behind it (one L2 round trip per element).
    constexpr int BT = 4;
    const int ts_start = c.ts_start, ts_end = c.ts_end, lb_start = c.lookback_start, lb_end = c.lookback_end;
    const float ts_bias = c.timeshift_bias;
    const unsigned char* __restrict__ vfl = p.vflags;
    float mm[2] = {-INFINITY, -INFINITY};                          // max of the previous step's scores, max of this step's
#pragma unroll 1
    for (int v0 = tid; v0 < V; v0 += BT * NT) {
        float xv[BT], lp[BT];
#pragma unroll
        for (int k = 0; k < BT; ++k) {
            const int v = v0 + k * NT;
            xv[k] = v < V ? s[v] : -INFINITY;
            lp[k] = (lb_apply && v < V) ? __ldcg(ls_prev + v) : -INFINITY;
        }
#pragma unroll
        for (int k = 0; k < BT; ++k) {
            const int v = v0 + k * NT;
            float x = xv[k];
            if (v >= ts_start && v < ts_end) {
                if (lts >= 0 && v < ts_start + lts) x = -INFINITY;
                if (ts_bias != 0.f) x += ts_bias;
            }
            x = x / temp;
            if (lb_plain && v >= lb_start && v < lb_end) x = -INFINITY;
            xv[k] = x;
            if (lb_apply && v < V) { mm[0] = fmaxf(mm[0], lp[k]); mm[1] = fmaxf(mm[1], x); }
        }
#pragma unroll
        for (int k = 0; k < BT; ++k) {
            const int v = v0 + k * NT;
            if (v < V) {
                s[v] = xv[k];
                if (lb_scores) ls_cur[v] = xv[k];
            }
        }
    }
    // (5) LookbackBias with the previous step's scores
    if (lb_apply) {
        block_reduce_fused<NT, 2>(mm, true, regions);
        const float m_last = mm[0], m_cur = mm[1];
        float zz[4] = {0.f, 0.f, 0.f, 0.f};                        // z_last, z_cur, e_last, o_cur
#pragma unroll 1
        for (int v0 = tid; v0 < V; v0 += BT * NT) {
            float xv[BT], lp[BT];
            unsigned char fl[BT];
#pragma unroll
            for (int k = 0; k < BT; ++k) {
                const int v = v0 + k * NT;
                xv[k] = v < V ? s[v] : -INFINITY;
                lp[k] = v < V ? __ldcg(ls_prev + v) : -INFINITY;
                fl[k] = v < V ? __ldg(vfl + v) : (unsigned char)0;
            }
#pragma unroll
            for (int k = 0; k < BT; ++k) {                         // (element order v0, v0 + NT, ... : the accumulation order of sample_body)
                const int v = v0 + k * NT;
                if (v < V) {
                    const float pl = expf(lp[k] - m_last);
                    const float pc = expf(xv[k] - m_cur);
                    zz[0] += pl; zz[1] += pc;
                    if (fl[k] & VF_LB_EOS) zz[2] += pl;
                    if (!(v >= lb_start && v < lb_end)) zz[3] += pc;
                }
            }
        }
        block_reduce_fused<NT, 4>(zz, false, regions + 4 * 32);
        const float prob_eos = zz[2] / zz[0];
        const float prob_event = 1.f - prob_eos;
        const float sc = 1.f / ((zz[3] / zz[1]) * prob_event + prob_eos);
        const float extra = fminf(fmaxf((sc - 1.f) * prob_eos / prob_event, 0.f), 1.f);
#pragma unroll 4
        for (int v = tid; v < V; v += NT) {
            float pr;
            if (v == lb_start) pr = extra;
            else if (v >= lb_start && v < lb_end) pr = 0.f;
            else pr = (expf(s[v] - m_cur) / zz[1]) * sc;
            s[v] = logf(pr);
        }
    }
    if (p.trace && tid == 0) p.trace[2] = (unsigned long long)clock64();
    // (6) argmax, first index on ties (torch.argmax)
    float best = -INFINITY; int bi = 0x7fffffff;
#pragma unroll 4
    for (int v = tid; v < V; v += NT) {
        const float xv = s[v];
        if (xv > best || (xv == best && v < bi)) { best = xv; bi = v; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if ((tid & 31) == 0) { sm.wb[tid >> 5] = best; sm.wi[tid >> 5] = bi; }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) {
        const float ob = sm.wb[w]; const int oi = sm.wi[w];
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    return bi == 0x7fffffff ? 0 : bi;
}

// vocabulary flags of batch row b: the call's one table, or the row's own in a ragged call (re-derived at every use: a pointer kept
// live across the chain costs the uniform instantiations a register)
template <bool RAGGED>
static __device__ __forceinline__ const unsigned char* row_vflags(const SampleParams& p, const SampleConfig& c, int b) {
    if (RAGGED) return p.vflags + (long long)b * c.vflags_ld;
    return p.vflags;
}

// The logits-processor chain of one batch row b (steps 0-5: min_new_tokens EOS mask, CFG, MonotonicTimeShift, TimeshiftBias,
// temperature decided on row 0, LookbackBias) from p.logits into sm.s.  Shared by the token selection below (on logits) and by the
// beam-search scores phase (beam.cu, on log-probs).
// RAGGED (mb200_model_generate_ragged): row b is its own batch-1 call — its own SampleConfig and vocabulary-flag row, and the
// conditional temperature decided on ITS last tokens (in a batch-1 call, "row 0" is the row itself).
template <int NT, bool RAGGED = false>
static __device__ __forceinline__ void logits_chain(const SampleParams& p, int b, SampleSmem& sm, int L, int st_step, int st_has_last,
                                                    bool suppress_eos) {
    float* s = sm.s;
    float* scratch = sm.scratch;
    const int tid = threadIdx.x;
    const SampleConfig& c = p.cfg[RAGGED ? b : 0];
    const int V = c.V, B = c.B;
    long long* ids_row = p.ids + (long long)b * c.ids_ld;
    // (0)+(1): min_new_tokens EOS suppression, then classifier-free guidance on raw logits
    if (p.ll_logits) {
        sample_poll_ll<NT>(p, b, s, suppress_eos);
    } else {
    _Pragma("unroll 1") for (int v = tid; v < V; v += NT) {
        float x;
        const bool eos = (row_vflags<RAGGED>(p, c, b)[v] & VF_EOS) != 0;
        if (c.use_cfg) {
            float cond = __ldcg(p.logits + (long long)b * p.logits_ld + v);          // first half = "conditional" in HF's processor
            float unc = __ldcg(p.logits + (long long)(B + b) * p.logits_ld + v);
            x = (suppress_eos && eos) ? -INFINITY : unc + (cond - unc) * c.cfg_scale;
        } else {
            x = __ldcg(p.logits + (long long)b * p.logits_ld + v);
            if (suppress_eos && eos) x = -INFINITY;
        }
        s[v] = x;
    }
    }
    // (2) MonotonicTimeShift, (3) TimeshiftBias, (4) temperature (decided on batch row 0)
    const int lts = p.last_ts[b];
    float temp = c.temperature;
    if (c.types_first) {
        for (int i = 0; i < c.n_cond; ++i) {
            const int off = c.cond_offset[i];
            if (L >= off) {
                long long t0 = __ldcg((RAGGED ? ids_row : p.ids) + (L - off));   // row 0 of the call
                if (t0 >= 0 && (row_vflags<RAGGED>(p, c, b)[t0] & c.cond_flag[i])) { temp = c.cond_temp[i]; break; }
            }
        }
    }
    __syncthreads();
    _Pragma("unroll 1") for (int v = tid; v < V; v += NT) {
        float x = s[v];
        if (v >= c.ts_start && v < c.ts_end) {
            if (lts >= 0 && v < c.ts_start + lts) x = -INFINITY;
            if (c.timeshift_bias != 0.f) x += c.timeshift_bias;
        }
        s[v] = x / temp;
    }
    __syncthreads();

    // (5) LookbackBias
    if (c.lookback_on) {
        if (!c.types_first) {
            _Pragma("unroll 1") for (int v = c.lookback_start + tid; v < c.lookback_end; v += NT) s[v] = -INFINITY;
            __syncthreads();
        } else {
            float* ls_cur = p.last_scores + ((long long)(st_step & 1) * B + b) * V;
            const float* ls_prev = p.last_scores + ((long long)((st_step + 1) & 1) * B + b) * V;
            _Pragma("unroll 1") for (int v = tid; v < V; v += NT) ls_cur[v] = s[v];
            const long long last_tok = L > 0 ? __ldcg(ids_row + (L - 1)) : -1;
            const bool timed = last_tok >= 0 && (row_vflags<RAGGED>(p, c, b)[last_tok] & VF_TIMED);
            if (st_has_last && timed) {
                float m_last = -INFINITY, m_cur = -INFINITY;
                _Pragma("unroll 1") for (int v = tid; v < V; v += NT) { m_last = fmaxf(m_last, __ldcg(ls_prev + v)); m_cur = fmaxf(m_cur, s[v]); }
                m_last = block_reduce<NT>(m_last, true, scratch);
                m_cur = block_reduce<NT>(m_cur, true, scratch);
                float z_last = 0.f, z_cur = 0.f, e_last = 0.f, o_cur = 0.f;
                _Pragma("unroll 1") for (int v = tid; v < V; v += NT) {
                    float pl = expf(__ldcg(ls_prev + v) - m_last);
                    float pc = expf(s[v] - m_cur);
                    z_last += pl; z_cur += pc;
                    if (row_vflags<RAGGED>(p, c, b)[v] & VF_LB_EOS) e_last += pl;
                    if (!(v >= c.lookback_start && v < c.lookback_end)) o_cur += pc;
                }
                z_last = block_reduce<NT>(z_last, false, scratch);
                z_cur = block_reduce<NT>(z_cur, false, scratch);
                e_last = block_reduce<NT>(e_last, false, scratch);
                o_cur = block_reduce<NT>(o_cur, false, scratch);
                const float prob_eos = e_last / z_last;
                const float prob_event = 1.f - prob_eos;
                const float sc = 1.f / ((o_cur / z_cur) * prob_event + prob_eos);
                const float extra = fminf(fmaxf((sc - 1.f) * prob_eos / prob_event, 0.f), 1.f);
                _Pragma("unroll 1") for (int v = tid; v < V; v += NT) {
                    float pr;
                    if (v == c.lookback_start) pr = extra;
                    else if (v >= c.lookback_start && v < c.lookback_end) pr = 0.f;
                    else pr = (expf(s[v] - m_cur) / z_cur) * sc;
                    s[v] = logf(pr);
                }
            }
            __syncthreads();
        }
    }
}

// The whole logits-processor chain + token selection + append for batch row b (one CTA of NT threads).
// Deliberately NOT inlined and with rolled vocabulary loops: it runs once per token on one CTA; inlined and unrolled it was 70 KB of
// the megakernel's 130 KB of code.  (A cold/warm re-run experiment later showed the per-layer phases are NOT instruction-fetch bound,
// so this is about code size and register pressure of the caller, not about the 32 KB L1.5 instruction cache.)
// Returns after the "last CTA" bookkeeping; the caller decides how the grid synchronises afterwards.
// NT = threads of the calling CTA (512 in the per-phase kernel and the barrier megakernel, 256 in the dataflow megakernel).
// RAGGED: lengths, limits, the finished flag, the step counter and the look-back flag are row b's own (ragged_rows(st)[b]); the draw
// uses the row's step and row index 0 in its counter, as the row's batch-1 call would; a finished row is frozen (nothing appended, its
// last embedding re-issued so the residual stream stays put).
template <int NT, bool RAGGED = false>
static __device__ __noinline__ void sample_body(const SampleParams& p, int b, SampleSmem& sm) {
    float* s = sm.s;
    int* sidx = sm.sidx;
    float* scratch = sm.scratch;
    const int tid = threadIdx.x;
    const SampleConfig& c = p.cfg[RAGGED ? b : 0];
    GenState* st = p.st;
    RowState* rs = ragged_rows(st) + b;                    // RAGGED only
    const int V = c.V, B = c.B;
    const int L = ld_state(RAGGED ? &rs->cur_len : &st->cur_len);
    const int st_prompt_len = ld_state(RAGGED ? &rs->prompt_len : &st->prompt_len);
    const int st_min_new = ld_state(RAGGED ? &rs->min_new_tokens : &st->min_new_tokens);
    const int st_step = ld_state(RAGGED ? &rs->step : &st->step), st_has_last = ld_state(RAGGED ? &rs->has_last_scores : &st->has_last_scores);
    const int st_max_length = ld_state(RAGGED ? &rs->max_length : &st->max_length);
    long long* ids_row = p.ids + (long long)b * c.ids_ld;
    const bool suppress_eos = st_min_new > 0 && (L - st_prompt_len) < st_min_new;

    if (p.trace && tid == 0) p.trace[6] = (unsigned long long)clock64();
    int chosen = 0;
    const bool frozen = RAGGED && ld_state(&rs->finished) != 0;      // uniform across the CTA
    const bool fast_greedy = !RAGGED && p.ll_logits != nullptr && !c.do_sample && p.dbg_scores == nullptr && V <= VMAX;
    if (frozen) {
        chosen = (int)__ldcg(ids_row + (L - 1));
    } else if (fast_greedy) {
        chosen = sample_greedy_regs<NT>(p, b, sm, L, st_step, st_has_last, suppress_eos);
    } else {
    logits_chain<NT, RAGGED>(p, b, sm, L, st_step, st_has_last, suppress_eos);

    // (6)-(7) selection
    if (!c.do_sample) {
        if (p.dbg_scores) { _Pragma("unroll 1") for (int v = tid; v < V; v += NT) p.dbg_scores[(long long)b * V + v] = s[v]; }
        // argmax, first index on ties (torch.argmax)
        float best = -INFINITY; int bi = 0x7fffffff;
        _Pragma("unroll 1") for (int v = tid; v < V; v += NT) {
            float x = s[v];
            if (x > best || (x == best && v < bi)) { best = x; bi = v; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best, o);
            int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        float* wb = sm.wb;
        int* wi = sm.wi;
        if ((tid & 31) == 0) { wb[tid >> 5] = best; wi[tid >> 5] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < NT / 32; ++w)
                if (wb[w] > best || (wb[w] == best && wi[w] < bi)) { best = wb[w]; bi = wi[w]; }
            sm.chosen_sh = (bi == 0x7fffffff) ? 0 : bi;
        }
        __syncthreads();
        chosen = sm.chosen_sh;
    } else {
        // sort ascending (bitonic over VMAX slots, padding = +inf at the top so real entries keep ascending order)
        _Pragma("unroll 1") for (int v = tid; v < VMAX; v += NT) { sidx[v] = v; if (v >= V) s[v] = INFINITY; }
        __syncthreads();
        const bool need_sort = c.top_k > 0 || c.top_p < 1.0f;
        if (need_sort) {
            for (int k = 2; k <= VMAX; k <<= 1) {
                for (int j = k >> 1; j > 0; j >>= 1) {
                    for (int i = tid; i < VMAX; i += NT) {
                        int ixj = i ^ j;
                        if (ixj > i) {
                            bool up = (i & k) == 0;
                            float a = s[i], bq = s[ixj];
                            int ia = sidx[i], ib = sidx[ixj];
                            bool gt = a > bq || (a == bq && ia > ib);
                            if (gt == up) { s[i] = bq; s[ixj] = a; sidx[i] = ib; sidx[ixj] = ia; }
                        }
                    }
                    __syncthreads();
                }
            }
            // real entries are now s[0..V-1] ascending
            if (c.top_k > 0) {
                int kk = min(c.top_k, V);
                float thr = s[V - kk];
                __syncthreads();
                _Pragma("unroll 1") for (int v = tid; v < V; v += NT) if (s[v] < thr) s[v] = -INFINITY;
                __syncthreads();
            }
        }
        // softmax statistics over the (possibly sorted) entries
        float m = -INFINITY;
        _Pragma("unroll 1") for (int v = tid; v < V; v += NT) m = fmaxf(m, s[v]);
        m = block_reduce<NT>(m, true, scratch);
        // Inclusive prefix sums of e[v] = exp(s[v] - m) in array order (ascending scores when sorted) by a block scan: thread t owns
        // the contiguous segment [t*SEG, (t+1)*SEG) (sequential inside, like the serial walk it replaces), warp shuffles scan the
        // segment totals, one warp scans the 16 warp totals.  The three serial thread-0 passes over V with expf (round 1) are gone.
        constexpr int SEG = VMAX / NT;
        const int lane = tid & 31, warp = tid >> 5;
        float loc[SEG];
        float run = 0.f;
#pragma unroll
        for (int j = 0; j < SEG; ++j) {
            const int v = tid * SEG + j;
            const float e = (v < V && s[v] != -INFINITY) ? expf(s[v] - m) : 0.f;
            run += e;
            loc[j] = run;
        }
        float incl = run;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        __syncthreads();
        if (lane == 31) scratch[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            float w = lane < NT / 32 ? scratch[lane] : 0.f;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            scratch[lane] = w;                               // inclusive scan of the warp totals; scratch[15] = z
        }
        __syncthreads();
        const float base = (incl - run) + (warp > 0 ? scratch[warp - 1] : 0.f);
        const float z = scratch[NT / 32 - 1];
        __syncthreads();
        // top-p (HF TopPLogitsWarper, min_tokens_to_keep = 1): in ascending order remove the longest prefix whose cumulative probability
        // is <= 1 - top_p; the last (largest) entry always stays.  The prefix sums are monotone, so its length is a count.
        int first_keep = 0;
        if (need_sort && c.top_p < 1.0f) {
            const float cut = c.top_p_cut;
            float cnt = 0.f;
#pragma unroll
            for (int j = 0; j < SEG; ++j) {
                const int v = tid * SEG + j;
                if (v < V - 1 && (base + loc[j]) / z <= cut) cnt += 1.f;
            }
            first_keep = (int)block_reduce<NT>(cnt, false, scratch);
        }
        if (p.dbg_scores) {       // parity hook (tests): the scores the selection sees, -inf = removed by top-k / top-p, original id order
            _Pragma("unroll 1") for (int v = tid; v < V; v += NT) p.dbg_scores[(long long)b * V + sidx[v]] = v < first_keep ? -INFINITY : s[v];
        }
        // mass below the kept set, then inverse-CDF draw over the kept entries
        if (tid == 0) scratch[33] = 0.f;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SEG; ++j)
            if (tid * SEG + j == first_keep - 1) scratch[33] = base + loc[j];
        __syncthreads();
        const float below = scratch[33];
        const unsigned long long r = splitmix64(c.seed ^ splitmix64(((unsigned long long)st_step << 20) ^ (unsigned long long)(RAGGED ? 0 : b)));
        const float u = below + (float)((r >> 40) + 0.5) * (1.0f / 16777216.0f) * (z - below);
        float cnt = 0.f;
#pragma unroll
        for (int j = 0; j < SEG; ++j) {
            const int v = tid * SEG + j;
            if (v >= first_keep && v < V && base + loc[j] < u) cnt += 1.f;
        }
        const int pick = min(V - 1, first_keep + (int)block_reduce<NT>(cnt, false, scratch));
        if (tid == 0) sm.chosen_sh = sidx[pick];
        __syncthreads();
        chosen = sm.chosen_sh;
    }

    }   // !fast_greedy

    if (p.trace && tid == 0) p.trace[3] = (unsigned long long)clock64();
    // (8) finished rows emit pad; append; EOS test; state updates; next-step embedding
    const bool was_finished = RAGGED ? false : p.finished[b] != 0;
    const long long tok = was_finished ? (long long)c.pad_id : (long long)chosen;
    __syncthreads();
    if (tid == 0 && !frozen) {
        ids_row[L] = tok;
        bool fin = was_finished || ((row_vflags<RAGGED>(p, c, b)[tok] & VF_EOS) != 0) || (L + 1 >= st_max_length);
        if (RAGGED) {
            rs->cur_len = L + 1;
            rs->step = st_step + 1;
            rs->has_last_scores = 1;
            if (fin) rs->finished = 1;
        } else if (fin && !was_finished) { p.finished[b] = 1; atomicAdd(&st->n_finished, 1); }
        // MonotonicTimeShift state (logit_processors.py:149-166): last time shift after the last SOS-type token
        const unsigned char fl = row_vflags<RAGGED>(p, c, b)[tok];
        if (fl & VF_SOS) p.last_ts[b] = -1;
        else if (tok >= c.ts_start && tok < c.ts_end) p.last_ts[b] = (int)(tok - c.ts_start);
    }
    // embedding of the token just appended, for every decoder row fed with it
    const int nrep = c.use_cfg ? 2 : 1;
    for (int rep = 0; rep < nrep; ++rep) {
        const int row = rep * B + b;
        int pos = frozen ? L - 1 : L;
        if (!RAGGED && c.pos_rule_cumsum && p.n_left_pad) pos = L - p.n_left_pad[row];
        const float4* te = reinterpret_cast<const float4*>(p.tok_emb + tok * p.d_model);
        const float4* pe = reinterpret_cast<const float4*>(p.pos_emb + (long long)pos * p.d_model);
        float4* xo = reinterpret_cast<float4*>(p.x_out + (long long)row * p.x_ld);
        for (int i = tid; i < p.d_model / 4; i += NT) {
            float4 a = te[i], q = pe[i];
            const float4 o = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
            xo[i] = o;
            if (p.ll_x_out) {
                for (int rep = 0; rep < p.ll_reps; ++rep) {
                    ll_t* lo = p.ll_x_out + rep * p.ll_x_rep + (long long)row * p.d_model + i * 4;
                    ll_store2(lo, o.x, o.y, p.ll_out_tag);
                    ll_store2(lo + 2, o.z, o.w, p.ll_out_tag);
                }
            }
        }
    }
    __syncthreads();
    if (p.trace && tid == 0) p.trace[4] = (unsigned long long)clock64();
    if (tid == 0) {
        // Last row to arrive publishes the next token's header.  Dataflow megakernel: the tagged header goes out FIRST (its consumers
        // synchronise on the tag, not on the fences); the plain state for the host / the per-phase kernels follows.
        // RAGGED: one CTA per row of the launch — every row of the state, or the rows of an admission's list
        const int n_cta = RAGGED ? (int)gridDim.x : B;
        if (n_cta > 1) __threadfence();                // this row's finished update before its ticket
        if (atomicAdd(&st->ticket, 1) == n_cta - 1) {
            int fin_all;
            if (RAGGED) {      // all rows of the state, launched or not; a vacant stream row is a finished row
                fin_all = 1;
                const int n = ld_state(&st->n_req);
                for (int r = 0; r < n; ++r)
                    if (!ld_state(&ragged_rows(st)[r].finished)) fin_all = 0;
            } else {
                fin_all = (ld_state(&st->n_finished) >= B || L + 1 >= st_max_length) ? 1 : 0;
            }
            if (p.ll_hdr) {        // token header of the dataflow megakernel: next cur_len, all-finished flag
                ll_store(p.ll_hdr + 0, __int_as_float(L + 1), p.ll_out_tag);
                ll_store(p.ll_hdr + 1, __int_as_float(fin_all), p.ll_out_tag);
            }
            st->ticket = 0;
            if (!RAGGED) st->cur_len = L + 1;
            if (!RAGGED) {     // a ragged row advanced its own step above
                st->step = st_step + 1;
                st->has_last_scores = 1;
            }
            if (fin_all) st->all_finished = 1;
            __threadfence();
        }
        if (p.trace) p.trace[5] = (unsigned long long)clock64();
    }
}


}  // namespace mb200
