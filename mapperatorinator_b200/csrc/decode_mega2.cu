// Dataflow token-loop megakernel: the same 98 dependent micro-phases per token as decode_mega.cu, the same device arithmetic
// (gemv_dot, the attention unit's score / softmax / PV order, the fused logits chain), but NO grid barrier between them.
//
// Why: ncu + the clock64 timeline of round 1 showed the barrier kernel at 348 us / token is latency-bound, and 27 % of a token is the
// barrier itself (98 x ~0.95 us = store drain + release atomic + acquire poll) with another ~0.3 us per phase for the activation load
// that can only start after it.  Here every value that crosses CTAs is an 8-byte pair {fp32 bits | tag << 32} written by ONE 64-bit
// store and polled by whoever needs it (NCCL's "LL" protocol): the consumer's load IS the wait, the producer never drains or
// releases, and a CTA that has nothing to consume in a phase simply runs ahead.  tag = (step + 1) * 128 + phase + 1 is unique per
// (token, phase), buffers are zeroed before every launch.
//
// Which CTA reads what, and why a buffer can be overwritten without a second copy: a version of a buffer is only overwritten by a
// phase whose inputs transitively require EVERY reader of that version to have produced its own output first (e.g. x after out_proj
// is read by the 128 CTAs that own rows of the cross-q projection; the next writer of x, the cross out_proj, needs the merged cross
// attention, which needs every row of cross-q).
//
// Structure of a CTA (one CTA per SM x 256 threads x 255 registers; DESIGN.md §4.1 has the measurements behind each choice):
//   * GEMV phases with a d_model-wide input (qkv, out, q_c, out_c, fc1, proj_out): threads 0..K/4-1 poll one float4 column each (pointers
//     precomputed per thread), LayerNorm statistics over a named barrier of the polling warps, the activation is published in shared
//     memory (the phase's one CTA barrier), then every warp takes whole weight rows with the activation in registers (gemv_dot's order)
//     and finishes its own rows: lane = row slot x replica, one store instruction writes all replicas  (m3_rw_tail);
//   * fc2 (ffn-wide input): K-split — a thread polls exactly the columns it multiplies with every row of the CTA's slab; a transposing
//     warp butterfly and 8 warp partials reduce them; warps 6 / 7 finish the rows  (m3_gemv_phase / m3_rows);
//   * weight slices: cp.async.bulk into two shared-memory buffers a phase ahead, handed over by an mbarrier every warp arrives on;
//   * attention units and the selection phase: m2_attention_unit / m2_attention_merge, sample_body<256> (decode_device.cuh).
//
// The K/V rows appended to the cache are the one thing readers pick up long after the fact (next token onwards) through plain
// ld.cg: their writer fences right after the plain stores (hidden: that warp then waits for the attention phase anyway) and the
// NEWEST row travels as tagged pairs (`kvnew`) like every other same-token value.
//
// Every wait is bounded; on a timeout the error flag is raised, every other wait sees it and the launch drains.
#include "common.cuh"
#include "kernels.h"
#include "decode_device.cuh"

namespace mb200 {

namespace {

constexpr int M2_THREADS = 256;                         // 8 warps, 255 registers per thread: the phases are chains of dependent latencies, not throughput
constexpr int M2_WARPS = M2_THREADS / 32;
constexpr int M2_NB_MAX = 2;
constexpr int M2_XS_FLOATS = M2_NB_MAX * 1024;
constexpr int M2_XRAW_FLOATS = M2_NB_MAX * 1024;
constexpr int M2_PART = 66;                             // pairs per split partial: o[64], m, l
constexpr int M3_SLOTS = 32;                            // K-split GEMV: output rows per thread (row slots), passes of 8
constexpr int M3_NS = 4;                                // K-split GEMV: float4 columns per thread (K <= 4 * 4 * 256)
constexpr int M3_ROWS = 32;                             // K-split GEMV: output rows per CTA and phase

struct __align__(16) M2Smem {
    float wbuf[2][MEGA_WBUF_FLOATS];
    union __align__(16) {
        float xs[M2_XS_FLOATS];
        SampleSmem sample;
        struct { __align__(16) float sc[128]; float red[4][64]; __align__(16) float qs[64]; float kns[64]; float vns[64]; float stat[2]; } attn;
    } u;
    __align__(16) float xraw[M2_XRAW_FLOATS];   // raw residual stream as of this CTA's last LayerNorm staging (residual source of its rows)
    Mega2Phase phase[3];                        // descriptor of phase i lives in slot i % 3 (the K-split mode has no end-of-phase barrier)
    SampleParams sample_params;
    int ctrl[8];                                // cur_len, all_finished, error, prompt_len, encoder slots
    float ln_red[32];
    // K-split GEMV mode (MODE 1): warp partial sums [parity][decoder row][row slot][warp] and the second LayerNorm statistic
    __align__(16) float red[2][M2_NB_MAX][M3_ROWS][M2_WARPS];     // [phase parity][decoder row][output row of this CTA][warp of the row's group]
    float ln_red2[32];
    unsigned long long mbar[2];
    unsigned long long wfree[2];                // weight buffer b has been read by every warp (arrive count = warps): the next bulk copy may overwrite it
    __align__(16) float xrw[2][M2_NB_MAX * 1024]; // row-per-warp GEMV phases: the (normalised) activation, double-buffered by phase parity
};

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("{ .reg .b64 t; mbarrier.arrive.shared::cta.b64 t, [%0]; }" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("{ .reg .b64 t; mbarrier.arrive.expect_tx.shared::cta.b64 t, [%0], %1; }" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
    unsigned ok;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    unsigned long long pol;      // weights stream through L2 once per token: evict-first keeps the small hot set (exchange buffers, K/V) resident
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void cta_rows(int N, int cta, int rpc, int& r0, int& r1) {
    r0 = min(N, cta * rpc);
    r1 = min(N, r0 + rpc);
}
// Weight slice of a GEMV phase inside the two-buffer arena: buffer 0 starts at the front, buffer 1 ends at the back.  Consecutive GEMV
// phases (always of opposite parity) therefore only need their two slices TOGETHER to fit the arena, which lets the vocabulary
// projection's larger slice share it with its neighbours (mega_eligible in engine_model.cu checks every consecutive pair).
// floats = rows per CTA x K of that phase.
__device__ __forceinline__ float* wslice(float (&wbuf)[2][MEGA_WBUF_FLOATS], int buf, int floats) {
    return buf ? &wbuf[0][0] + 2 * MEGA_WBUF_FLOATS - floats : &wbuf[0][0];
}
// floats of the arena a slice of `elems` weight elements takes (WBF16: two bf16 per float; K is a multiple of 8 there)
template <bool WBF16>
__device__ __forceinline__ int slice_floats(int elems) { return WBF16 ? elems >> 1 : elems; }
// WBF16: W holds bf16 bits; the slice is the same rows at half the bytes
template <bool WBF16>
__device__ __forceinline__ void prefetch_weights(const float* W, long long ldw, int N, int K, float* dst, unsigned long long* bar, int cta, int rpc) {
    int r0, r1;
    cta_rows(N, cta, rpc, r0, r1);
    const unsigned bytes = (unsigned)(r1 - r0) * (unsigned)K * (WBF16 ? 2u : 4u);
    if (bytes == 0 || (c_ll_debug & 1)) { mbar_arrive(bar); return; }
    mbar_arrive_expect_tx(bar, bytes);
    bulk_g2s(dst, gemv_wrow<WBF16>(W, (long long)r0 * ldw), bytes, bar);
}
__device__ __forceinline__ bool wait_weights(unsigned long long* bar, unsigned parity, int* error_flag) {
    for (long long spin = 0; spin < (1ll << 24); ++spin)
        if (mbar_try_wait(bar, parity)) return true;
    atomicCAS(error_flag, 0, 2);
    return false;
}

__device__ __forceinline__ unsigned ll_tag(int step, int pi) { return (unsigned)((step + 1) * 128 + pi + 1); }

__device__ __forceinline__ ll_t* ll_buf(const MegaLL& ll, int sel) {
    switch (sel) {
        case LL_X: return ll.x;
        case LL_Q: return ll.q;
        case LL_K: return ll.kvnew;
        case LL_V: return ll.kvnew;
        case LL_ATT: return ll.att;
        case LL_H: return ll.h;
        case LL_LOGITS: return ll.logits;
        default: return nullptr;
    }
}

// chunk partials of warps that hold no chunk (c0 >= K4 / 32) must read as zero: the fixed tree always adds eight of them
__device__ __forceinline__ void m2_clear_ln_red(float* red, int tid) {
    if (tid < 32) red[tid] = 0.f;
}

// Every poll below puts ALL of a thread's loads in flight before it looks at the first tag (a wait per value would serialise one L2
// round trip per value: measured +60 us / token).
__device__ __forceinline__ bool ll_tag_ok4(ll_t a, ll_t b, ll_t c, ll_t d, unsigned tag) {
    return (unsigned)(a >> 32) == tag && (unsigned)(b >> 32) == tag && (unsigned)(c >> 32) == tag && (unsigned)(d >> 32) == tag;
}
__device__ __forceinline__ float ll_val(ll_t a) { return __uint_as_float((unsigned)a); }

// ---- attention unit -------------------------------------------------------------------------------------------------------------
// (split s, head h, row r) exactly like decode_attention_body<16>: the same score chains, the same per-warp softmax statistics, the same
// four PV accumulation chains — only the operand sources differ: q and the newest K/V row are polled from the exchange buffers, the
// result leaves as tagged pairs (merged heads when one split covers the context, else a split partial that the split-0 CTA merges).
__device__ __forceinline__ void m2_attention_unit(const DecAttnParams& p, const MegaLL& ll, bool is_self, int s, int h, int r, int slot, int L, int P,
                                                  unsigned in_tag, unsigned out_tag, float* sc, float (*red)[64], float* stat, float* qs, float* kns,
                                                  float* vns, int tid, AttnRegs<M2_WARPS>& R, int* err, unsigned long long* trace = nullptr) {
    constexpr int NW = M2_WARPS;
    constexpr int SC_ITERS = AttnRegs<NW>::SC_ITERS, PV_PRE = AttnRegs<NW>::PV_PRE;
    const int lane = tid & 31, warp = tid >> 5;
    const int d = p.H * 64;
    const int k_begin = s * p.chunk, k_end = min(L, k_begin + p.chunk);
    const int nk = k_end - k_begin;
    const int newest = is_self ? (L - 1 - k_begin) : -1;           // index inside this split of the key appended by THIS token (self only)
    ll_t* part = ll.part + (((long long)r * p.H + h) * ll.max_splits + s) * M2_PART;
    ll_t* att = ll.att + (long long)r * d + h * 64;
    if (nk <= 0) {                                                 // empty split (uniform across the CTA)
        if (p.n_splits == 1) { if (tid < 64) for (int rep = 0; rep < ll.reps; ++rep) ll_store(att + rep * ll.x_rep + tid, 0.f, out_tag); return; }
        // No partial: the merge knows the split is empty (m_s = -inf, l_s = 0 contributes nothing) and does not poll it.  A store here
        // would depend on no input of this token, so a CTA with nothing else to wait for (no GEMV rows, no other unit) could run ahead
        // into the next layer's self attention and overwrite this slot before this phase's merge had read it.
        return;
    }
    const int tok = (int)p.tok_stride;
    const float* vb = p.vc + (long long)slot * p.row_stride + h * 64 + (long long)k_begin * tok;
    const int sub = lane & 7, kq = lane >> 3;
    // q and (self-attention) the key / value row this token appended are polled ONCE per CTA — warp 14 takes q, warp 15 the new K | V
    // row — into shared memory; everybody reads them from there after one CTA barrier.  (All 512 threads polling their own copy cost
    // 16x the L2 polling traffic and, with the prefetched cache rows live in registers, pushed the kernel into spills.)
    const bool has_new = newest >= 0 && newest < nk;
    if (warp == NW - 2) {
        const float2 v = ll_wait2(ll.q + (long long)r * d + h * 64 + lane * 2, in_tag, err);
        qs[lane * 2] = v.x; qs[lane * 2 + 1] = v.y;
    } else if (warp == NW - 1 && has_new) {
        const ll_t* kn = ll.kvnew + (long long)r * 2 * d + h * 64;
        ll_t w[4];
        long long spin = 0;
        while (true) {
            ll_load2(kn + lane * 2, w[0], w[1]);
            ll_load2(kn + d + lane * 2, w[2], w[3]);
            if (ll_tag_ok4(w[0], w[1], w[2], w[3], in_tag) || !ll_spin_check(spin, err, in_tag)) break;
        }
        kns[lane * 2] = ll_val(w[0]); kns[lane * 2 + 1] = ll_val(w[1]);
        vns[lane * 2] = ll_val(w[2]); vns[lane * 2 + 1] = ll_val(w[3]);
    }
    __syncthreads();
    if (trace && tid == 0) trace[2] = (unsigned long long)clock64();
    const float4 q0 = *reinterpret_cast<const float4*>(qs + sub * 8), q1 = *reinterpret_cast<const float4*>(qs + sub * 8 + 4);
#pragma unroll
    for (int it = 0; it < SC_ITERS; ++it) {
        const int kk = it * 4 * NW + warp * 4 + kq;
        const bool is_new = kk == newest;
        const float4 a = is_new ? *reinterpret_cast<const float4*>(kns + sub * 8) : R.ka[it];
        const float4 b = is_new ? *reinterpret_cast<const float4*>(kns + sub * 8 + 4) : R.kb4[it];
        float dd = q0.x * a.x;
        dd = fmaf(q0.y, a.y, dd); dd = fmaf(q0.z, a.z, dd); dd = fmaf(q0.w, a.w, dd);
        dd = fmaf(q1.x, b.x, dd); dd = fmaf(q1.y, b.y, dd); dd = fmaf(q1.z, b.z, dd); dd = fmaf(q1.w, b.w, dd);
        dd += __shfl_xor_sync(0xffffffffu, dd, 1);
        dd += __shfl_xor_sync(0xffffffffu, dd, 2);
        dd += __shfl_xor_sync(0xffffffffu, dd, 4);
        if (kk < nk && sub == 0) sc[kk] = (R.kvalid[it] || is_new) ? dd : -INFINITY;
    }
    __syncthreads();
    if (trace && tid == 0) trace[3] = (unsigned long long)clock64();
    if (warp < 4) {
        float pv[4];
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
        float2 o = make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < PV_PRE; ++i) {
            const int kk = warp + 4 * i;
            const float pk = __shfl_sync(0xffffffffu, pv[i >> 3], kk & 31);
            const float2 vv = kk == newest ? *reinterpret_cast<const float2*>(vns + lane * 2) : R.vpre[i];
            if (kk < nk) {
                o.x = fmaf(pk, vv.x, o.x);
                o.y = fmaf(pk, vv.y, o.y);
            }
        }
        if (nk > 64) {
#pragma unroll
            for (int t = 2; t < 4; ++t) {
                float2 vv[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int kk = 32 * t + warp + 4 * i;
                    vv[i] = make_float2(0.f, 0.f);
                    if (kk < nk) vv[i] = kk == newest ? *reinterpret_cast<const float2*>(vns + lane * 2) : ldcg2(vb + kk * tok + lane * 2);
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
    if (trace && tid == 0) trace[4] = (unsigned long long)clock64();
    if (tid < 64) {
        const float v = (red[0][tid] + red[1][tid]) + (red[2][tid] + red[3][tid]);
        if (p.n_splits == 1) {
            // one split holds the whole context: the merge degenerates to o / l (w = exp(m - m) = 1: the same bits as the general path)
            const float num = fmaf(1.f, v, 0.f), den = fmaf(1.f, stat[1], 0.f);
            const float o = (stat[1] > 0.f && den > 0.f) ? num / den : 0.f;
            for (int rep = 0; rep < ll.reps; ++rep) ll_store(att + rep * ll.x_rep + tid, o, out_tag);
        } else {
            ll_store(part + tid, v, out_tag);
            if (tid == 0) { ll_store(part + 64, stat[0], out_tag); ll_store(part + 65, stat[1], out_tag); }
        }
    }
}

// merge of the S split partials of (row r, head h) by the CTA that computed split 0: splits visited in index order,
// out = sum_s w_s o_s / sum_s w_s l_s with w_s = exp(m_s - max m) — decode_attention_merge's arithmetic, operands polled.
// Splits at or beyond key L are empty: they publish no partial and enter the sums as (m, l) = (-inf, 0), which is what the per-phase
// merge reads for them (same bits).
__device__ __forceinline__ void m2_attention_merge(const DecAttnParams& p, const MegaLL& ll, int h, int r, int L, unsigned tag,
                                                   float* msh /* >= 2 * 32 floats of shared memory */, int tid, int* err) {
    // called by the WHOLE CTA (uniform).  Threads 64 .. 64+S-1 poll the (m, l) pair of one split each into shared memory, threads 0..63
    // poll their output dim of every split (S <= 16: one batch; beyond that: rolled), then 64 threads combine.
    const int S = p.n_splits, d = p.H * 64;
    const int S_live = min(S, (L + p.chunk - 1) / p.chunk);        // splits that hold keys
    const ll_t* base = ll.part + ((long long)r * p.H + h) * ll.max_splits * M2_PART;
    for (int s0 = 0; s0 < S; s0 += 32) {
        const int s = s0 + (tid - 64);
        if (tid >= 64 && tid < 96 && s < S) {
            const float2 mv = s < S_live ? ll_wait2(base + (long long)s * M2_PART + 64, tag, err) : make_float2(-INFINITY, 0.f);
            if (s < 32) { msh[s] = mv.x; msh[32 + s] = mv.y; }
        }
    }
    constexpr int SB = 16;                             // splits merged with every load in flight at once (cross attention: 12 of them)
    float ov[SB];
    if (tid < 64 && S <= SB) {
        ll_t oo[SB];
        long long spin = 0;
        while (true) {
            bool ok = true;
#pragma unroll
            for (int s = 0; s < SB; ++s)
                if (s < S_live) asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(oo[s]) : "l"(base + (long long)s * M2_PART + tid) : "memory");
#pragma unroll
            for (int s = 0; s < SB; ++s)
                if (s < S_live) ok = ok && (unsigned)(oo[s] >> 32) == tag;
            if (ok || !ll_spin_check(spin, err, tag)) break;
        }
#pragma unroll
        for (int s = 0; s < SB; ++s) ov[s] = s < S_live ? ll_val(oo[s]) : 0.f;
    }
    __syncthreads();
    if (tid >= 64) return;
    float num = 0.f, den = 0.f;
    float mmax = -INFINITY;
    if (S <= SB) {
#pragma unroll
        for (int s = 0; s < SB; ++s) if (s < S) mmax = fmaxf(mmax, msh[s]);
#pragma unroll
        for (int s = 0; s < SB; ++s) {
            if (s < S && msh[32 + s] > 0.f) {
                const float w = expf(msh[s] - mmax);
                num = fmaf(w, ov[s], num);
                den = fmaf(w, msh[32 + s], den);
            }
        }
    } else {
#pragma unroll 1
        for (int s = 0; s < S; ++s) mmax = fmaxf(mmax, msh[s]);
#pragma unroll 1
        for (int s = 0; s < S_live; ++s) {                   // (empty splits: l = 0, nothing to add)
            const float o1 = ll_wait1(base + (long long)s * M2_PART + tid, tag, err);
            if (msh[32 + s] > 0.f) {
                const float w = expf(msh[s] - mmax);
                num = fmaf(w, o1, num);
                den = fmaf(w, msh[32 + s], den);
            }
        }
    }
    const float o = den > 0.f ? num / den : 0.f;
    for (int rep = 0; rep < ll.reps; ++rep) ll_store(ll.att + rep * ll.x_rep + (long long)r * d + h * 64 + tid, o, tag);
}


// ---- K-split GEMV phase (MODE 1) ---------------------------------------------------------------------------------------------------
// The row-per-warp form spends its time in shared memory: every output row re-reads the whole activation vector next to its weight
// row (2 x K x 4 bytes per row through a 128 B / clk port), only rows-per-CTA of the 16 warps have work (6 of 16 for the d x d
// projections), and the activation takes a detour through shared memory behind two or three CTA barriers.  Here the CTA's weight slab
// [R rows x K] is split along K instead: thread t owns float4 column(s) kq of EVERY row, keeps its 4 activation values in registers
// (polled straight from the exchange buffer: no staging pass), and the R partial sums per thread are reduced by a transposing warp
// butterfly (9 shuffles per 8 rows) plus one pass over <= 16 warp partials.  Summation order is fixed by the thread mapping.
//   K4 = K / 4 float4 columns.  "grouped" (K4 a multiple of 32, <= 256: the d_model-wide inputs): G = 512 / K4 row groups, group rg
//   takes rows rg, rg + G, ... and group 0 polls the activation for everybody (one CTA barrier).  Otherwise one group, thread t owns
//   columns t and t + 512 (K4 <= 1024) and polls exactly what it multiplies.
// CTA barrier over the first `count` threads only (named barrier 1): the LayerNorm statistics involve the warps that hold columns, not the
// epilogue warps, which may still be storing the previous phase's rows
__device__ __forceinline__ void m3_bar_cols(int count) { asm volatile("bar.sync 1, %0;" ::"r"(count) : "memory"); }
__device__ __forceinline__ float m3_dot4(const float4 w, const float4 x) {
    float t0 = w.x * x.x; t0 = fmaf(w.y, x.y, t0);
    float t1 = w.z * x.z; t1 = fmaf(w.w, x.w, t1);
    return t0 + t1;
}
__device__ __forceinline__ float m3_tree8(const float* r) { return ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7])); }

// P values per lane (P = 8, 16 or 32) -> one warp-wide sum per lane: the transposing butterfly halves the number of live values at every
// level (lanes with the mask bit set keep the upper half and send the lower half), then plain xor-adds once a single value is left.
// Every row is combined in the same order (xor 16, 8, 4, 2, 1) whatever P is, so a row's bits do not depend on how many rows ride along.
// The lane's row index is m3_ridx<P>(lane); 32 / P lanes hold each row redundantly.
template <int P>
__device__ __forceinline__ float m3_reduce(float (&a)[P], int lane) {
    int n = P;
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
        if (n > 1) {
            const bool hi = (lane & m) != 0;
            const int h = n / 2;
#pragma unroll
            for (int i = 0; i < P / 2; ++i) {
                if (i < h) {
                    const float send = hi ? a[i] : a[i + h], keep = hi ? a[i + h] : a[i];
                    a[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
                }
            }
            n = h;
        } else {
            a[0] += __shfl_xor_sync(0xffffffffu, a[0], m);
        }
    }
    return a[0];
}
template <int P>
__device__ __forceinline__ int m3_ridx(int lane) {
    int r = 0, n = P;
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1)
        if (n > 1) { n /= 2; r += (lane & m) ? n : 0; }
    return r;
}
template <int P>
__device__ __forceinline__ bool m3_rowner(int lane) { return (lane & (32 / P - 1)) == 0; }      // one writer per row

// Thread -> weight-column mapping of a K-wide input; K takes two values per model (d_model, ffn_dim): computed once per kernel.
struct M3Map { int K4, G, rg, kq0, NS, npw, wi; bool grouped, in_group, active_warp; };
__device__ __forceinline__ M3Map m3_make_map(int K, int tid) {
    M3Map m;
    m.K4 = K >> 2;
    m.grouped = (m.K4 & 31) == 0 && m.K4 <= 256;
    m.G = m.grouped ? M2_THREADS / m.K4 : 1;
    m.rg = m.grouped ? tid / m.K4 : 0;
    m.kq0 = tid - m.rg * m.K4;
    m.in_group = m.rg < m.G;
    m.NS = m.grouped ? 1 : (m.K4 + M2_THREADS - 1) / M2_THREADS;
    m.npw = m.grouped ? m.K4 >> 5 : min(M2_WARPS, (m.K4 + 31) >> 5);
    m.wi = m.grouped ? (tid >> 5) - m.rg * m.npw : (tid >> 5);
    m.active_warp = m.grouped ? m.in_group : (tid >> 5) < m.npw;
    return m;
}

// All row slots of the phase in one go (P = 8, 16 or 32 slots): weights are loaded in chunks of 8 rows (8 x LDS.128 in flight, branch-free:
// out-of-range rows re-read row 0 and are discarded by a select), every row slot keeps its own accumulator, and ONE butterfly reduces
// all of them at the end.  A phase is a chain of dependent latencies: one shuffle chain per phase instead of one per 8 rows.
// WBF16: the slice holds bf16 rows; column group kqc is read as 8 bytes and widened (the same products in the same order)
template <int NB, int P, bool WBF16 = false>
__device__ __forceinline__ void m3_rows(const float* wb, int K, int R, int G, int rg, int NS, const int (&kqc)[M3_NS], const float4 (&xv)[NB][M3_NS],
                                        float* red_b0, float* red_b1, int wi, int lane) {
    float acc[NB][P];
#pragma unroll
    for (int c = 0; c < P / 8; ++c) {
        const float4* wrow[8];
        const uint2* wrow16[8];
        bool valid[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int lr = (c * 8 + i) * G + rg;
            valid[i] = lr < R;
            if constexpr (WBF16) wrow16[i] = reinterpret_cast<const uint2*>(reinterpret_cast<const unsigned short*>(wb) + (valid[i] ? lr : 0) * K);
            else wrow[i] = reinterpret_cast<const float4*>(wb + (valid[i] ? lr : 0) * K);
#pragma unroll
            for (int b = 0; b < NB; ++b) acc[b][c * 8 + i] = 0.f;
        }
        if (c * 8 * G + rg < R) {             // (warp-uniform when G == 1; otherwise the selects below discard what the extra rows add)
#pragma unroll
            for (int s = 0; s < M3_NS; ++s) {
                if (s < NS) {
                    float4 w[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        if constexpr (WBF16) w[i] = bf16x4_to_float4(wrow16[i][kqc[s]]);
                        else w[i] = wrow[i][kqc[s]];
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int b = 0; b < NB; ++b) acc[b][c * 8 + i] += m3_dot4(w[i], xv[b][s]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int b = 0; b < NB; ++b) acc[b][c * 8 + i] = valid[i] ? acc[b][c * 8 + i] : 0.f;
    }
    const int lr = m3_ridx<P>(lane) * G + rg;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
        const float v = m3_reduce<P>(acc[b], lane);
        if (m3_rowner<P>(lane) && lr < R) (b == 0 ? red_b0 : red_b1)[lr * M2_WARPS + wi] = v;
    }
}

// Per-thread poll geometry, computed once per kernel: where this thread's columns of the three GEMV inputs live (its replica of the
// residual stream / merged heads / fc1 output) and which of its column slots exist.  A phase's first poll round is then two shared-memory
// reads (which input, how many CTAs own rows) away from the phase top.
struct M3Poll { const ll_t* x; const ll_t* att; const ll_t* h; unsigned mask_d, mask_f; };
__device__ __forceinline__ M3Poll m3_make_poll(const MegaLL& ll, const M3Map& md, const M3Map& mf, int rep_off) {
    M3Poll q;
    q.x = ll.x + (long long)rep_off * ll.x_rep + md.kq0 * 4;
    q.att = ll.att + (long long)rep_off * ll.x_rep + md.kq0 * 4;
    q.h = ll.h + (long long)rep_off * ll.h_rep + mf.kq0 * 4;
    q.mask_d = q.mask_f = 0;
#pragma unroll
    for (int s = 0; s < M3_NS; ++s) {
        // grouped mapping: group 0 polls for everybody (one column each); else a thread polls exactly the columns it multiplies
        if ((md.grouped ? md.rg == 0 && s == 0 : s < md.NS) && md.kq0 + s * M2_THREADS < md.K4) q.mask_d |= 1u << s;
        if ((mf.grouped ? mf.rg == 0 && s == 0 : s < mf.NS) && mf.kq0 + s * M2_THREADS < mf.K4) q.mask_f |= 1u << s;
    }
    return q;
}

// ---- row-per-warp GEMV phase (inputs as wide as d_model: qkv, out, q_c, out_c, fc1, proj_out) ------------------------------------------
// Measured on the K-split form (tools/mega3_trace.py): the multiply is instruction-issue bound, ~12 instructions per float4 product
// (address, select, butterfly share) with only 6 of 8 warps busy.  For the d_model-wide inputs the activation is small enough to sit in
// every warp's registers (K / 32 floats per lane), so each warp takes whole rows (warp, warp + 8, ...): one LDS.128 and four FFMA per
// float4 product — gemv_dot's arithmetic and summation order, i.e. the same bits as the per-phase kernels and the barrier megakernel —
// five shuffles per row, and the warp finishes its own rows (lane = row slot x replica: one store instruction writes every replica).
// No cross-warp reduction, no epilogue hand-over: the phase's only CTA barrier is the one that publishes the activation.
template <int NB, bool WBF16, typename SM>
__device__ __forceinline__ void m3_rw_tail(const Mega2Params& mp, const Mega2Phase& ph2, SM& sm, int cta, int tid, int buf, unsigned g_idx, int par,
                                           unsigned in_tag, unsigned out_tag, int cur_pos, int* err, unsigned long long* trace,
                                           ll_t (&w)[NB][M3_NS][4], const bool (&on)[NB][M3_NS], bool poller, const ll_t* in, int r0, int R) {
    const MegaPhase& ph = ph2.base;
    const GemvParams& g = ph.g;
    const int lane = tid & 31, warp = tid >> 5;
    const int d = mp.d_model, K = d, K4 = d >> 2;
    const bool ln = g.xmode == X_LAYERNORM;
    // ---- epilogue operands of this lane: row slot ei = lane / 8 (rows warp, warp + 8, warp + 16, warp + 24), replica rep = lane % 8 ----
    const int ei = lane >> 3, rep = lane & 7;
    const int erow = warp + M2_WARPS * ei;
    int act = 0;
    float alpha = 1.f, bias_v = 0.f, res_v[NB];
    ll_t* lo[NB];
    float* plain[NB];
    bool st0 = false, st1 = false;
    long long rs8 = 0;
#pragma unroll
    for (int b = 0; b < NB; ++b) { res_v[b] = 0.f; lo[b] = nullptr; plain[b] = nullptr; }
    if (erow < R) {
        const int n = r0 + erow;
        const int si = (int)(g.nseg > 1 && n >= g.seg[1].n_begin) + (int)(g.nseg > 2 && n >= g.seg[2].n_begin);
        const GemvSeg& sg = g.seg[si];
        const int col = n - sg.n_begin;
        if (g.bias) bias_v = __ldg(g.bias + n);
        act = sg.act; alpha = sg.alpha;
        const long long rs = ph2.out_rs[si];
        rs8 = 8 * rs;
        const bool has_out = ph2.out_sel[si] != LL_NONE;
        st0 = has_out && (rs ? rep < mp.ll.reps : rep == 0);
        st1 = has_out && rs && rep + 8 < mp.ll.reps;
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            if (b < mp.rows) {
                if (ph2.res_xraw) res_v[b] = sm.xraw[b * d + n];
                lo[b] = mp.ll.x + ph2.out_off[si] + (long long)b * ph2.out_bw[si] + col + rep * rs;
                if (ph2.plain_out[si] && rep == 0) plain[b] = sg.out + (long long)b * sg.out_bs + (long long)cur_pos * sg.pos_stride + col;
            }
        }
    }
    const int kq0 = tid;                                   // pollers: thread t holds float4 column t (t < K4 <= 256)
    float4 lw = make_float4(0, 0, 0, 0), lb = lw;
    if (ln && poller) {
        lw = __ldg(reinterpret_cast<const float4*>(g.ln_w) + kq0);
        lb = __ldg(reinterpret_cast<const float4*>(g.ln_b) + kq0);
    }
    if (trace && tid == 0) trace[2] = (unsigned long long)clock64();
    // ---- input ----
    if (poller) {
        long long spin = 0;
        while (true) {
            bool ok = true;
#pragma unroll
            for (int b = 0; b < NB; ++b)
                if (on[b][0]) ok = ok && ll_tag_ok4(w[b][0][0], w[b][0][1], w[b][0][2], w[b][0][3], in_tag);
            if (ok || !ll_spin_check(spin, err, in_tag)) break;
#pragma unroll
            for (int b = 0; b < NB; ++b)
                if (on[b][0]) {
                    const ll_t* src = in + (long long)b * K + kq0 * 4;
                    ll_load2(src, w[b][0][0], w[b][0][1]);
                    ll_load2(src + 2, w[b][0][2], w[b][0][3]);
                }
        }
        if (trace && tid == 0) { trace[4] = (unsigned long long)clock64(); trace[10] = (unsigned long long)spin; }
    }
    float* xs = sm.xrw[par];
    if (R > 0) {
        float4 raw[NB];
#pragma unroll
        for (int b = 0; b < NB; ++b)
            raw[b] = on[b][0] ? make_float4(ll_val(w[b][0][0]), ll_val(w[b][0][1]), ll_val(w[b][0][2]), ll_val(w[b][0][3])) : make_float4(0, 0, 0, 0);
        const int npl = (K4 + 31) >> 5;
        if (ln) {
            // LayerNorm with the reduction structure of gemv_stage_x (32-float4 chunks per warp, 8 chunk partials, fixed tree)
            if (warp < npl) {
                const float inv = 1.0f / (float)K;
#pragma unroll
                for (int b = 0; b < NB; ++b) {
                    const float sc = warp_sum((raw[b].x + raw[b].y) + (raw[b].z + raw[b].w));
                    if (lane == 0) sm.ln_red[b * 8 + warp] = sc;
                    if (poller) reinterpret_cast<float4*>(sm.xraw + b * K)[kq0] = raw[b];
                }
                m3_bar_cols(npl * 32);
                if (trace && tid == 0) trace[5] = (unsigned long long)clock64();
                float mean[NB];
#pragma unroll
                for (int b = 0; b < NB; ++b) {
                    mean[b] = m3_tree8(sm.ln_red + b * 8) * inv;
                    float q = 0.f;
                    if (poller && b < mp.rows) {
                        const float a0 = raw[b].x - mean[b], a1 = raw[b].y - mean[b], a2 = raw[b].z - mean[b], a3 = raw[b].w - mean[b];
                        q = (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
                    }
                    q = warp_sum(q);
                    if (lane == 0) sm.ln_red2[b * 8 + warp] = q;
                }
                m3_bar_cols(npl * 32);
                if (poller) {
#pragma unroll
                    for (int b = 0; b < NB; ++b) {
                        float4 o = make_float4(0, 0, 0, 0);
                        if (b < mp.rows) {
                            const float rstd = rsqrtf(m3_tree8(sm.ln_red2 + b * 8) * inv + g.eps);
                            o.x = (raw[b].x - mean[b]) * rstd * lw.x + lb.x; o.y = (raw[b].y - mean[b]) * rstd * lw.y + lb.y;
                            o.z = (raw[b].z - mean[b]) * rstd * lw.z + lb.z; o.w = (raw[b].w - mean[b]) * rstd * lw.w + lb.w;
                        }
                        reinterpret_cast<float4*>(xs + b * K)[kq0] = o;
                    }
                }
            }
        } else if (poller) {
#pragma unroll
            for (int b = 0; b < NB; ++b) reinterpret_cast<float4*>(xs + b * K)[kq0] = raw[b];
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");   // next phase's descriptor (issued at the top of the phase loop)
    __syncthreads();                                   // activation published; next descriptor landed
    if (trace && tid == 0) trace[6] = (unsigned long long)clock64();
    wait_weights(&sm.mbar[buf], (g_idx >> 1) & 1, err);
    if (trace && tid == 0) trace[3] = (unsigned long long)clock64();

    float sum[NB][4];
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
        for (int i = 0; i < 4; ++i) sum[b][i] = 0.f;
    if (R > 0 && warp < R && !(c_ll_debug & 4)) {
        constexpr int XS = 8;                              // float4 of the activation per lane (d_model <= 1024)
        const int nx = (K4 + 31) >> 5;
        float4 xr[NB][XS];
        const float4* xs4 = reinterpret_cast<const float4*>(xs);
#pragma unroll
        for (int j = 0; j < XS; ++j) {
            const int col = j * 32 + lane;
#pragma unroll
            for (int b = 0; b < NB; ++b) xr[b][j] = (j < nx && col < K4 && b < mp.rows) ? xs4[b * K4 + col] : make_float4(0, 0, 0, 0);
        }
        const float* wbs = wslice(sm.wbuf, buf, slice_floats<WBF16>(ph.rpc * K));
        const float4* wb4 = reinterpret_cast<const float4*>(wbs);
        const uint2* wb2 = reinterpret_cast<const uint2*>(wbs);
        float4 acc[NB][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int b = 0; b < NB; ++b) acc[b][i] = make_float4(0, 0, 0, 0);
            const int row = warp + M2_WARPS * i;
            if (row < R) {                                 // warp-uniform
                const float4* wrow = wb4 + row * K4;
                const uint2* wrow2 = wb2 + row * K4;
#pragma unroll
                for (int j = 0; j < XS; ++j) {
                    if (j < nx) {
                        const int col = j * 32 + lane;
                        float4 wv;                                       // (x is zero beyond K4)
                        if constexpr (WBF16) wv = bf16x4_to_float4(wrow2[col < K4 ? col : 0]);
                        else wv = wrow[col < K4 ? col : 0];
#pragma unroll
                        for (int b = 0; b < NB; ++b) {
                            acc[b][i].x = fmaf(wv.x, xr[b][j].x, acc[b][i].x); acc[b][i].y = fmaf(wv.y, xr[b][j].y, acc[b][i].y);
                            acc[b][i].z = fmaf(wv.z, xr[b][j].z, acc[b][i].z); acc[b][i].w = fmaf(wv.w, xr[b][j].w, acc[b][i].w);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int b = 0; b < NB; ++b) sum[b][i] = warp_sum((acc[b][i].x + acc[b][i].y) + (acc[b][i].z + acc[b][i].w));
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.wfree[buf]);            // this warp no longer reads the weight slice
    if (trace && tid == 0) trace[7] = (unsigned long long)clock64();
    // ---- epilogue in the warp that owns the rows ----
#pragma unroll
    for (int b = 0; b < NB; ++b) {
        if (lo[b]) {
            float v = ei == 0 ? sum[b][0] : (ei == 1 ? sum[b][1] : (ei == 2 ? sum[b][2] : sum[b][3]));
            v += bias_v;
            v = apply_act(v, act) * alpha;
            v += res_v[b];
            if (st0) ll_store(lo[b], v, out_tag);
            if (st1) ll_store(lo[b] + rs8, v, out_tag);
            if (plain[b]) {
                *plain[b] = v;
                __threadfence();                           // K/V cache rows are read by LATER tokens through plain loads (see the header comment)
            }
        }
    }
    if (trace && tid == 0) { trace[8] = (unsigned long long)clock64(); trace[9] = trace[8]; }
}

template <int NB, bool WBF16, typename SM>
__device__ __forceinline__ void m3_gemv_phase(const Mega2Params& mp, const Mega2Phase& ph2, SM& sm, const M3Map& mapd, const M3Map& mapf, const M3Poll& pl, int cta,
                                              int tid, unsigned g_idx, int par, unsigned in_tag, unsigned out_tag, int cur_pos, int* err,
                                              unsigned long long* trace /* null or [16] */) {
    // ---- the first poll round goes out before anything else: which input, does this CTA own rows — then the loads ----
    const int isel = ph2.in_sel;
    const bool has_rows = cta < ph2.n_active;
    const bool in_h = isel == LL_H;
    const ll_t* const pin = in_h ? pl.h : (isel == LL_ATT ? pl.att : pl.x);
    const unsigned pmask = has_rows ? (in_h ? pl.mask_f : pl.mask_d) : 0u;
    const int Kin = in_h ? mp.ffn_dim : mp.d_model;
    ll_t w[NB][M3_NS][4];
    bool on[NB][M3_NS];
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
        for (int s = 0; s < M3_NS; ++s) {
            on[b][s] = ((pmask >> s) & 1u) != 0 && b < mp.rows;
            w[b][s][0] = w[b][s][1] = w[b][s][2] = w[b][s][3] = 0;
            if (on[b][s]) {
                const ll_t* src = pin + (long long)b * Kin + s * (M2_THREADS * 4);
                ll_load2(src, w[b][s][0], w[b][s][1]);
                ll_load2(src + 2, w[b][s][2], w[b][s][3]);
            }
        }
    const bool poller = pmask != 0;
    const MegaPhase& ph = ph2.base;
    const GemvParams& g = ph.g;
    const int lane = tid & 31, warp = tid >> 5;
    const int buf = g_idx & 1;
    const int d = mp.d_model;
    const int K = g.K;
    const bool isd = !in_h;
    const int K4 = K >> 2;
    const bool grouped = isd ? mapd.grouped : mapf.grouped, in_group = isd ? mapd.in_group : mapf.in_group, active_warp = isd ? mapd.active_warp : mapf.active_warp;
    const int G = isd ? mapd.G : mapf.G, rg = isd ? mapd.rg : mapf.rg, kq0 = isd ? mapd.kq0 : mapf.kq0, NS = isd ? mapd.NS : mapf.NS,
              npw = isd ? mapd.npw : mapf.npw, wi = isd ? mapd.wi : mapf.wi;
    int r0, r1;
    cta_rows(g.N, cta, ph.rpc, r0, r1);
    const int R = r1 - r0;
    const bool ln = g.xmode == X_LAYERNORM;
    const bool shared = ln || grouped;
    const ll_t* in = pin - kq0 * 4;
    if (trace && tid == 0) trace[1] = (unsigned long long)clock64();
    // The next GEMV's weight slice goes into the buffer the PREVIOUS GEMV phase read: requested as soon as every warp has signalled that
    // it is done with it (a whole phase of lead for the copy).
    if (tid == M2_THREADS - 32) {
        if (g_idx > 0) wait_weights(&sm.wfree[buf ^ 1], ((g_idx - 1) >> 1) & 1, err);      // every warp has finished reading the slice of GEMV phase g_idx - 1
        prefetch_weights<WBF16>(ph.nx_W, ph.nx_ldw, ph.nx_N, ph.nx_K, wslice(sm.wbuf, buf ^ 1, slice_floats<WBF16>(ph.nx_rpc * ph.nx_K)), &sm.mbar[buf ^ 1], cta,
                                ph.nx_rpc);
    }
    if (isd) {
        m3_rw_tail<NB, WBF16>(mp, ph2, sm, cta, tid, buf, g_idx, par, in_tag, out_tag, cur_pos, err, trace, w, on, poller, in, r0, R);
        return;
    }
    const bool has_col = in_group && kq0 < K4;
    float4 lw = make_float4(0, 0, 0, 0), lb = lw;
    if (ln && has_col) {
        lw = __ldg(reinterpret_cast<const float4*>(g.ln_w) + kq0);
        lb = __ldg(reinterpret_cast<const float4*>(g.ln_b) + kq0);
    }

    // ---- epilogue operands, fetched NOW by the threads that will finish the rows (warps 6 / 7: thread 192 + e finishes decoder row e / R,
    //      output row e % R), so that nothing but the sum itself is left behind the barrier ----
    const int e = tid - (M2_THREADS - 64);
    bool epi = false;
    int eb = 0, elr = 0, act = 0, ll_nrep = 0;
    float bias_v = 0.f, res_v = 0.f, alpha = 1.f;
    ll_t* ll_out = nullptr;
    long long ll_rs = 0;
    float* plain = nullptr;
    if (e >= 0 && e < R * NB) {
        eb = (NB > 1 && e >= R) ? 1 : 0;
        elr = e - eb * R;
        epi = eb < g.B;
        if (epi) {
            const int n = r0 + elr;
            const int si = (int)(g.nseg > 1 && n >= g.seg[1].n_begin) + (int)(g.nseg > 2 && n >= g.seg[2].n_begin);
            const GemvSeg& sg = g.seg[si];
            const int col = n - sg.n_begin;
            if (g.bias) bias_v = __ldg(g.bias + n);
            if (ph2.res_xraw) res_v = sm.xraw[eb * d + n];
            act = sg.act; alpha = sg.alpha;
            if (ph2.out_sel[si] != LL_NONE) {
                ll_out = mp.ll.x + ph2.out_off[si] + (long long)eb * ph2.out_bw[si] + col;
                ll_rs = ph2.out_rs[si];
                ll_nrep = ph2.out_rs[si] ? mp.ll.reps : 1;
            }
            if (ph2.plain_out[si]) plain = sg.out + (long long)eb * sg.out_bs + (long long)cur_pos * sg.pos_stride + col;
        }
    }

    if (trace && tid == 0) trace[2] = (unsigned long long)clock64();
    if (active_warp) wait_weights(&sm.mbar[buf], (g_idx >> 1) & 1, err);        // requested a phase ago (only the warps that multiply need it)
    if (trace && tid == 0) trace[3] = (unsigned long long)clock64();

    // ---- input: polled straight into registers ----
    float4 xv[NB][M3_NS];
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
        for (int s = 0; s < M3_NS; ++s) xv[b][s] = make_float4(0, 0, 0, 0);
    if (poller) {
        long long spin = 0;
        while (true) {
            bool ok = true;
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int s = 0; s < M3_NS; ++s)
                    if (on[b][s]) ok = ok && ll_tag_ok4(w[b][s][0], w[b][s][1], w[b][s][2], w[b][s][3], in_tag);
            if (ok || !ll_spin_check(spin, err, in_tag)) break;
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int s = 0; s < M3_NS; ++s)
                    if (on[b][s]) {
                        const ll_t* src = in + (long long)b * K + (kq0 + s * M2_THREADS) * 4;
                        ll_load2(src, w[b][s][0], w[b][s][1]);
                        ll_load2(src + 2, w[b][s][2], w[b][s][3]);
                    }
        }
        if (trace && tid == 0) { trace[4] = (unsigned long long)clock64(); trace[10] = (unsigned long long)spin; }
    }
    const int ncols = grouped ? G * K4 : npw * 32;      // threads of the warps that hold columns (whole warps, from thread 0)
    if (R > 0 && active_warp) {
        if (shared) {
            float4 raw[NB];
#pragma unroll
            for (int b = 0; b < NB; ++b)
                raw[b] = on[b][0] ? make_float4(ll_val(w[b][0][0]), ll_val(w[b][0][1]), ll_val(w[b][0][2]), ll_val(w[b][0][3])) : make_float4(0, 0, 0, 0);
            const bool pol = poller;
            if (ln) {
                // LayerNorm with the reduction structure of gemv_stage_x (32-float4 chunks per warp, 8 chunk partials, fixed tree): the
                // normalised activations carry the same bits as in the other token-loop drivers.
                const int npl = (K4 + 31) >> 5;
                const float inv = 1.0f / (float)K;
                if (warp < npl) {
#pragma unroll
                    for (int b = 0; b < NB; ++b) {
                        const float sc = warp_sum((raw[b].x + raw[b].y) + (raw[b].z + raw[b].w));
                        if (lane == 0) sm.ln_red[b * 8 + warp] = sc;
                        if (pol) reinterpret_cast<float4*>(sm.xraw + b * K)[kq0] = raw[b];
                    }
                }
                m3_bar_cols(ncols);
                if (trace && tid == 0) trace[5] = (unsigned long long)clock64();
                float mean[NB];
#pragma unroll
                for (int b = 0; b < NB; ++b) mean[b] = m3_tree8(sm.ln_red + b * 8) * inv;
                if (warp < npl) {
#pragma unroll
                    for (int b = 0; b < NB; ++b) {
                        float q = 0.f;
                        if (pol && b < g.B) {
                            const float a0 = raw[b].x - mean[b], a1 = raw[b].y - mean[b], a2 = raw[b].z - mean[b], a3 = raw[b].w - mean[b];
                            q = (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
                        }
                        q = warp_sum(q);
                        if (lane == 0) sm.ln_red2[b * 8 + warp] = q;
                    }
                }
                m3_bar_cols(ncols);
                if (has_col) {
#pragma unroll
                    for (int b = 0; b < NB; ++b) {
                        if (b < g.B) {
                            const float rstd = rsqrtf(m3_tree8(sm.ln_red2 + b * 8) * inv + g.eps);
                            const float4 v = pol ? raw[b] : reinterpret_cast<const float4*>(sm.xraw + b * K)[kq0];
                            xv[b][0].x = (v.x - mean[b]) * rstd * lw.x + lb.x; xv[b][0].y = (v.y - mean[b]) * rstd * lw.y + lb.y;
                            xv[b][0].z = (v.z - mean[b]) * rstd * lw.z + lb.z; xv[b][0].w = (v.w - mean[b]) * rstd * lw.w + lb.w;
                        }
                    }
                }
            } else {
                if (G > 1) {            // more than one row group: hand the polled columns over through shared memory
                    if (pol) {
#pragma unroll
                        for (int b = 0; b < NB; ++b) reinterpret_cast<float4*>(sm.u.xs + b * K)[kq0] = raw[b];
                    }
                    m3_bar_cols(ncols);
                }
                if (has_col) {
#pragma unroll
                    for (int b = 0; b < NB; ++b) xv[b][0] = pol ? raw[b] : reinterpret_cast<const float4*>(sm.u.xs + b * K)[kq0];
                }
            }
        } else {
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int s = 0; s < M3_NS; ++s)
                    if (on[b][s]) xv[b][s] = make_float4(ll_val(w[b][s][0]), ll_val(w[b][s][1]), ll_val(w[b][s][2]), ll_val(w[b][s][3]));
        }
    }
    if (trace && tid == 0) trace[6] = (unsigned long long)clock64();

    // ---- multiply + reduce ----
    if (R > 0 && active_warp && !(c_ll_debug & 4)) {
        const int Pn = G == 1 ? R : (G == 2 ? (R + 1) >> 1 : (R + G - 1) / G);       // row slots per thread (host guarantees <= M3_SLOTS)
        const float* wb = wslice(sm.wbuf, buf, slice_floats<WBF16>(ph.rpc * K));
        int kqc[M3_NS];
#pragma unroll
        for (int s = 0; s < M3_NS; ++s) kqc[s] = kq0 + s * M2_THREADS < K4 ? kq0 + s * M2_THREADS : 0;
        float* red0 = &sm.red[par][0][0][0];
        float* red1 = &sm.red[par][NB - 1][0][0];
        if (Pn <= 8)       m3_rows<NB, 8, WBF16>(wb, K, R, G, rg, NS, kqc, xv, red0, red1, wi, lane);
        else if (Pn <= 16) m3_rows<NB, 16, WBF16>(wb, K, R, G, rg, NS, kqc, xv, red0, red1, wi, lane);
        else               m3_rows<NB, 32, WBF16>(wb, K, R, G, rg, NS, kqc, xv, red0, red1, wi, lane);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.wfree[buf]);        // this warp no longer reads the weight slice
    if (trace && tid == 0) trace[7] = (unsigned long long)clock64();
    asm volatile("cp.async.wait_all;" ::: "memory");   // next phase's descriptor (issued at the top of the phase loop)
    __syncthreads();
    if (trace && tid == 0) trace[8] = (unsigned long long)clock64();

    // ---- epilogue: sum of the warp partials (fixed tree over 8 slots, unused ones read as zero), bias / activation / residual, tagged store ----
    if (epi) {
        const float4* r4 = reinterpret_cast<const float4*>(&sm.red[par][eb][elr][0]);
        const float4 q0 = r4[0], q1 = r4[1];
        float t[M2_WARPS] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
        for (int i = 0; i < M2_WARPS; ++i) t[i] = i < npw ? t[i] : 0.f;
        float v = ((t[0] + t[1]) + (t[2] + t[3])) + ((t[4] + t[5]) + (t[6] + t[7]));
        v += bias_v;
        v = apply_act(v, act) * alpha;
        v += res_v;
        if (ll_nrep == 1) ll_store(ll_out, v, out_tag);
        else {
#pragma unroll
            for (int rep = 0; rep < MEGA_LL_MAX_REPS; ++rep)
                if (rep < ll_nrep) ll_store(ll_out + rep * ll_rs, v, out_tag);
        }
        if (plain) {
            *plain = v;
            __threadfence();                           // K/V cache rows are read by LATER tokens through plain loads (see the header comment)
        }
        if (trace && e == 0) trace[9] = (unsigned long long)clock64();
    }
}

// TRACE = true is a separate instantiation for tools/mega2_trace.py: CTAs 0, 1, 100 and 140 stamp clock64 at four points of every phase
// of token `trace_step` (phase start, input staged, weights landed, rows / units done); the production kernel carries no stamp code.
// WBF16: the phase table's weight matrices are the bf16 store (same rows per CTA, same schedule, half the bytes per slice)
template <int NB, bool TRACE, bool WBF16 = false>
__global__ void __launch_bounds__(M2_THREADS, 1) decode_megakernel_ll(Mega2Params mp) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    M2Smem& sm = *reinterpret_cast<M2Smem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, G = gridDim.x;
    const int d = mp.d_model;
    int* const err = mp.error_flag;

    if (tid == 0) {
        sm.sample_params = mp.sample;
        mbar_init(&sm.mbar[0], 1);
        mbar_init(&sm.mbar[1], 1);
        mbar_init(&sm.wfree[0], M2_WARPS);
        mbar_init(&sm.wfree[1], M2_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    m2_clear_ln_red(sm.ln_red, tid);
    m2_clear_ln_red(sm.ln_red2, tid);
    if (c_ll_debug & 1) for (int i = tid; i < 2 * MEGA_WBUF_FLOATS; i += M2_THREADS) (&sm.wbuf[0][0])[i] = 0.f;      // diagnostics: no weight stream, finite numbers
    __syncthreads();
    unsigned int g_idx = 0;          // running index of GEMV phases (selects weight buffer + mbarrier parity)
    if (tid == 0) {
        const MegaPhase* f = &mp.phases[0].base;
        prefetch_weights<WBF16>(f->g.W, f->g.ldw, f->g.N, f->g.K, wslice(sm.wbuf, 0, 0), &sm.mbar[0], cta, (f->g.N + G - 1) / G);
    }
    // CTA 0 publishes the residual stream left by the prefill (plain memory, written by an earlier kernel) and the first token header
    // under the tag the first phase of step 0 expects: "last phase of step -1"
    if (cta == 0) {
        const unsigned t0 = ll_tag(-1, mp.n_phases - 1);
        for (int rep = 0; rep < mp.ll.reps; ++rep)
            for (int i = tid; i < mp.rows * d; i += M2_THREADS) ll_store(mp.ll.x + rep * mp.ll.x_rep + i, mp.x_in[i], t0);
        if (tid == 0) {
            ll_store(mp.ll.hdr + 0, __int_as_float(ld_state(&mp.st->cur_len)), t0);
            ll_store(mp.ll.hdr + 1, __int_as_float(ld_state(&mp.st->all_finished)), t0);
        }
    }
    {
        const int* src = reinterpret_cast<const int*>(&mp.phases[0]);
        int* dst = reinterpret_cast<int*>(&sm.phase[0]);
        for (int i = tid; i < (int)(sizeof(Mega2Phase) / 4); i += M2_THREADS) dst[i] = src[i];
    }
    __syncthreads();
    int cur = 0;
    AttnRegs<M2_WARPS> areg;
    const M3Map mapd = m3_make_map(mp.d_model, tid), mapf = m3_make_map(mp.ffn_dim > 0 ? mp.ffn_dim : mp.d_model, tid);
    const M3Poll pl = m3_make_poll(mp.ll, mapd, mapf, cta % mp.ll.reps);

    for (int step = 0; step < mp.max_steps; ++step) {
        if (tid == 0) {      // token header: written by the selection phase of the previous token (or the prologue above)
            const unsigned th = ll_tag(step - 1, mp.n_phases - 1);
            sm.ctrl[0] = __float_as_int(ll_wait1(mp.ll.hdr + 0, th, err));
            sm.ctrl[1] = __float_as_int(ll_wait1(mp.ll.hdr + 1, th, err));
            sm.ctrl[2] = *reinterpret_cast<volatile int*>(err);
            sm.ctrl[3] = ld_state(&mp.st->prompt_len);
            sm.ctrl[4] = mp.row_slot[0]; sm.ctrl[5] = mp.rows > 1 ? mp.row_slot[1] : 0;
        }
        __syncthreads();
        const int cur_pos = sm.ctrl[0] - 1, fin = sm.ctrl[1], e = sm.ctrl[2], P = sm.ctrl[3];
        if (fin || e) break;
        const int tslot = cta == mp.trace_cta ? 0 : -1;
        const bool tracing = TRACE && mp.trace != nullptr && step == mp.trace_step && tslot >= 0 && tid == 0;
#define M2_TRACE(slot) do { if (tracing) mp.trace[(long long)pi * 16 + (slot)] = (unsigned long long)clock64(); } while (0)
        for (int pi = 0; pi < mp.n_phases; ++pi) {
            M2_TRACE(0);
            const Mega2Phase& ph2 = sm.phase[cur];
            const MegaPhase& ph = ph2.base;
            const unsigned in_tag = pi == 0 ? ll_tag(step - 1, mp.n_phases - 1) : ll_tag(step, pi - 1);
            const unsigned out_tag = ll_tag(step, pi);
            // next phase's descriptor: global -> shared asynchronously, drained before the end-of-phase CTA barrier
            constexpr int DESC_WORDS = (int)(sizeof(Mega2Phase) / 4);
            const int nxt = cur == 2 ? 0 : cur + 1;
            // (by warps 6 / 7, which hold no columns of the d_model-wide inputs, so the pollers start polling at once)
            for (int i = tid - (M2_THREADS - 64); i >= 0 && i < DESC_WORDS; i += 64) {
                const int* src = reinterpret_cast<const int*>(&mp.phases[pi + 1 < mp.n_phases ? pi + 1 : 0]) + i;
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(reinterpret_cast<int*>(&sm.phase[nxt]) + i)), "l"(src) : "memory");
            }
            if (ph.kind == 0) {
                // timeline (TRACE instantiation, CTA mp.trace_cta): 16 stamps per phase, see tools/mega3_trace.py
                unsigned long long* tr = nullptr;
                if (TRACE && mp.trace != nullptr && step == mp.trace_step && cta == mp.trace_cta) tr = mp.trace + (long long)pi * 16;
                m3_gemv_phase<NB, WBF16>(mp, ph2, sm, mapd, mapf, pl, cta, tid, g_idx, pi & 1, in_tag, out_tag, cur_pos, err, tr);
                ++g_idx;
            } else if (ph.kind == 1) {
                const DecAttnParams& a = ph.a;
                const bool is_self = a.fixed_len == 0;
                const int L = is_self ? cur_pos + 1 : a.fixed_len;
                const int units = a.rows * a.H * a.n_splits;
                for (int u = cta; u < units; u += G) {
                    const int hr = ph.magic_ns ? (int)__umulhi((unsigned)u, ph.magic_ns) : u;
                    const int s = u - hr * a.n_splits;
                    const int r = ph.magic_h ? (int)__umulhi((unsigned)hr, ph.magic_h) : hr;
                    const int h = hr - r * a.H;
                    const int slot = a.row_slot ? sm.ctrl[4 + r] : r;
                    // K/V of the cache first (they do not depend on this token's phases), q and the appended row are polled inside
                    decode_attention_load<M2_WARPS>(a, s, h, r, slot, L, P, tid, areg);
                    unsigned long long* tr = nullptr;
                    if (TRACE && mp.trace != nullptr && step == mp.trace_step && cta == mp.trace_cta && u == cta) tr = mp.trace + (long long)pi * 16;
                    if (tr && tid == 0) tr[1] = (unsigned long long)clock64();
                    m2_attention_unit(a, mp.ll, is_self, s, h, r, slot, L, P, in_tag, out_tag, sm.u.attn.sc, sm.u.attn.red, sm.u.attn.stat, sm.u.attn.qs,
                                      sm.u.attn.kns, sm.u.attn.vns, tid, areg, err, tr);
                    if (tr && tid == 0) tr[5] = (unsigned long long)clock64();
                    if (a.n_splits > 1 && s == 0) { __syncthreads(); m2_attention_merge(a, mp.ll, h, r, L, out_tag, sm.u.attn.sc, tid, err); if (tr && tid == 0) tr[6] = (unsigned long long)clock64(); }
                    __syncthreads();
                }
            } else {
                if (cta < sm.sample_params.cfg->B) {
                    if (tid == 0) {
                        sm.sample_params.ll_in_tag = in_tag; sm.sample_params.ll_out_tag = out_tag;
                        sm.sample_params.trace = (TRACE && mp.trace != nullptr && step == mp.trace_step && cta == mp.trace_cta) ? mp.trace + (long long)pi * 16 : nullptr;
                    }
                    __syncthreads();
                    sample_body<M2_THREADS>(sm.sample_params, cta, sm.u.sample);
                }
            }
            if (ph.kind != 0) {                           // (a GEMV phase ends with its own barrier, before its epilogue)
                asm volatile("cp.async.wait_all;" ::: "memory");
                __syncthreads();                          // attention / selection scratch free for the next phase; the next descriptor has landed
                M2_TRACE(8);
            }
            cur = nxt;
        }
    }
#undef M2_TRACE
    // drain the weight prefetch that is still in flight so no bulk copy outlives the CTA
    wait_weights(&sm.mbar[g_idx & 1], (g_idx >> 1) & 1, err);
}

}  // namespace

size_t mega2_smem_bytes() { return sizeof(M2Smem) + 128; }

int mega2_set_poll_sleep(int ns) {
    MB_CUDA_CHECK(cudaMemcpyToSymbol(c_ll_sleep_ns, &ns, sizeof(int)));
    return 0;
}
int mega2_set_debug(int bits) {
    MB_CUDA_CHECK(cudaMemcpyToSymbol(c_ll_debug, &bits, sizeof(int)));
    return 0;
}

template <int NB, bool TRACE, bool WBF16>
static const void* m2_configure() {
    const void* fn = (const void*)decode_megakernel_ll<NB, TRACE, WBF16>;
    static bool done = false;
    if (!done) {
        if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega2_smem_bytes()) != cudaSuccess) return nullptr;
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, M2_THREADS, mega2_smem_bytes()) != cudaSuccess || per_sm < 1) return nullptr;
        done = true;
    }
    return fn;
}

int launch_megakernel2(const Mega2Params& mp, int grid, cudaStream_t stream, bool w_bf16) {
    MB_REQUIRE(mp.rows >= 1 && mp.rows <= M2_NB_MAX, "megakernel handles 1 or 2 decoder rows");
    MB_REQUIRE(mp.n_phases <= 126, "tag layout holds at most 126 phases per token");
    MB_REQUIRE(mp.d_model <= 1024, "residual scratch holds d_model <= 1024");
    const bool tr = mp.trace != nullptr, one = mp.rows == 1;
    const void* fn = w_bf16 ? (tr ? (one ? m2_configure<1, true, true>() : m2_configure<2, true, true>())
                                  : (one ? m2_configure<1, false, true>() : m2_configure<2, false, true>()))
                            : (tr ? (one ? m2_configure<1, true, false>() : m2_configure<2, true, false>())
                                  : (one ? m2_configure<1, false, false>() : m2_configure<2, false, false>()));
    MB_REQUIRE(fn != nullptr, "dataflow megakernel does not fit on an SM");
    Mega2Params p = mp;
    void* args[] = {&p};
    // Cooperative launch for its co-residency guarantee: every CTA polls values that other CTAs produce, so all of them must be resident.
    MB_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(M2_THREADS), args, mega2_smem_bytes(), stream));
    ++g_launch_count;
    if (w_bf16) ++g_wbf16_launch_count;
    return 0;
}

// Limits of the K-split GEMV mapping for one phase (checked on the host when the phase table is built)
bool mega2_ksplit_ok(int N, int K, int rows, int grid) {
    const int K4 = K >> 2, rpc = (N + grid - 1) / grid;
    if ((K & 3) || K4 > M3_NS * M2_THREADS) return false;
    const bool grouped = (K4 & 31) == 0 && K4 <= 256;
    const int G = grouped ? M2_THREADS / K4 : 1;
    return (rpc + G - 1) / G <= M3_SLOTS && rpc <= M3_ROWS && rpc * rows <= 64;
}

}  // namespace mb200
