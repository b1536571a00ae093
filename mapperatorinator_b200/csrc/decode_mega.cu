// Persistent token-loop megakernel: the WHOLE autoregressive decode of one generate() call (every layer of every token,
// the logits-processor chain and the token selection) is ONE cooperative launch of one CTA per SM.
//
// Why: at batch 1-2 a decoder step is 98 dependent micro-phases moving ~4.7 MB each (464 MB of fp32 weights per token).  As
// separate kernels every phase pays launch + DRAM-latency ramp (~2.5 us) for ~0.7 us of HBM time.  Here the phases are
// separated by a ~1 us grid barrier instead, and — because each CTA knows statically which weight rows it owns in the NEXT
// GEMV phase — those rows are pulled into shared memory by the TMA bulk-copy engine (cp.async.bulk + mbarrier
// complete_tx) while the current phase is still computing / waiting at its barrier.  HBM therefore streams weights
// continuously across phase boundaries (2 x 78 KB in flight per SM, 132 SMs => ~20 MB outstanding), which is what the
// weight-streaming roofline needs; the math runs out of shared memory.
//
// Same arithmetic, same order as the per-kernel path (decode_device.cuh bodies are shared), so tokens are bit-identical.
// Every cross-CTA value is read through L2 (ld.global.cg) — L1 is not coherent across SMs inside one launch.
// All spin loops are bounded: on a timeout the kernel raises `error_flag`, falls through every remaining barrier and exits,
// so a logic error can never hang the GPU.
#include "common.cuh"
#include "kernels.h"
#include "decode_device.cuh"

namespace mb200 {

namespace {

constexpr int MEGA_THREADS = SAMPLE_THREADS;            // 512
constexpr int MEGA_WARPS = MEGA_THREADS / 32;
constexpr int MEGA_TRACE_SLOTS = 16;
constexpr int MEGA_NB_MAX = 2;                          // decoder rows handled: the kernel is instantiated for 1 and 2
constexpr int XS_FLOATS = MEGA_NB_MAX * 3072;

struct __align__(16) MegaSmem {
    float wbuf[2][MEGA_WBUF_FLOATS];
    union {
        float xs[XS_FLOATS];
        SampleSmem sample;
        struct { float sc[128]; float red[4][64]; float stat[2]; } attn;
    } u;
    MegaPhase phase[2];
    SampleParams sample_params;                 // shared copy: the chain is an out-of-line call and must not pin `mp` in local memory
    int ctrl[8];                                // all_finished, error, cur_len, prompt_len, encoder slot of row 0 / row 1
    float ln_red[32];                           // LayerNorm chunk partials
    unsigned long long mbar[2];
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
// The 464 MB of decoder weights stream through the 50 MB L2 once per token.  With the default policy they evict everything
// else — LayerNorm affine vectors, biases, phase descriptors, the K/V caches — so every small latency-critical load of the next
// token misses to DRAM.  Tagging the weight stream evict-first keeps that small hot set resident in L2.
__device__ __forceinline__ unsigned long long l2_evict_first_policy() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    const unsigned long long pol = l2_evict_first_policy();
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}

// rows [r0, r1) of an N-row GEMV owned by CTA `cta` of `G`
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

// thread 0: start streaming this CTA's weight rows of GEMV phase `ph` into wbuf[buf] (WBF16: W holds bf16 bits, half the bytes)
template <bool WBF16>
__device__ __forceinline__ void prefetch_weights(const float* W, long long ldw, int N, int K, float* dst, unsigned long long* bar, int cta,
                                                 int rpc) {
    int r0, r1;
    cta_rows(N, cta, rpc, r0, r1);
    const unsigned bytes = (unsigned)(r1 - r0) * (unsigned)K * (WBF16 ? 2u : 4u);
    if (bytes == 0) { mbar_arrive(bar); return; }
    mbar_arrive_expect_tx(bar, bytes);
    bulk_g2s(dst, gemv_wrow<WBF16>(W, (long long)r0 * ldw), bytes, bar);
}

__device__ __forceinline__ bool wait_weights(unsigned long long* bar, unsigned parity, int* error_flag) {
    for (long long spin = 0; spin < (1ll << 24); ++spin) {
        if (mbar_try_wait(bar, parity)) return true;
    }
    atomicExch(error_flag, 2);
    return false;
}

__device__ __forceinline__ unsigned long long gtimer() {
    // SM cycle counter: every stamp of a trace comes from CTA 0 (one SM), so clock64 is consistent and far finer than %globaltimer
    return (unsigned long long)clock64();
}
#define MEGA_TRACE(slot)                                                                              \
    do {                                                                                              \
        if (tracing && tid == 0) mp.trace[(long long)pi * MEGA_TRACE_SLOTS + (slot)] = gtimer();                     \
    } while (0)

// Grid barrier, split in two so that work which does not depend on other CTAs (the next phase's row range, its bias prefetch) runs
// between the arrival and the wait instead of behind the barrier.
// arrive = one fire-and-forget release reduction (cumulative over the CTA's writes through the bar.sync before it);
// wait = acquire polling by thread 0.  One L2 round trip after the last arrival, no separate fences.
__device__ __forceinline__ void grid_arrive(unsigned int* counter) {
    if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
}
__device__ __forceinline__ void grid_wait(unsigned int* counter, unsigned int target, int* error_flag) {
    if (threadIdx.x == 0) {
        unsigned int v = 0;
        long long spin = 0;
        while (true) {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            if (v >= target) break;
            if ((++spin & 0xFFF) == 0 && (spin > (1ll << 25) || *reinterpret_cast<volatile int*>(error_flag) != 0)) {
                atomicExch(error_flag, 1);
                break;
            }
        }
    }
    __syncthreads();
}

// TRACE = true is a separate instantiation used only by the phase-timeline tool: the production kernel carries no stamp code.
// WBF16: the phase table's weight matrices are the bf16 store (same rows per CTA, same prefetch schedule, half the bytes per slice).
template <int MEGA_NB, bool TRACE, bool WBF16 = false>
__global__ void __launch_bounds__(MEGA_THREADS, 1) decode_megakernel(MegaParams mp) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    MegaSmem& sm = *reinterpret_cast<MegaSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, G = gridDim.x;

    if (tid == 0) {
        sm.sample_params = mp.sample;
        mbar_init(&sm.mbar[0], 1);
        mbar_init(&sm.mbar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned int g_idx = 0;          // running index of GEMV phases (selects buffer + mbarrier parity)
    unsigned int sync_target = 0;
    if (tid == 0) {
        const MegaPhase* f = &mp.phases[mp.first_gemv];
        prefetch_weights<WBF16>(f->g.W, f->g.ldw, f->g.N, f->g.K, wslice(sm.wbuf, 0, 0), &sm.mbar[0], cta, (f->g.N + G - 1) / G);
    }

    // phase descriptors are double-buffered in shared memory: slot `cur` is the phase being executed, slot `cur ^ 1` is
    // filled with the NEXT phase's descriptor while this one runs (its latency never sits on the critical path)
    auto load_desc = [&](int pi, int slot) {
        const int* src = reinterpret_cast<const int*>(&mp.phases[pi]);
        int* dst = reinterpret_cast<int*>(&sm.phase[slot]);
        for (int i = tid; i < (int)(sizeof(MegaPhase) / 4); i += MEGA_THREADS) dst[i] = src[i];
    };
    int cur = 0;
    load_desc(0, 0);
    __syncthreads();
    // Prologue of a GEMV phase that needs nothing from other CTAs: this CTA's row range and the bias of this warp's rows (lane
    // j*NB + b holds it for the warp's j-th row).  Computed between the previous barrier's arrival and its wait.
    int pre_r0 = 0, pre_r1 = 0;
    float pre_bias = 0.f;
    // ... and of a cross-attention phase: its K/V are constants of the call (encoder states), so this CTA's first unit requests
    // them before the barrier; after it only q (the previous phase's output) is still to come.
    AttnRegs<MEGA_WARPS> areg;
    bool areg_valid = false;
    auto unit_of = [&](const MegaPhase& ph_, int u, int& s_, int& h_, int& r_) {      // exact for u < 2^16 (magic 0: divisor 1)
        const int hr = ph_.magic_ns ? (int)__umulhi((unsigned)u, ph_.magic_ns) : u;
        s_ = u - hr * ph_.a.n_splits;
        r_ = ph_.magic_h ? (int)__umulhi((unsigned)hr, ph_.magic_h) : hr;
        h_ = hr - r_ * ph_.a.H;
    };
    auto phase_prologue = [&](const MegaPhase& nx) {
        areg_valid = false;
        if (nx.kind == 0) {
            cta_rows(nx.g.N, cta, nx.rpc, pre_r0, pre_r1);
            pre_bias = 0.f;
            const int n = pre_r0 + warp + (lane / MEGA_NB) * MEGA_WARPS;
            if (n < pre_r1 && nx.g.bias) pre_bias = __ldg(nx.g.bias + n);
        } else if (nx.kind == 1 && nx.a.fixed_len > 0 && nx.a.key_valid == nullptr) {
            if (cta < nx.a.rows * nx.a.H * nx.a.n_splits) {
                int s_, h_, r_;
                unit_of(nx, cta, s_, h_, r_);
                decode_attention_load<MEGA_WARPS>(nx.a, s_, h_, r_, nx.a.row_slot ? sm.ctrl[4 + r_] : r_, nx.a.fixed_len, 0, tid, areg);
            }
            areg_valid = true;
        }
    };
    phase_prologue(sm.phase[0]);

    for (int step = 0; step < mp.max_steps; ++step) {
        // uniform across the grid: all three were written before the previous grid barrier
        if (tid == 0) {
            sm.ctrl[0] = ld_state(&mp.st->all_finished); sm.ctrl[1] = ld_state(mp.error_flag);
            sm.ctrl[2] = ld_state(&mp.st->cur_len); sm.ctrl[3] = ld_state(&mp.st->prompt_len);
            sm.ctrl[4] = mp.row_slot[0]; sm.ctrl[5] = mp.sample.rows > 1 ? mp.row_slot[1] : 0;
        }
        __syncthreads();
        const int fin = sm.ctrl[0], err = sm.ctrl[1], cur_pos = sm.ctrl[2] - 1, P = sm.ctrl[3];
        if (fin || err) break;
        const bool tracing = TRACE && mp.trace != nullptr && step == mp.trace_step && cta == 0;
        for (int pi = 0; pi < mp.n_phases; ++pi) {
            const MegaPhase& ph = sm.phase[cur];
            MEGA_TRACE(0);
            // next phase's descriptor: copied global -> shared asynchronously (cp.async, no register is held across the phase: under the
            // 128-register cap a held value was spilled to local memory right after its load, i.e. the phase WAITED for it) and
            // drained just before the end-of-phase barrier
            constexpr int DESC_WORDS = (int)(sizeof(MegaPhase) / 4);
            static_assert(DESC_WORDS <= MEGA_THREADS, "descriptor must fit one word per thread");
            if (tid < DESC_WORDS) {
                const int* src = reinterpret_cast<const int*>(&mp.phases[pi + 1 < mp.n_phases ? pi + 1 : 0]) + tid;
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(reinterpret_cast<int*>(&sm.phase[cur ^ 1]) + tid)), "l"(src) : "memory");
            }
            if (ph.kind == 0) {
                const int buf = g_idx & 1;
                const int r0 = pre_r0, r1 = pre_r1;
                // epilogue operands of this warp's rows: lane j*NB + b holds them for the warp's j-th row and batch row b (no per-row
                // register arrays -> one copy of the row code).  The bias came with the pre-barrier prologue; the residual is another
                // CTA's output of the previous phase and is requested now, together with the activations.
                constexpr int OPS_ROWS = 32 / MEGA_NB;
                const float bias_pref = pre_bias;
                float r_pref = 0.f;
                {
                    const int j = lane / MEGA_NB, b = lane - j * MEGA_NB;
                    const int n = r0 + warp + j * MEGA_WARPS;
                    if (n < r1 && b < ph.g.B && ph.g.R) r_pref = __ldcg(ph.g.R + (long long)b * ph.g.r_ld + n);
                }
                // trace mode runs the staging twice through the SAME code: pass 0 (slots 8, 9, 10) is what production pays, pass 1
                // (slots 6, 7, 1) repeats it with instruction cache / TLB / L2 state warm — measured: no difference, i.e. the phases are not fetch-bound
                for (int rep = tracing ? 0 : 1; rep < 2; ++rep) {
                    MEGA_TRACE(rep ? 6 : 8);
                    gemv_stage_x<MEGA_NB, MEGA_THREADS>(ph.g, 0, sm.u.xs, sm.ln_red, tid,
                                                        tracing ? &mp.trace[(long long)pi * MEGA_TRACE_SLOTS + (rep ? 7 : 9)] : nullptr);
                    MEGA_TRACE(rep ? 1 : 10);
                    __syncthreads();
                }
                MEGA_TRACE(2);
                // The next GEMV's weight slice is requested only now: issuing the ~5-9 MB bulk stream at the top of the phase
                // queues this phase's few small latency-critical loads (activations, LN affine, bias) behind it.  It still has
                // the rest of this phase plus the next prologue to land.
                // issued by the LAST warp (it owns the fewest rows), from fields already in shared memory
                if (tid == MEGA_THREADS - 32)
                    prefetch_weights<WBF16>(ph.nx_W, ph.nx_ldw, ph.nx_N, ph.nx_K, wslice(sm.wbuf, buf ^ 1, slice_floats<WBF16>(ph.nx_rpc * ph.nx_K)), &sm.mbar[buf ^ 1],
                                            cta, ph.nx_rpc);
                wait_weights(&sm.mbar[buf], (g_idx >> 1) & 1, mp.error_flag);   // on a timeout the error flag ends the loop at the next token
                MEGA_TRACE(3);
                for (int rep = tracing ? 0 : 1; rep < 2; ++rep) {      // trace mode: a cold pass (stamp 12) and a warm one; idempotent, the
                    int j = 0;                                          // residual operand was fetched before either pass stores
                    if (rep == 1) MEGA_TRACE(12);
#pragma unroll 1
                    for (int n = r0 + warp; n < r1; n += MEGA_WARPS, ++j) {
                        const bool pre = j < OPS_ROWS;
                        const float bias_v = __shfl_sync(0xffffffffu, bias_pref, (j * MEGA_NB) & 31);
                        const float r_v = __shfl_sync(0xffffffffu, r_pref, (j * MEGA_NB + (lane < MEGA_NB ? lane : 0)) & 31);
                        gemv_row<MEGA_NB, false, false, WBF16>(ph.g, n, gemv_wrow<WBF16>(wslice(sm.wbuf, buf, slice_floats<WBF16>(ph.rpc * ph.g.K)), (long long)(n - r0) * ph.g.K),
                                                               sm.u.xs, 0, lane, cur_pos, pre, bias_v, r_v,
                                                 (tracing && warp == 0 && rep == 1 && j == 0) ? &mp.trace[(long long)pi * MEGA_TRACE_SLOTS + 13] : nullptr);
                    }
                }
                ++g_idx;
            } else if (ph.kind == 1) {
                const DecAttnParams& a = ph.a;
                const int L = a.fixed_len > 0 ? a.fixed_len : cur_pos + 1;
                const int units = a.rows * a.H * a.n_splits;
                for (int u = cta; u < units; u += G) {
                    int s, h, r;
                    unit_of(ph, u, s, h, r);
                    const int slot = a.row_slot ? sm.ctrl[4 + r] : r;
                    if (!(areg_valid && u == cta)) decode_attention_load<MEGA_WARPS>(a, s, h, r, slot, L, P, tid, areg);
                    decode_attention_body<MEGA_WARPS>(a, s, h, r, slot, L, P, sm.u.attn.sc, sm.u.attn.red, sm.u.attn.stat, tid, areg,
                                                      tracing ? &mp.trace[(long long)pi * MEGA_TRACE_SLOTS + 6] : nullptr);
                    __syncthreads();
                }
            } else {
                if (cta < sm.sample_params.cfg->B) sample_body<SAMPLE_THREADS>(sm.sample_params, cta, sm.u.sample);
            }
            MEGA_TRACE(11);
            asm volatile("cp.async.wait_all;" ::: "memory");
            __syncthreads();                              // this CTA's stores are done; the next descriptor has landed
            MEGA_TRACE(4);
            sync_target += G;
            grid_arrive(mp.sync_counter);
            phase_prologue(sm.phase[cur ^ 1]);
            grid_wait(mp.sync_counter, sync_target, mp.error_flag);
            MEGA_TRACE(5);
            cur ^= 1;
        }
    }
    // drain the weight prefetch that is still in flight so no bulk copy outlives the CTA
    wait_weights(&sm.mbar[g_idx & 1], (g_idx >> 1) & 1, mp.error_flag);
}

}  // namespace

size_t mega_smem_bytes() { return sizeof(MegaSmem) + 128; }

template <bool WBF16>
static int launch_megakernel_impl(const MegaParams& mp, int grid, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        MB_CUDA_CHECK(cudaFuncSetAttribute(decode_megakernel<1, false, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem_bytes()));
        MB_CUDA_CHECK(cudaFuncSetAttribute(decode_megakernel<2, false, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem_bytes()));
        MB_CUDA_CHECK(cudaFuncSetAttribute(decode_megakernel<1, true, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem_bytes()));
        MB_CUDA_CHECK(cudaFuncSetAttribute(decode_megakernel<2, true, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem_bytes()));
        int per_sm = 0;
        MB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decode_megakernel<2, true, WBF16>, MEGA_THREADS, mega_smem_bytes()));
        MB_REQUIRE(per_sm >= 1, "megakernel does not fit on an SM");
        configured = true;
    }
    MB_REQUIRE(mp.sample.rows >= 1 && mp.sample.rows <= MEGA_NB_MAX, "megakernel handles 1 or 2 decoder rows");
    MegaParams p = mp;
    void* args[] = {&p};
    const void* fn = mp.trace ? (mp.sample.rows == 1 ? (const void*)decode_megakernel<1, true, WBF16> : (const void*)decode_megakernel<2, true, WBF16>)
                              : (mp.sample.rows == 1 ? (const void*)decode_megakernel<1, false, WBF16> : (const void*)decode_megakernel<2, false, WBF16>);
    MB_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(MEGA_THREADS), args, mega_smem_bytes(), stream));
    ++g_launch_count;
    if (WBF16) ++g_wbf16_launch_count;
    return 0;
}

int launch_megakernel(const MegaParams& mp, int grid, cudaStream_t stream, bool w_bf16) {
    return w_bf16 ? launch_megakernel_impl<true>(mp, grid, stream) : launch_megakernel_impl<false>(mp, grid, stream);
}

}  // namespace mb200
