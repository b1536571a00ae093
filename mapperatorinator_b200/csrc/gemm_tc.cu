// Tensor-core GEMM for the dense phases (encoder layers, conv stem, DiT blocks): Hopper wgmma (kind tf32) with fp32-grade accuracy
// through the 3xTF32 split
//        A.W^T  ~=  Ahi.Whi^T + Ahi.Wlo^T + Alo.Whi^T ,   x = xhi + xlo,  xhi = rn_tf32(x), xlo = rn_tf32(x - xhi).
// Both parts are rounded to nearest tf32 (cvt.rna) — weights once at load, activations by a tiny elementwise pass — because the
// tensor core would otherwise TRUNCATE the low 13 bits, and truncation bias adds up linearly over K.  Accumulation is fp32 in registers.
// The error vs fp64 is ~1e-6 relative — the same order as an fp32 FMA chain of that length — which is what bit-exact greedy decoding
// against the fp32 reference needs; plain TF32 (1e-3) flips tokens.
//
// Structure (one 128x128 output tile per CTA, 384 threads = 3 warpgroups):
//   warpgroup 0, thread 0 : TMA producer — 4 tiles per k-block (A, Alo, W, Wlo; 128 rows x 32 floats, SWIZZLE_128B) into a 3-stage ring
//   warpgroups 1, 2       : MMA + epilogue — warpgroup g owns output rows 64(g-1) .. +63: 12 x wgmma m64n128k8 per k-block into a
//                           64-register fp32 accumulator per thread; the stage is released (mbarrier, every consumer thread arrives)
//                           once the warpgroup's MMAs have completed.  Epilogue: accumulators -> shared memory (the idle pipeline
//                           stages) -> row by row with lane = column: bias / activation / gate / residual (same GemmParams epilogue
//                           as gemm.cu) and 128-byte coalesced loads and stores.
// A may be any RowMap (im2col-free conv over the padded buffer, batched rows) via a 3-D tensor map.
// Every wait is bounded: on a timeout the kernel sets an error flag and falls through, it can never hang the GPU.
#include <cuda.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <map>
#include <tuple>
#include <unordered_map>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace mb200 {

int g_tc_enabled = 1;

namespace {

constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 32, TC_STAGES = 3, TC_THREADS = 384, TC_CONSUMERS = 256;
constexpr int TC_TILE_BYTES = TC_BM * TC_BK * 4;          // 16 KB
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;         // A, Alo, W, Wlo
constexpr int TC_EPI_LD = TC_BN + 8;                      // epilogue staging row (floats): the fragment's float2 stores are conflict-free
static_assert(TC_BM * TC_EPI_LD * 4 <= TC_STAGES * TC_STAGE_BYTES, "epilogue staging fits the pipeline stages");

struct TcBarriers {
    unsigned long long full[TC_STAGES];
    unsigned long long empty[TC_STAGES];
};

__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool bar_wait(unsigned long long* bar, unsigned parity, int* err) {
    for (long long spin = 0; spin < (1ll << 22); ++spin) {
        unsigned ok;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
        if (ok) return true;
    }
    atomicExch(err, 3);
    return false;
}

__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_alo,
                   const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo, GemmParams p, int a_rpb, int* err) {
    extern __shared__ unsigned char tc_smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
    TcBarriers* bars = reinterpret_cast<TcBarriers*>(smem + TC_STAGES * TC_STAGE_BYTES);
    const int tid = threadIdx.x;
    const int n0 = blockIdx.x * TC_BN;
    const long long m0 = (long long)blockIdx.y * TC_BM;
    const int nkb_all = (p.K + TC_BK - 1) / TC_BK;
    // Split-K (kernels.h): k-range z = k-blocks [z*kpb, (z+1)*kpb) is summed on its own.  Grid split (under-filled grids): CTA
    // blockIdx.z owns range z and stores raw partials, gemm.cu's reduce kernel adds them in order.  In-tile split (large M): this CTA
    // walks every range, each range accumulating from zero; the running sum adds the range results in the same order.  Same
    // partial sums, same additions, same bits.
    const int kpb = p.splitk > 1 ? p.k_per_split / TC_BK : nkb_all;
    const bool grid_split = p.split_mode == 1, tile_split = p.split_mode == 2;
    const int kb0 = grid_split ? blockIdx.z * kpb : 0;
    const int nkb = grid_split ? max(0, min(nkb_all - kb0, kpb)) : nkb_all;

    if (tid == 0) {
        for (int s = 0; s < TC_STAGES; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&bars->full[s])));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(&bars->empty[s])), "r"(TC_CONSUMERS));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (tid < 128) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");      // the producer needs few registers; the accumulators get them
        if (tid == 0) {
            const int a_b = a_rpb > 0 ? (int)(m0 / a_rpb) : 0;
            const int a_t = a_rpb > 0 ? (int)(m0 - (long long)a_b * a_rpb) : (int)m0;
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % TC_STAGES;
                const unsigned ph = (kb / TC_STAGES) & 1;
                if (!bar_wait(&bars->empty[s], ph ^ 1, err)) break;
                unsigned char* st = smem + s * TC_STAGE_BYTES;
                const unsigned fb = s32(&bars->full[s]);
                asm volatile("{ .reg .b64 t; mbarrier.arrive.expect_tx.shared::cta.b64 t, [%0], %1; }" ::"r"(fb), "r"(TC_STAGE_BYTES) : "memory");
                const int k0 = (kb0 + kb) * TC_BK;
                asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                             ::"r"(s32(st)), "l"(&map_a), "r"(k0), "r"(a_t), "r"(a_b), "r"(fb) : "memory");
                asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                             ::"r"(s32(st + TC_TILE_BYTES)), "l"(&map_alo), "r"(k0), "r"(a_t), "r"(a_b), "r"(fb) : "memory");
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                             ::"r"(s32(st + 2 * TC_TILE_BYTES)), "l"(&map_w), "r"(k0), "r"(n0), "r"(fb) : "memory");
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                             ::"r"(s32(st + 3 * TC_TILE_BYTES)), "l"(&map_wlo), "r"(k0), "r"(n0), "r"(fb) : "memory");
            }
        }
        return;      // the bulk copies in flight complete on the mbarriers of this (still resident) CTA
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int ct = tid - 128;                          // consumer thread 0..255
    const int cg = ct >> 7;                            // consumer warpgroup: output rows 64 cg .. +63
    float acc[64], sum[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc[i] = 0.f; sum[i] = 0.f; }
#pragma unroll 1
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % TC_STAGES;
        const unsigned ph = (kb / TC_STAGES) & 1;
        if (!bar_wait(&bars->full[s], ph, err)) break;
        const unsigned base = s32(smem + s * TC_STAGE_BYTES);
        const unsigned a_off = (unsigned)cg * (64 * 128);                                 // 64 rows of 128 bytes
        const int z = tile_split ? kb / kpb : 0, kr = tile_split ? kb - z * kpb : kb;      // k-range and position inside it
        gmma_fence_regs(acc);
        gmma_fence();
#pragma unroll
        for (int sub = 0; sub < TC_BK / 8; ++sub) {
            const unsigned off = sub * 32;       // 8 tf32 = 32 bytes along K inside the 128-byte swizzle atom
            const unsigned long long a_hi = gmma_desc(base + a_off + off), a_lo = gmma_desc(base + TC_TILE_BYTES + a_off + off);
            const unsigned long long w_hi = gmma_desc(base + 2 * TC_TILE_BYTES + off), w_lo = gmma_desc(base + 3 * TC_TILE_BYTES + off);
            gmma_m64n128k8_ss(acc, a_hi, w_hi, (kr > 0 || sub > 0) ? 1u : 0u);
            gmma_m64n128k8_ss(acc, a_hi, w_lo, 1u);
            gmma_m64n128k8_ss(acc, a_lo, w_hi, 1u);
        }
        gmma_commit();
        gmma_wait<0>();
        gmma_fence_regs(acc);
        asm volatile("{ .reg .b64 t; mbarrier.arrive.shared::cta.b64 t, [%0]; }" ::"r"(s32(&bars->empty[s])) : "memory");
        if (kb == nkb - 1 || (tile_split && kr == kpb - 1)) {                            // a k-range is complete: ((r0 + r1) + r2) + r3
            if (z == 0) {
#pragma unroll
                for (int i = 0; i < 64; ++i) sum[i] = acc[i];
            } else {
#pragma unroll
                for (int i = 0; i < 64; ++i) sum[i] += acc[i];
            }
        }
    }

    // Epilogue.  Both consumer warpgroups are past their last MMA (every TMA load they waited for has landed), so the pipeline
    // stages are free: the tile goes through shared memory [128][TC_EPI_LD] and is then walked row by row with lane = column.
    asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory");
    float* stg = reinterpret_cast<float*>(smem);
    {
        const int w = (ct >> 5) & 3, lane = ct & 31, gid = lane >> 2, tig = lane & 3;
        const int r = cg * 64 + w * 16 + gid;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int c = 8 * j + 2 * tig;
            *reinterpret_cast<float2*>(stg + r * TC_EPI_LD + c) = make_float2(sum[4 * j], sum[4 * j + 1]);
            *reinterpret_cast<float2*>(stg + (r + 8) * TC_EPI_LD + c) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
        }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory");
    const int lane = ct & 31, cw = ct >> 5;            // consumer warp cw stores rows 16 cw .. +15
    const bool has_r = !grid_split && p.R.ptr != nullptr, has_g = !grid_split && p.gate != nullptr;
    float bias_v[TC_BN / 32];
#pragma unroll
    for (int c = 0; c < TC_BN / 32; ++c) {
        const int n = n0 + 32 * c + lane;
        bias_v[c] = (!grid_split && p.bias && n < p.N) ? __ldg(p.bias + n) : 0.f;
    }
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int row = cw * 16 + rr;
        const long long m = m0 + row;
        if (m >= p.M) break;
        float* crow = grid_split ? p.splitk_ws + ((long long)blockIdx.z * p.M + m) * p.N : p.C.row(m);
        const float* rrow = has_r ? p.R.row(m) : nullptr;
        const float* grow = has_g ? p.gate + (m / p.gate_rpb) * p.gate_ld : nullptr;
#pragma unroll
        for (int c = 0; c < TC_BN / 32; ++c) {
            const int n = n0 + 32 * c + lane;
            if (n >= p.N) continue;
            float x = stg[row * TC_EPI_LD + 32 * c + lane];
            if (!grid_split) {
                if (p.bias) x += bias_v[c];
                x = apply_act(x, p.act) * p.alpha;
                if (has_g) x *= __ldg(grow + n);
                if (has_r) x += rrow[n];
            }
            crow[n] = x;
        }
    }
}

// x = hi + lo with hi = round-to-nearest tf32(x) and lo = round-to-nearest tf32(x - hi).  Rounding (not truncating) both parts
// matters: truncation errors all point toward zero and add up linearly over K (measured 8e-6 relative at K = 3072, 70x the
// fp32 FMA kernel); rounded parts leave unbiased ~2^-22 errors that grow like sqrt(K).
__device__ __forceinline__ float rn_tf32(float x) {
    unsigned u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__global__ void tf32_split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, long long n4) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 h, l;
    h.x = rn_tf32(v.x); h.y = rn_tf32(v.y); h.z = rn_tf32(v.z); h.w = rn_tf32(v.w);
    l.x = rn_tf32(v.x - h.x); l.y = rn_tf32(v.y - h.y); l.z = rn_tf32(v.z - h.z); l.w = rn_tf32(v.w - h.w);
    reinterpret_cast<float4*>(hi)[i] = h;
    reinterpret_cast<float4*>(lo)[i] = l;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// [rows x K] fp32, K contiguous, optional batching: dims {K, rpb, batches}; box {32, 128, 1}; 128-byte swizzle; OOB reads give 0
int make_map(CUtensorMap* out, const float* base, long long K, long long rows_per_batch, long long ld, long long batches, long long bstride,
             int rank) {
    EncodeTiledFn fn = encode_fn();
    MB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows_per_batch, (cuuint64_t)batches};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)(bstride > 0 ? bstride : ld * rows_per_batch) * 4};
    cuuint32_t box[3] = {TC_BK, TC_BM, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return 0;
}

}  // namespace

// S of an (N, K) problem on the tensor-core path: the split that fills the machine for ONE encoder window (M = 512 rows = 4 row
// tiles), at least 8 k-blocks per range, at most 4 ranges.  A function of N and K only.
int gemm_splits_tc(int N, int K, int num_sms, int* k_per_split) {
    const int tiles_ref = 4 * ((N + TC_BN - 1) / TC_BN), nkb = (K + TC_BK - 1) / TC_BK;
    int splits = std::max(1, std::min({4, num_sms / std::max(1, tiles_ref), nkb / 8}));
    const int kpb = (nkb + splits - 1) / splits;                  // k-blocks per range
    splits = (nkb + kpb - 1) / kpb;                               // no empty range
    *k_per_split = kpb * TC_BK;
    return splits;
}

// One-time self test of the tensor-core path against a host fp64 product (grid split, in-tile split and unsplit shapes).  If the
// wgmma pipeline misbehaves on this driver / device the path is switched off LOUDLY and every GEMM stays on the fp32 SIMT kernel.
static int g_tc_tested = 0;
static void tc_self_test() {
    g_tc_tested = 1;
    GemmCtx ctx;
    ctx.num_sms = default_gemm_ctx()->num_sms;
    bool all_ok = true;
    const int shapes[3][3] = {{512, 128, 96}, {512, 128, 1024}, {2048, 256, 1024}};      // unsplit, grid split, in-tile split
    for (int t = 0; t < 3 && all_ok; ++t) {
        const int M = shapes[t][0], N = shapes[t][1], K = shapes[t][2];
        std::vector<float> a((size_t)M * K), w((size_t)N * K), c((size_t)M * N);
        unsigned s = 12345u + t;
        auto rnd = [&]() { s = s * 1664525u + 1013904223u; return (float)((s >> 8) & 0xFFFF) / 32768.0f - 1.0f; };
        for (auto& v : a) v = rnd();
        for (auto& v : w) v = rnd();
        float *da = nullptr, *dw = nullptr, *dc = nullptr;
        bool ok = cudaMalloc(&da, a.size() * 4) == cudaSuccess && cudaMalloc(&dw, w.size() * 4) == cudaSuccess && cudaMalloc(&dc, c.size() * 4) == cudaSuccess;
        if (ok) {
            cudaMemcpy(da, a.data(), a.size() * 4, cudaMemcpyHostToDevice);
            cudaMemcpy(dw, w.data(), w.size() * 4, cudaMemcpyHostToDevice);
            GemmParams g{};
            g.A = plain_map(da, K); g.W = dw; g.ldw = K; g.C = plain_map(dc, N); g.alpha = 1.f; g.gate_rpb = 1; g.M = M; g.N = N; g.K = K;
            ok = ctx.register_weight(dw, (long long)N * K) == 0 && launch_gemm_tc(g, nullptr, &ctx) == 0 && cudaDeviceSynchronize() == cudaSuccess &&
                 ctx.error() == 0;
            if (ok) {
                cudaMemcpy(c.data(), dc, c.size() * 4, cudaMemcpyDeviceToHost);
                double worst = 0;
                for (int m = 0; m < M; m += 37)
                    for (int n = 0; n < N; n += 5) {
                        double r = 0;
                        for (int k = 0; k < K; ++k) r += (double)a[(size_t)m * K + k] * (double)w[(size_t)n * K + k];
                        worst = std::max(worst, std::fabs(r - (double)c[(size_t)m * N + n]));
                    }
                ok = worst < 1e-3;
            }
        }
        if (da) cudaFree(da);
        if (dw) cudaFree(dw);
        if (dc) cudaFree(dc);
        all_ok = all_ok && ok;
    }
    ctx.destroy();
    if (!all_ok) {
        g_tc_enabled = 0;
        fprintf(stderr, "[mapperatorinator_b200] WARNING: wgmma GEMM self-test FAILED — tensor-core path disabled, using the fp32 SIMT GEMM\n");
        cudaGetLastError();
    }
}

bool tc_gemm_eligible(const GemmParams& p, GemmCtx* ctx) {
    if (g_tc_enabled && !g_tc_tested) tc_self_test();
    if (!g_tc_enabled || p.m_base != 0) return false;
    if (p.M < 512 || p.N < 64 || p.K < 32 || p.K % 4 != 0) return false;
    if (ctx->mirrors.find(p.W) == ctx->mirrors.end()) return false;
    if (p.A.rpb != 0 && (p.A.rpb % TC_BM) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(p.A.ptr) & 15) || (reinterpret_cast<uintptr_t>(p.W) & 15) || (p.A.ld % 4) || (p.ldw % 4)) return false;
    if (p.A.rpb != 0 && (p.A.bstride % 4)) return false;
    return true;
}

int launch_gemm_tc(const GemmParams& p, cudaStream_t stream, GemmCtx* ctx) {
    const Tf32Mirror wm = ctx->mirrors.at(p.W);
    // extent of the buffer A rows live in (rows may overlap: im2col-free conv) and its lo mirror
    const long long batches = p.A.rpb ? (p.M + p.A.rpb - 1) / p.A.rpb : 1;
    const long long rpb = p.A.rpb ? p.A.rpb : p.M;
    const long long extent = (batches - 1) * (p.A.rpb ? p.A.bstride : 0) + (rpb - 1) * p.A.ld + p.K;
    const long long n4 = (extent + 3) / 4;
    dim3 grid((p.N + TC_BN - 1) / TC_BN, (unsigned)((p.M + TC_BM - 1) / TC_BM));
    GemmParams q = p;
    q.splitk = gemm_splits_tc(p.N, p.K, ctx->num_sms, &q.k_per_split);
    q.split_mode = 0; q.splitk_ws = nullptr;
    if (q.splitk > 1) {
        // grid split while the tiles alone would leave SMs idle, in-tile split otherwise: same bits either way
        const int tiles = (int)(grid.x * grid.y);
        q.split_mode = tiles * 4 <= ctx->num_sms * 3 ? 1 : 2;
    } else {
        q.splitk = 1;
    }
    {
        const int s = ctx->reserve(q.split_mode == 1 ? (size_t)q.splitk * p.M * p.N * sizeof(float) : 0, (size_t)n4 * 32);      // hi and lo halves
        if (s) return s;
    }
    if (q.split_mode == 1) { q.splitk_ws = ctx->splitk_ws; grid.z = q.splitk; }
    float* a_hi = ctx->a_split;
    float* a_lo = ctx->a_split + n4 * 4;
    tf32_split_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(p.A.ptr, a_hi, a_lo, n4);
    MB_LAUNCH_CHECK();
    CUtensorMap ma, mal, mw, mwl;
    MB_REQUIRE(make_map(&ma, a_hi, p.K, rpb, p.A.ld, batches, p.A.rpb ? p.A.bstride : 0, 3) == 0, "tensor map Ahi");
    MB_REQUIRE(make_map(&mal, a_lo, p.K, rpb, p.A.ld, batches, p.A.rpb ? p.A.bstride : 0, 3) == 0, "tensor map Alo");
    MB_REQUIRE(make_map(&mw, wm.hi, p.K, p.N, p.ldw, 1, 0, 2) == 0, "tensor map Whi");
    MB_REQUIRE(make_map(&mwl, wm.lo, p.K, p.N, p.ldw, 1, 0, 2) == 0, "tensor map Wlo");
    static bool configured = false;
    const int smem = TC_STAGES * TC_STAGE_BYTES + (int)sizeof(TcBarriers) + 1024;      // stages | barriers | alignment slack
    if (!configured) {
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemm_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    gemm_tf32x3_kernel<<<grid, TC_THREADS, smem, stream>>>(ma, mal, mw, mwl, q, p.A.rpb, ctx->tc_err);
    MB_LAUNCH_CHECK();
    g_launch_count += 2;
    if (q.split_mode == 1) return launch_splitk_reduce(q, stream);
    return 0;
}

void GemmCtx::unregister_weight(const float* w) {
    auto it = mirrors.find(w);
    if (it == mirrors.end()) return;
    cudaFree(const_cast<float*>(it->second.hi));      // hi and lo share one allocation
    mirrors.erase(it);
}

// tf32 hi / lo mirror of a weight matrix (called once per weight at load; the owner unregisters it before freeing the weight)
int GemmCtx::register_weight(const float* w, long long numel) {
    unregister_weight(w);      // a recycled device address must never inherit a stale mirror
    float* buf = nullptr;
    const long long n4 = (numel + 3) / 4;
    MB_CUDA_CHECK(cudaMalloc(&buf, (size_t)n4 * 32));
    tf32_split_kernel<<<(unsigned)((n4 + 255) / 256), 256>>>(w, buf, buf + n4 * 4, n4);
    MB_LAUNCH_CHECK();
    mirrors[w] = Tf32Mirror{buf, buf + n4 * 4};
    return 0;
}

}  // namespace mb200
