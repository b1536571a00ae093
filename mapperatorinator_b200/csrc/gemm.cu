// fp32 GEMM with fused epilogues:  C = R + gate * ( act(A . W^T + bias) * alpha )
//
// Serves every dense projection of the hot path at fp32 accuracy (bit-exact-greedy parity needs fp32-grade sums;
// the reference's CPU path is fp32, SURVEY F4): encoder_embedder, conv1/conv2 (as im2col-free GEMMs over a padded
// token-major buffer, see RowMap), Whisper q/k/v/out/fc1/fc2 in encoder + prefill, DiT qkv/out/fc1/fc2/adaLN.
//   A: [M, K] via RowMap (K contiguous), W: [N, K] row-major (torch Linear layout), C/R: [M, N] via RowMap.
// Tile 128x128x16, 256 threads, 8x8 micro-tile, double-buffered shared memory with register prefetch.
#include <algorithm>
#include <cstdlib>
#include "common.cuh"
#include "kernels.h"

namespace mb200 {

namespace {

constexpr int BM = 128, BN = 128, BK = 16, PAD = 4;

// MH 64-row halves per tile: 2 = the 128x128 tile, 1 = a 64x128 tile for launches of at most one 128-row tile, whose padding rows
// would otherwise cost as many FMAs as the real ones.  Each output's sum runs over the same k in the same order either way.
template <int MH>
__global__ void __launch_bounds__(256, 2) gemm_f32_kernel(GemmParams p) {
    constexpr int TM = 64 * MH;
    __shared__ __align__(16) float As[2][BK][TM + PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + PAD];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const long long m0 = (long long)blockIdx.y * TM;
    const int n0 = blockIdx.x * BN;

    // global->smem loader coordinates: two rows per operand per thread, one float4 along K each
    const int lrow = tid >> 2;           // 0..63
    const int lk = (tid & 3) * 4;        // 0,4,8,12
    const float* a_ptr[2];
    const float* w_ptr[2];
    bool a_ok[2], w_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        long long m = m0 + lrow + h * 64;
        a_ok[h] = h < MH && m < p.M;
        a_ptr[h] = a_ok[h] ? p.A.row(p.m_base + m) : p.A.ptr;
        int n = n0 + lrow + h * 64;
        w_ok[h] = n < p.N;
        w_ptr[h] = p.W + (long long)(w_ok[h] ? n : 0) * p.ldw;
    }

    float acc[4 * MH][8];
#pragma unroll
    for (int i = 0; i < 4 * MH; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    float4 ra[2], rw[2];
    const int k_lo_ = p.splitk > 1 ? blockIdx.z * p.k_per_split : 0;
    const int k_hi_ = p.splitk > 1 ? min(p.K, k_lo_ + p.k_per_split) : p.K;
    auto gload = [&](int k0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int k = k_lo_ + k0 + lk;
            if (h < MH) ra[h] = (a_ok[h] && k < k_hi_) ? __ldg(reinterpret_cast<const float4*>(a_ptr[h] + k)) : make_float4(0, 0, 0, 0);
            rw[h] = (w_ok[h] && k < k_hi_) ? __ldg(reinterpret_cast<const float4*>(w_ptr[h] + k)) : make_float4(0, 0, 0, 0);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int r = lrow + h * 64;
            if (h < MH) { As[buf][lk + 0][r] = ra[h].x; As[buf][lk + 1][r] = ra[h].y; As[buf][lk + 2][r] = ra[h].z; As[buf][lk + 3][r] = ra[h].w; }
            Bs[buf][lk + 0][r] = rw[h].x; Bs[buf][lk + 1][r] = rw[h].y; Bs[buf][lk + 2][r] = rw[h].z; Bs[buf][lk + 3][r] = rw[h].w;
        }
    };

    const int k_lo = p.splitk > 1 ? blockIdx.z * p.k_per_split : 0;
    const int k_hi = p.splitk > 1 ? min(p.K, k_lo + p.k_per_split) : p.K;
    const int nk = (k_hi - k_lo + BK - 1) / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            float4 a1 = MH == 2 ? *reinterpret_cast<const float4*>(&As[buf][k][64 * (MH - 1) + ty * 4]) : a0;
            float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 4 * MH; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }

    // ---- epilogue --------------------------------------------------------------------------------------------------
    if (p.splitk > 1) {      // raw partial sums; gemm_splitk_reduce_kernel finishes the job
#pragma unroll
        for (int i = 0; i < 4 * MH; ++i) {
            long long m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
            if (m >= p.M) continue;
            float* wrow = p.splitk_ws + ((long long)blockIdx.z * p.M + m) * p.N;
#pragma unroll
            for (int jh = 0; jh < 2; ++jh)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    int nn = n0 + jh * 64 + tx * 4 + j;
                    if (nn < p.N) wrow[nn] = acc[i][jh * 4 + j];
                }
        }
        return;
    }
#pragma unroll
    for (int i = 0; i < 4 * MH; ++i) {
        long long m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (m >= p.M) continue;
        float* crow = p.C.row(p.m_base + m);
        const float* rrow = p.R.ptr ? p.R.row(p.m_base + m) : nullptr;
        const float* grow = p.gate ? p.gate + ((p.m_base + m) / p.gate_rpb) * p.gate_ld : nullptr;
#pragma unroll
        for (int jh = 0; jh < 2; ++jh) {
            int n = n0 + jh * 64 + tx * 4;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int nn = n + j;
                if (nn >= p.N) continue;
                float v = acc[i][jh * 4 + j];
                if (p.bias) v += __ldg(p.bias + nn);
                v = apply_act(v, p.act) * p.alpha;
                if (grow) v *= __ldg(grow + nn);
                if (rrow) v += rrow[nn];
                crow[nn] = v;
            }
        }
    }
}

__global__ void __launch_bounds__(256) gemm_splitk_reduce_kernel(GemmParams p) {
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= (long long)p.M * p.N) return;
    const long long m = idx / p.N;
    const int n = (int)(idx - m * p.N);
    float v = p.splitk_ws[m * p.N + n];
    for (int z = 1; z < p.splitk; ++z) v += p.splitk_ws[((long long)z * p.M + m) * p.N + n];   // fixed order: ((p0 + p1) + p2) + ...
    if (p.bias) v += __ldg(p.bias + n);
    v = apply_act(v, p.act) * p.alpha;
    if (p.gate) v *= __ldg(p.gate + ((p.m_base + m) / p.gate_rpb) * p.gate_ld + n);
    if (p.R.ptr) v += p.R.row(p.m_base + m)[n];
    p.C.row(p.m_base + m)[n] = v;
}

}  // namespace

// ---- per-engine scratch ------------------------------------------------------------------------------------------------
int GemmCtx::reserve(size_t splitk_need, size_t a_split_need) {
    auto grow = [&](float*& ptr, size_t& have, size_t need) -> int {
        if (need <= have) return 0;
        MB_REQUIRE(!frozen, "GEMM scratch is referenced by a captured CUDA graph and cannot grow (reserve the largest shape before capturing)");
        if (ptr) MB_CUDA_CHECK(cudaFree(ptr));
        ptr = nullptr; have = 0;
        MB_CUDA_CHECK(cudaMalloc(&ptr, need));
        have = need;
        return 0;
    };
    int s = grow(splitk_ws, splitk_bytes, splitk_need);
    if (s) return s;
    s = grow(a_split, a_split_bytes, a_split_need);
    if (s) return s;
    if (!tc_err) { MB_CUDA_CHECK(cudaMalloc(&tc_err, 4)); MB_CUDA_CHECK(cudaMemset(tc_err, 0, 4)); }
    return 0;
}

int GemmCtx::error() {
    if (!tc_err) return 0;
    int h = 0;
    cudaMemcpy(&h, tc_err, 4, cudaMemcpyDeviceToHost);
    return h;
}

void GemmCtx::destroy() {
    for (auto& kv : mirrors) cudaFree(const_cast<float*>(kv.second.hi));      // hi and lo share one allocation
    mirrors.clear();
    if (splitk_ws) cudaFree(splitk_ws);
    if (a_split) cudaFree(a_split);
    if (tc_err) cudaFree(tc_err);
    splitk_ws = a_split = nullptr; tc_err = nullptr; splitk_bytes = a_split_bytes = 0; frozen = false;
}

GemmCtx* default_gemm_ctx() {
    static GemmCtx ctx;
    static bool init = false;
    if (!init) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&ctx.num_sms, cudaDevAttrMultiProcessorCount, dev);
        init = true;
    }
    return &ctx;
}

// S of an (N, K) problem on the SIMT path: the split that fills the machine when M is one 128-row tile (decoder prefill, DiT
// conditioning) — chosen from N and K only, so a row's sum does not depend on how many rows share the launch.
int gemm_splits_simt(int N, int K, int num_sms, int* k_per_split) {
    const int tiles_n = (N + BN - 1) / BN;
    int splits = 1;
    if (tiles_n * 2 <= num_sms && K >= 64) splits = std::max(1, std::min((num_sms + tiles_n - 1) / tiles_n, K / 32));
    const int kps = ((K + splits - 1) / splits + BK - 1) / BK * BK;
    splits = (K + kps - 1) / kps;
    *k_per_split = kps;
    return splits;
}

int launch_splitk_reduce(const GemmParams& q, cudaStream_t stream) {
    gemm_splitk_reduce_kernel<<<(unsigned)(((long long)q.M * q.N + 255) / 256), 256, 0, stream>>>(q);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

int launch_gemm(const GemmParams& p, cudaStream_t stream, GemmCtx* ctx) {
    MB_REQUIRE(ctx != nullptr, "GEMM needs its engine's scratch context");
    MB_REQUIRE(p.K % 4 == 0, "GEMM K must be a multiple of 4 (float4 loads)");
    MB_REQUIRE(p.A.ld % 4 == 0 && p.ldw % 4 == 0, "GEMM operand row strides must be multiples of 4 floats");
    MB_REQUIRE((reinterpret_cast<uintptr_t>(p.A.ptr) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.W) & 15) == 0,
               "GEMM operands must be 16-byte aligned");
    if (p.M <= 0 || p.N <= 0) return 0;
    if (tc_gemm_eligible(p, ctx)) return launch_gemm_tc(p, stream, ctx);      // tensor cores (3xTF32)
    int kps = 0;
    const int splits = gemm_splits_simt(p.N, p.K, ctx->num_sms, &kps);
    const int tiles_n = (p.N + BN - 1) / BN;
    const bool half = p.M <= BM;      // one row tile: 64-row tiles halve the padded FMAs (and double the CTAs when M > 64)
    const int tm = half ? BM / 2 : BM;
    if (splits == 1) {
        dim3 grid(tiles_n, (unsigned)((p.M + tm - 1) / tm));
        if (half) gemm_f32_kernel<1><<<grid, 256, 0, stream>>>(p);
        else gemm_f32_kernel<2><<<grid, 256, 0, stream>>>(p);
        MB_LAUNCH_CHECK();
        ++g_launch_count;
        return 0;
    }
    // grid split; rows are processed in slices whose S partial planes fit the workspace (slicing M does not touch the arithmetic)
    const size_t row_bytes = (size_t)splits * p.N * sizeof(float);
    if (row_bytes * (size_t)p.M > ctx->splitk_bytes && !ctx->frozen) {
        const int s = ctx->reserve(std::max(row_bytes * (size_t)std::min(p.M, 2048), (size_t)64 << 20), 0);
        if (s) return s;
    }
    MB_REQUIRE(ctx->splitk_bytes >= row_bytes * BM, "split-K workspace smaller than one row tile");
    const long long rows_per_pass = std::min<long long>(p.M, (long long)(ctx->splitk_bytes / row_bytes) / BM * BM);
    for (long long m0 = 0; m0 < p.M; m0 += rows_per_pass) {
        GemmParams q = p;
        q.m_base = p.m_base + m0;
        q.M = (int)std::min<long long>(rows_per_pass, p.M - m0);
        q.splitk_ws = ctx->splitk_ws; q.splitk = splits; q.k_per_split = kps; q.split_mode = 1;
        const dim3 grid(tiles_n, (unsigned)((q.M + tm - 1) / tm), splits);
        if (half) gemm_f32_kernel<1><<<grid, 256, 0, stream>>>(q);
        else gemm_f32_kernel<2><<<grid, 256, 0, stream>>>(q);
        MB_LAUNCH_CHECK();
        ++g_launch_count;
        const int s = launch_splitk_reduce(q, stream);
        if (s) return s;
    }
    return 0;
}

}  // namespace mb200
