// Per-token scoring of a teacher-forced pass (MaiMod, `Processor.ai_mod`, osuT5/osuT5/inference/processor.py:519-525):
// for each logits row z of a chunk of vocabulary-projection rows, with p = softmax(z) in fp32 and y the next given token,
//   entropy   = -sum_v p_v * log2(p_v + 1e-10)
//   surprisal = -log2(p_y + 1e-10)
//   relative  = entropy > 0 ? surprisal / entropy : 0
//   suggested = argmax_v z_v (lowest index among equal maxima, as torch.argmax)
// written at the index of the scored token (row t of a sequence scores token t + 1).
//
// One CTA per row, 256 threads, the row held in registers (at most 16 values per thread: V <= 4096), so the row is read from
// HBM exactly once; the three block reductions (max / arg-max, sum of exp, entropy sum) run on the register copy.
#include "common.cuh"
#include "kernels.h"

namespace mb200 {
namespace {

constexpr int SC_THREADS = 256, SC_WARPS = SC_THREADS / 32, SC_PER_THREAD = 4096 / SC_THREADS;

__device__ __forceinline__ void argmax_merge(float& m, int& i, float om, int oi) {
    if (om > m || (om == m && oi < i)) { m = om; i = oi; }
}

__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();                       // red[] may still be read by the previous reduction
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float s = red[0];
#pragma unroll
    for (int w = 1; w < SC_WARPS; ++w) s += red[w];
    return s;
}

}  // namespace

// outside the anonymous namespace so the profiler shows one stable name: mb200::score_rows_kernel
__global__ void __launch_bounds__(SC_THREADS) score_rows_kernel(ScoreParams p) {
    __shared__ float red[SC_WARPS];
    __shared__ int redi[SC_WARPS];
    const long long r = p.row0 + blockIdx.x;              // global row = b * L + t
    const int tid = threadIdx.x;
    const float* z = p.logits + (long long)blockIdx.x * p.V;

    float v[SC_PER_THREAD];
    float m = -INFINITY;
    int mi = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < SC_PER_THREAD; ++k) {
        const int c = k * SC_THREADS + tid;
        v[k] = c < p.V ? __ldg(z + c) : -INFINITY;
        if (c < p.V && v[k] > m) { m = v[k]; mi = c; }   // ascending c: the first maximum of this thread's values
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        argmax_merge(m, mi, om, oi);
    }
    if ((tid & 31) == 0) { red[tid >> 5] = m; redi[tid >> 5] = mi; }
    __syncthreads();
    m = red[0]; mi = redi[0];
#pragma unroll
    for (int w = 1; w < SC_WARPS; ++w) argmax_merge(m, mi, red[w], redi[w]);

    float s = 0.f;
#pragma unroll
    for (int k = 0; k < SC_PER_THREAD; ++k) {
        v[k] = k * SC_THREADS + tid < p.V ? expf(v[k] - m) : 0.f;
        s += v[k];
    }
    const float sum = block_sum(s, red);

    const int t = (int)(r % p.L);
    const bool has_target = t + 1 < p.L;
    const long long y = has_target ? p.ids[r + 1] : -1;
    float e = 0.f, py = 0.f;
#pragma unroll
    for (int k = 0; k < SC_PER_THREAD; ++k) {
        const int c = k * SC_THREADS + tid;
        if (c < p.V) {
            const float pv = v[k] / sum;                   // torch softmax: exp(z - max) / sum
            e += pv * log2f(pv + 1e-10f);
            if (c == y) py = pv;
        }
    }
    const float entropy = -block_sum(e, red);

    if (t == 0 && tid == 0) {                              // column 0 has no logits row
        p.entropy[r] = NAN; p.surprisal[r] = NAN; p.relative[r] = NAN; p.suggested[r] = -1;
    }
    if (!has_target) return;
    if (tid == 0) {
        p.entropy[r + 1] = entropy;
        p.suggested[r + 1] = mi;
        if (y >= p.V) { p.surprisal[r + 1] = NAN; p.relative[r + 1] = NAN; }   // an input-only id has no output probability
    }
    if (y < p.V && tid == (int)(y % SC_THREADS)) {
        const float sp = -log2f(py + 1e-10f);
        p.surprisal[r + 1] = sp;
        p.relative[r + 1] = entropy > 0.f ? sp / entropy : 0.f;
    }
}

int launch_score_rows(const ScoreParams& p, int rows, cudaStream_t stream) {
    MB_REQUIRE(p.V >= 1 && p.V <= SC_THREADS * SC_PER_THREAD, "scoring holds a logits row in registers (V <= 4096)");
    if (rows <= 0) return 0;
    score_rows_kernel<<<rows, SC_THREADS, 0, stream>>>(p);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

}  // namespace mb200
