// Micro-benchmark behind the megakernel's phase design (DESIGN.md 4.1): what does one "everybody reads the activation vector
// right after a grid barrier" round trip cost, and why?
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o l2_hotspot_bench tools/l2_hotspot_bench.cu && ./l2_hotspot_bench
// One persistent cooperative grid (one CTA per SM x 512 threads).  Every iteration: producers write their slice of a 768-float vector,
// grid barrier (release add + acquire poll, as in decode_mega.cu), then warp 0 of every CTA loads the whole vector with ld.global.cg
// and we time issue -> data usable with clock64.  Modes:
//   0  all CTAs read the SAME freshly written vector                       (what LayerNorm staging does)
//   1  CTA c reads replica c % R of the freshly written vector (R = 8)     (producers store R copies)
//   2  all CTAs read the same vector, NOT rewritten (stays clean in L2)
//   3  every CTA reads its own private constant vector
// and each of them with / without a background bulk-copy weight stream (64 KB per CTA per iteration out of a 512 MB buffer).
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

constexpr int K = 768, R = 8, THREADS = 512, WB = 64 * 1024;

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// NC arrival counters (64 words apart: different L2 lines/slices); CTA c arrives on counter c % NC, lanes 0..NC-1 of warp 0 poll one each
__device__ __forceinline__ void grid_sync(unsigned* counter, unsigned round, int nc) {
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x, G = gridDim.x;
        if (lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter + (blockIdx.x % nc) * 64) : "memory");
        const unsigned per = lane < nc ? (unsigned)((G - lane + nc - 1) / nc) : 0u;      // CTAs that arrive on this lane's counter
        const unsigned target = per * round;
        bool ok;
        do {
            unsigned v = target;
            if (lane < nc) asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter + lane * 64) : "memory");
            ok = __all_sync(0xffffffffu, v >= target);
        } while (!ok);
    }
    __syncthreads();
}

struct Params {
    float* x;            // [R][K] replicas, written every iteration
    const float* priv;   // [grid][K] private constants
    const float* weights; size_t weight_floats;
    unsigned* counter;
    long long* lat;      // [grid] summed cycles
    long long* bar;      // [grid] summed barrier cycles
    float* sink;
    int mode, stream, iters, nc;
};

__global__ void __launch_bounds__(THREADS, 1) bench_kernel(Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ unsigned long long mbar;
    const int tid = threadIdx.x, lane = tid & 31, cta = blockIdx.x, G = gridDim.x;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned round = 0;
    long long lat = 0, bar = 0;
    float acc = 0.f;
    size_t woff = (size_t)cta * (WB / 4);
    for (int it = 0; it < p.iters; ++it) {
        // producers: CTA c owns elements [c*rpc, ...) of the vector; value depends on the iteration so the lines are really dirtied
        if (p.mode <= 1) {
            const int rpc = (K + G - 1) / G;
            if (tid < rpc && cta * rpc + tid < K) {
                const float v = (float)(it + cta);
                if (p.mode == 0) p.x[cta * rpc + tid] = v;
                else for (int r = 0; r < R; ++r) p.x[r * K + cta * rpc + tid] = v;
            }
        }
        if (p.stream && tid == 32) {          // background weight stream, one bulk copy per CTA per iteration
            asm volatile("{ .reg .b64 t; mbarrier.arrive.expect_tx.shared::cta.b64 t, [%0], %1; }" ::"r"(smem_u32(&mbar)), "r"(WB) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32(smem)), "l"(p.weights + woff), "r"(WB), "r"(smem_u32(&mbar)) : "memory");
            woff += (size_t)G * (WB / 4);
            if (woff + WB / 4 > p.weight_floats) woff = (size_t)cta * (WB / 4);
        }
        long long t0 = clock64();
        grid_sync(p.counter, ++round, p.nc);
        long long t1 = clock64();
        if (tid < 32) {
            const float* src = p.mode == 0 ? p.x : p.mode == 1 ? p.x + (cta % R) * K : p.mode == 2 ? p.x : p.priv + (size_t)cta * K;
            float4 v[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) v[i] = __ldcg(reinterpret_cast<const float4*>(src) + i * 32 + lane);
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 6; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            acc += s;
            long long t2 = clock64();
            if (lane == 0) { lat += t2 - t1; bar += t1 - t0; }
        }
        if (p.stream) {                        // wait for this iteration's bulk copy before the buffer is reused
            unsigned ok = 0;
            while (!ok) asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }"
                                     : "=r"(ok) : "r"(smem_u32(&mbar)), "r"(it & 1) : "memory");
        }
        grid_sync(p.counter, ++round, p.nc);          // readers done before the next overwrite
    }
    if (tid == 0) { p.lat[cta] = lat; p.bar[cta] = bar; }
    if (tid < 32) p.sink[cta * 32 + lane] = acc;
}

int main() {
    int dev = 0, sms = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int G = sms, iters = 2000;
    float *x, *priv, *weights, *sink;
    unsigned* counter; long long *lat, *bar;
    const size_t wfloats = (size_t)512 * 1024 * 1024 / 4;
    CK(cudaMalloc(&x, R * K * 4)); CK(cudaMemset(x, 0, R * K * 4));
    CK(cudaMalloc(&priv, (size_t)G * K * 4)); CK(cudaMemset(priv, 0, (size_t)G * K * 4));
    CK(cudaMalloc(&weights, wfloats * 4)); CK(cudaMemset(weights, 0, wfloats * 4));
    CK(cudaMalloc(&sink, G * 32 * 4)); CK(cudaMalloc(&counter, 64 * 64 * 4)); CK(cudaMalloc(&lat, G * 8)); CK(cudaMalloc(&bar, G * 8));
    CK(cudaFuncSetAttribute(bench_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WB));
    const char* names[4] = {"same vector, freshly written", "8 replicas, freshly written", "same vector, clean", "private vector per CTA"};
    for (int stream = 0; stream < 2; ++stream)
        for (int mode = 0; mode < 4; ++mode) {
            CK(cudaMemset(counter, 0, 64 * 64 * 4));
            Params p{x, priv, weights, wfloats, counter, lat, bar, sink, mode, stream, iters, 1};
            void* args[] = {&p};
            cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
            CK(cudaEventRecord(e0));
            CK(cudaLaunchCooperativeKernel((const void*)bench_kernel, dim3(G), dim3(THREADS), args, WB, 0));
            CK(cudaEventRecord(e1));
            CK(cudaDeviceSynchronize());
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            std::vector<long long> hl(G), hb(G);
            CK(cudaMemcpy(hl.data(), lat, G * 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(hb.data(), bar, G * 8, cudaMemcpyDeviceToHost));
            double sl = 0, mx = 0, sb = 0;
            for (int i = 0; i < G; ++i) { sl += hl[i]; sb += hb[i]; if (hl[i] > mx) mx = (double)hl[i]; }
            printf("stream=%d mode=%d (%-30s): load round trip mean %7.0f cyc, slowest CTA %7.0f cyc; barrier %7.0f cyc; %.2f us / iteration\n", stream, mode,
                   names[mode], sl / G / iters, mx / iters, sb / G / iters, 1000.0 * ms / iters);
        }
    for (int nc : {1, 2, 4, 8, 16, 32}) {          // barrier cost vs number of arrival counters (mode 3: private loads, no stream)
        CK(cudaMemset(counter, 0, 64 * 64 * 4));
        Params p{x, priv, weights, wfloats, counter, lat, bar, sink, 3, 0, iters, nc};
        void* args[] = {&p};
        cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        CK(cudaEventRecord(e0));
        CK(cudaLaunchCooperativeKernel((const void*)bench_kernel, dim3(G), dim3(THREADS), args, WB, 0));
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        std::vector<long long> hb(G);
        CK(cudaMemcpy(hb.data(), bar, G * 8, cudaMemcpyDeviceToHost));
        double sb = 0; for (int i = 0; i < G; ++i) sb += hb[i];
        printf("barrier with %2d arrival counters: %7.0f cyc mean per barrier; %.2f us / iteration (2 barriers + 1 load round trip)\n", nc, sb / G / iters, 1000.0 * ms / iters);
    }
    return 0;
}
