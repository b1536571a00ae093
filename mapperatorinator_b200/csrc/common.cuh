// Shared device/host helpers for the mapperatorinator_b200 engine (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>
#include <string>

namespace mb200 {

// ---- error plumbing: every C-ABI entry returns an int status; the message is kept per thread -------------------------
void set_last_error(const std::string& msg);

#define MB_CUDA_CHECK(expr)                                                                             \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess) {                                                                        \
            mb200::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + \
                                  ":" + std::to_string(__LINE__));                                      \
            return 1;                                                                                   \
        }                                                                                               \
    } while (0)

#define MB_REQUIRE(cond, msg)                                                                  \
    do {                                                                                       \
        if (!(cond)) {                                                                         \
            mb200::set_last_error(std::string("requirement failed: ") + #cond + " — " + (msg)); \
            return 2;                                                                          \
        }                                                                                      \
    } while (0)

#define MB_LAUNCH_CHECK() MB_CUDA_CHECK(cudaGetLastError())

// ---- measurement hooks: every launch_* bumps the counter; the step profiler brackets decode-path launches with events ----
extern long long g_launch_count;
extern long long g_wbf16_launch_count;      // the launches among them whose weights are a bf16 store (GEMV and megakernel)
struct StepProfiler {
    bool on = false;
    cudaEvent_t ev[1024];
    int cls[512];      // 0 gemv, 1 decode attention, 2 sample
    int n = 0;
    bool created = false;
};
extern StepProfiler g_prof;

// ---- captured CUDA graphs: a replay counts every node as a launch -------------------------------------------------------
struct CapturedGraph {
    cudaGraphExec_t exec = nullptr;
    long long nodes = 0;          // launches the body counted while it was captured
    long long wbf16_nodes = 0;    // ... of which read a bf16 weight store
    int launch(cudaStream_t st, int times = 1) {
        for (int i = 0; i < times; ++i) MB_CUDA_CHECK(cudaGraphLaunch(exec, st));
        g_launch_count += (long long)times * nodes;
        g_wbf16_launch_count += (long long)times * wbf16_nodes;
        return 0;
    }
};

// Captures `body(stream)` into *out on an engine-owned stream, created on first use (the caller's stream may be the legacy default
// stream, which cannot capture), once `st` has drained.  The capture launches nothing, so it leaves g_launch_count as it was.
template <typename Body>
int capture_graph(cudaStream_t& cap_stream, cudaStream_t st, Body&& body, CapturedGraph* out) {
    if (!cap_stream) MB_CUDA_CHECK(cudaStreamCreateWithFlags(&cap_stream, cudaStreamNonBlocking));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    cudaGraph_t graph;
    MB_CUDA_CHECK(cudaStreamBeginCapture(cap_stream, cudaStreamCaptureModeThreadLocal));
    const long long before = g_launch_count, before16 = g_wbf16_launch_count;
    const int rc = body(cap_stream);
    const cudaError_t e = cudaStreamEndCapture(cap_stream, &graph);
    out->nodes = g_launch_count - before;
    out->wbf16_nodes = g_wbf16_launch_count - before16;
    g_launch_count = before;
    g_wbf16_launch_count = before16;
    if (rc) {
        if (e == cudaSuccess) cudaGraphDestroy(graph);
        return rc;
    }
    MB_CUDA_CHECK(e);
    const cudaError_t ie = cudaGraphInstantiate(&out->exec, graph, 0);
    cudaGraphDestroy(graph);
    MB_CUDA_CHECK(ie);
    return 0;
}

// ---- activation ids shared by GEMM / GEMV epilogues ------------------------------------------------------------------
enum Act : int { ACT_NONE = 0, ACT_GELU_ERF = 1, ACT_GELU_TANH = 2, ACT_SILU = 3 };

__device__ __forceinline__ float apply_act(float x, int act) {
    switch (act) {
        case ACT_GELU_ERF:  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
        case ACT_GELU_TANH: {
            // torch gelu(approximate='tanh'): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
            const float k0 = 0.7978845608028654f, k1 = 0.044715f;
            float inner = k0 * (x + k1 * x * x * x);
            return 0.5f * x * (1.0f + tanhf(inner));
        }
        case ACT_SILU:      return x / (1.0f + expf(-x));
        default:            return x;
    }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Programmatic dependent launch hooks (no-ops when the launch does not carry the PDL attribute).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// A strided 2-D row map: logical row m of a [rows, cols] matrix lives at
//   ptr + (m / rpb) * bstride + (m % rpb) * ld      (rpb == 0 -> plain ptr + m * ld)
// Lets GEMM read im2col-free conv windows from a zero-padded [B, T+2, C] buffer, write K/V straight into the
// [B, Tmax, C] cache, or add a [T, C] position table to every batch item.
struct RowMap {
    float* ptr;
    long long ld;
    int rpb;
    long long bstride;
    __host__ __device__ __forceinline__ float* row(long long m) const {
        if (rpb == 0) return ptr + m * ld;
        long long b = m / rpb, t = m - b * rpb;
        return ptr + b * bstride + t * ld;
    }
};
static inline RowMap plain_map(const float* p, long long ld) { return RowMap{const_cast<float*>(p), ld, 0, 0}; }
static inline RowMap batched_map(const float* p, long long ld, int rpb, long long bstride) {
    return RowMap{const_cast<float*>(p), ld, rpb, bstride};
}

}  // namespace mb200
