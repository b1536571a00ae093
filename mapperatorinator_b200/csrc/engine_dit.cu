// Stage (iii): DiT forward + the ancestral sampling loop, entirely on the device.
//   reference: DiT.forward_with_cfg (osu_diffusion/utils/models.py:281-317), GaussianDiffusion.p_mean_variance / p_sample
//   (osu_diffusion/utils/diffusion/gaussian_diffusion.py:273-369, 420-467), the slider-free denoised_fn and in-paint mask of
//   DiffisionPipeline.sample_part (diffusion_pipeline.py:203-234).
// The conditioning vector silu(t_emb + y_emb) depends on the step only through t, so every adaLN modulation
// (12 blocks x 6 vectors + final 2) is computed for ALL steps up front with a handful of GEMMs; a step is then
//   first-layer embed -> 12 x [LN-modulate, qkv GEMM, band attention, gated out_proj GEMM, LN-modulate, fc1 GEMM + tanh-GELU,
//   gated fc2 GEMM] -> final LN-modulate -> 4-channel GEMM -> fused CFG-mix + learned-range variance + x0 + in-paint +
//   clamp(-2,2) + posterior mean + noise update, with no host round trip (the reference does ~25 tiny launches and several
//   numpy->tensor table gathers per step).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/mapperatorinator_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace mb200;

namespace {

struct DevBufD {
    void* p = nullptr; size_t bytes = 0;
    int ensure(size_t need) {
        if (need <= bytes) return 0;
        if (p) cudaFree(p);
        p = nullptr; bytes = 0;
        MB_CUDA_CHECK(cudaMalloc(&p, need));
        bytes = need;
        return 0;
    }
    float* f() const { return reinterpret_cast<float*>(p); }
    ~DevBufD() { if (p) cudaFree(p); }
};

#define MB_TRY(expr) do { int _s = (expr); if (_s) return _s; } while (0)

// A0[(n,t), :] = [cos|sin (x0*512*f) (128) , cos|sin (x1*512*f) (128) , c[n, :, t] (E)]   (FirstLayer.forward, models.py:204-209)
__global__ void dit_embed_kernel(const float* __restrict__ x, const float* __restrict__ c, const float* __restrict__ freqs, int N, int T, int C,
                                 int E, int FD, float* __restrict__ a0) {
    const int t = blockIdx.x, n = blockIdx.y;
    const int half_n = N / 2 > 0 ? N / 2 : 1;
    const int src = n % half_n;                      // forward_with_cfg feeds cat([half, half]) (models.py:306-307)
    const int K = C * FD + E, halfd = FD / 2;
    float* row = a0 + ((long long)n * T + t) * K;
    for (int j = threadIdx.x; j < K; j += blockDim.x) {
        float v;
        if (j < C * FD) {
            int ch = j / FD, k = j - ch * FD;
            float xv = x[((long long)src * C + ch) * T + t] * 512.0f;
            float arg = xv * freqs[k < halfd ? k : k - halfd];
            v = k < halfd ? cosf(arg) : sinf(arg);
        } else {
            v = c[((long long)n * E + (j - C * FD)) * T + t];
        }
        row[j] = v;
    }
}

// timestep_embedding(t, 256): row r -> [cos(t f) | sin(t f)]
__global__ void dit_temb_kernel(const float* __restrict__ tvals, const float* __restrict__ freqs, int FD, float* __restrict__ out) {
    const int r = blockIdx.x, halfd = FD / 2;
    const float t = tvals[r];
    for (int j = threadIdx.x; j < FD; j += blockDim.x) {
        float arg = t * freqs[j < halfd ? j : j - halfd];
        out[(long long)r * FD + j] = j < halfd ? cosf(arg) : sinf(arg);
    }
}

// b[r, :] = silu(te[r, :] + ye[r % N, :])   (DiT.forward: b = t + y, then adaLN_modulation[0] = SiLU)
__global__ void dit_cond_kernel(const float* __restrict__ te, const float* __restrict__ ye, int N, int d, float* __restrict__ b) {
    const int r = blockIdx.x;
    for (int j = threadIdx.x; j < d; j += blockDim.x) {
        float v = te[(long long)r * d + j] + ye[(long long)(r % N) * d + j];
        b[(long long)r * d + j] = v / (1.0f + expf(-v));
    }
}

// forward_with_cfg output assembly: out[n, ch, t] (models.py:312-317) from out4[(n,t), 4]
__global__ void dit_cfg_out_kernel(const float* __restrict__ o4, int N, int T, float cfg_scale, float* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * T) return;
    const int n = idx / T, t = idx - n * T, half_n = N / 2;
    for (int ch = 0; ch < 2; ++ch) {
        float cond = o4[((long long)(n % half_n) * T + t) * 4 + ch];
        float unc = o4[((long long)(half_n + n % half_n) * T + t) * 4 + ch];
        out[((long long)n * 4 + ch) * T + t] = unc + cfg_scale * (cond - unc);
        out[((long long)n * 4 + 2 + ch) * T + t] = o4[((long long)n * T + t) * 4 + 2 + ch];
    }
}

struct StepConst { float t, sqrt_recip, sqrt_recipm1, min_log, max_log, coef1, coef2, nonzero; };   // one row of the host schedule table

// Step-varying inputs are addressed through a device-resident step counter so that ONE captured CUDA graph serves every step:
// this kernel copies step k's adaLN modulation rows into the fixed buffers the graph's GEMM / LayerNorm nodes point at.
//   mods_all [depth][steps*N][6d] -> mods_cur [depth][N][6d];   fmod_all [steps*N][2d] -> fmod_cur [N][2d]
__global__ void dit_gather_mods_kernel(const float4* __restrict__ mods_all, const float4* __restrict__ fmod_all, const int* __restrict__ step_ptr,
                                       int depth, int steps, int N, int d4 /* d / 4 */, float4* __restrict__ mods_cur, float4* __restrict__ fmod_cur) {
    const int k = *step_ptr;
    const long long per_layer = (long long)N * 6 * d4, total_m = (long long)depth * per_layer, total = total_m + (long long)N * 2 * d4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if (i < total_m) {
            const long long l = i / per_layer, r = i - l * per_layer;
            mods_cur[i] = mods_all[(l * steps + k) * per_layer + r];
        } else {
            const long long r = i - total_m;
            fmod_cur[r] = fmod_all[(long long)k * N * 2 * d4 + r];
        }
    }
}

// one p_sample update (gaussian_diffusion.py:312-358, 454-466) for every (n, ch, t), in place (each element depends on its own
// index only); the step's constants and noise slice are read through the device step counter
__global__ void dit_update_kernel(const float* __restrict__ o4, float* __restrict__ x, const float* __restrict__ z,
                                  const unsigned char* __restrict__ inpaint, const float* __restrict__ noise, int N, int T, float cfg_scale,
                                  const StepConst* __restrict__ sched, const int* __restrict__ step_ptr) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * 2 * T) return;
    const int k = *step_ptr;
    const StepConst sc = sched[k];
    const int n = idx / (2 * T), rem = idx - n * 2 * T, ch = rem / T, t = rem - ch * T, half_n = N / 2;
    const float cond = o4[((long long)(n % half_n) * T + t) * 4 + ch];
    const float unc = o4[((long long)(half_n + n % half_n) * T + t) * 4 + ch];
    const float eps = unc + cfg_scale * (cond - unc);
    const float v = o4[((long long)n * T + t) * 4 + 2 + ch];
    const float frac = (v + 1.0f) / 2.0f;
    const float logvar = frac * sc.max_log + (1.0f - frac) * sc.min_log;
    const float xt = x[idx];
    float x0 = sc.sqrt_recip * xt - sc.sqrt_recipm1 * eps;
    if (inpaint && !inpaint[idx]) x0 = z[idx];
    x0 = fminf(fmaxf(x0, -2.0f), 2.0f);
    const float mean = sc.coef1 * x0 + sc.coef2 * xt;
    x[idx] = mean + sc.nonzero * expf(0.5f * logvar) * noise[(long long)k * N * 2 * T + idx];
}

// The same update in two halves around the slider recompute (denoised_fn with sliders, diffusion_pipeline.py:203-222):
//   (a) x0 = predicted x_start after the in-paint mask, for every (n, ch, t);
//   [slider.cu: conditional half -> pixels, slider ends recomputed, pixels written back to both halves of x0]
//   (b) clamp, posterior mean, noise.
__global__ void dit_x0_kernel(const float* __restrict__ o4, const float* __restrict__ x, const float* __restrict__ z,
                              const unsigned char* __restrict__ inpaint, int N, int T, float cfg_scale, const StepConst* __restrict__ sched,
                              const int* __restrict__ step_ptr, float* __restrict__ x0buf) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * 2 * T) return;
    const StepConst sc = sched[*step_ptr];
    const int n = idx / (2 * T), rem = idx - n * 2 * T, ch = rem / T, t = rem - ch * T, half_n = N / 2;
    const float cond = o4[((long long)(n % half_n) * T + t) * 4 + ch];
    const float unc = o4[((long long)(half_n + n % half_n) * T + t) * 4 + ch];
    const float eps = unc + cfg_scale * (cond - unc);
    float x0 = sc.sqrt_recip * x[idx] - sc.sqrt_recipm1 * eps;
    if (inpaint && !inpaint[idx]) x0 = z[idx];
    x0buf[idx] = x0;
}
__global__ void dit_finish_kernel(const float* __restrict__ o4, float* __restrict__ x, const float* __restrict__ x0buf, const float* __restrict__ noise,
                                  int N, int T, const StepConst* __restrict__ sched, const int* __restrict__ step_ptr) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * 2 * T) return;
    const int k = *step_ptr;
    const StepConst sc = sched[k];
    const int n = idx / (2 * T), rem = idx - n * 2 * T, ch = rem / T, t = rem - ch * T;
    const float v = o4[((long long)n * T + t) * 4 + 2 + ch];
    const float frac = (v + 1.0f) / 2.0f;
    const float logvar = frac * sc.max_log + (1.0f - frac) * sc.min_log;
    const float xt = x[idx];
    const float x0 = fminf(fmaxf(x0buf[idx], -2.0f), 2.0f);
    const float mean = sc.coef1 * x0 + sc.coef2 * xt;
    x[idx] = mean + sc.nonzero * expf(0.5f * logvar) * noise[(long long)k * N * 2 * T + idx];
}

__global__ void dit_step_advance_kernel(int* step_ptr) { *step_ptr += 1; }

struct BlockW { const float *in_w, *in_b, *out_w, *out_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b, *ada_w, *ada_b; };

}  // namespace

struct mb200_dit {
    mb200_dit_config cfg;
    std::unordered_map<std::string, std::vector<float>> host_w;
    bool finalized = false;
    DevBufD arena;
    // device pointers, resolved ONCE at finalize (no name lookups on the step path)
    const float *ctx_w = nullptr, *ctx_b = nullptr, *t0_w = nullptr, *t0_b = nullptr, *t2_w = nullptr, *t2_b = nullptr, *y0_w = nullptr,
                *y0_b = nullptr, *y2_w = nullptr, *y2_b = nullptr, *fada_w = nullptr, *fada_b = nullptr, *flin_w = nullptr, *flin_b = nullptr;
    std::vector<BlockW> blocks;
    const float *pos_freqs = nullptr, *t_freqs = nullptr;
    DevBufD a0, x, h, qkv, att, ffn, o4, temb, te1, te, ye1, ye, bcond, mods, fmod, tvals;
    // sampling loop: engine-owned copies of the call's inputs + the step-indexed tables, so the captured step graph never sees a
    // caller pointer
    DevBufD state, z_in, c_in, y_in, noise_in, inpaint_in, dense_in, sched, step_ctr, mods_cur, fmod_cur;
    std::map<std::tuple<int, int, int, int, int>, CapturedGraph> step_graphs;   // (N, T, mask mode, band, in-paint) -> graph
    // sliders of the current chunk (mb200_dit_set_sliders); the step graph is keyed by their presence, the arrays live in fixed buffers
    DevBufD sl_off, sl_idx, sl_end, sl_type, sl_len, sl_pix, sl_err, x0buf;
    int n_sliders = 0, sl_cap = 0, sl_cp_cap = 0;
    cudaStream_t cap_stream = nullptr;
    bool use_graph = true;
    float graph_cfg_scale = 0.f; const void* graph_noise = nullptr; const void* graph_mods = nullptr;   // what the cached graphs baked
    GemmCtx gemm;
    AttnCtx attn;                       // tensor-core attention scratch (head-major tf32 copies of q | k | v^T)
};

extern "C" int mb200_dit_create(mb200_dit** out, const mb200_dit_config* cfg) {
    MB_REQUIRE(out && cfg, "null argument");
    MB_REQUIRE(cfg->hidden == cfg->heads * 64, "kernels are specialised for head_dim 64 (DiT-B: 768 / 12)");
    MB_REQUIRE(cfg->hidden % 128 == 0 && cfg->hidden <= 1024, "hidden must be a multiple of 128 and <= 1024");
    MB_REQUIRE(cfg->in_channels == 2, "the position DiT has 2 input channels");
    MB_REQUIRE(cfg->class_size % 4 == 0 && cfg->context_size % 4 == 0, "class_size / context_size must be multiples of 4");
    mb200_dit* d = new mb200_dit();
    d->cfg = *cfg;
    *out = d;
    return 0;
}

extern "C" void mb200_dit_destroy(mb200_dit* d) {
    if (!d) return;
    for (auto& g : d->step_graphs) cudaGraphExecDestroy(g.second.exec);
    if (d->cap_stream) cudaStreamDestroy(d->cap_stream);
    d->gemm.destroy();
    d->attn.destroy();
    delete d;
}

extern "C" int mb200_dit_set_weight(mb200_dit* d, const char* name, const float* data, int64_t numel) {
    MB_REQUIRE(d && name && data && !d->finalized, "bad argument / state");
    d->host_w[name] = std::vector<float>(data, data + numel);
    return 0;
}

extern "C" int mb200_dit_finalize(mb200_dit* dd) {
    MB_REQUIRE(dd && !dd->finalized, "bad state");
    const auto& c = dd->cfg;
    const int d = c.hidden;
    std::vector<std::string> names = {
        "context_embedder.mlp.0.weight", "context_embedder.mlp.0.bias", "t_embedder.mlp.0.weight", "t_embedder.mlp.0.bias",
        "t_embedder.mlp.2.weight", "t_embedder.mlp.2.bias", "y_embedder.class_embedding.0.weight", "y_embedder.class_embedding.0.bias",
        "y_embedder.class_embedding.2.weight", "y_embedder.class_embedding.2.bias", "final_layer.adaLN_modulation.1.weight",
        "final_layer.adaLN_modulation.1.bias", "final_layer.linear.weight", "final_layer.linear.bias"};
    for (int i = 0; i < c.depth; ++i) {
        std::string p = "blocks." + std::to_string(i) + ".";
        for (const char* s : {"attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj.weight", "attn.out_proj.bias", "mlp.fc1.weight",
                              "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias", "adaLN_modulation.1.weight", "adaLN_modulation.1.bias"})
            names.push_back(p + s);
    }
    std::vector<float> pack;
    std::unordered_map<std::string, size_t> offs, sizes;
    for (const auto& n : names) {
        MB_REQUIRE(dd->host_w.count(n) == 1, "missing DiT weight " + n);
        std::vector<float> v = dd->host_w.at(n);
        // nn.MultiheadAttention scales q by head_dim^-0.5 = 1/8 (a power of two): fold it into the q rows, bit-exact
        if (n.find("attn.in_proj_weight") != std::string::npos) for (size_t i = 0; i < (size_t)d * d; ++i) v[i] *= 0.125f;
        if (n.find("attn.in_proj_bias") != std::string::npos) for (int i = 0; i < d; ++i) v[i] *= 0.125f;
        size_t off = (pack.size() + 63) & ~size_t(63);
        pack.resize(off + v.size());
        std::copy(v.begin(), v.end(), pack.begin() + off);
        offs[n] = off; sizes[n] = v.size();
    }
    // sinusoid frequency tables, same fp32 chain as positional_embedding.timestep_embedding (:40-46)
    auto freqs = [&](int dim) {
        std::vector<float> f(dim / 2);
        const float neg_log = (float)(-std::log(10000.0));
        for (int k = 0; k < dim / 2; ++k) f[k] = std::exp(neg_log * (float)k / (float)(dim / 2));
        return f;
    };
    for (auto pr : {std::make_pair(std::string("__pos_freqs"), c.pos_freq_dim), std::make_pair(std::string("__t_freqs"), c.t_freq_dim)}) {
        std::vector<float> v = freqs(pr.second);
        size_t off = (pack.size() + 63) & ~size_t(63);
        pack.resize(off + v.size());
        std::copy(v.begin(), v.end(), pack.begin() + off);
        offs[pr.first] = off;
    }
    MB_TRY(dd->arena.ensure(pack.size() * 4));
    MB_CUDA_CHECK(cudaMemcpy(dd->arena.p, pack.data(), pack.size() * 4, cudaMemcpyHostToDevice));
    auto W = [&](const std::string& n) -> const float* { return dd->arena.f() + offs.at(n); };
    dd->ctx_w = W("context_embedder.mlp.0.weight"); dd->ctx_b = W("context_embedder.mlp.0.bias");
    dd->t0_w = W("t_embedder.mlp.0.weight"); dd->t0_b = W("t_embedder.mlp.0.bias"); dd->t2_w = W("t_embedder.mlp.2.weight"); dd->t2_b = W("t_embedder.mlp.2.bias");
    dd->y0_w = W("y_embedder.class_embedding.0.weight"); dd->y0_b = W("y_embedder.class_embedding.0.bias");
    dd->y2_w = W("y_embedder.class_embedding.2.weight"); dd->y2_b = W("y_embedder.class_embedding.2.bias");
    dd->fada_w = W("final_layer.adaLN_modulation.1.weight"); dd->fada_b = W("final_layer.adaLN_modulation.1.bias");
    dd->flin_w = W("final_layer.linear.weight"); dd->flin_b = W("final_layer.linear.bias");
    for (int i = 0; i < c.depth; ++i) {
        const std::string p = "blocks." + std::to_string(i) + ".";
        dd->blocks.push_back(BlockW{W(p + "attn.in_proj_weight"), W(p + "attn.in_proj_bias"), W(p + "attn.out_proj.weight"), W(p + "attn.out_proj.bias"),
                                    W(p + "mlp.fc1.weight"), W(p + "mlp.fc1.bias"), W(p + "mlp.fc2.weight"), W(p + "mlp.fc2.bias"),
                                    W(p + "adaLN_modulation.1.weight"), W(p + "adaLN_modulation.1.bias")});
    }
    {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&dd->gemm.num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    // tf32 hi / lo mirrors for the tensor-core GEMMs (every 2-D weight of the blocks and the embedders)
    for (const auto& n : names)
        if (n.find("weight") != std::string::npos && sizes.at(n) >= (size_t)64 * 32) MB_TRY(dd->gemm.register_weight(W(n), (long long)sizes.at(n)));
    MB_CUDA_CHECK(cudaDeviceSynchronize());
    dd->pos_freqs = W("__pos_freqs"); dd->t_freqs = W("__t_freqs");
    MB_REQUIRE(dd->host_w.at("context_embedder.mlp.0.weight").size() == (size_t)d * (c.in_channels * c.pos_freq_dim + c.context_size),
               "context_embedder shape mismatch");
    {   // all scratch for the largest call, allocated once: the captured step graphs hold these pointers
        const size_t R = (size_t)std::max(2, c.max_batch) * c.max_seq_len;
        const size_t K0 = (size_t)c.in_channels * c.pos_freq_dim + c.context_size;
        MB_TRY(dd->gemm.reserve((size_t)64 << 20, R * std::max((size_t)d * c.mlp_ratio, K0) * 8 + 1024));
        dd->gemm.frozen = true;
        MB_TRY(dd->attn.reserve(attn_tc_workspace_bytes(std::max(2, c.max_batch), c.heads, c.max_seq_len, c.max_seq_len)));
        dd->attn.frozen = true;
    }
    dd->host_w.clear();
    dd->finalized = true;
    return 0;
}

namespace {

GemmParams gb(const float* A, long long lda, const float* W, long long ldw, float* C, long long ldc, const float* bias, int M, int N, int K) {
    GemmParams g{};
    g.A = plain_map(A, lda); g.W = W; g.ldw = ldw; g.C = plain_map(C, ldc); g.bias = bias; g.act = ACT_NONE; g.alpha = 1.f;
    g.gate = nullptr; g.gate_ld = 0; g.gate_rpb = 1; g.R = RowMap{nullptr, 0, 0, 0}; g.M = M; g.N = N; g.K = K;
    return g;
}

int ln_mod(const float* x, float* y, const float* shift, const float* scale, long long mod_ld, int T, int rows, int d, cudaStream_t st) {
    LayerNormParams p{};
    p.x = x; p.ldx = d; p.y = y; p.ldy = d; p.weight = nullptr; p.bias = nullptr; p.shift = shift; p.scale = scale; p.mod_ld = mod_ld;
    p.rows_per_batch = T; p.rows = rows; p.dim = d; p.eps = 1e-6f;
    return launch_layernorm(p, st);
}

// modulation vectors for `steps` timesteps: mods[l][step*N + n][6d], fmod[step*N + n][2d]
int prepare_conditioning(mb200_dit* dd, const float* tvals_host, int steps, int N, const float* y, cudaStream_t st) {
    const auto& c = dd->cfg;
    const int d = c.hidden, RS = steps * N;
    GemmCtx* gc = &dd->gemm;
    MB_TRY(dd->tvals.ensure((size_t)RS * 4)); MB_TRY(dd->temb.ensure((size_t)RS * c.t_freq_dim * 4));
    MB_TRY(dd->te1.ensure((size_t)RS * d * 4)); MB_TRY(dd->te.ensure((size_t)RS * d * 4));
    MB_TRY(dd->ye1.ensure((size_t)N * d * 4)); MB_TRY(dd->ye.ensure((size_t)N * d * 4));
    MB_TRY(dd->bcond.ensure((size_t)RS * d * 4));
    MB_TRY(dd->mods.ensure((size_t)c.depth * RS * 6 * d * 4)); MB_TRY(dd->fmod.ensure((size_t)RS * 2 * d * 4));
    MB_CUDA_CHECK(cudaMemcpyAsync(dd->tvals.p, tvals_host, (size_t)RS * 4, cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    dit_temb_kernel<<<RS, 128, 0, st>>>(dd->tvals.f(), dd->t_freqs, c.t_freq_dim, dd->temb.f());
    MB_LAUNCH_CHECK();
    {
        GemmParams g = gb(dd->temb.f(), c.t_freq_dim, dd->t0_w, c.t_freq_dim, dd->te1.f(), d, dd->t0_b, RS, d, c.t_freq_dim);
        g.act = ACT_SILU;
        MB_TRY(launch_gemm(g, st, gc));
        MB_TRY(launch_gemm(gb(dd->te1.f(), d, dd->t2_w, d, dd->te.f(), d, dd->t2_b, RS, d, d), st, gc));
        GemmParams gy = gb(y, c.class_size, dd->y0_w, c.class_size, dd->ye1.f(), d, dd->y0_b, N, d, c.class_size);
        gy.act = ACT_SILU;
        MB_TRY(launch_gemm(gy, st, gc));
        MB_TRY(launch_gemm(gb(dd->ye1.f(), d, dd->y2_w, d, dd->ye.f(), d, dd->y2_b, N, d, d), st, gc));
    }
    dit_cond_kernel<<<RS, 128, 0, st>>>(dd->te.f(), dd->ye.f(), N, d, dd->bcond.f());
    MB_LAUNCH_CHECK();
    for (int l = 0; l < c.depth; ++l)
        MB_TRY(launch_gemm(gb(dd->bcond.f(), d, dd->blocks[l].ada_w, d, dd->mods.f() + (size_t)l * RS * 6 * d, 6 * d, dd->blocks[l].ada_b, RS, 6 * d, d), st, gc));
    MB_TRY(launch_gemm(gb(dd->bcond.f(), d, dd->fada_w, d, dd->fmod.f(), 2 * d, dd->fada_b, RS, 2 * d, d), st, gc));
    return 0;
}

// activations for the largest (N, T) the engine was created for: allocated on first use, never moved afterwards
int ensure_work(mb200_dit* dd) {
    const auto& c = dd->cfg;
    const int d = c.hidden;
    const size_t R = (size_t)std::max(2, c.max_batch) * c.max_seq_len;
    const int K0 = c.in_channels * c.pos_freq_dim + c.context_size;
    MB_TRY(dd->a0.ensure(R * K0 * 4)); MB_TRY(dd->x.ensure(R * d * 4)); MB_TRY(dd->h.ensure(R * d * 4));
    MB_TRY(dd->qkv.ensure(R * 3 * d * 4)); MB_TRY(dd->att.ensure(R * d * 4)); MB_TRY(dd->ffn.ensure(R * d * c.mlp_ratio * 4));
    MB_TRY(dd->o4.ensure(R * 4 * 4));
    MB_TRY(dd->mods_cur.ensure((size_t)c.depth * c.max_batch * 6 * d * 4)); MB_TRY(dd->fmod_cur.ensure((size_t)c.max_batch * 2 * d * 4));
    return 0;
}

// one DiT forward with the modulation rows at mods [depth][N][6d] / fm [N][2d] -> o4[(n,t), 4]
int dit_forward(mb200_dit* dd, const float* xstate, const float* cctx, int N, int T, const float* mods, const float* fm,
                const mb200_dit_mask* mask, cudaStream_t st) {
    const auto& c = dd->cfg;
    const int d = c.hidden, f = d * c.mlp_ratio, R = N * T;
    const int K0 = c.in_channels * c.pos_freq_dim + c.context_size;
    GemmCtx* gc = &dd->gemm;
    dit_embed_kernel<<<dim3(T, N), 128, 0, st>>>(xstate, cctx, dd->pos_freqs, N, T, c.in_channels, c.context_size, c.pos_freq_dim, dd->a0.f());
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    MB_TRY(launch_gemm(gb(dd->a0.f(), K0, dd->ctx_w, K0, dd->x.f(), d, dd->ctx_b, R, d, K0), st, gc));
    for (int l = 0; l < c.depth; ++l) {
        const BlockW& w = dd->blocks[l];
        const float* mod = mods + (size_t)l * N * 6 * d;   // rows n = 0..N-1
        MB_TRY(ln_mod(dd->x.f(), dd->h.f(), mod + 0, mod + d, 6 * d, T, R, d, st));
        MB_TRY(launch_gemm(gb(dd->h.f(), d, w.in_w, d, dd->qkv.f(), 3 * d, w.in_b, R, 3 * d, d), st, gc));
        AttentionParams a{};
        a.q = dd->qkv.f(); a.q_ld = 3 * d; a.q_bs = (long long)T * 3 * d;
        a.k = dd->qkv.f() + d; a.k_ld = 3 * d; a.k_bs = a.q_bs;
        a.v = dd->qkv.f() + 2 * d; a.v_ld = 3 * d; a.v_bs = a.q_bs;
        a.o = dd->att.f(); a.o_ld = d; a.o_bs = (long long)T * d;
        a.B = N; a.H = c.heads; a.Tq = T; a.Tk = T; a.scale = 1.f;
        a.mask_mode = mask ? mask->mask_mode : MASK_NONE; a.band = mask ? mask->band : 0; a.dense = mask ? mask->dense_mask : nullptr;
        MB_TRY(launch_attention(a, st, &dd->attn));
        {
            GemmParams g = gb(dd->att.f(), d, w.out_w, d, dd->x.f(), d, w.out_b, R, d, d);
            g.gate = mod + 2 * d; g.gate_ld = 6 * d; g.gate_rpb = T; g.R = plain_map(dd->x.f(), d);
            MB_TRY(launch_gemm(g, st, gc));
        }
        MB_TRY(ln_mod(dd->x.f(), dd->h.f(), mod + 3 * d, mod + 4 * d, 6 * d, T, R, d, st));
        {
            GemmParams g = gb(dd->h.f(), d, w.fc1_w, d, dd->ffn.f(), f, w.fc1_b, R, f, d);
            g.act = ACT_GELU_TANH;
            MB_TRY(launch_gemm(g, st, gc));
        }
        {
            GemmParams g = gb(dd->ffn.f(), f, w.fc2_w, f, dd->x.f(), d, w.fc2_b, R, d, f);
            g.gate = mod + 5 * d; g.gate_ld = 6 * d; g.gate_rpb = T; g.R = plain_map(dd->x.f(), d);
            MB_TRY(launch_gemm(g, st, gc));
        }
    }
    MB_TRY(ln_mod(dd->x.f(), dd->h.f(), fm, fm + d, 2 * d, T, R, d, st));
    MB_TRY(launch_gemm(gb(dd->h.f(), d, dd->flin_w, d, dd->o4.f(), 4, dd->flin_b, R, 4, d), st, gc));
    return 0;
}

int check_shapes(mb200_dit* d, int N, int T) {
    MB_REQUIRE(d && d->finalized, "DiT not finalized");
    MB_REQUIRE(N >= 2 && N % 2 == 0 && N <= d->cfg.max_batch, "forward_with_cfg needs an even batch (cond | uncond) within max_batch");
    MB_REQUIRE(T >= 1 && T <= d->cfg.max_seq_len, "sequence longer than max_seq_len");
    return 0;
}

}  // namespace

extern "C" int mb200_dit_forward_with_cfg(mb200_dit* d, const float* x, const int32_t* t, const float* c, const float* y, int32_t N, int32_t T,
                                          float cfg_scale, const mb200_dit_mask* mask, float* out, void* stream) {
    MB_TRY(check_shapes(d, N, T));
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<float> tv(N);
    for (int i = 0; i < N; ++i) tv[i] = (float)t[i];
    MB_TRY(ensure_work(d));
    MB_TRY(prepare_conditioning(d, tv.data(), 1, N, y, st));
    MB_TRY(dit_forward(d, x, c, N, T, d->mods.f(), d->fmod.f(), mask, st));     // steps == 1: the all-steps tables ARE this step's rows
    dit_cfg_out_kernel<<<(N * T + 255) / 256, 256, 0, st>>>(d->o4.f(), N, T, cfg_scale, out);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

// The 100-step loop.  Every step is the SAME captured CUDA graph (gather this step's modulation rows -> DiT forward -> in-place
// p_sample update -> step counter + 1): one host launch per step, no host synchronisation inside the loop, no caller pointer in
// the graph (inputs are copied into engine-owned buffers first: 4 MB, once per call).
extern "C" int mb200_dit_sample_loop(mb200_dit* d, const float* z, const float* c, const float* y, const uint8_t* inpaint, int32_t N, int32_t T,
                                     float cfg_scale, const mb200_dit_mask* mask, const float* schedule, int32_t steps, const float* noise,
                                     float* out, void* stream) {
    MB_TRY(check_shapes(d, N, T));
    MB_REQUIRE(z && c && y && schedule && noise && out && steps >= 1, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const auto& cf = d->cfg;
    const int dm = cf.hidden;
    std::vector<float> tv((size_t)steps * N);
    for (int k = 0; k < steps; ++k)
        for (int n = 0; n < N; ++n) tv[(size_t)k * N + n] = schedule[(size_t)k * 8 + 0];
    MB_TRY(ensure_work(d));
    const size_t total = (size_t)N * 2 * T, state_bytes = total * 4;
    const size_t maxR = (size_t)cf.max_batch * cf.max_seq_len;
    MB_TRY(d->state.ensure(maxR * 2 * 4)); MB_TRY(d->z_in.ensure(maxR * 2 * 4)); MB_TRY(d->c_in.ensure(maxR * cf.context_size * 4));
    MB_TRY(d->inpaint_in.ensure(maxR * 2)); MB_TRY(d->dense_in.ensure((size_t)cf.max_seq_len * cf.max_seq_len));
    MB_TRY(d->step_ctr.ensure(64));
    MB_TRY(d->noise_in.ensure((size_t)steps * state_bytes));      // may grow with `steps`; graphs are dropped below when it moves
    MB_TRY(d->sched.ensure((size_t)steps * 8 * 4));
    MB_TRY(prepare_conditioning(d, tv.data(), steps, N, y, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(d->state.p, z, state_bytes, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(d->z_in.p, z, state_bytes, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(d->c_in.p, c, (size_t)N * cf.context_size * T * 4, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(d->noise_in.p, noise, (size_t)steps * state_bytes, cudaMemcpyDeviceToDevice, st));
    if (inpaint) MB_CUDA_CHECK(cudaMemcpyAsync(d->inpaint_in.p, inpaint, total, cudaMemcpyDeviceToDevice, st));
    mb200_dit_mask mk{MASK_NONE, 0, nullptr};
    if (mask) {
        mk = *mask;
        if (mk.mask_mode == MASK_DENSE) {
            MB_REQUIRE(mk.dense_mask != nullptr, "dense mask mode without a mask");
            MB_CUDA_CHECK(cudaMemcpyAsync(d->dense_in.p, mk.dense_mask, (size_t)T * T, cudaMemcpyDeviceToDevice, st));
            mk.dense_mask = reinterpret_cast<const uint8_t*>(d->dense_in.p);
        }
    }
    MB_CUDA_CHECK(cudaMemcpyAsync(d->sched.p, schedule, (size_t)steps * 8 * 4, cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaMemsetAsync(d->step_ctr.p, 0, 4, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));      // `schedule` is pageable host memory of the caller
    int* step_ptr = reinterpret_cast<int*>(d->step_ctr.p);
    const unsigned char* ip = inpaint ? reinterpret_cast<const unsigned char*>(d->inpaint_in.p) : nullptr;
    const int n_mods = (cf.depth * N * 6 + N * 2) * (dm / 4);
    SliderSet sl{};
    sl.n = d->n_sliders;
    if (sl.n > 0) {
        sl.cp_offsets = reinterpret_cast<const int*>(d->sl_off.p); sl.cp_index = reinterpret_cast<const int*>(d->sl_idx.p);
        sl.end_index = reinterpret_cast<const int*>(d->sl_end.p); sl.type = reinterpret_cast<const int*>(d->sl_type.p); sl.length = d->sl_len.f();
        MB_TRY(d->x0buf.ensure(maxR * 2 * 4)); MB_TRY(d->sl_pix.ensure((size_t)2 * cf.max_seq_len * 4));
        // the start state itself goes through the closure first (diffusion_pipeline.py:233: z_part = denoised_fn(z_part)); the in-paint
        // source of every later step is that corrected state (the closure reads the re-bound z_part)
        MB_TRY(launch_slider_recompute(sl, d->state.f(), N, T, d->sl_pix.f(), reinterpret_cast<int*>(d->sl_err.p), st));
        MB_CUDA_CHECK(cudaMemcpyAsync(d->z_in.p, d->state.p, state_bytes, cudaMemcpyDeviceToDevice, st));
    }
    auto one_step = [&](cudaStream_t s) -> int {
        dit_gather_mods_kernel<<<std::min(296, (n_mods + 255) / 256), 256, 0, s>>>(
            reinterpret_cast<const float4*>(d->mods.p), reinterpret_cast<const float4*>(d->fmod.p), step_ptr, cf.depth, steps, N, dm / 4,
            reinterpret_cast<float4*>(d->mods_cur.p), reinterpret_cast<float4*>(d->fmod_cur.p));
        MB_LAUNCH_CHECK();
        MB_TRY(dit_forward(d, d->state.f(), d->c_in.f(), N, T, d->mods_cur.f(), d->fmod_cur.f(), &mk, s));
        if (sl.n > 0) {
            dit_x0_kernel<<<((int)total + 255) / 256, 256, 0, s>>>(d->o4.f(), d->state.f(), d->z_in.f(), ip, N, T, cfg_scale,
                                                                  reinterpret_cast<const StepConst*>(d->sched.p), step_ptr, d->x0buf.f());
            MB_LAUNCH_CHECK();
            MB_TRY(launch_slider_recompute(sl, d->x0buf.f(), N, T, d->sl_pix.f(), reinterpret_cast<int*>(d->sl_err.p), s));
            dit_finish_kernel<<<((int)total + 255) / 256, 256, 0, s>>>(d->o4.f(), d->state.f(), d->x0buf.f(), d->noise_in.f(), N, T,
                                                                      reinterpret_cast<const StepConst*>(d->sched.p), step_ptr);
            MB_LAUNCH_CHECK();
            ++g_launch_count;
        } else {
            dit_update_kernel<<<((int)total + 255) / 256, 256, 0, s>>>(d->o4.f(), d->state.f(), d->z_in.f(), ip, d->noise_in.f(), N, T, cfg_scale,
                                                                      reinterpret_cast<const StepConst*>(d->sched.p), step_ptr);
            MB_LAUNCH_CHECK();
        }
        dit_step_advance_kernel<<<1, 1, 0, s>>>(step_ptr);
        MB_LAUNCH_CHECK();
        g_launch_count += 3;
        return 0;
    };
    if (!d->use_graph) {
        for (int k = 0; k < steps; ++k) MB_TRY(one_step(st));
    } else {
        // the graph bakes (N, T, mask, in-paint on/off, cfg_scale, steps, the mods / noise table addresses)
        const auto key = std::make_tuple((int)N, (int)T, (int)mk.mask_mode, (int)mk.band + 4096 * d->n_sliders, (inpaint ? 1 : 0) + 2 * steps);
        if (d->graph_cfg_scale != cfg_scale || d->graph_noise != d->noise_in.p || d->graph_mods != d->mods.p) {
            for (auto& g : d->step_graphs) cudaGraphExecDestroy(g.second.exec);
            d->step_graphs.clear();
            d->graph_cfg_scale = cfg_scale; d->graph_noise = d->noise_in.p; d->graph_mods = d->mods.p;
        }
        auto it = d->step_graphs.find(key);
        if (it == d->step_graphs.end()) {
            CapturedGraph g;
            MB_TRY(capture_graph(d->cap_stream, st, one_step, &g));
            if (d->step_graphs.size() >= 16) {      // bounded cache
                for (auto& old : d->step_graphs) cudaGraphExecDestroy(old.second.exec);
                d->step_graphs.clear();
            }
            it = d->step_graphs.emplace(key, g).first;
        }
        MB_TRY(it->second.launch(st, steps));
    }
    MB_CUDA_CHECK(cudaMemcpyAsync(out, d->state.p, state_bytes, cudaMemcpyDeviceToDevice, st));
    if (sl.n > 0) {
        int herr = 0;
        MB_CUDA_CHECK(cudaMemcpyAsync(&herr, d->sl_err.p, 4, cudaMemcpyDeviceToHost, st));
        MB_CUDA_CHECK(cudaStreamSynchronize(st));
        MB_REQUIRE(herr == 0, herr == 1 ? "a slider has more than 64 control points" : "a slider sub-path has more than 32 control points or needs more than 24 subdivision levels");
    }
    return 0;
}

// Sliders of the chunk about to be sampled (host arrays; n == 0 clears).  The caller filters them like the reference closure does
// (all control points and the end event inside the chunk, diffusion_pipeline.py:211-212) and passes chunk-relative indices.
extern "C" int mb200_dit_set_sliders(mb200_dit* d, int32_t n, const int32_t* cp_offsets, const int32_t* cp_index, const int32_t* end_index,
                                     const int32_t* type, const float* length) {
    MB_REQUIRE(d && d->finalized && n >= 0, "bad argument");
    d->n_sliders = 0;
    if (n == 0) return 0;
    MB_REQUIRE(cp_offsets && cp_index && end_index && type && length, "null argument");
    const int total = cp_offsets[n];
    for (int k = 0; k < n; ++k) {
        MB_REQUIRE(cp_offsets[k + 1] - cp_offsets[k] >= 1 && cp_offsets[k + 1] - cp_offsets[k] <= 64, "a slider needs 1..64 control points");
        MB_REQUIRE(type[k] >= 0 && type[k] <= 3, "unknown curve type");
        MB_REQUIRE(end_index[k] >= 0 && end_index[k] < d->cfg.max_seq_len, "slider end index outside the chunk");
    }
    for (int i = 0; i < total; ++i) MB_REQUIRE(cp_index[i] >= 0 && cp_index[i] < d->cfg.max_seq_len, "slider control point outside the chunk");
    // buffers only ever grow to the chunk capacity once: a captured step graph holds their addresses
    const size_t cap = (size_t)d->cfg.max_seq_len;
    MB_REQUIRE((size_t)n <= cap && (size_t)total <= 8 * cap, "more sliders / control points than the chunk can hold");
    MB_TRY(d->sl_off.ensure((cap + 1) * 4)); MB_TRY(d->sl_idx.ensure(8 * cap * 4)); MB_TRY(d->sl_end.ensure(cap * 4));
    MB_TRY(d->sl_type.ensure(cap * 4)); MB_TRY(d->sl_len.ensure(cap * 4)); MB_TRY(d->sl_err.ensure(64));
    MB_CUDA_CHECK(cudaMemcpy(d->sl_off.p, cp_offsets, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice));
    MB_CUDA_CHECK(cudaMemcpy(d->sl_idx.p, cp_index, (size_t)total * 4, cudaMemcpyHostToDevice));
    MB_CUDA_CHECK(cudaMemcpy(d->sl_end.p, end_index, (size_t)n * 4, cudaMemcpyHostToDevice));
    MB_CUDA_CHECK(cudaMemcpy(d->sl_type.p, type, (size_t)n * 4, cudaMemcpyHostToDevice));
    MB_CUDA_CHECK(cudaMemcpy(d->sl_len.p, length, (size_t)n * 4, cudaMemcpyHostToDevice));
    MB_CUDA_CHECK(cudaMemset(d->sl_err.p, 0, 4));
    d->n_sliders = n;
    return 0;
}

// The slider half of the closure on its own (Python-loop seam and parity tests): x DEVICE [N, 2, T] in place.
extern "C" int mb200_dit_apply_sliders(mb200_dit* d, float* x, int32_t N, int32_t T, void* stream) {
    MB_REQUIRE(d && d->finalized && x && N >= 1 && T >= 1 && T <= d->cfg.max_seq_len, "bad argument");
    if (d->n_sliders == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    MB_TRY(d->sl_pix.ensure((size_t)2 * d->cfg.max_seq_len * 4));
    SliderSet sl{d->n_sliders, reinterpret_cast<const int*>(d->sl_off.p), reinterpret_cast<const int*>(d->sl_idx.p),
                 reinterpret_cast<const int*>(d->sl_end.p), reinterpret_cast<const int*>(d->sl_type.p), d->sl_len.f()};
    MB_TRY(launch_slider_recompute(sl, x, N, T, d->sl_pix.f(), reinterpret_cast<int*>(d->sl_err.p), st));
    int herr = 0;
    MB_CUDA_CHECK(cudaMemcpyAsync(&herr, d->sl_err.p, 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    MB_REQUIRE(herr == 0, "slider path exceeds the device limits (64 control points, 32 per sub-path, 24 subdivision levels)");
    return 0;
}

extern "C" int mb200_dit_set_option(mb200_dit* d, const char* name, int32_t value) {
    MB_REQUIRE(d && name, "null argument");
    if (!strcmp(name, "graph")) { d->use_graph = value != 0; return 0; }
    set_last_error(std::string("unknown option ") + name);
    return 2;
}
