// C-ABI glue: error channel, the mel stage handle, and kernel-level entry points used by the parity tests.
#include <string>

#include "../../include/mapperatorinator_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace mb200 {
static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
long long g_launch_count = 0;
StepProfiler g_prof;
}  // namespace mb200

using namespace mb200;

struct mb200_mel {
    MelPlan* plan;
    mb200_mel_config cfg;
};

extern "C" int mb200_abi_version(void) { return MB200_ABI_VERSION; }
extern "C" int64_t mb200_launch_count(void) { return (int64_t)g_launch_count; }
extern "C" const char* mb200_last_error(void) { return g_last_error.c_str(); }

extern "C" int mb200_mel_create(mb200_mel** out, const mb200_mel_config* cfg, const float* mel_basis) {
    MB_REQUIRE(out && cfg && mel_basis, "null argument");
    MelPlan* plan = nullptr;
    int s = mel_plan_create(&plan, cfg->n_fft, cfg->hop_length, cfg->n_mels, cfg->pad_reflect, cfg->log_scale, mel_basis);
    if (s) return s;
    *out = new mb200_mel{plan, *cfg};
    return 0;
}

extern "C" void mb200_mel_destroy(mb200_mel* mel) {
    if (!mel) return;
    mel_plan_destroy(mel->plan);
    delete mel;
}

extern "C" int mb200_mel_forward(mb200_mel* mel, const float* pcm, int32_t batch, int32_t n_samples, float* out, void* stream) {
    MB_REQUIRE(mel && pcm && out, "null argument");
    const int frames = n_samples / mel->cfg.hop_length + 1;
    return launch_mel(mel->plan, pcm, n_samples, batch, n_samples, out, mel->cfg.n_mels, (long long)frames * mel->cfg.n_mels,
                      (cudaStream_t)stream);
}

extern "C" int mb200_op_gemm(const float* A, int64_t lda, const float* W, int64_t ldw, float* C, int64_t ldc, const float* bias, int32_t act,
                             float alpha, const float* residual, int64_t ldr, const float* gate, int64_t gate_ld, int32_t gate_rpb, int32_t M,
                             int32_t N, int32_t K, void* stream) {
    GemmParams g{};
    g.A = plain_map(A, lda); g.W = W; g.ldw = ldw; g.C = plain_map(C, ldc); g.bias = bias; g.act = act; g.alpha = alpha;
    g.gate = gate; g.gate_ld = gate_ld; g.gate_rpb = gate_rpb > 0 ? gate_rpb : 1;
    g.R = residual ? plain_map(residual, ldr) : RowMap{nullptr, 0, 0, 0};
    g.M = M; g.N = N; g.K = K;
    return launch_gemm(g, (cudaStream_t)stream, default_gemm_ctx());
}

extern "C" int mb200_op_gemm_tc(const float* A, int64_t lda, const float* W, int64_t ldw, float* C, int64_t ldc, const float* bias, int32_t act,
                                float alpha, const float* residual, int64_t ldr, int32_t M, int32_t N, int32_t K, void* stream) {
    GemmParams g{};
    g.A = plain_map(A, lda); g.W = W; g.ldw = ldw; g.C = plain_map(C, ldc); g.bias = bias; g.act = act; g.alpha = alpha;
    g.gate = nullptr; g.gate_ld = 0; g.gate_rpb = 1;
    g.R = residual ? plain_map(residual, ldr) : RowMap{nullptr, 0, 0, 0};
    g.M = M; g.N = N; g.K = K;
    GemmCtx* ctx = default_gemm_ctx();
    int s = ctx->register_weight(W, (long long)N * ldw);
    if (s) return s;
    if (!tc_gemm_eligible(g, ctx)) {
        ctx->unregister_weight(W);
        MB_REQUIRE(false, "problem not eligible for the wgmma path (M >= 512, K % 4 == 0, 16-byte aligned operands)");
    }
    s = launch_gemm_tc(g, (cudaStream_t)stream, ctx);
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
    ctx->unregister_weight(W);      // W belongs to the caller (a torch tensor whose address may be recycled)
    if (s) return s;
    MB_CUDA_CHECK(e);
    MB_REQUIRE(ctx->error() == 0, "wgmma GEMM pipeline wait timed out");
    return 0;
}

extern "C" int mb200_set_tensor_cores(int32_t enabled) { g_tc_enabled = enabled; return 0; }

extern "C" int mb200_op_layernorm(const float* x, float* y, const float* w, const float* b, const float* shift, const float* scale,
                                  int32_t rows_per_batch, int32_t rows, int32_t dim, float eps, void* stream) {
    LayerNormParams p{};
    p.x = x; p.ldx = dim; p.y = y; p.ldy = dim; p.weight = w; p.bias = b; p.shift = shift; p.scale = scale; p.mod_ld = dim;
    p.rows_per_batch = rows_per_batch > 0 ? rows_per_batch : 1; p.rows = rows; p.dim = dim; p.eps = eps;
    return launch_layernorm(p, (cudaStream_t)stream);
}

extern "C" int mb200_op_attention(const float* q, const float* k, const float* v, float* o, int32_t B, int32_t H, int32_t Tq, int32_t Tk,
                                  float scale, int32_t mask_mode, int32_t q_pos0, const uint8_t* key_valid, int32_t band,
                                  const uint8_t* dense_mask, void* stream) {
    AttentionParams a{};
    const long long D = (long long)H * 64;
    a.q = q; a.q_ld = D; a.q_bs = (long long)Tq * D;
    a.k = k; a.k_ld = D; a.k_bs = (long long)Tk * D;
    a.v = v; a.v_ld = D; a.v_bs = (long long)Tk * D;
    a.o = o; a.o_ld = D; a.o_bs = (long long)Tq * D;
    a.B = B; a.H = H; a.Tq = Tq; a.Tk = Tk; a.scale = scale; a.mask_mode = mask_mode; a.q_pos0 = q_pos0;
    a.key_valid = key_valid; a.key_valid_ld = Tk; a.band = band; a.dense = dense_mask; a.kv_slot = nullptr;
    static AttnCtx op_ctx;                    // scratch of this kernel-level test entry point
    const int rc = launch_attention(a, (cudaStream_t)stream, &op_ctx);
    if (rc) return rc;
    if (attn_tc_eligible(a, &op_ctx)) {       // surface a pipeline time-out of the tensor-core path as an error of the call
        MB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
        MB_REQUIRE(op_ctx.error() == 0, "tensor-core attention: a pipeline wait timed out");
    }
    return 0;
}
// tuning / tests: minimum query count for the tensor-core attention path (0 disables it)
extern "C" int mb200_set_attention_tc(int32_t enabled, int32_t min_queries) {
    g_attn_tc_enabled = enabled; g_attn_tc_min_t = min_queries;
    return 0;
}

// ---- audio ingest (SURVEY §8f N5) ----------------------------------------------------------------------------------------
extern "C" int64_t mb200_audio_out_frames(int64_t n_frames, int32_t in_rate, int32_t out_rate) {
    return (int64_t)mb200::audio_out_frames((long long)n_frames, in_rate, out_rate);
}
extern "C" int mb200_audio_ingest(const int16_t* pcm, int64_t n_frames, int32_t channels, int32_t in_rate, int32_t out_rate, int32_t normalize,
                                  float* out, int32_t* scratch, void* stream) {
    MB_REQUIRE(pcm && out && scratch, "null argument");
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return mb200::launch_audio_ingest(reinterpret_cast<const short*>(pcm), (long long)n_frames, channels, in_rate, out_rate, normalize, out,
                                      reinterpret_cast<int*>(scratch), sms, (cudaStream_t)stream);
}
