// C-ABI glue: error channel, the mel stage handle, and kernel-level entry points used by the parity tests.
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/mapperatorinator_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace mb200 {
static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
long long g_launch_count = 0;
long long g_wbf16_launch_count = 0;
StepProfiler g_prof;
}  // namespace mb200

using namespace mb200;
#define OP_TRY(expr) do { int _s = (expr); if (_s) return _s; } while (0)

struct mb200_mel {
    MelPlan* plan;
    mb200_mel_config cfg;
};

extern "C" int mb200_abi_version(void) { return MB200_ABI_VERSION; }
extern "C" int64_t mb200_launch_count(void) { return (int64_t)g_launch_count; }
extern "C" int64_t mb200_wbf16_launch_count(void) { return (int64_t)g_wbf16_launch_count; }
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

// One dense GEMM through the engine's own launch functions, with GemmParams filled from row maps as the encoder, the decoder prefill and
// the DiT fill them.  path 0: W gets a tf32 mirror as finalize gives the weights it registers, and launch_gemm picks what the engine would
// pick; 1: no mirror, so launch_gemm runs the fp32 SIMT kernel; 2: launch_gemm_tc, or an error naming why the problem is not eligible.
extern "C" int mb200_op_gemm_mapped(const mb200_rowmap* A, const float* W, int64_t ldw, const mb200_rowmap* C, const float* bias, int32_t act,
                                    float alpha, const mb200_rowmap* R, const float* gate, int64_t gate_ld, int32_t gate_rpb, int32_t M,
                                    int32_t N, int32_t K, int32_t path, void* stream) {
    MB_REQUIRE(A && A->ptr && W && C && C->ptr && (!R || R->ptr), "null argument");
    MB_REQUIRE(path >= 0 && path <= 2, "path is 0 (engine dispatch), 1 (SIMT) or 2 (tensor cores)");
    MB_REQUIRE(M >= 1 && N >= 1 && K >= 4 && K % 4 == 0, "need M >= 1, N >= 1 and K a positive multiple of 4");
    MB_REQUIRE(act >= ACT_NONE && act <= ACT_SILU, "unknown activation");
    for (const mb200_rowmap* m : {A, C, R}) {
        if (!m) continue;
        MB_REQUIRE(m->ld >= 1 && m->rpb >= 0 && m->bstride >= 0, "a row map needs ld >= 1, rpb >= 0 and bstride >= 0");
        MB_REQUIRE(m->rpb == 0 || m->rpb <= M, "a row map's rows per batch exceed M");
    }
    MB_REQUIRE(A->rpb == 0 || M % A->rpb == 0, "A's rows per batch must divide M (whole batches are read)");
    MB_REQUIRE(A->ld % 4 == 0 && (A->rpb == 0 || A->bstride % 4 == 0) && ldw % 4 == 0, "A and W row strides must be multiples of 4 floats");
    MB_REQUIRE(ldw >= K, "W's row stride is shorter than K");
    MB_REQUIRE(C->ld >= N && (!R || R->ld >= N), "an output or residual row stride is shorter than N");
    MB_REQUIRE(reinterpret_cast<uintptr_t>(A->ptr) % 16 == 0 && reinterpret_cast<uintptr_t>(W) % 16 == 0, "A and W must be 16-byte aligned");
    MB_REQUIRE(!gate || (gate_rpb >= 1 && gate_ld >= N), "a gate needs gate_rpb >= 1 and gate_ld >= N");
    GemmParams g{};
    g.A = batched_map(A->ptr, A->ld, A->rpb, A->bstride); g.W = W; g.ldw = ldw;
    g.C = batched_map(C->ptr, C->ld, C->rpb, C->bstride); g.bias = bias; g.act = act; g.alpha = alpha;
    g.gate = gate; g.gate_ld = gate ? gate_ld : 0; g.gate_rpb = gate ? gate_rpb : 1;
    g.R = R ? batched_map(R->ptr, R->ld, R->rpb, R->bstride) : RowMap{nullptr, 0, 0, 0};
    g.M = M; g.N = N; g.K = K;
    GemmCtx* ctx = default_gemm_ctx();
    if (path == 2) {      // eligibility apart from the mirror, judged before anything is launched
        const bool had = ctx->mirrors.count(W) != 0;
        if (!had) ctx->mirrors[W] = Tf32Mirror{nullptr, nullptr};
        const bool ok = tc_gemm_eligible(g, ctx);
        if (!had) ctx->mirrors.erase(W);
        MB_REQUIRE(ok, "problem not eligible for the wgmma path (tensor cores on, M >= 512, N >= 64, K >= 32, K % 4 == 0, A rows per batch a "
                       "multiple of 128, 16-byte aligned operands and strides)");
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (path != 1) OP_TRY(ctx->register_weight(W, (long long)(N - 1) * ldw + K));
    int s = path == 2 ? launch_gemm_tc(g, st, ctx) : launch_gemm(g, st, ctx);
    const cudaError_t e = cudaStreamSynchronize(st);
    ctx->unregister_weight(W);      // W belongs to the caller (a torch tensor whose address may be recycled)
    if (s) return s;
    MB_CUDA_CHECK(e);
    MB_REQUIRE(ctx->error() == 0, "wgmma GEMM pipeline wait timed out");
    return 0;
}

extern "C" int mb200_set_tensor_cores(int32_t enabled) { g_tc_enabled = enabled; return 0; }

extern "C" int mb200_op_layernorm(const float* x, float* y, const float* w, const float* b, const float* shift, const float* scale,
                                  int64_t mod_ld, int32_t rows_per_batch, int32_t rows, int32_t dim, float eps, void* stream) {
    MB_REQUIRE(x && y, "null argument");
    MB_REQUIRE(!shift == !scale, "modulate needs both shift and scale");
    MB_REQUIRE(!shift || mod_ld == 0 || mod_ld >= dim, "mod_ld is shorter than a row");
    LayerNormParams p{};
    p.x = x; p.ldx = dim; p.y = y; p.ldy = dim; p.weight = w; p.bias = b; p.shift = shift; p.scale = scale; p.mod_ld = mod_ld > 0 ? mod_ld : dim;
    p.rows_per_batch = rows_per_batch > 0 ? rows_per_batch : 1; p.rows = rows; p.dim = dim; p.eps = eps;
    return launch_layernorm(p, (cudaStream_t)stream);
}

extern "C" int mb200_op_attention(const float* q, int64_t q_ld, int64_t q_bs, const float* k, int64_t k_ld, int64_t k_bs, const float* v,
                                  int64_t v_ld, int64_t v_bs, float* o, int64_t o_ld, int64_t o_bs, int32_t B, int32_t H, int32_t Tq, int32_t Tk,
                                  float scale, int32_t mask_mode, int32_t q_pos0, const uint8_t* key_valid, int64_t key_valid_ld, int32_t band,
                                  const uint8_t* dense_mask, const int32_t* kv_slot, void* stream) {
    MB_REQUIRE(q && k && v && o, "null argument");
    MB_REQUIRE(B >= 1 && H >= 1 && Tq >= 1 && Tk >= 1, "need B, H, Tq and Tk >= 1");
    MB_REQUIRE(mask_mode >= MASK_NONE && mask_mode <= MASK_DENSE, "unknown mask mode");
    MB_REQUIRE(mask_mode != MASK_DENSE || dense_mask, "a dense mask mode needs the mask");
    MB_REQUIRE(!key_valid || key_valid_ld >= Tk, "key_valid_ld is shorter than Tk");
    const long long D = (long long)H * 64;
    MB_REQUIRE(q_ld >= D && k_ld >= D && v_ld >= D && o_ld >= D, "a token stride is shorter than H * 64");
    MB_REQUIRE(q_bs >= 0 && k_bs >= 0 && v_bs >= 0 && o_bs >= 0, "negative batch stride");
    for (const void* ptr : {(const void*)q, (const void*)k, (const void*)v, (const void*)o})
        MB_REQUIRE(reinterpret_cast<uintptr_t>(ptr) % 16 == 0, "q, k, v and o are read and written as float4: 16-byte alignment");
    MB_REQUIRE(q_ld % 4 == 0 && k_ld % 4 == 0 && v_ld % 4 == 0 && o_ld % 4 == 0 && q_bs % 4 == 0 && k_bs % 4 == 0 && v_bs % 4 == 0 &&
                   o_bs % 4 == 0, "attention strides must be multiples of 4");
    AttentionParams a{};
    a.q = q; a.q_ld = q_ld; a.q_bs = q_bs;
    a.k = k; a.k_ld = k_ld; a.k_bs = k_bs;
    a.v = v; a.v_ld = v_ld; a.v_bs = v_bs;
    a.o = o; a.o_ld = o_ld; a.o_bs = o_bs;
    a.B = B; a.H = H; a.Tq = Tq; a.Tk = Tk; a.scale = scale; a.mask_mode = mask_mode; a.q_pos0 = q_pos0;
    a.key_valid = key_valid; a.key_valid_ld = key_valid_ld; a.band = band; a.dense = dense_mask; a.kv_slot = kv_slot;
    static AttnCtx op_ctx;                    // scratch of this kernel-level test entry point
    const int rc = launch_attention(a, (cudaStream_t)stream, &op_ctx);
    if (rc) return rc;
    if (attn_tc_eligible(a, &op_ctx)) {       // surface a pipeline time-out of the tensor-core path as an error of the call
        MB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
        MB_REQUIRE(op_ctx.error() == 0, "tensor-core attention: a pipeline wait timed out");
    }
    return 0;
}

// One decode-attention phase through launch_decode_attention / launch_decode_attention_ragged, with the scratch a token step gives them
// (call state, split partials, tickets) owned here.
namespace {
struct OpScratch {
    void* p = nullptr; size_t bytes = 0;
    int ensure(size_t need) {
        if (need <= bytes) return 0;
        if (p) cudaFree(p);
        p = nullptr; bytes = 0;
        MB_CUDA_CHECK(cudaMalloc(&p, need));
        bytes = need;
        return 0;
    }
};
}  // namespace

extern "C" int mb200_op_decode_attention(const float* q, const float* kv, int32_t slots, int32_t t_max, int32_t H, int32_t rows,
                                         const int32_t* row_slot, int32_t cur_len, int32_t prompt_len, const uint8_t* key_valid,
                                         int64_t key_valid_ld, int32_t max_length, int32_t fixed_len, const int32_t* kv_src, int64_t kv_src_ld,
                                         const int32_t* ragged_cur_len, const int32_t* ragged_max_length, int32_t form, float* out,
                                         void* stream) {
    MB_REQUIRE(q && kv && out, "null argument");
    MB_REQUIRE(rows >= 1 && H >= 1 && slots >= 1 && t_max >= 1, "rows, heads, slots and cache length must be positive");
    const bool ragged = ragged_cur_len != nullptr;
    MB_REQUIRE(ragged == (ragged_max_length != nullptr), "a ragged call gives both per-row cur_len and max_length");
    MB_REQUIRE(!ragged || (fixed_len == 0 && !kv_src && form == ATTN_FORM_DEFAULT), "the ragged kernel is self attention without a table");
    MB_REQUIRE(!kv_src || fixed_len == 0, "the source-row table applies to self attention");
    const long long d = (long long)H * 64;
    DecAttnParams a{};
    a.q = q; a.q_ld = d; a.kc = kv; a.vc = kv + d; a.row_stride = (long long)t_max * 2 * d; a.tok_stride = 2 * d;
    a.key_valid = key_valid; a.key_valid_ld = key_valid_ld;
    a.kv_src = kv_src; a.kv_src_ld = kv_src_ld;
    a.rows = rows; a.H = H; a.out = out; a.out_ld = d;
    GenState gs{};
    std::vector<RowState> rs;
    if (ragged) {
        gs.n_req = rows;
        rs.resize(rows);
        int S = 1;
        for (int r = 0; r < rows; ++r) {
            MB_REQUIRE(ragged_cur_len[r] >= 1 && ragged_cur_len[r] <= ragged_max_length[r] && ragged_max_length[r] <= t_max,
                       "need 1 <= cur_len <= max_length <= cache length in every row");
            rs[r].cur_len = ragged_cur_len[r]; rs[r].prompt_len = 0; rs[r].max_length = ragged_max_length[r];
            S = std::max(S, self_splits(ragged_max_length[r]));
        }
        MB_REQUIRE(!row_slot, "a ragged row reads its own cache row");
        a.n_splits = S;                                  // the grid: the largest plan of the call
        a.chunk = self_split_chunk(S);                   // (not read by the ragged kernel)
    } else if (fixed_len > 0) {
        MB_REQUIRE(fixed_len <= t_max, "fixed_len exceeds the cache length");
        a.fixed_len = fixed_len; a.chunk = 64; a.n_splits = (fixed_len + 63) / 64;      // cross attention: 64-key splits
        gs.prompt_len = prompt_len;
    } else {
        MB_REQUIRE(cur_len >= 1 && cur_len <= max_length && max_length <= t_max, "need 1 <= cur_len <= max_length <= cache length");
        MB_REQUIRE(prompt_len >= 0 && prompt_len <= cur_len, "need 0 <= prompt_len <= cur_len");
        a.n_splits = self_splits(max_length);
        a.chunk = self_split_chunk(a.n_splits);
        gs.cur_len = cur_len; gs.prompt_len = prompt_len; gs.max_length = max_length;
    }
    a.row_slot = row_slot;
    cudaStream_t st = (cudaStream_t)stream;
    static OpScratch op_state, op_parts, op_tickets;
    const size_t n_units = (size_t)rows * H * a.n_splits;
    OP_TRY(op_state.ensure(sizeof(GenState) + (size_t)rows * sizeof(RowState)));
    OP_TRY(op_parts.ensure(n_units * 66 * sizeof(float)));
    OP_TRY(op_tickets.ensure((size_t)rows * H * sizeof(int)));
    MB_CUDA_CHECK(cudaMemcpyAsync(op_state.p, &gs, sizeof(GenState), cudaMemcpyHostToDevice, st));
    if (ragged) MB_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<GenState*>(op_state.p) + 1, rs.data(), rs.size() * sizeof(RowState), cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaMemsetAsync(op_tickets.p, 0, (size_t)rows * H * sizeof(int), st));
    a.st = reinterpret_cast<const GenState*>(op_state.p);
    a.part_o = reinterpret_cast<float*>(op_parts.p); a.part_ml = a.part_o + n_units * 64;
    a.ticket = reinterpret_cast<int*>(op_tickets.p);
    OP_TRY(ragged ? launch_decode_attention_ragged(a, st, false) : launch_decode_attention(a, st, false, form));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));      // the host-side state above goes out of scope
    return 0;
}

// One GEMV phase through launch_gemv, with the GemvParams a token step builds and the call state (GenState, RowStates) owned here.
// w_bf16: W holds bf16 bits (the token loop's bf16 store).
static int op_gemv(const float* x, int64_t x_ld, int32_t B, int32_t K, int32_t xmode, const float* ln_w, const float* ln_b, float eps,
                   const void* W, bool w_bf16, int64_t ldw, int32_t N, const float* bias, const float* R, int64_t r_ld,
                   const mb200_gemv_seg* segs, int32_t nseg, int32_t cur_len, const int32_t* ragged_cur_len,
                   const int32_t* ragged_finished, int32_t n_req, int32_t form, void* stream) {
    MB_REQUIRE(x && W && segs, "null argument");
    MB_REQUIRE(B >= 1 && N >= 1 && K >= 4, "need B >= 1, N >= 1, K >= 4");
    MB_REQUIRE(x_ld >= K && ldw >= K && (!R || r_ld >= N), "a row stride is shorter than its row");
    MB_REQUIRE(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(W) % 16 == 0, "x and W are read as float4");
    MB_REQUIRE(!w_bf16 || (K % 8 == 0 && ldw % 8 == 0), "bf16 weights are read 4 at a time from 16-byte rows: K and ldw must be multiples of 8");
    MB_REQUIRE(xmode == X_PLAIN || xmode == X_LAYERNORM, "unknown input mode");
    MB_REQUIRE(xmode != X_LAYERNORM || (ln_w && ln_b), "a LayerNorm input needs its weight and bias");
    MB_REQUIRE(nseg >= 1 && nseg <= 3, "1 to 3 output segments");
    const bool ragged = ragged_cur_len != nullptr;
    MB_REQUIRE(ragged == (ragged_finished != nullptr), "a ragged call gives both per-row cur_len and finished");
    bool positional = false;
    GemvParams g{};
    g.xmode = xmode; g.x = x; g.x_ld = x_ld; g.ln_w = ln_w; g.ln_b = ln_b; g.eps = eps;
    g.W = reinterpret_cast<const float*>(W); g.ldw = ldw; g.bias = bias; g.K = K; g.N = N; g.B = B; g.R = R; g.r_ld = r_ld;
    g.nseg = nseg;
    for (int i = 0; i < nseg; ++i) {
        const mb200_gemv_seg& s = segs[i];
        MB_REQUIRE(s.out, "a segment without an output");
        MB_REQUIRE(s.n_begin == (i ? segs[i - 1].n_end : 0) && s.n_begin < s.n_end && (i + 1 < nseg || s.n_end == N),
                   "the segments must tile [0, N) in order");
        MB_REQUIRE(s.act >= ACT_NONE && s.act <= ACT_SILU, "unknown activation");
        positional = positional || s.pos_stride != 0;
        g.seg[i] = GemvSeg{s.out, s.out_bs, s.pos_stride, s.n_begin, s.n_end, s.alpha, s.act};
    }
    GenState gs{};
    std::vector<RowState> rs;
    if (ragged) {
        MB_REQUIRE(n_req >= 1 && n_req <= B, "need 1 <= n_req <= B");
        gs.n_req = n_req;
        rs.resize(n_req);
        for (int r = 0; r < n_req; ++r) {
            MB_REQUIRE(ragged_cur_len[r] >= 1, "need cur_len >= 1 in every row");
            MB_REQUIRE(ragged_finished[r] == 0 || ragged_finished[r] == 1, "finished is 0 or 1");
            rs[r].cur_len = ragged_cur_len[r]; rs[r].finished = ragged_finished[r];
        }
    } else {
        MB_REQUIRE(!positional || cur_len >= 1, "a segment that writes at the cache position needs cur_len >= 1");
        gs.cur_len = cur_len;
    }
    cudaStream_t st = (cudaStream_t)stream;
    static OpScratch op_state;
    OP_TRY(op_state.ensure(sizeof(GenState) + rs.size() * sizeof(RowState)));
    MB_CUDA_CHECK(cudaMemcpyAsync(op_state.p, &gs, sizeof(GenState), cudaMemcpyHostToDevice, st));
    if (ragged) MB_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<GenState*>(op_state.p) + 1, rs.data(), rs.size() * sizeof(RowState), cudaMemcpyHostToDevice, st));
    g.st = reinterpret_cast<const GenState*>(op_state.p);
    const int rc = launch_gemv(g, st, false, ragged, form, w_bf16);     // also where the shape requirements of the kernels are checked
    MB_CUDA_CHECK(cudaStreamSynchronize(st));      // the host-side state above goes out of scope
    return rc;
}

extern "C" int mb200_op_gemv(const float* x, int64_t x_ld, int32_t B, int32_t K, int32_t xmode, const float* ln_w, const float* ln_b,
                             float eps, const float* W, int64_t ldw, int32_t N, const float* bias, const float* R, int64_t r_ld,
                             const mb200_gemv_seg* segs, int32_t nseg, int32_t cur_len, const int32_t* ragged_cur_len,
                             const int32_t* ragged_finished, int32_t n_req, int32_t form, void* stream) {
    return op_gemv(x, x_ld, B, K, xmode, ln_w, ln_b, eps, W, false, ldw, N, bias, R, r_ld, segs, nseg, cur_len, ragged_cur_len, ragged_finished,
                   n_req, form, stream);
}

extern "C" int mb200_op_gemv_bf16(const float* x, int64_t x_ld, int32_t B, int32_t K, int32_t xmode, const float* ln_w, const float* ln_b,
                                  float eps, const uint16_t* W, int64_t ldw, int32_t N, const float* bias, const float* R, int64_t r_ld,
                                  const mb200_gemv_seg* segs, int32_t nseg, int32_t cur_len, const int32_t* ragged_cur_len,
                                  const int32_t* ragged_finished, int32_t n_req, int32_t form, void* stream) {
    return op_gemv(x, x_ld, B, K, xmode, ln_w, ln_b, eps, W, true, ldw, N, bias, R, r_ld, segs, nseg, cur_len, ragged_cur_len, ragged_finished,
                   n_req, form, stream);
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
