// Host runtime of the osuT5 stage: weights, resident encoder/cross-KV slots, self-KV arena, encoder pass, decoder
// prefill, CUDA-graph token loop.  Mirrors what `server.model_generate` drives through HF `generate`
// (osuT5/osuT5/inference/server.py:83-156) — see include/mapperatorinator_b200.h for the boundary.
#include <algorithm>
#include <climits>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/mapperatorinator_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace mb200;

namespace {

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    int ensure(size_t need, bool zero = false) {
        if (need <= bytes) return 0;
        if (p) cudaFree(p);
        p = nullptr; bytes = 0;
        MB_CUDA_CHECK(cudaMalloc(&p, need));
        bytes = need;
        if (zero) MB_CUDA_CHECK(cudaMemset(p, 0, need));
        return 0;
    }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
    ~DevBuf() { if (p) cudaFree(p); }
};

struct LayerW {   // device pointers into the weight arena
    const float *ln1_w, *ln1_b, *wqkv, *bqkv, *wo, *bo;
    const float *ln2_w, *ln2_b, *wq_c, *bq_c, *wkv_c, *bkv_c, *wo_c, *bo_c;   // decoder cross attention only
    const float *ln3_w, *ln3_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
    // decoder only: the same packed matrices in the bf16 token-loop arena (bf16 bits behind a float pointer, as GemvParams::W carries
    // them), null when the engine has no bf16 store
    const float *wqkv16, *wo16, *wq_c16, *wo_c16, *fc1_w16, *fc2_w16;
};

}  // namespace

struct mb200_model {
    mb200_model_config cfg;
    MelPlan* mel = nullptr;
    std::unordered_map<std::string, std::vector<float>> host_w;   // until finalize()
    std::unordered_set<std::string> bf16_names;                   // weights that arrived as bf16 (until finalize())
    bool finalized = false;

    DevBuf arena;                       // all packed weights
    DevBuf arena16;                     // bf16 copies of the token loop's GEMV matrices (empty: the token loop reads the fp32 arena)
    const float* proj_out16 = nullptr;  // bf16 bits of proj_out in arena16
    const float *emb_w = nullptr, *emb_b = nullptr, *conv1_w = nullptr, *conv1_b = nullptr, *conv2_w = nullptr, *conv2_b = nullptr,
                *enc_pos = nullptr, *enc_ln_w = nullptr, *enc_ln_b = nullptr;
    const float *tok_emb = nullptr, *dec_pos = nullptr, *dec_ln_w = nullptr, *dec_ln_b = nullptr, *proj_out = nullptr;
    std::vector<LayerW> enc, dec;

    DevBuf cross_kv;                    // [dec_layers][max_windows][Ts][2d]   (k | v per token)
    DevBuf self_kv;                     // [dec_layers][max_rows][tgt][2d]
    int max_rows = 0;

    // encoder workspaces (chunk of windows)
    int enc_chunk = 0;
    DevBuf w_mel, w_embpad, w_c1pad, w_x, w_h, w_qkv, w_attn, w_ffn;
    // decoder workspaces
    DevBuf p_x, p_h, p_q, p_attn, p_ffn;          // prefill, sized rows * P
    DevBuf d_x, d_q, d_h, d_parto, d_partml, d_logits;   // decode step
    DevBuf d_attn, d_ticket;            // merged attention heads [rows, d] and the per-(row, head) arrival counters of the split merge
    DevBuf g_state, g_cfg, g_vflags, g_ids, g_prefill_ids, g_keyvalid, g_leftpad, g_rowslot, g_finished, g_lastts, g_lastscores;
    int* h_flag = nullptr;              // pinned
    unsigned char* h_stage = nullptr;   // pinned staging of a call's state (prompt ids, masks, slots, flags, GenState, SampleConfig, ...)
    size_t h_stage_bytes = 0;
    cudaEvent_t stage_ev = nullptr;     // recorded behind the staging copies: h_stage may be refilled once it has completed
    // graph keys carry B as well as rows: the captured sample kernel's grid is dim3(B), and a CFG call (B = 1, rows = 2) must
    // never replay the graph of a plain batch-2 call (B = 2, rows = 2)
    // ... and the beam count: a beam call ends its token step in the beam kernels and must never replay a greedy graph of equal rows
    std::map<std::tuple<int, int, int, int>, CapturedGraph> graphs;   // (rows, B, n_splits_self, num_beams) -> token-step graph
    bool use_pdl = false;
    cudaStream_t cap_stream = nullptr;
    std::map<std::tuple<int, int, int, int>, int> prefill_seen;                                   // (rows, B, P, position rule)
    std::map<std::tuple<int, int, int, int>, CapturedGraph> prefill_graphs;
    // persistent megakernel path
    int enc_graph = 1;                  // replay single-window encodes as a CUDA graph (option "enc_graph")
    int trace_cta = 0;                  // CTA whose phases the dataflow megakernel's TRACE instantiation stamps
    int use_mega = 2;                   // 0 = CUDA-graph replay per token, 1 = grid-barrier megakernel, 2 = dataflow (tagged-pair) megakernel
    DevBuf ll_arena;                    // exchange buffers of the dataflow megakernel (rows <= 2)
    MegaLL ll{};
    size_t ll_bytes = 0;
    // (driver, rows, B, n_splits_self) -> the megakernel's device phase table and its length
    std::map<std::tuple<int, int, int, int>, std::pair<std::unique_ptr<DevBuf>, int>> phase_tables;
    int num_sms = 0;                    // 0 = no cooperative launch -> no megakernel
    int num_sms_phys = 0;
    DevBuf g_megasync;                  // [0] grid-barrier counter, [8] error flag
    DevBuf mega_trace;                  // optional per-phase clock64 stamps (option "mega_trace")
    cudaEvent_t mega_ev[2] = {nullptr, nullptr};
    double mega_ms = 0.0; long long mega_launches = 0, mega_tokens = 0;   // CUDA-event time of every megakernel launch
    DevBuf w_pcm;                       // single-window encode: engine-owned copy of the window's PCM (the captured graph reads it)
    std::map<int, CapturedGraph> enc_graphs;   // slot -> captured single-window encode (the drop-in per-call pattern)
    std::map<int, int> enc_seen;
    // beam search state (allocated at the first beam call for max_batch rows, then fixed: captured graphs hold the pointers)
    DevBuf b_kvsrc, b_logprobs, b_cand, b_runscore, b_finids[2], b_finscore, b_finlen, b_finflag, b_unsat;
    DevBuf b_dbg;                       // beam-step parity hook outputs
    AttnCtx attn;                       // tensor-core attention scratch of the encoder (head-major tf32 copies of q | k | v^T)
    GemmCtx gemm;                       // this engine's GEMM scratch: split-K planes, tf32 activation copies, weight mirrors, error flag
    DevBuf s_logits;                    // token scoring: one chunk of vocabulary-projection rows [<= SCORE_CHUNK_ROWS, V]
    mb200_stream* live_stream = nullptr; // the open decode stream: it owns g_state, g_ids and the logits rows until closed

    int d() const { return cfg.d_model; }
    int Ts() const { return cfg.src_seq_len / 2; }
    size_t cross_layer_stride() const { return (size_t)cfg.max_windows * Ts() * 2 * d(); }
    size_t self_layer_stride() const { return (size_t)max_rows * cfg.tgt_seq_len * 2 * d(); }
};

namespace {

std::vector<std::string> required_names(const mb200_model_config& c) {
    std::vector<std::string> n = {
        "encoder_embedder.weight", "encoder_embedder.bias", "decoder_embedder.weight",
        "transformer.model.encoder.conv1.weight", "transformer.model.encoder.conv1.bias",
        "transformer.model.encoder.conv2.weight", "transformer.model.encoder.conv2.bias",
        "transformer.model.encoder.embed_positions.weight",
        "transformer.model.encoder.layer_norm.weight", "transformer.model.encoder.layer_norm.bias",
        "transformer.model.decoder.embed_positions.weight",
        "transformer.model.decoder.layer_norm.weight", "transformer.model.decoder.layer_norm.bias",
        "transformer.proj_out.weight"};
    auto attn = [&](const std::string& p) {
        n.push_back(p + "q_proj.weight"); n.push_back(p + "q_proj.bias"); n.push_back(p + "k_proj.weight");
        n.push_back(p + "v_proj.weight"); n.push_back(p + "v_proj.bias");
        n.push_back(p + "out_proj.weight"); n.push_back(p + "out_proj.bias");
    };
    auto ln = [&](const std::string& p) { n.push_back(p + "weight"); n.push_back(p + "bias"); };
    for (int side = 0; side < 2; ++side) {
        int L = side == 0 ? c.encoder_layers : c.decoder_layers;
        for (int i = 0; i < L; ++i) {
            std::string p = std::string("transformer.model.") + (side == 0 ? "encoder" : "decoder") + ".layers." + std::to_string(i) + ".";
            attn(p + "self_attn."); ln(p + "self_attn_layer_norm.");
            if (side == 1) { attn(p + "encoder_attn."); ln(p + "encoder_attn_layer_norm."); }
            n.push_back(p + "fc1.weight"); n.push_back(p + "fc1.bias"); n.push_back(p + "fc2.weight"); n.push_back(p + "fc2.bias");
            ln(p + "final_layer_norm.");
        }
    }
    return n;
}

GemmParams gemm_base(const RowMap& A, const float* W, long long ldw, const RowMap& C, const float* bias, int M, int N, int K) {
    GemmParams g{};
    g.A = A; g.W = W; g.ldw = ldw; g.C = C; g.bias = bias; g.act = ACT_NONE; g.alpha = 1.f;
    g.gate = nullptr; g.gate_ld = 0; g.gate_rpb = 1; g.R = RowMap{nullptr, 0, 0, 0};
    g.M = M; g.N = N; g.K = K;
    return g;
}

#define MB_TRY(expr) do { int _s = (expr); if (_s) return _s; } while (0)

int layernorm(const float* x, float* y, const float* w, const float* b, int rows, int dim, float eps, cudaStream_t st) {
    LayerNormParams p{};
    p.x = x; p.ldx = dim; p.y = y; p.ldy = dim; p.weight = w; p.bias = b; p.shift = nullptr; p.scale = nullptr; p.mod_ld = 0;
    p.rows_per_batch = 1; p.rows = rows; p.dim = dim; p.eps = eps;
    return launch_layernorm(p, st);
}

// Every call that writes the token loop's state (ids, GenState, SampleConfig, flag rows, logits rows, token-step graphs) refuses while a
// decode stream owns that state.
int token_loop_free(const mb200_model* m) {
    MB_REQUIRE(!m->live_stream, "a decode stream is open on this engine: close it first");
    return 0;
}

// A call's host state leaves from the engine's pinned staging buffer, so its copies are asynchronous and the launches behind them
// queue with no host wait.  One use: begin() waits until the previous use's copies have left the buffer; reserve() every record and
// check fits(), so that the capacity is checked before the first copy; fill the records; upload() each; end() records the event
// begin() waits for.
struct Stager {
    mb200_model* m;
    cudaStream_t st;
    size_t off = 0;
    int begin() {
        MB_CUDA_CHECK(cudaEventSynchronize(m->stage_ev));
        off = 0;
        return 0;
    }
    template <typename T> T* reserve(size_t n) {      // n elements, 16-byte aligned; past the capacity only fits() may be called
        off = (off + 15) & ~size_t(15);
        T* rec = reinterpret_cast<T*>(m->h_stage + off);
        off += n * sizeof(T);
        return rec;
    }
    int fits() const {
        MB_REQUIRE(off <= m->h_stage_bytes, "call state exceeds the staging buffer");
        return 0;
    }
    template <typename T> int upload(void* dst, const T* rec, size_t n) {
        MB_CUDA_CHECK(cudaMemcpyAsync(dst, rec, n * sizeof(T), cudaMemcpyHostToDevice, st));
        return 0;
    }
    int end() {
        MB_CUDA_CHECK(cudaEventRecord(m->stage_ev, st));
        return 0;
    }
};

// The prefill rows of a prompt call.  Row r holds item item_of(r) of `prompt` (of `neg_prompt` for the first n_neg rows, masked by
// `neg_mask` when given, else by `mask`): its P ids in pre [rows, P], its key mask in keyvalid [rows, tgt_seq_len] (1 from P on), the
// count of its leading masked keys in leftpad [rows] and its item's encoder slot in rowslot [rows].  Every slot and every token id is
// checked before any record is written.
template <typename ItemOf>
int build_prompt_rows(const mb200_model* m, int rows, int P, ItemOf item_of, int n_neg, const int32_t* slots, const int64_t* prompt,
                      const uint8_t* mask, const int64_t* neg_prompt, const uint8_t* neg_mask, long long* pre, unsigned char* keyvalid,
                      int* leftpad, int* rowslot) {
    const auto& c = m->cfg;
    const int ids_ld = c.tgt_seq_len;
    for (int r = 0; r < rows; ++r) {
        const int b = item_of(r);
        const int64_t* src = (r < n_neg ? neg_prompt : prompt) + (size_t)b * P;
        MB_REQUIRE(slots[b] >= 0 && slots[b] < c.max_windows, "encoder slot out of range");
        for (int t = 0; t < P; ++t) MB_REQUIRE(src[t] >= 0 && src[t] < c.vocab_size_in, "token id out of range");
    }
    for (int r = 0; r < rows; ++r) {
        const int b = item_of(r);
        const int64_t* src = (r < n_neg ? neg_prompt : prompt) + (size_t)b * P;
        const uint8_t* msk = r < n_neg && neg_mask ? neg_mask : mask;
        unsigned char* kv = keyvalid + (size_t)r * ids_ld;
        std::memset(kv, 1, ids_ld);
        int npad = 0; bool seen = false;
        for (int t = 0; t < P; ++t) {
            pre[(size_t)r * P + t] = src[t];
            kv[t] = msk ? (msk[(size_t)b * P + t] != 0) : 1;
            if (!kv[t] && !seen) ++npad; else seen = true;
        }
        leftpad[r] = npad;
        rowslot[r] = slots[b];
    }
    return 0;
}

}  // namespace

// =====================================================================================================================
extern "C" int mb200_model_create(mb200_model** out, const mb200_model_config* cfg, const float* mel_basis_host) {
    MB_REQUIRE(cfg && out, "null argument");
    MB_REQUIRE(cfg->d_model == cfg->heads * 64, "kernels are specialised for head_dim 64 (whisper-small: 768 / 12)");
    MB_REQUIRE(cfg->d_model % 128 == 0 && cfg->d_model <= 1024, "d_model must be a multiple of 128 and <= 1024");
    MB_REQUIRE(cfg->vocab_size_out <= 4096, "fused sampling kernel holds the vocabulary in shared memory (<= 4096 ids)");
    MB_REQUIRE(cfg->mel.n_mels % 4 == 0 && cfg->ffn_dim % 4 == 0, "n_mels / ffn_dim must be multiples of 4");
    mb200_model* m = new mb200_model();
    m->cfg = *cfg;
    int s = mel_plan_create(&m->mel, cfg->mel.n_fft, cfg->mel.hop_length, cfg->mel.n_mels, cfg->mel.pad_reflect, cfg->mel.log_scale,
                            mel_basis_host);
    if (s) { delete m; return s; }
    if (cudaMallocHost(&m->h_flag, 64) != cudaSuccess) { delete m; set_last_error("cudaMallocHost failed"); return 1; }
    {
        int dev = 0, coop = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&m->num_sms, cudaDevAttrMultiProcessorCount, dev);
        m->num_sms_phys = m->num_sms;
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
        if (!coop) m->num_sms = 0;
    }
    *out = m;
    return 0;
}

extern "C" void mb200_model_destroy(mb200_model* m) {
    if (!m) return;
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second.exec);
    for (auto& g : m->prefill_graphs) cudaGraphExecDestroy(g.second.exec);
    for (auto& g : m->enc_graphs) cudaGraphExecDestroy(g.second.exec);
    m->gemm.destroy();
    m->attn.destroy();
    for (auto& e : m->mega_ev) if (e) cudaEventDestroy(e);
    if (m->cap_stream) cudaStreamDestroy(m->cap_stream);
    mel_plan_destroy(m->mel);
    if (m->h_flag) cudaFreeHost(m->h_flag);
    if (m->h_stage) cudaFreeHost(m->h_stage);
    if (m->stage_ev) cudaEventDestroy(m->stage_ev);
    delete m;
}

extern "C" int mb200_model_set_weight(mb200_model* m, const char* name, const float* data, int64_t numel) {
    MB_REQUIRE(m && name && data, "null argument");
    MB_REQUIRE(!m->finalized, "model already finalized");
    m->host_w[name] = std::vector<float>(data, data + numel);
    m->bf16_names.erase(name);
    return 0;
}

extern "C" int mb200_model_set_weight_bf16(mb200_model* m, const char* name, const uint16_t* bits, int64_t numel) {
    MB_REQUIRE(m && name && bits, "null argument");
    MB_REQUIRE(!m->finalized, "model already finalized");
    std::vector<float> w((size_t)numel);
    for (int64_t i = 0; i < numel; ++i) {       // widening bf16 to fp32 is exact: the bits move to the top half
        const uint32_t u = (uint32_t)bits[i] << 16;
        std::memcpy(&w[(size_t)i], &u, 4);
    }
    m->host_w[name] = std::move(w);
    m->bf16_names.insert(name);
    return 0;
}

extern "C" int mb200_model_token_weight_bytes(const mb200_model* m, int32_t* bytes) {
    MB_REQUIRE(m && bytes, "null argument");
    MB_REQUIRE(m->finalized, "model not finalized");
    *bytes = m->arena16.p ? 2 : 4;
    return 0;
}

extern "C" int mb200_model_finalize(mb200_model* m) {
    MB_REQUIRE(m && !m->finalized, "bad model state");
    const auto& c = m->cfg;
    const int d = c.d_model, f = c.ffn_dim;
    for (const auto& n : required_names(c))
        MB_REQUIRE(m->host_w.count(n) == 1, std::string("missing weight ") + n);
    auto W = [&](const std::string& n) -> const std::vector<float>& { return m->host_w.at(n); };
    auto expect = [&](const std::string& n, size_t numel) -> int {
        MB_REQUIRE(W(n).size() == numel, "wrong element count for " + n);
        return 0;
    };
    MB_TRY(expect("encoder_embedder.weight", (size_t)d * c.mel.n_mels));
    MB_TRY(expect("decoder_embedder.weight", (size_t)c.vocab_size_in * d));
    MB_TRY(expect("transformer.proj_out.weight", (size_t)c.vocab_size_out * d));
    MB_TRY(expect("transformer.model.encoder.conv1.weight", (size_t)d * d * 3));
    MB_TRY(expect("transformer.model.encoder.embed_positions.weight", (size_t)(c.src_seq_len / 2) * d));
    MB_TRY(expect("transformer.model.decoder.embed_positions.weight", (size_t)c.tgt_seq_len * d));

    // ---- pack on the host ----
    std::vector<float> pack;
    auto push = [&](const std::vector<float>& v) -> size_t {
        size_t off = (pack.size() + 63) & ~size_t(63);   // 256-byte alignment
        pack.resize(off + v.size());
        std::copy(v.begin(), v.end(), pack.begin() + off);
        return off;
    };
    auto conv_pack = [&](const std::vector<float>& w) {   // [co][ci][3] -> [co][tap*C + ci]
        std::vector<float> o((size_t)d * 3 * d);
        for (int co = 0; co < d; ++co)
            for (int ci = 0; ci < d; ++ci)
                for (int j = 0; j < 3; ++j) o[(size_t)co * 3 * d + (size_t)j * d + ci] = w[((size_t)co * d + ci) * 3 + j];
        return o;
    };
    const float qs = 0.125f;   // head_dim^-0.5 for head_dim 64: a power of two, so folding it into Wq/bq is bit-exact
    auto qkv_pack = [&](const std::string& p, std::vector<float>& wq, std::vector<float>& bq) {
        wq.assign((size_t)3 * d * d, 0.f); bq.assign((size_t)3 * d, 0.f);
        const auto &q = W(p + "q_proj.weight"), &k = W(p + "k_proj.weight"), &v = W(p + "v_proj.weight");
        const auto &qb = W(p + "q_proj.bias"), &vb = W(p + "v_proj.bias");
        for (size_t i = 0; i < (size_t)d * d; ++i) { wq[i] = q[i] * qs; wq[(size_t)d * d + i] = k[i]; wq[(size_t)2 * d * d + i] = v[i]; }
        for (int i = 0; i < d; ++i) { bq[i] = qb[i] * qs; bq[2 * d + i] = vb[i]; }
    };
    struct Off { size_t v[20]; };
    std::vector<Off> eo(c.encoder_layers), dof(c.decoder_layers);
    size_t o_emb_w = push(W("encoder_embedder.weight")), o_emb_b = push(W("encoder_embedder.bias"));
    size_t o_c1w = push(conv_pack(W("transformer.model.encoder.conv1.weight"))), o_c1b = push(W("transformer.model.encoder.conv1.bias"));
    size_t o_c2w = push(conv_pack(W("transformer.model.encoder.conv2.weight"))), o_c2b = push(W("transformer.model.encoder.conv2.bias"));
    size_t o_epos = push(W("transformer.model.encoder.embed_positions.weight"));
    size_t o_elnw = push(W("transformer.model.encoder.layer_norm.weight")), o_elnb = push(W("transformer.model.encoder.layer_norm.bias"));
    size_t o_tok = push(W("decoder_embedder.weight")), o_dpos = push(W("transformer.model.decoder.embed_positions.weight"));
    size_t o_dlnw = push(W("transformer.model.decoder.layer_norm.weight")), o_dlnb = push(W("transformer.model.decoder.layer_norm.bias"));
    size_t o_proj = push(W("transformer.proj_out.weight"));
    for (int side = 0; side < 2; ++side) {
        int L = side == 0 ? c.encoder_layers : c.decoder_layers;
        for (int i = 0; i < L; ++i) {
            std::string p = std::string("transformer.model.") + (side == 0 ? "encoder" : "decoder") + ".layers." + std::to_string(i) + ".";
            Off& o = side == 0 ? eo[i] : dof[i];
            std::vector<float> wq, bq;
            qkv_pack(p + "self_attn.", wq, bq);
            o.v[0] = push(W(p + "self_attn_layer_norm.weight")); o.v[1] = push(W(p + "self_attn_layer_norm.bias"));
            o.v[2] = push(wq); o.v[3] = push(bq);
            o.v[4] = push(W(p + "self_attn.out_proj.weight")); o.v[5] = push(W(p + "self_attn.out_proj.bias"));
            if (side == 1) {
                qkv_pack(p + "encoder_attn.", wq, bq);
                o.v[6] = push(W(p + "encoder_attn_layer_norm.weight")); o.v[7] = push(W(p + "encoder_attn_layer_norm.bias"));
                o.v[8] = push(std::vector<float>(wq.begin(), wq.begin() + (size_t)d * d));
                o.v[9] = push(std::vector<float>(bq.begin(), bq.begin() + d));
                o.v[10] = push(std::vector<float>(wq.begin() + (size_t)d * d, wq.end()));
                o.v[11] = push(std::vector<float>(bq.begin() + d, bq.end()));
                o.v[12] = push(W(p + "encoder_attn.out_proj.weight")); o.v[13] = push(W(p + "encoder_attn.out_proj.bias"));
            }
            o.v[14] = push(W(p + "final_layer_norm.weight")); o.v[15] = push(W(p + "final_layer_norm.bias"));
            o.v[16] = push(W(p + "fc1.weight")); o.v[17] = push(W(p + "fc1.bias"));
            o.v[18] = push(W(p + "fc2.weight")); o.v[19] = push(W(p + "fc2.bias"));
            MB_REQUIRE(W(p + "fc1.weight").size() == (size_t)f * d, "wrong fc1 shape");
        }
    }
    MB_TRY(m->arena.ensure(pack.size() * sizeof(float)));
    MB_CUDA_CHECK(cudaMemcpy(m->arena.p, pack.data(), pack.size() * sizeof(float), cudaMemcpyHostToDevice));
    const float* base = m->arena.as<float>();
    m->emb_w = base + o_emb_w; m->emb_b = base + o_emb_b; m->conv1_w = base + o_c1w; m->conv1_b = base + o_c1b;
    m->conv2_w = base + o_c2w; m->conv2_b = base + o_c2b; m->enc_pos = base + o_epos; m->enc_ln_w = base + o_elnw; m->enc_ln_b = base + o_elnb;
    m->tok_emb = base + o_tok; m->dec_pos = base + o_dpos; m->dec_ln_w = base + o_dlnw; m->dec_ln_b = base + o_dlnb; m->proj_out = base + o_proj;
    auto fill = [&](const Off& o, bool cross) {
        LayerW l{};
        l.ln1_w = base + o.v[0]; l.ln1_b = base + o.v[1]; l.wqkv = base + o.v[2]; l.bqkv = base + o.v[3]; l.wo = base + o.v[4]; l.bo = base + o.v[5];
        if (cross) {
            l.ln2_w = base + o.v[6]; l.ln2_b = base + o.v[7]; l.wq_c = base + o.v[8]; l.bq_c = base + o.v[9];
            l.wkv_c = base + o.v[10]; l.bkv_c = base + o.v[11]; l.wo_c = base + o.v[12]; l.bo_c = base + o.v[13];
        }
        l.ln3_w = base + o.v[14]; l.ln3_b = base + o.v[15]; l.fc1_w = base + o.v[16]; l.fc1_b = base + o.v[17];
        l.fc2_w = base + o.v[18]; l.fc2_b = base + o.v[19];
        return l;
    };
    for (auto& o : eo) m->enc.push_back(fill(o, false));
    for (auto& o : dof) m->dec.push_back(fill(o, true));
    // ---- bf16 store of the token loop's GEMV matrices ----
    // Only when every matrix the token loop streams arrived as bf16 and every packed element (the q rows carry the folded 0.125) is
    // still a bf16 value: the bf16 GEMV widens each element and sums in the fp32 kernel's order, so both stores give the same bits.
    // The fp32 arena stays whole: the prefill GEMMs, the cross K/V projection and the teacher-forced passes read it.
    {
        std::vector<std::string> src = {"transformer.proj_out.weight"};
        for (int i = 0; i < c.decoder_layers; ++i) {
            const std::string p = "transformer.model.decoder.layers." + std::to_string(i) + ".";
            for (const char* n : {"self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.out_proj.weight",
                                  "encoder_attn.q_proj.weight", "encoder_attn.out_proj.weight", "fc1.weight", "fc2.weight"})
                src.push_back(p + n);
        }
        bool ok = d % 8 == 0 && f % 8 == 0;      // K of every matrix a multiple of 8: 16-byte rows for the 8-byte loads and bulk copies
        for (const auto& n : src) ok = ok && m->bf16_names.count(n) == 1;
        // (offset, element count) of every packed matrix in `pack`
        std::vector<std::pair<size_t, size_t>> mats = {{o_proj, (size_t)c.vocab_size_out * d}};
        for (const auto& o : dof) {
            mats.push_back({o.v[2], (size_t)3 * d * d}); mats.push_back({o.v[4], (size_t)d * d}); mats.push_back({o.v[8], (size_t)d * d});
            mats.push_back({o.v[12], (size_t)d * d}); mats.push_back({o.v[16], (size_t)f * d}); mats.push_back({o.v[18], (size_t)d * f});
        }
        std::vector<uint16_t> pack16;
        std::vector<size_t> off16;
        for (size_t k = 0; ok && k < mats.size(); ++k) {
            const size_t o16 = (pack16.size() + 127) & ~size_t(127);      // 256-byte alignment
            pack16.resize(o16 + mats[k].second);
            for (size_t i = 0; i < mats[k].second; ++i) {
                uint32_t u;
                std::memcpy(&u, &pack[mats[k].first + i], 4);
                if (u & 0xffffu) { ok = false; break; }
                pack16[o16 + i] = (uint16_t)(u >> 16);
            }
            off16.push_back(o16);
        }
        if (ok) {
            MB_TRY(m->arena16.ensure(pack16.size() * sizeof(uint16_t)));
            MB_CUDA_CHECK(cudaMemcpy(m->arena16.p, pack16.data(), pack16.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
            const uint16_t* b16 = m->arena16.as<uint16_t>();
            auto at = [&](size_t k) { return reinterpret_cast<const float*>(b16 + off16[k]); };
            m->proj_out16 = at(0);
            for (size_t l = 0; l < m->dec.size(); ++l) {
                LayerW& w = m->dec[l];
                w.wqkv16 = at(1 + 6 * l); w.wo16 = at(2 + 6 * l); w.wq_c16 = at(3 + 6 * l);
                w.wo_c16 = at(4 + 6 * l); w.fc1_w16 = at(5 + 6 * l); w.fc2_w16 = at(6 + 6 * l);
            }
        }
    }
    m->host_w.clear();
    m->bf16_names.clear();
    // tf32 "lo" mirrors of the weights that feed large (tensor-core) GEMMs: encoder stem + layers, cross K|V projections
    {
        const long long dd = (long long)d * d;
        auto reg = [&](const float* w, long long n) -> int { return m->gemm.register_weight(w, n); };
        MB_TRY(reg(m->emb_w, (long long)d * c.mel.n_mels));
        MB_TRY(reg(m->conv1_w, 3 * dd)); MB_TRY(reg(m->conv2_w, 3 * dd));
        for (const auto& l : m->enc) {
            MB_TRY(reg(l.wqkv, 3 * dd)); MB_TRY(reg(l.wo, dd));
            MB_TRY(reg(l.fc1_w, (long long)f * d)); MB_TRY(reg(l.fc2_w, (long long)f * d));
        }
        for (const auto& l : m->dec) MB_TRY(reg(l.wkv_c, 2 * dd));
        MB_CUDA_CHECK(cudaDeviceSynchronize());
        // Scratch for the largest encoder chunk, allocated once: captured prefill graphs hold the split-K workspace pointer, so
        // nothing in the context may move after this point.
        const size_t chunk = (size_t)std::min(std::max(1, c.max_windows), 16);
        const size_t a_floats = std::max({chunk * (size_t)(c.src_seq_len / 2) * f, chunk * (size_t)(c.src_seq_len + 2) * d,
                                          chunk * (size_t)c.src_seq_len * c.mel.n_mels});
        m->gemm.num_sms = std::max(1, m->num_sms_phys);
        MB_TRY(m->gemm.reserve((size_t)64 << 20, a_floats * 8 + 1024));
        m->gemm.frozen = true;
        MB_TRY(m->attn.reserve(attn_tc_workspace_bytes((int)chunk, c.heads, c.src_seq_len / 2, c.src_seq_len / 2)));
        m->attn.frozen = true;
    }

    // ---- resident state ----
    m->max_rows = std::max(1, c.max_batch);
    MB_TRY(m->cross_kv.ensure((size_t)c.decoder_layers * m->cross_layer_stride() * sizeof(float)));
    MB_TRY(m->self_kv.ensure((size_t)c.decoder_layers * m->self_layer_stride() * sizeof(float)));
    // sized for a ragged call (GenState + one RowState / SampleConfig / flag row per request); a uniform call uses element 0
    MB_TRY(m->g_state.ensure(sizeof(GenState) + (size_t)m->max_rows * sizeof(RowState)));
    MB_TRY(m->g_cfg.ensure((size_t)m->max_rows * sizeof(SampleConfig)));
    MB_TRY(m->g_vflags.ensure((size_t)m->max_rows * c.vocab_size_in));
    MB_TRY(m->g_ids.ensure((size_t)m->max_rows * c.tgt_seq_len * sizeof(long long)));
    MB_TRY(m->g_prefill_ids.ensure((size_t)m->max_rows * c.tgt_seq_len * sizeof(long long)));
    MB_TRY(m->g_keyvalid.ensure((size_t)m->max_rows * c.tgt_seq_len));
    MB_TRY(m->g_leftpad.ensure(m->max_rows * sizeof(int)));
    // [max_rows] decode rows, then one (slot, slot) pair per request for ragged prefills, then the row list of a stream admission
    MB_TRY(m->g_rowslot.ensure((size_t)4 * m->max_rows * sizeof(int)));
    MB_TRY(m->g_finished.ensure(m->max_rows));
    {
        const size_t tgt = (size_t)m->max_rows * c.tgt_seq_len;
        m->h_stage_bytes = tgt * 8 * 2 + tgt + (size_t)2 * m->max_rows * 4 + c.vocab_size_in + sizeof(GenState) + sizeof(SampleConfig) + 8 * 16;
        // a stream admission of up to max_rows requests: per row a flag row, RowState, SampleConfig, slot entries and their alignment
        m->h_stage_bytes += (size_t)m->max_rows * (c.vocab_size_in + sizeof(RowState) + sizeof(SampleConfig) + 16 + 5 * 16) + 16;
        // a beam call: its source-row table, the running and finished scores, and their alignment
        m->h_stage_bytes += tgt * 4 + (size_t)2 * m->max_rows * 4 + 3 * 16;
        MB_CUDA_CHECK(cudaMallocHost(&m->h_stage, m->h_stage_bytes));
        MB_CUDA_CHECK(cudaEventCreateWithFlags(&m->stage_ev, cudaEventDisableTiming));
    }
    MB_TRY(m->g_lastts.ensure(m->max_rows * sizeof(int)));
    MB_TRY(m->g_lastscores.ensure((size_t)2 * m->max_rows * c.vocab_size_out * sizeof(float)));
    MB_TRY(m->d_x.ensure((size_t)m->max_rows * d * sizeof(float)));
    MB_TRY(m->d_q.ensure((size_t)m->max_rows * d * sizeof(float)));
    MB_TRY(m->d_h.ensure((size_t)m->max_rows * f * sizeof(float)));
    MB_TRY(m->d_logits.ensure((size_t)m->max_rows * c.vocab_size_out * sizeof(float)));
    {   // prefill activations for the largest possible call, so captured prefill graphs never see a reallocation
        const size_t RPmax = (size_t)m->max_rows * c.tgt_seq_len;
        MB_TRY(m->p_x.ensure(RPmax * d * 4)); MB_TRY(m->p_h.ensure(RPmax * d * 4)); MB_TRY(m->p_q.ensure(RPmax * d * 4));
        MB_TRY(m->p_attn.ensure(RPmax * d * 4)); MB_TRY(m->p_ffn.ensure(RPmax * f * 4));
    }
    {   // split-KV partials sized for the longest possible context so captured graphs never see a reallocation
        const int max_splits = std::max((c.tgt_seq_len + 63) / 64, (c.src_seq_len / 2 + 63) / 64);
        MB_TRY(m->d_parto.ensure((size_t)m->max_rows * c.heads * max_splits * 64 * sizeof(float)));
        MB_TRY(m->d_partml.ensure((size_t)m->max_rows * c.heads * max_splits * 2 * sizeof(float)));
        MB_TRY(m->d_attn.ensure((size_t)m->max_rows * d * sizeof(float)));
        MB_TRY(m->d_ticket.ensure((size_t)m->max_rows * c.heads * sizeof(int)));
        MB_CUDA_CHECK(cudaMemset(m->d_ticket.p, 0, (size_t)m->max_rows * c.heads * sizeof(int)));
    }
    {   // exchange buffers of the dataflow megakernel: 8-byte {value | tag} pairs, two decoder rows
        const int R2 = 2, max_splits = std::max((c.tgt_seq_len + 63) / 64, (c.src_seq_len / 2 + 63) / 64);
        auto al = [](size_t n) { return (n + 15) & ~size_t(15); };
        const size_t n_x = al((size_t)R2 * d), n_kv = al((size_t)R2 * 2 * d), n_h = al((size_t)R2 * f), n_l = al((size_t)R2 * c.vocab_size_out),
                     n_p = al((size_t)R2 * c.heads * max_splits * 66), n_hdr = 16;
        const size_t RM = MEGA_LL_MAX_REPS;
        m->ll_bytes = ((2 * RM + 1) * n_x + n_kv + RM * n_h + n_l + n_p + n_hdr) * 8;
        MB_TRY(m->ll_arena.ensure(m->ll_bytes, true));
        unsigned long long* b = m->ll_arena.as<unsigned long long>();
        m->ll.x = b; b += RM * n_x; m->ll.att = b; b += RM * n_x; m->ll.q = b; b += n_x; m->ll.kvnew = b; b += n_kv; m->ll.h = b; b += RM * n_h;
        m->ll.logits = b; b += n_l; m->ll.part = b; b += n_p; m->ll.hdr = b;
        m->ll.max_splits = max_splits;
        m->ll.reps = 8; m->ll.x_rep = (long long)n_x; m->ll.h_rep = (long long)n_h;
    }
    m->finalized = true;
    return 0;
}

// =====================================================================================================================
// encoder
// =====================================================================================================================
static int encode_chunk(mb200_model* m, const float* pcm, int n, int slot_begin, float* enc_out, cudaStream_t st) {
    const auto& c = m->cfg;
    const int d = c.d_model, f = c.ffn_dim, H = c.heads, T2 = c.src_seq_len, T = T2 / 2, nm = c.mel.n_mels;
    const int n_samples = (c.src_seq_len - 1) * c.mel.hop_length;
    float* mel = m->w_mel.as<float>();
    float* embp = m->w_embpad.as<float>();
    float* c1p = m->w_c1pad.as<float>();
    float* x = m->w_x.as<float>();
    float* h = m->w_h.as<float>();
    float* qkv = m->w_qkv.as<float>();
    float* att = m->w_attn.as<float>();
    float* ffn = m->w_ffn.as<float>();
    const long long padrow = (long long)(T2 + 2) * d;

    MB_TRY(launch_mel(m->mel, pcm, n_samples, n, n_samples, mel, nm, (long long)T2 * nm, st));
    // encoder_embedder (modeling_mapperatorinator.py:433) written token-major into the zero-padded conv input
    {
        GemmParams g = gemm_base(plain_map(mel, nm), m->emb_w, nm, batched_map(embp + d, d, T2, padrow), m->emb_b, n * T2, d, nm);
        MB_TRY(launch_gemm(g, st, &m->gemm));
    }
    // conv1 k3 p1 + GELU  (row (b,t) of the padded buffer spans taps t-1, t, t+1 contiguously: K = 3d)
    {
        GemmParams g = gemm_base(batched_map(embp, d, T2, padrow), m->conv1_w, 3 * d, batched_map(c1p + d, d, T2, padrow), m->conv1_b,
                                 n * T2, d, 3 * d);
        g.act = ACT_GELU_ERF;
        MB_TRY(launch_gemm(g, st, &m->gemm));
    }
    // conv2 k3 s2 p1 + GELU + frozen positions
    {
        GemmParams g = gemm_base(batched_map(c1p, 2 * d, T, padrow), m->conv2_w, 3 * d, plain_map(x, d), m->conv2_b, n * T, d, 3 * d);
        g.act = ACT_GELU_ERF;
        g.R = batched_map(m->enc_pos, d, T, 0);
        MB_TRY(launch_gemm(g, st, &m->gemm));
    }
    const int rows = n * T;
    for (int l = 0; l < c.encoder_layers; ++l) {
        const LayerW& w = m->enc[l];
        MB_TRY(layernorm(x, h, w.ln1_w, w.ln1_b, rows, d, 1e-5f, st));
        MB_TRY(launch_gemm(gemm_base(plain_map(h, d), w.wqkv, d, plain_map(qkv, 3 * d), w.bqkv, rows, 3 * d, d), st, &m->gemm));
        AttentionParams a{};
        a.q = qkv; a.q_ld = 3 * d; a.q_bs = (long long)T * 3 * d;
        a.k = qkv + d; a.k_ld = 3 * d; a.k_bs = a.q_bs;
        a.v = qkv + 2 * d; a.v_ld = 3 * d; a.v_bs = a.q_bs;
        a.o = att; a.o_ld = d; a.o_bs = (long long)T * d;
        a.B = n; a.H = H; a.Tq = T; a.Tk = T; a.scale = 1.f; a.mask_mode = MASK_NONE;
        MB_TRY(launch_attention(a, st, &m->attn));
        {
            GemmParams g = gemm_base(plain_map(att, d), w.wo, d, plain_map(x, d), w.bo, rows, d, d);
            g.R = plain_map(x, d);
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
        MB_TRY(layernorm(x, h, w.ln3_w, w.ln3_b, rows, d, 1e-5f, st));
        {
            GemmParams g = gemm_base(plain_map(h, d), w.fc1_w, d, plain_map(ffn, f), w.fc1_b, rows, f, d);
            g.act = ACT_GELU_ERF;
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
        {
            GemmParams g = gemm_base(plain_map(ffn, f), w.fc2_w, f, plain_map(x, d), w.fc2_b, rows, d, f);
            g.R = plain_map(x, d);
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
    }
    float* enc = enc_out ? enc_out : h;
    MB_TRY(layernorm(x, enc, m->enc_ln_w, m->enc_ln_b, rows, d, 1e-5f, st));
    // cross-attention K|V of every decoder layer, straight into the resident slots
    for (int l = 0; l < c.decoder_layers; ++l) {
        float* dst = m->cross_kv.as<float>() + (size_t)l * m->cross_layer_stride() + (size_t)slot_begin * T * 2 * d;
        MB_TRY(launch_gemm(gemm_base(plain_map(enc, d), m->dec[l].wkv_c, d, plain_map(dst, 2 * d), m->dec[l].bkv_c, rows, 2 * d, d), st, &m->gemm));
    }
    return 0;
}

extern "C" int mb200_model_encode(mb200_model* m, const float* pcm, int32_t n_windows, int32_t slot_begin, float* enc_out, void* stream) {
    MB_REQUIRE(m && m->finalized, "model not finalized");
    MB_REQUIRE(slot_begin >= 0 && slot_begin + n_windows <= m->cfg.max_windows, "encoder slots out of range (raise max_windows)");
    cudaStream_t st = (cudaStream_t)stream;
    const auto& c = m->cfg;
    const int d = c.d_model, T2 = c.src_seq_len, T = T2 / 2;
    const int chunk = std::min(n_windows, 16);
    if (chunk > m->enc_chunk) {
        MB_TRY(m->w_mel.ensure((size_t)chunk * T2 * c.mel.n_mels * 4));
        MB_TRY(m->w_embpad.ensure((size_t)chunk * (T2 + 2) * d * 4, true));
        MB_TRY(m->w_c1pad.ensure((size_t)chunk * (T2 + 2) * d * 4, true));
        MB_TRY(m->w_x.ensure((size_t)chunk * T * d * 4));
        MB_TRY(m->w_h.ensure((size_t)chunk * T * d * 4));
        MB_TRY(m->w_qkv.ensure((size_t)chunk * T * 3 * d * 4));
        MB_TRY(m->w_attn.ensure((size_t)chunk * T * d * 4));
        MB_TRY(m->w_ffn.ensure((size_t)chunk * T * c.ffn_dim * 4));
        m->enc_chunk = chunk;
        for (auto& g : m->enc_graphs) cudaGraphExecDestroy(g.second.exec);      // the captured encodes point into the old workspaces
        m->enc_graphs.clear(); m->enc_seen.clear();
    }
    const long long n_samples = (long long)(c.src_seq_len - 1) * c.mel.hop_length;
    if (n_windows == 1 && enc_out == nullptr && m->enc_graph) {
        // The drop-in call pattern (`server.model_generate` encodes its one window per call): ~200 launches of 5-60 us.  The first call of
        // a slot runs eagerly, from the second on the same sequence is replayed as one CUDA graph over an engine-owned copy of the PCM.
        auto seen = m->enc_seen.find(slot_begin);
        if (seen == m->enc_seen.end()) {
            m->enc_seen[slot_begin] = 1;
            return encode_chunk(m, pcm, 1, slot_begin, nullptr, st);
        }
        MB_TRY(m->w_pcm.ensure((size_t)n_samples * sizeof(float)));
        auto git = m->enc_graphs.find(slot_begin);
        if (git == m->enc_graphs.end()) {
            CapturedGraph g;
            MB_TRY(capture_graph(m->cap_stream, st, [&](cudaStream_t cs) { return encode_chunk(m, m->w_pcm.as<float>(), 1, slot_begin, nullptr, cs); },
                                 &g));
            git = m->enc_graphs.emplace(slot_begin, g).first;
        }
        MB_CUDA_CHECK(cudaMemcpyAsync(m->w_pcm.p, pcm, (size_t)n_samples * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return git->second.launch(st);
    }
    for (int i = 0; i < n_windows; i += m->enc_chunk) {
        int n = std::min(m->enc_chunk, n_windows - i);
        MB_TRY(encode_chunk(m, pcm + (long long)i * n_samples, n, slot_begin + i, enc_out ? enc_out + (long long)i * T * d : nullptr, st));
    }
    return 0;
}

// =====================================================================================================================
// decoder prefill (shared by generate and forward_logits)
// =====================================================================================================================
// ids_dev [rows, P] int64, keyvalid_dev [rows, P], row_slot dev; afterwards p_x holds the final hidden states [rows*P, d]
// (pre final-LN) and the self cache holds positions [0, P).  Row i of the prefill writes self-cache row cache_row0 + i * cache_row_step
// and reads the encoder slot row_slot[i] (defaults: cache rows 0.., the call's slot table).
static int decoder_prefill(mb200_model* m, int rows, int P, const long long* ids_dev, int pos_rule, cudaStream_t st, int cache_row0 = 0,
                           int cache_row_step = 1, const int* row_slot = nullptr) {
    const auto& c = m->cfg;
    const int d = c.d_model, f = c.ffn_dim, H = c.heads, T = c.src_seq_len / 2;
    const size_t RP = (size_t)rows * P;
    MB_TRY(m->p_x.ensure(RP * d * 4)); MB_TRY(m->p_h.ensure(RP * d * 4)); MB_TRY(m->p_q.ensure(RP * d * 4));
    MB_TRY(m->p_attn.ensure(RP * d * 4)); MB_TRY(m->p_ffn.ensure(RP * f * 4));
    float *x = m->p_x.as<float>(), *h = m->p_h.as<float>(), *q = m->p_q.as<float>(), *att = m->p_attn.as<float>(), *ffn = m->p_ffn.as<float>();
    const unsigned char* kv_valid = m->g_keyvalid.as<unsigned char>();
    if (!row_slot) row_slot = m->g_rowslot.as<int>();
    MB_TRY(launch_embed(ids_dev, P, rows, rows, P, m->g_leftpad.as<int>(), pos_rule, m->tok_emb, m->dec_pos, d, x, st));
    const long long self_row = (long long)c.tgt_seq_len * 2 * d * cache_row_step;
    for (int l = 0; l < c.decoder_layers; ++l) {
        const LayerW& w = m->dec[l];
        float* skv = m->self_kv.as<float>() + (size_t)l * m->self_layer_stride() + (size_t)cache_row0 * c.tgt_seq_len * 2 * d;
        const float* ckv = m->cross_kv.as<float>() + (size_t)l * m->cross_layer_stride();
        MB_TRY(layernorm(x, h, w.ln1_w, w.ln1_b, (int)RP, d, 1e-5f, st));
        MB_TRY(launch_gemm(gemm_base(plain_map(h, d), w.wqkv, d, plain_map(q, d), w.bqkv, (int)RP, d, d), st, &m->gemm));
        MB_TRY(launch_gemm(gemm_base(plain_map(h, d), w.wqkv + (size_t)d * d, d, batched_map(skv, 2 * d, P, self_row), w.bqkv + d, (int)RP,
                                     2 * d, d), st, &m->gemm));
        AttentionParams a{};
        a.q = q; a.q_ld = d; a.q_bs = (long long)P * d;
        a.k = skv; a.k_ld = 2 * d; a.k_bs = self_row;
        a.v = skv + d; a.v_ld = 2 * d; a.v_bs = self_row;
        a.o = att; a.o_ld = d; a.o_bs = (long long)P * d;
        a.B = rows; a.H = H; a.Tq = P; a.Tk = P; a.scale = 1.f; a.mask_mode = MASK_CAUSAL; a.q_pos0 = 0;
        a.key_valid = kv_valid; a.key_valid_ld = c.tgt_seq_len;
        MB_TRY(launch_attention(a, st));
        {
            GemmParams g = gemm_base(plain_map(att, d), w.wo, d, plain_map(x, d), w.bo, (int)RP, d, d);
            g.R = plain_map(x, d);
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
        MB_TRY(layernorm(x, h, w.ln2_w, w.ln2_b, (int)RP, d, 1e-5f, st));
        MB_TRY(launch_gemm(gemm_base(plain_map(h, d), w.wq_c, d, plain_map(q, d), w.bq_c, (int)RP, d, d), st, &m->gemm));
        AttentionParams ca{};
        ca.q = q; ca.q_ld = d; ca.q_bs = (long long)P * d;
        ca.k = ckv; ca.k_ld = 2 * d; ca.k_bs = (long long)T * 2 * d;
        ca.v = ckv + d; ca.v_ld = 2 * d; ca.v_bs = ca.k_bs;
        ca.o = att; ca.o_ld = d; ca.o_bs = (long long)P * d;
        ca.B = rows; ca.H = H; ca.Tq = P; ca.Tk = T; ca.scale = 1.f; ca.mask_mode = MASK_NONE; ca.kv_slot = row_slot;
        MB_TRY(launch_attention(ca, st));
        {
            GemmParams g = gemm_base(plain_map(att, d), w.wo_c, d, plain_map(x, d), w.bo_c, (int)RP, d, d);
            g.R = plain_map(x, d);
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
        MB_TRY(layernorm(x, h, w.ln3_w, w.ln3_b, (int)RP, d, 1e-5f, st));
        {
            GemmParams g = gemm_base(plain_map(h, d), w.fc1_w, d, plain_map(ffn, f), w.fc1_b, (int)RP, f, d);
            g.act = ACT_GELU_ERF;
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
        {
            GemmParams g = gemm_base(plain_map(ffn, f), w.fc2_w, f, plain_map(x, d), w.fc2_b, (int)RP, d, f);
            g.R = plain_map(x, d);
            MB_TRY(launch_gemm(g, st, &m->gemm));
        }
    }
    return 0;
}

// =====================================================================================================================
// token step (captured into a CUDA graph)
// =====================================================================================================================
static GemvParams gemv_base(int xmode, const float* W, long long ldw, const float* bias, int K, int N, int B, const GenState* stt) {
    GemvParams g{};
    g.xmode = xmode; g.W = W; g.ldw = ldw; g.bias = bias; g.K = K; g.N = N; g.B = B; g.st = stt; g.eps = 1e-5f; g.nseg = 1;
    g.seg[0] = GemvSeg{nullptr, 0, 0, 0, N, 1.f, ACT_NONE};
    return g;
}

// Does the token loop stream the bf16 store?  Whenever the engine holds one: measured (tools/bf16_bench.py, README) faster than the
// fp32 copy on every driver and row count, megakernels and per-kernel GEMVs alike.
static bool token_bf16(const mb200_model* m) { return m->arena16.p != nullptr; }

// wbf: W is proj_out's bf16 copy (launch with w_bf16 = true)
static GemvParams final_logits_params(mb200_model* m, int rows, const float* x, long long x_ld, bool wbf) {
    const auto& c = m->cfg;
    GemvParams g = gemv_base(X_LAYERNORM, wbf ? m->proj_out16 : m->proj_out, c.d_model, nullptr, c.d_model, c.vocab_size_out, rows,
                             m->g_state.as<GenState>());
    g.x = x; g.x_ld = x_ld; g.ln_w = m->dec_ln_w; g.ln_b = m->dec_ln_b;
    g.seg[0].out = m->d_logits.as<float>(); g.seg[0].out_bs = c.vocab_size_out;
    return g;
}

static int final_logits(mb200_model* m, int rows, const float* x, long long x_ld, cudaStream_t st, bool pdl) {
    const bool wbf = token_bf16(m);
    return launch_gemv(final_logits_params(m, rows, x, x_ld, wbf), st, pdl, false, GEMV_FORM_KERNEL, wbf);
}

static SampleParams sample_params(mb200_model* m, int rows) {
    const auto& c = m->cfg;
    SampleParams s{};
    s.logits = m->d_logits.as<float>(); s.logits_ld = c.vocab_size_out;
    s.cfg = m->g_cfg.as<SampleConfig>(); s.st = m->g_state.as<GenState>(); s.vflags = m->g_vflags.as<unsigned char>();
    s.ids = m->g_ids.as<long long>(); s.finished = m->g_finished.as<unsigned char>(); s.last_ts = m->g_lastts.as<int>();
    s.last_scores = m->g_lastscores.as<float>(); s.n_left_pad = m->g_leftpad.as<int>();
    s.tok_emb = m->tok_emb; s.pos_emb = m->dec_pos; s.d_model = c.d_model;
    s.x_out = m->d_x.as<float>(); s.x_ld = c.d_model; s.rows = rows;
    return s;
}

// Either launches the 98 micro-phases of one token on `st` (eager / graph capture), or — when `collect` is given — records
// them as phase descriptors for the persistent megakernel.  One definition, so both paths run the same arithmetic.
// ragged: the step of a ragged call (per-phase kernels only) — n_splits_self is then the largest self-attention plan of the call.
static int token_step(mb200_model* m, int rows, int B, int n_splits_self, cudaStream_t st, bool pdl,
                      std::vector<MegaPhase>* collect = nullptr, const BeamParams* beam = nullptr, bool ragged = false) {
    // the weight store of this step's GEMVs (a megakernel's phase table carries it too)
    const bool wbf = token_bf16(m);
    auto TW = [&](const float* w32, const float* w16) { return wbf ? w16 : w32; };
    auto emit_gemv = [&](const GemvParams& g) -> int {
        // only the cache-writing GEMV reads the row's position
        if (!collect) return launch_gemv(g, st, pdl, ragged && g.nseg > 1, GEMV_FORM_KERNEL, wbf);
        MegaPhase ph{}; ph.kind = 0; ph.g = g; collect->push_back(ph);
        return 0;
    };
    auto emit_attn = [&](const DecAttnParams& a) -> int {
        if (!collect) return launch_decode_attention(a, st, pdl);
        MegaPhase ph{}; ph.kind = 1; ph.a = a;
        ph.magic_ns = a.n_splits > 1 ? (unsigned)((1ull << 32) / (unsigned)a.n_splits + 1) : 0u;       // 0 = divisor 1 (2^32 + 1 does not fit)
        ph.magic_h = a.H > 1 ? (unsigned)((1ull << 32) / (unsigned)a.H + 1) : 0u;
        collect->push_back(ph);
        return 0;
    };
    const auto& c = m->cfg;
    const int d = c.d_model, f = c.ffn_dim, H = c.heads, T = c.src_seq_len / 2;
    const GenState* gs = m->g_state.as<GenState>();
    float *x = m->d_x.as<float>(), *q = m->d_q.as<float>(), *hh = m->d_h.as<float>();
    float *po = m->d_parto.as<float>(), *pml = m->d_partml.as<float>(), *attn = m->d_attn.as<float>();
    int* ticket = m->d_ticket.as<int>();
    const int chunk = 64, n_splits_cross = (T + chunk - 1) / chunk;
    const long long self_row = (long long)c.tgt_seq_len * 2 * d;
    for (int l = 0; l < c.decoder_layers; ++l) {
        const LayerW& w = m->dec[l];
        float* skv = m->self_kv.as<float>() + (size_t)l * m->self_layer_stride();
        const float* ckv = m->cross_kv.as<float>() + (size_t)l * m->cross_layer_stride();
        {   // LN1 -> q | k | v  (k, v land in the self cache at position cur_len - 1)
            GemvParams g = gemv_base(X_LAYERNORM, TW(w.wqkv, w.wqkv16), d, w.bqkv, d, 3 * d, rows, gs);
            g.x = x; g.x_ld = d; g.ln_w = w.ln1_w; g.ln_b = w.ln1_b;
            g.nseg = 3;
            g.seg[0] = GemvSeg{q, d, 0, 0, d, 1.f, ACT_NONE};
            g.seg[1] = GemvSeg{skv, self_row, 2 * d, d, 2 * d, 1.f, ACT_NONE};
            g.seg[2] = GemvSeg{skv + d, self_row, 2 * d, 2 * d, 3 * d, 1.f, ACT_NONE};
            MB_TRY(emit_gemv(g));
        }
        {
            DecAttnParams a{};
            a.q = q; a.q_ld = d; a.kc = skv; a.vc = skv + d; a.row_stride = self_row; a.tok_stride = 2 * d; a.row_slot = nullptr;
            a.fixed_len = 0; a.st = gs; a.key_valid = m->g_keyvalid.as<unsigned char>(); a.key_valid_ld = c.tgt_seq_len;
            a.part_o = po; a.part_ml = pml; a.rows = rows; a.H = H; a.n_splits = n_splits_self;
            a.chunk = self_split_chunk(n_splits_self);      // contexts up to 128 tokens: one split per head, no merge step
            a.out = attn; a.out_ld = d; a.ticket = ticket;
            if (beam) { a.kv_src = beam->kv_src; a.kv_src_ld = beam->kv_src_ld; }
            if (ragged) {
                a.key_valid = nullptr;      // no pad keys in a ragged row
                MB_TRY(launch_decode_attention_ragged(a, st, pdl));
            } else
            MB_TRY(emit_attn(a));
        }
        {   // out_proj + residual (the heads were merged by the attention phase)
            GemvParams g = gemv_base(X_PLAIN, TW(w.wo, w.wo16), d, w.bo, d, d, rows, gs);
            g.x = attn; g.x_ld = d;
            g.seg[0].out = x; g.seg[0].out_bs = d; g.R = x; g.r_ld = d;
            MB_TRY(emit_gemv(g));
        }
        {   // LN2 -> cross q
            GemvParams g = gemv_base(X_LAYERNORM, TW(w.wq_c, w.wq_c16), d, w.bq_c, d, d, rows, gs);
            g.x = x; g.x_ld = d; g.ln_w = w.ln2_w; g.ln_b = w.ln2_b;
            g.seg[0].out = q; g.seg[0].out_bs = d;
            MB_TRY(emit_gemv(g));
        }
        {
            DecAttnParams a{};
            a.q = q; a.q_ld = d; a.kc = ckv; a.vc = ckv + d; a.row_stride = (long long)T * 2 * d; a.tok_stride = 2 * d;
            a.row_slot = m->g_rowslot.as<int>(); a.fixed_len = T; a.st = gs; a.key_valid = nullptr;
            a.part_o = po; a.part_ml = pml; a.rows = rows; a.H = H; a.n_splits = n_splits_cross; a.chunk = chunk;
            a.out = attn; a.out_ld = d; a.ticket = ticket;
            MB_TRY(emit_attn(a));
        }
        {
            GemvParams g = gemv_base(X_PLAIN, TW(w.wo_c, w.wo_c16), d, w.bo_c, d, d, rows, gs);
            g.x = attn; g.x_ld = d;
            g.seg[0].out = x; g.seg[0].out_bs = d; g.R = x; g.r_ld = d;
            MB_TRY(emit_gemv(g));
        }
        {   // LN3 -> fc1 + GELU
            GemvParams g = gemv_base(X_LAYERNORM, TW(w.fc1_w, w.fc1_w16), d, w.fc1_b, d, f, rows, gs);
            g.x = x; g.x_ld = d; g.ln_w = w.ln3_w; g.ln_b = w.ln3_b;
            g.seg[0] = GemvSeg{hh, f, 0, 0, f, 1.f, ACT_GELU_ERF};
            MB_TRY(emit_gemv(g));
        }
        {   // fc2 + residual
            GemvParams g = gemv_base(X_PLAIN, TW(w.fc2_w, w.fc2_w16), f, w.fc2_b, f, d, rows, gs);
            g.x = hh; g.x_ld = f;
            g.seg[0].out = x; g.seg[0].out_bs = d; g.R = x; g.r_ld = d;
            MB_TRY(emit_gemv(g));
        }
    }
    MB_TRY(emit_gemv(final_logits_params(m, rows, x, d, wbf)));
    if (collect) {
        MegaPhase ph{}; ph.kind = 2; collect->push_back(ph);
        const int n = (int)collect->size();
        for (int i = 0; i < n; ++i) {          // next GEMV phase after i, wrapping into the next token
            int j = (i + 1) % n;
            while ((*collect)[j].kind != 0) j = (j + 1) % n;
            (*collect)[i].next_gemv = j;
            (*collect)[i].nx_W = (*collect)[j].g.W; (*collect)[i].nx_ldw = (*collect)[j].g.ldw;
            (*collect)[i].nx_N = (*collect)[j].g.N; (*collect)[i].nx_K = (*collect)[j].g.K;
            (*collect)[i].nx_rpc = ((*collect)[j].g.N + m->num_sms - 1) / m->num_sms;
            (*collect)[i].rpc = (*collect)[i].kind == 0 ? ((*collect)[i].g.N + m->num_sms - 1) / m->num_sms : 0;
        }
        return 0;
    }
    if (beam) return launch_beam_step(*beam, B, st);
    MB_TRY(launch_sample(sample_params(m, rows), B, st, pdl, ragged));
    return 0;
}

// The device copy of a megakernel's phase table for (rows, B, n_splits_self): token_step's phase list, annotated by `annotate` for the
// kernel that reads it, built the first time the key is met.
template <typename Phase, typename Annotate>
static int phase_table(mb200_model* m, int driver, int rows, int B, int n_splits_self, cudaStream_t st, Annotate annotate,
                       const Phase** table, int* n_phases) {
    const auto key = std::make_tuple(driver, rows, B, n_splits_self);
    auto it = m->phase_tables.find(key);
    if (it == m->phase_tables.end()) {
        std::vector<MegaPhase> phases;
        MB_TRY(token_step(m, rows, B, n_splits_self, st, false, &phases));
        std::vector<Phase> annotated(phases.size());
        MB_TRY(annotate(phases, annotated));
        std::unique_ptr<DevBuf> buf(new DevBuf());
        MB_TRY(buf->ensure(annotated.size() * sizeof(Phase)));
        MB_CUDA_CHECK(cudaMemcpy(buf->p, annotated.data(), annotated.size() * sizeof(Phase), cudaMemcpyHostToDevice));
        it = m->phase_tables.emplace(key, std::make_pair(std::move(buf), (int)annotated.size())).first;
    }
    *table = it->second.first->template as<Phase>();
    *n_phases = it->second.second;
    return 0;
}

// One persistent launch of the token loop: clears the grid-sync words (g_megasync[0] the barrier counter, [8] the error flag, [9..11]
// where a timed-out wait was), times `launch` with CUDA events, reads cur_len before and after it into h_flag[2] / h_flag[3] and the
// error words into h_flag[1] / h_flag[4..6].  `before_sync` enqueues the caller's read-backs ahead of the closing sync, so the call
// needs only that one host wait.  The error flag is the caller's to interpret.
static int mega_launch(mb200_model* m, cudaStream_t st, const std::function<int()>& launch, const std::function<int()>& before_sync) {
    MB_TRY(m->g_megasync.ensure(64));
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_megasync.p, 0, 64, st));
    if (!m->mega_ev[0]) { MB_CUDA_CHECK(cudaEventCreate(&m->mega_ev[0])); MB_CUDA_CHECK(cudaEventCreate(&m->mega_ev[1])); }
    MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag + 2, &m->g_state.as<GenState>()->cur_len, 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaEventRecord(m->mega_ev[0], st));
    MB_TRY(launch());
    MB_CUDA_CHECK(cudaEventRecord(m->mega_ev[1], st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag + 1, m->g_megasync.as<int>() + 8, 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag + 4, m->g_megasync.as<int>() + 9, 12, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag + 3, &m->g_state.as<GenState>()->cur_len, 4, cudaMemcpyDeviceToHost, st));
    MB_TRY(before_sync());
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    float ms = 0.f;
    MB_CUDA_CHECK(cudaEventElapsedTime(&ms, m->mega_ev[0], m->mega_ev[1]));
    m->mega_ms += ms; m->mega_launches += 1; m->mega_tokens += m->h_flag[3] - m->h_flag[2];
    return 0;
}

// The persistent path: all remaining tokens of the call in one cooperative launch (rows <= 2, weight slices must fit).
static int run_megakernel(mb200_model* m, int rows, int B, int n_splits_self, int max_steps, cudaStream_t st,
                          const std::function<int()>& before_sync) {
    const MegaPhase* table = nullptr;
    int n_phases = 0;
    auto as_is = [](const std::vector<MegaPhase>& phases, std::vector<MegaPhase>& p1) { p1 = phases; return 0; };
    MB_TRY(phase_table(m, 1, rows, B, n_splits_self, st, as_is, &table, &n_phases));
    auto launch = [&]() -> int {
        MegaParams mp{};
        mp.phases = table; mp.n_phases = n_phases; mp.first_gemv = 0;
        mp.sample = sample_params(m, rows); mp.st = m->g_state.as<GenState>();
        mp.sync_counter = m->g_megasync.as<unsigned int>(); mp.error_flag = m->g_megasync.as<int>() + 8;
        mp.max_steps = max_steps; mp.row_slot = m->g_rowslot.as<int>();
        mp.trace = m->mega_trace.p ? m->mega_trace.as<unsigned long long>() : nullptr; mp.trace_step = 8;
        return launch_megakernel(mp, m->num_sms, st, token_bf16(m));
    };
    MB_TRY(mega_launch(m, st, launch, before_sync));
    MB_REQUIRE(m->h_flag[1] == 0, m->h_flag[1] == 1 ? "megakernel grid barrier timed out" : "megakernel weight copy timed out");
    return 0;
}

// The dataflow path: same phase list, each phase annotated with the exchange buffers it reads / writes.
static int run_megakernel2(mb200_model* m, int rows, int B, int n_splits_self, int max_steps, cudaStream_t st,
                           const std::function<int()>& before_sync) {
    auto annotate = [&](const std::vector<MegaPhase>& phases, std::vector<Mega2Phase>& p2) -> int {
        const float *dx = m->d_x.as<float>(), *dq = m->d_q.as<float>(), *dh = m->d_h.as<float>(), *datt = m->d_attn.as<float>(),
                    *dlog = m->d_logits.as<float>();
        for (size_t i = 0; i < phases.size(); ++i) {
            Mega2Phase& q = p2[i];
            q = Mega2Phase{};
            q.base = phases[i];
            if (phases[i].kind != 0) continue;
            const GemvParams& g = phases[i].g;
            q.in_sel = g.xmode == X_LAYERNORM ? LL_X : (g.x == datt ? LL_ATT : (g.x == dh ? LL_H : LL_NONE));
            MB_REQUIRE(q.in_sel != LL_NONE && (g.xmode != X_LAYERNORM || g.x == dx), "dataflow megakernel: unknown GEMV input buffer");
            q.res_xraw = g.R != nullptr;
            MB_REQUIRE(!g.R || g.R == dx, "dataflow megakernel: residual must be the residual stream");
            for (int sgi = 0; sgi < g.nseg; ++sgi) {
                const GemvSeg& sg = g.seg[sgi];
                if (sg.pos_stride != 0) { q.out_sel[sgi] = sgi == 1 ? LL_K : LL_V; q.plain_out[sgi] = 1; MB_REQUIRE(sgi >= 1, "cache segment order"); }
                else if (sg.out == dq) q.out_sel[sgi] = LL_Q;
                else if (sg.out == dx) q.out_sel[sgi] = LL_X;
                else if (sg.out == dh) q.out_sel[sgi] = LL_H;
                else if (sg.out == dlog) q.out_sel[sgi] = LL_LOGITS;
                else MB_REQUIRE(false, "dataflow megakernel: unknown GEMV output buffer");
                const int os = q.out_sel[sgi];
                const unsigned long long* ob = os == LL_X ? m->ll.x : os == LL_H ? m->ll.h : os == LL_Q ? m->ll.q : os == LL_LOGITS ? m->ll.logits : m->ll.kvnew;
                q.out_off[sgi] = (long long)(ob - m->ll.x) + (os == LL_V ? m->cfg.d_model : 0);
                q.out_rs[sgi] = os == LL_X ? m->ll.x_rep : (os == LL_H ? m->ll.h_rep : 0);
                q.out_bw[sgi] = os == LL_H ? g.N : (os == LL_K || os == LL_V ? 2 * m->cfg.d_model : (os == LL_LOGITS ? m->cfg.vocab_size_out : m->cfg.d_model));
            }
            {
                const unsigned long long* ib = q.in_sel == LL_H ? m->ll.h : (q.in_sel == LL_ATT ? m->ll.att : m->ll.x);
                q.in_off = (long long)(ib - m->ll.x);
                q.in_rs = q.in_sel == LL_H ? m->ll.h_rep : m->ll.x_rep;
                const int rpc = (g.N + m->num_sms - 1) / m->num_sms;
                q.n_active = (g.N + rpc - 1) / rpc;
            }
        }
        return 0;
    };
    const Mega2Phase* table = nullptr;
    int n_phases = 0;
    MB_TRY(phase_table(m, 2, rows, B, n_splits_self, st, annotate, &table, &n_phases));
    MB_CUDA_CHECK(cudaMemsetAsync(m->ll_arena.p, 0, m->ll_bytes, st));        // tag 0 = "nothing here yet"
    auto launch = [&]() -> int {
        Mega2Params mp{};
        mp.phases = table; mp.n_phases = n_phases;
        mp.sample = sample_params(m, rows); mp.st = m->g_state.as<GenState>();
        mp.ll = m->ll; mp.error_flag = m->g_megasync.as<int>() + 8;
        mp.sample.ll_logits = m->ll.logits; mp.sample.ll_x_out = m->ll.x; mp.sample.ll_hdr = m->ll.hdr; mp.sample.ll_err = mp.error_flag;
        mp.sample.ll_reps = m->ll.reps; mp.sample.ll_x_rep = m->ll.x_rep;
        mp.max_steps = max_steps; mp.row_slot = m->g_rowslot.as<int>(); mp.x_in = m->d_x.as<float>();
        mp.rows = rows; mp.d_model = m->cfg.d_model; mp.V = m->cfg.vocab_size_out; mp.ffn_dim = m->cfg.ffn_dim; mp.trace_cta = m->trace_cta;
        mp.trace = m->mega_trace.p ? m->mega_trace.as<unsigned long long>() : nullptr; mp.trace_step = 8;
        return launch_megakernel2(mp, m->num_sms, st, token_bf16(m));
    };
    MB_TRY(mega_launch(m, st, launch, before_sync));
    if (m->h_flag[1] == 4) {
        const unsigned tag = (unsigned)m->h_flag[6];
        MB_REQUIRE(false, "dataflow megakernel: a wait for tagged data timed out (CTA " + std::to_string(m->h_flag[4]) + ", thread " +
                              std::to_string(m->h_flag[5]) + ", expected tag " + std::to_string(tag) + " = step " + std::to_string((int)(tag / 128) - 1) +
                              " phase " + std::to_string((int)(tag % 128) - 1) + " of " + std::to_string(n_phases) + ", splits " +
                              std::to_string(n_splits_self) + ", rows " + std::to_string(rows) + ")");
    }
    MB_REQUIRE(m->h_flag[1] == 0, m->h_flag[1] == 2 ? "dataflow megakernel: weight copy timed out" : "dataflow megakernel: a wait for tagged data timed out");
    return 0;
}

static bool mega_eligible(const mb200_model* m, int rows) {
    if (!m->use_mega || rows > 2 || m->num_sms <= 0) return false;
    const auto& c = m->cfg;
    const int G = m->num_sms;
    // per-CTA weight slices of the token's GEMV phases; consecutive phases (qkv, out, cross q, cross out, fc1, fc2 per layer, then
    // the vocabulary projection, then the next token's qkv) share the two-buffer arena from opposite ends
    auto slice = [&](int N, int K) { return (size_t)((N + G - 1) / G) * K; };
    const int d = c.d_model, f = c.ffn_dim;
    const size_t qkv = slice(3 * d, d), dd = slice(d, d), fc1 = slice(f, d), fc2 = slice(d, f), voc = slice(c.vocab_size_out, d);
    auto pair = [&](size_t a, size_t b) { return a + b <= (size_t)2 * MEGA_WBUF_FLOATS; };
    return f <= 3072 && pair(qkv, dd) && pair(dd, dd) && pair(dd, fc1) && pair(fc1, fc2) && pair(fc2, qkv) && pair(fc2, voc) && pair(voc, qkv);
}

static SampleConfig make_sample_config(const mb200_generate_params* gp, int B, bool use_cfg, int V, int ids_ld) {
    SampleConfig sc{};
    sc.B = B; sc.use_cfg = use_cfg ? 1 : 0; sc.cfg_scale = gp->cfg_scale; sc.V = V; sc.ts_start = gp->time_shift_start; sc.ts_end = gp->time_shift_end;
    sc.timeshift_bias = gp->timeshift_bias; sc.types_first = gp->types_first; sc.temperature = gp->temperature;
    sc.n_cond = gp->n_cond;
    for (int i = 0; i < 3; ++i) { sc.cond_temp[i] = gp->cond_temp[i]; sc.cond_offset[i] = gp->cond_offset[i]; sc.cond_flag[i] = gp->cond_flag[i]; }
    sc.lookback_on = gp->lookback_on; sc.lookback_start = gp->lookback_start; sc.lookback_end = gp->lookback_end;
    sc.do_sample = gp->do_sample; sc.top_k = gp->top_k; sc.top_p = gp->top_p; sc.top_p_cut = gp->top_p_cut; sc.seed = gp->seed; sc.pad_id = gp->pad_token_id;
    sc.pos_rule_cumsum = gp->position_rule; sc.ids_ld = ids_ld; sc.vflags_ld = 0;
    return sc;
}

// Replays a token-step graph in bursts of 16 steps, the first one at least first_burst_min long, polling all_finished after each,
// until every row finished or `remaining` steps ran.
static int replay_until_finished(mb200_model* m, CapturedGraph& graph, int remaining, int first_burst_min, cudaStream_t st) {
    for (int burst_min = first_burst_min; remaining > 0; burst_min = 0) {
        const int burst = std::min(remaining, std::max(16, burst_min));
        MB_TRY(graph.launch(st, burst));
        remaining -= burst;
        MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag, &m->g_state.as<GenState>()->all_finished, 4, cudaMemcpyDeviceToHost, st));
        MB_CUDA_CHECK(cudaStreamSynchronize(st));
        if (*m->h_flag) break;
    }
    return 0;
}

// =====================================================================================================================
extern "C" int mb200_model_generate(mb200_model* m, const int32_t* slots, int32_t B, const int64_t* prompt, const uint8_t* prompt_mask,
                                    int32_t P, const int64_t* neg_prompt, const uint8_t* neg_mask, const uint8_t* vflags,
                                    const mb200_generate_params* gp, int64_t* out_ids, int32_t* out_len, void* stream) {
    MB_REQUIRE(m && m->finalized, "model not finalized");
    MB_TRY(token_loop_free(m));
    MB_REQUIRE(slots && prompt && vflags && gp && out_ids && out_len, "null argument");
    const auto& c = m->cfg;
    cudaStream_t st = (cudaStream_t)stream;
    const bool use_cfg = neg_prompt != nullptr;
    const int rows = use_cfg ? 2 * B : B;
    MB_REQUIRE(B >= 1 && rows <= m->max_rows, "batch exceeds max_batch (rows double under classifier-free guidance)");
    MB_REQUIRE(P >= 1 && P < gp->max_length && gp->max_length <= c.tgt_seq_len, "need 1 <= prompt_len < max_length <= tgt_seq_len");
    const int d = c.d_model, V = c.vocab_size_out;
    const int ids_ld = c.tgt_seq_len;

    // ---- call state: row r is item r % B; under CFG rows [0, B) carry the negative prompt (modeling_mapperatorinator.py:243-245) ----
    Stager sg{m, st};
    MB_TRY(sg.begin());
    long long* pre = sg.reserve<long long>((size_t)rows * P);
    long long* idsrow = sg.reserve<long long>((size_t)B * ids_ld);
    unsigned char* kv = sg.reserve<unsigned char>((size_t)rows * ids_ld);
    int* leftpad = sg.reserve<int>(rows);
    int* rowslot = sg.reserve<int>(rows);
    unsigned char* vf = sg.reserve<unsigned char>(c.vocab_size_in);
    GenState* gs = sg.reserve<GenState>(1);
    SampleConfig* sc = sg.reserve<SampleConfig>(1);
    MB_TRY(sg.fits());
    MB_TRY(build_prompt_rows(m, rows, P, [&](int r) { return r % B; }, use_cfg ? B : 0, slots, prompt, prompt_mask, neg_prompt, neg_mask,
                             pre, kv, leftpad, rowslot));
    for (int b = 0; b < B; ++b)
        for (int t = 0; t < ids_ld; ++t) idsrow[(size_t)b * ids_ld + t] = t < P ? prompt[(size_t)b * P + t] : gp->pad_token_id;
    std::memcpy(vf, vflags, c.vocab_size_in);
    *gs = GenState{};
    gs->cur_len = P; gs->prompt_len = P; gs->max_length = gp->max_length; gs->min_new_tokens = gp->min_new_tokens;
    *sc = make_sample_config(gp, B, use_cfg, V, ids_ld);
    MB_TRY(sg.upload(m->g_prefill_ids.p, pre, (size_t)rows * P));
    MB_TRY(sg.upload(m->g_ids.p, idsrow, (size_t)B * ids_ld));
    MB_TRY(sg.upload(m->g_keyvalid.p, kv, (size_t)rows * ids_ld));
    MB_TRY(sg.upload(m->g_leftpad.p, leftpad, rows));
    MB_TRY(sg.upload(m->g_rowslot.p, rowslot, rows));
    MB_TRY(sg.upload(m->g_vflags.p, vf, c.vocab_size_in));
    MB_TRY(sg.upload(m->g_state.p, gs, 1));
    MB_TRY(sg.upload(m->g_cfg.p, sc, 1));
    MB_TRY(sg.end());
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_finished.p, 0, m->max_rows, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->d_ticket.p, 0, (size_t)m->max_rows * m->cfg.heads * sizeof(int), st));   // self-resetting; cleared in case a previous call aborted

    const int n_splits_self = self_splits(gp->max_length);
    MB_TRY(launch_prompt_scan(m->g_ids.as<long long>(), ids_ld, B, P, m->g_vflags.as<unsigned char>(), sc->ts_start, sc->ts_end,
                              m->g_lastts.as<int>(), st));
    // prefill + first token: ~230 small launches.  The first call of a given (rows, P) shape runs eagerly (it may allocate);
    // from the second call on the same sequence is replayed as one CUDA graph (sequential windows reuse a few prompt lengths).
    {
        auto run_prefill = [&](cudaStream_t s) -> int {
            MB_TRY(decoder_prefill(m, rows, P, m->g_prefill_ids.as<long long>(), gp->position_rule, s));
            MB_TRY(final_logits(m, rows, m->p_x.as<float>() + (size_t)(P - 1) * d, (long long)P * d, s, false));
            MB_TRY(launch_sample(sample_params(m, rows), B, s, false));
            return 0;
        };
        const auto pkey = std::make_tuple(rows, (int)B, (int)P, (int)gp->position_rule);
        auto seen = m->prefill_seen.find(pkey);
        if (seen == m->prefill_seen.end()) {
            m->prefill_seen[pkey] = 1;
            MB_TRY(run_prefill(st));
        } else {
            auto git = m->prefill_graphs.find(pkey);
            if (git == m->prefill_graphs.end()) {
                CapturedGraph g;
                MB_TRY(capture_graph(m->cap_stream, st, run_prefill, &g));
                if (m->prefill_graphs.size() >= 48) {      // bounded cache: real songs see many prompt lengths; drop everything and re-learn
                    for (auto& old : m->prefill_graphs) cudaGraphExecDestroy(old.second.exec);
                    m->prefill_graphs.clear();
                    m->prefill_seen.clear();
                }
                git = m->prefill_graphs.emplace(pkey, g).first;
            }
            MB_TRY(git->second.launch(st));
        }
    }

    // ---- token loop, persistent path: every remaining token in ONE cooperative launch ----
    if (mega_eligible(m, rows) && gp->max_length - (P + 1) > 0) {
        bool dataflow = m->use_mega >= 2;
        if (dataflow) {     // every projection of this model must fit the K-split thread mapping, else the grid-barrier kernel takes the call
            const int G = m->num_sms;
            dataflow = mega2_ksplit_ok(3 * c.d_model, c.d_model, rows, G) && mega2_ksplit_ok(c.d_model, c.d_model, rows, G) &&
                       mega2_ksplit_ok(c.ffn_dim, c.d_model, rows, G) && mega2_ksplit_ok(c.d_model, c.ffn_dim, rows, G) &&
                       mega2_ksplit_ok(c.vocab_size_out, c.d_model, rows, G);
        }
        // (one 256-key attention unit per head for contexts of 129..256 tokens was tried: 365 vs 344 us / token against three 64-key units +
        //  merge — the V rows beyond the first 64 keys are fetched inside the PV loop, and the wider unit costs instructions in EVERY unit)
        // every row's ids up to max_length come back with {error flag, cur_len} ahead of the one sync; the final length is known only
        // then, so the rows are packed into out_ids ([B, cur_len]) on the host.  The staging copies of this call completed before the
        // megakernel started (stream order), so the pinned staging buffer is free to receive them.
        const int Lmax = gp->max_length;
        MB_REQUIRE((size_t)B * Lmax * 8 <= m->h_stage_bytes, "ids exceed the staging buffer");
        long long* ids_back = reinterpret_cast<long long*>(m->h_stage);
        auto read_ids = [&]() -> int {
            MB_CUDA_CHECK(cudaMemcpy2DAsync(ids_back, (size_t)Lmax * 8, m->g_ids.p, (size_t)ids_ld * 8, (size_t)Lmax * 8, B,
                                            cudaMemcpyDeviceToHost, st));
            return 0;
        };
        if (dataflow) MB_TRY(run_megakernel2(m, rows, B, n_splits_self, gp->max_length - (P + 1), st, read_ids));
        else MB_TRY(run_megakernel(m, rows, B, n_splits_self, gp->max_length - (P + 1), st, read_ids));
        const int Lm = m->h_flag[3];      // cur_len after the launch
        MB_REQUIRE(Lm >= P + 1 && Lm <= Lmax, "megakernel left an out-of-range length");
        for (int b = 0; b < B; ++b) std::memcpy(out_ids + (size_t)b * Lm, ids_back + (size_t)b * Lmax, (size_t)Lm * 8);
        *out_len = Lm;
        return 0;
    }
    // ---- token loop, graph path: one graph replay per token, flag polled every few tokens ----
    auto key = std::make_tuple(rows, (int)B, n_splits_self, 1);
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        CapturedGraph g;
        MB_TRY(capture_graph(m->cap_stream, st, [&](cudaStream_t cs) { return token_step(m, rows, B, n_splits_self, cs, m->use_pdl); }, &g));
        it = m->graphs.emplace(key, g).first;
    }
    // no EOS is possible before min_new_tokens are out, so the first poll can wait until then
    MB_TRY(replay_until_finished(m, it->second, gp->max_length - (P + 1), gp->min_new_tokens - 1, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag, &m->g_state.as<GenState>()->cur_len, 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    const int L = *m->h_flag;
    MB_CUDA_CHECK(cudaMemcpy2DAsync(out_ids, (size_t)L * 8, m->g_ids.p, (size_t)ids_ld * 8, (size_t)L * 8, B, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    *out_len = L;
    return 0;
}

// =====================================================================================================================
// Decode stream: a ragged token loop with a fixed row capacity N.  Requests are admitted into free rows between token steps and handed
// back as soon as they finish; each row's ids are bit-identical to its own batch-1 mb200_model_generate call, whatever step it joins at,
// whatever its neighbours do, and whatever the row held before.  Row r's state is its RowState (own length, plan, step counter and
// look-back flag), its SampleConfig and flag row, and its cache rows r (and N + r under classifier-free guidance).  A vacant row is a
// finished row: the step skips its self attention and leaves its cache and ids alone.  The ragged call below is one such stream that
// admits everything at once.  The two megakernels stay uniform (rows <= 2).
// =====================================================================================================================
struct mb200_stream {
    mb200_model* m = nullptr;
    int N = 0, rows = 0, cap = 0;
    bool use_cfg = false;
    CapturedGraph step;                      // the token-step graph; m->graphs owns its exec
    enum : int { FREE = 0, LIVE = 1, DONE = 2 };
    std::vector<int> status;                 // host view of each row
    std::vector<int> prompt_len, max_length, first_poll, selections;
    std::vector<int> done_len;               // DONE rows: final length
    RowState* h_rows = nullptr;              // pinned [N]: the rows' device state read back after each burst
};

namespace {

void stream_release(mb200_stream* s) {
    if (s->h_rows) cudaFreeHost(s->h_rows);
    s->h_rows = nullptr;
}

// The host-side bounds of n ragged requests (a ragged call's or a stream admission's), checked before anything is launched: every
// prompt 1 <= P < max_length <= cap, its encoder slot, guidance on every request or on none as the negative prompts say, its token ids.
int check_requests(const mb200_model* m, int n, const int32_t* slots, const int64_t* prompt, const int32_t* prompt_off,
                   const int64_t* neg_prompt, const mb200_generate_params* params, int cap) {
    const auto& c = m->cfg;
    MB_REQUIRE(prompt_off[0] == 0, "prompt offsets start at 0");
    for (int j = 0; j < n; ++j) {
        const mb200_generate_params& gp = params[j];
        const int P = prompt_off[j + 1] - prompt_off[j];
        MB_REQUIRE(P >= 1 && P < gp.max_length && gp.max_length <= cap,
                   "need 1 <= prompt_len < max_length <= the max_length cap (tgt_seq_len, or a stream's own) for every request");
        MB_REQUIRE(slots[j] >= 0 && slots[j] < c.max_windows, "encoder slot out of range");
        MB_REQUIRE((gp.cfg_scale > 1.0f) == (neg_prompt != nullptr), "classifier-free guidance on every request or on none");
        for (int t = prompt_off[j]; t < prompt_off[j + 1]; ++t) {
            MB_REQUIRE(prompt[t] >= 0 && prompt[t] < c.vocab_size_in, "prompt token id out of range");
            MB_REQUIRE(!neg_prompt || (neg_prompt[t] >= 0 && neg_prompt[t] < c.vocab_size_in), "negative prompt token id out of range");
        }
    }
    return 0;
}

// Fixes the shape (capacity N, guidance, max_length cap), captures the ragged step graph of (rows, N, self_splits(cap)) if this engine
// has none yet, and marks every row vacant.  Synchronises `st`.
int stream_open(mb200_model* m, mb200_stream* s, int N, bool use_cfg, int cap, cudaStream_t st) {
    const auto& c = m->cfg;
    const int rows = use_cfg ? 2 * N : N;
    MB_REQUIRE(N >= 1 && rows <= m->max_rows, "stream capacity exceeds max_batch (rows double under classifier-free guidance)");
    MB_REQUIRE(cap >= 2 && cap <= c.tgt_seq_len, "need 2 <= max_length cap <= tgt_seq_len");
    s->m = m; s->N = N; s->rows = rows; s->cap = cap; s->use_cfg = use_cfg;
    s->status.assign(N, mb200_stream::FREE);
    s->prompt_len.assign(N, 0); s->max_length.assign(N, 0); s->first_poll.assign(N, 0); s->selections.assign(N, 0); s->done_len.assign(N, 0);
    MB_CUDA_CHECK(cudaMallocHost(&s->h_rows, (size_t)N * sizeof(RowState)));
    const int ids_ld = c.tgt_seq_len, Vin = c.vocab_size_in;
    // vacant rows: finished, one valid token (the frozen selection re-issues the embedding of ids[r][cur_len - 1])
    std::vector<unsigned char> state(sizeof(GenState) + (size_t)N * sizeof(RowState), 0);
    GenState* gs = reinterpret_cast<GenState*>(state.data());
    gs->n_req = N; gs->all_finished = 1;
    RowState* rs = reinterpret_cast<RowState*>(gs + 1);
    for (int r = 0; r < N; ++r) { rs[r].cur_len = 1; rs[r].prompt_len = 1; rs[r].max_length = 2; rs[r].finished = 1; }
    SampleConfig base{};
    base.B = N; base.use_cfg = use_cfg ? 1 : 0; base.V = c.vocab_size_out; base.ids_ld = ids_ld; base.vflags_ld = Vin; base.temperature = 1.f;
    std::vector<SampleConfig> cfgs(N, base);
    MB_CUDA_CHECK(cudaMemcpyAsync(m->g_state.p, state.data(), state.size(), cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->g_cfg.p, cfgs.data(), cfgs.size() * sizeof(SampleConfig), cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_ids.p, 0, (size_t)N * ids_ld * 8, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_vflags.p, 0, (size_t)N * Vin, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_rowslot.p, 0, (size_t)4 * m->max_rows * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_keyvalid.p, 1, (size_t)m->max_rows * ids_ld, st));       // no pad keys in a stream row
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_leftpad.p, 0, m->max_rows * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->d_ticket.p, 0, (size_t)m->max_rows * c.heads * sizeof(int), st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));   // the host vectors above are pageable and go out of scope
    // the step graph; its key never meets a uniform (.., 1) or beam (.., K) graph
    auto key = std::make_tuple(rows, N, self_splits(cap), -1);
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        CapturedGraph g;
        MB_TRY(capture_graph(m->cap_stream, st, [&](cudaStream_t cs) {
            return token_step(m, rows, N, self_splits(cap), cs, m->use_pdl, nullptr, nullptr, true);
        }, &g));
        it = m->graphs.emplace(key, g).first;
    }
    s->step = it->second;
    return 0;
}

// Admits n requests into the lowest free rows (written to rows_out).  Every bound is checked before anything is launched; then the
// rows' state leaves from the engine's pinned staging buffer and the prompt scan, each request's prefill at its batch-1 shapes, its
// final-logits GEMV and the list selection of its first token queue behind it, with no host wait.
int stream_admit(mb200_stream* s, int n, const int32_t* slots, const int64_t* prompt, const int32_t* prompt_off, const int64_t* neg_prompt,
                 const uint8_t* vflags, const mb200_generate_params* params, int32_t* rows_out, cudaStream_t st) {
    mb200_model* m = s->m;
    const auto& c = m->cfg;
    MB_REQUIRE(slots && prompt && prompt_off && vflags && params && rows_out, "null argument");
    MB_REQUIRE((neg_prompt != nullptr) == s->use_cfg, "a negative prompt with every request of a guided stream and with none of an unguided one");
    std::vector<int> free_rows;
    for (int r = 0; r < s->N; ++r) if (s->status[r] == mb200_stream::FREE) free_rows.push_back(r);
    MB_REQUIRE(n >= 1 && n <= (int)free_rows.size(), "the stream has fewer free rows than requests to admit");
    MB_TRY(check_requests(m, n, slots, prompt, prompt_off, neg_prompt, params, s->cap));
    const int d = c.d_model, V = c.vocab_size_out, ids_ld = c.tgt_seq_len, Vin = c.vocab_size_in, N = s->N, nr = s->use_cfg ? 2 : 1;
    // ---- staging ----
    Stager sg{m, st};
    MB_TRY(sg.begin());
    int* list = sg.reserve<int>(n);
    std::vector<size_t> pre_off(n);
    size_t total = 0;
    for (int j = 0; j < n; ++j) { pre_off[j] = total; total += (size_t)nr * (prompt_off[j + 1] - prompt_off[j]); }
    long long* pre = sg.reserve<long long>(total);
    std::vector<long long*> h_ids(n); std::vector<RowState*> h_rs(n); std::vector<SampleConfig*> h_cfg(n); std::vector<int*> h_slot(n);
    std::vector<unsigned char*> h_vf(n);
    for (int j = 0; j < n; ++j) {
        h_ids[j] = sg.reserve<long long>(ids_ld);
        h_rs[j] = sg.reserve<RowState>(1);
        h_cfg[j] = sg.reserve<SampleConfig>(1);
        h_vf[j] = sg.reserve<unsigned char>(Vin);
        h_slot[j] = sg.reserve<int>(4);
    }
    MB_TRY(sg.fits());
    for (int j = 0; j < n; ++j) {
        const mb200_generate_params& gp = params[j];
        const int P = prompt_off[j + 1] - prompt_off[j], r = free_rows[j];
        list[j] = r;
        for (int i = 0; i < nr; ++i) {      // prefill rows of the request: the negative prompt first (modeling_mapperatorinator.py:243-245)
            const int64_t* src = (s->use_cfg && i == 0) ? neg_prompt : prompt;
            for (int t = 0; t < P; ++t) pre[pre_off[j] + (size_t)i * P + t] = src[prompt_off[j] + t];
        }
        for (int t = 0; t < ids_ld; ++t) h_ids[j][t] = t < P ? prompt[prompt_off[j] + t] : gp.pad_token_id;
        *h_rs[j] = RowState{};
        h_rs[j]->cur_len = P; h_rs[j]->prompt_len = P; h_rs[j]->max_length = gp.max_length; h_rs[j]->min_new_tokens = gp.min_new_tokens;
        *h_cfg[j] = make_sample_config(&gp, N, s->use_cfg, V, ids_ld);
        h_cfg[j]->pos_rule_cumsum = 0; h_cfg[j]->vflags_ld = Vin;
        std::memcpy(h_vf[j], vflags + (size_t)j * Vin, Vin);
        for (int i = 0; i < 4; ++i) h_slot[j][i] = slots[j];
    }
    GenState* gs = m->g_state.as<GenState>();
    int* rowslot = m->g_rowslot.as<int>();
    int* d_list = rowslot + 3 * m->max_rows;
    MB_TRY(sg.upload(d_list, list, n));
    MB_TRY(sg.upload(m->g_prefill_ids.p, pre, total));
    for (int j = 0; j < n; ++j) {
        const int r = list[j];
        MB_TRY(sg.upload(m->g_ids.as<long long>() + (size_t)r * ids_ld, h_ids[j], ids_ld));
        MB_TRY(sg.upload(ragged_rows(gs) + r, h_rs[j], 1));
        MB_TRY(sg.upload(m->g_cfg.as<SampleConfig>() + r, h_cfg[j], 1));
        MB_TRY(sg.upload(m->g_vflags.as<unsigned char>() + (size_t)r * Vin, h_vf[j], Vin));
        for (int i = 0; i < nr; ++i) MB_TRY(sg.upload(rowslot + r + i * N, h_slot[j], 1));      // decode rows r, N + r
        MB_TRY(sg.upload(rowslot + m->max_rows + 2 * r, h_slot[j], 2));                         // the prefill's (slot, slot) pair
    }
    MB_TRY(sg.end());
    for (int j = 0; j < n; ++j) {
        const int r = list[j];
        s->status[r] = mb200_stream::LIVE;
        s->prompt_len[r] = prompt_off[j + 1] - prompt_off[j];
        s->max_length[r] = params[j].max_length;
        s->first_poll[r] = std::min(std::max(params[j].min_new_tokens, 1), params[j].max_length - s->prompt_len[r]);   // no earlier stop
        s->selections[r] = 1;
    }
    // ---- launches ----
    MB_TRY(launch_prompt_scan_ragged(m->g_ids.as<long long>(), ids_ld, n, gs, m->g_vflags.as<unsigned char>(), Vin, params[0].time_shift_start,
                                     params[0].time_shift_end, m->g_lastts.as<int>(), st, d_list));
    // prefill of request j == the prefill of its batch-1 call, into cache rows r (and N + r); its last-position logits land in the
    // logits rows of the same index
    for (int j = 0; j < n; ++j) {
        const int P = prompt_off[j + 1] - prompt_off[j], r = list[j];
        MB_TRY(decoder_prefill(m, nr, P, m->g_prefill_ids.as<long long>() + pre_off[j], 0, st, r, N, rowslot + m->max_rows + 2 * r));
        const bool wbf = token_bf16(m);
        GemvParams g = final_logits_params(m, nr, m->p_x.as<float>() + (size_t)(P - 1) * d, (long long)P * d, wbf);
        g.seg[0].out += (size_t)r * V; g.seg[0].out_bs = (long long)N * V;
        MB_TRY(launch_gemv(g, st, false, false, GEMV_FORM_KERNEL, wbf));
    }
    // the list selection sets all_finished again if every row of the stream is finished after it
    MB_CUDA_CHECK(cudaMemsetAsync(&gs->all_finished, 0, sizeof(int), st));
    MB_TRY(launch_sample_rows(sample_params(m, s->rows), d_list, n, st));
    for (int j = 0; j < n; ++j) rows_out[j] = list[j];
    return 0;
}

// Replays the step graph for one burst (its length to *steps), then reads the rows' state back; the rows that finished are written to
// done_rows / done_len.
// The burst is short while requests wait for a row (`waiting` > 0), so a freed row is refilled within a step or two; otherwise it is 16
// steps, stretched until the first live row could stop and cut at the step where the last one must stop.
int stream_run(mb200_stream* s, int waiting, int32_t* done_rows, int32_t* done_len, int32_t* n_done, int32_t* steps, cudaStream_t st) {
    mb200_model* m = s->m;
    *n_done = 0;
    *steps = 0;
    int remaining = 0, earliest = INT32_MAX, live = 0;
    for (int r = 0; r < s->N; ++r) {
        if (s->status[r] != mb200_stream::LIVE) continue;
        ++live;
        remaining = std::max(remaining, s->max_length[r] - (s->prompt_len[r] + s->selections[r]));
        earliest = std::min(earliest, s->first_poll[r] - s->selections[r]);
    }
    if (!live) return 0;
    const int burst = std::max(0, std::min(remaining, std::max(waiting > 0 ? 2 : 16, earliest)));
    MB_TRY(s->step.launch(st, burst));
    *steps = burst;
    MB_CUDA_CHECK(cudaMemcpyAsync(s->h_rows, ragged_rows(m->g_state.as<GenState>()), (size_t)s->N * sizeof(RowState), cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int r = 0; r < s->N; ++r) {
        if (s->status[r] != mb200_stream::LIVE) continue;
        s->selections[r] += burst;
        const RowState& rs = s->h_rows[r];
        if (!rs.finished) continue;
        MB_REQUIRE(rs.cur_len > s->prompt_len[r] && rs.cur_len <= s->max_length[r], "a stream row finished with an out-of-range length");
        s->status[r] = mb200_stream::DONE;
        s->done_len[r] = rs.cur_len;
        done_rows[*n_done] = r; done_len[*n_done] = rs.cur_len; ++*n_done;
    }
    return 0;
}

// Copies a finished row's ids (prompt + generated, done_len of them) into out (host, out_ld wide) and frees the row.  Synchronises `st`.
int stream_take(mb200_stream* s, int row, int64_t* out, int32_t out_ld, cudaStream_t st) {
    MB_REQUIRE(row >= 0 && row < s->N && s->status[row] == mb200_stream::DONE, "the row holds no finished request");
    MB_REQUIRE(out && out_ld >= s->done_len[row], "output row is shorter than the request's ids");
    MB_CUDA_CHECK(cudaMemcpyAsync(out, s->m->g_ids.as<long long>() + (size_t)row * s->m->cfg.tgt_seq_len, (size_t)s->done_len[row] * 8,
                                  cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    s->status[row] = mb200_stream::FREE;
    return 0;
}

}  // namespace

extern "C" int mb200_stream_open(mb200_model* m, int32_t capacity, int32_t use_cfg, int32_t max_length, mb200_stream** out, void* stream) {
    MB_REQUIRE(m && m->finalized, "model not finalized");
    MB_REQUIRE(out, "null argument");
    MB_REQUIRE(!m->live_stream, "a decode stream is already open on this engine");
    mb200_stream* s = new mb200_stream();
    const int e = stream_open(m, s, capacity, use_cfg != 0, max_length, (cudaStream_t)stream);
    if (e) { stream_release(s); delete s; return e; }
    m->live_stream = s;
    *out = s;
    return 0;
}

extern "C" int mb200_stream_admit(mb200_stream* s, int32_t n, const int32_t* slots, const int64_t* prompt, const int32_t* prompt_off,
                                  const int64_t* neg_prompt, const uint8_t* vflags, const mb200_generate_params* params, int32_t* rows_out,
                                  void* stream) {
    MB_REQUIRE(s && s->m, "stream not open");
    return stream_admit(s, n, slots, prompt, prompt_off, neg_prompt, vflags, params, rows_out, (cudaStream_t)stream);
}

extern "C" int mb200_stream_run(mb200_stream* s, int32_t waiting, int32_t* done_rows, int32_t* done_len, int32_t* n_done, int32_t* steps,
                                void* stream) {
    MB_REQUIRE(s && s->m, "stream not open");
    MB_REQUIRE(done_rows && done_len && n_done && steps, "null argument");
    return stream_run(s, waiting, done_rows, done_len, n_done, steps, (cudaStream_t)stream);
}

extern "C" int mb200_stream_take(mb200_stream* s, int32_t row, int64_t* out_ids, int32_t out_ld, void* stream) {
    MB_REQUIRE(s && s->m, "stream not open");
    return stream_take(s, row, out_ids, out_ld, (cudaStream_t)stream);
}

extern "C" void mb200_stream_close(mb200_stream* s) {
    if (!s) return;
    if (s->m && s->m->live_stream == s) s->m->live_stream = nullptr;
    stream_release(s);
    delete s;
}

// Ragged batched generate: n_req INDEPENDENT requests in one token loop, each row bit-identical in its ids to its own batch-1
// mb200_model_generate call — a stream of capacity n_req and the largest max_length as its cap, every request admitted at once, run to
// the end.  Every bound is checked before anything is launched.
extern "C" int mb200_model_generate_ragged(mb200_model* m, int32_t n_req, const int32_t* slots, const int64_t* prompt, const int32_t* prompt_off,
                                           const int64_t* neg_prompt, const uint8_t* vflags, const mb200_generate_params* params,
                                           int64_t* out_ids, int32_t out_ld, int32_t* out_len, void* stream) {
    MB_REQUIRE(m && m->finalized, "model not finalized");
    MB_TRY(token_loop_free(m));
    MB_REQUIRE(slots && prompt && prompt_off && vflags && params && out_ids && out_len, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const bool use_cfg = neg_prompt != nullptr;
    const int N = n_req;
    MB_REQUIRE(N >= 1 && (use_cfg ? 2 * N : N) <= m->max_rows, "requests exceed max_batch (rows double under classifier-free guidance)");
    MB_TRY(check_requests(m, N, slots, prompt, prompt_off, neg_prompt, params, m->cfg.tgt_seq_len));
    int cap = 2;
    for (int r = 0; r < N; ++r) {
        MB_REQUIRE(params[r].max_length <= out_ld, "output rows are shorter than a request's max_length");
        cap = std::max(cap, (int)params[r].max_length);
    }
    mb200_stream s;
    int e = stream_open(m, &s, N, use_cfg, cap, st);
    std::vector<int32_t> rows(N), done_rows(N), done_len(N);
    if (!e) e = stream_admit(&s, N, slots, prompt, prompt_off, neg_prompt, vflags, params, rows.data(), st);
    int left = N;
    while (!e && left > 0) {
        int32_t n_done = 0, steps = 0;
        e = stream_run(&s, 0, done_rows.data(), done_len.data(), &n_done, &steps, st);
        for (int k = 0; !e && k < n_done; ++k) {
            const int j = done_rows[k];        // all admitted at once into an empty stream: request j holds row j
            e = stream_take(&s, done_rows[k], out_ids + (size_t)j * out_ld, out_ld, st);
            out_len[j] = done_len[k];
            --left;
        }
    }
    stream_release(&s);
    return e;
}

static int ensure_beam_buffers(mb200_model* m) {
    const size_t R = (size_t)m->max_rows, ld = (size_t)m->cfg.tgt_seq_len, V = (size_t)m->cfg.vocab_size_out;
    MB_TRY(m->b_kvsrc.ensure(R * ld * sizeof(int)));
    MB_TRY(m->b_logprobs.ensure(R * V * sizeof(float)));
    MB_TRY(m->b_cand.ensure(R * V * sizeof(float)));
    MB_TRY(m->b_runscore.ensure(R * sizeof(float)));
    MB_TRY(m->b_finids[0].ensure(R * ld * 8)); MB_TRY(m->b_finids[1].ensure(R * ld * 8));
    MB_TRY(m->b_finscore.ensure(R * sizeof(float))); MB_TRY(m->b_finlen.ensure(R * sizeof(int)));
    MB_TRY(m->b_finflag.ensure(R)); MB_TRY(m->b_unsat.ensure(R));
    return 0;
}

static BeamParams beam_params(mb200_model* m, int rows, int K) {
    const int V = m->cfg.vocab_size_out;
    BeamParams bp{};
    bp.sample = sample_params(m, rows);
    bp.sample.logits = m->b_logprobs.as<float>(); bp.sample.logits_ld = V;
    bp.logits = m->d_logits.as<float>(); bp.logits_ld = V;
    bp.logprobs = m->b_logprobs.as<float>(); bp.cand = m->b_cand.as<float>(); bp.run_score = m->b_runscore.as<float>();
    bp.kv_src = m->b_kvsrc.as<int>(); bp.kv_src_ld = m->cfg.tgt_seq_len;
    bp.fin_ids[0] = m->b_finids[0].as<long long>(); bp.fin_ids[1] = m->b_finids[1].as<long long>();
    bp.fin_score = m->b_finscore.as<float>(); bp.fin_len = m->b_finlen.as<int>(); bp.fin_flag = m->b_finflag.as<unsigned char>();
    bp.unsat = m->b_unsat.as<unsigned char>();
    bp.K = K; bp.V = V; bp.ids_ld = m->cfg.tgt_seq_len;
    return bp;
}

// =====================================================================================================================
// Beam search (num_beams = K in [2, 4]): HF's repeat_interleave expansion to B*K rows (2*B*K under classifier-free guidance),
// prefill, the first selection with running scores [0, -1e9, ...], then one CUDA-graph replay per token (per-phase kernels only;
// the megakernels stay greedy / sampling).  The self-attention cache is never copied: each row reads its history through the
// source-row table that the selection kernel gathers by parent.
extern "C" int mb200_model_generate_beams(mb200_model* m, const int32_t* slots, int32_t B, const int64_t* prompt, const uint8_t* prompt_mask,
                                          int32_t P, const int64_t* neg_prompt, const uint8_t* neg_mask, const uint8_t* vflags,
                                          const mb200_generate_params* gp, int32_t num_beams, int64_t fill_id, int64_t* out_ids,
                                          int32_t* out_len, float* out_scores, void* stream) {
    MB_REQUIRE(m && m->finalized, "model not finalized");
    MB_TRY(token_loop_free(m));
    MB_REQUIRE(slots && prompt && vflags && gp && out_ids && out_len && out_scores, "null argument");
    const auto& c = m->cfg;
    cudaStream_t st = (cudaStream_t)stream;
    const int K = num_beams;
    MB_REQUIRE(K >= 2 && K <= 4, "num_beams must be in [2, 4]");
    MB_REQUIRE(!gp->do_sample, "beam sampling (do_sample with num_beams > 1) is not supported");
    const bool use_cfg = neg_prompt != nullptr;
    const int BK = B * K, rows = use_cfg ? 2 * BK : BK;
    MB_REQUIRE(B >= 1 && rows <= m->max_rows, "batch * num_beams (x2 under classifier-free guidance) exceeds max_batch");
    MB_REQUIRE(P >= 1 && P < gp->max_length && gp->max_length <= c.tgt_seq_len, "need 1 <= prompt_len < max_length <= tgt_seq_len");
    const int d = c.d_model, V = c.vocab_size_out, ids_ld = c.tgt_seq_len;
    MB_REQUIRE(beam_select_smem_bytes(K, V, ids_ld) <= 220 * 1024, "beam candidates do not fit shared memory");
    MB_TRY(ensure_beam_buffers(m));

    // ---- call state: row r is beam (r mod B*K) % K of item (r mod B*K) / K; rows [0, B*K) carry the negative prompt under CFG ----
    Stager sg{m, st};
    MB_TRY(sg.begin());
    long long* pre = sg.reserve<long long>((size_t)rows * P);
    long long* idsrow = sg.reserve<long long>((size_t)BK * ids_ld);
    unsigned char* kv = sg.reserve<unsigned char>((size_t)rows * ids_ld);
    int* leftpad = sg.reserve<int>(rows);
    int* rowslot = sg.reserve<int>(rows);
    unsigned char* vf = sg.reserve<unsigned char>(c.vocab_size_in);
    GenState* gs = sg.reserve<GenState>(1);
    SampleConfig* sc = sg.reserve<SampleConfig>(1);
    int* kvsrc = sg.reserve<int>((size_t)rows * ids_ld);
    float* runscore = sg.reserve<float>(BK);
    float* finscore = sg.reserve<float>(BK);
    MB_TRY(sg.fits());
    MB_TRY(build_prompt_rows(m, rows, P, [&](int r) { return (r % BK) / K; }, use_cfg ? BK : 0, slots, prompt, prompt_mask, neg_prompt,
                             neg_mask, pre, kv, leftpad, rowslot));
    for (int r = 0; r < rows; ++r)      // every row reads its own prompt keys
        for (int t = 0; t < ids_ld; ++t) kvsrc[(size_t)r * ids_ld + t] = t < P ? r : 0;
    for (int j = 0; j < BK; ++j)
        for (int t = 0; t < ids_ld; ++t) idsrow[(size_t)j * ids_ld + t] = t < P ? prompt[(size_t)(j / K) * P + t] : gp->pad_token_id;
    for (int j = 0; j < BK; ++j) {
        runscore[j] = j % K == 0 ? 0.f : -1.0e9f;
        finscore[j] = -1.0e9f;
    }
    std::memcpy(vf, vflags, c.vocab_size_in);
    *gs = GenState{};
    gs->cur_len = P; gs->prompt_len = P; gs->max_length = gp->max_length; gs->min_new_tokens = gp->min_new_tokens;
    *sc = make_sample_config(gp, BK, use_cfg, V, ids_ld);
    MB_TRY(sg.upload(m->g_prefill_ids.p, pre, (size_t)rows * P));
    MB_TRY(sg.upload(m->g_ids.p, idsrow, (size_t)BK * ids_ld));
    MB_TRY(sg.upload(m->g_keyvalid.p, kv, (size_t)rows * ids_ld));
    MB_TRY(sg.upload(m->g_leftpad.p, leftpad, rows));
    MB_TRY(sg.upload(m->g_rowslot.p, rowslot, rows));
    MB_TRY(sg.upload(m->g_vflags.p, vf, c.vocab_size_in));
    MB_TRY(sg.upload(m->g_state.p, gs, 1));
    MB_TRY(sg.upload(m->g_cfg.p, sc, 1));
    MB_TRY(sg.upload(m->b_kvsrc.p, kvsrc, (size_t)rows * ids_ld));
    MB_TRY(sg.upload(m->b_runscore.p, runscore, BK));
    MB_TRY(sg.upload(m->b_finscore.p, finscore, BK));
    MB_TRY(sg.end());
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_finlen.p, 0, BK * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_finflag.p, 0, BK, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_unsat.p, 1, B, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->d_ticket.p, 0, (size_t)m->max_rows * m->cfg.heads * sizeof(int), st));

    const BeamParams bp = beam_params(m, rows, K);

    MB_TRY(launch_prompt_scan(m->g_ids.as<long long>(), ids_ld, BK, P, m->g_vflags.as<unsigned char>(), sc->ts_start, sc->ts_end,
                              m->g_lastts.as<int>(), st));
    MB_TRY(decoder_prefill(m, rows, P, m->g_prefill_ids.as<long long>(), gp->position_rule, st));
    MB_TRY(final_logits(m, rows, m->p_x.as<float>() + (size_t)(P - 1) * d, (long long)P * d, st, false));
    MB_TRY(launch_beam_step(bp, B, st));

    const int n_splits_self = self_splits(gp->max_length);
    auto key = std::make_tuple(rows, (int)B, n_splits_self, K);
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        CapturedGraph g;
        MB_TRY(capture_graph(m->cap_stream, st, [&](cudaStream_t cs) { return token_step(m, rows, B, n_splits_self, cs, m->use_pdl, nullptr, &bp); },
                             &g));
        it = m->graphs.emplace(key, g).first;
    }
    int remaining = gp->max_length - (P + 1);
    MB_CUDA_CHECK(cudaMemcpyAsync(m->h_flag, &m->g_state.as<GenState>()->all_finished, 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (*m->h_flag) remaining = 0;
    MB_TRY(replay_until_finished(m, it->second, remaining, 0, st));
    GenState fin{};
    MB_CUDA_CHECK(cudaMemcpyAsync(&fin, m->g_state.p, sizeof(fin), cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    // the finished store the last selection wrote (parity of the step count)
    std::vector<long long> fids((size_t)BK * ids_ld);
    std::vector<float> fscore(BK);
    std::vector<int> flen(BK);
    std::vector<unsigned char> fflag(BK);
    MB_CUDA_CHECK(cudaMemcpyAsync(fids.data(), m->b_finids[fin.step & 1].p, fids.size() * 8, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(fscore.data(), m->b_finscore.p, BK * 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(flen.data(), m->b_finlen.p, BK * 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(fflag.data(), m->b_finflag.p, BK, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    // best hypothesis per item, padded to P + the longest generated length with the filler id
    int gen_max = 0;
    for (int b = 0; b < B; ++b) {
        MB_REQUIRE(fflag[(size_t)b * K], "beam search ended without a finished hypothesis");
        gen_max = std::max(gen_max, flen[(size_t)b * K]);
    }
    const int Lout = P + gen_max;
    for (int b = 0; b < B; ++b) {
        const long long* h = fids.data() + (size_t)b * K * ids_ld;
        const int Lb = P + flen[(size_t)b * K];
        for (int t = 0; t < Lout; ++t) out_ids[(size_t)b * Lout + t] = t < Lb ? h[t] : fill_id;
        out_scores[b] = fscore[(size_t)b * K];
    }
    *out_len = Lout;
    return 0;
}

// Teacher-forced pass up to the final LayerNorm: stages ids / key mask / left padding / slots, runs the decoder prefill and leaves
// the normalised hidden states of all B * len positions in p_h (what the vocabulary projection reads).
static int teacher_forced_hidden(mb200_model* m, const int32_t* slots, int32_t B, const int64_t* ids, const uint8_t* mask, int32_t len,
                                 int32_t position_rule, cudaStream_t st) {
    MB_REQUIRE(m && m->finalized, "model not finalized");
    MB_TRY(token_loop_free(m));
    MB_REQUIRE(B >= 1 && B <= m->max_rows && len >= 1 && len <= m->cfg.tgt_seq_len, "bad batch / length");
    const auto& c = m->cfg;
    const int ids_ld = c.tgt_seq_len, d = c.d_model;
    Stager sg{m, st};
    MB_TRY(sg.begin());
    long long* pre = sg.reserve<long long>((size_t)B * len);
    unsigned char* kv = sg.reserve<unsigned char>((size_t)B * ids_ld);
    int* leftpad = sg.reserve<int>(B);
    int* rowslot = sg.reserve<int>(B);
    MB_TRY(sg.fits());
    MB_TRY(build_prompt_rows(m, B, len, [](int r) { return r; }, 0, slots, ids, mask, nullptr, nullptr, pre, kv, leftpad, rowslot));
    MB_TRY(sg.upload(m->g_prefill_ids.p, pre, (size_t)B * len));
    MB_TRY(sg.upload(m->g_keyvalid.p, kv, (size_t)B * ids_ld));
    MB_TRY(sg.upload(m->g_leftpad.p, leftpad, B));
    MB_TRY(sg.upload(m->g_rowslot.p, rowslot, B));
    MB_TRY(sg.end());
    MB_TRY(decoder_prefill(m, B, len, m->g_prefill_ids.as<long long>(), position_rule, st));
    MB_TRY(layernorm(m->p_x.as<float>(), m->p_h.as<float>(), m->dec_ln_w, m->dec_ln_b, B * len, d, 1e-5f, st));
    return 0;
}

extern "C" int mb200_model_forward_logits(mb200_model* m, const int32_t* slots, int32_t B, const int64_t* ids, const uint8_t* mask,
                                          int32_t len, int32_t position_rule, float* logits_out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    MB_TRY(teacher_forced_hidden(m, slots, B, ids, mask, len, position_rule, st));
    const auto& c = m->cfg;
    const int d = c.d_model;
    const int R = B * len;
    MB_TRY(launch_gemm(gemm_base(plain_map(m->p_h.as<float>(), d), m->proj_out, d, plain_map(logits_out, c.vocab_size_out), nullptr, R,
                                 c.vocab_size_out, d), st, &m->gemm));
    return 0;
}

// Rows of one projection chunk in mb200_model_score_tokens.  >= 512 so that every chunk of a call of more rows is a tensor-core GEMM,
// as the unchunked projection of forward_logits is; not a divisor of the usual B * L (powers of two), so the tests meet the overlapping
// last chunk.
static constexpr int SCORE_CHUNK_ROWS = 3072;

extern "C" int mb200_model_score_tokens(mb200_model* m, const int32_t* slots, int32_t B, const int64_t* ids, const uint8_t* mask,
                                        int32_t len, int32_t position_rule, float* entropy, float* surprisal, float* relative,
                                        int64_t* suggested, void* stream) {
    MB_REQUIRE(entropy && surprisal && relative && suggested, "null output");
    cudaStream_t st = (cudaStream_t)stream;
    MB_TRY(teacher_forced_hidden(m, slots, B, ids, mask, len, position_rule, st));
    const auto& c = m->cfg;
    const int d = c.d_model, V = c.vocab_size_out, R = B * len;
    const int chunk = std::min(R, SCORE_CHUNK_ROWS);
    MB_TRY(m->s_logits.ensure((size_t)chunk * V * sizeof(float)));
    ScoreParams sp{};
    sp.logits = m->s_logits.as<float>(); sp.ids = m->g_prefill_ids.as<long long>(); sp.L = len; sp.V = V;
    sp.entropy = entropy; sp.surprisal = surprisal; sp.relative = relative; sp.suggested = reinterpret_cast<long long*>(suggested);
    // Every chunk has the same M (the last one overlaps its predecessor instead of being short) and starts at m_base 0 of its own
    // A pointer: tc_gemm_eligible sends m_base != 0 or M < 512 to the SIMT kernel, whose sums differ in the last bits, so this keeps
    // each row on the GEMM path the single [R, V] projection of forward_logits takes, and every logit bit-identical to it.
    for (int r0 = 0; r0 < R; r0 += chunk) {
        const int row0 = std::min(r0, R - chunk);
        MB_TRY(launch_gemm(gemm_base(plain_map(m->p_h.as<float>() + (size_t)row0 * d, d), m->proj_out, d, plain_map(m->s_logits.as<float>(), V),
                                     nullptr, chunk, V, d), st, &m->gemm));
        sp.row0 = row0;
        MB_TRY(launch_score_rows(sp, chunk, st));
    }
    return 0;
}

// test / tuning hooks (not part of the reference-facing boundary)
extern "C" int mb200_model_set_option(mb200_model* m, const char* name, int value) {
    MB_REQUIRE(m && name, "null argument");
    if (!strcmp(name, "pdl")) {
        MB_TRY(token_loop_free(m));      // the toggle destroys every token-step graph, the open stream's among them
        if (m->use_pdl != (value != 0)) {
            for (auto& g : m->graphs) cudaGraphExecDestroy(g.second.exec);
            m->graphs.clear();
        }
        m->use_pdl = value != 0;
        return 0;
    }
    if (!strcmp(name, "mega")) { m->use_mega = value; return 0; }
    if (!strcmp(name, "ll_sleep")) return mega2_set_poll_sleep(value);
    if (!strcmp(name, "enc_graph")) { m->enc_graph = value; return 0; }
    if (!strcmp(name, "trace_cta")) { m->trace_cta = value; return 0; }
    if (!strcmp(name, "ll_debug")) return mega2_set_debug(value);
    if (!strcmp(name, "ll_reps")) {
        MB_REQUIRE(value >= 1 && value <= MEGA_LL_MAX_REPS && value * 2 <= 32, "ll_reps must be in [1, 16]");
        m->ll.reps = value;
        return 0;
    }
    if (!strcmp(name, "mega_trace")) {
        if (value) { MB_TRY(m->mega_trace.ensure(128 * 16 * 8)); MB_CUDA_CHECK(cudaMemset(m->mega_trace.p, 0, 128 * 16 * 8)); }
        return 0;
    }
    set_last_error(std::string("unknown option ") + name);
    return 2;
}

// Measurement hook for bench.py: replays the token step EAGERLY `iters` times on the state left by the last generate() call,
// bracketing every decode-path launch with CUDA events on the launching stream.  out_us[0..2] = device microseconds per token
// spent in {gemv, split-KV attention, logits/sample} kernels, out_us[3] = their launch counts packed as gemv*1e6 + attn*1e3 + sample.
extern "C" int mb200_model_profile_step(mb200_model* m, int32_t rows, int32_t B, int32_t max_length, int32_t iters, float* out_us, void* stream) {
    MB_REQUIRE(m && m->finalized && out_us && iters >= 1, "bad argument");
    MB_TRY(token_loop_free(m));
    cudaStream_t st = (cudaStream_t)stream;
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    GenState gs{};
    MB_CUDA_CHECK(cudaMemcpy(&gs, m->g_state.p, sizeof(gs), cudaMemcpyDeviceToHost));
    const int cur0 = gs.prompt_len + 1;
    double acc[3] = {0, 0, 0}; long long cnt[3] = {0, 0, 0};
    if (!g_prof.created) { for (auto& e : g_prof.ev) MB_CUDA_CHECK(cudaEventCreate(&e)); g_prof.created = true; }
    const int n_splits_self = self_splits(max_length);
    for (int it = 0; it < iters; ++it) {
        gs.cur_len = cur0 + it; gs.all_finished = 0; gs.n_finished = 0; gs.ticket = 0; gs.max_length = m->cfg.tgt_seq_len; gs.min_new_tokens = 0;
        MB_CUDA_CHECK(cudaMemcpy(m->g_state.p, &gs, sizeof(gs), cudaMemcpyHostToDevice));
        MB_CUDA_CHECK(cudaMemset(m->g_finished.p, 0, m->max_rows));
        g_prof.n = 0; g_prof.on = true;
        int s = token_step(m, rows, B, n_splits_self, st, false);
        g_prof.on = false;
        if (s) return s;
        MB_CUDA_CHECK(cudaStreamSynchronize(st));
        for (int i = 0; i < g_prof.n; ++i) {
            float ms = 0.f;
            MB_CUDA_CHECK(cudaEventElapsedTime(&ms, g_prof.ev[2 * i], g_prof.ev[2 * i + 1]));
            acc[g_prof.cls[i]] += ms * 1000.0; cnt[g_prof.cls[i]]++;
        }
    }
    for (int c = 0; c < 3; ++c) out_us[c] = (float)(acc[c] / iters);
    out_us[3] = (float)((cnt[0] / iters) * 1000000LL + (cnt[1] / iters) * 1000LL + (cnt[2] / iters));
    return 0;
}

// debug: copy the megakernel phase trace (option "mega_trace") to host: out[n_phases][16] SM-cycle stamps
extern "C" int mb200_model_read_trace(mb200_model* m, uint64_t* out, int32_t n_phases) {
    MB_REQUIRE(m && out && m->mega_trace.p && n_phases <= 128, "trace not enabled");
    MB_CUDA_CHECK(cudaDeviceSynchronize());
    MB_CUDA_CHECK(cudaMemcpy(out, m->mega_trace.p, (size_t)n_phases * 16 * 8, cudaMemcpyDeviceToHost));
    return 0;
}

// Measurement hook: CUDA-event totals of the persistent token-loop kernel since the last reset:
// out[0] = launches, out[1] = total device milliseconds, out[2] = tokens decoded inside those launches.
extern "C" int mb200_model_mega_stats(mb200_model* m, double* out, int32_t reset) {
    MB_REQUIRE(m && out, "null argument");
    out[0] = (double)m->mega_launches; out[1] = m->mega_ms; out[2] = (double)m->mega_tokens;
    if (reset) { m->mega_launches = 0; m->mega_ms = 0.0; m->mega_tokens = 0; }
    return 0;
}

// Parity hook for the fused logits-processor chain (tests; not part of the reference-facing boundary): runs ONE selection step of
// `sample_body` on caller-supplied logits.  logits: DEVICE [rows, V] (rows = 2B under CFG, negative-prompt rows first);
// ids: HOST [B, L] the tokens so far (prompt + generated); `step` / `has_last_scores` select the look-back-bias state left by the
// previous call (scores are double-buffered by step parity, exactly as in generation).  Outputs: scores_out DEVICE [B, V] = the scores
// the selection sees (-inf where MinNewTokens / MonotonicTimeShift / LookbackBias / top-k / top-p removed the id), chosen_out HOST [B].
extern "C" int mb200_model_logits_chain(mb200_model* m, const float* logits, int32_t B, int32_t use_cfg, const int64_t* ids, int32_t L,
                                        int32_t prompt_len, const uint8_t* vflags, const mb200_generate_params* gp, int32_t step,
                                        int32_t has_last_scores, float* scores_out, int64_t* chosen_out, void* stream) {
    MB_REQUIRE(m && m->finalized && logits && ids && vflags && gp && scores_out && chosen_out, "null argument");
    MB_TRY(token_loop_free(m));
    const auto& c = m->cfg;
    const int rows = use_cfg ? 2 * B : B, V = c.vocab_size_out, ids_ld = c.tgt_seq_len;
    MB_REQUIRE(B >= 1 && rows <= m->max_rows && L >= 1 && L < ids_ld, "bad batch / length");
    cudaStream_t st = (cudaStream_t)stream;
    Stager sg{m, st};
    MB_TRY(sg.begin());
    long long* idsrow = sg.reserve<long long>((size_t)B * ids_ld);
    unsigned char* vf = sg.reserve<unsigned char>(c.vocab_size_in);
    GenState* gs = sg.reserve<GenState>(1);
    SampleConfig* sc = sg.reserve<SampleConfig>(1);
    MB_TRY(sg.fits());
    for (int b = 0; b < B; ++b)
        for (int t = 0; t < ids_ld; ++t) idsrow[(size_t)b * ids_ld + t] = t < L ? ids[(size_t)b * L + t] : gp->pad_token_id;
    std::memcpy(vf, vflags, c.vocab_size_in);
    *gs = GenState{};
    gs->cur_len = L; gs->prompt_len = prompt_len; gs->max_length = gp->max_length; gs->min_new_tokens = gp->min_new_tokens;
    gs->step = step; gs->has_last_scores = has_last_scores;
    *sc = make_sample_config(gp, B, use_cfg != 0, V, ids_ld);
    MB_TRY(sg.upload(m->g_ids.p, idsrow, (size_t)B * ids_ld));
    MB_TRY(sg.upload(m->g_vflags.p, vf, c.vocab_size_in));
    MB_TRY(sg.upload(m->g_state.p, gs, 1));
    MB_TRY(sg.upload(m->g_cfg.p, sc, 1));
    MB_TRY(sg.end());
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_leftpad.p, 0, rows * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_finished.p, 0, m->max_rows, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->d_logits.p, logits, (size_t)rows * V * 4, cudaMemcpyDeviceToDevice, st));
    MB_TRY(launch_prompt_scan(m->g_ids.as<long long>(), ids_ld, B, L, m->g_vflags.as<unsigned char>(), sc->ts_start, sc->ts_end, m->g_lastts.as<int>(), st));
    SampleParams sp = sample_params(m, rows);
    sp.dbg_scores = scores_out;
    MB_TRY(launch_sample(sp, B, st, false));
    std::vector<long long> chosen(B);
    MB_CUDA_CHECK(cudaMemcpy2DAsync(chosen.data(), 8, m->g_ids.as<long long>() + L, (size_t)ids_ld * 8, 8, B, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b) chosen_out[b] = chosen[b];
    return 0;
}

// Parity hook for beam search (tests; not part of the reference-facing boundary): ONE selection step of the beam kernels on
// caller-supplied logits, from an empty finished store.  logits DEVICE [rows, V] (rows = 2*B*K under CFG, negative-prompt rows first);
// ids HOST [B*K, L] the running sequences; run_scores HOST [B*K]; `step` / `has_last_scores` as in mb200_model_logits_chain.
// Outputs: logprobs_out DEVICE [B*K, V] = the processed log-probs (before the running score is added); HOST [B*K]: top_out = the first
// K candidates of each item (flat index beam * V + token, in order), parent_out = the batch row each new running beam continues,
// token_out / score_out = its token and running score, fin_score_out / fin_len_out / fin_flag_out = the finished store
// (-1e9 / 0 / 0 where empty); fin_ids_out HOST [B*K, L + 1] its ids.
extern "C" int mb200_model_beam_step(mb200_model* m, const float* logits, int32_t B, int32_t num_beams, int32_t use_cfg, const int64_t* ids,
                                     int32_t L, int32_t prompt_len, const uint8_t* vflags, const mb200_generate_params* gp,
                                     const float* run_scores, int32_t step, int32_t has_last_scores, float* logprobs_out, int32_t* top_out,
                                     int32_t* parent_out, int64_t* token_out, float* score_out, float* fin_score_out, int32_t* fin_len_out,
                                     uint8_t* fin_flag_out, int64_t* fin_ids_out, void* stream) {
    MB_REQUIRE(m && m->finalized && logits && ids && vflags && gp && run_scores && logprobs_out && top_out && parent_out && token_out &&
               score_out && fin_score_out && fin_len_out && fin_flag_out && fin_ids_out, "null argument");
    MB_TRY(token_loop_free(m));
    const auto& c = m->cfg;
    const int K = num_beams, BK = B * K, rows = use_cfg ? 2 * BK : BK, V = c.vocab_size_out, ids_ld = c.tgt_seq_len;
    MB_REQUIRE(K >= 2 && K <= 4, "num_beams must be in [2, 4]");
    MB_REQUIRE(B >= 1 && rows <= m->max_rows && prompt_len >= 1 && L >= prompt_len && L < ids_ld && L < gp->max_length, "bad batch / length");
    MB_REQUIRE(beam_select_smem_bytes(K, V, ids_ld) <= 220 * 1024, "beam candidates do not fit shared memory");
    cudaStream_t st = (cudaStream_t)stream;
    MB_TRY(ensure_beam_buffers(m));
    Stager sg{m, st};
    MB_TRY(sg.begin());
    long long* idsrow = sg.reserve<long long>((size_t)BK * ids_ld);
    unsigned char* vf = sg.reserve<unsigned char>(c.vocab_size_in);
    GenState* gs = sg.reserve<GenState>(1);
    SampleConfig* sc = sg.reserve<SampleConfig>(1);
    float* runscore = sg.reserve<float>(BK);
    float* finscore = sg.reserve<float>(BK);
    MB_TRY(sg.fits());
    for (int j = 0; j < BK; ++j)
        for (int t = 0; t < ids_ld; ++t) idsrow[(size_t)j * ids_ld + t] = t < L ? ids[(size_t)j * L + t] : gp->pad_token_id;
    std::memcpy(vf, vflags, c.vocab_size_in);
    *gs = GenState{};
    gs->cur_len = L; gs->prompt_len = prompt_len; gs->max_length = gp->max_length; gs->min_new_tokens = gp->min_new_tokens;
    gs->step = step; gs->has_last_scores = has_last_scores;
    *sc = make_sample_config(gp, BK, use_cfg != 0, V, ids_ld);
    std::memcpy(runscore, run_scores, BK * sizeof(float));
    for (int j = 0; j < BK; ++j) finscore[j] = -1.0e9f;      // an empty finished store
    MB_TRY(sg.upload(m->g_ids.p, idsrow, (size_t)BK * ids_ld));
    MB_TRY(sg.upload(m->g_vflags.p, vf, c.vocab_size_in));
    MB_TRY(sg.upload(m->g_state.p, gs, 1));
    MB_TRY(sg.upload(m->g_cfg.p, sc, 1));
    MB_TRY(sg.upload(m->b_runscore.p, runscore, BK));
    MB_TRY(sg.upload(m->b_finscore.p, finscore, BK));
    MB_TRY(sg.end());
    MB_CUDA_CHECK(cudaMemsetAsync(m->g_leftpad.p, 0, rows * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_kvsrc.p, 0, (size_t)rows * ids_ld * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_finlen.p, 0, BK * sizeof(int), st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_finflag.p, 0, BK, st));
    MB_CUDA_CHECK(cudaMemsetAsync(m->b_unsat.p, 1, B, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(m->d_logits.p, logits, (size_t)rows * V * 4, cudaMemcpyDeviceToDevice, st));
    MB_TRY(launch_prompt_scan(m->g_ids.as<long long>(), ids_ld, BK, L, m->g_vflags.as<unsigned char>(), sc->ts_start, sc->ts_end,
                              m->g_lastts.as<int>(), st));
    BeamParams bp = beam_params(m, rows, K);
    bp.dbg_logprobs = logprobs_out;
    MB_TRY(m->b_dbg.ensure((size_t)2 * m->max_rows * sizeof(int)));
    bp.dbg_top = m->b_dbg.as<int>(); bp.dbg_parent = m->b_dbg.as<int>() + m->max_rows;
    MB_TRY(launch_beam_step(bp, B, st));
    std::vector<int> dbg((size_t)2 * m->max_rows);
    std::vector<long long> tok((size_t)BK * ids_ld), fids((size_t)BK * ids_ld);
    MB_CUDA_CHECK(cudaMemcpyAsync(dbg.data(), m->b_dbg.p, dbg.size() * 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(tok.data(), m->g_ids.p, tok.size() * 8, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(fids.data(), m->b_finids[1 - (step & 1)].p, fids.size() * 8, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(score_out, m->b_runscore.p, BK * 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(fin_score_out, m->b_finscore.p, BK * 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(fin_len_out, m->b_finlen.p, BK * 4, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(fin_flag_out, m->b_finflag.p, BK, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int j = 0; j < BK; ++j) {
        top_out[j] = dbg[j]; parent_out[j] = dbg[m->max_rows + j]; token_out[j] = tok[(size_t)j * ids_ld + L];
        for (int t = 0; t <= L; ++t) fin_ids_out[(size_t)j * (L + 1) + t] = fids[(size_t)j * ids_ld + t];
    }
    return 0;
}
