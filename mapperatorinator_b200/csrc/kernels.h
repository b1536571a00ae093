// Internal kernel-launch API of the engine (C++ side; the public C ABI is include/mapperatorinator_b200.h).
#pragma once
#include <unordered_map>
#include "common.cuh"

namespace mb200 {

// ---- gemm.cu ---------------------------------------------------------------------------------------------------------
struct GemmParams {
    RowMap A;               // [M, K]
    const float* W;         // [N, K] row-major
    long long ldw;
    RowMap C;               // [M, N]
    const float* bias;      // [N] or null
    int act;                // Act
    float alpha;            // applied after the activation
    const float* gate;      // per-sample channel gate: gate[(m / gate_rpb) * gate_ld + n], or null
    long long gate_ld;
    int gate_rpb;
    RowMap R;               // residual (ptr == null -> none)
    int M, N, K;
    // Split-K.  `splitk` = S is part of the ARITHMETIC of a (N, K) problem — it is chosen from N and K only, never from M or the grid
    // fill, so a row's result does not depend on how many other rows share the launch (one encoder window alone == the same
    // window inside a 16-window chunk, bit for bit).  k-range z = [z*k_per_split, (z+1)*k_per_split) is summed on its own and the
    // S partial sums are added in index order.  HOW the partials are realised is a launch decision that does not change a bit:
    //   split_mode 1 ("grid"):    CTA z = blockIdx.z writes raw partials to ws[z][M][N]; gemm_splitk_reduce_kernel adds them in order
    //                             and applies the epilogue (under-filled grids);
    //   split_mode 2 ("in-tile"): one CTA walks all of K with S accumulators (tensor-core path: one range at a time, a running sum in registers) and its epilogue
    //                             adds them in the same order (large M).
    float* splitk_ws; int splitk; int k_per_split; int split_mode;
    long long m_base;       // logical row of local row 0 (launch_gemm slices M when the partial planes of a grid split exceed the workspace)
};

// Per-engine GEMM scratch.  Nothing in here is shared between engines, devices or streams (round-1 had process globals: two
// engines on two streams raced on them, and a reallocation could pull memory from under a captured CUDA graph).
struct Tf32Mirror { const float* hi; const float* lo; };
struct GemmCtx {
    int num_sms = 132;
    float* splitk_ws = nullptr; size_t splitk_bytes = 0;        // [S][M][N] partial sums of the grid split
    float* a_split = nullptr; size_t a_split_bytes = 0;         // tf32 hi | lo copies of the activation operand (tensor-core path)
    int* tc_err = nullptr;                                      // device flag: 0 fine, 3 = a pipeline wait timed out
    bool frozen = false;                                        // set once a CUDA graph holds these pointers: reserve() may no longer move them
    std::unordered_map<const float*, Tf32Mirror> mirrors;       // weight matrix -> its tf32 hi / lo arrays (filled at finalize)
    int reserve(size_t splitk_need, size_t a_split_need);       // grow-only; fails loudly when frozen and too small
    int register_weight(const float* w, long long numel);
    void unregister_weight(const float* w);
    int error();                                                // reads tc_err
    void destroy();
};
GemmCtx* default_gemm_ctx();                                    // scratch of the kernel-level test entry points (mb200_op_gemm*)
int launch_gemm(const GemmParams& p, cudaStream_t stream, GemmCtx* ctx);
// gemm_tc.cu — wgmma 3xTF32 path (fp32-grade accuracy on the tensor cores); launch_gemm dispatches to it for large problems
// whose weight matrix has a registered tf32 "lo" mirror
extern int g_tc_enabled;
int launch_splitk_reduce(const GemmParams& q, cudaStream_t stream);
bool tc_gemm_eligible(const GemmParams& p, GemmCtx* ctx);
int launch_gemm_tc(const GemmParams& p, cudaStream_t stream, GemmCtx* ctx);
int gemm_splits_tc(int N, int K, int num_sms, int* k_per_split);      // S of the tensor-core path for an (N, K) problem
int gemm_splits_simt(int N, int K, int num_sms, int* k_per_split);    // S of the fp32 SIMT path

// ---- norm.cu ---------------------------------------------------------------------------------------------------------
// y[m, :] = LN(x[m, :]) * w + b                       (affine; w/b may be null)
// y[m, :] = LN(x[m, :]) * (1 + scale[b, :]) + shift[b, :]   (adaLN modulate; b = m / rows_per_batch)
struct LayerNormParams {
    const float* x; long long ldx;
    float* y; long long ldy;
    const float* weight; const float* bias;
    const float* shift; const float* scale; long long mod_ld; int rows_per_batch;
    int rows, dim;
    float eps;
};
int launch_layernorm(const LayerNormParams& p, cudaStream_t stream);

// ---- attention.cu ----------------------------------------------------------------------------------------------------
enum MaskMode : int { MASK_NONE = 0, MASK_CAUSAL = 1, MASK_BAND = 2, MASK_DENSE = 3 };
struct AttentionParams {
    // token-major operands: element (b, t, h, d) at ptr + b*bstride + t*ld + h*64 + d ; head_dim is fixed at 64
    const float* q; long long q_ld, q_bs;
    const float* k; long long k_ld, k_bs;
    const float* v; long long v_ld, v_bs;
    float* o; long long o_ld, o_bs;
    int B, H, Tq, Tk;
    float scale;                   // multiplies q.k (1.0 when q is pre-scaled like HF Whisper)
    int mask_mode;
    int q_pos0;                    // MASK_CAUSAL: absolute position of query row 0 (keys are absolute 0..Tk-1)
    const unsigned char* key_valid; long long key_valid_ld;   // [B, Tk] 1 = real token (null = all valid)
    int band;                      // MASK_BAND: query r sees key c iff c - band <= r < c + band
    const unsigned char* dense;    // MASK_DENSE: [Tq, Tk] 1 = blocked
    const int* kv_slot;            // optional: K/V batch index of batch row b (cross attention over resident encoder slots)
};
// Per-engine scratch of the tensor-core attention path (attention_tc.cu): head-major tf32 hi / lo copies of q, k and v^T.
struct AttnCtx {
    void* ws = nullptr; size_t ws_bytes = 0;
    int* err = nullptr;                              // device flag: 0 fine, 5 = a pipeline wait timed out
    bool frozen = false;                             // set once a CUDA graph holds the workspace address
    int reserve(size_t bytes);                       // grow-only; fails loudly when frozen and too small
    int error();
    void destroy();
};
extern int g_attn_tc_enabled, g_attn_tc_min_t;
size_t attn_tc_workspace_bytes(int B, int H, int Tq, int Tk);
bool attn_tc_eligible(const AttentionParams& p, const AttnCtx* ctx);
int launch_attention_tc(const AttentionParams& p, cudaStream_t stream, AttnCtx* ctx);
// ctx != null and an eligible problem (no dense mask, no kv_slot gather, enough queries): wgmma flash attention; else the fp32 SIMT kernel
int launch_attention(const AttentionParams& p, cudaStream_t stream, AttnCtx* ctx = nullptr);

// ---- slider.cu: slider end-point recompute of the diffusion denoised_fn (diffusion_pipeline.py:203-222) -------------------
struct SliderSet {                 // device arrays describing the sliders that lie fully inside the current chunk
    int n;
    const int* cp_offsets;         // [n + 1] prefix offsets into cp_index
    const int* cp_index;           // chunk-relative sequence index of every control point (head, anchors ..., last anchor)
    const int* end_index;          // [n] chunk-relative sequence index of the slider-end event
    const int* type;               // [n] 0 Bezier, 1 PerfectCurve, 2 Catmull, 3 Linear
    const float* length;           // [n] slider length in osu! pixels
};
// x: DEVICE [N, 2, T] normalised coordinates, updated in place: conditional half -> pixels, every slider end moved to
// position_at(length / max_length) of its path, pixels written back to BOTH halves.  pix_scratch: >= 2*T floats.
int launch_slider_recompute(const SliderSet& sl, float* x, int N, int T, float* pix_scratch, int* error_flag, cudaStream_t st);

// ---- audio.cu: PCM at the file's rate -> mono float32 at the model rate (the CPU tail of data_utils.py:80-101 load_audio_file) ----
long long audio_out_frames(long long n_in, int in_rate, int out_rate);
// pcm: DEVICE int16 [n_frames, channels] interleaved; out: DEVICE float32 [audio_out_frames]; scratch: DEVICE int (peak)
int launch_audio_ingest(const short* pcm, long long n_frames, int channels, int in_rate, int out_rate, int normalize, float* out, int* scratch,
                        int num_sms, cudaStream_t stream);

// ---- mel.cu ----------------------------------------------------------------------------------------------------------
struct MelPlan;   // opaque (filterbank in CSR form + twiddles on device)
int mel_plan_create(MelPlan** out, int n_fft, int hop, int n_mels, int pad_reflect, int log_scale,
                    const float* mel_basis_host /* [n_mels, n_fft/2+1] */);
void mel_plan_destroy(MelPlan* p);
// pcm [B, n_samples] (row stride pcm_ld) -> mel [B, frames, n_mels] via RowMap-like strides (frames = n_samples/hop + 1)
int launch_mel(const MelPlan* plan, const float* pcm, long long pcm_ld, int B, int n_samples, float* mel, long long mel_ld,
               long long mel_bs, cudaStream_t stream);

// ---- score.cu: per-token statistics of a teacher-forced pass (processor.py:519-525) ------------------------------------
struct ScoreParams {
    const float* logits;           // [rows, V]: the projection rows row0 .. row0 + rows - 1 of the call
    long long row0;                // global row (b * L + t) of logits row 0
    const long long* ids;          // DEVICE [B * L] given ids (row r's target is ids[r + 1] when t + 1 < L)
    int L, V;
    float *entropy, *surprisal, *relative;   // DEVICE [B * L], indexed by the scored token
    long long* suggested;
};
int launch_score_rows(const ScoreParams& p, int rows, cudaStream_t stream);

}  // namespace mb200

// =====================================================================================================================
// decode.cu — the per-token path (B small): weight-streaming GEMV family, split-KV decode attention, fused
// logits-processor chain + token selection.  All step-varying scalars live in device memory (GenState) so that one
// captured CUDA graph replays for every token of every generate() call.
// =====================================================================================================================
namespace mb200 {

// vocabulary flag bits (host builds vflags[vocab_in] per call; only VF_EOS changes between calls)
enum : unsigned char { VF_EOS = 1, VF_TIMED = 2, VF_SOS = 4, VF_LB_EOS = 8, VF_BEAT = 16, VF_MANIA = 32, VF_SCROLL = 64 };

struct GenState {            // device-resident, one per engine
    int cur_len;             // tokens currently in every ids row (prompt + generated); next token goes to ids[b][cur_len]
    int prompt_len;          // P
    int max_length;
    int min_new_tokens;
    int n_finished;
    int ticket;              // last-CTA detection in the sampling kernel
    int all_finished;
    int has_last_scores;
    int step;                // decode steps since the start of this call (RNG counter; a ragged row counts its own in RowState)
    int n_req;               // ragged call: un-doubled rows of the call (0 in a uniform call)
    int pad_[6];
};

// Ragged call and decode stream (mb200_model_generate_ragged, mb200_stream_*): every request is its own batch-1 call.  The GenState
// above keeps what the rows share (the tickets, all_finished, n_req); what differs per row follows it IN THE SAME device buffer, so a
// kernel that holds the GenState pointer finds row b's state at ragged_rows(st)[b].  Decoder row r (2B rows under CFG) belongs to
// request r % B.  Each row counts its own steps, so a request admitted into a running stream draws and looks back as its own call.
struct RowState {
    int cur_len;             // tokens in this row's ids (prompt + generated); its next token goes to ids[b][cur_len]
    int prompt_len;
    int max_length;
    int min_new_tokens;
    int finished;            // stopped on its own EOS set or max_length (or a vacant stream row): appends nothing, to its ids or cache
    int step;                // selections made since the row's prefill (RNG counter, parity of its look-back scores)
    int has_last_scores;     // the look-back bias has this row's previous scores
    int pad_;
};
__host__ __device__ inline const RowState* ragged_rows(const GenState* st) { return reinterpret_cast<const RowState*>(st + 1); }
__host__ __device__ inline RowState* ragged_rows(GenState* st) { return reinterpret_cast<RowState*>(st + 1); }

// split-KV layout of the self-attention cache of ONE call: one 128-key split while the context fits, 64-key splits beyond.  A ragged
// row keeps the plan of its own max_length, whatever its neighbours need: its partials and their merge order are its own call's.
__host__ __device__ inline int self_splits(int max_length) { return max_length <= 128 ? 1 : (max_length + 63) / 64; }
// keys per split of that plan: the single split holds all 128, every plan of several splits cuts 64-key chunks
__host__ __device__ inline int self_split_chunk(int n_splits) { return n_splits == 1 ? 128 : 64; }

struct SampleConfig {        // device-resident, rewritten by the host once per generate() call
    int B;                   // un-doubled batch rows
    int use_cfg;             // decoder rows = 2B; rows [0,B) carry the negative prompt (modeling_mapperatorinator.py:243-245)
    float cfg_scale;
    int V;                   // vocab_size_out
    int ts_start, ts_end;    // time-shift id range
    float timeshift_bias;
    int types_first;
    float temperature;
    int n_cond;              // conditional temperatures (logit_processors.py:62-71), evaluated on batch row 0 only
    float cond_temp[3]; int cond_offset[3]; int cond_flag[3];   // flag = VF_BEAT / VF_MANIA / VF_SCROLL
    int lookback_on; int lookback_start, lookback_end;           // LookbackBiasLogitsWarper range
    int do_sample; int top_k; float top_p; float top_p_cut;      // top_p_cut = (float)(1.0 - (double)top_p), see mb200_generate_params
    unsigned long long seed;
    int pad_id;
    int pos_rule_cumsum;     // 0: position = index (transformers 5.x), 1: index - n_left_pad[b] (4.5x)
    int ids_ld;              // row stride of the ids buffer
    int vflags_ld;           // ragged call: one SampleConfig and one vocabulary-flag row per request, flags of request b at vflags + b * vflags_ld
};

enum XMode : int { X_PLAIN = 0, X_LAYERNORM = 1 };

struct GemvSeg {
    float* out;              // row b at out + b * out_bs + (pos ? (cur_len - 1) * pos_stride : 0)
    long long out_bs;
    long long pos_stride;    // != 0: write at the cache position of the token being processed
    int n_begin, n_end;      // output columns [n_begin, n_end) of the stacked weight
    float alpha;
    int act;
};

struct GemvParams {
    int xmode;
    const float* x; long long x_ld;                 // PLAIN / LAYERNORM input rows
    const float* ln_w; const float* ln_b; float eps;
    const float* W; long long ldw; const float* bias;
    int K, N, B;
    int nseg; GemvSeg seg[3];
    const float* R; long long r_ld;                 // residual rows for segment 0 (null = none)
    const GenState* st;
};
// Which kernel body runs the rows.  KERNEL is the per-phase gemv_kernel (4 warps, weights read from global memory); MEGA is the barrier
// megakernel's phase body (16 warps, each CTA's weight rows copied to shared memory first; B <= 2, not ragged), which the kernel-level
// tests compare with KERNEL bit for bit.
enum GemvForm : int { GEMV_FORM_KERNEL = 0, GEMV_FORM_MEGA = 1 };
// ragged: p.st heads a ragged state; segments with pos_stride write row b at ITS cache position, and not at all once it has finished
// w_bf16: p.W holds bf16 bits ([N, ldw] elements, K and ldw multiples of 8, 16-byte aligned); the sums are the bits of the fp32 kernel
// on the widened weights
int launch_gemv(const GemvParams& p, cudaStream_t stream, bool pdl, bool ragged = false, int form = GEMV_FORM_KERNEL, bool w_bf16 = false);

struct DecAttnParams {
    const float* q; long long q_ld;                 // [rows, d_model], already scaled
    const float* kc; const float* vc;               // cache base for this layer
    long long row_stride;                           // stride between cache rows / slots
    long long tok_stride;                           // stride between tokens (d_model)
    const int* row_slot;                            // per decoder row: which cache row/slot to read (null = row index)
    int fixed_len;                                  // >0: number of keys (cross attention); 0: use st->cur_len
    const GenState* st;
    const unsigned char* key_valid; long long key_valid_ld;   // [rows, >=P] validity of prompt positions (null = all valid)
    float* part_o; float* part_ml;                  // [rows, H, n_splits, 64], [rows, H, n_splits, 2]
    int rows, H, n_splits, chunk;
    float* out; long long out_ld;                   // merged heads [rows, H*64], written by the LAST split of each (row, head) to arrive
    int* ticket;                                    // [rows, H] arrival counters, zero on entry, reset by the last arriver
    const int* kv_src; long long kv_src_ld;         // beam search: [rows, kv_src_ld] cache row holding key position t of row r (null = row r)
};
// Which kernel body runs the units.  DEFAULT is the engine's own choice (the CTA body, KMAX from the chunk; the one-warp batch form for
// rows > 2 when MB200_ATTN_BATCH is set); the others force one body — the kernel-level tests compare them bit for bit.
enum DecAttnForm : int { ATTN_FORM_DEFAULT = 0, ATTN_FORM_CTA128 = 1, ATTN_FORM_CTA64 = 2, ATTN_FORM_WARP = 3 };
int launch_decode_attention(const DecAttnParams& p, cudaStream_t stream, bool pdl, int form = ATTN_FORM_DEFAULT);
// Ragged self attention: p.st heads a ragged state; row r attends to its own cur_len keys with the split plan of its own max_length.
// p.n_splits = splits of the grid (the largest plan of the call; also the row stride of the partials); p.chunk is not read.
int launch_decode_attention_ragged(const DecAttnParams& p, cudaStream_t stream, bool pdl);

struct SampleParams {
    const float* logits; long long logits_ld;       // [rows(2B if cfg), V]
    const SampleConfig* cfg;
    GenState* st;
    const unsigned char* vflags;                    // [vocab_in]
    long long* ids;                                 // [B, ids_ld] int64 like the reference's LongTensor
    unsigned char* finished;                        // [B]
    int* last_ts;                                   // [B] value of the last time-shift token after the last SOS-type token, -1 if none
    float* last_scores;                             // [2, B, V] double-buffered by step parity
    const int* n_left_pad;                          // [rows] (pos_rule_cumsum only)
    const float* tok_emb; const float* pos_emb; int d_model;   // decoder_embedder / embed_positions
    float* x_out; long long x_ld;                   // [rows, d_model] residual stream input of the next step
    int rows;
    float* dbg_scores;                              // parity hook, null in production: [B, V] scores the selection sees (-inf = removed)
    // dataflow megakernel only (null otherwise): logits arrive as tagged pairs, and the next step's embedding + the token header leave
    // as tagged pairs (see decode_mega2.cu)
    const unsigned long long* ll_logits; unsigned ll_in_tag;
    unsigned long long* ll_x_out; unsigned long long* ll_hdr; unsigned ll_out_tag;
    int ll_reps; long long ll_x_rep;                // replicas of the residual-stream buffer and their stride (see MegaLL)
    int* ll_err;
    unsigned long long* trace;                      // tools/mega3_trace.py: clock64 stamps inside the selection phase (null in production)
};
// ragged: cfg / vflags are per-request arrays, st heads a ragged state; row b runs the chain of its own batch-1 call
int launch_sample(const SampleParams& p, int B, cudaStream_t stream, bool pdl, bool ragged = false);
// the ragged selection of the n rows in the DEVICE list `rows` only (first token of rows just prefilled into a running stream): one CTA
// per listed row; no other row's ids, state, embedding or look-back scores are touched
int launch_sample_rows(const SampleParams& p, const int* rows, int n, cudaStream_t stream);

// ---- beam.cu: beam search (num_beams K <= 4) after the decoder's final logits ---------------------------------------------
struct BeamParams {
    SampleParams sample;                            // chain state with logits = logprobs, cfg->B = B*K beam rows, ids [B*K, ids_ld]
    const float* logits; long long logits_ld;       // decoder logits [rows (2*B*K under CFG), V]
    float* logprobs;                                // [rows, V] log_softmax of every decoder row
    float* cand;                                    // [B*K, V] processed log-probs + running beam score
    float* run_score;                               // [B*K] running beam scores
    int* kv_src; long long kv_src_ld;               // [rows, kv_src_ld] self-attention source-row table
    long long* fin_ids[2];                          // finished hypotheses [B*K, ids_ld], double-buffered by step parity
    float* fin_score; int* fin_len; unsigned char* fin_flag;   // [B*K]: score, generated tokens, real hypothesis
    unsigned char* unsat;                           // [B] early-stop heuristic not yet satisfied
    int K, V, ids_ld;
    float* dbg_logprobs;                            // parity hook, null in production: [B*K, V] processed log-probs
    int* dbg_parent;                                // parity hook, null in production: [B*K] parent row of each new beam
    int* dbg_top;                                   // parity hook, null in production: [B*K] first K candidates per item (flat index)
};
size_t beam_select_smem_bytes(int K, int V, int ids_ld);
int launch_beam_step(const BeamParams& bp, int B, cudaStream_t stream);

// ---- decode_mega.cu: the persistent token-loop megakernel ----------------------------------------------------------------
constexpr int MEGA_WBUF_FLOATS = 19968;       // 78 KB per buffer, two buffers per CTA (one arena: see wslice in decode_mega.cu)
struct MegaPhase {                            // one dependent micro-phase of a token (built on the host)
    int kind;                                 // 0 GEMV, 1 split-KV attention, 2 logits chain + token selection
    int next_gemv;                            // index of the next GEMV phase (wraps into the next token)
    const float* nx_W; long long nx_ldw; int nx_N, nx_K;   // its weight matrix, so the prefetch needs no extra global reads
    unsigned magic_ns, magic_h;               // floor(2^32 / d) + 1 for d = n_splits, H (0 when d == 1): unit -> (split, head, row) without integer division
    int rpc, nx_rpc;                          // output rows per CTA of this / the next GEMV phase (ceil(N / grid), host-computed)
    GemvParams g;
    DecAttnParams a;
};
struct MegaParams {
    const MegaPhase* phases; int n_phases; int first_gemv;
    SampleParams sample;
    GenState* st;
    unsigned int* sync_counter;               // zeroed by the host before every launch
    int* error_flag;                          // 0 ok, 1 grid-barrier timeout, 2 weight-copy timeout
    int max_steps;
    const int* row_slot;                      // encoder slot of each decoder row (read once per token)
    unsigned long long* trace;                // optional [n_phases][6] globaltimer stamps of CTA 0 at token `trace_step`
    int trace_step;
};
size_t mega_smem_bytes();
// w_bf16: the phase table carries the bf16 store
int launch_megakernel(const MegaParams& mp, int grid, cudaStream_t stream, bool w_bf16 = false);

// ---- decode_mega2.cu: the DATAFLOW token-loop megakernel ----------------------------------------------------------------
// Same phases, same arithmetic, no grid barrier: every value that crosses CTAs travels as an 8-byte {fp32 bits | tag << 32} pair
// written by one 64-bit store and polled by its consumers, so the data IS the synchronisation (one L2 store + one L2 load between
// producer and consumer instead of store-drain + release atomic + acquire poll + load).
struct MegaLL {                                   // engine-owned exchange buffers, zeroed by the host before every launch (tag 0 = invalid)
    unsigned long long* x;                        // [rows][d]      residual stream
    unsigned long long* q;                        // [rows][d]      self / cross query
    unsigned long long* kvnew;                    // [rows][2d]     k | v of the token being processed (also stored plainly into the cache)
    unsigned long long* att;                      // [rows][d]      merged attention heads
    unsigned long long* h;                        // [rows][ffn]    fc1 output
    unsigned long long* logits;                   // [rows][V]
    unsigned long long* part;                     // [rows][H][max_splits][66]  split-KV partials: o[64], m, l
    unsigned long long* hdr;                      // [0] cur_len, [1] all_finished of the NEXT token (written by the selection phase)
    int max_splits;
    // x, att and h are read by (almost) every CTA.  Every SM polling the same 6 KB turns its L2 lines into a hot spot (the tagged
    // stores become visible late under that read pressure), so these three buffers exist `reps` times; producers store
    // every replica, CTA c polls replica c % reps.
    int reps;
    long long x_rep, h_rep;                       // replica strides of x / att (2 * d) and h (2 * ffn), in pairs
};
constexpr int MEGA_LL_MAX_REPS = 16;
enum MegaLLSel : int { LL_NONE = 0, LL_X = 1, LL_Q = 2, LL_K = 3, LL_V = 4, LL_ATT = 5, LL_H = 6, LL_LOGITS = 7 };
struct Mega2Phase {
    MegaPhase base;                               // the barrier kernel's descriptor (weights, segments, attention geometry, prefetch chain)
    int in_sel;                                   // GEMV input buffer: LL_X (LayerNorm prologue), LL_ATT, LL_H
    int out_sel[3];                               // per output segment: which exchange buffer receives the tagged copy (LL_NONE = plain only)
    int res_xraw;                                 // epilogue adds the residual from the raw x this CTA staged at the last LL_X input
    int plain_out[3];                             // per segment: also store plainly through seg.out (the K/V cache)
    // host-resolved exchange-buffer geometry, in pairs relative to MegaLL::x (the start of the arena), so the kernel's prologue is a
    // few adds instead of chains of shared-memory loads and selects
    long long in_off, in_rs;                      // GEMV input buffer and its replica stride
    int n_active;                                 // CTAs that own output rows in this GEMV phase: ceil(N / rows-per-CTA)
    long long out_off[3], out_rs[3], out_bw[3];   // per segment: tagged output buffer (incl. the V half of kvnew), replica stride (0 = one copy), pairs per decoder row
};
struct Mega2Params {
    const Mega2Phase* phases; int n_phases;
    SampleParams sample;
    GenState* st;
    MegaLL ll;
    int* error_flag;
    int max_steps;
    const int* row_slot;
    const float* x_in;                            // [rows][d] plain residual stream left by the prefill's selection kernel
    int rows, d_model, V, ffn_dim;
    unsigned long long* trace; int trace_step, trace_cta;    // optional [n_phases][16] clock64 stamps of one CTA (tools/mega3_trace.py)
};
size_t mega2_smem_bytes();
// w_bf16: the phase table carries the bf16 store
int launch_megakernel2(const Mega2Params& mp, int grid, cudaStream_t stream, bool w_bf16 = false);
bool mega2_ksplit_ok(int N, int K, int rows, int grid);   // does one GEMV phase fit the K-split thread mapping?
int mega2_set_debug(int bits);                    // diagnostics (decode_device.cuh, c_ll_debug)
int mega2_set_poll_sleep(int ns);                 // tuning: nanoseconds to back off after a failed poll (0 = spin)

// one-time per call: scan the prompt for the MonotonicTimeShift state (logit_processors.py:149-166)
int launch_prompt_scan(const long long* ids, long long ids_ld, int B, int P, const unsigned char* vflags, int ts_start, int ts_end,
                       int* last_ts, cudaStream_t stream);
// the same per request of a ragged call: own prompt length (ragged state `st`) and own flag row; rows = DEVICE list of the n rows to
// scan (null: rows 0 .. n - 1)
int launch_prompt_scan_ragged(const long long* ids, long long ids_ld, int n, const GenState* st, const unsigned char* vflags, long long vflags_ld,
                              int ts_start, int ts_end, int* last_ts, cudaStream_t stream, const int* rows = nullptr);
// prefill embedding: x[b, t] = tok_emb[ids[b, t]] + pos_emb[pos(b, t)]
int launch_embed(const long long* ids, long long ids_ld, int rows, int B_ids, int P, const int* n_left_pad, int pos_rule_cumsum,
                 const float* tok_emb, const float* pos_emb, int d_model, float* x, cudaStream_t stream);

}  // namespace mb200
