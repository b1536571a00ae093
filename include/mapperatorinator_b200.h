/* mapperatorinator_b200 — C ABI of the H100-native (sm_90a) engine for the Mapperatorinator inference hot path.
 *
 * The reference (OliBomby/Mapperatorinator) has no FFI layer: its boundary is a Python object protocol (SURVEY §8b).
 * Each entry point below names the reference call it replaces.  All pointers are plain device or host pointers owned by
 * the caller (torch tensors on the Python side); the engine owns only its weights copy, KV arena and workspaces.
 * Every function returns 0 on success; on failure a non-zero status, with mb200_last_error() giving the message
 * (the Python host raises RuntimeError — the reference convention "raise; the inference server turns any exception into
 * RETRY_SIGNAL", osuT5/osuT5/inference/server.py:411-417).  One caller thread and one CUDA stream per engine
 * (server.py:384: a single batch thread); no re-entrancy.
 */
#ifndef MAPPERATORINATOR_B200_H
#define MAPPERATORINATOR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_ABI_VERSION 2

int mb200_abi_version(void);
const char* mb200_last_error(void);

/* ------------------------------------------------------------------------------------------------------------------
 * Stage (i): raw PCM -> mel.  Replaces MelSpectrogram.forward (osuT5/osuT5/model/spectrogram.py:63-83), i.e. nnAudio
 * features.MelSpectrogram (v29) or torchaudio.transforms.MelSpectrogram (v30+) + optional log1p + permute(0, 2, 1).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct mb200_mel mb200_mel;
typedef struct {
    int32_t n_fft;        /* 1024 */
    int32_t hop_length;   /* 128 */
    int32_t n_mels;
    int32_t pad_reflect;  /* 0 = constant zero padding (v29), 1 = reflect (v30+) */
    int32_t log_scale;    /* spectrogram.py:80-81 */
} mb200_mel_config;
/* mel_basis: HOST float32 [n_mels, n_fft/2+1], the filterbank buffer of the reference module
 * (state_dict key spectrogram.transform.mel_basis / .mel_scale.fb^T). */
int mb200_mel_create(mb200_mel** out, const mb200_mel_config* cfg, const float* mel_basis);
void mb200_mel_destroy(mb200_mel* mel);
/* pcm: DEVICE f32 [batch, n_samples]; out: DEVICE f32 [batch, n_samples / hop + 1, n_mels]. */
int mb200_mel_forward(mb200_mel* mel, const float* pcm, int32_t batch, int32_t n_samples, float* out, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Stage (ii): the osuT5 model.  Replaces Mapperatorinator (osuT5/osuT5/model/modeling_mapperatorinator.py:60-443) with
 * the stock HF Whisper backbone of v29, as driven by server.model_generate / model_forward (server.py:83-181).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct mb200_model mb200_model;
typedef struct {
    int32_t d_model, encoder_layers, decoder_layers, heads, ffn_dim;
    int32_t src_seq_len;      /* mel frames per window (1024); max_source_positions = src_seq_len / 2 */
    int32_t tgt_seq_len;      /* max_target_positions (2048) */
    int32_t vocab_size_in, vocab_size_out;
    mb200_mel_config mel;
    int32_t max_windows;      /* encoder-state slots kept resident (cross-attention K/V of every window of the song(s)) */
    int32_t max_batch;        /* decoder rows of one generate() call (2x under classifier-free guidance) */
} mb200_model_config;

int mb200_model_create(mb200_model** out, const mb200_model_config* cfg, const float* mel_basis_host);
void mb200_model_destroy(mb200_model* m);
/* Upload one tensor by its reference state_dict() name (SURVEY Appendix A.7); data is HOST float32. Unknown names that
 * the inference path does not read (loss_fn.weight, decoder.embed_tokens.weight, spectrogram.*) are accepted and ignored. */
int mb200_model_set_weight(mb200_model* m, const char* name, const float* data, int64_t numel);
/* The same for a tensor held in bf16 (a model loaded at bf16 precision): bits are HOST bf16 bit patterns. The engine keeps the
 * widened (exact) fp32 values and remembers that the tensor arrived as bf16. */
int mb200_model_set_weight_bf16(mb200_model* m, const char* name, const uint16_t* bits, int64_t numel);
/* Checks that every required tensor was set and packs fused weights (q|k|v stacking, conv tap-major layout).
 * When every matrix the token loop streams arrived as bf16 (q|k|v, out, cross q, cross out, fc1 and fc2 of every decoder layer, and
 * proj_out), every packed element is still a bf16 value and every row length is a multiple of 8, the engine also keeps a bf16 copy of
 * those matrices, which every token-loop driver streams (half the bytes, the same result bits); the prefill, the cross K/V projection
 * and the teacher-forced passes read the fp32 weights. */
int mb200_model_finalize(mb200_model* m);
/* 2 when the engine holds the bf16 token-loop store, else 4. After finalize. */
int mb200_model_token_weight_bytes(const mb200_model* m, int32_t* bytes);

/* OsuTEncoder.forward (modeling_mapperatorinator.py:392-443) + the cross-attention K/V projection of every decoder
 * layer (HF modeling_whisper.py:331-338), for `n_windows` windows of raw PCM, written to slots
 * [slot_begin, slot_begin + n_windows).   pcm: DEVICE f32 [n_windows, (src_seq_len-1)*hop].
 * enc_out (optional, may be NULL): DEVICE f32 [n_windows, src_seq_len/2, d_model] receives the encoder hidden states. */
int mb200_model_encode(mb200_model* m, const float* pcm, int32_t n_windows, int32_t slot_begin, float* enc_out, void* cuda_stream);

typedef struct {
    /* generate_kwargs of server.model_generate (server.py:91-101) */
    float cfg_scale;
    float timeshift_bias;
    int32_t types_first;
    float temperature, timing_temperature, mania_column_temperature, taiko_hit_temperature;
    int32_t lookback_on;          /* lookback_time > 0 */
    int32_t lookback_start, lookback_end;   /* LookbackBiasLogitsWarper range (logit_processors.py:91-94) */
    int32_t do_sample, top_k;
    float top_p;
    int32_t max_length, min_new_tokens;
    int32_t pad_token_id;
    uint64_t seed;
    /* tokenizer facts (TokenLayout) */
    int32_t time_shift_start, time_shift_end;
    int32_t n_cond;               /* registered conditional temperatures in processor order */
    float cond_temp[3]; int32_t cond_offset[3]; int32_t cond_flag[3];   /* flag: 16 beat, 32 mania, 64 scroll-speed */
    int32_t position_rule;        /* 0 = arange (transformers 5.x), 1 = mask cumsum (4.5x) */
    float top_p_cut;              /* (float)(1.0 - top_p) evaluated in DOUBLE like HF's `cumulative_probs <= (1 - self.top_p)` with a Python
                                     float top_p (logits_process.py TopPLogitsWarper): 1.0f - (float)0.95 is one ulp away from it */
} mb200_generate_params;

/* GenerationMixin.generate as called by server.model_generate (server.py:143-150): prefill + token loop with the fused
 * logits-processor chain.  All arrays are HOST memory (the reference hands CPU tensors in and gets a CPU tensor back,
 * server.py:86,153).
 *   slots[batch]                  encoder-state slot of each row (from mb200_model_encode)
 *   prompt[batch, prompt_len]     int64 left-padded decoder_input_ids;  prompt_mask: uint8, 1 = real token
 *   neg_prompt / neg_mask         negative prompt for CFG or NULL
 *   vflags[vocab_size_in]         uint8 per-token flags: 1 EOS-set, 2 timed, 4 SOS-type, 8 lookback-eos, 16/32/64 cond. temp sets
 *   out_ids[batch, max_length]    int64, prompt + generated, rows padded with pad_token_id after their EOS
 *   out_len                       number of columns written (uniform across rows, like the reference's result tensor)
 */
int mb200_model_generate(mb200_model* m, const int32_t* slots, int32_t batch, const int64_t* prompt, const uint8_t* prompt_mask,
                         int32_t prompt_len, const int64_t* neg_prompt, const uint8_t* neg_mask, const uint8_t* vflags,
                         const mb200_generate_params* params, int64_t* out_ids, int32_t* out_len, void* cuda_stream);

/* The same call with HF beam search (generate(num_beams=K, do_sample=False), length_penalty 1.0, early_stopping False), 2 <= K <= 4:
 * the engine runs batch * K decoder rows (2x under classifier-free guidance; max_batch must cover them).  Same inputs as
 * mb200_model_generate plus
 *   num_beams                     K
 *   fill_id                       the id written past a shorter hypothesis (HF: pad_token_id, or the first EOS id when that is 0)
 * and returns the best finished hypothesis of every item:
 *   out_ids[batch, out_len]       int64, prompt + generated, out_len = prompt_len + the longest generated length in the batch
 *   out_scores[batch]             its score (sum of processed log-probs / generated length), HF's sequences_scores
 */
int mb200_model_generate_beams(mb200_model* m, const int32_t* slots, int32_t batch, const int64_t* prompt, const uint8_t* prompt_mask,
                               int32_t prompt_len, const int64_t* neg_prompt, const uint8_t* neg_mask, const uint8_t* vflags,
                               const mb200_generate_params* params, int32_t num_beams, int64_t fill_id, int64_t* out_ids,
                               int32_t* out_len, float* out_scores, void* cuda_stream);

/* Ragged batched generate: n_req independent requests in ONE token loop.  Request r has its own prompt (no padding), its own
 * generate params (max_length, min_new_tokens, EOS set and look-back range, temperatures, time-shift bias, sampling settings and
 * seed, cfg_scale) and its own encoder slot; row r of the result is bit-identical in its ids to mb200_model_generate called with
 * batch 1 for that request alone (positions 0..P_r-1 then P_r.., conditional temperature decided on the row itself, the sampling
 * counter of batch row 0, stop on its own EOS set or max_length).  All arrays are HOST memory.
 *   slots[n_req]                  encoder-state slot of each request
 *   prompt / prompt_off           int64 prompt ids of all requests back to back; request r owns [prompt_off[r], prompt_off[r+1])
 *   neg_prompt                    NULL, or the negative-prompt rows at the same offsets (the request's prompt with its leading tokens
 *                                 replaced, as for mb200_model_generate).  Either every request has cfg_scale > 1 and a negative row
 *                                 or none has: a mixed call is rejected.
 *   vflags[n_req, vocab_size_in]  per-request token flags (only the EOS bits differ between requests)
 *   params[n_req]                 per-request parameters; position_rule is not used (there is no padding)
 *   out_ids[n_req, out_ld]        int64, prompt + generated of each request; out_len[n_req] = its length
 * Rejected before anything is launched: more decoder rows than max_batch (n_req, doubled under CFG), prompt_len >= max_length,
 * max_length > tgt_seq_len or out_ld, mixed CFG.  Beam search stays on mb200_model_generate_beams. */
int mb200_model_generate_ragged(mb200_model* m, int32_t n_req, const int32_t* slots, const int64_t* prompt, const int32_t* prompt_off,
                                const int64_t* neg_prompt, const uint8_t* vflags, const mb200_generate_params* params,
                                int64_t* out_ids, int32_t out_ld, int32_t* out_len, void* cuda_stream);

/* Decode stream: continuous batching in the token loop.  A ragged token loop with a fixed row capacity: requests are admitted into free
 * rows between token steps and handed back as soon as they finish, and their rows are reused.  Every request's ids are bit-identical to
 * its own batch-1 mb200_model_generate call, whatever step it joins at, whatever the other rows do and whatever its row held before.
 * One stream per engine: while it is open, generate / generate_beams / generate_ragged / forward_logits / score_tokens, the parity
 * hooks, mb200_model_profile_step and the option "pdl" refuse; mb200_model_encode into slots no live row reads stays allowed.  Beam
 * search does not run in a stream.
 *   open:  capacity requests (2 * capacity decoder rows when use_cfg: every request guided, or none), each with max_length <= the
 *          max_length cap.  Captures the stream's token-step graph the first time this shape is seen; synchronises the stream.
 *   admit: n requests, arguments as for mb200_model_generate_ragged (HOST memory), into the lowest free rows (rows_out[n]).  Stages
 *          the rows and queues their prompt scan, batch-1 prefill and first-token selection with no host wait.  Rejected before
 *          anything is launched: fewer free rows than n, prompt_len >= max_length, max_length above the cap, a guidance mismatch
 *          with the stream, token ids out of range; the stream stays usable.
 *   run:   one burst of *steps token steps (short while `waiting` requests wait for a row, else up to 16), then the rows that
 *          finished in it: done_rows[n_done], done_len[n_done] (capacity entries each).  Synchronises the stream.
 *   take:  copies a finished row's ids (prompt + generated, done_len of them) to out_ids (HOST, out_ld wide) and frees the row.
 *   close: frees the stream; the engine's other token-loop calls work again. */
typedef struct mb200_stream mb200_stream;
int mb200_stream_open(mb200_model* m, int32_t capacity, int32_t use_cfg, int32_t max_length, mb200_stream** out, void* cuda_stream);
int mb200_stream_admit(mb200_stream* s, int32_t n, const int32_t* slots, const int64_t* prompt, const int32_t* prompt_off,
                       const int64_t* neg_prompt, const uint8_t* vflags, const mb200_generate_params* params, int32_t* rows_out,
                       void* cuda_stream);
int mb200_stream_run(mb200_stream* s, int32_t waiting, int32_t* done_rows, int32_t* done_len, int32_t* n_done, int32_t* steps,
                     void* cuda_stream);
int mb200_stream_take(mb200_stream* s, int32_t row, int64_t* out_ids, int32_t out_ld, void* cuda_stream);
void mb200_stream_close(mb200_stream* s);

/* Mapperatorinator.forward teacher-forced logits (server.model_forward, server.py:159-181), no CFG mixing.
 * ids: HOST int64 [batch, len]; mask HOST uint8; logits_out: DEVICE f32 [batch, len, vocab_size_out]. */
int mb200_model_forward_logits(mb200_model* m, const int32_t* slots, int32_t batch, const int64_t* ids, const uint8_t* mask,
                               int32_t len, int32_t position_rule, float* logits_out, void* cuda_stream);

/* Per-token scores of the same teacher-forced pass (MaiMod's Processor.ai_mod, processor.py:519-525), without ever holding the
 * call's [batch, len, vocab_size_out] logits: the projection runs in row chunks, each reduced on the device.  Same inputs as
 * mb200_model_forward_logits.  Outputs: DEVICE [batch, len], indexed by the scored token j; for j >= 1, with
 * p = softmax(logits[b, j - 1]) and y = ids[b, j]:
 *   entropy   = -sum p log2(p + 1e-10);   surprisal = -log2(p_y + 1e-10);   relative = entropy > 0 ? surprisal / entropy : 0;
 *   suggested = argmax logits[b, j - 1] (lowest index among ties).
 * Column 0 is NaN (suggested -1); a target y >= vocab_size_out has NaN surprisal and relative.  The logits behind the scores are
 * bit-identical to mb200_model_forward_logits' output for the same call. */
int mb200_model_score_tokens(mb200_model* m, const int32_t* slots, int32_t batch, const int64_t* ids, const uint8_t* mask, int32_t len,
                             int32_t position_rule, float* entropy, float* surprisal, float* relative, int64_t* suggested,
                             void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Stage (iii): DiT + sampling loop.  Replaces DiT.forward_with_cfg (osu_diffusion/utils/models.py:301-317) and
 * SpacedDiffusion.p_sample_loop as called by DiffisionPipeline.sample_part (diffusion_pipeline.py:243-252).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct mb200_dit mb200_dit;
typedef struct {
    int32_t hidden, depth, heads, mlp_ratio;
    int32_t in_channels, context_size, class_size;
    int32_t pos_freq_dim, t_freq_dim;
    int32_t max_seq_len;      /* longest chunk (diffusion_pipeline max_seq_len = 1024) */
    int32_t max_batch;        /* CFG pair = 2 */
} mb200_dit_config;

int mb200_dit_create(mb200_dit** out, const mb200_dit_config* cfg);
void mb200_dit_destroy(mb200_dit* d);
int mb200_dit_set_weight(mb200_dit* d, const char* name, const float* data, int64_t numel);   /* DiT.state_dict() names */
int mb200_dit_finalize(mb200_dit* d);

typedef struct {
    int32_t mask_mode;        /* 0 none, 2 band (|.| as diffusion_pipeline.py:146-148), 3 dense bool mask */
    int32_t band;             /* 128 */
    const uint8_t* dense_mask;/* DEVICE [T, T], 1 = blocked (mask_mode 3) */
} mb200_dit_mask;

/* DiT.forward_with_cfg: x DEVICE [N, 2, T], t HOST int32 [N] (model timesteps), c DEVICE [N, context, T],
 * y DEVICE [N, class_size]; out DEVICE [N, 4, T]. */
int mb200_dit_forward_with_cfg(mb200_dit* d, const float* x, const int32_t* t, const float* c, const float* y, int32_t N, int32_t T,
                               float cfg_scale, const mb200_dit_mask* mask, float* out, void* cuda_stream);

/* p_sample_loop with the slider-free denoised_fn (x0 <- where(inpaint, x0, z)) run entirely on the device.
 *   z DEVICE [N, 2, T] start state (also the in-paint source), inpaint DEVICE uint8 [N, 2, T] (1 = generate) or NULL,
 *   schedule HOST f32 [steps, 8] rows {t_model, sqrt_recip_acp, sqrt_recipm1_acp, posterior_log_var_clipped, log_beta,
 *   posterior_mean_coef1, posterior_mean_coef2, nonzero} for loop iteration order (first row = highest timestep),
 *   noise DEVICE f32 [steps, N, 2, T] (noise[k] = what th.randn_like returns at iteration k; gaussian_diffusion.py:454),
 *   out DEVICE [N, 2, T]. */
int mb200_dit_sample_loop(mb200_dit* d, const float* z, const float* c, const float* y, const uint8_t* inpaint, int32_t N, int32_t T,
                          float cfg_scale, const mb200_dit_mask* mask, const float* schedule, int32_t steps, const float* noise,
                          float* out, void* cuda_stream);

/* Slider end-point recompute of the denoised_fn closure (diffusion_pipeline.py:203-222: SliderPath(curve_type, control points)
 * .position_at(length / max_length), osuT5/osuT5/inference/slider_path.py:57-99, path_approximator.py:12-253) on the device.
 * mb200_dit_set_sliders registers the sliders of the chunk about to be sampled (HOST arrays, chunk-relative sequence indices; n = 0
 * clears): cp_offsets [n+1] prefix offsets into cp_index, end_index [n], type [n] (0 Bezier, 1 PerfectCurve, 2 Catmull, 3 Linear),
 * length [n] in osu! pixels.  The next mb200_dit_sample_loop then applies the recompute to the start state and to every step's
 * predicted x_start, inside the loop.  mb200_dit_apply_sliders runs the recompute once on x (DEVICE [N, 2, T], in place). */
int mb200_dit_set_sliders(mb200_dit* d, int32_t n, const int32_t* cp_offsets, const int32_t* cp_index, const int32_t* end_index,
                          const int32_t* type, const float* length);
int mb200_dit_apply_sliders(mb200_dit* d, float* x, int32_t N, int32_t T, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Measurement / tuning hooks used by bench.py (not part of the reference-facing boundary).
 * ------------------------------------------------------------------------------------------------------------------ */
/* Number of engine kernels launched by this process so far (graph replays count every node). */
int64_t mb200_launch_count(void);
/* The launches among those whose weights are a bf16 token-loop store (bf16 GEMVs and bf16 megakernels). */
int64_t mb200_wbf16_launch_count(void);
/* option "pdl": 1 = capture the token-step graph with programmatic dependent launch edges. */
int mb200_model_set_option(mb200_model* m, const char* name, int32_t value);
/* Parity hook for the fused logits-processor chain (server.py:106-134 + HF min-new-tokens / top-k / top-p + selection): ONE selection
 * step on caller-supplied logits.  logits DEVICE [rows, V] (rows = 2B under CFG, negative-prompt rows first); ids HOST [B, L];
 * `step` / `has_last_scores` select the look-back-bias state left by the previous call.  scores_out DEVICE [B, V] = the scores the
 * selection sees (-inf = removed), chosen_out HOST [B]. */
int mb200_model_logits_chain(mb200_model* m, const float* logits, int32_t B, int32_t use_cfg, const int64_t* ids, int32_t L, int32_t prompt_len,
                             const uint8_t* vflags, const mb200_generate_params* gp, int32_t step, int32_t has_last_scores, float* scores_out,
                             int64_t* chosen_out, void* cuda_stream);
/* Parity hook for beam search: ONE selection step of the beam kernels on caller-supplied logits, from an empty finished store.
 * logits DEVICE [rows, V] (rows = 2*B*K under CFG, negative-prompt rows first); ids HOST [B*K, L] running sequences; run_scores HOST [B*K].
 * logprobs_out DEVICE [B*K, V] processed log-probs; HOST [B*K]: top_out first K candidates per item (flat index beam * V + token),
 * parent_out batch row each new running beam continues, token_out / score_out its token and running score, fin_score_out /
 * fin_len_out / fin_flag_out the finished store (-1e9 / 0 / 0 where empty); fin_ids_out HOST [B*K, L + 1]. */
int mb200_model_beam_step(mb200_model* m, const float* logits, int32_t B, int32_t num_beams, int32_t use_cfg, const int64_t* ids, int32_t L,
                          int32_t prompt_len, const uint8_t* vflags, const mb200_generate_params* gp, const float* run_scores, int32_t step,
                          int32_t has_last_scores, float* logprobs_out, int32_t* top_out, int32_t* parent_out, int64_t* token_out,
                          float* score_out, float* fin_score_out, int32_t* fin_len_out, uint8_t* fin_flag_out, int64_t* fin_ids_out,
                          void* cuda_stream);
/* option "graph": 1 (default) = every step of mb200_dit_sample_loop is one replay of a captured CUDA graph, 0 = eager launches. */
int mb200_dit_set_option(mb200_dit* d, const char* name, int32_t value);
/* Re-runs the token step eagerly `iters` times on the state of the last generate() call with CUDA events around every
 * decode-path launch: out_us[0..2] = device us per token in {gemv, split-KV attention, logits+sample} kernels,
 * out_us[3] = launches per token packed as gemv*1e6 + attention*1e3 + sample. */
int mb200_model_profile_step(mb200_model* m, int32_t rows, int32_t batch, int32_t max_length, int32_t iters, float* out_us,
                             void* cuda_stream);

/* options "mega" (1 = persistent token-loop megakernel for <= 2 decoder rows, default) and "mega_trace" (1 = record
 * clock64 stamps of CTA 0 for every micro-phase of the 9th token); read them back as out[n_phases][16] SM cycles:
 * {phase start, activations staged, CTA sync passed, weights landed, math done, grid barrier passed, staging start,
 *  LayerNorm loads landed (0 for non-LayerNorm phases), then the same three staging stamps {start, loads landed, staged} of a
 *  first (cold) pass that trace mode runs in front of the timed one, slot 11 = this warp's rows done, slot 12 = end of a first
 *  (cold) pass over the rows that trace mode runs in front of the timed one; the rest spare}. */
int mb200_model_read_trace(mb200_model* m, uint64_t* out, int32_t n_phases);
/* CUDA-event totals of the persistent token-loop kernel (recorded on the launching stream around every launch):
 * out[0] = launches, out[1] = device milliseconds, out[2] = tokens decoded inside them; reset != 0 clears the counters. */
int mb200_model_mega_stats(mb200_model* m, double* out, int32_t reset);

/* ------------------------------------------------------------------------------------------------------------------
 * Kernel-level entry points (parity tests of the individual kernels; not needed by an integrator).
 * ------------------------------------------------------------------------------------------------------------------ */
/* Rows of a matrix operand as the engine addresses them: logical row m at ptr + (m / rpb) * bstride + (m % rpb) * ld (rpb 0: ptr + m * ld).
 * Rows may overlap (the conv stem reads a 3-tap window of a padded buffer as one row of 3 * ld floats) and bstride may be 0 (one table
 * added to every batch item). */
typedef struct mb200_rowmap {
    float* ptr;
    int64_t ld;
    int32_t rpb;
    int64_t bstride;
} mb200_rowmap;
/* One dense GEMM through the engine's own launch functions (gemm.cu / gemm_tc.cu):
 *   C[m, n] = act(A[m, :] . W[n, :] + bias[n]) * alpha [* gate[(m / gate_rpb) * gate_ld + n]] [+ R[m, n]],  m < M, n < N
 * A, C and R (null = none; it may be C itself) are row maps; W [N rows of K at stride ldw]; bias [N] or null.
 * path 0: W gets a tf32 mirror as the engine's registered weights have, and the engine's dispatch picks the kernel; 1: no mirror, the
 * fp32 SIMT kernel; 2: the wgmma 3xTF32 kernel, or an error if the problem is not eligible for it.  Every argument is checked before
 * anything is launched.  All pointers are DEVICE.  Synchronises the stream and reports a pipeline time-out of the tensor-core path. */
int mb200_op_gemm_mapped(const mb200_rowmap* A, const float* W, int64_t ldw, const mb200_rowmap* C, const float* bias, int32_t act,
                         float alpha, const mb200_rowmap* R, const float* gate, int64_t gate_ld, int32_t gate_rpb, int32_t M, int32_t N,
                         int32_t K, int32_t path, void* cuda_stream);
/* 0 = route every GEMM through the fp32 SIMT kernel (A/B comparisons), 1 = tensor cores where eligible (default) */
int mb200_set_tensor_cores(int32_t enabled);
/* LayerNorm of rows x [rows, dim] (contiguous) into y: affine with w / b, or the adaLN modulate y = LN(x) * (1 + scale) + shift with
 * shift / scale rows of batch item m / rows_per_batch at stride mod_ld (0 = dim). */
int mb200_op_layernorm(const float* x, float* y, const float* w, const float* b, const float* shift, const float* scale, int64_t mod_ld,
                       int32_t rows_per_batch, int32_t rows, int32_t dim, float eps, void* cuda_stream);
/* Dense attention (attention.cu / attention_tc.cu), head_dim 64: element (b, t, h, d) of q / k / v / o at ptr + b * bs + t * ld + h * 64 + d.
 * key_valid [B rows of key_valid_ld] (1 = real key) or null; kv_slot (DEVICE int32 [B], or null): batch row b reads K / V of batch index
 * kv_slot[b].  mask_mode 0 none, 1 causal (query t sees keys <= q_pos0 + t), 2 band, 3 dense [Tq, Tk] (1 = blocked).
 * The tensor-core path runs where it is eligible (see mb200_set_attention_tc). */
int mb200_op_attention(const float* q, int64_t q_ld, int64_t q_bs, const float* k, int64_t k_ld, int64_t k_bs, const float* v, int64_t v_ld,
                       int64_t v_bs, float* o, int64_t o_ld, int64_t o_bs, int32_t B, int32_t H, int32_t Tq, int32_t Tk, float scale,
                       int32_t mask_mode, int32_t q_pos0, const uint8_t* key_valid, int64_t key_valid_ld, int32_t band,
                       const uint8_t* dense_mask, const int32_t* kv_slot, void* cuda_stream);
/* One split-KV decode-attention phase of the token loop (decode.cu), through the engine's own launch functions and split plan.
 * q [rows, H*64] already scaled; kv: K|V cache [slots, t_max, 2*H*64] (token stride 2*H*64, V at offset H*64); row_slot [rows] cache
 * row of each decoder row (null = row r); out [rows, H*64] merged heads.  All pointers are DEVICE except ragged_cur_len /
 * ragged_max_length (host).
 *   self attention (fixed_len == 0): keys [0, cur_len); the split plan is that of max_length (one 128-key split up to 128, else
 *     64-key splits); key_valid [rows, key_valid_ld] masks prompt positions t < prompt_len (null = all valid); kv_src [rows,
 *     kv_src_ld] optional source-row table (beam search: key t of row r lives in cache row kv_src[r][t]);
 *   cross attention (fixed_len > 0): keys [0, fixed_len) in 64-key splits;
 *   ragged (ragged_cur_len and ragged_max_length given, host int32 [rows]): row r attends to its own cur_len keys with the plan of its
 *     own max_length, no prompt mask, row_slot null;
 *   form: 0 the engine's choice, 1 the CTA body with room for 128 keys, 2 the CTA body with 64, 3 the one-warp batch form.
 * Synchronises the stream before it returns. */
int mb200_op_decode_attention(const float* q, const float* kv, int32_t slots, int32_t t_max, int32_t H, int32_t rows, const int32_t* row_slot,
                              int32_t cur_len, int32_t prompt_len, const uint8_t* key_valid, int64_t key_valid_ld, int32_t max_length,
                              int32_t fixed_len, const int32_t* kv_src, int64_t kv_src_ld, const int32_t* ragged_cur_len,
                              const int32_t* ragged_max_length, int32_t form, float* out, void* cuda_stream);
/* One output segment of mb200_op_gemv: stacked-weight columns [n_begin, n_end) go to out, row b at
 * out + b * out_bs + (pos_stride ? (cur_len - 1) * pos_stride : 0) + (n - n_begin), as act(.) * alpha (+ the residual). */
typedef struct mb200_gemv_seg {
    float* out;
    int64_t out_bs;
    int64_t pos_stride;       /* != 0: write at the cache position of the token being processed */
    int32_t n_begin, n_end;
    float alpha;
    int32_t act;              /* 0 none, 1 GELU (erf), 2 GELU (tanh), 3 SiLU */
} mb200_gemv_seg;
/* One weight-streaming GEMV phase of the token loop (decode.cu), through the engine's own launch_gemv:
 *   out[b, n] = act(W[n, :] . X(x[b, :]) + bias[n]) * alpha + R[b, n],  b < B, n < N
 * x [B rows of K at stride x_ld]; xmode 0 takes X = x, xmode 1 the LayerNorm X = LN(x) * ln_w + ln_b (K <= 1024); W [N rows of K
 * at stride ldw]; bias [N] or null; R [B rows at stride r_ld] or null (it may be the output of segment 0: in-place residual).
 * segs (host, 1 to 3) must tile [0, N) in order; cur_len >= 1 places the segments with a pos_stride.
 * Ragged (ragged_cur_len and ragged_finished given, host int32 [n_req]): rows r and r + n_req share the state of request r % n_req;
 * a positional segment writes row b at its own cur_len - 1, and not at all once the row has finished.
 * form: 0 the per-phase kernel, 1 the barrier megakernel's phase body (B <= 2, not ragged).
 * All pointers except segs / ragged_* are DEVICE.  Synchronises the stream before it returns. */
int mb200_op_gemv(const float* x, int64_t x_ld, int32_t B, int32_t K, int32_t xmode, const float* ln_w, const float* ln_b, float eps,
                  const float* W, int64_t ldw, int32_t N, const float* bias, const float* R, int64_t r_ld, const mb200_gemv_seg* segs,
                  int32_t nseg, int32_t cur_len, const int32_t* ragged_cur_len, const int32_t* ragged_finished, int32_t n_req,
                  int32_t form, void* cuda_stream);
/* mb200_op_gemv with W given as bf16 bits (DEVICE uint16 [N rows of K at stride ldw]), through the bf16 GEMV the token loop runs on a
 * bf16 store. K and ldw must be multiples of 8 and W 16-byte aligned. */
int mb200_op_gemv_bf16(const float* x, int64_t x_ld, int32_t B, int32_t K, int32_t xmode, const float* ln_w, const float* ln_b, float eps,
                       const uint16_t* W, int64_t ldw, int32_t N, const float* bias, const float* R, int64_t r_ld, const mb200_gemv_seg* segs,
                       int32_t nseg, int32_t cur_len, const int32_t* ragged_cur_len, const int32_t* ragged_finished, int32_t n_req,
                       int32_t form, void* cuda_stream);
/* Tuning / tests: tensor-core (wgmma, 3xTF32) flash attention on or off, and the minimum number of queries for which it is used
   (attention_tc.cu; replaces the SIMT kernel for the encoder self-attention of HF modeling_whisper.py:286-358 and the DiT band of
   osu_diffusion/utils/models.py:145-151). */
int mb200_set_attention_tc(int32_t enabled, int32_t min_queries);

/* ---- audio ingest (SURVEY.md §8f N5) ---------------------------------------------------------------------------------------------
   Replaces the CPU tail of the reference's `load_audio_file` (osuT5/osuT5/dataset/data_utils.py:80-101, called by Preprocessor.load,
   osuT5/osuT5/inference/preprocessor.py:39): pydub `set_frame_rate` (audioop.ratecv) -> `set_channels(1)` (audioop.tomono) -> float32 ->
   `normalize_audio_samples` (:132-137).  File decoding (ffmpeg) stays with the caller: `pcm` is what
   `AudioSegment.from_file(path).get_array_of_samples()` holds.  Bit-identical to the reference's arithmetic.
   pcm: DEVICE int16 [n_frames, channels] interleaved (channels 1 or 2); in_rate = int(file rate * speed); out: DEVICE float32
   [mb200_audio_out_frames(n_frames, in_rate, out_rate)]; scratch: DEVICE int32 (1 element). */
int64_t mb200_audio_out_frames(int64_t n_frames, int32_t in_rate, int32_t out_rate);
int mb200_audio_ingest(const int16_t* pcm, int64_t n_frames, int32_t channels, int32_t in_rate, int32_t out_rate, int32_t normalize,
                       float* out, int32_t* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MAPPERATORINATOR_B200_H */
