// Per-token decode path of the osuT5 decoder (reference: HF WhisperDecoderLayer x12 + proj_out called once per token by
// GenerationMixin._sample, ~330 launches + a host sync per token — SURVEY §3.2).  Here one token = 8 kernels per layer:
//   gemv[LN1 -> q|k|v, k/v written in place into the self cache]  ->  split-KV self attention  ->
//   gemv[out_proj + residual]  ->  gemv[LN2 -> cross q]  ->  split-KV cross attention (+ merge)  ->
//   gemv[out_proj + residual]  ->  gemv[LN3 -> fc1 + GELU]  ->  gemv[fc2 + residual]
// then gemv[final LN -> proj_out] and ONE kernel that runs the whole logits-processor chain (server.py:106-134 +
// HF min_new_tokens / top-k / top-p), selects the token, tests the EOS set, appends to `ids`, and writes the next step's
// embedding.  No host synchronisation per token; every step-varying scalar is read from GenState in device memory.
//
// The GEMVs are weight-streaming (HBM-bound): one warp per output row, float4 coalesced reads of the [N, K] row-major
// weight, activations for up to 8 batch rows staged in shared memory, fp32 accumulation in a fixed order.
#include <algorithm>
#include <cstdlib>
#include "common.cuh"
#include "kernels.h"
#include "decode_device.cuh"

namespace mb200 {
namespace {

constexpr int GEMV_THREADS = 128, GEMV_WARPS = GEMV_THREADS / 32;

// WBF16: p.W holds bf16 bits, row n at element n * p.ldw (decode_device.cuh gemv_dot)
template <int NB, bool RAGGED = false, bool WBF16 = false>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_kernel(GemvParams p) {
    extern __shared__ __align__(16) float xs[];   // [NB][K] activations, then 32 floats of LayerNorm reduction scratch
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_launch_dependents();
    pdl_wait();
    const int cur_pos = (p.st && !RAGGED) ? p.st->cur_len - 1 : 0;
    for (int b0 = 0; b0 < p.B; b0 += NB) {
        gemv_stage_x<NB, GEMV_THREADS>(p, b0, xs, xs + NB * p.K, tid);
        __syncthreads();
        for (int n = blockIdx.x * GEMV_WARPS + warp; n < p.N; n += gridDim.x * GEMV_WARPS)
            gemv_row<NB, true, RAGGED, WBF16>(p, n, gemv_wrow<WBF16>(p.W, (long long)n * p.ldw), xs, b0, lane, cur_pos);
        __syncthreads();
    }
}

// The barrier megakernel's GEMV phase (decode_mega.cu) as a kernel of its own: the megakernel's 512 threads stage the activations, CTA c
// holds weight rows [c * rpc, (c + 1) * rpc), rpc = ceil(N / grid), in shared memory (the megakernel streams them there with bulk
// copies; plain loads here) and warp w runs gemv_row on rows r0 + w, r0 + w + 16, ...  Only the kernel-level tests launch it, to hold
// the two forms to the same bits.
constexpr int MEGA_GEMV_THREADS = SAMPLE_THREADS;      // decode_mega.cu's MEGA_THREADS

// WBF16: the rows are bf16 bits (K a multiple of 8), copied to shared memory as they are: half the bytes of the fp32 slice.
template <int NB, bool WBF16 = false>
__global__ void __launch_bounds__(MEGA_GEMV_THREADS) gemv_mega_body_kernel(GemvParams p) {
    extern __shared__ __align__(16) float sm[];   // [rpc][K] weight rows, [NB][K] activations, 32 floats of LayerNorm reduction scratch
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_launch_dependents();
    pdl_wait();
    const int rpc = (p.N + (int)gridDim.x - 1) / (int)gridDim.x;
    const int r0 = min(p.N, (int)blockIdx.x * rpc), r1 = min(p.N, r0 + rpc);
    const int KV = WBF16 ? p.K >> 3 : p.K >> 2;     // 16-byte vectors per weight row
    float* wbuf = sm;
    float* xs = sm + (WBF16 ? (long long)rpc * (p.K >> 1) : (long long)rpc * p.K);
    for (int e = tid; e < (r1 - r0) * KV; e += MEGA_GEMV_THREADS) {
        const int r = e / KV, c = e - r * KV;
        reinterpret_cast<float4*>(wbuf)[e] = __ldg(reinterpret_cast<const float4*>(gemv_wrow<WBF16>(p.W, (long long)(r0 + r) * p.ldw)) + c);
    }
    gemv_stage_x<NB, MEGA_GEMV_THREADS>(p, 0, xs, xs + NB * p.K, tid);
    __syncthreads();
    const int cur_pos = p.st ? p.st->cur_len - 1 : 0;
    for (int n = r0 + warp; n < r1; n += MEGA_GEMV_THREADS / 32)
        gemv_row<NB, false, false, WBF16>(p, n, gemv_wrow<WBF16>(wbuf, (long long)(n - r0) * p.K), xs, 0, lane, cur_pos);
}

template <int KMAX, bool TABLE = false>
__global__ void __launch_bounds__(128, KMAX == 64 ? 6 : 4) decode_attention_kernel(DecAttnParams p) {
    __shared__ float sc[128];
    __shared__ float red[4][64];
    __shared__ float stat[2];
    pdl_launch_dependents();
    pdl_wait();
    const int L = p.fixed_len > 0 ? p.fixed_len : p.st->cur_len;
    const int P = p.st ? p.st->prompt_len : 0;
    const int r = blockIdx.z;
    const int slot = p.row_slot ? p.row_slot[r] : r;
    AttnRegs<4, KMAX> regs;
    decode_attention_load<4, KMAX, TABLE>(p, blockIdx.x, blockIdx.y, r, slot, L, P, threadIdx.x, regs);
    decode_attention_body<4, KMAX, TABLE>(p, blockIdx.x, blockIdx.y, r, slot, L, P, sc, red, stat, threadIdx.x, regs);
}

// batch form: one warp per (split, head, row) unit, 8 units per CTA (see decode_attention_warp_body)
__global__ void __launch_bounds__(256) decode_attention_warp_kernel(DecAttnParams p) {
    __shared__ float sc[8][128];
    pdl_launch_dependents();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u = blockIdx.x * 8 + warp;
    if (u >= p.rows * p.H * p.n_splits) return;
    const int L = p.fixed_len > 0 ? p.fixed_len : p.st->cur_len;
    const int P = p.st ? p.st->prompt_len : 0;
    const int hr = u / p.n_splits, s = u - hr * p.n_splits, r = hr / p.H, h = hr - r * p.H;
    decode_attention_warp_body(p, s, h, r, p.row_slot ? p.row_slot[r] : r, L, P, sc[warp], lane);
}

// Ragged self attention: the unit (split s, head h, row r) of the grid runs with the geometry of row r's OWN call — key count
// cur_len_r, the split plan of max_length_r — so its partials and their merge order are that call's, bit for bit.  Splits of the grid
// beyond the row's plan do not exist for it (no partial, no ticket); an empty split inside the plan contributes nothing, as always.
// One instantiation with room for 128 keys: rows with the single 128-key split and rows with 64-key splits share a launch, and the
// per-row geometry does not fit the 80 registers that give the uniform 64-key kernel its extra resident CTAs anyway.
__global__ void __launch_bounds__(128, 4) decode_attention_ragged_kernel(DecAttnParams p) {
    constexpr int KMAX = 128;
    __shared__ float sc[128];
    __shared__ float red[4][64];
    __shared__ float stat[2];
    pdl_launch_dependents();
    pdl_wait();
    const int s = blockIdx.x, h = blockIdx.y, r = blockIdx.z;
    const RowState* rs = ragged_rows(p.st) + r % p.st->n_req;
    // a finished row (or a vacant stream row) appends nothing and its output is never read: no keys, no ticket
    if (rs->finished) return;
    const int L = rs->cur_len;
    const int S = self_splits(rs->max_length);
    if (s >= S) return;                                // uniform across the CTA
    // partials stay at (row, head) stride p.n_splits while the body indexes them with the row's own split count
    const long long shift = ((long long)r * p.H + h) * (p.n_splits - S);
    p.part_o += shift * 64; p.part_ml += shift * 2;
    p.n_splits = S;
    p.chunk = self_split_chunk(S);
    AttnRegs<4, KMAX> regs;
    decode_attention_load<4, KMAX, false>(p, s, h, r, r, L, 0, threadIdx.x, regs);
    decode_attention_body<4, KMAX, false>(p, s, h, r, r, L, 0, sc, red, stat, threadIdx.x, regs);
}

template <bool RAGGED>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(SampleParams p) {
    __shared__ SampleSmem sm;
    pdl_launch_dependents();
    pdl_wait();
    if (p.st->all_finished) return;   // replays past the end of a call are no-ops (uniform across the grid)
    sample_body<SAMPLE_THREADS, RAGGED>(p, blockIdx.x, sm);
}

// the ragged selection of the listed rows only (decode stream admissions): CTA i runs row rows[i] at whatever step that row is at
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_rows_kernel(SampleParams p, const int* rows) {
    __shared__ SampleSmem sm;
    sample_body<SAMPLE_THREADS, true>(p, rows[blockIdx.x], sm);
}

__global__ void prompt_scan_kernel(const long long* ids, long long ids_ld, int P, const unsigned char* vflags, int ts_start, int ts_end,
                                   int* last_ts) {
    const int b = blockIdx.x;
    if (threadIdx.x != 0) return;
    int lt = -1;
    for (int t = 0; t < P; ++t) {
        long long tok = ids[(long long)b * ids_ld + t];
        if (vflags[tok] & VF_SOS) lt = -1;
        else if (tok >= ts_start && tok < ts_end) lt = (int)(tok - ts_start);
    }
    last_ts[b] = lt;
}

__global__ void prompt_scan_ragged_kernel(const long long* ids, long long ids_ld, const GenState* st, const unsigned char* vflags, long long vflags_ld,
                                          int ts_start, int ts_end, int* last_ts, const int* rows) {
    const int b = rows ? rows[blockIdx.x] : blockIdx.x;
    if (threadIdx.x != 0) return;
    const int P = ragged_rows(st)[b].prompt_len;
    const unsigned char* vf = vflags + b * vflags_ld;
    int lt = -1;
    for (int t = 0; t < P; ++t) {
        long long tok = ids[(long long)b * ids_ld + t];
        if (vf[tok] & VF_SOS) lt = -1;
        else if (tok >= ts_start && tok < ts_end) lt = (int)(tok - ts_start);
    }
    last_ts[b] = lt;
}

__global__ void embed_kernel(const long long* ids, long long ids_ld, int P, const int* n_left_pad, int pos_rule_cumsum,
                             const float* tok_emb, const float* pos_emb, int d_model, float* x) {
    const int t = blockIdx.x, r = blockIdx.y;
    const long long tok = ids[(long long)r * ids_ld + t];
    int pos = t;
    if (pos_rule_cumsum && n_left_pad) pos = max(0, t - n_left_pad[r]);
    const float4* te = reinterpret_cast<const float4*>(tok_emb + tok * d_model);
    const float4* pe = reinterpret_cast<const float4*>(pos_emb + (long long)pos * d_model);
    float4* xo = reinterpret_cast<float4*>(x + ((long long)r * P + t) * d_model);
    for (int i = threadIdx.x; i < d_model / 4; i += blockDim.x) {
        float4 a = te[i], q = pe[i];
        xo[i] = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
    }
}

static int g_prof_class = 0;

template <typename Kern, typename Params>
int launch_with_attrs(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, const Params& p) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    if (pdl) {
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
    }
    ++g_launch_count;
    const bool prof = g_prof.on && g_prof.n < 512;
    if (prof) MB_CUDA_CHECK(cudaEventRecord(g_prof.ev[2 * g_prof.n], stream));
    MB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, p));
    if (prof) { MB_CUDA_CHECK(cudaEventRecord(g_prof.ev[2 * g_prof.n + 1], stream)); g_prof.cls[g_prof.n++] = g_prof_class; }
    return 0;
}

}  // namespace

template <bool WBF16>
static int launch_gemv_impl(const GemvParams& p, cudaStream_t stream, bool pdl, bool ragged, int form) {
    if (form == GEMV_FORM_MEGA) {
        // a 132-CTA grid like the megakernel's on an H100, more CTAs when that many rows per CTA would not fit shared memory
        const size_t limit = 200 * 1024, fixed = ((size_t)p.B * p.K + 32) * sizeof(float), row = (size_t)p.K * (WBF16 ? 2 : sizeof(float));
        MB_REQUIRE(fixed + row <= limit, "GEMV activation tile does not fit shared memory");
        const int rpc = (int)std::min<size_t>((p.N + 131) / 132, (limit - fixed) / row);
        static bool mega_configured = false;
        if (!mega_configured) {
            MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_mega_body_kernel<1, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
            MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_mega_body_kernel<2, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
            mega_configured = true;
        }
        const dim3 grid((p.N + rpc - 1) / rpc);       // the kernel's ceil(N / grid) is at most rpc
        const size_t smem = fixed + rpc * row;
        g_prof_class = 0;
        return p.B == 1 ? launch_with_attrs(gemv_mega_body_kernel<1, WBF16>, grid, dim3(MEGA_GEMV_THREADS), smem, stream, pdl, p)
                        : launch_with_attrs(gemv_mega_body_kernel<2, WBF16>, grid, dim3(MEGA_GEMV_THREADS), smem, stream, pdl, p);
    }
    int nb = p.B >= 8 ? 8 : (p.B > 4 ? 8 : (p.B > 2 ? 4 : p.B));
    const size_t smem = ((size_t)nb * p.K + 32) * sizeof(float);
    const int blocks = (p.N + GEMV_WARPS - 1) / GEMV_WARPS;
    static bool configured = false;
    if (!configured) {
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<1, false, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<2, false, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<4, false, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<8, false, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<1, true, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<2, true, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<4, true, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MB_CUDA_CHECK(cudaFuncSetAttribute(gemv_kernel<8, true, WBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        configured = true;
    }
    MB_REQUIRE(smem <= 200 * 1024, "GEMV activation tile does not fit shared memory");
    g_prof_class = 0;
    if (ragged) {
        MB_REQUIRE(p.st, "ragged GEMV needs the ragged state");
        switch (nb) {
            case 1: return launch_with_attrs(gemv_kernel<1, true, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
            case 2: return launch_with_attrs(gemv_kernel<2, true, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
            case 4: return launch_with_attrs(gemv_kernel<4, true, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
            default: return launch_with_attrs(gemv_kernel<8, true, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
        }
    }
    switch (nb) {
        case 1: return launch_with_attrs(gemv_kernel<1, false, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
        case 2: return launch_with_attrs(gemv_kernel<2, false, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
        case 4: return launch_with_attrs(gemv_kernel<4, false, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
        default: return launch_with_attrs(gemv_kernel<8, false, WBF16>, dim3(blocks), dim3(GEMV_THREADS), smem, stream, pdl, p);
    }
}

int launch_gemv(const GemvParams& p, cudaStream_t stream, bool pdl, bool ragged, int form, bool w_bf16) {
    MB_REQUIRE(p.K % 4 == 0 && p.ldw % 4 == 0 && p.x_ld % 4 == 0, "GEMV K / ldw / x_ld must be multiples of 4");
    MB_REQUIRE(!w_bf16 || (p.K % 8 == 0 && p.ldw % 8 == 0 && reinterpret_cast<uintptr_t>(p.W) % 16 == 0),
               "bf16 GEMV weights need K and ldw multiples of 8 and 16-byte aligned rows");
    MB_REQUIRE(p.xmode != X_LAYERNORM || p.K <= 1024, "fused LayerNorm prologue supports K <= 1024");
    MB_REQUIRE(form == GEMV_FORM_KERNEL || form == GEMV_FORM_MEGA, "unknown GEMV form");
    MB_REQUIRE(form != GEMV_FORM_MEGA || (!ragged && p.B <= 2), "the megakernel's GEMV body runs 1 or 2 rows, not ragged");
    if (p.B <= 0 || p.N <= 0) return 0;
    if (!w_bf16) return launch_gemv_impl<false>(p, stream, pdl, ragged, form);
    const int rc = launch_gemv_impl<true>(p, stream, pdl, ragged, form);
    if (rc == 0) ++g_wbf16_launch_count;
    return rc;
}

int launch_decode_attention(const DecAttnParams& p, cudaStream_t stream, bool pdl, int form) {
    MB_REQUIRE(p.chunk > 0 && p.chunk <= 128, "decode attention chunk must be in (0, 128]");
    MB_REQUIRE(p.out && p.ticket, "decode attention needs the merged-output buffer and its tickets");
    MB_REQUIRE(form >= ATTN_FORM_DEFAULT && form <= ATTN_FORM_WARP, "unknown decode attention form");
    MB_REQUIRE(form != ATTN_FORM_CTA64 || p.chunk <= 64, "the KMAX 64 body cannot hold a chunk of more than 64 keys");
    MB_REQUIRE(form != ATTN_FORM_WARP || !p.kv_src, "the one-warp body has no source-row table");
    if (p.rows <= 0) return 0;
    g_prof_class = 1;
    const dim3 grid(p.n_splits, p.H, p.rows);
    if (form == ATTN_FORM_CTA128)
        return p.kv_src ? launch_with_attrs(decode_attention_kernel<128, true>, grid, dim3(128), 0, stream, pdl, p)
                        : launch_with_attrs(decode_attention_kernel<128>, grid, dim3(128), 0, stream, pdl, p);
    if (form == ATTN_FORM_CTA64)
        return p.kv_src ? launch_with_attrs(decode_attention_kernel<64, true>, grid, dim3(128), 0, stream, pdl, p)
                        : launch_with_attrs(decode_attention_kernel<64>, grid, dim3(128), 0, stream, pdl, p);
    if (form == ATTN_FORM_WARP)
        return launch_with_attrs(decode_attention_warp_kernel, dim3((p.rows * p.H * p.n_splits + 7) / 8), dim3(256), 0, stream, pdl, p);
    // Default: one CTA per unit with everything prefetched (the megakernel's phase body).  MB200_ATTN_BATCH=1 selects the
    // one-warp-per-unit form for rows > 2 — the same arithmetic value for value (parity-tested), kept as the starting point for a
    // persistent multi-unit kernel.
    static const int batch_form = [] { const char* e = getenv("MB200_ATTN_BATCH"); return e ? atoi(e) : 0; }();
    if (p.kv_src) {        // beam search: self attention through the source-row table
        if (p.chunk <= 64) return launch_with_attrs(decode_attention_kernel<64, true>, dim3(p.n_splits, p.H, p.rows), dim3(128), 0, stream, pdl, p);
        return launch_with_attrs(decode_attention_kernel<128, true>, dim3(p.n_splits, p.H, p.rows), dim3(128), 0, stream, pdl, p);
    }
    if (p.rows > 2 && batch_form) {
        const int units = p.rows * p.H * p.n_splits;
        return launch_with_attrs(decode_attention_warp_kernel, dim3((units + 7) / 8), dim3(256), 0, stream, pdl, p);
    }
    // 64-key chunks (every split launch) take the instantiation with half the K registers: 6 resident CTAs per SM instead of 4
    if (p.chunk <= 64) return launch_with_attrs(decode_attention_kernel<64>, dim3(p.n_splits, p.H, p.rows), dim3(128), 0, stream, pdl, p);
    return launch_with_attrs(decode_attention_kernel<128>, dim3(p.n_splits, p.H, p.rows), dim3(128), 0, stream, pdl, p);
}

int launch_decode_attention_ragged(const DecAttnParams& p, cudaStream_t stream, bool pdl) {
    MB_REQUIRE(p.st && p.out && p.ticket && !p.kv_src && p.fixed_len == 0, "ragged decode attention is the self attention of a ragged state");
    if (p.rows <= 0) return 0;
    g_prof_class = 1;
    return launch_with_attrs(decode_attention_ragged_kernel, dim3(p.n_splits, p.H, p.rows), dim3(128), 0, stream, pdl, p);
}

int launch_sample(const SampleParams& p, int B, cudaStream_t stream, bool pdl, bool ragged) {
    g_prof_class = 2;
    if (ragged) return launch_with_attrs(sample_kernel<true>, dim3(B), dim3(SAMPLE_THREADS), 0, stream, pdl, p);
    return launch_with_attrs(sample_kernel<false>, dim3(B), dim3(SAMPLE_THREADS), 0, stream, pdl, p);
}

int launch_sample_rows(const SampleParams& p, const int* rows, int n, cudaStream_t stream) {
    if (n <= 0) return 0;
    g_prof_class = 2;
    sample_rows_kernel<<<n, SAMPLE_THREADS, 0, stream>>>(p, rows);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

int launch_prompt_scan(const long long* ids, long long ids_ld, int B, int P, const unsigned char* vflags, int ts_start, int ts_end,
                       int* last_ts, cudaStream_t stream) {
    prompt_scan_kernel<<<B, 32, 0, stream>>>(ids, ids_ld, P, vflags, ts_start, ts_end, last_ts);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

int launch_prompt_scan_ragged(const long long* ids, long long ids_ld, int n, const GenState* st, const unsigned char* vflags, long long vflags_ld,
                              int ts_start, int ts_end, int* last_ts, cudaStream_t stream, const int* rows) {
    if (n <= 0) return 0;
    prompt_scan_ragged_kernel<<<n, 32, 0, stream>>>(ids, ids_ld, st, vflags, vflags_ld, ts_start, ts_end, last_ts, rows);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

int launch_embed(const long long* ids, long long ids_ld, int rows, int B_ids, int P, const int* n_left_pad, int pos_rule_cumsum,
                 const float* tok_emb, const float* pos_emb, int d_model, float* x, cudaStream_t stream) {
    (void)B_ids;
    if (rows <= 0 || P <= 0) return 0;
    embed_kernel<<<dim3(P, rows), 128, 0, stream>>>(ids, ids_ld, P, n_left_pad, pos_rule_cumsum, tok_emb, pos_emb, d_model, x);
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

}  // namespace mb200
