// Beam search in the token loop: HF `GenerationMixin._beam_search` (transformers 5.5.0 generation/utils.py:3076-3380 and its
// helpers at :2856-3075) with num_beams = K <= 4, do_sample = False, length_penalty = 1.0, early_stopping = False.
// Two kernels per token, after the decoder's final logits:
//   beam_scores_kernel  (one CTA per beam row j of the B*K):  log_softmax of the row (and of its negative-prompt row under CFG),
//                       the fused logits-processor chain on the log-probs (decode_device.cuh::logits_chain), + running score;
//   beam_select_kernel  (one CTA per batch item):  candidate selection over the K*V (score, flat index) pairs, the finished-hypothesis
//                       store, the early-stop heuristic, and the reorder: ids rows, MonotonicTimeShift state and the self-attention
//                       source-row table gathered by parent, the next step's embeddings written.
// Candidate order: score descending, then flat index (beam * V + token) ascending.
//
// Selection.  HF takes the top beams_to_keep = max(2, 1 + n_eos) * K candidates, then (a) the running beams = the top K of
// score + hit * -1e9 among them, (b) the finished candidates = those of the first K that hit a stopping criterion.  Among the first
// beams_to_keep candidates at most K * n_eos can hit (one hit per EOS id and beam) unless the max length is reached, so the first K
// candidates that do not hit are always inside the kept set; ranking every candidate by (score + hit * -1e9, then candidate order)
// therefore yields exactly HF's running beams, including the all-hit step at max_length.  Both selections are K rounds of a block
// arg-max over the K*V pairs held in shared memory: exact, and no sort of the beams_to_keep survivors is needed.
#include "common.cuh"
#include "kernels.h"
#include "decode_device.cuh"

namespace mb200 {
namespace {

constexpr int BEAM_THREADS = 512;

// block-wide log_softmax of one row of V logits (torch's x - max - log(sum(exp(x - max)))) into out
__device__ void log_softmax_row(const float* x, float* out, int V, float* scratch) {
    float m = -INFINITY;
    for (int v = threadIdx.x; v < V; v += BEAM_THREADS) m = fmaxf(m, __ldcg(x + v));
    m = block_reduce<BEAM_THREADS>(m, true, scratch);
    float z = 0.f;
    for (int v = threadIdx.x; v < V; v += BEAM_THREADS) z += expf(__ldcg(x + v) - m);
    z = block_reduce<BEAM_THREADS>(z, false, scratch);
    const float lz = logf(z);
    for (int v = threadIdx.x; v < V; v += BEAM_THREADS) out[v] = (__ldcg(x + v) - m) - lz;
}

__global__ void __launch_bounds__(BEAM_THREADS) beam_scores_kernel(BeamParams bp) {
    __shared__ SampleSmem sm;
    const SampleParams& p = bp.sample;
    GenState* st = p.st;
    if (st->all_finished) return;                  // replays past the end of a call are no-ops
    const SampleConfig& c = *p.cfg;
    const int j = blockIdx.x, V = c.V, BK = c.B;
    log_softmax_row(bp.logits + (long long)j * bp.logits_ld, bp.logprobs + (long long)j * V, V, sm.scratch);
    if (c.use_cfg) log_softmax_row(bp.logits + (long long)(BK + j) * bp.logits_ld, bp.logprobs + (long long)(BK + j) * V, V, sm.scratch);
    __syncthreads();
    const int L = ld_state(&st->cur_len);
    const int st_min_new = ld_state(&st->min_new_tokens);
    const bool suppress_eos = st_min_new > 0 && (L - ld_state(&st->prompt_len)) < st_min_new;
    logits_chain<BEAM_THREADS>(p, j, sm, L, ld_state(&st->step), ld_state(&st->has_last_scores), suppress_eos);
    __syncthreads();
    const float run = bp.run_score[j];
    for (int v = threadIdx.x; v < V; v += BEAM_THREADS) {
        if (bp.dbg_logprobs) bp.dbg_logprobs[(long long)j * V + v] = sm.s[v];
        bp.cand[(long long)j * V + v] = sm.s[v] + run;
    }
}

struct Cand { float key; float score; int idx; };

__device__ __forceinline__ bool cand_better(const Cand& a, const Cand& b) {
    if (a.key != b.key) return a.key > b.key;
    if (a.score != b.score) return a.score > b.score;
    return a.idx < b.idx;
}

// K rounds of arg-max over the K*V candidates in shared memory; running = rank by score + hit * -1e9 instead of score
__device__ void select_top(const float* cs, int n, int V, int K, int L, int max_length, const unsigned char* vflags, bool running,
                           Cand* out, Cand* wbest) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int k = 0; k < K; ++k) {
        Cand best{-INFINITY, -INFINITY, 0x7fffffff};
        for (int i = tid; i < n; i += BEAM_THREADS) {
            bool taken = false;
            for (int q = 0; q < k; ++q) taken |= out[q].idx == i;
            if (taken) continue;
            const float s = cs[i];
            const bool hit = (vflags[i % V] & VF_EOS) != 0 || L + 1 >= max_length;
            const Cand c{running && hit ? s + -1.0e9f : s, s, i};
            if (best.idx == 0x7fffffff || cand_better(c, best)) best = c;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            Cand x{__shfl_xor_sync(0xffffffffu, best.key, o), __shfl_xor_sync(0xffffffffu, best.score, o), __shfl_xor_sync(0xffffffffu, best.idx, o)};
            if (x.idx != 0x7fffffff && (best.idx == 0x7fffffff || cand_better(x, best))) best = x;
        }
        if (lane == 0) wbest[warp] = best;
        __syncthreads();
        if (tid == 0) {
            Cand b = wbest[0];
            for (int w = 1; w < BEAM_THREADS / 32; ++w)
                if (wbest[w].idx != 0x7fffffff && (b.idx == 0x7fffffff || cand_better(wbest[w], b))) b = wbest[w];
            out[k] = b;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(BEAM_THREADS) beam_select_kernel(BeamParams bp) {
    extern __shared__ __align__(16) unsigned char beam_smem[];
    __shared__ Cand top[4], run[4], wbest[BEAM_THREADS / 32];
    __shared__ int src_slot[4], src_cand[4], parent[4];      // new finished slot k <- old slot / candidate rank; running beam parent
    __shared__ long long tok[4];
    const SampleParams& p = bp.sample;
    GenState* st = p.st;
    if (st->all_finished) return;
    const SampleConfig& c = *p.cfg;
    const int b = blockIdx.x, K = bp.K, V = c.V, BK = c.B, ld = c.ids_ld, tid = threadIdx.x;
    const int L = ld_state(&st->cur_len), P = ld_state(&st->prompt_len), max_length = ld_state(&st->max_length);
    float* cs = reinterpret_cast<float*>(beam_smem);                                    // [K*V] candidate scores of item b
    long long* region = reinterpret_cast<long long*>(beam_smem + (((size_t)K * V * 4 + 15) & ~size_t(15)));   // [K][ld] staging rows
    const int n = K * V;
    for (int i = tid; i < n; i += BEAM_THREADS) cs[i] = __ldcg(bp.cand + (long long)b * K * V + i);
    __syncthreads();
    select_top(cs, n, V, K, L, max_length, p.vflags, false, top, wbest);
    select_top(cs, n, V, K, L, max_length, p.vflags, true, run, wbest);

    float* fs = bp.fin_score + b * K;
    int* fl = bp.fin_len + b * K;
    unsigned char* ff = bp.fin_flag + b * K;
    const int rd = ld_state(&st->step) & 1;                        // finished ids: read parity rd, write 1 - rd
    const long long* fin_in = bp.fin_ids[rd] + (long long)b * K * ld;
    long long* fin_out = bp.fin_ids[1 - rd] + (long long)b * K * ld;
    if (tid == 0) {
        // finished hypotheses: the old store merged with those of the first K candidates that hit (HF's top_num_beam_mask),
        // score / (cur_len + 1 - P) ** 1.0; the old entries come first among equal scores.  Candidates that do not finish carry
        // HF's -1e9 sentinels and never outrank a real hypothesis, so only real ones are merged.
        const bool unsat = bp.unsat[b] != 0;
        const float denom = (float)(L + 1 - P);
        float ms[8]; int msrc[8]; int mcand[8]; int m = 0;
        for (int k = 0; k < K; ++k) { ms[m] = fs[k]; msrc[m] = k; mcand[m] = -1; ++m; }
        for (int k = 0; k < K; ++k) {
            const int t = top[k].idx % V;
            const bool hit = (p.vflags[t] & VF_EOS) != 0 || L + 1 >= max_length;
            if (hit && unsat && top[k].score / denom > -1.0e9f) { ms[m] = top[k].score / denom; msrc[m] = -1; mcand[m] = k; ++m; }
        }
        float nfs[4]; int nfl[4]; unsigned char nff[4];
        bool used[8] = {false, false, false, false, false, false, false, false};
        for (int k = 0; k < K; ++k) {
            int bi = -1;
            for (int q = 0; q < m; ++q)
                if (!used[q] && (bi < 0 || ms[q] > ms[bi])) bi = q;
            used[bi] = true;
            nfs[k] = ms[bi];
            src_slot[k] = msrc[bi]; src_cand[k] = mcand[bi];
            if (msrc[bi] >= 0) { nfl[k] = fl[msrc[bi]]; nff[k] = ff[msrc[bi]]; }
            else { nfl[k] = L + 1 - P; nff[k] = 1; }
        }
        for (int k = 0; k < K; ++k) { fs[k] = nfs[k]; fl[k] = nfl[k]; ff[k] = nff[k]; }
        // running beams
        for (int k = 0; k < K; ++k) {
            parent[k] = run[k].idx / V;
            tok[k] = run[k].idx % V;
            bp.run_score[b * K + k] = run[k].key;
            if (bp.dbg_parent) bp.dbg_parent[b * K + k] = b * K + parent[k];
            if (bp.dbg_top) bp.dbg_top[b * K + k] = top[k].idx;
        }
        // early-stop heuristic (early_stopping False): the best running beam at the current length against the worst finished one
        float worst = fs[0];
        for (int k = 1; k < K; ++k) worst = fminf(worst, fs[k]);
        const float best_running = run[0].key / (float)(L + 1 - P);
        bool any = false;
        for (int k = 0; k < K; ++k) any |= best_running > (ff[k] ? worst : -1.0e9f);
        if (unsat && !any) { bp.unsat[b] = 0; atomicAdd(&st->n_finished, 1); }
    }
    __syncthreads();
    // finished store: rows from the old store (staged) or from the candidate's parent row + its token
    for (int i = tid; i < K * (L + 1); i += BEAM_THREADS) region[(i / (L + 1)) * ld + i % (L + 1)] = fin_in[(i / (L + 1)) * ld + i % (L + 1)];
    __syncthreads();
    for (int k = 0; k < K; ++k) {
        long long* dst = fin_out + (long long)k * ld;
        if (src_slot[k] >= 0) {
            for (int t = tid; t <= L; t += BEAM_THREADS) dst[t] = region[(long long)src_slot[k] * ld + t];
        } else {
            const int ci = top[src_cand[k]].idx;
            const long long* srow = p.ids + (long long)(b * K + ci / V) * ld;
            for (int t = tid; t < L; t += BEAM_THREADS) dst[t] = srow[t];
            if (tid == 0) dst[L] = ci % V;
        }
    }
    __syncthreads();
    // ids rows gathered by parent, new token appended
    long long* ids = p.ids + (long long)b * K * ld;
    for (int i = tid; i < K * L; i += BEAM_THREADS) region[(i / L) * ld + i % L] = ids[(i / L) * ld + i % L];
    __syncthreads();
    for (int i = tid; i < K * L; i += BEAM_THREADS) ids[(i / L) * ld + i % L] = region[parent[i / L] * ld + i % L];
    if (tid < K) ids[(long long)tid * ld + L] = tok[tid];
    __syncthreads();
    // source-row table: rows of item b (and, under CFG, their conditional twins, which take the NEGATIVE rows' history:
    // MapperatorinatorCache.reorder_cache reorders with beam_idx.repeat(2)); the new position of row r points to r itself
    int* tab = reinterpret_cast<int*>(region);
    const int* ks = bp.kv_src + (long long)b * K * bp.kv_src_ld;
    for (int i = tid; i < K * L; i += BEAM_THREADS) tab[(i / L) * ld + i % L] = ks[(i / L) * bp.kv_src_ld + i % L];
    __syncthreads();
    const int nrep = c.use_cfg ? 2 : 1;
    for (int rep = 0; rep < nrep; ++rep) {
        int* kd = bp.kv_src + ((long long)rep * BK + b * K) * bp.kv_src_ld;
        for (int i = tid; i < K * (L + 1); i += BEAM_THREADS) {
            const int k = i / (L + 1), t = i % (L + 1);
            kd[(long long)k * bp.kv_src_ld + t] = t < L ? tab[parent[k] * ld + t] : rep * BK + b * K + k;
        }
    }
    // MonotonicTimeShift state follows each beam's own sequence
    if (tid == 0) {
        int lt[4];
        for (int k = 0; k < K; ++k) lt[k] = p.last_ts[b * K + parent[k]];
        for (int k = 0; k < K; ++k) {
            const long long t = tok[k];
            if (p.vflags[t] & VF_SOS) lt[k] = -1;
            else if (t >= c.ts_start && t < c.ts_end) lt[k] = (int)(t - c.ts_start);
            p.last_ts[b * K + k] = lt[k];
        }
    }
    // embedding of each beam's new token for every decoder row fed with it
    for (int rep = 0; rep < nrep; ++rep)
        for (int k = 0; k < K; ++k) {
            const int row = rep * BK + b * K + k;
            int pos = L;
            if (c.pos_rule_cumsum && p.n_left_pad) pos = L - p.n_left_pad[row];
            const float4* te = reinterpret_cast<const float4*>(p.tok_emb + tok[k] * p.d_model);
            const float4* pe = reinterpret_cast<const float4*>(p.pos_emb + (long long)pos * p.d_model);
            float4* xo = reinterpret_cast<float4*>(p.x_out + (long long)row * p.x_ld);
            for (int i = tid; i < p.d_model / 4; i += BEAM_THREADS) {
                const float4 a = te[i], q = pe[i];
                xo[i] = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
            }
        }
    __syncthreads();
    if (tid == 0) {
        // last item to arrive advances the call state: the loop ends when no item can improve or every kept candidate stops
        const int B = BK / K;
        if (B > 1) __threadfence();
        if (atomicAdd(&st->ticket, 1) == B - 1) {
            const int fin_all = (ld_state(&st->n_finished) >= B || L + 1 >= max_length) ? 1 : 0;
            st->ticket = 0;
            st->cur_len = L + 1;
            st->step = ld_state(&st->step) + 1;
            st->has_last_scores = 1;
            if (fin_all) st->all_finished = 1;
            __threadfence();
        }
    }
}

}  // namespace

size_t beam_select_smem_bytes(int K, int V, int ids_ld) {
    return (((size_t)K * V * 4 + 15) & ~size_t(15)) + (size_t)K * ids_ld * 8;
}

int launch_beam_step(const BeamParams& bp, int B, cudaStream_t stream) {
    const size_t smem = beam_select_smem_bytes(bp.K, bp.V, bp.ids_ld);
    MB_REQUIRE(bp.K >= 2 && bp.K <= 4, "beam search takes 2..4 beams");
    MB_REQUIRE(smem <= 220 * 1024, "beam candidates do not fit shared memory");
    static size_t configured = 0;
    if (smem > configured) {
        MB_CUDA_CHECK(cudaFuncSetAttribute(beam_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    beam_scores_kernel<<<B * bp.K, BEAM_THREADS, 0, stream>>>(bp);
    MB_LAUNCH_CHECK();
    beam_select_kernel<<<B, BEAM_THREADS, smem, stream>>>(bp);
    MB_LAUNCH_CHECK();
    g_launch_count += 2;
    return 0;
}

}  // namespace mb200
