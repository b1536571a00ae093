// Tensor-core flash attention (head_dim 64) for the dense phases: Whisper encoder self-attention (T = 512, HF modeling_whisper.py:286-358),
// the DiT blocks' +-128 band (osu_diffusion/utils/models.py:145-151) and causal / key-padded self-attention.  fp32 in, fp32 out, both
// contractions on Hopper wgmma (kind tf32) with the 3xTF32 split of gemm_tc.cu (x = hi + lo, hi.hi + hi.lo + lo.hi), fp32 accumulators
// in registers.
//
//   attn_prep_kernel   one pass over q | k | v (token-major, the projection GEMM's layout): scale + tf32 hi / lo split, written head-major
//                      as Q [2][B*H][Tq_pad][64], K [2][B*H][Tk_pad][64] and V TRANSPOSED VT [2][B*H][64][Tk_pad] (so that V is a K-major
//                      B operand of the second contraction), zero padded to whole tiles.  Inside every group of 8 keys VT holds the keys
//                      in the order 0 2 4 6 1 3 5 7: that is the order in which a thread's score accumulators (keys 2t, 2t+1) sit in the
//                      A-operand fragment of the P.V MMA (columns t, t+4), so P goes from the score registers into the MMA unshuffled.
//   attention_tc_kernel  one CTA = 128 queries of one (batch, head), 64-key tiles, 384 threads (3 warpgroups):
//       warpgroup 0, thread 0 : TMA producer — Q once (4 x [128 x 32 floats]), then per KV tile 4 K tiles + 4 VT tiles (2-stage ring)
//       warpgroups 1, 2       : 64 query rows each: S = Q K^T (24 x wgmma m64n64k8, both operands in shared memory) -> mask -> online
//                               softmax in registers (a row lives in the 4 threads of a quad) -> O = O * alpha + P V (24 x wgmma
//                               m64n64k8, P hi / lo from registers) -> normalise -> store.
// Every wait is bounded (error flag + fall through), like gemm_tc.cu.  Dense boolean masks and K/V gathered through kv_slot stay on the
// fp32 SIMT kernel (attention.cu).
#include <cuda.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace mb200 {

namespace {

constexpr int FA_BM = 128, FA_BN = 64, FA_HD = 64, FA_THREADS = 384, FA_CONSUMERS = 256, FA_STAGES = 2;
constexpr int FA_Q_TILE = FA_BM * 32 * 4;                 // 16 KB: 128 rows x 32 floats
constexpr int FA_Q_BYTES = 4 * FA_Q_TILE;                 // hi d0-31 | hi d32-63 | lo d0-31 | lo d32-63
constexpr int FA_KV_TILE = FA_BN * 32 * 4;                // 8 KB: 64 rows x 32 floats
constexpr int FA_STAGE_BYTES = 8 * FA_KV_TILE;            // K: hi d0, hi d1, lo d0, lo d1 | VT: hi k0, hi k1, lo k0, lo k1

struct FaBarriers {
    unsigned long long q_full;
    unsigned long long kv_full[FA_STAGES], kv_empty[FA_STAGES];
};

__device__ __forceinline__ unsigned fa_s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool fa_wait(unsigned long long* bar, unsigned parity, int* err) {
    for (long long spin = 0; spin < (1ll << 22); ++spin) {
        unsigned ok;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok) : "r"(fa_s32(bar)), "r"(parity) : "memory");
        if (ok) return true;
    }
    atomicExch(err, 5);
    return false;
}
__device__ __forceinline__ float fa_rn_tf32(float x) {
    unsigned u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float fa_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct FaParams {
    float* o; long long o_ld, o_bs;
    int B, H, Tq, Tk, Tq_pad, Tk_pad;
    int mask_mode, q_pos0, band;
    const unsigned char* key_valid; long long key_valid_ld;
};

__global__ void __launch_bounds__(FA_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_vt,
                    FaParams p, int* err) {
    extern __shared__ unsigned char fa_smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(fa_smem_raw) + 1023) & ~uintptr_t(1023));
    unsigned char* q_s = smem;
    unsigned char* kv_s = smem + FA_Q_BYTES;
    FaBarriers* bars = reinterpret_cast<FaBarriers*>(smem + FA_Q_BYTES + FA_STAGES * FA_STAGE_BYTES);
    const int tid = threadIdx.x;
    const int q0 = blockIdx.x * FA_BM, bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;

    // KV tile range the mask allows for this query tile
    int kt_begin = 0, kt_end = (p.Tk + FA_BN - 1) / FA_BN;
    if (p.mask_mode == MASK_CAUSAL) {
        const int last = p.q_pos0 + min(q0 + FA_BM - 1, p.Tq - 1);
        kt_end = min(kt_end, last / FA_BN + 1);
    } else if (p.mask_mode == MASK_BAND) {
        const int lo = q0 - p.band + 1, hi = min(q0 + FA_BM - 1, p.Tq - 1) + p.band;
        kt_begin = max(0, lo) / FA_BN;
        kt_end = min(kt_end, hi / FA_BN + 1);
    }
    const int ntiles = max(0, kt_end - kt_begin);

    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(fa_s32(&bars->q_full)));
        for (int s = 0; s < FA_STAGES; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(fa_s32(&bars->kv_full[s])));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fa_s32(&bars->kv_empty[s])), "r"(FA_CONSUMERS));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (tid < 128) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (tid == 0 && ntiles > 0) {
            // Q: rows bh * Tq_pad + q0 .. +127, halves d0-31 / d32-63, hi (plane 0) then lo (plane 1)
            const unsigned qb = fa_s32(&bars->q_full);
            asm volatile("{ .reg .b64 t; mbarrier.arrive.expect_tx.shared::cta.b64 t, [%0], %1; }" ::"r"(qb), "r"(FA_Q_BYTES) : "memory");
            const int qrow = bh * p.Tq_pad + q0;
            for (int t = 0; t < 4; ++t)
                asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                             ::"r"(fa_s32(q_s + t * FA_Q_TILE)), "l"(&map_q), "r"((t & 1) * 32), "r"(qrow), "r"(t >> 1), "r"(qb) : "memory");
            for (int i = 0; i < ntiles; ++i) {
                const int s = i % FA_STAGES;
                const unsigned ph = (i / FA_STAGES) & 1;
                if (!fa_wait(&bars->kv_empty[s], ph ^ 1, err)) break;
                unsigned char* st = kv_s + s * FA_STAGE_BYTES;
                const unsigned fb = fa_s32(&bars->kv_full[s]);
                asm volatile("{ .reg .b64 t; mbarrier.arrive.expect_tx.shared::cta.b64 t, [%0], %1; }" ::"r"(fb), "r"(FA_STAGE_BYTES) : "memory");
                const int k0 = (kt_begin + i) * FA_BN;
                const int krow = bh * p.Tk_pad + k0;
                for (int t = 0; t < 4; ++t)      // K tiles: [64 keys x 32 dims]
                    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                                 ::"r"(fa_s32(st + t * FA_KV_TILE)), "l"(&map_k), "r"((t & 1) * 32), "r"(krow), "r"(t >> 1), "r"(fb) : "memory");
                for (int t = 0; t < 4; ++t)      // V^T tiles: [64 dims x 32 keys]
                    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                                 ::"r"(fa_s32(st + (4 + t) * FA_KV_TILE)), "l"(&map_vt), "r"(k0 + (t & 1) * 32), "r"(bh * FA_HD), "r"(t >> 1), "r"(fb) : "memory");
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ---- consumer warpgroup g: query rows 64 g .. +63 of the tile.  Thread (warp w, lane = 4 gid + tig) holds rows r = 16 w + gid and
    //      r + 8, score / output columns 8 j + 2 tig + {0, 1} (j = 0..7); a row's max and sum are reduced over its quad.
    //      Scores arrive in the log2 domain (scale * log2 e folded into Q by the prep pass): p = ex2(s - m) is one MUFU instruction.
    const int ct = tid - 128, g = ct >> 7, w = (ct >> 5) & 3, lane = ct & 31, gid = lane >> 2, tig = lane & 3;
    const int qr[2] = {q0 + g * 64 + w * 16 + gid, q0 + g * 64 + w * 16 + gid + 8};
    const unsigned qa = fa_s32(q_s) + (unsigned)g * (64 * 128);           // this warpgroup's 64 Q rows inside each Q tile
    const unsigned char* kvalid = p.key_valid ? p.key_valid + (long long)b * p.key_valid_ld : nullptr;
    // keys a row may see form one interval [k_lo, k_hi) (none / causal / band); key padding is applied on top when present
    int k_lo[2], k_hi[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int q = qr[e];
        k_lo[e] = 0; k_hi[e] = p.Tk;
        if (p.mask_mode == MASK_CAUSAL) k_hi[e] = min(k_hi[e], p.q_pos0 + q + 1);
        else if (p.mask_mode == MASK_BAND) { k_lo[e] = max(k_lo[e], q - p.band + 1); k_hi[e] = min(k_hi[e], q + p.band + 1); }
        if (q >= p.Tq) k_hi[e] = k_lo[e];
    }
    float o[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) o[j] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    bool ok = ntiles == 0 || fa_wait(&bars->q_full, 0, err);
#pragma unroll 1
    for (int i = 0; i < ntiles && ok; ++i) {
        const int s = i % FA_STAGES;
        ok = fa_wait(&bars->kv_full[s], (i / FA_STAGES) & 1, err);
        if (!ok) break;
        const unsigned kb = fa_s32(kv_s + s * FA_STAGE_BYTES), vb = kb + 4 * FA_KV_TILE;
        float sc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) sc[j] = 0.f;
        gmma_fence_regs(sc);
        gmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {         // 8 k-steps of 8 dims: tile ks / 4, 32-byte sub-step ks % 4
            const unsigned qo = (ks >> 2) * FA_Q_TILE + (ks & 3) * 32, ko = (ks >> 2) * FA_KV_TILE + (ks & 3) * 32;
            const unsigned long long q_hi = gmma_desc(qa + qo), q_lo = gmma_desc(qa + 2 * FA_Q_TILE + qo);
            const unsigned long long k_hi = gmma_desc(kb + ko), k_lo = gmma_desc(kb + 2 * FA_KV_TILE + ko);
            gmma_m64n64k8_ss(sc, q_hi, k_hi, ks > 0 ? 1u : 0u);
            gmma_m64n64k8_ss(sc, q_hi, k_lo, 1u);
            gmma_m64n64k8_ss(sc, q_lo, k_hi, 1u);
        }
        gmma_commit();
        gmma_wait<0>();
        gmma_fence_regs(sc);

        const int k0 = (kt_begin + i) * FA_BN;
        float alpha[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {            // row e: accumulators 4 j + 2 e + {0, 1}
            const int c_lo = k_lo[e] - k0, c_hi = k_hi[e] - k0;
            float mx = -INFINITY;
            if (c_lo <= 0 && c_hi >= FA_BN && kvalid == nullptr) {
#pragma unroll
                for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * e], sc[4 * j + 2 * e + 1]));
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int c = 8 * j + 2 * tig + u;
                        bool allowed = c >= c_lo && c < c_hi;
                        if (kvalid) allowed = allowed && kvalid[min(k0 + c, p.Tk - 1)] != 0;
                        const float v = allowed ? sc[4 * j + 2 * e + u] : -INFINITY;
                        sc[4 * j + 2 * e + u] = v;
                        mx = fmaxf(mx, v);
                    }
                }
            }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[e], mx);
            const float m_use = (m_new == -INFINITY) ? 0.f : m_new;    // fully masked so far: every s is -inf, ex2(-inf - 0) = 0
            alpha[e] = fa_ex2(m_run[e] - m_use);                        // m_run = -inf -> 0 (o and l are 0 anyway)
            float psum = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const float pr = fa_ex2(sc[4 * j + 2 * e + u] - m_use);
                    psum += pr;
                    sc[4 * j + 2 * e + u] = pr;
                }
            }
            l_run[e] = l_run[e] * alpha[e] + psum;                      // this thread's share of the row sum
            m_run[e] = m_new;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0]; o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
        }
        // O += P V: k-step j covers keys 8 j .. 8 j + 7; A fragment (rows r, r + 8; columns tig, tig + 4) = keys 2 tig, 2 tig + 1 (VT order).
        // The hi / lo fragments are all formed before the first MMA is issued, so the MMA batch runs without register hazards.
        unsigned ph[8][4], pl[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int src[4] = {4 * j, 4 * j + 2, 4 * j + 1, 4 * j + 3};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float x = sc[src[u]], hi = fa_rn_tf32(x);
                ph[j][u] = __float_as_uint(hi);
                pl[j][u] = __float_as_uint(fa_rn_tf32(x - hi));
            }
        }
        gmma_fence_regs(o);
        gmma_fence();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned vo = (j >> 2) * FA_KV_TILE + (j & 3) * 32;
            const unsigned long long v_hi = gmma_desc(vb + vo), v_lo = gmma_desc(vb + 2 * FA_KV_TILE + vo);
            gmma_m64n64k8_rs(o, ph[j], v_hi, 1u);
            gmma_m64n64k8_rs(o, ph[j], v_lo, 1u);
            gmma_m64n64k8_rs(o, pl[j], v_hi, 1u);
        }
        gmma_commit();
        gmma_wait<0>();
        gmma_fence_regs(o);
        asm volatile("{ .reg .b64 t; mbarrier.arrive.shared::cta.b64 t, [%0]; }" ::"r"(fa_s32(&bars->kv_empty[s])) : "memory");
    }
    // row sums over the quad, then normalise; fully masked rows (left-pad queries) produce 0 like torch SDPA
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        float l = l_run[e];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        if (qr[e] < p.Tq) {
            const float inv = (ok && l > 0.f) ? 1.0f / l : 0.f;
            float* orow = p.o + (long long)b * p.o_bs + (long long)qr[e] * p.o_ld + h * FA_HD + 2 * tig;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(o[4 * j + 2 * e] * inv, o[4 * j + 2 * e + 1] * inv);
        }
    }
}

// q | k | v (token-major, strided) -> scaled tf32 hi / lo planes, head-major, V transposed; zero padded to whole tiles.
// grid (ceil(max(Tq_pad, Tk_pad) / 64), B * H), 256 threads: each CTA handles 64 tokens of one (batch, head).
struct PrepParams {
    const float* q; long long q_ld, q_bs;
    const float* k; long long k_ld, k_bs;
    const float* v; long long v_ld, v_bs;
    float* qw; float* kw; float* vtw;             // workspaces: [2][BH][Tq_pad][64], [2][BH][Tk_pad][64], [2][BH][64][Tk_pad]
    int B, H, Tq, Tk, Tq_pad, Tk_pad;
    float scale;
};
__global__ void __launch_bounds__(256) attn_prep_kernel(PrepParams p) {
    __shared__ float vt_hi[64][65], vt_lo[64][65];
    const int t0 = blockIdx.x * 64, bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;
    const int tid = threadIdx.x, r = tid >> 4, d4 = (tid & 15) * 4;
    const long long BH = (long long)p.B * p.H;
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        const int row = r + rr * 16, t = t0 + row;
        if (t < p.Tq_pad) {
            float4 x = make_float4(0, 0, 0, 0);
            if (t < p.Tq) x = *reinterpret_cast<const float4*>(p.q + (long long)b * p.q_bs + (long long)t * p.q_ld + h * 64 + d4);
            x.x *= p.scale; x.y *= p.scale; x.z *= p.scale; x.w *= p.scale;
            float4 hi = make_float4(fa_rn_tf32(x.x), fa_rn_tf32(x.y), fa_rn_tf32(x.z), fa_rn_tf32(x.w));
            float4 lo = make_float4(fa_rn_tf32(x.x - hi.x), fa_rn_tf32(x.y - hi.y), fa_rn_tf32(x.z - hi.z), fa_rn_tf32(x.w - hi.w));
            float* dst = p.qw + ((long long)bh * p.Tq_pad + t) * 64 + d4;
            *reinterpret_cast<float4*>(dst) = hi;
            *reinterpret_cast<float4*>(dst + BH * p.Tq_pad * 64) = lo;
        }
        if (t < p.Tk_pad) {
            float4 x = make_float4(0, 0, 0, 0), y = x;
            if (t < p.Tk) {
                x = *reinterpret_cast<const float4*>(p.k + (long long)b * p.k_bs + (long long)t * p.k_ld + h * 64 + d4);
                y = *reinterpret_cast<const float4*>(p.v + (long long)b * p.v_bs + (long long)t * p.v_ld + h * 64 + d4);
            }
            float4 hi = make_float4(fa_rn_tf32(x.x), fa_rn_tf32(x.y), fa_rn_tf32(x.z), fa_rn_tf32(x.w));
            float4 lo = make_float4(fa_rn_tf32(x.x - hi.x), fa_rn_tf32(x.y - hi.y), fa_rn_tf32(x.z - hi.z), fa_rn_tf32(x.w - hi.w));
            float* dst = p.kw + ((long long)bh * p.Tk_pad + t) * 64 + d4;
            *reinterpret_cast<float4*>(dst) = hi;
            *reinterpret_cast<float4*>(dst + BH * p.Tk_pad * 64) = lo;
            const float yv[4] = {y.x, y.y, y.z, y.w};
            const int col = (row & ~7) | ((row & 7) >> 1) | ((row & 1) << 2);      // key 2t -> column t, key 2t + 1 -> column t + 4
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float vh = fa_rn_tf32(yv[c]);
                vt_hi[d4 + c][col] = vh;
                vt_lo[d4 + c][col] = fa_rn_tf32(yv[c] - vh);
            }
        }
    }
    __syncthreads();
    if (t0 < p.Tk_pad) {
        // transposed write: dim = r + 16 * rr, 4 consecutive keys per thread
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
            const int dim = r + rr * 16, kq = (tid & 15) * 4;
            float* dst = p.vtw + ((long long)bh * 64 + dim) * p.Tk_pad + t0 + kq;
            *reinterpret_cast<float4*>(dst) = make_float4(vt_hi[dim][kq], vt_hi[dim][kq + 1], vt_hi[dim][kq + 2], vt_hi[dim][kq + 3]);
            *reinterpret_cast<float4*>(dst + BH * 64 * p.Tk_pad) = make_float4(vt_lo[dim][kq], vt_lo[dim][kq + 1], vt_lo[dim][kq + 2], vt_lo[dim][kq + 3]);
        }
    }
}

typedef CUresult (*FaEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
FaEncodeTiledFn fa_encode_fn() {
    static FaEncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<FaEncodeTiledFn>(p);
    }
    return fn;
}
// [2 planes][rows][cols] fp32, cols contiguous; box {32, box_rows, 1}; 128-byte swizzle
int fa_make_map(CUtensorMap* out, const float* base, long long cols, long long rows, int box_rows) {
    FaEncodeTiledFn fn = fa_encode_fn();
    MB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, 2};
    cuuint64_t strides[2] = {(cuuint64_t)cols * 4, (cuuint64_t)cols * rows * 4};
    cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return 0;
}

}  // namespace

int g_attn_tc_enabled = 1;
int g_attn_tc_min_t = 256;        // below this many queries the launch is a handful of CTAs either way: stay on the SIMT kernel

size_t attn_tc_workspace_bytes(int B, int H, int Tq, int Tk) {
    const size_t tq = (size_t)(Tq + FA_BM - 1) / FA_BM * FA_BM, tk = (size_t)(Tk + FA_BN - 1) / FA_BN * FA_BN;
    return (size_t)B * H * 64 * 4 * 2 * (tq + 2 * tk) + 1024;
}

int AttnCtx::reserve(size_t bytes) {
    if (bytes <= ws_bytes) return 0;
    MB_REQUIRE(!frozen, "attention workspace is frozen (a CUDA graph holds its address) and too small for this launch");
    if (ws) cudaFree(ws);
    ws = nullptr; ws_bytes = 0;
    MB_CUDA_CHECK(cudaMalloc(&ws, bytes));
    ws_bytes = bytes;
    if (!err) { MB_CUDA_CHECK(cudaMalloc(&err, sizeof(int))); MB_CUDA_CHECK(cudaMemset(err, 0, sizeof(int))); }
    return 0;
}
void AttnCtx::destroy() {
    if (ws) cudaFree(ws);
    if (err) cudaFree(err);
    ws = nullptr; err = nullptr; ws_bytes = 0;
}
int AttnCtx::error() {
    if (!err) return 0;
    int e = 0;
    if (cudaMemcpy(&e, err, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return e;
}

bool attn_tc_eligible(const AttentionParams& p, const AttnCtx* ctx) {
    if (!ctx || !g_attn_tc_enabled) return false;
    if (p.mask_mode == MASK_DENSE || p.kv_slot != nullptr) return false;
    if (p.Tq < g_attn_tc_min_t || p.Tk < 1) return false;
    if ((reinterpret_cast<uintptr_t>(p.q) & 15) || (reinterpret_cast<uintptr_t>(p.k) & 15) || (reinterpret_cast<uintptr_t>(p.v) & 15) ||
        (reinterpret_cast<uintptr_t>(p.o) & 15))
        return false;
    if ((p.q_bs % 4) || (p.k_bs % 4) || (p.v_bs % 4) || (p.o_bs % 4)) return false;
    if ((p.q_ld % 4) || (p.k_ld % 4) || (p.v_ld % 4) || (p.o_ld % 4)) return false;      // float4 loads / float2 stores per row
    return true;
}

int launch_attention_tc(const AttentionParams& p, cudaStream_t stream, AttnCtx* ctx) {
    const int Tq_pad = (p.Tq + FA_BM - 1) / FA_BM * FA_BM, Tk_pad = (p.Tk + FA_BN - 1) / FA_BN * FA_BN;
    const long long BH = (long long)p.B * p.H;
    { const int rs = ctx->reserve(attn_tc_workspace_bytes(p.B, p.H, p.Tq, p.Tk)); if (rs) return rs; }
    float* qw = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ctx->ws) + 1023) & ~uintptr_t(1023));
    float* kw = qw + 2 * BH * Tq_pad * 64;
    float* vtw = kw + 2 * BH * Tk_pad * 64;
    // softmax(scale q.k) = 2^(log2e scale q.k - max) / sum: the kernel works in the log2 domain (one ex2 per score)
    PrepParams pp{p.q, p.q_ld, p.q_bs, p.k, p.k_ld, p.k_bs, p.v, p.v_ld, p.v_bs, qw, kw, vtw, p.B, p.H, p.Tq, p.Tk, Tq_pad, Tk_pad, p.scale * 1.4426950408889634f};
    dim3 pgrid((unsigned)((std::max(Tq_pad, Tk_pad) + 63) / 64), (unsigned)BH);
    attn_prep_kernel<<<pgrid, 256, 0, stream>>>(pp);
    MB_LAUNCH_CHECK();
    CUtensorMap mq, mk, mvt;
    MB_REQUIRE(fa_make_map(&mq, qw, 64, BH * Tq_pad, FA_BM) == 0, "tensor map Q");
    MB_REQUIRE(fa_make_map(&mk, kw, 64, BH * Tk_pad, FA_BN) == 0, "tensor map K");
    MB_REQUIRE(fa_make_map(&mvt, vtw, Tk_pad, BH * 64, FA_HD) == 0, "tensor map V^T");
    static bool configured = false;
    const int smem = FA_Q_BYTES + FA_STAGES * FA_STAGE_BYTES + (int)sizeof(FaBarriers) + 1024;
    if (!configured) {
        MB_CUDA_CHECK(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    FaParams fp{p.o, p.o_ld, p.o_bs, p.B, p.H, p.Tq, p.Tk, Tq_pad, Tk_pad, p.mask_mode, p.q_pos0, p.band, p.key_valid, p.key_valid_ld};
    dim3 grid((unsigned)(Tq_pad / FA_BM), (unsigned)BH);
    attention_tc_kernel<<<grid, FA_THREADS, smem, stream>>>(mq, mk, mvt, fp, ctx->err);
    MB_LAUNCH_CHECK();
    g_launch_count += 2;
    return 0;
}

}  // namespace mb200
