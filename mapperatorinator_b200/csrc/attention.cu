// fp32 flash attention for the dense phases of the hot path (head_dim 64):
//   * Whisper encoder self-attention (T = 512, bidirectional)            HF modeling_whisper.py:286-358
//   * decoder prefill: causal + left-pad key mask, and cross-attention    HF modeling_whisper.py:417-507
//   * DiT blocks: +-128 band mask of diffusion_pipeline.py:146-148 (or any dense bool mask)   models.py:145-151
// One CTA = 64 queries of one (batch, head); K/V streamed in 64-key tiles through shared memory; online softmax in
// fp32 registers; KV tiles that the mask rules out entirely are skipped.  Operands are token-major ([B, T, H*64]), the
// layout the projection GEMMs write, so no head transposes exist anywhere in the engine.
#include "common.cuh"
#include "kernels.h"

namespace mb200 {
namespace {

constexpr int TQ = 64, TK = 64, HD = 64, LDS_ = 68;   // 68 = 64 + 4 pad (keeps float4 alignment)

__device__ __forceinline__ bool mask_allowed(const AttentionParams& p, int b, int q, int k) {
    if (k >= p.Tk) return false;
    if (p.key_valid && !p.key_valid[(long long)b * p.key_valid_ld + k]) return false;
    switch (p.mask_mode) {
        case MASK_CAUSAL: return k <= p.q_pos0 + q;
        case MASK_BAND:   return (q >= k - p.band) && (q < k + p.band);
        case MASK_DENSE:  return q < p.Tq && !p.dense[(long long)q * p.Tk + k];
        default:          return true;
    }
}

// QPT queries per thread (4: one CTA = 64 queries; 1: one CTA = 16 queries, for launches that would leave most SMs idle).  Lane tx
// always owns keys tx*4..+3 of a tile and output dims tx*4..+3, so every query's arithmetic is the same for both instantiations.
template <int QPT>
__global__ void __launch_bounds__(256) attention_kernel(AttentionParams p) {
    constexpr int TQ_ = 16 * QPT;
    extern __shared__ __align__(16) float smem[];
    float (*Qt)[LDS_] = reinterpret_cast<float (*)[LDS_]>(smem);                    // [d][q]
    float (*Kt)[LDS_] = reinterpret_cast<float (*)[LDS_]>(smem + HD * LDS_);        // [d][k]
    float (*Vs)[LDS_] = reinterpret_cast<float (*)[LDS_]>(smem + 2 * HD * LDS_);    // [k][d]
    float (*Ps)[LDS_] = reinterpret_cast<float (*)[LDS_]>(smem + 3 * HD * LDS_);    // [q][k]

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int q0 = blockIdx.x * TQ_, h = blockIdx.y, b = blockIdx.z;
    const float* qb = p.q + (long long)b * p.q_bs + h * HD;
    const int kvb = p.kv_slot ? p.kv_slot[b] : b;
    const float* kb = p.k + (long long)kvb * p.k_bs + h * HD;
    const float* vb = p.v + (long long)kvb * p.v_bs + h * HD;

    // ---- stage Q^T (pre-multiplied by scale) ----
    {
        const int r = tid >> 4, dq = (tid & 15) * 4;
#pragma unroll
        for (int rr = 0; rr < QPT; ++rr) {
            int row = r + rr * 16, q = q0 + row;
            float4 v = q < p.Tq ? *reinterpret_cast<const float4*>(qb + (long long)q * p.q_ld + dq) : make_float4(0, 0, 0, 0);
            Qt[dq + 0][row] = v.x * p.scale; Qt[dq + 1][row] = v.y * p.scale;
            Qt[dq + 2][row] = v.z * p.scale; Qt[dq + 3][row] = v.w * p.scale;
        }
    }

    // ---- KV tile range allowed by the mask ----
    int kt_begin = 0, kt_end = (p.Tk + TK - 1) / TK;
    if (p.mask_mode == MASK_CAUSAL) {
        int last = p.q_pos0 + min(q0 + TQ_ - 1, p.Tq - 1);
        kt_end = min(kt_end, last / TK + 1);
    } else if (p.mask_mode == MASK_BAND) {
        int lo = q0 - p.band + 1, hi = min(q0 + TQ_ - 1, p.Tq - 1) + p.band;
        kt_begin = max(0, lo) / TK;
        kt_end = min(kt_end, hi / TK + 1);
    }

    float m_i[QPT], l_i[QPT], o[QPT][4];
#pragma unroll
    for (int i = 0; i < QPT; ++i) {
        m_i[i] = -INFINITY; l_i[i] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
    }

    // K/V tiles go through registers; with QPT = 1 one tile ahead, so the next tile's global reads overlap this tile's math (with
    // QPT = 4 the extra registers would cost a resident CTA per SM)
    constexpr bool AHEAD = QPT == 1;
    float4 kr[4], vr[4];
    auto gload = [&](int k0) {
        const int r = tid >> 4, dq = (tid & 15) * 4;
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
            int k = k0 + r + rr * 16;
            kr[rr] = make_float4(0, 0, 0, 0); vr[rr] = make_float4(0, 0, 0, 0);
            if (k < p.Tk) {
                kr[rr] = *reinterpret_cast<const float4*>(kb + (long long)k * p.k_ld + dq);
                vr[rr] = *reinterpret_cast<const float4*>(vb + (long long)k * p.v_ld + dq);
            }
        }
    };
    if (AHEAD && kt_begin < kt_end) gload(kt_begin * TK);

    for (int kt = kt_begin; kt < kt_end; ++kt) {
        const int k0 = kt * TK;
        __syncthreads();   // previous tile fully consumed (also orders the Q^T staging before first use)
        if (!AHEAD) gload(k0);
        {
            const int r = tid >> 4, dq = (tid & 15) * 4;
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) {
                int row = r + rr * 16;
                Kt[dq + 0][row] = kr[rr].x; Kt[dq + 1][row] = kr[rr].y; Kt[dq + 2][row] = kr[rr].z; Kt[dq + 3][row] = kr[rr].w;
                *reinterpret_cast<float4*>(&Vs[row][dq]) = vr[rr];
            }
        }
        __syncthreads();
        if (AHEAD && kt + 1 < kt_end) gload(k0 + TK);

        // ---- S = Q K^T for this thread's QPT x 4 block ----
        float s[QPT][4];
#pragma unroll
        for (int i = 0; i < QPT; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 16
        for (int d = 0; d < HD; ++d) {
            float qv[QPT];
            if constexpr (QPT == 4) {
                float4 qa = *reinterpret_cast<const float4*>(&Qt[d][ty * 4]);
                qv[0] = qa.x; qv[1] = qa.y; qv[2] = qa.z; qv[3] = qa.w;
            } else {
                qv[0] = Qt[d][ty];
            }
            float4 ka = *reinterpret_cast<const float4*>(&Kt[d][tx * 4]);
            float kv[4] = {ka.x, ka.y, ka.z, ka.w};
#pragma unroll
            for (int i = 0; i < QPT; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
        }

        // ---- mask, online softmax ----
#pragma unroll
        for (int i = 0; i < QPT; ++i) {
            const int q = q0 + ty * QPT + i;
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (!mask_allowed(p, b, q, k0 + tx * 4 + j)) s[i][j] = -INFINITY;
                mx = fmaxf(mx, s[i][j]);
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float m_new = fmaxf(m_i[i], mx);
            const float corr = (m_new == -INFINITY) ? 1.f : expf(m_i[i] - m_new);
            float psum = 0.f;
            float pr[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                pr[j] = (s[i][j] == -INFINITY) ? 0.f : expf(s[i][j] - m_new);
                psum += pr[j];
            }
            l_i[i] = fmaf(l_i[i], corr, psum);      // spelled out: the compiler contracts it in one instantiation and not the other
            m_i[i] = m_new;
#pragma unroll
            for (int j = 0; j < 4; ++j) o[i][j] *= corr;
            *reinterpret_cast<float4*>(&Ps[ty * QPT + i][tx * 4]) = make_float4(pr[0], pr[1], pr[2], pr[3]);
        }
        __syncthreads();

        // ---- O += P V ----
#pragma unroll 4
        for (int c4 = 0; c4 < TK / 4; ++c4) {
            float4 pa[QPT], va[4];
#pragma unroll
            for (int i = 0; i < QPT; ++i) pa[i] = *reinterpret_cast<const float4*>(&Ps[ty * QPT + i][c4 * 4]);
#pragma unroll
            for (int c = 0; c < 4; ++c) va[c] = *reinterpret_cast<const float4*>(&Vs[c4 * 4 + c][tx * 4]);
#pragma unroll
            for (int i = 0; i < QPT; ++i) {
                const float pv[4] = {pa[i].x, pa[i].y, pa[i].z, pa[i].w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    o[i][0] = fmaf(pv[c], va[c].x, o[i][0]); o[i][1] = fmaf(pv[c], va[c].y, o[i][1]);
                    o[i][2] = fmaf(pv[c], va[c].z, o[i][2]); o[i][3] = fmaf(pv[c], va[c].w, o[i][3]);
                }
            }
        }
    }

    // ---- normalise and store; fully masked rows (left-pad queries) produce 0 like torch SDPA ----
    float* ob = p.o + (long long)b * p.o_bs + h * HD;
#pragma unroll
    for (int i = 0; i < QPT; ++i) {
        float l = l_i[i];
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) l += __shfl_xor_sync(0xffffffffu, l, off);
        const int q = q0 + ty * QPT + i;
        if (q >= p.Tq) continue;
        const float inv = l > 0.f ? 1.0f / l : 0.f;
        *reinterpret_cast<float4*>(ob + (long long)q * p.o_ld + tx * 4) =
            make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
    }
}

}  // namespace

int launch_attention(const AttentionParams& p, cudaStream_t stream, AttnCtx* ctx) {
    MB_REQUIRE(p.q_ld % 4 == 0 && p.k_ld % 4 == 0 && p.v_ld % 4 == 0 && p.o_ld % 4 == 0, "attention strides must be multiples of 4");
    if (p.B <= 0 || p.Tq <= 0) return 0;
    if (attn_tc_eligible(p, ctx)) return launch_attention_tc(p, stream, ctx);
    static bool configured = false;
    static int num_sms = 0;
    const int smem_bytes = 4 * HD * LDS_ * (int)sizeof(float);
    if (!configured) {
        MB_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        MB_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        int dev = 0;
        MB_CUDA_CHECK(cudaGetDevice(&dev));
        MB_CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        configured = true;
    }
    // short query runs (decoder prefill: one (batch, head) pair per CTA would fill a tenth of the SMs): 16 queries per CTA
    if ((long long)((p.Tq + TQ - 1) / TQ) * p.H * p.B < num_sms) {
        attention_kernel<1><<<dim3((p.Tq + 15) / 16, p.H, p.B), 256, smem_bytes, stream>>>(p);
    } else {
        attention_kernel<4><<<dim3((p.Tq + TQ - 1) / TQ, p.H, p.B), 256, smem_bytes, stream>>>(p);
    }
    MB_LAUNCH_CHECK();
    ++g_launch_count;
    return 0;
}

}  // namespace mb200
