// Masked multi-head self-attention with partial RoPE (models/diffusion_transformer.py:58-79,
// 107-108, 123-198), flash-style: never materialises the (B,1,T,T) float mask or the scores.
//
// Semantics reproduced from the reference:
//   * head h = channels [64h, 64h+64); RoPE rotates dims [0,32) in pairs (j, j+16), position =
//     frame index from 0; dims [32,64) pass through (rope_cs == nullptr: no RoPE at all);
//   * softmax(QK^T / sqrt(64) + M) V, M = -FLT_MAX where query OR key is padded.  For a valid
//     query only valid keys contribute (exp underflows to exactly 0 for the others); a padded
//     query's row is multiplied by mask afterwards (:111), so we write 0 there.
//
// v1 engine (fp32 SIMT): one thread per query, K/V tiles broadcast from shared memory.
#include "common.cuh"
#include <math_constants.h>

namespace st {

constexpr int AT_Q = 128;    // queries per block (one per thread)
constexpr int AT_K = 32;     // keys per smem tile
constexpr int DH = 64;       // head dim
constexpr int DROT = 32;     // rotated dims

__global__ void __launch_bounds__(AT_Q) attention_simt_kernel(AttnArgs a) {
    pdl_trigger(); pdl_wait();
    __shared__ __align__(16) float Ks[AT_K][DH];
    __shared__ __align__(16) float Vs[AT_K][DH];
    __shared__ float Mk[AT_K];
    const int bb = blockIdx.z, h = blockIdx.y;
    const int b = bb % a.B;
    const int q = blockIdx.x * AT_Q + threadIdx.x;
    const int H3 = 3 * a.H;
    const int kvlen = a.kvlen[b];
    const bool q_in = q < a.T;
    const bool q_valid = q_in && a.mask[(long)b * a.T + q] != 0.f;

    float qr[DH], acc[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = 0.f;
    if (q_valid) {
        const float* qp = a.qkv + ((long)bb * a.T + q) * H3 + h * DH;
#pragma unroll
        for (int d4 = 0; d4 < DH / 4; ++d4) {
            float4 v = *reinterpret_cast<const float4*>(qp + d4 * 4);
            qr[d4 * 4 + 0] = v.x; qr[d4 * 4 + 1] = v.y; qr[d4 * 4 + 2] = v.z; qr[d4 * 4 + 3] = v.w;
        }
        const float* cs = a.rope_cs ? a.rope_cs + (long)q * (DROT / 2) * 2 : nullptr;
#pragma unroll
        for (int j = 0; j < (a.rope_cs ? DROT / 2 : 0); ++j) {
            float c = cs[j * 2], s = cs[j * 2 + 1];
            float x0 = qr[j], x1 = qr[j + DROT / 2];
            qr[j] = x0 * c - x1 * s;
            qr[j + DROT / 2] = x1 * c + x0 * s;
        }
#pragma unroll
        for (int d = 0; d < DH; ++d) qr[d] *= 0.125f;      // 1/sqrt(64), SDPA default scale (:77)
    } else {
#pragma unroll
        for (int d = 0; d < DH; ++d) qr[d] = 0.f;
    }
    float m_run = -CUDART_INF_F, l_run = 0.f;

    for (int k0 = 0; k0 < kvlen; k0 += AT_K) {
        __syncthreads();
        // load K, V tile (raw), 4 float4 per thread each
        for (int i = threadIdx.x; i < AT_K * DH / 4; i += AT_Q) {
            int r = i / (DH / 4), c4 = i % (DH / 4);
            int kj = k0 + r;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (kj < kvlen) {
                const float* base = a.qkv + ((long)bb * a.T + kj) * H3 + h * DH + c4 * 4;
                kv = *reinterpret_cast<const float4*>(base + a.H);
                vv = *reinterpret_cast<const float4*>(base + 2 * a.H);
            }
            *reinterpret_cast<float4*>(&Ks[r][c4 * 4]) = kv;
            *reinterpret_cast<float4*>(&Vs[r][c4 * 4]) = vv;
        }
        if (threadIdx.x < AT_K) {
            int kj = k0 + threadIdx.x;
            Mk[threadIdx.x] = (kj < kvlen) ? a.mask[(long)b * a.T + kj] : 0.f;
        }
        __syncthreads();
        // RoPE on the K tile in place: AT_K * 16 pairs (none without a table: nn.MultiheadAttention of the style encoder)
        for (int i = threadIdx.x; a.rope_cs && i < AT_K * (DROT / 2); i += AT_Q) {
            int r = i / (DROT / 2), j = i % (DROT / 2);
            int kj = k0 + r;
            if (kj < kvlen) {
                const float* cs = a.rope_cs + ((long)kj * (DROT / 2) + j) * 2;
                float c = cs[0], s = cs[1];
                float x0 = Ks[r][j], x1 = Ks[r][j + DROT / 2];
                Ks[r][j] = x0 * c - x1 * s;
                Ks[r][j + DROT / 2] = x1 * c + x0 * s;
            }
        }
        __syncthreads();
        if (!q_valid) continue;
#pragma unroll 1
        for (int c0 = 0; c0 < AT_K; c0 += 8) {
            float sc[8];
            float cmax = -CUDART_INF_F;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                float s = 0.f;
#pragma unroll
                for (int d4 = 0; d4 < DH / 4; ++d4) {
                    float4 kv = *reinterpret_cast<const float4*>(&Ks[c0 + jj][d4 * 4]);
                    s = fmaf(qr[d4 * 4 + 0], kv.x, s); s = fmaf(qr[d4 * 4 + 1], kv.y, s);
                    s = fmaf(qr[d4 * 4 + 2], kv.z, s); s = fmaf(qr[d4 * 4 + 3], kv.w, s);
                }
                s = (Mk[c0 + jj] != 0.f) ? s : -CUDART_INF_F;
                sc[jj] = s;
                cmax = fmaxf(cmax, s);
            }
            if (cmax == -CUDART_INF_F) continue;
            const float m_new = fmaxf(m_run, cmax);
            const float corr = expf(m_run - m_new);
            l_run *= corr;
#pragma unroll
            for (int d = 0; d < DH; ++d) acc[d] *= corr;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                float p = expf(sc[jj] - m_new);
                l_run += p;
#pragma unroll
                for (int d4 = 0; d4 < DH / 4; ++d4) {
                    float4 vv = *reinterpret_cast<const float4*>(&Vs[c0 + jj][d4 * 4]);
                    acc[d4 * 4 + 0] = fmaf(p, vv.x, acc[d4 * 4 + 0]); acc[d4 * 4 + 1] = fmaf(p, vv.y, acc[d4 * 4 + 1]);
                    acc[d4 * 4 + 2] = fmaf(p, vv.z, acc[d4 * 4 + 2]); acc[d4 * 4 + 3] = fmaf(p, vv.w, acc[d4 * 4 + 3]);
                }
            }
            m_run = m_new;
        }
    }
    if (!q_in) return;
    const float inv = (q_valid && l_run > 0.f) ? 1.0f / l_run : 0.f;
    const long o = ((long)bb * a.T + q) * a.H + h * DH;
#pragma unroll
    for (int d4 = 0; d4 < DH / 4; ++d4) {
        float v0 = acc[d4 * 4 + 0] * inv, v1 = acc[d4 * 4 + 1] * inv, v2 = acc[d4 * 4 + 2] * inv, v3 = acc[d4 * 4 + 3] * inv;
        if (a.out_f32) *reinterpret_cast<float4*>(a.out_f32 + o + d4 * 4) = make_float4(v0, v1, v2, v3);
        if (a.out_hi) {
            bf16 hh[4], ll[4];
            split_bf16(v0, hh[0], ll[0]); split_bf16(v1, hh[1], ll[1]); split_bf16(v2, hh[2], ll[2]); split_bf16(v3, hh[3], ll[3]);
#pragma unroll
            for (int e = 0; e < 4; ++e) { a.out_hi[o + d4 * 4 + e] = hh[e]; a.out_lo[o + d4 * 4 + e] = ll[e]; }
        }
    }
}

cudaError_t launch_attention_simt(const AttnArgs& a, cudaStream_t s) {
    if (a.H != a.n_heads * DH) return cudaErrorInvalidValue;
    if (a.BB == 0 || a.T == 0) return cudaSuccess;
    dim3 grid((a.T + AT_Q - 1) / AT_Q, a.n_heads, a.BB);
    attention_simt_kernel<<<grid, AT_Q, 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace st
