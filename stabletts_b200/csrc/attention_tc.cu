// wgmma masked multi-head attention (models/diffusion_transformer.py:58-79,107-108) — flash-style,
// split-bf16 operands, fp32 softmax in the exp2 domain.
//
// Input: the QKV projection's own output planes (BB, T, 3H) as split-bf16 (hi, lo).  RoPE and the
// softmax scale are already applied by the GEMM epilogue (EPI_ROPE, gemm_epilogue.cuh), so Q, K and V
// tiles are plain TMA boxes of that tensor — no re-layout pass:
//     Q tile  [128 queries][64 dims]  channels [64h, 64h+64)        K-major A operand
//     K tile  [ 64 keys   ][64 dims]  channels [H + 64h, ...)       K-major B operand of S = Q·K^T
//     V tile  [ 64 keys   ][64 dims]  channels [2H + 64h, ...)      MN-major B operand of O += P·V
// One CTA per (128-query tile, head, batch row): two warpgroups of 64 queries each share the K / V
// tiles, which one thread brings in by TMA into a ring of two (block j + 2 is requested as soon as
// both warpgroups have finished block j).
//   * S = Q·K^T lands in the warpgroup's registers (wgmma m64n64k16, three products per k-step); a
//     query row lives in the four lanes of a quad, so row max / row sum are two shuffles;
//   * online softmax on registers: the O accumulator is rescaled in place when the running max moves;
//   * P never leaves the registers: the S accumulator layout IS the wgmma A-fragment layout, so the
//     split-bf16 words of P feed O += P·V directly (A from registers, V transposed by the MMA).
// Mask semantics: keys with mask == 0 get probability exactly 0; query rows with mask == 0 are written
// as 0 (the reference multiplies them by the mask afterwards, :111).
#include "common.cuh"
#include "tc_ptx.cuh"
#include "gemm_epilogue.cuh"     // kQScale
#include <math_constants.h>
#include <mutex>
#include <string>
#include <cstring>
#include <cstdlib>
#include <cstdio>

namespace st {

bool tmap_encode_bf16(const void* ptr, int rank, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1,
                      CUtensorMap* out);    // gemm_tc.cu (cached)
const char* gemm_tc_last_error();

namespace {

using namespace ptx;

constexpr int AQ = 128;          // queries per CTA (two warpgroups x 64)
constexpr int AK = 64;           // keys per block
constexpr int DH = 64;
constexpr int A_THREADS = 256;
constexpr int K_BYTES = AK * DH * 2;        // 8 KB per plane

struct AttMaps { CUtensorMap q_hi, q_lo, kv_hi, kv_lo; };

struct AttParams {
    int BB, B, T, H, n_heads;
    const float* mask; const int* kvlen; const int* prefix;
    float* out_f32; bf16* out_hi; bf16* out_lo;
};

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// ----------------------------------------------------------------------------------------------
// fp32 packed qkv (BB, T, 3H) -> RoPE'd, q-scaled split-bf16 planes of the same shape.  Used by the
// kernel-level test hook and when the QKV projection ran on the SIMT engine; the product path gets
// this from the QKV GEMM epilogue instead.
// ----------------------------------------------------------------------------------------------
__global__ void rope_split_kernel(const float* __restrict__ qkv, const float* __restrict__ rope_cs, bf16* __restrict__ hi,
                                  bf16* __restrict__ lo, long rows, int T, int H) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // one thread per (row, column pair)
    const int H3 = 3 * H, half = H3 / 2;
    if (i >= rows * half) return;
    const long row = i / half;
    const int c = (int)(i % half) * 2;
    const int t = (int)(row % T);
    float x[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int n = c + e, d = n & 63;
        float v = qkv[row * H3 + n];
        if (n < 2 * H && d < 32) {
            const int j = d & 15;
            const float cs = rope_cs[((long)t * 16 + j) * 2], sn = rope_cs[((long)t * 16 + j) * 2 + 1];
            const float o = (d < 16) ? -qkv[row * H3 + n + 16] : qkv[row * H3 + n - 16];
            v = v * cs + o * sn;
        }
        if (n < H) v *= kQScale;
        x[e] = v;
    }
    uint32_t h2, l2;
    split_bf16x2(x[0], x[1], h2, l2);
    *reinterpret_cast<uint32_t*>(hi + row * H3 + c) = h2;
    *reinterpret_cast<uint32_t*>(lo + row * H3 + c) = l2;
}

constexpr int Q_BYTES = AQ * DH * 2;         // 16 KB per plane
constexpr int ATT_SMEM = 2 * Q_BYTES + 4 * K_BYTES + 4 * K_BYTES + 64 /*barriers*/ + 1024 /*align slack*/;

__global__ void __launch_bounds__(A_THREADS, 2)
attention_wgmma_kernel(const __grid_constant__ AttMaps maps, const AttParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;                  // [hi 16K | lo 16K]
    uint8_t* sK = sQ + 2 * Q_BYTES;      // ring of 2: [hi 8K | lo 8K]
    uint8_t* sV = sK + 4 * K_BYTES;      // ring of 2: [hi 8K | lo 8K]
    uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + 4 * K_BYTES);
    uint64_t* kv_full = q_full + 1;      // [2]
    pdl_trigger(); pdl_wait();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bb = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AQ;
    const int b = bb % p.B;
    const int kvlen = p.kvlen[b];
    const int ck = p.H + h * DH, cv = 2 * p.H + h * DH;     // channel offsets of this head's K and V

    if (q0 >= kvlen) {
        // whole query tile is padding (or the utterance is empty): exact zeros, no pipeline needed
        for (int i = threadIdx.x; i < AQ * (DH / 4); i += A_THREADS) {
            const int r = i / (DH / 4), c4 = (i % (DH / 4)) * 4, t = q0 + r;
            if (t < p.T) {
                const long o = ((long)bb * p.T + t) * p.H + h * DH + c4;
                if (p.out_f32) *reinterpret_cast<float4*>(p.out_f32 + o) = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.out_hi) { *reinterpret_cast<uint2*>(p.out_hi + o) = make_uint2(0, 0); *reinterpret_cast<uint2*>(p.out_lo + o) = make_uint2(0, 0); }
            }
        }
        return;
    }
    const int nb = (kvlen + AK - 1) / AK;

    auto issue_kv = [&](int j) {         // K and V tiles of key block j -> ring slot j & 1
        const int slot = j & 1;
        mbar_expect_tx(&kv_full[slot], 4 * K_BYTES);
        tma_load_3d(&maps.kv_hi, &kv_full[slot], sK + slot * 2 * K_BYTES, ck, j * AK, bb);
        tma_load_3d(&maps.kv_lo, &kv_full[slot], sK + slot * 2 * K_BYTES + K_BYTES, ck, j * AK, bb);
        tma_load_3d(&maps.kv_hi, &kv_full[slot], sV + slot * 2 * K_BYTES, cv, j * AK, bb);
        tma_load_3d(&maps.kv_lo, &kv_full[slot], sV + slot * 2 * K_BYTES + K_BYTES, cv, j * AK, bb);
    };
    if (threadIdx.x == 0) {
        mbar_init(q_full, 1); mbar_init(&kv_full[0], 1); mbar_init(&kv_full[1], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(q_full, 2 * Q_BYTES);
        tma_load_3d(&maps.q_hi, q_full, sQ, h * DH, q0, bb);
        tma_load_3d(&maps.q_lo, q_full, sQ + Q_BYTES, h * DH, q0, bb);
        for (int j = 0; j < 2 && j < nb; ++j) issue_kv(j);
    }

    // thread <-> rows 16w + lane / 4 (+ 8) of its warpgroup's 64 queries, column pairs 8jj + 2(lane % 4) + {0, 1}
    const int wgi = warp >> 2, cq = 2 * (lane & 3);
    const int row0 = q0 + wgi * 64 + (warp & 3) * 16 + (lane >> 2);
    const int prefix = p.prefix[b];
    const float* mrow = p.mask + (long)b * p.T;
    const uint32_t aQ = smem_u32(sQ) + (uint32_t)wgi * (64 * 128);
    const uint64_t dQh = make_sw128_desc(aQ), dQl = make_sw128_desc(aQ + Q_BYTES);
    constexpr uint64_t v_adv = (uint64_t)((16 * 128) >> 4);      // MN-major V tile: 16 keys = +2048 B
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};

    mbar_wait(q_full, 0);
    for (int j = 0; j < nb; ++j) {
        const int slot = j & 1;
        mbar_wait(&kv_full[slot], (j >> 1) & 1);
        const uint64_t dKh = make_sw128_desc(smem_u32(sK + slot * 2 * K_BYTES));
        const uint64_t dKl = make_sw128_desc(smem_u32(sK + slot * 2 * K_BYTES + K_BYTES));
        float s[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DH / 16; ++k) {
            const uint64_t adv = (uint64_t)(k * 2);
            wgmma_m64n64k16_ss(s, dQl + adv, dKh + adv, k != 0);     // small terms first
            wgmma_m64n64k16_ss(s, dQh + adv, dKl + adv, 1);
            wgmma_m64n64k16_ss(s, dQh + adv, dKh + adv, 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        // key validity (only blocks reaching past the all-ones prefix of the mask need it)
        if (j * AK + AK > prefix) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int key = j * AK + 8 * jj + cq + e;
                    if (!(key < kvlen && __ldg(mrow + min(key, p.T - 1)) != 0.f)) { s[4 * jj + e] = -CUDART_INF_F; s[4 * jj + 2 + e] = -CUDART_INF_F; }
                }
            }
        }
        uint32_t ph[4][4], pl[4][4];                       // split-bf16 P as wgmma A fragments, one per 16-key step
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float mx = -CUDART_INF_F;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * r], s[4 * jj + 2 * r + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[r], mx);
            const float m_eff = (m_new == -CUDART_INF_F) ? 0.f : m_new;
            const float factor = (m_run[r] == -CUDART_INF_F) ? 1.f : ex2_approx(m_run[r] - m_new);
            m_run[r] = m_new;
            float ps = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                o[4 * jj + 2 * r] *= factor; o[4 * jj + 2 * r + 1] *= factor;
                const float p0 = ex2_approx(s[4 * jj + 2 * r] - m_eff), p1 = ex2_approx(s[4 * jj + 2 * r + 1] - m_eff);
                ps += p0 + p1;
                // S accumulator -> A fragment: column group jj is k-step jj / 2, registers (jj & 1) * 2 + r
                split_bf16x2(p0, p1, ph[jj >> 1][(jj & 1) * 2 + r], pl[jj >> 1][(jj & 1) * 2 + r]);
            }
            l_run[r] = l_run[r] * factor + ps;             // this thread's share of the row sum (quad-reduced at the end)
        }
        const uint64_t dVh = make_sw128_desc(smem_u32(sV + slot * 2 * K_BYTES));
        const uint64_t dVl = make_sw128_desc(smem_u32(sV + slot * 2 * K_BYTES + K_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AK / 16; ++k) {
            const uint64_t va = (uint64_t)k * v_adv;
            wgmma_m64n64k16_rs_tb(o, pl[k], dVh + va, 1);
            wgmma_m64n64k16_rs_tb(o, ph[k], dVl + va, 1);
            wgmma_m64n64k16_rs_tb(o, ph[k], dVh + va, 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncthreads();                                   // both warpgroups have finished reading ring slot j & 1
        if (threadIdx.x == 0 && j + 2 < nb) issue_kv(j + 2);
    }

#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float lsum = l_run[r];
        lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
        lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
        const int t = row0 + 8 * r;
        if (t >= p.T) continue;
        const float inv = (mrow[t] != 0.f && lsum > 0.f) ? 1.0f / lsum : 0.f;
        const long ob = ((long)bb * p.T + t) * p.H + h * DH + cq;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const float f0 = o[4 * jj + 2 * r] * inv, f1 = o[4 * jj + 2 * r + 1] * inv;
            if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + ob + 8 * jj) = make_float2(f0, f1);
            if (p.out_hi) {
                uint32_t h2, l2;
                split_bf16x2(f0, f1, h2, l2);
                *reinterpret_cast<uint32_t*>(p.out_hi + ob + 8 * jj) = h2;
                *reinterpret_cast<uint32_t*>(p.out_lo + ob + 8 * jj) = l2;
            }
        }
    }
}

std::mutex g_att_mu;
std::atomic<uint64_t> g_att_attr{0};    // one bit per device
std::string g_att_err;

}  // namespace

const char* attention_tc_last_error() { return g_att_err.c_str(); }

cudaError_t launch_rope_split(const float* qkv, const float* rope_cs, bf16* hi, bf16* lo, int BB, int T, int H, cudaStream_t s) {
    const long rows = (long)BB * T, n = rows * (3 * H / 2);
    if (n == 0) return cudaSuccess;
    rope_split_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(qkv, rope_cs, hi, lo, rows, T, H);
    return cudaGetLastError();
}

// a.qkv_hi / a.qkv_lo: RoPE'd, q-scaled split planes (BB, T, 3H)
cudaError_t launch_attention_tc(const AttnArgs& a, cudaStream_t s) {
    std::lock_guard<std::mutex> lk(g_att_mu);
    if (a.H != a.n_heads * DH) return cudaErrorInvalidValue;
    if (a.BB == 0 || a.T == 0) return cudaSuccess;
    if (!a.qkv_hi || !a.qkv_lo) { g_att_err = "split qkv planes missing"; return cudaErrorInvalidValue; }
    AttMaps maps;
    const uint64_t C3 = 3 * (uint64_t)a.H;
    bool ok = true;
    ok = ok && tmap_encode_bf16(a.qkv_hi, 3, C3, (uint64_t)a.T, (uint64_t)a.BB, DH, AQ, &maps.q_hi);
    ok = ok && tmap_encode_bf16(a.qkv_lo, 3, C3, (uint64_t)a.T, (uint64_t)a.BB, DH, AQ, &maps.q_lo);
    ok = ok && tmap_encode_bf16(a.qkv_hi, 3, C3, (uint64_t)a.T, (uint64_t)a.BB, DH, AK, &maps.kv_hi);
    ok = ok && tmap_encode_bf16(a.qkv_lo, 3, C3, (uint64_t)a.T, (uint64_t)a.BB, DH, AK, &maps.kv_lo);
    if (!ok) { g_att_err = gemm_tc_last_error(); return cudaErrorInvalidValue; }
    AttParams p;
    p.BB = a.BB; p.B = a.B; p.T = a.T; p.H = a.H; p.n_heads = a.n_heads;
    p.mask = a.mask; p.kvlen = a.kvlen; p.prefix = a.prefix;
    p.out_f32 = a.out_f32; p.out_hi = a.out_hi; p.out_lo = a.out_lo;
    {
        cudaError_t e = ensure_dyn_smem(attention_wgmma_kernel, ATT_SMEM, g_att_attr);
        if (e != cudaSuccess) { g_att_err = "cudaFuncSetAttribute failed for the attention kernel"; return e; }
    }
    dim3 grid((a.T + AQ - 1) / AQ, a.n_heads, a.BB);
    return launch_k(attention_wgmma_kernel, grid, dim3(A_THREADS), (size_t)ATT_SMEM, s, maps, p);
}

}  // namespace st
