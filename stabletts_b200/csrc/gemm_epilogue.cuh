// Fused conv-GEMM epilogue of the wgmma kernel (gemm_tc.cu), run on the accumulator registers.
//
// A consumer warpgroup owns 64 frames x BN channels.  In the wgmma accumulator layout thread (warp w, lane l) holds, for
// every 8-column group j, the column pair 8j + 2(l % 4) + {0, 1} of rows 16w + l / 4 and 16w + l / 4 + 8, so
//   * all math runs on registers — bias / SiLU / GELU / FiLM / mask / gate / residual, and the partial RoPE of the QKV
//     projection (the rotation partners c, c + 16 of a head live in the same thread);
//   * per-column vectors and residual rows are read as 8-byte pairs, results leave as 8-byte fp32 pairs and / or packed
//     split-bf16 (or fp16) words; the four lanes of a row cover one 32-byte sector per column group;
//   * when the tile spans all N = BN channels a row lives in the four lanes of one quad, so the LayerNorm + adaLN-modulate
//     that follows O / conv_2 / the long-skip conv / in_proj in the reference (models/diffusion_transformer.py:111-112,
//     119-121) is fused: the finished row stays in the accumulator registers, mean and variance are two quad reductions,
//     and the split-bf16 operand of the next GEMM is emitted directly — no separate LayerNorm kernel, no HBM round trip.
// One code instance per mode (plain / SiLU / GELU / RoPE / residual / LayerNorm-fused); a launch executes exactly one.
#pragma once
#include "common.cuh"
#include <cstdlib>
#include "tc_ptx.cuh"

namespace st {

enum : int { EM_PLAIN = 0, EM_SILU = 1, EM_GELU = 2, EM_ROPE = 3, EM_LN = 4, EM_RESID = 5 };   // EM_RESID: plain + residual rows

struct TcParams {
    int n_src, Cs0, Cs1, taps, N, a_bmod, BB, T;
    int m_tiles_per_b, n_tiles, total_tiles;
    int flags, B, film_H, c_clamp, resid_clamp, rope_H, tap_outer;
    long film_bstride, gate_bstride;
    const float *bias, *mask, *film, *gate, *resid, *rope_cs;
    int mode;                         // EM_* (kernel-uniform)
    float* out_f32; bf16* out_hi; bf16* out_lo;       // (BB, T, N) outputs; out16: out_hi is ONE fp16 plane (GemmArgs::prec)
    int out16, u16;
    // EM_LN: u = ((x - mean) * rstd * (1 + scale) + shift) [* mask] over the finished row -> u_hi / u_lo;
    // film2: x2 = (gamma2 * x + beta2) * mask first (the NEXT block's time fusion, models/estimator.py:16) -> out2_f32, LN over x2
    int ln_mask_out;
    const float *ln_shift, *ln_scale, *film2;
    float* out2_f32; bf16* u_hi; bf16* u_lo;
    long ada_bstride, film2_bstride;
    int ksplit, split_bb;             // split-K: batch index = slice * split_bb + real batch; slice picks the K range
};

inline int epilogue_mode(const GemmArgs& g) {
    if (g.flags & EPI_ROPE) return EM_ROPE;
    if (g.ln) return EM_LN;
    if (g.flags & EPI_SILU) return EM_SILU;
    if (g.flags & EPI_GELU) return EM_GELU;
    if (g.flags & EPI_RESID) return EM_RESID;
    return EM_PLAIN;
}

inline void fill_tc_params(TcParams& p, const GemmArgs& g) {
    p.n_src = g.n_src; p.Cs0 = g.Cs[0]; p.Cs1 = g.Cs[1]; p.taps = g.taps; p.N = g.N; p.a_bmod = g.a_bmod; p.BB = g.BB; p.T = g.T;
    p.flags = g.flags; p.B = g.B; p.film_H = g.film_H; p.c_clamp = g.c_clamp; p.resid_clamp = g.resid_clamp; p.rope_H = g.rope_H;
    p.film_bstride = g.film_bstride; p.gate_bstride = g.gate_bstride;
    p.bias = g.bias; p.mask = g.mask; p.film = g.film; p.gate = g.gate; p.resid = g.resid; p.rope_cs = g.rope_cs;
    p.mode = epilogue_mode(g);
    p.out_f32 = g.out_f32; p.out_hi = g.out_hi; p.out_lo = g.out_lo;
    p.out16 = g.out16; p.u16 = g.u16;
    p.ln_mask_out = g.ln_mask_out;
    p.ln_shift = g.ln_shift; p.ln_scale = g.ln_scale; p.film2 = g.film2;
    p.out2_f32 = g.out2_f32; p.u_hi = g.u_hi; p.u_lo = g.u_lo;
    p.ada_bstride = g.ada_bstride; p.film2_bstride = g.film2_bstride;
    p.ksplit = 1; p.split_bb = g.BB;
    static int tap_outer = -1;
    if (tap_outer < 0) { const char* e = getenv("STABLETTS_B200_TAP_OUTER"); tap_outer = (e && e[0] == '1') ? 1 : 0; }
    p.tap_outer = tap_outer;
}

// softmax scale folded into q: 1/sqrt(64) * log2(e) (attention runs in the exp2 domain)
constexpr float kQScale = 0.125f * 1.4426950408889634f;

namespace epi {

__device__ __forceinline__ float2 ld2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// a column pair leaves as split-bf16 words in two planes, or as one saturated fp16 word
__device__ __forceinline__ void store_planes(bf16* hi, bf16* lo, int f16, long o, float a, float b) {
    if (f16) {
        *reinterpret_cast<uint32_t*>(hi + o) = pack_f16x2_sat(a, b);
    } else {
        uint32_t h, l;
        split_bf16x2(a, b, h, l);
        *reinterpret_cast<uint32_t*>(hi + o) = h;
        *reinterpret_cast<uint32_t*>(lo + o) = l;
    }
}

}  // namespace epi

// Drains one finished accumulator: this warpgroup's 64 frames (first frame t0) x BN channels (first channel n0) of batch
// row bb.  acc[128h + 4j + 2r + e] (BN = 256: two 128-column halves h) is row 16w + l / 4 + 8r, column 128h + 8j + 2(l % 4) + e.
template <int BN, int MODE>
__device__ __forceinline__ void epilogue_tile(const TcParams& p, int bb, int t0, int n0, float (&acc)[BN / 2]) {
    using namespace epi;
    constexpr bool ROPE = MODE == EM_ROPE, LN = MODE == EM_LN, RES = MODE == EM_RESID || MODE == EM_LN;
    constexpr int NJ = BN / 8;                         // column groups of the tile
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int cq = 2 * (lane & 3);
    const int mb = bb % p.B;
    const bool plain = ROPE || (p.flags & (EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID)) == 0;
    const bool mask_only = !ROPE && (p.flags & (EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID)) == EPI_MASK;
    const bool has_resid = RES && (p.flags & EPI_RESID);
    const float* film = p.film + (long)mb * p.film_bstride;
    const float* gate = p.gate + (long)min(bb, p.c_clamp) * p.gate_bstride;
    const float* film2 = p.film2 + (long)mb * p.film2_bstride;

#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int t = t0 + 16 * w + (lane >> 2) + 8 * r;
        const bool row_ok = t < p.T;
        const int tcl = min(t, p.T - 1);               // clamped for the loads; stores are guarded
        const float mrow = (!ROPE && p.mask) ? __ldg(p.mask + (long)mb * p.T + tcl) : 1.f;
        const float m = (p.flags & EPI_MASK) ? mrow : 1.f;
        const long orow = ((long)bb * p.T + tcl) * p.N;
        const float* resid_row = p.resid + ((long)min(bb, p.resid_clamp) * p.T + tcl) * p.N;
        const float* cs = p.rope_cs + (long)tcl * 32;
        float s1 = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int i = (j / 16) * 64 + (j % 16) * 4 + 2 * r;      // accumulator index of this pair
            const int n = n0 + 8 * j + cq;
            const bool ok = row_ok && n < p.N;
            const int nc = min(n, p.N - 2);
            float x0 = acc[i], x1 = acc[i + 1];
            if (p.flags & EPI_BIAS) { const float2 b = ld2(p.bias + nc); x0 += b.x; x1 += b.y; }
            if constexpr (ROPE) {
                // partial RoPE on the first 32 dims of every 64-wide head of q and k (columns [0, 2H)): pairs (c, c + 16),
                // theta index c (models/diffusion_transformer.py:173-198); the partner pair sits two column groups further
                // in the same thread and is rotated together with this one.  q additionally carries the softmax scale.
                if (n < 2 * p.rope_H && (n & 63) < 16) {
                    const int i2 = ((j + 2) / 16) * 64 + ((j + 2) % 16) * 4 + 2 * r;
                    float y0 = acc[i2], y1 = acc[i2 + 1];
                    if (p.flags & EPI_BIAS) { const float2 b = ld2(p.bias + min(n + 16, p.N - 2)); y0 += b.x; y1 += b.y; }
                    const float4 c4 = __ldg(reinterpret_cast<const float4*>(cs + 2 * (n & 63)));     // (cos, sin) of c, c + 1
                    acc[i] = x0 * c4.x - y0 * c4.y; acc[i + 1] = x1 * c4.z - y1 * c4.w;
                    acc[i2] = y0 * c4.x + x0 * c4.y; acc[i2 + 1] = y1 * c4.z + x1 * c4.w;
                    x0 = acc[i]; x1 = acc[i + 1];
                } else if (n < 2 * p.rope_H && (n & 63) < 32) {
                    x0 = acc[i]; x1 = acc[i + 1];      // rotated (bias included) with its partner above
                }
                if (n < p.rope_H) { x0 *= kQScale; x1 *= kQScale; }
            } else {
                if constexpr (MODE == EM_SILU) { x0 = silu_fast(x0); x1 = silu_fast(x1); }
                if constexpr (MODE == EM_GELU) { x0 = gelu_f(x0); x1 = gelu_f(x1); }
                if (mask_only) {                       // (h * mask): the FFN hidden activation, cond features
                    x0 *= m; x1 *= m;
                } else if (!plain) {
                    if (p.flags & EPI_FILM) {          // x = gamma * x + beta
                        const float2 fg = ld2(film + nc), fb = ld2(film + p.film_H + nc);
                        x0 = fmaf(fg.x, x0, fb.x); x1 = fmaf(fg.y, x1, fb.y);
                    }
                    float g0 = m, g1 = m;              // gate * mask
                    if (p.flags & EPI_GATE) { const float2 g2 = ld2(gate + nc); g0 *= g2.x; g1 *= g2.y; }
                    if constexpr (RES) {
                        float2 rr = make_float2(0.f, 0.f);
                        if (has_resid) rr = ld2(resid_row + nc);
                        x0 = fmaf(x0, g0, rr.x); x1 = fmaf(x1, g1, rr.y);
                    } else {
                        x0 *= g0; x1 *= g1;
                    }
                }
            }
            if (ok) {
                if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + orow + n) = make_float2(x0, x1);
                if (p.out_hi) store_planes(p.out_hi, p.out_lo, p.out16, orow + n, x0, x1);
            }
            if constexpr (LN) {
                if (p.film2) {                         // the next block's FiLM·mask on the finished residual stream
                    const float2 fg = ld2(film2 + nc), fb = ld2(film2 + p.film_H + nc);
                    x0 = (fg.x * x0 + fb.x) * mrow; x1 = (fg.y * x1 + fb.y) * mrow;
                    if (ok) *reinterpret_cast<float2*>(p.out2_f32 + orow + n) = make_float2(x0, x1);
                }
                acc[i] = x0; acc[i + 1] = x1;          // the row stays in registers for the normalisation
                s1 += x0 + x1;
            }
        }
        if constexpr (LN) {
            // LayerNorm(C = N = BN, no affine, eps 1e-5) over the row held by the four lanes of this quad (two-pass:
            // mean, then centred squares), adaLN modulate [+ FFN input mask] -> the next GEMM's operand planes
            s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
            const float mean = s1 * (1.0f / (float)BN);
            float s2 = 0.f;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int i = (j / 16) * 64 + (j % 16) * 4 + 2 * r;
                const float d0 = acc[i] - mean, d1 = acc[i + 1] - mean;
                s2 = fmaf(d0, d0, s2); s2 = fmaf(d1, d1, s2);
            }
            s2 += __shfl_xor_sync(0xffffffffu, s2, 1); s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
            const float rstd = rsqrtf(s2 * (1.0f / (float)BN) + 1e-5f);
            const float mo = p.ln_mask_out ? mrow : 1.0f;
            const float* sh = p.ln_shift + (long)min(bb, p.c_clamp) * p.ada_bstride;
            const float* sc = p.ln_scale + (long)min(bb, p.c_clamp) * p.ada_bstride;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int i = (j / 16) * 64 + (j % 16) * 4 + 2 * r;
                const int n = 8 * j + cq;
                const float2 s4 = ld2(sh + n), c4 = ld2(sc + n);
                const float u0 = ((acc[i] - mean) * rstd * (1.f + c4.x) + s4.x) * mo;
                const float u1 = ((acc[i + 1] - mean) * rstd * (1.f + c4.y) + s4.y) * mo;
                if (row_ok) store_planes(p.u_hi, p.u_lo, p.u16, orow + n, u0, u1);
            }
        }
    }
}

}  // namespace st
