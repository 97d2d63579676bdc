// Fused conv-GEMM epilogue of the wgmma kernel (gemm_tc.cu), run on the accumulator registers.
//
// A consumer warpgroup owns 64 frames x BN channels.  In the wgmma accumulator layout thread (warp w, lane l) holds, for
// every 8-column group j, the column pair 8j + 2(l % 4) + {0, 1} of rows 16w + l / 4 and 16w + l / 4 + 8, so
//   * all math runs on registers — bias / SiLU / GELU / FiLM / mask / gate / residual, and the partial RoPE of the QKV
//     projection (the rotation partners c, c + 16 of a head live in the same thread);
//   * per-column vectors and residual rows are read as 8-byte pairs, results leave as 8-byte fp32 pairs and / or packed
//     split-bf16 (or fp16) words; the four lanes of a row cover one 32-byte sector per column group;
//   * on 256-channel tiles the per-column vectors (bias, FiLM, gate, film2, adaLN shift / scale) are staged in shared
//     memory once per tile (EpiVec) instead of being re-read from global memory for every column group of both rows;
//   * residual pairs are loaded several column groups ahead of their use, so their HBM round trips overlap;
//   * when the tile spans all N = BN channels a row lives in the four lanes of one quad, so the LayerNorm + adaLN-modulate
//     that follows O / conv_2 / the long-skip conv / in_proj in the reference (models/diffusion_transformer.py:111-112,
//     119-121) is fused: the finished row stays in the accumulator registers, mean and variance are two quad reductions,
//     and the split-bf16 operand of the next GEMM is emitted directly — no separate LayerNorm kernel, no HBM round trip.
// One code instance per mode (plain / SiLU / GELU / Mish / RoPE / residual / LayerNorm-fused); a launch executes exactly one.
#pragma once
#include "common.cuh"
#include <type_traits>
#include "tc_ptx.cuh"

namespace st {

enum : int { EM_PLAIN = 0, EM_SILU = 1, EM_GELU = 2, EM_ROPE = 3, EM_LN = 4, EM_RESID = 5,   // EM_RESID: plain + residual rows
             EM_SILU_OUT = 6,     // EM_RESID whose split planes / out2_f32 receive silu(v) (EPI_SILU_OUT)
             EM_MISH = 7 };       // EM_PLAIN with Mish after the bias (128-channel tiles only)

struct TcParams {
    int n_src, Cs0, Cs1, taps, dil, N, a_bmod, BB, T;
    int m_tiles_per_b, n_tiles, total_tiles;
    int flags, B, film_H, c_clamp, resid_clamp, rope_H;
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
    if (g.flags & EPI_SILU_OUT) return EM_SILU_OUT;
    if (g.flags & EPI_SILU) return EM_SILU;
    if (g.flags & EPI_GELU) return EM_GELU;
    if (g.flags & EPI_MISH) return EM_MISH;
    if (g.flags & EPI_RESID) return EM_RESID;
    return EM_PLAIN;
}

inline void fill_tc_params(TcParams& p, const GemmArgs& g) {
    p.n_src = g.n_src; p.Cs0 = g.Cs[0]; p.Cs1 = g.Cs[1]; p.taps = g.taps; p.dil = g.dil; p.N = g.N; p.a_bmod = g.a_bmod; p.BB = g.BB; p.T = g.T;
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
}

// softmax scale folded into q: 1/sqrt(64) * log2(e) (attention runs in the exp2 domain)
constexpr float kQScale = 0.125f * 1.4426950408889634f;

namespace epi {

__device__ __forceinline__ float2 ld2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// the same load when `on` (else 0), kept where it is issued: the compiler sinks a plain read-only load next to its first
// use.  One predicated instruction and no branch, so no copy at a branch join waits on the loaded value before its use
__device__ __forceinline__ float2 ld2_ahead(const float* p, bool on) {
    float2 v;
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\tmov.f32 %0, 0f00000000;\n\tmov.f32 %1, 0f00000000;\n\t"
                 "@q ld.global.nc.v2.f32 {%0, %1}, [%2];\n\t}"
                 : "=f"(v.x), "=f"(v.y) : "l"(p), "r"((int)on));
    return v;
}

// ld2_ahead as a coherent load, for the ring of epilogue_wide: ptxas may hoist a read-only (.nc) load above the
// warpgroup barrier and ahead of the stores it could alias, which collapses the ring into one burst per row; a coherent
// load stays where it is written, RD column groups ahead of its use
__device__ __forceinline__ float2 ld2_ring(const float* p, bool on, float fill) {
    float2 v;
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\tmov.f32 %0, %4;\n\tmov.f32 %1, %4;\n\t"
                 "@q ld.global.v2.f32 {%0, %1}, [%2];\n\t}"
                 : "=f"(v.x), "=f"(v.y) : "l"(p), "r"((int)on), "f"(fill));
    return v;
}

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

// shared-memory load that the compiler neither merges across rows nor moves across the (volatile) barriers
__device__ __forceinline__ float2 lds2(uint32_t a) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a));
    return v;
}

// the same as a volatile load, which ptxas keeps where it is as well: the LayerNorm modulate loop reads the same 64 pairs
// for both rows, and with plain loads ptxas keeps them in registers across rows, spilling 408 bytes beside the accumulators
__device__ __forceinline__ float2 lds2_volatile(uint32_t a) {
    float2 v;
    asm volatile("ld.volatile.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a));
    return v;
}

__device__ __forceinline__ void named_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// row base pointer base + off elements, formed by an opaque add once per row: the compiler then neither keeps row 0's
// pointers live into row 1 (beside the accumulators they would spill) nor re-derives them per column group, so every
// access of the row is [base + immediate].  A null base stays unused: every access through it is predicated off
template <typename T>
__device__ __forceinline__ T* row_ptr(T* base, long off) {
    T* r;
    asm volatile("add.s64 %0, %1, %2;" : "=l"(r) : "l"(base), "l"(off * (long)sizeof(T)));
    return r;
}

// global stores under a predicate the caller evaluates once per row: one instruction each, no branch
__device__ __forceinline__ void st2_if(float* a, float x, float y, bool on) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\t@q st.global.v2.f32 [%0], {%1, %2};\n\t}"
                 ::"l"(a), "f"(x), "f"(y), "r"((int)on));
}
__device__ __forceinline__ void st1_if(bf16* a, uint32_t v, bool on) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q st.global.b32 [%0], %1;\n\t}" ::"l"(a), "r"(v), "r"((int)on));
}
__device__ __forceinline__ void st2w_if(bf16* a, uint32_t v0, uint32_t v1, bool on) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\t@q st.global.v2.b32 [%0], {%1, %2};\n\t}"
                 ::"l"(a), "r"(v0), "r"(v1), "r"((int)on));
}

}  // namespace epi

// Per-column vectors of a 256-channel tile in shared memory, one copy per consumer warpgroup: EV_COUNT rows of BN fp32.
// Measured on H100 80GB HBM3: reading them from global memory in every column group is what the epilogue of these tiles
// waited on most (DESIGN.md §5).  The adaLN shift / scale of the fused LayerNorm are per-column vectors too.
enum : int { EV_BIAS = 0, EV_FILM_G, EV_FILM_B, EV_GATE, EV_FILM2_G, EV_FILM2_B, EV_LN_SHIFT, EV_LN_SCALE, EV_COUNT };
constexpr int EPI_VEC_BYTES = EV_COUNT * 256 * 4;

// Stages the vectors of one tile (batch row bb, first channel n0) into the warpgroup's copy at shared address `vs`: each of
// the 128 threads loads one column pair of every vector the epilogue reads, all loads in flight at once.  Called by the
// whole warpgroup at tile start, before the main loop; the barrier orders it after the previous tile's epilogue reads.
template <int BN, int MODE>
__device__ __forceinline__ void stage_epi_vectors(const TcParams& p, int bb, int n0, uint32_t vs, int bar_id) {
    static_assert(BN == 256 && MODE != EM_ROPE, "one column pair per thread of the warpgroup (RoPE: stage_rope_bias)");
    epi::named_bar_sync(bar_id);
    const int c = 2 * (threadIdx.x & 127);
    const int mb = bb % p.B, cb = min(bb, p.c_clamp);
    auto put = [&](int v, const float* src) {
        const float2 x = epi::ld2(src + c);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(vs + (v * BN + c) * 4), "f"(x.x), "f"(x.y) : "memory");
    };
    if (p.flags & EPI_BIAS) put(EV_BIAS, p.bias + n0);
    if (p.flags & EPI_FILM) {
        const float* film = p.film + (long)mb * p.film_bstride + n0;
        put(EV_FILM_G, film); put(EV_FILM_B, film + p.film_H);
    }
    if (p.flags & EPI_GATE) put(EV_GATE, p.gate + (long)cb * p.gate_bstride + n0);
    if (MODE == EM_LN) {                   // (N = BN: n0 = 0)
        const long ab = (long)cb * p.ada_bstride;
        put(EV_LN_SHIFT, p.ln_shift + ab); put(EV_LN_SCALE, p.ln_scale + ab);
        if (p.film2) {
            const float* film2 = p.film2 + (long)mb * p.film2_bstride;
            put(EV_FILM2_G, film2); put(EV_FILM2_B, film2 + p.film_H);
        }
    }
}

// epilogue_tile of a 256-channel tile, as straight-line code.  The epilogue is time in which the SM's tensor cores idle
// (DESIGN.md §5) and it issues from 8 warps per SM, so what counts is the instructions each column group issues:
//   * no bounds work on columns: 256-channel tiles run for N % 256 == 0 only (launch_bn<256> refuses anything else), so
//     every column of the tile exists.  Rows keep their guard, one predicate per row;
//   * every plane a row reads or writes has one base pointer per row, and each column group accesses [base + immediate];
//   * kernel-uniform choices (flags, output planes, film2) are predicates evaluated once per tile or row; the column loop
//     runs predicated instructions, and branches only per row (the format of the 2-byte planes, where the row loop holds
//     no residual loads).
// The floating-point operations and their order are those of epilogue_narrow.  (The QKV projection's RoPE epilogue runs
// on 128-channel half-tiles: epilogue_rope_half.)
template <int MODE>
__device__ __forceinline__ void epilogue_wide(const TcParams& p, int bb, int t0, int n0, float (&acc)[128], uint32_t vs,
                                              int bar_id) {
    using namespace epi;
    static_assert(MODE != EM_ROPE, "RoPE: epilogue_rope_half");
    constexpr int BN = 256, NJ = BN / 8;               // column groups of the tile
    named_bar_sync(bar_id);                            // the tile's vectors are staged
    constexpr bool LN = MODE == EM_LN, SO = MODE == EM_SILU_OUT;
    constexpr bool RES = MODE == EM_RESID || MODE == EM_LN || SO;
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int cq = 2 * (lane & 3);
    const int mb = bb % p.B;
    const int f = p.flags;
    const bool bias = f & EPI_BIAS, film = f & EPI_FILM, gate = f & EPI_GATE;
    const bool plain = (f & (EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID)) == 0;
    const bool has_resid = RES && (f & EPI_RESID);
    // RES: every flag combination runs x = fma(x, gate * mask, residual), so that the residual loads exist once.  Without a
    // residual it adds 0, as epilogue_narrow does; -0 where epilogue_narrow computes x (plain) or x * mask (mask only):
    // fma(x, 1, -0) = x and fma(x, m, -0) = x * m bit for bit, which +0 is not for a product of -0
    const float rfill = plain || (f & (EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID)) == EPI_MASK ? -0.f : 0.f;
    const bool f16 = p.out16 != 0, has_film2 = LN && p.film2;
    // once per tile: tested per row, ptxas may sink this pointer test into row 1's column chains
    const bool has_2 = p.out2_f32 && (SO || has_film2);
    // Residual pairs are loaded RD column groups ahead of their use, through a ring of RD register pairs per row.  Loaded
    // where they are used, each one was waited on alone, one HBM round trip per column group.  Reading ahead is safe when
    // the residual is the fp32 output itself: each (row, column) pair is read, and then written, by this thread only.  The
    // ring restarts per row: carried into row 1, it stays live across row 0's LayerNorm passes, which then spill 184 bytes.
    // RD = 4 and 16 measured no faster than 8 (DESIGN.md §5); tests/test_gemm_epilogue_sass.py checks the distance.
    constexpr int RD = 8;
    enum : int { FMT_ANY, FMT_F16, FMT_SPLIT };        // 2-byte planes: either format (predicated), or one of them

#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int t = t0 + 16 * w + (lane >> 2) + 8 * r;
        const bool row_ok = t < p.T;
        const int tcl = min(t, p.T - 1);               // clamped for the loads; stores are guarded
        const float mrow = p.mask ? __ldg(p.mask + (long)mb * p.T + tcl) : 1.f;
        const float m = (f & EPI_MASK) ? mrow : 1.f;
        const long orow = ((long)bb * p.T + tcl) * p.N + n0 + cq;
        const bool st_f32 = row_ok && p.out_f32, st_f16 = row_ok && p.out_hi && f16, st_split = row_ok && p.out_hi && !f16;
        const bool st_2 = row_ok && has_2;
        float* const of = row_ptr(p.out_f32, orow);
        float* const o2 = SO || LN ? row_ptr(p.out2_f32, orow) : nullptr;
        bf16* const oh = row_ptr(p.out_hi, orow);
        bf16* const ol = row_ptr(p.out_lo, orow);
        const float* const rs = RES ? row_ptr(p.resid, ((long)min(bb, p.resid_clamp) * p.T + tcl) * p.N + n0 + cq) : nullptr;
        uint32_t vsr;
        asm volatile("mov.b32 %0, %1;" : "=r"(vsr) : "r"(vs + cq * 4));
        auto vec = [&](int v, int j) { return lds2(vsr + (v * BN + 8 * j) * 4); };     // column pair of group j
        float s1 = 0.f;

        auto row = [&](auto fmt) {
            float2 ring[RD];
            if constexpr (RES) {
#pragma unroll
                for (int j = 0; j < RD; ++j) ring[j] = ld2_ring(rs + 8 * j, has_resid, rfill);
            }
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int i = (j / 16) * 64 + (j % 16) * 4 + 2 * r;  // accumulator index of this pair
                float2 rr;
                if constexpr (RES) {
                    rr = ring[j % RD];
                    if (j + RD < NJ) ring[j % RD] = ld2_ring(rs + 8 * (j + RD), has_resid, rfill);
                }
                // in place on acc (dead after the epilogue): a predicated instruction then needs no copy beside it
                float &a0 = acc[i], &a1 = acc[i + 1];
                if (bias) { const float2 b = vec(EV_BIAS, j); a0 += b.x; a1 += b.y; }
                if constexpr (MODE == EM_SILU) { a0 = silu_fast(a0); a1 = silu_fast(a1); }
                if constexpr (MODE == EM_GELU) { a0 = gelu_f(a0); a1 = gelu_f(a1); }
                // (plain: no FiLM, no gate; mask only: g = m)
                if (film) {
                    const float2 fg = vec(EV_FILM_G, j), fb = vec(EV_FILM_B, j);
                    a0 = fmaf(fg.x, a0, fb.x); a1 = fmaf(fg.y, a1, fb.y);
                }
                float g0 = m, g1 = m;
                if (gate) { const float2 g2 = vec(EV_GATE, j); g0 *= g2.x; g1 *= g2.y; }
                if constexpr (RES) {
                    a0 = fmaf(a0, g0, rr.x); a1 = fmaf(a1, g1, rr.y);
                } else if (!plain) {
                    a0 *= g0; a1 *= g1;
                }
                float x0 = a0, x1 = a1;
                st2_if(of + 8 * j, x0, x1, st_f32);
                float h0 = x0, h1 = x1;                // what the 2-byte planes receive
                if constexpr (SO) { h0 = silu_fast(x0); h1 = silu_fast(x1); st2_if(o2 + 8 * j, h0, h1, st_2); }
                if constexpr (decltype(fmt)::value != FMT_SPLIT) st1_if(oh + 8 * j, pack_f16x2_sat(h0, h1), st_f16);
                if constexpr (decltype(fmt)::value != FMT_F16) {
                    uint32_t hw, lw;
                    split_bf16x2(h0, h1, hw, lw);
                    st1_if(oh + 8 * j, hw, st_split); st1_if(ol + 8 * j, lw, st_split);
                }
                if constexpr (LN) {
                    if (has_film2) {                   // the next block's FiLM·mask on the finished residual stream
                        const float2 fg = vec(EV_FILM2_G, j), fb = vec(EV_FILM2_B, j);
                        x0 = (fg.x * x0 + fb.x) * mrow; x1 = (fg.y * x1 + fb.y) * mrow;
                    }
                    st2_if(o2 + 8 * j, x0, x1, st_2);
                    acc[i] = x0; acc[i + 1] = x1;      // the row stays in registers for the normalisation
                    s1 += x0 + x1;
                }
            }
        };
        if constexpr (RES) {
            row(std::integral_constant<int, FMT_ANY>());
        } else if (f16) {
            row(std::integral_constant<int, FMT_F16>());
        } else {
            row(std::integral_constant<int, FMT_SPLIT>());
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
            bf16* const uh = row_ptr(p.u_hi, orow);
            bf16* const ul = row_ptr(p.u_lo, orow);
            auto u_pair = [&](int j, float& u0, float& u1) {
                const int i = (j / 16) * 64 + (j % 16) * 4 + 2 * r;
                const float2 s4 = lds2_volatile(vsr + (EV_LN_SHIFT * BN + 8 * j) * 4);
                const float2 c4 = lds2_volatile(vsr + (EV_LN_SCALE * BN + 8 * j) * 4);
                u0 = ((acc[i] - mean) * rstd * (1.f + c4.x) + s4.x) * mo;
                u1 = ((acc[i + 1] - mean) * rstd * (1.f + c4.y) + s4.y) * mo;
            };
            if (p.u16) {                               // one branch per row: fp16 u (O), split bf16 u (conv_2)
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    float u0, u1;
                    u_pair(j, u0, u1);
                    st1_if(uh + 8 * j, pack_f16x2_sat(u0, u1), row_ok);
                }
            } else {
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    float u0, u1;
                    uint32_t hw, lw;
                    u_pair(j, u0, u1);
                    split_bf16x2(u0, u1, hw, lw);
                    st1_if(uh + 8 * j, hw, row_ok); st1_if(ul + 8 * j, lw, row_ok);
                }
            }
        }
    }
}

// The bias of the QKV projection's 128-channel half-tile (first channel n0) into the warpgroup's 512-byte copy at shared
// address vs, one column per thread.  Called by the whole warpgroup before the main loop; the barrier orders it after the
// previous half-tile's epilogue reads.
__device__ __forceinline__ void stage_rope_bias(const TcParams& p, int n0, uint32_t vs, int bar_id) {
    epi::named_bar_sync(bar_id);
    if (p.flags & EPI_BIAS) {
        const int c = threadIdx.x & 127;
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(vs + 4 * c), "f"(__ldg(p.bias + n0 + c)) : "memory");
    }
}

// Epilogue of the QKV projection's 128 x 128 half-tile (gemm_wgmma_kernel<256, EM_ROPE, 0>): the warpgroup holds all 128
// frames (first frame t0) x 128 channels (first channel n0) of batch row bb as two m64n128 accumulators, acc[64 rh + 4j +
// 2r + e] = row 64 rh + 16w + l / 4 + 8r, column 8j + 2(l % 4) + e; the bias comes from the copy stage_rope_bias made.
// Straight-line as epilogue_wide is: one base pointer per row and plane, predicated stores, no bounds work on columns
// (N % 256 == 0), and kernel-uniform choices per 64-column head: rotation (columns < 2 rope_H) and q scale (columns <
// rope_H) hold for whole heads, as rope_H is a multiple of 64 (launch_bn<256> checks it).  The two 64-row halves run as one
// loop body: after the first, the second accumulator moves down into acc[0, 64).  The floating-point operations and
// their order are those of epilogue_narrow.
// The 2-byte planes leave in whole 32-byte sectors: the two lanes of a pair (l, l ^ 1) swap words across column groups
// j, j + 1, so that the even lane stores 4 columns of group j and the odd lane 4 of group j + 1, and the four lanes of a
// row write 32 contiguous bytes per instruction.  Stored as one 4-byte word per lane and group, each row wrote half
// sectors, and with only one warpgroup draining at a time this epilogue, not the MMAs, set the pace (DESIGN.md §5).
__device__ __forceinline__ void epilogue_rope_half(const TcParams& p, int bb, int t0, int n0, float (&acc)[128], uint32_t vs,
                                                   int bar_id) {
    using namespace epi;
    constexpr int NJ = 128 / 8;                        // column groups of the half-tile
    named_bar_sync(bar_id);                            // the half-tile's bias is staged
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int cq = 2 * (lane & 3);
    const bool odd = lane & 1;                         // stores the column group j + 1 of each pair (j, j + 1)
    const bool bias = p.flags & EPI_BIAS, f16 = p.out16 != 0;
    const int rope_rot = 2 * p.rope_H - n0, rope_q = p.rope_H - n0;   // head hh starts at column n0 + 64 hh
    enum : int { FMT_F16, FMT_SPLIT };

#pragma unroll 1
    for (int rh = 0; rh < 2; ++rh) {
        // both rows' clamps ahead of the first row's stores (opaque moves keep them there): ptxas otherwise schedules row
        // 1's clamp amid row 0's column chains
        int tcl2[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int tc = min(t0 + 64 * rh + 16 * w + (lane >> 2) + 8 * r, p.T - 1);
            asm volatile("mov.b32 %0, %1;" : "=r"(tcl2[r]) : "r"(tc));
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int t = t0 + 64 * rh + 16 * w + (lane >> 2) + 8 * r;
            const bool row_ok = t < p.T;
            const int tcl = tcl2[r];                   // clamped for the loads; stores are guarded
            const long orow = ((long)bb * p.T + tcl) * p.N + n0 + cq;
            const float* cs = p.rope_cs + (long)tcl * 32;
            const float4 cs4[2] = {__ldg(reinterpret_cast<const float4*>(cs + 2 * cq)),
                                   __ldg(reinterpret_cast<const float4*>(cs + 2 * (8 + cq)))};
            const bool st_f32 = row_ok && p.out_f32, st_f16 = row_ok && p.out_hi && f16, st_split = row_ok && p.out_hi && !f16;
            float* const of = row_ptr(p.out_f32, orow);
            // 2-byte planes: the even lane's 4 columns of group j start at column cq of the group, the odd lane's 4 of group
            // j + 1 at column cq - 2 of that group, 8 + cq - 2 = cq + 6 columns after group j
            bf16* const oh = row_ptr(p.out_hi, orow + (odd ? 6 : 0));
            bf16* const ol = row_ptr(p.out_lo, orow + (odd ? 6 : 0));
            uint32_t vsr;
            asm volatile("mov.b32 %0, %1;" : "=r"(vsr) : "r"(vs + cq * 4));
            auto vec = [&](int j) { return lds2(vsr + 8 * j * 4); };      // bias pair of column group j
            // words w0 (group j) and w1 (group j + 1) of this lane -> 8 bytes at [o + 8j]: the even lane keeps w0 and takes
            // its partner's w0 (columns cq + 2, cq + 3 of group j), the odd lane takes its partner's w1 and keeps its own
            auto st_pair = [&](bf16* o, int j, uint32_t w0, uint32_t w1, bool on) {
                const uint32_t got = __shfl_xor_sync(0xffffffffu, odd ? w0 : w1, 1);
                st2w_if(o + 8 * j, odd ? got : w0, odd ? w1 : got, on);
            };

            auto row = [&](auto fmt) {
                uint32_t wh = 0, wl = 0;               // the words of the even group j of the current pair
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    const int i = 4 * j + 2 * r;       // accumulator index of this pair
                    const int jj = j % 8, hh = j / 8;
                    const bool rot = 64 * hh < rope_rot;
                    if (jj == 0 && rot) {
                        // one branch per head: the pairs (c, c + 16) of groups 8 hh + {0, 1} and 8 hh + {2, 3} sit in the
                        // same thread and are rotated together, bias included; their groups then store what is left in acc
#pragma unroll
                        for (int k = 0; k < 2; ++k) {
                            const int ia = 4 * (j + k) + 2 * r, i2 = 4 * (j + k + 2) + 2 * r;
                            float u0 = acc[ia], u1 = acc[ia + 1], y0 = acc[i2], y1 = acc[i2 + 1];
                            if (bias) { const float2 b = vec(j + k); u0 += b.x; u1 += b.y; }
                            if (bias) { const float2 b = vec(j + k + 2); y0 += b.x; y1 += b.y; }
                            const float4 c4 = cs4[k];  // (cos, sin) of c, c + 1
                            acc[ia] = u0 * c4.x - y0 * c4.y; acc[ia + 1] = u1 * c4.z - y1 * c4.w;
                            acc[i2] = y0 * c4.x + u0 * c4.y; acc[i2 + 1] = y1 * c4.z + u1 * c4.w;
                        }
                    }
                    float x0 = acc[i], x1 = acc[i + 1];
                    if (bias && !(jj < 4 && rot)) { const float2 b = vec(j); x0 += b.x; x1 += b.y; }
                    if (64 * hh < rope_q) { x0 *= kQScale; x1 *= kQScale; }
                    st2_if(of + 8 * j, x0, x1, st_f32);
                    uint32_t hw, lw = 0;
                    if constexpr (decltype(fmt)::value == FMT_F16) {
                        hw = pack_f16x2_sat(x0, x1);
                    } else {
                        split_bf16x2(x0, x1, hw, lw);
                    }
                    if (j % 2 == 0) {
                        wh = hw; wl = lw;
                    } else if constexpr (decltype(fmt)::value == FMT_F16) {
                        st_pair(oh, j - 1, wh, hw, st_f16);
                    } else {
                        st_pair(oh, j - 1, wh, hw, st_split); st_pair(ol, j - 1, wl, lw, st_split);
                    }
                }
            };
            if (f16) {                                 // one branch per row: the format of the 2-byte planes
                row(std::integral_constant<int, FMT_F16>());
            } else {
                row(std::integral_constant<int, FMT_SPLIT>());
            }
        }
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = acc[64 + i];     // the second row half, for the second pass
    }
}

// Drains one finished accumulator of a tile of at most 128 channels: this warpgroup's 64 frames (first frame t0) x BN
// channels (first channel n0) of batch row bb.  acc[4j + 2r + e] is row 16w + l / 4 + 8r, column 8j + 2(l % 4) + e.
template <int BN, int MODE>
__device__ __forceinline__ void epilogue_narrow(const TcParams& p, int bb, int t0, int n0, float (&acc)[BN / 2]) {
    using namespace epi;
    constexpr bool ROPE = MODE == EM_ROPE, SO = MODE == EM_SILU_OUT;
    constexpr bool RES = MODE == EM_RESID || SO;
    static_assert(BN <= 128 && MODE != EM_LN, "the fused LayerNorm runs on full-row 256-channel tiles (epilogue_wide)");
    constexpr int NJ = BN / 8;                         // column groups of the tile
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int cq = 2 * (lane & 3);
    const int mb = bb % p.B;
    const bool plain = ROPE || (p.flags & (EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID)) == 0;
    const bool mask_only = !ROPE && (p.flags & (EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID)) == EPI_MASK;
    const bool has_resid = RES && (p.flags & EPI_RESID);
    const float* film = p.film + (long)mb * p.film_bstride;
    const float* gate = p.gate + (long)min(bb, p.c_clamp) * p.gate_bstride;

    constexpr int RD = 8;                              // residual pairs loaded ahead: see epilogue_wide

#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int t = t0 + 16 * w + (lane >> 2) + 8 * r;
        const bool row_ok = t < p.T;
        const int tcl = min(t, p.T - 1);               // clamped for the loads; stores are guarded
        const float mrow = (!ROPE && p.mask) ? __ldg(p.mask + (long)mb * p.T + tcl) : 1.f;
        const float m = (p.flags & EPI_MASK) ? mrow : 1.f;
        const long orow = ((long)bb * p.T + tcl) * p.N;
        // RoPE: n0 is a multiple of 64, so the rotated pairs of every head are those of column groups j % 8 = 0, 1 and read
        // the same two (cos, sin) float4 of the row: (c, c + 1) for c = cq and c = 8 + cq
        float4 cs4[2];
        if constexpr (ROPE) {
            const float* cs = p.rope_cs + (long)tcl * 32;
            cs4[0] = __ldg(reinterpret_cast<const float4*>(cs + 2 * cq));
            cs4[1] = __ldg(reinterpret_cast<const float4*>(cs + 2 * (8 + cq)));
        }
        // the column base passes through an opaque move once per row: otherwise the compiler keeps the column-derived values
        // of row r = 0 (32 column groups) live into row r = 1 instead of recomputing them, and beside the accumulators they
        // spill to local memory, whose round trips miss the small L1 left beside the 160-192 KB of pipeline stages.  This
        // steers a compiler decision (checked with CUDA 12.9); tests/test_gemm_spills.py fails if the spills come back
        int n0r;
        asm volatile("mov.b32 %0, %1;" : "=r"(n0r) : "r"(n0));
        const float* resid_row = p.resid + ((long)min(bb, p.resid_clamp) * p.T + tcl) * p.N;
        auto resid_pair = [&](int j) { return ld2_ahead(resid_row + min(n0r + 8 * j + cq, p.N - 2), has_resid); };
        float2 ring[RD];
        if constexpr (RES) {
#pragma unroll
            for (int j = 0; j < RD; ++j) ring[j] = resid_pair(j);
        }
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int i = (j / 16) * 64 + (j % 16) * 4 + 2 * r;      // accumulator index of this pair
            const int n = n0r + 8 * j + cq;
            const bool ok = row_ok && n < p.N;
            const int nc = min(n, p.N - 2);
            float x0 = acc[i], x1 = acc[i + 1];
            float2 rr;                                 // residual pair (RES), loaded RD groups ago
            if constexpr (RES) {
                rr = ring[j % RD];
                if (j + RD < NJ) ring[j % RD] = resid_pair(j + RD);
            }
            if (p.flags & EPI_BIAS) { const float2 b = ld2(p.bias + nc); x0 += b.x; x1 += b.y; }
            if constexpr (ROPE) {
                // partial RoPE on the first 32 dims of every 64-wide head of q and k (columns [0, 2H)): pairs (c, c + 16),
                // theta index c (models/diffusion_transformer.py:173-198); the partner pair sits two column groups further
                // in the same thread and is rotated together with this one.  q additionally carries the softmax scale.
                if (n < 2 * p.rope_H && j % 8 < 2) {       // (n & 63) < 16
                    const int i2 = ((j + 2) / 16) * 64 + ((j + 2) % 16) * 4 + 2 * r;
                    float y0 = acc[i2], y1 = acc[i2 + 1];
                    if (p.flags & EPI_BIAS) { const float2 b = ld2(p.bias + min(n + 16, p.N - 2)); y0 += b.x; y1 += b.y; }
                    const float4 c4 = cs4[j % 2];      // (cos, sin) of c, c + 1
                    acc[i] = x0 * c4.x - y0 * c4.y; acc[i + 1] = x1 * c4.z - y1 * c4.w;
                    acc[i2] = y0 * c4.x + x0 * c4.y; acc[i2 + 1] = y1 * c4.z + x1 * c4.w;
                    x0 = acc[i]; x1 = acc[i + 1];
                } else if (n < 2 * p.rope_H && j % 8 < 4) {    // (n & 63) < 32
                    x0 = acc[i]; x1 = acc[i + 1];      // rotated (bias included) with its partner above
                }
                if (n < p.rope_H) { x0 *= kQScale; x1 *= kQScale; }
            } else {
                if constexpr (MODE == EM_SILU) { x0 = silu_fast(x0); x1 = silu_fast(x1); }
                if constexpr (MODE == EM_GELU) { x0 = gelu_f(x0); x1 = gelu_f(x1); }
                if constexpr (MODE == EM_MISH) { x0 = mish_f(x0); x1 = mish_f(x1); }
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
                        x0 = fmaf(x0, g0, rr.x); x1 = fmaf(x1, g1, rr.y);
                    } else {
                        x0 *= g0; x1 *= g1;
                    }
                }
            }
            if (ok) {
                if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + orow + n) = make_float2(x0, x1);
                if constexpr (SO) {
                    const float s0 = silu_fast(x0), s1 = silu_fast(x1);
                    if (p.out_hi) store_planes(p.out_hi, p.out_lo, p.out16, orow + n, s0, s1);
                    if (p.out2_f32) *reinterpret_cast<float2*>(p.out2_f32 + orow + n) = make_float2(s0, s1);
                } else {
                    if (p.out_hi) store_planes(p.out_hi, p.out_lo, p.out16, orow + n, x0, x1);
                }
            }
        }
    }
}

// Drains one finished accumulator (epilogue_wide for 256-channel tiles, whose per-column vectors come from the
// warpgroup's staged copy at shared address vs, stage_epi_vectors; epilogue_narrow below that)
template <int BN, int MODE>
__device__ __forceinline__ void epilogue_tile(const TcParams& p, int bb, int t0, int n0, float (&acc)[BN / 2], uint32_t vs,
                                              int bar_id) {
    if constexpr (BN == 256) {
        epilogue_wide<MODE>(p, bb, t0, n0, acc, vs, bar_id);
    } else {
        epilogue_narrow<BN, MODE>(p, bb, t0, n0, acc);
    }
}

}  // namespace st
