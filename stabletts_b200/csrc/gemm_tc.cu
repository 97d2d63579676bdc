// wgmma / TMA conv-GEMM engine (sm_90a) — the product path for every dense contraction of the
// estimator (cond_proj, in_proj, QKV, O, conv_1, conv_2, long-skip convs, final_proj).
//
//   D[128 frames x BN channels] (fp32, registers) += A[128 x 64] (bf16, smem, K-major, SW128)
//                                                   · B[BN x 64]^T (bf16, smem, K-major, SW128)
//
// * split-bf16 ("bf16x3"): every operand travels as hi = bf16(x), lo = bf16(x - hi); each k-step
//   issues Alo·Bhi + Ahi·Blo + Ahi·Bhi into the same fp32 accumulator (~16 mantissa bits;
//   plain bf16 cannot meet the 1e-3 parity bar, SURVEY.md fact 3).
// * k-tap Conv1d = taps shifted accumulating GEMMs: the A tile of tap j is the TMA box at frame
//   coordinate t0 + j - pad of a 3-D (C, T, batch) tensor map; frames outside [0, T) are zero-filled
//   by TMA — exactly the reference's zero padding at TENSOR edges (not utterance edges).
// * the U-Net long-skip concat is never materialised: k-blocks walk two A tensor maps.
// * persistent, warp-specialised CTA (one per SM): warpgroup 0 = TMA producer (one thread, registers
//   released with setmaxnreg), warpgroups 1-2 = consumers: each issues the wgmma stream of its own 64
//   frames x BN channels and then runs the fused epilogue on its accumulator registers
//   (bias/SiLU/FiLM/mask/gate/residual[/LayerNorm] -> fp32 and/or split-bf16 global stores) while the
//   producer already fills the pipeline for the next tile.
// * tile widths: BN = 128 (three smem stages), and BN = 256 (two stages; two 128-column wgmma
//   halves per k-step) for wide outputs with enough tiles to fill the SMs — it halves the A re-reads
//   and owns whole 256-channel rows, which the fused LayerNorm and the two-pass fp16 FFN mode need;
//   narrow outputs of exactly 16, 32 or 64 channels (the FireflyGAN head's late stages) run on BN = N
//   tiles (m64nNk16, four stages) instead of padding the MMA and the B tile to 128 columns.
// * the QKV projection's 256-channel instance (RoPE, bf16x3) keeps its A rows resident and runs the two consumer
//   warpgroups on alternate 128-channel half-tiles, one draining while the other issues MMAs (rope_tiles).
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <mutex>
#include <unordered_map>
#include <string>
#include <cstring>
#include <cstdlib>

namespace st {

static_assert(ST_TEST_MODE_PLAIN == EM_PLAIN && ST_TEST_MODE_SILU == EM_SILU && ST_TEST_MODE_GELU == EM_GELU &&
              ST_TEST_MODE_ROPE == EM_ROPE && ST_TEST_MODE_LN == EM_LN && ST_TEST_MODE_RESID == EM_RESID &&
              ST_TEST_MODE_SILU_OUT == EM_SILU_OUT && ST_TEST_MODE_MISH == EM_MISH,
              "st_test_gemm_plan::mode reports the EM_* epilogue instances");

bool tmap_encode_bf16(const void* ptr, int rank, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1,
                      CUtensorMap* out);

namespace {

using namespace ptx;     // PTX wrappers shared with the attention kernel (tc_ptx.cuh)

constexpr int BLOCK_M = 128;            // two consumer warpgroups x 64 frames
constexpr int BLOCK_K = 64;             // bf16 elements = 128 bytes = one SW128 row
constexpr int WG_K = 16;
constexpr int NUM_THREADS = 384;        // warpgroup 0: TMA producer; warpgroups 1-2: wgmma + epilogue
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;     // 16 KB

struct TcMaps {
    CUtensorMap a_hi[2], a_lo[2], w_hi, w_lo;
};

// PREC = 1: the opt-in two-pass FFN precision — ONE fp16 A plane, fp16 hi / lo weight planes, two wgmmas per k-step
// (A16·Wlo + A16·Whi)
template <int BN, int PREC> struct Cfg {
    static constexpr int B_TILE_BYTES = BN * BLOCK_K * 2;
    static constexpr int A_BYTES = (PREC ? 1 : 2) * A_TILE_BYTES;            // offset of the B tiles inside a stage
    static constexpr int STAGE_BYTES = A_BYTES + 2 * B_TILE_BYTES;           // 64 KB (BN 128) / 96 KB (BN 256) of 227 KB
    static constexpr int STAGES = BN == 256 ? 2 : BN == 128 ? 3 : 4;
    static constexpr int VEC_OFF = STAGES * STAGE_BYTES;                     // BN 256: EpiVec copies of the two consumer warpgroups
    static constexpr int BAR_OFF = VEC_OFF + (BN == 256 ? 2 * EPI_VEC_BYTES : 0);
    static constexpr int SMEM_BYTES = BAR_OFF + 64 /*barriers*/ + 1024 /*align slack*/;
    static_assert(SMEM_BYTES <= 227 * 1024, "above the 227 KB of shared memory a block may use on sm_90");
};

// The QKV projection's instance (BN 256, EM_ROPE, bf16x3; rope_tiles below): the A slab of one 128-frame block stays
// resident, W streams through a ring of 128-channel stages
struct RopeCfg {
    static constexpr int SLAB_KB = 4;                        // k-blocks of the slab: K loops of at most 256 (wide_tile)
    static constexpr int KB_BYTES = 2 * A_TILE_BYTES;        // hi + lo of one A k-block: 32 KB
    static constexpr int W_TILE_BYTES = 128 * BLOCK_K * 2;   // 16 KB
    static constexpr int STAGE_BYTES = 2 * W_TILE_BYTES;     // 32 KB
    static constexpr int STAGES = 3;
    static constexpr int RING_OFF = SLAB_KB * KB_BYTES;      // 128 KB of A, then the ring
    static constexpr int VEC_OFF = RING_OFF + STAGES * STAGE_BYTES;    // the bias of each warpgroup's half-tile
    static constexpr int BAR_OFF = VEC_OFF + 2 * 128 * 4;
    static constexpr int SMEM_BYTES = BAR_OFF + 2 * (STAGES + SLAB_KB) * 8 + 1024 /*align slack*/;
    static_assert(SMEM_BYTES <= 227 * 1024, "above the 227 KB of shared memory a block may use on sm_90");
};

template <int BN, int MODE, int PREC> constexpr bool kRopeTiles = BN == 256 && MODE == EM_ROPE && PREC == 0;
template <int BN, int MODE, int PREC> constexpr int kSmemBytes = kRopeTiles<BN, MODE, PREC> ? RopeCfg::SMEM_BYTES : Cfg<BN, PREC>::SMEM_BYTES;

constexpr int ORDER_BAR = 3;           // named barriers 3, 4: ordered MMA issue of rope_tiles (1, 2: each warpgroup's own)

__device__ __forceinline__ void bar_arrive_n(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_sync_n(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// ----------------------------------------------------------------------------------------------
// The QKV projection on 256-channel tiles.  Its K loop is 4 k-blocks, so draining a 128 x 256 tile took about as long as
// its MMAs, and with both consumer warpgroups draining at once no MMA issued meanwhile (DESIGN.md §5).  Here:
//   * a CTA takes a contiguous range of the tile index (n fastest), so consecutive tiles share their 128-frame block.
//     Each tile splits into two 128 x 128 half-tiles; warpgroup 1 takes the even half-tiles of the range, warpgroup 2 the
//     odd ones, each over all 128 frames (two m64n128 accumulators, one per 64-row half);
//   * the A rows of the current frame block stay resident: a slab of up to 4 k-blocks x (hi + lo) = 128 KB, loaded once
//     per frame block.  K-block kb of the next block is loaded as soon as the MMAs on kb of both warpgroups' last
//     half-tiles of the block have retired (a_empty[kb]: 4 warps x 2 warpgroups);
//   * W streams through a ring of 128-channel stages in half-tile order; a stage is read by one warpgroup (4 warps);
//   * ordered MMA issue: a warpgroup starts a half-tile's MMAs only after the other has issued all of the previous
//     half-tile's (named barrier ORDER_BAR + its index), so one warpgroup's epilogue runs beside the other's MMAs.
// Phase invariant.  The producer and both warpgroups derive ring stage and phase from one enumeration of the CTA's
// half-tiles: ring position = (half-tile - first half-tile) x k-blocks + kb.  A warpgroup waits on a position only after
// every earlier position has been waited on (by itself, or by the other warpgroup before the handoff), so those fills
// have completed and the stage's full barrier is in the phase of this position: a parity wait cannot pass on an older
// phase, and the next fill of the stage needs this position's release first.  Likewise each warpgroup works on every frame
// block of the range (both halves of every tile) and releases each slab k-block once per block, so a_full[kb] cannot
// complete the next block before both warpgroups have waited on the current one.
__device__ __forceinline__ void rope_tiles(const TcMaps& maps, const TcParams& p, uint8_t* smem) {
    using C = RopeCfg;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
    uint64_t* empty_bar = full_bar + C::STAGES;
    uint64_t* a_full = empty_bar + C::STAGES;
    uint64_t* a_empty = a_full + C::SLAB_KB;
    const int wg = threadIdx.x >> 7;
    const int kb0 = (p.Cs0 + BLOCK_K - 1) / BLOCK_K;
    const int kb1 = p.n_src > 1 ? (p.Cs1 + BLOCK_K - 1) / BLOCK_K : 0;
    const int num_kb = p.taps * (kb0 + kb1);                    // <= SLAB_KB: wide_tile sends longer K loops to BN 128
    const int pad = p.taps / 2;
    const int hpb = 2 * p.n_tiles;                               // half-tiles per frame block
    const int h_begin = 2 * (int)((long)blockIdx.x * p.total_tiles / gridDim.x);
    const int h_end = 2 * (int)((long)(blockIdx.x + 1) * p.total_tiles / gridDim.x);

    if (threadIdx.x == 0) {
        prefetch_tmap(&maps.a_hi[0]); prefetch_tmap(&maps.a_lo[0]); prefetch_tmap(&maps.w_hi); prefetch_tmap(&maps.w_lo);
        if (p.n_src > 1) { prefetch_tmap(&maps.a_hi[1]); prefetch_tmap(&maps.a_lo[1]); }
        for (int i = 0; i < C::STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
        for (int i = 0; i < C::SLAB_KB; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 8); }
        mbar_fence_init();
    }
    __syncthreads();
    pdl_wait();                        // predecessors complete: operands are valid from here on

    if (wg == 0) {
        // ================= TMA producer =================
        reg_dealloc<40>();
        if (threadIdx.x == 0) {
            int stage = 0, slab = -1; uint32_t phase = 0, a_phase = 0;
            for (int h = h_begin; h < h_end; ++h) {
                const int m_tile = h / hpb, n0 = (h % hpb) * 128;
                const int bb = m_tile / p.m_tiles_per_b, t0 = (m_tile % p.m_tiles_per_b) * BLOCK_M;
                const bool load_a = m_tile != slab;
                for (int it = 0; it < num_kb; ++it) {
                    const int kb = it / p.taps, tap = it % p.taps;        // channel block outer, tap inner, as in gemm_wgmma_kernel
                    const int src = kb >= kb0 ? 1 : 0;
                    const int kc = (src ? kb - kb0 : kb) * BLOCK_K;
                    const int kw = (src ? p.Cs0 : 0) + kc;
                    if (load_a) {
                        mbar_wait(&a_empty[it], a_phase ^ 1);
                        uint8_t* s = smem + it * C::KB_BYTES;
                        mbar_expect_tx(&a_full[it], C::KB_BYTES);
                        const int ta = t0 + (tap - pad) * p.dil;
                        tma_load_3d(&maps.a_hi[src], &a_full[it], s, kc, ta, bb % p.a_bmod);
                        tma_load_3d(&maps.a_lo[src], &a_full[it], s + A_TILE_BYTES, kc, ta, bb % p.a_bmod);
                    }
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* s = smem + C::RING_OFF + stage * C::STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
                    tma_load_2d(&maps.w_hi, &full_bar[stage], s, kw, tap * p.N + n0);
                    tma_load_2d(&maps.w_lo, &full_bar[stage], s + C::W_TILE_BYTES, kw, tap * p.N + n0);
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
                }
                if (load_a) { slab = m_tile; a_phase ^= 1; }
            }
        }
    } else {
        // ================= consumers: alternate half-tiles, MMAs issued in half-tile order =================
        reg_alloc<232>();
        const int cw = wg - 1;
        const uint32_t vs = smem_u32(smem + C::VEC_OFF + cw * 128 * 4);
        float acc[128];                                          // acc[64 rh + ...]: rows [64 rh, 64 rh + 64) of the half-tile
        int slab = -1; uint32_t a_phase = 0;
        for (int h = h_begin + cw; h < h_end; h += 2) {
            const int m_tile = h / hpb, n0 = (h % hpb) * 128;
            const int bb = m_tile / p.m_tiles_per_b, t0 = (m_tile % p.m_tiles_per_b) * BLOCK_M;
            if (m_tile != slab) { a_phase ^= slab >= 0; slab = m_tile; }
            const bool last_of_slab = h + 2 >= h_end || (h + 2) / hpb != m_tile;
            stage_rope_bias(p, n0, vs, 1 + cw);                  // lands during the main loop
            const int pos = (h - h_begin) * num_kb;
            int stage = pos % C::STAGES, prev = 0;
            uint32_t phase = (pos / C::STAGES) & 1;
            if (h > h_begin) bar_sync_n(ORDER_BAR + cw, 256);    // the other warpgroup has issued the previous half-tile
            for (int it = 0; it < num_kb; ++it) {
                mbar_wait(&a_full[it], a_phase);
                mbar_wait(&full_bar[stage], phase);
                const uint32_t sa = smem_u32(smem + it * C::KB_BYTES);
                const uint32_t sb = smem_u32(smem + C::RING_OFF + stage * C::STAGE_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BLOCK_K / WG_K; ++k) {
                    const uint64_t adv = (uint64_t)((k * WG_K * 2) >> 4);   // +32 B per K step inside the 128 B row
                    const uint64_t b_hi = make_sw128_desc(sb) + adv, b_lo = make_sw128_desc(sb + C::W_TILE_BYTES) + adv;
#pragma unroll
                    for (int rh = 0; rh < 2; ++rh) {
                        float (&d)[64] = *reinterpret_cast<float (*)[64]>(&acc[64 * rh]);
                        const uint64_t a_hi = make_sw128_desc(sa + rh * (64 * 128)) + adv;
                        const uint64_t a_lo = make_sw128_desc(sa + A_TILE_BYTES + rh * (64 * 128)) + adv;
                        wgmma_m64n128k16_ss<false>(d, a_lo, b_hi, (it | k) != 0);   // small terms first
                        wgmma_m64n128k16_ss<false>(d, a_hi, b_lo, 1);
                        wgmma_m64n128k16_ss<false>(d, a_hi, b_hi, 1);
                    }
                }
                wgmma_commit();
                // keep this k-block in flight and release the previous one: a stage holds 32 KB of W only
                wgmma_wait<1>();
                if (it > 0 && (threadIdx.x & 31) == 0) {
                    mbar_arrive(&empty_bar[prev]);
                    if (last_of_slab) mbar_arrive(&a_empty[it - 1]);
                }
                prev = stage;
                if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
            }
            if (h + 1 < h_end) bar_arrive_n(ORDER_BAR + 1 - cw, 256);   // the other warpgroup may issue the next half-tile
            wgmma_wait<0>();
            if ((threadIdx.x & 31) == 0) {
                mbar_arrive(&empty_bar[prev]);
                if (last_of_slab) mbar_arrive(&a_empty[num_kb - 1]);
            }
            epilogue_rope_half(p, bb, t0, n0, acc, vs, 1 + cw);
        }
    }
}

// ----------------------------------------------------------------------------------------------
// One kernel instance per (tile width, epilogue mode): a combined kernel that switched over the modes at run time would
// make ptxas keep every mode's temporaries live beside the 64 / 128 accumulator registers.
template <int BN, int MODE, int PREC>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ TcMaps maps, const TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    pdl_trigger();                     // successor may start its prologue now; it waits for us before touching memory
    if constexpr (kRopeTiles<BN, MODE, PREC>) {
        rope_tiles(maps, p, smem);
    } else {
        using C = Cfg<BN, PREC>;
        uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
        uint64_t* empty_bar = full_bar + C::STAGES;

        const int wg = threadIdx.x >> 7;
        const int kb0 = (p.Cs0 + BLOCK_K - 1) / BLOCK_K;
        const int kb1 = p.n_src > 1 ? (p.Cs1 + BLOCK_K - 1) / BLOCK_K : 0;
        const int kb_per_tap = kb0 + kb1;
        const int num_kb = p.taps * kb_per_tap;
        const int it_per = (num_kb + p.ksplit - 1) / p.ksplit;     // split-K: a "batch" owns one slice of the K loop
        const int pad = p.taps / 2;

        if (threadIdx.x == 0) {
            prefetch_tmap(&maps.a_hi[0]); prefetch_tmap(&maps.a_lo[0]); prefetch_tmap(&maps.w_hi); prefetch_tmap(&maps.w_lo);
            if (p.n_src > 1) { prefetch_tmap(&maps.a_hi[1]); prefetch_tmap(&maps.a_lo[1]); }
            for (int i = 0; i < C::STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }   // one arrive per consumer warp
            mbar_fence_init();
        }
        __syncthreads();
        pdl_wait();                        // predecessors complete: operands / residuals are valid from here on

        if (wg == 0) {
            // ================= TMA producer =================
            reg_dealloc<40>();
            if (threadIdx.x == 0) {
                int stage = 0; uint32_t phase = 0;
                for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                    const int n_tile = tile % p.n_tiles, m_tile = tile / p.n_tiles;
                    const int bb = m_tile / p.m_tiles_per_b, t0 = (m_tile % p.m_tiles_per_b) * BLOCK_M;
                    const int ab = (bb % p.split_bb) % p.a_bmod, n0 = n_tile * BN;
                    const int it0 = (bb / p.split_bb) * it_per, it1 = min(num_kb, it0 + it_per);
                    // channel block OUTER, tap INNER: the k taps of one channel block read the same A rows shifted by one
                    // frame, back to back, so taps 1.. hit L2 (tap-outer order re-reads the whole A slab per tap)
                    for (int it = it0; it < it1; ++it) {
                        const int kb = it / p.taps, tap = it % p.taps;
                        const int src = kb >= kb0 ? 1 : 0;
                        const int kc = (src ? kb - kb0 : kb) * BLOCK_K;          // channel offset inside the source
                        const int kw = (src ? p.Cs0 : 0) + kc;                   // column in the packed weight
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        uint8_t* s = smem + stage * C::STAGE_BYTES;
                        mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
                        const int ta = t0 + (tap - pad) * p.dil;                 // first frame of this tap's A rows
                        tma_load_3d(&maps.a_hi[src], &full_bar[stage], s, kc, ta, ab);          // PREC: the fp16 plane
                        if (!PREC) tma_load_3d(&maps.a_lo[src], &full_bar[stage], s + A_TILE_BYTES, kc, ta, ab);
                        tma_load_2d(&maps.w_hi, &full_bar[stage], s + C::A_BYTES, kw, tap * p.N + n0);
                        tma_load_2d(&maps.w_lo, &full_bar[stage], s + C::A_BYTES + C::B_TILE_BYTES, kw, tap * p.N + n0);
                        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        } else {
            // ================= consumers: wgmma main loop + epilogue on the accumulator registers =================
            reg_alloc<232>();
            const int cw = wg - 1;                          // frames [64 cw, 64 cw + 64) of the tile
            float acc[BN / 2];
            int stage = 0; uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                const int n_tile = tile % p.n_tiles, m_tile = tile / p.n_tiles;
                const int bb = m_tile / p.m_tiles_per_b, t0 = (m_tile % p.m_tiles_per_b) * BLOCK_M + cw * 64;
                const uint32_t vs = smem_u32(smem + C::VEC_OFF + cw * EPI_VEC_BYTES);
                if constexpr (BN == 256) stage_epi_vectors<BN, MODE>(p, bb, n_tile * BN, vs, 1 + cw);   // lands during the main loop
                const int it0 = (bb / p.split_bb) * it_per;
                const int n_it = min(num_kb, it0 + it_per) - it0;
                for (int kb = 0; kb < n_it; ++kb) {
                    mbar_wait(&full_bar[stage], phase);
                    const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES) + (uint32_t)cw * (64 * 128);
                    const uint32_t sb = smem_u32(smem + stage * C::STAGE_BYTES) + C::A_BYTES;
                    const uint64_t a_hi = make_sw128_desc(sa), a_lo = make_sw128_desc(sa + A_TILE_BYTES);
                    wgmma_fence();
    #pragma unroll
                    for (int k = 0; k < BLOCK_K / WG_K; ++k) {
                        const uint64_t adv = (uint64_t)((k * WG_K * 2) >> 4);   // +32 B per K step inside the 128 B row
                        if constexpr (BN < 128) {          // narrow tile: one m64nBNk16 per pass
                            const uint64_t b_hi = make_sw128_desc(sb) + adv, b_lo = make_sw128_desc(sb + C::B_TILE_BYTES) + adv;
                            const int acc_in = (kb | k) != 0;
                            if constexpr (BN == 64) {
                                wgmma_m64n64k16_ss(acc, a_lo + adv, b_hi, acc_in);
                                wgmma_m64n64k16_ss(acc, a_hi + adv, b_lo, 1);
                                wgmma_m64n64k16_ss(acc, a_hi + adv, b_hi, 1);
                            } else if constexpr (BN == 32) {
                                wgmma_m64n32k16_ss(acc, a_lo + adv, b_hi, acc_in);
                                wgmma_m64n32k16_ss(acc, a_hi + adv, b_lo, 1);
                                wgmma_m64n32k16_ss(acc, a_hi + adv, b_hi, 1);
                            } else {
                                wgmma_m64n16k16_ss(acc, a_lo + adv, b_hi, acc_in);
                                wgmma_m64n16k16_ss(acc, a_hi + adv, b_lo, 1);
                                wgmma_m64n16k16_ss(acc, a_hi + adv, b_hi, 1);
                            }
                        }
    #pragma unroll
                        for (int h = 0; h < BN / 128; ++h) {
                            float (&d)[64] = *reinterpret_cast<float (*)[64]>(&acc[64 * h]);
                            const uint64_t b_hi = make_sw128_desc(sb + h * (128 * 128)) + adv;
                            const uint64_t b_lo = make_sw128_desc(sb + C::B_TILE_BYTES + h * (128 * 128)) + adv;
                            if (PREC) {                    // fp16 operands: A16·Wlo + A16·Whi (small term first)
                                wgmma_m64n128k16_ss<true>(d, a_hi + adv, b_lo, (kb | k) != 0);
                                wgmma_m64n128k16_ss<true>(d, a_hi + adv, b_hi, 1);
                            } else {
                                wgmma_m64n128k16_ss<false>(d, a_lo + adv, b_hi, (kb | k) != 0);   // small terms first
                                wgmma_m64n128k16_ss<false>(d, a_hi + adv, b_lo, 1);
                                wgmma_m64n128k16_ss<false>(d, a_hi + adv, b_hi, 1);
                            }
                        }
                    }
                    wgmma_commit();
                    // the stage is handed back as soon as its own MMAs have retired.  Keeping this k-block in flight across the
                    // next stage's wait (wait_group 1, release of the PREVIOUS stage) was measured slower on H100 80GB HBM3
                    // (700 W; separate runs, attention — untouched by it — 20.6 ms in both): cfg1 185 vs 167 ms per solve, GEMM
                    // class 151 vs 133 ms — with two or three 64-96 KB stages a stage held one block longer is
                    // a stage the producer cannot prefetch into; the two consumer warpgroups already overlap each other
                    wgmma_wait<0>();
                    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty_bar[stage]);      // this warp's share of the stage reads has retired
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
                }
                epilogue_tile<BN, MODE>(p, bb, t0, n_tile * BN, acc, vs, 1 + cw);
            }
        }
    }
}

// ----------------------------------------------------------------------------------------------
// host side: tensor-map construction (cached) and launch
// ----------------------------------------------------------------------------------------------
std::string g_err = "";
std::recursive_mutex g_mu;          // held for a whole launch_gemm_tc (g_err, the map cache); the map cache re-enters it
PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

struct MapKey {
    const void* ptr; uint64_t d0, d1, d2; uint32_t b0, b1; int rank;
    bool operator==(const MapKey& o) const {
        return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && b0 == o.b0 && b1 == o.b1 && rank == o.rank;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = std::hash<const void*>()(k.ptr);
        h ^= k.d0 * 0x9E3779B97F4A7C15ull + (h << 6); h ^= k.d1 * 0xC2B2AE3D27D4EB4Full + (h >> 3);
        h ^= k.d2 * 0x165667B19E3779F9ull + (h << 9); h ^= ((size_t)k.b0 << 20) ^ ((size_t)k.b1 << 4) ^ (size_t)k.rank;
        return h;
    }
};
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
GemmPlan g_inst;                    // the instance the last launch_inst launched (under g_mu)

bool ensure_encode() {
    if (g_encode) return true;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
        g_err = "cuTensorMapEncodeTiled driver entry point unavailable";
        return false;
    }
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    return true;
}

// 2-byte-element operand tile, 128-byte swizzle; dim0 contiguous.  rank 3: (d0, d1, d2) box (b0, b1, 1); rank 2: (d0, d1) box (b0, b1).
bool get_map(const void* ptr, int rank, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1, CUtensorMap* out) {
    MapKey key{ptr, d0, d1, d2, b0, b1, rank};
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return true; }
    const uint64_t es = 2;
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {d0 * es, d0 * d1 * es};
    cuuint32_t box[3] = {b0, b1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUtensorMap m;
    CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank,
                          const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        g_err = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r) + " (rank " + std::to_string(rank) +
                ", dims " + std::to_string(d0) + "x" + std::to_string(d1) + "x" + std::to_string(d2) + ")";
        return false;
    }
    if (g_maps.size() > 4096) g_maps.clear();
    g_maps.emplace(key, m);
    *out = m;
    return true;
}

template <int BN, int MODE, int PREC>
cudaError_t launch_inst(const TcMaps& maps, const TcParams& p, int grid, cudaStream_t s) {
    constexpr int SMEM = kSmemBytes<BN, MODE, PREC>;
    static std::atomic<uint64_t> attr_done{0};      // one bit per device (per template instance)
    cudaError_t e = ensure_dyn_smem(gemm_wgmma_kernel<BN, MODE, PREC>, SMEM, attr_done);
    if (e != cudaSuccess) { g_err = "cudaFuncSetAttribute(max dynamic smem) failed"; return e; }
    g_inst.engine = ST_ENGINE_TCGEN05; g_inst.bn = BN; g_inst.mode = MODE; g_inst.prec = PREC; g_inst.ksplit = p.ksplit; g_inst.grid = grid;
    return launch_k(gemm_wgmma_kernel<BN, MODE, PREC>, dim3(grid), dim3(NUM_THREADS), (size_t)SMEM, s, maps, p);
}

template <int BN>
cudaError_t launch_bn(const GemmArgs& g, int num_sms, cudaStream_t s, int split_bb = 0) {
    TcMaps maps;
    for (int i = 0; i < g.n_src; ++i) {            // (a 2-byte-element map serves bf16 and fp16 planes alike)
        if (!tmap_encode_bf16(g.A_hi[i], 3, (uint64_t)g.Cs[i], (uint64_t)g.T, (uint64_t)g.a_bmod, BLOCK_K, BLOCK_M, &maps.a_hi[i])) return cudaErrorInvalidValue;
        if (g.prec) maps.a_lo[i] = maps.a_hi[i];
        else if (!tmap_encode_bf16(g.A_lo[i], 3, (uint64_t)g.Cs[i], (uint64_t)g.T, (uint64_t)g.a_bmod, BLOCK_K, BLOCK_M, &maps.a_lo[i])) return cudaErrorInvalidValue;
    }
    if (g.n_src == 1) { maps.a_hi[1] = maps.a_hi[0]; maps.a_lo[1] = maps.a_lo[0]; }
    const uint32_t wrows = BN == 256 && (g.flags & EPI_ROPE) ? 128 : BN;     // rope_tiles streams W in 128-channel stages
    if (!tmap_encode_bf16(g.W_hi, 2, (uint64_t)g.Ktot, (uint64_t)g.taps * g.N, 1, BLOCK_K, wrows, &maps.w_hi)) return cudaErrorInvalidValue;
    if (!tmap_encode_bf16(g.W_lo, 2, (uint64_t)g.Ktot, (uint64_t)g.taps * g.N, 1, BLOCK_K, wrows, &maps.w_lo)) return cudaErrorInvalidValue;
    TcParams p;
    fill_tc_params(p, g);
    if (split_bb > 0) { p.ksplit = g.ksplit; p.split_bb = split_bb; }
    p.m_tiles_per_b = (g.T + BLOCK_M - 1) / BLOCK_M;
    p.n_tiles = (g.N + BN - 1) / BN;
    p.total_tiles = g.BB * p.m_tiles_per_b * p.n_tiles;
    const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
    if (p.mode == EM_MISH) {           // one instance: launch_gemm_tc routes Mish to 128-channel tiles
        if constexpr (BN == 128) return launch_inst<BN, EM_MISH, 0>(maps, p, grid, s);
        g_err = "EPI_MISH runs on 128-channel tiles only"; return cudaErrorInvalidValue;
    }
    if constexpr (BN == 256) {
        // epilogue_wide does no bounds work on columns; epilogue_rope_half rotates / scales whole 64-wide RoPE heads
        if (g.N % 256) { g_err = "256-channel tiles need N % 256 == 0"; return cudaErrorInvalidValue; }
        if ((g.flags & EPI_ROPE) && g.rope_H % 64) { g_err = "RoPE on 256-channel tiles needs rope_H % 64 == 0"; return cudaErrorInvalidValue; }
        if (g.prec) {                  // two-pass fp16 FFN convs: conv_1 (SiLU), conv_2 (residual, with or without the fused LayerNorm)
            switch (p.mode) {
                case EM_SILU:  return launch_inst<BN, EM_SILU, 1>(maps, p, grid, s);
                case EM_LN:    return launch_inst<BN, EM_LN, 1>(maps, p, grid, s);
                case EM_RESID: return launch_inst<BN, EM_RESID, 1>(maps, p, grid, s);
                case EM_PLAIN: return launch_inst<BN, EM_PLAIN, 1>(maps, p, grid, s);      // long-skip conv without the fused LayerNorm
                default: g_err = "the two-pass fp16 precision is built for the FFN and long-skip convs only"; return cudaErrorInvalidValue;
            }
        }
        if (p.mode == EM_LN) return launch_inst<BN, EM_LN, 0>(maps, p, grid, s);           // needs full rows: wide tile only
    }
    if constexpr (BN < 128) {          // narrow tiles: the conv epilogues only (RoPE needs 64-column head groups, LN full rows)
        switch (p.mode) {
            case EM_SILU: return launch_inst<BN, EM_SILU, 0>(maps, p, grid, s);
            case EM_GELU: return launch_inst<BN, EM_GELU, 0>(maps, p, grid, s);
            case EM_RESID: return launch_inst<BN, EM_RESID, 0>(maps, p, grid, s);
            case EM_SILU_OUT: return launch_inst<BN, EM_SILU_OUT, 0>(maps, p, grid, s);
            case EM_PLAIN: return launch_inst<BN, EM_PLAIN, 0>(maps, p, grid, s);
            default: g_err = "narrow tiles: unsupported epilogue"; return cudaErrorInvalidValue;
        }
    }
    switch (p.mode) {                  // one kernel instance per epilogue mode
        case EM_ROPE: return launch_inst<BN, EM_ROPE, 0>(maps, p, grid, s);
        case EM_SILU: return launch_inst<BN, EM_SILU, 0>(maps, p, grid, s);
        case EM_GELU: return launch_inst<BN, EM_GELU, 0>(maps, p, grid, s);
        case EM_RESID: return launch_inst<BN, EM_RESID, 0>(maps, p, grid, s);
        case EM_SILU_OUT: return launch_inst<BN, EM_SILU_OUT, 0>(maps, p, grid, s);
        default:      return launch_inst<BN, EM_PLAIN, 0>(maps, p, grid, s);
    }
}

}  // namespace

const char* gemm_tc_last_error() { return g_err.c_str(); }

// shared with attention_tc.cu (cached, mutex-free: callers serialise through their own launch mutex)
bool tmap_encode_bf16(const void* ptr, int rank, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1,
                      CUtensorMap* out) {
    std::lock_guard<std::recursive_mutex> lk(g_mu);
    if (!ensure_encode()) return false;
    return get_map(ptr, rank, d0, d1, d2, b0, b1, out);
}

// wide (256-channel) tiles: outputs that are a multiple of 256 channels, with enough tiles to give every SM one (not for Mish,
// nor for RoPE with a K loop longer than the resident A slab of rope_tiles)
static bool wide_tile(const GemmArgs& g, int num_sms) {
    if (!g.A_hi[0] || !g.W_hi || g.N % 256 || (g.flags & EPI_MISH)) return false;     // (Mish: 128-channel tiles only)
    const int kblocks = (g.Cs[0] + BLOCK_K - 1) / BLOCK_K + (g.n_src > 1 ? (g.Cs[1] + BLOCK_K - 1) / BLOCK_K : 0);
    if ((g.flags & EPI_ROPE) && g.taps * kblocks > RopeCfg::SLAB_KB) return false;
    return (long)g.BB * ((g.T + BLOCK_M - 1) / BLOCK_M) * (g.N / 256) >= num_sms;
}

bool gemm_tc_wide_tile(const GemmArgs& g, int num_sms) { return wide_tile(g, num_sms); }

bool gemm_tc_ln_fusable(const GemmArgs& g, int num_sms) { return g.N == 256 && wide_tile(g, num_sms); }

static cudaError_t launch_gemm_tc_locked(const GemmArgs& g, int num_sms, cudaStream_t s);

cudaError_t launch_gemm_tc(const GemmArgs& g, int num_sms, cudaStream_t s) {
    if (g.BB == 0 || g.T == 0) return cudaSuccess;
    std::lock_guard<std::recursive_mutex> lk(g_mu);
    g_inst = GemmPlan();
    const cudaError_t e = launch_gemm_tc_locked(g, num_sms, s);
    if (e == cudaSuccess && g.plan) *g.plan = g_inst;
    return e;
}

static cudaError_t launch_gemm_tc_locked(const GemmArgs& g, int num_sms, cudaStream_t s) {
    if (const char* why = gemm_flags_error(g)) { g_err = why; return cudaErrorInvalidValue; }
    const bool wide = wide_tile(g, num_sms);
    if (g.dil < 1) { g_err = "tap dilation must be >= 1"; return cudaErrorInvalidValue; }
    if (g.ln && g.N != 256) {          // the epilogue normalises over one 256-channel tile: a wider row would be cut in halves
        g_err = "fused LayerNorm needs N == 256 (check gemm_tc_ln_fusable before setting GemmArgs::ln)";
        return cudaErrorInvalidValue;
    }
    if (g.out16 && g.ksplit > 1) {     // the reduce kernel writes split-bf16 planes only
        g_err = "split-K does not write the fp16 output plane (out16)";
        return cudaErrorInvalidValue;
    }
    if ((g.ln || g.prec) && !wide) {
        g_err = g.ln ? "fused LayerNorm needs full-row 256-channel tiles (check gemm_tc_ln_fusable before setting GemmArgs::ln)"
                     : "the two-pass fp16 FFN precision runs on the 256-channel tile only (check gemm_tc_wide_tile before setting GemmArgs::prec)";
        return cudaErrorInvalidValue;
    }
    if (g.ln && (!g.u_hi || (!g.u16 && !g.u_lo) || (g.film2 && !g.out2_f32))) { g_err = "fused LayerNorm: missing output plane"; return cudaErrorInvalidValue; }
    if (!ensure_encode()) return cudaErrorNotSupported;
    for (int i = 0; i < g.n_src; ++i) {
        if (!g.A_hi[i] || (!g.prec && !g.A_lo[i])) { g_err = "split-bf16 A planes missing"; return cudaErrorInvalidValue; }
        if (g.Cs[i] % 8) { g_err = "A channels must be a multiple of 8 (16-byte TMA stride)"; return cudaErrorInvalidValue; }
        if (i == 0 && g.n_src > 1 && g.Cs[0] % BLOCK_K) { g_err = "first concat source must be a multiple of 64 channels"; return cudaErrorInvalidValue; }
    }
    if (!g.W_hi || !g.W_lo || g.Ktot % 8 || g.N % 8) { g_err = "bad weight operand"; return cudaErrorInvalidValue; }
    if (!g.out_f32 && !g.out_hi) { g_err = "no output plane"; return cudaErrorInvalidValue; }
    if (g.out_hi && !g.out16 && !g.out_lo) { g_err = "split output needs both planes"; return cudaErrorInvalidValue; }
    if (wide) {
        if (g.ksplit > 1) { g_err = "split-K runs on 128-channel tiles; this problem takes 256-channel tiles"; return cudaErrorInvalidValue; }
        return launch_bn<256>(g, num_sms, s);
    }
    if (g.ksplit > 1) {                // split-K: raw fp32 partial tiles of ksplit x BB "batches", then the reduce + epilogue kernel
        if (!g.part || (g.flags & EPI_ROPE)) { g_err = "split-K needs a partial buffer and a non-RoPE epilogue"; return cudaErrorInvalidValue; }
        const int nkb = g.taps * ((g.Cs[0] + BLOCK_K - 1) / BLOCK_K + (g.n_src > 1 ? (g.Cs[1] + BLOCK_K - 1) / BLOCK_K : 0));
        if (nkb % g.ksplit) {          // an empty K slice would never complete its accumulator: refuse instead of hanging
            g_err = "split-K factor does not divide the K loop"; return cudaErrorInvalidValue;
        }
        GemmArgs q = g;
        q.BB = g.ksplit * g.BB; q.flags = 0; q.out_f32 = g.part; q.out_hi = nullptr; q.out_lo = nullptr; q.ksplit = g.ksplit;
        cudaError_t e = launch_bn<128>(q, num_sms, s, g.BB);
        if (e != cudaSuccess) return e;
        e = launch_splitk_reduce(g, s);
        if (e != cudaSuccess) g_err = "split-K reduce launch failed";
        return e;
    }
    if (!g.ln && !g.prec && !(g.flags & (EPI_ROPE | EPI_MISH))) {   // outputs of exactly 16 / 32 / 64 channels: narrow tiles
        if (g.N == 64) return launch_bn<64>(g, num_sms, s);
        if (g.N == 32) return launch_bn<32>(g, num_sms, s);
        if (g.N == 16) return launch_bn<16>(g, num_sms, s);
    }
    return launch_bn<128>(g, num_sms, s);
}

}  // namespace st
