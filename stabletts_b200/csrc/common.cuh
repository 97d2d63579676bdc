// Shared declarations for libstabletts_b200.so (sm_90a only).
//
// Internal data layout: every activation is TOKEN-MAJOR (B, T, C) with C contiguous — one mel
// frame is one GEMM row — while the C-ABI boundary keeps the reference's channel-major (B, C, T).
// Tensor-core GEMM operands are carried as split-bf16 plane pairs (hi = bf16(x), lo = bf16(x - hi))
// because plain bf16 operands cannot meet the 1e-3 parity bar (SURVEY.md fact 3).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <map>
#include <atomic>

#include "../../include/stabletts_b200.h"

namespace st {

typedef __nv_bfloat16 bf16;

// ----------------------------------------------------------------------------------------------
// conv-GEMM problem:  out[bb, t, n] = epi( sum_{tap, src, k} A_src[bb % a_bmod, t + (tap - taps/2) * dil, k]
//                                                          * W[tap][n][koff_src + k] )
// rows outside [0, T) read as zero (the reference's Conv1d zero padding at TENSOR edges).
// ----------------------------------------------------------------------------------------------
enum : int {
    EPI_BIAS  = 1 << 0,   // v += bias[n]
    EPI_SILU  = 1 << 1,   // v = v * sigmoid(v)
    EPI_FILM  = 1 << 2,   // v = gamma[n] * v + beta[n]
    EPI_MASK  = 1 << 3,   // v *= mask[bb % B, t]
    EPI_GATE  = 1 << 4,   // v *= gate[min(bb, c_clamp), n]
    EPI_RESID = 1 << 5,   // v += resid[min(bb, resid_clamp), t, n]
    EPI_ROPE  = 1 << 6,   // partial RoPE on q/k column blocks (QKV projection only; TC engine)
    EPI_GELU  = 1 << 7,   // v = 0.5 v (1 + erf(v / sqrt 2)): nn.GELU() exact form (Vocos ConvNeXt block, module.py:26)
    EPI_SILU_OUT = 1 << 8,   // after the whole epilogue: v -> out_f32, silu(v) -> the split planes and / or out2_f32
                             // (FireflyGAN ResBlock1: the residual stream and the operand of the next conv, head.py:94-98)
    EPI_MISH = 1 << 9,    // v = v tanh(softplus(v)), softplus(v) = v for v > 20 (nn.Mish; MelStyleEncoder.spectral,
                          // models/reference_encoder.py:47-52)
};
// Allowed sets (every engine refuses the others, gemm_flags_error): at most one activation (SILU, GELU or MISH), and it
// excludes RESID and SILU_OUT, because the wgmma engine has one epilogue instance per mode; ROPE combines with BIAS only;
// the fused LayerNorm (GemmArgs::ln) excludes the activations, SILU_OUT and ROPE.  MISH runs on 128-channel tiles only
// (its one wgmma instance; launch_gemm_tc routes it there).
constexpr int EPI_ALL = EPI_BIAS | EPI_SILU | EPI_FILM | EPI_MASK | EPI_GATE | EPI_RESID | EPI_ROPE | EPI_GELU | EPI_SILU_OUT |
                        EPI_MISH;

// the launch that ran (filled by launch_gemm_tc / launch_gemm_simt when GemmArgs::plan is set; st_test_gemm_ex reports it)
struct GemmPlan {
    int engine = -1;                  // ST_ENGINE_*
    int bn = 0;                       // tile width in output channels
    int mode = -1;                    // EM_* epilogue instance of the wgmma kernel (gemm_epilogue.cuh); -1 for the SIMT engine
    int prec = 0;                     // 1: two-pass fp16 operands
    int ksplit = 1;                   // > 1: split-K partial pass (mode is then the partial pass's) + reduce-and-epilogue kernel
    int grid = 0;                     // CTAs launched (persistent wgmma kernel: min(tiles, SMs))
};

struct GemmArgs {
    // A: n_src sources concatenated along channels, each (a_batches, T, Cs[i]) token-major.
    const float* A_f32[2] = {nullptr, nullptr};   // SIMT engine
    const bf16*  A_hi[2]  = {nullptr, nullptr};   // tensor-core engine: split planes
    const bf16*  A_lo[2]  = {nullptr, nullptr};
    int Cs[2] = {0, 0};
    int n_src = 1;
    int a_bmod = 0;                               // A batch index = bb % a_bmod
    // W: packed [taps][N][Ktot], K contiguous
    const float* W_f32 = nullptr;
    const bf16*  W_hi = nullptr;
    const bf16*  W_lo = nullptr;
    const float* bias = nullptr;
    int taps = 1, N = 0, Ktot = 0;
    int dil = 1;                                  // tap spacing in frames (dilated Conv1d)
    int BB = 0, T = 0;
    // epilogue
    int flags = 0;
    const float* mask = nullptr; int B = 1;       // (B, T)
    const float* film = nullptr; long film_bstride = 0; int film_H = 0;   // gamma[n], beta[film_H + n]
    const float* gate = nullptr; long gate_bstride = 0; int c_clamp = 0;
    const float* resid = nullptr; int resid_clamp = 0;
    const float* rope_cs = nullptr; int rope_H = 0; // (T, 16, 2) cos/sin table; columns [0,2*rope_H) are q|k (EPI_ROPE)
    float* out_f32 = nullptr;
    bf16*  out_hi = nullptr;
    bf16*  out_lo = nullptr;
    // fused LayerNorm(C = N, no affine, eps 1e-5) + adaLN modulate of the finished output row (tensor-core engine, tiles that span
    // all N = 256 channels: gemm_tc_ln_fusable): u = ((x - mean) rstd (1 + scale) + shift) [* mask] -> u_hi / u_lo.
    // film2 (optional): x2 = (gamma2 x + beta2) * mask first — the NEXT block's time fusion (models/estimator.py:16) —
    // written to out2_f32, and the LayerNorm runs over x2.
    int ln = 0, ln_mask_out = 0;
    const float* ln_shift = nullptr; const float* ln_scale = nullptr; long ada_bstride = 0;
    bf16* u_hi = nullptr; bf16* u_lo = nullptr;
    const float* film2 = nullptr; long film2_bstride = 0; float* out2_f32 = nullptr;
    // (film2 and ln_mask_out multiply by mask[bb % B, t] whenever `mask` is set, with or without EPI_MASK)
    // opt-in two-pass FFN precision (ST_PRECISION_FFN_FP16X2, 256-channel tiles only): prec = 1 -> the A operand is ONE fp16
    // plane (A_hi[i] points to it, A_lo is ignored), the weights are an fp16 hi / lo pair (W_hi / W_lo point to them) and
    // each k-step issues A16·Wlo + A16·Whi (wgmma with fp16 operands).  out16: the split output becomes one fp16 plane
    // written to out_hi (out_lo ignored); u16: likewise for the fused LayerNorm output u_hi.
    int prec = 0, out16 = 0, u16 = 0;
    // split-K for latency-bound small problems (128-channel tiles): the K loop (taps x channel blocks) is cut into `ksplit`
    // slices that run as ksplit x BB "batches" writing raw fp32 partial tiles into `part` ((ksplit*BB, T, N)); a reduce
    // kernel then sums the slices in a fixed order and applies this GemmArgs' epilogue (launch_splitk_reduce).  Deterministic.
    int ksplit = 1; float* part = nullptr;
    // 1: run_gemm never chooses split-K for this GEMM, so an utterance's result does not depend on how many others share
    // the call (split-K is picked from the tile count, i.e. the batch size, and changes the summation order)
    int batch_invariant = 0;
    // 0: run_gemm decides split-K itself; 1: never; 2..4: exactly that factor (kernel-level tests: st_test_gemm_ex)
    int force_ksplit = 0;
    GemmPlan* plan = nullptr;                     // optional: receives the launch that ran
};

// nullptr when the epilogue flags and switches form an allowed set (see EPI_*), else why not
inline const char* gemm_flags_error(const GemmArgs& g) {
    const int f = g.flags;
    if (f & ~EPI_ALL) return "unknown EPI_* flag";
    const int acts = f & (EPI_SILU | EPI_GELU | EPI_MISH);
    const bool act = acts != 0;
    if (acts & (acts - 1)) return "EPI_SILU, EPI_GELU and EPI_MISH are alternatives (one activation per GEMM)";
    if (act && (f & EPI_RESID)) return "EPI_RESID does not combine with EPI_SILU / EPI_GELU / EPI_MISH";
    if (act && (f & EPI_SILU_OUT)) return "EPI_SILU_OUT does not combine with EPI_SILU / EPI_GELU / EPI_MISH";
    if ((f & EPI_ROPE) && (f & ~(EPI_ROPE | EPI_BIAS))) return "EPI_ROPE combines with EPI_BIAS only (the QKV epilogue variant)";
    if (g.ln && (act || (f & (EPI_SILU_OUT | EPI_ROPE)))) return "the fused LayerNorm does not combine with EPI_SILU / EPI_GELU / EPI_MISH / EPI_SILU_OUT / EPI_ROPE";
    return nullptr;
}

// engines
// nullptr when the SIMT engine supports this problem, else why not (it has no fused LayerNorm, fp16 planes or RoPE)
const char* gemm_simt_unsupported(const GemmArgs& g);
cudaError_t launch_gemm_simt(const GemmArgs& g, cudaStream_t s);
// out = epilogue(sum_s part[s]) with g's flags (bias, SiLU / GELU / Mish, FiLM, mask, gate, residual) -> fp32 and / or split planes
cudaError_t launch_splitk_reduce(const GemmArgs& g, cudaStream_t s);
// returns cudaErrorNotSupported if the tensor-map driver entry point is unavailable
cudaError_t launch_gemm_tc(const GemmArgs& g, int num_sms, cudaStream_t s);
const char* gemm_tc_last_error();
// true when launch_gemm_tc would run this problem on full-row (256-channel) tiles, i.e. GemmArgs::ln may be set
bool gemm_tc_ln_fusable(const GemmArgs& g, int num_sms);
// true when launch_gemm_tc would run this problem on 256-channel tiles at all (GemmArgs::prec / out16 need them)
bool gemm_tc_wide_tile(const GemmArgs& g, int num_sms);

// ----------------------------------------------------------------------------------------------
// elementwise / reduction kernels (elementwise.cu)
// ----------------------------------------------------------------------------------------------
// (B, C, T) -> (B', T, C) with optional extra broadcast row: if bcast != null, batch index B is
// filled with bcast[c] for every t (the CFG fake_content, models/flow_matching.py:60).
cudaError_t launch_bct_to_btc(const float* in, float* out_f32, bf16* out_hi, bf16* out_lo, int B, int C, int T,
                              const float* bcast, cudaStream_t s);
cudaError_t launch_btc_to_bct(const float* in, float* out, int B, int C, int T, cudaStream_t s);

struct LnArgs {
    const float* xin = nullptr;   // (BB, T, H)
    float* xout = nullptr;        // residual stream written when has_film (may alias xin)
    const float* film = nullptr; long film_bstride = 0;     // gamma[0..H), beta[H..2H)
    const float* shift = nullptr; const float* scale = nullptr; long ada_bstride = 0; int c_clamp = 0;
    const float* mask = nullptr; int B = 1;
    int has_film = 0;             // x = (gamma*xin+beta)*mask  (models/estimator.py:16)
    int mask_out = 0;             // u *= mask (FFN input, models/diffusion_transformer.py:26)
    float* u_f32 = nullptr; bf16* u_hi = nullptr; bf16* u_lo = nullptr;
    int u16 = 0;                  // u_hi receives ONE fp16 plane instead of the bf16 hi / lo pair (two-pass FFN mode)
    int BB = 0, T = 0, H = 0;
};
cudaError_t launch_film_ln_mod(const LnArgs& a, cudaStream_t s);

// y[r * y_rstride + n] = post( bias[n] + sum_k pre(x[r, k]) * W[n, k] ),  pre/post in {none, silu}
cudaError_t launch_gemv(const float* x, const float* W, const float* bias, float* y, long y_rstride, int R, int K, int N,
                        int silu_in, int silu_out, cudaStream_t s);
// sinusoidal embedding of n_t times (models/estimator.py:41-49): out (n_t, H)
cudaError_t launch_time_embed(const float* t, int n_t, int H, float* out, cudaStream_t s);
// cos/sin table (T, 16, 2) of models/diffusion_transformer.py:150-171 with d = 32
cudaError_t launch_rope_table(float* cs, int T, int d_rot, cudaStream_t s);
// kvlen[b] = 1 + last index with mask != 0 (0 if none); prefix[b] = first index with mask == 0 (T if none)
cudaError_t launch_mask_lengths(const float* mask, int* kvlen, int* prefix, int B, int T, cudaStream_t s);
// K_out = uncond + s*(cond - uncond) (models/flow_matching.py:66) or copy when !cfg
cudaError_t launch_cfg_combine(const float* V, float* K_out, int B, long per_batch, int cfg, float s_cfg, cudaStream_t s);
// dst = y + sum_i coef[i] * K[i]   (n <= 6)
cudaError_t launch_lincomb(float* dst, const float* y, const float* const* K, const float* coef, int n, long numel,
                           cudaStream_t s);
// TextEncoder front end: x (B,T,H) = emb[ids] * scale * mask, mask (B,T) = t < lens[b]
cudaError_t launch_embed(const int64_t* ids, const int64_t* lens, const float* emb, int n_vocab, int B, int T, int H, float scale,
                         float* x, float* mask, cudaStream_t s);
// *out = sum_e ((sum_i coef_i K_i[e]) / (atol + rtol max(|u[e]|,|v[e]|)))^2   (n <= 7; out is zeroed first)
cudaError_t launch_scaled_sumsq(const float* const* K, const float* coef, int n, const float* u, const float* v, float atol,
                                float rtol, long numel, double* out, cudaStream_t s);
// fp32 -> split bf16 planes
cudaError_t launch_cfm_mix(const float* x1, const float* z, const float* t, float sigma_min, int B, long per_batch, float* y,
                           cudaStream_t s);
cudaError_t launch_cfm_loss(const float* v, const float* x1, const float* z, const float* mask, float sigma_min, int B, int C,
                            int T, double* acc2, float* loss, cudaStream_t s);
cudaError_t launch_split(const float* in, bf16* hi, bf16* lo, long numel, cudaStream_t s);
// fp32 -> fp16 hi / lo planes (hi = fp16(x), lo = fp16(x - hi)), stored in 2-byte slots typed bf16* like every plane here
cudaError_t launch_split_f16(const float* in, bf16* hi, bf16* lo, long numel, cudaStream_t s);

// duration -> alignment -> mu_y expansion (align.cu; models/model.py:81-95)
cudaError_t launch_align_lengths(const float* logw, const float* x_mask, float length_scale, int B, int Tx, float* cum,
                                 long long* ylen, cudaStream_t s);
cudaError_t launch_align_expand(const float* mu_x, const float* x_mask, const float* cum, const long long* ylen, int B, int M,
                                int Tx, int Ty, float* mu_y, float* y_mask, float* attn, cudaStream_t s);

// monotonic alignment search of the training forward (mas.cu; models/model.py:148-176, monotonic_align/core.py)
int mas_max_tx();
size_t mas_workspace_bytes(int B, int Ty, int Tx);
cudaError_t launch_mas_scores(const float* y, const float* mu_x, float* neg_cent, int B, int D, int Ty, int Tx, cudaStream_t s);
cudaError_t launch_maximum_path(const float* neg_cent, const float* mask, const long long* xlen, const long long* ylen, float* path,
                                float* dur, float* cum, void* ws, int B, int Ty, int Tx, cudaStream_t s);
cudaError_t launch_mas_losses(const float* y, const float* mu_y, const float* y_mask, const float* logw, const float* x_mask,
                              const float* dur, const long long* x_lengths, void* ws, int B, int M, int Ty, int Tx, float* prior_loss,
                              float* dur_loss, cudaStream_t s);

// ----------------------------------------------------------------------------------------------
// attention (attention.cu): qkv (BB, T, 3H) fp32 -> out (BB, T, H); partial RoPE fused on load.
// ----------------------------------------------------------------------------------------------
struct AttnArgs {
    const float* qkv = nullptr;       // SIMT engine: raw fp32 projections (RoPE applied on load)
    const bf16* qkv_hi = nullptr;     // tensor-core engine: RoPE'd, q-scaled split planes (BB, T, 3H)
    const bf16* qkv_lo = nullptr;
    const float* rope_cs = nullptr;   // (T, 16, 2); SIMT engine: nullptr = no RoPE
    const float* mask = nullptr;      // (B, T)
    const int* kvlen = nullptr;       // (B) 1 + last index with mask != 0
    const int* prefix = nullptr;      // (B) first index with mask == 0 (T if none): keys below it need no mask test
    float* out_f32 = nullptr; bf16* out_hi = nullptr; bf16* out_lo = nullptr;
    int BB = 0, B = 1, T = 0, H = 0, n_heads = 0;
};
cudaError_t launch_attention_simt(const AttnArgs& a, cudaStream_t s);

// tensor-core engine (attention_tc.cu)
cudaError_t launch_attention_tc(const AttnArgs& a, cudaStream_t s);
const char* attention_tc_last_error();

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch: every kernel of the path (1) lets its successor start launching
// immediately and (2) waits for ALL its predecessors to complete before its first global access, so
// launch latency, smem carve-up, barrier init and tensor-map prefetch of kernel N+1
// overlap the tail of kernel N.  Without the launch attribute both instructions are no-ops.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <class... KArgs, class... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: opt in once per (kernel, device), so that a
// second handle on another device of the same process launches with the raised limit too (`done` = one bit per device).
template <class K>
inline cudaError_t ensure_dyn_smem(K kernel, int bytes, std::atomic<uint64_t>& done) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const uint64_t bit = 1ull << (dev & 63);
    if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
    return e;
}

__device__ __forceinline__ float silu_f(float v) { return __fdividef(v, 1.0f + __expf(-v)); }
// SiLU on the two SFU approximations directly (ex2.approx + rcp.approx, ~3e-7 relative): no range-fix-up code around them.
// v -> -inf: ex2(+big) = +inf, rcp(inf) = 0, v * 0 = -0;  v -> +inf: ex2(-big) = 0, v * rcp(1) = v.
__device__ __forceinline__ float silu_fast(float v) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return v * r;
}
__device__ __forceinline__ float gelu_f(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f)); }
// nn.Mish: v tanh(softplus(v)) with torch's softplus (threshold 20: softplus(v) = v above it), accurate libm forms
__device__ __forceinline__ float mish_f(float v) { return v * tanhf(v > 20.f ? v : log1pf(expf(v))); }

// two floats -> packed (hi0,hi1) and (lo0,lo1) bf16x2 words: one cvt.rn.bf16x2 per plane
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<uint32_t*>(&h);
    const float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xFFFF0000u);
    __nv_bfloat162 l = __floats2bfloat162_rn(a - ha, b - hb);
    lo = *reinterpret_cast<uint32_t*>(&l);
}

// two floats -> one packed fp16x2 word, saturated to the finite fp16 range (fp16 overflows at 65504 where bf16 does not)
__device__ __forceinline__ uint32_t pack_f16x2_sat(float a, float b) {
    a = fminf(fmaxf(a, -65504.f), 65504.f); b = fminf(fmaxf(b, -65504.f), 65504.f);
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));       // low half = a, high half = b
    return r;
}

__device__ __forceinline__ void split_bf16(float v, bf16& hi, bf16& lo) {
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

}  // namespace st
