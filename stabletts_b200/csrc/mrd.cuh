// Kernels of the multi-resolution discriminator (vocoders/vocos/models/discriminator.py:112-171, DiscriminatorR); the
// 32 -> 32 band convs run on the conv-GEMM engines (mrd_api.cu).  Layouts:
//   spec    (B, 2 = [re, im], T', F) fp32: the reference's view_as_real + permute(0, 3, 2, 1) of the STFT
//   NCHW    the reference's (B, 32, T', W) fp32 band activations: the fmaps the caller keeps, their gradients
//   rows    token-major (BB = B T' sequences, G groups, K): sequence bb = b T' + t is one row of a band along F.  Group g
//           holds `lanes` consecutive columns [lanes g, lanes g + lanes) of the three time rows t - 1, t, t + 1:
//           channel (l 3 + dt) 32 + c = X[b, c, t + dt - 1, lanes g + l], zero outside [0, T') x [0, W)
//   Planes  a rows tensor as the selected engine reads it: fp32 (SIMT) or split-bf16 hi / lo (wgmma)
#pragma once
#include "common.cuh"

namespace st {

struct MrdPlanes { float* f = nullptr; bf16* hi = nullptr; bf16* lo = nullptr; };

struct MrdGeo { int B = 0, T = 0; };     // T = T' frames of the STFT

// A band slice of a (B, C, T', Wtot) tensor: columns [off, off + W).
struct MrdBand { int off = 0, W = 0; };

// ---- STFT -------------------------------------------------------------------------------------------------------------
// spec (B, 2, T', n_fft / 2 + 1) of x (B, L): centred frames (reflect pad n_fft / 2), the given window, mel.cuh's FFT
cudaError_t launch_mrd_stft(const float* x, long long L, MrdGeo g, int log2M, const float* window, const float2* tw, float* spec,
                            cudaStream_t s);
// frame gradients gf (B, T', n_fft) = window · (the rfft adjoint of gspec (B, 2, T', F)); mel_loss's gather folds them
cudaError_t launch_mrd_stft_adj(const float* gspec, MrdGeo g, int log2M, const float* window, const float2* tw, float* gf,
                                cudaStream_t s);

// ---- layer 0 (2 -> 32, (3, 9), pad (1, 4)) and conv_post (32 -> 1, (3, 3), pad (1, 1)) in fp32 ------------------------
// fmap0 (B, 32, T', W) = leaky(conv(spec[..., band]))
cudaError_t launch_mrd_conv0_fwd(const float* spec, int F, MrdGeo g, MrdBand bd, const float* w, const float* b, float* fmap0,
                                 cudaStream_t s);
// gspec[..., band] = the input gradient of dz0 (B, 32, T', W)
cudaError_t launch_mrd_conv0_dgrad(const float* dz0, MrdGeo g, MrdBand bd, int F, const float* w, float* gspec, cudaStream_t s);
// dw (32, 2, 3, 9), db (32): fixed-order block reductions
cudaError_t launch_mrd_conv0_wgrad(const float* dz0, const float* spec, int F, MrdGeo g, MrdBand bd, float* dw, float* db,
                                   cudaStream_t s);
// The five band outputs (B, 32, T', W_k) as one tensor concatenated along F, for conv_post.
struct MrdCat { const float* f[5]; int off[6]; };          // band k holds columns [off[k], off[k + 1])
cudaError_t launch_mrd_post_fwd(MrdCat cat, MrdGeo g, const float* w, const float* b, float* post, cudaStream_t s);
// G (B, 32, T', W) of band `k` = conv_post's input gradient from gpost (B, 1, T', Wtot), reading across the seams
cudaError_t launch_mrd_post_dgrad(const float* gpost, MrdCat cat, int k, MrdGeo g, const float* w, float* G, cudaStream_t s);
cudaError_t launch_mrd_post_wgrad(const float* gpost, MrdCat cat, MrdGeo g, float* dw, float* db, cudaStream_t s);

// ---- the GEMM layers 1-4 ----------------------------------------------------------------------------------------------
// Layer kinds: lanes 2, taps 5 (the (3, 9) stride-(1, 2) convs 1-3) or lanes 1, taps 3 (the (3, 3) conv 4).  Kx = lanes 96.
// rows (BB, G, Kx) of X (B, 32, T', W), G = ceil(W / lanes)
cudaError_t launch_mrd_expand(const float* X, MrdGeo g, int W, int lanes, MrdPlanes out, cudaStream_t s);
// weight (32, 32, 3, kw) -> packed fp32: forward [taps][32][Kx] (tap t, channel (l, dt, c) = w[n, c, dt, lanes t + l],
// zero when lanes t + l >= kw), or dgrad [taps][Kx][32] = the forward's tap taps - 1 - t transposed
cudaError_t launch_mrd_pack(const float* w, int lanes, int dgrad, float* out, cudaStream_t s);
// fmap (B, 32, T', W) = leaky(Y (BB, W, 32)) (slope 1: the layout change alone, for the single-conv hook)
cudaError_t launch_mrd_act_fwd(const float* Y, MrdGeo g, int W, float* fmap, cudaStream_t s, float slope = 0.1f);
// dZ = (G + gfmap) · leaky'(fmap), all (B, 32, T', W); gfmap may be null, a null fmap means slope 1.  Writes any of: dZ rows
// (BB, W, 32), the transposed planes dZT [32][Kr] (column r = bb W + o; the caller zeroes r >= BB W) and dZ in NCHW.
cudaError_t launch_mrd_act_bwd(const float* G, const float* gfmap, const float* fmap, MrdGeo g, int W, MrdPlanes dz, MrdPlanes dzT,
                               long long Kr, float* dz_nchw, cudaStream_t s);
// the adjoint of launch_mrd_expand: dX (B, 32, T', W) = Σ_dt dR (BB, G, Kx) in ascending dt
cudaError_t launch_mrd_fold(const float* dR, MrdGeo g, int W, int lanes, float* dX, cudaStream_t s);
// the wgrad GEMM's W operand [taps Kx + 8][Kr]: row (t, kx), column r = bb G + o holds rows(X)[bb, o + t - taps / 2, kx]
// (zero outside [0, G)); row taps Kx is ones (the bias gradient), the last 7 rows zero
cudaError_t launch_mrd_im2col_t(const float* X, MrdGeo g, int W, int lanes, long long Kr, MrdPlanes out, cudaStream_t s);
// dWp [32][taps Kx + 8] -> dw (32, 32, 3, kw), db (32)
cudaError_t launch_mrd_unpack_wgrad(const float* dWp, int lanes, float* dw, float* db, cudaStream_t s);

__host__ __device__ inline int mrd_taps(int lanes) { return lanes == 2 ? 5 : 3; }
__host__ __device__ inline int mrd_kw(int lanes) { return lanes == 2 ? 9 : 3; }

}  // namespace st
