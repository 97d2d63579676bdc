// Row kernels of the multi-period discriminator (vocoders/vocos/models/discriminator.py::DiscriminatorP); the dense
// convolutions run on the conv-GEMM engines (mpd_api.cu).  Layouts:
//   NCHW    the reference's (B, C, H, p) fp32 tensors: the fmaps the caller keeps, their gradients
//   rows    token-major (BB = B·p columns, rows, C): column bb = b·p + j is one independent 1-D sequence along H
//   Planes  a rows tensor as the selected engine reads it: fp32 (SIMT) or split-bf16 hi / lo (wgmma)
#pragma once
#include "common.cuh"

namespace st {

struct MpdPlanes { float* f = nullptr; bf16* hi = nullptr; bf16* lo = nullptr; };

struct MpdGeo { int B = 0, p = 0; long long L = 0; int Hin = 0; };   // Hin = (L + reflect pad) / p

// conv 0 (1 -> 32, (5, 1), stride 3, pad 2) + leaky ReLU on the reflect-padded input x (B, L):
// fmap0 (B, 32, H0, p) and the rows of conv 1's input, (BB, R, 32) with rows [H0, R) zero
cudaError_t launch_mpd_conv0_fwd(const float* x, MpdGeo g, int H0, int R, const float* w, const float* b, float* fmap0,
                                 MpdPlanes out, cudaStream_t s);
// leaky ReLU of the GEMM output Y (BB, H, C) -> fmap (B, C, H, p); when `out` has a plane, also rows (BB, R, C), [H, R) zero
// (slope 1: the layout change alone, for the single-conv test hook)
cudaError_t launch_mpd_act_fwd(const float* Y, MpdGeo g, int H, int C, int R, float* fmap, MpdPlanes out, cudaStream_t s,
                               float slope = 0.1f);
// fmap (B, C, H, p) -> rows (BB, R, C), rows [H, R) zero, without an activation (the single-conv test hook's inputs)
cudaError_t launch_mpd_nchw_to_rows(const float* fmap, MpdGeo g, int H, int C, int R, MpdPlanes out, cudaStream_t s);
// conv_post (1024 -> 1, (3, 1), pad 1) on fmap4 (B, 1024, H, p) -> post (B, 1, H, p)
cudaError_t launch_mpd_post_fwd(const float* fmap4, MpdGeo g, int H, const float* w, const float* b, float* post, cudaStream_t s);

// weight (Cout, Cin, 5) -> packed fp32 [taps][N][K] of one of the four GEMM packings (MPD_PACK_*, see mpd.cu)
enum { MPD_PACK_FWD_S3 = 0, MPD_PACK_FWD_S1 = 1, MPD_PACK_DGRAD_S3 = 2, MPD_PACK_DGRAD_S1 = 3 };
cudaError_t launch_mpd_pack(const float* w, int Cout, int Cin, int mode, float* out, cudaStream_t s);

// d fmap4 from conv_post: G (BB, H, 1024) = Σ_k w[c, k] gpost[h - k + 1]
cudaError_t launch_mpd_post_dgrad(const float* gpost, MpdGeo g, int H, const float* w, float* G, cudaStream_t s);
// conv_post's weight and bias gradients, fixed-order block reductions
cudaError_t launch_mpd_post_wgrad(const float* gpost, const float* fmap4, MpdGeo g, int H, float* dw, float* db, cudaStream_t s);
// dZ = (G + gfmap) · leaky'(fmap) of one hidden layer (H rows, C channels).  G is rows-laid with `Rg` rows per column and
// row h at Rg-row `h + off`; gfmap (NCHW) may be null; a null fmap means slope 1 (the test hook).  Writes any of: dZ rows
// (BB, H + 1, C) with row H zero, the transposed planes dZT [C][Kr] (column r = bb·H + h; the caller zeroes r >= BB·H), and
// dZ in NCHW.
cudaError_t launch_mpd_act_bwd(const float* G, int Rg, int off, const float* gfmap, const float* fmap, MpdGeo g, int H, int C,
                               MpdPlanes dz, MpdPlanes dzT, long long Kr, float* dz_nchw, cudaStream_t s);
// the wgrad GEMM's W operand [5 Cin + 8][Kr]: row (k, c), column r = bb·H + o holds X[bb, s·o + k - 2, c] (zero outside
// [0, Hx)), from the layer input X = fmap (B, Cin, Hx, p); row 5 Cin is ones (the bias gradient), the last 7 rows zero
cudaError_t launch_mpd_im2col_t(const float* fmap, MpdGeo g, int Hx, int Cin, int H, int stride, long long Kr, MpdPlanes out,
                                cudaStream_t s);
// dWp [Cout][5 Cin + 8] -> dW (Cout, Cin, 5) and db (Cout)
cudaError_t launch_mpd_unpack_wgrad(const float* dWp, int Cout, int Cin, float* dw, float* db, cudaStream_t s);
// conv 0's weight / bias gradients from dz0 (B, 32, H0, p), fixed-order block reductions
cudaError_t launch_mpd_conv0_wgrad(const float* dz0, const float* x, MpdGeo g, int H0, float* dw, float* db, cudaStream_t s);
// conv 0's input gradient, with the reflect pad's adjoint folded in: gx (B, L)
cudaError_t launch_mpd_conv0_dgrad(const float* dz0, const float* w, MpdGeo g, int H0, float* gx, cudaStream_t s);

}  // namespace st
