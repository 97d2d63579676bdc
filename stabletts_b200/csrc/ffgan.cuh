// Row / packing kernels of the FireflyGAN vocoder (ffgan.cu); the contractions run on the conv-GEMM engines.
#pragma once
#include "common.cuh"

namespace st {

// W = g * v / ||v|| per dim-0 row of `rows` x `len` (torch weight_norm, dim = 0)
cudaError_t launch_weight_norm_fold(const float* g, const float* v, float* out, int rows, int len, cudaStream_t s);
// ConvTranspose1d weight (Cin, Cout, 2u) -> packed 3-tap conv weight out[tau][r * Cout + c][i] (K = Cin contiguous),
// = w[i, c, r + u/2 - (tau - 1) u] where that kernel index lies in [0, 2u), else 0
cudaError_t launch_pack_polyphase(const float* w, float* out, int Cin, int Cout, int u, cudaStream_t s);
// ParralelBlock mean + the SiLU that follows it: v = silu((r0 + r1 + r2) / 3) -> out_f32 and / or split planes (n % 4 == 0)
cudaError_t launch_mean3_silu(const float* r0, const float* r1, const float* r2, long n, float* out_f32, bf16* out_hi,
                              bf16* out_lo, cudaStream_t s);
// conv_post + tanh on the SiLU'd last stage: x (B, L, C) token-major, w (1, C, k) reference layout -> audio (B, L)
cudaError_t launch_post_conv_tanh(const float* x, const float* w, const float* bias, int B, long L, int C, int k, float* audio,
                                  cudaStream_t s);

}  // namespace st
