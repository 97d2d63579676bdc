// Row kernels of the vocoder hand-off (vocos.cu) and of its backward pass (vocos_grad.cu); orchestration in vocos_api.cu.
#pragma once
#include "common.cuh"

namespace st {

struct DwLnArgs {
    const float* x = nullptr;        // (B, T, C) fp32
    const float* dw_w = nullptr;     // [7][C] depthwise taps (null: LayerNorm only)
    const float* dw_b = nullptr;     // [C]
    const float* ln_w = nullptr; const float* ln_b = nullptr;
    float* out_f32 = nullptr; bf16* out_hi = nullptr; bf16* out_lo = nullptr;
    int B = 0, T = 0, C = 0;
    float eps = 1e-6f;
};
cudaError_t launch_dwconv_ln(const DwLnArgs& a, cudaStream_t s);
cudaError_t launch_spectrum(const float* x, int Nh, int Kp, int K, int K2, long rows, float* s_f32, bf16* s_hi, bf16* s_lo,
                            cudaStream_t s);
cudaError_t launch_idft_basis(const float* window, int n_fft, int K, int K2, float* W, cudaStream_t s);
cudaError_t launch_overlap_add(const float* frames, const float* window, int B, int T, int n_fft, int hop, float* audio,
                               cudaStream_t s);

// The LayerNorm input of row `row` (one warp, lane `lane`, channels (j 32 + lane) 4 + e in v[j 4 + e]): with dw_w, the
// depthwise conv y[t, c] = bias[c] + sum_k w[k][c] x[t + k - 3, c], zero padded at the utterance's edges; else x itself.
// The forward (dwconv_ln_kernel) and the backward (ln_bwd_kernel) share it, so both see the same bits.
template <int C>
__device__ __forceinline__ void dwconv_or_load(const float* x, const float* dw_w, const float* dw_b, int B, int T, long row,
                                               int lane, float* v) {
    constexpr int G = C / 128;
    if (dw_w) {
        const int b = (int)(row / T), t = (int)(row - (long)b * T);
#pragma unroll
        for (int j = 0; j < G; ++j) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(dw_b + (j * 32 + lane) * 4));
            v[j * 4 + 0] = b4.x; v[j * 4 + 1] = b4.y; v[j * 4 + 2] = b4.z; v[j * 4 + 3] = b4.w;
        }
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            const int ts = t + k - 3;
            if (ts < 0 || ts >= T) continue;             // warp-uniform
            const float* xr = x + ((long)b * T + ts) * C;
            const float* wr = dw_w + (long)k * C;
#pragma unroll
            for (int j = 0; j < G; ++j) {
                const int c = (j * 32 + lane) * 4;
                const float4 x4 = __ldg(reinterpret_cast<const float4*>(xr + c));
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(wr + c));
                v[j * 4 + 0] = fmaf(w4.x, x4.x, v[j * 4 + 0]); v[j * 4 + 1] = fmaf(w4.y, x4.y, v[j * 4 + 1]);
                v[j * 4 + 2] = fmaf(w4.z, x4.z, v[j * 4 + 2]); v[j * 4 + 3] = fmaf(w4.w, x4.w, v[j * 4 + 3]);
            }
        }
    } else {
        const float* xr = x + row * C;
#pragma unroll
        for (int j = 0; j < G; ++j) {
            const float4 x4 = __ldg(reinterpret_cast<const float4*>(xr + (j * 32 + lane) * 4));
            v[j * 4 + 0] = x4.x; v[j * 4 + 1] = x4.y; v[j * 4 + 2] = x4.z; v[j * 4 + 3] = x4.w;
        }
    }
}

// ---- backward (vocos_grad.cu) ----
// dF (B T, n_fft): the gradient of the frames for the audio gradient g (B, T hop)
cudaError_t launch_frame_grad(const float* g, const float* window, int B, int T, int n_fft, int hop, float* dF, cudaStream_t s);
// dS (rows, K2) = (dre | dim), x = the head output (rows, Nh) -> dx (rows, Nh): dlogmag at [0, K), dphase at [Kp, Kp + K), 0 else
cudaError_t launch_spectrum_grad(const float* dS, const float* x, int Nh, int Kp, int K, int K2, long rows, float* dx,
                                 cudaStream_t s);
struct LnBwdArgs {
    const float* x = nullptr;        // (B, T, C) the LayerNorm input, or the depthwise conv's input with dw_w
    const float* dw_w = nullptr;     // [7][C] (null: LayerNorm only)
    const float* dw_b = nullptr;
    const float* ln_w = nullptr;
    const float* g = nullptr;        // (B, T, C) the output gradient
    float* dx = nullptr;             // (B, T, C) the LayerNorm input's gradient (may not alias g)
    float* zhat = nullptr;           // (B, T, C) or null: the normalised input, for the affine gradients
    int B = 0, T = 0, C = 0;         // C = 512, 768 or 1024
    float eps = 1e-6f;
};
cudaError_t launch_ln_bwd(const LnBwdArgs& a, cudaStream_t s);
// dx (B, T, C) += sum_k w[k][c] dz[t + 3 - k, c]; w = [7][C]; C % 4 == 0
cudaError_t launch_dwconv_adj(const float* dz, const float* w, int B, int T, int C, float* dx, cudaStream_t s);
// out[c] = sum_r a[r, c] b[r, c] (b null: sum_r a[r, c]), a fixed-order sum over the rows
cudaError_t launch_col_sum(const float* a, const float* b, long rows, int C, float* out, cudaStream_t s);
// dw (C, 1, 7), db (C): the depthwise conv's weight and bias gradients of dz for the input x, both (B, T, C)
cudaError_t launch_dwconv_wgrad(const float* dz, const float* x, int B, int T, int C, float* dw, float* db, cudaStream_t s);
// y (rows, C) = x * gamma[c]
cudaError_t launch_scale_cols(const float* x, const float* gamma, long rows, int C, float* y, cudaStream_t s);
// dh = dg (Phi(h) + h phi(h)), n elements
cudaError_t launch_gelu_bwd(const float* dg, const float* h, long n, float* dh, cudaStream_t s);
struct TransposeArgs {
    const float* src_f32 = nullptr;  // (B, T, Cx) token-major: fp32, or the split planes src_hi / src_lo
    const bf16* src_hi = nullptr; const bf16* src_lo = nullptr;
    float* dst_f32 = nullptr;        // [Nd][Kr]: fp32 and / or split planes (split-plane sources: planes only)
    bf16* dst_hi = nullptr; bf16* dst_lo = nullptr;
    int B = 0, T = 0, Cx = 0;
    int taps = 1;                    // 1, or 7: row k Cx + c holds frame t + k - 3 of the same utterance
    int ones = 0;                    // row taps Cx is 1 for every real column
    int Nd = 0;                      // >= taps Cx (+ 1 with ones); rows past the data are 0
    long Kr = 0;                     // >= B T; columns past B T are 0
};
cudaError_t launch_transpose_rows(const TransposeArgs& a, cudaStream_t s);
// dWp [Np][taps Cx + 8] -> gw (Nref, Cx, taps), gb (Nref); split > 0: reference row n >= split reads packed row Kp + n - split
cudaError_t launch_unpack_wgrad(const float* dWp, int Nref, int Cx, int taps, int split, int Kp, float* gw, float* gb,
                                cudaStream_t s);

}  // namespace st
