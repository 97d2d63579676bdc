// HBM-bound row kernels of the vocoder hand-off (SURVEY.md §8 row f4; reference: vocoders/vocos/models/):
//   dwconv_ln_kernel  depthwise k=7 conv along frames (module.py:21,36) + LayerNorm(C, affine, eps 1e-6) (:23,38),
//                     or the LayerNorm alone (backbone.py:31,43,51,55) — one warp per frame, warp-shuffle reductions
//   spectrum_kernel   ISTFTHead's (log-magnitude, phase) -> (re, im) with the 1e2 clip (head.py:103-113), written as the
//                     split-bf16 A operand of the inverse-DFT GEMM
//   idft_basis_kernel the windowed inverse-real-DFT basis (what irfft + window computes, head.py:62-63) as a GEMM weight
//   overlap_add_kernel fold + window-envelope normalisation + "same" trimming (head.py:66-81) as a 4-frame gather
// The dense contractions between them (embed conv k=7, pwconv1 + GELU, pwconv2 + layer scale + residual, head Linear,
// frames = [re | im] · W) run on the conv-GEMM engine of gemm_tc.cu.
#include "common.cuh"
#include "vocos.cuh"

namespace st {

template <int C>
__global__ void __launch_bounds__(256) dwconv_ln_kernel(DwLnArgs a) {
    pdl_trigger(); pdl_wait();
    constexpr int G = C / 128;         // float4 groups per lane
    const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long rows = (long)a.B * a.T;
    if (warp >= rows) return;
    float v[G * 4];
    dwconv_or_load<C>(a.x, a.dw_w, a.dw_b, a.B, a.T, warp, lane, v);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < G * 4; ++j) sum += v[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * (1.0f / C);
    float var = 0.f;
#pragma unroll
    for (int j = 0; j < G * 4; ++j) { const float d = v[j] - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = rsqrtf(var * (1.0f / C) + a.eps);
#pragma unroll
    for (int j = 0; j < G; ++j) {
        const int c = (j * 32 + lane) * 4;
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(a.ln_w + c));
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.ln_b + c));
        const float u0 = (v[j * 4 + 0] - mean) * rstd * w4.x + b4.x, u1 = (v[j * 4 + 1] - mean) * rstd * w4.y + b4.y;
        const float u2 = (v[j * 4 + 2] - mean) * rstd * w4.z + b4.z, u3 = (v[j * 4 + 3] - mean) * rstd * w4.w + b4.w;
        const long o = warp * C + c;
        if (a.out_f32) *reinterpret_cast<float4*>(a.out_f32 + o) = make_float4(u0, u1, u2, u3);
        if (a.out_hi) {
            uint32_t h01, l01, h23, l23;
            split_bf16x2(u0, u1, h01, l01); split_bf16x2(u2, u3, h23, l23);
            *reinterpret_cast<uint2*>(a.out_hi + o) = make_uint2(h01, h23);
            *reinterpret_cast<uint2*>(a.out_lo + o) = make_uint2(l01, l23);
        }
    }
}

cudaError_t launch_dwconv_ln(const DwLnArgs& a, cudaStream_t s) {
    const long rows = (long)a.B * a.T;
    if (rows == 0) return cudaSuccess;
    const dim3 grid((unsigned)((rows * 32 + 255) / 256)), block(256);
    switch (a.C) {
        case 128: return launch_k(dwconv_ln_kernel<128>, grid, block, 0, s, a);
        case 256: return launch_k(dwconv_ln_kernel<256>, grid, block, 0, s, a);
        case 384: return launch_k(dwconv_ln_kernel<384>, grid, block, 0, s, a);
        case 512: return launch_k(dwconv_ln_kernel<512>, grid, block, 0, s, a);
        case 768: return launch_k(dwconv_ln_kernel<768>, grid, block, 0, s, a);
        case 1024: return launch_k(dwconv_ln_kernel<1024>, grid, block, 0, s, a);
        default: return cudaErrorInvalidValue;
    }
}

// head: x (rows, Nh) with log-magnitudes at columns [0, K) and phases at [Kp, Kp + K)  ->  S (rows, K2) split planes
// (+ fp32 for the SIMT engine) with re = min(exp(m), 1e2) cos(p) at [0, K), im = ... sin(p) at [K2/2, K2/2 + K), 0 elsewhere.
__global__ void spectrum_kernel(const float* __restrict__ x, int Nh, int Kp, int K, int K2, long rows, float* __restrict__ s_f32,
                                bf16* __restrict__ s_hi, bf16* __restrict__ s_lo) {
    pdl_trigger(); pdl_wait();
    const int half = K2 / 2;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * half) return;
    const long r = i / half;
    const int k = (int)(i - r * half);
    float re = 0.f, im = 0.f;
    if (k < K) {
        const float m = fminf(expf(x[r * Nh + k]), 1e2f);             // head.py:105-106
        float sn, cs;
        sincosf(x[r * Nh + Kp + k], &sn, &cs);                        // :108-109
        re = m * cs; im = m * sn;                                     // :113
    }
    const long o0 = r * K2 + k, o1 = o0 + half;
    if (s_f32) { s_f32[o0] = re; s_f32[o1] = im; }
    if (s_hi) {
        bf16 h, l;
        split_bf16(re, h, l); s_hi[o0] = h; s_lo[o0] = l;
        split_bf16(im, h, l); s_hi[o1] = h; s_lo[o1] = l;
    }
}

cudaError_t launch_spectrum(const float* x, int Nh, int Kp, int K, int K2, long rows, float* s_f32, bf16* s_hi, bf16* s_lo,
                            cudaStream_t s) {
    const long n = rows * (K2 / 2);
    if (n == 0) return cudaSuccess;
    return launch_k(spectrum_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, x, Nh, Kp, K, K2, rows, s_f32, s_hi, s_lo);
}

// W[n][kk], n < n_fft (GEMM output column = sample within the frame), kk < K2 (GEMM K):
//   kk = k        < K : window[n] * c_k * cos(2 pi k n / n_fft) / n_fft
//   kk = K2/2 + k     : -window[n] * c_k * sin(2 pi k n / n_fft) / n_fft, and 0 for the DC / Nyquist bins (irfft ignores them)
// with c_0 = c_{K-1} = 1, c_k = 2 otherwise — so that frames = [re | im] · W^T equals window * irfft(S, norm="backward").
__global__ void idft_basis_kernel(const float* __restrict__ window, int n_fft, int K, int K2, float* __restrict__ W) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n_fft * K2) return;
    const int n = (int)(i / K2), kk = (int)(i - (long)n * K2);
    const int half = K2 / 2;
    const int k = kk < half ? kk : kk - half;
    double v = 0.0;
    if (k < K) {
        const double c = (k == 0 || k == K - 1) ? 1.0 : 2.0;
        const long kn = ((long)k * n) % n_fft;                       // exact argument reduction
        double sn, cs;
        sincospi(2.0 * (double)kn / (double)n_fft, &sn, &cs);
        if (kk < half) v = c * cs / n_fft;
        else v = (k == 0 || k == K - 1) ? 0.0 : -c * sn / n_fft;
        v *= (double)window[n];
    }
    W[i] = (float)v;
}

cudaError_t launch_idft_basis(const float* window, int n_fft, int K, int K2, float* W, cudaStream_t s) {
    const long n = (long)n_fft * K2;
    idft_basis_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(window, n_fft, K, K2, W);
    return cudaGetLastError();
}

// audio[b, s] = (sum over the n_fft/hop frames covering sample s of frames[b, t, n]) / (sum of window[n]^2 over the same
// frames), s in [0, T*hop): position s + pad of the un-trimmed fold output, pad = (n_fft - hop) / 2 (head.py:46,66-81)
__global__ void overlap_add_kernel(const float* __restrict__ frames, const float* __restrict__ window, int B, int T, int n_fft,
                                   int hop, float* __restrict__ audio) {
    pdl_trigger(); pdl_wait();
    const long L = (long)T * hop;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * L) return;
    const int b = (int)(i / L);
    const long s = i - (long)b * L;
    const long pos = s + (n_fft - hop) / 2;
    const int tq = (int)(pos / hop);
    float acc = 0.f, env = 0.f;
    for (int j = 0; j < n_fft / hop; ++j) {
        const int t = tq - j;
        const int n = (int)(pos - (long)t * hop);
        if (t >= 0 && t < T) {
            acc += frames[((long)b * T + t) * n_fft + n];
            const float w = __ldg(window + n);
            env = fmaf(w, w, env);
        }
    }
    audio[i] = acc / env;
}

cudaError_t launch_overlap_add(const float* frames, const float* window, int B, int T, int n_fft, int hop, float* audio,
                               cudaStream_t s) {
    const long n = (long)B * T * hop;
    if (n == 0) return cudaSuccess;
    return launch_k(overlap_add_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, frames, window, B, T, n_fft, hop, audio);
}

}  // namespace st
