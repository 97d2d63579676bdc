// Row and packing kernels of the FireflyGAN vocoder (reference: vocoders/ffgan/head.py):
//   weight_norm_fold_kernel  W = g v / ||v|| (the weight_norm parametrization, folded once at st_finalize_weights)
//   pack_polyphase_kernel    ConvTranspose1d(k = 2u, stride u, padding u/2) as a 3-tap conv at the input rate with
//                            N = u * C_out (oracle/ffgan_ref.py polyphase_weight)
//   mean3_silu_kernel        ParralelBlock's mean of three ResBlock1 outputs (head.py:133-134) in a fixed order, then the
//                            SiLU of the next ups / conv_post (head.py:230, 244)
//   post_conv_tanh_kernel    conv_post (C -> 1, k = 13) + tanh (head.py:245-246), written straight to (B, T * 512)
#include "ffgan.cuh"

namespace st {

__global__ void __launch_bounds__(256) weight_norm_fold_kernel(const float* __restrict__ g, const float* __restrict__ v,
                                                               float* __restrict__ out, int len) {
    __shared__ double red[8];
    const long row = blockIdx.x;
    const float* vr = v + row * len;
    double ss = 0.0;
    for (int i = threadIdx.x; i < len; i += blockDim.x) ss += (double)vr[i] * vr[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    double tot = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    const float scale = (float)((double)g[row] / sqrt(tot));
    for (int i = threadIdx.x; i < len; i += blockDim.x) out[row * len + i] = vr[i] * scale;
}

cudaError_t launch_weight_norm_fold(const float* g, const float* v, float* out, int rows, int len, cudaStream_t s) {
    weight_norm_fold_kernel<<<rows, 256, 0, s>>>(g, v, out, len);
    return cudaGetLastError();
}

__global__ void pack_polyphase_kernel(const float* __restrict__ w, float* __restrict__ out, int Cin, int Cout, int u) {
    const long total = 3L * u * Cout * Cin;
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int i = (int)(idx % Cin);
    const long rn = idx / Cin;
    const int n = (int)(rn % ((long)u * Cout)), tau = (int)(rn / ((long)u * Cout));
    const int r = n / Cout, c = n - r * Cout;
    const int kk = r + u / 2 - (tau - 1) * u;
    out[idx] = (kk >= 0 && kk < 2 * u) ? w[((long)i * Cout + c) * 2 * u + kk] : 0.f;
}

cudaError_t launch_pack_polyphase(const float* w, float* out, int Cin, int Cout, int u, cudaStream_t s) {
    const long total = 3L * u * Cout * Cin;
    pack_polyphase_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w, out, Cin, Cout, u);
    return cudaGetLastError();
}

__global__ void mean3_silu_kernel(const float4* __restrict__ r0, const float4* __restrict__ r1, const float4* __restrict__ r2,
                                  long n4, float* __restrict__ out_f32, bf16* __restrict__ out_hi, bf16* __restrict__ out_lo) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 a = r0[i], b = r1[i], c = r2[i];
    const float v0 = silu_f((a.x + b.x + c.x) / 3.0f), v1 = silu_f((a.y + b.y + c.y) / 3.0f);
    const float v2 = silu_f((a.z + b.z + c.z) / 3.0f), v3 = silu_f((a.w + b.w + c.w) / 3.0f);
    if (out_f32) reinterpret_cast<float4*>(out_f32)[i] = make_float4(v0, v1, v2, v3);
    if (out_hi) {
        uint32_t h01, l01, h23, l23;
        split_bf16x2(v0, v1, h01, l01); split_bf16x2(v2, v3, h23, l23);
        reinterpret_cast<uint2*>(out_hi)[i] = make_uint2(h01, h23);
        reinterpret_cast<uint2*>(out_lo)[i] = make_uint2(l01, l23);
    }
}

cudaError_t launch_mean3_silu(const float* r0, const float* r1, const float* r2, long n, float* out_f32, bf16* out_hi,
                              bf16* out_lo, cudaStream_t s) {
    const long n4 = n / 4;
    if (n % 4) return cudaErrorInvalidValue;
    if (n4 == 0) return cudaSuccess;
    return launch_k(mean3_silu_kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, s, reinterpret_cast<const float4*>(r0),
                    reinterpret_cast<const float4*>(r1), reinterpret_cast<const float4*>(r2), n4, out_f32, out_hi, out_lo);
}

// one thread per output sample; the (C, k) weights sit in shared memory, C = 16 channels are four float4 loads per tap
template <int C, int K>
__global__ void __launch_bounds__(256) post_conv_tanh_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                             const float* __restrict__ bias, int B, long L, float* __restrict__ audio) {
    pdl_trigger(); pdl_wait();
    __shared__ float ws[K][C];
    for (int i = threadIdx.x; i < C * K; i += blockDim.x) ws[i % K][i / K] = w[i];     // w[c * K + k] -> ws[k][c]
    __syncthreads();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * L) return;
    const long b = i / L, s = i - b * L;
    float acc = bias[0];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const long t = s + k - K / 2;
        if (t < 0 || t >= L) continue;
        const float4* xr = reinterpret_cast<const float4*>(x + (b * L + t) * C);
#pragma unroll
        for (int c4 = 0; c4 < C / 4; ++c4) {
            const float4 v = __ldg(xr + c4);
            acc = fmaf(ws[k][4 * c4 + 0], v.x, acc); acc = fmaf(ws[k][4 * c4 + 1], v.y, acc);
            acc = fmaf(ws[k][4 * c4 + 2], v.z, acc); acc = fmaf(ws[k][4 * c4 + 3], v.w, acc);
        }
    }
    audio[i] = tanhf(acc);
}

cudaError_t launch_post_conv_tanh(const float* x, const float* w, const float* bias, int B, long L, int C, int k, float* audio,
                                  cudaStream_t s) {
    if (C != 16 || k != 13) return cudaErrorInvalidValue;                     // the reference's one configuration
    const long n = (long)B * L;
    if (n == 0) return cudaSuccess;
    return launch_k(post_conv_tanh_kernel<16, 13>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, x, w, bias, B, L, audio);
}

}  // namespace st
