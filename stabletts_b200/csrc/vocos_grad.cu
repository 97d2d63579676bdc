// fp32 row kernels of the Vocos generator's backward pass (DESIGN.md §8 row f12; orchestration in vocos_api.cu).  Every
// reduction over rows runs in a fixed order with no atomics, so a repeated backward is bitwise identical.
//   frame_grad_kernel     dF[t, n] = g[s] / env[s], s = t hop + n - pad inside [0, L), else 0: the adjoint of the
//                         overlap-add, envelope division and "same" trim (head.py:66-81)
//   spectrum_grad_kernel  (dre, dim) -> (dlogmag, dphase) of exp / clip / cos / sin (head.py:103-113), pad columns 0
//   ln_bwd_kernel         LayerNorm backward (affine, biased variance), recomputing the depthwise-conv output first for
//                         the block LayerNorms (module.py:36-38)
//   dwconv_adj_kernel     dx += the depthwise k = 7 conv's adjoint of dz (zero padding at each utterance's edges)
//   col_sum_kernel        out[c] = sum over rows of a[r, c] (* b[r, c]): LayerNorm affine and layer-scale gradients
//   dwconv_wgrad_kernel   the depthwise conv's weight (C, 1, 7) and bias gradients
//   scale_cols_kernel     dP = dX' * gamma (the layer scale, module.py:44)
//   gelu_bwd_kernel       dh = dG (Phi(h) + h phi(h)), the exact-erf GELU (module.py:40)
//   transpose_rows_kernel token-major rows -> transposed GEMM planes with Kr columns, optionally 7-tap shifted (the
//                         embed conv's input) and with a row of ones (the bias gradient): the W operand and the dY^T A
//                         operand of a weight-gradient GEMM
//   wgrad_unpack_kernel   a weight-gradient GEMM's [N][taps Cx + 8] output -> the reference's weight and bias layouts
#include "common.cuh"
#include "vocos.cuh"

namespace st {

__global__ void frame_grad_kernel(const float* __restrict__ g, const float* __restrict__ window, int B, int T, int n_fft,
                                  int hop, float* __restrict__ dF) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * T * n_fft) return;
    const long r = i / n_fft;
    const int n = (int)(i - r * n_fft);
    const int b = (int)(r / T), t = (int)(r - (long)b * T);
    const long L = (long)T * hop, pad = (n_fft - hop) / 2;
    const long s = (long)t * hop + n - pad;
    float v = 0.f;
    if (s >= 0 && s < L) {                 // the envelope exactly as overlap_add_kernel sums it
        const long pos = s + pad;
        const int tq = (int)(pos / hop);
        float env = 0.f;
        for (int j = 0; j < n_fft / hop; ++j) {
            const int tt = tq - j;
            if (tt >= 0 && tt < T) {
                const float w = __ldg(window + (int)(pos - (long)tt * hop));
                env = fmaf(w, w, env);
            }
        }
        v = g[(long)b * L + s] / env;
    }
    dF[i] = v;
}

cudaError_t launch_frame_grad(const float* g, const float* window, int B, int T, int n_fft, int hop, float* dF, cudaStream_t s) {
    const long n = (long)B * T * n_fft;
    if (n == 0) return cudaSuccess;
    return launch_k(frame_grad_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, g, window, B, T, n_fft, hop, dF);
}

__global__ void spectrum_grad_kernel(const float* __restrict__ dS, const float* __restrict__ x, int Nh, int Kp, int K, int K2,
                                     long rows, float* __restrict__ dx) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * Kp) return;
    const long r = i / Kp;
    const int k = (int)(i - r * Kp);
    float dm = 0.f, dp = 0.f;
    if (k < K) {
        const float e = expf(x[r * Nh + k]);
        const float a = fminf(e, 1e2f);
        float sn, cs;
        sincosf(x[r * Nh + Kp + k], &sn, &cs);
        const float dre = dS[r * K2 + k], dim = dS[r * K2 + K2 / 2 + k];
        const float da = dre * cs + dim * sn;
        dp = a * (dim * cs - dre * sn);
        dm = e <= 1e2f ? da * a : 0.f;      // torch.clip passes the gradient where the value equals the bound
    }
    dx[r * Nh + k] = dm;
    dx[r * Nh + Kp + k] = dp;
}

cudaError_t launch_spectrum_grad(const float* dS, const float* x, int Nh, int Kp, int K, int K2, long rows, float* dx,
                                 cudaStream_t s) {
    const long n = rows * Kp;
    if (n == 0) return cudaSuccess;
    return launch_k(spectrum_grad_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, dS, x, Nh, Kp, K, K2, rows, dx);
}

template <int C>
__global__ void __launch_bounds__(256) ln_bwd_kernel(LnBwdArgs a) {
    pdl_trigger(); pdl_wait();
    constexpr int G = C / 128;
    const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= (long)a.B * a.T) return;
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
    float gw[G * 4], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < G; ++j) {
        const int c = (j * 32 + lane) * 4;
        const float4 g4 = *reinterpret_cast<const float4*>(a.g + warp * C + c);
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(a.ln_w + c));
        gw[j * 4 + 0] = g4.x * w4.x; gw[j * 4 + 1] = g4.y * w4.y; gw[j * 4 + 2] = g4.z * w4.z; gw[j * 4 + 3] = g4.w * w4.w;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            v[j * 4 + e] = (v[j * 4 + e] - mean) * rstd;          // zhat
            s1 += gw[j * 4 + e];
            s2 = fmaf(gw[j * 4 + e], v[j * 4 + e], s2);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 * (1.0f / C), m2 = s2 * (1.0f / C);
#pragma unroll
    for (int j = 0; j < G; ++j) {
        const int c = (j * 32 + lane) * 4;
        const long o = warp * C + c;
        float d[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) d[e] = rstd * (gw[j * 4 + e] - m1 - v[j * 4 + e] * m2);
        *reinterpret_cast<float4*>(a.dx + o) = make_float4(d[0], d[1], d[2], d[3]);
        if (a.zhat) *reinterpret_cast<float4*>(a.zhat + o) = make_float4(v[j * 4 + 0], v[j * 4 + 1], v[j * 4 + 2], v[j * 4 + 3]);
    }
}

cudaError_t launch_ln_bwd(const LnBwdArgs& a, cudaStream_t s) {
    const long rows = (long)a.B * a.T;
    if (rows == 0) return cudaSuccess;
    const dim3 grid((unsigned)((rows * 32 + 255) / 256)), block(256);
    switch (a.C) {
        case 512: return launch_k(ln_bwd_kernel<512>, grid, block, 0, s, a);
        case 768: return launch_k(ln_bwd_kernel<768>, grid, block, 0, s, a);
        case 1024: return launch_k(ln_bwd_kernel<1024>, grid, block, 0, s, a);
        default: return cudaErrorInvalidValue;
    }
}

// dx[t, c] += sum_k w[k][c] dz[t + 3 - k, c] over the taps whose frame lies in the utterance; one thread per 4 channels
__global__ void dwconv_adj_kernel(const float* __restrict__ dz, const float* __restrict__ w, int B, int T, int C, float* dx) {
    pdl_trigger(); pdl_wait();
    const int C4 = C / 4;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * T * C4) return;
    const long r = i / C4;
    const int c = (int)(i - r * C4) * 4;
    const int b = (int)(r / T), t = (int)(r - (long)b * T);
    float4 acc = *reinterpret_cast<const float4*>(dx + r * C + c);
#pragma unroll
    for (int k = 0; k < 7; ++k) {
        const int ts = t + 3 - k;
        if (ts < 0 || ts >= T) continue;
        const float4 d4 = *reinterpret_cast<const float4*>(dz + ((long)b * T + ts) * C + c);
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(w + (long)k * C + c));
        acc.x = fmaf(w4.x, d4.x, acc.x); acc.y = fmaf(w4.y, d4.y, acc.y);
        acc.z = fmaf(w4.z, d4.z, acc.z); acc.w = fmaf(w4.w, d4.w, acc.w);
    }
    *reinterpret_cast<float4*>(dx + r * C + c) = acc;
}

cudaError_t launch_dwconv_adj(const float* dz, const float* w, int B, int T, int C, float* dx, cudaStream_t s) {
    const long n = (long)B * T * (C / 4);
    if (n == 0) return cudaSuccess;
    if (C % 4) return cudaErrorInvalidValue;
    return launch_k(dwconv_adj_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, dz, w, B, T, C, dx);
}

// Column reductions: a block of 32 columns x kColLanes row lanes; lane y sums rows y, y + kColLanes, ... in order, then
// lane 0 adds the lanes' partials in order.  The order depends on the row count only.
constexpr int kColLanes = 16;

__global__ void __launch_bounds__(32 * kColLanes) col_sum_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                 long rows, int C, float* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    __shared__ float part[kColLanes][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    float acc = 0.f;
    if (c < C)
        for (long r = threadIdx.y; r < rows; r += kColLanes) {
            const float v = a[r * C + c];
            acc = b ? fmaf(v, b[r * C + c], acc) : acc + v;
        }
    part[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float s = part[0][threadIdx.x];
        for (int y = 1; y < kColLanes; ++y) s += part[y][threadIdx.x];
        out[c] = s;
    }
}

cudaError_t launch_col_sum(const float* a, const float* b, long rows, int C, float* out, cudaStream_t s) {
    if (C == 0) return cudaSuccess;
    return launch_k(col_sum_kernel, dim3((unsigned)((C + 31) / 32)), dim3(32, kColLanes), 0, s, a, b, rows, C, out);
}

// dw[c][0][k] = sum_r dz[r, c] x[r + k - 3, c] (frames inside the utterance), db[c] = sum_r dz[r, c]
__global__ void __launch_bounds__(32 * kColLanes) dwconv_wgrad_kernel(const float* __restrict__ dz, const float* __restrict__ x,
                                                                      int B, int T, int C, float* __restrict__ dw,
                                                                      float* __restrict__ db) {
    pdl_trigger(); pdl_wait();
    __shared__ float part[kColLanes][8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    const long rows = (long)B * T;
    if (c < C)
        for (long r = threadIdx.y; r < rows; r += kColLanes) {
            const int t = (int)(r % T);
            const float d = dz[r * C + c];
#pragma unroll
            for (int k = 0; k < 7; ++k) {
                const int ts = t + k - 3;
                if (ts >= 0 && ts < T) acc[k] = fmaf(d, x[(r + k - 3) * C + c], acc[k]);
            }
            acc[7] += d;
        }
#pragma unroll
    for (int k = 0; k < 8; ++k) part[threadIdx.y][k][threadIdx.x] = acc[k];
    __syncthreads();
    if (threadIdx.y < 8 && c < C) {
        const int k = threadIdx.y;
        float s = part[0][k][threadIdx.x];
        for (int y = 1; y < kColLanes; ++y) s += part[y][k][threadIdx.x];
        if (k < 7) dw[(long)c * 7 + k] = s; else db[c] = s;
    }
}

cudaError_t launch_dwconv_wgrad(const float* dz, const float* x, int B, int T, int C, float* dw, float* db, cudaStream_t s) {
    if (C == 0) return cudaSuccess;
    return launch_k(dwconv_wgrad_kernel, dim3((unsigned)((C + 31) / 32)), dim3(32, kColLanes), 0, s, dz, x, B, T, C, dw, db);
}

__global__ void scale_cols_kernel(const float* __restrict__ x, const float* __restrict__ gamma, long rows, int C,
                                  float* __restrict__ y) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * C) return;
    y[i] = x[i] * __ldg(gamma + (int)(i % C));
}

cudaError_t launch_scale_cols(const float* x, const float* gamma, long rows, int C, float* y, cudaStream_t s) {
    const long n = rows * C;
    if (n == 0) return cudaSuccess;
    return launch_k(scale_cols_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, x, gamma, rows, C, y);
}

__global__ void gelu_bwd_kernel(const float* __restrict__ dg, const float* __restrict__ h, long n, float* __restrict__ dh) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = h[i];
    const float cdf = 0.5f * (1.0f + erff(v * 0.70710678118654752f));
    const float pdf = 0.39894228040143268f * expf(-0.5f * v * v);
    dh[i] = dg[i] * fmaf(v, pdf, cdf);
}

cudaError_t launch_gelu_bwd(const float* dg, const float* h, long n, float* dh, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    return launch_k(gelu_bwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, dg, h, n, dh);
}

// dst row j < taps Cx, column r < rows: src[r + k - 3 (taps = 7) or r, c] with j = k Cx + c, 0 where that frame leaves
// r's utterance; row taps Cx: 1 (with `ones`); the 7 rows after it and the columns [rows, Kr): 0.  32 x 32 tiles through
// shared memory, so both the reads (along c) and the writes (along r) are coalesced.  Split planes are transposed plane
// by plane (exact); an fp32 source is written as fp32 or split on the way out.
__global__ void __launch_bounds__(256) transpose_rows_kernel(TransposeArgs a) {
    pdl_trigger(); pdl_wait();
    __shared__ float th[32][33], tl[32][33];
    const int j0 = blockIdx.y * 32;
    const long r0 = (long)blockIdx.x * 32;
    const long rows = (long)a.B * a.T;
    const int Nv = a.taps * a.Cx;
    const bool planes_in = a.src_hi != nullptr;
    for (int i = threadIdx.y; i < 32; i += 8) {          // tile row = column r0 + i, tile column = row j0 + threadIdx.x
        const long r = r0 + i;
        const int j = j0 + threadIdx.x;
        float h = 0.f, l = 0.f;
        if (r < rows) {
            if (j < Nv) {
                const int k = a.taps == 7 ? j / a.Cx : 3, c = j - (a.taps == 7 ? k : 0) * a.Cx;
                const int t = (int)(r % a.T), ts = t + k - 3;
                if (ts >= 0 && ts < a.T) {
                    const long o = (r + k - 3) * a.Cx + c;
                    if (planes_in) { h = __bfloat162float(a.src_hi[o]); l = __bfloat162float(a.src_lo[o]); }
                    else h = a.src_f32[o];
                }
            } else if (a.ones && j == Nv) {
                h = 1.f;
            }
        }
        th[i][threadIdx.x] = h; tl[i][threadIdx.x] = l;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int j = j0 + i;
        const long r = r0 + threadIdx.x;
        if (j >= a.Nd || r >= a.Kr) continue;
        const long o = (long)j * a.Kr + r;
        const float h = th[threadIdx.x][i], l = tl[threadIdx.x][i];
        if (a.dst_f32) a.dst_f32[o] = h;
        if (a.dst_hi) {
            if (planes_in) { a.dst_hi[o] = __float2bfloat16_rn(h); a.dst_lo[o] = __float2bfloat16_rn(l); }
            else { bf16 hh, ll; split_bf16(h, hh, ll); a.dst_hi[o] = hh; a.dst_lo[o] = ll; }
        }
    }
}

cudaError_t launch_transpose_rows(const TransposeArgs& a, cudaStream_t s) {
    if ((a.taps != 1 && a.taps != 7) || (a.src_hi && a.dst_f32) || (!a.src_hi && !a.src_f32) || (!a.dst_f32 && !a.dst_hi) ||
        a.Nd < a.taps * a.Cx + (a.ones ? 1 : 0) || a.Kr < (long)a.B * a.T)
        return cudaErrorInvalidValue;
    if (a.Nd == 0 || a.Kr == 0) return cudaSuccess;
    const dim3 grid((unsigned)((a.Kr + 31) / 32), (unsigned)((a.Nd + 31) / 32)), block(32, 8);
    return launch_k(transpose_rows_kernel, grid, block, 0, s, a);
}

// gw[n][c][k] = dWp[m(n)][k Cx + c], gb[n] = dWp[m(n)][taps Cx], row stride ld = taps Cx + 8; m(n) = n, or for the head
// (split > 0) n below `split` stays and n >= split moves to Kp + n - split (the phase column group)
__global__ void wgrad_unpack_kernel(const float* __restrict__ dWp, int Nref, int Cx, int taps, int split, int Kp,
                                    float* __restrict__ gw, float* __restrict__ gb) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long per = (long)Cx * taps + 1;
    if (i >= (long)Nref * per) return;
    const int n = (int)(i / per);
    const int e = (int)(i - (long)n * per);
    const int m = (split > 0 && n >= split) ? Kp + n - split : n;
    const long ld = (long)taps * Cx + 8;
    if (e == per - 1) { gb[n] = dWp[m * ld + (long)taps * Cx]; return; }
    const int c = e / taps, k = e - c * taps;
    gw[(long)n * Cx * taps + e] = dWp[m * ld + (long)k * Cx + c];
}

cudaError_t launch_unpack_wgrad(const float* dWp, int Nref, int Cx, int taps, int split, int Kp, float* gw, float* gb,
                                cudaStream_t s) {
    const long n = (long)Nref * ((long)Cx * taps + 1);
    if (n == 0) return cudaSuccess;
    return launch_k(wgrad_unpack_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, dWp, Nref, Cx, taps, split, Kp, gw, gb);
}

}  // namespace st
