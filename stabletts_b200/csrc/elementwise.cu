// HBM-bound glue kernels of the CFM/DiT path: layout changes at the boundary, mask·FiLM →
// LayerNorm → adaLN-modulate (one pass, warp-shuffle reductions), tiny GEMVs for the
// t-/c-conditioning vectors, CFG combine and Runge–Kutta linear combinations.
#include "common.cuh"
#include <cuda_fp16.h>
#include <algorithm>

namespace st {

// ---------------------------------------------------------------------------------------------
// (B, C, T) <-> (B, T, C) tiled transposes (32x32 smem tile, +1 padding: conflict-free)
// ---------------------------------------------------------------------------------------------
__global__ void bct_to_btc_kernel(const float* __restrict__ in, float* __restrict__ out_f32, bf16* __restrict__ out_hi,
                                  bf16* __restrict__ out_lo, int B, int C, int T, const float* __restrict__ bcast) {
    pdl_trigger(); pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const bool is_bcast = (b == B);
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int c = c0 + i, t = t0 + threadIdx.x;
        float v = 0.f;
        if (c < C && t < T) v = is_bcast ? bcast[c] : in[((long)b * C + c) * T + t];
        tile[i][threadIdx.x] = v;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int t = t0 + i, c = c0 + threadIdx.x;
        if (c < C && t < T) {
            float v = tile[threadIdx.x][i];
            long o = ((long)b * T + t) * C + c;
            if (out_f32) out_f32[o] = v;
            if (out_hi) { bf16 h, l; split_bf16(v, h, l); out_hi[o] = h; out_lo[o] = l; }
        }
    }
}

cudaError_t launch_bct_to_btc(const float* in, float* out_f32, bf16* out_hi, bf16* out_lo, int B, int C, int T,
                              const float* bcast, cudaStream_t s) {
    const int rows = B + (bcast ? 1 : 0);
    if (rows == 0 || C == 0 || T == 0) return cudaSuccess;
    dim3 grid((T + 31) / 32, (C + 31) / 32, rows), block(32, 8);
    return launch_k(bct_to_btc_kernel, grid, block, 0, s, in, out_f32, out_hi, out_lo, B, C, T, bcast);
}

__global__ void btc_to_bct_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int T) {
    pdl_trigger(); pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int t = t0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (c < C && t < T) ? in[((long)b * T + t) * C + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int c = c0 + i, t = t0 + threadIdx.x;
        if (c < C && t < T) out[((long)b * C + c) * T + t] = tile[threadIdx.x][i];
    }
}

cudaError_t launch_btc_to_bct(const float* in, float* out, int B, int C, int T, cudaStream_t s) {
    if (B == 0 || C == 0 || T == 0) return cudaSuccess;
    dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
    return launch_k(btc_to_bct_kernel, grid, block, 0, s, in, out, B, C, T);
}

// ---------------------------------------------------------------------------------------------
// mask·FiLM → LayerNorm(C, no affine, eps 1e-5) → modulate.   One warp per frame (row); H = 256
// → 8 channels per lane as two float4; mean / variance by warp shuffles (two-pass, in registers).
// Reference: models/estimator.py:16,30-33 (FiLM), models/diffusion_transformer.py:106,111-112,
// 119-121 (x*mask, LN, modulate), :26 (FFN input mask).
// ---------------------------------------------------------------------------------------------
template <int H>
__global__ void __launch_bounds__(256) film_ln_mod_kernel(LnArgs a) {
    pdl_trigger(); pdl_wait();
    constexpr int V = H / 32;          // channels per lane
    constexpr int R = 2;               // frames per warp: two independent 1 KB row streams in flight per warp
    static_assert(V % 4 == 0, "H must be a multiple of 128");
    const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long rows = (long)a.BB * a.T;
    const long row0 = warp * R;
    if (row0 >= rows) return;
    float x[R][V];
    float m[R];
    int cb[R];
    bool ok[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const long row = row0 + r;
        ok[r] = row < rows;
        const long rw = ok[r] ? row : rows - 1;
        const int bb = (int)(rw / a.T), t = (int)(rw - (long)bb * a.T);
        m[r] = a.mask[(long)(bb % a.B) * a.T + t];
        cb[r] = min(bb, a.c_clamp);
        const float* xr = a.xin + rw * H;
#pragma unroll
        for (int j = 0; j < V / 4; ++j) {
            float4 v = __ldg(reinterpret_cast<const float4*>(xr + (j * 32 + lane) * 4));
            x[r][j * 4 + 0] = v.x; x[r][j * 4 + 1] = v.y; x[r][j * 4 + 2] = v.z; x[r][j * 4 + 3] = v.w;
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (!ok[r]) continue;
        const long row = row0 + r;
        const int bb = (int)(row / a.T);
        if (a.has_film) {
            const float* f = a.film + (long)(bb % a.B) * a.film_bstride;
#pragma unroll
            for (int j = 0; j < V / 4; ++j) {
                int c = (j * 32 + lane) * 4;
                float4 g = __ldg(reinterpret_cast<const float4*>(f + c));
                float4 be = __ldg(reinterpret_cast<const float4*>(f + H + c));
                x[r][j * 4 + 0] = (g.x * x[r][j * 4 + 0] + be.x) * m[r];
                x[r][j * 4 + 1] = (g.y * x[r][j * 4 + 1] + be.y) * m[r];
                x[r][j * 4 + 2] = (g.z * x[r][j * 4 + 2] + be.z) * m[r];
                x[r][j * 4 + 3] = (g.w * x[r][j * 4 + 3] + be.w) * m[r];
            }
            float* xo = a.xout + row * H;
#pragma unroll
            for (int j = 0; j < V / 4; ++j)
                *reinterpret_cast<float4*>(xo + (j * 32 + lane) * 4) =
                    make_float4(x[r][j * 4 + 0], x[r][j * 4 + 1], x[r][j * 4 + 2], x[r][j * 4 + 3]);
        }
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) sum += x[r][j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float mean = sum * (1.0f / H);
        float var = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) { float d = x[r][j] - mean; var += d * d; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
        const float rstd = rsqrtf(var * (1.0f / H) + 1e-5f);
        const float* sh = a.shift + (long)cb[r] * a.ada_bstride;
        const float* sc = a.scale + (long)cb[r] * a.ada_bstride;
        const float mo = a.mask_out ? m[r] : 1.0f;
#pragma unroll
        for (int j = 0; j < V / 4; ++j) {
            int c = (j * 32 + lane) * 4;
            float4 s4 = __ldg(reinterpret_cast<const float4*>(sh + c));
            float4 c4 = __ldg(reinterpret_cast<const float4*>(sc + c));
            float u0 = ((x[r][j * 4 + 0] - mean) * rstd * (1.f + c4.x) + s4.x) * mo;
            float u1 = ((x[r][j * 4 + 1] - mean) * rstd * (1.f + c4.y) + s4.y) * mo;
            float u2 = ((x[r][j * 4 + 2] - mean) * rstd * (1.f + c4.z) + s4.z) * mo;
            float u3 = ((x[r][j * 4 + 3] - mean) * rstd * (1.f + c4.w) + s4.w) * mo;
            long o = row * H + c;
            if (a.u_f32) *reinterpret_cast<float4*>(a.u_f32 + o) = make_float4(u0, u1, u2, u3);
            if (a.u_hi && a.u16) {
                *reinterpret_cast<uint2*>(a.u_hi + o) = make_uint2(pack_f16x2_sat(u0, u1), pack_f16x2_sat(u2, u3));
            } else if (a.u_hi) {
                uint32_t h01, l01, h23, l23;
                split_bf16x2(u0, u1, h01, l01); split_bf16x2(u2, u3, h23, l23);
                *reinterpret_cast<uint2*>(a.u_hi + o) = make_uint2(h01, h23);
                *reinterpret_cast<uint2*>(a.u_lo + o) = make_uint2(l01, l23);
            }
        }
    }
}

cudaError_t launch_film_ln_mod(const LnArgs& a, cudaStream_t s) {
    if (a.H != 256) return cudaErrorInvalidValue;
    long rows = (long)a.BB * a.T;
    if (rows == 0) return cudaSuccess;
    int blocks = (int)((((rows + 1) / 2) * 32 + 255) / 256);      // two frames per warp
    return launch_k(film_ln_mod_kernel<256>, dim3(blocks), dim3(256), 0, s, a);
}

// ---------------------------------------------------------------------------------------------
// small GEMV batch: one warp per (row r, output n)
// ---------------------------------------------------------------------------------------------
__global__ void gemv_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias,
                            float* __restrict__ y, long y_rstride, int R, int K, int N, int silu_in, int silu_out) {
    pdl_trigger(); pdl_wait();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (gw >= R * N) return;
    const int r = gw / N, n = gw - r * N;
    const float* xr = x + (long)r * K;
    const float* wr = W + (long)n * K;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) {
        float xv = xr[k];
        if (silu_in) xv = xv / (1.0f + expf(-xv));
        acc = fmaf(xv, wr[k], acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        float v = acc + (bias ? bias[n] : 0.f);
        if (silu_out) v = v / (1.0f + expf(-v));
        y[(long)r * y_rstride + n] = v;
    }
}

cudaError_t launch_gemv(const float* x, const float* W, const float* bias, float* y, long y_rstride, int R, int K, int N,
                        int silu_in, int silu_out, cudaStream_t s) {
    long warps = (long)R * N;
    if (warps == 0) return cudaSuccess;
    int blocks = (int)((warps * 32 + 255) / 256);
    return launch_k(gemv_kernel, dim3(blocks), dim3(256), 0, s, x, W, bias, y, y_rstride, R, K, N, silu_in, silu_out);
}

// models/estimator.py:41-49: emb = 1000 * t * exp(-i * ln(1e4)/(half-1)); cat(sin, cos)
__global__ void time_embed_kernel(const float* __restrict__ t, int n_t, int H, float* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int half = H / 2;
    if (i >= n_t * half) return;
    int r = i / half, j = i - r * half;
    float step = (float)(9.210340371976184 / (double)(half - 1));     // ln(10000)/(half-1)
    float w = expf((float)j * -step);
    float e = 1000.0f * t[r] * w;
    out[(long)r * H + j] = sinf(e);
    out[(long)r * H + half + j] = cosf(e);
}

cudaError_t launch_time_embed(const float* t, int n_t, int H, float* out, cudaStream_t s) {
    int n = n_t * (H / 2);
    return launch_k(time_embed_kernel, dim3((n + 127) / 128), dim3(128), 0, s, t, n_t, H, out);
}

// models/diffusion_transformer.py:157-171: theta_i = 1/base^(2i/d); angle = pos * theta_i
__global__ void rope_table_kernel(float* __restrict__ cs, int T, int d_rot) {
    pdl_trigger(); pdl_wait();
    int half = d_rot / 2;
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T * half) return;
    int pos = i / half, j = i - pos * half;
    float theta = 1.0f / powf(10000.0f, (float)(2 * j) / (float)d_rot);
    float ang = (float)pos * theta;
    cs[(long)i * 2 + 0] = (float)cos((double)ang);
    cs[(long)i * 2 + 1] = (float)sin((double)ang);
}

cudaError_t launch_rope_table(float* cs, int T, int d_rot, cudaStream_t s) {
    int n = T * (d_rot / 2);
    if (n == 0) return cudaSuccess;
    return launch_k(rope_table_kernel, dim3((n + 127) / 128), dim3(128), 0, s, cs, T, d_rot);
}

__global__ void mask_lengths_kernel(const float* __restrict__ mask, int* __restrict__ kvlen, int* __restrict__ prefix, int B, int T) {
    pdl_trigger(); pdl_wait();
    int b = blockIdx.x;
    int best = 0, first0 = T;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        if (mask[(long)b * T + t] != 0.f) best = max(best, t + 1);
        else first0 = min(first0, t);
    }
    __shared__ int red[32], red2[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
        first0 = min(first0, __shfl_xor_sync(0xffffffffu, first0, o));
    }
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = best; red2[threadIdx.x >> 5] = first0; }
    __syncthreads();
    if (threadIdx.x < 32) {
        int v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0;
        int w = threadIdx.x < (blockDim.x >> 5) ? red2[threadIdx.x] : T;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
            w = min(w, __shfl_xor_sync(0xffffffffu, w, o));
        }
        if (threadIdx.x == 0) { kvlen[b] = v; prefix[b] = w; }
    }
}

cudaError_t launch_mask_lengths(const float* mask, int* kvlen, int* prefix, int B, int T, cudaStream_t s) {
    return launch_k(mask_lengths_kernel, dim3(B), dim3(256), 0, s, mask, kvlen, prefix, B, T);
}

// TextEncoder front end (models/text_encoder.py:35-37): x = emb[id] * sqrt(H) * mask, mask = t < x_lengths[b]
__global__ void embed_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ lens, const float* __restrict__ emb,
                             int n_vocab, int B, int T, int H, float scale, float* __restrict__ x, float* __restrict__ mask) {
    pdl_trigger(); pdl_wait();
    const long row = blockIdx.x;                 // (b, t)
    const int b = (int)(row / T), t = (int)(row % T);
    const float m = t < lens[b] ? 1.f : 0.f;
    long id = ids[row];
    id = id < 0 ? 0 : (id >= n_vocab ? n_vocab - 1 : id);
    for (int c = threadIdx.x; c < H; c += blockDim.x) x[row * H + c] = emb[id * H + c] * scale * m;
    if (threadIdx.x == 0) mask[row] = m;
}

cudaError_t launch_embed(const int64_t* ids, const int64_t* lens, const float* emb, int n_vocab, int B, int T, int H, float scale,
                         float* x, float* mask, cudaStream_t s) {
    if ((long)B * T == 0) return cudaSuccess;
    return launch_k(embed_kernel, dim3((unsigned)((long)B * T)), dim3(64), 0, s, ids, lens, emb, n_vocab, B, T, H, scale, x, mask);
}

__global__ void cfg_combine_kernel(const float* __restrict__ V, float* __restrict__ K, long n, int cfg, float s_cfg) {
    pdl_trigger(); pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float c = V[i];
    if (cfg) { float u = V[n + i]; c = u + s_cfg * (c - u); }
    K[i] = c;
}

cudaError_t launch_cfg_combine(const float* V, float* K_out, int B, long per_batch, int cfg, float s_cfg, cudaStream_t s) {
    long n = (long)B * per_batch;
    if (n == 0) return cudaSuccess;
    return launch_k(cfg_combine_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, V, K_out, n, cfg, s_cfg);
}

struct LinArgs { const float* K[6]; float coef[6]; int n; };

__global__ void lincomb_kernel(float* __restrict__ dst, const float* __restrict__ y, LinArgs a, long numel) {
    pdl_trigger(); pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numel) return;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 6; ++j) if (j < a.n) acc = fmaf(a.coef[j], a.K[j][i], acc);
    dst[i] = y[i] + acc;
}

cudaError_t launch_lincomb(float* dst, const float* y, const float* const* K, const float* coef, int n, long numel,
                           cudaStream_t s) {
    if (n > 6) return cudaErrorInvalidValue;
    if (numel == 0) return cudaSuccess;
    LinArgs a;
    for (int j = 0; j < 6; ++j) { a.K[j] = j < n ? K[j] : nullptr; a.coef[j] = j < n ? coef[j] : 0.f; }
    a.n = n;
    return launch_k(lincomb_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, s, dst, y, a, numel);
}

// sum over all elements of ( (sum_i coef_i * K_i[e]) / (atol + rtol * max(|u[e]|, |v[e]|)) )^2  -> *out (double, atomic)
// (the RMS mixed error norm of the adaptive Dormand–Prince controller; also Hairer's initial-step norms)
struct NormArgs { const float* K[7]; float coef[7]; int n; };

__global__ void scaled_sumsq_kernel(NormArgs a, const float* __restrict__ u, const float* __restrict__ v, float atol, float rtol,
                                    long numel, double* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    double acc = 0.0;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += (long)gridDim.x * blockDim.x) {
        float num = 0.f;
#pragma unroll
        for (int j = 0; j < 7; ++j) if (j < a.n) num = fmaf(a.coef[j], a.K[j][i], num);
        const float tol = atol + rtol * fmaxf(fabsf(u[i]), fabsf(v[i]));
        const float r = num / tol;
        acc += (double)r * (double)r;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
        atomicAdd(out, t);
    }
}

cudaError_t launch_scaled_sumsq(const float* const* K, const float* coef, int n, const float* u, const float* v, float atol,
                                float rtol, long numel, double* out, cudaStream_t s) {
    if (n > 7) return cudaErrorInvalidValue;
    NormArgs a;
    for (int j = 0; j < 7; ++j) { a.K[j] = j < n ? K[j] : nullptr; a.coef[j] = j < n ? coef[j] : 0.f; }
    a.n = n;
    cudaError_t e = cudaMemsetAsync(out, 0, sizeof(double), s);
    if (e != cudaSuccess) return e;
    const int blocks = (int)std::min<long>((numel + 255) / 256, 592);
    return launch_k(scaled_sumsq_kernel, dim3(blocks > 0 ? blocks : 1), dim3(256), 0, s, a, u, v, atol, rtol, numel, out);
}

__global__ void split_kernel(const float* __restrict__ in, bf16* __restrict__ hi, bf16* __restrict__ lo, long n) {
    pdl_trigger(); pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bf16 h, l;
    split_bf16(in[i], h, l);
    hi[i] = h; lo[i] = l;
}

cudaError_t launch_split(const float* in, bf16* hi, bf16* lo, long numel, cudaStream_t s) {
    if (numel == 0) return cudaSuccess;
    return launch_k(split_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, s, in, hi, lo, numel);
}

// fp16 hi / lo planes of a weight tensor (two-pass FFN precision): hi = fp16(x), lo = fp16(x - hi); 22 mantissa bits
// while |x - hi| stays above the fp16 subnormal step 2^-24.  From |x| >= 65520 on hi rounds to inf and lo to -inf, so the
// pair no longer stands for x: such an x (or a NaN) sets *out_of_range, whose owner then keeps these planes out of use.
__global__ void split_f16_kernel(const float* __restrict__ in, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, long n,
                                 int* __restrict__ out_of_range) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = in[i];
    const __half h = __float2half_rn(x);
    const __half l = __float2half_rn(x - __half2float(h));
    hi[i] = __half_as_ushort(h); lo[i] = __half_as_ushort(l);
    if (out_of_range && !(fabsf(x) < 65520.f)) *out_of_range = 1;
}

cudaError_t launch_split_f16(const float* in, bf16* hi, bf16* lo, long numel, cudaStream_t s, int* out_of_range) {
    if (numel == 0) return cudaSuccess;
    split_f16_kernel<<<(unsigned)((numel + 255) / 256), 256, 0, s>>>(in, reinterpret_cast<uint16_t*>(hi), reinterpret_cast<uint16_t*>(lo), numel,
                                                                     out_of_range);
    return cudaGetLastError();
}

// ----- conditional-flow-matching objective (models/flow_matching.py:69-100), forward value only -----
// y = (1 - (1 - sigma_min) t_b) z + t_b x1  on (B, C, T) tensors, t per sample (:96)
__global__ void cfm_mix_kernel(const float* __restrict__ x1, const float* __restrict__ z, const float* __restrict__ t,
                               float sigma_min, long per_batch, long numel, float* __restrict__ y) {
    pdl_trigger(); pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numel) return;
    const float tb = t[i / per_batch];
    y[i] = (1.f - (1.f - sigma_min) * tb) * z[i] + tb * x1[i];
}

cudaError_t launch_cfm_mix(const float* x1, const float* z, const float* t, float sigma_min, int B, long per_batch, float* y,
                           cudaStream_t s) {
    const long n = (long)B * per_batch;
    if (n == 0) return cudaSuccess;
    return launch_k(cfm_mix_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, x1, z, t, sigma_min, per_batch, n, y);
}

// acc[0] += sum (v - u)^2 with u = x1 - (1 - sigma_min) z over ALL positions (the reference's mse_loss(reduction="sum")
// runs over padded frames too, :97-99); acc[1] += sum(mask).  v, x1, z: (B, C, T); mask: (B, 1, T).
__global__ void cfm_loss_kernel(const float* __restrict__ v, const float* __restrict__ x1, const float* __restrict__ z,
                                const float* __restrict__ mask, float sigma_min, long numel, long n_mask,
                                double* __restrict__ acc) {
    pdl_trigger(); pdl_wait();
    double a = 0.0, m = 0.0;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
        const float d = v[i] - (x1[i] - (1.f - sigma_min) * z[i]);
        a += (double)d * (double)d;
    }
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_mask; i += stride) m += (double)mask[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); m += __shfl_xor_sync(0xffffffffu, m, o); }
    __shared__ double red[2][8];
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = m; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ta = 0.0, tm = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { ta += red[0][w]; tm += red[1][w]; }
        atomicAdd(acc, ta); atomicAdd(acc + 1, tm);
    }
}

// loss = sumsq / (sum(mask) * C)   (:97-99)
__global__ void cfm_loss_final_kernel(const double* __restrict__ acc, int C, float* __restrict__ loss) {
    pdl_trigger(); pdl_wait();
    if (threadIdx.x == 0 && blockIdx.x == 0) loss[0] = (float)(acc[0] / (acc[1] * (double)C));
}

cudaError_t launch_cfm_loss(const float* v, const float* x1, const float* z, const float* mask, float sigma_min, int B, int C,
                            int T, double* acc2, float* loss, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(acc2, 0, 2 * sizeof(double), s);
    if (e != cudaSuccess) return e;
    const long numel = (long)B * C * T, n_mask = (long)B * T;
    const int blocks = (int)std::max<long>(1, std::min<long>((numel + 255) / 256, 592));
    e = launch_k(cfm_loss_kernel, dim3(blocks), dim3(256), 0, s, v, x1, z, mask, sigma_min, numel, n_mask, acc2);
    if (e != cudaSuccess) return e;
    return launch_k(cfm_loss_final_kernel, dim3(1), dim3(32), 0, s, (const double*)acc2, C, loss);
}

}  // namespace st
