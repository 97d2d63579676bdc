// Kernels of the multi-resolution discriminator (see mrd.cuh; reference: vocoders/vocos/models/discriminator.py:112-171).
// The STFT and its adjoint are mel.cuh's per-frame device code; every reduction runs in a fixed order and no kernel uses
// atomics, so a repeated call is bitwise identical.
#include "mrd.cuh"
#include "mel.cuh"

namespace st {

namespace {

constexpr float kSlope = 0.1f;              // the leaky_relu slope of DiscriminatorR.forward
constexpr int kRedThreads = 256;

__device__ __forceinline__ void put(const MrdPlanes& P, long long i, float v) {
    if (P.f) P.f[i] = v;
    if (P.hi) { bf16 h, l; split_bf16(v, h, l); P.hi[i] = h; P.lo[i] = l; }
}

// slot layout of the STFT kernels: mel.cuh's complex buffer | magnitudes | X (M + 1 complex)
__host__ __device__ inline int stft_xoff(int lm) { return mel_zfloats(lm) + mel_magfloats(lm); }
__host__ __device__ inline int stft_stride(int lm) { return stft_xoff(lm) + ((1 << lm) + 1) * 2 / 4 * 4 + 4; }

__global__ void __launch_bounds__(MEL_THREADS) mrd_stft_kernel(const float* __restrict__ x, long long L, MrdGeo g, int lm,
                                                               const float* __restrict__ window, const float2* __restrict__ tw,
                                                               float* __restrict__ spec) {
    extern __shared__ float4 smem4[];
    float* sm = reinterpret_cast<float*>(smem4);
    const int M = 1 << lm, MP = M + 1, P = frames_per_cta(lm), FS = stft_stride(lm), XO = stft_xoff(lm);
    const int b = blockIdx.y, t0 = blockIdx.x * P, nf = min(P, g.T - t0);
    const float* row = x + (long long)b * L;
    // hop n_fft / 4 = M / 2, centre pad n_fft / 2 = M
    mel_load_frames(sm, lm, P, FS, window, L, M / 2, M, [&](int f, const float*& xp, int& t) {
        xp = row; t = t0 + f;
        return f < nf;
    });
    mel_fft(sm, lm, P, FS, tw);
    mel_half_spectrum(sm, lm, P, FS, tw, XO);
    for (int i = threadIdx.x; i < 2 * P * MP; i += MEL_THREADS) {
        const int ri = i / (P * MP), f = (i / MP) % P, k = i % MP;
        if (f >= nf) continue;
        const float2 X = reinterpret_cast<const float2*>(sm + f * FS + XO)[k];
        spec[(((long long)b * 2 + ri) * g.T + t0 + f) * MP + k] = ri ? X.y : X.x;
    }
}

__global__ void __launch_bounds__(MEL_THREADS) mrd_stft_adj_kernel(const float* __restrict__ gspec, MrdGeo g, int lm,
                                                                   const float* __restrict__ window, const float2* __restrict__ tw,
                                                                   float* __restrict__ gf) {
    extern __shared__ float4 smem4[];
    float* sm = reinterpret_cast<float*>(smem4);
    const int M = 1 << lm, MP = M + 1, N = 2 * M, P = frames_per_cta(lm), FS = stft_stride(lm), XO = stft_xoff(lm);
    const int b = blockIdx.y, t0 = blockIdx.x * P, nf = min(P, g.T - t0);
    for (int i = threadIdx.x; i < P * MP; i += MEL_THREADS) {
        const int f = i / MP, k = i % MP;
        float2 y = make_float2(0.f, 0.f);
        if (f < nf) {
            const float* gs = gspec + ((long long)b * 2 * g.T + t0 + f) * MP + k;
            y = make_float2(gs[0], gs[(long long)g.T * MP]);
        }
        reinterpret_cast<float2*>(sm + f * FS + XO)[k] = y;
    }
    __syncthreads();
    mel_irfft(sm, lm, P, FS, XO, tw);
    for (int i = threadIdx.x; i < P * N; i += MEL_THREADS) {
        const int f = i >> (lm + 1), n = i & (N - 1);
        if (f >= nf) continue;
        gf[((long long)b * g.T + t0 + f) * N + n] = mel_irfft_sample(sm + f * FS, lm, n) * __ldg(window + n);
    }
}

// one thread per (b, t, w) of the band: all 32 output channels
__global__ void mrd_conv0_fwd_kernel(const float* __restrict__ spec, int F, MrdGeo g, MrdBand bd, const float* __restrict__ w,
                                     const float* __restrict__ bias, float* __restrict__ fmap0) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.T * bd.W) return;
    const int x = (int)(i % bd.W), t = (int)((i / bd.W) % g.T), b = (int)(i / ((long long)bd.W * g.T));
    float in[2][3][9];
    for (int ch = 0; ch < 2; ++ch)
        for (int dt = 0; dt < 3; ++dt)
            for (int k = 0; k < 9; ++k) {
                const int tt = t + dt - 1, xx = x + k - 4;
                in[ch][dt][k] = tt >= 0 && tt < g.T && xx >= 0 && xx < bd.W
                                    ? spec[(((long long)b * 2 + ch) * g.T + tt) * F + bd.off + xx] : 0.f;
            }
    for (int n = 0; n < 32; ++n) {
        float v = __ldg(bias + n);
        for (int ch = 0; ch < 2; ++ch)
            for (int dt = 0; dt < 3; ++dt)
                for (int k = 0; k < 9; ++k) v = fmaf(__ldg(w + ((n * 2 + ch) * 3 + dt) * 9 + k), in[ch][dt][k], v);
        v = v > 0.f ? v : v * kSlope;
        fmap0[(((long long)b * 32 + n) * g.T + t) * bd.W + x] = v;
    }
}

__global__ void mrd_conv0_dgrad_kernel(const float* __restrict__ dz0, MrdGeo g, MrdBand bd, int F, const float* __restrict__ w,
                                       float* __restrict__ gspec) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.T * bd.W) return;
    const int x = (int)(i % bd.W), t = (int)((i / bd.W) % g.T), b = (int)(i / ((long long)bd.W * g.T));
    float v[2] = {0.f, 0.f};
    for (int n = 0; n < 32; ++n)
        for (int dt = 0; dt < 3; ++dt) {
            const int tt = t - dt + 1;
            if (tt < 0 || tt >= g.T) continue;
            const float* d = dz0 + (((long long)b * 32 + n) * g.T + tt) * bd.W;
            for (int k = 0; k < 9; ++k) {
                const int xx = x - k + 4;
                if (xx < 0 || xx >= bd.W) continue;
                const float dv = d[xx];
                for (int ch = 0; ch < 2; ++ch) v[ch] = fmaf(__ldg(w + ((n * 2 + ch) * 3 + dt) * 9 + k), dv, v[ch]);
            }
        }
    for (int ch = 0; ch < 2; ++ch) gspec[(((long long)b * 2 + ch) * g.T + t) * F + bd.off + x] = v[ch];
}

// fixed-order tree over one block's partial sums (kRedThreads entries per row of `sm`)
template <int NV>
__device__ void block_sum(float (*sm)[kRedThreads], float* acc) {
    for (int v = 0; v < NV; ++v) sm[v][threadIdx.x] = acc[v];
    __syncthreads();
    for (int st = kRedThreads / 2; st > 0; st >>= 1) {
        if (threadIdx.x < st)
            for (int v = 0; v < NV; ++v) sm[v][threadIdx.x] += sm[v][threadIdx.x + st];
        __syncthreads();
    }
}

// block (n, ch, dt): dw[n, ch, dt, k] = Σ_{b, t, x} dz0[b, n, t, x] spec[b, ch, t + dt - 1, off + x + k - 4]; the block
// (n, 0, 0) also sums db[n] = Σ dz0[b, n, t, x]
__global__ void __launch_bounds__(kRedThreads) mrd_conv0_wgrad_kernel(const float* __restrict__ dz0, const float* __restrict__ spec,
                                                                      int F, MrdGeo g, MrdBand bd, float* __restrict__ dw,
                                                                      float* __restrict__ db) {
    __shared__ float sm[10][kRedThreads];
    const int n = blockIdx.x, ch = blockIdx.y, dt = blockIdx.z;
    const int TW = g.T * bd.W;
    const long long cnt = (long long)g.B * TW;
    float acc[10] = {};
    for (long long i = threadIdx.x; i < cnt; i += kRedThreads) {
        const int b = (int)(i / TW), q = (int)(i % TW), t = q / bd.W, x = q % bd.W;
        const float d = dz0[((long long)b * 32 + n) * TW + q];
        acc[9] += d;
        const int tt = t + dt - 1;
        if (tt < 0 || tt >= g.T) continue;
        const float* s = spec + (((long long)b * 2 + ch) * g.T + tt) * F + bd.off;
        for (int k = 0; k < 9; ++k) {
            const int xx = x + k - 4;
            if (xx >= 0 && xx < bd.W) acc[k] = fmaf(d, s[xx], acc[k]);
        }
    }
    block_sum<10>(sm, acc);
    if (threadIdx.x == 0) {
        for (int k = 0; k < 9; ++k) dw[((n * 2 + ch) * 3 + dt) * 9 + k] = sm[k][0];
        if (ch == 0 && dt == 0) db[n] = sm[9][0];
    }
}

// value of the concatenated band outputs at channel c, frame t, column col (zero outside)
__device__ __forceinline__ float cat_at(const MrdCat& cat, const MrdGeo& g, int b, int c, int t, int col) {
    if (t < 0 || t >= g.T || col < 0 || col >= cat.off[5]) return 0.f;
    int k = 0;
    while (col >= cat.off[k + 1]) ++k;
    const int W = cat.off[k + 1] - cat.off[k];
    return cat.f[k][(((long long)b * 32 + c) * g.T + t) * W + col - cat.off[k]];
}

__global__ void mrd_post_fwd_kernel(MrdCat cat, MrdGeo g, const float* __restrict__ w, const float* __restrict__ bias,
                                    float* __restrict__ post) {
    const int Wt = cat.off[5];
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.T * Wt) return;
    const int x = (int)(i % Wt), t = (int)((i / Wt) % g.T), b = (int)(i / ((long long)Wt * g.T));
    float v = 0.f;
    for (int c = 0; c < 32; ++c)
        for (int dt = 0; dt < 3; ++dt)
            for (int dk = 0; dk < 3; ++dk) v = fmaf(__ldg(w + (c * 3 + dt) * 3 + dk), cat_at(cat, g, b, c, t + dt - 1, x + dk - 1), v);
    post[i] = v + __ldg(bias);
}

__global__ void mrd_post_dgrad_kernel(const float* __restrict__ gpost, MrdCat cat, int k, MrdGeo g, const float* __restrict__ w,
                                      float* __restrict__ G) {
    const int W = cat.off[k + 1] - cat.off[k], Wt = cat.off[5];
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * 32 * g.T * W) return;
    const int x = (int)(i % W), t = (int)((i / W) % g.T), c = (int)((i / ((long long)W * g.T)) % 32);
    const int b = (int)(i / (32LL * W * g.T)), X = cat.off[k] + x;
    float v = 0.f;
    for (int dt = 0; dt < 3; ++dt) {
        const int tt = t - dt + 1;
        if (tt < 0 || tt >= g.T) continue;
        for (int dk = 0; dk < 3; ++dk) {
            const int xx = X - dk + 1;
            if (xx >= 0 && xx < Wt) v = fmaf(__ldg(w + (c * 3 + dt) * 3 + dk), gpost[((long long)b * g.T + tt) * Wt + xx], v);
        }
    }
    G[i] = v;
}

// block c < 32: dw[c, dt, dk] = Σ gpost[b, t, x] cat[b, c, t + dt - 1, x + dk - 1]; block 32: db = Σ gpost
__global__ void __launch_bounds__(kRedThreads) mrd_post_wgrad_kernel(const float* __restrict__ gpost, MrdCat cat, MrdGeo g,
                                                                     float* __restrict__ dw, float* __restrict__ db) {
    __shared__ float sm[9][kRedThreads];
    const int c = blockIdx.x, Wt = cat.off[5], TW = g.T * Wt;
    const long long cnt = (long long)g.B * TW;
    float acc[9] = {};
    for (long long i = threadIdx.x; i < cnt; i += kRedThreads) {
        const float gv = gpost[i];
        if (c == 32) { acc[0] += gv; continue; }
        const int b = (int)(i / TW), q = (int)(i % TW), t = q / Wt, x = q % Wt;
        for (int dt = 0; dt < 3; ++dt)
            for (int dk = 0; dk < 3; ++dk) acc[dt * 3 + dk] = fmaf(gv, cat_at(cat, g, b, c, t + dt - 1, x + dk - 1), acc[dt * 3 + dk]);
    }
    block_sum<9>(sm, acc);
    if (threadIdx.x == 0) {
        if (c == 32) db[0] = sm[0][0];
        else for (int j = 0; j < 9; ++j) dw[c * 9 + j] = sm[j][0];
    }
}

// rows(X)[bb, gg, kx] of mrd.cuh (zero outside)
__device__ __forceinline__ float rows_at(const float* __restrict__ X, const MrdGeo& g, int W, int lanes, int bb, int gg, int kx) {
    const int c = kx % 32, ldt = kx / 32, l = ldt / 3, dt = ldt % 3;
    const int b = bb / g.T, t = bb % g.T + dt - 1, col = lanes * gg + l;
    if (t < 0 || t >= g.T || col >= W) return 0.f;
    return X[(((long long)b * 32 + c) * g.T + t) * W + col];
}

__global__ void mrd_expand_kernel(const float* __restrict__ X, MrdGeo g, int W, int lanes, MrdPlanes out) {
    const int G = (W + lanes - 1) / lanes, Kx = 96 * lanes;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.T * G * Kx) return;
    const int kx = (int)(i % Kx), gg = (int)((i / Kx) % G), bb = (int)(i / ((long long)Kx * G));
    put(out, i, rows_at(X, g, W, lanes, bb, gg, kx));
}

__global__ void mrd_pack_kernel(const float* __restrict__ w, int lanes, int dgrad, float* __restrict__ out) {
    const int taps = mrd_taps(lanes), kw = mrd_kw(lanes), Kx = 96 * lanes;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= taps * 32 * Kx) return;
    int t, n, kx;
    if (!dgrad) { kx = i % Kx; n = (i / Kx) % 32; t = i / (Kx * 32); }
    else { n = i % 32; kx = (i / 32) % Kx; t = taps - 1 - i / (32 * Kx); }
    const int c = kx % 32, ldt = kx / 32, l = ldt / 3, dt = ldt % 3, k = lanes * t + l;
    out[i] = k < kw ? w[((n * 32 + c) * 3 + dt) * kw + k] : 0.f;
}

__global__ void mrd_act_fwd_kernel(const float* __restrict__ Y, MrdGeo g, int W, float slope, float* __restrict__ fmap) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * 32 * g.T * W) return;
    const int x = (int)(i % W), t = (int)((i / W) % g.T), n = (int)((i / ((long long)W * g.T)) % 32);
    const int b = (int)(i / (32LL * W * g.T));
    const float v = Y[(((long long)b * g.T + t) * W + x) * 32 + n];
    fmap[i] = v > 0.f ? v : v * slope;
}

__global__ void mrd_act_bwd_kernel(const float* __restrict__ G, const float* __restrict__ gfmap, const float* __restrict__ fmap,
                                   MrdGeo g, int W, MrdPlanes dz, MrdPlanes dzT, long long Kr, float* __restrict__ dz_nchw) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * 32 * g.T * W) return;
    const int x = (int)(i % W), t = (int)((i / W) % g.T), n = (int)((i / ((long long)W * g.T)) % 32);
    const int b = (int)(i / (32LL * W * g.T));
    float v = G[i];
    if (gfmap) v += gfmap[i];
    if (fmap) v = fmap[i] > 0.f ? v : v * kSlope;
    const long long r = ((long long)b * g.T + t) * W + x;
    put(dz, r * 32 + n, v);
    put(dzT, (long long)n * Kr + r, v);
    if (dz_nchw) dz_nchw[i] = v;
}

__global__ void mrd_fold_kernel(const float* __restrict__ dR, MrdGeo g, int W, int lanes, float* __restrict__ dX) {
    const int G = (W + lanes - 1) / lanes, Kx = 96 * lanes;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * 32 * g.T * W) return;
    const int x = (int)(i % W), t = (int)((i / W) % g.T), c = (int)((i / ((long long)W * g.T)) % 32);
    const int b = (int)(i / (32LL * W * g.T));
    float v = 0.f;
    for (int dt = 0; dt < 3; ++dt) {
        const int tr = t - dt + 1;
        if (tr >= 0 && tr < g.T) v += dR[(((long long)b * g.T + tr) * G + x / lanes) * Kx + ((x % lanes) * 3 + dt) * 32 + c];
    }
    dX[i] = v;
}

__global__ void mrd_im2col_t_kernel(const float* __restrict__ X, MrdGeo g, int W, int lanes, long long Kr, MrdPlanes out) {
    const int G = (W + lanes - 1) / lanes, Kx = 96 * lanes, taps = mrd_taps(lanes);
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)(taps * Kx + 8) * Kr) return;
    const long long r = i % Kr;
    const int row = (int)(i / Kr);
    float v = 0.f;
    if (r < (long long)g.B * g.T * G) {
        if (row < taps * Kx) {
            const int bb = (int)(r / G), gg = (int)(r % G) + row / Kx - taps / 2;
            if (gg >= 0 && gg < G) v = rows_at(X, g, W, lanes, bb, gg, row % Kx);
        } else if (row == taps * Kx) {
            v = 1.f;
        }
    }
    put(out, i, v);
}

__global__ void mrd_unpack_wgrad_kernel(const float* __restrict__ dWp, int lanes, float* __restrict__ dw, float* __restrict__ db) {
    const int taps = mrd_taps(lanes), kw = mrd_kw(lanes), Kx = 96 * lanes, Np = taps * Kx + 8;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 32 * 32 * 3 * kw) return;
    const int k = i % kw, dt = (i / kw) % 3, c = (i / (3 * kw)) % 32, n = i / (96 * kw);
    dw[i] = dWp[n * Np + (k / lanes) * Kx + ((k % lanes) * 3 + dt) * 32 + c];
    if (c == 0 && dt == 0 && k == 0) db[n] = dWp[n * Np + taps * Kx];
}

inline unsigned blocks(long long n) { return (unsigned)((n + 255) / 256); }

}  // namespace

cudaError_t launch_mrd_stft(const float* x, long long L, MrdGeo g, int log2M, const float* window, const float2* tw, float* spec,
                            cudaStream_t s) {
    static std::atomic<uint64_t> smem_done{0};
    cudaError_t e = ensure_dyn_smem(mrd_stft_kernel, MEL_LOSS_MAX_SMEM, smem_done);
    if (e != cudaSuccess) return e;
    const int P = frames_per_cta(log2M);
    mrd_stft_kernel<<<dim3((unsigned)((g.T + P - 1) / P), (unsigned)g.B), MEL_THREADS, (size_t)P * stft_stride(log2M) * 4, s>>>(
        x, L, g, log2M, window, tw, spec);
    return cudaGetLastError();
}

cudaError_t launch_mrd_stft_adj(const float* gspec, MrdGeo g, int log2M, const float* window, const float2* tw, float* gf,
                                cudaStream_t s) {
    static std::atomic<uint64_t> smem_done{0};
    cudaError_t e = ensure_dyn_smem(mrd_stft_adj_kernel, MEL_LOSS_MAX_SMEM, smem_done);
    if (e != cudaSuccess) return e;
    const int P = frames_per_cta(log2M);
    mrd_stft_adj_kernel<<<dim3((unsigned)((g.T + P - 1) / P), (unsigned)g.B), MEL_THREADS, (size_t)P * stft_stride(log2M) * 4, s>>>(
        gspec, g, log2M, window, tw, gf);
    return cudaGetLastError();
}

cudaError_t launch_mrd_conv0_fwd(const float* spec, int F, MrdGeo g, MrdBand bd, const float* w, const float* b, float* fmap0,
                                 cudaStream_t s) {
    mrd_conv0_fwd_kernel<<<blocks((long long)g.B * g.T * bd.W), 256, 0, s>>>(spec, F, g, bd, w, b, fmap0);
    return cudaGetLastError();
}

cudaError_t launch_mrd_conv0_dgrad(const float* dz0, MrdGeo g, MrdBand bd, int F, const float* w, float* gspec, cudaStream_t s) {
    mrd_conv0_dgrad_kernel<<<blocks((long long)g.B * g.T * bd.W), 256, 0, s>>>(dz0, g, bd, F, w, gspec);
    return cudaGetLastError();
}

cudaError_t launch_mrd_conv0_wgrad(const float* dz0, const float* spec, int F, MrdGeo g, MrdBand bd, float* dw, float* db,
                                   cudaStream_t s) {
    mrd_conv0_wgrad_kernel<<<dim3(32, 2, 3), kRedThreads, 0, s>>>(dz0, spec, F, g, bd, dw, db);
    return cudaGetLastError();
}

cudaError_t launch_mrd_post_fwd(MrdCat cat, MrdGeo g, const float* w, const float* b, float* post, cudaStream_t s) {
    mrd_post_fwd_kernel<<<blocks((long long)g.B * g.T * cat.off[5]), 256, 0, s>>>(cat, g, w, b, post);
    return cudaGetLastError();
}

cudaError_t launch_mrd_post_dgrad(const float* gpost, MrdCat cat, int k, MrdGeo g, const float* w, float* G, cudaStream_t s) {
    mrd_post_dgrad_kernel<<<blocks((long long)g.B * 32 * g.T * (cat.off[k + 1] - cat.off[k])), 256, 0, s>>>(gpost, cat, k, g, w, G);
    return cudaGetLastError();
}

cudaError_t launch_mrd_post_wgrad(const float* gpost, MrdCat cat, MrdGeo g, float* dw, float* db, cudaStream_t s) {
    mrd_post_wgrad_kernel<<<33, kRedThreads, 0, s>>>(gpost, cat, g, dw, db);
    return cudaGetLastError();
}

cudaError_t launch_mrd_expand(const float* X, MrdGeo g, int W, int lanes, MrdPlanes out, cudaStream_t s) {
    const long long n = (long long)g.B * g.T * ((W + lanes - 1) / lanes) * 96 * lanes;
    mrd_expand_kernel<<<blocks(n), 256, 0, s>>>(X, g, W, lanes, out);
    return cudaGetLastError();
}

cudaError_t launch_mrd_pack(const float* w, int lanes, int dgrad, float* out, cudaStream_t s) {
    mrd_pack_kernel<<<blocks((long long)mrd_taps(lanes) * 32 * 96 * lanes), 256, 0, s>>>(w, lanes, dgrad, out);
    return cudaGetLastError();
}

cudaError_t launch_mrd_act_fwd(const float* Y, MrdGeo g, int W, float* fmap, cudaStream_t s, float slope) {
    mrd_act_fwd_kernel<<<blocks((long long)g.B * 32 * g.T * W), 256, 0, s>>>(Y, g, W, slope, fmap);
    return cudaGetLastError();
}

cudaError_t launch_mrd_act_bwd(const float* G, const float* gfmap, const float* fmap, MrdGeo g, int W, MrdPlanes dz, MrdPlanes dzT,
                               long long Kr, float* dz_nchw, cudaStream_t s) {
    mrd_act_bwd_kernel<<<blocks((long long)g.B * 32 * g.T * W), 256, 0, s>>>(G, gfmap, fmap, g, W, dz, dzT, Kr, dz_nchw);
    return cudaGetLastError();
}

cudaError_t launch_mrd_fold(const float* dR, MrdGeo g, int W, int lanes, float* dX, cudaStream_t s) {
    mrd_fold_kernel<<<blocks((long long)g.B * 32 * g.T * W), 256, 0, s>>>(dR, g, W, lanes, dX);
    return cudaGetLastError();
}

cudaError_t launch_mrd_im2col_t(const float* X, MrdGeo g, int W, int lanes, long long Kr, MrdPlanes out, cudaStream_t s) {
    mrd_im2col_t_kernel<<<blocks((long long)(mrd_taps(lanes) * 96 * lanes + 8) * Kr), 256, 0, s>>>(X, g, W, lanes, Kr, out);
    return cudaGetLastError();
}

cudaError_t launch_mrd_unpack_wgrad(const float* dWp, int lanes, float* dw, float* db, cudaStream_t s) {
    mrd_unpack_wgrad_kernel<<<blocks(32LL * 32 * 3 * mrd_kw(lanes)), 256, 0, s>>>(dWp, lanes, dw, db);
    return cudaGetLastError();
}

}  // namespace st
