// Row kernels of the multi-period discriminator (see mpd.cuh; reference: vocoders/vocos/models/discriminator.py:33-79).
// Every reduction runs in a fixed order and no kernel uses atomics, so a repeated call is bitwise identical.
#include "mpd.cuh"

namespace st {

namespace {

constexpr float kSlope = 0.1f;              // DiscriminatorP.lrelu_slope
constexpr int kRedThreads = 256;

__device__ __forceinline__ void put(const MpdPlanes& P, long long i, float v) {
    if (P.f) P.f[i] = v;
    if (P.hi) { bf16 h, l; split_bf16(v, h, l); P.hi[i] = h; P.lo[i] = l; }
}

// sample hin of column j of batch row b after the right reflect pad (padded sample L + i = x[L - 2 - i]); zero outside [0, Hin)
__device__ __forceinline__ float x_in(const float* __restrict__ x, const MpdGeo& g, int b, int j, int hin) {
    if (hin < 0 || hin >= g.Hin) return 0.f;
    long long t = (long long)hin * g.p + j;
    if (t >= g.L) t = 2 * g.L - 2 - t;
    return x[(long long)b * g.L + t];
}

__global__ void conv0_fwd_kernel(const float* __restrict__ x, MpdGeo g, int H0, int R, const float* __restrict__ w,
                                 const float* __restrict__ bias, float* __restrict__ fmap0, MpdPlanes out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.p * R * 32) return;
    const int c = (int)(i % 32), h = (int)((i / 32) % R), bb = (int)(i / (32LL * R));
    const int b = bb / g.p, j = bb % g.p;
    float v = 0.f;
    if (h < H0) {
        v = bias[c];
        for (int k = 0; k < 5; ++k) v = fmaf(w[c * 5 + k], x_in(x, g, b, j, 3 * h + k - 2), v);
        v = v > 0.f ? v : v * kSlope;
        fmap0[(((long long)b * 32 + c) * H0 + h) * g.p + j] = v;
    }
    put(out, i, v);
}

__global__ void act_fwd_kernel(const float* __restrict__ Y, MpdGeo g, int H, int C, int R, float slope, float* __restrict__ fmap,
                               MpdPlanes out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.p * R * C) return;
    const int c = (int)(i % C), h = (int)((i / C) % R), bb = (int)(i / ((long long)C * R));
    float v = 0.f;
    if (h < H) {
        v = Y[((long long)bb * H + h) * C + c];
        v = v > 0.f ? v : v * slope;
        const int b = bb / g.p, j = bb % g.p;
        fmap[(((long long)b * C + c) * H + h) * g.p + j] = v;
    }
    put(out, i, v);
}

// one block: 32 consecutive (h, j) positions of one batch row; warp w sums channels [128 w, 128 w + 128), lanes the positions
__global__ void __launch_bounds__(256) post_fwd_kernel(const float* __restrict__ f, MpdGeo g, int H, const float* __restrict__ w,
                                                       const float* __restrict__ bias, float* __restrict__ post) {
    __shared__ float part[8][32];
    const int b = blockIdx.y, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const int HP = H * g.p, q = blockIdx.x * 32 + lane;
    const int h = q / g.p;
    float acc = 0.f;
    if (q < HP) {
        const float* base = f + (long long)b * 1024 * HP + q;
        for (int c = wp * 128; c < wp * 128 + 128; ++c) {
            const float* fc = base + (long long)c * HP;
            if (h > 0) acc = fmaf(w[c * 3 + 0], fc[-g.p], acc);
            acc = fmaf(w[c * 3 + 1], fc[0], acc);
            if (h + 1 < H) acc = fmaf(w[c * 3 + 2], fc[g.p], acc);
        }
    }
    part[wp][lane] = acc;
    __syncthreads();
    if (wp == 0 && q < HP) {
        float v = 0.f;
        for (int i = 0; i < 8; ++i) v += part[i][lane];
        post[(long long)b * HP + q] = v + bias[0];
    }
}

// packings (W = the reference weight (Cout, Cin, 5)):
//   FWD_S3   [2][Cout][3 Cin]  stride-3 conv as a 2-tap conv over lane groups of 3 rows: tap 0 reads group o - 1 (lane l is
//            kernel tap l - 1; lane 0 is outside the kernel: zero), tap 1 reads group o (kernel tap l + 2)
//   FWD_S1   [5][Cout][Cin]    plain 5-tap conv
//   DGRAD_S3 [2][3 Cin][Cout]  the adjoint of FWD_S3: output row r = input group r - 1; tap 0 reads dZ[r - 1] = dZ[group]
//            (kernel tap l + 2), tap 1 reads dZ[group + 1] (kernel tap l - 1; zero for lane 0)
//   DGRAD_S1 [5][Cin][Cout]    flipped, transposed taps
__global__ void pack_kernel(const float* __restrict__ w, int Cout, int Cin, int mode, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool s3 = mode == MPD_PACK_FWD_S3 || mode == MPD_PACK_DGRAD_S3;
    const int K3 = s3 ? 3 * Cin : Cin, taps = s3 ? 2 : 5;
    if (i >= (long long)taps * Cout * K3) return;
    int n, c, l = 0, tap, k;
    if (mode == MPD_PACK_FWD_S3 || mode == MPD_PACK_FWD_S1) {
        const int kk = (int)(i % K3);
        n = (int)((i / K3) % Cout);
        tap = (int)(i / ((long long)K3 * Cout));
        c = kk % Cin; l = kk / Cin;
        k = s3 ? (tap == 0 ? l - 1 : l + 2) : tap;
    } else {
        n = (int)(i % Cout);
        const int kk = (int)((i / Cout) % K3);
        tap = (int)(i / ((long long)K3 * Cout));
        c = kk % Cin; l = kk / Cin;
        k = s3 ? (tap == 0 ? l + 2 : l - 1) : 4 - tap;
    }
    out[i] = k < 0 ? 0.f : w[((long long)n * Cin + c) * 5 + k];
}

__global__ void post_dgrad_kernel(const float* __restrict__ gpost, MpdGeo g, int H, const float* __restrict__ w, float* __restrict__ G) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.p * H * 1024) return;
    const int c = (int)(i % 1024), h = (int)((i / 1024) % H), bb = (int)(i / (1024LL * H));
    const int b = bb / g.p, j = bb % g.p;
    const float* gp = gpost + (long long)b * H * g.p + j;
    float v = 0.f;
    for (int k = 0; k < 3; ++k) {
        const int o = h - k + 1;
        if (o >= 0 && o < H) v = fmaf(w[c * 3 + k], gp[(long long)o * g.p], v);
    }
    G[i] = v;
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

// block c: dw[c, k] = Σ_{b, h, j} gpost[b, h, j] fmap4[b, c, h + k - 1, j]; block 1024: db = Σ gpost
__global__ void __launch_bounds__(kRedThreads) post_wgrad_kernel(const float* __restrict__ gpost, const float* __restrict__ f,
                                                                 MpdGeo g, int H, float* __restrict__ dw, float* __restrict__ db) {
    __shared__ float sm[3][kRedThreads];
    const int c = blockIdx.x, HP = H * g.p;
    const long long n = (long long)g.B * HP;
    float acc[3] = {0.f, 0.f, 0.f};
    for (long long i = threadIdx.x; i < n; i += kRedThreads) {
        const int b = (int)(i / HP), q = (int)(i % HP), h = q / g.p;
        const float gv = gpost[i];
        if (c == 1024) { acc[0] += gv; continue; }
        const float* fc = f + ((long long)b * 1024 + c) * HP + q;
        if (h > 0) acc[0] = fmaf(gv, fc[-g.p], acc[0]);
        acc[1] = fmaf(gv, fc[0], acc[1]);
        if (h + 1 < H) acc[2] = fmaf(gv, fc[g.p], acc[2]);
    }
    block_sum<3>(sm, acc);
    if (threadIdx.x == 0) {
        if (c == 1024) db[0] = sm[0][0];
        else for (int k = 0; k < 3; ++k) dw[c * 3 + k] = sm[k][0];
    }
}

__global__ void act_bwd_kernel(const float* __restrict__ G, int Rg, int off, const float* __restrict__ gfmap,
                               const float* __restrict__ fmap, MpdGeo g, int H, int C, MpdPlanes dz, MpdPlanes dzT, long long Kr,
                               float* __restrict__ dz_nchw) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.p * (H + 1) * C) return;
    const int c = (int)(i % C), h = (int)((i / C) % (H + 1)), bb = (int)(i / ((long long)C * (H + 1)));
    if (h == H) { put(dz, i, 0.f); return; }
    const int b = bb / g.p, j = bb % g.p;
    const long long q = (((long long)b * C + c) * H + h) * g.p + j;
    float v = G[((long long)bb * Rg + h + off) * C + c];
    if (gfmap) v += gfmap[q];
    if (fmap) v = fmap[q] > 0.f ? v : v * kSlope;
    put(dz, i, v);
    put(dzT, (long long)c * Kr + (long long)bb * H + h, v);
    if (dz_nchw) dz_nchw[q] = v;
}

__global__ void im2col_t_kernel(const float* __restrict__ f, MpdGeo g, int Hx, int Cin, int H, int stride, long long Kr, MpdPlanes out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)(5 * Cin + 8) * Kr) return;
    const long long r = i % Kr;
    const int row = (int)(i / Kr);
    const long long valid = (long long)g.B * g.p * H;
    float v = 0.f;
    if (r < valid) {
        if (row < 5 * Cin) {
            const int k = row / Cin, c = row % Cin, bb = (int)(r / H), o = (int)(r % H);
            const int hx = stride * o + k - 2;
            if (hx >= 0 && hx < Hx) v = f[(((long long)(bb / g.p) * Cin + c) * Hx + hx) * g.p + bb % g.p];
        } else if (row == 5 * Cin) {
            v = 1.f;
        }
    }
    put(out, i, v);
}

__global__ void unpack_wgrad_kernel(const float* __restrict__ dWp, int Cout, int Cin, float* __restrict__ dw, float* __restrict__ db) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)Cout * Cin * 5) return;
    const int k = (int)(i % 5), c = (int)((i / 5) % Cin), n = (int)(i / (5LL * Cin));
    const long long Np = 5LL * Cin + 8;
    dw[i] = dWp[n * Np + (long long)k * Cin + c];
    if (c == 0 && k == 0) db[n] = dWp[n * Np + 5LL * Cin];
}

// block c: dw[c, k] = Σ dz0[b, c, h, j] x_in(3h + k - 2), db[c] = Σ dz0[b, c, h, j]
__global__ void __launch_bounds__(kRedThreads) conv0_wgrad_kernel(const float* __restrict__ dz0, const float* __restrict__ x,
                                                                  MpdGeo g, int H0, float* __restrict__ dw, float* __restrict__ db) {
    __shared__ float sm[6][kRedThreads];
    const int c = blockIdx.x, HP = H0 * g.p;
    const long long n = (long long)g.B * HP;
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long i = threadIdx.x; i < n; i += kRedThreads) {
        const int b = (int)(i / HP), q = (int)(i % HP), h = q / g.p, j = q % g.p;
        const float d = dz0[((long long)b * 32 + c) * HP + q];
        for (int k = 0; k < 5; ++k) acc[k] = fmaf(d, x_in(x, g, b, j, 3 * h + k - 2), acc[k]);
        acc[5] += d;
    }
    block_sum<6>(sm, acc);
    if (threadIdx.x == 0) {
        for (int k = 0; k < 5; ++k) dw[c * 5 + k] = sm[k][0];
        db[c] = sm[5][0];
    }
}

__device__ float conv0_dgrad_at(const float* __restrict__ dz0, const float* __restrict__ w, const MpdGeo& g, int H0, int b, long long t) {
    const int hin = (int)(t / g.p), j = (int)(t % g.p);
    float v = 0.f;
    for (int k = 0; k < 5; ++k) {
        const int num = hin + 2 - k;
        if (num < 0 || num % 3) continue;
        const int h = num / 3;
        if (h >= H0) continue;
        const float* d = dz0 + ((long long)b * 32 * H0 + h) * g.p + j;
        for (int c = 0; c < 32; ++c) v = fmaf(w[c * 5 + k], d[(long long)c * H0 * g.p], v);
    }
    return v;
}

__global__ void conv0_dgrad_kernel(const float* __restrict__ dz0, const float* __restrict__ w, MpdGeo g, int H0, float* __restrict__ gx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.L) return;
    const int b = (int)(i / g.L);
    const long long t = i % g.L;
    float v = conv0_dgrad_at(dz0, w, g, H0, b, t);
    const long long t2 = 2 * g.L - 2 - t;                   // the padded sample that mirrors t
    if (t2 >= g.L && t2 < (long long)g.Hin * g.p) v += conv0_dgrad_at(dz0, w, g, H0, b, t2);
    gx[i] = v;
}

__global__ void nchw_to_rows_kernel(const float* __restrict__ f, MpdGeo g, int H, int C, int R, MpdPlanes out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)g.B * g.p * R * C) return;
    const int c = (int)(i % C), h = (int)((i / C) % R), bb = (int)(i / ((long long)C * R));
    put(out, i, h < H ? f[(((long long)(bb / g.p) * C + c) * H + h) * g.p + bb % g.p] : 0.f);
}

inline unsigned blocks(long long n) { return (unsigned)((n + 255) / 256); }

}  // namespace

cudaError_t launch_mpd_conv0_fwd(const float* x, MpdGeo g, int H0, int R, const float* w, const float* b, float* fmap0,
                                 MpdPlanes out, cudaStream_t s) {
    conv0_fwd_kernel<<<blocks((long long)g.B * g.p * R * 32), 256, 0, s>>>(x, g, H0, R, w, b, fmap0, out);
    return cudaGetLastError();
}

cudaError_t launch_mpd_act_fwd(const float* Y, MpdGeo g, int H, int C, int R, float* fmap, MpdPlanes out, cudaStream_t s,
                               float slope) {
    act_fwd_kernel<<<blocks((long long)g.B * g.p * R * C), 256, 0, s>>>(Y, g, H, C, R, slope, fmap, out);
    return cudaGetLastError();
}

cudaError_t launch_mpd_nchw_to_rows(const float* fmap, MpdGeo g, int H, int C, int R, MpdPlanes out, cudaStream_t s) {
    nchw_to_rows_kernel<<<blocks((long long)g.B * g.p * R * C), 256, 0, s>>>(fmap, g, H, C, R, out);
    return cudaGetLastError();
}

cudaError_t launch_mpd_post_fwd(const float* fmap4, MpdGeo g, int H, const float* w, const float* b, float* post, cudaStream_t s) {
    post_fwd_kernel<<<dim3((unsigned)((H * g.p + 31) / 32), (unsigned)g.B), 256, 0, s>>>(fmap4, g, H, w, b, post);
    return cudaGetLastError();
}

cudaError_t launch_mpd_pack(const float* w, int Cout, int Cin, int mode, float* out, cudaStream_t s) {
    const bool s3 = mode == MPD_PACK_FWD_S3 || mode == MPD_PACK_DGRAD_S3;
    const long long n = (long long)(s3 ? 6 : 5) * Cout * Cin;
    pack_kernel<<<blocks(n), 256, 0, s>>>(w, Cout, Cin, mode, out);
    return cudaGetLastError();
}

cudaError_t launch_mpd_post_dgrad(const float* gpost, MpdGeo g, int H, const float* w, float* G, cudaStream_t s) {
    post_dgrad_kernel<<<blocks((long long)g.B * g.p * H * 1024), 256, 0, s>>>(gpost, g, H, w, G);
    return cudaGetLastError();
}

cudaError_t launch_mpd_post_wgrad(const float* gpost, const float* fmap4, MpdGeo g, int H, float* dw, float* db, cudaStream_t s) {
    post_wgrad_kernel<<<1025, kRedThreads, 0, s>>>(gpost, fmap4, g, H, dw, db);
    return cudaGetLastError();
}

cudaError_t launch_mpd_act_bwd(const float* G, int Rg, int off, const float* gfmap, const float* fmap, MpdGeo g, int H, int C,
                               MpdPlanes dz, MpdPlanes dzT, long long Kr, float* dz_nchw, cudaStream_t s) {
    act_bwd_kernel<<<blocks((long long)g.B * g.p * (H + 1) * C), 256, 0, s>>>(G, Rg, off, gfmap, fmap, g, H, C, dz, dzT, Kr, dz_nchw);
    return cudaGetLastError();
}

cudaError_t launch_mpd_im2col_t(const float* fmap, MpdGeo g, int Hx, int Cin, int H, int stride, long long Kr, MpdPlanes out,
                                cudaStream_t s) {
    im2col_t_kernel<<<blocks((long long)(5 * Cin + 8) * Kr), 256, 0, s>>>(fmap, g, Hx, Cin, H, stride, Kr, out);
    return cudaGetLastError();
}

cudaError_t launch_mpd_unpack_wgrad(const float* dWp, int Cout, int Cin, float* dw, float* db, cudaStream_t s) {
    unpack_wgrad_kernel<<<blocks((long long)Cout * Cin * 5), 256, 0, s>>>(dWp, Cout, Cin, dw, db);
    return cudaGetLastError();
}

cudaError_t launch_mpd_conv0_wgrad(const float* dz0, const float* x, MpdGeo g, int H0, float* dw, float* db, cudaStream_t s) {
    conv0_wgrad_kernel<<<32, kRedThreads, 0, s>>>(dz0, x, g, H0, dw, db);
    return cudaGetLastError();
}

cudaError_t launch_mpd_conv0_dgrad(const float* dz0, const float* w, MpdGeo g, int H0, float* gx, cudaStream_t s) {
    conv0_dgrad_kernel<<<blocks((long long)g.B * g.L), 256, 0, s>>>(dz0, w, g, H0, gx);
    return cudaGetLastError();
}

}  // namespace st
