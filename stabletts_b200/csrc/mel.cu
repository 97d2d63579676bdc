// Log-mel spectrogram of utils/audio.py::LogMelSpectrogram (center = False, reflect padding), fp32, one kernel:
//
//   mel_kernel      a CTA takes P consecutive frames of one batch row (P = 8, or 4 at n_fft = 4096) and, in shared memory:
//                   1. loads each frame with the reflect padding folded into the index (F.pad(..., "reflect")), times the
//                      window;
//                   2. runs the real FFT of size N = n_fft as an M = N/2 point complex FFT of z[n] = x[2n] + i x[2n+1]:
//                      decimation in frequency, in place, radix-2 stages fused pairwise into radix-4 butterflies (the same
//                      arithmetic as the radix-2 stages, half the passes over shared memory), output in bit-reversed order;
//                   3. splits Z into the half spectrum X[k], k = 0..M, and writes |X| = sqrt(re^2 + im^2 + 1e-6);
//                   4. either writes |X| (LinearSpectrogram) or sums each mel filter over its non-zero band [k0, k1) in
//                      ascending k and writes log(max(., 1e-5)).
//                   Writes go to (B, C, T) with T fastest: P consecutive frames of one row per 32 / 16-byte segment.
//   mel_twiddles    exp(-2 pi i t / N), t < M, evaluated in double with exact argument reduction and rounded to fp32
//   mel_pack_fb     mel_scale.fb (n_freqs, n_mels) -> per-filter rows and non-zero bands
//
// There is no tensor-core path: the magnitude feeds a log, which turns absolute error in re / im into large relative error
// in spectral valleys, so the transform stays in fp32 throughout.
#include "mel.cuh"

namespace st {

constexpr int MEL_THREADS = 256;

__device__ __forceinline__ int fpad(int i) { return i + (i >> 4); }      // one float2 of padding per 16: conflict-free strides

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 w) { return make_float2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x); }

__host__ __device__ inline int frames_per_cta(int log2M) { return log2M <= 10 ? 8 : 4; }
// floats of shared memory per frame: the padded complex buffer, then M + 1 magnitudes (rounded up to 16 bytes)
__host__ __device__ inline int frame_stride(int log2M) {
    const int M = 1 << log2M;
    return 2 * (M + M / 16) + (M + 1 + 3) / 4 * 4;
}

__global__ void __launch_bounds__(MEL_THREADS) mel_kernel(MelArgs a) {
    extern __shared__ float4 smem4[];
    float* sm = reinterpret_cast<float*>(smem4);
    const int lm = a.log2M, M = 1 << lm, N = 2 * M, P = frames_per_cta(lm), FS = frame_stride(lm);
    const int b = blockIdx.y, t0 = blockIdx.x * P;
    const int nf = min(P, a.T - t0);
    const float* x = a.wav + (long long)b * a.L;
    pdl_trigger(); pdl_wait();

    // 1. windowed frames; padded-signal sample t*hop + n is input sample t*hop + n - pad, reflected at both edges
    for (int i = threadIdx.x; i < P * N; i += MEL_THREADS) {
        const int f = i >> (lm + 1), n = i & (N - 1);
        float v = 0.f;
        if (f < nf) {
            long long s = (long long)(t0 + f) * a.hop + n - a.pad;
            if (s < 0) s = -s;
            else if (s >= a.L) s = 2 * (a.L - 1) - s;
            v = __ldg(x + s) * __ldg(a.window + n);
        }
        sm[f * FS + 2 * fpad(n >> 1) + (n & 1)] = v;
    }
    __syncthreads();

    // 2. M-point complex FFT.  Radix-2 DIF stage of span h: (u, v) -> (u + v, (u - v) W_2h^j).  Two consecutive stages (h,
    //    h/2) on the four points i0, i0 + h/2, i0 + h, i0 + 3h/2 make one radix-4 butterfly; W_2h^(j + h/2) = -i W_2h^j.
    int lh = lm - 1;                                                     // log2 of the current span
    for (; lh >= 1; lh -= 2) {
        const int h = 1 << lh, h2 = h >> 1, tws = M >> lh;              // W_2h^j = tw[j M / h], W_h^j = tw[2 j M / h]
        for (int i = threadIdx.x; i < P * (M / 4); i += MEL_THREADS) {
            const int f = i >> (lm - 2), q = i & (M / 4 - 1);
            float2* z = reinterpret_cast<float2*>(sm + f * FS);
            const int j = q & (h2 - 1);
            const int i0 = ((q >> (lh - 1)) << (lh + 1)) + j;
            const float2 x0 = z[fpad(i0)], x1 = z[fpad(i0 + h2)], x2 = z[fpad(i0 + h)], x3 = z[fpad(i0 + h + h2)];
            const float2 w1 = __ldg(a.tw + j * tws), w2 = __ldg(a.tw + 2 * j * tws);
            const float2 a0 = cadd(x0, x2), a1 = cadd(x1, x3);
            const float2 a2 = cmul(csub(x0, x2), w1);
            const float2 d = csub(x1, x3);
            const float2 a3 = cmul(make_float2(d.y, -d.x), w1);
            z[fpad(i0)] = cadd(a0, a1);
            z[fpad(i0 + h2)] = cmul(csub(a0, a1), w2);
            z[fpad(i0 + h)] = cadd(a2, a3);
            z[fpad(i0 + h + h2)] = cmul(csub(a2, a3), w2);
        }
        __syncthreads();
    }
    if (lh == 0) {                                                       // odd log2 M: a last radix-2 stage of span 1
        for (int i = threadIdx.x; i < P * (M / 2); i += MEL_THREADS) {
            const int f = i >> (lm - 1), q = i & (M / 2 - 1);
            float2* z = reinterpret_cast<float2*>(sm + f * FS);
            const float2 u = z[fpad(2 * q)], v = z[fpad(2 * q + 1)];
            z[fpad(2 * q)] = cadd(u, v);
            z[fpad(2 * q + 1)] = csub(u, v);
        }
        __syncthreads();
    }

    // 3. half spectrum X[k] = E[k] + W_N^k O[k], E = (Z[k] + conj Z[M-k]) / 2, O = -i (Z[k] - conj Z[M-k]) / 2 (Z[M] = Z[0],
    //    W_N^M = -1); Z[k] sits at bit-reversed position
    const int MP = M + 1;
    for (int i = threadIdx.x; i < P * MP; i += MEL_THREADS) {
        const int f = i / MP, k = i - f * MP;
        const float2* z = reinterpret_cast<const float2*>(sm + f * FS);
        const int r = (int)(__brev((unsigned)(k & (M - 1))) >> (32 - lm));
        const int rm = (int)(__brev((unsigned)((M - k) & (M - 1))) >> (32 - lm));
        const float2 zk = z[fpad(r)], zm = z[fpad(rm)];
        const float2 e = make_float2((zk.x + zm.x) * 0.5f, (zk.y - zm.y) * 0.5f);
        const float2 o = make_float2((zk.y + zm.y) * 0.5f, (zm.x - zk.x) * 0.5f);
        const float2 w = k < M ? __ldg(a.tw + k) : make_float2(-1.f, 0.f);
        const float2 X = cadd(e, cmul(o, w));
        sm[f * FS + 2 * (M + M / 16) + k] = sqrtf(X.x * X.x + X.y * X.y + 1e-6f);
    }
    __syncthreads();

    // 4. output rows, frames fastest
    const float* mag = sm + 2 * (M + M / 16);
    const int lp = P == 8 ? 3 : 2;
    if (a.linear) {
        float* out = a.out + (long long)b * MP * a.T + t0;
        for (int i = threadIdx.x; i < MP * P; i += MEL_THREADS) {
            const int k = i >> lp, f = i & (P - 1);
            if (f < nf) out[(long long)k * a.T + f] = mag[f * FS + k];
        }
        return;
    }
    float* out = a.out + (long long)b * a.n_mels * a.T + t0;
    for (int i = threadIdx.x; i < a.n_mels * P; i += MEL_THREADS) {
        const int m = i >> lp, f = i & (P - 1);
        if (f >= nf) continue;
        const int2 band = __ldg(a.band + m);
        const float* w = a.fbT + (long long)m * MP;
        const float* mg = mag + f * FS;
        float acc = 0.f;
        for (int k = band.x; k < band.y; ++k) acc = fmaf(__ldg(w + k), mg[k], acc);
        out[(long long)m * a.T + f] = logf(acc < 1e-5f ? 1e-5f : acc);       // torch.clamp(min=1e-5) keeps NaN
    }
}

__global__ void mel_twiddles_kernel(int n_fft, float2* __restrict__ tw) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_fft / 2) return;
    double sn, cs;
    sincospi(2.0 * (double)t / (double)n_fft, &sn, &cs);                // t < n_fft: the argument is already reduced
    tw[t] = make_float2((float)cs, (float)-sn);
}

__global__ void mel_pack_fb_kernel(const float* __restrict__ fb, int n_freqs, int n_mels, float* __restrict__ fbT,
                                   int2* __restrict__ band) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_mels) return;
    int k0 = n_freqs, k1 = 0;
    for (int k = 0; k < n_freqs; ++k) {
        const float v = fb[(long long)k * n_mels + m];
        fbT[(long long)m * n_freqs + k] = v;
        if (v != 0.f) { k0 = min(k0, k); k1 = k + 1; }
    }
    band[m] = k1 > 0 ? make_int2(k0, k1) : make_int2(0, 0);
}

cudaError_t launch_mel(const MelArgs& a, cudaStream_t s) {
    static std::atomic<uint64_t> smem_done{0};
    const int P = frames_per_cta(a.log2M);
    const int bytes = P * frame_stride(a.log2M) * 4;
    constexpr int kMaxBytes = 8 * (2 * (1024 + 64) + 1028) * 4;            // the largest of any supported n_fft
    static_assert(kMaxBytes >= 4 * (2 * (2048 + 128) + 2052) * 4, "n_fft = 4096 must fit");
    cudaError_t e = ensure_dyn_smem(mel_kernel, kMaxBytes, smem_done);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)((a.T + P - 1) / P), (unsigned)a.B);
    return launch_k(mel_kernel, grid, dim3(MEL_THREADS), (size_t)bytes, s, a);
}

cudaError_t launch_mel_twiddles(int n_fft, float2* tw, cudaStream_t s) {
    mel_twiddles_kernel<<<(n_fft / 2 + 255) / 256, 256, 0, s>>>(n_fft, tw);
    return cudaGetLastError();
}

cudaError_t launch_mel_pack_fb(const float* fb, int n_freqs, int n_mels, float* fbT, int2* band, cudaStream_t s) {
    mel_pack_fb_kernel<<<(n_mels + 127) / 128, 128, 0, s>>>(fb, n_freqs, n_mels, fbT, band);
    return cudaGetLastError();
}

}  // namespace st
