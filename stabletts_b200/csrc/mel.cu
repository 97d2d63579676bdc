// Log-mel spectrogram of utils/audio.py::LogMelSpectrogram (center = False, reflect padding), fp32, one kernel:
//
//   mel_kernel      a CTA takes P consecutive frames of one batch row (P = 8, 4 at n_fft = 4096, 2048 / n_fft below n_fft =
//                   256) and, in shared memory (steps 1-3 and the mel sum are mel.cuh's, shared with mel_loss.cu):
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
//   mel_pack_fb     mel_scale.fb (n_freqs, n_mels) -> per-filter rows and non-zero bands (and, for the loss, the range of
//                   filters that are non-zero at each bin)
//
// There is no tensor-core path: the magnitude feeds a log, which turns absolute error in re / im into large relative error
// in spectral valleys, so the transform stays in fp32 throughout.
#include "mel.cuh"

namespace st {

// floats of shared memory per frame: the padded complex buffer, then M + 1 magnitudes (rounded up to 16 bytes)
__host__ __device__ inline int frame_stride(int log2M) { return mel_zfloats(log2M) + mel_magfloats(log2M); }

__global__ void __launch_bounds__(MEL_THREADS) mel_kernel(MelArgs a) {
    extern __shared__ float4 smem4[];
    float* sm = reinterpret_cast<float*>(smem4);
    const int lm = a.log2M, M = 1 << lm, P = frames_per_cta(lm), FS = frame_stride(lm);
    const int b = blockIdx.y, t0 = blockIdx.x * P;
    const int nf = min(P, a.T - t0);
    const float* xrow = a.wav + (long long)b * a.L;
    pdl_trigger(); pdl_wait();

    mel_load_frames(sm, lm, P, FS, a.window, a.L, a.hop, a.pad, [&](int f, const float*& x, int& t) {
        x = xrow; t = t0 + f;
        return f < nf;
    });
    mel_fft(sm, lm, P, FS, a.tw);
    mel_half_spectrum(sm, lm, P, FS, a.tw, 0);

    // 4. output rows, frames fastest
    const int MP = M + 1;
    const float* mag = sm + mel_zfloats(lm);
    const int lp = __ffs(P) - 1;
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
        out[(long long)m * a.T + f] = mel_log(mel_band_sum(a.fbT, a.band, mag + f * FS, m, MP));
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
                                   int2* __restrict__ band, int2* __restrict__ kband) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m < n_mels) {
        int k0 = n_freqs, k1 = 0;
        for (int k = 0; k < n_freqs; ++k) {
            const float v = fb[(long long)k * n_mels + m];
            fbT[(long long)m * n_freqs + k] = v;
            if (v != 0.f) { k0 = min(k0, k); k1 = k + 1; }
        }
        band[m] = k1 > 0 ? make_int2(k0, k1) : make_int2(0, 0);
    }
    if (kband && m < n_freqs) {                                          // the loss's fb^T product: filters non-zero at bin m
        int m0 = n_mels, m1 = 0;
        for (int j = 0; j < n_mels; ++j)
            if (fb[(long long)m * n_mels + j] != 0.f) { m0 = min(m0, j); m1 = j + 1; }
        kband[m] = m1 > 0 ? make_int2(m0, m1) : make_int2(0, 0);
    }
}

cudaError_t launch_mel(const MelArgs& a, cudaStream_t s) {
    static std::atomic<uint64_t> smem_done{0};
    const int P = frames_per_cta(a.log2M);
    const int bytes = P * frame_stride(a.log2M) * 4;
    constexpr int kMaxBytes = 8 * (2 * (1024 + 64) + 1028) * 4;            // the largest of any supported n_fft
    static_assert(kMaxBytes >= 4 * (2 * (2048 + 128) + 2052) * 4, "n_fft = 4096 must fit");
    static_assert(kMaxBytes >= 64 * (2 * (16 + 1) + 20) * 4, "n_fft = 32 must fit");
    cudaError_t e = ensure_dyn_smem(mel_kernel, kMaxBytes, smem_done);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)((a.T + P - 1) / P), (unsigned)a.B);
    return launch_k(mel_kernel, grid, dim3(MEL_THREADS), (size_t)bytes, s, a);
}

cudaError_t launch_mel_twiddles(int n_fft, float2* tw, cudaStream_t s) {
    mel_twiddles_kernel<<<(n_fft / 2 + 255) / 256, 256, 0, s>>>(n_fft, tw);
    return cudaGetLastError();
}

cudaError_t launch_mel_pack_fb(const float* fb, int n_freqs, int n_mels, float* fbT, int2* band, int2* kband, cudaStream_t s) {
    const int n = kband ? max(n_mels, n_freqs) : n_mels;
    mel_pack_fb_kernel<<<(n + 127) / 128, 128, 0, s>>>(fb, n_freqs, n_mels, fbT, band, kband);
    return cudaGetLastError();
}

}  // namespace st
