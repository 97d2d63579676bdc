// Log-mel / linear spectrogram kernels (mel.cu), the multi-scale mel loss (mel_loss.cu); orchestration in mel_api.cu.
// The per-frame device code (windowed load, FFT, real split, banded mel sum, log) is shared here so that the loss's log-mels
// are bit for bit the ones LogMelSpectrogram writes.
#pragma once
#include "common.cuh"

namespace st {

struct MelArgs {
    const float* wav = nullptr;        // (B, L) fp32
    const float* window = nullptr;     // (n_fft)
    const float2* tw = nullptr;        // (n_fft / 2) twiddles exp(-2 pi i t / n_fft)
    const float* fbT = nullptr;        // (n_mels, n_fft / 2 + 1): mel_scale.fb transposed
    const int2* band = nullptr;        // (n_mels) [k0, k1): the bins where filter m is non-zero
    float* out = nullptr;              // (B, n_mels, T) log-mel, or (B, n_fft / 2 + 1, T) magnitude when linear
    long long L = 0;
    int B = 0, T = 0, hop = 0, pad = 0, log2M = 0, n_mels = 0, linear = 0;
};
cudaError_t launch_mel(const MelArgs& a, cudaStream_t s);
cudaError_t launch_mel_twiddles(int n_fft, float2* tw, cudaStream_t s);
cudaError_t launch_mel_pack_fb(const float* fb, int n_freqs, int n_mels, float* fbT, int2* band, int2* kband, cudaStream_t s);

constexpr int MEL_THREADS = 256;
constexpr int MEL_LOSS_MAX_SCALES = 16;
constexpr int MEL_LOSS_MAX_SMEM = 220 * 1024;             // dynamic shared memory of one CTA; the opt-in limit is 227 KB

// One scale of the multi-scale loss: frames of x and y through the log-mel of MelArgs, |Δ| partial sums, and (when gfx /
// gfy are set) the per-frame waveform gradient of mean |Δ| for a unit upstream gradient.
struct MelLossArgs {
    const float* x = nullptr; const float* y = nullptr;      // (B, L)
    const float* window = nullptr; const float2* tw = nullptr; const float* fbT = nullptr; const int2* band = nullptr;
    const float* fb = nullptr;         // (n_freqs, n_mels) as loaded
    const int2* kband = nullptr;       // (n_freqs) [m0, m1): the filters that are non-zero at bin k
    double* part = nullptr;            // (B, ceil(T / Q)) per-CTA sums of |Δ|
    float* gfx = nullptr; float* gfy = nullptr;              // (B, T, n_fft) frame gradients, or nullptr
    long long L = 0;
    int B = 0, T = 0, hop = 0, pad = 0, log2M = 0, n_mels = 0;
    float inv_n = 0.f;                 // 1 / (B n_mels T) in fp32, as torch's mean backward forms it
};
struct MelLossScale { const float* gf; int T, hop, pad, log2N; };
struct MelLossGatherArgs {
    MelLossScale sc[MEL_LOSS_MAX_SCALES];
    float* grad = nullptr;             // (B, L)
    long long L = 0;
    int B = 0, n_scales = 0;
};
struct MelLossFinalArgs {
    const double* part = nullptr;
    long long off[MEL_LOSS_MAX_SCALES + 1];                  // scale s owns part[off[s], off[s + 1])
    double numel[MEL_LOSS_MAX_SCALES];                       // B n_mels T of scale s
    float* loss = nullptr;
    int n_scales = 0;
};
int mel_loss_frames_per_input(int log2M);                    // Q: frames of x (and of y) per CTA
int mel_loss_smem_bytes(int log2M, int n_mels);
cudaError_t launch_mel_loss(const MelLossArgs& a, cudaStream_t s);
cudaError_t launch_mel_loss_final(const MelLossFinalArgs& a, cudaStream_t s);
cudaError_t launch_mel_loss_gather(const MelLossGatherArgs& a, cudaStream_t s);

// ---- shared per-frame device code --------------------------------------------------------------------------------------

__device__ __forceinline__ int fpad(int i) { return i + (i >> 4); }      // one float2 of padding per 16: conflict-free strides

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 w) { return make_float2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x); }

// frames per CTA: 8 (4 at n_fft = 4096), and 2048 / n_fft below n_fft = 256 so that a CTA still loads >= 2048 samples
__host__ __device__ inline int frames_per_cta(int log2M) { return log2M < 7 ? 1 << (10 - log2M) : log2M <= 10 ? 8 : 4; }
// floats of the padded complex buffer of one frame; the M + 1 magnitudes follow it
__host__ __device__ inline int mel_zfloats(int log2M) { const int M = 1 << log2M; return 2 * (M + M / 16); }
__host__ __device__ inline int mel_magfloats(int log2M) { return ((1 << log2M) + 1 + 3) / 4 * 4; }

// 1. windowed frames: slot f of P takes frame t of row `row` when src(f, row, t) is true, else zeros; padded-signal sample
//    t*hop + n is input sample t*hop + n - pad, reflected at both edges
template <class Src>
__device__ __forceinline__ void mel_load_frames(float* sm, int lm, int P, int FS, const float* __restrict__ window, long long L,
                                                int hop, int pad, Src src) {
    const int N = 2 << lm;
    for (int i = threadIdx.x; i < P * N; i += MEL_THREADS) {
        const int f = i >> (lm + 1), n = i & (N - 1);
        float v = 0.f;
        const float* x; int t;
        if (src(f, x, t)) {
            long long s = (long long)t * hop + n - pad;
            if (s < 0) s = -s;
            else if (s >= L) s = 2 * (L - 1) - s;
            v = __ldg(x + s) * __ldg(window + n);
        }
        sm[f * FS + 2 * fpad(n >> 1) + (n & 1)] = v;
    }
    __syncthreads();
}

// 2. M-point complex FFT of every slot, in place.  Radix-2 DIF stage of span h: (u, v) -> (u + v, (u - v) W_2h^j).  Two
//    consecutive stages (h, h/2) on the four points i0, i0 + h/2, i0 + h, i0 + 3h/2 make one radix-4 butterfly;
//    W_2h^(j + h/2) = -i W_2h^j.  Natural order in, bit-reversed order out.
__device__ __forceinline__ void mel_fft(float* sm, int lm, int P, int FS, const float2* __restrict__ tw) {
    const int M = 1 << lm;
    int lh = lm - 1;                                                     // log2 of the current span
    for (; lh >= 1; lh -= 2) {
        const int h = 1 << lh, h2 = h >> 1, tws = M >> lh;              // W_2h^j = tw[j M / h], W_h^j = tw[2 j M / h]
        for (int i = threadIdx.x; i < P * (M / 4); i += MEL_THREADS) {
            const int f = i >> (lm - 2), q = i & (M / 4 - 1);
            float2* z = reinterpret_cast<float2*>(sm + f * FS);
            const int j = q & (h2 - 1);
            const int i0 = ((q >> (lh - 1)) << (lh + 1)) + j;
            const float2 x0 = z[fpad(i0)], x1 = z[fpad(i0 + h2)], x2 = z[fpad(i0 + h)], x3 = z[fpad(i0 + h + h2)];
            const float2 w1 = __ldg(tw + j * tws), w2 = __ldg(tw + 2 * j * tws);
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
}

__device__ __forceinline__ int mel_brev(int k, int lm) { return (int)(__brev((unsigned)k) >> (32 - lm)); }

// 3. half spectrum X[k] = E[k] + W_N^k O[k], E = (Z[k] + conj Z[M-k]) / 2, O = -i (Z[k] - conj Z[M-k]) / 2 (Z[M] = Z[0],
//    W_N^M = -1); Z[k] sits at bit-reversed position.  Writes |X| = sqrt(re^2 + im^2 + 1e-6) after the complex buffer and,
//    when xoff > 0, X itself at float offset xoff of the slot.
__device__ __forceinline__ void mel_half_spectrum(float* sm, int lm, int P, int FS, const float2* __restrict__ tw, int xoff) {
    const int M = 1 << lm, MP = M + 1, zf = mel_zfloats(lm);
    for (int i = threadIdx.x; i < P * MP; i += MEL_THREADS) {
        const int f = i / MP, k = i - f * MP;
        const float2* z = reinterpret_cast<const float2*>(sm + f * FS);
        const int r = mel_brev(k & (M - 1), lm);
        const int rm = mel_brev((M - k) & (M - 1), lm);
        const float2 zk = z[fpad(r)], zm = z[fpad(rm)];
        const float2 e = make_float2((zk.x + zm.x) * 0.5f, (zk.y - zm.y) * 0.5f);
        const float2 o = make_float2((zk.y + zm.y) * 0.5f, (zm.x - zk.x) * 0.5f);
        const float2 w = k < M ? __ldg(tw + k) : make_float2(-1.f, 0.f);
        const float2 X = cadd(e, cmul(o, w));
        sm[f * FS + zf + k] = sqrtf(X.x * X.x + X.y * X.y + 1e-6f);
        if (xoff > 0) reinterpret_cast<float2*>(sm + f * FS + xoff)[k] = X;
    }
    __syncthreads();
}

// 4. filter m summed over its non-zero band in ascending k, and the log of the clamped sum (torch.clamp(min=1e-5) keeps NaN)
__device__ __forceinline__ float mel_band_sum(const float* __restrict__ fbT, const int2* __restrict__ band, const float* mg,
                                              int m, int MP) {
    const int2 bd = __ldg(band + m);
    const float* w = fbT + (long long)m * MP;
    float acc = 0.f;
    for (int k = bd.x; k < bd.y; ++k) acc = fmaf(__ldg(w + k), mg[k], acc);
    return acc;
}
__device__ __forceinline__ float mel_log(float acc) { return logf(acc < 1e-5f ? 1e-5f : acc); }

// 5. the adjoint of 1-3 for the ns slots at `sm`: Y_k (M + 1 complex at float offset yoff of each slot) ->
//    c_j = d_{2j} + i d_{2j+1}, d_n = Re Σ_{k=0}^{M} Y_k e^{+2πikn/N} (the one-sided rfft's adjoint, before the window).
//    d is the inverse real DFT of V (V_0 = Re Y_0, V_M = Re Y_M, V_k = Y_k / 2, V_{N−k} = conj V_k); it packs V into
//    C_k = (V_k + conj V_{M−k}) + i e^{+2πik/N} (V_k − conj V_{M−k}) (k < M) and runs mel_fft with conjugates on both sides,
//    c = conj(FFT(conj C)).  mel_irfft_sample reads d_n back (Z bit-reversed).
__device__ __forceinline__ void mel_irfft(float* sm, int lm, int ns, int FS, int yoff, const float2* __restrict__ tw) {
    const int M = 1 << lm;
    for (int i = threadIdx.x; i < ns * M; i += MEL_THREADS) {
        const int f = i >> lm, k = i & (M - 1);
        const float2* Y = reinterpret_cast<const float2*>(sm + f * FS + yoff);
        const float2 yk = Y[k], ym = Y[M - k];
        const float2 vk = k == 0 ? make_float2(yk.x, 0.f) : make_float2(0.5f * yk.x, 0.5f * yk.y);
        const float2 vm = k == 0 ? make_float2(ym.x, 0.f) : make_float2(0.5f * ym.x, 0.5f * ym.y);
        const float2 A = make_float2(vk.x + vm.x, vk.y - vm.y);             // V_k + conj V_{M-k}
        const float2 Bv = make_float2(vk.x - vm.x, vk.y + vm.y);            // V_k - conj V_{M-k}
        const float2 w = __ldg(tw + k);
        const float2 wb = cmul(Bv, make_float2(w.x, -w.y));                 // e^{+2 pi i k / N} B
        const float2 C = make_float2(A.x - wb.y, A.y + wb.x);               // A + i wb
        reinterpret_cast<float2*>(sm + f * FS)[fpad(k)] = make_float2(C.x, -C.y);
    }
    __syncthreads();
    mel_fft(sm, lm, ns, FS, tw);
}
__device__ __forceinline__ float mel_irfft_sample(const float* slot, int lm, int n) {
    const float2 z = reinterpret_cast<const float2*>(slot)[fpad(mel_brev(n >> 1, lm))];
    return (n & 1) ? -z.y : z.x;
}

}  // namespace st
