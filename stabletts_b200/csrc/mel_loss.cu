// Multi-scale mel loss of vocoders/vocos/models/loss.py (MultiScaleMelSpectrogramLoss), forward and waveform gradient:
//
//   loss = Σ_s mean |mel_s(x) − mel_s(y)|,   mel_s = log(clamp(fb_s^T |STFT_s|, 1e-5))   (utils/audio.py::LogMelSpectrogram)
//
//   mel_loss_kernel        one launch per scale.  A CTA takes Q consecutive frames of one row of x and the same frames of y
//                          (2Q = P slots of mel.cu's tile) through mel.cuh's load -> FFT -> half spectrum -> band sum, so the
//                          log-mels are bit for bit LogMelSpectrogram's; |Δ| of its Q x n_mels cells is summed in double
//                          (fixed tree) into one partial per CTA.  With a gradient requested the same CTA goes on (below).
//   mel_loss_final_kernel  one CTA: each scale's partials in a fixed order, / (B n_mels T), scales ascending -> fp32 loss
//   mel_loss_gather_kernel each waveform sample sums its frame gradients (<= 4 frames per padded position, frames ascending,
//                          the reflect-pad images after the direct position), then the scales in ascending order
//
// The adjoint, per frame (unit upstream gradient; for x the sign of g flips and x's own spectrum is used):
//   g_m = −sgn(Δ_m) / N_s · [mel_m >= 1e-5] / mel_m          sgn(0) = 0; torch.clamp passes the gradient at exactly 1e-5
//   G_k = Σ_m fb[k, m] g_m, over the filters non-zero at k, ascending m
//   Y_k = (G_k / |X_k|) X_k                                   |X_k| = sqrt(re² + im² + 1e-6), the forward's magnitude
//   d_n = w_n Re Σ_{k=0}^{M} Y_k e^{+2πikn/N}                 the adjoint of the one-sided rfft: interior bins not doubled
// d is the inverse real DFT of V (V_0 = Re Y_0, V_M = Re Y_M, V_k = Y_k / 2, V_{N−k} = conj V_k).  As the forward packs the
// real input into an M-point complex FFT, the inverse packs V into C_k = (V_k + conj V_{M−k}) + i e^{+2πik/N} (V_k − conj V_{M−k})
// (k < M), so that c_j = d_{2j} + i d_{2j+1} = Σ_k C_k e^{+2πijk/M} (mel.cuh::mel_irfft).  That inverse runs on mel_fft itself, with
// conjugates on both sides: c = conj(FFT(conj C)).  The frame gradients go to (B, T, n_fft) workspace and the gather adds
// them; no float atomics, so every output is repeatable bit for bit.
#include "mel.cuh"

namespace st {

namespace {

__host__ __device__ inline int loss_frame_stride(int lm, int n_mels) {
    // complex buffer | magnitudes | X (M + 1 complex, kept for the gradient) | mel sums, then g
    return mel_zfloats(lm) + mel_magfloats(lm) + ((1 << lm) + 1) * 2 / 4 * 4 + 4 + (n_mels + 3) / 4 * 4;
}
__host__ __device__ inline int loss_xoff(int lm) { return mel_zfloats(lm) + mel_magfloats(lm); }
__host__ __device__ inline int loss_meloff(int lm) { return loss_xoff(lm) + ((1 << lm) + 1) * 2 / 4 * 4 + 4; }

__device__ double block_sum_double(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(~0u, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < nw ? red[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(~0u, v, o);
    }
    return v;                                            // valid in thread 0
}

__global__ void __launch_bounds__(MEL_THREADS) mel_loss_kernel(MelLossArgs a) {
    extern __shared__ float4 smem4[];
    __shared__ double red[MEL_THREADS / 32];
    float* sm = reinterpret_cast<float*>(smem4);
    const int lm = a.log2M, M = 1 << lm, N = 2 * M, MP = M + 1, P = frames_per_cta(lm), Q = P / 2, lq = __ffs(Q) - 1;
    const int FS = loss_frame_stride(lm, a.n_mels), XO = loss_xoff(lm), MO = loss_meloff(lm), ZF = mel_zfloats(lm);
    const int b = blockIdx.y, t0 = blockIdx.x * Q;
    const int nf = min(Q, a.T - t0);
    const float* xrow = a.x + (long long)b * a.L;
    const float* yrow = a.y + (long long)b * a.L;
    pdl_trigger(); pdl_wait();

    // slots [0, Q) hold frames t0.. of x, slots [Q, 2Q) the same frames of y
    mel_load_frames(sm, lm, P, FS, a.window, a.L, a.hop, a.pad, [&](int f, const float*& x, int& t) {
        x = f < Q ? xrow : yrow; t = t0 + (f & (Q - 1));
        return (f & (Q - 1)) < nf;
    });
    mel_fft(sm, lm, P, FS, a.tw);
    mel_half_spectrum(sm, lm, P, FS, a.tw, XO);
    for (int i = threadIdx.x; i < a.n_mels * P; i += MEL_THREADS) {
        const int m = i / P, f = i - m * P;
        if ((f & (Q - 1)) < nf) sm[f * FS + MO + m] = mel_band_sum(a.fbT, a.band, sm + f * FS + ZF, m, MP);
    }
    __syncthreads();

    // |Δ| and, in place of the mel sums, g for the inputs that want a gradient
    double acc = 0.0;
    for (int i = threadIdx.x; i < a.n_mels * Q; i += MEL_THREADS) {
        const int m = i >> lq, f = i & (Q - 1);
        if (f >= nf) continue;
        float* px = sm + f * FS + MO + m;
        float* py = sm + (f + Q) * FS + MO + m;
        const float mx = *px, my = *py;
        const float d = mel_log(mx) - mel_log(my);
        acc += (double)fabsf(d);
        const float sg = (float)((d > 0.f) - (d < 0.f)) * a.inv_n;
        if (a.gfx) *px = mx >= 1e-5f ? sg / mx : 0.f;
        if (a.gfy) *py = my >= 1e-5f ? -sg / my : 0.f;
    }
    acc = block_sum_double(acc, red);
    if (threadIdx.x == 0) a.part[(long long)b * gridDim.x + blockIdx.x] = acc;
    if (!a.gfx && !a.gfy) return;
    __syncthreads();
    const int f_lo = a.gfx ? 0 : Q, f_hi = a.gfy ? P : Q;           // the slots whose input wants a gradient
    const int ns = f_hi - f_lo;
    const int nm = a.n_mels;

    // Y_k = (G_k / |X_k|) X_k over the stored X
    for (int i = threadIdx.x; i < ns * MP; i += MEL_THREADS) {
        const int f = f_lo + i / MP, k = i % MP;
        if ((f & (Q - 1)) >= nf) continue;
        const float* g = sm + f * FS + MO;
        const int2 kb = __ldg(a.kband + k);
        const float* w = a.fb + (long long)k * nm;
        float G = 0.f;
        for (int m = kb.x; m < kb.y; ++m) G = fmaf(__ldg(w + m), g[m], G);
        const float sc = G / sm[f * FS + ZF + k];
        float2* X = reinterpret_cast<float2*>(sm + f * FS + XO);
        X[k] = make_float2(X[k].x * sc, X[k].y * sc);
    }
    __syncthreads();

    // the inverse real DFT of every Y (mel.cuh), then times the window, to the frame gradients
    mel_irfft(sm + f_lo * FS, lm, ns, FS, XO, a.tw);
    for (int i = threadIdx.x; i < ns * N; i += MEL_THREADS) {
        const int f = f_lo + (i >> (lm + 1)), n = i & (N - 1), fr = f & (Q - 1);
        if (fr >= nf) continue;
        const float d = mel_irfft_sample(sm + f * FS, lm, n);
        float* gf = f < Q ? a.gfx : a.gfy;
        gf[((long long)b * a.T + t0 + fr) * N + n] = d * __ldg(a.window + n);
    }
}

__global__ void mel_loss_final_kernel(MelLossFinalArgs a) {
    __shared__ double red[32];
    pdl_trigger(); pdl_wait();
    double loss = 0.0;
    for (int s = 0; s < a.n_scales; ++s) {
        double v = 0.0;
        for (long long i = a.off[s] + threadIdx.x; i < a.off[s + 1]; i += blockDim.x) v += a.part[i];
        v = block_sum_double(v, red);
        loss += v / a.numel[s];                                          // meaningful in thread 0
    }
    if (threadIdx.x == 0) *a.loss = (float)loss;
}

__global__ void __launch_bounds__(256) mel_loss_gather_kernel(MelLossGatherArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    pdl_trigger(); pdl_wait();
    if (i >= a.L) return;
    const long long L = a.L;
    float total = 0.f;
    for (int s = 0; s < a.n_scales; ++s) {
        const MelLossScale c = a.sc[s];
        const int N = 1 << c.log2N;
        const float* gf = c.gf + (long long)b * c.T * N;
        // padded positions that read sample i: the direct one, then the left and right reflect images
        long long pos[3];
        int np = 0;
        pos[np++] = i + c.pad;
        if (i >= 1 && i <= c.pad) pos[np++] = c.pad - i;
        if (i <= L - 2 && i >= L - 1 - c.pad) pos[np++] = 2 * (L - 1) - i + c.pad;
        float acc = 0.f;
        for (int q = 0; q < np; ++q) {
            const long long p = pos[q];
            long long tlo = p - N + 1 <= 0 ? 0 : (p - N + c.hop) / c.hop;    // ceil((p - N + 1) / hop)
            long long thi = min(p / c.hop, (long long)c.T - 1);
            for (long long t = tlo; t <= thi; ++t) acc += gf[t * N + (p - t * c.hop)];
        }
        total += acc;
    }
    a.grad[(long long)b * L + i] = total;
}

}  // namespace

int mel_loss_frames_per_input(int log2M) { return frames_per_cta(log2M) / 2; }

int mel_loss_smem_bytes(int log2M, int n_mels) { return frames_per_cta(log2M) * loss_frame_stride(log2M, n_mels) * 4; }

cudaError_t launch_mel_loss(const MelLossArgs& a, cudaStream_t s) {
    static std::atomic<uint64_t> smem_done{0};
    cudaError_t e = ensure_dyn_smem(mel_loss_kernel, MEL_LOSS_MAX_SMEM, smem_done);
    if (e != cudaSuccess) return e;
    const int Q = mel_loss_frames_per_input(a.log2M);
    const dim3 grid((unsigned)((a.T + Q - 1) / Q), (unsigned)a.B);
    return launch_k(mel_loss_kernel, grid, dim3(MEL_THREADS), (size_t)mel_loss_smem_bytes(a.log2M, a.n_mels), s, a);
}

cudaError_t launch_mel_loss_final(const MelLossFinalArgs& a, cudaStream_t s) {
    return launch_k(mel_loss_final_kernel, dim3(1), dim3(256), 0, s, a);
}

cudaError_t launch_mel_loss_gather(const MelLossGatherArgs& a, cudaStream_t s) {
    const dim3 grid((unsigned)((a.L + 255) / 256), (unsigned)a.B);
    return launch_k(mel_loss_gather_kernel, grid, dim3(256), 0, s, a);
}

}  // namespace st
