// Log-mel / linear spectrogram kernels (mel.cu); orchestration in mel_api.cu.
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
cudaError_t launch_mel_pack_fb(const float* fb, int n_freqs, int n_mels, float* fbT, int2* band, cudaStream_t s);

}  // namespace st
