// C-ABI of the log-mel front end (utils/audio.py::LogMelSpectrogram / LinearSpectrogram, api.py:72-73, preprocess.py:50-73):
// the handle keeps the window, the twiddle table and the mel filters packed by band; st_mel_forward is one launch of
// mel_kernel (mel.cu).
#include "handle.cuh"
#include "mel.cuh"

using namespace st;

namespace st {

struct MelState {
    st_mel_dims d;
    int log2M = 0, n_freqs = 0;
    float* window = nullptr;           // the raw copy of spectrogram.window (owned by h->raw)
    float2* tw = nullptr;
    float* fbT = nullptr;
    int2* band = nullptr;
};

void mel_free(st_handle* h) {
    delete (MelState*)h->mel;
    h->mel = nullptr;
}

int mel_finalize(st_handle* h, cudaStream_t s) {
    MelState* m = (MelState*)h->mel;
    if (!m) return fail(h, "internal: mel state missing");
    const st_mel_dims& d = m->d;
    if (get_raw(h, "spectrogram.window", d.n_fft, &m->window)) return 1;
    if (dev_alloc(h, &m->tw, (size_t)d.n_fft / 2)) return 1;
    ST_CUDA(launch_mel_twiddles(d.n_fft, m->tw, s));
    if (d.n_mels > 0) {
        float* fb;
        if (get_raw(h, "mel_scale.fb", (int64_t)m->n_freqs * d.n_mels, &fb)) return 1;
        if (dev_alloc(h, &m->fbT, (size_t)m->n_freqs * d.n_mels) || dev_alloc(h, &m->band, (size_t)d.n_mels)) return 1;
        ST_CUDA(launch_mel_pack_fb(fb, m->n_freqs, d.n_mels, m->fbT, m->band, s));
    }
    return 0;
}

}  // namespace st

extern "C" {

int st_create_mel(const st_mel_dims* dims, int device, st_handle** out) {
    if (!dims || !out) return fail(nullptr, "st_create_mel: null argument");
    const st_mel_dims& d = *dims;
    if (d.n_fft < 256 || d.n_fft > 4096 || (d.n_fft & (d.n_fft - 1)))
        return fail(nullptr, "n_fft must be a power of two in [256, 4096]");
    if (d.hop_length <= 0) return fail(nullptr, "hop_length must be positive");
    if (d.pad < 0) return fail(nullptr, "pad must be non-negative");
    if (d.n_mels < 0 || d.n_mels > 4096) return fail(nullptr, "n_mels must be in [0, 4096] (0: linear spectrogram only)");
    // a CFM-estimator-shaped handle carries the device / error plumbing; its dims are the reference ModelConfig's
    st_dims base = {80, 256, 1024, 4, 6, 3, 256};
    int rc = st_create(&base, device, out);
    if (rc) return rc;
    st_handle* h = *out;
    h->kind = 6;
    MelState* m = new MelState();
    m->d = d;
    while ((2 << m->log2M) < d.n_fft) ++m->log2M;                       // M = n_fft / 2 = 1 << log2M
    m->n_freqs = d.n_fft / 2 + 1;
    h->mel = m;
    return 0;
}

int st_mel_forward(st_handle* h, const float* wav, float* out, int B, int64_t L, int linear, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (h->kind != 6 || !h->mel) return fail(h, "handle is not a mel spectrogram");
    if (!h->finalized) return fail(h, "weights not finalized (call st_finalize_weights)");
    if (!wav || !out) return fail(h, "st_mel_forward: null pointer");
    const MelState* m = (const MelState*)h->mel;
    const st_mel_dims& d = m->d;
    if (!linear && d.n_mels == 0) return fail(h, "this handle was created with n_mels = 0: only the linear spectrogram");
    if (B <= 0 || B > 65535) return fail(h, "B must be in [1, 65535]");
    if (L <= (int64_t)d.pad)
        return fail(h, "reflect padding needs pad < L (pad " + std::to_string(d.pad) + ", L " + std::to_string(L) + ")");
    if (L + 2 * (int64_t)d.pad < d.n_fft)
        return fail(h, "input too short: L + 2 pad = " + std::to_string(L + 2 * (int64_t)d.pad) + " < n_fft = " +
                           std::to_string(d.n_fft) + " gives no frame");
    const int64_t T = (L + 2 * (int64_t)d.pad - d.n_fft) / d.hop_length + 1;
    if (T > ((int64_t)1 << 30)) return fail(h, "input too long");
    MelArgs a;
    a.wav = wav; a.window = m->window; a.tw = m->tw; a.fbT = m->fbT; a.band = m->band; a.out = out;
    a.L = L; a.B = B; a.T = (int)T; a.hop = d.hop_length; a.pad = d.pad; a.log2M = m->log2M; a.n_mels = d.n_mels;
    a.linear = linear ? 1 : 0;
    ST_LAUNCH(launch_mel(a, (cudaStream_t)stream));
    return 0;
}

}  // extern "C"
