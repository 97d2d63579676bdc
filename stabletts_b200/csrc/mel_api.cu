// C-ABI of the log-mel front end (utils/audio.py::LogMelSpectrogram / LinearSpectrogram, api.py:72-73, preprocess.py:50-73):
// the handle keeps the window, the twiddle table and the mel filters packed by band; st_mel_forward is one launch of
// mel_kernel (mel.cu).  The multi-scale mel loss (vocoders/vocos/models/loss.py) keeps one such state per scale;
// st_mel_loss_forward is one mel_loss_kernel launch per scale, the loss reduction and, with gradients, one gather per input
// (mel_loss.cu).
#include "handle.cuh"
#include "mel.cuh"

using namespace st;

namespace st {

// one scale: the transform's dims and its packed tables
struct MelScale {
    st_mel_dims d;
    int log2M = 0, n_freqs = 0;
    float* window = nullptr;           // the raw copy of spectrogram.window (owned by h->raw)
    float2* tw = nullptr;
    float* fbT = nullptr;
    int2* band = nullptr;
    float* fb = nullptr;               // the raw copy of mel_scale.fb (loss handles only)
    int2* kband = nullptr;             // loss handles only: per bin, the filters that are non-zero there
};

namespace {

const char* mel_dims_error(const st_mel_dims& d) {
    if (d.n_fft < 32 || d.n_fft > 4096 || (d.n_fft & (d.n_fft - 1))) return "n_fft must be a power of two in [32, 4096]";
    if (d.hop_length <= 0) return "hop_length must be positive";
    if (d.pad < 0) return "pad must be non-negative";
    if (d.n_mels < 0 || d.n_mels > 4096) return "n_mels must be in [0, 4096] (0: linear spectrogram only)";
    return nullptr;
}

void mel_init(MelScale* m, const st_mel_dims& d) {
    m->d = d;
    while ((2 << m->log2M) < d.n_fft) ++m->log2M;                       // M = n_fft / 2 = 1 << log2M
    m->n_freqs = d.n_fft / 2 + 1;
}

// `prefix` + "spectrogram.window" / "mel_scale.fb" -> window, twiddles, band-packed filters (and the loss's per-bin bands)
int mel_pack(st_handle* h, MelScale* m, const std::string& prefix, bool loss, cudaStream_t s) {
    const st_mel_dims& d = m->d;
    if (get_raw(h, prefix + "spectrogram.window", d.n_fft, &m->window)) return 1;
    if (dev_alloc(h, &m->tw, (size_t)d.n_fft / 2)) return 1;
    ST_CUDA(launch_mel_twiddles(d.n_fft, m->tw, s));
    if (d.n_mels > 0) {
        float* fb;
        if (get_raw(h, prefix + "mel_scale.fb", (int64_t)m->n_freqs * d.n_mels, &fb)) return 1;
        if (dev_alloc(h, &m->fbT, (size_t)m->n_freqs * d.n_mels) || dev_alloc(h, &m->band, (size_t)d.n_mels)) return 1;
        m->fb = fb;
        if (loss && dev_alloc(h, &m->kband, (size_t)m->n_freqs)) return 1;
        ST_CUDA(launch_mel_pack_fb(fb, m->n_freqs, d.n_mels, m->fbT, m->band, loss ? m->kband : nullptr, s));
    }
    return 0;
}

}  // namespace

// the log-mel spectrogram
struct MelState : Model {
    MelScale m;
    explicit MelState(const st_mel_dims& d) { mel_init(&m, d); }
    int finalize(st_handle* h, cudaStream_t s) override { return mel_pack(h, &m, "", false, s); }
};

// the multi-scale mel loss: one scale per transform
struct MelLossState : Model {
    std::vector<MelScale> sc;
    int finalize(st_handle* h, cudaStream_t s) override {
        for (size_t i = 0; i < sc.size(); ++i)
            if (mel_pack(h, &sc[i], "mel_transforms." + std::to_string(i) + ".", true, s)) return 1;
        return 0;
    }
};

}  // namespace st

extern "C" {

int st_create_mel(const st_mel_dims* dims, int device, st_handle** out) {
    if (!dims || !out) return fail(nullptr, "st_create_mel: null argument");
    const st_mel_dims& d = *dims;
    if (const char* e = mel_dims_error(d)) return fail(nullptr, e);
    return create_handle(device, std::make_unique<MelState>(d), out);
}

int st_mel_forward(st_handle* h, const float* wav, float* out, int B, int64_t L, int linear, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    const MelState* mel = ready_model<MelState>(h, "mel spectrogram");
    if (!mel) return 1;
    if (!wav || !out) return fail(h, "st_mel_forward: null pointer");
    const MelScale* m = &mel->m;
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

int st_create_mel_loss(int n_scales, const st_mel_dims* dims, int device, st_handle** out) {
    if (!dims || !out) return fail(nullptr, "st_create_mel_loss: null argument");
    if (n_scales < 1 || n_scales > MEL_LOSS_MAX_SCALES)
        return fail(nullptr, "n_scales must be in [1, " + std::to_string(MEL_LOSS_MAX_SCALES) + "]");
    auto L = std::make_unique<MelLossState>();
    L->sc.resize(n_scales);
    for (int i = 0; i < n_scales; ++i) {
        const st_mel_dims& d = dims[i];
        const char* e = mel_dims_error(d);
        if (!e && d.n_mels == 0) e = "n_mels must be positive";
        mel_init(&L->sc[i], d);
        if (!e && mel_loss_smem_bytes(L->sc[i].log2M, d.n_mels) > MEL_LOSS_MAX_SMEM)
            e = "n_mels too large for this n_fft: the frames of one CTA do not fit in shared memory";
        if (e) return fail(nullptr, "scale " + std::to_string(i) + ": " + e);
    }
    return create_handle(device, std::move(L), out);
}

namespace {

struct LossPlan { int64_t T[MEL_LOSS_MAX_SCALES]; size_t part_off[MEL_LOSS_MAX_SCALES + 1], gf_off[MEL_LOSS_MAX_SCALES + 1]; };

// workspace: the per-CTA partial sums (double) of every scale, then the frame gradients of x and of y (fp32)
size_t loss_plan(const MelLossState* L, int B, int64_t Lw, LossPlan* p) {
    p->part_off[0] = 0; p->gf_off[0] = 0;
    const int n = (int)L->sc.size();
    for (int i = 0; i < n; ++i) {
        const st_mel_dims& d = L->sc[i].d;
        const int64_t T = (Lw + 2 * (int64_t)d.pad - d.n_fft) / d.hop_length + 1;
        const int Q = mel_loss_frames_per_input(L->sc[i].log2M);
        p->T[i] = T;
        p->part_off[i + 1] = p->part_off[i] + (size_t)B * (size_t)((T + Q - 1) / Q);
        p->gf_off[i + 1] = p->gf_off[i] + (size_t)B * (size_t)T * d.n_fft;
    }
    const size_t part_bytes = (p->part_off[n] * sizeof(double) + 255) / 256 * 256;
    return part_bytes + 2 * p->gf_off[n] * sizeof(float);
}

}  // namespace

size_t st_mel_loss_workspace_bytes(const st_handle* h, int B, int64_t L) {
    const MelLossState* S = h ? dynamic_cast<const MelLossState*>(h->model.get()) : nullptr;
    if (!S || B <= 0 || L <= 0) return 0;
    LossPlan p;
    return loss_plan(S, B, L, &p);
}

int st_mel_loss_forward(st_handle* h, const float* x, const float* y, int B, int64_t L, float* loss_out, float* gx, float* gy,
                        void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    const MelLossState* S = ready_model<MelLossState>(h, "mel loss");
    if (!S) return 1;
    if (!x || !y || !loss_out) return fail(h, "st_mel_loss_forward: null pointer");
    if (B <= 0 || B > 65535) return fail(h, "B must be in [1, 65535]");
    const int n = (int)S->sc.size();
    for (int i = 0; i < n; ++i) {
        const st_mel_dims& d = S->sc[i].d;
        if (L <= (int64_t)d.pad)
            return fail(h, "reflect padding needs pad < L (scale " + std::to_string(i) + ": pad " + std::to_string(d.pad) +
                               ", L " + std::to_string(L) + ")");
        if (L + 2 * (int64_t)d.pad < d.n_fft)
            return fail(h, "input too short for scale " + std::to_string(i) + ": L + 2 pad = " +
                               std::to_string(L + 2 * (int64_t)d.pad) + " < n_fft = " + std::to_string(d.n_fft));
    }
    if (L > ((int64_t)1 << 30)) return fail(h, "input too long");
    LossPlan p;
    const size_t need = loss_plan(S, B, L, &p);
    if (!h->ws_ptr || h->ws_bytes < need)
        return fail(h, "attached workspace too small: st_mel_loss_workspace_bytes = " + std::to_string(need));
    cudaStream_t s = (cudaStream_t)stream;
    void* ws = h->ws_ptr;
    double* part = (double*)ws;
    float* gfx = (float*)((char*)ws + (p.part_off[n] * sizeof(double) + 255) / 256 * 256);
    float* gfy = gfx + p.gf_off[n];
    MelLossFinalArgs fa;
    fa.part = part; fa.loss = loss_out; fa.n_scales = n;
    MelLossGatherArgs gx_args, gy_args;
    gx_args.L = gy_args.L = L; gx_args.B = gy_args.B = B; gx_args.n_scales = gy_args.n_scales = n;
    gx_args.grad = gx; gy_args.grad = gy;
    for (int i = 0; i < n; ++i) {
        const MelScale& m = S->sc[i];
        const st_mel_dims& d = m.d;
        MelLossArgs a;
        a.x = x; a.y = y; a.window = m.window; a.tw = m.tw; a.fbT = m.fbT; a.band = m.band; a.fb = m.fb; a.kband = m.kband;
        a.part = part + p.part_off[i];
        a.gfx = gx ? gfx + p.gf_off[i] : nullptr;
        a.gfy = gy ? gfy + p.gf_off[i] : nullptr;
        a.L = L; a.B = B; a.T = (int)p.T[i]; a.hop = d.hop_length; a.pad = d.pad; a.log2M = m.log2M; a.n_mels = d.n_mels;
        a.inv_n = 1.f / (float)((double)B * d.n_mels * p.T[i]);
        ST_LAUNCH(launch_mel_loss(a, s));
        fa.off[i] = (long long)p.part_off[i]; fa.off[i + 1] = (long long)p.part_off[i + 1];
        fa.numel[i] = (double)B * d.n_mels * (double)p.T[i];
        gx_args.sc[i] = {a.gfx, a.T, d.hop_length, d.pad, m.log2M + 1};
        gy_args.sc[i] = {a.gfy, a.T, d.hop_length, d.pad, m.log2M + 1};
    }
    ST_LAUNCH(launch_mel_loss_final(fa, s));
    if (gx) ST_LAUNCH(launch_mel_loss_gather(gx_args, s));
    if (gy) ST_LAUNCH(launch_mel_loss_gather(gy_args, s));
    return 0;
}

}  // extern "C"
