// C-ABI of the multi-resolution discriminator (vocoders/vocos/models/discriminator.py:112-171, DiscriminatorR): one handle
// per window length N.  The weights and the window arrive as device pointers on every call and are packed by that call, so
// an optimizer step between two calls is always seen; the handle keeps only the twiddle table of its N, and everything
// backward needs (the spectrum and the band activations) stays in the caller's tensors.
//
// Per band, layer i maps W[i-1] columns to W[i] = ceil(W[i-1] / 2) (convs 1-3, stride (1, 2)) or W[i] = W[i-1] (convs 0,
// 4).  Convs 1-4 and their input and weight gradients run on the conv-GEMM engine (run_gemm) with BB = B T' batches: each
// (b, t') row of a band is one independent sequence along F, whose rows outside [0, W) read as zero (the frequency
// padding).  The three time taps fold into the channels (mrd.cuh "rows": K = lanes 3 C_in, zero rows at t' = -1 and T').
//   forward  convs 1-3: the stride-2, 9-tap conv is a 5-tap conv over lane groups of 2 columns, K = 2 3 32 = 192; tap t lane
//            l is kernel column 2 t + l, so tap 4 lane 1 is a zero weight.  At odd widths the last group's second lane
//            reads the zero column W.  conv 4: a plain 3-tap conv, K = 96
//   dgrad    the same convs with flipped, transposed taps (N = K of the forward), then the fold: each input element sums its
//            three time-tap copies in ascending dt
//   wgrad    dWp[n][(t, kx)] = Σ_r dZ[r, n] rows[r + t - taps / 2, kx] over every row r = (bb, o) of the band: a GEMM with
//            the transposed planes dZ^T as A (T = 32, K = rows) and the transposed, shifted rows as W (N = taps K + 8, the
//            extra row of ones yielding the bias gradient); run_gemm splits its K loop when few tiles cover it
// Conv 0 (2 input channels), conv_post (1 output channel, across the band seams), the STFT and its adjoint are fp32 kernels
// (mrd.cu); the STFT runs on mel.cuh's FFT and its adjoint ends in mel_loss.cu's overlap-add / reflect gather.
#include "handle.cuh"
#include "mel.cuh"
#include "mrd.cuh"

using namespace st;

namespace st {

struct MrdModel : Model {
    int n_fft, lm;                      // lm = log2(n_fft / 2)
    float2* tw = nullptr;               // (n_fft / 2) twiddles, made by the first call
    explicit MrdModel(int n) : n_fft(n), lm(__builtin_ctz((unsigned)n) - 1) {}
    int finalize(st_handle*, cudaStream_t) override { return 0; }   // weights come with every call
};

}  // namespace st

namespace {

constexpr double kBands[6] = {0.0, 0.1, 0.25, 0.5, 0.75, 1.0};

// Shapes of one call and the workspace carved for it.
struct MrdPlan {
    MrdGeo g;
    long long L = 0;
    int F = 0, BB = 0;
    MrdBand band[5];
    int W[5][5] = {};                   // W[k][i]: the width of layer i's output in band k
    float* wf = nullptr; bf16* whi = nullptr; bf16* wlo = nullptr;   // one packed weight
    MrdPlanes rows, dz, dzT, wt;
    float* Y = nullptr;                 // GEMM output: forward activations, then the dgrad results
    float* dWp = nullptr;
    float* G = nullptr;                 // (B, 32, T', W) gradient of the current layer's output
    float* dz0 = nullptr;
    float* gspec = nullptr;             // (B, 2, T', F)
    float* gf = nullptr;                // (B, T', N) frame gradients
    size_t bytes = 0;
};

long long round256(long long n) { return (n + 255) / 256 * 256; }

const char* mrd_shape_error(int n_fft, int B, long long L) {
    if (B <= 0 || B > 65535) return "B must be in [1, 65535]";
    if (L <= n_fft / 2) return "L must be above n_fft / 2: the centred STFT reflect-pads n_fft / 2 samples on each side";
    if (L > (1LL << 30)) return "L must be at most 2^30";
    if ((long long)B * (L / (n_fft / 4) + 1) > 65535) return "B * frames must be at most 65535";
    return nullptr;
}

// The forward carves the packed weight, the rows and a 32-wide Y; the backward the packed weight, the dZ planes, the wgrad
// operand, a Kx-wide Y and the gradient buffers (it never reads the rows).
size_t mrd_plan(int n_fft, int B, long long L, bool tc, bool bwd, void* base, MrdPlan* P) {
    P->L = L;
    P->g.B = B;
    P->g.T = (int)(L / (n_fft / 4) + 1);
    P->F = n_fft / 2 + 1;
    P->BB = B * P->g.T;
    for (int k = 0; k < 5; ++k) {
        const int lo = (int)(kBands[k] * P->F), hi = (int)(kBands[k + 1] * P->F);
        P->band[k].off = lo; P->band[k].W = hi - lo;
        P->W[k][0] = hi - lo;
        for (int i = 1; i < 5; ++i) P->W[k][i] = i < 4 ? (P->W[k][i - 1] + 1) / 2 : P->W[k][i - 1];
    }
    const long long BB = P->BB;
    size_t rows = 0, y = 0, dz = 0, dzT = 0, wt = 0, dwp = 0, gmax = 0;
    for (int k = 0; k < 5; ++k) {
        gmax = std::max<size_t>(gmax, (size_t)B * 32 * P->g.T * P->W[k][0]);
        for (int i = 1; i < 5; ++i) {
            const int lanes = i < 4 ? 2 : 1, Kx = 96 * lanes, taps = mrd_taps(lanes);
            const long long G = P->W[k][i], Kr = round256(BB * G);
            rows = std::max<size_t>(rows, (size_t)(BB * G * Kx));
            y = std::max<size_t>(y, (size_t)(BB * G * (bwd ? Kx : 32)));
            dz = std::max<size_t>(dz, (size_t)(BB * G * 32));
            dzT = std::max<size_t>(dzT, (size_t)(32 * Kr));
            wt = std::max<size_t>(wt, (size_t)((taps * Kx + 8) * Kr));
            dwp = std::max<size_t>(dwp, (size_t)(32 * (taps * Kx + 8)));
        }
    }
    const size_t wmax = 5 * 32 * 192;
    Bump bp(base, SIZE_MAX);
    auto planes = [&](MrdPlanes& q, size_t n) {
        q = MrdPlanes();
        if (tc) { q.hi = bp.take<bf16>(n); q.lo = bp.take<bf16>(n); }
        else q.f = bp.take<float>(n);
    };
    P->wf = bp.take<float>(wmax);
    if (tc) { P->whi = bp.take<bf16>(wmax); P->wlo = bp.take<bf16>(wmax); }
    P->Y = bp.take<float>(y);
    if (!bwd) {
        planes(P->rows, rows);
    } else {
        planes(P->dz, dz);
        planes(P->dzT, dzT);
        planes(P->wt, wt);
        P->dWp = bp.take<float>(dwp);
        P->G = bp.take<float>(gmax);
        P->dz0 = bp.take<float>(gmax);
        P->gspec = bp.take<float>((size_t)B * 2 * P->g.T * P->F);
        P->gf = bp.take<float>((size_t)B * P->g.T * n_fft);
    }
    P->bytes = bp.off + 256;
    return P->bytes;
}

int mrd_enter(st_handle* h, const char* fn, const void* x, const void* window, int B, long long L, bool bwd, MrdPlan* P,
              cudaStream_t s) {
    MrdModel* m = static_cast<MrdModel*>(h->model.get());
    if (!x || !window) return fail(h, std::string(fn) + ": null pointer");
    if (const char* e = mrd_shape_error(m->n_fft, B, L)) return fail(h, std::string(fn) + ": " + e);
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t need = mrd_plan(m->n_fft, B, L, tc, bwd, nullptr, P);
    if (!h->ws_ptr || h->ws_bytes < need)
        return fail(h, std::string("attached workspace too small: st_mrd_workspace_bytes(") + (bwd ? "backward" : "forward") +
                           ") = " + std::to_string(need));
    mrd_plan(m->n_fft, B, L, tc, bwd, h->ws_ptr, P);
    if (!m->tw) {
        if (dev_alloc(h, &m->tw, (size_t)m->n_fft / 2)) return 1;
        ST_CUDA(launch_mel_twiddles(m->n_fft, m->tw, s));
    }
    return 0;
}

int mrd_pack(st_handle* h, const MrdPlan& P, const float* w, int lanes, bool dgrad, GemmW* out, cudaStream_t s) {
    const int Kx = 96 * lanes, taps = mrd_taps(lanes);
    ST_LAUNCH(launch_mrd_pack(w, lanes, dgrad, P.wf, s));
    if (P.whi) ST_LAUNCH(launch_split(P.wf, P.whi, P.wlo, (long)taps * 32 * Kx, s));
    *out = GemmW();
    out->f32 = P.wf; out->hi = P.whi; out->lo = P.wlo;
    out->taps = taps;
    out->N = dgrad ? Kx : 32;
    out->K = dgrad ? 32 : Kx;
    return 0;
}

Act act_of(const MrdPlanes& q, int C) { Act a; a.f32 = q.f; a.hi = q.hi; a.lo = q.lo; a.C = C; return a; }

// Y (BB, G, 32) = the layer's conv of X (B, 32, T', W) + bias, through P.rows
int mrd_fwd_gemm(st_handle* h, const MrdPlan& P, const float* X, int W, int lanes, const float* w, const float* b, cudaStream_t s) {
    const int G = (W + lanes - 1) / lanes;
    ST_LAUNCH(launch_mrd_expand(X, P.g, W, lanes, P.rows, s));
    GemmW Wp;
    if (mrd_pack(h, P, w, lanes, false, &Wp, s)) return 1;
    Wp.bias = const_cast<float*>(b);
    GemmArgs ga;
    ga.BB = P.BB; ga.T = G; ga.a_bmod = P.BB; ga.B = P.BB; ga.flags = EPI_BIAS; ga.batch_invariant = 1;
    const Act a = act_of(P.rows, Wp.K);
    Act y; y.f32 = P.Y; y.C = 32;
    return run_gemm(h, ga, Wp, &a, nullptr, y, s);
}

// dX (B, 32, T', W) = the layer's input gradient of the dZ rows in P.dz (BB, G, 32)
int mrd_dgrad(st_handle* h, const MrdPlan& P, int W, int lanes, const float* w, float* dX, cudaStream_t s) {
    GemmW Wp;
    if (mrd_pack(h, P, w, lanes, true, &Wp, s)) return 1;
    GemmArgs ga;
    ga.BB = P.BB; ga.T = (W + lanes - 1) / lanes; ga.a_bmod = P.BB; ga.B = P.BB; ga.batch_invariant = 1;
    const Act a = act_of(P.dz, 32);
    Act o; o.f32 = P.Y; o.C = Wp.N;
    if (run_gemm(h, ga, Wp, &a, nullptr, o, s)) return 1;
    ST_LAUNCH(launch_mrd_fold(P.Y, P.g, W, lanes, dX, s));
    return 0;
}

// the layer's weight and bias gradients from P.dzT (32 x Kr, columns >= BB G zero) and its input X (B, 32, T', W)
int mrd_wgrad(st_handle* h, const MrdPlan& P, const float* X, int W, int lanes, long long Kr, float* gw, float* gb, cudaStream_t s) {
    ST_LAUNCH(launch_mrd_im2col_t(X, P.g, W, lanes, Kr, P.wt, s));
    GemmW Wo;
    Wo.f32 = P.wt.f; Wo.hi = P.wt.hi; Wo.lo = P.wt.lo; Wo.taps = 1; Wo.N = mrd_taps(lanes) * 96 * lanes + 8; Wo.K = (int)Kr;
    GemmArgs ga;
    ga.BB = 1; ga.T = 32; ga.a_bmod = 1; ga.B = 1;
    const Act a = act_of(P.dzT, (int)Kr);
    Act o; o.f32 = P.dWp; o.C = Wo.N;
    if (run_gemm(h, ga, Wo, &a, nullptr, o, s)) return 1;
    ST_LAUNCH(launch_mrd_unpack_wgrad(P.dWp, lanes, gw, gb, s));
    return 0;
}

int zero_planes(st_handle* h, const MrdPlanes& q, size_t n, cudaStream_t s) {
    if (q.hi) { ST_CUDA(cudaMemsetAsync(q.hi, 0, n * sizeof(bf16), s)); ST_CUDA(cudaMemsetAsync(q.lo, 0, n * sizeof(bf16), s)); }
    if (q.f) ST_CUDA(cudaMemsetAsync(q.f, 0, n * sizeof(float), s));
    return 0;
}

MrdCat cat_of(const MrdPlan& P, const float* const* fmaps) {
    MrdCat c;
    c.off[0] = 0;
    for (int k = 0; k < 5; ++k) { c.f[k] = fmaps[5 * k + 4]; c.off[k + 1] = c.off[k] + P.W[k][4]; }
    return c;
}

}  // namespace

extern "C" {

int st_create_mrd(int n_fft, int device, st_handle** out) {
    if (!out) return fail(nullptr, "st_create_mrd: null argument");
    if (n_fft < 256 || n_fft > 4096 || (n_fft & (n_fft - 1)))
        return fail(nullptr, "n_fft must be a power of two in [256, 4096]");
    return create_handle(device, std::make_unique<MrdModel>(n_fft), out);
}

size_t st_mrd_workspace_bytes(const st_handle* h, int B, int64_t L, int backward) {
    const MrdModel* m = h ? dynamic_cast<const MrdModel*>(h->model.get()) : nullptr;
    if (!m || mrd_shape_error(m->n_fft, B, L)) return 0;
    MrdPlan P;
    return mrd_plan(m->n_fft, B, L, h->engine == ST_ENGINE_TCGEN05, backward != 0, nullptr, &P);
}

int st_mrd_forward(st_handle* h, const float* x, int B, int64_t L, const float* window, const float* const* w,
                   const float* const* b, float* spec, float* const* fmaps, float* post, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    MrdModel* m = model_of<MrdModel>(h, "multi-resolution discriminator");
    if (!m) return 1;
    if (!w || !b || !fmaps || !spec || !post) return fail(h, "st_mrd_forward: null pointer");
    for (int i = 0; i < 26; ++i)
        if (!w[i] || !b[i] || (i < 25 && !fmaps[i])) return fail(h, "st_mrd_forward: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    MrdPlan P;
    if (mrd_enter(h, "st_mrd_forward", x, window, B, L, false, &P, s)) return 1;
    ST_LAUNCH(launch_mrd_stft(x, L, P.g, m->lm, window, m->tw, spec, s));
    for (int k = 0; k < 5; ++k) {
        ST_LAUNCH(launch_mrd_conv0_fwd(spec, P.F, P.g, P.band[k], w[5 * k], b[5 * k], fmaps[5 * k], s));
        for (int i = 1; i < 5; ++i) {
            const int lanes = i < 4 ? 2 : 1;
            if (mrd_fwd_gemm(h, P, fmaps[5 * k + i - 1], P.W[k][i - 1], lanes, w[5 * k + i], b[5 * k + i], s)) return 1;
            ST_LAUNCH(launch_mrd_act_fwd(P.Y, P.g, P.W[k][i], fmaps[5 * k + i], s));
        }
    }
    ST_LAUNCH(launch_mrd_post_fwd(cat_of(P, fmaps), P.g, w[25], b[25], post, s));
    return 0;
}

int st_mrd_backward(st_handle* h, const float* x, int B, int64_t L, const float* window, const float* const* w,
                    const float* spec, const float* const* fmaps, const float* gpost, const float* const* gfmaps, float* gx,
                    float* const* gw, float* const* gb, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    MrdModel* m = model_of<MrdModel>(h, "multi-resolution discriminator");
    if (!m) return 1;
    if (!w || !fmaps || !gpost || !spec) return fail(h, "st_mrd_backward: null pointer");
    for (int i = 0; i < 26; ++i)
        if (!w[i] || (i < 25 && !fmaps[i])) return fail(h, "st_mrd_backward: null pointer");
    if (!gw != !gb) return fail(h, "st_mrd_backward: gw and gb are both given or both NULL");
    if (gw)
        for (int i = 0; i < 26; ++i)
            if (!gw[i] || !gb[i]) return fail(h, "st_mrd_backward: null gradient pointer");
    if (!gw && !gx) return fail(h, "st_mrd_backward: nothing to compute (gx, gw and gb are NULL)");
    cudaStream_t s = (cudaStream_t)stream;
    MrdPlan P;
    if (mrd_enter(h, "st_mrd_backward", x, window, B, L, true, &P, s)) return 1;
    const MrdCat cat = cat_of(P, fmaps);
    if (gw) ST_LAUNCH(launch_mrd_post_wgrad(gpost, cat, P.g, gw[25], gb[25], s));
    for (int k = 0; k < 5; ++k) {
        ST_LAUNCH(launch_mrd_post_dgrad(gpost, cat, k, P.g, w[25], P.G, s));
        for (int i = 4; i >= 1; --i) {
            const int lanes = i < 4 ? 2 : 1, Wo = P.W[k][i];
            const long long Kr = round256((long long)P.BB * Wo);
            if (gw && zero_planes(h, P.dzT, (size_t)32 * Kr, s)) return 1;
            ST_LAUNCH(launch_mrd_act_bwd(P.G, gfmaps ? gfmaps[4 * k + i - 1] : nullptr, fmaps[5 * k + i], P.g, Wo, P.dz,
                                         gw ? P.dzT : MrdPlanes(), Kr, nullptr, s));
            if (gw && mrd_wgrad(h, P, fmaps[5 * k + i - 1], P.W[k][i - 1], lanes, Kr, gw[5 * k + i], gb[5 * k + i], s)) return 1;
            if (mrd_dgrad(h, P, P.W[k][i - 1], lanes, w[5 * k + i], P.G, s)) return 1;
        }
        ST_LAUNCH(launch_mrd_act_bwd(P.G, nullptr, fmaps[5 * k], P.g, P.W[k][0], MrdPlanes(), MrdPlanes(), 0, P.dz0, s));
        if (gw) ST_LAUNCH(launch_mrd_conv0_wgrad(P.dz0, spec, P.F, P.g, P.band[k], gw[5 * k], gb[5 * k], s));
        if (gx) ST_LAUNCH(launch_mrd_conv0_dgrad(P.dz0, P.g, P.band[k], P.F, w[5 * k], P.gspec, s));
    }
    if (gx) {
        ST_LAUNCH(launch_mrd_stft_adj(P.gspec, P.g, m->lm, window, m->tw, P.gf, s));
        MelLossGatherArgs ga;
        ga.sc[0] = MelLossScale{P.gf, P.g.T, m->n_fft / 4, m->n_fft / 2, m->lm + 1};
        ga.grad = gx; ga.L = L; ga.B = B; ga.n_scales = 1;
        ST_LAUNCH(launch_mel_loss_gather(ga, s));
    }
    return 0;
}

int st_test_mrd_conv(st_handle* h, int mode, int layer, int B, int T, int W, const float* x, const float* dz, const float* w,
                     const float* b, float* out, float* out_b, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!model_of<MrdModel>(h, "multi-resolution discriminator")) return 1;
    if (mode < 0 || mode > 2) return fail(h, "st_test_mrd_conv: mode must be 0 (forward), 1 (dgrad) or 2 (wgrad)");
    if (layer < 1 || layer > 4) return fail(h, "st_test_mrd_conv: layer must be in [1, 4]");
    if (B < 1 || T < 1 || W < 1 || (long long)B * T > 65535 || W > 4097) return fail(h, "st_test_mrd_conv: bad B, T or W");
    if (!out || (mode != 1 && !x) || (mode != 0 && !dz) || (mode != 2 && !w) || (mode == 0 && !b) || (mode == 2 && !out_b))
        return fail(h, "st_test_mrd_conv: null pointer");
    const int lanes = layer < 4 ? 2 : 1, Kx = 96 * lanes, taps = mrd_taps(lanes), G = (W + lanes - 1) / lanes;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    MrdPlan P;
    P.g.B = B; P.g.T = T; P.BB = B * T;
    const long long BB = P.BB, Kr = round256(BB * G);
    const size_t wn = (size_t)taps * 32 * Kx, rn = (size_t)BB * G * Kx, dzn = (size_t)BB * G * 32, dzTn = (size_t)32 * Kr;
    const size_t wtn = (size_t)(taps * Kx + 8) * Kr;
    TestBufs bufs;
    auto planes = [&](MrdPlanes& q, size_t n) {
        if (tc) { q.hi = bufs.take<bf16>(n); q.lo = bufs.take<bf16>(n); } else q.f = bufs.take<float>(n);
    };
    P.wf = bufs.take<float>(wn);
    if (tc) { P.whi = bufs.take<bf16>(wn); P.wlo = bufs.take<bf16>(wn); }
    planes(P.rows, rn); planes(P.dz, dzn); planes(P.dzT, dzTn); planes(P.wt, wtn);
    P.Y = bufs.take<float>(rn); P.dWp = bufs.take<float>((size_t)32 * (taps * Kx + 8));
    if (!bufs.ok) return fail(h, "st_test_mrd_conv: out of memory");
    cudaStream_t s = (cudaStream_t)stream;
    if (mode == 0) {                          // out (B, 32, T, G) = conv(x) + b, no activation
        if (mrd_fwd_gemm(h, P, x, W, lanes, w, b, s)) return 1;
        ST_CUDA(launch_mrd_act_fwd(P.Y, P.g, G, out, s, 1.f));
    } else if (mode == 1) {                   // out (B, 32, T, W) = the input gradient of dz (B, 32, T, G)
        ST_CUDA(launch_mrd_act_bwd(dz, nullptr, nullptr, P.g, G, P.dz, MrdPlanes(), 0, nullptr, s));
        if (mrd_dgrad(h, P, W, lanes, w, out, s)) return 1;
    } else {                                  // out (32, 32, 3, kw), out_b (32): the weight and bias gradients
        if (zero_planes(h, P.dzT, dzTn, s)) return 1;
        ST_CUDA(launch_mrd_act_bwd(dz, nullptr, nullptr, P.g, G, MrdPlanes(), P.dzT, Kr, nullptr, s));
        if (mrd_wgrad(h, P, x, W, lanes, Kr, out, out_b, s)) return 1;
    }
    return hook_done(h, s, "st_test_mrd_conv");
}

}  // extern "C"
