// C-ABI of the multi-period discriminator (vocoders/vocos/models/discriminator.py:33-79, DiscriminatorP): one handle per
// period.  The weights arrive as device pointers on every call and are packed by that call, so an optimizer step between
// two calls is always seen; the handle keeps no state between calls, and everything backward needs (the input and the
// fmaps) stays in the caller's tensors.
//
// Per column (b, j) of the (B, 1, H, p) view, layer i maps H[i-1] rows to H[i] = ceil(H[i-1] / 3) rows (convs 0-3, stride 3)
// or H[i] = H[i-1] (conv 4, conv_post).  Convs 1-4 and their input and weight gradients run on the conv-GEMM engine
// (run_gemm) with BB = B p batches of one column each; conv 0 and conv_post are fp32 row kernels (mpd.cu).
//   forward  convs 1-3: a stride-3 conv is a 2-tap conv over the input viewed in lane groups of 3 rows, K = 3 Cin
//            conv 4: a plain 5-tap conv
//   dgrad    convs 1-3: the adjoint 2-tap conv with N = 3 Cin whose output row r is input group r - 1 (dZ gets one zero
//            row at its end); conv 4: flipped, transposed taps
//   wgrad    dWp[n][(k, c)] = Σ_r dZ[r, n] X[s o + k - 2, c] over every row r = (bb, o) of the batch: a GEMM with the
//            transposed planes dZ^T as A (T = Cout, K = rows) and the transposed, shifted input as W (N = 5 Cin + 8, the
//            extra row of ones yielding the bias gradient); run_gemm splits its K loop when few tiles cover it
#include "handle.cuh"
#include "mpd.cuh"

using namespace st;

namespace st {

struct MpdModel : Model {
    int period;
    explicit MpdModel(int p) : period(p) {}
    int finalize(st_handle*, cudaStream_t) override { return 0; }   // weights come with every call
};

}  // namespace st

namespace {

constexpr int kCin[5] = {1, 32, 128, 512, 1024};
constexpr int kCout[5] = {32, 128, 512, 1024, 1024};
constexpr int kStride[5] = {3, 3, 3, 3, 1};

// Shapes of one call and the workspace carved for it.
struct MpdPlan {
    MpdGeo g;
    int BB = 0, H[5] = {};
    long long Kr[5] = {};          // wgrad K of layers 1-4: BB H[i] rounded up to 256 (split-K needs whole 64-column blocks)
    float* wf = nullptr; bf16* whi = nullptr; bf16* wlo = nullptr;   // one packed weight
    MpdPlanes act, dz, dzT, wt;
    float* Y = nullptr;            // GEMM output: forward activations, then the dgrad results
    float* dWp = nullptr;
    float* dz0 = nullptr;
    size_t bytes = 0;
};

const char* mpd_shape_error(int p, int B, long long L) {
    if (B <= 0 || B > 65535) return "B must be in [1, 65535]";
    if (L <= 0 || L > (1LL << 30)) return "L must be in [1, 2^30]";
    const long long npad = L % p ? p - L % p : 0;
    if (npad >= L) return "L too short for the reflect pad: the pad p - L % p must be below L";
    if ((long long)B * p > 65535) return "B * period must be at most 65535";
    return nullptr;
}

size_t mpd_plan(int p, int B, long long L, bool tc, void* base, MpdPlan* P) {
    P->g.B = B; P->g.p = p; P->g.L = L;
    const long long Lp = L % p ? L + p - L % p : L;
    P->g.Hin = (int)(Lp / p);
    P->BB = B * p;
    int prev = P->g.Hin;
    for (int i = 0; i < 5; ++i) { P->H[i] = kStride[i] == 3 ? (prev + 2) / 3 : prev; prev = P->H[i]; }
    const long long BB = P->BB;
    size_t wmax = 0, act = 0, y = 0, dz = 0, dzT = 0, wt = 0, dwp = 0;
    for (int i = 1; i < 5; ++i) {
        const long long Ci = kCin[i], Co = kCout[i], H = P->H[i];
        const bool s3 = kStride[i] == 3;
        P->Kr[i] = (BB * H + 255) / 256 * 256;
        wmax = std::max<size_t>(wmax, (size_t)(s3 ? 6 : 5) * Ci * Co);
        act = std::max<size_t>(act, (size_t)(BB * (s3 ? 3 * H : H) * Ci));
        y = std::max<size_t>(y, (size_t)(BB * H * Co));
        y = std::max<size_t>(y, (size_t)(BB * (H + 1) * (s3 ? 3 * Ci : Ci)));
        dz = std::max<size_t>(dz, (size_t)(BB * (H + 1) * Co));
        dzT = std::max<size_t>(dzT, (size_t)(Co * P->Kr[i]));
        wt = std::max<size_t>(wt, (size_t)((5 * Ci + 8) * P->Kr[i]));
        dwp = std::max<size_t>(dwp, (size_t)(Co * (5 * Ci + 8)));
    }
    y = std::max<size_t>(y, (size_t)(BB * P->H[4] * 1024));      // conv_post's dgrad
    Bump bp(base, SIZE_MAX);
    auto planes = [&](MpdPlanes& q, size_t n) {
        q = MpdPlanes();
        if (tc) { q.hi = bp.take<bf16>(n); q.lo = bp.take<bf16>(n); }
        else q.f = bp.take<float>(n);
    };
    P->wf = bp.take<float>(wmax);
    if (tc) { P->whi = bp.take<bf16>(wmax); P->wlo = bp.take<bf16>(wmax); }
    planes(P->act, act);
    planes(P->dz, dz);
    planes(P->dzT, dzT);
    planes(P->wt, wt);
    P->Y = bp.take<float>(y);
    P->dWp = bp.take<float>(dwp);
    P->dz0 = bp.take<float>((size_t)B * 32 * P->H[0] * p);
    P->bytes = bp.off + 256;
    return P->bytes;
}

// common checks of forward and backward; fills the plan over the attached workspace
int mpd_enter(st_handle* h, const char* fn, const void* x, int B, long long L, MpdPlan* P) {
    const MpdModel* m = static_cast<const MpdModel*>(h->model.get());
    if (!x) return fail(h, std::string(fn) + ": null pointer");
    if (const char* e = mpd_shape_error(m->period, B, L)) return fail(h, std::string(fn) + ": " + e);
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t need = mpd_plan(m->period, B, L, tc, nullptr, P);
    if (!h->ws_ptr || h->ws_bytes < need)
        return fail(h, std::string("attached workspace too small: st_mpd_workspace_bytes = ") + std::to_string(need));
    mpd_plan(m->period, B, L, tc, h->ws_ptr, P);
    return 0;
}

// packs layer i's weight in `mode` into the plan's weight buffer (and its split planes on the wgmma engine)
int mpd_pack(st_handle* h, const MpdPlan& P, const float* w, int i, int mode, GemmW* out, cudaStream_t s) {
    const bool s3 = kStride[i] == 3, fwd = mode == MPD_PACK_FWD_S3 || mode == MPD_PACK_FWD_S1;
    const long long n = (long long)(s3 ? 6 : 5) * kCin[i] * kCout[i];
    ST_LAUNCH(launch_mpd_pack(w, kCout[i], kCin[i], mode, P.wf, s));
    if (P.whi) ST_LAUNCH(launch_split(P.wf, P.whi, P.wlo, n, s));
    *out = GemmW();
    out->f32 = P.wf; out->hi = P.whi; out->lo = P.wlo;
    out->taps = s3 ? 2 : 5;
    out->N = fwd ? kCout[i] : (s3 ? 3 : 1) * kCin[i];
    out->K = fwd ? (s3 ? 3 : 1) * kCin[i] : kCout[i];
    return 0;
}

Act act_of(const MpdPlanes& q, int C) { Act a; a.f32 = q.f; a.hi = q.hi; a.lo = q.lo; a.C = C; return a; }

// layer i's weight and bias gradients from the transposed planes P.dzT (C_out x Kr, columns >= BB H zero) and the layer
// input X = fmap (B, C_in, Hx, p): the transposed, shifted input, one GEMM, the unpack
int mpd_wgrad(st_handle* h, const MpdPlan& P, int i, const float* X, int Hx, int H, long long Kr, float* gw, float* gb,
              cudaStream_t s) {
    const int Ci = kCin[i], Co = kCout[i];
    ST_LAUNCH(launch_mpd_im2col_t(X, P.g, Hx, Ci, H, kStride[i], Kr, P.wt, s));
    GemmW W;
    W.f32 = P.wt.f; W.hi = P.wt.hi; W.lo = P.wt.lo; W.taps = 1; W.N = 5 * Ci + 8; W.K = (int)Kr;
    GemmArgs ga;
    ga.BB = 1; ga.T = Co; ga.a_bmod = 1; ga.B = 1;
    const Act a = act_of(P.dzT, (int)Kr);
    Act o; o.f32 = P.dWp; o.C = W.N;
    if (run_gemm(h, ga, W, &a, nullptr, o, s)) return 1;
    ST_LAUNCH(launch_mpd_unpack_wgrad(P.dWp, Co, Ci, gw, gb, s));
    return 0;
}

// layer i's input gradient from the dZ rows P.dz (BB, H + 1, C_out) into P.Y; *Rg / *off: where input row h lands
int mpd_dgrad(st_handle* h, const MpdPlan& P, int i, const float* w, int H, int* Rg, int* off, cudaStream_t s) {
    const bool s3 = kStride[i] == 3;
    GemmW W;
    if (mpd_pack(h, P, w, i, s3 ? MPD_PACK_DGRAD_S3 : MPD_PACK_DGRAD_S1, &W, s)) return 1;
    GemmArgs ga;
    ga.BB = P.BB; ga.T = H + 1; ga.a_bmod = P.BB; ga.B = P.BB; ga.batch_invariant = 1;
    const Act a = act_of(P.dz, kCout[i]);
    Act o; o.f32 = P.Y; o.C = W.N;
    if (run_gemm(h, ga, W, &a, nullptr, o, s)) return 1;
    *Rg = s3 ? 3 * (H + 1) : H + 1;                            // input row h is output row h + off of its column
    *off = s3 ? 3 : 0;
    return 0;
}

// layer i's forward GEMM from the rows in P.act into P.Y (BB, H[i], C_out), bias in the epilogue
int mpd_fwd_gemm(st_handle* h, const MpdPlan& P, int i, const float* w, const float* b, int H, cudaStream_t s) {
    const bool s3 = kStride[i] == 3;
    GemmW W;
    if (mpd_pack(h, P, w, i, s3 ? MPD_PACK_FWD_S3 : MPD_PACK_FWD_S1, &W, s)) return 1;
    W.bias = const_cast<float*>(b);
    GemmArgs ga;
    ga.BB = P.BB; ga.T = H; ga.a_bmod = P.BB; ga.B = P.BB; ga.flags = EPI_BIAS; ga.batch_invariant = 1;
    const Act a = act_of(P.act, W.K);
    Act y; y.f32 = P.Y; y.C = kCout[i];
    return run_gemm(h, ga, W, &a, nullptr, y, s);
}

int zero_planes(st_handle* h, const MpdPlanes& q, size_t n, cudaStream_t s) {
    if (q.hi) { ST_CUDA(cudaMemsetAsync(q.hi, 0, n * sizeof(bf16), s)); ST_CUDA(cudaMemsetAsync(q.lo, 0, n * sizeof(bf16), s)); }
    if (q.f) ST_CUDA(cudaMemsetAsync(q.f, 0, n * sizeof(float), s));
    return 0;
}

// st_test_mpd_row_ex: what each kind reads and writes, and the checks of its descriptor
enum : unsigned { IN_X = 1, IN_W = 2, IN_B = 4, IN_Y = 8, IN_G = 16, IN_GPOST = 32, IN_FMAP = 64, IN_DZ0 = 128, IN_DWP = 256 };
enum : unsigned { OUT_F = 1, OUT_B = 2, OUT_ROWS = 4, OUT_TR = 8 };

struct MpdRowKind { unsigned in, writes, needs; };   // in: IN_* required; writes: OUT_* allowed; needs: OUT_* required
constexpr MpdRowKind kMpdRowKinds[] = {
    {IN_X | IN_W | IN_B, OUT_F | OUT_ROWS, OUT_F},
    {IN_Y, OUT_F | OUT_ROWS, OUT_F},
    {IN_FMAP, OUT_ROWS, OUT_ROWS},
    {IN_FMAP | IN_W | IN_B, OUT_F, OUT_F},
    {IN_W, OUT_F, OUT_F},
    {IN_GPOST | IN_W, OUT_F, OUT_F},
    {IN_GPOST | IN_FMAP, OUT_F | OUT_B, OUT_F | OUT_B},
    {IN_G, OUT_F | OUT_ROWS | OUT_TR, 0},
    {IN_FMAP, OUT_TR, OUT_TR},
    {IN_DWP, OUT_F | OUT_B, OUT_F | OUT_B},
    {IN_DZ0 | IN_X, OUT_F | OUT_B, OUT_F | OUT_B},
    {IN_DZ0 | IN_W, OUT_F, OUT_F},
};
static_assert(sizeof(kMpdRowKinds) / sizeof(kMpdRowKinds[0]) == ST_TEST_MPD_ROW_CONV0_DGRAD + 1, "one entry per kind");

// fills *g (and *H0) for the kinds with a geometry; nullptr when the descriptor is inside the contract
const char* test_mpd_row_error(const st_test_mpd_row_desc& d, MpdGeo* g, int* H0) {
    if (d.kind < 0 || d.kind > ST_TEST_MPD_ROW_CONV0_DGRAD) return "unknown kind";
    const MpdRowKind& k = kMpdRowKinds[d.kind];
    if (!d.rows_hi != !d.rows_lo || !d.tr_hi != !d.tr_lo) return "a plane set's hi and lo go together";
    const unsigned in = (d.x ? IN_X : 0) | (d.w ? IN_W : 0) | (d.b ? IN_B : 0) | (d.Y ? IN_Y : 0) | (d.G ? IN_G : 0) |
                        (d.gpost ? IN_GPOST : 0) | (d.fmap ? IN_FMAP : 0) | (d.dz0 ? IN_DZ0 : 0) | (d.dWp ? IN_DWP : 0);
    const unsigned out = (d.out ? OUT_F : 0) | (d.out_b ? OUT_B : 0) | (d.rows_f || d.rows_hi ? OUT_ROWS : 0) |
                         (d.tr_f || d.tr_hi ? OUT_TR : 0);
    if (k.in & ~in) return "a required input is NULL";
    if (k.needs & ~out) return "a required output is NULL";
    if (out & ~k.writes) return "an output this kind does not write is given";
    if (!out) return "no output requested";
    if (d.kind == ST_TEST_MPD_ROW_PACK || d.kind == ST_TEST_MPD_ROW_UNPACK_WGRAD) {
        if (d.Cout < 1 || d.Cin < 1) return "Cout, Cin >= 1";
        if (d.kind == ST_TEST_MPD_ROW_PACK && (d.mode < MPD_PACK_FWD_S3 || d.mode > MPD_PACK_DGRAD_S1)) return "unknown pack mode";
        return nullptr;
    }
    if (d.p < 1 || d.p > 4096) return "p must be in [1, 4096]";
    if (const char* e = mpd_shape_error(d.p, d.B, d.L)) return e;
    MpdPlan P;
    mpd_plan(d.p, d.B, d.L, false, nullptr, &P);             // Hin as st_mpd_forward derives it
    *g = P.g;
    *H0 = P.H[0];
    const long long BBH = (long long)d.B * d.p * d.H;
    switch (d.kind) {
    case ST_TEST_MPD_ROW_CONV0_FWD:
    case ST_TEST_MPD_ROW_CONV0_WGRAD:
    case ST_TEST_MPD_ROW_CONV0_DGRAD:
        if (d.H != P.H[0]) return "H must be H0 = ceil(ceil(L / p) / 3)";
        if (d.kind == ST_TEST_MPD_ROW_CONV0_FWD && d.R < d.H) return "R must be >= H";
        return nullptr;
    case ST_TEST_MPD_ROW_ACT_FWD:
    case ST_TEST_MPD_ROW_NCHW_TO_ROWS:
        if (d.H < 1 || d.C < 1) return "H, C >= 1";
        if (d.R < d.H) return "R must be >= H";
        return nullptr;
    case ST_TEST_MPD_ROW_POST_FWD:
    case ST_TEST_MPD_ROW_POST_DGRAD:
    case ST_TEST_MPD_ROW_POST_WGRAD:
        if (d.C != 1024) return "C must be 1024, conv_post's one input width";
        if (d.H < 1) return "H >= 1";
        return nullptr;
    case ST_TEST_MPD_ROW_ACT_BWD:
        if (d.H < 1 || d.C < 1 || d.off < 0) return "H, C >= 1 and off >= 0";
        if (d.Rg < d.H + d.off) return "Rg must be >= H + off";
        if ((out & OUT_TR) && d.Kr < BBH) return "Kr must be >= B p H";
        return nullptr;
    case ST_TEST_MPD_ROW_IM2COL_T:
        if (d.stride != 1 && d.stride != 3) return "stride must be 1 or 3";
        if (d.Cin < 1 || d.Hx < 1) return "Cin, Hx >= 1";
        if (d.H != (d.stride == 3 ? (d.Hx + 2) / 3 : d.Hx)) return "H must be ceil(Hx / 3) (stride 3) or Hx (stride 1)";
        if (d.Kr < BBH) return "Kr must be >= B p H";
        return nullptr;
    }
    return "unknown kind";
}

}  // namespace

extern "C" {

int st_create_mpd(int period, int device, st_handle** out) {
    if (!out) return fail(nullptr, "st_create_mpd: null argument");
    if (period < 1 || period > 4096) return fail(nullptr, "period must be in [1, 4096]");
    return create_handle(device, std::make_unique<MpdModel>(period), out);
}

size_t st_mpd_workspace_bytes(const st_handle* h, int B, int64_t L) {
    const MpdModel* m = h ? dynamic_cast<const MpdModel*>(h->model.get()) : nullptr;
    if (!m || mpd_shape_error(m->period, B, L)) return 0;
    MpdPlan P;
    return mpd_plan(m->period, B, L, h->engine == ST_ENGINE_TCGEN05, nullptr, &P);
}

int st_mpd_forward(st_handle* h, const float* x, int B, int64_t L, const float* const* w, const float* const* b,
                   float* const* fmaps, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!model_of<MpdModel>(h, "multi-period discriminator")) return 1;
    if (!w || !b || !fmaps) return fail(h, "st_mpd_forward: null pointer");
    for (int i = 0; i < 6; ++i)
        if (!w[i] || !b[i] || !fmaps[i]) return fail(h, "st_mpd_forward: null pointer");
    MpdPlan P;
    if (mpd_enter(h, "st_mpd_forward", x, B, L, &P)) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    const MpdGeo& g = P.g;
    ST_LAUNCH(launch_mpd_conv0_fwd(x, g, P.H[0], 3 * P.H[1], w[0], b[0], fmaps[0], P.act, s));
    for (int i = 1; i < 5; ++i) {
        if (mpd_fwd_gemm(h, P, i, w[i], b[i], P.H[i], s)) return 1;
        const int R = i < 3 ? 3 * P.H[i + 1] : P.H[i];          // rows per column of the next layer's input
        ST_LAUNCH(launch_mpd_act_fwd(P.Y, g, P.H[i], kCout[i], R, fmaps[i], i < 4 ? P.act : MpdPlanes(), s));
    }
    ST_LAUNCH(launch_mpd_post_fwd(fmaps[4], g, P.H[4], w[5], b[5], fmaps[5], s));
    return 0;
}

int st_mpd_backward(st_handle* h, const float* x, int B, int64_t L, const float* const* w, const float* const* fmaps,
                    const float* gpost, const float* const* gfmaps, float* gx, float* const* gw, float* const* gb, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!model_of<MpdModel>(h, "multi-period discriminator")) return 1;
    if (!w || !fmaps || !gpost) return fail(h, "st_mpd_backward: null pointer");
    for (int i = 0; i < 6; ++i)
        if (!w[i] || (i < 5 && !fmaps[i])) return fail(h, "st_mpd_backward: null pointer");
    if (!gw != !gb) return fail(h, "st_mpd_backward: gw and gb are both given or both NULL");
    if (gw)
        for (int i = 0; i < 6; ++i)
            if (!gw[i] || !gb[i]) return fail(h, "st_mpd_backward: null gradient pointer");
    if (!gw && !gx) return fail(h, "st_mpd_backward: nothing to compute (gx, gw and gb are NULL)");
    MpdPlan P;
    if (mpd_enter(h, "st_mpd_backward", x, B, L, &P)) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    const MpdGeo& g = P.g;
    ST_LAUNCH(launch_mpd_post_dgrad(gpost, g, P.H[4], w[5], P.Y, s));
    if (gw) ST_LAUNCH(launch_mpd_post_wgrad(gpost, fmaps[4], g, P.H[4], gw[5], gb[5], s));
    int Rg = P.H[4], off = 0;                                   // where P.Y holds the gradient of layer i's output
    for (int i = 4; i >= 1; --i) {
        const int H = P.H[i];
        if (gw && zero_planes(h, P.dzT, (size_t)kCout[i] * P.Kr[i], s)) return 1;
        ST_LAUNCH(launch_mpd_act_bwd(P.Y, Rg, off, gfmaps ? gfmaps[i - 1] : nullptr, fmaps[i], g, H, kCout[i], P.dz,
                                     gw ? P.dzT : MpdPlanes(), P.Kr[i], nullptr, s));
        if (gw && mpd_wgrad(h, P, i, fmaps[i - 1], P.H[i - 1], H, P.Kr[i], gw[i], gb[i], s)) return 1;
        if (mpd_dgrad(h, P, i, w[i], H, &Rg, &off, s)) return 1;
    }
    ST_LAUNCH(launch_mpd_act_bwd(P.Y, Rg, off, nullptr, fmaps[0], g, P.H[0], 32, MpdPlanes(), MpdPlanes(), 0, P.dz0, s));
    if (gw) ST_LAUNCH(launch_mpd_conv0_wgrad(P.dz0, x, g, P.H[0], gw[0], gb[0], s));
    if (gx) ST_LAUNCH(launch_mpd_conv0_dgrad(P.dz0, w[0], g, P.H[0], gx, s));
    return 0;
}

int st_test_mpd_conv(st_handle* h, int mode, int layer, int B, int Hx, const float* x, const float* dz, const float* w,
                     const float* b, float* out, float* out_b, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    const MpdModel* m = model_of<MpdModel>(h, "multi-period discriminator");
    if (!m) return 1;
    if (mode < 0 || mode > 2) return fail(h, "st_test_mpd_conv: mode must be 0 (forward), 1 (dgrad) or 2 (wgrad)");
    if (layer < 1 || layer > 4) return fail(h, "st_test_mpd_conv: layer must be in [1, 4]");
    if (B < 1 || Hx < 1 || (long long)B * m->period > 65535 || (long long)Hx * m->period > (1LL << 30))
        return fail(h, "st_test_mpd_conv: bad B or Hx");
    if (!out || (mode != 1 && !x) || (mode != 0 && !dz) || (mode != 2 && !w) || (mode == 0 && !b) || (mode == 2 && !out_b))
        return fail(h, "st_test_mpd_conv: null pointer");
    const int Ci = kCin[layer], Co = kCout[layer];
    const bool s3 = kStride[layer] == 3, tc = h->engine == ST_ENGINE_TCGEN05;
    const int H = s3 ? (Hx + 2) / 3 : Hx;
    MpdPlan P;
    P.g.B = B; P.g.p = m->period; P.g.L = (long long)Hx * m->period; P.g.Hin = Hx;
    P.BB = B * m->period;
    const long long BB = P.BB, Kr = (BB * H + 255) / 256 * 256;
    const size_t wn = (size_t)(s3 ? 6 : 5) * Ci * Co;
    const size_t act = (size_t)BB * (s3 ? 3 * H : H) * Ci, dzn = (size_t)BB * (H + 1) * Co, dzTn = (size_t)Co * Kr;
    const size_t wtn = (size_t)(5 * Ci + 8) * Kr, yn = std::max((size_t)BB * H * Co, (size_t)BB * (H + 1) * (s3 ? 3 : 1) * Ci);
    TestBufs bufs;
    auto planes = [&](MpdPlanes& q, size_t n) {
        if (tc) { q.hi = bufs.take<bf16>(n); q.lo = bufs.take<bf16>(n); } else q.f = bufs.take<float>(n);
    };
    P.wf = bufs.take<float>(wn);
    if (tc) { P.whi = bufs.take<bf16>(wn); P.wlo = bufs.take<bf16>(wn); }
    planes(P.act, act); planes(P.dz, dzn); planes(P.dzT, dzTn); planes(P.wt, wtn);
    P.Y = bufs.take<float>(yn); P.dWp = bufs.take<float>((size_t)Co * (5 * Ci + 8));
    if (!bufs.ok) return fail(h, "st_test_mpd_conv: out of memory");
    cudaStream_t s = (cudaStream_t)stream;
    if (mode == 0) {                          // out (B, C_out, H, p) = conv(x) + b, no activation
        ST_CUDA(launch_mpd_nchw_to_rows(x, P.g, Hx, Ci, s3 ? 3 * H : H, P.act, s));
        if (mpd_fwd_gemm(h, P, layer, w, b, H, s)) return 1;
        ST_CUDA(launch_mpd_act_fwd(P.Y, P.g, H, Co, H, out, MpdPlanes(), s, 1.f));
    } else if (mode == 1) {                   // out (B, C_in, Hx, p) = the input gradient of dz (B, C_out, H, p)
        ST_CUDA(launch_mpd_nchw_to_rows(dz, P.g, H, Co, H + 1, P.dz, s));
        int Rg = 0, off = 0;
        if (mpd_dgrad(h, P, layer, w, H, &Rg, &off, s)) return 1;
        ST_CUDA(launch_mpd_act_bwd(P.Y, Rg, off, nullptr, nullptr, P.g, Hx, Ci, MpdPlanes(), MpdPlanes(), 0, out, s));
    } else {                                  // out (C_out, C_in, 5), out_b (C_out): the weight and bias gradients
        MpdPlanes yrows; yrows.f = P.Y;
        ST_CUDA(launch_mpd_nchw_to_rows(dz, P.g, H, Co, H, yrows, s));
        if (zero_planes(h, P.dzT, dzTn, s)) return 1;
        ST_CUDA(launch_mpd_act_bwd(P.Y, H, 0, nullptr, nullptr, P.g, H, Co, MpdPlanes(), P.dzT, Kr, nullptr, s));
        if (mpd_wgrad(h, P, layer, x, Hx, H, Kr, out, out_b, s)) return 1;
    }
    return hook_done(h, s, "st_test_mpd_conv");
}

int st_test_mpd_row_ex(st_handle* h, const st_test_mpd_row_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_mpd_row_ex: null descriptor");
    const st_test_mpd_row_desc& d = *dp;
    MpdGeo g;
    int H0 = 0;
    if (const char* why = test_mpd_row_error(d, &g, &H0)) return fail(h, std::string("st_test_mpd_row_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    MpdPlanes rows, tr;
    rows.f = d.rows_f; rows.hi = (bf16*)d.rows_hi; rows.lo = (bf16*)d.rows_lo;
    tr.f = d.tr_f; tr.hi = (bf16*)d.tr_hi; tr.lo = (bf16*)d.tr_lo;
    cudaError_t e = cudaSuccess;
    switch (d.kind) {
    case ST_TEST_MPD_ROW_CONV0_FWD: e = launch_mpd_conv0_fwd(d.x, g, H0, d.R, d.w, d.b, d.out, rows, s); break;
    case ST_TEST_MPD_ROW_ACT_FWD: e = launch_mpd_act_fwd(d.Y, g, d.H, d.C, d.R, d.out, rows, s, d.slope); break;
    case ST_TEST_MPD_ROW_NCHW_TO_ROWS: e = launch_mpd_nchw_to_rows(d.fmap, g, d.H, d.C, d.R, rows, s); break;
    case ST_TEST_MPD_ROW_POST_FWD: e = launch_mpd_post_fwd(d.fmap, g, d.H, d.w, d.b, d.out, s); break;
    case ST_TEST_MPD_ROW_PACK: e = launch_mpd_pack(d.w, d.Cout, d.Cin, d.mode, d.out, s); break;
    case ST_TEST_MPD_ROW_POST_DGRAD: e = launch_mpd_post_dgrad(d.gpost, g, d.H, d.w, d.out, s); break;
    case ST_TEST_MPD_ROW_POST_WGRAD: e = launch_mpd_post_wgrad(d.gpost, d.fmap, g, d.H, d.out, d.out_b, s); break;
    case ST_TEST_MPD_ROW_ACT_BWD:
        e = launch_mpd_act_bwd(d.G, d.Rg, d.off, d.gfmap, d.fmap, g, d.H, d.C, rows, tr, d.Kr, d.out, s);
        break;
    case ST_TEST_MPD_ROW_IM2COL_T: e = launch_mpd_im2col_t(d.fmap, g, d.Hx, d.Cin, d.H, d.stride, d.Kr, tr, s); break;
    case ST_TEST_MPD_ROW_UNPACK_WGRAD: e = launch_mpd_unpack_wgrad(d.dWp, d.Cout, d.Cin, d.out, d.out_b, s); break;
    case ST_TEST_MPD_ROW_CONV0_WGRAD: e = launch_mpd_conv0_wgrad(d.dz0, d.x, g, H0, d.out, d.out_b, s); break;
    case ST_TEST_MPD_ROW_CONV0_DGRAD: e = launch_mpd_conv0_dgrad(d.dz0, d.w, g, H0, d.out, s); break;
    }
    if (e != cudaSuccess) return fail(h, std::string("st_test_mpd_row_ex: launch failed: ") + cudaGetErrorString(e));
    return hook_done(h, s, "st_test_mpd_row_ex");
}

}  // extern "C"
