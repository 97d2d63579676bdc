// C-ABI + orchestration of the FireflyGAN vocoder, the reference's default vocoder (vocoders/ffgan/model.py:45-56), at
// its one configuration (config_dict, model.py:7-29).  Token-major throughout; one GEMM row is one frame (backbone) or one
// sample at the stage's rate (head).
//
//   mel (B, 128, T) -> token-major operand planes
//   ConvNeXtEncoder (backbone.py:206-214), dims 128 / 256 / 384 / 512, depths 3 / 3 / 9 / 3:
//     stem Conv1d(128 -> 128, k = 7)                              conv-GEMM, 7 taps
//     channels-first LayerNorm (eps 1e-6, :69-74)                 row kernel (dwconv_ln_kernel without the conv)
//     downsample i: LayerNorm + Conv1d(1x1)                       row kernel + GEMM
//     ConvNeXt block (:124-143): dwconv k = 7 + LayerNorm         row kernel
//                                pwconv1 + exact GELU             GEMM, EPI_GELU
//                                pwconv2 * gamma + residual       GEMM, EPI_GATE | EPI_RESID
//     final LayerNorm                                             row kernel
//   HiFiGANGenerator (head.py:225-249, use_template = False):
//     conv_pre (512 -> 512, k = 13) + the SiLU of ups[0]          GEMM, 13 taps, EPI_SILU
//     ups[i]: ConvTranspose1d(C -> C/2, k = 2u, stride u)         GEMM, 3 taps at the input rate, N = u * C/2 (polyphase
//                                                                 packing): its (T, u C/2) output IS the (u T, C/2) input of
//                                                                 the stage; emits x (fp32) and silu(x) (operand)
//     ParralelBlock i: 3 x ResBlock1 (k = 3, 7, 11), each 3 x
//       convs1[j] (dilation 1 / 3 / 5) -> silu                    GEMM, dilated taps, EPI_SILU
//       convs2[j] + residual                                      GEMM, EPI_RESID | EPI_SILU_OUT: x + y (fp32 residual
//                                                                 stream) and silu(x + y) (operand of convs1[j + 1])
//     mean of the three, then SiLU                                row kernel, fixed summation order
//     conv_post (16 -> 1, k = 13) + tanh                          row kernel, writes (B, 512 T)
#include "handle.cuh"
#include "ffgan.cuh"
#include "vocos.cuh"

using namespace st;

namespace st {

namespace {

constexpr int kDims[4] = {128, 256, 384, 512}, kDepths[4] = {3, 3, 9, 3};
constexpr int kUps[5] = {8, 8, 2, 2, 2}, kResK[3] = {3, 7, 11}, kResD[3] = {1, 3, 5};
constexpr int kMel = 128, kC0 = 512, kPreK = 13, kPostK = 13, kHop = 512;
constexpr int kStageWidth = 8192;           // C_i * (samples per mel frame) of every head stage but the first (2048)

}  // namespace

struct FfganState : Model {
    GemmW stem, down[4], pre, ups[5], c1[5][3][3], c2[5][3][3];
    std::vector<GemmW> pw1, pw2;
    std::vector<float*> dw_w, dw_b, ln_w, ln_b, gamma;
    float *lnc_w[4] = {}, *lnc_b[4] = {};   // channels-first LayerNorms: stem (index 0), downsample 1..3
    float *norm_w = nullptr, *norm_b = nullptr, *post_w = nullptr, *post_b = nullptr;
    void* ws = nullptr; size_t ws_bytes = 0;
    ~FfganState() override { if (ws) cudaFree(ws); }
    int finalize(st_handle* h, cudaStream_t s) override;
};

namespace {

const std::string kG = ".parametrizations.weight.original0", kV = ".parametrizations.weight.original1";

// weight-normed Conv1d (Cout, Cin, k): fold W = g v / ||v|| (g per output channel), then pack [k][Cout][Cin] + split planes
int pack_wn_conv(st_handle* h, GemmW* w, const std::string& name, int Cout, int Cin, int k, cudaStream_t s) {
    float *g, *v, *b, *tmp;
    const size_t n = (size_t)Cout * Cin * k;
    if (get_raw(h, name + kG, Cout, &g) || get_raw(h, name + kV, (int64_t)n, &v) || get_raw(h, name + ".bias", Cout, &b)) return 1;
    if (dev_alloc(h, &tmp, n) || alloc_gemm_w(h, w, k, Cout, Cin, true)) return 1;
    ST_CUDA(launch_weight_norm_fold(g, v, tmp, Cout, Cin * k, s));
    ST_CUDA(launch_pack_conv(tmp, w->f32, Cout, Cin, k, Cout, 0, 0, Cin, s));
    ST_CUDA(cudaMemcpyAsync(w->bias, b, (size_t)Cout * 4, cudaMemcpyDeviceToDevice, s));
    ST_CUDA(launch_split(w->f32, w->hi, w->lo, (long)n, s));
    return 0;
}

// weight-normed ConvTranspose1d (Cin, Cout, 2u), g per INPUT channel -> 3-tap polyphase conv, N = u Cout, bias tiled u times
int pack_wn_ups(st_handle* h, GemmW* w, const std::string& name, int Cin, int Cout, int u, cudaStream_t s) {
    float *g, *v, *b, *tmp;
    const size_t nv = (size_t)Cin * Cout * 2 * u, n = (size_t)3 * u * Cout * Cin;
    if (get_raw(h, name + kG, Cin, &g) || get_raw(h, name + kV, (int64_t)nv, &v) || get_raw(h, name + ".bias", Cout, &b)) return 1;
    if (dev_alloc(h, &tmp, nv) || alloc_gemm_w(h, w, 3, u * Cout, Cin, true)) return 1;
    ST_CUDA(launch_weight_norm_fold(g, v, tmp, Cin, Cout * 2 * u, s));
    ST_CUDA(launch_pack_polyphase(tmp, w->f32, Cin, Cout, u, s));
    for (int r = 0; r < u; ++r) ST_CUDA(cudaMemcpyAsync(w->bias + (size_t)r * Cout, b, (size_t)Cout * 4, cudaMemcpyDeviceToDevice, s));
    ST_CUDA(launch_split(w->f32, w->hi, w->lo, (long)n, s));
    return 0;
}

}  // namespace

int FfganState::finalize(st_handle* h, cudaStream_t s) {
    const int nb = kDepths[0] + kDepths[1] + kDepths[2] + kDepths[3];
    pw1.assign(nb, GemmW()); pw2.assign(nb, GemmW());
    dw_w.assign(nb, nullptr); dw_b.assign(nb, nullptr); ln_w.assign(nb, nullptr); ln_b.assign(nb, nullptr);
    gamma.assign(nb, nullptr);
    const std::string dl = "backbone.downsample_layers.";
    if (pack_gemm(h, &stem, {dl + "0.0"}, kDims[0], kMel, 7, 0, kMel, true, s)) return 1;             // backbone.py:160-169
    if (get_raw(h, dl + "0.1.weight", kDims[0], &lnc_w[0]) || get_raw(h, dl + "0.1.bias", kDims[0], &lnc_b[0])) return 1;
    for (int i = 1; i < 4; ++i) {                                                                          // :172-177
        const std::string p = dl + std::to_string(i) + ".";
        if (get_raw(h, p + "0.weight", kDims[i - 1], &lnc_w[i]) || get_raw(h, p + "0.bias", kDims[i - 1], &lnc_b[i])) return 1;
        if (pack_gemm(h, &down[i], {p + "1"}, kDims[i], kDims[i - 1], 1, 0, kDims[i - 1], true, s)) return 1;
    }
    for (int i = 0, l = 0; i < 4; ++i) {
        const int C = kDims[i];
        for (int j = 0; j < kDepths[i]; ++j, ++l) {                                                        // :183-196
            const std::string p = "backbone.stages." + std::to_string(i) + "." + std::to_string(j) + ".";
            if (pack_dw7(h, p + "dwconv.weight", C, &dw_w[l], s)) return 1;
            if (get_raw(h, p + "dwconv.bias", C, &dw_b[l])) return 1;
            if (get_raw(h, p + "norm.weight", C, &ln_w[l]) || get_raw(h, p + "norm.bias", C, &ln_b[l])) return 1;
            if (get_raw(h, p + "gamma", C, &gamma[l])) return 1;
            if (pack_gemm(h, &pw1[l], {p + "pwconv1"}, 4 * C, C, 1, 0, C, true, s)) return 1;
            if (pack_gemm(h, &pw2[l], {p + "pwconv2"}, C, 4 * C, 1, 0, 4 * C, true, s)) return 1;
        }
    }
    if (get_raw(h, "backbone.norm.weight", kC0, &norm_w) || get_raw(h, "backbone.norm.bias", kC0, &norm_b)) return 1;
    if (pack_wn_conv(h, &pre, "head.conv_pre", kC0, kC0, kPreK, s)) return 1;                           // head.py:162-170
    for (int i = 0; i < 5; ++i) {
        const int cin = kC0 >> i, c = kC0 >> (i + 1);
        if (pack_wn_ups(h, &ups[i], "head.ups." + std::to_string(i), cin, c, kUps[i], s)) return 1;     // :176-186
        for (int b = 0; b < 3; ++b)
            for (int j = 0; j < 3; ++j) {                                                                  // :26-80
                const std::string p = "head.resblocks." + std::to_string(i) + ".blocks." + std::to_string(b) + ".";
                if (pack_wn_conv(h, &c1[i][b][j], p + "convs1." + std::to_string(j), c, c, kResK[b], s)) return 1;
                if (pack_wn_conv(h, &c2[i][b][j], p + "convs2." + std::to_string(j), c, c, kResK[b], s)) return 1;
            }
    }
    {   // conv_post (1, 16, 13): folded in place of a packed weight; the row kernel reads the reference layout
        float *g, *v;
        const int C = kC0 >> 5;
        if (get_raw(h, "head.conv_post" + kG, 1, &g) || get_raw(h, "head.conv_post" + kV, (int64_t)C * kPostK, &v)) return 1;
        if (get_raw(h, "head.conv_post.bias", 1, &post_b)) return 1;
        if (dev_alloc(h, &post_w, (size_t)C * kPostK)) return 1;
        ST_CUDA(launch_weight_norm_fold(g, v, post_w, 1, C * kPostK, s));
    }
    return 0;
}

}  // namespace st

namespace {

// Eight equal slots of 8192 values per mel frame (the widest head stage; every slot holds an fp32 tensor or a pair of
// split-bf16 planes), reused by the backbone.  Head: Xu (ups output, fp32), Xs (its SiLU, operand), R[3] (the three
// ResBlock1 residual streams), Rs (silu(R), operand), Hd (silu(convs1), operand), S (silu(mean), operand of the next ups).
struct FfganWs { float* slot[8] = {}; size_t slot_vals = 0, bytes = 0; };

void layout_ffgan_ws(FfganWs& w, void* base, int B, int T) {
    Bump bp(base, 0);
    w.slot_vals = (size_t)B * T * kStageWidth;
    for (int i = 0; i < 8; ++i) w.slot[i] = bp.take<float>(w.slot_vals);
    w.bytes = bp.off + 256;
}

// an activation of `rows` x C in a slot: fp32 for the SIMT engine, split planes (hi, then lo) for the wgmma engine
Act act(float* slot, size_t rows, int C, bool tc) {
    Act a; a.C = C;
    if (tc) { a.hi = (bf16*)slot; a.lo = a.hi + rows * C; } else a.f32 = slot;
    return a;
}
Act act_f32(float* slot, int C) { Act a; a.C = C; a.f32 = slot; return a; }

}  // namespace

extern "C" {

int st_create_ffgan(int device, st_handle** out) {
    if (!out) return fail(nullptr, "st_create_ffgan: null argument");
    return create_handle(device, std::make_unique<FfganState>(), out);
}

size_t st_ffgan_workspace_bytes(const st_handle* h, int B, int T) {
    (void)h;
    FfganWs w;
    layout_ffgan_ws(w, nullptr, B, T);
    return w.bytes;
}

int st_ffgan_forward(st_handle* h, const float* mel, float* audio, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    FfganState* f = ready_model<FfganState>(h, "FireflyGAN vocoder");
    if (!f) return 1;
    if (!mel || !audio) return fail(h, "st_ffgan_forward: null pointer");
    if (B <= 0 || T <= 0 || B > 32767 || (long)T * kHop > (1L << 30)) return fail(h, "B and T must be positive (and T * 512 < 2^30)");
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    FfganWs w;
    layout_ffgan_ws(w, nullptr, B, T);
    if (grow_ws_synced(h, &f->ws, &f->ws_bytes, w.bytes, s)) return 1;
    layout_ffgan_ws(w, f->ws, B, T);
    auto base = [&](int flags, int Tg) {
        GemmArgs g = utt_gemm(B, Tg, flags);
        g.batch_invariant = 1;         // an utterance's audio must not depend on its batch (the deep head amplifies reordering)
        return g;
    };
    const size_t rows = (size_t)B * T;

    // ---------------- ConvNeXtEncoder (backbone.py:206-214) ----------------
    int cat = ST_PROF_FFGAN_BACKBONE;
    Act M = act(w.slot[6], rows, kMel, tc), E = act_f32(w.slot[0], kDims[0]), X = act_f32(w.slot[2], kDims[0]);
    ST_LAUNCH_P(cat, 0, (double)rows * kMel * 8, s,
                launch_bct_to_btc(mel, M.f32, M.hi, M.lo, B, kMel, T, nullptr, s));
    {
        GemmArgs g = base(EPI_BIAS, T);
        if (run_gemm(h, g, f->stem, &M, nullptr, E, s, cat)) return 1;
    }
    auto ln = [&](const float* x, int C, const float* lw, const float* lb, const float* dw_w, const float* dw_b, const Act& o) {
        DwLnArgs a;
        a.B = B; a.T = T; a.C = C; a.eps = 1e-6f;
        a.x = x; a.dw_w = dw_w; a.dw_b = dw_b; a.ln_w = lw; a.ln_b = lb;
        a.out_f32 = o.f32; a.out_hi = o.hi; a.out_lo = o.lo;
        return launch_dwconv_ln(a, s);
    };
    ST_LAUNCH_P(cat, 0, (double)rows * kDims[0] * 8, s, ln(E.f32, kDims[0], f->lnc_w[0], f->lnc_b[0], nullptr, nullptr, X));
    for (int i = 0, l = 0; i < 4; ++i) {
        const int C = kDims[i];
        if (i > 0) {                   // downsample: channels-first LayerNorm, then Conv1d 1x1 (backbone.py:173-176)
            Act U = act(w.slot[1], rows, kDims[i - 1], tc);
            ST_LAUNCH_P(cat, 0, (double)rows * kDims[i - 1] * 8, s, ln(X.f32, kDims[i - 1], f->lnc_w[i], f->lnc_b[i], nullptr, nullptr, U));
            X = act_f32(w.slot[i % 2 ? 3 : 2], C);
            GemmArgs g = base(EPI_BIAS, T);
            if (run_gemm(h, g, f->down[i], &U, nullptr, X, s, cat)) return 1;
        }
        for (int j = 0; j < kDepths[i]; ++j, ++l) {                                    // backbone.py:124-143
            Act U = act(w.slot[1], rows, C, tc), Hid = act(w.slot[4], rows, 4 * C, tc);
            ST_LAUNCH_P(cat, 0, (double)rows * C * 8, s, ln(X.f32, C, f->ln_w[l], f->ln_b[l], f->dw_w[l], f->dw_b[l], U));
            {
                GemmArgs g = base(EPI_BIAS | EPI_GELU, T);
                if (run_gemm(h, g, f->pw1[l], &U, nullptr, Hid, s, cat)) return 1;
            }
            {
                GemmArgs g = base(EPI_BIAS | EPI_GATE | EPI_RESID, T);
                g.gate = f->gamma[l]; g.gate_bstride = 0; g.resid = X.f32;
                if (run_gemm(h, g, f->pw2[l], &Hid, nullptr, X, s, cat)) return 1;
            }
        }
    }
    Act U = act(w.slot[1], rows, kC0, tc);
    ST_LAUNCH_P(cat, 0, (double)rows * kC0 * 8, s, ln(X.f32, kC0, f->norm_w, f->norm_b, nullptr, nullptr, U));   // backbone.py:198,214

    // ---------------- HiFiGANGenerator (head.py:225-249) ----------------
    Act S = act(w.slot[7], rows, kC0, tc);
    {   // conv_pre, then the SiLU that opens the first upsampling step (head.py:226, 230)
        GemmArgs g = base(EPI_BIAS | EPI_SILU, T);
        if (run_gemm(h, g, f->pre, &U, nullptr, S, s, ST_PROF_FFGAN_PRE)) return 1;
    }
    int Tin = T;
    for (int i = 0; i < 5; ++i) {
        cat = ST_PROF_FFGAN_STAGE0 + i;
        const int u = kUps[i], C = kC0 >> (i + 1), Ti = Tin * u;
        const size_t ri = (size_t)B * Ti;
        Act Xu = act_f32(w.slot[0], C), Xs = act(w.slot[1], ri, C, tc);
        {   // ups[i] as the 3-tap polyphase conv at the input rate: (B, Tin, u C) == (B, Ti, C)
            Act Xu_in = act_f32(Xu.f32, u * C), Xs_in = Xs;
            Xs_in.C = u * C;
            GemmArgs g = base(EPI_BIAS | EPI_SILU_OUT, Tin);
            Act o = Xu_in; o.hi = Xs_in.hi; o.lo = Xs_in.lo;
            if (!tc) g.out2_f32 = Xs.f32;
            if (run_gemm(h, g, f->ups[i], &S, nullptr, o, s, cat)) return 1;
        }
        Act R[3];
        for (int b = 0; b < 3; ++b) {                  // ResBlock1 (head.py:92-99)
            R[b] = act_f32(w.slot[2 + b], C);
            for (int j = 0; j < 3; ++j) {
                Act Hd = act(w.slot[6], ri, C, tc), Rs = act(w.slot[5], ri, C, tc);
                {
                    GemmArgs g = base(EPI_BIAS | EPI_SILU, Ti);
                    g.dil = kResD[j];
                    if (run_gemm(h, g, f->c1[i][b][j], j == 0 ? &Xs : &Rs, nullptr, Hd, s, cat)) return 1;
                }
                {   // x = x + convs2(.); the last one of the block needs no operand of its SiLU
                    const bool last = j == 2;
                    GemmArgs g = base(EPI_BIAS | EPI_RESID | (last ? 0 : EPI_SILU_OUT), Ti);
                    g.resid = j == 0 ? Xu.f32 : R[b].f32;
                    Act o = R[b];
                    if (!last) { o.hi = Rs.hi; o.lo = Rs.lo; if (!tc) g.out2_f32 = Rs.f32; }
                    if (run_gemm(h, g, f->c2[i][b][j], &Hd, nullptr, o, s, cat)) return 1;
                }
            }
        }
        const bool post = i == 4;                       // the last stage feeds conv_post's row kernel (fp32)
        S = post ? act_f32(w.slot[7], C) : act(w.slot[7], ri, C, tc);
        ST_LAUNCH_P(cat, 0, (double)ri * C * 16, s, launch_mean3_silu(R[0].f32, R[1].f32, R[2].f32, (long)ri * C, S.f32, S.hi, S.lo, s));
        Tin = Ti;
    }
    ST_LAUNCH_P(ST_PROF_FFGAN_POST, 2.0 * rows * kHop * 16 * kPostK, (double)rows * kHop * (16 + 1) * 4, s,
                launch_post_conv_tanh(S.f32, f->post_w, f->post_b, B, (long)T * kHop, 16, kPostK, audio, s));
    return 0;
}

}  // extern "C"
