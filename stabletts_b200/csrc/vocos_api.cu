// C-ABI + orchestration of the vocoder hand-off (SURVEY.md §8 row f4): the reference's Vocos
// (vocoders/vocos/models/model.py:11-20) on the mel this library's CFM path emits (api.py:76).
//
//   mel (B, n_mel, T) -> token-major split planes
//   embed Conv1d k=7 (backbone.py:30,50)                       conv-GEMM, 7 taps, K = n_mel, N = dim
//   LayerNorm(dim, eps 1e-6) (:31,51)                          row kernel
//   12 x ConvNeXtBlock (module.py:34-46):
//       depthwise k=7 conv + LayerNorm                         row kernel (one pass, split-bf16 out)
//       pwconv1 + exact GELU                                   GEMM K = dim, N = intermediate, EPI_GELU
//       pwconv2, * gamma, + residual                           GEMM K = intermediate, N = dim, EPI_GATE | EPI_RESID
//   final LayerNorm (backbone.py:43,55)                        row kernel
//   head Linear dim -> n_fft + 2 (head.py:96-101)              GEMM, log-magnitudes and phases in two 128-aligned column
//                                                              groups ([0, K) and [Kp, Kp + K), K = n_fft/2 + 1)
//   exp / clip / cos / sin (head.py:103-113)                   elementwise, emits the split [re | im] operand
//   irfft * window (head.py:62-63)                             ONE GEMM against the windowed inverse-DFT basis
//                                                              (oracle/vocoder_ref.py idft_basis: exact in float64)
//   fold / envelope / trim (head.py:66-81)                     4-frame gather
// Training (DESIGN.md §8 row f12): st_vocos_forward_train runs the same forward into a caller-owned `saved` buffer, and
// st_vocos_backward walks it back (vocos_backward below; row kernels in vocos_grad.cu).
#include "handle.cuh"
#include "vocos.cuh"
#include <cmath>

using namespace st;

namespace st {

struct VocosState : Model {
    st_vocos_dims d;
    int K = 0, Kp = 0, Nh = 0, K2 = 0;         // bins, phase column offset, padded head width, padded spectrum width
    GemmW embed, head, basis;
    std::vector<GemmW> pw1, pw2;
    std::vector<float*> dw_w, dw_b, ln_w, ln_b, gamma;
    float *norm_w = nullptr, *norm_b = nullptr, *fln_w = nullptr, *fln_b = nullptr, *window = nullptr;
    void* ws = nullptr; size_t ws_bytes = 0;
    // backward: transposed weight packs (made by the first backward after each finalize) and the backward scratch
    bool grad_packed = false;
    GemmW headT, basisT;
    std::vector<GemmW> pw1T, pw2T;
    void* bws = nullptr; size_t bws_bytes = 0;
    explicit VocosState(const st_vocos_dims& dims)
        : d(dims), K(dims.n_fft / 2 + 1),
          Kp((K + 127) / 128 * 128),           // phases start at a 128-aligned column
          Nh(2 * Kp),
          K2(2 * ((K + 63) / 64 * 64)) {}      // [re | im], each half padded to the GEMM's 64-channel K block
    ~VocosState() override { if (ws) cudaFree(ws); if (bws) cudaFree(bws); }
    int finalize(st_handle* h, cudaStream_t s) override;
    int pack_grad(st_handle* h, cudaStream_t s);
};

const char* vocos_stft_error(int n_fft, int hop) {
    if (hop <= 0 || n_fft <= 0 || n_fft % 128 || n_fft % hop || n_fft / hop > 16 || (n_fft - hop) % 2)
        return "Vocos n_fft must be a multiple of 128 and of hop_length, with at most 16 overlapping frames";
    // "same" padding trims (n_fft - hop) / 2 samples off each end with [pad:-pad] (head.py:46,62): at pad = 0 that slice
    // is empty, so the reference returns a (B, 0) signal, where the overlap-add here would divide by a zero envelope
    if (hop >= n_fft)
        return "Vocos hop_length must be below n_fft: at hop_length == n_fft the reference's \"same\" ISTFT returns an empty "
               "(B, 0) signal (pad = 0 and y[pad:-pad] is empty)";
    return nullptr;
}

int VocosState::finalize(st_handle* h, cudaStream_t s) {
    const int L = d.n_layers, C = d.dim, I = d.intermediate;
    grad_packed = false;                       // st_finalize_weights freed the transposed packs with the rest
    pw1.assign(L, GemmW()); pw2.assign(L, GemmW());
    dw_w.assign(L, nullptr); dw_b.assign(L, nullptr); ln_w.assign(L, nullptr); ln_b.assign(L, nullptr);
    gamma.assign(L, nullptr);
    if (pack_gemm(h, &embed, {"backbone.embed"}, C, d.n_mel, 7, 0, d.n_mel, true, s)) return 1;
    if (get_raw(h, "backbone.norm.weight", C, &norm_w) || get_raw(h, "backbone.norm.bias", C, &norm_b)) return 1;
    for (int l = 0; l < L; ++l) {
        const std::string p = "backbone.convnext." + std::to_string(l) + ".";
        if (pack_dw7(h, p + "dwconv.weight", C, &dw_w[l], s)) return 1;
        if (get_raw(h, p + "dwconv.bias", C, &dw_b[l])) return 1;
        if (get_raw(h, p + "norm.weight", C, &ln_w[l]) || get_raw(h, p + "norm.bias", C, &ln_b[l])) return 1;
        if (get_raw(h, p + "gamma", C, &gamma[l])) return 1;
        if (pack_gemm(h, &pw1[l], {p + "pwconv1"}, I, C, 1, 0, C, true, s)) return 1;
        if (pack_gemm(h, &pw2[l], {p + "pwconv2"}, C, I, 1, 0, I, true, s)) return 1;
    }
    if (get_raw(h, "backbone.final_layer_norm.weight", C, &fln_w) || get_raw(h, "backbone.final_layer_norm.bias", C, &fln_b)) return 1;
    if (get_raw(h, "head.istft.window", d.n_fft, &window)) return 1;
    {   // head.out (n_fft + 2, dim): rows [0, K) = log-magnitudes, [K, 2K) = phases (chunk(2, dim=1), head.py:102) -> two
        // 128-aligned column groups of a zero-filled (Nh, dim) matrix
        float *w, *b;
        if (get_raw(h, "head.out.weight", (int64_t)2 * K * C, &w) || get_raw(h, "head.out.bias", 2 * K, &b)) return 1;
        GemmW& g = head;
        const size_t n = (size_t)Nh * C;
        if (alloc_gemm_w(h, &g, 1, Nh, C, true)) return 1;
        ST_CUDA(cudaMemsetAsync(g.f32, 0, n * 4, s));
        ST_CUDA(cudaMemsetAsync(g.bias, 0, (size_t)Nh * 4, s));
        ST_CUDA(launch_pack_conv(w, g.f32, K, C, 1, Nh, 0, 0, C, s));
        ST_CUDA(launch_pack_conv(w + (size_t)K * C, g.f32, K, C, 1, Nh, Kp, 0, C, s));
        ST_CUDA(cudaMemcpyAsync(g.bias, b, (size_t)K * 4, cudaMemcpyDeviceToDevice, s));
        ST_CUDA(cudaMemcpyAsync(g.bias + Kp, b + K, (size_t)K * 4, cudaMemcpyDeviceToDevice, s));
        ST_CUDA(launch_split(g.f32, g.hi, g.lo, (long)n, s));
    }
    {   // windowed inverse-DFT basis (n_fft outputs x K2)
        GemmW& g = basis;
        const size_t n = (size_t)d.n_fft * K2;
        if (alloc_gemm_w(h, &g, 1, d.n_fft, K2, false)) return 1;
        ST_CUDA(launch_idft_basis(window, d.n_fft, K, K2, g.f32, s));
        ST_CUDA(launch_split(g.f32, g.hi, g.lo, (long)n, s));
    }
    return 0;
}

// The dgrad GEMMs' weights: each forward weight [N][K] transposed to [K][N] (the head's zero rows at its padded columns
// become zero columns, the basis's zero imaginary DC / Nyquist columns zero rows).  Inference never pays for them.
int VocosState::pack_grad(st_handle* h, cudaStream_t s) {
    auto tr = [&](const GemmW& w, GemmW* t) -> int {
        if (alloc_gemm_w(h, t, 1, w.K, w.N, false)) return 1;
        ST_CUDA(launch_btc_to_bct(w.f32, t->f32, 1, w.K, w.N, s));
        ST_CUDA(launch_split(t->f32, t->hi, t->lo, (long)w.N * w.K, s));
        return 0;
    };
    pw1T.assign(d.n_layers, GemmW()); pw2T.assign(d.n_layers, GemmW());
    if (tr(head, &headT) || tr(basis, &basisT)) return 1;
    for (int l = 0; l < d.n_layers; ++l)
        if (tr(pw1[l], &pw1T[l]) || tr(pw2[l], &pw2T[l])) return 1;
    grad_packed = true;
    return 0;
}

}  // namespace st

namespace {

struct VocosWs { Act mel, E, X, U, Hid, Hd, S, F; size_t bytes = 0; };

void layout_vocos_ws(const st_handle* h, const VocosState* v, VocosWs& w, void* base, int B, int T) {
    const st_vocos_dims& d = v->d;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t rows = (size_t)B * T;
    Bump bp(base, 0);
    w.mel = take_act(bp, rows, d.n_mel, !tc, tc);
    w.E = take_act(bp, rows, d.dim, true, false);
    w.X = take_act(bp, rows, d.dim, true, false);
    w.U = take_act(bp, rows, d.dim, !tc, tc);
    w.Hid = take_act(bp, rows, d.intermediate, !tc, tc);
    w.Hd = take_act(bp, rows, v->Nh, true, false);
    w.S = take_act(bp, rows, v->K2, !tc, tc);
    w.F = take_act(bp, rows, d.n_fft, true, false);
    w.bytes = bp.off + 256;
}

// What st_vocos_forward_train keeps for st_vocos_backward, in the caller's buffer: every GEMM operand and LayerNorm input
// of the forward.  An operand is fp32 on the SIMT engine and split-bf16 planes on the wgmma engine: 4 bytes per element
// either way.
struct VocosSaved {
    Act mel;                          // (rows, n_mel) the embed conv's operand
    std::vector<float*> X;            // X[0] = LayerNorm(embed(mel)), X[l + 1] = block l's output: (rows, dim) fp32
    std::vector<Act> U, G;            // block l's LayerNorm output (rows, dim) and GELU(h) (rows, intermediate)
    Act Uf;                           // the final LayerNorm's output (rows, dim)
    Act Hd;                           // the head's output (rows, Nh) fp32
    size_t bytes = 0;
};

void layout_vocos_saved(const st_handle* h, const VocosState* v, VocosSaved& sv, void* base, int B, int T) {
    const st_vocos_dims& d = v->d;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t rows = (size_t)B * T;
    Bump bp(base, 0);
    sv.mel = take_act(bp, rows, d.n_mel, !tc, tc);
    sv.X.assign(d.n_layers + 1, nullptr);
    for (auto& x : sv.X) x = bp.take<float>(rows * d.dim);
    sv.U.assign(d.n_layers, Act()); sv.G.assign(d.n_layers, Act());
    for (int l = 0; l < d.n_layers; ++l) {
        sv.U[l] = take_act(bp, rows, d.dim, !tc, tc);
        sv.G[l] = take_act(bp, rows, d.intermediate, !tc, tc);
    }
    sv.Uf = take_act(bp, rows, d.dim, !tc, tc);
    sv.Hd = take_act(bp, rows, v->Nh, true, false);
    sv.bytes = (bp.off + 255) & ~size_t(255);
}

Act f32_act(float* p, int C) { Act a; a.f32 = p; a.C = C; return a; }

// The one forward.  sv == nullptr: every intermediate lives in the handle's workspace (inference); else the same launches
// write the operands st_vocos_backward needs into sv, and the audio is bitwise the same.
int vocos_forward(st_handle* h, VocosState* v, const float* mel, float* audio, int B, int T, const VocosSaved* sv,
                  cudaStream_t s) {
    const st_vocos_dims& d = v->d;
    VocosWs w;
    layout_vocos_ws(h, v, w, nullptr, B, T);
    if (grow_ws_synced(h, &v->ws, &v->ws_bytes, w.bytes, s)) return 1;
    layout_vocos_ws(h, v, w, v->ws, B, T);
    const long rows = (long)B * T;
    const Act& melA = sv ? sv->mel : w.mel;
    ST_LAUNCH(launch_bct_to_btc(mel, melA.f32, melA.hi, melA.lo, B, d.n_mel, T, nullptr, s));
    {   // embed: Conv1d(n_mel -> dim, k = 7, padding 3) (backbone.py:30,50)
        GemmArgs g = utt_gemm(B, T, EPI_BIAS);
        if (run_gemm(h, g, v->embed, &melA, nullptr, w.E, s)) return 1;
    }
    DwLnArgs ln;
    ln.B = B; ln.T = T; ln.C = d.dim; ln.eps = 1e-6f;
    ln.x = w.E.f32; ln.ln_w = v->norm_w; ln.ln_b = v->norm_b; ln.out_f32 = sv ? sv->X[0] : w.X.f32;
    ST_LAUNCH_P(ST_PROF_LN, 0, (double)rows * d.dim * 8, s, launch_dwconv_ln(ln, s));              // backbone.py:51
    for (int l = 0; l < d.n_layers; ++l) {                                                         // module.py:34-46
        const Act X = sv ? f32_act(sv->X[l], d.dim) : w.X, Xn = sv ? f32_act(sv->X[l + 1], d.dim) : w.X;
        const Act& U = sv ? sv->U[l] : w.U;
        const Act& Hid = sv ? sv->G[l] : w.Hid;
        DwLnArgs a;
        a.B = B; a.T = T; a.C = d.dim; a.eps = 1e-6f;
        a.x = X.f32; a.dw_w = v->dw_w[l]; a.dw_b = v->dw_b[l]; a.ln_w = v->ln_w[l]; a.ln_b = v->ln_b[l];
        a.out_f32 = U.f32; a.out_hi = U.hi; a.out_lo = U.lo;
        ST_LAUNCH_P(ST_PROF_LN, 0, (double)rows * d.dim * 8, s, launch_dwconv_ln(a, s));
        {
            GemmArgs g = utt_gemm(B, T, EPI_BIAS | EPI_GELU);
            if (run_gemm(h, g, v->pw1[l], &U, nullptr, Hid, s, ST_PROF_GEMM_C1)) return 1;
        }
        {   // x = residual + gamma * pwconv2(h)
            GemmArgs g = utt_gemm(B, T, EPI_BIAS | EPI_GATE | EPI_RESID);
            g.gate = v->gamma[l]; g.gate_bstride = 0; g.resid = X.f32;
            if (run_gemm(h, g, v->pw2[l], &Hid, nullptr, Xn, s, ST_PROF_GEMM_C2)) return 1;
        }
    }
    const Act& Uf = sv ? sv->Uf : w.U;
    ln.x = sv ? sv->X[d.n_layers] : w.X.f32; ln.ln_w = v->fln_w; ln.ln_b = v->fln_b;
    ln.out_f32 = Uf.f32; ln.out_hi = Uf.hi; ln.out_lo = Uf.lo;
    ST_LAUNCH_P(ST_PROF_LN, 0, (double)rows * d.dim * 8, s, launch_dwconv_ln(ln, s));              // backbone.py:55
    const Act& Hd = sv ? sv->Hd : w.Hd;
    {   // head.out (head.py:101)
        GemmArgs g = utt_gemm(B, T, EPI_BIAS);
        if (run_gemm(h, g, v->head, &Uf, nullptr, Hd, s)) return 1;
    }
    ST_LAUNCH(launch_spectrum(Hd.f32, v->Nh, v->Kp, v->K, v->K2, rows, w.S.f32, w.S.hi, w.S.lo, s));
    {   // frames = window * irfft(S) as one contraction
        GemmArgs g = utt_gemm(B, T, 0);
        if (run_gemm(h, g, v->basis, &w.S, nullptr, w.F, s)) return 1;
    }
    ST_LAUNCH(launch_overlap_add(w.F.f32, v->window, B, T, d.n_fft, d.hop, audio, s));
    return 0;
}

// Backward scratch.  Kr: the weight-gradient GEMMs' K, the rows rounded up to 256 (split-K needs whole 64-column blocks).
struct VocosGradWs {
    long long Kr = 0;
    float *f1 = nullptr, *f2 = nullptr, *f3 = nullptr;   // (rows, widest) fp32: row-kernel and GEMM results
    float *dX = nullptr, *zh = nullptr;                  // (rows, dim): the residual stream's gradient, a LayerNorm's zhat
    Act pA;                                              // (rows, widest) split planes of a dgrad GEMM's A (wgmma engine)
    Act tA, tW;                                          // [.][Kr] transposed operands of a wgrad GEMM: dY^T, [X^T; 1]
    float* dWp = nullptr;                                // a wgrad GEMM's output
    size_t bytes = 0;
};

void layout_vocos_grad_ws(const st_handle* h, const VocosState* v, VocosGradWs& w, void* base, int B, int T) {
    const st_vocos_dims& d = v->d;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t rows = (size_t)B * T;
    const int C = d.dim, I = d.intermediate;
    const int widest = std::max(std::max(d.n_fft, v->K2), std::max(v->Nh, std::max(C, I)));
    w.Kr = ((long long)rows + 255) / 256 * 256;
    const int nA = std::max(v->Nh, std::max(C, I)), nW = std::max(std::max(C, I) + 8, 7 * d.n_mel + 8);
    const size_t dwp = std::max(std::max((size_t)v->Nh * (C + 8), (size_t)C * (I + 8)),
                                std::max((size_t)I * (C + 8), (size_t)C * (7 * d.n_mel + 8)));
    Bump bp(base, 0);
    w.f1 = bp.take<float>(rows * widest);
    w.f2 = bp.take<float>(rows * widest);
    w.f3 = bp.take<float>(rows * std::max(C, I));
    w.dX = bp.take<float>(rows * C);
    w.zh = bp.take<float>(rows * C);
    w.pA = take_act(bp, tc ? rows : 0, widest, false, tc);
    w.tA = take_act(bp, (size_t)w.Kr, nA, !tc, tc);
    w.tW = take_act(bp, (size_t)w.Kr, nW, !tc, tc);
    w.dWp = bp.take<float>(dwp);
    w.bytes = bp.off + 256;
}

// A dgrad GEMM's A operand from fp32 rows f (rows, C): the rows themselves (SIMT) or their split planes (wgmma)
int grad_operand(st_handle* h, const VocosGradWs& w, float* f, long rows, int C, Act* a, cudaStream_t s) {
    a->f32 = f; a->C = C; a->hi = a->lo = nullptr;
    if (h->engine == ST_ENGINE_TCGEN05) {
        ST_LAUNCH(launch_split(f, w.pA.hi, w.pA.lo, rows * C, s));
        a->f32 = nullptr; a->hi = w.pA.hi; a->lo = w.pA.lo;
    }
    return 0;
}

// out = A · W^T for the token-major operand A (rows, W.K) into fp32 rows (rows, W.N)
int grad_gemm(st_handle* h, const GemmW& W, const Act& A, float* out, int B, int T, int flags, cudaStream_t s) {
    GemmArgs g = utt_gemm(B, T, flags);
    return run_gemm(h, g, W, &A, nullptr, f32_act(out, W.N), s);
}

// transposed GEMM planes [Nd][Kr] of the rows (rows, Cx) in fp32 `f` or in the saved operand `x`
int grad_transpose(st_handle* h, const VocosGradWs& w, const Act* x, const float* f, int B, int T, int Cx, int taps, bool ones,
                   const Act& dst, cudaStream_t s) {
    TransposeArgs a;
    a.src_f32 = f ? f : x->f32;
    if (!f && x->hi) { a.src_f32 = nullptr; a.src_hi = x->hi; a.src_lo = x->lo; }
    a.dst_f32 = dst.f32; a.dst_hi = dst.hi; a.dst_lo = dst.lo;
    a.B = B; a.T = T; a.Cx = Cx; a.taps = taps; a.ones = ones ? 1 : 0;
    a.Nd = taps * Cx + (ones ? 8 : 0); a.Kr = w.Kr;
    ST_LAUNCH(launch_transpose_rows(a, s));
    return 0;
}

// The weight and bias gradients of a layer from its output gradient (fp32 rows dY (rows, Ny)) and its input (the saved
// operand x or fp32 rows, (rows, Cx), taps 1 or 7): dWp [Ny][taps Cx + 8] = dY^T · [X^T; 1]^T as one GEMM over the rows
// (T = Ny output rows, K = Kr), then the reference layouts (wgrad_unpack_kernel).
int grad_wgrad(st_handle* h, const VocosGradWs& w, const float* dY, int Ny, const Act* x, int Cx, int taps, int B, int T,
               int Nref, int split, int Kp, float* gw, float* gb, cudaStream_t s) {
    const Act tA = [&] { Act a = w.tA; a.C = (int)w.Kr; return a; }();
    if (grad_transpose(h, w, nullptr, dY, B, T, Ny, 1, false, tA, s)) return 1;
    if (grad_transpose(h, w, x, nullptr, B, T, Cx, taps, true, w.tW, s)) return 1;
    GemmW W;
    W.f32 = w.tW.f32; W.hi = w.tW.hi; W.lo = w.tW.lo; W.taps = 1; W.N = taps * Cx + 8; W.K = (int)w.Kr;
    GemmArgs ga;
    ga.BB = 1; ga.T = Ny; ga.a_bmod = 1; ga.B = 1;
    if (run_gemm(h, ga, W, &tA, nullptr, f32_act(w.dWp, W.N), s)) return 1;
    ST_LAUNCH(launch_unpack_wgrad(w.dWp, Nref, Cx, taps, split, Kp, gw, gb, s));
    return 0;
}

// The backward of vocos_forward: grads in _param_shapes order (vocos.py), each overwritten.  gx = the running gradient of
// the residual stream.
int vocos_backward(st_handle* h, VocosState* v, const VocosSaved& sv, const VocosGradWs& w, const float* d_audio, int B, int T,
                   float* const* grads, cudaStream_t s) {
    const st_vocos_dims& d = v->d;
    const int L = d.n_layers, C = d.dim, I = d.intermediate;
    const long rows = (long)B * T;
    float* const* gl = grads + 4;                         // block l's nine gradients at gl[9 l ..]
    float* const* gt = grads + 4 + 9 * L;                 // final LayerNorm, head
    Act A;
    // ISTFT adjoint: frame gradient, then dS = dF · W (the basis's transpose as the GEMM weight)
    ST_LAUNCH(launch_frame_grad(d_audio, v->window, B, T, d.n_fft, d.hop, w.f1, s));
    if (grad_operand(h, w, w.f1, rows, d.n_fft, &A, s) || grad_gemm(h, v->basisT, A, w.f2, B, T, 0, s)) return 1;
    // spectrum -> dHd (rows, Nh) in f1
    ST_LAUNCH(launch_spectrum_grad(w.f2, sv.Hd.f32, v->Nh, v->Kp, v->K, v->K2, rows, w.f1, s));
    // head Linear: weight / bias gradients in the reference's (n_fft + 2, dim) layout, then dU = dHd · W_head
    if (grad_wgrad(h, w, w.f1, v->Nh, &sv.Uf, C, 1, B, T, 2 * v->K, v->K, v->Kp, gt[2], gt[3], s)) return 1;
    if (grad_operand(h, w, w.f1, rows, v->Nh, &A, s) || grad_gemm(h, v->headT, A, w.f2, B, T, 0, s)) return 1;
    // final LayerNorm: dX = its input's gradient
    LnBwdArgs ln;
    ln.B = B; ln.T = T; ln.C = C; ln.eps = 1e-6f;
    ln.x = sv.X[L]; ln.ln_w = v->fln_w; ln.g = w.f2; ln.dx = w.dX; ln.zhat = w.zh;
    ST_LAUNCH(launch_ln_bwd(ln, s));
    ST_LAUNCH(launch_col_sum(w.f2, w.zh, rows, C, gt[0], s));
    ST_LAUNCH(launch_col_sum(w.f2, nullptr, rows, C, gt[1], s));
    for (int l = L - 1; l >= 0; --l) {
        float* const* g = gl + 9 * l;                     // gamma, dwconv.{w, b}, norm.{w, b}, pwconv1.{w, b}, pwconv2.{w, b}
        // layer scale: P = pwconv2(GELU(h)) + b2 recomputed; dgamma = sum dX' P, dP = dX' gamma
        if (grad_gemm(h, v->pw2[l], sv.G[l], w.f3, B, T, EPI_BIAS, s)) return 1;
        ST_LAUNCH(launch_col_sum(w.dX, w.f3, rows, C, g[0], s));
        ST_LAUNCH(launch_scale_cols(w.dX, v->gamma[l], rows, C, w.f1, s));
        // pwconv2: weight / bias gradients, then dGELU = dP · W2
        if (grad_wgrad(h, w, w.f1, C, &sv.G[l], I, 1, B, T, C, 0, 0, g[7], g[8], s)) return 1;
        if (grad_operand(h, w, w.f1, rows, C, &A, s) || grad_gemm(h, v->pw2T[l], A, w.f2, B, T, 0, s)) return 1;
        // GELU: h = pwconv1(U) + b1 recomputed; dh = dGELU gelu'(h)
        if (grad_gemm(h, v->pw1[l], sv.U[l], w.f3, B, T, EPI_BIAS, s)) return 1;
        ST_LAUNCH(launch_gelu_bwd(w.f2, w.f3, rows * I, w.f1, s));
        // pwconv1: weight / bias gradients, then dU = dh · W1
        if (grad_wgrad(h, w, w.f1, I, &sv.U[l], C, 1, B, T, I, 0, 0, g[5], g[6], s)) return 1;
        if (grad_operand(h, w, w.f1, rows, I, &A, s) || grad_gemm(h, v->pw1T[l], A, w.f2, B, T, 0, s)) return 1;
        // LayerNorm over the recomputed depthwise-conv output: dz in f1, affine gradients
        ln.x = sv.X[l]; ln.dw_w = v->dw_w[l]; ln.dw_b = v->dw_b[l]; ln.ln_w = v->ln_w[l]; ln.g = w.f2; ln.dx = w.f1;
        ST_LAUNCH(launch_ln_bwd(ln, s));
        ST_LAUNCH(launch_col_sum(w.f2, w.zh, rows, C, g[3], s));
        ST_LAUNCH(launch_col_sum(w.f2, nullptr, rows, C, g[4], s));
        // depthwise conv: weight / bias gradients, then dX = dX' (residual) + the conv's adjoint of dz
        ST_LAUNCH(launch_dwconv_wgrad(w.f1, sv.X[l], B, T, C, g[1], g[2], s));
        ST_LAUNCH(launch_dwconv_adj(w.f1, v->dw_w[l], B, T, C, w.dX, s));
    }
    // post-embed LayerNorm over the recomputed embed output E = embed(mel) + b
    if (grad_gemm(h, v->embed, sv.mel, w.f3, B, T, EPI_BIAS, s)) return 1;
    ln.x = w.f3; ln.dw_w = nullptr; ln.dw_b = nullptr; ln.ln_w = v->norm_w; ln.g = w.dX; ln.dx = w.f1;
    ST_LAUNCH(launch_ln_bwd(ln, s));
    ST_LAUNCH(launch_col_sum(w.dX, w.zh, rows, C, grads[2], s));
    ST_LAUNCH(launch_col_sum(w.dX, nullptr, rows, C, grads[3], s));
    // embed conv: weight / bias gradients against the 7-tap shifted transpose of the mel
    return grad_wgrad(h, w, w.f1, C, &sv.mel, d.n_mel, 7, B, T, C, 0, 0, grads[0], grads[1], s);
}

}  // namespace

extern "C" {

int st_create_vocos(const st_vocos_dims* dims, int device, st_handle** out) {
    if (!dims || !out) return fail(nullptr, "st_create_vocos: null argument");
    const st_vocos_dims& d = *dims;
    if (d.dim != 512 && d.dim != 768 && d.dim != 1024) return fail(nullptr, "Vocos dim must be 512, 768 or 1024 (reference VocosConfig: 768)");
    if (d.n_mel <= 0 || d.n_mel % 16) return fail(nullptr, "Vocos input_channels must be a positive multiple of 16");
    if (d.intermediate <= 0 || d.intermediate % 64) return fail(nullptr, "Vocos intermediate_dim must be a multiple of 64");
    if (d.n_layers <= 0 || d.n_layers > 64) return fail(nullptr, "Vocos num_layers out of range");
    if (const char* why = vocos_stft_error(d.n_fft, d.hop)) return fail(nullptr, why);
    return create_handle(device, std::make_unique<VocosState>(d), out);
}

int st_vocos_forward(st_handle* h, const float* mel, float* audio, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    VocosState* v = ready_model<VocosState>(h, "Vocos vocoder");
    if (!v) return 1;
    if (!mel || !audio) return fail(h, "st_vocos_forward: null pointer");
    if (B <= 0 || T <= 0 || B > 32767) return fail(h, "B and T must be positive");
    return vocos_forward(h, v, mel, audio, B, T, nullptr, (cudaStream_t)stream);
}

size_t st_vocos_saved_bytes(st_handle* h, int B, int T) {
    VocosState* v = h ? dynamic_cast<VocosState*>(h->model.get()) : nullptr;
    if (!v || B <= 0 || T <= 0 || B > 32767) return 0;
    VocosSaved sv;
    layout_vocos_saved(h, v, sv, nullptr, B, T);
    return sv.bytes;
}

int st_vocos_forward_train(st_handle* h, const float* mel, float* audio, int B, int T, void* saved, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    VocosState* v = ready_model<VocosState>(h, "Vocos vocoder");
    if (!v) return 1;
    if (!mel || !audio || !saved) return fail(h, "st_vocos_forward_train: null pointer");
    if (B <= 0 || T <= 0 || B > 32767) return fail(h, "B and T must be positive");
    VocosSaved sv;
    layout_vocos_saved(h, v, sv, saved, B, T);
    return vocos_forward(h, v, mel, audio, B, T, &sv, (cudaStream_t)stream);
}

int st_vocos_backward(st_handle* h, const void* saved, const float* d_audio, int B, int T, float* const* grads, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    VocosState* v = ready_model<VocosState>(h, "Vocos vocoder");
    if (!v) return 1;
    if (!saved || !d_audio || !grads) return fail(h, "st_vocos_backward: null pointer");
    if (B <= 0 || T <= 0 || B > 32767) return fail(h, "B and T must be positive");
    const int L = v->d.n_layers, np = 4 + 9 * L + 4;
    for (int i = 0; i < np; ++i)
        if (!grads[i]) return fail(h, "st_vocos_backward: null gradient pointer");
    cudaStream_t s = (cudaStream_t)stream;
    if (!v->grad_packed && v->pack_grad(h, s)) return 1;
    VocosSaved sv;
    layout_vocos_saved(h, v, sv, const_cast<void*>(saved), B, T);
    VocosGradWs w;
    layout_vocos_grad_ws(h, v, w, nullptr, B, T);
    if (grow_ws_synced(h, &v->bws, &v->bws_bytes, w.bytes, s)) return 1;
    layout_vocos_grad_ws(h, v, w, v->bws, B, T);
    return vocos_backward(h, v, sv, w, d_audio, B, T, grads, s);
}

int st_test_vocos_grad_ex(st_handle* h, const st_test_vocos_grad_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_vocos_grad_ex: null descriptor");
    const st_test_vocos_grad_desc& d = *dp;
    auto need = [&](bool ok) { return ok ? 0 : fail(h, "st_test_vocos_grad_ex: a required input or output is NULL"); };
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaSuccess;
    switch (d.kind) {
    case ST_TEST_VOCOS_GRAD_FRAME_GRAD:
        if (need(d.x && d.w && d.out_f32)) return 1;
        if (d.n_fft <= 0 || d.hop <= 0 || d.n_fft % d.hop || d.hop >= d.n_fft) return fail(h, "st_test_vocos_grad_ex: bad n_fft / hop");
        e = launch_frame_grad(d.x, d.w, d.B, d.T, d.n_fft, d.hop, d.out_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_SPECTRUM_GRAD:
        if (need(d.x && d.x1 && d.out_f32)) return 1;
        if (d.K > d.Kp || 2 * d.Kp > d.Nh || 2 * d.K > d.K2) return fail(h, "st_test_vocos_grad_ex: need K <= Kp, 2 Kp <= Nh, 2 K <= K2");
        e = launch_spectrum_grad(d.x, d.x1, d.Nh, d.Kp, d.K, d.K2, d.rows, d.out_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_LN_BWD: {
        if (need(d.x && d.x1 && d.x2 && d.out_f32 && (!d.w == !d.bias))) return 1;
        LnBwdArgs a;
        a.x = d.x; a.dw_w = d.w; a.dw_b = d.bias; a.ln_w = d.x1; a.g = d.x2; a.dx = d.out_f32; a.zhat = d.out2_f32;
        a.B = d.B; a.T = d.T; a.C = d.C; a.eps = d.eps;
        e = launch_ln_bwd(a, s);
        break;
    }
    case ST_TEST_VOCOS_GRAD_DWCONV_ADJ:
        if (need(d.x && d.w && d.out_f32)) return 1;
        e = launch_dwconv_adj(d.x, d.w, d.B, d.T, d.C, d.out_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_COL_SUM:
        if (need(d.x && d.out_f32)) return 1;
        e = launch_col_sum(d.x, d.x1, d.rows, d.C, d.out_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_DWCONV_WGRAD:
        if (need(d.x && d.x1 && d.out_f32 && d.out2_f32)) return 1;
        e = launch_dwconv_wgrad(d.x, d.x1, d.B, d.T, d.C, d.out_f32, d.out2_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_SCALE_COLS:
        if (need(d.x && d.w && d.out_f32)) return 1;
        e = launch_scale_cols(d.x, d.w, d.rows, d.C, d.out_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_GELU_BWD:
        if (need(d.x && d.x1 && d.out_f32)) return 1;
        e = launch_gelu_bwd(d.x, d.x1, d.rows, d.out_f32, s);
        break;
    case ST_TEST_VOCOS_GRAD_TRANSPOSE_ROWS: {
        if (need((d.x || d.x_hi) && (d.out_f32 || d.out_hi)) || need(!d.x_hi == !d.x_lo && !d.out_hi == !d.out_lo)) return 1;
        TransposeArgs a;
        a.src_f32 = d.x; a.src_hi = (const bf16*)d.x_hi; a.src_lo = (const bf16*)d.x_lo;
        a.dst_f32 = d.out_f32; a.dst_hi = (bf16*)d.out_hi; a.dst_lo = (bf16*)d.out_lo;
        a.B = d.B; a.T = d.T; a.Cx = d.C; a.taps = d.taps; a.ones = d.ones; a.Nd = d.Nd; a.Kr = d.Kr;
        if (d.B < 1 || d.T < 1 || d.C < 1) return fail(h, "st_test_vocos_grad_ex: B, T, C >= 1");
        e = launch_transpose_rows(a, s);
        break;
    }
    case ST_TEST_VOCOS_GRAD_WGRAD_UNPACK:
        if (need(d.x && d.out_f32 && d.out2_f32)) return 1;
        if (d.taps != 1 && d.taps != 7) return fail(h, "st_test_vocos_grad_ex: taps must be 1 or 7");
        e = launch_unpack_wgrad(d.x, d.Nref, d.C, d.taps, d.split, d.Kp, d.out_f32, d.out2_f32, s);
        break;
    default:
        return fail(h, "st_test_vocos_grad_ex: unknown kind");
    }
    if (e != cudaSuccess) return fail(h, std::string("st_test_vocos_grad_ex: launch failed: ") + cudaGetErrorString(e));
    return hook_done(h, s, "st_test_vocos_grad_ex");
}

}  // extern "C"
