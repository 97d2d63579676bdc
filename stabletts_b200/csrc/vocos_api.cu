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
    explicit VocosState(const st_vocos_dims& dims)
        : d(dims), K(dims.n_fft / 2 + 1),
          Kp((K + 127) / 128 * 128),           // phases start at a 128-aligned column
          Nh(2 * Kp),
          K2(2 * ((K + 63) / 64 * 64)) {}      // [re | im], each half padded to the GEMM's 64-channel K block
    ~VocosState() override { if (ws) cudaFree(ws); }
    int finalize(st_handle* h, cudaStream_t s) override;
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
    const st_vocos_dims& d = v->d;
    cudaStream_t s = (cudaStream_t)stream;
    VocosWs w;
    layout_vocos_ws(h, v, w, nullptr, B, T);
    if (grow_ws_synced(h, &v->ws, &v->ws_bytes, w.bytes, s)) return 1;
    layout_vocos_ws(h, v, w, v->ws, B, T);
    const long rows = (long)B * T;
    ST_LAUNCH(launch_bct_to_btc(mel, w.mel.f32, w.mel.hi, w.mel.lo, B, d.n_mel, T, nullptr, s));
    {   // embed: Conv1d(n_mel -> dim, k = 7, padding 3) (backbone.py:30,50)
        GemmArgs g = utt_gemm(B, T, EPI_BIAS);
        if (run_gemm(h, g, v->embed, &w.mel, nullptr, w.E, s)) return 1;
    }
    DwLnArgs ln;
    ln.B = B; ln.T = T; ln.C = d.dim; ln.eps = 1e-6f;
    ln.x = w.E.f32; ln.ln_w = v->norm_w; ln.ln_b = v->norm_b; ln.out_f32 = w.X.f32;
    ST_LAUNCH_P(ST_PROF_LN, 0, (double)rows * d.dim * 8, s, launch_dwconv_ln(ln, s));              // backbone.py:51
    for (int l = 0; l < d.n_layers; ++l) {                                                         // module.py:34-46
        DwLnArgs a;
        a.B = B; a.T = T; a.C = d.dim; a.eps = 1e-6f;
        a.x = w.X.f32; a.dw_w = v->dw_w[l]; a.dw_b = v->dw_b[l]; a.ln_w = v->ln_w[l]; a.ln_b = v->ln_b[l];
        a.out_f32 = w.U.f32; a.out_hi = w.U.hi; a.out_lo = w.U.lo;
        ST_LAUNCH_P(ST_PROF_LN, 0, (double)rows * d.dim * 8, s, launch_dwconv_ln(a, s));
        {
            GemmArgs g = utt_gemm(B, T, EPI_BIAS | EPI_GELU);
            if (run_gemm(h, g, v->pw1[l], &w.U, nullptr, w.Hid, s, ST_PROF_GEMM_C1)) return 1;
        }
        {   // x = residual + gamma * pwconv2(h)
            GemmArgs g = utt_gemm(B, T, EPI_BIAS | EPI_GATE | EPI_RESID);
            g.gate = v->gamma[l]; g.gate_bstride = 0; g.resid = w.X.f32;
            if (run_gemm(h, g, v->pw2[l], &w.Hid, nullptr, w.X, s, ST_PROF_GEMM_C2)) return 1;
        }
    }
    ln.x = w.X.f32; ln.ln_w = v->fln_w; ln.ln_b = v->fln_b; ln.out_f32 = w.U.f32; ln.out_hi = w.U.hi; ln.out_lo = w.U.lo;
    ST_LAUNCH_P(ST_PROF_LN, 0, (double)rows * d.dim * 8, s, launch_dwconv_ln(ln, s));              // backbone.py:55
    {   // head.out (head.py:101)
        GemmArgs g = utt_gemm(B, T, EPI_BIAS);
        if (run_gemm(h, g, v->head, &w.U, nullptr, w.Hd, s)) return 1;
    }
    ST_LAUNCH(launch_spectrum(w.Hd.f32, v->Nh, v->Kp, v->K, v->K2, rows, w.S.f32, w.S.hi, w.S.lo, s));
    {   // frames = window * irfft(S) as one contraction
        GemmArgs g = utt_gemm(B, T, 0);
        if (run_gemm(h, g, v->basis, &w.S, nullptr, w.F, s)) return 1;
    }
    ST_LAUNCH(launch_overlap_add(w.F.f32, v->window, B, T, d.n_fft, d.hop, audio, s));
    return 0;
}

}  // extern "C"
