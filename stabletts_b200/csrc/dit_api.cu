// C-ABI + host-side orchestration of the DiT models: the CFM estimator and the text encoder (see include/stabletts_b200.h).
//
// What runs where (reference: models/flow_matching.py:24-67, models/estimator.py:103-137):
//   per solve   : layout change (B,C,T)->(B,T,C); cond_proj(mu) and cond_proj(fake_content) ONCE
//                 (t-independent; exact hoist); in_proj's mu-half P = W_mu·mu' + b ONCE; adaLN(c)
//                 ONCE; time-MLP + FiLM (gamma,beta) for every stage time of the grid up front.
//   per eval    : in_proj x-half + P -> 6 x [ (lsc conv) FiLM·mask, LN, modulate, QKV, RoPE+masked
//                 attention, O+gate+residual, LN, modulate, conv_1+SiLU, conv_2+gate+residual ]
//                 -> final_proj.  With CFG the cond and uncond branches are ONE doubled batch.
// The ODE drivers that call these per solve and per evaluation are in solve.cu.
#include "dit.cuh"
#include <cmath>

using namespace st;

namespace {

// ----- workspace ----------------------------------------------------------------------------------
void layout_ws(const st_handle* h, const DitModel& m, Workspace& w, void* base, size_t cap, int B, int T, int cfg) {
    const st_dims& d = m.d;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    w.B = B; w.T = T; w.cfg = cfg; w.BB = cfg ? 2 * B : B; w.Bc = B + (cfg ? 1 : 0);
    w.NT = std::max(MAX_EVAL_TABLE, B);
    Bump bp(base, cap);
    const size_t bt = (size_t)B * T, bbt = (size_t)w.BB * T, bct = (size_t)w.Bc * T;
    w.xt = take_act(bp, bt, d.n_mel, true, false);
    w.ytmp = take_act(bp, bt, d.n_mel, true, false);
    w.xs = take_act(bp, bt, d.n_mel, false, tc);
    w.V = take_act(bp, bbt, d.n_mel, true, false);
    for (int i = 0; i < 10; ++i) w.Kst[i] = bp.take<float>(bt * d.n_mel);
    w.dscal = bp.take<double>(2);
    w.mut = take_act(bp, bct, d.n_mel, !tc, tc);
    w.C1 = take_act(bp, bct, d.filter, !tc, tc);
    w.C2 = take_act(bp, bct, d.filter, !tc, tc);
    w.C3 = take_act(bp, bct, d.hidden, !tc, tc);
    w.P = take_act(bp, bct, d.hidden, true, false);
    for (int i = 0; i < 5; ++i) w.X[i] = take_act(bp, bbt, d.hidden, true, tc);
    w.U = take_act(bp, bbt, d.hidden, !tc, tc);
    w.QKV = take_act(bp, bbt, 3 * d.hidden, !tc, tc);   // tensor-core engine: RoPE'd split planes straight from the GEMM epilogue
    w.AO = take_act(bp, bbt, d.hidden, !tc, tc);
    w.Hid = take_act(bp, bbt, d.filter, !tc, tc);
    w.kvlen = bp.take<int>(B);
    w.prefix = bp.take<int>(B);
    w.rope_cs = bp.take<float>((size_t)T * 32);
    w.temb = bp.take<float>((size_t)w.NT * d.hidden);
    w.tmid = bp.take<float>((size_t)w.NT * d.filter);
    w.tvec = bp.take<float>((size_t)w.NT * d.hidden);
    w.film = bp.take<float>((size_t)w.NT * d.n_layers * 2 * d.hidden);
    w.ada = bp.take<float>((size_t)w.Bc * d.n_layers * 6 * d.hidden);
    w.cin = bp.take<float>((size_t)w.Bc * d.gin);
    w.h_z = bp.take<float>(bt * d.n_mel);
    w.h_mu = bp.take<float>(bt * d.n_mel);
    w.h_mask = bp.take<float>(bt);
    w.h_c = bp.take<float>((size_t)B * d.gin);
    w.h_fc = bp.take<float>(d.n_mel);
    w.h_fs = bp.take<float>(d.gin);
    w.bytes = bp.off + 256;
}

}  // namespace

int st::ensure_ws(st_handle* h, DitModel& m, Workspace& w, int B, int T, int cfg) {
    Workspace probe;
    layout_ws(h, m, probe, nullptr, 0, B, T, cfg);
    if (h->ws_ptr == nullptr || h->ws_bytes < probe.bytes) {
        if (h->ws_ptr && !h->ws_owned)
            return fail(h, "attached workspace too small: need " + std::to_string(probe.bytes) + " bytes");
        m.drop_cached();
        if (h->ws_ptr) { cudaFree(h->ws_ptr); h->ws_ptr = nullptr; }
        ST_CUDA(cudaMalloc(&h->ws_ptr, probe.bytes));
        h->ws_bytes = probe.bytes; h->ws_owned = true;
    }
    layout_ws(h, m, w, h->ws_ptr, h->ws_bytes, B, T, cfg);
    return 0;
}

// fp16 hi / lo planes of a packed weight (the FFN convs; used by ST_PRECISION_FFN_FP16X2)
int DitModel::pack_f16_planes(st_handle* h, GemmW* w, cudaStream_t s) {
    const size_t n = (size_t)w->taps * w->N * w->K;
    if (dev_alloc(h, &w->h_hi, n) || dev_alloc(h, &w->h_lo, n)) return 1;
    ST_CUDA(launch_split_f16(w->f32, w->h_hi, w->h_lo, (long)n, s, f16_range));
    return 0;
}

int DitModel::begin_f16_range(st_handle* h, cudaStream_t s) {
    if (dev_alloc(h, &f16_range, 1)) return 1;
    ST_CUDA(cudaMemsetAsync(f16_range, 0, sizeof(int), s));
    return 0;
}

int DitModel::end_f16_range(st_handle* h, cudaStream_t s) {
    int out = 0;
    ST_CUDA(cudaMemcpyAsync(&out, f16_range, sizeof(int), cudaMemcpyDeviceToHost, s));
    ST_CUDA(cudaStreamSynchronize(s));
    f16_ok = out == 0;
    return 0;
}

int DitModel::pack_block(st_handle* h, int l, const std::string& p, cudaStream_t s) {
    const int H = d.hidden, F = d.filter, k = d.kernel;
    if (pack_gemm(h, &qkv[l], {p + "attn.conv_q", p + "attn.conv_k", p + "attn.conv_v"}, H, H, 1, 0, H, true, s)) return 1;
    if (pack_gemm(h, &wo[l], {p + "attn.conv_o"}, H, H, 1, 0, H, true, s)) return 1;
    if (pack_gemm(h, &c1[l], {p + "mlp.conv_1"}, F, H, k, 0, H, true, s)) return 1;
    if (pack_gemm(h, &c2[l], {p + "mlp.conv_2"}, H, F, k, 0, F, true, s)) return 1;
    if (pack_f16_planes(h, &c1[l], s) || pack_f16_planes(h, &c2[l], s)) return 1;
    if (get_raw(h, p + "adaLN_modulation.2.weight", (int64_t)6 * H * H, &ada_w[l])) return 1;
    return get_raw(h, p + "adaLN_modulation.2.bias", 6 * H, &ada_b[l]);
}

int CfmModel::finalize(st_handle* h, cudaStream_t s) {
    const int H = d.hidden, F = d.filter, M = d.n_mel, k = d.kernel, L = d.n_layers;
    qkv.assign(L, GemmW()); wo.assign(L, GemmW()); c1.assign(L, GemmW()); c2.assign(L, GemmW()); lsc.assign(L / 2, GemmW());
    film_w.assign(L, nullptr); film_b.assign(L, nullptr); ada_w.assign(L, nullptr); ada_b.assign(L, nullptr);
    if (begin_f16_range(h, s)) return 1;
    if (pack_gemm(h, &cond0, {"cond_proj.0"}, F, M, k, 0, M, true, s)) return 1;
    if (pack_gemm(h, &cond2, {"cond_proj.2"}, F, F, k, 0, F, true, s)) return 1;
    if (pack_gemm(h, &cond4, {"cond_proj.4"}, H, F, k, 0, F, true, s)) return 1;
    // in_proj acts on cat(x, mu') (models/estimator.py:120): columns [0,M) multiply x, [M, M+H) multiply mu'
    if (pack_gemm(h, &inx, {"in_proj"}, H, M + H, 1, 0, M, false, s)) return 1;
    if (pack_gemm(h, &inmu, {"in_proj"}, H, M + H, 1, M, H, true, s)) return 1;
    if (pack_gemm(h, &fin, {"final_proj"}, M, H, 1, 0, H, true, s)) return 1;
    for (int l = 0; l < L; ++l) {
        std::string p = "blocks." + std::to_string(l) + ".";
        if (pack_block(h, l, p + "block.", s)) return 1;
        if (get_raw(h, p + "time_fusion.film.weight", (int64_t)2 * H * H, &film_w[l])) return 1;
        if (get_raw(h, p + "time_fusion.film.bias", 2 * H, &film_b[l])) return 1;
    }
    for (int i = 0; i < L / 2; ++i) {
        if (pack_gemm(h, &lsc[i], {"lsc_layers." + std::to_string(i)}, H, 2 * H, k, 0, 2 * H, true, s)) return 1;
        if (pack_f16_planes(h, &lsc[i], s)) return 1;
    }
    if (get_raw(h, "time_mlp.layer.0.weight", (int64_t)F * H, &tm0_w)) return 1;
    if (get_raw(h, "time_mlp.layer.0.bias", F, &tm0_b)) return 1;
    if (get_raw(h, "time_mlp.layer.2.weight", (int64_t)H * F, &tm2_w)) return 1;
    if (get_raw(h, "time_mlp.layer.2.bias", H, &tm2_b)) return 1;
    return end_f16_range(h, s);
}

// models/text_encoder.py:22-26: emb, n_layers DiTConVBlocks, proj
int TextEncoderModel::finalize(st_handle* h, cudaStream_t s) {
    const int H = d.hidden, L = d.n_layers;
    qkv.assign(L, GemmW()); wo.assign(L, GemmW()); c1.assign(L, GemmW()); c2.assign(L, GemmW());
    ada_w.assign(L, nullptr); ada_b.assign(L, nullptr);
    if (begin_f16_range(h, s)) return 1;
    for (int l = 0; l < L; ++l)
        if (pack_block(h, l, "encoder." + std::to_string(l) + ".", s)) return 1;
    if (pack_gemm(h, &fin, {"proj"}, d.n_mel, H, 1, 0, H, true, s)) return 1;
    if (get_raw(h, "emb.weight", (int64_t)n_vocab * H, &emb)) return 1;
    return end_f16_range(h, s);
}

CfmModel::~CfmModel() {
    drop_cached();
    if (cap_stream) cudaStreamDestroy(cap_stream);
    if (pinned) cudaFreeHost(pinned);
    if (pin_buf) cudaFreeHost(pin_buf);
}

void CfmModel::drop_cached() { for (auto& g : graphs) cudaGraphExecDestroy(g.exec); graphs.clear(); }

GemmArgs st::dit_gemm(const Workspace& w, const float* mask, int flags) {
    GemmArgs g;
    g.BB = w.BB; g.T = w.T; g.a_bmod = w.BB; g.B = w.B; g.mask = mask; g.flags = flags;
    g.c_clamp = w.B; g.resid_clamp = w.BB - 1; g.film_H = w.U.C; g.rope_cs = w.rope_cs;
    return g;
}

// ----- per-solve precompute -------------------------------------------------------------------------
// cond features (models/estimator.py:118) for B real rows + (cfg) the broadcast fake_content row;
// P = W_in[:, M:]·mu' + b_in (models/estimator.py:120-121, mu-half); adaLN(c) (diffusion_transformer.py:110)
int st::precompute_cond(st_handle* h, const CfmModel& m, Workspace& w, const float* mu, const float* mask, const float* c,
                        const float* fake_content, const float* fake_speaker, cudaStream_t s) {
    const st_dims& d = m.d;
    ST_LAUNCH(launch_bct_to_btc(mu, w.mut.f32, w.mut.hi, w.mut.lo, w.B, d.n_mel, w.T, w.cfg ? fake_content : nullptr, s));
    ST_LAUNCH(launch_mask_lengths(mask, w.kvlen, w.prefix, w.B, w.T, s));
    ST_LAUNCH(launch_rope_table(w.rope_cs, w.T, 32, s));
    GemmArgs g;
    g.BB = w.Bc; g.T = w.T; g.a_bmod = w.Bc; g.B = w.B; g.resid_clamp = w.Bc - 1;
    g.flags = EPI_BIAS | EPI_SILU;
    if (run_gemm(h, g, m.cond0, &w.mut, nullptr, w.C1, s, ST_PROF_GEMM_COND)) return 1;
    if (run_gemm(h, g, m.cond2, &w.C1, nullptr, w.C2, s, ST_PROF_GEMM_COND)) return 1;
    g.flags = EPI_BIAS;
    if (run_gemm(h, g, m.cond4, &w.C2, nullptr, w.C3, s, ST_PROF_GEMM_COND)) return 1;
    if (run_gemm(h, g, m.inmu, &w.C3, nullptr, w.P, s, ST_PROF_GEMM_COND)) return 1;
    // adaLN: rows = c (B) [+ fake_speaker]
    ST_CUDA(cudaMemcpyAsync(w.cin, c, sizeof(float) * (size_t)w.B * d.gin, cudaMemcpyDeviceToDevice, s));
    if (w.cfg)
        ST_CUDA(cudaMemcpyAsync(w.cin + (size_t)w.B * d.gin, fake_speaker, sizeof(float) * d.gin, cudaMemcpyDeviceToDevice, s));
    for (int l = 0; l < d.n_layers; ++l)   // ada layout (Bc, L, 6H)
        ST_LAUNCH(launch_gemv(w.cin, m.ada_w[l], m.ada_b[l], w.ada + (size_t)l * 6 * d.hidden, (long)d.n_layers * 6 * d.hidden,
                              w.Bc, d.gin, 6 * d.hidden, 1, 0, s));
    return 0;
}

// time-MLP + FiLM vectors for n_t times already embedded in w.temb (models/estimator.py:55-62,30-31)
int st::precompute_film(st_handle* h, const CfmModel& m, Workspace& w, int n_t, cudaStream_t s) {
    const st_dims& d = m.d;
    ST_LAUNCH(launch_gemv(w.temb, m.tm0_w, m.tm0_b, w.tmid, d.filter, n_t, d.hidden, d.filter, 0, 1, s));
    ST_LAUNCH(launch_gemv(w.tmid, m.tm2_w, m.tm2_b, w.tvec, d.hidden, n_t, d.filter, d.hidden, 0, 0, s));
    for (int l = 0; l < d.n_layers; ++l)   // film layout (n_t, L, 2H)
        ST_LAUNCH(launch_gemv(w.tvec, m.film_w[l], m.film_b[l], w.film + (size_t)l * 2 * d.hidden, (long)d.n_layers * 2 * d.hidden,
                              n_t, d.hidden, 2 * d.hidden, 0, 0, s));
    return 0;
}

namespace {

// the adaLN-Zero conditioning and the fused LayerNorm's output planes of a GEMM whose epilogue runs a block's LN1 / LN2
void set_u(GemmArgs& g, const Workspace& w, long ada_bs) { g.ada_bstride = ada_bs; g.u_hi = w.U.hi; g.u_lo = w.U.lo; }

// The LayerNorm + adaLN modulate that FOLLOWS a GEMM whose tile owns whole 256-channel rows rides in that GEMM's epilogue
// (gemm_epilogue.cuh, EM_LN): O -> LN2, conv_2 / in_proj -> the next block's [FiLM·mask +] LN1, long-skip conv -> LN1.
// Small problems (fewer 128 x 256 tiles than SMs: they run on 128 x 128 tiles) and the SIMT engine keep the separate kernel.
bool ln_fusion_on(const st_handle* h, const st_dims& d, const Workspace& w) {
    if (h->engine != ST_ENGINE_TCGEN05) return false;
    GemmArgs g;
    g.BB = w.BB; g.T = w.T; g.N = d.hidden; g.Ktot = d.hidden; g.Cs[0] = d.hidden; g.n_src = 1;
    g.A_hi[0] = w.U.hi; g.W_hi = w.U.hi;           // non-null placeholders: only shapes matter here
    return gemm_tc_ln_fusable(g, h->num_sms);
}

// The two-pass FFN precision applies when both FFN convs of this problem run on 256-channel tiles, and every weight with
// fp16 planes lies in their range (DitModel::f16_ok).
bool ffn16_on(const st_handle* h, const DitModel& m, const Workspace& w) {
    if (h->precision != ST_PRECISION_FFN_FP16X2 || h->engine != ST_ENGINE_TCGEN05 || !m.f16_ok) return false;
    const st_dims& d = m.d;
    const int H = d.hidden, F = d.filter;
    GemmArgs g1, g2;
    g1.BB = g2.BB = w.BB; g1.T = g2.T = w.T; g1.n_src = g2.n_src = 1;
    g1.N = F; g1.Ktot = H; g1.Cs[0] = H; g2.N = H; g2.Ktot = F; g2.Cs[0] = F;
    g1.A_hi[0] = g2.A_hi[0] = w.U.hi; g1.W_hi = g2.W_hi = w.U.hi;       // non-null placeholders: only shapes matter
    return gemm_tc_wide_tile(g1, h->num_sms) && gemm_tc_wide_tile(g2, h->num_sms);
}

struct NextLn {                 // the LayerNorm that directly follows this block's conv_2 (nullptr: none / not fused)
    const float* film2; long film2_bs; float* x2_out;   // the next block's FiLM (estimator blocks < L/2), else nullptr
    const float* shift; const float* scale;
};

// One adaLN-Zero DiT block on the residual stream X[xb] (models/diffusion_transformer.py:98-117): LN1+modulate -> QKV (+RoPE)
// -> masked attention -> O·gate + residual -> LN2+modulate·mask -> conv_1+SiLU·mask -> conv_2·mask·gate + residual.
// `ln` describes LN1 for the separate kernel (plain, or FiLM·mask fused); with `ln1_done` the previous GEMM's epilogue has
// already written U.  `fuse`: LN2 rides in O's epilogue, and `next` (if any) in conv_2's.
int dit_block_core(st_handle* h, const DitModel& m, Workspace& w, int l, LnArgs ln, const float* ada_l, long ada_bs, int xb,
                   const float* mask, cudaStream_t s, bool fuse = false, bool ln1_done = false, const NextLn* next = nullptr,
                   bool x16 = false) {
    const st_dims& d = m.d;
    const int H = d.hidden;
    const bool f16 = ffn16_on(h, m, w);   // LN2's U and the hidden activation travel as ONE fp16 plane (in the hi buffers)
    auto base = [&](int flags) {
        GemmArgs g = dit_gemm(w, mask, flags);
        set_u(g, w, ada_bs);
        return g;
    };
    ln.shift = ada_l; ln.scale = ada_l + H;
    ln.u_f32 = w.U.f32; ln.u_hi = w.U.hi; ln.u_lo = w.U.lo;
    if (!ln1_done)
        ST_LAUNCH_P(ST_PROF_LN, 0, (double)w.BB * w.T * H * (4 + (ln.has_film ? 4 : 0) + 4), s, launch_film_ln_mod(ln, s));
    {   // q,k,v projections as one N=3H GEMM (models/diffusion_transformer.py:59-61)
        // tensor-core engine: partial RoPE + softmax scale fused in the epilogue, split-bf16 output
        GemmArgs g = base(h->engine == ST_ENGINE_TCGEN05 ? (EPI_BIAS | EPI_ROPE) : EPI_BIAS);
        g.rope_H = H;
        if (run_gemm(h, g, m.qkv[l], &w.U, nullptr, w.QKV, s, ST_PROF_GEMM_QKV)) return 1;
    }
    {
        AttnArgs a;
        a.qkv = w.QKV.f32; a.qkv_hi = w.QKV.hi; a.qkv_lo = w.QKV.lo;
        a.rope_cs = w.rope_cs; a.mask = mask; a.kvlen = w.kvlen; a.prefix = w.prefix;
        a.out_f32 = w.AO.f32; a.out_hi = w.AO.hi; a.out_lo = w.AO.lo;
        a.BB = w.BB; a.B = w.B; a.T = w.T; a.H = H; a.n_heads = d.n_heads;
        if (h->engine == ST_ENGINE_TCGEN05) {
            ST_LAUNCH_P(ST_PROF_ATTN, 4.0 * w.BB * (double)w.T * w.T * H, (double)w.BB * w.T * H * 16, s, launch_attention_tc(a, s));
        } else {
            ST_LAUNCH_P(ST_PROF_ATTN, 4.0 * w.BB * (double)w.T * w.T * H, (double)w.BB * w.T * H * 16, s, launch_attention_simt(a, s));
        }
    }
    {   // x += gate_msa * conv_o(attn) * mask   (:65, :111)  [+ LN2 + modulate, FFN input mask (:112, :26) in the epilogue]
        GemmArgs g = base(EPI_BIAS | EPI_MASK | EPI_GATE | EPI_RESID);
        g.gate = ada_l + 2 * H; g.gate_bstride = ada_bs; g.resid = w.X[xb].f32;
        if (fuse) { g.ln = 1; g.ln_mask_out = 1; g.ln_shift = ada_l + 3 * H; g.ln_scale = ada_l + 4 * H; g.u16 = f16; }
        Act out = w.X[xb]; out.hi = nullptr; out.lo = nullptr;
        if (run_gemm(h, g, m.wo[l], &w.AO, nullptr, out, s, ST_PROF_GEMM_O)) return 1;
    }
    if (!fuse) {   // LN2 + modulate, FFN input mask (:112, :26)
        LnArgs l2 = ln;
        l2.xin = w.X[xb].f32; l2.xout = nullptr; l2.has_film = 0; l2.mask_out = 1; l2.u16 = f16;
        l2.shift = ada_l + 3 * H; l2.scale = ada_l + 4 * H;
        ST_LAUNCH_P(ST_PROF_LN, 0, (double)w.BB * w.T * H * 8, s, launch_film_ln_mod(l2, s));
    }
    {   // conv_1 + SiLU, (h * mask) feeds conv_2 (:26-29)
        GemmArgs g = base(EPI_BIAS | EPI_SILU | EPI_MASK);
        if (f16) { g.prec = 1; g.out16 = 1; }
        if (run_gemm(h, g, m.c1[l], &w.U, nullptr, w.Hid, s, ST_PROF_GEMM_C1)) return 1;
    }
    {   // x += gate_mlp * (conv_2(h) * mask)   (:29-30, :112)  [+ the next block's (FiLM·mask,) LN1 + modulate in the epilogue]
        GemmArgs g = base(EPI_BIAS | EPI_MASK | EPI_GATE | EPI_RESID);
        g.gate = ada_l + 5 * H; g.gate_bstride = ada_bs; g.resid = w.X[xb].f32;
        if (f16) g.prec = 1;
        if (f16 && x16) g.out16 = 1;   // the residual stream's operand plane feeds a two-pass long-skip conv: ONE fp16 plane
        if (fuse && next) {
            g.ln = 1; g.ln_mask_out = 0; g.ln_shift = next->shift; g.ln_scale = next->scale;
            g.film2 = next->film2; g.film2_bstride = next->film2_bs; g.out2_f32 = next->x2_out;
        }
        if (run_gemm(h, g, m.c2[l], &w.Hid, nullptr, w.X[xb], s, ST_PROF_GEMM_C2)) return 1;
    }
    return 0;
}

// nullptr when the DiT blocks are built for these dims (n_layers is each creator's own check)
const char* dit_dims_error(const st_dims& d) {
    if (d.hidden != 256 || d.n_heads * 64 != d.hidden)
        return "only hidden=256, head_dim=64 is built (reference ModelConfig, config.py:22-30)";
    if (d.gin != d.hidden) return "gin_channels must equal hidden_channels";
    if (d.kernel != 3 && d.kernel != 1) return "kernel_size must be 1 or 3";
    if (d.n_mel % 16 || d.n_mel <= 0 || d.n_mel > 256) return "n_mel must be a multiple of 16, <= 256";
    if (d.filter % 64 || d.filter <= 0) return "filter_channels must be a multiple of 64";
    return nullptr;
}

}  // namespace

// ----- one estimator evaluation (models/estimator.py:120-137) ------------------------------------------
int st::estimator_eval(st_handle* h, const CfmModel& m, Workspace& w, const Act& xin, const float* mask, const float* film,
                       long film_bstride, cudaStream_t s) {
    const st_dims& d = m.d;
    const int H = d.hidden, L = d.n_layers, n_lsc = L / 2;
    const long ada_bs = (long)L * 6 * H;
    const bool fuse = ln_fusion_on(h, d, w);
    // two-pass precision: the long-skip convs (models/estimator.py:131-132) take their two A sources — the residual stream
    // and the popped skip — as fp16 planes too, so every producer of those planes (in_proj, conv_2 of blocks 0..L-2) emits
    // ONE fp16 plane; the last block's conv_2 keeps hi / lo for the three-pass final_proj
    const bool f16 = ffn16_on(h, m, w);
    // in_proj: x-half GEMM + hoisted P (cond rows P[b], uncond rows P[B])  [+ block 0's FiLM·mask and LN1 in the epilogue]
    {
        GemmArgs g = dit_gemm(w, mask, EPI_RESID);
        g.a_bmod = w.B; g.resid = w.P.f32; g.resid_clamp = w.B;
        g.out16 = f16;
        if (fuse) {
            set_u(g, w, ada_bs);
            g.ln = 1; g.ln_shift = w.ada; g.ln_scale = w.ada + H;
            g.film2 = film; g.film2_bstride = film_bstride; g.out2_f32 = w.X[1].f32;
        }
        if (run_gemm(h, g, m.inx, &xin, nullptr, w.X[0], s)) return 1;
    }
    // buffer plan (skips are block INPUTS, models/estimator.py:128-131):
    //   X0 = in_proj out (skip for block 5), X1 = block0 out (skip for block 4), X2 = block1 out (skip for block 3)
    int cur = 0;
    for (int l = 0; l < L; ++l) {
        const float* film_l = film + (size_t)l * 2 * H;
        const float* ada_l = w.ada + (size_t)l * 6 * H;
        int xb;                        // buffer holding this block's residual stream
        LnArgs ln;
        ln.BB = w.BB; ln.T = w.T; ln.H = H; ln.mask = mask; ln.B = w.B; ln.c_clamp = w.B; ln.ada_bstride = ada_bs;
        if (l < n_lsc) {
            xb = cur + 1;              // FiLM·mask written to a fresh buffer so the block input survives as a skip
            ln.xin = w.X[cur].f32; ln.xout = w.X[xb].f32; ln.has_film = 1; ln.film = film_l; ln.film_bstride = film_bstride;
        } else {
            // long skip: x = Conv1d(k=3)(cat(x, skip)) UNMASKED (models/estimator.py:131-132), FiLM·mask fused in the epilogue
            // [+ LN1 + modulate]
            const int sk = L - 1 - l;      // pop order: block-(L-1-l) input
            xb = (cur == n_lsc) ? n_lsc + 1 : n_lsc;
            GemmArgs g = dit_gemm(w, mask, EPI_BIAS | EPI_FILM | EPI_MASK);
            g.film = film_l; g.film_bstride = film_bstride;
            if (f16) g.prec = 1;
            if (fuse) { set_u(g, w, ada_bs); g.ln = 1; g.ln_shift = ada_l; g.ln_scale = ada_l + H; }
            Act out = w.X[xb]; out.hi = nullptr; out.lo = nullptr;     // consumed by LN only
            if (run_gemm(h, g, m.lsc[l - n_lsc], &w.X[cur], &w.X[sk], out, s, ST_PROF_GEMM_LSC)) return 1;
            ln.xin = w.X[xb].f32; ln.has_film = 0;
        }
        // the LN1 of block l+1 follows this block's conv_2 directly when that block has no long-skip conv in between
        NextLn nx;
        const bool has_next = fuse && (l + 1 < n_lsc);
        if (has_next) {
            nx.film2 = film + (size_t)(l + 1) * 2 * H; nx.film2_bs = film_bstride; nx.x2_out = w.X[xb + 1].f32;
            nx.shift = w.ada + (size_t)(l + 1) * 6 * H; nx.scale = nx.shift + H;
        }
        if (dit_block_core(h, m, w, l, ln, ada_l, ada_bs, xb, mask, s, fuse, fuse, has_next ? &nx : nullptr, /*x16=*/l + 1 < L)) return 1;
        cur = xb;
    }
    {   // final_proj(x * mask) * mask (:136-137); x is already masked at this point
        GemmArgs g = dit_gemm(w, mask, EPI_BIAS | EPI_MASK);
        if (run_gemm(h, g, m.fin, &w.X[cur], nullptr, w.V, s)) return 1;
    }
    return 0;
}

int st::check_bt(st_handle* h, int B, int T) {
    if (B <= 0 || T <= 0) return fail(h, "B and T must be positive");
    if (B > 32767) return fail(h, "B too large");
    return 0;
}

// =================================================================================================
extern "C" {

int st_create(const st_dims* dims, int device, st_handle** out) {
    if (!dims || !out) return fail(nullptr, "null argument");
    if (dims->n_layers <= 0 || dims->n_layers % 2 || dims->n_layers > 6) return fail(nullptr, "n_layers must be even and <= 6");
    if (const char* why = dit_dims_error(*dims)) return fail(nullptr, why);
    return create_handle(device, std::make_unique<CfmModel>(*dims), out);
}

int st_create_text_encoder(const st_dims* dims, int n_vocab, int device, st_handle** out) {
    if (!dims || !out || n_vocab <= 0) return fail(nullptr, "st_create_text_encoder: bad argument");
    if (dims->n_layers <= 0 || dims->n_layers > 6) return fail(nullptr, "n_layers must be in [1, 6]");
    if (const char* why = dit_dims_error(*dims)) return fail(nullptr, why);
    return create_handle(device, std::make_unique<TextEncoderModel>(*dims, n_vocab), out);
}

size_t st_workspace_bytes(const st_handle* h, int B, int T, int cfg) {
    const DitModel* m = h ? dynamic_cast<const DitModel*>(h->model.get()) : nullptr;
    if (!m || B <= 0 || T <= 0) return 0;
    Workspace w;
    layout_ws(h, *m, w, nullptr, 0, B, T, cfg);
    return w.bytes;
}

int st_estimator_forward(st_handle* h, const float* t, int t_count, const float* x, const float* mask, const float* mu,
                         const float* c, float* out, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = ready_model<CfmModel>(h, "CFM estimator");
    if (!m || check_bt(h, B, T)) return 1;
    if (!t || !x || !mask || !mu || !c || !out) return fail(h, "st_estimator_forward: null pointer");
    if (t_count != 1 && t_count != B) return fail(h, "t must have 1 or B elements (models/estimator.py:107)");
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, 0)) return 1;
    const st_dims& d = m->d;
    if (precompute_cond(h, *m, w, mu, mask, c, nullptr, nullptr, s)) return 1;
    ST_LAUNCH(launch_time_embed(t, t_count, d.hidden, w.temb, s));
    if (precompute_film(h, *m, w, t_count, s)) return 1;
    ST_LAUNCH(launch_bct_to_btc(x, w.xt.f32, w.xs.hi, w.xs.lo, B, d.n_mel, T, nullptr, s));
    Act xin = w.xt; xin.hi = w.xs.hi; xin.lo = w.xs.lo;
    if (estimator_eval(h, *m, w, xin, mask, w.film, t_count == 1 ? 0 : (long)d.n_layers * 2 * d.hidden, s)) return 1;
    ST_LAUNCH(launch_btc_to_bct(w.V.f32, out, B, d.n_mel, T, s));
    return 0;
}

// CFMDecoder.compute_loss's forward value (models/flow_matching.py:69-100) for given draws t (already warped, :92-93)
// and z (:96): y = (1-(1-sigma)t) z + t x1 -> estimator(t, y, mask, mu, c) -> sum((v-u)^2) / (sum(mask) * n_mel).
int st_cfm_loss(st_handle* h, const float* x1, const float* z, const float* t, const float* mask, const float* mu, const float* c,
                float sigma_min, float* y_out, float* loss_out, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = ready_model<CfmModel>(h, "CFM estimator");
    if (!m || check_bt(h, B, T)) return 1;
    if (!x1 || !z || !t || !mask || !mu || !c || !y_out || !loss_out) return fail(h, "st_cfm_loss: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const st_dims& d = m->d;
    ST_LAUNCH(launch_cfm_mix(x1, z, t, sigma_min, B, (long)d.n_mel * T, y_out, s));
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, 0)) return 1;
    // the estimator's (B, n_mel, T) output lands in the workspace (Kst[0] is only used by the ODE drivers)
    if (st_estimator_forward(h, t, B, y_out, mask, mu, c, w.Kst[0], B, T, stream)) return 1;
    ST_LAUNCH(launch_cfm_loss(w.Kst[0], x1, z, mask, sigma_min, B, d.n_mel, T, w.dscal, loss_out, s));
    return 0;
}

// models/text_encoder.py:34-44: emb(x)*sqrt(H) -> n_layers DiTConVBlocks(x, c, x_mask) -> proj(x)*x_mask
int st_text_encoder_forward(st_handle* h, const int64_t* ids, const float* c, const int64_t* x_lengths, float* x_out,
                            float* mu_out, float* mask_out, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    TextEncoderModel* m = ready_model<TextEncoderModel>(h, "text encoder");
    if (!m || check_bt(h, B, T)) return 1;
    if (!ids || !c || !x_lengths || !x_out || !mu_out || !mask_out) return fail(h, "st_text_encoder_forward: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, 0)) return 1;
    const st_dims& d = m->d;
    const int H = d.hidden, L = d.n_layers;
    const long ada_bs = (long)L * 6 * H;
    // x_mask = sequence_mask(x_lengths) (:37) and the masked, scaled embedding (:35; DiTConVBlock masks its input, :106)
    ST_LAUNCH(launch_embed(ids, x_lengths, m->emb, m->n_vocab, B, T, H, sqrtf((float)H), w.X[0].f32, mask_out, s));
    ST_LAUNCH(launch_mask_lengths(mask_out, w.kvlen, w.prefix, B, T, s));
    ST_LAUNCH(launch_rope_table(w.rope_cs, T, 32, s));
    for (int l = 0; l < L; ++l)        // adaLN(c) for every layer: (B, L, 6H)
        ST_LAUNCH(launch_gemv(c, m->ada_w[l], m->ada_b[l], w.ada + (size_t)l * 6 * H, ada_bs, B, d.gin, 6 * H, 1, 0, s));
    const bool fuse = ln_fusion_on(h, d, w);
    for (int l = 0; l < L; ++l) {
        LnArgs ln;
        ln.BB = w.BB; ln.T = w.T; ln.H = H; ln.mask = mask_out; ln.B = w.B; ln.c_clamp = w.B; ln.ada_bstride = ada_bs;
        ln.xin = w.X[0].f32; ln.has_film = 0;
        NextLn nx;                     // block l+1's LN1 rides in this block's conv_2 epilogue (no FiLM in the text encoder)
        nx.film2 = nullptr; nx.film2_bs = 0; nx.x2_out = nullptr;
        nx.shift = w.ada + (size_t)(l + 1) * 6 * H; nx.scale = nx.shift + H;
        if (dit_block_core(h, *m, w, l, ln, w.ada + (size_t)l * 6 * H, ada_bs, 0, mask_out, s, fuse, fuse && l > 0,
                           (fuse && l + 1 < L) ? &nx : nullptr)) return 1;
    }
    {   // mu_x = proj(x) * x_mask (:42)
        GemmArgs g = dit_gemm(w, mask_out, EPI_BIAS | EPI_MASK);
        if (run_gemm(h, g, m->fin, &w.X[0], nullptr, w.V, s)) return 1;
    }
    ST_LAUNCH(launch_btc_to_bct(w.X[0].f32, x_out, B, H, T, s));
    ST_LAUNCH(launch_btc_to_bct(w.V.f32, mu_out, B, d.n_mel, T, s));
    return 0;
}

}  // extern "C"
