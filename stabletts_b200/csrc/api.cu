// C-ABI + host-side orchestration of the CFM/DiT hot path (see include/stabletts_b200.h).
//
// What runs where (reference: models/flow_matching.py:24-67, models/estimator.py:103-137):
//   per solve   : layout change (B,C,T)->(B,T,C); cond_proj(mu) and cond_proj(fake_content) ONCE
//                 (t-independent; exact hoist); in_proj's mu-half P = W_mu·mu' + b ONCE; adaLN(c)
//                 ONCE; time-MLP + FiLM (gamma,beta) for every stage time of the grid up front.
//   per eval    : in_proj x-half + P -> 6 x [ (lsc conv) FiLM·mask, LN, modulate, QKV, RoPE+masked
//                 attention, O+gate+residual, LN, modulate, conv_1+SiLU, conv_2+gate+residual ]
//                 -> final_proj.  With CFG the cond and uncond branches are ONE doubled batch.
//   ODE driver  : explicit Runge–Kutta on the caller's grid, all device-resident: stage times are
//                 baked into kernel arguments, nothing is copied or synchronised between steps.
#include "handle.cuh"
#include "ffgan.cuh"
#include "vocos.cuh"
#include <cmath>
#include <mutex>

using namespace st;

namespace {

std::string g_create_error;
std::mutex g_mutex;

constexpr int MAX_EVAL_TABLE = 1024;

struct Workspace {
    int B = 0, T = 0, cfg = 0, BB = 0, Bc = 0, NT = 0;
    Act xt, ytmp, xs, V, mut, C1, C2, C3, P, X[5], U, QKV, AO, Hid;
    float* Kst[10] = {};               // RK stage derivatives (+ spare state buffers for the adaptive solver)
    double* dscal = nullptr;           // device scalar for norm reductions
    int* kvlen = nullptr; int* prefix = nullptr;
    float *rope_cs = nullptr, *temb = nullptr, *tmid = nullptr, *tvec = nullptr, *film = nullptr, *ada = nullptr;
    float *cin = nullptr;    // (Bc, gin): c rows + fake_speaker row
    // host staging for st_solve_host
    float *h_z = nullptr, *h_mu = nullptr, *h_mask = nullptr, *h_c = nullptr, *h_fc = nullptr, *h_fs = nullptr;
    size_t bytes = 0;
};

}  // namespace

int st::fail(st_handle* h, const std::string& msg) {
    if (h) h->err = msg; else g_create_error = msg;
    return 1;
}

int st::create_handle(int device, std::unique_ptr<Model> model, st_handle** out) {
    std::lock_guard<std::mutex> lk(g_mutex);
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(nullptr, std::string("no CUDA device (this library has no CPU fallback): ") + cudaGetErrorString(e));
    if (device < 0 || device >= n) return fail(nullptr, "bad device index");
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, device) != cudaSuccess) return fail(nullptr, "cudaGetDeviceProperties failed");
    if (p.major != 9) return fail(nullptr, "device is not sm_90-class (Hopper H100 required: the kernels are built for sm_90a)");
    st_handle* h = new st_handle();
    h->device = device; h->num_sms = p.multiProcessorCount;
    if (const char* e = getenv("STABLETTS_B200_PRECISION")) {
        if (!strcmp(e, "bf16x3")) h->precision = ST_PRECISION_BF16X3;
        else if (!strcmp(e, "ffn_fp16x2")) h->precision = ST_PRECISION_FFN_FP16X2;
    }
    h->model = std::move(model);
    *out = h;
    return 0;
}

int st::grow_ws_synced(st_handle* h, void** ws, size_t* have, size_t need, cudaStream_t s) {
    if (need <= *have) return 0;
    if (*ws) { ST_CUDA(cudaStreamSynchronize(s)); cudaFree(*ws); *ws = nullptr; *have = 0; }
    ST_CUDA(cudaMalloc(ws, need));
    *have = need;
    return 0;
}

namespace {

// ----- weight packing ---------------------------------------------------------------------------
// in: (Nsrc, Csrc, k) reference Conv1d / Linear layout -> out[tap][n_off + n][c] for c in [c_off, c_off+Cc)
__global__ void pack_conv_kernel(const float* __restrict__ in, float* __restrict__ out, int Nsrc, int Csrc, int k,
                                 int Ntot, int n_off, int c_off, int Cc) {
    pdl_trigger(); pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    long total = (long)k * Nsrc * Cc;
    if (i >= total) return;
    int c = (int)(i % Cc);
    long r = i / Cc;
    int n = (int)(r % Nsrc);
    int tap = (int)(r / Nsrc);
    out[((long)tap * Ntot + n_off + n) * Cc + c] = in[((long)n * Csrc + c_off + c) * k + tap];
}

struct TArr { float v[256]; };
__global__ void time_embed_val_kernel(TArr t, int n_t, int H, float* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int half = H / 2;
    if (i >= n_t * half) return;
    int r = i / half, j = i - r * half;
    float step = (float)(9.210340371976184 / (double)(half - 1));
    float w = expf((float)j * -step);
    float e = 1000.0f * t.v[r] * w;
    out[(long)r * H + j] = sinf(e);
    out[(long)r * H + half + j] = cosf(e);
}

}  // namespace

cudaError_t st::launch_pack_conv(const float* in, float* out, int Nsrc, int Csrc, int k, int Ntot, int n_off, int c_off, int Cc,
                                 cudaStream_t s) {
    const long total = (long)k * Nsrc * Cc;
    if (total == 0) return cudaSuccess;
    pack_conv_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, out, Nsrc, Csrc, k, Ntot, n_off, c_off, Cc);
    return cudaGetLastError();
}

int st::get_raw(st_handle* h, const std::string& name, int64_t expect, float** out) {
    auto it = h->raw.find(name);
    if (it == h->raw.end()) return fail(h, "missing weight: " + name);
    if (it->second.second != expect) {
        char b[256];
        snprintf(b, sizeof b, "weight %s has %lld elements, expected %lld", name.c_str(), (long long)it->second.second,
                 (long long)expect);
        return fail(h, b);
    }
    *out = it->second.first;
    return 0;
}

// Packs `parts` reference tensors (each (N_i, Csrc, k)) stacked along N, taking channels [c_off, c_off+Cc).
int st::pack_gemm(st_handle* h, GemmW* w, const std::vector<std::string>& names, int N_each, int Csrc, int k, int c_off,
                  int Cc, bool with_bias, cudaStream_t s) {
    int parts = (int)names.size();
    w->taps = k; w->N = N_each * parts; w->K = Cc;
    size_t n = (size_t)k * w->N * Cc;
    if (dev_alloc(h, &w->f32, n)) return 1;
    if (dev_alloc(h, &w->hi, n)) return 1;
    if (dev_alloc(h, &w->lo, n)) return 1;
    if (with_bias && dev_alloc(h, &w->bias, (size_t)w->N)) return 1;
    for (int p = 0; p < parts; ++p) {
        float* src;
        if (get_raw(h, names[p] + ".weight", (int64_t)N_each * Csrc * k, &src)) return 1;
        long total = (long)k * N_each * Cc;
        pack_conv_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(src, w->f32, N_each, Csrc, k, w->N, p * N_each,
                                                                         c_off, Cc);
        ST_CUDA(cudaGetLastError());
        if (with_bias) {
            float* bsrc;
            if (get_raw(h, names[p] + ".bias", N_each, &bsrc)) return 1;
            ST_CUDA(cudaMemcpyAsync(w->bias + (size_t)p * N_each, bsrc, sizeof(float) * N_each, cudaMemcpyDeviceToDevice, s));
        }
    }
    ST_CUDA(launch_split(w->f32, w->hi, w->lo, (long)n, s));
    return 0;
}

namespace {

// ----- models -------------------------------------------------------------------------------------
// What the CFM estimator and the text encoder share: DiT blocks (models/diffusion_transformer.py:98-117) and a final
// 1x1 projection.
struct DitModel : Model {
    st_dims d;
    std::vector<GemmW> qkv, wo, c1, c2;
    std::vector<float*> ada_w, ada_b;
    GemmW fin;
    explicit DitModel(const st_dims& dims) : d(dims) {}
    // the weights of block l under `p` ("blocks.<l>.block." / "encoder.<l>.")
    int pack_block(st_handle* h, int l, const std::string& p, cudaStream_t s);
};

// Decoder (models/estimator.py:65-137) with the ODE drivers' per-handle state.
struct CfmModel : DitModel {
    GemmW cond0, cond2, cond4, inmu, inx;
    std::vector<GemmW> lsc;
    std::vector<float*> film_w, film_b;
    float *tm0_w = nullptr, *tm0_b = nullptr, *tm2_w = nullptr, *tm2_b = nullptr;
    // CUDA-graph cache for launch-bound (small) solves: key -> instantiated graph + its launch count
    struct GraphEntry { std::string key; cudaGraphExec_t exec; int64_t launches; };
    std::vector<GraphEntry> graphs;
    std::vector<std::string> graph_seen;   // keys enqueued directly once (kernels loaded, attributes set) before capture
    cudaStream_t cap_stream = nullptr;   // capture happens on a private stream (the caller's may be the legacy stream)
    int graph_mode = -1;               // -1: read STABLETTS_B200_GRAPH on first use; 0 off; 1 always; 2 auto (small problems)
    double* pinned = nullptr;          // 16 B of pinned host memory: norm read-back of the adaptive controller
    char* pin_buf = nullptr; size_t pin_bytes = 0;   // pinned staging of st_solve_host for callers with pageable buffers
    using DitModel::DitModel;
    ~CfmModel() override {
        drop_cached();
        if (cap_stream) cudaStreamDestroy(cap_stream);
        if (pinned) cudaFreeHost(pinned);
        if (pin_buf) cudaFreeHost(pin_buf);
    }
    void drop_cached() override { for (auto& g : graphs) cudaGraphExecDestroy(g.exec); graphs.clear(); }
    int finalize(st_handle* h, cudaStream_t s) override;
};

// TextEncoder (models/text_encoder.py:8-44): an embedding, n_layers DiT blocks without FiLM, proj
struct TextEncoderModel : DitModel {
    int n_vocab;
    float* emb = nullptr;
    TextEncoderModel(const st_dims& dims, int vocab) : DitModel(dims), n_vocab(vocab) {}
    int finalize(st_handle* h, cudaStream_t s) override;
};

// ----- workspace ----------------------------------------------------------------------------------
void layout_ws(const st_handle* h, const DitModel& m, Workspace& w, void* base, size_t cap, int B, int T, int cfg) {
    const st_dims& d = m.d;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    w.B = B; w.T = T; w.cfg = cfg; w.BB = cfg ? 2 * B : B; w.Bc = B + (cfg ? 1 : 0);
    w.NT = std::max(MAX_EVAL_TABLE, B);
    Bump bp(base, cap);
    const size_t bt = (size_t)B * T, bbt = (size_t)w.BB * T, bct = (size_t)w.Bc * T;
    auto mk = [&](Act& a, size_t rows, int C, bool f32, bool split) {
        a.C = C;
        a.f32 = f32 ? bp.take<float>(rows * C) : nullptr;
        a.hi = split ? bp.take<bf16>(rows * C) : nullptr;
        a.lo = split ? bp.take<bf16>(rows * C) : nullptr;
    };
    mk(w.xt, bt, d.n_mel, true, false);
    mk(w.ytmp, bt, d.n_mel, true, false);
    mk(w.xs, bt, d.n_mel, false, tc);
    mk(w.V, bbt, d.n_mel, true, false);
    for (int i = 0; i < 10; ++i) w.Kst[i] = bp.take<float>(bt * d.n_mel);
    w.dscal = bp.take<double>(2);
    mk(w.mut, bct, d.n_mel, !tc, tc);
    mk(w.C1, bct, d.filter, !tc, tc);
    mk(w.C2, bct, d.filter, !tc, tc);
    mk(w.C3, bct, d.hidden, !tc, tc);
    mk(w.P, bct, d.hidden, true, false);
    for (int i = 0; i < 5; ++i) mk(w.X[i], bbt, d.hidden, true, tc);
    mk(w.U, bbt, d.hidden, !tc, tc);
    mk(w.QKV, bbt, 3 * d.hidden, !tc, tc);       // tensor-core engine: RoPE'd split planes straight from the GEMM epilogue
    mk(w.AO, bbt, d.hidden, !tc, tc);
    mk(w.Hid, bbt, d.filter, !tc, tc);
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

int ensure_ws(st_handle* h, DitModel& m, Workspace& w, int B, int T, int cfg) {
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

}  // namespace

// fp16 hi / lo planes of a packed weight (the FFN convs; used by ST_PRECISION_FFN_FP16X2)
static int pack_f16_planes(st_handle* h, GemmW* w, cudaStream_t s) {
    const size_t n = (size_t)w->taps * w->N * w->K;
    if (dev_alloc(h, &w->h_hi, n) || dev_alloc(h, &w->h_lo, n)) return 1;
    ST_CUDA(launch_split_f16(w->f32, w->h_hi, w->h_lo, (long)n, s));
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
    return get_raw(h, "time_mlp.layer.2.bias", H, &tm2_b);
}

// models/text_encoder.py:22-26: emb, n_layers DiTConVBlocks, proj
int TextEncoderModel::finalize(st_handle* h, cudaStream_t s) {
    const int H = d.hidden, L = d.n_layers;
    qkv.assign(L, GemmW()); wo.assign(L, GemmW()); c1.assign(L, GemmW()); c2.assign(L, GemmW());
    ada_w.assign(L, nullptr); ada_b.assign(L, nullptr);
    for (int l = 0; l < L; ++l)
        if (pack_block(h, l, "encoder." + std::to_string(l) + ".", s)) return 1;
    if (pack_gemm(h, &fin, {"proj"}, d.n_mel, H, 1, 0, H, true, s)) return 1;
    return get_raw(h, "emb.weight", (int64_t)n_vocab * H, &emb);
}

// ----- GEMM dispatch -------------------------------------------------------------------------------
// S x tiles <= num_sms tiles of at most 128 x 128 fp32: one buffer of num_sms x 64 KB (8.7 MB on 132 SMs) covers every shape
// run_gemm splits, so it is allocated once and never moves (captured graphs keep pointing at it).  Not inside a stream
// capture (cudaMalloc is not capturable): run_gemm runs such a call unsplit.
static int ensure_part_buf(st_handle* h) {
    if (h->part_buf) return 0;
    h->part_bytes = (size_t)h->num_sms * 128 * 128 * sizeof(float);
    ST_CUDA(cudaMalloc((void**)&h->part_buf, h->part_bytes));
    return 0;
}

int st::run_gemm(st_handle* h, GemmArgs& g, const GemmW& w, const Act* a0, const Act* a1, const Act& out, cudaStream_t s,
                 int prof_cat) {
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    g.n_src = a1 ? 2 : 1;
    const Act* as[2] = {a0, a1};
    int ktot = 0;
    for (int i = 0; i < g.n_src; ++i) {
        g.A_f32[i] = as[i]->f32; g.A_hi[i] = as[i]->hi; g.A_lo[i] = as[i]->lo; g.Cs[i] = as[i]->C;
        ktot += as[i]->C;
        if (tc ? (!as[i]->hi) : (!as[i]->f32)) return fail(h, "internal: GEMM operand plane missing for engine");
    }
    if (ktot != w.K) return fail(h, "internal: GEMM K mismatch");
    g.W_f32 = w.f32; g.W_hi = w.hi; g.W_lo = w.lo; g.bias = w.bias;
    if (g.prec) {
        if (!w.h_hi) return fail(h, "internal: fp16 weight planes missing for the two-pass FFN precision");
        g.W_hi = w.h_hi; g.W_lo = w.h_lo;
    }
    if ((g.flags & EPI_BIAS) && !w.bias) return fail(h, "internal: bias requested but absent");
    g.taps = w.taps; g.N = w.N; g.Ktot = w.K;
    g.out_f32 = out.f32; g.out_hi = out.hi; g.out_lo = out.lo;
    if (out.C != w.N) return fail(h, "internal: GEMM N mismatch");
    // Latency-bound small problems (a handful of 128 x 128 tiles, e.g. one 300-frame utterance): a long K loop
    // on 12 SMs is serial time; cut it into slices that run side by side and sum them in a fixed order afterwards.
    if (const char* why = gemm_flags_error(g)) return fail(h, std::string("GEMM refused: ") + why);
    g.ksplit = 1; g.part = nullptr;    // callers reuse one GemmArgs for several GEMMs: the decision is per call
    // split-K's reduce kernel writes fp32 and split-bf16 planes only: never for an fp16 output plane (out16 / u16)
    const bool splittable = tc && !g.ln && !g.prec && !g.out16 && !g.u16 && !(g.flags & EPI_ROPE) && g.N % 4 == 0 &&
                            !gemm_tc_wide_tile(g, h->num_sms);
    if (g.force_ksplit > 1 && !splittable)
        return fail(h, "split-K is not available for this GEMM (SIMT engine, RoPE, LayerNorm, fp16 planes, N % 4 or 256-channel tiles)");
    if (splittable && g.force_ksplit != 1 && (g.force_ksplit > 1 || !g.batch_invariant)) {
        static int env = -1;
        if (env < 0) { const char* e = getenv("STABLETTS_B200_SPLITK"); env = e ? atoi(e) : 1; }   // 0: off, 1: auto, 2..4: only that factor
        const int kb = g.taps * ((g.Cs[0] + 63) / 64 + (g.n_src > 1 ? (g.Cs[1] + 63) / 64 : 0));
        const long tiles = (long)g.BB * ((g.T + 127) / 128) * ((g.N + 127) / 128);
        int S = 1;
        for (int cand = 4; cand >= 2 && env; --cand)
            if ((env == 1 || env == cand) && kb % cand == 0 && kb / cand >= 3 && tiles * cand <= h->num_sms) { S = cand; break; }
        if (g.force_ksplit > 1) S = g.force_ksplit;     // launch_gemm_tc refuses a factor that does not divide the K loop
        if (S > 1 && !h->part_buf) {
            cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
            ST_CUDA(cudaStreamIsCapturing(s, &cap));
            if (cap != cudaStreamCaptureStatusNone) S = 1;
            else if (ensure_part_buf(h)) return 1;
        }
        if (S > 1) {
            if ((size_t)S * g.BB * g.T * g.N * sizeof(float) > h->part_bytes) return fail(h, "internal: split-K partial buffer too small");
            g.ksplit = S; g.part = h->part_buf;
            h->launches++;             // the reduce + epilogue kernel
            if (getenv("STABLETTS_B200_DEBUG"))
                fprintf(stderr, "[stabletts_b200] split-K x%d: BB %d T %d N %d K %d taps %d n_src %d a_bmod %d flags 0x%x\n", S, g.BB, g.T, g.N,
                        g.Ktot, g.taps, g.n_src, g.a_bmod, g.flags);
        }
    }
    st_handle::ProfRec pr{prof_cat, 2.0 * g.BB * g.T * (double)g.N * g.Ktot * g.taps,
                          (double)g.BB * g.T * ((double)g.Ktot * 4 + (double)g.N * ((out.f32 ? 4 : 0) + (out.hi ? 4 : 0))), nullptr, nullptr};
    if (tc) pr.issued = pr.flops * (g.prec ? 2.0 : 3.0);   // split operands: A_lo*W_hi + A_hi*W_lo + A_hi*W_hi, or A16*W_lo + A16*W_hi
    if (h->prof_on) { pr.e0 = h->take_event(); pr.e1 = h->take_event(); cudaEventRecord(pr.e0, s); }
    h->launches++;
    static int dbg = -1;
    if (dbg < 0) { const char* e = getenv("STABLETTS_B200_DEBUG"); dbg = e ? atoi(e) : 0; }
    if (dbg >= 2) {
        cudaError_t e = cudaStreamSynchronize(s);
        fprintf(stderr, "[stabletts_b200] gemm BB %d T %d N %d K %d taps %d flags 0x%x ln %d prec %d ksplit %d (before: %s) ... ", g.BB, g.T, g.N,
                g.Ktot, g.taps, g.flags, g.ln ? 1 : 0, g.prec, g.ksplit, cudaGetErrorString(e));
        fflush(stderr);
    }
    if (tc) {
        cudaError_t e = launch_gemm_tc(g, h->num_sms, s);
        if (e != cudaSuccess) return fail(h, std::string("wgmma GEMM launch failed: ") + cudaGetErrorString(e) + " / " + gemm_tc_last_error());
    } else {
        if (const char* why = gemm_simt_unsupported(g)) return fail(h, std::string("SIMT GEMM refused: ") + why);
        cudaError_t e = launch_gemm_simt(g, s);
        if (e != cudaSuccess) return fail(h, std::string("SIMT GEMM launch failed: ") + cudaGetErrorString(e));
    }
    if (dbg >= 2) { cudaError_t e = cudaStreamSynchronize(s); fprintf(stderr, "%s\n", cudaGetErrorString(e)); }
    if (h->prof_on) { cudaEventRecord(pr.e1, s); h->prof.push_back(pr); }
    return 0;
}

namespace {

// ----- per-solve precompute -------------------------------------------------------------------------
// cond features (models/estimator.py:118) for B real rows + (cfg) the broadcast fake_content row;
// P = W_in[:, M:]·mu' + b_in (models/estimator.py:120-121, mu-half); adaLN(c) (diffusion_transformer.py:110)
int precompute_cond(st_handle* h, const CfmModel& m, Workspace& w, const float* mu, const float* mask, const float* c,
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
int precompute_film(st_handle* h, const CfmModel& m, Workspace& w, int n_t, cudaStream_t s) {
    const st_dims& d = m.d;
    ST_LAUNCH(launch_gemv(w.temb, m.tm0_w, m.tm0_b, w.tmid, d.filter, n_t, d.hidden, d.filter, 0, 1, s));
    ST_LAUNCH(launch_gemv(w.tmid, m.tm2_w, m.tm2_b, w.tvec, d.hidden, n_t, d.filter, d.hidden, 0, 0, s));
    for (int l = 0; l < d.n_layers; ++l)   // film layout (n_t, L, 2H)
        ST_LAUNCH(launch_gemv(w.tvec, m.film_w[l], m.film_b[l], w.film + (size_t)l * 2 * d.hidden, (long)d.n_layers * 2 * d.hidden,
                              n_t, d.hidden, 2 * d.hidden, 0, 0, s));
    return 0;
}

// The LayerNorm + adaLN modulate that FOLLOWS a GEMM whose tile owns whole 256-channel rows rides in that GEMM's epilogue
// (gemm_epilogue.cuh, EM_LN): O -> LN2, conv_2 / in_proj -> the next block's [FiLM·mask +] LN1, long-skip conv -> LN1.
// Small problems (fewer 128 x 256 tiles than SMs: they run on 128 x 128 tiles) and the SIMT engine keep the separate kernel.
bool ln_fusion_on(const st_handle* h, const st_dims& d, const Workspace& w) {
    static int env = -1;
    if (env < 0) { const char* e = getenv("STABLETTS_B200_FUSE_LN"); env = (e && !strcmp(e, "0")) ? 0 : 1; }
    if (!env || h->engine != ST_ENGINE_TCGEN05) return false;
    GemmArgs g;
    g.BB = w.BB; g.T = w.T; g.N = d.hidden; g.Ktot = d.hidden; g.Cs[0] = d.hidden; g.n_src = 1;
    g.A_hi[0] = w.U.hi; g.W_hi = w.U.hi;           // non-null placeholders: only shapes matter here
    return gemm_tc_ln_fusable(g, h->num_sms);
}

// The opt-in two-pass FFN precision applies when both FFN convs of this problem run on 256-channel tiles.
bool ffn16_on(const st_handle* h, const st_dims& d, const Workspace& w) {
    if (h->precision != ST_PRECISION_FFN_FP16X2 || h->engine != ST_ENGINE_TCGEN05) return false;
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
    const bool f16 = ffn16_on(h, d, w);   // LN2's U and the hidden activation travel as ONE fp16 plane (in the hi buffers)
    auto base = [&](int flags) {
        GemmArgs g;
        g.BB = w.BB; g.T = w.T; g.a_bmod = w.BB; g.B = w.B; g.mask = mask; g.flags = flags;
        g.c_clamp = w.B; g.resid_clamp = w.BB - 1; g.film_H = H; g.rope_cs = w.rope_cs;
        g.ada_bstride = ada_bs; g.u_hi = w.U.hi; g.u_lo = w.U.lo;
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

// ----- one estimator evaluation (models/estimator.py:120-137) ------------------------------------------
// xin: (B, T, M) stage input (fp32 [+ split planes for the tensor engine]); writes w.V (BB, T, M).
// film: table row for this eval, (L, 2H); film_bstride != 0 when t is per-sample.
int estimator_eval(st_handle* h, const CfmModel& m, Workspace& w, const Act& xin, const float* mask, const float* film,
                   long film_bstride, cudaStream_t s) {
    const st_dims& d = m.d;
    const int H = d.hidden, L = d.n_layers, n_lsc = L / 2;
    const long ada_bs = (long)L * 6 * H;
    auto base = [&](int flags) {
        GemmArgs g;
        g.BB = w.BB; g.T = w.T; g.a_bmod = w.BB; g.B = w.B; g.mask = mask; g.flags = flags;
        g.c_clamp = w.B; g.resid_clamp = w.BB - 1; g.film_H = H; g.rope_cs = w.rope_cs;
        return g;
    };
    const bool fuse = ln_fusion_on(h, d, w);
    // two-pass precision: the long-skip convs (models/estimator.py:131-132) take their two A sources — the residual stream
    // and the popped skip — as fp16 planes too, so every producer of those planes (in_proj, conv_2 of blocks 0..L-2) emits
    // ONE fp16 plane; the last block's conv_2 keeps hi / lo for the three-pass final_proj
    const bool f16 = ffn16_on(h, d, w);
    auto set_u = [&](GemmArgs& g) { g.ada_bstride = ada_bs; g.u_hi = w.U.hi; g.u_lo = w.U.lo; };
    // in_proj: x-half GEMM + hoisted P (cond rows P[b], uncond rows P[B])  [+ block 0's FiLM·mask and LN1 in the epilogue]
    {
        GemmArgs g = base(EPI_RESID);
        g.a_bmod = w.B; g.resid = w.P.f32; g.resid_clamp = w.B;
        g.out16 = f16;
        if (fuse) {
            set_u(g);
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
            GemmArgs g = base(EPI_BIAS | EPI_FILM | EPI_MASK);
            g.film = film_l; g.film_bstride = film_bstride;
            if (f16) g.prec = 1;
            if (fuse) { set_u(g); g.ln = 1; g.ln_shift = ada_l; g.ln_scale = ada_l + H; }
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
        GemmArgs g = base(EPI_BIAS | EPI_MASK);
        if (run_gemm(h, g, m.fin, &w.X[cur], nullptr, w.V, s)) return 1;
    }
    return 0;
}

struct Tableau { int S; float c[6]; float a[6][5]; float b[6]; };

Tableau tableau_for(int method) {
    Tableau t{};
    if (method == ST_EULER) { t.S = 1; t.b[0] = 1.f; }
    else if (method == ST_MIDPOINT) { t.S = 2; t.c[1] = 0.5f; t.a[1][0] = 0.5f; t.b[1] = 1.f; }
    else if (method == ST_RK4) {   // torchdiffeq "rk4" = 3/8 rule
        t.S = 4; t.c[1] = 1.f / 3; t.c[2] = 2.f / 3; t.c[3] = 1.f;
        t.a[1][0] = 1.f / 3; t.a[2][0] = -1.f / 3; t.a[2][1] = 1.f; t.a[3][0] = 1.f; t.a[3][1] = -1.f; t.a[3][2] = 1.f;
        t.b[0] = 0.125f; t.b[1] = 0.375f; t.b[2] = 0.375f; t.b[3] = 0.125f;
    } else {                       // Dormand–Prince 5(4) stages 1..6, 5th-order weights, no error control
        t.S = 6;
        const double c[6] = {0, 1. / 5, 3. / 10, 4. / 5, 8. / 9, 1};
        const double a[6][5] = {{0}, {1. / 5}, {3. / 40, 9. / 40}, {44. / 45, -56. / 15, 32. / 9},
                                {19372. / 6561, -25360. / 2187, 64448. / 6561, -212. / 729},
                                {9017. / 3168, -355. / 33, 46732. / 5247, 49. / 176, -5103. / 18656}};
        const double b[6] = {35. / 384, 0, 500. / 1113, 125. / 192, -2187. / 6784, 11. / 84};
        for (int i = 0; i < 6; ++i) { t.c[i] = (float)c[i]; t.b[i] = (float)b[i]; for (int j = 0; j < 5; ++j) t.a[i][j] = (float)a[i][j]; }
    }
    return t;
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

int check_common(st_handle* h, int B, int T) {
    if (!h->finalized) return fail(h, "weights not finalized (call st_finalize_weights)");
    if (B <= 0 || T <= 0) return fail(h, "B and T must be positive");
    if (B > 32767) return fail(h, "B too large");
    return 0;
}

}  // namespace

// =================================================================================================
extern "C" {

int st_version(void) { return 20600; }

const char* st_last_error(const st_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

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

int st_destroy(st_handle* h) {
    if (!h) return 0;
    {
    ST_ENTER(h);
    cudaDeviceSynchronize();
    h->model.reset();
    for (auto& kv : h->raw) cudaFree(kv.second.first);
    for (void* p : h->owned) cudaFree(p);
    for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
    if (h->part_buf) cudaFree(h->part_buf);
    if (h->ws_ptr && h->ws_owned) cudaFree(h->ws_ptr);
    }
    delete h;
    return 0;
}

int st_set_engine(st_handle* h, int engine) {
    if (!h) return 1;
    h->model->drop_cached();
    if (engine != ST_ENGINE_TCGEN05 && engine != ST_ENGINE_SIMT) return fail(h, "unknown engine");
    h->engine = engine;
    return 0;
}

int st_set_precision(st_handle* h, int precision) {
    if (!h) return 1;
    if (precision != ST_PRECISION_BF16X3 && precision != ST_PRECISION_FFN_FP16X2) return fail(h, "unknown precision mode");
    h->model->drop_cached();           // cached graphs bake the kernel instances in
    h->precision = precision;
    return 0;
}

int64_t st_launch_count(const st_handle* h) { return h ? h->launches : 0; }

int st_profile_begin(st_handle* h) {
    if (!h) return 1;
    h->prof.clear(); h->ev_used = 0; h->prof_on = true;
    return 0;
}

int st_profile_end(st_handle* h, double* ms, double* flops, double* bytes, int64_t* launches) {
    if (!h) return 1;
    h->prof_on = false;
    ST_ENTER(h);
    ST_CUDA(cudaDeviceSynchronize());
    for (int i = 0; i < ST_PROF_NCAT; ++i) { ms[i] = 0; flops[i] = 0; bytes[i] = 0; launches[i] = 0; h->prof_issued[i] = 0; }
    for (auto& r : h->prof) {
        float t = 0.f;
        ST_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
        ms[r.cat] += t; flops[r.cat] += r.flops; bytes[r.cat] += r.bytes; launches[r.cat] += 1;
        h->prof_issued[r.cat] += r.issued;
    }
    h->prof.clear(); h->ev_used = 0;
    return 0;
}

int st_profile_issued(st_handle* h, double* issued) {
    if (!h || !issued) return 1;
    for (int i = 0; i < ST_PROF_NCAT; ++i) issued[i] = h->prof_issued[i];
    return 0;
}

int st_load_weight(st_handle* h, const char* name, const float* data, int64_t numel, void* stream) {
    if (!h || !name || !data || numel <= 0) return fail(h, "st_load_weight: bad argument");
    ST_ENTER(h);
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, data) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        return fail(h, std::string("st_load_weight: ") + name + " is not a device pointer (no CPU path)");
    }
    float* p;
    ST_CUDA(cudaMalloc((void**)&p, sizeof(float) * numel));
    {
        cudaError_t ce = cudaMemcpyAsync(p, data, sizeof(float) * numel, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
        if (ce != cudaSuccess) { cudaFree(p); return fail(h, std::string("st_load_weight: copy of ") + name + " failed: " + cudaGetErrorString(ce)); }
    }
    auto it = h->raw.find(name);
    if (it != h->raw.end()) { cudaFree(it->second.first); }
    h->raw[name] = {p, numel};
    h->finalized = false;
    return 0;
}

int st_finalize_weights(st_handle* h, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    h->model->drop_cached();           // cached graphs hold pointers into the old packed weights
    for (void* p : h->owned) cudaFree(p);
    h->owned.clear();
    if (h->model->finalize(h, (cudaStream_t)stream)) return 1;
    h->finalized = true;
    return 0;
}

size_t st_workspace_bytes(const st_handle* h, int B, int T, int cfg) {
    const DitModel* m = h ? dynamic_cast<const DitModel*>(h->model.get()) : nullptr;
    if (!m || B <= 0 || T <= 0) return 0;
    Workspace w;
    layout_ws(h, *m, w, nullptr, 0, B, T, cfg);
    return w.bytes;
}

int st_attach_workspace(st_handle* h, void* dev_ptr, size_t bytes) {
    if (!h) return 1;
    ST_ENTER(h);
    if (h->ws_ptr && h->ws_owned) cudaFree(h->ws_ptr);
    h->model->drop_cached();           // cached graphs hold pointers into the old workspace
    h->ws_ptr = dev_ptr; h->ws_bytes = dev_ptr ? bytes : 0; h->ws_owned = false;
    return 0;
}

int st_estimator_forward(st_handle* h, const float* t, int t_count, const float* x, const float* mask, const float* mu,
                         const float* c, float* out, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = model_of<CfmModel>(h, "CFM estimator");
    if (!m || check_common(h, B, T)) return 1;
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
    CfmModel* m = model_of<CfmModel>(h, "CFM estimator");
    if (!m || check_common(h, B, T)) return 1;
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

// enqueues one complete solve on `s` (no host synchronisation, capturable into a CUDA graph)
static int solve_impl(st_handle* h, const CfmModel& m, Workspace& w, float* z_inout, const float* mu, const float* mask, const float* c,
                      const float* fake_content, const float* fake_speaker, float cfg_strength, const float* t_span_host,
                      int n_steps, int method, int B, int T, int cfg, cudaStream_t s) {
    const st_dims& d = m.d;
    const Tableau tb = tableau_for(method);
    const long numel = (long)B * T * d.n_mel;

    if (precompute_cond(h, m, w, mu, mask, c, fake_content, fake_speaker, s)) return 1;
    ST_LAUNCH(launch_bct_to_btc(z_inout, w.xt.f32, nullptr, nullptr, B, d.n_mel, T, nullptr, s));

    // stage times, fp32 arithmetic as torchdiffeq's fixed-grid solvers evaluate them
    std::vector<float> tv((size_t)n_steps * tb.S);
    for (int i = 0; i < n_steps; ++i) {
        const float t0 = t_span_host[i], t1 = t_span_host[i + 1], dt = t1 - t0;
        for (int st = 0; st < tb.S; ++st) tv[(size_t)i * tb.S + st] = (tb.c[st] == 1.f) ? t1 : t0 + tb.c[st] * dt;
    }
    const int n_eval = n_steps * tb.S;
    const long film_row = (long)d.n_layers * 2 * d.hidden;
    int table_lo = 0, table_hi = 0;      // evals [lo, hi) currently in the FiLM table
    for (int e = 0; e < n_eval; ++e) {
        if (e >= table_hi) {             // (re)fill the t-conditioning table: no copies, times travel as kernel args
            table_lo = e; table_hi = std::min(n_eval, e + MAX_EVAL_TABLE);
            for (int off = table_lo; off < table_hi; off += 256) {
                TArr ta; int n = std::min(256, table_hi - off);
                for (int i = 0; i < n; ++i) ta.v[i] = tv[off + i];
                int cnt = n * (d.hidden / 2);
                h->launches++;
                time_embed_val_kernel<<<(cnt + 127) / 128, 128, 0, s>>>(ta, n, d.hidden, w.temb + (size_t)(off - table_lo) * d.hidden);
                ST_CUDA(cudaGetLastError());
            }
            if (precompute_film(h, m, w, table_hi - table_lo, s)) return 1;
        }
        const int step = e / tb.S, st = e % tb.S;
        const float dt = t_span_host[step + 1] - t_span_host[step];
        Act xin = w.xt;
        if (st > 0) {                    // stage input y + dt * sum_j a[st][j] K_j
            float coef[6]; const float* Ks[6];
            for (int j = 0; j < st; ++j) { coef[j] = dt * tb.a[st][j]; Ks[j] = w.Kst[j]; }
            ST_LAUNCH(launch_lincomb(w.ytmp.f32, w.xt.f32, Ks, coef, st, numel, s));
            xin = w.ytmp;
        }
        if (h->engine == ST_ENGINE_TCGEN05) {
            ST_LAUNCH(launch_split(xin.f32, w.xs.hi, w.xs.lo, numel, s));
            xin.hi = w.xs.hi; xin.lo = w.xs.lo;
        }
        if (estimator_eval(h, m, w, xin, mask, w.film + (size_t)(e - table_lo) * film_row, 0, s)) return 1;
        ST_LAUNCH(launch_cfg_combine(w.V.f32, w.Kst[st], B, (long)T * d.n_mel, cfg, cfg_strength, s));
        if (st == tb.S - 1) {            // y += dt * sum_j b_j K_j
            float coef[6]; const float* Ks[6]; int n = 0;
            for (int j = 0; j < tb.S; ++j) if (tb.b[j] != 0.f) { coef[n] = dt * tb.b[j]; Ks[n] = w.Kst[j]; ++n; }
            ST_LAUNCH(launch_lincomb(w.xt.f32, w.xt.f32, Ks, coef, n, numel, s));
        }
    }
    ST_LAUNCH(launch_btc_to_bct(w.xt.f32, z_inout, B, d.n_mel, T, s));
    return 0;
}

// models/text_encoder.py:34-44: emb(x)*sqrt(H) -> n_layers DiTConVBlocks(x, c, x_mask) -> proj(x)*x_mask
int st_text_encoder_forward(st_handle* h, const int64_t* ids, const float* c, const int64_t* x_lengths, float* x_out,
                            float* mu_out, float* mask_out, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    TextEncoderModel* m = model_of<TextEncoderModel>(h, "text encoder");
    if (!m || check_common(h, B, T)) return 1;
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
        GemmArgs g;
        g.BB = w.BB; g.T = w.T; g.a_bmod = w.BB; g.B = w.B; g.mask = mask_out; g.flags = EPI_BIAS | EPI_MASK;
        g.c_clamp = w.B; g.resid_clamp = w.BB - 1;
        if (run_gemm(h, g, m->fin, &w.X[0], nullptr, w.V, s)) return 1;
    }
    ST_LAUNCH(launch_btc_to_bct(w.X[0].f32, x_out, B, H, T, s));
    ST_LAUNCH(launch_btc_to_bct(w.V.f32, mu_out, B, d.n_mel, T, s));
    return 0;
}

int st_solve(st_handle* h, float* z_inout, const float* mu, const float* mask, const float* c, const float* fake_content,
             const float* fake_speaker, float cfg_strength, const float* t_span_host, int n_steps, int method, int B, int T,
             void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = model_of<CfmModel>(h, "CFM estimator");
    if (!m || check_common(h, B, T)) return 1;
    if (!z_inout || !mu || !mask || !c || !t_span_host) return fail(h, "st_solve: null pointer");
    if (n_steps <= 0) return fail(h, "n_timesteps must be positive");
    if (method < ST_EULER || method > ST_DOPRI5_FIXED) return fail(h, "unknown ODE method");
    const int cfg = (fake_content && fake_speaker) ? 1 : 0;
    if (!cfg && (fake_content || fake_speaker)) return fail(h, "CFG needs both fake_content and fake_speaker");
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, cfg)) return 1;
    const st_dims& d = m->d;
    if (m->graph_mode < 0) {
        const char* e = getenv("STABLETTS_B200_GRAPH");
        m->graph_mode = !e ? 2 : (!strcmp(e, "0") ? 0 : (!strcmp(e, "1") ? 1 : 2));
    }
    // Small problems are launch-bound (~90 kernels per evaluation, a few microseconds each): replay the whole
    // solve as one CUDA graph.  Inputs are staged into workspace-owned buffers so the graph's pointers are stable.
    const long rows = (long)(cfg ? 2 * B : B) * T;
    const bool use_graph = !h->prof_on && (m->graph_mode == 1 || (m->graph_mode == 2 && rows <= 24576));
    if (!use_graph)
        return solve_impl(h, *m, w, z_inout, mu, mask, c, fake_content, fake_speaker, cfg_strength, t_span_host, n_steps, method, B, T, cfg, s);

    const size_t n = (size_t)B * T * d.n_mel;
    if (z_inout != w.h_z) ST_CUDA(cudaMemcpyAsync(w.h_z, z_inout, n * 4, cudaMemcpyDeviceToDevice, s));
    if (mu != w.h_mu) ST_CUDA(cudaMemcpyAsync(w.h_mu, mu, n * 4, cudaMemcpyDeviceToDevice, s));
    if (mask != w.h_mask) ST_CUDA(cudaMemcpyAsync(w.h_mask, mask, (size_t)B * T * 4, cudaMemcpyDeviceToDevice, s));
    if (c != w.h_c) ST_CUDA(cudaMemcpyAsync(w.h_c, c, (size_t)B * d.gin * 4, cudaMemcpyDeviceToDevice, s));
    if (cfg) {
        if (fake_content != w.h_fc) ST_CUDA(cudaMemcpyAsync(w.h_fc, fake_content, (size_t)d.n_mel * 4, cudaMemcpyDeviceToDevice, s));
        if (fake_speaker != w.h_fs) ST_CUDA(cudaMemcpyAsync(w.h_fs, fake_speaker, (size_t)d.gin * 4, cudaMemcpyDeviceToDevice, s));
    }
    std::string key((const char*)t_span_host, sizeof(float) * (n_steps + 1));
    char meta[160];
    unsigned cfg_bits;
    memcpy(&cfg_bits, &cfg_strength, sizeof cfg_bits);
    snprintf(meta, sizeof meta, "|%d,%d,%d,%d,%d,%d,%08x,%p", B, T, cfg, method, n_steps, h->engine, cfg_bits, h->ws_ptr);
    key += meta;
    CfmModel::GraphEntry* ge = nullptr;
    for (auto& g : m->graphs) if (g.key == key) { ge = &g; break; }
    if (!ge) {
        bool seen = false;
        for (auto& k : m->graph_seen) if (k == key) { seen = true; break; }
        if (!seen) {                   // first occurrence: plain enqueue (module loading / attribute calls stay out of capture)
            if (m->graph_seen.size() >= 32) m->graph_seen.clear();
            m->graph_seen.push_back(key);
            return solve_impl(h, *m, w, z_inout, mu, mask, c, fake_content, fake_speaker, cfg_strength, t_span_host, n_steps, method, B, T, cfg, s);
        }
        const int64_t l0 = h->launches;
        cudaGraph_t graph = nullptr;
        if (!m->cap_stream) ST_CUDA(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        ST_CUDA(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
        int rc = solve_impl(h, *m, w, w.h_z, w.h_mu, w.h_mask, w.h_c, cfg ? w.h_fc : nullptr, cfg ? w.h_fs : nullptr, cfg_strength,
                            t_span_host, n_steps, method, B, T, cfg, m->cap_stream);
        cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &graph);
        const int64_t captured = h->launches - l0;
        h->launches = l0;
        if (rc || ce != cudaSuccess || !graph) {
            if (graph) cudaGraphDestroy(graph);
            cudaGetLastError();
            m->graph_mode = 0;                         // do not retry: fall back to direct enqueue for this handle
            if (getenv("STABLETTS_B200_DEBUG"))
                fprintf(stderr, "[stabletts_b200] graph capture failed (%s / %s); falling back to direct enqueue\n",
                        cudaGetErrorString(ce), h->err.c_str());
            return solve_impl(h, *m, w, z_inout, mu, mask, c, fake_content, fake_speaker, cfg_strength, t_span_host, n_steps, method, B, T, cfg, s);
        }
        cudaGraphExec_t exec = nullptr;
        cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) { cudaGetLastError(); m->graph_mode = 0; return fail(h, std::string("cudaGraphInstantiate failed: ") + cudaGetErrorString(ie)); }
        if (m->graphs.size() >= 8) { cudaGraphExecDestroy(m->graphs.front().exec); m->graphs.erase(m->graphs.begin()); }
        m->graphs.push_back({key, exec, captured});
        ge = &m->graphs.back();
    }
    ST_CUDA(cudaGraphLaunch(ge->exec, s));
    h->launches += ge->launches;
    if (z_inout != w.h_z) ST_CUDA(cudaMemcpyAsync(z_inout, w.h_z, n * 4, cudaMemcpyDeviceToDevice, s));
    return 0;
}

// ---- adaptive embedded Runge–Kutta solvers: the reference's default `solver=None` -> torchdiffeq dopri5
// (models/flow_matching.py:54) and the other adaptive strings webui.py:110 offers (bosh3, fehlberg2, adaptive_heun).
// torchdiffeq is absent and unpinned, so this follows its PUBLISHED algorithm (oracle/adaptive_ref.py restates the same
// and is what the tests compare against): one generic stepper over a Butcher tableau (alpha, beta, c_sol, c_error,
// c_mid, order) — stage k_{i+1} = f(t_i, y + dt sum_j beta_ij k_j), t_i = t1 exactly when alpha_i = 1; the solution is
// the last stage input when c_sol equals the last beta row (Dormand–Prince), else y + dt sum c_sol_j k_j; the LAST
// stage derivative is carried over as the next step's f0 for every tableau (what torchdiffeq's rk_common does, also
// for the tableaux that are not strictly FSAL) — RMS mixed error norm over all elements, I-controller (safety 0.9,
// factor in [0.2, 10], exponent 1/order), Hairer's initial step, evaluation at t_end through the 4th-order Hermite
// interpolant fitted to (y0, y1, y_mid, f0, f1).  Like torchdiffeq on a GPU, accept/reject needs ONE host-visible
// scalar per step (8 bytes, pinned).
namespace {
struct AdTab { int S, order; double alpha[6], beta[6][6], csol[7], cerr[7], cmid[7]; bool sol_is_last_stage; };

AdTab adaptive_tableau(int method) {
    AdTab t{};
    if (method == ST_ADAPT_BOSH3) {            // Bogacki–Shampine 3(2)
        t.S = 3; t.order = 3;
        const double al[3] = {1. / 2, 3. / 4, 1.};
        const double be[3][3] = {{1. / 2}, {0., 3. / 4}, {2. / 9, 1. / 3, 4. / 9}};
        const double cs[4] = {2. / 9, 1. / 3, 4. / 9, 0.};
        const double ce[4] = {2. / 9 - 7. / 24, 1. / 3 - 1. / 4, 4. / 9 - 1. / 3, -1. / 8};
        const double cm[4] = {0., 0.5, 0., 0.};
        for (int i = 0; i < 3; ++i) { t.alpha[i] = al[i]; for (int j = 0; j < 3; ++j) t.beta[i][j] = be[i][j]; }
        for (int i = 0; i < 4; ++i) { t.csol[i] = cs[i]; t.cerr[i] = ce[i]; t.cmid[i] = cm[i]; }
        t.sol_is_last_stage = true;
    } else if (method == ST_ADAPT_FEHLBERG2) { // Fehlberg 2(1)
        t.S = 2; t.order = 2;
        t.alpha[0] = 0.5; t.alpha[1] = 1.0;
        t.beta[0][0] = 0.5; t.beta[1][0] = 1. / 256; t.beta[1][1] = 255. / 256;
        t.csol[0] = 1. / 512; t.csol[1] = 255. / 256; t.csol[2] = 1. / 512;
        t.cerr[0] = -1. / 512; t.cerr[1] = 0.; t.cerr[2] = 1. / 512;
        t.cmid[0] = 0.; t.cmid[1] = 0.5; t.cmid[2] = 0.;
        t.sol_is_last_stage = false;
    } else if (method == ST_ADAPT_HEUN) {      // Heun–Euler 2(1)
        t.S = 1; t.order = 2;
        t.alpha[0] = 1.0; t.beta[0][0] = 1.0;
        t.csol[0] = 0.5; t.csol[1] = 0.5;
        t.cerr[0] = 0.5; t.cerr[1] = -0.5;
        t.cmid[0] = 0.5; t.cmid[1] = 0.;
        t.sol_is_last_stage = false;
    } else {                                   // Dormand–Prince 5(4), Shampine's embedded weights
        t.S = 6; t.order = 5;
        const double al[6] = {1. / 5, 3. / 10, 4. / 5, 8. / 9, 1.0, 1.0};
        const double be[6][6] = {{1. / 5}, {3. / 40, 9. / 40}, {44. / 45, -56. / 15, 32. / 9},
                                 {19372. / 6561, -25360. / 2187, 64448. / 6561, -212. / 729},
                                 {9017. / 3168, -355. / 33, 46732. / 5247, 49. / 176, -5103. / 18656},
                                 {35. / 384, 0, 500. / 1113, 125. / 192, -2187. / 6784, 11. / 84}};
        const double ce[7] = {35. / 384 - 1951. / 21600, 0, 500. / 1113 - 22642. / 50085, 125. / 192 - 451. / 720,
                              -2187. / 6784 + 12231. / 42400, 11. / 84 - 649. / 6300, -1. / 60};
        const double cm[7] = {6025192743. / 30085553152. / 2, 0, 51252292925. / 65400821598. / 2, -2691868925. / 45128329728. / 2,
                              187940372067. / 1594534317056. / 2, -1776094331. / 19743644256. / 2, 11237099. / 235043384. / 2};
        for (int i = 0; i < 6; ++i) { t.alpha[i] = al[i]; t.csol[i] = be[5][i]; for (int j = 0; j < 6; ++j) t.beta[i][j] = be[i][j]; }
        for (int i = 0; i < 7; ++i) { t.cerr[i] = ce[i]; t.cmid[i] = cm[i]; }
        t.sol_is_last_stage = true;
    }
    return t;
}
}  // namespace

int st_solve_adaptive_ex(st_handle* h, int method, float* z_inout, const float* mu, const float* mask, const float* c,
                         const float* fake_content, const float* fake_speaker, float cfg_strength, double t_start, double t_end,
                         double rtol, double atol, int max_steps, int B, int T, void* stream, int64_t* stats) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = model_of<CfmModel>(h, "CFM estimator");
    if (!m || check_common(h, B, T)) return 1;
    if (!z_inout || !mu || !mask || !c) return fail(h, "st_solve_adaptive: null pointer");
    if (method < ST_ADAPT_DOPRI5 || method > ST_ADAPT_HEUN) return fail(h, "st_solve_adaptive: unknown adaptive method");
    if (!(t_end > t_start) || rtol <= 0 || atol <= 0 || max_steps <= 0) return fail(h, "st_solve_adaptive: bad tolerances / interval");
    const int cfg = (fake_content && fake_speaker) ? 1 : 0;
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, cfg)) return 1;
    if (!m->pinned) ST_CUDA(cudaMallocHost((void**)&m->pinned, 16));
    const st_dims& d = m->d;
    const long numel = (long)B * T * d.n_mel;
    const AdTab tb = adaptive_tableau(method);
    const int S = tb.S;
    int64_t nfe = 0, n_acc = 0, n_rej = 0;
    // The step-size controller compares an embedded error estimate with rtol = atol = 1e-5: the two-pass FFN mode's
    // evaluation noise (~2e-4 relative) would feed straight into that estimate, so adaptive solves evaluate the vector
    // field with three passes everywhere, whatever the handle's precision mode (restored on every return path).
    struct PrecisionGuard {
        st_handle* h; int saved;
        explicit PrecisionGuard(st_handle* h_) : h(h_), saved(h_->precision) { h->precision = ST_PRECISION_BF16X3; }
        ~PrecisionGuard() { h->precision = saved; }
    } precision_guard(h);

    if (precompute_cond(h, *m, w, mu, mask, c, fake_content, fake_speaker, s)) return 1;
    // state buffers (token-major): y, y1 and S+1 stage derivatives rotate through Kst[]
    float* y = w.xt.f32; float* y1 = w.Kst[7]; float* ymid = w.Kst[8]; float* ysave = w.Kst[9];
    float* k[7]; for (int i = 0; i < 7; ++i) k[i] = w.Kst[i];
    ST_LAUNCH(launch_bct_to_btc(z_inout, y, nullptr, nullptr, B, d.n_mel, T, nullptr, s));

    auto feval = [&](double t, const float* yin, float* kout) -> int {        // kout = f(t, yin) (CFG-combined)
        TArr ta; ta.v[0] = (float)t;
        h->launches++;
        time_embed_val_kernel<<<(d.hidden / 2 + 127) / 128, 128, 0, s>>>(ta, 1, d.hidden, w.temb);
        if (cudaGetLastError() != cudaSuccess) return fail(h, "time embedding launch failed");
        if (precompute_film(h, *m, w, 1, s)) return 1;
        Act xin = w.xt; xin.f32 = const_cast<float*>(yin);
        if (h->engine == ST_ENGINE_TCGEN05) {
            if (launch_split(yin, w.xs.hi, w.xs.lo, numel, s) != cudaSuccess) return fail(h, "split failed");
            h->launches++;
            xin.hi = w.xs.hi; xin.lo = w.xs.lo;
        }
        if (estimator_eval(h, *m, w, xin, mask, w.film, 0, s)) return 1;
        if (launch_cfg_combine(w.V.f32, kout, B, (long)T * d.n_mel, cfg, cfg_strength, s) != cudaSuccess) return fail(h, "cfg combine failed");
        h->launches++; ++nfe;
        return 0;
    };
    auto norm = [&](const float* const* K, const float* coef, int n, const float* u, const float* v, double* out) -> int {
        if (launch_scaled_sumsq(K, coef, n, u, v, (float)atol, (float)rtol, numel, w.dscal, s) != cudaSuccess) return fail(h, "norm launch failed");
        h->launches++;
        if (cudaMemcpyAsync(m->pinned, w.dscal, sizeof(double), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
            cudaStreamSynchronize(s) != cudaSuccess) return fail(h, "norm read-back failed");
        *out = std::sqrt(m->pinned[0] / (double)numel);
        return 0;
    };
    // dst = base + dt * sum_j w[j] k[j] over the non-zero weights (j < n)
    auto combine = [&](float* dst, const float* base, const double* wts, int n, double dt) -> int {
        float coef[7]; const float* Ks[7]; int m = 0;
        for (int j = 0; j < n; ++j) if (wts[j] != 0.0) { coef[m] = (float)(dt * wts[j]); Ks[m] = k[j]; ++m; }
        if (m > 6) return fail(h, "internal: too many terms in a stage combination");
        ST_LAUNCH(launch_lincomb(dst, base, Ks, coef, m, numel, s));
        return 0;
    };

    double t0 = t_start;
    if (feval(t0, y, k[0])) return 1;
    double dt;
    {   // Hairer's initial step; torchdiffeq passes order - 1, so the exponent is 1 / order
        double d0, d1, d2;
        const float one = 1.f; const float* Ky[1] = {y}; const float* Kf[1] = {k[0]};
        if (norm(Ky, &one, 1, y, y, &d0) || norm(Kf, &one, 1, y, y, &d1)) return 1;
        const double h0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
        const float c1 = (float)h0; const float* K1[1] = {k[0]};
        ST_LAUNCH(launch_lincomb(y1, y, K1, &c1, 1, numel, s));
        if (feval(t0 + h0, y1, k[1])) return 1;
        const float pm[2] = {1.f, -1.f}; const float* Kd[2] = {k[1], k[0]};
        if (norm(Kd, pm, 2, y, y, &d2)) return 1;
        d2 /= h0;
        const double h1 = (d1 <= 1e-15 && d2 <= 1e-15) ? std::max(1e-6, h0 * 1e-3) : std::pow(0.01 / std::max(d1, d2), 1.0 / tb.order);
        dt = std::min(100 * h0, h1);
    }
    double ia_t0 = t0, ia_t1 = t0, ia_dt = 0;      // interval of the last accepted step (dense output)
    while (true) {
        if (n_acc + n_rej >= max_steps) return fail(h, "st_solve_adaptive: max_steps exceeded");
        const double t1 = t0 + dt;
        for (int i = 0; i < S; ++i) {
            // the last stage input IS the solution when c_sol equals the last beta row (Dormand–Prince, Bogacki–Shampine)
            float* dst = (i == S - 1 && tb.sol_is_last_stage) ? y1 : w.ytmp.f32;
            if (combine(dst, y, tb.beta[i], i + 1, dt)) return 1;
            if (feval(tb.alpha[i] == 1.0 ? t1 : t0 + tb.alpha[i] * dt, dst, k[i + 1])) return 1;
        }
        if (!tb.sol_is_last_stage && combine(y1, y, tb.csol, S + 1, dt)) return 1;
        double ratio;
        {
            float coef[7]; const float* Ks[7]; int n = 0;
            for (int j = 0; j <= S; ++j) if (tb.cerr[j] != 0.0) { coef[n] = (float)(dt * tb.cerr[j]); Ks[n] = k[j]; ++n; }
            if (norm(Ks, coef, n, y, y1, &ratio)) return 1;
        }
        const bool accept = ratio <= 1.0;
        double factor;
        if (ratio == 0.0) factor = 10.0;
        else factor = std::min(10.0, std::max(0.9 / std::pow(ratio, 1.0 / tb.order), ratio < 1.0 ? 1.0 : 0.2));
        if (accept) {
            ++n_acc;
            if (combine(ymid, y, tb.cmid, S + 1, dt)) return 1;      // y_mid for the dense output
            // keep (y_a = y, y_b = y1, f_a = k0, f_b = k_S) alive for the interpolant; advance by pointer rotation
            ia_t0 = t0; ia_t1 = t1; ia_dt = dt;
            std::swap(y, ysave);        // ysave now holds y_a ... (y pointer will be replaced below)
            std::swap(y, y1);           // y = y_b (new state); y1 = old ysave buffer (free)
            std::swap(k[0], k[S]);      // f0 <- last stage derivative; k[S] now holds f_a
            t0 = t1;
        } else {
            ++n_rej;
        }
        dt *= factor;
        if (accept && t0 >= t_end) break;
    }
    {   // 4th-order dense output at t_end on the last accepted interval (y_a = ysave, y_b = y, f_a = k[S], f_b = k[0])
        const double hh = ia_dt, x = (t_end - ia_t0) / (ia_t1 - ia_t0);
        const double x2 = x * x, x3 = x2 * x, x4 = x3 * x;
        // out = ya + x d + x^2 c + x^3 b + x^4 a with a,b,c,d linear in (ya, yb, ym, fa, fb)
        const double cya = 1.0 - 11 * x2 + 18 * x3 - 8 * x4;
        const double cyb = -5 * x2 + 14 * x3 - 8 * x4;
        const double cym = 16 * x2 - 32 * x3 + 16 * x4;
        const double cfa = hh * (x - 4 * x2 + 5 * x3 - 2 * x4);
        const double cfb = hh * (x2 - 3 * x3 + 2 * x4);
        float coef[5] = {(float)(cya - 1.0), (float)cyb, (float)cym, (float)cfa, (float)cfb};
        const float* Ks[5] = {ysave, y, ymid, k[S], k[0]};
        ST_LAUNCH(launch_lincomb(w.ytmp.f32, ysave, Ks, coef, 5, numel, s));
    }
    ST_LAUNCH(launch_btc_to_bct(w.ytmp.f32, z_inout, B, d.n_mel, T, s));
    if (stats) { stats[0] = n_acc; stats[1] = n_rej; stats[2] = nfe; }
    return 0;
}

int st_solve_adaptive(st_handle* h, float* z_inout, const float* mu, const float* mask, const float* c,
                      const float* fake_content, const float* fake_speaker, float cfg_strength, double t_start, double t_end,
                      double rtol, double atol, int max_steps, int B, int T, void* stream, int64_t* stats) {
    return st_solve_adaptive_ex(h, ST_ADAPT_DOPRI5, z_inout, mu, mask, c, fake_content, fake_speaker, cfg_strength, t_start, t_end,
                                rtol, atol, max_steps, B, T, stream, stats);
}

int st_solve_host_io(st_handle* h, const float* z_in_host, float* out_host, const float* mu_host, const float* mask_host, const float* c_host,
                  const float* fake_content_host, const float* fake_speaker_host, float cfg_strength,
                  const float* t_span_host, int n_steps, int method, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = model_of<CfmModel>(h, "CFM estimator");
    if (!m || check_common(h, B, T)) return 1;
    if (!z_in_host || !out_host || !mu_host || !mask_host || !c_host) return fail(h, "st_solve_host: null pointer");
    const int cfg = (fake_content_host && fake_speaker_host) ? 1 : 0;
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, cfg)) return 1;
    const st_dims& d = m->d;
    const size_t n = (size_t)B * T * d.n_mel;
    // Host buffers that are not page-locked are staged through a pinned buffer the handle owns (a pageable
    // cudaMemcpyAsync is staged by the driver in small chunks and serialises with the stream); pinned callers
    // (cudaHostAlloc / torch pin_memory) are copied from directly.
    auto is_pinned = [](const void* p) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return at.type == cudaMemoryTypeHost;
    };
    const size_t sizes[6] = {n * 4, n * 4, (size_t)B * T * 4, (size_t)B * d.gin * 4, (size_t)d.n_mel * 4, (size_t)d.gin * 4};
    const void* src[6] = {z_in_host, mu_host, mask_host, c_host, cfg ? fake_content_host : nullptr, cfg ? fake_speaker_host : nullptr};
    void* dst[6] = {w.h_z, w.h_mu, w.h_mask, w.h_c, w.h_fc, w.h_fs};
    size_t need = 0;
    bool pinned_in[6];
    for (int i = 0; i < 6; ++i) { pinned_in[i] = !src[i] || is_pinned(src[i]); if (!pinned_in[i]) need += (sizes[i] + 255) & ~size_t(255); }
    const bool out_pinned = is_pinned(out_host);
    size_t out_off = 0;
    if (!out_pinned) { out_off = need; need += (n * 4 + 255) & ~size_t(255); }     // the result is staged too
    if (need > m->pin_bytes) {
        if (m->pin_buf) { ST_CUDA(cudaStreamSynchronize(s)); cudaFreeHost(m->pin_buf); m->pin_buf = nullptr; m->pin_bytes = 0; }
        ST_CUDA(cudaMallocHost((void**)&m->pin_buf, need));
        m->pin_bytes = need;
    }
    size_t off = 0;
    for (int i = 0; i < 6; ++i) {
        if (!src[i]) continue;
        const void* from = src[i];
        if (!pinned_in[i]) {
            memcpy(m->pin_buf + off, src[i], sizes[i]);
            from = m->pin_buf + off;
            off += (sizes[i] + 255) & ~size_t(255);
        }
        ST_CUDA(cudaMemcpyAsync(dst[i], from, sizes[i], cudaMemcpyHostToDevice, s));
    }
    if (st_solve(h, w.h_z, w.h_mu, w.h_mask, w.h_c, cfg ? w.h_fc : nullptr, cfg ? w.h_fs : nullptr, cfg_strength, t_span_host,
                 n_steps, method, B, T, stream))
        return 1;
    ST_CUDA(cudaMemcpyAsync(out_pinned ? (void*)out_host : (void*)(m->pin_buf + out_off), w.h_z, n * 4, cudaMemcpyDeviceToHost, s));
    ST_CUDA(cudaStreamSynchronize(s));
    if (!out_pinned) memcpy(out_host, m->pin_buf + out_off, n * 4);
    return 0;
}

int st_solve_host(st_handle* h, float* z_inout_host, const float* mu_host, const float* mask_host, const float* c_host,
                  const float* fake_content_host, const float* fake_speaker_host, float cfg_strength,
                  const float* t_span_host, int n_steps, int method, int B, int T, void* stream) {
    return st_solve_host_io(h, z_inout_host, z_inout_host, mu_host, mask_host, c_host, fake_content_host, fake_speaker_host, cfg_strength,
                            t_span_host, n_steps, method, B, T, stream);
}

// ---- caller-side glue of the path (SURVEY.md §8 row f1); stateless: errors go to st_last_error(NULL) ----
int st_align_lengths(const float* logw, const float* x_mask, float length_scale, int B, int Tx, float* cum, int64_t* y_lengths,
                     void* stream) {
    st_handle* h = nullptr;
    if (!logw || !x_mask || !cum || !y_lengths || B < 0 || Tx <= 0) return fail(h, "st_align_lengths: bad argument");
    ST_CUDA(launch_align_lengths(logw, x_mask, length_scale, B, Tx, cum, (long long*)y_lengths, (cudaStream_t)stream));
    return 0;
}

int st_align_expand(const float* mu_x, const float* x_mask, const float* cum, const int64_t* y_lengths, int B, int M, int Tx,
                    int Ty, float* mu_y, float* y_mask, float* attn, void* stream) {
    st_handle* h = nullptr;
    if (!mu_x || !x_mask || !cum || !y_lengths || !mu_y || !y_mask || B < 0 || M <= 0 || Tx <= 0 || Ty < 0)
        return fail(h, "st_align_expand: bad argument");
    ST_CUDA(launch_align_expand(mu_x, x_mask, cum, (const long long*)y_lengths, B, M, Tx, Ty, mu_y, y_mask, attn, (cudaStream_t)stream));
    return 0;
}

// ---- monotonic alignment search of the training forward (SURVEY.md §8 row f8); stateless like st_align_* ----
size_t st_mas_workspace_bytes(int B, int Ty, int Tx) {
    return B <= 0 || Ty <= 0 || Tx <= 0 ? 0 : mas_workspace_bytes(B, Ty, Tx);
}

int st_mas_scores(const float* y, const float* mu_x, float* neg_cent, int B, int D, int Ty, int Tx, void* stream) {
    st_handle* h = nullptr;
    if (!y || !mu_x || !neg_cent || B < 0 || D <= 0 || Ty < 0 || Tx < 0) return fail(h, "st_mas_scores: bad argument");
    ST_CUDA(launch_mas_scores(y, mu_x, neg_cent, B, D, Ty, Tx, (cudaStream_t)stream));
    return 0;
}

int st_maximum_path(const float* neg_cent, const float* mask, const int64_t* x_lengths, const int64_t* y_lengths, float* path,
                    float* dur, float* cum, void* ws, size_t ws_bytes, int B, int Ty, int Tx, void* stream) {
    st_handle* h = nullptr;
    if (!neg_cent || B < 0 || Ty < 0 || Tx < 0) return fail(h, "st_maximum_path: bad argument");
    const bool by_mask = mask && !x_lengths && !y_lengths, by_lengths = !mask && x_lengths && y_lengths;
    if (!by_mask && !by_lengths)
        return fail(h, "st_maximum_path: pass either mask or both x_lengths and y_lengths");
    if (Tx > mas_max_tx())
        return fail(h, "st_maximum_path: Tx = " + std::to_string(Tx) + " exceeds the " + std::to_string(mas_max_tx()) +
                           " tokens whose score rows fit in shared memory");
    if (B == 0 || Ty == 0 || Tx == 0) return 0;
    if (!ws || ws_bytes < mas_workspace_bytes(B, Ty, Tx))
        return fail(h, "st_maximum_path: workspace smaller than st_mas_workspace_bytes(B, Ty, Tx)");
    ST_CUDA(launch_maximum_path(neg_cent, mask, (const long long*)x_lengths, (const long long*)y_lengths, path, dur, cum, ws, B, Ty,
                                Tx, (cudaStream_t)stream));
    return 0;
}

int st_mas_losses(const float* y, const float* mu_y, const float* y_mask, const float* logw, const float* x_mask, const float* dur,
                  const int64_t* x_lengths, void* ws, size_t ws_bytes, int B, int M, int Ty, int Tx, float* prior_loss,
                  float* dur_loss, void* stream) {
    st_handle* h = nullptr;
    if (!y || !mu_y || !y_mask || !logw || !x_mask || !dur || !x_lengths || !prior_loss || !dur_loss || B <= 0 || M <= 0 || Ty <= 0 ||
        Tx <= 0)
        return fail(h, "st_mas_losses: bad argument");
    if (!ws || ws_bytes < mas_workspace_bytes(B, Ty, Tx))
        return fail(h, "st_mas_losses: workspace smaller than st_mas_workspace_bytes(B, Ty, Tx)");
    ST_CUDA(launch_mas_losses(y, mu_y, y_mask, logw, x_mask, dur, (const long long*)x_lengths, ws, B, M, Ty, Tx, prior_loss, dur_loss,
                              (cudaStream_t)stream));
    return 0;
}

// ---- kernel-level test hooks ------------------------------------------------------------------------
int st_test_conv(st_handle* h, const float* x, const float* wgt, const float* bias, float* out, int B, int Cin, int Cout,
                 int T, int k, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t nx = (size_t)B * T * Cin, nw = (size_t)k * Cout * Cin, no = (size_t)B * T * Cout;
    float *xt, *wp, *ot; bf16 *xh, *xl, *wh, *wl;
    ST_CUDA(cudaMalloc(&xt, nx * 4)); ST_CUDA(cudaMalloc(&wp, nw * 4)); ST_CUDA(cudaMalloc(&ot, no * 4));
    ST_CUDA(cudaMalloc(&xh, nx * 2)); ST_CUDA(cudaMalloc(&xl, nx * 2)); ST_CUDA(cudaMalloc(&wh, nw * 2)); ST_CUDA(cudaMalloc(&wl, nw * 2));
    int rc = 0;
    do {
        if (launch_bct_to_btc(x, xt, xh, xl, B, Cin, T, nullptr, s) != cudaSuccess) { rc = fail(h, "transpose failed"); break; }
        long total = (long)k * Cout * Cin;
        pack_conv_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(wgt, wp, Cout, Cin, k, Cout, 0, 0, Cin);
        if (launch_split(wp, wh, wl, (long)nw, s) != cudaSuccess) { rc = fail(h, "split failed"); break; }
        GemmArgs g;
        g.BB = B; g.T = T; g.a_bmod = B; g.B = B; g.resid_clamp = B - 1; g.flags = bias ? EPI_BIAS : 0;
        GemmW w; w.f32 = wp; w.hi = wh; w.lo = wl; w.bias = const_cast<float*>(bias); w.taps = k; w.N = Cout; w.K = Cin;
        Act a; a.C = Cin; a.f32 = xt; a.hi = tc ? xh : nullptr; a.lo = tc ? xl : nullptr;
        Act o; o.C = Cout; o.f32 = ot;
        if (run_gemm(h, g, w, &a, nullptr, o, s)) { rc = 1; break; }
        if (launch_btc_to_bct(ot, out, B, Cout, T, s) != cudaSuccess) { rc = fail(h, "transpose failed"); break; }
    } while (0);
    cudaStreamSynchronize(s);
    cudaError_t e = cudaGetLastError();
    if (!rc && e != cudaSuccess) rc = fail(h, std::string("st_test_conv: ") + cudaGetErrorString(e));
    cudaFree(xt); cudaFree(wp); cudaFree(ot); cudaFree(xh); cudaFree(xl); cudaFree(wh); cudaFree(wl);
    return rc;
}

int st_test_gemm(st_handle* h, const float* A, const float* W, const float* bias, float* out, int R, int K, int N, int silu,
                 void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const size_t na = (size_t)R * K, nw = (size_t)N * K;
    bf16 *ah, *al, *wh, *wl;
    ST_CUDA(cudaMalloc(&ah, na * 2)); ST_CUDA(cudaMalloc(&al, na * 2)); ST_CUDA(cudaMalloc(&wh, nw * 2)); ST_CUDA(cudaMalloc(&wl, nw * 2));
    int rc = 0;
    do {
        if (launch_split(A, ah, al, (long)na, s) != cudaSuccess || launch_split(W, wh, wl, (long)nw, s) != cudaSuccess) {
            rc = fail(h, "split failed"); break;
        }
        GemmArgs g;   // one "utterance" of R frames
        g.BB = 1; g.T = R; g.a_bmod = 1; g.B = 1; g.resid_clamp = 0; g.flags = (bias ? EPI_BIAS : 0) | (silu ? EPI_SILU : 0);
        GemmW w; w.f32 = const_cast<float*>(W); w.hi = wh; w.lo = wl; w.bias = const_cast<float*>(bias); w.taps = 1; w.N = N; w.K = K;
        Act a; a.C = K; a.f32 = const_cast<float*>(A); a.hi = tc ? ah : nullptr; a.lo = tc ? al : nullptr;
        Act o; o.C = N; o.f32 = out;
        if (run_gemm(h, g, w, &a, nullptr, o, s)) { rc = 1; break; }
    } while (0);
    cudaStreamSynchronize(s);
    cudaError_t e = cudaGetLastError();
    if (!rc && e != cudaSuccess) rc = fail(h, std::string("st_test_gemm: ") + cudaGetErrorString(e));
    cudaFree(ah); cudaFree(al); cudaFree(wh); cudaFree(wl);
    return rc;
}

static_assert(ST_TEST_EPI_BIAS == EPI_BIAS && ST_TEST_EPI_SILU == EPI_SILU && ST_TEST_EPI_FILM == EPI_FILM &&
              ST_TEST_EPI_MASK == EPI_MASK && ST_TEST_EPI_GATE == EPI_GATE && ST_TEST_EPI_RESID == EPI_RESID &&
              ST_TEST_EPI_ROPE == EPI_ROPE && ST_TEST_EPI_GELU == EPI_GELU && ST_TEST_EPI_SILU_OUT == EPI_SILU_OUT &&
              ST_TEST_EPI_MISH == EPI_MISH,
              "st_test_gemm_desc::flags are the EPI_* bits");

// device scratch of a test hook, freed on every exit (cudaFree waits for the work that uses it)
struct TestBufs {
    std::vector<void*> p;
    void* take(size_t bytes) {
        void* q = nullptr;
        if (cudaMalloc(&q, std::max<size_t>(bytes, 4)) != cudaSuccess) return nullptr;
        p.push_back(q);
        return q;
    }
    ~TestBufs() { for (void* q : p) cudaFree(q); }
};

static const char* test_gemm_desc_error(const st_test_gemm_desc& d) {
    if (d.B < 1 || d.BB < 1 || d.T < 1 || d.a_bmod < 1 || d.a_bmod > d.BB) return "B, BB, T >= 1 and 1 <= a_bmod <= BB";
    if ((d.n_src != 1 && d.n_src != 2) || d.C0 < 1 || (d.n_src == 2 ? d.C1 < 1 : d.C1 != 0)) return "n_src 1 (C1 = 0) or 2, channels >= 1";
    if (!d.A0 || (d.n_src == 2 && !d.A1) || !d.W) return "A0 [, A1] and W are required";
    if (d.N < 1 || d.taps < 1 || d.dil < 1) return "N, taps, dil >= 1";
    if (d.flags & ~EPI_ALL) return "unknown flag";
    if (d.c_clamp < 0 || d.resid_clamp < 0 || d.film_bstride < 0 || d.gate_bstride < 0 || d.ada_bstride < 0 || d.film2_bstride < 0)
        return "clamps and batch strides must be >= 0";
    if ((d.flags & EPI_BIAS) && !d.bias) return "EPI_BIAS needs bias";
    if ((d.flags & EPI_MASK) && !d.mask) return "EPI_MASK needs mask";
    if ((d.flags & EPI_FILM) && !d.film) return "EPI_FILM needs film";
    if (((d.flags & EPI_FILM) || d.film2) && d.film_H < d.N) return "film_H (the beta offset) must be >= N";
    if ((d.flags & EPI_GATE) && !d.gate) return "EPI_GATE needs gate";
    if ((d.flags & EPI_RESID) && !d.resid) return "EPI_RESID needs resid";
    if ((d.flags & EPI_ROPE) && (d.rope_H < 64 || d.rope_H % 64 || 2 * d.rope_H > d.N)) return "EPI_ROPE needs rope_H % 64 == 0, 2 rope_H <= N";
    if (d.ln && (!d.ln_shift || !d.ln_scale || !d.u_hi || (!d.u16 && !d.u_lo))) return "ln needs ln_shift, ln_scale and the u planes";
    if (!d.ln && (d.u_hi || d.u_lo || d.u16 || d.film2 || d.ln_mask_out)) return "u planes, u16, film2 and ln_mask_out belong to ln";
    if (d.film2 && !d.out2_f32) return "film2 needs out2_f32";
    if (d.out2_f32 && !d.film2 && !(d.flags & EPI_SILU_OUT)) return "out2_f32 is written by EPI_SILU_OUT or film2 only";
    if (d.out16 && !d.out_hi) return "out16 needs out_hi";
    if (d.out_hi && !d.out16 && !d.out_lo) return "out_hi needs out_lo (or out16)";
    if (!d.out_f32 && !d.out_hi && !d.out2_f32 && !d.u_hi) return "no output requested";
    if (d.ksplit < 0 || d.ksplit > 4 || d.num_sms < 0) return "ksplit in [0, 4], num_sms >= 0";
    return nullptr;
}

int st_test_gemm_ex(st_handle* h, const st_test_gemm_desc* dp, st_test_gemm_plan* plan, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_gemm_ex: null descriptor");
    const st_test_gemm_desc& d = *dp;
    if (const char* why = test_gemm_desc_error(d)) return fail(h, std::string("st_test_gemm_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const int Cs[2] = {d.C0, d.C1}, Ktot = d.C0 + d.C1;
    const size_t nw = (size_t)d.taps * d.N * Ktot;
    TestBufs bufs;
    auto take = [&](size_t bytes) { return bufs.take(bytes); };
    // W: (N, Ktot, taps) Conv1d layout -> packed [taps][N][Ktot], then its planes
    GemmW w; w.taps = d.taps; w.N = d.N; w.K = Ktot; w.bias = const_cast<float*>(d.bias);
    w.f32 = (float*)take(nw * 4); w.hi = (bf16*)take(nw * 2); w.lo = (bf16*)take(nw * 2);
    if (d.prec) { w.h_hi = (bf16*)take(nw * 2); w.h_lo = (bf16*)take(nw * 2); }
    if (!w.f32 || !w.hi || !w.lo || (d.prec && (!w.h_hi || !w.h_lo))) return fail(h, "st_test_gemm_ex: out of memory");
    ST_CUDA(launch_pack_conv(d.W, w.f32, d.N, Ktot, d.taps, d.N, 0, 0, Ktot, s));
    ST_CUDA(launch_split(w.f32, w.hi, w.lo, (long)nw, s));
    if (d.prec) ST_CUDA(launch_split_f16(w.f32, w.h_hi, w.h_lo, (long)nw, s));
    // A: fp32 for the SIMT engine; split-bf16 planes, or with prec ONE fp16 plane (the hi plane of the fp16 split)
    Act a[2];
    for (int i = 0; i < d.n_src; ++i) {
        const float* src = i ? d.A1 : d.A0;
        const size_t n = (size_t)d.a_bmod * d.T * Cs[i];
        a[i].C = Cs[i]; a[i].f32 = const_cast<float*>(src);
        if (!tc) continue;
        a[i].hi = (bf16*)take(n * 2); a[i].lo = (bf16*)take(n * 2);
        if (!a[i].hi || !a[i].lo) return fail(h, "st_test_gemm_ex: out of memory");
        ST_CUDA(d.prec ? launch_split_f16(src, a[i].hi, a[i].lo, (long)n, s) : launch_split(src, a[i].hi, a[i].lo, (long)n, s));
    }
    GemmArgs g;
    g.BB = d.BB; g.T = d.T; g.a_bmod = d.a_bmod; g.B = d.B; g.flags = d.flags; g.dil = d.dil;
    g.mask = d.mask; g.film = d.film; g.film_bstride = d.film_bstride; g.film_H = d.film_H;
    g.gate = d.gate; g.gate_bstride = d.gate_bstride; g.c_clamp = d.c_clamp; g.resid = d.resid; g.resid_clamp = d.resid_clamp;
    g.rope_H = d.rope_H;
    if (d.flags & EPI_ROPE) {
        float* cs = (float*)take((size_t)d.T * 32 * 4);
        if (!cs) return fail(h, "st_test_gemm_ex: out of memory");
        ST_CUDA(launch_rope_table(cs, d.T, 32, s));
        g.rope_cs = cs;
    }
    g.ln = d.ln; g.ln_mask_out = d.ln_mask_out; g.ln_shift = d.ln_shift; g.ln_scale = d.ln_scale; g.ada_bstride = d.ada_bstride;
    g.u_hi = (bf16*)d.u_hi; g.u_lo = (bf16*)d.u_lo; g.film2 = d.film2; g.film2_bstride = d.film2_bstride; g.out2_f32 = d.out2_f32;
    g.prec = d.prec; g.out16 = d.out16; g.u16 = d.u16;
    g.force_ksplit = d.ksplit;
    GemmPlan gp;
    g.plan = &gp;
    Act o; o.C = d.N; o.f32 = d.out_f32; o.hi = (bf16*)d.out_hi; o.lo = (bf16*)d.out_lo;
    // the split-K partial buffer is sized by the real SM count, before any override; a handle serves one caller at a time
    // (as every entry point assumes), so the override only has to be undone on every exit
    if (tc && ensure_part_buf(h)) return 1;
    struct SmsRestore {
        st_handle* h; int saved;
        ~SmsRestore() { h->num_sms = saved; }
    } restore{h, h->num_sms};
    if (d.num_sms > 0) h->num_sms = d.num_sms;
    int rc = run_gemm(h, g, w, &a[0], d.n_src == 2 ? &a[1] : nullptr, o, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (!rc && e != cudaSuccess) rc = fail(h, std::string("st_test_gemm_ex: ") + cudaGetErrorString(e));
    if (!rc && plan) {
        plan->engine = gp.engine; plan->bn = gp.bn; plan->mode = gp.mode; plan->prec = gp.prec; plan->ksplit = gp.ksplit; plan->grid = gp.grid;
    }
    return rc;
}

__global__ void fill_pattern_kernel(float* p, long n, uint32_t seed) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u + seed;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    p[i] = ((float)(x & 0xFFFF) / 32768.0f - 1.0f);
}

// Times `reps` launches of the selected engine's conv-GEMM on synthetic data (token-major operands are
// generated on the device): (B, T, Cin) x [k][Cout][Cin] -> (B, T, Cout).  epi 1: conv_2-style epilogue (bias, mask, gate,
// residual, fp32 + split outputs); 2: conv_1-style (bias, SiLU, mask, split output); 3: O-style (residual, mask, gate,
// fp32 output + fused LayerNorm / modulate); 0: bias-only split output.  prec = 1: the two-pass fp16 operands (one fp16 A
// plane, fp16 hi / lo weights) with fp16 output planes, as ST_PRECISION_FFN_FP16X2 runs the FFN convs.
int st_bench_conv(st_handle* h, int B, int Cin, int Cout, int T, int k, int epi, int prec, int reps, float* ms_out) {
    if (!h || !ms_out) return 1;
    ST_ENTER(h);
    cudaStream_t s = 0;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    if (prec && !tc) return fail(h, "st_bench_conv: the two-pass fp16 precision runs on the wgmma engine only");
    const size_t nx = (size_t)B * T * Cin, nw = (size_t)k * Cout * Cin, no = (size_t)B * T * Cout;
    float *xf, *wf, *of, *bias, *mask, *gate; bf16 *xh, *xl, *wh, *wl, *oh, *ol;
    ST_CUDA(cudaMalloc(&xf, nx * 4)); ST_CUDA(cudaMalloc(&wf, nw * 4)); ST_CUDA(cudaMalloc(&of, no * 4));
    ST_CUDA(cudaMalloc(&xh, nx * 2)); ST_CUDA(cudaMalloc(&xl, nx * 2)); ST_CUDA(cudaMalloc(&wh, nw * 2)); ST_CUDA(cudaMalloc(&wl, nw * 2));
    ST_CUDA(cudaMalloc(&oh, no * 2)); ST_CUDA(cudaMalloc(&ol, no * 2));
    ST_CUDA(cudaMalloc(&bias, Cout * 4)); ST_CUDA(cudaMalloc(&gate, (size_t)B * Cout * 4)); ST_CUDA(cudaMalloc(&mask, (size_t)B * T * 4));
    fill_pattern_kernel<<<(unsigned)((nx + 255) / 256), 256, 0, s>>>(xf, (long)nx, 1u);
    fill_pattern_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(wf, (long)nw, 2u);
    fill_pattern_kernel<<<(unsigned)((no + 255) / 256), 256, 0, s>>>(of, (long)no, 3u);
    fill_pattern_kernel<<<(Cout + 255) / 256, 256, 0, s>>>(bias, Cout, 4u);
    fill_pattern_kernel<<<(unsigned)(((size_t)B * Cout + 255) / 256), 256, 0, s>>>(gate, (long)B * Cout, 5u);
    ST_CUDA(cudaMemsetAsync(mask, 0x3f, (size_t)B * T * 4, s));       // 0.747 everywhere: a non-trivial multiplier
    int rc = 0;
    do {
        // prec: one fp16 A plane (xh) and fp16 hi / lo weight planes, 2-byte outputs as one fp16 plane (the FFN convs' mode)
        auto split = prec ? launch_split_f16 : launch_split;
        if (split(xf, xh, xl, (long)nx, s) != cudaSuccess || split(wf, wh, wl, (long)nw, s) != cudaSuccess) { rc = fail(h, "split failed"); break; }
        GemmArgs g;
        g.BB = B; g.T = T; g.a_bmod = B; g.B = B; g.resid_clamp = B - 1; g.c_clamp = B - 1; g.mask = mask;
        g.flags = (epi == 1 || epi == 3) ? (EPI_BIAS | EPI_MASK | EPI_GATE | EPI_RESID) : (epi == 2 ? (EPI_BIAS | EPI_SILU | EPI_MASK) : EPI_BIAS);
        g.gate = gate; g.gate_bstride = Cout; g.resid = of;
        if (epi == 3) {                // O-style: fp32 residual stream out + fused LayerNorm/modulate -> split-bf16 U
            g.ln = 1; g.ln_mask_out = 1; g.ln_shift = gate; g.ln_scale = gate; g.ada_bstride = Cout; g.u_hi = oh; g.u_lo = ol;
        }
        GemmW w; w.f32 = wf; w.hi = wh; w.lo = wl; w.bias = bias; w.taps = k; w.N = Cout; w.K = Cin;
        if (prec) { g.prec = 1; g.out16 = 1; g.u16 = 1; w.h_hi = wh; w.h_lo = wl; }
        Act a; a.C = Cin; a.f32 = xf; a.hi = tc ? xh : nullptr; a.lo = tc ? xl : nullptr;
        Act o; o.C = Cout; o.f32 = (epi == 1 || epi == 3) ? of : nullptr; o.hi = epi == 3 ? nullptr : oh; o.lo = epi == 3 ? nullptr : ol;
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int i = 0; i < 2 && !rc; ++i) rc = run_gemm(h, g, w, &a, nullptr, o, s);
        if (rc) break;
        cudaEventRecord(e0, s);
        for (int i = 0; i < reps && !rc; ++i) rc = run_gemm(h, g, w, &a, nullptr, o, s);
        cudaEventRecord(e1, s);
        cudaEventSynchronize(e1);
        float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1);
        *ms_out = ms / (reps > 0 ? reps : 1);
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    } while (0);
    cudaStreamSynchronize(s);
    cudaError_t e = cudaGetLastError();
    if (!rc && e != cudaSuccess) rc = fail(h, std::string("st_bench_conv: ") + cudaGetErrorString(e));
    cudaFree(xf); cudaFree(wf); cudaFree(of); cudaFree(xh); cudaFree(xl); cudaFree(wh); cudaFree(wl); cudaFree(oh); cudaFree(ol);
    cudaFree(bias); cudaFree(gate); cudaFree(mask);
    return rc;
}


static const char* test_attn_desc_error(const st_test_attn_desc& d, bool tc) {
    if (d.n_heads < 1 || d.n_heads > 65535 || d.H != 64 * d.n_heads) return "H must be 64 n_heads (n_heads >= 1)";
    if (d.B < 1 || d.T < 1 || d.BB < 1 || d.BB % d.B || d.BB > 65535) return "B, T >= 1 and BB a positive multiple of B (<= 65535)";
    if (!d.mask) return "mask is required";
    if (!d.out_f32 && !d.out_hi && !d.out_lo) return "no output requested";
    if (!d.out_hi != !d.out_lo) return "out_hi and out_lo go together";
    if (d.rope != 0 && d.rope != 1) return "rope is 0 or 1";
    if (tc && (!d.qkv_hi || !d.qkv_lo)) return "the wgmma engine needs the split planes qkv_hi and qkv_lo";
    if (tc && d.rope) return "the wgmma engine takes planes that are already RoPE'd: rope must be 0";
    if (!tc && !d.qkv) return "the SIMT engine needs the fp32 qkv";
    return nullptr;
}

int st_test_attention_ex(st_handle* h, const st_test_attn_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_attention_ex: null descriptor");
    const st_test_attn_desc& d = *dp;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    if (const char* why = test_attn_desc_error(d, tc)) return fail(h, std::string("st_test_attention_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    TestBufs bufs;
    int* kvlen = d.kvlen_out ? d.kvlen_out : (int*)bufs.take(sizeof(int) * d.B);
    int* prefix = d.prefix_out ? d.prefix_out : (int*)bufs.take(sizeof(int) * d.B);
    float* cs = d.rope ? (float*)bufs.take(sizeof(float) * d.T * 32) : nullptr;
    if (!kvlen || !prefix || (d.rope && !cs)) return fail(h, "st_test_attention_ex: out of memory");
    ST_CUDA(launch_mask_lengths(d.mask, kvlen, prefix, d.B, d.T, s));
    if (d.rope) ST_CUDA(launch_rope_table(cs, d.T, 32, s));
    AttnArgs a;
    a.qkv = d.qkv; a.qkv_hi = (const bf16*)d.qkv_hi; a.qkv_lo = (const bf16*)d.qkv_lo; a.rope_cs = cs;
    a.mask = d.mask; a.kvlen = kvlen; a.prefix = prefix;
    a.out_f32 = d.out_f32; a.out_hi = (bf16*)d.out_hi; a.out_lo = (bf16*)d.out_lo;
    a.BB = d.BB; a.B = d.B; a.T = d.T; a.H = d.H; a.n_heads = d.n_heads;
    cudaError_t e = tc ? launch_attention_tc(a, s) : launch_attention_simt(a, s);
    if (e != cudaSuccess)
        return fail(h, std::string("st_test_attention_ex: launch failed: ") + cudaGetErrorString(e) + (tc ? std::string(" / ") + attention_tc_last_error() : ""));
    e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, std::string("st_test_attention_ex: ") + cudaGetErrorString(e));
    return 0;
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

static const char* test_row_desc_error(const st_test_row_desc& d) {
    const bool planes = d.out_hi || d.out_lo;
    if (d.u16 && d.kind != ST_TEST_ROW_ADALN) return "u16 belongs to ADALN";
    if (d.u16 && d.out_lo) return "u16 writes one fp16 plane to out_hi: out_lo must be NULL";
    if (!d.u16 && !d.out_hi != !d.out_lo) return "out_hi and out_lo go together";
    switch (d.kind) {
    case ST_TEST_ROW_ADALN:
        if (d.C != 256) return "ADALN: H (C) must be 256, the one width film_ln_mod_kernel is instantiated for";
        if (d.B < 1 || d.BB < 1 || d.T < 1) return "ADALN: B, BB, T >= 1";
        if (!d.x || !d.mask || !d.shift || !d.scale) return "ADALN: x, mask, shift and scale are required";
        if (d.has_film != 0 && d.has_film != 1) return "ADALN: has_film is 0 or 1";
        if (d.has_film && (!d.film || !d.xout)) return "ADALN: has_film needs film and xout";
        if (!d.has_film && (d.film || d.xout)) return "ADALN: film and xout belong to has_film";
        if (d.c_clamp < 0 || d.film_bstride < 0 || d.ada_bstride < 0) return "ADALN: c_clamp and batch strides must be >= 0";
        if (d.u16 && !d.out_hi) return "ADALN: u16 needs out_hi";
        if (!d.out_f32 && !d.out_hi) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.xout) || !aligned16(d.film) || !aligned16(d.shift) || !aligned16(d.scale) ||
            !aligned16(d.out_f32) || !aligned16(d.out_hi) || !aligned16(d.out_lo) || d.film_bstride % 4 || d.ada_bstride % 4)
            return "ADALN: buffers must be 16-byte aligned and batch strides multiples of 4";
        return nullptr;
    case ST_TEST_ROW_DWCONV_LN:
        if (d.C != 128 && d.C != 256 && d.C != 384 && d.C != 512 && d.C != 768 && d.C != 1024)
            return "DWCONV_LN: C must be 128, 256, 384, 512, 768 or 1024 (the instantiated widths)";
        if (d.B < 1 || d.T < 1) return "DWCONV_LN: B, T >= 1";
        if (!d.x || !d.ln_w || !d.ln_b || (d.w && !d.bias)) return "DWCONV_LN: x, ln_w, ln_b (and bias with w) are required";
        if (!(d.eps > 0.f)) return "DWCONV_LN: eps must be positive";
        if (!d.out_f32 && !planes) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.bias) || !aligned16(d.ln_w) || !aligned16(d.ln_b) || !aligned16(d.out_f32) ||
            !aligned16(d.out_hi) || !aligned16(d.out_lo))
            return "DWCONV_LN: buffers must be 16-byte aligned";
        return nullptr;
    case ST_TEST_ROW_SPECTRUM:
        if (d.B < 1 || d.T < 1) return "SPECTRUM: B, T >= 1";
        if (!d.x) return "SPECTRUM: x is required";
        if (d.K < 1 || d.Kp < d.K || d.Nh < d.Kp + d.K || d.K2 < 2 * d.K || d.K2 % 2)
            return "SPECTRUM: needs 1 <= K <= Kp, Kp + K <= Nh, K2 even and K <= K2/2";
        if (!d.out_f32 && !planes) return "no output requested";
        return nullptr;
    case ST_TEST_ROW_IDFT_BASIS:
        if (d.n_fft < 2 || d.n_fft % 2) return "IDFT_BASIS: n_fft must be even";
        if (d.K2 % 2 || d.K2 < 2 * (d.n_fft / 2 + 1)) return "IDFT_BASIS: K2 must be even, with n_fft/2 + 1 <= K2/2";
        if (!d.window) return "IDFT_BASIS: window is required";
        if (!d.out_f32 || planes) return "IDFT_BASIS: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_OVERLAP_ADD:
        if (const char* why = vocos_stft_error(d.n_fft, d.hop)) return why;
        if (d.B < 1 || d.T < 1) return "OVERLAP_ADD: B, T >= 1";
        if (!d.x || !d.window) return "OVERLAP_ADD: x (frames) and window are required";
        if (!d.out_f32 || planes) return "OVERLAP_ADD: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_MEAN3_SILU:
        if (d.n < 1 || d.n % 4) return "MEAN3_SILU: n must be a positive multiple of 4";
        if (!d.x || !d.x1 || !d.x2) return "MEAN3_SILU: x, x1 and x2 are required";
        if (!d.out_f32 && !planes) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.x1) || !aligned16(d.x2) || !aligned16(d.out_f32) || !aligned16(d.out_hi) || !aligned16(d.out_lo))
            return "MEAN3_SILU: buffers must be 16-byte aligned";
        return nullptr;
    case ST_TEST_ROW_POST_TANH:
        if (d.C != 16) return "POST_TANH: C must be 16, conv_post's one input width";
        if (d.B < 1 || d.T < 1) return "POST_TANH: B, T >= 1";
        if (!d.x || !d.w || !d.bias) return "POST_TANH: x, w and bias are required";
        if (!d.out_f32 || planes) return "POST_TANH: writes out_f32 only";
        if (!aligned16(d.x)) return "POST_TANH: x must be 16-byte aligned";
        return nullptr;
    default:
        return "unknown kind";
    }
}

int st_test_row_ex(st_handle* h, const st_test_row_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_row_ex: null descriptor");
    const st_test_row_desc& d = *dp;
    if (const char* why = test_row_desc_error(d)) return fail(h, std::string("st_test_row_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    bf16* hi = (bf16*)d.out_hi; bf16* lo = (bf16*)d.out_lo;
    TestBufs bufs;
    cudaError_t e = cudaSuccess;
    switch (d.kind) {
    case ST_TEST_ROW_ADALN: {
        LnArgs a;
        a.xin = d.x; a.xout = d.xout; a.film = d.film; a.film_bstride = d.film_bstride;
        a.shift = d.shift; a.scale = d.scale; a.ada_bstride = d.ada_bstride; a.c_clamp = d.c_clamp;
        a.mask = d.mask; a.B = d.B; a.has_film = d.has_film; a.mask_out = d.mask_out;
        a.u_f32 = d.out_f32; a.u_hi = hi; a.u_lo = lo; a.u16 = d.u16;
        a.BB = d.BB; a.T = d.T; a.H = d.C;
        e = launch_film_ln_mod(a, s);
        break;
    }
    case ST_TEST_ROW_DWCONV_LN: {
        DwLnArgs a;
        a.B = d.B; a.T = d.T; a.C = d.C; a.eps = d.eps;
        a.x = d.x; a.dw_b = d.bias; a.ln_w = d.ln_w; a.ln_b = d.ln_b;
        a.out_f32 = d.out_f32; a.out_hi = hi; a.out_lo = lo;
        if (d.w) {                     // (C, 1, 7) -> [7][C], as vocos_finalize / ffgan_finalize pack it
            float* packed = (float*)bufs.take((size_t)7 * d.C * 4);
            if (!packed) return fail(h, "st_test_row_ex: out of memory");
            ST_CUDA(launch_pack_conv(d.w, packed, d.C, 1, 7, d.C, 0, 0, 1, s));
            a.dw_w = packed;
        }
        e = launch_dwconv_ln(a, s);
        break;
    }
    case ST_TEST_ROW_SPECTRUM:
        e = launch_spectrum(d.x, d.Nh, d.Kp, d.K, d.K2, (long)d.B * d.T, d.out_f32, hi, lo, s);
        break;
    case ST_TEST_ROW_IDFT_BASIS:
        e = launch_idft_basis(d.window, d.n_fft, d.n_fft / 2 + 1, d.K2, d.out_f32, s);
        break;
    case ST_TEST_ROW_OVERLAP_ADD:
        e = launch_overlap_add(d.x, d.window, d.B, d.T, d.n_fft, d.hop, d.out_f32, s);
        break;
    case ST_TEST_ROW_MEAN3_SILU:
        e = launch_mean3_silu(d.x, d.x1, d.x2, (long)d.n, d.out_f32, hi, lo, s);
        break;
    case ST_TEST_ROW_POST_TANH:
        e = launch_post_conv_tanh(d.x, d.w, d.bias, d.B, (long)d.T, d.C, 13, d.out_f32, s);
        break;
    }
    if (e != cudaSuccess) return fail(h, std::string("st_test_row_ex: launch failed: ") + cudaGetErrorString(e));
    e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, std::string("st_test_row_ex: ") + cudaGetErrorString(e));
    return 0;
}

}  // extern "C"
