// The ODE drivers of the CFM decoder (models/flow_matching.py:24-67) over the estimator of dit_api.cu: explicit
// Runge–Kutta on the caller's grid, all device-resident (stage times are baked into kernel arguments, nothing is copied
// or synchronised between steps; small solves replay as one CUDA graph), its host-I/O variant, and the adaptive
// embedded solvers.
#include "dit.cuh"
#include <cmath>

using namespace st;

namespace {

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

// the sinusoidal embedding (launch_time_embed) of n_t <= 256 times given on the host: they travel as a kernel argument
cudaError_t st::launch_time_embed_vals(const float* t_host, int n_t, int H, float* out, cudaStream_t s) {
    if (n_t < 1 || n_t > (int)(sizeof(TArr::v) / sizeof(float))) return cudaErrorInvalidValue;
    TArr ta;
    for (int i = 0; i < n_t; ++i) ta.v[i] = t_host[i];
    const int cnt = n_t * (H / 2);
    time_embed_val_kernel<<<(cnt + 127) / 128, 128, 0, s>>>(ta, n_t, H, out);
    return cudaGetLastError();
}

namespace {

// Dormand–Prince 5(4): the stage times c_2..c_6 (then 1 again: the FSAL stage of the adaptive solver) and the rows of the
// Butcher tableau for stages 2..6; the last row is also the 5th-order solution weights.
constexpr double kDpAlpha[6] = {1. / 5, 3. / 10, 4. / 5, 8. / 9, 1.0, 1.0};
constexpr double kDpBeta[6][6] = {{1. / 5}, {3. / 40, 9. / 40}, {44. / 45, -56. / 15, 32. / 9},
                                  {19372. / 6561, -25360. / 2187, 64448. / 6561, -212. / 729},
                                  {9017. / 3168, -355. / 33, 46732. / 5247, 49. / 176, -5103. / 18656},
                                  {35. / 384, 0, 500. / 1113, 125. / 192, -2187. / 6784, 11. / 84}};

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
        for (int i = 0; i < 6; ++i) {
            t.c[i] = i ? (float)kDpAlpha[i - 1] : 0.f;
            t.b[i] = (float)kDpBeta[5][i];
            for (int j = 0; j < 5; ++j) t.a[i][j] = i ? (float)kDpBeta[i - 1][j] : 0.f;
        }
    }
    return t;
}

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
        const double ce[7] = {35. / 384 - 1951. / 21600, 0, 500. / 1113 - 22642. / 50085, 125. / 192 - 451. / 720,
                              -2187. / 6784 + 12231. / 42400, 11. / 84 - 649. / 6300, -1. / 60};
        const double cm[7] = {6025192743. / 30085553152. / 2, 0, 51252292925. / 65400821598. / 2, -2691868925. / 45128329728. / 2,
                              187940372067. / 1594534317056. / 2, -1776094331. / 19743644256. / 2, 11237099. / 235043384. / 2};
        for (int i = 0; i < 6; ++i) { t.alpha[i] = kDpAlpha[i]; t.csol[i] = kDpBeta[5][i]; for (int j = 0; j < 6; ++j) t.beta[i][j] = kDpBeta[i][j]; }
        for (int i = 0; i < 7; ++i) { t.cerr[i] = ce[i]; t.cmid[i] = cm[i]; }
        t.sol_is_last_stage = true;
    }
    return t;
}

}  // namespace

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
            for (int off = table_lo; off < table_hi; off += 256)
                ST_LAUNCH(launch_time_embed_vals(tv.data() + off, std::min(256, table_hi - off), d.hidden,
                                                 w.temb + (size_t)(off - table_lo) * d.hidden, s));
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

extern "C" {

int st_solve(st_handle* h, float* z_inout, const float* mu, const float* mask, const float* c, const float* fake_content,
             const float* fake_speaker, float cfg_strength, const float* t_span_host, int n_steps, int method, int B, int T,
             void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = ready_model<CfmModel>(h, "CFM estimator");
    if (!m || check_bt(h, B, T)) return 1;
    if (!z_inout || !mu || !mask || !c || !t_span_host) return fail(h, "st_solve: null pointer");
    if (n_steps <= 0) return fail(h, "n_timesteps must be positive");
    if (method < ST_EULER || method > ST_DOPRI5_FIXED) return fail(h, "unknown ODE method");
    const int cfg = (fake_content && fake_speaker) ? 1 : 0;
    if (!cfg && (fake_content || fake_speaker)) return fail(h, "CFG needs both fake_content and fake_speaker");
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (ensure_ws(h, *m, w, B, T, cfg)) return 1;
    const st_dims& d = m->d;
    auto direct = [&] {
        return solve_impl(h, *m, w, z_inout, mu, mask, c, fake_content, fake_speaker, cfg_strength, t_span_host, n_steps, method, B, T, cfg, s);
    };
    // Small problems are launch-bound (~90 kernels per evaluation, a few microseconds each): replay the whole
    // solve as one CUDA graph.  Inputs are staged into workspace-owned buffers so the graph's pointers are stable.
    const long rows = (long)(cfg ? 2 * B : B) * T;
    const bool use_graph = !h->prof_on && !m->graphs_disabled && rows <= 24576;
    if (!use_graph) return direct();

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
            return direct();
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
            m->graphs_disabled = true;                 // do not retry: fall back to direct enqueue for this handle
            if (getenv("STABLETTS_B200_DEBUG"))
                fprintf(stderr, "[stabletts_b200] graph capture failed (%s / %s); falling back to direct enqueue\n",
                        cudaGetErrorString(ce), h->err.c_str());
            return direct();
        }
        cudaGraphExec_t exec = nullptr;
        cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) { cudaGetLastError(); m->graphs_disabled = true; return fail(h, std::string("cudaGraphInstantiate failed: ") + cudaGetErrorString(ie)); }
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
int st_solve_adaptive_ex(st_handle* h, int method, float* z_inout, const float* mu, const float* mask, const float* c,
                         const float* fake_content, const float* fake_speaker, float cfg_strength, double t_start, double t_end,
                         double rtol, double atol, int max_steps, int B, int T, void* stream, int64_t* stats) {
    if (!h) return 1;
    ST_ENTER(h);
    CfmModel* m = ready_model<CfmModel>(h, "CFM estimator");
    if (!m || check_bt(h, B, T)) return 1;
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
        const float tf = (float)t;
        ST_LAUNCH(launch_time_embed_vals(&tf, 1, d.hidden, w.temb, s));
        if (precompute_film(h, *m, w, 1, s)) return 1;
        Act xin = w.xt; xin.f32 = const_cast<float*>(yin);
        if (h->engine == ST_ENGINE_TCGEN05) {
            ST_LAUNCH(launch_split(yin, w.xs.hi, w.xs.lo, numel, s));
            xin.hi = w.xs.hi; xin.lo = w.xs.lo;
        }
        if (estimator_eval(h, *m, w, xin, mask, w.film, 0, s)) return 1;
        ST_LAUNCH(launch_cfg_combine(w.V.f32, kout, B, (long)T * d.n_mel, cfg, cfg_strength, s));
        ++nfe;
        return 0;
    };
    auto norm = [&](const float* const* K, const float* coef, int n, const float* u, const float* v, double* out) -> int {
        ST_LAUNCH(launch_scaled_sumsq(K, coef, n, u, v, (float)atol, (float)rtol, numel, w.dscal, s));
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
    CfmModel* m = ready_model<CfmModel>(h, "CFM estimator");
    if (!m || check_bt(h, B, T)) return 1;
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

}  // extern "C"
