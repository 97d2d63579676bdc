// What every model's C-ABI shares: handle creation and the generic entry points (destroy, engine / precision modes,
// launch counting and profiling, weight loading and finalizing, an attached workspace), weight lookup and packing, and
// the conv-GEMM dispatch.
#include "handle.cuh"
#include <mutex>

using namespace st;

namespace {

std::string g_create_error;
std::mutex g_mutex;

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

int st::grow_ws(st_handle* h, void** ws, size_t* have, size_t need, cudaStream_t s) {
    if (need <= *have) return 0;
    if (*ws) { ST_CUDA(cudaFreeAsync(*ws, s)); *ws = nullptr; *have = 0; }
    ST_CUDA(cudaMallocAsync(ws, need, s));
    *have = need;
    return 0;
}

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

int st::alloc_gemm_w(st_handle* h, GemmW* w, int taps, int N, int K, bool with_bias) {
    w->taps = taps; w->N = N; w->K = K;
    const size_t n = (size_t)taps * N * K;
    if (dev_alloc(h, &w->f32, n) || dev_alloc(h, &w->hi, n) || dev_alloc(h, &w->lo, n)) return 1;
    return with_bias ? dev_alloc(h, &w->bias, (size_t)N) : 0;
}

// Packs `parts` reference tensors (each (N_i, Csrc, k)) stacked along N, taking channels [c_off, c_off+Cc).
int st::pack_gemm(st_handle* h, GemmW* w, const std::vector<std::string>& names, int N_each, int Csrc, int k, int c_off,
                  int Cc, bool with_bias, cudaStream_t s) {
    const int parts = (int)names.size();
    if (alloc_gemm_w(h, w, k, N_each * parts, Cc, with_bias)) return 1;
    for (int p = 0; p < parts; ++p) {
        float* src;
        if (get_raw(h, names[p] + ".weight", (int64_t)N_each * Csrc * k, &src)) return 1;
        ST_CUDA(launch_pack_conv(src, w->f32, N_each, Csrc, k, w->N, p * N_each, c_off, Cc, s));
        if (with_bias) {
            float* bsrc;
            if (get_raw(h, names[p] + ".bias", N_each, &bsrc)) return 1;
            ST_CUDA(cudaMemcpyAsync(w->bias + (size_t)p * N_each, bsrc, sizeof(float) * N_each, cudaMemcpyDeviceToDevice, s));
        }
    }
    ST_CUDA(launch_split(w->f32, w->hi, w->lo, (long)k * w->N * Cc, s));
    return 0;
}

int st::pack_dw7(st_handle* h, const std::string& name, int C, float** out, cudaStream_t s) {
    float* dw;
    if (get_raw(h, name, (int64_t)C * 7, &dw) || dev_alloc(h, out, (size_t)7 * C)) return 1;
    ST_CUDA(launch_pack_conv(dw, *out, C, 1, 7, C, 0, 0, 1, s));
    return 0;
}

// ----- GEMM dispatch -------------------------------------------------------------------------------
// S x tiles <= num_sms tiles of at most 128 x 128 fp32: one buffer of num_sms x 64 KB (8.7 MB on 132 SMs) covers every shape
// run_gemm splits, so it is allocated once and never moves (captured graphs keep pointing at it).  Not inside a stream
// capture (cudaMalloc is not capturable): run_gemm runs such a call unsplit.
int st::ensure_part_buf(st_handle* h) {
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
        const int kb = g.taps * ((g.Cs[0] + 63) / 64 + (g.n_src > 1 ? (g.Cs[1] + 63) / 64 : 0));
        const long tiles = (long)g.BB * ((g.T + 127) / 128) * ((g.N + 127) / 128);
        int S = 1;
        for (int cand = 4; cand >= 2; --cand)
            if (kb % cand == 0 && kb / cand >= 3 && tiles * cand <= h->num_sms) { S = cand; break; }
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

int st::hook_done(st_handle* h, cudaStream_t s, const char* fn) {
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}

// =================================================================================================
extern "C" {

int st_version(void) { return 20800; }

const char* st_last_error(const st_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

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


int st_attach_workspace(st_handle* h, void* dev_ptr, size_t bytes) {
    if (!h) return 1;
    ST_ENTER(h);
    if (h->ws_ptr && h->ws_owned) cudaFree(h->ws_ptr);
    h->model->drop_cached();           // cached graphs hold pointers into the old workspace
    h->ws_ptr = dev_ptr; h->ws_bytes = dev_ptr ? bytes : 0; h->ws_owned = false;
    return 0;
}
}  // extern "C"
