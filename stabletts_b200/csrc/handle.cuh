// Host-side state shared by the C-ABI translation units: the handle every entry point takes, and the model it carries.
#pragma once
#include "common.cuh"
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <map>
#include <memory>

namespace st {

struct GemmW {           // one packed conv/linear weight
    float* f32 = nullptr; bf16* hi = nullptr; bf16* lo = nullptr; float* bias = nullptr;
    bf16 *h_hi = nullptr, *h_lo = nullptr;      // fp16 hi / lo planes (FFN convs only; the opt-in two-pass precision)
    int taps = 1, N = 0, K = 0;
};

struct Act {             // an activation buffer: fp32 and/or split-bf16 planes, (batch, T, C)
    float* f32 = nullptr; bf16* hi = nullptr; bf16* lo = nullptr; int C = 0;
};

struct Bump {
    char* base; size_t off = 0, cap;
    Bump(void* p, size_t c) : base((char*)p), cap(c) {}
    template <class T> T* take(size_t n) {
        off = (off + 255) & ~size_t(255);
        T* r = base ? (T*)(base + off) : nullptr;
        off += n * sizeof(T);
        return r;
    }
};


// What a handle of one kind holds beyond the common state of st_handle: its dims, its weights packed from h->raw into
// h->owned, and whatever else it allocates (freed by the destructor, which st_destroy runs on the handle's device).
struct Model {
    virtual ~Model() = default;
    virtual int finalize(st_handle* h, cudaStream_t s) = 0;   // packs h->raw into h->owned (emptied before the call)
    virtual void drop_cached() {}                             // forgets state that bakes in weights, workspace or modes
};

}  // namespace st

struct st_handle {
    int device = 0, engine = ST_ENGINE_TCGEN05, num_sms = 132;
    int precision = ST_PRECISION_FFN_FP16X2;
    std::string err;
    std::map<std::string, std::pair<float*, int64_t>> raw;   // name -> (device copy, numel)
    bool finalized = false;
    std::vector<void*> owned;
    void* ws_ptr = nullptr; size_t ws_bytes = 0; bool ws_owned = false;
    int64_t launches = 0;
    float* part_buf = nullptr; size_t part_bytes = 0;   // split-K partial tiles of latency-bound small GEMMs (run_gemm)
    // optional per-launch CUDA-event profiling (bench.py roofline): category, flops, bytes, event pair
    bool prof_on = false;
    struct ProfRec { int cat; double flops, bytes; cudaEvent_t e0, e1; double issued = 0; };   // issued: tensor-core FLOPs actually
                                                                                             // issued (passes x algorithmic), 0 = not an MMA launch
    double prof_issued[32] = {0};                       // per class, filled by st_profile_end (st_profile_issued reads it)
    std::vector<ProfRec> prof;
    std::vector<cudaEvent_t> ev_pool; size_t ev_used = 0;
    cudaEvent_t take_event() {
        if (ev_used == ev_pool.size()) { cudaEvent_t e; cudaEventCreate(&e); ev_pool.push_back(e); }
        return ev_pool[ev_used++];
    }
    std::unique_ptr<st::Model> model;
};

namespace st {

int fail(st_handle* h, const std::string& msg);          // records the message (st_last_error) and returns 1

// The handle's model as an M, or nullptr after recording "handle is not a <what>".  Every typed entry point asks this
// first, before it looks at weights, shapes or pointers.
template <class M> M* model_of(st_handle* h, const char* what) {
    M* m = dynamic_cast<M*>(h->model.get());
    if (!m) fail(h, std::string("handle is not a ") + what);
    return m;
}

// Creates a handle on `device` (an sm_90 GPU) that carries `model`; the model's creator has validated its arguments.
int create_handle(int device, std::unique_ptr<Model> model, st_handle** out);

#define ST_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            char buf__[512];                                                                  \
            snprintf(buf__, sizeof buf__, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, \
                     cudaGetErrorString(e__));                                                \
            return fail(h, buf__);                                                            \
        }                                                                                     \
    } while (0)

#define ST_LAUNCH(call) do { h->launches++; ST_CUDA(call); } while (0)

// profiled launch: brackets `call` with events on the launching stream when profiling is enabled
#define ST_LAUNCH_P(cat, flops_, bytes_, s_, call)                                             \
    do {                                                                                      \
        st_handle::ProfRec pr__{cat, (double)(flops_), (double)(bytes_), nullptr, nullptr};   \
        if (h->prof_on) { pr__.e0 = h->take_event(); pr__.e1 = h->take_event(); cudaEventRecord(pr__.e0, s_); } \
        h->launches++;                                                                        \
        ST_CUDA(call);                                                                        \
        if (h->prof_on) { cudaEventRecord(pr__.e1, s_); h->prof.push_back(pr__); }            \
    } while (0)

// Every entry point runs on the handle's device and RESTORES the caller's current device on return (a torch caller
// whose current device is cuda:0 must not find it switched to cuda:1 because a module lives there).
struct DevGuard {
    int prev = -1, dev;
    explicit DevGuard(int d) : dev(d) { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; if (prev != d) cudaSetDevice(d); }
    ~DevGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
    DevGuard(const DevGuard&) = delete; DevGuard& operator=(const DevGuard&) = delete;
};
#define ST_ENTER(h) DevGuard dev_guard__((h)->device)

template <class T> int dev_alloc(st_handle* h, T** p, size_t n) {
    ST_CUDA(cudaMalloc((void**)p, std::max<size_t>(n, 1) * sizeof(T)));
    h->owned.push_back(*p);
    return 0;
}

// The handle's model as an M once its weights are packed: model_of, then "weights not finalized" (nullptr after either).
template <class M> M* ready_model(st_handle* h, const char* what) {
    M* m = model_of<M>(h, what);
    if (m && !h->finalized) {
        fail(h, "weights not finalized (call st_finalize_weights)");
        return nullptr;
    }
    return m;
}

// handle.cu: raw (reference-layout) tensor lookup, conv/linear weight packing into [tap][N][K] fp32 + split planes, GEMM dispatch
int get_raw(st_handle* h, const std::string& name, int64_t expect, float** out);
// Allocates w's fp32 and split-bf16 planes for [taps][N][K] (and an N-float bias) from the handle's packed-weight memory.
// The caller fills f32 (and bias), then splits it with launch_split.
int alloc_gemm_w(st_handle* h, GemmW* w, int taps, int N, int K, bool with_bias);
int pack_gemm(st_handle* h, GemmW* w, const std::vector<std::string>& names, int N_each, int Csrc, int k, int c_off, int Cc,
              bool with_bias, cudaStream_t s);
// depthwise Conv1d weight `name` (C, 1, 7) -> [7][C]: dwconv_ln_kernel reads float4 groups over channels
int pack_dw7(st_handle* h, const std::string& name, int C, float** out, cudaStream_t s);
int run_gemm(st_handle* h, GemmArgs& g, const GemmW& w, const Act* a0, const Act* a1, const Act& out, cudaStream_t s,
             int prof_cat = ST_PROF_GEMM);
// Allocates the split-K partial buffer run_gemm uses (once per handle; a no-op after that).
int ensure_part_buf(st_handle* h);

// out[tap][n_off + n][c] = in[n][c_off + c][tap]: (Nsrc, Csrc, k) reference Conv1d / Linear layout -> packed [k][Ntot][Cc]
cudaError_t launch_pack_conv(const float* in, float* out, int Nsrc, int Csrc, int k, int Ntot, int n_off, int c_off, int Cc,
                             cudaStream_t s);

// An activation of rows x C carved from `bp`: an fp32 plane (the SIMT engine's operand, or an fp32 result) and / or the
// split-bf16 hi / lo planes (the wgmma engine's operand).
inline Act take_act(Bump& bp, size_t rows, int C, bool f32, bool planes) {
    Act a; a.C = C;
    a.f32 = f32 ? bp.take<float>(rows * C) : nullptr;
    a.hi = planes ? bp.take<bf16>(rows * C) : nullptr;
    a.lo = planes ? bp.take<bf16>(rows * C) : nullptr;
    return a;
}

// GemmArgs of a GEMM with one batch row per utterance: B batches of T frames, no CFG doubling, no broadcast rows.
inline GemmArgs utt_gemm(int B, int T, int flags) {
    GemmArgs g;
    g.BB = B; g.T = T; g.a_bmod = B; g.B = B; g.resid_clamp = B - 1; g.flags = flags;
    return g;
}

// Grows a workspace the handle's model owns to `need` bytes.  Both keep the old block until the work queued on `s` is done.
// grow_ws_synced synchronises `s` and frees the old block before it allocates the new one, so the two are never held at
// once: for the vocoders, whose workspaces grow with the mel length (FireflyGAN takes 256 KB per mel frame); free it with
// cudaFree.  grow_ws is stream-ordered (cudaFreeAsync / cudaMallocAsync on `s`) and never blocks the host: for the small
// front-end workspaces; free it with cudaFreeAsync.
int grow_ws_synced(st_handle* h, void** ws, size_t* have, size_t need, cudaStream_t s);
int grow_ws(st_handle* h, void** ws, size_t* have, size_t need, cudaStream_t s);

// nullptr when st_create_vocos accepts this (n_fft, hop) pair, else why not (also the overlap-add test hook's contract)
const char* vocos_stft_error(int n_fft, int hop);

// Device scratch of a kernel-level test hook, freed on every exit (cudaFree waits for the work that uses it).  `ok` turns
// false when an allocation fails.
struct TestBufs {
    std::vector<void*> p;
    bool ok = true;
    template <class T> T* take(size_t n) {
        void* q = nullptr;
        if (cudaMalloc(&q, std::max<size_t>(n * sizeof(T), 4)) != cudaSuccess) { ok = false; return nullptr; }
        p.push_back(q);
        return (T*)q;
    }
    ~TestBufs() { for (void* q : p) cudaFree(q); }
};

// The end of a test hook: waits for `s`, then reports a launch or execution error as "<fn>: <error>".
int hook_done(st_handle* h, cudaStream_t s, const char* fn);

}  // namespace st
