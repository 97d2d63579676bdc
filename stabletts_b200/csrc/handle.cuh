// Host-side state shared by the C-ABI translation units (api.cu: CFM estimator / text encoder; vocos_api.cu: vocoder).
#pragma once
#include "common.cuh"
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <map>

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


}  // namespace st

struct st_handle {
    st_dims d;
    int kind = 0;                      // 0 = CFM estimator (Decoder), 1 = TextEncoder (SURVEY.md §8 row f2), 2 = Vocos vocoder (row f4)
    void* vocos = nullptr;             // kind 2: st::VocosState (vocos_api.cu)
    int n_vocab = 0; float* emb = nullptr;
    int device = 0, engine = ST_ENGINE_TCGEN05, num_sms = 132;
    int precision = ST_PRECISION_FFN_FP16X2;
    std::string err;
    std::map<std::string, std::pair<float*, int64_t>> raw;   // name -> (device copy, numel)
    bool finalized = false;
    st::GemmW cond0, cond2, cond4, inmu, inx, fin;
    std::vector<st::GemmW> qkv, wo, c1, c2, lsc;
    std::vector<float*> film_w, film_b, ada_w, ada_b;
    float *tm0_w = nullptr, *tm0_b = nullptr, *tm2_w = nullptr, *tm2_b = nullptr;
    std::vector<void*> owned;
    void* ws_ptr = nullptr; size_t ws_bytes = 0; bool ws_owned = false;
    int64_t launches = 0;
    // CUDA-graph cache for launch-bound (small) solves: key -> instantiated graph + its launch count
    struct GraphEntry { std::string key; cudaGraphExec_t exec; int64_t launches; };
    std::vector<GraphEntry> graphs;
    std::vector<std::string> graph_seen;   // keys enqueued directly once (kernels loaded, attributes set) before capture
    double* pinned = nullptr;          // 16 B of pinned host memory: norm read-back of the adaptive controller
    char* pin_buf = nullptr; size_t pin_bytes = 0;   // pinned staging of st_solve_host for callers with pageable buffers
    float* part_buf = nullptr; size_t part_bytes = 0;   // split-K partial tiles of latency-bound small GEMMs (run_gemm)
    cudaStream_t cap_stream = nullptr;   // capture happens on a private stream (the caller's may be the legacy stream)
    int graph_mode = -1;               // -1: read STABLETTS_B200_GRAPH on first use; 0 off; 1 always; 2 auto (small problems)
    void drop_graphs() { for (auto& g : graphs) cudaGraphExecDestroy(g.exec); graphs.clear(); }
    // optional per-launch CUDA-event profiling (bench.py roofline): category, flops, bytes, event pair
    bool prof_on = false;
    struct ProfRec { int cat; double flops, bytes; cudaEvent_t e0, e1; double issued = 0; };   // issued: tensor-core FLOPs actually
                                                                                             // issued (passes x algorithmic), 0 = not an MMA launch
    double prof_issued[16] = {0};                       // per class, filled by st_profile_end (st_profile_issued reads it)
    std::vector<ProfRec> prof;
    std::vector<cudaEvent_t> ev_pool; size_t ev_used = 0;
    cudaEvent_t take_event() {
        if (ev_used == ev_pool.size()) { cudaEvent_t e; cudaEventCreate(&e); ev_pool.push_back(e); }
        return ev_pool[ev_used++];
    }
};

namespace st {

int fail(st_handle* h, const std::string& msg);          // records the message (st_last_error) and returns 1

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

// api.cu: raw (reference-layout) tensor lookup, conv/linear weight packing into [tap][N][K] fp32 + split planes, GEMM dispatch
int get_raw(st_handle* h, const std::string& name, int64_t expect, float** out);
int pack_gemm(st_handle* h, GemmW* w, const std::vector<std::string>& names, int N_each, int Csrc, int k, int c_off, int Cc,
              bool with_bias, cudaStream_t s);
int run_gemm(st_handle* h, GemmArgs& g, const GemmW& w, const Act* a0, const Act* a1, const Act& out, cudaStream_t s,
             int prof_cat = ST_PROF_GEMM);

// out[tap][n_off + n][c] = in[n][c_off + c][tap]: (Nsrc, Csrc, k) reference Conv1d / Linear layout -> packed [k][Ntot][Cc]
cudaError_t launch_pack_conv(const float* in, float* out, int Nsrc, int Csrc, int k, int Ntot, int n_off, int c_off, int Cc,
                             cudaStream_t s);

// vocos_api.cu: the vocoder's per-handle state (created by st_create_vocos, packed by st_finalize_weights)
int vocos_finalize(st_handle* h, cudaStream_t s);
void vocos_free(st_handle* h);

}  // namespace st
