// The DiT models (the CFM estimator and the text encoder, dit_api.cu) and what the ODE drivers (solve.cu) use of them.
#pragma once
#include "handle.cuh"

namespace st {

constexpr int MAX_EVAL_TABLE = 1024;   // evaluations whose time conditioning (temb, FiLM vectors) the workspace holds at once

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

// What the CFM estimator and the text encoder share: DiT blocks (models/diffusion_transformer.py:98-117) and a final
// 1x1 projection.
struct DitModel : Model {
    st_dims d;
    std::vector<GemmW> qkv, wo, c1, c2;
    std::vector<float*> ada_w, ada_b;
    GemmW fin;
    // false when a weight with fp16 planes (conv_1, conv_2, long skips) lies outside what those planes represent: the
    // model then runs ST_PRECISION_FFN_FP16X2 as three passes everywhere.  f16_range is its device flag during finalize.
    bool f16_ok = true;
    int* f16_range = nullptr;
    explicit DitModel(const st_dims& dims) : d(dims) {}
    // the weights of block l under `p` ("blocks.<l>.block." / "encoder.<l>.")
    int pack_block(st_handle* h, int l, const std::string& p, cudaStream_t s);
    // fp16 hi / lo planes of a packed weight, noting in f16_range whether they represent it
    int pack_f16_planes(st_handle* h, GemmW* w, cudaStream_t s);
    // around a finalize's packing: clear f16_range first, then read it once into f16_ok
    int begin_f16_range(st_handle* h, cudaStream_t s);
    int end_f16_range(st_handle* h, cudaStream_t s);
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
    bool graphs_disabled = false;      // set by a failed capture or instantiate: direct enqueue from then on
    double* pinned = nullptr;          // 16 B of pinned host memory: norm read-back of the adaptive controller
    char* pin_buf = nullptr; size_t pin_bytes = 0;   // pinned staging of st_solve_host for callers with pageable buffers
    using DitModel::DitModel;
    ~CfmModel() override;
    void drop_cached() override;
    int finalize(st_handle* h, cudaStream_t s) override;
};

// TextEncoder (models/text_encoder.py:8-44): an embedding, n_layers DiT blocks without FiLM, proj
struct TextEncoderModel : DitModel {
    int n_vocab;
    float* emb = nullptr;
    TextEncoderModel(const st_dims& dims, int vocab) : DitModel(dims), n_vocab(vocab) {}
    int finalize(st_handle* h, cudaStream_t s) override;
};

// Lays out w for (B, T, cfg) over the handle's workspace, (re)allocating an owned one that is too small.
int ensure_ws(st_handle* h, DitModel& m, Workspace& w, int B, int T, int cfg);
// the batch checks every DiT entry point makes after ready_model
int check_bt(st_handle* h, int B, int T);
// GemmArgs of a DiT GEMM: BB = B rows (2B with CFG: cond rows, then uncond rows), the conditioning of rows >= B clamped
// to row B (the uncond row), `mask` over the B real rows
GemmArgs dit_gemm(const Workspace& w, const float* mask, int flags);

// per solve: cond features, the in_proj mu-half P and adaLN(c) for B real rows (+ the uncond row with CFG)
int precompute_cond(st_handle* h, const CfmModel& m, Workspace& w, const float* mu, const float* mask, const float* c,
                    const float* fake_content, const float* fake_speaker, cudaStream_t s);
// time-MLP + FiLM vectors for n_t times already embedded in w.temb
int precompute_film(st_handle* h, const CfmModel& m, Workspace& w, int n_t, cudaStream_t s);
// one estimator evaluation on the stage input xin (B, T, M) -> w.V (BB, T, M); film: this evaluation's FiLM row (L, 2H),
// film_bstride != 0 when t is per-sample
int estimator_eval(st_handle* h, const CfmModel& m, Workspace& w, const Act& xin, const float* mask, const float* film,
                   long film_bstride, cudaStream_t s);

}  // namespace st
