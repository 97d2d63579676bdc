/*
 * stabletts_b200.h — C ABI of the CUDA-native (H100, sm_90a) CFM/DiT mel-denoiser (libstabletts_b200.so).
 *
 * The reference (KdaiP/StableTTS) has no FFI: its boundary for this path is a Python class
 * surface.  Each entry point below names the reference interface it replaces
 * (paths relative to the reference checkout).  INTEGRATION.md shows the ctypes stub a
 * maintainer adds on the reference side.
 *
 * Conventions
 *  - every tensor argument is a raw DEVICE pointer to contiguous fp32 in the reference's own
 *    boundary layout (B, C, T), T fastest, owned by the caller; the library never frees or
 *    retains caller pointers past the call (weights are copied + repacked at load time);
 *  - all work is enqueued on the `stream` passed (a cudaStream_t cast to void*); no entry point
 *    except st_create / st_destroy / st_*_host synchronises the device;
 *  - every function returns 0 on success, non-zero on failure; st_last_error() gives the text.
 *    No exceptions cross the ABI.  There is NO CPU fallback: without a CUDA device st_create fails.
 *  - `mask` is the reference's float prefix mask (B,1,T) == (B,T), values in {0,1}.
 */
#ifndef STABLETTS_B200_H_
#define STABLETTS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct st_handle st_handle;

/* Constructor arguments of models/estimator.py:66 `Decoder.__init__` (as built by
 * models/flow_matching.py:22 from CFMDecoder's own arguments). */
typedef struct st_dims {
    int32_t n_mel;      /* noise_channels == cond_channels == out_channels (models/model.py:40) */
    int32_t hidden;     /* hidden_channels, 256 (config.py:23) */
    int32_t filter;     /* filter_channels, 1024 (config.py:24) */
    int32_t n_heads;    /* 4 */
    int32_t n_layers;   /* n_dec_layers, 6 (even: U-Net long skips, models/estimator.py:92) */
    int32_t kernel;     /* kernel_size, 3 */
    int32_t gin;        /* gin_channels, 256 (must equal hidden: adaLN_modulation.0 is Identity,
                           models/diffusion_transformer.py:93) */
} st_dims;

/* ODE methods — the `solver` strings of models/flow_matching.py:54 / webui.py:110 that have a
 * fixed grid; ST_DOPRI5_FIXED is the Dormand–Prince tableau stepped on the grid without error
 * control (BASELINE.json cfg2's "dopri5-equiv"), NOT torchdiffeq's adaptive dopri5. */
enum { ST_EULER = 0, ST_MIDPOINT = 1, ST_RK4 = 2, ST_DOPRI5_FIXED = 3 };

/* GEMM engines (both hand-written sm_90a CUDA in this library; a debugging switch, not a
 * backend dispatch): 0 = wgmma/TMA split-bf16 tensor-core path (default; the constant keeps its historical name),
 * 1 = fp32 SIMT. */
enum { ST_ENGINE_TCGEN05 = 0, ST_ENGINE_SIMT = 1 };

/* Replaces: Decoder.__init__ (models/estimator.py:66-96).  Creates the per-device handle. */
int st_create(const st_dims* dims, int device, st_handle** out);

/* Replaces: nn.Module teardown. Frees packed weights and any internally owned workspace. */
int st_destroy(st_handle* h);

/* Last error text for this handle (or for st_create when h == NULL).  Never NULL. */
const char* st_last_error(const st_handle* h);

/* Library/ABI version (major*10000 + minor*100 + patch). */
int st_version(void);

/* Replaces: load_state_dict of the `decoder.estimator.*` tensors (api.py:49; inventory in
 * models/estimator.py:66-96).  `name` is the reference key relative to `estimator.` (e.g.
 * "blocks.3.block.mlp.conv_1.weight"); `data` is a device fp32 tensor in the reference layout
 * with `numel` elements.  The library converts/packs into buffers it owns. */
int st_load_weight(st_handle* h, const char* name, const float* data, int64_t numel, void* stream);

/* Must be called after all 116 (for 6 layers) tensors are loaded; fails listing a missing key. */
int st_finalize_weights(st_handle* h, void* stream);

/* Selects the GEMM engine (see enum above).  Default ST_ENGINE_TCGEN05. */
int st_set_engine(st_handle* h, int engine);

/* Precision of the tensor-core engine's operands.
 *   ST_PRECISION_FFN_FP16X2 (the default since round 2): every contraction runs split-bf16 x 3 (hi / lo planes of both
 *     operands, three MMA passes, ~16 mantissa bits) EXCEPT the two k = 3 FFN convs of every DiT block
 *     (models/diffusion_transformer.py:20-30; 48-55 % of the FLOPs) and the three U-Net long-skip convs
 *     (models/estimator.py:131-132), which take their activations as ONE fp16 plane against fp16 hi / lo weights: two MMA
 *     passes and half the operand traffic.  tests/test_gpu_parity.py::test_ffn_fp16x2_margin_at_maximum_sizes holds the
 *     error against the reference under 5e-4 (2x margin below the 1e-3 bar) at the largest supported sizes.  Applies to
 *     problems large enough for the 256-channel GEMM tiles; smaller ones run three passes everywhere.
 *   ST_PRECISION_BF16X3: three passes everywhere: the round-1 behaviour, for callers who want
 *     the widest margin.  The environment variable STABLETTS_B200_PRECISION=bf16x3|ffn_fp16x2 sets the initial mode.
 *   The adaptive solvers (st_solve_adaptive[_ex]) always evaluate the vector field in ST_PRECISION_BF16X3: their step-size
 *   controller compares an error estimate with rtol = atol = 1e-5, below the two-pass mode's evaluation noise. */
enum { ST_PRECISION_BF16X3 = 0, ST_PRECISION_FFN_FP16X2 = 1 };
int st_set_precision(st_handle* h, int precision);

/* Workspace: bytes needed for a (B, T) problem (cfg != 0 doubles the estimator batch), and
 * attachment of a caller-owned device buffer of at least that size (e.g. a torch uint8 tensor).
 * The buffer must stay alive until the next attach or st_destroy. */
size_t st_workspace_bytes(const st_handle* h, int B, int T, int cfg);
int st_attach_workspace(st_handle* h, void* dev_ptr, size_t bytes);

/* Replaces: Decoder.forward(t, x, mask, mu, c) (models/estimator.py:103-137).
 *   t: device fp32, t_count == 1 (the 0-dim t of odeint) or == B (training-style per-sample t)
 *   x, mu, out: (B, n_mel, T);  mask: (B, T);  c: (B, gin). */
int st_estimator_forward(st_handle* h, const float* t, int t_count, const float* x, const float* mask,
                         const float* mu, const float* c, float* out, int B, int T, void* stream);

/* Replaces: the forward VALUE of CFMDecoder.compute_loss (models/flow_matching.py:69-100) in eval mode (no dropout,
 * no autograd): given the caller's draws t (B values, already cosine-warped, :92-93) and z (:96) it forms
 * y = (1-(1-sigma_min) t) z + t x1 (written to y_out, (B, n_mel, T)), evaluates the estimator at per-sample t and writes
 * sum((v - u)^2) / (sum(mask) * n_mel), u = x1 - (1-sigma_min) z, to the DEVICE scalar loss_out.  No host sync. */
int st_cfm_loss(st_handle* h, const float* x1, const float* z, const float* t, const float* mask, const float* mu,
                const float* c, float sigma_min, float* y_out, float* loss_out, int B, int T, void* stream);

/* Replaces: CFMDecoder.forward's `odeint(estimator | cfg_wrapper, z, t_span, method=solver)` and
 * `trajectory[-1]` (models/flow_matching.py:46-55) together with cfg_wrapper (:58-67).
 *   z_inout: (B, n_mel, T) — in: z = randn_like(mu)*temperature (UNMASKED, :45); out: the sample
 *   fake_content (n_mel) / fake_speaker (gin): device, or NULL for no CFG (cfg_kwargs is None)
 *   t_span_host: n_steps+1 fp32 values on the HOST (torch.linspace(0,1,n+1), :46)
 * The whole solve is device-resident: no host synchronisation between steps. */
int st_solve(st_handle* h, float* z_inout, const float* mu, const float* mask, const float* c,
             const float* fake_content, const float* fake_speaker, float cfg_strength,
             const float* t_span_host, int n_steps, int method, int B, int T, void* stream);

/* Replaces the reference's DEFAULT solver: `odeint(..., method=None)` = torchdiffeq's adaptive dopri5 with
 * rtol = atol = 1e-5 (models/flow_matching.py:54).  torchdiffeq is absent/unpinned: this follows its published
 * algorithm (see oracle/adaptive_ref.py; parity unpinned).  One 8-byte host read per step (accept/reject), as
 * torchdiffeq itself does on a GPU.  stats (host, may be NULL): [accepted steps, rejected steps, NFE]. */
int st_solve_adaptive(st_handle* h, float* z_inout, const float* mu, const float* mask, const float* c,
                      const float* fake_content, const float* fake_speaker, float cfg_strength, double t_start,
                      double t_end, double rtol, double atol, int max_steps, int B, int T, void* stream, int64_t* stats);

/* The other adaptive `solver` strings the reference's UI offers (webui.py:110) are further embedded tableaux on the
 * same controller: Bogacki–Shampine 3(2) ("bosh3"), Fehlberg 2(1) ("fehlberg2"), Heun–Euler 2(1) ("adaptive_heun");
 * stats: [accepted, rejected, NFE] with NFE = 2 + stages*(accepted+rejected).  "implicit_adams" (a multistep
 * predictor-corrector with its own history) is NOT built: the Python surface raises for it. */
enum { ST_ADAPT_DOPRI5 = 0, ST_ADAPT_BOSH3 = 1, ST_ADAPT_FEHLBERG2 = 2, ST_ADAPT_HEUN = 3 };
int st_solve_adaptive_ex(st_handle* h, int method, float* z_inout, const float* mu, const float* mask, const float* c,
                         const float* fake_content, const float* fake_speaker, float cfg_strength, double t_start,
                         double t_end, double rtol, double atol, int max_steps, int B, int T, void* stream, int64_t* stats);

/* Same as st_solve with HOST buffers: copies inputs host->device and the sample device->host on
 * `stream` and synchronises it before returning (the end-to-end form bench.py's `e2e` times).  Page-locked host
 * buffers are copied from/to directly; pageable ones are staged through a pinned buffer the handle owns. */
int st_solve_host(st_handle* h, float* z_inout_host, const float* mu_host, const float* mask_host,
                  const float* c_host, const float* fake_content_host, const float* fake_speaker_host,
                  float cfg_strength, const float* t_span_host, int n_steps, int method, int B, int T,
                  void* stream);
/* The same with separate noise input and sample output buffers (a serving loop keeps its request buffers intact). */
int st_solve_host_io(st_handle* h, const float* z_in_host, float* out_host, const float* mu_host, const float* mask_host,
                     const float* c_host, const float* fake_content_host, const float* fake_speaker_host,
                     float cfg_strength, const float* t_span_host, int n_steps, int method, int B, int T,
                     void* stream);

/* ---- caller-side glue (SURVEY.md §8 row f1): StableTTS.synthesise's duration -> alignment -> mu_y ----
 * Replaces models/model.py:83-85 + the cumsum of generate_path (:19):
 *   logw, x_mask: (B, Tx) device fp32 (the reference's (B,1,Tx));  cum out (B, Tx) fp32 cumulative
 *   ceil-durations;  y_lengths out (B) int64 = clamp_min(sum(ceil(exp(logw)*mask)*length_scale), 1). */
int st_align_lengths(const float* logw, const float* x_mask, float length_scale, int B, int Tx, float* cum,
                     int64_t* y_lengths, void* stream);
/* Replaces models/model.py:89-95 (sequence_mask, generate_path :17-27, attn^T·mu_x as a gather):
 *   mu_x (B, M, Tx) -> mu_y (B, M, Ty), y_mask (B, Ty); attn (B, Tx, Ty) dense path or NULL. */
int st_align_expand(const float* mu_x, const float* x_mask, const float* cum, const int64_t* y_lengths, int B, int M,
                    int Tx, int Ty, float* mu_y, float* y_mask, float* attn, void* stream);

/* ---- SURVEY.md §8 row f2: TextEncoder (models/text_encoder.py:8-44) on the same kernels ---------------
 * dims: n_mel = out_channels, n_layers = n_enc_layers (3).  Weights are loaded with st_load_weight under the
 * reference keys relative to `encoder.`: "emb.weight", "encoder.{i}.attn.conv_{q,k,v,o}.{weight,bias}",
 * "encoder.{i}.mlp.conv_{1,2}.*", "encoder.{i}.adaLN_modulation.2.*", "proj.*"; then st_finalize_weights. */
int st_create_text_encoder(const st_dims* dims, int n_vocab, int device, st_handle** out);
/* Replaces TextEncoder.forward(x, c, x_lengths) (:34-44): ids (B,T) int64, c (B,gin), x_lengths (B) int64 ->
 * x_out (B, hidden, T), mu_out (B, n_mel, T), mask_out (B, T). */
int st_text_encoder_forward(st_handle* h, const int64_t* ids, const float* c, const int64_t* x_lengths, float* x_out,
                            float* mu_out, float* mask_out, int B, int T, void* stream);

/* ---- SURVEY.md §8 row f4: the vocoder hand-off, api.py:76 `self.vocoder_model(mel_output)` --------------------------
 * Replaces Vocos.__init__ / forward (vocoders/vocos/models/model.py:11-20: VocosBackbone backbone.py:21-56, ConvNeXtBlock
 * module.py:15-46, ISTFTHead / ISTFT with "same" padding head.py:21-117).  dims = VocosConfig + MelConfig
 * (vocoders/vocos/config.py): input_channels, dim, intermediate_dim, num_layers, n_fft, hop_length.
 * Weights are loaded with st_load_weight under the reference's state_dict keys ("backbone.embed.weight",
 * "backbone.norm.*", "backbone.convnext.{i}.{gamma,dwconv.*,norm.*,pwconv1.*,pwconv2.*}", "backbone.final_layer_norm.*",
 * "head.out.*", "head.istft.window"), then st_finalize_weights.  The handle owns its workspace. */
typedef struct st_vocos_dims {
    int32_t n_mel, dim, intermediate, n_layers, n_fft, hop;
} st_vocos_dims;
int st_create_vocos(const st_vocos_dims* dims, int device, st_handle** out);
/* mel (B, n_mel, T) device fp32 -> audio (B, T * hop) device fp32; enqueued on `stream`, no host synchronisation
 * (except when the internal workspace has to grow). */
int st_vocos_forward(st_handle* h, const float* mel, float* audio, int B, int T, void* stream);

/* Number of kernels this library launched since the handle was created (bench.py gpu_launches). */
int64_t st_launch_count(const st_handle* h);

/* Per-kernel-class CUDA-event profiling (bench.py's roofline): between begin and end every launch of
 * the listed classes is bracketed by events on the launching stream.  st_profile_end synchronises
 * the device and fills four arrays of ST_PROF_NCAT entries: summed milliseconds, algorithmic FLOPs,
 * algorithmic bytes and launch counts per class. */
enum { ST_PROF_GEMM = 0 /* in_proj, final_proj, test hooks */, ST_PROF_ATTN = 1 /* prep + attention */, ST_PROF_LN = 2,
       ST_PROF_GEMM_QKV = 3, ST_PROF_GEMM_O = 4, ST_PROF_GEMM_C1 = 5, ST_PROF_GEMM_C2 = 6, ST_PROF_GEMM_LSC = 7,
       ST_PROF_GEMM_COND = 8 /* per-solve cond_proj + in_proj mu-half */, ST_PROF_NCAT = 9 };
int st_profile_begin(st_handle* h);
int st_profile_end(st_handle* h, double* ms, double* flops, double* bytes, int64_t* launches);
/* Tensor-core FLOPs ISSUED per class by the launches of the last st_profile_begin/end bracket (ST_PROF_NCAT entries):
 * algorithmic FLOPs x the number of MMA passes of the operand precision (3 for split-bf16, 2 for the fp16 two-pass
 * convs; 0 for classes without tensor-core GEMM launches).  issued / time against the bf16 peak is the tensor-pipe
 * utilisation; flops / time is the algorithmic roofline figure. */
int st_profile_issued(st_handle* h, double* issued);

/* ---- kernel-level test hooks (used by tests/ only; same kernels the path uses) ------------- */

/* out(R,N) = [silu]( A(R,K)·W(N,K)^T + bias ) through the selected engine's conv-GEMM with
 * taps==1: exercises the wgmma/TMA pipeline in isolation.  All device fp32, row-major. */
int st_test_gemm(st_handle* h, const float* A, const float* W, const float* bias, float* out,
                 int R, int K, int N, int silu, void* stream);

/* k-tap conv1d, zero padded: x (B,Cin,T), w (Cout,Cin,k), out (B,Cout,T) — reference layouts. */
int st_test_conv(st_handle* h, const float* x, const float* w, const float* bias, float* out,
                 int B, int Cin, int Cout, int T, int k, void* stream);

/* Times `reps` launches of the selected engine's conv-GEMM on device-generated synthetic operands:
 * (B,T,Cin) x [k][Cout][Cin] -> (B,T,Cout); epi != 0 uses the conv_2-style epilogue (bias, mask, gate,
 * residual, fp32 + split-bf16 outputs), epi == 2 the conv_1-style one (bias, SiLU, mask, split-bf16 output), epi == 0 bias +
 * split-bf16 output.  *ms_out = ms per launch. */
int st_bench_conv(st_handle* h, int B, int Cin, int Cout, int T, int k, int epi, int reps, float* ms_out);

/* Masked multi-head attention with partial RoPE on packed qkv (B,T,3*hidden) -> (B,T,hidden). */
int st_test_attention(st_handle* h, const float* qkv, const float* mask, float* out, int B, int T,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STABLETTS_B200_H_ */
