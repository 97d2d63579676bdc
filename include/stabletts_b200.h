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

/* Library/ABI version (major*10000 + minor*100 + patch): 2.8.0 = 20800. */
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
 *     problems large enough for the 256-channel GEMM tiles; smaller ones run three passes everywhere.  fp16 hi / lo planes
 *     represent a weight only while |w| < 65520 (beyond it hi rounds to inf and every output the weight touches would be
 *     NaN): a model with a conv_1, conv_2 or long-skip weight outside that range, or a NaN one, runs three passes
 *     everywhere, exactly as ST_PRECISION_BF16X3.  st_finalize_weights decides this anew at every (re-)finalize.
 *   ST_PRECISION_BF16X3: three passes everywhere: the round-1 behaviour, for callers who want
 *     the widest margin.
 *   The adaptive solvers (st_solve_adaptive[_ex]) always evaluate the vector field in ST_PRECISION_BF16X3: their step-size
 *   controller compares an error estimate with rtol = atol = 1e-5, below the two-pass mode's evaluation noise. */
enum { ST_PRECISION_BF16X3 = 0, ST_PRECISION_FFN_FP16X2 = 1 };
int st_set_precision(st_handle* h, int precision);

/* Workspace: bytes needed for a (B, T) problem (cfg != 0 doubles the estimator batch), and
 * attachment of a caller-owned device buffer of at least that size (e.g. a torch uint8 tensor).
 * The buffer must stay alive until the next attach or st_destroy.
 * st_workspace_bytes is 0 for a handle that is neither a CFM estimator nor a text encoder. */
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
 *   logw, x_mask: (B, Tx) device fp32 (the reference's (B,1,Tx));  cum out (B, Tx) fp32 cumulative (accumulated in double,
 *   each prefix rounded to fp32: torch.cumsum's CPU result)
 *   ceil-durations;  y_lengths out (B) int64 = clamp_min(sum(ceil(exp(logw)*mask)*length_scale), 1). */
int st_align_lengths(const float* logw, const float* x_mask, float length_scale, int B, int Tx, float* cum,
                     int64_t* y_lengths, void* stream);
/* Replaces models/model.py:89-95 (sequence_mask, generate_path :17-27, attn^T·mu_x as a gather):
 *   mu_x (B, M, Tx) -> mu_y (B, M, Ty), y_mask (B, Ty); attn (B, Tx, Ty) dense path or NULL. */
int st_align_expand(const float* mu_x, const float* x_mask, const float* cum, const int64_t* y_lengths, int B, int M,
                    int Tx, int Ty, float* mu_y, float* y_mask, float* attn, void* stream);

/* ---- SURVEY.md §8 row f8: monotonic alignment search of StableTTS's training forward ---------------------------------
 * Handle-less like st_align_*: each runs on the device of its pointers, is enqueued on `stream`, never synchronises the
 * host and never allocates.  Scratch is a caller device buffer of at least st_mas_workspace_bytes(B, Ty, Tx) bytes (one
 * size serves st_maximum_path and st_mas_losses); it may be 0 for an empty problem.  Errors go to st_last_error(NULL). */
size_t st_mas_workspace_bytes(int B, int Ty, int Tx);
/* Replaces the `neg_cent` of models/model.py:150-155 (s_p_sq_r = 1):
 *   y (B, D, Ty), mu_x (B, D, Tx) -> neg_cent (B, Ty, Tx) = -0.5 log(2π) D - 0.5 Σ_d y² + Σ_d y·mu_x - 0.5 Σ_d mu_x²,
 *   the four terms summed left to right in fp32 (each contraction an fp32 FMA chain over d, not torch's einsum order). */
int st_mas_scores(const float* y, const float* mu_x, float* neg_cent, int B, int D, int Ty, int Tx, void* stream);
/* Replaces monotonic_align.maximum_path(neg_cent, mask) (monotonic_align/__init__.py:7-16, core.py:14-46), bit for bit:
 *   neg_cent (B, Ty, Tx) fp32.  Lengths come from EITHER mask (B, Ty, Tx) fp32 — t_y = (int) Σ_y mask[b,y,0],
 *   t_x = (int) Σ_x mask[b,0,x], as the reference derives them — OR from x_lengths / y_lengths (B) int64 with mask NULL,
 *   which gives the lengths the training forward's mask x_mask ⊗ y_mask would (model.py:157: both 0 when either is 0).
 *   Outputs, each optional (NULL): path (B, Ty, Tx) fp32 0/1; dur (B, Tx) fp32 frames per token (attn.sum(2),
 *   model.py:162); cum (B, Tx) fp32 inclusive prefix sums of dur (st_align_expand's `cum`).
 *   Degenerate lengths behave as the reference: t_x > t_y walks the raw scores (row -1 read as row Ty-1, numpy's
 *   wrap-around); t_y == 0 gives an all-zero path.  t_x == 0 with t_y > 0 (a mask whose row 0 is empty while column 0 is
 *   not: no product of two prefix masks) makes the reference read out of bounds; here the path is all zeros.
 *   Tx is limited to the rows that fit in shared memory (9632 tokens); Ty is not limited. */
int st_maximum_path(const float* neg_cent, const float* mask, const int64_t* x_lengths, const int64_t* y_lengths, float* path,
                    float* dur, float* cum, void* ws, size_t ws_bytes, int B, int Ty, int Tx, void* stream);
/* Replaces the two closed-form losses of the training forward, eval mode (model.py:162-163 with duration_predictor.py:38-40,
 * and :175-176), written to device scalars:
 *   prior_loss = Σ 0.5 ((y - mu_y)² + log 2π) y_mask / (Σ y_mask · M)       y, mu_y (B, M, Ty); y_mask (B, Ty)
 *   dur_loss   = Σ (logw - log(1e-8 + dur) x_mask)² / Σ x_lengths           logw, x_mask, dur (B, Tx); x_lengths (B) int64
 * Each term in fp32 as the reference forms it, summed in double in a fixed order (repeatable bit for bit). */
int st_mas_losses(const float* y, const float* mu_y, const float* y_mask, const float* logw, const float* x_mask, const float* dur,
                  const int64_t* x_lengths, void* ws, size_t ws_bytes, int B, int M, int Ty, int Tx, float* prior_loss,
                  float* dur_loss, void* stream);

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
 * "head.out.*", "head.istft.window"), then st_finalize_weights.  The handle owns its workspace.
 * api.py's get_vocoder builds Vocos(VocosConfig(), MelConfig()) from the reference's top-level config.py (dim 512,
 * intermediate 1536, 8 layers); vocoders/vocos/config.py (768 / 2048 / 12) is the vocos training configuration.
 * st_create_vocos accepts dim 512, 768 or 1024 and an n_fft that is a multiple of 128 and of hop, with hop < n_fft and at
 * most 16 overlapping frames.  hop == n_fft is refused: there the reference's "same" ISTFT trims nothing off an empty
 * slice and returns a (B, 0) signal.  Known difference: the reference asserts that the window envelope stays above 1e-11;
 * this library does not check a loaded window, so a window that is zero where only one frame covers a sample gives
 * non-finite audio there instead of an assertion. */
typedef struct st_vocos_dims {
    int32_t n_mel, dim, intermediate, n_layers, n_fft, hop;
} st_vocos_dims;
int st_create_vocos(const st_vocos_dims* dims, int device, st_handle** out);
/* mel (B, n_mel, T) device fp32 -> audio (B, T * hop) device fp32; enqueued on `stream`, no host synchronisation
 * (except when the internal workspace has to grow). */
int st_vocos_forward(st_handle* h, const float* mel, float* audio, int B, int T, void* stream);

/* ---- DESIGN.md §8 row f12: training the Vocos generator (vocoders/vocos/train.py:94 `audios_fake = generator(mels)`) ----
 * A forward that keeps what its backward needs, and that backward.  Both take a Vocos handle only (any other kind fails
 * with "handle is not a Vocos vocoder") whose weights are finalized; the engine (st_set_engine) must not change between
 * a forward and its backward, because it decides how `saved` holds each GEMM operand.
 *
 * st_vocos_saved_bytes: the size of `saved` for one (B, T) forward on the handle's current engine, 0 for a bad argument:
 *   4 B T (n_mel + (L + 1) dim + L (dim + intermediate) + dim + Nh) bytes, Nh = 2 ceil((n_fft/2 + 1) / 128) 128, L =
 *   n_layers, with each of its regions rounded up to 256 bytes.  It holds the mel operand, X_0 ... X_L (fp32: the output
 *   of the post-embed LayerNorm and of every ConvNeXt block), each block's LayerNorm output U and GELU(h), the final
 *   LayerNorm's output and the head output (fp32); each operand is fp32 on the SIMT engine and split-bf16 planes on the
 *   wgmma engine, 4 bytes per element either way.
 * st_vocos_forward_train: st_vocos_forward with the same launches, writing those into the caller's `saved`; its audio is
 *   bitwise equal to st_vocos_forward's.
 * st_vocos_backward: d_audio (B, T hop) device fp32 -> grads[i] OVERWRITTEN with the gradient of every parameter, in the
 *   order of the state_dict keys above without the window ("backbone.embed.weight", ".bias", "backbone.norm.weight",
 *   ".bias", then per block "gamma", "dwconv.weight", "dwconv.bias", "norm.weight", "norm.bias", "pwconv1.weight",
 *   "pwconv1.bias", "pwconv2.weight", "pwconv2.bias", then "backbone.final_layer_norm.weight", ".bias", "head.out.weight",
 *   ".bias": 8 + 9 L pointers), each in the reference's layout.  The mel gradient is not computed.  It reads only `saved`
 *   (unchanged) and the handle's weights, which must be those of the forward.  The first backward after each
 *   st_finalize_weights makes the transposed weight packs of the input-gradient GEMMs (pwconv1, pwconv2, the head, the
 *   inverse-DFT basis); inference never makes them.  Every sum over rows runs in a fixed order without atomics: a
 *   repeated backward is bitwise identical.  Enqueued on `stream` with no host synchronisation except when its internal
 *   scratch has to grow (as st_vocos_forward's workspace does). */
size_t st_vocos_saved_bytes(st_handle* h, int B, int T);
int st_vocos_forward_train(st_handle* h, const float* mel, float* audio, int B, int T, void* saved, void* stream);
int st_vocos_backward(st_handle* h, const void* saved, const float* d_audio, int B, int T, float* const* grads, void* stream);

/* The backward's row kernels and packings (vocos_grad.cu) through the library's own launchers, one kernel per call
 * (kernel-level tests; any handle kind works: the hook needs only the device).  Buffers are caller-owned device memory,
 * NULL = not given; fp32, rows contiguous; rows = B T unless stated.
 *   FRAME_GRAD: x = g (B, T hop), w = window (n_fft) -> out_f32 = dF (B T, n_fft): g[b, s] / env[s], s = t hop + n - pad
 *     inside [0, T hop), else 0; env[s] = sum of window[n']^2 over the frames covering s (pad = (n_fft - hop) / 2).
 *   SPECTRUM_GRAD: x = dS (rows, K2), x1 = the head output (rows, Nh) -> out_f32 (rows, Nh): dm at [0, K), dp at
 *     [Kp, Kp + K), 0 at the other columns (the formulas at st_vocos_backward's contract, DESIGN.md row f12).
 *   LN_BWD: x (B, T, C), C = 512, 768 or 1024, w / bias = the depthwise taps [7][C] / bias (C) or NULL, x1 = ln_w (C),
 *     x2 = g (B, T, C), eps -> out_f32 = dx, out2_f32 = zhat or NULL: the LayerNorm backward over z = dwconv(x) (w given)
 *     or z = x.
 *   DWCONV_ADJ: x = dz (B, T, C), w = [7][C], C % 4 == 0 -> out_f32 (B, T, C) += sum_k w[k][c] dz[t + 3 - k, c]
 *     (frames inside the utterance; out_f32 holds the residual gradient on entry).
 *   COL_SUM: x = a (rows, C), x1 = b (rows, C) or NULL -> out_f32 (C) = sum_r a[r, c] b[r, c] (or a[r, c]).
 *   DWCONV_WGRAD: x = dz, x1 = the conv input, both (B, T, C) -> out_f32 = dw (C, 1, 7), out2_f32 = db (C).
 *   SCALE_COLS: x (rows, C), w = gamma (C) -> out_f32 = x gamma.
 *   GELU_BWD: x = dg, x1 = h (rows elements) -> out_f32 = dg (Phi(h) + h phi(h)).
 *   TRANSPOSE_ROWS: x (B, T, C) fp32 or x_hi / x_lo split planes, taps 1 or 7, ones 0 / 1, Nd >= taps C + ones, Kr >= B T
 *     -> out_f32 and / or out_hi / out_lo [Nd][Kr] (planes only for a planes source): row k C + c, column r = x[r + k - 3
 *     (taps 7) or r, c] inside r's utterance, else 0; row taps C = 1 on columns < B T with ones; everything else 0.
 *   WGRAD_UNPACK: x = dWp [Np][taps C + 8], Nref, taps, split, Kp -> out_f32 = gw (Nref, C, taps) = dWp[m(n)][k C + c],
 *     out2_f32 = gb (Nref) = dWp[m(n)][taps C]; m(n) = n, or Kp + n - split for n >= split when split > 0.
 * Returns non-zero with st_last_error set when an input or output the kind needs is NULL, the kind is unknown or the
 * launcher refuses the shape.  Synchronises `stream`. */
enum { ST_TEST_VOCOS_GRAD_FRAME_GRAD = 0, ST_TEST_VOCOS_GRAD_SPECTRUM_GRAD = 1, ST_TEST_VOCOS_GRAD_LN_BWD = 2,
       ST_TEST_VOCOS_GRAD_DWCONV_ADJ = 3, ST_TEST_VOCOS_GRAD_COL_SUM = 4, ST_TEST_VOCOS_GRAD_DWCONV_WGRAD = 5,
       ST_TEST_VOCOS_GRAD_SCALE_COLS = 6, ST_TEST_VOCOS_GRAD_GELU_BWD = 7, ST_TEST_VOCOS_GRAD_TRANSPOSE_ROWS = 8,
       ST_TEST_VOCOS_GRAD_WGRAD_UNPACK = 9 };
typedef struct st_test_vocos_grad_desc {
    const float *x, *x1, *x2, *w, *bias;
    const uint16_t *x_hi, *x_lo;
    float *out_f32, *out2_f32;
    uint16_t *out_hi, *out_lo;
    int64_t rows, Kr;
    int32_t kind, B, T, C, n_fft, hop, Nh, Kp, K, K2, taps, ones, Nd, Nref, split;
    float eps;
} st_test_vocos_grad_desc;
int st_test_vocos_grad_ex(st_handle* h, const st_test_vocos_grad_desc* d, void* stream);

/* ---- the FireflyGAN vocoder, the reference's DEFAULT vocoder (api.py get_vocoder / StableTTSAPI, vocoder_name='ffgan') ----
 * Replaces FireflyGANBase.__init__ / forward (vocoders/ffgan/model.py:45-56) at its one configuration (config_dict,
 * model.py:7-29): ConvNeXtEncoder (backbone.py:146-214: k = 7 stem conv, channels-first LayerNorms, 1x1 downsample convs,
 * 3 / 3 / 9 / 3 ConvNeXt blocks at 128 / 256 / 384 / 512 channels) and HiFiGANGenerator (head.py:137-249 with
 * use_template = False: weight-normed conv_pre k = 13, five SiLU -> ConvTranspose1d ups (u = 8, 8, 2, 2, 2), five
 * ParralelBlocks of three ResBlock1 (k = 3, 7, 11; dilations 1 / 3 / 5), SiLU -> conv_post k = 13 -> tanh).  No dims: the
 * reference supports no other configuration.  Weights are loaded with st_load_weight under the reference's state_dict
 * keys, weight-normed convs as their parametrization ("head.ups.{i}.parametrizations.weight.original0" = g,
 * "...original1" = v), then st_finalize_weights folds W = g v / ||v|| (norm over all dims but dim 0, which is C_in for
 * the ConvTranspose1d weights) and packs every transposed conv as a 3-tap polyphase conv at its input rate. */
int st_create_ffgan(int device, st_handle** out);
/* mel (B, 128, T) device fp32 -> audio (B, T * 512) device fp32; enqueued on `stream`, no host synchronisation except
 * when the handle-owned workspace has to grow.  st_ffgan_workspace_bytes gives its size: eight slots of 8192 fp32 values
 * per mel frame, 256 KB per frame (B = 32, T = 1000: 8.4 GB). */
int st_ffgan_forward(st_handle* h, const float* mel, float* audio, int B, int T, void* stream);
size_t st_ffgan_workspace_bytes(const st_handle* h, int B, int T);

/* ---- the front end of StableTTS.synthesise (models/model.py:78-80): speaker vector and token durations ------------------
 * Replaces MelStyleEncoder.__init__ / forward (models/reference_encoder.py:25-92) as StableTTS builds it (models/model.py:38:
 * style_hidden 128, style_vector_dim 256, style_kernel_size 5, 2 heads; eval mode).  Weights are loaded with st_load_weight
 * under the reference keys relative to `ref_encoder.` ("spectral.{0,3}.*", "temporal.{0,1}.conv1.*",
 * "slf_attn.in_proj_weight", "slf_attn.in_proj_bias", "slf_attn.out_proj.*", "fc.*"), then st_finalize_weights (which folds
 * the softmax scale into the packed q rows).  n_mel: a positive multiple of 16. */
int st_create_style_encoder(int n_mel, int device, st_handle** out);
/* y (B, n_mel, T) device fp32 reference mel, y_mask (B, T) or NULL (the `x_mask=None` of synthesise, model.py:79: every frame
 * is a key and the mean runs over all T) -> c_out (B, 256).  The Conv1dGLU convs are unmasked, as in the reference.  Enqueued
 * on `stream`; no host synchronisation (the handle's workspace grows stream-ordered). */
int st_style_encoder_forward(st_handle* h, const float* y, const float* y_mask, float* c_out, int B, int T, void* stream);
/* Replaces DurationPredictor.__init__ / forward (models/duration_predictor.py:5-36) as StableTTS builds it (model.py:39):
 * dims: hidden = in_channels = 256, filter = 1024, kernel = 3, gin = 256 (the other fields are ignored).  Weights under the
 * reference keys relative to `dp.` ("conv1.*", "norm1.*", "conv2.*", "norm2.*", "proj.*", "cond.*"), then
 * st_finalize_weights.  An utterance's logw does not depend on the other utterances of the batch (no split-K). */
int st_create_duration_predictor(const st_dims* dims, int device, st_handle** out);
/* x (B, 256, Tx) text encoding, x_mask (B, Tx), g (B, 256) speaker vector -> logw_out (B, Tx) (the reference's (B, 1, Tx)).
 * Enqueued on `stream`; no host synchronisation. */
int st_duration_predictor_forward(st_handle* h, const float* x, const float* x_mask, const float* g, float* logw_out, int B,
                                  int Tx, void* stream);

/* ---- the reference-audio front end (api.py:72-73) and the corpus feature extractor (preprocess.py:50-73) ------------------
 * Replaces utils/audio.py::LogMelSpectrogram / LinearSpectrogram (center = False, pad_mode "reflect", win_length = n_fft):
 * F.pad(reflect, pad) -> frames of n_fft every hop_length -> window -> rfft -> sqrt(re^2 + im^2 + 1e-6) [-> mel_scale.fb ->
 * log(clamp(., 1e-5))].  n_fft: a power of two in [32, 4096]; n_mels = 0 makes a handle for the linear spectrogram only.
 * Weights under the reference's state_dict keys: "spectrogram.window" (n_fft) and, when n_mels > 0, "mel_scale.fb"
 * (n_fft / 2 + 1, n_mels), then st_finalize_weights (builds the twiddles and packs each filter's non-zero band from the
 * loaded fb).  The whole transform runs in fp32 CUDA cores; st_set_engine has no effect on this handle. */
typedef struct st_mel_dims {
    int32_t n_fft, hop_length, pad, n_mels;
} st_mel_dims;
int st_create_mel(const st_mel_dims* dims, int device, st_handle** out);
/* wav (B, L) device fp32 -> out (B, n_mels, T) log-mel, or (B, n_fft / 2 + 1, T) magnitude when `linear` != 0, with
 * T = (L + 2 pad - n_fft) / hop_length + 1.  Needs pad < L (torch's reflect padding) and L + 2 pad >= n_fft.  A batch row's
 * output depends only on that row.  Enqueued on `stream`; no host synchronisation. */
int st_mel_forward(st_handle* h, const float* wav, float* out, int B, int64_t L, int linear, void* stream);

/* ---- the Vocos training loss (vocoders/vocos/train.py:115, models/loss.py:10-35) ---------------------------------------
 * Replaces MultiScaleMelSpectrogramLoss / SingleScaleMelSpectrogramLoss: loss = Σ_s mean |mel_s(x) − mel_s(y)|, scales in
 * ascending order, with mel_s the log-mel of st_mel_forward at dims[s] (n_mels > 0), bit for bit.  Weights under the
 * reference keys "mel_transforms.{s}.spectrogram.window" and "mel_transforms.{s}.mel_scale.fb", then st_finalize_weights.
 * At most 16 scales; a scale whose frames do not fit one CTA's shared memory (very large n_mels) is refused. */
int st_create_mel_loss(int n_scales, const st_mel_dims* dims, int device, st_handle** out);
/* Bytes of the workspace that st_attach_workspace must give st_mel_loss_forward for (B, L) inputs: the per-CTA partial sums
 * and two sets of frame gradients, 8 · Σ_s B · T_s · n_fft_s bytes for the latter (B = 32, L = 20480, 7 scales: 147 MB). */
size_t st_mel_loss_workspace_bytes(const st_handle* h, int B, int64_t L);
/* x, y (B, L) device fp32 -> *loss_out (device fp32 scalar) and, when gx / gy are not NULL, d loss / dx and d loss / dy
 * (B, L) for a unit upstream gradient.  Needs pad < L and L + 2 pad >= n_fft at every scale.  Partial sums are reduced in
 * double in a fixed order and every gradient sample sums its frame contributions in a fixed order: no float atomics, so a
 * repeated call is bitwise identical.  Enqueued on `stream`; no host synchronisation. */
int st_mel_loss_forward(st_handle* h, const float* x, const float* y, int B, int64_t L, float* loss_out, float* gx, float* gy,
                        void* stream);

/* ---- the Vocos multi-period discriminator (vocoders/vocos/models/discriminator.py:33-79, DiscriminatorP) ---------------
 * One handle per period p.  Input x (B, L) device fp32; when L % p != 0 it is reflect-padded on the right by p - L % p
 * samples (needs p - L % p < L) and viewed as (B, 1, H, p), H = ceil(L / p).  Layer i maps H[i-1] rows to H[i]:
 * convs 0-3 (kernel (5, 1), stride 3, pad 2) give H[i] = ceil(H[i-1] / 3), conv 4 (stride 1) and conv_post keep H.
 * Channels: 1 -> 32 -> 128 -> 512 -> 1024 -> 1024 -> 1, each conv but conv_post followed by leaky ReLU 0.1.
 * Weights are the EFFECTIVE (weight-normed) conv weights, index 0-4 = convs.0-4 (C_out, C_in, 5) and 5 = conv_post
 * (1, 1024, 3), with their biases; they are read and packed on every call, so no state carries over between calls.
 * "fmaps" are the post-activation outputs of convs 0-4, (B, C_i, H[i], p) each, and post (B, 1, H[4], p): the reference's
 * fmap list is fmaps 1-4 and post, its score post flattened.  Convs 1-4 and their gradients run on the engine that
 * st_set_engine selects (wgmma: split-bf16 operands in three passes; SIMT: fp32); convs 0 and conv_post are fp32 kernels.
 * Every reduction runs in a fixed order and there are no atomics: a repeated call is bitwise identical.  The workspace
 * (st_attach_workspace) is scratch only; calls with a handle must be ordered on one stream. */
int st_create_mpd(int period, int device, st_handle** out);
/* Bytes of the workspace st_mpd_forward / st_mpd_backward need for (B, L) on the handle's current engine; 0 for a handle of
 * another kind or a bad shape.  (B = 32, L = 20480, p = 2: about 0.5 GB.) */
size_t st_mpd_workspace_bytes(const st_handle* h, int B, int64_t L);
/* w[6], b[6]: device pointers (host arrays) of the weights above; fmaps[6]: outputs, fmaps of convs 0-4 then post.
 * Errors: B outside [1, 65535], B p > 65535, L outside [1, 2^30] or too short for the reflect pad, a NULL pointer,
 * a workspace below st_mpd_workspace_bytes.  Enqueued on `stream`; no host synchronisation. */
int st_mpd_forward(st_handle* h, const float* x, int B, int64_t L, const float* const* w, const float* const* b,
                   float* const* fmaps, void* stream);
/* The gradients of one forward call: x, w and fmaps[0..4] as that call had them; gpost (B, 1, H[4], p) the gradient of
 * post (score and last fmap together); gfmaps[4] (host array, may be NULL, entries may be NULL = zero) the gradients of
 * the fmaps of convs 1-4.  Writes gx (B, L) unless NULL (the reflect pad's samples fold back onto x[L - 2 - i]) and, unless
 * gw and gb are NULL, the weight and bias gradients gw[6] / gb[6] in the layouts of w and b.  At least one of them is
 * wanted.  The leaky ReLU's slope is read from the sign of the saved fmap.  Enqueued on `stream`; no host sync. */
int st_mpd_backward(st_handle* h, const float* x, int B, int64_t L, const float* const* w, const float* const* fmaps,
                    const float* gpost, const float* const* gfmaps, float* gx, float* const* gw, float* const* gb, void* stream);

/* ---- the multi-resolution discriminator of Vocos training (vocoders/vocos/models/discriminator.py:112-171) -------------
 * One handle per DiscriminatorR(window_length = n_fft) (n_fft a power of two in [256, 4096]); MultiResolutionDiscriminator
 * (lines 78-109) runs three.  Replaces, per call of train.py:102 / :123:
 *   spectrogram (lines 142-154): spec (B, 2, T', F) = [re, im] of torchaudio Spectrogram(n_fft, hop = n_fft / 4, power =
 *     None): centred frames (reflect pad n_fft / 2 on both sides, so L > n_fft / 2), the window buffer given (`window`,
 *     n_fft floats: the module's loaded spec_fn.window), not normalised, one-sided; T' = L / hop + 1, F = n_fft / 2 + 1.
 *     Band k is bins [int(b0 F), int(b1 F)) of (0, .1, .25, .5, .75, 1).
 *   per band (lines 158-166): convs 0-4 ((3, 9) pad (1, 4); three (3, 9) stride (1, 2) pad (1, 4); (3, 3) pad (1, 1)),
 *     each followed by leaky_relu(0.1); widths W0 = band width, W_i = ceil(W_{i-1} / 2) for i = 1-3, W4 = W3
 *   conv_post (lines 167-169) over the band outputs concatenated along F: its frequency taps read the neighbouring band.
 * Weights are the EFFECTIVE (weight-normed) conv weights, index 5 k + i = band_convs.k.i (32, C_in, 3, kw) and 25 =
 * conv_post (1, 32, 3, 3), with their biases; they are read and packed on every call.  "fmaps" are the post-activation
 * outputs of every band conv, index 5 k + i, (B, 32, T', W_i) each: the reference's fmap list is entries 5 k + 1..4 for
 * k = 0..4, then post (B, 1, T', Σ_k W4_k), which is also the score.  Convs 1-4 and their gradients run on the engine
 * st_set_engine selects (wgmma: split-bf16 operands in three passes; SIMT: fp32); the STFT, conv 0 and conv_post are fp32
 * kernels.  Every reduction runs in a fixed order and there are no atomics: a repeated call is bitwise identical.  The
 * workspace (st_attach_workspace) is scratch only; calls with a handle must be ordered on one stream. */
int st_create_mrd(int n_fft, int device, st_handle** out);
/* Bytes of the workspace st_mrd_forward (backward = 0) or st_mrd_backward (backward != 0) needs for (B, L) on the handle's
 * current engine; 0 for a handle of another kind or a bad shape.  The backward's is larger: it holds the weight-gradient
 * GEMM's transposed operand ((5 192 + 8) x B T' W1 values, about 0.7 GB in split bf16 at B = 32, L = 20480, n_fft = 512). */
size_t st_mrd_workspace_bytes(const st_handle* h, int B, int64_t L, int backward);
/* w[26], b[26]: device pointers (host arrays) of the weights above; spec (B, 2, T', F), fmaps[25] and post: outputs.
 * Errors: B outside [1, 65535], L <= n_fft / 2 or above 2^30, B T' > 65535, a NULL pointer, a workspace below
 * st_mrd_workspace_bytes(.., 0).  Enqueued on `stream`; no host synchronisation. */
int st_mrd_forward(st_handle* h, const float* x, int B, int64_t L, const float* window, const float* const* w,
                   const float* const* b, float* spec, float* const* fmaps, float* post, void* stream);
/* The gradients of one forward call: x, window, w, spec and fmaps[25] as that call had them; gpost (B, 1, T', Σ W4) the
 * gradient of post (score and last fmap together); gfmaps[20] (host array, may be NULL, entries may be NULL = zero) the
 * gradients of the reference's fmaps 0-19 (entry 4 k + i - 1 = band k, conv i).  Writes gx (B, L) unless NULL (the STFT
 * adjoint: d_n = w_n Re Σ_k (gRe_k + i gIm_k) e^{+2πikn/N} per frame, the overlap-add of the frames, the reflect pad's
 * samples folded back onto their mirror samples) and, unless gw and gb are NULL, gw[26] / gb[26] in the layouts of w and
 * b.  At least one of them is wanted.  The leaky ReLU's slope is read from the sign of the saved fmap.  Enqueued on
 * `stream`; no host sync. */
int st_mrd_backward(st_handle* h, const float* x, int B, int64_t L, const float* window, const float* const* w,
                    const float* spec, const float* const* fmaps, const float* gpost, const float* const* gfmaps, float* gx,
                    float* const* gw, float* const* gb, void* stream);

/* ---- resampling of the reference audio (api.py:72) and of every corpus clip (preprocess.py:65) -------------------------
 * Replaces torchaudio.functional.resample(x, orig_freq, new_freq) as utils/audio.py:73 calls it (sinc_interp_hann,
 * lowpass_filter_width 6, rolloff 0.99) and torchaudio.transforms.Resample.  With g = gcd(orig, new), O = orig / g,
 * N = new / g, base = 0.99 min(O, N) and width = ceil(6 O / base) (Python float arithmetic, as torchaudio):
 *   xpad[m] = x[m - width] for 0 <= m - width < L, else 0
 *   y[i N + j] = Σ_{k = 0}^{2 width + O - 1} coef[j][k] · xpad[i O + k],  output length ceil(N L / O) (integers)
 *   t = clamp(((k - width) / O - j / N) · base, -6, 6),  coef[j][k] = sinc(t) · cos²(t π / 12) · base / O,
 *   sinc(t) = sin(π t) / (π t), 1 at t = 0.
 * st_create_resample evaluates the coefficients in double on the host and rounds each once to fp32; each phase j keeps only
 * its band [k0_j, k1_j) of non-zero coefficients.  A table of more than ST_RESAMPLE_MAX_TABLE coefficients (N x the widest
 * band) is refused: 12345 -> 44100 needs 38 220, and every pair between {8000, 11025, 16000, 22050, 24000, 32000, 44100,
 * 48000, 88200, 96000, 192000} and {16000, 22050, 24000, 44100} fits (torchaudio's dense kernel for 44101 -> 44100 would
 * take 7.8 GB).  A pair whose block of N outputs reads more than 49 152 input samples is refused too (shared memory; only
 * pairs with O in the tens of thousands).  orig_freq == new_freq is refused: resampling is the identity.
 * st_load_weight(h, "kernel", (N, 1, 2 width + O) fp32) then st_finalize_weights replaces the table by the bands of the
 * loaded buffer (torchaudio.transforms.Resample's state_dict), used exactly as loaded; st_finalize_weights reads that buffer
 * back to the host once to find its bands. */
#define ST_RESAMPLE_MAX_TABLE (1 << 18)
int st_create_resample(int32_t orig_freq, int32_t new_freq, int device, st_handle** out);
/* ceil(N L / O): the output length for L input samples; -1 for a bad handle or L < 0. */
int64_t st_resample_out_length(const st_handle* h, int64_t L);
/* x (rows, L) device fp32 -> y (rows, st_resample_out_length(L)) device fp32.  Every output sums its band in ascending k
 * with fp32 FMA; no atomics, so a repeated call is bitwise identical and a row's output depends only on that row.
 * Enqueued on `stream`; no host synchronisation (capturable in a CUDA graph). */
int st_resample_forward(st_handle* h, const float* x, float* y, int64_t rows, int64_t L, void* stream);

/* Number of kernels this library launched since the handle was created (bench.py gpu_launches). */
int64_t st_launch_count(const st_handle* h);

/* Per-kernel-class CUDA-event profiling (bench.py's roofline): between begin and end every launch of
 * the listed classes is bracketed by events on the launching stream.  st_profile_end synchronises
 * the device and fills four arrays of ST_PROF_NCAT entries: summed milliseconds, algorithmic FLOPs,
 * algorithmic bytes and launch counts per class. */
enum { ST_PROF_GEMM = 0 /* in_proj, final_proj, test hooks */, ST_PROF_ATTN = 1 /* prep + attention */, ST_PROF_LN = 2,
       ST_PROF_GEMM_QKV = 3, ST_PROF_GEMM_O = 4, ST_PROF_GEMM_C1 = 5, ST_PROF_GEMM_C2 = 6, ST_PROF_GEMM_LSC = 7,
       ST_PROF_GEMM_COND = 8 /* per-solve cond_proj + in_proj mu-half */,
       /* FireflyGAN stages: the ConvNeXt encoder, conv_pre, ups[i] + ParralelBlock i (i = 0..4), conv_post + tanh */
       ST_PROF_FFGAN_BACKBONE = 9, ST_PROF_FFGAN_PRE = 10, ST_PROF_FFGAN_STAGE0 = 11, ST_PROF_FFGAN_POST = 16,
       ST_PROF_NCAT = 17 };
int st_profile_begin(st_handle* h);
int st_profile_end(st_handle* h, double* ms, double* flops, double* bytes, int64_t* launches);
/* Tensor-core FLOPs ISSUED per class by the launches of the last st_profile_begin/end bracket (ST_PROF_NCAT entries):
 * algorithmic FLOPs x the number of MMA passes of the operand precision (3 for split-bf16, 2 for the fp16 two-pass
 * convs; 0 for classes without tensor-core GEMM launches).  issued / time against the bf16 peak is the tensor-pipe
 * utilisation; flops / time is the algorithmic roofline figure. */
int st_profile_issued(st_handle* h, double* issued);

/* ---- kernel-level test hooks (used by tests/ only; same kernels the path uses) ------------- */

/* Conv1d / ConvTranspose1d through the FireflyGAN head's conv-GEMM path (reference layouts, device fp32):
 *   transposed == 0: x (B,Cin,T), w (Cout,Cin,k), dilation `dil`, padding dil*(k-1)/2 -> out (B,Cout,T)
 *   transposed == 1: x (B,Cin,T), w (Cin,Cout,2u) with u = `dil`, stride u, padding u/2 -> out (B,Cout,u*T), run as the
 *                    3-tap polyphase conv with N = u*Cout. */
int st_test_conv_ex(st_handle* h, const float* x, const float* w, const float* bias, float* out, int B, int Cin, int Cout,
                    int T, int k, int dil, int transposed, void* stream);

/* The whole conv-GEMM contract through the selected engine (kernel-level tests of every instance and epilogue).
 *   out[bb, t, n] = epi( sum_{tap, src, k} A_src[bb % a_bmod, t + (tap - taps/2) * dil, k] * W[n, koff_src + k, tap] ),
 *   rows outside [0, T) read as zero; A0 (a_bmod, T, C0) and A1 (a_bmod, T, C1) are token-major and concatenated along
 *   channels (n_src = 2); W (N, C0 + C1, taps) is in the Conv1d layout.  Epilogue, in order: + bias[n]; SiLU or GELU (exact
 *   erf) or Mish (v tanh(softplus(v)), softplus
 *   threshold 20; 128-channel tiles); FiLM film[mb * film_bstride + n] * v + film[mb * film_bstride + film_H + n]; * mask[mb, t]; * gate[cb * gate_bstride
 *   + n]; + resid[rb, t, n] with mb = bb % B, cb = min(bb, c_clamp), rb = min(bb, resid_clamp).  ROPE (with BIAS only): the
 *   partial RoPE of the QKV projection on columns < 2 rope_H, q columns (< rope_H) scaled by log2(e) / 8.  SILU_OUT: v ->
 *   out_f32, silu(v) -> out planes / out2_f32.  ln (N = 256, wgmma engine): x2 = (film2 gamma x + beta) * mask -> out2_f32 when
 *   film2 is set, then u = LayerNorm(x2) (eps 1e-5, no affine) * (1 + ln_scale[cb]) + ln_shift[cb] [* mask] -> u planes.
 * The hook makes the operand planes itself (split bf16; with prec one fp16 A plane and fp16 hi / lo weights).
 * Outputs are caller-owned device buffers (BB, T, N), NULL = not requested: out_f32, the raw 2-byte planes out_hi / out_lo
 * (bf16 hi / lo; out16: one fp16 plane in out_hi), out2_f32, u_hi / u_lo (u16: one fp16 plane in u_hi).
 * ksplit: 0 = the library's own decision, 1 = never, 2..4 = exactly that split-K factor.  num_sms > 0: the tile-width choice
 * and the persistent grid behave as on a GPU with that many SMs.  `plan` (may be NULL) receives the launch that ran.
 * Returns non-zero with st_last_error set, launching nothing, when the problem is outside the contract. */
enum { ST_TEST_EPI_BIAS = 1, ST_TEST_EPI_SILU = 2, ST_TEST_EPI_FILM = 4, ST_TEST_EPI_MASK = 8, ST_TEST_EPI_GATE = 16,
       ST_TEST_EPI_RESID = 32, ST_TEST_EPI_ROPE = 64, ST_TEST_EPI_GELU = 128, ST_TEST_EPI_SILU_OUT = 256,
       ST_TEST_EPI_MISH = 512 };
/* st_test_gemm_plan.mode: the epilogue instance of the wgmma kernel (-1: SIMT engine) */
enum { ST_TEST_MODE_PLAIN = 0, ST_TEST_MODE_SILU = 1, ST_TEST_MODE_GELU = 2, ST_TEST_MODE_ROPE = 3, ST_TEST_MODE_LN = 4,
       ST_TEST_MODE_RESID = 5, ST_TEST_MODE_SILU_OUT = 6, ST_TEST_MODE_MISH = 7 };
typedef struct st_test_gemm_desc {
    const float *A0, *A1, *W, *bias, *mask, *film, *gate, *resid, *ln_shift, *ln_scale, *film2;
    float* out_f32; uint16_t* out_hi; uint16_t* out_lo; float* out2_f32; uint16_t* u_hi; uint16_t* u_lo;
    int64_t film_bstride, gate_bstride, ada_bstride, film2_bstride;
    int32_t B, BB, T, a_bmod, n_src, C0, C1, N, taps, dil;
    int32_t flags, c_clamp, resid_clamp, film_H, rope_H;
    int32_t ln, ln_mask_out, prec, out16, u16;
    int32_t ksplit, num_sms;
} st_test_gemm_desc;
typedef struct st_test_gemm_plan {
    int32_t engine, bn, mode, prec, ksplit, grid;   /* ST_ENGINE_*, tile width, ST_TEST_MODE_*, fp16 operands, split-K factor, CTAs */
} st_test_gemm_plan;
int st_test_gemm_ex(st_handle* h, const st_test_gemm_desc* d, st_test_gemm_plan* plan, void* stream);

/* Times `reps` launches of the selected engine's conv-GEMM on device-generated synthetic operands:
 * (B,T,Cin) x [k][Cout][Cin] -> (B,T,Cout); epi != 0 uses the conv_2-style epilogue (bias, mask, gate,
 * residual, fp32 + split-bf16 outputs), epi == 2 the conv_1-style one (bias, SiLU, mask, split-bf16 output), epi == 3 the
 * O-style one (residual, mask, gate, fp32 output + fused LayerNorm / modulate), epi == 0 bias + split-bf16 output.
 * prec = 1: the two-pass fp16 operands (ST_PRECISION_FFN_FP16X2's FFN convs; 256-channel tiles only), 2-byte outputs as
 * one fp16 plane.  *ms_out = ms per launch. */
int st_bench_conv(st_handle* h, int B, int Cin, int Cout, int T, int k, int epi, int prec, int reps, float* ms_out);

/* The whole masked multi-head attention contract (AttnArgs) through the selected engine (kernel-level tests of both engines).
 *   Operands (BB, T, 3H) are token-major; head h reads q / k / v at columns 64h, H + 64h and 2H + 64h (H = 64 n_heads).
 *   Row bb uses mask row b = bb % B (BB = B, or 2B under classifier-free guidance).  Key j counts for row bb only if
 *   j < kvlen[b] and mask[b, j] != 0 (-0.0 counts as zero), with kvlen[b] = 1 + the last index where mask[b] != 0 (0 if none)
 *   and prefix[b] = the first index where mask[b] == 0 (T if none).  A query row with mask == 0 is written as zero.
 *   wgmma engine: qkv_hi / qkv_lo are split-bf16 planes already RoPE'd and q-scaled, as the producer GEMM writes them
 *     (EPI_ROPE, or the style encoder's pre-scaled q rows); out = softmax_2(q k^T) v with softmax base 2 on the plane values
 *     hi + lo, no further scale.
 *   SIMT engine: qkv holds the raw fp32 projections; with rope the hook builds the (T, 16) cos / sin table of
 *     launch_rope_table and rotates the pairs (j, j + 16), j < 16, of every head's q and k by the frame index; then q is
 *     multiplied by 1/8 and out = softmax_e(q k^T) v with natural exp.
 * Outputs are caller-owned device buffers (BB, T, H), NULL = not requested: out_f32, and the split-bf16 planes out_hi / out_lo
 * (hi = bf16(x), lo = bf16(x - hi); together).  kvlen_out / prefix_out (B), optional, receive the lengths the mask gave.
 * Returns non-zero with st_last_error set, launching nothing, when the problem is outside the contract. */
typedef struct st_test_attn_desc {
    const float* qkv;                           /* SIMT engine: raw fp32 projections (BB, T, 3H) */
    const uint16_t *qkv_hi, *qkv_lo;            /* wgmma engine: split-bf16 planes, already RoPE'd and q-scaled */
    const float* mask;                          /* (B, T), required */
    float* out_f32; uint16_t *out_hi, *out_lo;  /* (BB, T, H); any non-empty subset, hi and lo together */
    int32_t* kvlen_out; int32_t* prefix_out;    /* optional (B) */
    int32_t BB, B, T, H, n_heads, rope;         /* rope: SIMT engine only (0 or 1) */
} st_test_attn_desc;
int st_test_attention_ex(st_handle* h, const st_test_attn_desc* d, void* stream);

/* The row kernels through the library's own launchers (kernel-level tests of the fp32 row kernels; any handle kind works:
 * the hook needs only the device).  One problem per call, selected by `kind`.  Inputs and outputs are caller-owned device
 * fp32 buffers, NULL = not requested; rows are contiguous.  Split planes: hi = bf16(v), lo = bf16(v - hi), together.
 *   ADALN (FiLM·mask -> LayerNorm -> adaLN modulate, the CFM estimator's row kernel): x (BB, T, C), C = 256, mask (B, T).
 *     For row bb: mb = bb % B, cb = min(bb, c_clamp).  With has_film: x2 = (film[mb * film_bstride + c] x
 *     + film[mb * film_bstride + C + c]) * mask[mb, t], written to xout (which may be x itself); else x2 = x.
 *     u = LayerNorm(x2, eps 1e-5, no affine) * (1 + scale[cb * ada_bstride + c]) + shift[cb * ada_bstride + c], times
 *     mask[mb, t] when mask_out.  Outputs: out_f32, the split planes, or with u16 ONE fp16 plane in out_hi:
 *     cvt.rn(clamp(u, +-65504)).  x, mask, shift and scale are 16-byte aligned.
 *   DWCONV_LN (depthwise k = 7 conv + affine LayerNorm, the vocoders' ConvNeXt row kernel): x (B, T, C),
 *     C in {128, 256, 384, 512, 768, 1024}.  w (C, 1, 7) is the reference's depthwise Conv1d weight (packed by the hook as
 *     st_finalize_weights packs it) and bias (C) its bias: y = conv1d(x, w, bias, padding 3) along T, zero padded at each
 *     utterance's own edges; with w NULL, y = x.  u = LayerNorm(y, eps) * ln_w + ln_b (the vocoders use eps 1e-6) ->
 *     out_f32 and / or the split planes.  x, w, bias, ln_w, ln_b 16-byte aligned.
 *   SPECTRUM (the Vocos head's exp / clip / cos / sin): x (B·T, Nh) with log-magnitudes m at columns [0, K) and phases p at
 *     [Kp, Kp + K) -> (B·T, K2): min(exp(m), 1e2) cos(p) at [0, K), min(exp(m), 1e2) sin(p) at [K2/2, K2/2 + K), exact
 *     zeros elsewhere; no other input column is read.  Needs K <= Kp, Kp + K <= Nh, K2 even, K <= K2/2.  Outputs: out_f32
 *     and / or the split planes.
 *   IDFT_BASIS (the Vocos inverse-DFT GEMM weight): window (n_fft) -> out_f32 (n_fft, K2), K = n_fft/2 + 1, K2 even,
 *     K <= K2/2: W[n][k] = window[n] c_k cos(2 pi k n / n_fft) / n_fft, W[n][K2/2 + k] = -window[n] c_k sin(...) / n_fft
 *     for 0 < k < K - 1 and 0 for k = 0, K - 1 (c_0 = c_{K-1} = 1, else 2); 0 in the padding.  Evaluated in double and
 *     rounded once.
 *   OVERLAP_ADD (the Vocos ISTFT's fold, envelope and "same" trim): x = frames (B, T, n_fft), window (n_fft) ->
 *     out_f32 (B, T·hop): sample s sums frames[b, t, s + pad - t hop] over the frames t in [0, T) that cover position
 *     s + pad, pad = (n_fft - hop)/2, and divides by the sum of window^2 over the same frames.  n_fft and hop as
 *     st_create_vocos accepts them.
 *   MEAN3_SILU (FireflyGAN's ParralelBlock mean + SiLU): x, x1, x2 (n) -> silu((x + x1 + x2)/3) -> out_f32 and / or the
 *     split planes; n a positive multiple of 4, buffers 16-byte aligned.
 *   POST_TANH (FireflyGAN's conv_post + tanh): x (B, T, 16) token-major, w (1, 16, 13) reference layout, bias (1) ->
 *     out_f32 (B, T) = tanh(conv1d(x, w, bias, padding 6)), zero padded at each utterance's own edges.  x 16-byte aligned.
 * The MelStyleEncoder and DurationPredictor row kernels (rows = B·T):
 *   GLU_RESID (Conv1dGLU tail): x = the conv output (rows, 2C) = [a | g], x1 = the residual (rows, C) ->
 *     x1 + a sigmoid(g) -> out_f32 and / or the split planes; C even, buffers 8-byte aligned.
 *   MASKED_MEAN (temporal pool): x (B, T, C), mask (B, T) or NULL -> out_f32 (B, C) = the sum of x over the frames with
 *     mask != 0 (all T without a mask) over their count; 0 / 0 when no frame is valid.  1 <= C <= 128.
 *   COND_TRANSPOSE (DurationPredictor input): x (B, C, T), bias = cond (B, C), mask (B, T) -> (B, T, C) token-major
 *     (x[b, c, t] + cond[b, c]) mask[b, t] -> out_f32 and / or the split planes.
 *   RELU_LN: x (B, T, C), C = 1024, ln_w, ln_b (C), mask (B, T) -> LayerNorm(relu(x), eps 1e-5, biased variance) ln_w
 *     + ln_b, times mask -> out_f32 and / or the split planes.  Buffers 16-byte aligned.
 *   RELU_LN_PROJ: as RELU_LN, then w = proj weight (C) and bias = proj bias (1) -> out_f32 (B, T) =
 *     (mask sum_c u[c] w[c] + bias) mask: logw.
 * The CFM conditioning and solver kernels:
 *   GEMV: x (B, K), w (N, K), bias (N) or NULL -> out_f32[r y_rstride + n] = act_out(sum_k act_in(x[r, k]) w[n, k]
 *     + bias[n]) for r < B, n < N; act_in / act_out are SiLU when silu_in / silu_out, else the identity.  y_rstride >= N.
 *   TIME_EMBED: x = t (n_t) on the device; TIME_EMBED_VALS: t_host = t (n_t <= 256) in host memory, passed as a kernel
 *     argument.  -> out_f32 (n_t, C): e_j = 1000 t exp(-j ln(1e4) / (C/2 - 1)), [sin e | cos e]; C even, >= 4.
 *   ROPE_TABLE: out_f32 (T, 16, 2) = (cos, sin)(pos 10000^(-2j / 32)) for pos < T, j < 16.  C = 32.
 *   LINCOMB: x = y (n), terms[0..n_terms) (n), n_terms <= 6 -> out_f32 = y + sum_j coef[j] terms[j]; out_f32 may be x.
 *   SCALED_SUMSQ: terms[0..n_terms) (n), 1 <= n_terms <= 7, x = u, x1 = v (n) -> out_f64 (1) = sum_e ((sum_j coef[j]
 *     terms[j][e]) / (atol + rtol max(|u[e]|, |v[e]|)))^2.
 *   CFG_COMBINE: x = V (B n, or 2 B n with cfg: the cond rows, then the uncond rows) -> out_f32 (B n) = u + s_cfg (c - u)
 *     with cfg, else c.
 *   CFM_MIX: x = x1, x1 = z (B, C, T), x2 = t (B) -> out_f32 = (1 - (1 - sigma_min) t_b) z + t_b x1.
 *   CFM_LOSS: x = x1, x1 = z, x2 = v (B, C, T), mask (B, T) -> out_f64 (2) = (sum over every position of
 *     (v - (x1 - (1 - sigma_min) z))^2, sum mask) and out_f32 (1) = out_f64[0] / (out_f64[1] C).
 * Returns non-zero with st_last_error set, launching nothing, when the problem is outside the contract.  Synchronises
 * `stream`. */
enum { ST_TEST_ROW_ADALN = 0, ST_TEST_ROW_DWCONV_LN = 1, ST_TEST_ROW_SPECTRUM = 2, ST_TEST_ROW_IDFT_BASIS = 3,
       ST_TEST_ROW_OVERLAP_ADD = 4, ST_TEST_ROW_MEAN3_SILU = 5, ST_TEST_ROW_POST_TANH = 6,
       ST_TEST_ROW_GLU_RESID = 7, ST_TEST_ROW_MASKED_MEAN = 8, ST_TEST_ROW_COND_TRANSPOSE = 9, ST_TEST_ROW_RELU_LN = 10,
       ST_TEST_ROW_RELU_LN_PROJ = 11, ST_TEST_ROW_GEMV = 12, ST_TEST_ROW_TIME_EMBED = 13, ST_TEST_ROW_TIME_EMBED_VALS = 14,
       ST_TEST_ROW_ROPE_TABLE = 15, ST_TEST_ROW_LINCOMB = 16, ST_TEST_ROW_SCALED_SUMSQ = 17, ST_TEST_ROW_CFG_COMBINE = 18,
       ST_TEST_ROW_CFM_MIX = 19, ST_TEST_ROW_CFM_LOSS = 20 };
typedef struct st_test_row_desc {
    const float *x, *x1, *x2;                   /* inputs (x1, x2: MEAN3_SILU's second and third operand) */
    const float *w, *bias, *ln_w, *ln_b;        /* DWCONV_LN, POST_TANH */
    const float *film, *shift, *scale, *mask;   /* ADALN */
    const float* window;                         /* IDFT_BASIS, OVERLAP_ADD */
    float* xout;                                 /* ADALN with has_film */
    float* out_f32; uint16_t *out_hi, *out_lo;
    int64_t film_bstride, ada_bstride, n;       /* n: MEAN3_SILU's element count */
    int32_t kind, B, BB, T, C;                   /* BB: ADALN only */
    int32_t c_clamp, has_film, mask_out, u16;    /* ADALN */
    int32_t Nh, Kp, K, K2, n_fft, hop;           /* SPECTRUM (Nh, Kp, K, K2), IDFT_BASIS (n_fft, K2), OVERLAP_ADD */
    float eps;                                   /* DWCONV_LN */
    /* GLU_RESID .. CFM_LOSS (appended: the fields above keep their offsets) */
    const float* terms[7]; float coef[7];        /* LINCOMB, SCALED_SUMSQ */
    const float* t_host;                         /* TIME_EMBED_VALS: host memory */
    double* out_f64;                             /* SCALED_SUMSQ, CFM_LOSS */
    int64_t y_rstride;                           /* GEMV */
    int32_t N, silu_in, silu_out;                /* GEMV (K: the inner dimension) */
    int32_t n_terms, n_t, cfg;                   /* LINCOMB / SCALED_SUMSQ, TIME_EMBED[_VALS], CFG_COMBINE */
    float atol, rtol, sigma_min, s_cfg;          /* SCALED_SUMSQ, CFM_MIX / CFM_LOSS, CFG_COMBINE */
} st_test_row_desc;
int st_test_row_ex(st_handle* h, const st_test_row_desc* d, void* stream);

/* One hidden conv of the multi-period discriminator (layer 1-4 of st_create_mpd's handle: C_in -> C_out, (5, 1) kernel,
 * stride 3 for layers 1-3 and 1 for layer 4, pad 2) through the same packings, kernels and engine (st_set_engine) as
 * st_mpd_forward / st_mpd_backward, with the handle's period p.  Hx input rows give H = ceil(Hx / 3) (stride 3) or Hx
 * output rows.  mode 0 (forward): out (B, C_out, H, p) = conv(x) + b, x (B, C_in, Hx, p), no activation.  mode 1 (dgrad):
 * out (B, C_in, Hx, p) = the input gradient of dz (B, C_out, H, p).  mode 2 (wgrad): out (C_out, C_in, 5) and out_b
 * (C_out) = the weight and bias gradients of dz for input x.  w (C_out, C_in, 5).  Allocates its scratch and synchronises
 * `stream`. */
int st_test_mpd_conv(st_handle* h, int mode, int layer, int B, int Hx, const float* x, const float* dz, const float* w,
                     const float* b, float* out, float* out_b, void* stream);

/* One GEMM conv of the multi-resolution discriminator (band conv 1-4 of st_create_mrd's handle: 32 -> 32, (3, 9) stride
 * (1, 2) pad (1, 4) for layers 1-3, (3, 3) pad (1, 1) for layer 4) through the same packings, kernels and engine
 * (st_set_engine) as st_mrd_forward / st_mrd_backward.  W input columns give G = ceil(W / 2) (layers 1-3) or W output
 * columns.  mode 0 (forward): out (B, 32, T, G) = conv(x) + b, x (B, 32, T, W), no activation.  mode 1 (dgrad): out
 * (B, 32, T, W) = the input gradient of dz (B, 32, T, G).  mode 2 (wgrad): out (32, 32, 3, kw) and out_b (32) = the weight
 * and bias gradients of dz for input x.  w (32, 32, 3, kw).  Allocates its scratch and synchronises `stream`. */
int st_test_mrd_conv(st_handle* h, int mode, int layer, int B, int T, int W, const float* x, const float* dz, const float* w,
                     const float* b, float* out, float* out_b, void* stream);

/* The multi-period discriminator's fp32 row kernels (mpd.cu) through the library's own launchers, one kernel per call
 * (kernel-level tests; any handle kind works: the hook needs only the device).  Buffers are caller-owned device fp32, NULL =
 * not requested.  Geometry of every kind but PACK and UNPACK_WGRAD: B, p and L as st_mpd_forward checks them; Hin =
 * ceil(L / p) rows of the reflect-padded view, H0 = ceil(Hin / 3); BB = B p columns, column bb = b p + j.  A plane set
 * {f, hi, lo} is fp32 and / or split bf16 (hi = bf16(v), lo = bf16(v - hi), together): `rows` holds rows (BB, R, C)
 * token-major, `tr` transposed planes with Kr columns.  Slopes are f32(0.1) (`slope` only for ACT_FWD).
 *   CONV0_FWD: x (B, L), w (32, 1, 5), b (32); H = H0 -> out = fmap0 (B, 32, H0, p) = leaky(conv2d(reflect-pad view of x,
 *     w, b, stride (3, 1), pad (2, 0))); rows (BB, R, 32), R >= H0, rows [H0, R) +0.
 *   ACT_FWD: Y (BB, H, C) -> out = fmap (B, C, H, p) = where(Y > 0, Y, Y f32(slope)); rows (BB, R, C), R >= H, [H, R) +0.
 *   NCHW_TO_ROWS: fmap (B, C, H, p) -> rows (BB, R, C), R >= H, rows [H, R) +0.
 *   POST_FWD: fmap = fmap4 (B, 1024, H, p), w (1, 1024, 3), b (1); C = 1024 -> out = post (B, 1, H, p), conv_post with
 *     taps (3, 1), pad (1, 0).
 *   PACK: w (Cout, Cin, 5), mode 0-3 = FWD_S3, FWD_S1, DGRAD_S3, DGRAD_S1 -> out: FWD_S3 [2][Cout][3 Cin], FWD_S1
 *     [5][Cout][Cin] = w.permute(2, 0, 1), DGRAD_S3 [2][3 Cin][Cout], DGRAD_S1 [5][Cin][Cout] (oracle/mpd_ref.py pack_*).
 *   POST_DGRAD: gpost (B, 1, H, p), w (1, 1024, 3); C = 1024 -> out = G (BB, H, 1024) = Σ_k w[c, k] gpost[h - k + 1].
 *   POST_WGRAD: gpost (B, 1, H, p), fmap = fmap4 (B, 1024, H, p); C = 1024 -> out = dw (1024 · 3) and out_b = db (1).
 *   ACT_BWD: G (BB, Rg, C) with row h at Rg-row h + off (Rg >= H + off), gfmap (B, C, H, p) or NULL, fmap (B, C, H, p) or
 *     NULL (slope 1): v = (G + gfmap) · (fmap > 0 ? 1 : f32(0.1)) -> any of: rows = dZ (BB, H + 1, C) with row H +0; tr
 *     = dZ^T [C][Kr], Kr >= BB H, v at column bb H + h, columns >= BB H not written; out = dZ (B, C, H, p).
 *   IM2COL_T: fmap = X (B, Cin, Hx, p), stride 3 (H = ceil(Hx / 3)) or 1 (H = Hx), Kr >= BB H -> tr [5 Cin + 8][Kr]:
 *     row k Cin + c, column bb H + o holds X[b, c, s o + k - 2, j] (+0 outside [0, Hx)); row 5 Cin is 1; the last 7
 *     rows and the columns [BB H, Kr) +0.
 *   UNPACK_WGRAD: dWp [Cout][5 Cin + 8] -> out = dw (Cout, Cin, 5) = dWp[n][k Cin + c], out_b = db (Cout) = dWp[n][5 Cin].
 *   CONV0_WGRAD: dz0 (B, 32, H0, p), x (B, L); H = H0 -> out = dw (32, 5), out_b = db (32): conv 0's weight and bias
 *     gradients through the reflect pad.
 *   CONV0_DGRAD: dz0 (B, 32, H0, p), w (32, 1, 5); H = H0 -> out = gx (B, L): conv 0's input gradient, the reflect pad's
 *     adjoint folded in.
 * Returns non-zero with st_last_error set, launching nothing, when the problem is outside the contract (a geometry
 * st_mpd_forward refuses, R < H, Kr < BB H, Rg < H + off, an unknown kind or pack mode, hi without lo, a missing input or
 * output, an output the kind does not write).  Synchronises `stream`. */
enum { ST_TEST_MPD_ROW_CONV0_FWD = 0, ST_TEST_MPD_ROW_ACT_FWD = 1, ST_TEST_MPD_ROW_NCHW_TO_ROWS = 2, ST_TEST_MPD_ROW_POST_FWD = 3,
       ST_TEST_MPD_ROW_PACK = 4, ST_TEST_MPD_ROW_POST_DGRAD = 5, ST_TEST_MPD_ROW_POST_WGRAD = 6, ST_TEST_MPD_ROW_ACT_BWD = 7,
       ST_TEST_MPD_ROW_IM2COL_T = 8, ST_TEST_MPD_ROW_UNPACK_WGRAD = 9, ST_TEST_MPD_ROW_CONV0_WGRAD = 10,
       ST_TEST_MPD_ROW_CONV0_DGRAD = 11 };
typedef struct st_test_mpd_row_desc {
    const float *x, *w, *b, *Y, *G, *gpost, *fmap, *gfmap, *dz0, *dWp;   /* inputs, by kind */
    float *out, *out_b;                                                   /* out_b: the bias gradients */
    float* rows_f; uint16_t *rows_hi, *rows_lo;                           /* rows plane set */
    float* tr_f; uint16_t *tr_hi, *tr_lo;                                 /* transposed plane set */
    int64_t L, Kr;
    int32_t kind, B, p, H, C, R, Rg, off, Hx, Cin, Cout, stride, mode;
    float slope;                                                          /* ACT_FWD */
} st_test_mpd_row_desc;
int st_test_mpd_row_ex(st_handle* h, const st_test_mpd_row_desc* d, void* stream);

/* The layout, operand-split and weight-packing kernels through the library's own launchers, one kernel per call
 * (kernel-level tests; any handle kind works: the hook needs only the device).  Buffers are caller-owned device memory,
 * NULL = not requested; fp32 unless stated, rows contiguous.  Every kind is exact: no arithmetic beyond what it states.
 *   BCT_TO_BTC: x (B, C, T) -> (B [+1], T, C) out_f32 and / or the split planes out_hi / out_lo (hi = bf16_rn(v), lo =
 *     bf16_rn(v - hi), together).  With bcast (C), row B is bcast[c] for every t.  B >= 0 (x may be NULL when B = 0).
 *   BTC_TO_BCT: x (B, T, C) -> out_f32 (B, C, T).
 *   EMBED: ids, lens (int64: (B, T), (B)), x = emb (n_vocab, C) -> out_f32 (B, T, C): x[b, t, :] = emb[clamp(id, 0,
 *     n_vocab - 1)] · scale · m, with m = [t < lens[b]], and out2_f32 = mask (B, T) = m.  The product order is the
 *     reference's, so -0 and NaN follow torch.
 *   SPLIT_BF16: x (n) -> out_hi, out_lo (bf16): hi = bf16_rn(x), lo = bf16_rn(x - hi).
 *   SPLIT_F16: x (n) -> out_hi, out_lo (fp16): hi = fp16_rn(x), lo = fp16_rn(x - hi) for |x| < 65520, plus the range
 *     flag: out_i32 (1) or NULL = 1 when some x is NaN or |x| >= 65520 (the planes then do not represent it), else 0.
 *   PACK_CONV: x (Nsrc, Csrc, k) -> out_f32 [k][Ntot][Cc]: out[tap][n_off + n][c] = x[n][c_off + c][tap].  Rows outside
 *     [n_off, n_off + Nsrc) are left untouched.
 *   WEIGHT_NORM: g (rows), x = v (rows, len) -> out_f32 (rows, len): W[r, i] = v[r, i] · fl32(g[r] / ||v_r||), with ||v_r||
 *     accumulated in double.
 *   POLYPHASE: x = w (Cin, Cout, 2u), u even >= 2 -> out_f32 [3][u Cout][Cin]: out[tau][r Cout + c][i] = w[i, c, r + u/2 -
 *     (tau - 1) u] where that tap lies in [0, 2u), else 0 (oracle/ffgan_ref.py::polyphase_weight, tap-major).
 *   MEL_TWIDDLES: n_fft -> out_f32 (n_fft/2, 2): tw[t] = fl32(cos 2 pi t / n_fft) - i fl32(sin 2 pi t / n_fft).
 *   MEL_PACK_FB: x = fb (n_fft/2 + 1, n_mels) -> out_f32 = fbT (n_mels, n_fft/2 + 1) = fb^T; out_i32 = band (n_mels, 2):
 *     [first, last + 1) of the entries != 0 of filter m, or (0, 0) if there are none; out2_i32 = kband (n_fft/2 + 1, 2) or
 *     NULL: the same over the filters at bin k.
 * Returns non-zero with st_last_error set, launching nothing, when the problem is outside the contract (a missing input or
 * output, hi without lo, negative sizes, n_off + Nsrc > Ntot, c_off + Cc > Csrc, an odd u or u < 2, n_fft not a power of
 * two in [32, 4096], an unknown kind).  Synchronises `stream`. */
enum { ST_TEST_PACK_BCT_TO_BTC = 0, ST_TEST_PACK_BTC_TO_BCT = 1, ST_TEST_PACK_EMBED = 2, ST_TEST_PACK_SPLIT_BF16 = 3,
       ST_TEST_PACK_SPLIT_F16 = 4, ST_TEST_PACK_PACK_CONV = 5, ST_TEST_PACK_WEIGHT_NORM = 6, ST_TEST_PACK_POLYPHASE = 7,
       ST_TEST_PACK_MEL_TWIDDLES = 8, ST_TEST_PACK_MEL_PACK_FB = 9 };
typedef struct st_test_pack_desc {
    const float *x, *bcast, *g;                  /* x: every kind's source (EMBED: emb, WEIGHT_NORM: v, MEL_PACK_FB: fb) */
    const int64_t *ids, *lens;                   /* EMBED */
    float *out_f32, *out2_f32;                   /* out2_f32: EMBED's mask */
    uint16_t *out_hi, *out_lo;
    int32_t *out_i32, *out2_i32;                 /* SPLIT_F16: the range flag; MEL_PACK_FB: band, kband */
    int64_t n;                                   /* SPLIT_BF16, SPLIT_F16 */
    int32_t kind, B, C, T, n_vocab;              /* BCT_TO_BTC, BTC_TO_BCT, EMBED */
    int32_t Nsrc, Csrc, k, Ntot, n_off, c_off, Cc;   /* PACK_CONV */
    int32_t rows, len;                           /* WEIGHT_NORM */
    int32_t Cin, Cout, u;                        /* POLYPHASE */
    int32_t n_fft, n_mels;                       /* MEL_TWIDDLES, MEL_PACK_FB */
    float scale;                                 /* EMBED */
} st_test_pack_desc;
int st_test_pack_ex(st_handle* h, const st_test_pack_desc* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STABLETTS_B200_H_ */
