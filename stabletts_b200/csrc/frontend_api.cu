// C-ABI + orchestration of the two small front-end modules of StableTTS.synthesise (models/model.py:78-80) that run
// before the TextEncoder's output reaches the alignment: the MelStyleEncoder (speaker vector c from the reference mel)
// and the DurationPredictor (logw from the text encoding).  Token-major throughout; one GEMM row is one frame / token.
//
// MelStyleEncoder (models/reference_encoder.py:25-92; style_hidden 128, style_vector_dim 256, kernel 5, 2 heads):
//   y (B, M, T) -> token-major planes
//   spectral: Linear(M -> 128) + Mish, Linear(128 -> 128) + Mish        GEMM, EPI_MISH (x2)
//   temporal: 2 x Conv1dGLU: Conv1d(128 -> 256, k = 5, UNMASKED)        GEMM, 5 taps, fp32 out
//             x + a * sigmoid(g)                                        row kernel (fp32 residual + split planes)
//   slf_attn: in_proj (q | k | v rows), q rows pre-scaled by log2(e)/8  GEMM, plain bias
//             2 heads x 64, key_padding_mask = ~x_mask                  attention_wgmma_kernel (no RoPE)
//   pool first, then project: mean_t(fc(out_proj(a))) = fc(out_proj(mean_t(a))) (both affine: exact algebra)
//             masked mean over the valid frames (all T without a mask)  row kernel, fixed summation order
//             out_proj (128 -> 128), fc (128 -> 256)                    gemv_kernel (x2)
// DurationPredictor (models/duration_predictor.py:5-36; in 256, filter 1024, k = 3):
//   x' = (x + cond(g)) * m                                              gemv_kernel (cond) + transpose row kernel
//   conv1 (256 -> 1024, k = 3)                                          GEMM, batch-invariant
//   ReLU -> LayerNorm(1024, affine, eps 1e-5) -> * m                    row kernel -> operand of conv2
//   conv2 (1024 -> 1024, k = 3)                                         GEMM, batch-invariant
//   ReLU -> LayerNorm -> proj (1024 -> 1) on (. * m) -> * m             row kernel, writes logw (B, Tx)
#include "handle.cuh"

using namespace st;

namespace st {

namespace {

constexpr int kSH = 128, kSOut = 256, kSK = 5, kSHeads = 2;        // MelStyleEncoder as models/model.py:38 builds it
constexpr int kDIn = 256, kDF = 1024, kDK = 3;                      // DurationPredictor(hidden 256, filter 1024, k 3)

// ---------------------------------------------------------------------------------------------------------------------
// row kernels
// ---------------------------------------------------------------------------------------------------------------------
// Conv1dGLU tail (reference_encoder.py:16-21): out = resid + a * sigmoid(g), conv output (rows, 2C) = [a | g]
__global__ void glu_residual_kernel(const float* __restrict__ ag, const float* __restrict__ resid, float* __restrict__ out,
                                    bf16* __restrict__ hi, bf16* __restrict__ lo, long rows, int C) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // one thread per channel pair
    const int hc = C / 2;
    if (i >= rows * hc) return;
    const long r = i / hc;
    const int c = (int)(i - r * hc) * 2;
    const float2 a = *reinterpret_cast<const float2*>(ag + r * 2 * C + c);
    const float2 g = *reinterpret_cast<const float2*>(ag + r * 2 * C + C + c);
    const float2 x = *reinterpret_cast<const float2*>(resid + r * C + c);
    const float v0 = x.x + a.x / (1.0f + expf(-g.x)), v1 = x.y + a.y / (1.0f + expf(-g.y));
    if (out) *reinterpret_cast<float2*>(out + r * C + c) = make_float2(v0, v1);
    if (hi) {
        uint32_t h, l;
        split_bf16x2(v0, v1, h, l);
        *reinterpret_cast<uint32_t*>(hi + r * C + c) = h;
        *reinterpret_cast<uint32_t*>(lo + r * C + c) = l;
    }
}

// temporal_avg_pool (reference_encoder.py:71-75): out[b, c] = sum over frames with mask != 0 of x[b, t, c] / their count
// (mask == nullptr: all T).  Block (C, 8): thread (c, j) sums frames j, j + 8, ... in order, then the eight partials are
// added in a fixed order — the result does not depend on the batch or on scheduling.
constexpr int kPoolG = 8;
__global__ void masked_mean_kernel(const float* __restrict__ x, const float* __restrict__ mask, float* __restrict__ out, int T, int C) {
    pdl_trigger(); pdl_wait();
    extern __shared__ float part[];                                  // [kPoolG][C] sums, then [kPoolG] counts
    const int b = blockIdx.x, c = threadIdx.x, j = threadIdx.y;
    float s = 0.f, n = 0.f;
    const float* xb = x + (long)b * T * C;
#pragma unroll 4
    for (int t = j; t < T; t += kPoolG) {
        const bool ok = !mask || mask[(long)b * T + t] != 0.f;
        s += ok ? xb[(long)t * C + c] : 0.f;
        n += ok ? 1.f : 0.f;
    }
    part[j * C + c] = s;
    if (c == 0) part[kPoolG * C + j] = n;
    __syncthreads();
    if (j == 0) {
        float sum = 0.f, cnt = 0.f;
#pragma unroll
        for (int k = 0; k < kPoolG; ++k) { sum += part[k * C + c]; cnt += part[kPoolG * C + k]; }
        out[(long)b * C + c] = sum / cnt;
    }
}

// DurationPredictor input (duration_predictor.py:24-25): (B, C, T) x -> token-major (x + cond[b, c]) * mask[b, t]
__global__ void cond_mask_transpose_kernel(const float* __restrict__ in, const float* __restrict__ cond, const float* __restrict__ mask,
                                           float* __restrict__ out_f32, bf16* __restrict__ out_hi, bf16* __restrict__ out_lo,
                                           int C, int T) {
    pdl_trigger(); pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, t = t0 + threadIdx.x;
        float v = 0.f;
        if (c < C && t < T) v = (in[((long)b * C + c) * T + t] + cond[(long)b * C + c]) * mask[(long)b * T + t];
        tile[i][threadIdx.x] = v;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int t = t0 + i, c = c0 + threadIdx.x;
        if (c < C && t < T) {
            const float v = tile[threadIdx.x][i];
            const long o = ((long)b * T + t) * C + c;
            if (out_f32) out_f32[o] = v;
            if (out_hi) { bf16 h, l; split_bf16(v, h, l); out_hi[o] = h; out_lo[o] = l; }
        }
    }
}

// ReLU -> LayerNorm(C, affine, eps 1e-5) -> * mask, one warp per token (the dwconv_ln_kernel layout: lane owns float4
// groups j * 32 + lane).  PROJ = 0: the result is the operand of the next conv (fp32 and / or split planes).
// PROJ = 1: logw[row] = (mask * sum_c u[c] w[c] + b) * mask (proj on (x * mask), then * mask; duration_predictor.py:33-35).
template <int C, int PROJ>
__global__ void __launch_bounds__(256) relu_ln_kernel(const float* __restrict__ x, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                                                      const float* __restrict__ mask, long rows, float* __restrict__ out_f32,
                                                      bf16* __restrict__ out_hi, bf16* __restrict__ out_lo,
                                                      const float* __restrict__ proj_w, const float* __restrict__ proj_b,
                                                      float* __restrict__ logw) {
    pdl_trigger(); pdl_wait();
    constexpr int G = C / 128;
    const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float v[G * 4];
    const float* xr = x + row * C;
#pragma unroll
    for (int j = 0; j < G; ++j) {
        const float4 x4 = __ldg(reinterpret_cast<const float4*>(xr + (j * 32 + lane) * 4));
        v[j * 4 + 0] = fmaxf(x4.x, 0.f); v[j * 4 + 1] = fmaxf(x4.y, 0.f); v[j * 4 + 2] = fmaxf(x4.z, 0.f); v[j * 4 + 3] = fmaxf(x4.w, 0.f);
    }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < G * 4; ++j) sum += v[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * (1.0f / C);
    float var = 0.f;
#pragma unroll
    for (int j = 0; j < G * 4; ++j) { const float d = v[j] - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = rsqrtf(var * (1.0f / C) + 1e-5f);
    const float m = mask[row];
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < G; ++j) {
        const int c = (j * 32 + lane) * 4;
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(ln_w + c));
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(ln_b + c));
        const float u0 = (v[j * 4 + 0] - mean) * rstd * w4.x + b4.x, u1 = (v[j * 4 + 1] - mean) * rstd * w4.y + b4.y;
        const float u2 = (v[j * 4 + 2] - mean) * rstd * w4.z + b4.z, u3 = (v[j * 4 + 3] - mean) * rstd * w4.w + b4.w;
        if constexpr (PROJ) {
            const float4 p4 = __ldg(reinterpret_cast<const float4*>(proj_w + c));
            dot = fmaf(u0, p4.x, dot); dot = fmaf(u1, p4.y, dot); dot = fmaf(u2, p4.z, dot); dot = fmaf(u3, p4.w, dot);
        } else {
            const long o = row * C + c;
            if (out_f32) *reinterpret_cast<float4*>(out_f32 + o) = make_float4(u0 * m, u1 * m, u2 * m, u3 * m);
            if (out_hi) {
                uint32_t h01, l01, h23, l23;
                split_bf16x2(u0 * m, u1 * m, h01, l01); split_bf16x2(u2 * m, u3 * m, h23, l23);
                *reinterpret_cast<uint2*>(out_hi + o) = make_uint2(h01, h23);
                *reinterpret_cast<uint2*>(out_lo + o) = make_uint2(l01, l23);
            }
        }
    }
    if constexpr (PROJ) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        if (lane == 0) logw[row] = (m * dot + __ldg(proj_b)) * m;
    }
}

__global__ void fill_kernel(float* __restrict__ p, long n, float v) {
    pdl_trigger(); pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

__global__ void scale_kernel(float* __restrict__ p, long n, float s) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] *= s;
}

unsigned blocks_for(long n, int per = 256) { return (unsigned)((n + per - 1) / per); }

}  // namespace

cudaError_t launch_glu_residual(const float* ag, const float* resid, float* out_f32, bf16* out_hi, bf16* out_lo, long rows, int C,
                                cudaStream_t s) {
    if (C < 2 || C % 2) return cudaErrorInvalidValue;
    if (rows == 0) return cudaSuccess;
    return launch_k(glu_residual_kernel, dim3(blocks_for(rows * C / 2)), dim3(256), 0, s, ag, resid, out_f32, out_hi, out_lo, rows, C);
}

cudaError_t launch_masked_mean(const float* x, const float* mask, float* out, int B, int T, int C, cudaStream_t s) {
    if (C < 1 || C > 1024 / kPoolG) return cudaErrorInvalidValue;
    if (B == 0) return cudaSuccess;
    return launch_k(masked_mean_kernel, dim3(B), dim3(C, kPoolG), (size_t)(kPoolG * C + kPoolG) * 4, s, x, mask, out, T, C);
}

cudaError_t launch_cond_mask_transpose(const float* x, const float* cond, const float* mask, float* out_f32, bf16* out_hi,
                                       bf16* out_lo, int B, int C, int T, cudaStream_t s) {
    if ((long)B * C * T == 0) return cudaSuccess;
    return launch_k(cond_mask_transpose_kernel, dim3((T + 31) / 32, (C + 31) / 32, B), dim3(32, 8), 0, s, x, cond, mask, out_f32,
                    out_hi, out_lo, C, T);
}

cudaError_t launch_relu_ln(const float* x, const float* ln_w, const float* ln_b, const float* mask, long rows, int C, float* out_f32,
                           bf16* out_hi, bf16* out_lo, const float* proj_w, const float* proj_b, float* logw, cudaStream_t s) {
    if (C != kDF) return cudaErrorInvalidValue;
    if (rows == 0) return cudaSuccess;
    const dim3 grid(blocks_for(rows * 32)), block(256);
    if (logw)
        return launch_k(relu_ln_kernel<kDF, 1>, grid, block, 0, s, x, ln_w, ln_b, mask, rows, (float*)nullptr, (bf16*)nullptr,
                        (bf16*)nullptr, proj_w, proj_b, logw);
    return launch_k(relu_ln_kernel<kDF, 0>, grid, block, 0, s, x, ln_w, ln_b, mask, rows, out_f32, out_hi, out_lo,
                    (const float*)nullptr, (const float*)nullptr, (float*)nullptr);
}

// ---------------------------------------------------------------------------------------------------------------------
// per-handle state
// ---------------------------------------------------------------------------------------------------------------------
// the workspaces grow stream-ordered (grow_ws) and are freed with cudaFreeAsync; the device is idle when st_destroy
// runs the destructors
struct StyleState : Model {
    int n_mel;
    GemmW sp0, sp3, glu[2], qkv, qkv_tc;    // qkv: reference rows (SIMT engine); qkv_tc: q rows x log2(e)/8 (wgmma engine)
    float *wo = nullptr, *bo = nullptr, *wfc = nullptr, *bfc = nullptr;
    void* ws = nullptr; size_t ws_bytes = 0;
    explicit StyleState(int m) : n_mel(m) {}
    ~StyleState() override { if (ws) cudaFreeAsync(ws, 0); }
    int finalize(st_handle* h, cudaStream_t s) override {
        const int M = n_mel;
        if (pack_gemm(h, &sp0, {"spectral.0"}, kSH, M, 1, 0, M, true, s)) return 1;                         // :47
        if (pack_gemm(h, &sp3, {"spectral.3"}, kSH, kSH, 1, 0, kSH, true, s)) return 1;                     // :50
        for (int i = 0; i < 2; ++i)                                                                          // :56-59
            if (pack_gemm(h, &glu[i], {"temporal." + std::to_string(i) + ".conv1"}, 2 * kSH, kSH, kSK, 0, kSH, true, s)) return 1;
        float *w, *b;                                                                                        // :61-66
        if (get_raw(h, "slf_attn.in_proj_weight", (int64_t)3 * kSH * kSH, &w) || get_raw(h, "slf_attn.in_proj_bias", 3 * kSH, &b)) return 1;
        const size_t n = (size_t)3 * kSH * kSH;
        for (GemmW* q : {&qkv, &qkv_tc}) {
            if (alloc_gemm_w(h, q, 1, 3 * kSH, kSH, true)) return 1;
            ST_CUDA(launch_pack_conv(w, q->f32, 3 * kSH, kSH, 1, 3 * kSH, 0, 0, kSH, s));
            ST_CUDA(cudaMemcpyAsync(q->bias, b, (size_t)3 * kSH * 4, cudaMemcpyDeviceToDevice, s));
            if (q == &qkv_tc) {
                // attention_wgmma_kernel expects q carrying the softmax scale in the exp2 domain; the RoPE QKV epilogue applies
                // it elsewhere, here it is folded into the q rows and the q bias once, so the QKV GEMM is a plain bias GEMM
                scale_kernel<<<blocks_for((long)kSH * kSH), 256, 0, s>>>(q->f32, (long)kSH * kSH, 0.125f * 1.4426950408889634f);
                scale_kernel<<<1, kSH, 0, s>>>(q->bias, kSH, 0.125f * 1.4426950408889634f);
                ST_CUDA(cudaGetLastError());
            }
            ST_CUDA(launch_split(q->f32, q->hi, q->lo, (long)n, s));
        }
        if (get_raw(h, "slf_attn.out_proj.weight", (int64_t)kSH * kSH, &wo) || get_raw(h, "slf_attn.out_proj.bias", kSH, &bo)) return 1;
        return get_raw(h, "fc.weight", (int64_t)kSOut * kSH, &wfc) || get_raw(h, "fc.bias", kSOut, &bfc);                // :68
    }
};

struct DpState : Model {
    GemmW c1, c2;
    float *cond_w = nullptr, *cond_b = nullptr, *n1w = nullptr, *n1b = nullptr, *n2w = nullptr, *n2b = nullptr;
    float *proj_w = nullptr, *proj_b = nullptr;
    void* ws = nullptr; size_t ws_bytes = 0;
    ~DpState() override { if (ws) cudaFreeAsync(ws, 0); }
    int finalize(st_handle* h, cudaStream_t s) override {
        if (pack_gemm(h, &c1, {"conv1"}, kDF, kDIn, kDK, 0, kDIn, true, s)) return 1;                       // :17
        if (pack_gemm(h, &c2, {"conv2"}, kDF, kDF, kDK, 0, kDF, true, s)) return 1;                         // :19
        if (get_raw(h, "norm1.weight", kDF, &n1w) || get_raw(h, "norm1.bias", kDF, &n1b) ||
            get_raw(h, "norm2.weight", kDF, &n2w) || get_raw(h, "norm2.bias", kDF, &n2b)) return 1;
        if (get_raw(h, "proj.weight", kDF, &proj_w) || get_raw(h, "proj.bias", 1, &proj_b)) return 1;       // :21
        return get_raw(h, "cond.weight", (int64_t)kDIn * kDIn, &cond_w) || get_raw(h, "cond.bias", kDIn, &cond_b);   // :23
    }
};

}  // namespace st

namespace {

struct StyleWs { Act Y, S1, X[2], G, QKV, AO; float *ones, *pool, *op; int *kvlen, *prefix; size_t bytes; };

void layout_style_ws(StyleWs& w, void* base, int B, int T, int M, bool tc) {
    Bump bp(base, 0);
    const size_t r = (size_t)B * T;
    w.Y = take_act(bp, r, M, true, tc);
    w.S1 = take_act(bp, r, kSH, !tc, tc);
    w.X[0] = take_act(bp, r, kSH, true, tc);
    w.X[1] = take_act(bp, r, kSH, true, tc);
    w.G = take_act(bp, r, 2 * kSH, true, false);
    w.QKV = take_act(bp, r, 3 * kSH, !tc, tc);
    w.AO = take_act(bp, r, kSH, true, false);
    w.ones = bp.take<float>(r);
    w.pool = bp.take<float>((size_t)B * kSH);
    w.op = bp.take<float>((size_t)B * kSH);
    w.kvlen = bp.take<int>(B);
    w.prefix = bp.take<int>(B);
    w.bytes = bp.off + 256;
}

struct DpWs { Act X0, H, U; float* cg; size_t bytes; };

void layout_dp_ws(DpWs& w, void* base, int B, int T, bool tc) {
    Bump bp(base, 0);
    const size_t r = (size_t)B * T;
    w.X0 = take_act(bp, r, kDIn, !tc, tc);
    w.H = take_act(bp, r, kDF, true, false);
    w.U = take_act(bp, r, kDF, !tc, tc);
    w.cg = bp.take<float>((size_t)B * kDIn);
    w.bytes = bp.off + 256;
}

}  // namespace

extern "C" {

int st_create_style_encoder(int n_mel, int device, st_handle** out) {
    if (!out) return fail(nullptr, "st_create_style_encoder: null argument");
    if (n_mel <= 0 || n_mel % 16 || n_mel > 1024) return fail(nullptr, "st_create_style_encoder: n_mel must be a positive multiple of 16, <= 1024");
    return create_handle(device, std::make_unique<StyleState>(n_mel), out);
}

int st_create_duration_predictor(const st_dims* dims, int device, st_handle** out) {
    if (!dims || !out) return fail(nullptr, "st_create_duration_predictor: null argument");
    if (dims->hidden != kDIn || dims->filter != kDF || dims->kernel != kDK || dims->gin != kDIn)
        return fail(nullptr, "st_create_duration_predictor: only in_channels = gin_channels = 256, filter_channels = 1024, kernel_size = 3 is built");
    return create_handle(device, std::make_unique<DpState>(), out);
}

// models/reference_encoder.py:77-92 (eval: dropout is the identity)
int st_style_encoder_forward(st_handle* h, const float* y, const float* y_mask, float* c_out, int B, int T, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    StyleState* f = ready_model<StyleState>(h, "MelStyleEncoder");
    if (!f) return 1;
    if (!y || !c_out) return fail(h, "st_style_encoder_forward: null pointer");
    if (B <= 0 || T <= 0 || B > 65535 || (long)B * T > (1L << 26)) return fail(h, "B and T must be positive (B * T < 2^26)");
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const int M = f->n_mel;
    StyleWs w;
    layout_style_ws(w, nullptr, B, T, M, tc);
    if (grow_ws(h, &f->ws, &f->ws_bytes, w.bytes, s)) return 1;
    layout_style_ws(w, f->ws, B, T, M, tc);
    const long rows = (long)B * T;
    ST_LAUNCH(launch_bct_to_btc(y, w.Y.f32, w.Y.hi, w.Y.lo, B, M, T, nullptr, s));          // x.transpose(1, 2) (:78)
    {   // spectral (:47-52): Linear + Mish, twice; the second one's output is also the temporal residual stream
        GemmArgs g = utt_gemm(B, T, EPI_BIAS | EPI_MISH);
        if (run_gemm(h, g, f->sp0, &w.Y, nullptr, w.S1, s)) return 1;
        if (run_gemm(h, g, f->sp3, &w.S1, nullptr, w.X[0], s)) return 1;
    }
    for (int i = 0; i < 2; ++i) {      // temporal (:56-59): Conv1dGLU on the full tensor, padded frames included (unmasked)
        GemmArgs g = utt_gemm(B, T, EPI_BIAS);
        if (run_gemm(h, g, f->glu[i], &w.X[i], nullptr, w.G, s)) return 1;
        const Act& o = w.X[1 - i];
        ST_LAUNCH(launch_glu_residual(w.G.f32, w.X[i].f32, o.f32, o.hi, o.lo, rows, kSH, s));
    }
    const Act& X = w.X[0];             // after two GLU layers the stream is back in X[0]
    // slf_attn (:61-66, :86-87).  key_padding_mask = ~x_mask; without a mask every key is valid (an all-ones mask).
    const float* mask = y_mask;
    if (!mask) {
        ST_LAUNCH(launch_k(fill_kernel, dim3(blocks_for(rows)), dim3(256), 0, s, w.ones, rows, 1.0f));
        mask = w.ones;
    }
    ST_LAUNCH(launch_mask_lengths(mask, w.kvlen, w.prefix, B, T, s));
    {
        GemmArgs g = utt_gemm(B, T, EPI_BIAS);
        if (run_gemm(h, g, tc ? f->qkv_tc : f->qkv, &X, nullptr, w.QKV, s)) return 1;
    }
    {
        AttnArgs a;
        a.qkv = w.QKV.f32; a.qkv_hi = w.QKV.hi; a.qkv_lo = w.QKV.lo; a.rope_cs = nullptr;
        a.mask = mask; a.kvlen = w.kvlen; a.prefix = w.prefix; a.out_f32 = w.AO.f32;
        a.BB = B; a.B = B; a.T = T; a.H = kSH; a.n_heads = kSHeads;
        // frames with mask == 0 come out as zeros (the reference computes them, attending to the valid keys); harmless:
        // the pool below never reads them
        ST_LAUNCH(tc ? launch_attention_tc(a, s) : launch_attention_simt(a, s));
    }
    // pool first, then project (out_proj and fc are affine, so the masked mean commutes with both; :68, :89-90)
    ST_LAUNCH(launch_masked_mean(w.AO.f32, y_mask, w.pool, B, T, kSH, s));
    ST_LAUNCH(launch_gemv(w.pool, f->wo, f->bo, w.op, kSH, B, kSH, kSH, 0, 0, s));
    ST_LAUNCH(launch_gemv(w.op, f->wfc, f->bfc, c_out, kSOut, B, kSH, kSOut, 0, 0, s));
    return 0;
}

// models/duration_predictor.py:22-36 (eval: dropout is the identity)
int st_duration_predictor_forward(st_handle* h, const float* x, const float* x_mask, const float* g_in, float* logw, int B, int Tx,
                                  void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    DpState* f = ready_model<DpState>(h, "DurationPredictor");
    if (!f) return 1;
    if (!x || !x_mask || !g_in || !logw) return fail(h, "st_duration_predictor_forward: null pointer");
    if (B <= 0 || Tx <= 0 || B > 65535 || (long)B * Tx > (1L << 24)) return fail(h, "B and Tx must be positive (B * Tx < 2^24)");
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    DpWs w;
    layout_dp_ws(w, nullptr, B, Tx, tc);
    if (grow_ws(h, &f->ws, &f->ws_bytes, w.bytes, s)) return 1;
    layout_dp_ws(w, f->ws, B, Tx, tc);
    auto base = [&]() {
        GemmArgs g = utt_gemm(B, Tx, EPI_BIAS);
        g.batch_invariant = 1;         // logw goes through ceil(exp(.)): a batch-dependent summation order could move a duration
        return g;
    };
    const long rows = (long)B * Tx;
    ST_LAUNCH(launch_gemv(g_in, f->cond_w, f->cond_b, w.cg, kDIn, B, kDIn, kDIn, 0, 0, s));                 // cond(g) (:24)
    ST_LAUNCH(launch_cond_mask_transpose(x, w.cg, x_mask, w.X0.f32, w.X0.hi, w.X0.lo, B, kDIn, Tx, s));        // (x + cond) * m
    {
        GemmArgs g = base();
        if (run_gemm(h, g, f->c1, &w.X0, nullptr, w.H, s)) return 1;                                            // conv1 (:25)
    }
    ST_LAUNCH(launch_relu_ln(w.H.f32, f->n1w, f->n1b, x_mask, rows, kDF, w.U.f32, w.U.hi, w.U.lo, nullptr, nullptr, nullptr, s));  // :26-29
    {
        GemmArgs g = base();
        if (run_gemm(h, g, f->c2, &w.U, nullptr, w.H, s)) return 1;                                             // conv2 (:29)
    }
    ST_LAUNCH(launch_relu_ln(w.H.f32, f->n2w, f->n2b, x_mask, rows, kDF, nullptr, nullptr, nullptr, f->proj_w, f->proj_b, logw, s));   // :30-35
    return 0;
}

}  // extern "C"
