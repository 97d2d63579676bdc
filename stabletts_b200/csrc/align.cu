// Duration -> alignment -> mu_y expansion of StableTTS.synthesise (models/model.py:81-95 with
// generate_path :17-27), the immediate caller-side glue of the CFM path (SURVEY.md §8 row f1).
//
// The reference materialises a dense (B, T_x, T_y) 0/1 path from cumulative durations and multiplies
// it with mu_x; the path has exactly one 1 per output frame, so the product is a gather:
//     mu_y[b, :, t] = mu_x[b, :, i(t)],   i(t) = the token with cum[i-1] <= t < cum[i]
// Kernel 1 (one thread per utterance):
//     w = exp(logw) * x_mask;  w_ceil = ceil(w) * length_scale (fp32, as the reference);  cum = cumsum(w_ceil);
//     y_len = (int64) max(sum(w_ceil), 1)
//   The prefix sum accumulates in double and stores each prefix rounded to fp32: that is what torch.cumsum computes for
//   an fp32 tensor on the CPU, bit for bit.  A sequential fp32 sum differs from it in the last bit often enough to move
//   a frame boundary whenever the durations are fractional (length_scale = 1.15: cum = 23 in exact arithmetic comes out
//   22.999998 or 23.000002).  y_len truncates the same double total rounded to fp32; the reference's torch.sum uses an
//   fp32 cascade whose order depends on the platform, which agrees except when the exact total is an integer.
// Kernel 2: per output frame a binary search over cum, then a coalesced gather; also emits the float
//     prefix mask y_mask and, on request, the dense attn path the reference returns to its caller.
#include "handle.cuh"

namespace st {

__global__ void align_lengths_kernel(const float* __restrict__ logw, const float* __restrict__ x_mask, float length_scale,
                                     int B, int Tx, float* __restrict__ cum, long long* __restrict__ ylen) {
    pdl_trigger(); pdl_wait();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double acc = 0.0;
    for (int i = 0; i < Tx; ++i) {
        const float w = expf(logw[(long)b * Tx + i]) * x_mask[(long)b * Tx + i];     // models/model.py:83
        const float wc = ceilf(w) * length_scale;                                     // :84
        acc += (double)wc;                                                             // generate_path cumsum (:19)
        cum[(long)b * Tx + i] = (float)acc;
    }
    ylen[b] = (long long)fmaxf((float)acc, 1.0f);                                     // :85 clamp_min(...,1).long()
}

__global__ void align_expand_kernel(const float* __restrict__ mu_x, const float* __restrict__ x_mask,
                                    const float* __restrict__ cum, const long long* __restrict__ ylen, int B, int M, int Tx,
                                    int Ty, float* __restrict__ mu_y, float* __restrict__ y_mask, float* __restrict__ attn) {
    pdl_trigger(); pdl_wait();
    extern __shared__ int tok[];              // token index per frame of this tile, -1 = no token
    const int b = blockIdx.y, t0 = blockIdx.x * blockDim.x, t = t0 + threadIdx.x;
    const float* cb = cum + (long)b * Tx;
    int idx = -1;
    if (t < Ty) {
        const bool in_len = t < ylen[b];                                              // sequence_mask(y_lengths) :89
        // smallest i with t < cum[i]  (path[b,i,t] = [t < cum[i]] - [t < cum[i-1]], generate_path :22-25)
        int lo = 0, hi = Tx;
        const float tf = (float)t;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (tf < cb[mid]) hi = mid; else lo = mid + 1; }
        if (in_len && lo < Tx && x_mask[(long)b * Tx + lo] != 0.f) idx = lo;         // attn_mask = x_mask * y_mask (:90)
        y_mask[(long)b * Ty + t] = in_len ? 1.f : 0.f;
    }
    tok[threadIdx.x] = idx;
    __syncthreads();
    // gather: thread = frame, loop over channels: writes are contiguous along T (the (B, M, T) boundary layout)
    if (t < Ty) {
        for (int m = 0; m < M; ++m)
            mu_y[((long)b * M + m) * Ty + t] = idx >= 0 ? __ldg(mu_x + ((long)b * M + m) * Tx + idx) : 0.f;
    }
    if (attn) {                               // dense path (B, Tx, Ty), only when the caller wants it back
        const int n = min((int)blockDim.x, Ty - t0);
        for (int i = 0; i < Tx; ++i)
            for (int j = threadIdx.x; j < n; j += blockDim.x)
                attn[((long)b * Tx + i) * Ty + t0 + j] = tok[j] == i ? 1.f : 0.f;
    }
}

cudaError_t launch_align_lengths(const float* logw, const float* x_mask, float length_scale, int B, int Tx, float* cum,
                                 long long* ylen, cudaStream_t s) {
    if (B == 0) return cudaSuccess;
    return launch_k(align_lengths_kernel, dim3((B + 63) / 64), dim3(64), 0, s, logw, x_mask, length_scale, B, Tx, cum, ylen);
}

cudaError_t launch_align_expand(const float* mu_x, const float* x_mask, const float* cum, const long long* ylen, int B, int M,
                                int Tx, int Ty, float* mu_y, float* y_mask, float* attn, cudaStream_t s) {
    if (B == 0 || Ty == 0) return cudaSuccess;
    return launch_k(align_expand_kernel, dim3((Ty + 127) / 128, B), dim3(128), 128 * sizeof(int), s, mu_x, x_mask, cum, ylen, B, M,
                    Tx, Ty, mu_y, y_mask, attn);
}

}  // namespace st

using namespace st;

extern "C" {

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

}  // extern "C"
