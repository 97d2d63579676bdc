// Monotonic alignment search of StableTTS's training forward (models/model.py:148-162; monotonic_align/__init__.py and
// core.py), SURVEY.md §8 row f8.  Three stages, all device-resident:
//
// 1. mas_scores_kernel: neg_cent[b, y, x] = c0 + (-0.5 Σ_d y[b,d,y]²) + Σ_d y[b,d,y] mu[b,d,x] + (-0.5 Σ_d mu[b,d,x]²),
//    c0 = -0.5 log(2π) D, the four terms of model.py:151-155 summed left to right in fp32.  64 x 64 output tiles over all
//    SMs, fp32 FMAs on CUDA cores: the path is discontinuous in the scores, so no split-bf16 tensor-core contraction.
//
// 2. mas_dp_kernel: one CTA per utterance runs the dynamic program of core.py:26-39 row by row.  Row y depends only on
//    row y-1, and only on the band x ∈ [max(0, t_x + y - t_y), min(t_x, y + 1)); threads span the band.  The arithmetic is
//    the reference's exactly:  value[y,x] = value[y,x] + (v_cur > v_prev ? v_cur : v_prev) as one fp32 add (numba forms
//    it in double and rounds once, which is the correctly rounded fp32 sum), with Python's max order (NaN / ±0 pick
//    v_prev).  The rows of neg_cent stream through a 4-row shared-memory ring by cp.async, three rows ahead of use.
//    The backtrack (core.py:41-46) needs, per visited cell, only the bit  x != 0 && (x == y || value[y-1,x] <
//    value[y-1,x-1])  — both operands lie in row y-1's band whenever t_x <= t_y — so the forward pass stores that bit per
//    band cell (shared memory while T_y·⌈T_x/32⌉ words fit, workspace otherwise) and never keeps the value matrix.  One
//    thread then walks the bits, writes the chosen token of each frame to workspace, and the CTA emits the per-token
//    frame counts d and their prefix sums cum.
//    Degenerate lengths, as the reference behaves:  t_x > t_y leaves every band empty and the walk compares the RAW
//    scores, reading row -1 at y = 0 as numpy does, i.e. the last padded row neg_cent[b, T_y - 1, ·];  t_y == 0 gives
//    an all-zero path.  t_x == 0 with t_y > 0 (a mask whose row 0 is empty but column 0 is not; no product of two prefix
//    masks gives it) makes the reference index negative columns out of bounds: here the path is all zeros.
//
// 3. mas_path_kernel: the dense 0/1 path (B, T_y, T_x) from the per-frame tokens, over all SMs.
//
// mas_loss_partial_kernel / mas_loss_final_kernel: prior_loss (model.py:175-176) and dur_loss (:162-163,
// duration_predictor.py:38-40) in double with a fixed summation order (fixed grid, fixed tree), so repeated calls are
// bit-identical.
#include "handle.cuh"
#include <algorithm>
#include <cmath>

namespace st {

namespace {

constexpr int MAS_THREADS = 512;
constexpr int MAS_RING = 4;                              // neg_cent rows in flight: the current one and three ahead
constexpr int MAS_SMEM_BUDGET = 227 * 1024 - 1024;       // sm_90 opt-in limit, less the static scan scratch
constexpr int LOSS_GRID = 264;                           // fixed: the partial sums' order must not depend on the device

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ int band_lo(int tx, int ty, int y) { return max(0, tx + y - ty); }
__device__ __forceinline__ int band_hi(int tx, int y) { return min(tx, y + 1); }

// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mas_scores_kernel(const float* __restrict__ y, const float* __restrict__ mu, int D, int Ty,
                                                         int Tx, float c0, float* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    constexpr int TILE = 64, DK = 16;
    __shared__ float ys[DK][TILE], ms[DK][TILE];
    const int b = blockIdx.z, y0 = blockIdx.y * TILE, x0 = blockIdx.x * TILE;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const float* yb = y + (long)b * D * Ty;
    const float* mb = mu + (long)b * D * Tx;
    float dot[4][4] = {}, sy[4] = {}, sm[4] = {};
    for (int d0 = 0; d0 < D; d0 += DK) {
        for (int i = threadIdx.x; i < DK * TILE; i += 256) {
            const int d = d0 + i / TILE, t = i % TILE;
            ys[i / TILE][t] = (d < D && y0 + t < Ty) ? yb[(long)d * Ty + y0 + t] : 0.f;
            ms[i / TILE][t] = (d < D && x0 + t < Tx) ? mb[(long)d * Tx + x0 + t] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < DK; ++k) {
            float a[4], m[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = ys[k][ty + 16 * i]; m[i] = ms[k][tx + 16 * i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                sy[i] = fmaf(a[i], a[i], sy[i]);
                sm[i] = fmaf(m[i], m[i], sm[i]);
#pragma unroll
                for (int j = 0; j < 4; ++j) dot[i][j] = fmaf(a[i], m[j], dot[i][j]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int yy = y0 + ty + 16 * i;
        if (yy >= Ty) continue;
        const float row = __fadd_rn(c0, -0.5f * sy[i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int xx = x0 + tx + 16 * j;
            if (xx < Tx) out[((long)b * Ty + yy) * Tx + xx] = __fadd_rn(__fadd_rn(row, dot[i][j]), -0.5f * sm[j]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// inclusive scan of one int per thread across the CTA (MAS_THREADS threads); returns the thread's inclusive prefix
__device__ int block_inclusive_scan(int v, int* warp_tot) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(~0u, v, o);
        if (lane >= o) v += n;
    }
    if (lane == 31) warp_tot[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int w = lane < MAS_THREADS / 32 ? warp_tot[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(~0u, w, o);
            if (lane >= o) w += n;
        }
        if (lane < MAS_THREADS / 32) warp_tot[lane] = w;
    }
    __syncthreads();
    return v + (warp > 0 ? warp_tot[warp - 1] : 0);
}

__device__ double block_sum_double(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(~0u, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < nw ? red[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(~0u, v, o);
    }
    return v;                                            // valid in thread 0
}

struct MasArgs {
    const float* nc; const float* mask; const long long* xlen; const long long* ylen;
    float* dur; float* cum;
    int* tok;                 // (B, Ty) workspace: chosen token of every frame, -1 where the path row is empty
    uint32_t* gbits;          // (B, Ty, W) workspace, or nullptr when the decision bits live in shared memory
    int Ty, Tx, W;
};

__global__ void __launch_bounds__(MAS_THREADS) mas_dp_kernel(MasArgs a) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) float smem[];
    __shared__ int warp_tot[32];
    __shared__ double red[32];
    __shared__ int s_len[2];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int Ty = a.Ty, Tx = a.Tx, W = a.W;
    const float* nc = a.nc + (long)b * Ty * Tx;

    // lengths: (int) sum(mask[b, :, 0]) and (int) sum(mask[b, 0, :]) (monotonic_align/__init__.py:13-14), or the length
    // vectors as the training forward's masks give them (t_x counts row 0 of x_mask ⊗ y_mask, so it is 0 when t_y is)
    if (a.mask) {
        const float* mb = a.mask + (long)b * Ty * Tx;
        double sy = 0.0, sx = 0.0;
        for (int i = tid; i < Ty; i += MAS_THREADS) sy += (double)mb[(long)i * Tx];
        for (int i = tid; i < Tx; i += MAS_THREADS) sx += (double)mb[i];
        sy = block_sum_double(sy, red);
        __syncthreads();
        sx = block_sum_double(sx, red);
        if (tid == 0) {
            s_len[0] = (int)fmin(fmax(sy, 0.0), (double)Ty);
            s_len[1] = (int)fmin(fmax(sx, 0.0), (double)Tx);
        }
    } else if (tid == 0) {
        const long long ly = min(max(a.ylen[b], 0ll), (long long)Ty), lx = min(max(a.xlen[b], 0ll), (long long)Tx);
        s_len[0] = lx > 0 ? (int)ly : 0;
        s_len[1] = ly > 0 ? (int)lx : 0;
    }
    __syncthreads();
    const int ty = s_len[0], tx = s_len[1];

    float* vals = smem;                                  // two rows of value: row y-1 and row y
    float* ring = smem + 2 * Tx;                         // MAS_RING rows of neg_cent
    uint32_t* bits = a.gbits ? a.gbits + (long)b * Ty * W : reinterpret_cast<uint32_t*>(smem + (2 + MAS_RING) * Tx);
    int* dcount = reinterpret_cast<int*>(smem);          // per-token frame counts, reusing `vals` after the DP

    const bool dp = tx >= 1 && tx <= ty;
    if (dp) {
        auto issue = [&](int r) {
            if (r < ty) {
                const int lo = band_lo(tx, ty, r), hi = band_hi(tx, r);
                float* dst = ring + (r % MAS_RING) * Tx;
                for (int x = lo + tid; x < hi; x += MAS_THREADS) cp_async4(dst + x, nc + (long)r * Tx + x);
            }
            cp_async_commit();
        };
        for (int r = 0; r < MAS_RING - 1; ++r) issue(r);
        for (int y = 0; y < ty; ++y) {
            cp_async_wait<MAS_RING - 2>();
            __syncthreads();                             // row y landed; row y-1 of value is complete; slot (y-1) is free
            issue(y + MAS_RING - 1);
            const float* row = ring + (y % MAS_RING) * Tx;
            const float* prv = vals + ((y + 1) & 1) * Tx;
            float* cur = vals + (y & 1) * Tx;
            const int lo = band_lo(tx, ty, y), hi = band_hi(tx, y);
            for (int x = (lo & ~31) + tid; x - lane < hi; x += MAS_THREADS) {
                bool bit = false;
                if (x >= lo && x < hi) {
                    const float v_cur = x == y ? -1e9f : prv[x];                                  // core.py:28-31
                    const float v_prev = x == 0 ? (y == 0 ? 0.f : -1e9f) : prv[x - 1];            // :32-38
                    cur[x] = __fadd_rn(row[x], v_cur > v_prev ? v_cur : v_prev);                  // :39
                    bit = x != 0 && (x == y || prv[x] < prv[x - 1]);                              // :43-45
                }
                const uint32_t word = __ballot_sync(~0u, bit);
                if (lane == 0) bits[(long)y * W + ((x - lane) >> 5)] = word;
            }
        }
        cp_async_wait<0>();
    }
    __syncthreads();
    for (int x = tid; x < Tx; x += MAS_THREADS) dcount[x] = 0;
    __syncthreads();

    // backtrack (core.py:41-46): one thread; tok[b, y] = the token of frame y
    int* tok = a.tok + (long)b * Ty;
    if (tid == 0) {
        int index = tx - 1, y = ty - 1;
        if (tx >= 1) {
            for (; y >= 0; --y) {
                tok[y] = index;
                ++dcount[index];
                bool dec;
                if (dp) {
                    dec = (bits[(long)y * W + (index >> 5)] >> (index & 31)) & 1u;
                } else {                                 // t_x > t_y: raw scores, row -1 is the last padded row
                    const float* pr = nc + (long)(y == 0 ? Ty - 1 : y - 1) * Tx;
                    dec = index != 0 && (index == y || pr[index] < pr[index - 1]);
                }
                if (dec) --index;
            }
        }
        for (y = max(ty, 0); y < Ty; ++y) tok[y] = -1;
        if (tx < 1) for (y = 0; y < ty; ++y) tok[y] = -1;
    }
    __syncthreads();

    // d (attn.sum over frames, model.py:162) and its inclusive prefix sums (exact: integers below 2^24)
    if (a.dur || a.cum) {
        const int chunk = (Tx + MAS_THREADS - 1) / MAS_THREADS, x0 = tid * chunk, x1 = min(x0 + chunk, Tx);
        int s = 0;
        for (int x = x0; x < x1; ++x) s += dcount[x];
        int run = block_inclusive_scan(s, warp_tot) - s;
        for (int x = x0; x < x1; ++x) {
            run += dcount[x];
            if (a.dur) a.dur[(long)b * Tx + x] = (float)dcount[x];
            if (a.cum) a.cum[(long)b * Tx + x] = (float)run;
        }
    }
}

__global__ void mas_path_kernel(const int* __restrict__ tok, long rows, int Tx, float* __restrict__ path) {
    pdl_trigger(); pdl_wait();
    for (long r = blockIdx.y; r < rows; r += gridDim.y) {
        const int t = tok[r];
        for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < Tx; x += gridDim.x * blockDim.x) path[r * Tx + x] = x == t ? 1.f : 0.f;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mas_loss_partial_kernel(const float* __restrict__ y, const float* __restrict__ mu_y,
                                                               const float* __restrict__ y_mask, const float* __restrict__ logw,
                                                               const float* __restrict__ x_mask, const float* __restrict__ dur,
                                                               int B, int M, int Ty, int Tx, double* __restrict__ part) {
    pdl_trigger(); pdl_wait();
    __shared__ double red[32];
    const long stride = (long)gridDim.x * blockDim.x, i0 = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const float log2pi = 1.8378770664093453f;
    double sp = 0.0, sm = 0.0, sd = 0.0;
    const long n_prior = (long)B * M * Ty;
    for (long i = i0; i < n_prior; i += stride) {        // 0.5 ((y - mu_y)^2 + log 2π) y_mask   (model.py:175)
        const long t = i % Ty, b = i / ((long)M * Ty);
        const float m = y_mask[b * Ty + t];
        const float d = y[i] - mu_y[i];
        sp += (double)(0.5f * (d * d + log2pi) * m);
    }
    for (long i = i0; i < (long)B * Ty; i += stride) sm += (double)y_mask[i];
    for (long i = i0; i < (long)B * Tx; i += stride) {   // (logw - log(1e-8 + d) x_mask)^2   (model.py:162, dp.py:39)
        const float xm = x_mask[i];
        const float e = logw[i] - logf(1e-8f + dur[i]) * xm;
        sd += (double)(e * e);
    }
    sp = block_sum_double(sp, red);
    __syncthreads();
    sm = block_sum_double(sm, red);
    __syncthreads();
    sd = block_sum_double(sd, red);
    if (threadIdx.x == 0) {
        part[blockIdx.x * 3 + 0] = sp;
        part[blockIdx.x * 3 + 1] = sm;
        part[blockIdx.x * 3 + 2] = sd;
    }
}

__global__ void mas_loss_final_kernel(const double* __restrict__ part, const long long* __restrict__ x_lengths, int B, int M,
                                      float* __restrict__ prior_loss, float* __restrict__ dur_loss) {
    pdl_trigger(); pdl_wait();
    __shared__ double red[32];
    double sp = 0.0, sm = 0.0, sd = 0.0;
    for (int i = threadIdx.x; i < LOSS_GRID; i += blockDim.x) { sp += part[3 * i]; sm += part[3 * i + 1]; sd += part[3 * i + 2]; }
    sp = block_sum_double(sp, red);
    __syncthreads();
    sm = block_sum_double(sm, red);
    __syncthreads();
    sd = block_sum_double(sd, red);
    if (threadIdx.x == 0) {
        long long nx = 0;
        for (int b = 0; b < B; ++b) nx += x_lengths[b];
        *prior_loss = (float)(sp / (sm * (double)M));
        *dur_loss = (float)(sd / (double)nx);
    }
}

std::atomic<uint64_t> g_dp_smem_done{0};

int mas_words(int Tx) { return (Tx + 31) / 32; }
size_t mas_base_smem(int Tx) { return (size_t)(2 + MAS_RING) * Tx * sizeof(float); }
bool mas_bits_in_smem(int Ty, int Tx) {
    return mas_base_smem(Tx) + (size_t)Ty * mas_words(Tx) * 4 <= (size_t)MAS_SMEM_BUDGET;
}

}  // namespace

int mas_max_tx() { return MAS_SMEM_BUDGET / (int)((2 + MAS_RING) * sizeof(float)) / 32 * 32; }

size_t mas_workspace_bytes(int B, int Ty, int Tx) {
    const size_t tok = ((size_t)B * Ty * sizeof(int) + 255) / 256 * 256;
    const size_t bits = mas_bits_in_smem(Ty, Tx) ? 0 : (size_t)B * Ty * mas_words(Tx) * 4;
    const size_t loss = (size_t)LOSS_GRID * 3 * sizeof(double);
    return std::max(tok + bits, loss);
}

cudaError_t launch_mas_scores(const float* y, const float* mu_x, float* neg_cent, int B, int D, int Ty, int Tx, cudaStream_t s) {
    if (B == 0 || Ty == 0 || Tx == 0) return cudaSuccess;
    const float c0 = (float)(-0.5 * std::log(2.0 * 3.14159265358979323846) * D);
    return launch_k(mas_scores_kernel, dim3((Tx + 63) / 64, (Ty + 63) / 64, B), dim3(256), 0, s, y, mu_x, D, Ty, Tx, c0, neg_cent);
}

cudaError_t launch_maximum_path(const float* neg_cent, const float* mask, const long long* xlen, const long long* ylen, float* path,
                                float* dur, float* cum, void* ws, int B, int Ty, int Tx, cudaStream_t s) {
    if (B == 0 || Ty == 0 || Tx == 0) return cudaSuccess;
    MasArgs a{};
    a.nc = neg_cent; a.mask = mask; a.xlen = xlen; a.ylen = ylen; a.dur = dur; a.cum = cum;
    a.Ty = Ty; a.Tx = Tx; a.W = mas_words(Tx);
    a.tok = static_cast<int*>(ws);
    const bool in_smem = mas_bits_in_smem(Ty, Tx);
    a.gbits = in_smem ? nullptr
                      : reinterpret_cast<uint32_t*>(static_cast<char*>(ws) + ((size_t)B * Ty * sizeof(int) + 255) / 256 * 256);
    const size_t smem = mas_base_smem(Tx) + (in_smem ? (size_t)Ty * a.W * 4 : 0);
    cudaError_t e = ensure_dyn_smem(mas_dp_kernel, MAS_SMEM_BUDGET, g_dp_smem_done);
    if (e != cudaSuccess) return e;
    e = launch_k(mas_dp_kernel, dim3(B), dim3(MAS_THREADS), smem, s, a);
    if (e != cudaSuccess || !path) return e;
    const long rows = (long)B * Ty;
    return launch_k(mas_path_kernel, dim3(std::min((Tx + 127) / 128, 8), (unsigned)std::min<long>(rows, 8192)), dim3(128), 0, s,
                    (const int*)a.tok, rows, Tx, path);
}

cudaError_t launch_mas_losses(const float* y, const float* mu_y, const float* y_mask, const float* logw, const float* x_mask,
                              const float* dur, const long long* x_lengths, void* ws, int B, int M, int Ty, int Tx, float* prior_loss,
                              float* dur_loss, cudaStream_t s) {
    double* part = static_cast<double*>(ws);
    cudaError_t e = launch_k(mas_loss_partial_kernel, dim3(LOSS_GRID), dim3(256), 0, s, y, mu_y, y_mask, logw, x_mask, dur, B, M,
                             Ty, Tx, part);
    if (e != cudaSuccess) return e;
    return launch_k(mas_loss_final_kernel, dim3(1), dim3(256), 0, s, (const double*)part, x_lengths, B, M, prior_loss, dur_loss);
}

}  // namespace st

using namespace st;

extern "C" {

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

}  // extern "C"
