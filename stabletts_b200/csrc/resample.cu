// Band-limited polyphase resampling: torchaudio.functional.resample (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99)
// as the reference calls it in utils/audio.py:73 (load_and_resample_audio: api.py:72, preprocess.py:65), and
// torchaudio.transforms.Resample.  The contract is in include/stabletts_b200.h and oracle/resample_ref.py.
//
// The coefficient table keeps, for every phase j, only its band [k0_j, k0_j + cnt_j) of non-zero fp32 coefficients (the
// taps clamped to t = ±6 are exactly 0 in fp32): 14 taps per output at 48 kHz -> 44.1 kHz, where torchaudio's dense
// conv1d runs 174.  The default table is evaluated in double on the host and rounded once; a loaded `kernel` buffer
// replaces it at st_finalize_weights and is used as loaded.
//
// resample_kernel: a CTA takes I consecutive blocks of N outputs of one row.  It stages their input span into shared memory
// with one coalesced load (zeros outside [0, L)), stages the table too when it fits, and each thread writes outputs
// q, q + 256, ... of the run: consecutive threads write consecutive outputs.  Each output sums its band in ascending k with
// fp32 FMA.  No atomics and no host synchronisation; a row's output depends only on that row.
#include "handle.cuh"

#include <cmath>

using namespace st;

namespace st {

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_TARGET_OUT = 4096;            // outputs per CTA to aim for
constexpr int RS_SPAN_TARGET = 8192;           // input floats per CTA to aim for (32 KB)
constexpr int RS_SPAN_MAX = 48 * 1024;         // input floats of one block of N outputs, at most (192 KB)
constexpr int RS_TABLE_SMEM = 32 * 1024;       // the table goes to shared memory when it takes at most this many bytes
constexpr int RS_SMEM_MAX = 220 * 1024;

struct ResampleArgs {
    const float* x = nullptr;      // (rows, L)
    float* y = nullptr;            // (rows, out_len)
    const float* coef = nullptr;   // (bw, N): tap c of phase j at c * N + j
    const int2* band = nullptr;    // (N): (k0_j - kmin, cnt_j)
    long long L = 0, out_len = 0, rows = 0;
    int O = 0, N = 0, width = 0, kmin = 0, bw = 0, I = 0, span = 0;
};

template <bool SMEM_TABLE>
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(ResampleArgs a) {
    extern __shared__ __align__(16) float rs_sm[];
    float* xs = rs_sm;
    const float* coef = a.coef;
    const int2* band = a.band;
    if (SMEM_TABLE) {
        int2* bs = (int2*)(rs_sm + ((a.span + 3) & ~3));
        float* cs = (float*)(bs + a.N);
        for (int t = threadIdx.x; t < a.N; t += RS_THREADS) bs[t] = a.band[t];
        for (int t = threadIdx.x; t < a.N * a.bw; t += RS_THREADS) cs[t] = __ldg(a.coef + t);
        coef = cs;
        band = bs;
    }
    const long long i0 = (long long)blockIdx.x * a.I;            // first block of N outputs of this CTA
    const long long s0 = i0 * a.O + a.kmin - a.width;            // x index of xs[0]
    const long long p0 = i0 * a.N;
    const int P = (int)min((long long)a.I * a.N, a.out_len - p0);
    for (long long row = blockIdx.y; row < a.rows; row += gridDim.y) {
        const float* x = a.x + row * a.L;
        for (int t = threadIdx.x; t < a.span; t += RS_THREADS) {
            const long long m = s0 + t;
            xs[t] = (m >= 0 && m < a.L) ? __ldg(x + m) : 0.f;
        }
        __syncthreads();
        float* y = a.y + row * a.out_len + p0;
        for (int q = threadIdx.x; q < P; q += RS_THREADS) {
            const int i = q / a.N, j = q - i * a.N;
            const int2 b = SMEM_TABLE ? band[j] : __ldg(band + j);
            const float* xp = xs + i * a.O + b.x;
            const float* cp = coef + j;
            float acc = 0.f;
            for (int c = 0; c < b.y; ++c) acc = fmaf(SMEM_TABLE ? cp[c * a.N] : __ldg(cp + (long long)c * a.N), xp[c], acc);
            y[q] = acc;
        }
        __syncthreads();
    }
}

cudaError_t launch_resample(const ResampleArgs& a, bool smem_table, cudaStream_t s) {
    const long long blocks = (a.out_len + a.N - 1) / a.N;
    const dim3 grid((unsigned)((blocks + a.I - 1) / a.I), (unsigned)std::min<long long>(a.rows, 65535));
    size_t smem = (size_t)((a.span + 3) & ~3) * 4;
    if (smem_table) smem += (size_t)a.N * 8 + (size_t)a.N * a.bw * 4;
    auto kern = smem_table ? resample_kernel<true> : resample_kernel<false>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    kern<<<grid, RS_THREADS, smem, s>>>(a);
    return cudaGetLastError();
}

}  // namespace

struct ResampleState : Model {
    int O = 0, N = 0, width = 0;
    double base = 0;
    // the packed table on the host: the default (float64 formula rounded once) and the one in use
    std::vector<float> def_coef; std::vector<int2> def_band; int def_bw = 0;
    // in use, on the device
    float* coef = nullptr; int2* band = nullptr;
    int bw = 0, kmin = 0, kspan = 0, I = 1, span = 0;
    bool smem_table = false;
    int finalize(st_handle* h, cudaStream_t s) override;
};

namespace {

// the contract's coefficient of phase j, tap k, in double, in the order oracle/resample_ref.py states it
double rs_coef(const ResampleState& r, int j, int k) {
    double t = ((double)(k - r.width) / r.O - (double)j / r.N) * r.base;
    t = std::min(6.0, std::max(-6.0, t));
    const double w = std::cos(t * M_PI / 6 / 2);
    const double window = w * w;
    const double pt = t * M_PI;
    const double sinc = pt == 0 ? 1.0 : std::sin(pt) / pt;
    return sinc * (window * (r.base / r.O));
}

// phase j's taps come from row(j)[0 .. 2 width + O); packs the non-zero band of every phase into coef [bw][N] / band [N]
template <class Row>
const char* rs_pack(const ResampleState& r, Row row, std::vector<float>& coef, std::vector<int2>& band, int& bw) {
    band.assign(r.N, int2{0, 0});
    bw = 0;
    std::vector<std::pair<int, int>> lim(r.N);
    for (int j = 0; j < r.N; ++j) {
        int k0 = -1, k1 = 0;
        row(j, [&](int k, float c) { if (c != 0.f) { if (k0 < 0) k0 = k; k1 = k + 1; } });
        if (k0 < 0) k0 = k1 = 0;
        lim[j] = {k0, k1};
        bw = std::max(bw, k1 - k0);
        if ((int64_t)r.N * bw > ST_RESAMPLE_MAX_TABLE) return "the table of this pair exceeds the bound: N x band > ST_RESAMPLE_MAX_TABLE";
    }
    coef.assign((size_t)std::max(bw, 1) * r.N, 0.f);
    for (int j = 0; j < r.N; ++j) {
        band[j] = int2{lim[j].first, lim[j].second - lim[j].first};
        row(j, [&](int k, float c) { if (k >= lim[j].first && k < lim[j].second) coef[(size_t)(k - lim[j].first) * r.N + j] = c; });
    }
    return nullptr;
}

// the default table: phase j is non-zero only where |t| < 6, k in (width + O j / N - 6 O / base, width + O j / N + 6 O / base)
const char* rs_default_table(ResampleState& r) {
    const int K = 2 * r.width + r.O;
    const int64_t grid = (int64_t)std::ceil(12.0 * r.O / r.base) + 3;
    // every phase has at least 5/8 of its evaluation grid non-zero, so a grid over 4x the bound is a table over the bound
    if (r.N > ST_RESAMPLE_MAX_TABLE || (int64_t)r.N * grid > 4 * (int64_t)ST_RESAMPLE_MAX_TABLE)
        return "the table of this pair exceeds the bound: N x band > ST_RESAMPLE_MAX_TABLE";
    auto row = [&](int j, auto&& emit) {
        const int lo = std::max(0, (int)std::floor(r.width + (double)r.O * j / r.N - 6.0 * r.O / r.base) - 1);
        const int hi = std::min<int64_t>(K, lo + grid);
        for (int k = lo; k < hi; ++k) emit(k, (float)rs_coef(r, j, k));
    };
    return rs_pack(r, row, r.def_coef, r.def_band, r.def_bw);
}

// device copy of a packed table + the launch geometry it implies
int rs_install(st_handle* h, ResampleState& r, const std::vector<float>& coef, std::vector<int2> band, int bw) {
    int kmin = INT32_MAX, kmax = 0;
    for (const int2& b : band) { kmin = std::min(kmin, b.x); kmax = std::max(kmax, b.x + b.y); }
    if (kmin > kmax) kmin = kmax;
    for (int2& b : band) b.x -= kmin;
    r.bw = bw; r.kmin = kmin; r.kspan = kmax - kmin;
    if ((int64_t)r.O + r.kspan > RS_SPAN_MAX)
        return fail(h, "the input span of one block of outputs (O + the table's tap span = " + std::to_string(r.O + r.kspan) +
                           " samples) exceeds " + std::to_string(RS_SPAN_MAX) + " (shared memory)");
    int64_t I = std::max<int64_t>(1, (RS_TARGET_OUT + r.N - 1) / r.N);
    I = std::min<int64_t>(I, std::max<int64_t>(1, (RS_SPAN_TARGET - r.kspan) / r.O));
    r.I = (int)I;
    r.span = (int)(I * r.O + r.kspan);
    const size_t table_bytes = (size_t)r.N * 8 + coef.size() * 4;
    r.smem_table = table_bytes <= RS_TABLE_SMEM && (size_t)((r.span + 3) & ~3) * 4 + table_bytes <= RS_SMEM_MAX;
    if (dev_alloc(h, &r.coef, coef.size()) || dev_alloc(h, &r.band, band.size())) return 1;
    ST_CUDA(cudaMemcpy(r.coef, coef.data(), coef.size() * 4, cudaMemcpyHostToDevice));
    ST_CUDA(cudaMemcpy(r.band, band.data(), band.size() * sizeof(int2), cudaMemcpyHostToDevice));
    return 0;
}

}  // namespace

// a loaded "kernel" ((N, 1, 2 width + O) as torchaudio.transforms.Resample) replaces the default table; without one the
// default table is re-installed (st_finalize_weights frees every packed buffer first)
int ResampleState::finalize(st_handle* h, cudaStream_t s) {
    if (h->raw.find("kernel") == h->raw.end()) return rs_install(h, *this, def_coef, def_band, def_bw);
    const int K = 2 * width + O;
    float* kd;
    if (get_raw(h, "kernel", (int64_t)N * K, &kd)) return 1;
    std::vector<float> kh((size_t)N * K);
    ST_CUDA(cudaMemcpyAsync(kh.data(), kd, kh.size() * 4, cudaMemcpyDeviceToHost, s));
    ST_CUDA(cudaStreamSynchronize(s));
    std::vector<float> coef; std::vector<int2> band; int bw = 0;
    auto row = [&](int j, auto&& emit) { for (int k = 0; k < K; ++k) emit(k, kh[(size_t)j * K + k]); };
    if (const char* e = rs_pack(*this, row, coef, band, bw)) return fail(h, std::string("loaded kernel: ") + e);
    return rs_install(h, *this, coef, band, bw);
}

}  // namespace st

extern "C" {

int st_create_resample(int32_t orig_freq, int32_t new_freq, int device, st_handle** out) {
    if (!out) return fail(nullptr, "st_create_resample: null argument");
    if (orig_freq <= 0 || new_freq <= 0) return fail(nullptr, "sample rates must be positive");
    if (orig_freq == new_freq) return fail(nullptr, "orig_freq == new_freq: resampling is the identity (no handle needed)");
    auto r = std::make_unique<ResampleState>();
    int64_t a = orig_freq, b = new_freq;
    while (b) { int64_t t = a % b; a = b; b = t; }
    r->O = (int)(orig_freq / a); r->N = (int)(new_freq / a);
    r->base = std::min(r->O, r->N) * 0.99;
    r->width = (int)std::ceil(6 * (double)r->O / r->base);
    if (const char* e = rs_default_table(*r))
        return fail(nullptr, std::string(e) + " (" + std::to_string(orig_freq) + " -> " + std::to_string(new_freq) + ")");
    if (int rc = create_handle(device, std::move(r), out)) return rc;
    st_handle* h = *out;
    ST_ENTER(h);
    if (h->model->finalize(h, nullptr)) {                 // the default table
        std::string e = h->err;
        st_destroy(h);
        *out = nullptr;
        return fail(nullptr, e);
    }
    h->finalized = true;
    return 0;
}

int64_t st_resample_out_length(const st_handle* h, int64_t L) {
    const ResampleState* r = h ? dynamic_cast<const ResampleState*>(h->model.get()) : nullptr;
    if (!r || L < 0) return -1;
    return (r->N * L + r->O - 1) / r->O;
}

int st_resample_forward(st_handle* h, const float* x, float* y, int64_t rows, int64_t L, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    const ResampleState* r = ready_model<ResampleState>(h, "resampler");
    if (!r) return 1;
    if (rows < 0 || L < 0) return fail(h, "rows and L must be non-negative");
    if (L > ((int64_t)1 << 40) / std::max(1, r->N)) return fail(h, "input too long");
    const int64_t out_len = (r->N * L + r->O - 1) / r->O;
    if (rows == 0 || out_len == 0) return 0;
    if (!x || !y) return fail(h, "st_resample_forward: null pointer");
    ResampleArgs a;
    a.x = x; a.y = y; a.coef = r->coef; a.band = r->band;
    a.L = L; a.out_len = out_len; a.rows = rows;
    a.O = r->O; a.N = r->N; a.width = r->width; a.kmin = r->kmin; a.bw = r->bw; a.I = r->I; a.span = r->span;
    ST_LAUNCH(launch_resample(a, r->smem_table, (cudaStream_t)stream));
    return 0;
}

}  // extern "C"
