// fp32 SIMT conv-GEMM engine: the straightforward, obviously-correct implementation of the
// GemmArgs contract (k-tap Conv1d as shifted accumulating GEMMs, dual-source A for the long-skip
// concat, fused bias/SiLU/FiLM/mask/gate/residual epilogue).  It is the on-device cross-check for
// the wgmma engine (tests compare both against the oracle) and a debugging engine
// (st_set_engine); the wgmma engine in gemm_tc.cu is the product path.
#include "common.cuh"

namespace st {

constexpr int SM_BM = 64, SM_BN = 64, SM_BK = 16;

__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmArgs g) {
    pdl_trigger(); pdl_wait();
    __shared__ __align__(16) float As[SM_BK][SM_BM + 4];
    __shared__ __align__(16) float Ws[SM_BK][SM_BN + 4];
    const int bb = blockIdx.z;
    const int t0 = blockIdx.x * SM_BM, n0 = blockIdx.y * SM_BN;
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    const int lrow = tid >> 2, lk = (tid & 3) * 4;
    const int ab = bb % g.a_bmod;
    const int pad = g.taps / 2;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int tap = 0; tap < g.taps; ++tap) {
        int koff = 0;
        for (int src = 0; src < g.n_src; ++src) {
            const int C = g.Cs[src];
            const float* Ab = g.A_f32[src] + (long)ab * g.T * C;
            const int ta = t0 + lrow + (tap - pad) * g.dil;
            const bool arow_ok = (ta >= 0 && ta < g.T);
            const int wn = n0 + lrow;
            const float* Wr = g.W_f32 + ((long)tap * g.N + min(wn, g.N - 1)) * g.Ktot + koff;
            for (int kc = 0; kc < C; kc += SM_BK) {
                float4 av = make_float4(0.f, 0.f, 0.f, 0.f), wv = make_float4(0.f, 0.f, 0.f, 0.f);
                if (arow_ok) av = *reinterpret_cast<const float4*>(Ab + (long)ta * C + kc + lk);
                if (wn < g.N) wv = *reinterpret_cast<const float4*>(Wr + kc + lk);
                __syncthreads();
                As[lk + 0][lrow] = av.x; As[lk + 1][lrow] = av.y; As[lk + 2][lrow] = av.z; As[lk + 3][lrow] = av.w;
                Ws[lk + 0][lrow] = wv.x; Ws[lk + 1][lrow] = wv.y; Ws[lk + 2][lrow] = wv.z; Ws[lk + 3][lrow] = wv.w;
                __syncthreads();
#pragma unroll
                for (int k = 0; k < SM_BK; ++k) {
                    float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
                    float4 b4 = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
                    float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
                }
            }
            koff += C;
        }
    }

    const int mb = bb % g.B;
    const int cb = min(bb, g.c_clamp);
    const int rb = min(bb, g.resid_clamp);
    const float* film = (g.flags & EPI_FILM) ? g.film + (long)mb * g.film_bstride : nullptr;
    const float* gate = (g.flags & EPI_GATE) ? g.gate + (long)cb * g.gate_bstride : nullptr;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + ty * 4 + i;
        if (t >= g.T) continue;
        const float m = (g.flags & EPI_MASK) ? g.mask[(long)mb * g.T + t] : 1.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= g.N) continue;
            float v = acc[i][j];
            if (g.flags & EPI_BIAS) v += g.bias[n];
            if (g.flags & EPI_SILU) v = silu_f(v);
            else if (g.flags & EPI_GELU) v = gelu_f(v);
            else if (g.flags & EPI_MISH) v = mish_f(v);
            if (g.flags & EPI_FILM) v = film[n] * v + film[g.film_H + n];
            if (g.flags & EPI_MASK) v *= m;
            if (g.flags & EPI_GATE) v *= gate[n];
            if (g.flags & EPI_RESID) v += g.resid[((long)rb * g.T + t) * g.N + n];
            const long o = ((long)bb * g.T + t) * g.N + n;
            if (g.out_f32) g.out_f32[o] = v;
            if (g.flags & EPI_SILU_OUT) {
                v = silu_f(v);
                if (g.out2_f32) g.out2_f32[o] = v;
            }
            if (g.out_hi) { bf16 h, l; split_bf16(v, h, l); g.out_hi[o] = h; g.out_lo[o] = l; }
        }
    }
}

// Second half of a split-K conv-GEMM: sums the ksplit raw partial tiles in slice order (deterministic) and applies the
// epilogue of the SIMT engine above; one thread per 4 consecutive channels of a frame.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(GemmArgs g) {
    pdl_trigger(); pdl_wait();
    const long n4 = g.N / 4;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)g.BB * g.T * n4) return;
    const int n = (int)(i % n4) * 4;
    const long row = i / n4;
    const int bb = (int)(row / g.T), t = (int)(row - (long)bb * g.T);
    const long o = row * g.N + n;
    const long slice = (long)g.BB * g.T * g.N;
    float4 a = *reinterpret_cast<const float4*>(g.part + o);
    for (int s = 1; s < g.ksplit; ++s) {
        const float4 b = *reinterpret_cast<const float4*>(g.part + s * slice + o);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    float v[4] = {a.x, a.y, a.z, a.w};
    const int mb = bb % g.B;
    const float m = (g.flags & EPI_MASK) ? g.mask[(long)mb * g.T + t] : 1.f;
    const float* film = (g.flags & EPI_FILM) ? g.film + (long)mb * g.film_bstride : nullptr;
    const float* gate = (g.flags & EPI_GATE) ? g.gate + (long)min(bb, g.c_clamp) * g.gate_bstride : nullptr;
    const float* resid = (g.flags & EPI_RESID) ? g.resid + ((long)min(bb, g.resid_clamp) * g.T + t) * g.N : nullptr;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float x = v[e];
        if (g.flags & EPI_BIAS) x += g.bias[n + e];
        if (g.flags & EPI_SILU) x = silu_f(x);
        else if (g.flags & EPI_GELU) x = gelu_f(x);
        else if (g.flags & EPI_MISH) x = mish_f(x);
        if (g.flags & EPI_FILM) x = film[n + e] * x + film[g.film_H + n + e];
        if (g.flags & EPI_MASK) x *= m;
        if (g.flags & EPI_GATE) x *= gate[n + e];
        if (g.flags & EPI_RESID) x += resid[n + e];
        v[e] = x;
    }
    if (g.out_f32) *reinterpret_cast<float4*>(g.out_f32 + o) = make_float4(v[0], v[1], v[2], v[3]);
    if (g.flags & EPI_SILU_OUT) {
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = silu_f(v[e]);
        if (g.out2_f32) *reinterpret_cast<float4*>(g.out2_f32 + o) = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (g.out_hi) {
        uint32_t h01, l01, h23, l23;
        split_bf16x2(v[0], v[1], h01, l01); split_bf16x2(v[2], v[3], h23, l23);
        *reinterpret_cast<uint2*>(g.out_hi + o) = make_uint2(h01, h23);
        *reinterpret_cast<uint2*>(g.out_lo + o) = make_uint2(l01, l23);
    }
}

cudaError_t launch_splitk_reduce(const GemmArgs& g, cudaStream_t s) {
    if (g.N % 4 || !g.part || g.ksplit < 2) return cudaErrorInvalidValue;
    const long n = (long)g.BB * g.T * (g.N / 4);
    if (n == 0) return cudaSuccess;
    return launch_k(splitk_reduce_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, g);
}

const char* gemm_simt_unsupported(const GemmArgs& g) {
    if (const char* why = gemm_flags_error(g)) return why;
    if (g.ln || g.prec || g.out16 || g.u16 || (g.flags & EPI_ROPE))
        return "the SIMT engine has no fused LayerNorm, fp16 planes (prec / out16 / u16) or RoPE epilogue";
    for (int i = 0; i < g.n_src; ++i)
        if (g.Cs[i] % SM_BK != 0 || !g.A_f32[i]) return "SIMT engine: A channels must be a multiple of 16 (fp32 A planes required)";
    if (!g.W_f32 || g.Ktot % 4 != 0 || g.dil < 1) return "SIMT engine: bad weight operand or dilation";
    return nullptr;
}

cudaError_t launch_gemm_simt(const GemmArgs& g, cudaStream_t s) {
    if (g.BB == 0 || g.T == 0) return cudaSuccess;
    if (gemm_simt_unsupported(g)) return cudaErrorInvalidValue;
    dim3 grid((g.T + SM_BM - 1) / SM_BM, (g.N + SM_BN - 1) / SM_BN, g.BB);
    gemm_simt_kernel<<<grid, 256, 0, s>>>(g);
    if (g.plan) { *g.plan = GemmPlan(); g.plan->engine = ST_ENGINE_SIMT; g.plan->bn = SM_BN; g.plan->grid = (int)(grid.x * grid.y * grid.z); }
    return cudaGetLastError();
}

}  // namespace st
