// Kernel-level test hooks of the C-ABI: the conv-GEMM (st_test_gemm_ex, and st_test_conv_ex for dilated and transposed
// convs), attention, the row kernels and the layout / split / packing kernels on caller-given operands, and a conv-GEMM
// timing loop on synthetic data (st_bench_conv).  Each allocates its scratch per call and waits for its work before it returns.
#include "handle.cuh"
#include "ffgan.cuh"
#include "vocos.cuh"
#include "mel.cuh"

using namespace st;

namespace {

static_assert(ST_TEST_EPI_BIAS == EPI_BIAS && ST_TEST_EPI_SILU == EPI_SILU && ST_TEST_EPI_FILM == EPI_FILM &&
              ST_TEST_EPI_MASK == EPI_MASK && ST_TEST_EPI_GATE == EPI_GATE && ST_TEST_EPI_RESID == EPI_RESID &&
              ST_TEST_EPI_ROPE == EPI_ROPE && ST_TEST_EPI_GELU == EPI_GELU && ST_TEST_EPI_SILU_OUT == EPI_SILU_OUT &&
              ST_TEST_EPI_MISH == EPI_MISH,
              "st_test_gemm_desc::flags are the EPI_* bits");

const char* test_gemm_desc_error(const st_test_gemm_desc& d) {
    if (d.B < 1 || d.BB < 1 || d.T < 1 || d.a_bmod < 1 || d.a_bmod > d.BB) return "B, BB, T >= 1 and 1 <= a_bmod <= BB";
    if ((d.n_src != 1 && d.n_src != 2) || d.C0 < 1 || (d.n_src == 2 ? d.C1 < 1 : d.C1 != 0)) return "n_src 1 (C1 = 0) or 2, channels >= 1";
    if (!d.A0 || (d.n_src == 2 && !d.A1) || !d.W) return "A0 [, A1] and W are required";
    if (d.N < 1 || d.taps < 1 || d.dil < 1) return "N, taps, dil >= 1";
    if (d.flags & ~EPI_ALL) return "unknown flag";
    if (d.c_clamp < 0 || d.resid_clamp < 0 || d.film_bstride < 0 || d.gate_bstride < 0 || d.ada_bstride < 0 || d.film2_bstride < 0)
        return "clamps and batch strides must be >= 0";
    if ((d.flags & EPI_BIAS) && !d.bias) return "EPI_BIAS needs bias";
    if ((d.flags & EPI_MASK) && !d.mask) return "EPI_MASK needs mask";
    if ((d.flags & EPI_FILM) && !d.film) return "EPI_FILM needs film";
    if (((d.flags & EPI_FILM) || d.film2) && d.film_H < d.N) return "film_H (the beta offset) must be >= N";
    if ((d.flags & EPI_GATE) && !d.gate) return "EPI_GATE needs gate";
    if ((d.flags & EPI_RESID) && !d.resid) return "EPI_RESID needs resid";
    if ((d.flags & EPI_ROPE) && (d.rope_H < 64 || d.rope_H % 64 || 2 * d.rope_H > d.N)) return "EPI_ROPE needs rope_H % 64 == 0, 2 rope_H <= N";
    if (d.ln && (!d.ln_shift || !d.ln_scale || !d.u_hi || (!d.u16 && !d.u_lo))) return "ln needs ln_shift, ln_scale and the u planes";
    if (!d.ln && (d.u_hi || d.u_lo || d.u16 || d.film2 || d.ln_mask_out)) return "u planes, u16, film2 and ln_mask_out belong to ln";
    if (d.film2 && !d.out2_f32) return "film2 needs out2_f32";
    if (d.out2_f32 && !d.film2 && !(d.flags & EPI_SILU_OUT)) return "out2_f32 is written by EPI_SILU_OUT or film2 only";
    if (d.out16 && !d.out_hi) return "out16 needs out_hi";
    if (d.out_hi && !d.out16 && !d.out_lo) return "out_hi needs out_lo (or out16)";
    if (!d.out_f32 && !d.out_hi && !d.out2_f32 && !d.u_hi) return "no output requested";
    if (d.ksplit < 0 || d.ksplit > 4 || d.num_sms < 0) return "ksplit in [0, 4], num_sms >= 0";
    return nullptr;
}

const char* test_attn_desc_error(const st_test_attn_desc& d, bool tc) {
    if (d.n_heads < 1 || d.n_heads > 65535 || d.H != 64 * d.n_heads) return "H must be 64 n_heads (n_heads >= 1)";
    if (d.B < 1 || d.T < 1 || d.BB < 1 || d.BB % d.B || d.BB > 65535) return "B, T >= 1 and BB a positive multiple of B (<= 65535)";
    if (!d.mask) return "mask is required";
    if (!d.out_f32 && !d.out_hi && !d.out_lo) return "no output requested";
    if (!d.out_hi != !d.out_lo) return "out_hi and out_lo go together";
    if (d.rope != 0 && d.rope != 1) return "rope is 0 or 1";
    if (tc && (!d.qkv_hi || !d.qkv_lo)) return "the wgmma engine needs the split planes qkv_hi and qkv_lo";
    if (tc && d.rope) return "the wgmma engine takes planes that are already RoPE'd: rope must be 0";
    if (!tc && !d.qkv) return "the SIMT engine needs the fp32 qkv";
    return nullptr;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }
bool aligned8(const void* p) { return ((uintptr_t)p & 7) == 0; }

const char* test_row_desc_error(const st_test_row_desc& d) {
    const bool planes = d.out_hi || d.out_lo;
    if (d.u16 && d.kind != ST_TEST_ROW_ADALN) return "u16 belongs to ADALN";
    if (d.u16 && d.out_lo) return "u16 writes one fp16 plane to out_hi: out_lo must be NULL";
    if (!d.u16 && !d.out_hi != !d.out_lo) return "out_hi and out_lo go together";
    switch (d.kind) {
    case ST_TEST_ROW_ADALN:
        if (d.C != 256) return "ADALN: H (C) must be 256, the one width film_ln_mod_kernel is instantiated for";
        if (d.B < 1 || d.BB < 1 || d.T < 1) return "ADALN: B, BB, T >= 1";
        if (!d.x || !d.mask || !d.shift || !d.scale) return "ADALN: x, mask, shift and scale are required";
        if (d.has_film != 0 && d.has_film != 1) return "ADALN: has_film is 0 or 1";
        if (d.has_film && (!d.film || !d.xout)) return "ADALN: has_film needs film and xout";
        if (!d.has_film && (d.film || d.xout)) return "ADALN: film and xout belong to has_film";
        if (d.c_clamp < 0 || d.film_bstride < 0 || d.ada_bstride < 0) return "ADALN: c_clamp and batch strides must be >= 0";
        if (d.u16 && !d.out_hi) return "ADALN: u16 needs out_hi";
        if (!d.out_f32 && !d.out_hi) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.xout) || !aligned16(d.film) || !aligned16(d.shift) || !aligned16(d.scale) ||
            !aligned16(d.out_f32) || !aligned16(d.out_hi) || !aligned16(d.out_lo) || d.film_bstride % 4 || d.ada_bstride % 4)
            return "ADALN: buffers must be 16-byte aligned and batch strides multiples of 4";
        return nullptr;
    case ST_TEST_ROW_DWCONV_LN:
        if (d.C != 128 && d.C != 256 && d.C != 384 && d.C != 512 && d.C != 768 && d.C != 1024)
            return "DWCONV_LN: C must be 128, 256, 384, 512, 768 or 1024 (the instantiated widths)";
        if (d.B < 1 || d.T < 1) return "DWCONV_LN: B, T >= 1";
        if (!d.x || !d.ln_w || !d.ln_b || (d.w && !d.bias)) return "DWCONV_LN: x, ln_w, ln_b (and bias with w) are required";
        if (!(d.eps > 0.f)) return "DWCONV_LN: eps must be positive";
        if (!d.out_f32 && !planes) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.bias) || !aligned16(d.ln_w) || !aligned16(d.ln_b) || !aligned16(d.out_f32) ||
            !aligned16(d.out_hi) || !aligned16(d.out_lo))
            return "DWCONV_LN: buffers must be 16-byte aligned";
        return nullptr;
    case ST_TEST_ROW_SPECTRUM:
        if (d.B < 1 || d.T < 1) return "SPECTRUM: B, T >= 1";
        if (!d.x) return "SPECTRUM: x is required";
        if (d.K < 1 || d.Kp < d.K || d.Nh < d.Kp + d.K || d.K2 < 2 * d.K || d.K2 % 2)
            return "SPECTRUM: needs 1 <= K <= Kp, Kp + K <= Nh, K2 even and K <= K2/2";
        if (!d.out_f32 && !planes) return "no output requested";
        return nullptr;
    case ST_TEST_ROW_IDFT_BASIS:
        if (d.n_fft < 2 || d.n_fft % 2) return "IDFT_BASIS: n_fft must be even";
        if (d.K2 % 2 || d.K2 < 2 * (d.n_fft / 2 + 1)) return "IDFT_BASIS: K2 must be even, with n_fft/2 + 1 <= K2/2";
        if (!d.window) return "IDFT_BASIS: window is required";
        if (!d.out_f32 || planes) return "IDFT_BASIS: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_OVERLAP_ADD:
        if (const char* why = vocos_stft_error(d.n_fft, d.hop)) return why;
        if (d.B < 1 || d.T < 1) return "OVERLAP_ADD: B, T >= 1";
        if (!d.x || !d.window) return "OVERLAP_ADD: x (frames) and window are required";
        if (!d.out_f32 || planes) return "OVERLAP_ADD: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_MEAN3_SILU:
        if (d.n < 1 || d.n % 4) return "MEAN3_SILU: n must be a positive multiple of 4";
        if (!d.x || !d.x1 || !d.x2) return "MEAN3_SILU: x, x1 and x2 are required";
        if (!d.out_f32 && !planes) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.x1) || !aligned16(d.x2) || !aligned16(d.out_f32) || !aligned16(d.out_hi) || !aligned16(d.out_lo))
            return "MEAN3_SILU: buffers must be 16-byte aligned";
        return nullptr;
    case ST_TEST_ROW_POST_TANH:
        if (d.C != 16) return "POST_TANH: C must be 16, conv_post's one input width";
        if (d.B < 1 || d.T < 1) return "POST_TANH: B, T >= 1";
        if (!d.x || !d.w || !d.bias) return "POST_TANH: x, w and bias are required";
        if (!d.out_f32 || planes) return "POST_TANH: writes out_f32 only";
        if (!aligned16(d.x)) return "POST_TANH: x must be 16-byte aligned";
        return nullptr;
    case ST_TEST_ROW_GLU_RESID:
        if (d.C < 2 || d.C % 2) return "GLU_RESID: C must be even and positive";
        if (d.B < 1 || d.T < 1) return "GLU_RESID: B, T >= 1";
        if (!d.x || !d.x1) return "GLU_RESID: x ([a | g]) and x1 (the residual) are required";
        if (!d.out_f32 && !planes) return "no output requested";
        if (!aligned8(d.x) || !aligned8(d.x1) || !aligned8(d.out_f32) || !aligned8(d.out_hi) || !aligned8(d.out_lo))
            return "GLU_RESID: buffers must be 8-byte aligned";
        return nullptr;
    case ST_TEST_ROW_MASKED_MEAN:
        if (d.C < 1 || d.C > 128) return "MASKED_MEAN: C must be in [1, 128]";
        if (d.B < 1 || d.T < 1) return "MASKED_MEAN: B, T >= 1";
        if (!d.x) return "MASKED_MEAN: x is required";
        if (!d.out_f32 || planes) return "MASKED_MEAN: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_COND_TRANSPOSE:
        if (d.B < 1 || d.C < 1 || d.T < 1 || d.B > 65535) return "COND_TRANSPOSE: B, C, T >= 1 (B <= 65535)";
        if (!d.x || !d.bias || !d.mask) return "COND_TRANSPOSE: x, bias (cond) and mask are required";
        if (!d.out_f32 && !planes) return "no output requested";
        return nullptr;
    case ST_TEST_ROW_RELU_LN:
    case ST_TEST_ROW_RELU_LN_PROJ: {
        const bool proj = d.kind == ST_TEST_ROW_RELU_LN_PROJ;
        if (d.C != 1024) return "RELU_LN: C must be 1024, the one width relu_ln_kernel is instantiated for";
        if (d.B < 1 || d.T < 1) return "RELU_LN: B, T >= 1";
        if (!d.x || !d.ln_w || !d.ln_b || !d.mask) return "RELU_LN: x, ln_w, ln_b and mask are required";
        if (proj && (!d.w || !d.bias)) return "RELU_LN_PROJ: w (proj weight) and bias (proj bias) are required";
        if (proj && (!d.out_f32 || planes)) return "RELU_LN_PROJ: writes out_f32 (logw) only";
        if (!d.out_f32 && !planes) return "no output requested";
        if (!aligned16(d.x) || !aligned16(d.ln_w) || !aligned16(d.ln_b) || (proj && !aligned16(d.w)) ||
            (!proj && (!aligned16(d.out_f32) || !aligned16(d.out_hi) || !aligned16(d.out_lo))))
            return "RELU_LN: buffers must be 16-byte aligned";
        return nullptr;
    }
    case ST_TEST_ROW_GEMV:
        if (d.B < 1 || d.K < 1 || d.N < 1 || (long)d.B * d.N > (1L << 26)) return "GEMV: B, K, N >= 1 and B N <= 2^26";
        if (d.y_rstride < d.N) return "GEMV: y_rstride must be >= N";
        if ((d.silu_in != 0 && d.silu_in != 1) || (d.silu_out != 0 && d.silu_out != 1)) return "GEMV: silu_in and silu_out are 0 or 1";
        if (!d.x || !d.w) return "GEMV: x and w are required";
        if (!d.out_f32 || planes) return "GEMV: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_TIME_EMBED:
    case ST_TEST_ROW_TIME_EMBED_VALS:
        if (d.C < 4 || d.C % 2) return "TIME_EMBED: C must be even and >= 4";
        if (d.kind == ST_TEST_ROW_TIME_EMBED && (d.n_t < 1 || (long)d.n_t * d.C > (1L << 30)))
            return "TIME_EMBED: n_t >= 1 (n_t C <= 2^30)";
        if (d.kind == ST_TEST_ROW_TIME_EMBED ? !d.x : !d.t_host) return "TIME_EMBED: x (device) or t_host (TIME_EMBED_VALS) is required";
        if (!d.out_f32 || planes) return "TIME_EMBED: writes out_f32 only";
        return nullptr;               // TIME_EMBED_VALS: launch_time_embed_vals itself refuses n_t outside [1, 256]
    case ST_TEST_ROW_ROPE_TABLE:
        if (d.C != 32) return "ROPE_TABLE: C must be 32, the rotary width";
        if (d.T < 1 || d.T > (1 << 24)) return "ROPE_TABLE: T in [1, 2^24]";
        if (!d.out_f32 || planes) return "ROPE_TABLE: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_LINCOMB:
    case ST_TEST_ROW_SCALED_SUMSQ: {
        const bool norm = d.kind == ST_TEST_ROW_SCALED_SUMSQ;
        if (norm ? (d.n_terms < 1 || d.n_terms > 7) : (d.n_terms < 0 || d.n_terms > 6))
            return "LINCOMB: n_terms in [0, 6]; SCALED_SUMSQ: n_terms in [1, 7]";
        if (d.n < 1) return "LINCOMB / SCALED_SUMSQ: n >= 1";
        for (int j = 0; j < d.n_terms; ++j)
            if (!d.terms[j]) return "LINCOMB / SCALED_SUMSQ: terms[0 .. n_terms) are required";
        if (!d.x || (norm && !d.x1)) return "LINCOMB: x (y) is required; SCALED_SUMSQ: x (u) and x1 (v) are required";
        if (norm && !(d.atol > 0.f && d.rtol >= 0.f)) return "SCALED_SUMSQ: atol > 0 and rtol >= 0";
        if (norm ? (!d.out_f64 || d.out_f32 || planes) : (!d.out_f32 || planes))
            return "LINCOMB writes out_f32 only, SCALED_SUMSQ out_f64 only";
        return nullptr;
    }
    case ST_TEST_ROW_CFG_COMBINE:
        if (d.B < 1 || d.n < 1) return "CFG_COMBINE: B, n >= 1";
        if (d.cfg != 0 && d.cfg != 1) return "CFG_COMBINE: cfg is 0 or 1";
        if (!d.x) return "CFG_COMBINE: x (V) is required";
        if (!d.out_f32 || planes) return "CFG_COMBINE: writes out_f32 only";
        return nullptr;
    case ST_TEST_ROW_CFM_MIX:
    case ST_TEST_ROW_CFM_LOSS: {
        const bool loss = d.kind == ST_TEST_ROW_CFM_LOSS;
        if (d.B < 1 || d.C < 1 || d.T < 1) return "CFM_MIX / CFM_LOSS: B, C, T >= 1";
        if (!d.x || !d.x1 || !d.x2 || (loss && !d.mask)) return "CFM_MIX: x, x1 and x2 are required (CFM_LOSS: and mask)";
        if (loss ? (!d.out_f32 || !d.out_f64 || planes) : (!d.out_f32 || planes || d.out_f64))
            return "CFM_MIX writes out_f32 only, CFM_LOSS out_f32 and out_f64";
        return nullptr;
    }
    default:
        return "unknown kind";
    }
}

const char* test_pack_desc_error(const st_test_pack_desc& d) {
    const bool planes = d.out_hi || d.out_lo;
    if (!d.out_hi != !d.out_lo) return "out_hi and out_lo go together";
    const bool pow2_fft = d.n_fft >= 32 && d.n_fft <= 4096 && !(d.n_fft & (d.n_fft - 1));
    switch (d.kind) {
    case ST_TEST_PACK_BCT_TO_BTC:
        if (d.B < 0 || d.B > 65534 || d.C < 1 || d.T < 1) return "BCT_TO_BTC: 0 <= B < 65535, C, T >= 1";
        if (d.B > 0 && !d.x) return "BCT_TO_BTC: x is required when B > 0";
        if (!d.out_f32 && !planes) return "no output requested";
        return nullptr;
    case ST_TEST_PACK_BTC_TO_BCT:
        if (d.B < 1 || d.B > 65535 || d.C < 1 || d.T < 1) return "BTC_TO_BCT: B in [1, 65535], C, T >= 1";
        if (!d.x) return "BTC_TO_BCT: x is required";
        if (!d.out_f32 || planes) return "BTC_TO_BCT: writes out_f32 only";
        return nullptr;
    case ST_TEST_PACK_EMBED:
        if (d.B < 1 || d.T < 1 || d.C < 1 || d.n_vocab < 1 || (long)d.B * d.T > INT32_MAX) return "EMBED: B, T, C, n_vocab >= 1";
        if (!d.ids || !d.lens || !d.x) return "EMBED: ids, lens and x (emb) are required";
        if (!d.out_f32 || !d.out2_f32 || planes) return "EMBED: writes out_f32 (x) and out2_f32 (mask)";
        return nullptr;
    case ST_TEST_PACK_SPLIT_BF16:
    case ST_TEST_PACK_SPLIT_F16:
        if (d.n < 0 || d.n > (1L << 40)) return "SPLIT: n >= 0";
        if (!d.x) return "SPLIT: x is required";
        if (!planes || d.out_f32) return "SPLIT: writes out_hi and out_lo";
        if (d.out_i32 && d.kind != ST_TEST_PACK_SPLIT_F16) return "out_i32 (the range flag) belongs to SPLIT_F16";
        return nullptr;
    case ST_TEST_PACK_PACK_CONV:
        if (d.Nsrc < 1 || d.Csrc < 1 || d.k < 1 || d.Cc < 1 || d.n_off < 0 || d.c_off < 0) return "PACK_CONV: Nsrc, Csrc, k, Cc >= 1, offsets >= 0";
        if ((long)d.n_off + d.Nsrc > d.Ntot) return "PACK_CONV: n_off + Nsrc must be <= Ntot";
        if ((long)d.c_off + d.Cc > d.Csrc) return "PACK_CONV: c_off + Cc must be <= Csrc";
        if (!d.x) return "PACK_CONV: x is required";
        if (!d.out_f32 || planes) return "PACK_CONV: writes out_f32 only";
        return nullptr;
    case ST_TEST_PACK_WEIGHT_NORM:
        if (d.rows < 1 || d.len < 1) return "WEIGHT_NORM: rows, len >= 1";
        if (!d.g || !d.x) return "WEIGHT_NORM: g and x (v) are required";
        if (!d.out_f32 || planes) return "WEIGHT_NORM: writes out_f32 only";
        return nullptr;
    case ST_TEST_PACK_POLYPHASE:
        if (d.u < 2 || d.u % 2) return "POLYPHASE: u must be even and >= 2";
        if (d.Cin < 1 || d.Cout < 1 || 3L * d.u * d.Cout * d.Cin > (1L << 40)) return "POLYPHASE: Cin, Cout >= 1";
        if (!d.x) return "POLYPHASE: x (w) is required";
        if (!d.out_f32 || planes) return "POLYPHASE: writes out_f32 only";
        return nullptr;
    case ST_TEST_PACK_MEL_TWIDDLES:
        if (!pow2_fft) return "MEL_TWIDDLES: n_fft must be a power of two in [32, 4096]";
        if (!d.out_f32 || planes) return "MEL_TWIDDLES: writes out_f32 only";
        return nullptr;
    case ST_TEST_PACK_MEL_PACK_FB:
        if (!pow2_fft) return "MEL_PACK_FB: n_fft must be a power of two in [32, 4096]";
        if (d.n_mels < 1 || d.n_mels > 4096) return "MEL_PACK_FB: n_mels in [1, 4096]";
        if (!d.x) return "MEL_PACK_FB: x (fb) is required";
        if (!d.out_f32 || !d.out_i32 || planes) return "MEL_PACK_FB: writes out_f32 (fbT) and out_i32 (band) [, out2_i32 (kband)]";
        return nullptr;
    default:
        return "unknown kind";
    }
}

}  // namespace

extern "C" {

__global__ void fill_pattern_kernel(float* p, long n, uint32_t seed) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u + seed;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    p[i] = ((float)(x & 0xFFFF) / 32768.0f - 1.0f);
}

int st_test_gemm_ex(st_handle* h, const st_test_gemm_desc* dp, st_test_gemm_plan* plan, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_gemm_ex: null descriptor");
    const st_test_gemm_desc& d = *dp;
    if (const char* why = test_gemm_desc_error(d)) return fail(h, std::string("st_test_gemm_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const int Cs[2] = {d.C0, d.C1}, Ktot = d.C0 + d.C1;
    const size_t nw = (size_t)d.taps * d.N * Ktot;
    TestBufs bufs;
    // W: (N, Ktot, taps) Conv1d layout -> packed [taps][N][Ktot], then its planes
    GemmW w; w.taps = d.taps; w.N = d.N; w.K = Ktot; w.bias = const_cast<float*>(d.bias);
    w.f32 = bufs.take<float>(nw); w.hi = bufs.take<bf16>(nw); w.lo = bufs.take<bf16>(nw);
    if (d.prec) { w.h_hi = bufs.take<bf16>(nw); w.h_lo = bufs.take<bf16>(nw); }
    if (!bufs.ok) return fail(h, "st_test_gemm_ex: out of memory");
    ST_CUDA(launch_pack_conv(d.W, w.f32, d.N, Ktot, d.taps, d.N, 0, 0, Ktot, s));
    ST_CUDA(launch_split(w.f32, w.hi, w.lo, (long)nw, s));
    if (d.prec) ST_CUDA(launch_split_f16(w.f32, w.h_hi, w.h_lo, (long)nw, s));
    // A: fp32 for the SIMT engine; split-bf16 planes, or with prec ONE fp16 plane (the hi plane of the fp16 split)
    Act a[2];
    for (int i = 0; i < d.n_src; ++i) {
        const float* src = i ? d.A1 : d.A0;
        const size_t n = (size_t)d.a_bmod * d.T * Cs[i];
        a[i].C = Cs[i]; a[i].f32 = const_cast<float*>(src);
        if (!tc) continue;
        a[i].hi = bufs.take<bf16>(n); a[i].lo = bufs.take<bf16>(n);
        if (!bufs.ok) return fail(h, "st_test_gemm_ex: out of memory");
        ST_CUDA(d.prec ? launch_split_f16(src, a[i].hi, a[i].lo, (long)n, s) : launch_split(src, a[i].hi, a[i].lo, (long)n, s));
    }
    GemmArgs g;
    g.BB = d.BB; g.T = d.T; g.a_bmod = d.a_bmod; g.B = d.B; g.flags = d.flags; g.dil = d.dil;
    g.mask = d.mask; g.film = d.film; g.film_bstride = d.film_bstride; g.film_H = d.film_H;
    g.gate = d.gate; g.gate_bstride = d.gate_bstride; g.c_clamp = d.c_clamp; g.resid = d.resid; g.resid_clamp = d.resid_clamp;
    g.rope_H = d.rope_H;
    if (d.flags & EPI_ROPE) {
        float* cs = bufs.take<float>((size_t)d.T * 32);
        if (!bufs.ok) return fail(h, "st_test_gemm_ex: out of memory");
        ST_CUDA(launch_rope_table(cs, d.T, 32, s));
        g.rope_cs = cs;
    }
    g.ln = d.ln; g.ln_mask_out = d.ln_mask_out; g.ln_shift = d.ln_shift; g.ln_scale = d.ln_scale; g.ada_bstride = d.ada_bstride;
    g.u_hi = (bf16*)d.u_hi; g.u_lo = (bf16*)d.u_lo; g.film2 = d.film2; g.film2_bstride = d.film2_bstride; g.out2_f32 = d.out2_f32;
    g.prec = d.prec; g.out16 = d.out16; g.u16 = d.u16;
    g.force_ksplit = d.ksplit;
    GemmPlan gp;
    g.plan = &gp;
    Act o; o.C = d.N; o.f32 = d.out_f32; o.hi = (bf16*)d.out_hi; o.lo = (bf16*)d.out_lo;
    // the split-K partial buffer is sized by the real SM count, before any override; a handle serves one caller at a time
    // (as every entry point assumes), so the override only has to be undone on every exit
    if (tc && ensure_part_buf(h)) return 1;
    struct SmsRestore {
        st_handle* h; int saved;
        ~SmsRestore() { h->num_sms = saved; }
    } restore{h, h->num_sms};
    if (d.num_sms > 0) h->num_sms = d.num_sms;
    if (run_gemm(h, g, w, &a[0], d.n_src == 2 ? &a[1] : nullptr, o, s) || hook_done(h, s, "st_test_gemm_ex")) return 1;
    if (plan) {
        plan->engine = gp.engine; plan->bn = gp.bn; plan->mode = gp.mode; plan->prec = gp.prec; plan->ksplit = gp.ksplit; plan->grid = gp.grid;
    }
    return 0;
}

int st_test_attention_ex(st_handle* h, const st_test_attn_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_attention_ex: null descriptor");
    const st_test_attn_desc& d = *dp;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    if (const char* why = test_attn_desc_error(d, tc)) return fail(h, std::string("st_test_attention_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    TestBufs bufs;
    int* kvlen = d.kvlen_out ? d.kvlen_out : bufs.take<int>(d.B);
    int* prefix = d.prefix_out ? d.prefix_out : bufs.take<int>(d.B);
    float* cs = d.rope ? bufs.take<float>((size_t)d.T * 32) : nullptr;
    if (!bufs.ok) return fail(h, "st_test_attention_ex: out of memory");
    ST_CUDA(launch_mask_lengths(d.mask, kvlen, prefix, d.B, d.T, s));
    if (d.rope) ST_CUDA(launch_rope_table(cs, d.T, 32, s));
    AttnArgs a;
    a.qkv = d.qkv; a.qkv_hi = (const bf16*)d.qkv_hi; a.qkv_lo = (const bf16*)d.qkv_lo; a.rope_cs = cs;
    a.mask = d.mask; a.kvlen = kvlen; a.prefix = prefix;
    a.out_f32 = d.out_f32; a.out_hi = (bf16*)d.out_hi; a.out_lo = (bf16*)d.out_lo;
    a.BB = d.BB; a.B = d.B; a.T = d.T; a.H = d.H; a.n_heads = d.n_heads;
    cudaError_t e = tc ? launch_attention_tc(a, s) : launch_attention_simt(a, s);
    if (e != cudaSuccess)
        return fail(h, std::string("st_test_attention_ex: launch failed: ") + cudaGetErrorString(e) + (tc ? std::string(" / ") + attention_tc_last_error() : ""));
    return hook_done(h, s, "st_test_attention_ex");
}

int st_test_row_ex(st_handle* h, const st_test_row_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_row_ex: null descriptor");
    const st_test_row_desc& d = *dp;
    if (const char* why = test_row_desc_error(d)) return fail(h, std::string("st_test_row_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    bf16* hi = (bf16*)d.out_hi; bf16* lo = (bf16*)d.out_lo;
    TestBufs bufs;
    cudaError_t e = cudaSuccess;
    switch (d.kind) {
    case ST_TEST_ROW_ADALN: {
        LnArgs a;
        a.xin = d.x; a.xout = d.xout; a.film = d.film; a.film_bstride = d.film_bstride;
        a.shift = d.shift; a.scale = d.scale; a.ada_bstride = d.ada_bstride; a.c_clamp = d.c_clamp;
        a.mask = d.mask; a.B = d.B; a.has_film = d.has_film; a.mask_out = d.mask_out;
        a.u_f32 = d.out_f32; a.u_hi = hi; a.u_lo = lo; a.u16 = d.u16;
        a.BB = d.BB; a.T = d.T; a.H = d.C;
        e = launch_film_ln_mod(a, s);
        break;
    }
    case ST_TEST_ROW_DWCONV_LN: {
        DwLnArgs a;
        a.B = d.B; a.T = d.T; a.C = d.C; a.eps = d.eps;
        a.x = d.x; a.dw_b = d.bias; a.ln_w = d.ln_w; a.ln_b = d.ln_b;
        a.out_f32 = d.out_f32; a.out_hi = hi; a.out_lo = lo;
        if (d.w) {                     // (C, 1, 7) -> [7][C], as pack_dw7 packs it
            float* packed = bufs.take<float>((size_t)7 * d.C);
            if (!bufs.ok) return fail(h, "st_test_row_ex: out of memory");
            ST_CUDA(launch_pack_conv(d.w, packed, d.C, 1, 7, d.C, 0, 0, 1, s));
            a.dw_w = packed;
        }
        e = launch_dwconv_ln(a, s);
        break;
    }
    case ST_TEST_ROW_SPECTRUM:
        e = launch_spectrum(d.x, d.Nh, d.Kp, d.K, d.K2, (long)d.B * d.T, d.out_f32, hi, lo, s);
        break;
    case ST_TEST_ROW_IDFT_BASIS:
        e = launch_idft_basis(d.window, d.n_fft, d.n_fft / 2 + 1, d.K2, d.out_f32, s);
        break;
    case ST_TEST_ROW_OVERLAP_ADD:
        e = launch_overlap_add(d.x, d.window, d.B, d.T, d.n_fft, d.hop, d.out_f32, s);
        break;
    case ST_TEST_ROW_MEAN3_SILU:
        e = launch_mean3_silu(d.x, d.x1, d.x2, (long)d.n, d.out_f32, hi, lo, s);
        break;
    case ST_TEST_ROW_POST_TANH:
        e = launch_post_conv_tanh(d.x, d.w, d.bias, d.B, (long)d.T, d.C, 13, d.out_f32, s);
        break;
    case ST_TEST_ROW_GLU_RESID:
        e = launch_glu_residual(d.x, d.x1, d.out_f32, hi, lo, (long)d.B * d.T, d.C, s);
        break;
    case ST_TEST_ROW_MASKED_MEAN:
        e = launch_masked_mean(d.x, d.mask, d.out_f32, d.B, d.T, d.C, s);
        break;
    case ST_TEST_ROW_COND_TRANSPOSE:
        e = launch_cond_mask_transpose(d.x, d.bias, d.mask, d.out_f32, hi, lo, d.B, d.C, d.T, s);
        break;
    case ST_TEST_ROW_RELU_LN:
        e = launch_relu_ln(d.x, d.ln_w, d.ln_b, d.mask, (long)d.B * d.T, d.C, d.out_f32, hi, lo, nullptr, nullptr, nullptr, s);
        break;
    case ST_TEST_ROW_RELU_LN_PROJ:
        e = launch_relu_ln(d.x, d.ln_w, d.ln_b, d.mask, (long)d.B * d.T, d.C, nullptr, nullptr, nullptr, d.w, d.bias, d.out_f32, s);
        break;
    case ST_TEST_ROW_GEMV:
        e = launch_gemv(d.x, d.w, d.bias, d.out_f32, (long)d.y_rstride, d.B, d.K, d.N, d.silu_in, d.silu_out, s);
        break;
    case ST_TEST_ROW_TIME_EMBED:
        e = launch_time_embed(d.x, d.n_t, d.C, d.out_f32, s);
        break;
    case ST_TEST_ROW_TIME_EMBED_VALS:
        e = launch_time_embed_vals(d.t_host, d.n_t, d.C, d.out_f32, s);
        break;
    case ST_TEST_ROW_ROPE_TABLE:
        e = launch_rope_table(d.out_f32, d.T, d.C, s);
        break;
    case ST_TEST_ROW_LINCOMB:
        e = launch_lincomb(d.out_f32, d.x, d.terms, d.coef, d.n_terms, (long)d.n, s);
        break;
    case ST_TEST_ROW_SCALED_SUMSQ:
        e = launch_scaled_sumsq(d.terms, d.coef, d.n_terms, d.x, d.x1, d.atol, d.rtol, (long)d.n, d.out_f64, s);
        break;
    case ST_TEST_ROW_CFG_COMBINE:
        e = launch_cfg_combine(d.x, d.out_f32, d.B, (long)d.n, d.cfg, d.s_cfg, s);
        break;
    case ST_TEST_ROW_CFM_MIX:
        e = launch_cfm_mix(d.x, d.x1, d.x2, d.sigma_min, d.B, (long)d.C * d.T, d.out_f32, s);
        break;
    case ST_TEST_ROW_CFM_LOSS:
        e = launch_cfm_loss(d.x2, d.x, d.x1, d.mask, d.sigma_min, d.B, d.C, d.T, d.out_f64, d.out_f32, s);
        break;
    }
    if (e != cudaSuccess) return fail(h, std::string("st_test_row_ex: launch failed: ") + cudaGetErrorString(e));
    return hook_done(h, s, "st_test_row_ex");
}

int st_test_pack_ex(st_handle* h, const st_test_pack_desc* dp, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (!dp) return fail(h, "st_test_pack_ex: null descriptor");
    const st_test_pack_desc& d = *dp;
    if (const char* why = test_pack_desc_error(d)) return fail(h, std::string("st_test_pack_ex: ") + why);
    cudaStream_t s = (cudaStream_t)stream;
    bf16* hi = (bf16*)d.out_hi; bf16* lo = (bf16*)d.out_lo;
    cudaError_t e = cudaSuccess;
    switch (d.kind) {
    case ST_TEST_PACK_BCT_TO_BTC:
        e = launch_bct_to_btc(d.x, d.out_f32, hi, lo, d.B, d.C, d.T, d.bcast, s);
        break;
    case ST_TEST_PACK_BTC_TO_BCT:
        e = launch_btc_to_bct(d.x, d.out_f32, d.B, d.C, d.T, s);
        break;
    case ST_TEST_PACK_EMBED:
        e = launch_embed(d.ids, d.lens, d.x, d.n_vocab, d.B, d.T, d.C, d.scale, d.out_f32, d.out2_f32, s);
        break;
    case ST_TEST_PACK_SPLIT_BF16:
        e = launch_split(d.x, hi, lo, (long)d.n, s);
        break;
    case ST_TEST_PACK_SPLIT_F16:
        if (d.out_i32) ST_CUDA(cudaMemsetAsync(d.out_i32, 0, sizeof(int32_t), s));
        e = launch_split_f16(d.x, hi, lo, (long)d.n, s, d.out_i32);
        break;
    case ST_TEST_PACK_PACK_CONV:
        e = launch_pack_conv(d.x, d.out_f32, d.Nsrc, d.Csrc, d.k, d.Ntot, d.n_off, d.c_off, d.Cc, s);
        break;
    case ST_TEST_PACK_WEIGHT_NORM:
        e = launch_weight_norm_fold(d.g, d.x, d.out_f32, d.rows, d.len, s);
        break;
    case ST_TEST_PACK_POLYPHASE:
        e = launch_pack_polyphase(d.x, d.out_f32, d.Cin, d.Cout, d.u, s);
        break;
    case ST_TEST_PACK_MEL_TWIDDLES:
        e = launch_mel_twiddles(d.n_fft, reinterpret_cast<float2*>(d.out_f32), s);
        break;
    case ST_TEST_PACK_MEL_PACK_FB:
        e = launch_mel_pack_fb(d.x, d.n_fft / 2 + 1, d.n_mels, d.out_f32, reinterpret_cast<int2*>(d.out_i32),
                               reinterpret_cast<int2*>(d.out2_i32), s);
        break;
    }
    if (e != cudaSuccess) return fail(h, std::string("st_test_pack_ex: launch failed: ") + cudaGetErrorString(e));
    return hook_done(h, s, "st_test_pack_ex");
}

// Times `reps` launches of the selected engine's conv-GEMM on synthetic data (token-major operands are
// generated on the device): (B, T, Cin) x [k][Cout][Cin] -> (B, T, Cout).  epi 1: conv_2-style epilogue (bias, mask, gate,
// residual, fp32 + split outputs); 2: conv_1-style (bias, SiLU, mask, split output); 3: O-style (residual, mask, gate,
// fp32 output + fused LayerNorm / modulate); 0: bias-only split output.  prec = 1: the two-pass fp16 operands (one fp16 A
// plane, fp16 hi / lo weights) with fp16 output planes, as ST_PRECISION_FFN_FP16X2 runs the FFN convs.
int st_bench_conv(st_handle* h, int B, int Cin, int Cout, int T, int k, int epi, int prec, int reps, float* ms_out) {
    if (!h || !ms_out) return 1;
    ST_ENTER(h);
    cudaStream_t s = 0;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    if (prec && !tc) return fail(h, "st_bench_conv: the two-pass fp16 precision runs on the wgmma engine only");
    const size_t nx = (size_t)B * T * Cin, nw = (size_t)k * Cout * Cin, no = (size_t)B * T * Cout;
    TestBufs bufs;
    float *xf = bufs.take<float>(nx), *wf = bufs.take<float>(nw), *of = bufs.take<float>(no);
    bf16 *xh = bufs.take<bf16>(nx), *xl = bufs.take<bf16>(nx), *wh = bufs.take<bf16>(nw), *wl = bufs.take<bf16>(nw);
    bf16 *oh = bufs.take<bf16>(no), *ol = bufs.take<bf16>(no);
    float *bias = bufs.take<float>(Cout), *gate = bufs.take<float>((size_t)B * Cout), *mask = bufs.take<float>((size_t)B * T);
    if (!bufs.ok) return fail(h, "st_bench_conv: out of memory");
    fill_pattern_kernel<<<(unsigned)((nx + 255) / 256), 256, 0, s>>>(xf, (long)nx, 1u);
    fill_pattern_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(wf, (long)nw, 2u);
    fill_pattern_kernel<<<(unsigned)((no + 255) / 256), 256, 0, s>>>(of, (long)no, 3u);
    fill_pattern_kernel<<<(Cout + 255) / 256, 256, 0, s>>>(bias, Cout, 4u);
    fill_pattern_kernel<<<(unsigned)(((size_t)B * Cout + 255) / 256), 256, 0, s>>>(gate, (long)B * Cout, 5u);
    ST_CUDA(cudaMemsetAsync(mask, 0x3f, (size_t)B * T * 4, s));       // 0.747 everywhere: a non-trivial multiplier
    // prec: one fp16 A plane (xh) and fp16 hi / lo weight planes, 2-byte outputs as one fp16 plane (the FFN convs' mode)
    auto split = [&](const float* in, bf16* hi, bf16* lo, long n) {
        return prec ? launch_split_f16(in, hi, lo, n, s) : launch_split(in, hi, lo, n, s);
    };
    ST_CUDA(split(xf, xh, xl, (long)nx));
    ST_CUDA(split(wf, wh, wl, (long)nw));
    GemmArgs g = utt_gemm(B, T, (epi == 1 || epi == 3) ? (EPI_BIAS | EPI_MASK | EPI_GATE | EPI_RESID)
                                                       : (epi == 2 ? (EPI_BIAS | EPI_SILU | EPI_MASK) : EPI_BIAS));
    g.c_clamp = B - 1; g.mask = mask; g.gate = gate; g.gate_bstride = Cout; g.resid = of;
    if (epi == 3) {                    // O-style: fp32 residual stream out + fused LayerNorm/modulate -> split-bf16 U
        g.ln = 1; g.ln_mask_out = 1; g.ln_shift = gate; g.ln_scale = gate; g.ada_bstride = Cout; g.u_hi = oh; g.u_lo = ol;
    }
    GemmW w; w.f32 = wf; w.hi = wh; w.lo = wl; w.bias = bias; w.taps = k; w.N = Cout; w.K = Cin;
    if (prec) { g.prec = 1; g.out16 = 1; g.u16 = 1; w.h_hi = wh; w.h_lo = wl; }
    Act a; a.C = Cin; a.f32 = xf; a.hi = tc ? xh : nullptr; a.lo = tc ? xl : nullptr;
    Act o; o.C = Cout; o.f32 = (epi == 1 || epi == 3) ? of : nullptr; o.hi = epi == 3 ? nullptr : oh; o.lo = epi == 3 ? nullptr : ol;
    for (int i = 0; i < 2; ++i)
        if (run_gemm(h, g, w, &a, nullptr, o, s)) return 1;
    int rc = 0;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0, s);
    for (int i = 0; i < reps && !rc; ++i) rc = run_gemm(h, g, w, &a, nullptr, o, s);
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1);
    *ms_out = ms / (reps > 0 ? reps : 1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return rc ? rc : hook_done(h, s, "st_bench_conv");
}

// dilated / transposed conv through the conv-GEMM
int st_test_conv_ex(st_handle* h, const float* x, const float* wgt, const float* bias, float* out, int B, int Cin, int Cout,
                    int T, int k, int dil, int transposed, void* stream) {
    if (!h) return 1;
    ST_ENTER(h);
    if (B <= 0 || T <= 0 || Cin <= 0 || Cout <= 0 || dil < 1 || (transposed ? (k != 2 * dil || dil % 2) : (k % 2 == 0)))
        return fail(h, "st_test_conv_ex: bad shape (odd k for a conv; k = 2u, even u for a transposed conv)");
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = h->engine == ST_ENGINE_TCGEN05;
    const int u = transposed ? dil : 1, taps = transposed ? 3 : k, N = u * Cout;
    const size_t nx = (size_t)B * T * Cin, nw = (size_t)taps * N * Cin, no = (size_t)B * T * N;
    TestBufs bufs;
    float *xt = bufs.take<float>(nx), *wp = bufs.take<float>(nw), *ot = bufs.take<float>(no), *bt = bufs.take<float>(N);
    bf16 *xh = bufs.take<bf16>(nx), *xl = bufs.take<bf16>(nx), *wh = bufs.take<bf16>(nw), *wl = bufs.take<bf16>(nw);
    if (!bufs.ok) return fail(h, "st_test_conv_ex: out of memory");
    ST_CUDA(launch_bct_to_btc(x, xt, xh, xl, B, Cin, T, nullptr, s));
    ST_CUDA(transposed ? launch_pack_polyphase(wgt, wp, Cin, Cout, u, s) : launch_pack_conv(wgt, wp, Cout, Cin, k, Cout, 0, 0, Cin, s));
    ST_CUDA(launch_split(wp, wh, wl, (long)nw, s));
    if (bias)
        for (int r = 0; r < u; ++r) ST_CUDA(cudaMemcpyAsync(bt + (size_t)r * Cout, bias, (size_t)Cout * 4, cudaMemcpyDeviceToDevice, s));
    GemmArgs g = utt_gemm(B, T, bias ? EPI_BIAS : 0);
    g.dil = transposed ? 1 : dil;
    GemmW w; w.f32 = wp; w.hi = wh; w.lo = wl; w.bias = bias ? bt : nullptr; w.taps = taps; w.N = N; w.K = Cin;
    Act a; a.C = Cin; a.f32 = xt; a.hi = tc ? xh : nullptr; a.lo = tc ? xl : nullptr;
    Act o; o.C = N; o.f32 = ot;
    if (run_gemm(h, g, w, &a, nullptr, o, s)) return 1;
    // (B, T, u Cout) == (B, u T, Cout) token-major -> (B, Cout, u T)
    ST_CUDA(launch_btc_to_bct(ot, out, B, Cout, u * T, s));
    return hook_done(h, s, "st_test_conv_ex");
}

}  // extern "C"
