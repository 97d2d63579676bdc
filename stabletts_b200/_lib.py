"""ctypes binding of libstabletts_b200.so (C ABI: include/stabletts_b200.h)."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

ST_EULER, ST_MIDPOINT, ST_RK4, ST_DOPRI5_FIXED = 0, 1, 2, 3
ST_ENGINE_TCGEN05, ST_ENGINE_SIMT = 0, 1
ST_PRECISION_BF16X3, ST_PRECISION_FFN_FP16X2 = 0, 1
ST_ADAPT_DOPRI5, ST_ADAPT_BOSH3, ST_ADAPT_FEHLBERG2, ST_ADAPT_HEUN = 0, 1, 2, 3
ST_PROF_NAMES = ("gemm_other", "attention", "ln", "gemm_qkv", "gemm_o", "gemm_conv1", "gemm_conv2", "gemm_lsc", "gemm_cond",
                 "ffgan_backbone", "ffgan_conv_pre", "ffgan_stage0", "ffgan_stage1", "ffgan_stage2", "ffgan_stage3", "ffgan_stage4",
                 "ffgan_post")
ST_PROF_NCAT = len(ST_PROF_NAMES)
ST_RESAMPLE_MAX_TABLE = 1 << 18      # include/stabletts_b200.h: coefficients of a resampler's table, at most

# every symbol include/stabletts_b200.h declares (tests check the .so exports all of them)
EXPORTS = [
    "st_create", "st_destroy", "st_last_error", "st_version", "st_load_weight", "st_finalize_weights",
    "st_set_engine", "st_set_precision", "st_workspace_bytes", "st_attach_workspace", "st_estimator_forward", "st_cfm_loss", "st_solve",
    "st_solve_host", "st_solve_host_io", "st_solve_adaptive", "st_solve_adaptive_ex", "st_align_lengths", "st_align_expand", "st_mas_workspace_bytes", "st_mas_scores", "st_maximum_path", "st_mas_losses", "st_create_text_encoder", "st_text_encoder_forward", "st_create_vocos", "st_vocos_forward", "st_create_ffgan", "st_ffgan_forward", "st_ffgan_workspace_bytes", "st_create_style_encoder", "st_style_encoder_forward", "st_create_duration_predictor", "st_duration_predictor_forward", "st_create_mel", "st_mel_forward", "st_create_mel_loss", "st_mel_loss_workspace_bytes", "st_mel_loss_forward", "st_create_mpd", "st_mpd_workspace_bytes", "st_mpd_forward", "st_mpd_backward", "st_create_resample", "st_resample_out_length", "st_resample_forward", "st_launch_count", "st_profile_begin", "st_profile_end", "st_profile_issued", "st_test_gemm_ex", "st_test_conv_ex", "st_test_attention_ex", "st_test_row_ex", "st_test_mpd_conv", "st_bench_conv",
]


class StDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_mel", "hidden", "filter", "n_heads", "n_layers", "kernel", "gin")]


class StVocosDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_mel", "dim", "intermediate", "n_layers", "n_fft", "hop")]


class StMelDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_fft", "hop_length", "pad", "n_mels")]


ST_TEST_EPI_BIAS, ST_TEST_EPI_SILU, ST_TEST_EPI_FILM, ST_TEST_EPI_MASK, ST_TEST_EPI_GATE = 1, 2, 4, 8, 16
ST_TEST_EPI_RESID, ST_TEST_EPI_ROPE, ST_TEST_EPI_GELU, ST_TEST_EPI_SILU_OUT, ST_TEST_EPI_MISH = 32, 64, 128, 256, 512
ST_TEST_MODE_NAMES = ("PLAIN", "SILU", "GELU", "ROPE", "LN", "RESID", "SILU_OUT", "MISH")     # st_test_gemm_plan.mode


class StTestGemmDesc(C.Structure):
    """st_test_gemm_desc: one conv-GEMM problem of st_test_gemm_ex (device pointers as integers, 0 = absent)."""
    _fields_ = ([(n, C.c_void_p) for n in ("A0", "A1", "W", "bias", "mask", "film", "gate", "resid", "ln_shift", "ln_scale",
                                          "film2", "out_f32", "out_hi", "out_lo", "out2_f32", "u_hi", "u_lo")]
                + [(n, C.c_int64) for n in ("film_bstride", "gate_bstride", "ada_bstride", "film2_bstride")]
                + [(n, C.c_int32) for n in ("B", "BB", "T", "a_bmod", "n_src", "C0", "C1", "N", "taps", "dil", "flags", "c_clamp",
                                            "resid_clamp", "film_H", "rope_H", "ln", "ln_mask_out", "prec", "out16", "u16",
                                            "ksplit", "num_sms")])


class StTestGemmPlan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("engine", "bn", "mode", "prec", "ksplit", "grid")]


class StTestAttnDesc(C.Structure):
    """st_test_attn_desc: one attention problem of st_test_attention_ex (device pointers as integers, 0 = absent)."""
    _fields_ = ([(n, C.c_void_p) for n in ("qkv", "qkv_hi", "qkv_lo", "mask", "out_f32", "out_hi", "out_lo", "kvlen_out",
                                          "prefix_out")]
                + [(n, C.c_int32) for n in ("BB", "B", "T", "H", "n_heads", "rope")])


ST_TEST_ROW_KINDS = ("ADALN", "DWCONV_LN", "SPECTRUM", "IDFT_BASIS", "OVERLAP_ADD", "MEAN3_SILU", "POST_TANH")  # st_test_row_desc.kind


class StTestRowDesc(C.Structure):
    """st_test_row_desc: one row-kernel problem of st_test_row_ex (device pointers as integers, 0 = absent)."""
    _fields_ = ([(n, C.c_void_p) for n in ("x", "x1", "x2", "w", "bias", "ln_w", "ln_b", "film", "shift", "scale", "mask",
                                          "window", "xout", "out_f32", "out_hi", "out_lo")]
                + [(n, C.c_int64) for n in ("film_bstride", "ada_bstride", "n")]
                + [(n, C.c_int32) for n in ("kind", "B", "BB", "T", "C", "c_clamp", "has_film", "mask_out", "u16", "Nh", "Kp",
                                            "K", "K2", "n_fft", "hop")]
                + [("eps", C.c_float)])


def library_path() -> str:
    """The in-tree library; STABLETTS_B200_LIB=<file name or path> selects another build of it (A/B runs of kernel
    generations on one box — never a different backend)."""
    override = os.environ.get("STABLETTS_B200_LIB")
    if override:
        return override if os.path.isabs(override) else os.path.join(_HERE, override)
    return os.path.join(_HERE, "libstabletts_b200.so")


def load_library() -> C.CDLL:
    """Loads the in-tree shared library; raises if it has not been built (no fallback)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). stabletts_b200 has no CPU/PyTorch fallback.")
    lib = C.CDLL(path)
    if os.environ.get("STABLETTS_B200_LIB"):       # an older build may lack the newest debug hooks: bind what it has
        class _Tolerant:
            def __init__(self, inner): object.__setattr__(self, "_inner", inner)
            def __getattr__(self, name):
                try:
                    return getattr(self._inner, name)
                except AttributeError:
                    return type("_Missing", (), {"argtypes": None, "restype": None})()
        real, lib = lib, _Tolerant(lib)
        bind = lib
    vp, f32p, i64, i32 = C.c_void_p, C.c_void_p, C.c_int64, C.c_int
    lib.st_create.argtypes = [C.POINTER(StDims), i32, C.POINTER(vp)]
    lib.st_destroy.argtypes = [vp]
    lib.st_last_error.argtypes = [vp]
    lib.st_last_error.restype = C.c_char_p
    lib.st_version.restype = i32
    lib.st_load_weight.argtypes = [vp, C.c_char_p, f32p, i64, vp]
    lib.st_finalize_weights.argtypes = [vp, vp]
    lib.st_set_engine.argtypes = [vp, i32]
    lib.st_set_precision.argtypes = [vp, i32]
    lib.st_workspace_bytes.argtypes = [vp, i32, i32, i32]
    lib.st_workspace_bytes.restype = C.c_size_t
    lib.st_attach_workspace.argtypes = [vp, vp, C.c_size_t]
    lib.st_estimator_forward.argtypes = [vp, f32p, i32, f32p, f32p, f32p, f32p, f32p, i32, i32, vp]
    lib.st_cfm_loss.argtypes = [vp, f32p, f32p, f32p, f32p, f32p, f32p, C.c_float, f32p, f32p, i32, i32, vp]
    lib.st_solve.argtypes = [vp, f32p, f32p, f32p, f32p, f32p, f32p, C.c_float, C.POINTER(C.c_float), i32, i32, i32, i32, vp]
    lib.st_solve_host.argtypes = lib.st_solve.argtypes
    lib.st_solve_host_io.argtypes = [vp, f32p] + lib.st_solve.argtypes[1:]
    lib.st_solve_adaptive.argtypes = [vp, f32p, f32p, f32p, f32p, f32p, f32p, C.c_float, C.c_double, C.c_double, C.c_double, C.c_double,
                                      i32, i32, i32, vp, C.POINTER(C.c_int64)]
    lib.st_solve_adaptive_ex.argtypes = [vp, i32] + lib.st_solve_adaptive.argtypes[1:]
    lib.st_align_lengths.argtypes = [f32p, f32p, C.c_float, i32, i32, f32p, vp, vp]
    lib.st_align_expand.argtypes = [f32p, f32p, f32p, vp, i32, i32, i32, i32, f32p, f32p, f32p, vp]
    lib.st_mas_workspace_bytes.argtypes = [i32, i32, i32]
    lib.st_mas_workspace_bytes.restype = C.c_size_t
    lib.st_mas_scores.argtypes = [f32p, f32p, f32p, i32, i32, i32, i32, vp]
    lib.st_maximum_path.argtypes = [f32p, f32p, vp, vp, f32p, f32p, f32p, vp, C.c_size_t, i32, i32, i32, vp]
    lib.st_mas_losses.argtypes = [f32p, f32p, f32p, f32p, f32p, f32p, vp, vp, C.c_size_t, i32, i32, i32, i32, f32p, f32p, vp]
    lib.st_create_text_encoder.argtypes = [C.POINTER(StDims), i32, i32, C.POINTER(vp)]
    lib.st_text_encoder_forward.argtypes = [vp, vp, f32p, vp, f32p, f32p, f32p, i32, i32, vp]
    lib.st_create_vocos.argtypes = [C.POINTER(StVocosDims), i32, C.POINTER(vp)]
    lib.st_vocos_forward.argtypes = [vp, f32p, f32p, i32, i32, vp]
    lib.st_create_ffgan.argtypes = [i32, C.POINTER(vp)]
    lib.st_ffgan_forward.argtypes = [vp, f32p, f32p, i32, i32, vp]
    lib.st_ffgan_workspace_bytes.argtypes = [vp, i32, i32]
    lib.st_ffgan_workspace_bytes.restype = C.c_size_t
    lib.st_create_style_encoder.argtypes = [i32, i32, C.POINTER(vp)]
    lib.st_style_encoder_forward.argtypes = [vp, f32p, f32p, f32p, i32, i32, vp]
    lib.st_create_duration_predictor.argtypes = [C.POINTER(StDims), i32, C.POINTER(vp)]
    lib.st_duration_predictor_forward.argtypes = [vp, f32p, f32p, f32p, f32p, i32, i32, vp]
    lib.st_create_mel.argtypes = [C.POINTER(StMelDims), i32, C.POINTER(vp)]
    lib.st_mel_forward.argtypes = [vp, f32p, f32p, i32, i64, i32, vp]
    lib.st_create_mel_loss.argtypes = [i32, C.POINTER(StMelDims), i32, C.POINTER(vp)]
    lib.st_mel_loss_workspace_bytes.argtypes = [vp, i32, i64]
    lib.st_mel_loss_workspace_bytes.restype = C.c_size_t
    lib.st_mel_loss_forward.argtypes = [vp, f32p, f32p, i32, i64, f32p, f32p, f32p, vp]
    lib.st_create_mpd.argtypes = [i32, i32, C.POINTER(vp)]
    lib.st_mpd_workspace_bytes.argtypes = [vp, i32, i64]
    lib.st_mpd_workspace_bytes.restype = C.c_size_t
    lib.st_mpd_forward.argtypes = [vp, f32p, i32, i64, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), vp]
    lib.st_mpd_backward.argtypes = [vp, f32p, i32, i64, C.POINTER(vp), C.POINTER(vp), f32p, C.POINTER(vp), f32p, C.POINTER(vp),
                                    C.POINTER(vp), vp]
    lib.st_create_resample.argtypes = [i32, i32, i32, C.POINTER(vp)]
    lib.st_resample_out_length.argtypes = [vp, i64]
    lib.st_resample_out_length.restype = i64
    lib.st_resample_forward.argtypes = [vp, f32p, f32p, i64, i64, vp]
    lib.st_launch_count.argtypes = [vp]
    lib.st_launch_count.restype = i64
    lib.st_profile_begin.argtypes = [vp]
    lib.st_profile_end.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    lib.st_profile_issued.argtypes = [vp, C.POINTER(C.c_double)]
    lib.st_test_gemm_ex.argtypes = [vp, C.POINTER(StTestGemmDesc), C.POINTER(StTestGemmPlan), vp]
    lib.st_test_conv_ex.argtypes = [vp, f32p, f32p, f32p, f32p, i32, i32, i32, i32, i32, i32, i32, vp]
    lib.st_bench_conv.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32, C.POINTER(C.c_float)]
    lib.st_test_attention_ex.argtypes = [vp, C.POINTER(StTestAttnDesc), vp]
    lib.st_test_row_ex.argtypes = [vp, C.POINTER(StTestRowDesc), vp]
    lib.st_test_mpd_conv.argtypes = [vp, i32, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, f32p, vp]
    for name in EXPORTS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("st_version",):
            fn.restype = C.c_int
    if os.environ.get("STABLETTS_B200_LIB"):
        lib = real
    _LIB = lib
    return lib


def check(lib, handle, rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.st_last_error(handle)
        raise RuntimeError(f"{what} failed: {msg.decode() if msg else 'unknown error'}")
