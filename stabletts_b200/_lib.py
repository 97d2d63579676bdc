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
ST_PROF_NAMES = ("gemm_other", "attention", "ln", "gemm_qkv", "gemm_o", "gemm_conv1", "gemm_conv2", "gemm_lsc", "gemm_cond")
ST_PROF_NCAT = len(ST_PROF_NAMES)

# every symbol include/stabletts_b200.h declares (tests check the .so exports all of them)
EXPORTS = [
    "st_create", "st_destroy", "st_last_error", "st_version", "st_load_weight", "st_finalize_weights",
    "st_set_engine", "st_set_precision", "st_workspace_bytes", "st_attach_workspace", "st_estimator_forward", "st_cfm_loss", "st_solve",
    "st_solve_host", "st_solve_host_io", "st_solve_adaptive", "st_solve_adaptive_ex", "st_align_lengths", "st_align_expand", "st_create_text_encoder", "st_text_encoder_forward", "st_create_vocos", "st_vocos_forward", "st_launch_count", "st_profile_begin", "st_profile_end", "st_profile_issued", "st_test_gemm", "st_test_conv", "st_test_attention", "st_bench_conv",
]


class StDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_mel", "hidden", "filter", "n_heads", "n_layers", "kernel", "gin")]


class StVocosDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_mel", "dim", "intermediate", "n_layers", "n_fft", "hop")]


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
    lib.st_create_text_encoder.argtypes = [C.POINTER(StDims), i32, i32, C.POINTER(vp)]
    lib.st_text_encoder_forward.argtypes = [vp, vp, f32p, vp, f32p, f32p, f32p, i32, i32, vp]
    lib.st_create_vocos.argtypes = [C.POINTER(StVocosDims), i32, C.POINTER(vp)]
    lib.st_vocos_forward.argtypes = [vp, f32p, f32p, i32, i32, vp]
    lib.st_launch_count.argtypes = [vp]
    lib.st_launch_count.restype = i64
    lib.st_profile_begin.argtypes = [vp]
    lib.st_profile_end.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    lib.st_profile_issued.argtypes = [vp, C.POINTER(C.c_double)]
    lib.st_test_gemm.argtypes = [vp, f32p, f32p, f32p, f32p, i32, i32, i32, i32, vp]
    lib.st_test_conv.argtypes = [vp, f32p, f32p, f32p, f32p, i32, i32, i32, i32, i32, vp]
    lib.st_bench_conv.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, C.POINTER(C.c_float)]
    lib.st_test_attention.argtypes = [vp, f32p, f32p, f32p, i32, i32, vp]
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
