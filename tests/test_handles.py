"""Every typed entry point refuses a handle of another kind, first: one handle of each of the nine kinds (created, never
finalized) is passed to every entry point that does not take it, and each call returns 1 with that entry point's
"handle is not a ..." text before it looks at weights, shapes or pointers.  The workspace and length queries answer 0 / -1
for the kinds they do not belong to."""
import ctypes as C

import pytest
import torch

from kernel_harness import dev  # noqa: F401 (a fixture)

pytestmark = pytest.mark.gpu

B, T, L_WAV = 1, 8, 4096
N = 1 << 16                       # floats per buffer: more than any of these B = 1, T = 8 calls reads or writes


def _handles(lib, _lib):
    dit = _lib.StDims(80, 256, 1024, 4, 2, 3, 256)
    make = {
        "estimator": lambda h: lib.st_create(C.byref(dit), 0, h),
        "text_encoder": lambda h: lib.st_create_text_encoder(C.byref(_lib.StDims(80, 256, 1024, 4, 1, 3, 256)), 10, 0, h),
        "vocos": lambda h: lib.st_create_vocos(C.byref(_lib.StVocosDims(128, 512, 1536, 1, 512, 128)), 0, h),
        "ffgan": lambda h: lib.st_create_ffgan(0, h),
        "style": lambda h: lib.st_create_style_encoder(80, 0, h),
        "duration": lambda h: lib.st_create_duration_predictor(C.byref(_lib.StDims(80, 256, 1024, 4, 6, 3, 256)), 0, h),
        "mel": lambda h: lib.st_create_mel(C.byref(_lib.StMelDims(1024, 256, 384, 100)), 0, h),
        "mel_loss": lambda h: lib.st_create_mel_loss(1, (_lib.StMelDims * 1)(_lib.StMelDims(64, 16, 24, 5)), 0, h),
        "resample": lambda h: lib.st_create_resample(2, 3, 0, h),
    }
    out = {}
    for kind, create in make.items():
        h = C.c_void_p()
        _lib.check(lib, None, create(C.byref(h)), f"create {kind}")
        out[kind] = h
    return out


def test_every_entry_point_refuses_other_kinds_first(dev):
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    s = torch.cuda.current_stream(dev).cuda_stream
    d = [torch.zeros(N, device=dev) for _ in range(8)]
    p = [t.data_ptr() for t in d]
    hb = [torch.zeros(N) for _ in range(6)]
    q = [t.data_ptr() for t in hb]
    t_span = (C.c_float * 2)(0.0, 1.0)
    stats = (C.c_int64 * 3)()
    # (entry point, the kind it takes, the call)
    calls = [
        ("st_estimator_forward", "estimator", "CFM estimator",
         lambda h: lib.st_estimator_forward(h, p[0], 1, p[1], p[2], p[3], p[4], p[5], B, T, s)),
        ("st_cfm_loss", "estimator", "CFM estimator",
         lambda h: lib.st_cfm_loss(h, p[0], p[1], p[2], p[3], p[4], p[5], 1e-4, p[6], p[7], B, T, s)),
        ("st_solve", "estimator", "CFM estimator",
         lambda h: lib.st_solve(h, p[0], p[1], p[2], p[3], None, None, 1.0, t_span, 1, _lib.ST_EULER, B, T, s)),
        ("st_solve_host", "estimator", "CFM estimator",
         lambda h: lib.st_solve_host(h, q[0], q[1], q[2], q[3], None, None, 1.0, t_span, 1, _lib.ST_EULER, B, T, s)),
        ("st_solve_host_io", "estimator", "CFM estimator",
         lambda h: lib.st_solve_host_io(h, q[0], q[4], q[1], q[2], q[3], None, None, 1.0, t_span, 1, _lib.ST_EULER, B, T, s)),
        ("st_solve_adaptive_ex", "estimator", "CFM estimator",
         lambda h: lib.st_solve_adaptive_ex(h, _lib.ST_ADAPT_DOPRI5, p[0], p[1], p[2], p[3], None, None, 1.0, 0.0, 1.0, 1e-5,
                                            1e-5, 100, B, T, s, stats)),
        ("st_text_encoder_forward", "text_encoder", "text encoder",
         lambda h: lib.st_text_encoder_forward(h, p[0], p[1], p[2], p[3], p[4], p[5], B, T, s)),
        ("st_vocos_forward", "vocos", "Vocos vocoder", lambda h: lib.st_vocos_forward(h, p[0], p[1], B, T, s)),
        ("st_ffgan_forward", "ffgan", "FireflyGAN vocoder", lambda h: lib.st_ffgan_forward(h, p[0], p[1], B, T, s)),
        ("st_style_encoder_forward", "style", "MelStyleEncoder",
         lambda h: lib.st_style_encoder_forward(h, p[0], None, p[1], B, T, s)),
        ("st_duration_predictor_forward", "duration", "DurationPredictor",
         lambda h: lib.st_duration_predictor_forward(h, p[0], p[1], p[2], p[3], B, T, s)),
        ("st_mel_forward", "mel", "mel spectrogram", lambda h: lib.st_mel_forward(h, p[0], p[1], B, L_WAV, 0, s)),
        ("st_mel_loss_forward", "mel_loss", "mel loss",
         lambda h: lib.st_mel_loss_forward(h, p[0], p[1], B, L_WAV, p[2], p[3], p[4], s)),
        ("st_resample_forward", "resample", "resampler", lambda h: lib.st_resample_forward(h, p[0], p[1], B, T, s)),
    ]
    handles = _handles(lib, _lib)
    try:
        wrong = []
        for name, own, what, call in calls:
            for kind, h in handles.items():
                if kind == own:
                    continue
                rc = call(h)
                err = lib.st_last_error(h).decode()
                if rc != 1 or err != f"handle is not a {what}":
                    wrong.append((name, kind, rc, err))
        assert not wrong, wrong
        for kind, h in handles.items():
            ws = lib.st_workspace_bytes(h, B, T, 0)
            assert (ws > 0) if kind in ("estimator", "text_encoder") else ws == 0, (kind, ws)
            ml = lib.st_mel_loss_workspace_bytes(h, B, L_WAV)
            assert (ml > 0) if kind == "mel_loss" else ml == 0, (kind, ml)
            n = lib.st_resample_out_length(h, T)
            assert n == (12 if kind == "resample" else -1), (kind, n)
    finally:
        for h in handles.values():
            lib.st_destroy(h)
        torch.cuda.synchronize()
