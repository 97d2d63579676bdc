"""The log-mel front end: LogMelSpectrogram / LinearSpectrogram on the fp32 FFT kernel (mel.cu).

CPU: the float64 oracle (oracle/mel_ref.py) against the fixtures of the unmodified reference module (tests/golden/mel_*.npz;
recipe oracle/make_golden_mel.py), the package's default filterbank against the reference's, the state_dict inventory and
the refusals.
GPU: every fixture case within max(1e-4, 4 E32) absolute log-mel error of the reference's float64 output (E32: the
reference module's own fp32 error on that case), the LinearSpectrogram magnitude, edges against the oracle, exact
properties (batch independence, determinism, (B, 1, L) input, a zeroed filter, a non-Hann window) and the composition
waveform -> LogMelSpectrogram -> MelStyleEncoder against the reference modules."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import rel_errs
from oracle import mel_ref as M, style_ref, weights


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _wave(cs):
    return M.make_batch(cs["kinds"], cs["seed"], cs["L"], M.CONFIGS[cs["cfg"]]["sample_rate"])


def _hann(cfg):
    return torch.hann_window(cfg["n_fft"])                     # the reference's fp32 buffer


# ------------------------------------------------------------------ CPU ------------------------------------------------------

@pytest.mark.parametrize("name", list(M.CASES))
def test_oracle_vs_reference_golden(name, golden_dir):
    cs, g = M.CASES[name], _golden(golden_dir, name)
    cfg = M.CONFIGS[cs["cfg"]]
    x = _wave(cs)
    np.testing.assert_allclose(M.checksum(x), g["wave_checksum"], rtol=1e-12)
    out = M.log_mel(x, _hann(cfg), torch.from_numpy(g["fb"]), cfg)
    assert float((out - torch.from_numpy(g["out64"])).abs().max()) <= 1e-9


@pytest.mark.parametrize("name", list(M.LINEAR_CASES))
def test_oracle_linear_vs_reference_golden(name, golden_dir):
    cs, g = M.LINEAR_CASES[name], _golden(golden_dir, name)
    cfg = M.CONFIGS[cs["cfg"]]
    x = _wave(cs)
    np.testing.assert_allclose(M.checksum(x), g["wave_checksum"], rtol=1e-12)
    out = M.magnitude(x, _hann(cfg), cfg["n_fft"], cfg["hop_length"], cfg["pad"])
    assert max(rel_errs(out, torch.from_numpy(g["linear64"]))) <= 1e-12


@pytest.mark.parametrize("cfg_name,case", [("default", "mel_noise"), ("22k", "mel_22k"), ("n512", "mel_n512")])
def test_default_filterbank_vs_reference(cfg_name, case, golden_dir):
    """The formulas evaluated in fp32 (torchaudio's precision) give the reference's fb bit for bit; the package evaluates
    them in float64, which differs from torchaudio's fp32 arithmetic by its rounding (3.6e-6 at the default config)."""
    from stabletts_b200.audio import LogMelSpectrogram, slaney_mel_filterbank
    cfg = M.CONFIGS[cfg_name]
    ref = torch.from_numpy(_golden(golden_dir, case)["fb"])
    n_freqs = cfg["n_fft"] // 2 + 1
    f32 = slaney_mel_filterbank(n_freqs, cfg["f_min"], float(cfg["sample_rate"] // 2), cfg["n_mels"], cfg["sample_rate"], torch.float32)
    assert torch.equal(f32, ref)
    assert torch.equal(M.slaney_fb(cfg, torch.float32), ref)
    fb = LogMelSpectrogram(**cfg).mel_scale.fb
    assert fb.dtype == torch.float32 and tuple(fb.shape) == tuple(ref.shape)
    assert rel_errs(fb, ref)[0] <= 1e-5
    assert torch.equal(fb, M.slaney_fb(cfg).float())


def test_state_dict_matches_reference_inventory(golden_dir):
    from stabletts_b200 import LogMelSpectrogram
    from stabletts_b200.audio import LinearSpectrogram
    m = LogMelSpectrogram(**M.CONFIGS["default"])
    sd = m.state_dict()
    assert list(sd) == ["spectrogram.window", "mel_scale.fb"]
    assert tuple(sd["spectrogram.window"].shape) == (2048,) and tuple(sd["mel_scale.fb"].shape) == (1025, 128)
    assert torch.equal(sd["spectrogram.window"], torch.hann_window(2048))
    assert isinstance(m.spectrogram, LinearSpectrogram)
    assert list(m.parameters()) == []
    fb = torch.from_numpy(_golden(golden_dir, "mel_noise")["fb"])
    m.load_state_dict({"spectrogram.window": torch.hann_window(2048), "mel_scale.fb": fb}, strict=True)
    assert torch.equal(m.mel_scale.fb, fb)
    x = torch.randn(2, 5000)
    assert torch.equal(m.decompress(m.compress(x.abs() + 1e-3)), torch.exp(torch.log(torch.clamp(x.abs() + 1e-3, min=1e-5))))


@pytest.mark.parametrize("override", [dict(center=True), dict(pad_mode="constant"), dict(win_length=1024),
                                      dict(mel_scale="htk"), dict(n_fft=1000, win_length=1000), dict(n_fft=8192, win_length=8192)])
def test_refused_configurations(override):
    from stabletts_b200 import LogMelSpectrogram
    with pytest.raises(ValueError):
        LogMelSpectrogram(**{**M.CONFIGS["default"], **override})


def test_cpu_tensor_raises():
    from stabletts_b200 import LogMelSpectrogram
    m = LogMelSpectrogram(**M.CONFIGS["default"])
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 44100))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.spectrogram(torch.randn(1, 44100))


# ------------------------------------------------------------------ GPU ------------------------------------------------------

def _module(cfg, fb=None, window=None):
    from stabletts_b200 import LogMelSpectrogram
    m = LogMelSpectrogram(**cfg)
    if fb is not None:
        m.mel_scale.fb.copy_(fb)
    if window is not None:
        m.spectrogram.window.copy_(window)
    return m.cuda()


def _bar(e32):
    return max(1e-4, 4 * e32)


_GROUPS = {"default": [n for n, c in M.CASES.items() if c["cfg"] == "default"], "22k": ["mel_22k"], "n512": ["mel_n512"]}


@pytest.mark.gpu
@pytest.mark.parametrize("group", list(_GROUPS))
def test_gpu_vs_reference_golden(group, golden_dir):
    worst = []
    for name in _GROUPS[group]:
        cs, g = M.CASES[name], _golden(golden_dir, name)
        cfg = M.CONFIGS[cs["cfg"]]
        m = _module(cfg, fb=torch.from_numpy(g["fb"]))
        out = m(_wave(cs).cuda())
        ref = torch.from_numpy(g["out64"])
        assert out.shape == ref.shape and out.dtype == torch.float32
        err = float((out.double().cpu() - ref).abs().max())
        bar = _bar(float(g["E32"]))
        worst.append((err / bar, name, err, bar))
        assert err <= bar, (name, err, bar)
    r, name, err, bar = max(worst)
    print(f"[mel {group}] worst ratio to the bar {r:.3f} ({name}: {err:.3e} vs {bar:.3e})")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(M.LINEAR_CASES))
def test_gpu_linear_vs_reference_golden(name, golden_dir):
    from stabletts_b200 import LinearSpectrogram
    cs, g = M.LINEAR_CASES[name], _golden(golden_dir, name)
    cfg = M.CONFIGS[cs["cfg"]]
    m = LinearSpectrogram(cfg["n_fft"], cfg["win_length"], cfg["hop_length"], cfg["pad"], False, "reflect").cuda()
    out = m(_wave(cs).cuda())
    e = rel_errs(out, torch.from_numpy(g["linear64"]))
    print(f"[linear {name}] rel_errs {e[0]:.3e} / {e[1]:.3e}")
    assert max(e) <= 1e-5


def _oracle_bar(x, window, fb, cfg):
    """the fixture tests' bar for an oracle case: max(1e-4, 4 E32) with E32 the error of the same transform computed by
    torch in fp32 (torch.fft.rfft, matmul) against float64 — tonal inputs put fp32 error of ~1e-3 into spectral valleys"""
    e32 = float((M.log_mel(x, window, fb, cfg, torch.float32).double() - M.log_mel(x, window, fb, cfg)).abs().max())
    return _bar(e32)


def _edge_check(cfg, x, fb=None, frames=None):
    """(max abs error against the float64 oracle, bar)"""
    fb = M.slaney_fb(cfg).float() if fb is None else fb
    m = _module(cfg, fb=fb)
    out = m(x.cuda()).double().cpu()
    assert out.shape[-1] == M.n_frames(cfg, x.shape[-1])
    if frames is None:
        ref = M.log_mel(x, _hann(cfg), fb, cfg)
        bar = _oracle_bar(x, _hann(cfg), fb, cfg)
    else:                                           # the oracle on just the frames that read the sampled outputs
        hop, n_fft, pad = cfg["hop_length"], cfg["n_fft"], cfg["pad"]
        xp = torch.nn.functional.pad(x.double().unsqueeze(1), (pad, pad), "reflect").squeeze(1)
        segs = torch.stack([xp[:, t * hop:t * hop + n_fft] for t in frames], -1)       # (B, n_fft, k)
        X = torch.fft.rfft(segs * _hann(cfg).double()[None, :, None], dim=1)
        mag = torch.sqrt(X.real ** 2 + X.imag ** 2 + 1e-6)
        ref = torch.log(torch.clamp(torch.einsum("bkt,km->bmt", mag, fb.double()), min=1e-5))
        out = out[..., frames]
        bar = 1e-4
    return float((out - ref).abs().max()), bar


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", list(M.CONFIGS))
def test_gpu_edges_vs_oracle(cfg_name):
    cfg = M.CONFIGS[cfg_name]
    n_fft, pad, hop, sr = cfg["n_fft"], cfg["pad"], cfg["hop_length"], cfg["sample_rate"]
    L1 = max(pad + 1, n_fft - 2 * pad)                          # the shortest legal input: T = 1
    assert M.n_frames(cfg, L1) == 1
    cases = {
        "T1": M.make_batch(["noise", "lowpass"], 201, L1, sr),
        "T1+hop-1": M.make_batch(["noise"], 202, L1 + hop - 1, sr),            # still one frame
        "ragged": M.make_batch(["noise", "sine"], 203, 7 * hop + 333, sr),     # L not a multiple of hop
        "both_pads": M.make_batch(["lowpass"], 204, pad + 5, sr),             # every frame reads both reflect pads
    }
    for k, x in cases.items():
        err, bar = _edge_check(cfg, x)
        print(f"[mel edge {cfg_name} {k}] L {x.shape[-1]} max abs {err:.3e}, bar {bar:.3e}")
        assert err <= bar, (k, err, bar)


@pytest.mark.gpu
def test_gpu_ten_minute_clip():
    cfg = M.CONFIGS["default"]
    L = 600 * cfg["sample_rate"]
    x = M.make_batch(["speech"], 205, L)
    T = M.n_frames(cfg, L)
    assert 51000 < T < 52000
    frames = [0, 1, 2, 1000, 25837, T // 2 + 3, T - 9, T - 2, T - 1]
    err, bar = _edge_check(cfg, x, frames=frames)
    print(f"[mel 10 min] T {T}, sampled frames max abs {err:.3e}")
    assert err <= bar


@pytest.mark.gpu
def test_gpu_exact_properties():
    cfg = M.CONFIGS["default"]
    m = _module(cfg)
    x = M.make_batch(["noise", "sine", "speech", "quiet"], 301, 20000).cuda()
    full = m(x)
    for b in range(x.shape[0]):                                             # an utterance alone equals its batch row
        assert torch.equal(m(x[b:b + 1])[0], full[b])
    assert torch.equal(m(x), full)                                          # repeated runs are bit-identical
    assert torch.equal(m(x.unsqueeze(1)), full)                             # (B, 1, L) as the reference's squeeze(1)
    assert m(x[:0]).shape == (0, 128, full.shape[-1])                       # B = 0
    fb = m.mel_scale.fb.clone()                                             # a zeroed filter gives log(1e-5) exactly
    m.mel_scale.fb[:, 17] = 0
    z = m(x)
    assert torch.all(z[:, 17] == torch.tensor(1e-5, dtype=torch.float32).log())
    keep = [i for i in range(128) if i != 17]
    assert torch.equal(z[:, keep], full[:, keep])
    m.mel_scale.fb.copy_(fb)
    assert torch.equal(m(x), full)
    with pytest.raises(TypeError):
        m(x.double())
    with pytest.raises(ValueError):
        m(x[:, :cfg["pad"]])                                                # reflect padding needs pad < L
    with pytest.raises(ValueError):
        m(x[:, :2])


@pytest.mark.gpu
def test_gpu_loaded_window_is_honoured():
    cfg = M.CONFIGS["22k"]
    n = torch.arange(cfg["n_fft"], dtype=torch.float64)
    win = (0.54 - 0.46 * torch.cos(2 * math.pi * n / cfg["n_fft"])).float()     # Hamming
    fb = M.slaney_fb(cfg).float()
    m = _module(cfg, fb=fb, window=win)
    x = M.make_batch(["noise", "sine"], 302, 9000, cfg["sample_rate"])
    err = float((m(x.cuda()).double().cpu() - M.log_mel(x, win, fb, cfg)).abs().max())
    bar = _oracle_bar(x, win, fb, cfg)
    print(f"[mel hamming window] max abs {err:.3e}, bar {bar:.3e}")
    assert err <= bar
    assert float((M.log_mel(x, win, fb, cfg) - M.log_mel(x, _hann(cfg), fb, cfg)).abs().max()) > 1e-2


@pytest.mark.gpu
def test_gpu_composed_with_style_encoder(golden_dir):
    """waveform -> LogMelSpectrogram -> MelStyleEncoder (api.py:72-73, models/model.py:79), both this library's"""
    from stabletts_b200 import LogMelSpectrogram, MelStyleEncoder
    cs = M.COMPOSED
    g = _golden(golden_dir, cs["name"])
    cfg = M.CONFIGS[cs["cfg"]]
    x = _wave(cs)
    np.testing.assert_allclose(M.checksum(x), g["wave_checksum"], rtol=1e-12)
    st = style_ref.make_state(n_mel=cfg["n_mels"])
    assert float(g["weight_checksum"]) == pytest.approx(weights.checksum(st), rel=1e-12)
    mel = LogMelSpectrogram(**cfg).cuda()
    enc = MelStyleEncoder(cfg["n_mels"], 128, 256, 5, 2, 0.1).eval()
    enc.load_state_dict(st, strict=True)
    enc = enc.cuda()
    with torch.inference_mode():
        c = enc(mel(x.cuda()), None)
    e = rel_errs(c, torch.from_numpy(g["c"]))
    print(f"[mel -> style encoder] c rel_errs {e[0]:.3e} / {e[1]:.3e}")
    assert max(e) <= 1e-4
