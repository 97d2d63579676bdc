"""CPU oracle for the log-mel front end (TEST INFRASTRUCTURE ONLY): float64 restatement of utils/audio.py's
LogMelSpectrogram / LinearSpectrogram (center = False, reflect padding), plus the seeded test waveforms.  Pinned by
tests/test_mel.py against tests/golden/mel_*.npz, which oracle/make_golden_mel.py writes from the unmodified reference
module."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def mel_config(sample_rate=44100, n_fft=2048, hop_length=512, n_mels=128):
    """asdict(MelConfig(...)) of the reference's config.py: pad defaults to (n_fft - hop_length) // 2."""
    return dict(sample_rate=sample_rate, n_fft=n_fft, win_length=n_fft, hop_length=hop_length, f_min=0.0, f_max=None,
                pad=(n_fft - hop_length) // 2, n_mels=n_mels, center=False, pad_mode="reflect", mel_scale="slaney")


CONFIGS = {
    "default": mel_config(),                                                   # config.py MelConfig()
    "22k": mel_config(sample_rate=22050, n_fft=1024, hop_length=256, n_mels=80),
    "n512": mel_config(n_fft=512, hop_length=128, n_mels=80),                  # narrow filters: the 1e-5 clamp is active
}


def n_frames(cfg, L):
    return (L + 2 * cfg["pad"] - cfg["n_fft"]) // cfg["hop_length"] + 1


def slaney_fb(cfg, dtype=torch.float64):
    """torchaudio.functional.melscale_fbanks(n_fft//2+1, f_min, f_max or sr//2, n_mels, sr, "slaney", "slaney"), restated."""
    sr, n_mels, n_freqs = cfg["sample_rate"], cfg["n_mels"], cfg["n_fft"] // 2 + 1
    f_max = float(sr // 2) if cfg["f_max"] is None else float(cfg["f_max"])
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0

    def hz_to_mel(f):
        return f / f_sp if f < min_log_hz else min_log_mel + math.log(f / min_log_hz) / logstep

    m = torch.linspace(hz_to_mel(cfg["f_min"]), hz_to_mel(f_max), n_mels + 2, dtype=dtype)
    f_pts = torch.where(m >= min_log_mel, min_log_hz * torch.exp(logstep * (m - min_log_mel)), f_sp * m)
    freqs = torch.linspace(0, sr // 2, n_freqs, dtype=dtype)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - freqs[:, None]
    fb = torch.clamp(torch.minimum(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]), min=0.0)
    return fb * (2.0 / (f_pts[2:n_mels + 2] - f_pts[:n_mels]))[None, :]


def magnitude(wav, window, n_fft, hop_length, pad, dtype=torch.float64):
    """LinearSpectrogram.forward (audio.py:19-26) in float64 (or `dtype`): (B, L) or (B, 1, L) -> (B, n_fft // 2 + 1, T)."""
    x = wav.to(dtype)
    if x.ndim == 3:
        x = x.squeeze(1)
    x = F.pad(x.unsqueeze(1), (pad, pad), "reflect").squeeze(1)
    frames = x.unfold(-1, n_fft, hop_length) * window.to(dtype)                 # (B, T, n_fft)
    X = torch.fft.rfft(frames, dim=-1)
    return torch.sqrt(X.real ** 2 + X.imag ** 2 + 1e-6).transpose(1, 2)


def log_mel(wav, window, fb, cfg, dtype=torch.float64):
    """LogMelSpectrogram.forward (audio.py:53-57) in float64 (or `dtype`) with the given window and fb -> (B, n_mels, T)."""
    mag = magnitude(wav, window, cfg["n_fft"], cfg["hop_length"], cfg["pad"], dtype)
    mel = torch.matmul(mag.transpose(1, 2), fb.to(dtype)).transpose(1, 2)
    return torch.log(torch.clamp(mel, min=1e-5))


def make_wave(kind, seed, L, sample_rate=44100):
    """One seeded fp32 waveform (L,) of the named kind."""
    g = torch.Generator().manual_seed(seed)
    n = torch.arange(L, dtype=torch.float64)
    if kind == "noise":
        return torch.randn(L, generator=g) * 0.1
    if kind == "quiet":
        return torch.randn(L, generator=g) * 1e-4
    if kind == "silence":
        return torch.zeros(L)
    if kind == "sine":
        return (0.9 * torch.sin(2 * math.pi * 440.0 * n / sample_rate)).float()
    if kind == "lowpass":                                                       # white noise through a 64-tap Hann FIR
        w = torch.hann_window(64, dtype=torch.float64) / 32
        x = torch.randn(1, 1, L + 63, generator=g, dtype=torch.float64)
        return (0.3 * F.conv1d(x, w.view(1, 1, -1)).view(L)).float()
    if kind == "square":                                                        # exactly +-1, period 100 samples
        return ((n // 50) % 2 * -2.0 + 1.0).float()
    if kind == "speech":                                                        # a decaying harmonic stack + noise
        f0 = 110.0 + 40.0 * torch.rand(1, generator=g, dtype=torch.float64)
        x = sum(0.3 / k * torch.sin(2 * math.pi * k * f0 * n / sample_rate + float(k)) for k in range(1, 16))
        x = x * (0.6 + 0.4 * torch.sin(2 * math.pi * 3.0 * n / sample_rate)) + 0.01 * torch.randn(L, generator=g, dtype=torch.float64)
        return x.float()
    raise ValueError(kind)


def make_batch(kinds, seed, L, sample_rate=44100):
    return torch.stack([make_wave(k, seed + i, L, sample_rate) for i, k in enumerate(kinds)])


def checksum(wav):
    """(sum |x|, sum x * (1 + n mod 7)) in float64: detects a drifted generator."""
    x = wav.double().reshape(-1)
    return torch.stack([x.abs().sum(), (x * (1 + torch.arange(x.numel(), dtype=torch.float64) % 7)).sum()]).numpy()


L_CASE = 30000                                                                  # not a multiple of any hop
CASES = {
    "mel_noise":     dict(cfg="default", kinds=["noise"], seed=101, L=L_CASE),
    "mel_sine440":   dict(cfg="default", kinds=["sine"], seed=102, L=L_CASE),
    "mel_silence":   dict(cfg="default", kinds=["silence"], seed=103, L=L_CASE),
    "mel_quiet":     dict(cfg="default", kinds=["quiet"], seed=104, L=L_CASE),
    "mel_lowpass":   dict(cfg="default", kinds=["lowpass"], seed=105, L=L_CASE),
    "mel_square":    dict(cfg="default", kinds=["square"], seed=106, L=L_CASE),
    "mel_batch3":    dict(cfg="default", kinds=["noise", "sine", "quiet"], seed=107, L=L_CASE),
    "mel_22k":       dict(cfg="22k", kinds=["noise", "lowpass"], seed=108, L=15000),
    "mel_n512":      dict(cfg="n512", kinds=["noise", "silence", "quiet"], seed=109, L=8000),
}
# LinearSpectrogram fixtures: short clips (the magnitude has n_fft / 2 + 1 rows)
LINEAR_CASES = {
    "mel_linear_default": dict(cfg="default", kinds=["noise", "sine"], seed=111, L=8192),
    "mel_linear_n512":    dict(cfg="n512", kinds=["lowpass"], seed=112, L=4096),
}
# waveform -> LogMelSpectrogram -> MelStyleEncoder (style_ref's seeded weights, 128 mels), as api.py:72-73 + model.py:79
COMPOSED = dict(name="mel_style_composed", cfg="default", kinds=["speech", "noise"], seed=121, L=44100)
