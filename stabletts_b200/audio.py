"""Drop-ins for the reference's feature extractor, ``utils/audio.py``: ``LogMelSpectrogram`` (api.py:72-73 turns the
reference audio into the mel the style encoder reads; preprocess.py:50-73 extracts the mel of every training clip) and its
``LinearSpectrogram``.

Same constructor arguments (``LogMelSpectrogram(**asdict(MelConfig()))`` works), the same ``compress`` / ``decompress``
and exactly the reference's state_dict: the buffers ``spectrogram.window`` (periodic Hann) and ``mel_scale.fb`` (the
slaney-normalised slaney-scale filterbank, (n_fft / 2 + 1, n_mels)).  The default ``fb`` is computed here, in float64, by
the formulas of torchaudio's ``melscale_fbanks``; a loaded ``fb`` or ``window`` is used as loaded.  ``forward`` is one
call into the CUDA library (``st_mel_forward``: frames -> fp32 FFT -> magnitude -> banded mel sum -> log, one kernel).

Built: ``center=False``, ``pad_mode="reflect"``, ``win_length == n_fft`` (a power of two in [32, 4096]) and
``mel_scale="slaney"`` — the reference's ``MelConfig``.  Other settings raise ``ValueError``.  Input: fp32 CUDA waveforms
(B, L) or (B, 1, L).  No CPU fallback."""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from . import _lib
from ._native import NativeModule, _Node


def _hz_to_mel_slaney(f: float) -> float:
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    if f < min_log_hz:
        return f / f_sp
    return min_log_hz / f_sp + math.log(f / min_log_hz) / (math.log(6.4) / 27.0)


def _mel_to_hz_slaney(m: torch.Tensor) -> torch.Tensor:
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0
    return torch.where(m >= min_log_mel, min_log_hz * torch.exp(logstep * (m - min_log_mel)), f_sp * m)


def slaney_mel_filterbank(n_freqs: int, f_min: float, f_max: float, n_mels: int, sample_rate: int,
                          dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """(n_freqs, n_mels): triangular filters equally spaced on the slaney mel scale, each divided by its width in Hz over 2
    (slaney area normalisation) — torchaudio.functional.melscale_fbanks(norm="slaney", mel_scale="slaney").  torchaudio
    evaluates these formulas in float32, 3.6e-6 (max-norm relative) from float64 at the default MelConfig; the module uses
    float64 and rounds once."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs, dtype=dtype)
    m_pts = torch.linspace(_hz_to_mel_slaney(f_min), _hz_to_mel_slaney(f_max), n_mels + 2, dtype=dtype)
    f_pts = _mel_to_hz_slaney(m_pts)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    down = -slopes[:, :-2] / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    fb = torch.clamp(torch.minimum(down, up), min=0.0)
    return fb * (2.0 / (f_pts[2:n_mels + 2] - f_pts[:n_mels]))[None, :]


def _check_config(n_fft, win_length, hop_length, pad, center, pad_mode):
    if center:
        raise ValueError("center=True is not built: the reference's MelConfig uses center=False with explicit reflect padding")
    if pad_mode != "reflect":
        raise ValueError(f"pad_mode={pad_mode!r} is not built: only 'reflect' (the reference's MelConfig)")
    if win_length != n_fft:
        raise ValueError(f"win_length={win_length} != n_fft={n_fft} is not built")
    if not isinstance(n_fft, int) or n_fft < 32 or n_fft > 4096 or n_fft & (n_fft - 1):
        raise ValueError(f"n_fft must be a power of two in [32, 4096], got {n_fft}")
    if hop_length <= 0 or pad < 0:
        raise ValueError("hop_length must be positive and pad non-negative")


class _SpectrogramBase(NativeModule):
    """Handle plumbing shared by both modules: buffers instead of parameters, no workspace."""

    def _native_buffers(self):
        raise NotImplementedError

    def _sync_weights(self, lib, h, stream: int, force: bool = False) -> None:
        if force:
            self._synced.clear()
        dirty = False
        for name, t in self._native_buffers():
            if t.device.type != "cuda" or t.dtype != torch.float32:
                raise RuntimeError(f"buffer {name} must be CUDA fp32 (got {t.device}, {t.dtype}); call .to('cuda')")
            tag = (t.data_ptr(), t._version)
            if self._synced.get(name) != tag:
                tc = t.detach().contiguous()
                _lib.check(lib, h, lib.st_load_weight(h, name.encode(), tc.data_ptr(), tc.numel(), stream), f"st_load_weight({name})")
                self._synced[name] = tag
                dirty = True
        if dirty:
            _lib.check(lib, h, lib.st_finalize_weights(h, stream), "st_finalize_weights")

    def set_engine(self, name: str) -> None:
        """Accepted for interface parity with the other modules and ignored: the spectrogram has one engine, fp32 CUDA
        cores (a tensor-core DFT would lose the accuracy the log needs in spectral valleys)."""
        if name not in ("tcgen05", "simt"):
            raise KeyError(name)

    def _run(self, x: torch.Tensor, channels: int, linear: int) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or x.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError(f"the waveform must be float32, got {x.dtype}")
        if x.ndim == 3 and x.shape[1] == 1:                      # (B, 1, L), as the reference's squeeze(1)
            x = x[:, 0]
        if x.ndim != 2:
            raise ValueError(f"the waveform must be (B, L) or (B, 1, L), got shape {tuple(x.shape)}")
        B, L = x.shape
        if L <= self.pad:
            raise ValueError(f"reflect padding needs pad < L: pad {self.pad}, L {L}")
        if L + 2 * self.pad < self.n_fft:
            raise ValueError(f"input too short: L + 2 pad = {L + 2 * self.pad} < n_fft = {self.n_fft} gives no frame")
        T = (L + 2 * self.pad - self.n_fft) // self.hop_length + 1
        out = torch.empty(B, channels, T, device=x.device, dtype=torch.float32)
        if B == 0:
            return out
        with torch.no_grad():
            wav = x.detach().contiguous()
            lib, h, stream = self._prepare(x)
            _lib.check(lib, h, lib.st_mel_forward(h, wav.data_ptr(), out.data_ptr(), B, L, linear, stream), "st_mel_forward")
        return out

    def _make_handle(self, lib, index, n_mels):
        dims = _lib.StMelDims(self.n_fft, self.hop_length, self.pad, n_mels)
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_mel(C.byref(dims), index, C.byref(h)), "st_create_mel")
        return h


class LinearSpectrogram(_SpectrogramBase):
    """utils/audio.py::LinearSpectrogram: waveform (B, L) or (B, 1, L) -> magnitude (B, n_fft / 2 + 1, T),
    sqrt(re^2 + im^2 + 1e-6) of the reflect-padded, Hann-windowed frames."""

    def __init__(self, n_fft, win_length, hop_length, pad, center, pad_mode):
        super().__init__()
        _check_config(n_fft, win_length, hop_length, pad, center, pad_mode)
        self.n_fft, self.win_length, self.hop_length, self.pad = n_fft, win_length, hop_length, pad
        self.center, self.pad_mode = center, pad_mode
        self.register_buffer("window", torch.hann_window(win_length))
        self._init_native()

    def _native_buffers(self):
        return [("spectrogram.window", self.window)]

    def _create_handle(self, lib, index):
        return self._make_handle(lib, index, 0)

    def forward(self, waveform: torch.Tensor) -> torch.Tensor:
        return self._run(waveform, self.n_fft // 2 + 1, 1)


class LogMelSpectrogram(_SpectrogramBase):
    """utils/audio.py::LogMelSpectrogram: waveform (B, L) or (B, 1, L) -> log-mel (B, n_mels, T),
    log(clamp(fb^T |STFT|, 1e-5)).  ``set_engine`` has no effect: the transform has one engine (fp32)."""

    def __init__(self, sample_rate, n_fft, win_length, hop_length, f_min, f_max, pad, n_mels, center, pad_mode, mel_scale):
        super().__init__()
        _check_config(n_fft, win_length, hop_length, pad, center, pad_mode)
        if mel_scale != "slaney":
            raise ValueError(f"mel_scale={mel_scale!r} is not built: only 'slaney' (the reference's MelConfig; its MelScale "
                             "passes mel_scale as the norm too, which torchaudio accepts only for 'slaney')")
        if n_mels <= 0 or n_mels > 4096:
            raise ValueError("n_mels must be in [1, 4096]")
        self.sample_rate = sample_rate
        self.n_fft = n_fft
        self.win_length = win_length
        self.hop_length = hop_length
        self.f_min = f_min
        self.f_max = f_max
        self.pad = pad
        self.n_mels = n_mels
        self.center = center
        self.pad_mode = pad_mode
        self.spectrogram = LinearSpectrogram(n_fft, win_length, hop_length, pad, center, pad_mode)
        self.mel_scale = _Node()                                  # torchaudio.transforms.MelScale: holds the buffer fb
        f_max_ = float(sample_rate // 2) if f_max is None else float(f_max)
        fb = slaney_mel_filterbank(n_fft // 2 + 1, float(f_min), f_max_, n_mels, sample_rate)
        self.mel_scale.register_buffer("fb", fb.to(torch.float32))
        self._init_native()

    def compress(self, x: torch.Tensor) -> torch.Tensor:
        return torch.log(torch.clamp(x, min=1e-5))

    def decompress(self, x: torch.Tensor) -> torch.Tensor:
        return torch.exp(x)

    def _native_buffers(self):
        return [("spectrogram.window", self.spectrogram.window), ("mel_scale.fb", self.mel_scale.fb)]

    def _create_handle(self, lib, index):
        return self._make_handle(lib, index, self.n_mels)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self._run(x, self.n_mels, 0)
