"""Drop-ins for the Vocos training loss, ``vocoders/vocos/models/loss.py``: ``MultiScaleMelSpectrogramLoss`` (train.py:115
calls it on every generator step) and ``SingleScaleMelSpectrogramLoss``.

    loss = Σ_s mean |mel_s(x) − mel_s(y)|        mel_s: utils/audio.py's LogMelSpectrogram at MelConfig(n_mels=m_s,
                                                 n_fft=win_length=w_s, hop_length=w_s // 4), pad = 3 w_s / 8

Same constructor (defaults n_mels [5 … 320], window_lengths [32 … 2048]) and exactly the reference's state_dict:
``mel_transforms`` is an ``nn.ModuleList`` of this package's ``LogMelSpectrogram``, so the keys are
``mel_transforms.{i}.spectrogram.window`` and ``mel_transforms.{i}.mel_scale.fb``.  ``forward(x, y)`` is one call into the
CUDA library (``st_mel_loss_forward``): every scale's log-mels of x and y (bit for bit the drop-in ``LogMelSpectrogram``'s),
the L1 sums in double, and, when autograd wants them, the waveform gradients from the same pass.  The gradients are for a
unit upstream gradient; backward scales them by ``grad_output`` (``once_differentiable``: no double backward).  Repeated
calls are bitwise identical.

Input: fp32 CUDA waveforms (B, L) or (B, 1, L), x and y of one shape; gradients come back in that shape.  CPU tensors raise
``RuntimeError``, other dtypes ``TypeError``, an L too short for a scale's reflect padding or frame ``ValueError``.  The
module has no parameters, so it runs the same in ``train()`` and ``eval()`` mode."""
from __future__ import annotations

import ctypes as C
from typing import List

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from .audio import LogMelSpectrogram, _SpectrogramBase


def _mel_config(n_mels: int, n_fft: int) -> dict:
    """asdict(MelConfig(n_mels=n_mels, n_fft=n_fft, win_length=n_fft, hop_length=n_fft // 4)) of vocoders/vocos/config.py
    (its __post_init__ turns pad = 0 into (n_fft - hop_length) // 2)."""
    hop = n_fft // 4
    return dict(sample_rate=44100, n_fft=n_fft, win_length=n_fft, hop_length=hop, f_min=0.0, f_max=None,
                pad=(n_fft - hop) // 2, n_mels=n_mels, center=False, pad_mode="reflect", mel_scale="slaney")


class _MelLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, module, need_x, need_y):
        loss, gx, gy = module._compute(x, y, need_x, need_y)
        ctx.save_for_backward(gx, gy)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        gx, gy = ctx.saved_tensors
        return (None if gx is None else gx * grad_output, None if gy is None else gy * grad_output, None, None, None)


class _MelLossBase(_SpectrogramBase):
    """Handle plumbing of both losses: one st_mel_loss handle over the scales of ``_transforms()``."""

    def _transforms(self) -> List[LogMelSpectrogram]:
        raise NotImplementedError

    def _native_buffers(self):
        out = []
        for i, t in enumerate(self._transforms()):
            out += [(f"mel_transforms.{i}.spectrogram.window", t.spectrogram.window),
                    (f"mel_transforms.{i}.mel_scale.fb", t.mel_scale.fb)]
        return out

    def _create_handle(self, lib, index):
        ts = self._transforms()
        dims = (_lib.StMelDims * len(ts))(*[_lib.StMelDims(t.n_fft, t.hop_length, t.pad, t.n_mels) for t in ts])
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_mel_loss(len(ts), dims, index, C.byref(h)), "st_create_mel_loss")
        return h

    def _check(self, x: torch.Tensor, name: str) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or x.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError(f"{name} must be float32, got {x.dtype}")
        if not (x.ndim == 2 or (x.ndim == 3 and x.shape[1] == 1)):
            raise ValueError(f"{name} must be (B, L) or (B, 1, L), got shape {tuple(x.shape)}")
        return x.reshape(x.shape[0], x.shape[-1])

    def _compute(self, x, y, need_x: bool, need_y: bool):
        x2, y2 = x.detach().contiguous().view(x.shape[0], -1), y.detach().contiguous().view(y.shape[0], -1)
        B, L = x2.shape
        lib, h, stream = self._prepare(x)
        self._attach_workspace(lib, h, int(lib.st_mel_loss_workspace_bytes(h, B, L)), x.device)
        loss = torch.empty((), device=x.device, dtype=torch.float32)
        gx = torch.empty_like(x2) if need_x else None
        gy = torch.empty_like(y2) if need_y else None
        _lib.check(lib, h, lib.st_mel_loss_forward(h, x2.data_ptr(), y2.data_ptr(), B, L, loss.data_ptr(),
                                                    0 if gx is None else gx.data_ptr(), 0 if gy is None else gy.data_ptr(),
                                                    stream), "st_mel_loss_forward")
        return loss, None if gx is None else gx.view(x.shape), None if gy is None else gy.view(y.shape)

    def forward(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        xs, ys = self._check(x, "x"), self._check(y, "y")
        if xs.shape != ys.shape or x.device != y.device:
            raise ValueError(f"x and y must have one shape and device, got {tuple(x.shape)} on {x.device} and "
                             f"{tuple(y.shape)} on {y.device}")
        B, L = xs.shape
        if B == 0:
            raise ValueError("empty batch")
        for i, t in enumerate(self._transforms()):
            if L <= t.pad or L + 2 * t.pad < t.n_fft:
                raise ValueError(f"L = {L} is too short for scale {i} (n_fft {t.n_fft}): the reference's reflect padding "
                                 f"needs L > pad = {t.pad} and a frame needs L + 2 pad >= n_fft")
        grad = torch.is_grad_enabled()
        need_x, need_y = grad and x.requires_grad, grad and y.requires_grad
        if not (need_x or need_y):
            return self._compute(x, y, False, False)[0]
        return _MelLoss.apply(x, y, self, need_x, need_y)


class MultiScaleMelSpectrogramLoss(_MelLossBase):
    """models/loss.py::MultiScaleMelSpectrogramLoss: Σ over the scales of the L1 distance of the log-mels of x and y."""

    def __init__(self, n_mels: List[int] = [5, 10, 20, 40, 80, 160, 320],
                 window_lengths: List[int] = [32, 64, 128, 256, 512, 1024, 2048]):
        super().__init__()
        assert len(n_mels) == len(window_lengths), "n_mels and window_lengths must have the same length"
        self.mel_transforms = nn.ModuleList([LogMelSpectrogram(**_mel_config(m, w)) for m, w in zip(n_mels, window_lengths)])
        self._init_native()

    def _transforms(self):
        return list(self.mel_transforms)


class SingleScaleMelSpectrogramLoss(_MelLossBase):
    """models/loss.py::SingleScaleMelSpectrogramLoss: the L1 distance of the log-mels at the default MelConfig."""

    def __init__(self):
        super().__init__()
        self.mel_transform = LogMelSpectrogram(**_mel_config(128, 2048))
        self._init_native()

    def _transforms(self):
        return [self.mel_transform]
