"""Drop-ins for the Vocos training discriminator, ``vocoders/vocos/models/discriminator.py``: ``MultiPeriodDiscriminator``
and ``DiscriminatorP``, ``MultiResolutionDiscriminator`` and ``DiscriminatorR`` (train.py runs both on real and generated
audio in both half-steps).

The parameter tree is the reference's: ``convs.{0..4}`` and ``conv_post`` are real ``nn.Conv2d`` modules under
``torch.nn.utils.parametrizations.weight_norm``, so the state_dict keys (``….parametrizations.weight.original0`` / ``original1``
/ ``.bias``), parameter identity, optimizers, ``clip_grad_norm_`` and DDP behave as there.  Their forward is never called:
``conv.weight`` (torch computes the weight norm and its backward) and ``conv.bias`` go into one autograd Function whose
forward and backward are calls into the CUDA library (``st_mpd_forward`` / ``st_mpd_backward``).  The weights are packed on
every call, so optimizer steps are always seen.

The Function returns the fmaps of convs 1-4 and ``post``; the score is ``torch.flatten(post, 1)`` outside it, so gradients
on the score and on the last fmap add up as in the reference.  Backward saves the input and the fmaps of convs 0-4, nothing
else (per DiscriminatorP and sample: 4 (L + Σ_i C_i H_i p) bytes, the fmaps the caller holds anyway plus conv 0's).  It
computes the input gradient only when x requires grad and the weight gradients only when a parameter does
(``once_differentiable``: no double backward).

Input: fp32 CUDA (B, 1, L).  CPU tensors raise ``RuntimeError``; other shapes, an L too short for the reflect pad and
constructor arguments other than the reference's defaults raise ``ValueError``."""
from __future__ import annotations

import ctypes as C
from typing import List, Tuple

import torch
import torch.nn as nn
from torch import Tensor
from torch.autograd.function import once_differentiable
from torch.nn.utils.parametrizations import weight_norm

from . import _lib
from ._native import NativeModule


def _ptrs(ts) -> "C.Array":
    return (C.c_void_p * len(ts))(*[0 if t is None else t.data_ptr() for t in ts])


class _MPDFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, module, *wb):
        ws, bs = [w.detach().contiguous() for w in wb[:6]], [b.detach().contiguous() for b in wb[6:]]
        x2 = x.detach().contiguous().view(x.shape[0], x.shape[-1])
        fm = module._forward(x2, ws, bs)
        ctx.module = module
        ctx.save_for_backward(x2, *ws, *fm[:5])
        ctx.bshapes = [b.shape for b in bs]
        ctx.xshape = x.shape
        return tuple(fm[1:])

    @staticmethod
    @once_differentiable
    def backward(ctx, g1, g2, g3, g4, gpost):
        x2, *rest = ctx.saved_tensors
        ws, fm = rest[:6], rest[6:]
        need_x = ctx.needs_input_grad[0]
        need_w = any(ctx.needs_input_grad[2:])
        gx, gw, gb = ctx.module._backward(x2, ws, fm, [g1, g2, g3, g4], gpost, need_x, need_w)
        gx = None if gx is None else gx.view(ctx.xshape)
        gw = gw if gw is not None else [None] * 6
        gb = gb if gb is not None else [None] * 6
        return (gx, None, *gw, *gb)


class DiscriminatorP(NativeModule):
    """models/discriminator.py::DiscriminatorP on sm_90a.  ``forward(x)`` -> ``(score, fmap)`` with score (B, H_post p) and
    fmap the post-activation outputs of convs 1-4 plus conv_post's, NCHW (B, C, H_i, p)."""

    def __init__(self, period: int, in_channels: int = 1, kernel_size: int = 5, stride: int = 3, lrelu_slope: float = 0.1):
        super().__init__()
        if (in_channels, kernel_size, stride, lrelu_slope) != (1, 5, 3, 0.1):
            raise ValueError("this DiscriminatorP is built for the reference's defaults only: in_channels=1, kernel_size=5, "
                             f"stride=3, lrelu_slope=0.1 (got {in_channels}, {kernel_size}, {stride}, {lrelu_slope})")
        if not isinstance(period, int) or not 1 <= period <= 4096:
            raise ValueError(f"period must be an int in [1, 4096], got {period!r}")
        self.period = period
        self.lrelu_slope = lrelu_slope
        chans = [1, 32, 128, 512, 1024, 1024]
        self.convs = nn.ModuleList([
            weight_norm(nn.Conv2d(chans[i], chans[i + 1], (5, 1), (3 if i < 4 else 1, 1), padding=(2, 0))) for i in range(5)])
        self.conv_post = weight_norm(nn.Conv2d(1024, 1, (3, 1), 1, padding=(1, 0)))
        self._init_native()
        self._shapes = {}                 # no weights live in the handle: every call passes them

    def _create_handle(self, lib, index):
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_mpd(self.period, index, C.byref(h)), "st_create_mpd")
        return h

    def _layers(self):
        return list(self.convs) + [self.conv_post]

    def _heights(self, L: int) -> List[int]:
        H = -(-L // self.period)
        out = []
        for i in range(5):
            H = -(-H // 3) if i < 4 else H
            out.append(H)
        return out

    def _call_prep(self, x2: Tensor):
        B, L = x2.shape
        lib, h, stream = self._prepare(x2)
        need = int(lib.st_mpd_workspace_bytes(h, B, L))
        if need == 0:
            raise RuntimeError(f"st_mpd_workspace_bytes refused B = {B}, L = {L}: {lib.st_last_error(h).decode()}")
        ws = torch.empty(need, dtype=torch.uint8, device=x2.device)   # per call: the caching allocator shares it between periods
        _lib.check(lib, h, lib.st_attach_workspace(h, ws.data_ptr(), ws.numel()), "st_attach_workspace")
        return lib, h, stream, ws

    def _forward(self, x2: Tensor, ws, bs) -> List[Tensor]:
        B, L = x2.shape
        H = self._heights(L)
        chans = [32, 128, 512, 1024, 1024]
        fm = [torch.empty((B, chans[i], H[i], self.period), device=x2.device, dtype=torch.float32) for i in range(5)]
        fm.append(torch.empty((B, 1, H[4], self.period), device=x2.device, dtype=torch.float32))
        lib, h, stream, work = self._call_prep(x2)
        _lib.check(lib, h, lib.st_mpd_forward(h, x2.data_ptr(), B, L, _ptrs(ws), _ptrs(bs), _ptrs(fm), stream), "st_mpd_forward")
        del work
        return fm

    def _backward(self, x2, ws, fm, gf, gpost, need_x: bool, need_w: bool):
        B, L = x2.shape
        gpost = torch.zeros_like(fm[4][:, :1]) if gpost is None else gpost.contiguous().float()
        gf = [None if g is None else g.contiguous().float() for g in gf]
        gx = torch.empty_like(x2) if need_x else None
        gw = [torch.empty_like(w) for w in ws] if need_w else None
        gb = [torch.empty(w.shape[0], device=w.device, dtype=torch.float32) for w in ws] if need_w else None
        lib, h, stream, work = self._call_prep(x2)
        _lib.check(lib, h, lib.st_mpd_backward(h, x2.data_ptr(), B, L, _ptrs(ws), _ptrs(fm), gpost.data_ptr(), _ptrs(gf),
                                               0 if gx is None else gx.data_ptr(), _ptrs(gw) if need_w else None,
                                               _ptrs(gb) if need_w else None, stream), "st_mpd_backward")
        del work
        return gx, gw, gb

    def forward(self, x: Tensor) -> Tuple[Tensor, List[Tensor]]:
        if not isinstance(x, torch.Tensor) or x.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError(f"x must be float32, got {x.dtype}")
        if x.ndim != 3 or x.shape[1] != 1 or x.shape[0] == 0:
            raise ValueError(f"x must be (B, 1, L) with B >= 1, got shape {tuple(x.shape)}")
        L = x.shape[-1]
        n_pad = (self.period - L % self.period) % self.period
        if L == 0 or n_pad >= L:
            raise ValueError(f"L = {L} is too short for the reflect pad of period {self.period}: the pad {n_pad} must be below L")
        layers = self._layers()
        ws = [m.weight for m in layers]
        bs = [m.bias for m in layers]
        f1, f2, f3, f4, post = _MPDFunction.apply(x, self, *ws, *bs)
        return torch.flatten(post, 1, -1), [f1, f2, f3, f4, post]


class MultiPeriodDiscriminator(nn.Module):
    """models/discriminator.py::MultiPeriodDiscriminator: one DiscriminatorP per period, each run on y then y_hat."""

    def __init__(self, periods: Tuple[int, ...] = (2, 3, 5, 7, 11)):
        super().__init__()
        self.discriminators = nn.ModuleList([DiscriminatorP(period=p) for p in periods])

    def set_engine(self, name: str) -> None:
        for d in self.discriminators:
            d.set_engine(name)

    def forward(self, y: Tensor, y_hat: Tensor):
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
        for d in self.discriminators:
            y_d_r, fmap_r = d(y)
            y_d_g, fmap_g = d(y_hat)
            y_d_rs.append(y_d_r)
            fmap_rs.append(fmap_r)
            y_d_gs.append(y_d_g)
            fmap_gs.append(fmap_g)
        return y_d_rs, y_d_gs, fmap_rs, fmap_gs


# ---------------------------------------------------------------------------------------------------------------------------
# the multi-resolution discriminator (models/discriminator.py:78-171)
# ---------------------------------------------------------------------------------------------------------------------------
_MRD_BANDS = ((0.0, 0.1), (0.1, 0.25), (0.25, 0.5), (0.5, 0.75), (0.75, 1.0))


class _Spectrogram(nn.Module):
    """Holds ``spec_fn.window`` as torchaudio's Spectrogram does (a buffer, in the state_dict); never called."""

    def __init__(self, n_fft: int):
        super().__init__()
        self.register_buffer("window", torch.hann_window(n_fft))


class _MRDFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, module, window, *wb):
        ws, bs = [w.detach().contiguous() for w in wb[:26]], [b.detach().contiguous() for b in wb[26:]]
        x2 = x.detach().contiguous().view(x.shape[0], x.shape[-1])
        win = window.detach().contiguous().float()
        spec, fm, post = module._forward(x2, win, ws, bs)
        ctx.module = module
        ctx.set_materialize_grads(False)       # an output without a cotangent reaches the library as NULL, not as zeros
        ctx.save_for_backward(x2, win, spec, *ws, *fm)
        ctx.xshape = x.shape
        return (post, *[fm[5 * k + i] for k in range(5) for i in range(1, 5)])

    @staticmethod
    @once_differentiable
    def backward(ctx, gpost, *gf):
        x2, win, spec, *rest = ctx.saved_tensors
        ws, fm = rest[:26], rest[26:]
        need_x = ctx.needs_input_grad[0]
        need_w = any(ctx.needs_input_grad[3:])
        gx, gw, gb = ctx.module._backward(x2, win, spec, ws, fm, gpost, list(gf), need_x, need_w)
        gx = None if gx is None else gx.view(ctx.xshape)
        gw = gw if gw is not None else [None] * 26
        gb = gb if gb is not None else [None] * 26
        return (gx, None, None, *gw, *gb)


class DiscriminatorR(NativeModule):
    """models/discriminator.py::DiscriminatorR on sm_90a.  ``forward(x)`` -> ``(score, fmap)``: score (B, 1, T', Σ W4) is
    conv_post's output over the concatenated bands, fmap the 20 band activations (B, 32, T', W_i) of convs 1-4 of each band
    followed by the score.  The STFT reads the loaded ``spec_fn.window`` buffer; ``spec_fn`` itself is never called."""

    def __init__(self, window_length: int, channels: int = 32, hop_factor: float = 0.25,
                 bands: Tuple[Tuple[float, float], ...] = _MRD_BANDS):
        super().__init__()
        if channels != 32 or hop_factor != 0.25 or tuple(tuple(float(v) for v in b) for b in bands) != _MRD_BANDS:
            raise ValueError("this DiscriminatorR is built for the reference's defaults only: channels=32, hop_factor=0.25 "
                             f"and the five default bands (got {channels}, {hop_factor}, {bands})")
        if not isinstance(window_length, int) or window_length < 256 or window_length > 4096 or window_length & (window_length - 1):
            raise ValueError(f"window_length must be a power of two in [256, 4096], got {window_length!r}")
        self.window_length = window_length
        self.hop_factor = hop_factor
        self.spec_fn = _Spectrogram(window_length)
        n_fft = window_length // 2 + 1
        self.bands = [(int(b[0] * n_fft), int(b[1] * n_fft)) for b in bands]
        convs = lambda: nn.ModuleList([
            weight_norm(nn.Conv2d(2, channels, (3, 9), (1, 1), padding=(1, 4))),
            weight_norm(nn.Conv2d(channels, channels, (3, 9), (1, 2), padding=(1, 4))),
            weight_norm(nn.Conv2d(channels, channels, (3, 9), (1, 2), padding=(1, 4))),
            weight_norm(nn.Conv2d(channels, channels, (3, 9), (1, 2), padding=(1, 4))),
            weight_norm(nn.Conv2d(channels, channels, (3, 3), (1, 1), padding=(1, 1))),
        ])
        self.band_convs = nn.ModuleList([convs() for _ in range(len(self.bands))])
        self.conv_post = weight_norm(nn.Conv2d(channels, 1, (3, 3), (1, 1), padding=(1, 1)))
        self._init_native()
        self._shapes = {}                 # no weights live in the handle: every call passes them

    def _create_handle(self, lib, index):
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_mrd(self.window_length, index, C.byref(h)), "st_create_mrd")
        return h

    def _layers(self):
        return [c for stack in self.band_convs for c in stack] + [self.conv_post]

    def _widths(self) -> List[List[int]]:
        out = []
        for lo, hi in self.bands:
            w = [hi - lo]
            for i in range(1, 5):
                w.append(-(-w[-1] // 2) if i < 4 else w[-1])
            out.append(w)
        return out

    def _call_prep(self, x2: Tensor, backward: bool):
        B, L = x2.shape
        lib, h, stream = self._prepare(x2)
        need = int(lib.st_mrd_workspace_bytes(h, B, L, int(backward)))
        if need == 0:
            raise RuntimeError(f"st_mrd_workspace_bytes refused B = {B}, L = {L}: {lib.st_last_error(h).decode()}")
        ws = torch.empty(need, dtype=torch.uint8, device=x2.device)   # per call: the caching allocator shares it
        _lib.check(lib, h, lib.st_attach_workspace(h, ws.data_ptr(), ws.numel()), "st_attach_workspace")
        return lib, h, stream, ws

    def _forward(self, x2: Tensor, win: Tensor, ws, bs):
        B, L = x2.shape
        T = L // (self.window_length // 4) + 1
        dev = x2.device
        spec = torch.empty((B, 2, T, self.window_length // 2 + 1), device=dev, dtype=torch.float32)
        W = self._widths()
        fm = [torch.empty((B, 32, T, W[k][i]), device=dev, dtype=torch.float32) for k in range(5) for i in range(5)]
        post = torch.empty((B, 1, T, sum(w[4] for w in W)), device=dev, dtype=torch.float32)
        lib, h, stream, work = self._call_prep(x2, False)
        _lib.check(lib, h, lib.st_mrd_forward(h, x2.data_ptr(), B, L, win.data_ptr(), _ptrs(ws), _ptrs(bs), spec.data_ptr(),
                                              _ptrs(fm), post.data_ptr(), stream), "st_mrd_forward")
        del work
        return spec, fm, post

    def _backward(self, x2, win, spec, ws, fm, gpost, gf, need_x: bool, need_w: bool):
        B, L = x2.shape
        W = self._widths()
        T = spec.shape[2]
        gpost = (torch.zeros((B, 1, T, sum(w[4] for w in W)), device=x2.device, dtype=torch.float32) if gpost is None
                 else gpost.contiguous().float())
        gf = [None if g is None else g.contiguous().float() for g in gf]
        gx = torch.empty_like(x2) if need_x else None
        gw = [torch.empty_like(w) for w in ws] if need_w else None
        gb = [torch.empty(w.shape[0], device=w.device, dtype=torch.float32) for w in ws] if need_w else None
        lib, h, stream, work = self._call_prep(x2, True)
        _lib.check(lib, h, lib.st_mrd_backward(h, x2.data_ptr(), B, L, win.data_ptr(), _ptrs(ws), spec.data_ptr(), _ptrs(fm),
                                               gpost.data_ptr(), _ptrs(gf), 0 if gx is None else gx.data_ptr(),
                                               _ptrs(gw) if need_w else None, _ptrs(gb) if need_w else None, stream),
                   "st_mrd_backward")
        del work
        return gx, gw, gb

    def forward(self, x: Tensor) -> Tuple[Tensor, List[Tensor]]:
        if not isinstance(x, torch.Tensor) or x.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError(f"x must be float32, got {x.dtype}")
        if x.ndim != 3 or x.shape[1] != 1 or x.shape[0] == 0:
            raise ValueError(f"x must be (B, 1, L) with B >= 1, got shape {tuple(x.shape)}")
        L = x.shape[-1]
        if L <= self.window_length // 2:
            raise ValueError(f"L = {L} is too short for the centred STFT of window {self.window_length}: L must be above "
                             f"{self.window_length // 2}")
        layers = self._layers()
        ws = [m.weight for m in layers]
        bs = [m.bias for m in layers]
        post, *fmaps = _MRDFunction.apply(x, self, self.spec_fn.window, *ws, *bs)
        return post, fmaps + [post]


class MultiResolutionDiscriminator(nn.Module):
    """models/discriminator.py::MultiResolutionDiscriminator: one DiscriminatorR per window length, each run on y then
    y_hat."""

    def __init__(self, fft_sizes: Tuple[int, ...] = (2048, 1024, 512)):
        super().__init__()
        self.discriminators = nn.ModuleList([DiscriminatorR(window_length=w) for w in fft_sizes])

    def set_engine(self, name: str) -> None:
        for d in self.discriminators:
            d.set_engine(name)

    def forward(self, y: Tensor, y_hat: Tensor):
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
        for d in self.discriminators:
            y_d_r, fmap_r = d(x=y)
            y_d_g, fmap_g = d(x=y_hat)
            y_d_rs.append(y_d_r)
            fmap_rs.append(fmap_r)
            y_d_gs.append(y_d_g)
            fmap_gs.append(fmap_g)
        return y_d_rs, y_d_gs, fmap_rs, fmap_gs
