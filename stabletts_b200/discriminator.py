"""Drop-ins for the Vocos training discriminator, ``vocoders/vocos/models/discriminator.py``: ``MultiPeriodDiscriminator``
and ``DiscriminatorP`` (train.py runs it on real and generated audio in both half-steps).

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
