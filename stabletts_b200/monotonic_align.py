"""Drop-in for the reference's ``monotonic_align`` package (monotonic_align/__init__.py, core.py): monotonic alignment
search on the GPU (SURVEY.md §8 row f8).  The reference copies ``neg_cent`` to the host, runs a one-thread numba dynamic
program utterance after utterance and copies the path back; here the whole search runs in ``st_maximum_path`` on the
tensor's own device with no host read, so it can be captured in a CUDA graph.  The path is bit for bit the reference's.

One line in the reference's ``models/model.py`` swaps it in:

    from stabletts_b200 import monotonic_align          # was: import monotonic_align

The reference calls it under ``torch.no_grad()`` (model.py:149-158), so autograd never sees it and its own DDP training
loop runs unchanged.
"""
from __future__ import annotations

import torch

from . import _lib


def _require_cuda(t, what):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise RuntimeError(f"{what}: stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")


def workspace(B: int, Ty: int, Tx: int, device) -> torch.Tensor:
    """The scratch buffer of st_maximum_path / st_mas_losses for a (B, Ty, Tx) problem."""
    lib = _lib.load_library()
    return torch.empty(max(int(lib.st_mas_workspace_bytes(B, Ty, Tx)), 1), device=device, dtype=torch.uint8)


def scores(y: torch.Tensor, mu_x: torch.Tensor) -> torch.Tensor:
    """``neg_cent`` of models/model.py:150-155: y (B, D, T_y), mu_x (B, D, T_x) -> (B, T_y, T_x) fp32 (st_mas_scores)."""
    _require_cuda(y, "mas scores")
    B, D, Ty = y.shape
    Tx = mu_x.shape[2]
    if tuple(mu_x.shape) != (B, D, Tx) or mu_x.device != y.device:
        raise ValueError(f"mu_x must be (B, D, T_x) = ({B}, {D}, T_x) on {y.device}, got {tuple(mu_x.shape)} on {mu_x.device}")
    y_ = y.detach().to(torch.float32).contiguous()
    mu_ = mu_x.detach().to(torch.float32).contiguous()
    out = torch.empty(B, Ty, Tx, device=y.device, dtype=torch.float32)
    lib = _lib.load_library()
    stream = torch.cuda.current_stream(y.device).cuda_stream
    _lib.check(lib, None, lib.st_mas_scores(y_.data_ptr(), mu_.data_ptr(), out.data_ptr(), B, D, Ty, Tx, stream), "st_mas_scores")
    return out


def search(neg_cent: torch.Tensor, mask: torch.Tensor | None = None, x_lengths: torch.Tensor | None = None,
           y_lengths: torch.Tensor | None = None, want_path: bool = True, ws: torch.Tensor | None = None):
    """st_maximum_path on fp32 contiguous ``neg_cent`` (B, T_y, T_x), lengths from ``mask`` or from the int64 length
    vectors.  Returns (path (B, T_y, T_x) fp32 or None, dur (B, T_x) fp32, cum (B, T_x) fp32)."""
    B, Ty, Tx = neg_cent.shape
    dev = neg_cent.device
    path = torch.empty(B, Ty, Tx, device=dev, dtype=torch.float32) if want_path else None
    dur = torch.empty(B, Tx, device=dev, dtype=torch.float32)
    cum = torch.empty(B, Tx, device=dev, dtype=torch.float32)
    if ws is None:
        ws = workspace(B, Ty, Tx, dev)
    lib = _lib.load_library()
    stream = torch.cuda.current_stream(dev).cuda_stream
    ptr = lambda t: None if t is None else t.data_ptr()
    _lib.check(lib, None, lib.st_maximum_path(neg_cent.data_ptr(), ptr(mask), ptr(x_lengths), ptr(y_lengths), ptr(path), dur.data_ptr(),
                                              cum.data_ptr(), ws.data_ptr(), ws.numel(), B, Ty, Tx, stream), "st_maximum_path")
    return path, dur, cum


def maximum_path(neg_cent: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """monotonic_align/__init__.py:7-16.  neg_cent, mask: (B, T_y, T_x) on one CUDA device, any float dtype and any
    strides (fp16 / bf16 scores are widened to fp32 exactly, as the reference's ``astype(float32)`` does).  Returns the
    0/1 path in ``neg_cent``'s dtype on its device.  The lengths are t_y = (int) Σ mask[b, :, 0] and
    t_x = (int) Σ mask[b, 0, :], summed on the device (exactly, for any 0/1 mask).  A mask whose row 0 is empty while
    its column 0 is not (t_x = 0 < t_y; no product of two prefix masks gives one) makes the reference read out of
    bounds: here that utterance's path is all zeros."""
    if neg_cent.dim() != 3 or tuple(mask.shape) != tuple(neg_cent.shape):
        raise ValueError(f"neg_cent and mask must both be (B, T_y, T_x); got {tuple(neg_cent.shape)} and {tuple(mask.shape)}")
    _require_cuda(neg_cent, "maximum_path")
    _require_cuda(mask, "maximum_path")
    if mask.device != neg_cent.device:
        raise ValueError(f"mask is on {mask.device}, neg_cent on {neg_cent.device}")
    if not neg_cent.is_floating_point():
        raise ValueError(f"neg_cent must be a floating-point tensor, got {neg_cent.dtype}")
    B, Ty, Tx = neg_cent.shape
    if B * Ty * Tx == 0:
        return torch.zeros_like(neg_cent)
    nc = neg_cent.detach().to(torch.float32).contiguous()
    m = mask.detach().to(torch.float32).contiguous()
    path, _, _ = search(nc, mask=m)
    return path if neg_cent.dtype == torch.float32 else path.to(neg_cent.dtype)


def losses(y, mu_y, y_mask, logw, x_mask, dur, x_lengths, ws):
    """st_mas_losses: (prior_loss, dur_loss) as fp32 device scalars (models/model.py:162-163, 175-176)."""
    B, M, Ty = y.shape
    Tx = logw.shape[-1]
    prior = torch.empty((), device=y.device, dtype=torch.float32)
    dur_loss = torch.empty((), device=y.device, dtype=torch.float32)
    lib = _lib.load_library()
    stream = torch.cuda.current_stream(y.device).cuda_stream
    _lib.check(lib, None, lib.st_mas_losses(y.data_ptr(), mu_y.data_ptr(), y_mask.data_ptr(), logw.data_ptr(), x_mask.data_ptr(),
                                            dur.data_ptr(), x_lengths.data_ptr(), ws.data_ptr(), ws.numel(), B, M, Ty, Tx,
                                            prior.data_ptr(), dur_loss.data_ptr(), stream), "st_mas_losses")
    return prior, dur_loss
