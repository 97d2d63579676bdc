"""Duration -> alignment -> ``mu_y`` expansion: the caller-side glue of the CFM path inside
``StableTTS.synthesise`` (models/model.py:81-95, ``generate_path`` :17-27) as two small CUDA kernels
(SURVEY.md §8 row f1).  The reference builds a dense (B, T_x, T_y) path and multiplies; here the path
is never materialised unless the caller asks for ``attn`` back.

    mu_y, y_mask, y_lengths, attn = expand_by_durations(logw, x_mask, mu_x, length_scale)

``max_length=None`` reproduces the reference (one host read of ``y_lengths.max()``, model.py:86);
passing ``max_length`` keeps the whole thing device-resident (outputs padded to that length).
"""
from __future__ import annotations

import torch

from . import _lib


def expand_by_durations(logw: torch.Tensor, x_mask: torch.Tensor, mu_x: torch.Tensor, length_scale: float = 1.0,
                        max_length: int | None = None, return_attn: bool = False):
    """logw, x_mask: (B, 1, T_x); mu_x: (B, M, T_x), all CUDA fp32.
    Returns mu_y (B, M, T_y), y_mask (B, 1, T_y), y_lengths (B,) int64, attn (B, 1, T_x, T_y) or None."""
    if logw.device.type != "cuda":
        raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
    lib = _lib.load_library()
    B, M, Tx = mu_x.shape
    logw_ = logw.detach().float().reshape(B, Tx).contiguous()
    mask_ = x_mask.detach().float().reshape(B, Tx).contiguous()
    mu_ = mu_x.detach().float().contiguous()
    stream = torch.cuda.current_stream(mu_x.device).cuda_stream
    cum = torch.empty(B, Tx, device=mu_x.device, dtype=torch.float32)
    y_lengths = torch.empty(B, device=mu_x.device, dtype=torch.int64)
    _lib.check(lib, None, lib.st_align_lengths(logw_.data_ptr(), mask_.data_ptr(), float(length_scale), B, Tx, cum.data_ptr(),
                                               y_lengths.data_ptr(), stream), "st_align_lengths")
    Ty = int(y_lengths.max()) if max_length is None else int(max_length)           # models/model.py:86 (host read)
    mu_y = torch.empty(B, M, Ty, device=mu_x.device, dtype=torch.float32)
    y_mask = torch.empty(B, 1, Ty, device=mu_x.device, dtype=torch.float32)
    attn = torch.empty(B, 1, Tx, Ty, device=mu_x.device, dtype=torch.float32) if return_attn else None
    _lib.check(lib, None, lib.st_align_expand(mu_.data_ptr(), mask_.data_ptr(), cum.data_ptr(), y_lengths.data_ptr(), B, M, Tx, Ty,
                                              mu_y.data_ptr(), y_mask.data_ptr(), None if attn is None else attn.data_ptr(), stream),
               "st_align_expand")
    return mu_y, y_mask, y_lengths, attn
