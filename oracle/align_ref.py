"""CPU oracle for the caller-side glue of the path (TEST INFRASTRUCTURE ONLY): duration ->
alignment -> mu_y inside ``StableTTS.synthesise`` (models/model.py:81-95) with ``generate_path``
(models/model.py:17-27) and ``sequence_mask`` (utils/mask.py:4-8), restated functionally.

Pinned by tests/test_align.py: against tests/golden/align_*.npz generated from the reference's own
``generate_path`` / ``sequence_mask``.
"""
from __future__ import annotations

import torch


def sequence_mask(length: torch.Tensor, max_length=None) -> torch.Tensor:
    """utils/mask.py:4-8."""
    if max_length is None:
        max_length = length.max()
    x = torch.arange(max_length, dtype=length.dtype, device=length.device)
    return x.unsqueeze(0) < length.unsqueeze(1)


def generate_path(duration: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """models/model.py:17-27.  duration (B, T_x), mask (B, T_x, T_y) -> 0/1 path (B, T_x, T_y)."""
    b, t_x, t_y = mask.shape
    cum = torch.cumsum(duration, 1)
    path = sequence_mask(cum.view(b * t_x), t_y).to(mask.dtype).view(b, t_x, t_y)
    path = path - torch.nn.functional.pad(path, (0, 0, 1, 0, 0, 0))[:, :-1]
    return path * mask


def expand_by_durations(logw: torch.Tensor, x_mask: torch.Tensor, mu_x: torch.Tensor, length_scale: float = 1.0, exp=torch.exp):
    """models/model.py:83-95.  logw, x_mask (B,1,T_x); mu_x (B,M,T_x) -> mu_y (B,M,T_y), y_mask (B,1,T_y),
    y_lengths (B,), attn (B,1,T_x,T_y).  `exp` evaluates exp(logw) (e.g. on the device the reference would run on)."""
    w = exp(logw) * x_mask
    w_ceil = torch.ceil(w) * length_scale
    y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()
    y_max_length = y_lengths.max()
    y_mask = sequence_mask(y_lengths, y_max_length).unsqueeze(1).to(x_mask.dtype)
    attn_mask = x_mask.unsqueeze(-1) * y_mask.unsqueeze(2)
    attn = generate_path(w_ceil.squeeze(1), attn_mask.squeeze(1)).unsqueeze(1)
    mu_y = torch.matmul(attn.squeeze(1).transpose(1, 2), mu_x.transpose(1, 2)).transpose(1, 2)
    return mu_y, y_mask, y_lengths, attn


def make_align_inputs(seed: int, B: int, Tx: int, M: int, lens=None):
    g = torch.Generator().manual_seed(seed)
    lens = torch.as_tensor(lens if lens is not None else [Tx] * B)
    x_mask = (torch.arange(Tx)[None] < lens[:, None]).float().unsqueeze(1)
    logw = torch.randn(B, 1, Tx, generator=g) * 0.7 + 0.5           # durations ~ 1..6 frames
    mu_x = torch.randn(B, M, Tx, generator=g) * x_mask
    return logw * x_mask, x_mask, mu_x


ALIGN_CASES = {
    "align_basic":   dict(seed=41, B=3, Tx=37, M=80, lens=[37, 21, 5], length_scale=1.0),
    "align_scale":   dict(seed=42, B=2, Tx=64, M=128, lens=[64, 40], length_scale=1.5),
    "align_single":  dict(seed=43, B=1, Tx=1, M=80, lens=[1], length_scale=1.0),
    "align_empty":   dict(seed=44, B=2, Tx=9, M=16, lens=[9, 0], length_scale=1.0),
    "align_long":    dict(seed=45, B=2, Tx=129, M=80, lens=[129, 100], length_scale=1.0),
}
