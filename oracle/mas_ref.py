"""CPU oracle of monotonic alignment search and of StableTTS's training-forward losses (TEST INFRASTRUCTURE ONLY).

``maximum_path`` restates monotonic_align/core.py's dynamic program row-parallel and vectorised over the batch, in numpy
fp32: row y is a function of row y-1 alone, so every band cell of a row is updated at once with the reference's own
operations (value += (v_cur > v_prev ? v_cur : v_prev), one fp32 add; the strict comparison in the backtrack; row -1
read as the last padded row).  It returns the value matrix too, so the fixtures can state their margins.
``neg_cent64`` is the fp64 statement of models/model.py:150-155, and ``forward_losses`` composes the value of the training
``forward`` (models/model.py:114-178, eval mode) from the encoder oracles of synth_ref.  Pinned by tests/test_mas.py against
tests/golden/mas_*.npz and fwd_*.npz (oracle/make_golden_mas.py, unmodified reference)."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import duration_ref, estimator_ref, style_ref, text_encoder_ref
from oracle.synth_ref import sub

NEG = np.float32(-1e9)


def lengths_from_mask(mask: np.ndarray):
    """t_y = (int) Σ_y mask[b, y, 0], t_x = (int) Σ_x mask[b, 0, x] (monotonic_align/__init__.py:13-14)."""
    m = np.asarray(mask, dtype=np.float64)
    return m[:, :, 0].sum(1).astype(np.int64), m[:, 0, :].sum(1).astype(np.int64)


def maximum_path(neg_cent, mask=None, t_y=None, t_x=None, return_value=False):
    """neg_cent (B, T_y, T_x) -> 0/1 int32 path of the same shape (and the DP's value matrix).  Lengths from ``mask`` or
    given.  t_x == 0 < t_y (the reference reads out of bounds) gives an all-zero path, as the CUDA kernel does."""
    value = np.array(neg_cent, dtype=np.float32, copy=True)
    B, Ty, Tx = value.shape
    if mask is not None:
        t_y, t_x = lengths_from_mask(mask)
    t_y, t_x = np.asarray(t_y, dtype=np.int64), np.asarray(t_x, dtype=np.int64)
    xs = np.arange(Tx)
    for y in range(Ty):
        lo = np.maximum(0, t_x + y - t_y)[:, None]
        hi = np.minimum(t_x, y + 1)[:, None]
        band = (xs[None] >= lo) & (xs[None] < hi)
        if not band.any():
            continue
        prev = value[:, y - 1, :] if y > 0 else np.zeros((B, Tx), np.float32)
        v_cur = np.where(xs[None] == y, NEG, prev)
        shifted = np.concatenate([np.zeros((B, 1), np.float32), prev[:, :-1]], axis=1)
        v_prev = np.where(xs[None] == 0, np.float32(0.0) if y == 0 else NEG, shifted)
        with np.errstate(invalid="ignore"):
            m = np.where(v_cur > v_prev, v_cur, v_prev).astype(np.float32)
        value[:, y, :] = np.where(band, value[:, y, :] + m, value[:, y, :])
    path = np.zeros((B, Ty, Tx), np.int32)
    index = t_x - 1
    bi = np.arange(B)
    live = (t_x >= 1)
    for y in range(Ty - 1, -1, -1):
        on = live & (y < t_y)
        path[bi[on], y, index[on]] = 1
        i = np.clip(index, 1, max(Tx - 1, 1)) if Tx > 1 else np.zeros_like(index)
        with np.errstate(invalid="ignore"):
            less = value[bi, y - 1, i] < value[bi, y - 1, np.maximum(i - 1, 0)]
        dec = on & (index != 0) & ((index == y) | less)
        index = index - dec.astype(np.int64)
    return (path, value) if return_value else path


def backtrack_gap(value, path, t_y):
    """Per utterance: the smallest |value[y-1, i] - value[y-1, i-1]| over the backtrack's comparisons along the chosen
    path (rows where i != 0 and i != y), i.e. how far the scores could move before the path changes (inf: none made)."""
    gaps = []
    for b in range(path.shape[0]):
        g = math.inf
        for y in range(1, int(t_y[b])):
            i = int(np.argmax(path[b, y]))
            if i != 0 and i != y:
                g = min(g, abs(float(value[b, y - 1, i]) - float(value[b, y - 1, i - 1])))
        gaps.append(g)
    return np.array(gaps)


def neg_cent64(y: torch.Tensor, mu_x: torch.Tensor) -> torch.Tensor:
    """models/model.py:150-155 in fp64: y (B, D, T_y), mu_x (B, D, T_x) -> (B, T_y, T_x)."""
    y, mu = y.double(), mu_x.double()
    D = y.shape[1]
    return (-0.5 * math.log(2 * math.pi) * D - 0.5 * (y * y).sum(1)[:, :, None] + torch.einsum("bdt,bds->bts", y, mu)
            - 0.5 * (mu * mu).sum(1)[:, None, :])


def sequence_mask(lengths, T):
    return (torch.arange(T)[None] < torch.as_tensor(lengths)[:, None]).float()


def forward_losses(state, ids, x_lengths, y, y_lengths, z, z_lengths, u_cfg, u_t, noise, cfg_dropout=0.2):
    """The value of models/model.py:114-178 in eval mode with its three random draws passed in: ``u_cfg`` (B, 1) behind the
    cfg dropout mask (:138), ``u_t`` (B, 1, 1) and ``noise`` (B, n_mel, T_y) behind compute_loss's t and z.
    Returns (dur_loss, diff_loss, prior_loss, attn (B, T_x, T_y)) and, for the fixtures' margins, (neg_cent, mask)."""
    with torch.inference_mode():
        B, M, Ty = y.shape
        keep = u_cfg > cfg_dropout
        z_mask = sequence_mask(z_lengths, z.shape[2]).unsqueeze(1)
        c = style_ref.style_forward(sub(state, "ref_encoder."), z, z_mask) * keep + ~keep * state["fake_speaker"].repeat(B, 1)
        x, mu_x, x_mask = text_encoder_ref.text_encoder_forward(sub(state, "encoder."), ids, c, x_lengths)
        logw = duration_ref.dp_forward(sub(state, "dp."), x, x_mask, c)
        y_mask = sequence_mask(y_lengths, Ty)
        nc = neg_cent64(y, mu_x).float()
        mask = x_mask[:, 0, None, :] * y_mask[:, :, None]
        path = torch.from_numpy(maximum_path(nc.numpy(), mask.numpy())).float()          # (B, T_y, T_x)
        d = path.sum(1, keepdim=True)                                                    # (B, 1, T_x)
        dur_loss = ((logw - torch.log(1e-8 + d) * x_mask) ** 2).double().sum() / torch.as_tensor(x_lengths).sum()
        mu_y = torch.einsum("bts,bds->bdt", path.double(), mu_x.double()).float()
        prior = (0.5 * ((y - mu_y) ** 2 + math.log(2 * math.pi)) * y_mask[:, None]).double().sum() / (y_mask.double().sum() * M)
        k = keep[:, :, None]
        mu_y_masked = mu_y * k + ~k * state["fake_content"].repeat(B, 1, Ty)
        diff, _ = estimator_ref.cfm_loss(sub(state, "decoder.estimator."), y, y_mask[:, None], mu_y_masked, c, u_t, noise)
    return (float(dur_loss), float(diff), float(prior), path.transpose(1, 2)), (nc, mask)
