"""CPU oracle of the multi-scale mel loss (TEST INFRASTRUCTURE ONLY): a float64 restatement of vocoders/vocos/models/loss.py's
MultiScaleMelSpectrogramLoss with its gradient written out as an explicit adjoint, plus the seeded fixture cases.  Pinned by
tests/test_mel_loss.py against tests/golden/mlw_*.npz (recipe oracle/make_golden_mel_loss.py, the unmodified reference)
and against torch autograd of the same float64 forward.

Per scale s (n_fft N, hop N / 4, pad 3N / 8, filters fb (N/2 + 1, m)), for one frame of y:
    g_m = −sgn(Δ_m) / (B m T) · [mel_m >= 1e-5] / mel_m,  Δ = log-mel(x) − log-mel(y), mel_m the pre-log filter sum
    G_k = Σ_m fb[k, m] g_m,  Y_k = G_k X_k / |X_k|,  |X_k| = sqrt(re² + im² + 1e-6)
    d_n = w_n Re Σ_{k=0}^{N/2} Y_k e^{+2πikn/N}
then overlap-add of the frames and the adjoint of the reflect padding.  `signs` and `clamps` replace sgn(Δ) and the clamp
masks (per scale, (B, T, m)), so a test can take them from another implementation's log-mels."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import mel_ref as M

N_MELS = [5, 10, 20, 40, 80, 160, 320]
WINDOWS = [32, 64, 128, 256, 512, 1024, 2048]


def scale_config(n_mels, n_fft):
    """asdict(MelConfig(n_mels=n_mels, n_fft=n_fft, win_length=n_fft, hop_length=n_fft // 4)): pad = (n_fft - hop) // 2."""
    return M.mel_config(n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels)


MULTI = [scale_config(m, w) for m, w in zip(N_MELS, WINDOWS)]
SINGLE = [M.mel_config()]


def _frames(wav, cfg):
    """(B, L) -> reflect-padded frames (B, T, N) and each frame sample's input index (T, N)."""
    N, hop, pad = cfg["n_fft"], cfg["hop_length"], cfg["pad"]
    L = wav.shape[-1]
    xp = F.pad(wav.unsqueeze(1), (pad, pad), "reflect").squeeze(1)
    fr = xp.unfold(-1, N, hop)
    T = fr.shape[1]
    s = (torch.arange(T)[:, None] * hop + torch.arange(N)[None, :]) - pad
    s = torch.where(s < 0, -s, s)
    s = torch.where(s >= L, 2 * (L - 1) - s, s)
    return fr, s


def _scale_forward(wav, window, fb, cfg):
    """(X (B, T, K) complex, |X| (B, T, K), mel (B, T, m) before the log)"""
    fr, _ = _frames(wav, cfg)
    X = torch.fft.rfft(fr * window, dim=-1)
    mag = torch.sqrt(X.real ** 2 + X.imag ** 2 + 1e-6)
    return X, mag, mag @ fb


def log_mels(wav, windows, fbs, cfgs):
    """[(B, n_mels, T)] per scale, float64: the reference's LogMelSpectrogram outputs."""
    wav = wav.double().reshape(wav.shape[0], -1)
    return [torch.log(torch.clamp(_scale_forward(wav, w.double(), fb.double(), c)[2], min=1e-5)).transpose(1, 2)
            for w, fb, c in zip(windows, fbs, cfgs)]


def loss(x, y, windows, fbs, cfgs):
    """Σ_s mean |mel_s(x) − mel_s(y)| in float64 (a 0-dim tensor; differentiable)."""
    lx, ly = log_mels(x, windows, fbs, cfgs), log_mels(y, windows, fbs, cfgs)
    return sum((a - b).abs().mean() for a, b in zip(lx, ly))


def frame_adjoint(g, X, mag, window, fb):
    """g (B, T, m), the gradient at the filter sums -> the gradient at each frame's input samples (B, T, N)."""
    N = window.shape[0]
    G = g @ fb.T                                                              # (B, T, K)
    Y = G / mag * X
    k = torch.arange(N // 2 + 1, dtype=torch.float64)
    n = torch.arange(N, dtype=torch.float64)
    E = torch.exp(1j * 2 * math.pi * k[:, None] * n[None, :] / N)          # e^{+2 pi i k n / N}, (K, N)
    return (Y @ E).real * window


def scatter_frames(d, idx, L):
    """The adjoint of framing + reflect padding: (B, T, N) frame gradients onto (B, L), every sample its own sum."""
    B = d.shape[0]
    out = torch.zeros(B, L, dtype=torch.float64)
    out.index_add_(1, idx.reshape(-1), d.reshape(B, -1))
    return out


def gradients(x, y, windows, fbs, cfgs, signs=None, clamps_x=None, clamps_y=None):
    """(loss, d loss / dx, d loss / dy) in float64 by the explicit adjoint.  signs[s]: sgn(Δ) of scale s, (B, T, m);
    clamps_x[s] / clamps_y[s]: the masks [mel >= 1e-5]; None computes them from this oracle's own float64 log-mels."""
    x = x.double().reshape(x.shape[0], -1)
    y = y.double().reshape(y.shape[0], -1)
    B, L = x.shape
    total = torch.zeros((), dtype=torch.float64)
    gx, gy = torch.zeros_like(x), torch.zeros_like(y)
    for s, (w, fb, c) in enumerate(zip(windows, fbs, cfgs)):
        w, fb = w.double(), fb.double()
        Xx, mx_mag, mx = _scale_forward(x, w, fb, c)
        Xy, my_mag, my = _scale_forward(y, w, fb, c)
        delta = torch.log(torch.clamp(mx, min=1e-5)) - torch.log(torch.clamp(my, min=1e-5))
        total = total + delta.abs().mean()
        sg = torch.sign(delta) if signs is None else signs[s].double()
        cx = (mx >= 1e-5) if clamps_x is None else clamps_x[s]
        cy = (my >= 1e-5) if clamps_y is None else clamps_y[s]
        n = delta.numel()
        g_x = torch.where(cx, sg / n / mx, torch.zeros_like(mx))
        g_y = torch.where(cy, -sg / n / my, torch.zeros_like(my))
        _, idx = _frames(x, c)
        gx += scatter_frames(frame_adjoint(g_x, Xx, mx_mag, w, fb), idx, L)
        gy += scatter_frames(frame_adjoint(g_y, Xy, my_mag, w, fb), idx, L)
    return total, gx, gy


def flip_bound(y, deltas, windows, fbs, cfgs, tol=1e-4):
    """Σ over the cells with |Δ| <= tol of 2 ‖∂(Δ / n_s)/∂y‖₂: the most that sgn(Δ) decided differently at those cells can
    move d loss / dy (float64).  deltas: [(B, T, m)] per scale."""
    y = y.double().reshape(y.shape[0], -1)
    L = y.shape[-1]
    bound = 0.0
    for d, w, fb, c in zip(deltas, windows, fbs, cfgs):
        w, fb = w.double(), fb.double()
        X, mag, mel = _scale_forward(y, w, fb, c)
        _, idx = _frames(y, c)
        sel = (d.abs() <= tol).nonzero()                                         # (E, 3): b, t, m
        for chunk in sel.split(4096):
            b, t, m = chunk[:, 0], chunk[:, 1], chunk[:, 2]
            mm = mel[b, t, m]
            g = torch.zeros(len(chunk), 1, fb.shape[1], dtype=torch.float64)
            g[torch.arange(len(chunk)), 0, m] = torch.where(mm >= 1e-5, 1.0 / mm, torch.zeros_like(mm)) / d.numel()
            rows = frame_adjoint(g, X[b, t][:, None], mag[b, t][:, None], w, fb)[:, 0]    # (E, N)
            pos = idx[t]                                                               # input index of each frame sample
            local = pos - pos.min(dim=1, keepdim=True).values
            acc = torch.zeros_like(rows).scatter_add_(1, local, rows)                # reflect images of one sample merged
            bound += float(2 * acc.norm(dim=1).sum())
    return bound


# ---- the fixture cases (waveforms from mel_ref's seeded generators; L = 20480 is TrainConfig.segment_size) --------------
def make_pair(case):
    L, B, seed = case["L"], case["B"], case["seed"]
    g = torch.Generator().manual_seed(seed + 1000)
    x = M.make_batch([case["kind"]] * B, seed, L)
    y = x + case["noise"] * torch.randn(B, L, generator=g)
    for r in case.get("half_rows", []):
        y[r] = 0.5 * x[r]
    for r in case.get("equal_rows", []):
        y[r] = x[r]
    return x, y.float()


CASES = {
    "mlw_b2_segment": dict(scales="multi", B=2, L=20480, kind="speech", seed=401, noise=0.02),
    "mlw_b3_half":    dict(scales="multi", B=3, L=8192, kind="noise", seed=402, noise=0.02, half_rows=[1]),
    "mlw_equal_row":  dict(scales="multi", B=2, L=8192, kind="lowpass", seed=403, noise=0.05, equal_rows=[0], grad_x=True),
    "mlw_quiet":      dict(scales="multi", B=2, L=8192, kind="silence", seed=404, noise=1e-5),
    "mlw_shortest":   dict(scales="multi", B=2, L=769, kind="noise", seed=405, noise=0.05),   # pad + 1 at n_fft 2048
    "mlw_single":     dict(scales="single", B=2, L=8192, kind="speech", seed=406, noise=0.02),
}


def scale_configs(case):
    return MULTI if case["scales"] == "multi" else SINGLE


def hann_windows(cfgs):
    return [torch.hann_window(c["n_fft"]) for c in cfgs]
