"""Float64 restatement of the Vocos multi-resolution discriminator (vocoders/vocos/models/discriminator.py:78-171) and of
the packings its CUDA path uses (stabletts_b200/csrc/mrd_api.cu, mrd.cuh).  Test-side only: nothing under stabletts_b200/
imports it.

``discriminator_r`` follows DiscriminatorR: the complex spectrogram (lines 142-154: torchaudio Spectrogram(n_fft = N,
hop = N / 4, power=None) is torch.stft with center=True, reflect padding, the given window, normalized=False, onesided;
view_as_real, permute(0, 3, 2, 1)), the band split (line 153), five convs per band with leaky ReLU 0.1 (lines 160-166),
conv_post over the concatenated bands (lines 167-169).  ``masks`` replaces each leaky ReLU's sign test by a given pattern
(True = slope 1), so a backward can be taken with another implementation's activation signs."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle.mpd_ref import checksums, fixture_quantities, seeded, upstream_loss, weight_norm  # noqa: F401

FFT_SIZES = (2048, 1024, 512)
BANDS = ((0.0, 0.1), (0.1, 0.25), (0.25, 0.5), (0.5, 0.75), (0.75, 1.0))
SLOPE = 0.1


def band_edges(N: int) -> List[Tuple[int, int]]:
    F_ = N // 2 + 1
    return [(int(a * F_), int(b * F_)) for a, b in BANDS]


def effective_params(sd: Dict[str, torch.Tensor], prefix: str = "") -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """(weight, bias) of band_convs.k.i (index 5 k + i) and conv_post (index 25) from a DiscriminatorR state_dict."""
    out = []
    for name in [f"band_convs.{k}.{i}" for k in range(5) for i in range(5)] + ["conv_post"]:
        p = prefix + name
        out.append((weight_norm(sd[p + ".parametrizations.weight.original0"], sd[p + ".parametrizations.weight.original1"]),
                    sd[p + ".bias"]))
    return out


def spectrogram(x: torch.Tensor, window: torch.Tensor, N: int) -> torch.Tensor:
    """(B, 1, L) -> (B, 2, T', N / 2 + 1)."""
    X = torch.stft(x.squeeze(1), N, hop_length=N // 4, win_length=N, window=window.to(x.dtype), center=True,
                   pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
    return torch.view_as_real(X).permute(0, 3, 2, 1)


def discriminator_r(x, window, params, N: int, masks: Optional[List[torch.Tensor]] = None):
    """-> (score, fmaps (the reference's 21: convs 1-4 of each band, then the score), pre-activations of the 25 band convs)."""
    spec = spectrogram(x, window, N)
    fmaps, pres, outs = [], [], []
    for k, (lo, hi) in enumerate(band_edges(N)):
        h = spec[..., lo:hi]
        for i in range(5):
            w, b = params[5 * k + i]
            z = F.conv2d(h, w, b, stride=(1, 2) if 1 <= i <= 3 else 1, padding=(1, 4) if i < 4 else (1, 1))
            pres.append(z)
            pos = (z > 0) if masks is None else masks[5 * k + i]
            h = torch.where(pos, z, SLOPE * z)
            if i > 0:
                fmaps.append(h)
        outs.append(h)
    w, b = params[25]
    post = F.conv2d(torch.cat(outs, dim=-1), w, b, padding=(1, 1))
    fmaps.append(post)
    return post, fmaps, pres


# ---------------------------------------------------------------- packing identities (mrd_api.cu) --------------------------
# One band activation X (B, C, T', W); rows (B T', G, lanes 3 C): channel (l 3 + dt) C + c of group g of sequence b T' + t
# is X[b, c, t + dt - 1, lanes g + l], zero outside.

def conv_band(X: torch.Tensor, Wt: torch.Tensor, lanes: int) -> torch.Tensor:
    """Direct statement: the reference's layer, (3, 9) stride (1, 2) pad (1, 4) (lanes 2) or (3, 3) pad (1, 1) (lanes 1)."""
    return F.conv2d(X, Wt, stride=(1, 2) if lanes == 2 else 1, padding=(1, 4) if lanes == 2 else (1, 1))


def expand(X: torch.Tensor, lanes: int) -> torch.Tensor:
    B, C, T, W = X.shape
    G = -(-W // lanes)
    Xp = torch.zeros(B, C, T + 2, lanes * G, dtype=X.dtype)
    Xp[:, :, 1:T + 1, :W] = X
    R = torch.zeros(B, T, G, lanes, 3, C, dtype=X.dtype)
    for dt in range(3):
        v = Xp[:, :, dt:dt + T, :].reshape(B, C, T, G, lanes)            # [b, c, t, g, l] = X[b, c, t + dt - 1, lanes g + l]
        R[:, :, :, :, dt, :] = v.permute(0, 2, 3, 4, 1)
    return R.reshape(B * T, G, lanes * 3 * C)


def taps_of(lanes: int) -> int:
    return 5 if lanes == 2 else 3


def pack_fwd(Wt: torch.Tensor, lanes: int) -> torch.Tensor:
    """[taps][C_out][lanes 3 C_in]: tap t, channel (l, dt, c) = Wt[n, c, dt, lanes t + l], zero past the kernel."""
    Co, Ci, _, kw = Wt.shape
    taps = taps_of(lanes)
    P = torch.zeros(taps, Co, lanes, 3, Ci, dtype=Wt.dtype)
    for t in range(taps):
        for l in range(lanes):
            k = lanes * t + l
            if k < kw:
                P[t, :, l] = Wt[:, :, :, k].permute(0, 2, 1)
    return P.reshape(taps, Co, lanes * 3 * Ci)


def pack_dgrad(Wt: torch.Tensor, lanes: int) -> torch.Tensor:
    """[taps][lanes 3 C_in][C_out]: the forward's taps flipped and transposed."""
    return pack_fwd(Wt, lanes).flip(0).transpose(1, 2).contiguous()


def engine_conv(A: torch.Tensor, Wp: torch.Tensor) -> torch.Tensor:
    """The conv-GEMM engine's contract, batched: out[bb, o, n] = Σ_{tap, k} A[bb, o + tap - taps // 2, k] Wp[tap, n, k]."""
    taps, G = Wp.shape[0], A.shape[1]
    out = torch.zeros(A.shape[0], G, Wp.shape[1], dtype=A.dtype)
    for tap in range(taps):
        sh = tap - taps // 2
        src = torch.zeros_like(A)
        lo, hi = max(0, -sh), min(G, G - sh)
        if hi > lo:
            src[:, lo:hi] = A[:, lo + sh:hi + sh]
        out += src @ Wp[tap].t()
    return out


def rows_to_nchw(Y: torch.Tensor, B: int, T: int) -> torch.Tensor:
    BB, G, C = Y.shape
    return Y.reshape(B, T, G, C).permute(0, 3, 1, 2)


def nchw_to_rows(Z: torch.Tensor) -> torch.Tensor:
    B, C, T, G = Z.shape
    return Z.permute(0, 2, 3, 1).reshape(B * T, G, C)


def fold(dR: torch.Tensor, B: int, C: int, T: int, W: int, lanes: int) -> torch.Tensor:
    """The adjoint of expand: dX[b, c, t, w] = Σ_dt dR[b T + t - dt + 1, w / lanes, ((w % lanes) 3 + dt) C + c]."""
    G = dR.shape[1]
    R = dR.reshape(B, T, G, lanes, 3, C)
    dX = torch.zeros(B, C, T + 2, lanes * G, dtype=dR.dtype)
    for dt in range(3):
        dX[:, :, dt:dt + T, :] += R[:, :, :, :, dt, :].permute(0, 4, 1, 2, 3).reshape(B, C, T, lanes * G)
    return dX[:, :, 1:T + 1, :W]


def forward_engine(X, Wt, b, lanes):
    B, _, T, _ = X.shape
    return rows_to_nchw(engine_conv(expand(X, lanes), pack_fwd(Wt, lanes)), B, T) + b.view(1, -1, 1, 1)


def dgrad_engine(dZ, Wt, W, lanes):
    B, _, T, _ = dZ.shape
    return fold(engine_conv(nchw_to_rows(dZ), pack_dgrad(Wt, lanes)), B, Wt.shape[1], T, W, lanes)


def wgrad_engine(dZ, X, lanes):
    """The transposed GEMM: A = dZ^T (C_out, rows), W operand [taps K + 1][rows] with row (t, k) = rows(X)[r + t - taps/2, k]
    and a row of ones; returns dW (C_out, C_in, 3, kw), db (C_out)."""
    taps, kw = taps_of(lanes), 9 if lanes == 2 else 3
    R = expand(X, lanes)
    BB, G, K = R.shape
    Ci = X.shape[1]
    ops = []
    for t in range(taps):
        sh = t - taps // 2
        src = torch.zeros_like(R)
        lo, hi = max(0, -sh), min(G, G - sh)
        if hi > lo:
            src[:, lo:hi] = R[:, lo + sh:hi + sh]
        ops.append(src.reshape(BB * G, K))
    Wop = torch.cat(ops + [torch.ones(BB * G, 1, dtype=X.dtype)], dim=1)
    out = nchw_to_rows(dZ).reshape(BB * G, -1).t() @ Wop                   # (C_out, taps K + 1)
    P = out[:, :taps * K].reshape(-1, taps, lanes, 3, Ci)
    dW = torch.zeros(out.shape[0], Ci, 3, kw, dtype=X.dtype)
    for k in range(kw):
        dW[:, :, :, k] = P[:, k // lanes, k % lanes].permute(0, 2, 1)
    return dW, out[:, taps * K]


def post_across_seams(outs: List[torch.Tensor], w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """conv_post as mrd_post_fwd_kernel states it, without a concatenated tensor: post[b, 0, t, x] = bias + Σ_{c, dt, dk}
    w[0, c, dt, dk] band_k(x + dk - 1)[b, c, t + dt - 1], where column x + dk - 1 is read from the band k that holds it
    (the neighbouring band across a seam), zero outside [0, Σ W) and [0, T')."""
    offs = [0]
    for o in outs:
        offs.append(offs[-1] + o.shape[-1])
    B, _, T, _ = outs[0].shape
    post = torch.zeros(B, 1, T, offs[-1], dtype=outs[0].dtype) + b.view(1, 1, 1, 1)
    for x in range(offs[-1]):
        for dk in range(3):
            col = x + dk - 1
            if col < 0 or col >= offs[-1]:
                continue
            k = max(i for i in range(len(outs)) if offs[i] <= col)
            src = outs[k][:, :, :, col - offs[k]]                                 # (B, C, T)
            for dt in range(3):
                lo, hi = max(0, 1 - dt), min(T, T + 1 - dt)                      # rows t with 0 <= t + dt - 1 < T
                post[:, 0, lo:hi, x] += torch.einsum("c,bct->bt", w[0, :, dt, dk], src[:, :, lo + dt - 1:hi + dt - 1])
    return post


def post_dgrad_band(gpost: torch.Tensor, w: torch.Tensor, widths: List[int], k: int) -> torch.Tensor:
    """conv_post's input gradient for band k as mrd_post_dgrad_kernel states it: G[b, c, t, x] = Σ_{dt, dk} w[0, c, dt, dk]
    gpost[b, 0, t - dt + 1, off_k + x - dk + 1], reading the score columns across the band's seams."""
    off, Wt = sum(widths[:k]), sum(widths)
    B, _, T, _ = gpost.shape
    G = torch.zeros(B, w.shape[1], T, widths[k], dtype=gpost.dtype)
    for x in range(widths[k]):
        for dk in range(3):
            X = off + x - dk + 1
            if X < 0 or X >= Wt:
                continue
            for dt in range(3):
                lo, hi = max(0, dt - 1), min(T, T + dt - 1)                      # rows t with 0 <= t - dt + 1 < T
                G[:, :, lo:hi, x] += w[0, :, dt, dk].view(1, -1, 1) * gpost[:, :, lo - dt + 1:hi - dt + 1, X]
    return G


def stft_adjoint(gspec: torch.Tensor, window: torch.Tensor, N: int, L: int) -> torch.Tensor:
    """The input gradient of spectrogram for the cotangent gspec (B, 2, T', F): per frame d_n = w_n Re Σ_k (gRe_k +
    i gIm_k) e^{+2πikn/N}, the overlap-add of the frames, the reflect pad folded back onto its mirror samples."""
    B, _, T, Fq = gspec.shape
    hop, pad = N // 4, N // 2
    k = torch.arange(Fq, dtype=torch.float64)
    n = torch.arange(N, dtype=torch.float64)
    ang = 2 * torch.pi * k[:, None] * n[None, :] / N
    g = gspec.permute(0, 2, 3, 1)                                          # (B, T, F, 2)
    d = (g[..., 0] @ torch.cos(ang) - g[..., 1] @ torch.sin(ang)) * window.to(torch.float64)   # (B, T, N)
    padded = torch.zeros(B, L + 2 * pad, dtype=torch.float64)
    for t in range(T):
        padded[:, t * hop:t * hop + N] += d[:, t]
    gx = padded[:, pad:pad + L].clone()
    gx[:, 1:pad + 1] += padded[:, :pad].flip(1)                            # padded p < pad reads x[pad - p]
    gx[:, L - 1 - pad:L - 1] += padded[:, L + pad:].flip(1)                # padded p >= L + pad reads x[2 (L - 1) - (p - pad)]
    return gx


# ---------------------------------------------------------------- fixture cases (oracle/make_golden_mrd.py) ----------------
# weights: the reference's own init of a MultiResolutionDiscriminator built right after torch.manual_seed(weight_seed); the
# drop-in builds the same modules in the same order, so it regenerates them exactly
CASES = {
    "mrd_b2_l20480": dict(B=2, L=20480, seed=21, weight_seed=0),
    "mrd_b3_l1100": dict(B=3, L=1100, seed=22, weight_seed=1),
    "mrd_b2_l5003": dict(B=2, L=5003, seed=23, weight_seed=2),
}


def make_wave(cs) -> torch.Tensor:
    return (0.3 * seeded((cs["B"], 1, cs["L"]), cs["seed"], 0)).float().double()   # fp32-representable, as the GPU sees it
