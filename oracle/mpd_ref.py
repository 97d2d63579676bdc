"""Float64 restatement of the Vocos multi-period discriminator (vocoders/vocos/models/discriminator.py:33-79) and of the
GEMM packings its CUDA path uses (stabletts_b200/csrc/mpd_api.cu).  Test-side only: nothing under stabletts_b200/ imports it.

``discriminator_p`` follows DiscriminatorP.forward: reflect pad on the right when L % p != 0 (lines 62-66), the
(B, 1, L / p, p) view (line 67), five (5, 1) convs with leaky ReLU 0.1 (lines 69-73), conv_post (line 74), flatten
(line 76).  ``masks`` replaces each leaky ReLU's sign test by a given boolean pattern (True = slope 1), so a backward can be
taken with another implementation's activation signs: a pre-activation that lands on the other side of zero in fp32 then
cannot make a gradient comparison flaky."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

PERIODS = (2, 3, 5, 7, 11)
CHANS = (1, 32, 128, 512, 1024, 1024)
SLOPE = 0.1


def weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """torch.nn.utils.parametrizations.weight_norm with dim = 0: g v / ||v|| over every dim but the first."""
    return g * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))


def effective_params(sd: Dict[str, torch.Tensor], prefix: str = "") -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """(weight, bias) of convs 0-4 and conv_post from a DiscriminatorP state_dict (keys under `prefix`)."""
    out = []
    for name in [f"convs.{i}" for i in range(5)] + ["conv_post"]:
        p = prefix + name
        out.append((weight_norm(sd[p + ".parametrizations.weight.original0"], sd[p + ".parametrizations.weight.original1"]),
                    sd[p + ".bias"]))
    return out


def pad_view(x: torch.Tensor, p: int) -> torch.Tensor:
    """(B, 1, L) -> (B, 1, ceil(L / p), p), reflect-padded on the right (discriminator.py:62-67)."""
    b, c, t = x.shape
    if t % p:
        x = F.pad(x, (0, p - t % p), "reflect")
        t = x.shape[-1]
    return x.view(b, c, t // p, p)


def discriminator_p(x: torch.Tensor, params, p: int, masks: Optional[List[torch.Tensor]] = None):
    """-> (score, fmaps of convs 0-4 + post, pre-activations of convs 0-4).  fmaps[1:] is the reference's fmap list."""
    h = pad_view(x, p)
    fmaps, pres = [], []
    for i in range(5):
        w, b = params[i]
        z = F.conv2d(h, w, b, stride=(3 if i < 4 else 1, 1), padding=(2, 0))
        pres.append(z)
        pos = (z > 0) if masks is None else masks[i]
        h = torch.where(pos, z, SLOPE * z)
        fmaps.append(h)
    w, b = params[5]
    post = F.conv2d(h, w, b, stride=1, padding=(1, 0))
    fmaps.append(post)
    return torch.flatten(post, 1, -1), fmaps, pres


# ---------------------------------------------------------------- packing identities (mpd_api.cu) --------------------------
# rows of one column: X (H_in, C_in) token-major; a (5, 1) conv with stride s and pad 2 along H.

def conv_rows(X: torch.Tensor, W: torch.Tensor, stride: int) -> torch.Tensor:
    """Direct statement: Y[o, n] = Σ_{k, c} W[n, c, k] X[s o + k - 2, c], rows outside [0, H_in) zero.  X (H_in, C_in),
    W (C_out, C_in, 5)."""
    return F.conv1d(X.t()[None], W, stride=stride, padding=2)[0].t()


def engine_conv(A: torch.Tensor, Wp: torch.Tensor) -> torch.Tensor:
    """The conv-GEMM engine's contract for one batch: out[t, n] = Σ_{tap, k} A[t + tap - taps // 2, k] Wp[tap, n, k]."""
    taps, T = Wp.shape[0], A.shape[0]
    out = torch.zeros(T, Wp.shape[1], dtype=A.dtype)
    for tap in range(taps):
        sh = tap - taps // 2
        src = torch.zeros_like(A)
        lo, hi = max(0, -sh), min(T, T - sh)
        if hi > lo:
            src[lo:hi] = A[lo + sh:hi + sh]
        out += src @ Wp[tap].t()
    return out


def pack_fwd_s3(W: torch.Tensor) -> torch.Tensor:
    """[2][C_out][3 C_in]: tap 0 (group o - 1), lane l -> kernel tap l - 1 (lane 0: zero); tap 1 (group o) -> l + 2."""
    Co, Ci, _ = W.shape
    P = torch.zeros(2, Co, 3, Ci, dtype=W.dtype)
    P[0, :, 1] = W[:, :, 0]
    P[0, :, 2] = W[:, :, 1]
    for l in range(3):
        P[1, :, l] = W[:, :, l + 2]
    return P.reshape(2, Co, 3 * Ci)


def pack_dgrad_s3(W: torch.Tensor) -> torch.Tensor:
    """[2][3 C_in][C_out]: output row r = input group r - 1; tap 0 reads dZ[group] (kernel tap l + 2), tap 1 reads
    dZ[group + 1] (kernel tap l - 1, zero for lane 0)."""
    Co, Ci, _ = W.shape
    P = torch.zeros(2, 3, Ci, Co, dtype=W.dtype)
    for l in range(3):
        P[0, l] = W[:, :, l + 2].t()
    P[1, 1] = W[:, :, 0].t()
    P[1, 2] = W[:, :, 1].t()
    return P.reshape(2, 3 * Ci, Co)


def pack_dgrad_s1(W: torch.Tensor) -> torch.Tensor:
    """[5][C_in][C_out]: flipped, transposed taps."""
    return W.flip(2).permute(2, 1, 0).contiguous()


def strided_forward(X: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """Stride-3 conv as the engine runs it: X zero-padded to 3 G rows and viewed as (G, 3 C_in), a 2-tap conv."""
    H, Ci = X.shape
    G = -(-H // 3)
    Xg = torch.zeros(3 * G, Ci, dtype=X.dtype)
    Xg[:H] = X
    return engine_conv(Xg.reshape(G, 3 * Ci), pack_fwd_s3(W))


def strided_dgrad(dZ: torch.Tensor, W: torch.Tensor, H_in: int) -> torch.Tensor:
    """Input gradient of the stride-3 conv as the engine runs it: dZ with one zero row appended, the DGRAD_S3 2-tap conv,
    output row r = group r - 1 viewed as rows, input row h at row h + 3."""
    G, Co = dZ.shape
    Ci = W.shape[1]
    A = torch.cat([dZ, torch.zeros(1, Co, dtype=dZ.dtype)])
    out = engine_conv(A, pack_dgrad_s3(W)).reshape(3 * (G + 1), Ci)
    return out[3:3 + H_in]


def s1_dgrad(dZ: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    return engine_conv(dZ, pack_dgrad_s1(W))


def wgrad(dZs: List[torch.Tensor], Xs: List[torch.Tensor], stride: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Weight and bias gradients as the transposed GEMM: A = dZ^T (C_out, rows of every column), W operand [5 C_in + 1][rows]
    with row (k, c) = X[s o + k - 2, c] and a row of ones; returns dW (C_out, C_in, 5), db (C_out)."""
    cols = []
    for X, dZ in zip(Xs, dZs):
        H, Ci = dZ.shape[0], X.shape[1]
        M = torch.zeros(5 * Ci + 1, H, dtype=X.dtype)
        for k in range(5):
            for o in range(H):
                hx = stride * o + k - 2
                if 0 <= hx < X.shape[0]:
                    M[k * Ci:(k + 1) * Ci, o] = X[hx]
        M[5 * Ci] = 1
        cols.append(M)
    Wop = torch.cat(cols, dim=1)
    AT = torch.cat([d.t() for d in dZs], dim=1)
    out = AT @ Wop.t()
    Ci = Xs[0].shape[1]
    return out[:, :5 * Ci].reshape(-1, 5, Ci).permute(0, 2, 1).contiguous(), out[:, 5 * Ci]


# ---------------------------------------------------------------- fixture cases (oracle/make_golden_mpd.py) ----------------
# weights: the reference's own init (nn.Conv2d defaults under weight_norm) of a MultiPeriodDiscriminator built right after
# torch.manual_seed(weight_seed); the drop-in builds the same modules in the same order, so it regenerates them exactly
CASES = {
    "mpd_b2_l4096": dict(B=2, L=4096, kind="noise", seed=11, weight_seed=0),
    "mpd_b3_l4099": dict(B=3, L=4099, kind="noise", seed=12, weight_seed=0),
    "mpd_b2_l12": dict(B=2, L=12, kind="noise", seed=13, weight_seed=1),
    "mpd_b2_tone": dict(B=2, L=4096, kind="tone", seed=14, weight_seed=1),
}


def seeded(shape, seed: int, k: int) -> torch.Tensor:
    """N(0, 1) float64 draw number k of a case (upstream gradients and probe tensors)."""
    return torch.randn(tuple(shape), generator=torch.Generator().manual_seed(seed * 100003 + k), dtype=torch.float64)


def make_wave(cs) -> torch.Tensor:
    x = 0.3 * seeded((cs["B"], 1, cs["L"]), cs["seed"], 0)
    if cs["kind"] == "tone":
        t = torch.arange(cs["L"], dtype=torch.float64) / 24000.0
        x = 0.5 * torch.sin(2 * torch.pi * 440.0 * t).expand_as(x) + 0.05 * x
    return x.float().double()                     # fp32-representable, as the GPU sees it


def checksums(sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    return torch.tensor([[float(v.double().sum()), float(v.double().square().sum())] for v in sd.values()], dtype=torch.float64)


def fixture_quantities(score_fmaps, x_grad, param_grads, seed: int) -> Dict[str, torch.Tensor]:
    """What a fixture stores: per period the score in full and (norm, dot with a seeded probe) of each fmap; the input
    gradient in full; (norm, dot) of every parameter gradient in state_dict order."""
    out, k = {}, 1000
    for pi, (score, fmaps) in enumerate(score_fmaps):
        out[f"score{pi}"] = score.detach()
        st = []
        for f in fmaps:
            st.append([float(f.detach().norm()), float((f.detach() * seeded(f.shape, seed, k)).sum())])
            k += 1
        out[f"fmap_stats{pi}"] = torch.tensor(st, dtype=torch.float64)
    out["gx"] = x_grad.detach()
    st, k = [], 5000
    for g in param_grads:
        st.append([float(g.norm()), float((g.detach() * seeded(g.shape, seed, k)).sum())])
        k += 1
    out["grad_stats"] = torch.tensor(st, dtype=torch.float64)
    return out


def upstream_loss(score_fmaps, seed: int) -> torch.Tensor:
    """Σ over periods of <score, g_s> + Σ <fmap_i, g_i>, every upstream gradient a seeded N(0, 1) draw."""
    loss, k = 0.0, 2000
    for score, fmaps in score_fmaps:
        loss = loss + (score * seeded(score.shape, seed, k).to(score)).sum()
        k += 1
        for f in fmaps:
            loss = loss + (f * seeded(f.shape, seed, k).to(f)).sum()
            k += 1
    return loss
