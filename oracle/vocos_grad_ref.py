"""fp64 oracle of the Vocos generator's backward pass (DESIGN.md §8 row f12; TEST INFRASTRUCTURE ONLY).

``oracle_grads`` is torch's float64 autograd through ``vocoder_ref.vocos_forward`` (the reference's own irfft / fold ISTFT).
The functions below it state the adjoints st_vocos_backward computes, one per row kernel or packing, in the notation of
include/stabletts_b200.h (rows are the B·T tokens):

    frame gradient    dF[t, n] = g[s] / env[s], s = t·hop + n − pad inside [0, L), else 0
    spectrum          a = min(exp(m), 1e2); da = dre·cos p + dim·sin p; dp = a·(dim·cos p − dre·sin p);
                      dm = da·a·[exp(m) ≤ 1e2]
    LayerNorm         dx = rstd·(g·w − mean(g·w) − ẑ·mean(g·w·ẑ)); dw = Σ_rows g·ẑ; db = Σ_rows g
    depthwise conv    dx[t, c] = Σ_k w[c, k]·dz[t + 3 − k, c]; dw[c, k] = Σ dz[t, c]·x[t + k − 3, c]; db = Σ dz
                      (zero padding 3 at each utterance's edges)
    GELU              gelu'(h) = Φ(h) + h·φ(h)
    wgrad packing     [Xᵀ; 1] with 7-tap shifts for the embed conv: row k·C + c, column b·T + t = x[b, t + k − 3, c]
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch
import torch.nn.functional as F

from oracle import vocoder_ref as V

LN_CLIP = math.log(1e2)


def seeded(shape, seed: int, k: int) -> torch.Tensor:
    """N(0, 1) float64 draw number k of a case (upstream gradients, probe tensors)."""
    return torch.randn(tuple(shape), generator=torch.Generator().manual_seed(seed * 100003 + k), dtype=torch.float64)


def param_names(dims) -> List[str]:
    return [n for n in V.param_shapes(**dims) if n != "head.istft.window"]


def param_sizes(dims) -> List[int]:
    return [math.prod(s) for n, s in V.param_shapes(**dims).items() if n != "head.istft.window"]


def oracle_grads(state, mel: torch.Tensor, g: torch.Tensor, n_fft: int, hop: int):
    """(audio, {name: gradient}) of <vocos_forward(mel), g> in float64"""
    st = {k: v.detach().double().clone().requires_grad_(k != "head.istft.window") for k, v in state.items()}
    audio = V.vocos_forward(st, mel.double(), n_fft, hop)
    (audio * g.double()).sum().backward()
    return audio.detach(), {k: v.grad for k, v in st.items() if k != "head.istft.window"}


def clip_margin(state, mel: torch.Tensor) -> float:
    """the smallest |log-magnitude − ln 100| over every (frame, bin): how far the input is from flipping a clip decision"""
    with torch.no_grad():
        st = {k: v.double() for k, v in state.items()}
        return float((V.head_log_magnitudes(st, mel.double()) - LN_CLIP).abs().min())


def make_clean_mel(state, seed: int, B: int, T: int, dims, margin: float = 1e-3) -> torch.Tensor:
    """the first of the mels V.make_mel(seed + 1000 i) whose log-magnitudes all stay `margin` away from ln 100, so that no
    clip decision depends on rounding (float32-representable)"""
    for i in range(64):
        mel = V.make_mel(seed + 1000 * i, B, T, dims["input_channels"])
        if clip_margin(state, mel) >= margin:
            return mel
    raise RuntimeError("no mel clear of the clip boundary")


def checksums(state) -> "np.ndarray":
    return torch.tensor([[float(v.double().sum()), float(v.double().square().sum())] for v in state.values()],
                        dtype=torch.float64).numpy()


def grad_stats(grads, seed: int) -> torch.Tensor:
    """(norm, dot with a seeded probe) of every gradient, in order"""
    return torch.tensor([[float(g.norm()), float((g.double() * seeded(g.shape, seed, 5000 + i)).sum())]
                         for i, g in enumerate(grads)], dtype=torch.float64)


# fixtures of the unmodified reference (make_golden_vocos_grad.py): name -> dims, B, T, seeds, head gain
FIXTURES = {
    "vocos_grad_train_b2_t40": dict(dims={}, B=2, T=40, seed=61, weight_seed=21, head_gain=0.5),
    "vocos_grad_api_b1_t1": dict(dims=V.API_DIMS, B=1, T=1, seed=62, weight_seed=22, head_gain=0.5),
    "vocos_grad_api_b2_t16_clip": dict(dims=V.API_DIMS, B=2, T=16, seed=63, weight_seed=23, head_gain=V.HEAD_GAIN_CLIP),
}


def case_dims(cs):
    d = dict(V.DIMS)
    d.update(cs["dims"])
    return d


def case_state(cs):
    return V.make_state(cs["weight_seed"], head_gain=cs["head_gain"], **cs["dims"])


def case_mel(cs) -> torch.Tensor:
    return make_clean_mel(case_state(cs), cs["seed"], cs["B"], cs["T"], case_dims(cs)).double()


# ---- the explicit adjoints ------------------------------------------------------------------------------------------
def envelope(window: torch.Tensor, T: int, n_fft: int, hop: int) -> torch.Tensor:
    """env[s], s in [0, T·hop): Σ window[n]² over the frames covering sample s + pad of the untrimmed signal"""
    pad = (n_fft - hop) // 2
    s = torch.arange(T * hop) + pad
    env = torch.zeros(T * hop, dtype=torch.float64)
    for j in range(n_fft // hop):
        t = s // hop - j
        ok = (t >= 0) & (t < T)
        env += torch.where(ok, window.double()[s - t * hop].square(), torch.zeros((), dtype=torch.float64))
    return env


def frame_grad(g: torch.Tensor, window: torch.Tensor, T: int, n_fft: int, hop: int) -> torch.Tensor:
    """g (B, T·hop) -> dF (B, T, n_fft)"""
    B = g.shape[0]
    pad = (n_fft - hop) // 2
    env = envelope(window, T, n_fft, hop)
    s = torch.arange(T)[:, None] * hop + torch.arange(n_fft)[None, :] - pad
    ok = (s >= 0) & (s < T * hop)
    sc = s.clamp(0, T * hop - 1)
    return torch.where(ok[None], (g.double() / env[None])[:, sc], torch.zeros((), dtype=torch.float64))


def spectrum_grad(dre, dim, m, p):
    """(dlogmag, dphase) of re = a cos p, im = a sin p, a = min(exp(m), 1e2); all (…, K)"""
    e = torch.exp(m)
    a = torch.clamp(e, max=1e2)
    da = dre * torch.cos(p) + dim * torch.sin(p)
    dp = a * (dim * torch.cos(p) - dre * torch.sin(p))
    return torch.where(e <= 1e2, da * a, torch.zeros_like(da)), dp


def ln_bwd(x, w, g, eps: float = 1e-6):
    """(dx, dw, db) of LayerNorm over the last dim (affine, biased variance); x, g (rows, C)"""
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
    zh = (x - mean) * rstd
    gw = g * w
    dx = rstd * (gw - gw.mean(-1, keepdim=True) - zh * (gw * zh).mean(-1, keepdim=True))
    return dx, (g * zh).sum(0), g.sum(0)


def dwconv_bwd(x, w, dz):
    """(dx, dw (C, 1, 7), db) of the depthwise k = 7 conv with zero padding 3 per utterance; x, dz (B, T, C)"""
    B, T, C = x.shape
    xp = F.pad(x, (0, 0, 3, 3))
    dzp = F.pad(dz, (0, 0, 3, 3))
    dx = torch.zeros_like(x)
    dw = torch.zeros(C, 1, 7, dtype=x.dtype)
    for k in range(7):
        dx += w[:, 0, k] * dzp[:, 6 - k: 6 - k + T]               # dz[t + 3 - k]
        dw[:, 0, k] = (dz * xp[:, k: k + T]).sum((0, 1))          # x[t + k - 3]
    return dx, dw, dz.sum((0, 1))


def gelu_bwd(h, dg):
    return dg * (0.5 * (1 + torch.erf(h / math.sqrt(2))) + h * torch.exp(-0.5 * h * h) / math.sqrt(2 * math.pi))


def wgrad_operand(x, taps: int, Kr: int) -> torch.Tensor:
    """[Xᵀ; 1] (taps·C + 8, Kr) of x (B, T, C): row k·C + c, column b·T + t = x[b, t + k − 3, c] (taps 7) or x[b, t, c]
    (taps 1), 0 outside the utterance; row taps·C is 1 on the B·T real columns; the rest 0"""
    B, T, C = x.shape
    out = torch.zeros(taps * C + 8, Kr, dtype=x.dtype)
    xp = F.pad(x, (0, 0, 3, 3))
    for k in range(taps):
        sh = k if taps == 7 else 3
        out[k * C:(k + 1) * C, :B * T] = xp[:, sh: sh + T].reshape(B * T, C).T
    out[taps * C, :B * T] = 1
    return out


def unpack_wgrad(dWp, Nref: int, Cx: int, taps: int, split: int = 0, Kp: int = 0):
    """[Np][taps·Cx + 8] -> (gw (Nref, Cx, taps), gb (Nref,)); split > 0: row n >= split reads packed row Kp + n − split"""
    n = torch.arange(Nref)
    m = torch.where((n >= split) & (split > 0), Kp + n - split, n)
    rows = dWp[m]
    gw = rows[:, :taps * Cx].reshape(Nref, taps, Cx).permute(0, 2, 1)
    return gw, rows[:, taps * Cx]
