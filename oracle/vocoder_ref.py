"""CPU oracle for SURVEY.md §8 row f4, the vocoder hand-off (TEST INFRASTRUCTURE ONLY; the CUDA path for this row
is NOT built yet — this file and its fixtures are the groundwork: the restated algorithm, pinned against the
unmodified reference, in the form the tensor-core path will compute it).

Restates the reference's Vocos (vocoders/vocos/models/model.py:11-20): ``VocosBackbone``
(vocoders/vocos/models/backbone.py:21-56: k=7 embed conv, LayerNorm, 12 ConvNeXt blocks, final LayerNorm),
``ConvNeXtBlock`` (vocoders/vocos/models/module.py:15-46: depthwise k=7 conv, LayerNorm, Linear 768->2048, GELU,
Linear 2048->768, layer scale, residual) and ``ISTFTHead`` / ``ISTFT`` with "same" padding
(vocoders/vocos/models/head.py:21-117).

``istft_same_as_gemm`` is the same inverse STFT written as ONE dense contraction with a windowed inverse-DFT basis
(2·(n_fft/2+1) x n_fft) followed by a 4-frame overlap-add gather — the formulation a split-bf16 wgmma GEMM can
run — and tests/test_vocoder_oracle.py shows it equals the reference's ``irfft`` + ``fold`` path.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

DIMS = dict(input_channels=128, dim=768, intermediate_dim=2048, num_layers=12, n_fft=2048, hop_length=512)   # vocoders/vocos/config.py:4-27
# The Vocos that api.py builds: get_vocoder(..., 'vocos') runs `from config import VocosConfig, MelConfig` from the reference
# root, i.e. the top-level config.py (VocosConfig at its end: dim 512, intermediate_dim 1536, num_layers 8), not
# vocoders/vocos/config.py, which is the vocos training configuration (DIMS).
API_DIMS = dict(dim=512, intermediate_dim=1536, num_layers=8)
HEAD_GAIN_CLIP = 8.0                 # 16 % of the clip fixture's (frame, bin) magnitudes exceed 1e2


def param_shapes(input_channels=128, dim=768, intermediate_dim=2048, num_layers=12, n_fft=2048, hop_length=512):
    s = OrderedDict()
    s["backbone.embed.weight"] = (dim, input_channels, 7); s["backbone.embed.bias"] = (dim,)
    s["backbone.norm.weight"] = (dim,); s["backbone.norm.bias"] = (dim,)
    for i in range(num_layers):
        p = f"backbone.convnext.{i}."
        s[p + "gamma"] = (dim,)
        s[p + "dwconv.weight"] = (dim, 1, 7); s[p + "dwconv.bias"] = (dim,)
        s[p + "norm.weight"] = (dim,); s[p + "norm.bias"] = (dim,)
        s[p + "pwconv1.weight"] = (intermediate_dim, dim); s[p + "pwconv1.bias"] = (intermediate_dim,)
        s[p + "pwconv2.weight"] = (dim, intermediate_dim); s[p + "pwconv2.bias"] = (dim,)
    s["backbone.final_layer_norm.weight"] = (dim,); s["backbone.final_layer_norm.bias"] = (dim,)
    s["head.out.weight"] = (n_fft + 2, dim); s["head.out.bias"] = (n_fft + 2,)
    s["head.istft.window"] = (n_fft,)
    return s


def make_state(seed: int = 11, head_gain: float = 0.5, **dims):
    """Seeded synthetic weights under the reference's parameter names: U(+-1/sqrt(fan_in)) matrices, LayerNorm affine
    near (1, 0), layer scale ~ 1/num_layers (backbone.py:32).  The head weight is scaled by head_gain: the default 0.5 keeps
    exp(mag) off the 1e2 clip; a larger gain drives a share of the (frame, bin) magnitudes onto it."""
    d = dict(DIMS); d.update(dims)
    g = torch.Generator().manual_seed(seed)
    st = OrderedDict()
    for name, shape in param_shapes(**d).items():
        if name == "head.istft.window":
            st[name] = torch.hann_window(d["n_fft"])                                     # head.py:28-29
        elif name.endswith("gamma"):
            st[name] = (1.0 / d["num_layers"]) * (1 + 0.2 * torch.randn(shape, generator=g))
        elif ".norm." in name or "final_layer_norm" in name:
            st[name] = (1 + 0.1 * torch.randn(shape, generator=g)) if name.endswith("weight") else 0.1 * torch.randn(shape, generator=g)
        elif name.endswith(".weight"):
            fan = 1
            for k in shape[1:]:
                fan *= k
            st[name] = (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(fan) * (head_gain if name.startswith("head") else 1.0)
        else:
            st[name] = 0.1 * (torch.rand(shape, generator=g) * 2 - 1)
    return st


def make_mel(seed: int, B: int, T: int, n_mel: int = 128) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, n_mel, T, generator=g)


def backbone_forward(state, x: torch.Tensor) -> torch.Tensor:
    """backbone.py:49-56 / module.py:34-46.  x: (B, n_mel, T) -> (B, T, dim)."""
    dim = state["backbone.norm.weight"].shape[0]
    n_layers = 1 + max(int(k.split(".")[2]) for k in state if k.startswith("backbone.convnext."))
    x = F.conv1d(x, state["backbone.embed.weight"], state["backbone.embed.bias"], padding=3)        # :50
    x = F.layer_norm(x.transpose(1, 2), (dim,), state["backbone.norm.weight"], state["backbone.norm.bias"], 1e-6).transpose(1, 2)
    for i in range(n_layers):
        p = f"backbone.convnext.{i}."
        r = x
        h = F.conv1d(x, state[p + "dwconv.weight"], state[p + "dwconv.bias"], padding=3, groups=dim)   # module.py:36
        h = F.layer_norm(h.transpose(1, 2), (dim,), state[p + "norm.weight"], state[p + "norm.bias"], 1e-6)
        h = F.linear(h, state[p + "pwconv1.weight"], state[p + "pwconv1.bias"])
        h = F.gelu(h)                                                                                  # exact (erf) GELU
        h = F.linear(h, state[p + "pwconv2.weight"], state[p + "pwconv2.bias"])
        h = state[p + "gamma"] * h
        x = r + h.transpose(1, 2)
    return F.layer_norm(x.transpose(1, 2), (dim,), state["backbone.final_layer_norm.weight"],
                        state["backbone.final_layer_norm.bias"], 1e-6)                                # :55


def head_spectrum(state, h: torch.Tensor):
    """head.py:96-113: Linear -> (log-magnitude, phase) -> real / imaginary parts.  h: (B, T, dim) -> two (B, N, T)."""
    x = F.linear(h, state["head.out.weight"], state["head.out.bias"]).transpose(1, 2)
    mag, p = x.chunk(2, dim=1)
    mag = torch.clip(torch.exp(mag), max=1e2)
    return mag * torch.cos(p), mag * torch.sin(p)


def istft_same_reference(re: torch.Tensor, im: torch.Tensor, window: torch.Tensor, n_fft: int, hop: int) -> torch.Tensor:
    """head.py:31-83 ("same" padding, win_length = n_fft), literally: irfft, window, fold, envelope."""
    B, N, T = re.shape
    pad = (n_fft - hop) // 2
    ifft = torch.fft.irfft(torch.complex(re, im), n_fft, dim=1, norm="backward") * window[None, :, None]
    size = (T - 1) * hop + n_fft
    y = F.fold(ifft, output_size=(1, size), kernel_size=(1, n_fft), stride=(1, hop))[:, 0, 0, pad:-pad]
    wsq = window.square().expand(1, T, -1).transpose(1, 2)
    env = F.fold(wsq, output_size=(1, size), kernel_size=(1, n_fft), stride=(1, hop)).squeeze()[pad:-pad]
    return y / env


def idft_basis(window: torch.Tensor, n_fft: int, dtype=torch.float64) -> torch.Tensor:
    """(2·(n_fft/2+1), n_fft) matrix W with  frame[n] = sum_k re[k]·W[k, n] + im[k]·W[K+k, n]  ==  window[n]·irfft(S)[n].
    irfft ignores the imaginary parts of the DC and Nyquist bins and counts the interior bins twice."""
    K = n_fft // 2 + 1
    k = torch.arange(K, dtype=dtype)[:, None]
    n = torch.arange(n_fft, dtype=dtype)[None, :]
    ang = 2 * math.pi * k * n / n_fft
    c = torch.full((K, 1), 2.0, dtype=dtype); c[0] = 1.0; c[-1] = 1.0
    wr = c * torch.cos(ang) / n_fft
    wi = -c * torch.sin(ang) / n_fft
    wi[0] = 0.0; wi[-1] = 0.0
    return (torch.cat([wr, wi], 0) * window.to(dtype)[None, :])


def istft_same_as_gemm(re: torch.Tensor, im: torch.Tensor, window: torch.Tensor, n_fft: int, hop: int) -> torch.Tensor:
    """The same ISTFT as one GEMM + a gather: frames = [re | im]^T · W (rows = frames), then every output sample
    sums the n_fft/hop frames that overlap it and divides by the (input-independent) window envelope."""
    B, N, T = re.shape
    W = idft_basis(window, n_fft, torch.float64).to(re.dtype)
    frames = torch.cat([re, im], 1).transpose(1, 2) @ W                 # (B, T, n_fft): the GEMM
    pad = (n_fft - hop) // 2
    L = T * hop                                                         # (T-1)·hop + n_fft - 2·pad
    s = torch.arange(L) + pad                                           # position in the un-trimmed signal
    out = torch.zeros(B, L, dtype=re.dtype)
    env = torch.zeros(L, dtype=re.dtype)
    for j in range(n_fft // hop):                                       # the frames covering sample s: t = s//hop - j
        t = s // hop - j
        n = s - t * hop
        ok = (t >= 0) & (t < T)
        tc = t.clamp(0, T - 1)
        out += torch.where(ok[None, :], frames[:, tc, n], torch.zeros((), dtype=re.dtype))
        env += torch.where(ok, window[n].square(), torch.zeros((), dtype=re.dtype))
    return out / env


def vocos_forward(state, mel: torch.Tensor, n_fft: int = 2048, hop: int = 512, gemm_istft: bool = False) -> torch.Tensor:
    """model.py:17-20: mel (B, n_mel, T) -> audio (B, T·hop)."""
    re, im = head_spectrum(state, backbone_forward(state, mel))
    f = istft_same_as_gemm if gemm_istft else istft_same_reference
    return f(re, im, state["head.istft.window"], n_fft, hop)


def head_log_magnitudes(state, mel: torch.Tensor) -> torch.Tensor:
    """the head's log-magnitudes (B, K, T) before exp and the clip (head.py:101-105)"""
    x = F.linear(backbone_forward(state, mel), state["head.out.weight"], state["head.out.bias"]).transpose(1, 2)
    return x.chunk(2, dim=1)[0]


# name -> mel seed, B, T and the make_state arguments beyond the seed (none: DIMS with head_gain 0.5)
CASES = {
    "vocos_b2_t24": dict(seed=41, B=2, T=24),
    "vocos_b1_t7": dict(seed=42, B=1, T=7),
}
API_CASES = {
    "vocos_api_b2_t24": dict(seed=51, B=2, T=24, state=dict(API_DIMS)),
    "vocos_api_b1_t1": dict(seed=52, B=1, T=1, state=dict(API_DIMS)),        # one frame: every dwconv tap but the centre is off
    "vocos_api_b2_t64_clip": dict(seed=53, B=2, T=64, state=dict(API_DIMS, head_gain=HEAD_GAIN_CLIP)),
}
