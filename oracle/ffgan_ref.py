"""CPU oracle for the FireflyGAN vocoder (TEST INFRASTRUCTURE ONLY): a functional, weight-dict-driven restatement of the
reference's ``FireflyGANBase`` (vocoders/ffgan/model.py:45-56) — ``ConvNeXtEncoder`` (vocoders/ffgan/backbone.py:146-214)
followed by ``HiFiGANGenerator`` (vocoders/ffgan/head.py:137-257) at the one configuration the reference ships
(``config_dict``, model.py:7-29).

Two formulations of the transposed convolutions (head.py:176-186) are kept side by side:
  * ``F.conv_transpose1d``, literally as the reference runs it;
  * the polyphase form the CUDA path runs: in token-major layout ``ConvTranspose1d(C_in -> C_out, k = 2u, stride u,
    padding u/2)`` is a 3-tap conv at the INPUT rate with N = u·C_out outputs per frame, whose (T, u·C_out) result is the
    (u·T, C_out) token-major input of the next stage (``polyphase_weight``).
"""
from __future__ import annotations

import math
import re
from collections import OrderedDict

import torch
import torch.nn.functional as F

DEPTHS, DIMS = (3, 3, 9, 3), (128, 256, 384, 512)                 # model.py:9-13
N_MEL, HOP = 128, 512
UPS = ((8, 16), (8, 16), (2, 4), (2, 4), (2, 4))                   # (upsample rate u, kernel 2u), model.py:18-19
RES_K, RES_D = (3, 7, 11), (1, 3, 5)                               # model.py:20-21
PRE_K = POST_K = 13                                                # model.py:25-26
C0 = 512                                                           # upsample_initial_channel


def _wn(s, name, w_shape):
    """weight_norm parametrization keys (torch.nn.utils.parametrizations.weight_norm, dim 0): g then v."""
    s[name + ".parametrizations.weight.original0"] = (w_shape[0], 1, 1)
    s[name + ".parametrizations.weight.original1"] = w_shape


def param_shapes():
    """The reference's state_dict inventory (471 tensors), in its registration order."""
    s = OrderedDict()
    s["backbone.downsample_layers.0.0.weight"] = (DIMS[0], N_MEL, 7); s["backbone.downsample_layers.0.0.bias"] = (DIMS[0],)
    s["backbone.downsample_layers.0.1.weight"] = (DIMS[0],); s["backbone.downsample_layers.0.1.bias"] = (DIMS[0],)
    for i in range(1, 4):                                                                    # backbone.py:172-177
        p = f"backbone.downsample_layers.{i}."
        s[p + "0.weight"] = (DIMS[i - 1],); s[p + "0.bias"] = (DIMS[i - 1],)
        s[p + "1.weight"] = (DIMS[i], DIMS[i - 1], 1); s[p + "1.bias"] = (DIMS[i],)
    for i, (depth, d) in enumerate(zip(DEPTHS, DIMS)):                                       # backbone.py:183-196
        for j in range(depth):
            p = f"backbone.stages.{i}.{j}."
            s[p + "gamma"] = (d,)
            s[p + "dwconv.weight"] = (d, 1, 7); s[p + "dwconv.bias"] = (d,)
            s[p + "norm.weight"] = (d,); s[p + "norm.bias"] = (d,)
            s[p + "pwconv1.weight"] = (4 * d, d); s[p + "pwconv1.bias"] = (4 * d,)
            s[p + "pwconv2.weight"] = (d, 4 * d); s[p + "pwconv2.bias"] = (d,)
    s["backbone.norm.weight"] = (DIMS[-1],); s["backbone.norm.bias"] = (DIMS[-1],)
    s["head.conv_pre.bias"] = (C0,); _wn(s, "head.conv_pre", (C0, C0, PRE_K))                  # head.py:162-170
    for i, (u, k) in enumerate(UPS):                                                         # head.py:176-186
        cin, cout = C0 >> i, C0 >> (i + 1)
        s[f"head.ups.{i}.bias"] = (cout,); _wn(s, f"head.ups.{i}", (cin, cout, k))
    for i in range(len(UPS)):                                                                # head.py:207-212
        c = C0 >> (i + 1)
        for b, k in enumerate(RES_K):
            for which in ("convs1", "convs2"):
                for j in range(3):
                    name = f"head.resblocks.{i}.blocks.{b}.{which}.{j}"
                    s[name + ".bias"] = (c,); _wn(s, name, (c, c, k))
    s["head.conv_post.bias"] = (1,); _wn(s, "head.conv_post", (1, C0 >> len(UPS), POST_K))   # head.py:215-223
    return s


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """W = g · v / ||v||, the norm over every dim except dim 0 (torch._weight_norm, dim = 0).  Dim 0 is C_out for Conv1d
    but C_in for ConvTranspose1d (whose weight is (C_in, C_out, k)): g is per INPUT channel there."""
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape((-1,) + (1,) * (v.dim() - 1))
    return v * (g / n)


def conv_weight(state, name: str) -> torch.Tensor:
    return fold_weight_norm(state[name + ".parametrizations.weight.original0"], state[name + ".parametrizations.weight.original1"])


def polyphase_weight(w: torch.Tensor, u: int) -> torch.Tensor:
    """ConvTranspose1d weight (C_in, C_out, 2u) -> (u·C_out, C_in, 3) Conv1d weight (padding 1, input rate) with
    W'[r·C_out + c, i, tau] = w[i, c, r + u/2 - (tau - 1)·u] where that index lies in [0, 2u), else 0."""
    cin, cout, k = w.shape
    assert k == 2 * u and u % 2 == 0
    out = torch.zeros(u, cout, cin, 3, dtype=w.dtype)
    for tau in range(3):
        for r in range(u):
            kk = r + u // 2 - (tau - 1) * u
            if 0 <= kk < k:
                out[r, :, :, tau] = w[:, :, kk].t()
    return out.reshape(u * cout, cin, 3)


def conv_transpose_polyphase(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, u: int) -> torch.Tensor:
    """Same result as F.conv_transpose1d(x, w, bias, stride=u, padding=u//2) for k = 2u, via the 3-tap polyphase conv:
    x (B, C_in, T) -> (B, C_out, u·T)."""
    B, _, T = x.shape
    cout = w.shape[1]
    y = F.conv1d(x, polyphase_weight(w, u), bias.repeat(u), padding=1)        # (B, u·C_out, T), row r·C_out + c
    return y.reshape(B, u, cout, T).permute(0, 2, 3, 1).reshape(B, cout, T * u)


def _ln_channels_first(x, w, b, eps=1e-6):
    """backbone.py:69-74."""
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    return w[:, None] * ((x - u) / torch.sqrt(s + eps)) + b[:, None]


def backbone_forward(state, x: torch.Tensor, skip_block=None) -> torch.Tensor:
    """backbone.py:206-214 (ConvNeXtBlock :124-143; DropPath is the identity in eval mode).  x (B, 128, T) -> (B, 512, T).
    skip_block = (stage, j) drops that block's residual branch (tests: every block matters)."""
    for i in range(4):
        p = f"backbone.downsample_layers.{i}."
        if i == 0:
            x = F.conv1d(x, state[p + "0.weight"], state[p + "0.bias"], padding=3)
            x = _ln_channels_first(x, state[p + "1.weight"], state[p + "1.bias"])
        else:
            x = _ln_channels_first(x, state[p + "0.weight"], state[p + "0.bias"])
            x = F.conv1d(x, state[p + "1.weight"], state[p + "1.bias"])
        d = DIMS[i]
        for j in range(DEPTHS[i]):
            if skip_block == (i, j):
                continue
            q = f"backbone.stages.{i}.{j}."
            h = F.conv1d(x, state[q + "dwconv.weight"], state[q + "dwconv.bias"], padding=3, groups=d)
            h = F.layer_norm(h.transpose(1, 2), (d,), state[q + "norm.weight"], state[q + "norm.bias"], 1e-6)
            h = F.gelu(F.linear(h, state[q + "pwconv1.weight"], state[q + "pwconv1.bias"]))
            h = state[q + "gamma"] * F.linear(h, state[q + "pwconv2.weight"], state[q + "pwconv2.bias"])
            x = x + h.transpose(1, 2)
    return _ln_channels_first(x, state["backbone.norm.weight"], state["backbone.norm.bias"])


def resblock1(state, name: str, x: torch.Tensor, k: int, skip=False) -> torch.Tensor:
    """head.py:92-99: three times x += conv2(silu(conv1(silu(x)))) with conv1 dilated 1 / 3 / 5."""
    if skip:
        return x
    for j, d in enumerate(RES_D):
        xt = F.conv1d(F.silu(x), conv_weight(state, f"{name}.convs1.{j}"), state[f"{name}.convs1.{j}.bias"],
                      padding=d * (k - 1) // 2, dilation=d)
        xt = F.conv1d(F.silu(xt), conv_weight(state, f"{name}.convs2.{j}"), state[f"{name}.convs2.{j}.bias"],
                      padding=(k - 1) // 2)
        x = xt + x
    return x


def head_forward(state, x: torch.Tensor, polyphase: bool = False, skip_resblock=None) -> torch.Tensor:
    """head.py:225-249 with use_template = False: (B, 512, T) -> (B, 1, 512·T)."""
    x = F.conv1d(x, conv_weight(state, "head.conv_pre"), state["head.conv_pre.bias"], padding=(PRE_K - 1) // 2)
    for i, (u, k) in enumerate(UPS):
        x = F.silu(x)
        w, b = conv_weight(state, f"head.ups.{i}"), state[f"head.ups.{i}.bias"]
        x = conv_transpose_polyphase(x, w, b, u) if polyphase else F.conv_transpose1d(x, w, b, stride=u, padding=(k - u) // 2)
        rs = [resblock1(state, f"head.resblocks.{i}.blocks.{bi}", x, kk, skip=skip_resblock == (i, bi))
              for bi, kk in enumerate(RES_K)]
        x = torch.stack(rs, 0).mean(0)                                         # ParralelBlock, head.py:133-134
    x = F.conv1d(F.silu(x), conv_weight(state, "head.conv_post"), state["head.conv_post.bias"], padding=(POST_K - 1) // 2)
    return torch.tanh(x)


def ffgan_forward(state, mel: torch.Tensor, polyphase: bool = False, skip_block=None, skip_resblock=None) -> torch.Tensor:
    """model.py:51-56: mel (B, 128, T) -> audio (B, 512·T)."""
    return head_forward(state, backbone_forward(state, mel, skip_block), polyphase, skip_resblock).squeeze(1)


def _is_layer_norm(name: str) -> bool:
    """backbone LayerNorm affines: the stem's (downsample_layers.0.1), the downsample layers' (downsample_layers.{1,2,3}.0),
    the blocks' (stages.*.norm) and the final one (backbone.norm)."""
    return bool(re.match(r"backbone\.(downsample_layers\.(0\.1|[123]\.0)\.|stages\.\d+\.\d+\.norm\.|norm\.)", name))


def make_state(seed: int = 21):
    """Seeded weights under the reference keys with O(1) gain per layer.  The reference's own init is nearly inert
    (layer scale 1e-6, HiFiGAN convs N(0, 0.01) with g = ||v||: audio std ~0.002), so fixtures from it would test
    almost nothing.  Here: conv / linear weights U(+-1/sqrt(fan_in)); LayerNorm affine near (1, 0); layer scale
    gamma ~ 0.3; weight-norm g of order 1 per dim-0 row.  The gains are kept low enough that the network stays well
    conditioned (a 1e-5 relative perturbation of every weight moves the audio by ~1e-4 max-rel), so that fixture parity
    pins the arithmetic rather than the rounding noise of an ill-conditioned network."""
    g = torch.Generator().manual_seed(seed)
    st = OrderedDict()

    def rnd(shape, lo=-1.0, hi=1.0):
        return lo + (hi - lo) * torch.rand(shape, generator=g)

    for name, shape in param_shapes().items():
        if name.endswith("original0"):
            continue                                           # drawn together with its v below
        if name.endswith("original1"):
            fan = shape[1] * shape[2]
            st[name] = rnd(shape) / math.sqrt(fan)
            gname = name[:-1] + "0"
            if ".ups." in name:
                # per INPUT channel: one output sample sees 2 of the 2u taps of all C_in rows -> gain^2 = g^2 C_in / (u C_out)
                u = shape[2] // 2
                gain = 1.2 * math.sqrt(u * shape[1] / shape[0])
            elif ".convs2." in name:
                gain = 0.5                                     # nine residual additions per ResBlock1
            else:
                gain = 6.0 if "conv_post" in name else 1.0     # conv_post: into tanh's nonlinear range
            st[gname] = gain * (1 + 0.1 * torch.randn(shape[0], 1, 1, generator=g))
        elif name.endswith("gamma"):
            st[name] = 0.3 * (1 + 0.3 * torch.randn(shape, generator=g))
        elif _is_layer_norm(name):
            st[name] = (1 + 0.1 * torch.randn(shape, generator=g)) if name.endswith("weight") else 0.1 * torch.randn(shape, generator=g)
        elif name.endswith(".weight"):
            fan = 1
            for k in shape[1:]:
                fan *= k
            st[name] = rnd(shape) / math.sqrt(fan)
        else:
            st[name] = 0.1 * rnd(shape)
    return OrderedDict((k, st[k]) for k in param_shapes())


def make_mel(seed: int, B: int, T: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N_MEL, T, generator=g)


def weight_checksum(state) -> float:
    return float(sum(float(v.double().sum()) for v in state.values()))


CASES = {
    "ffgan_b1_t1": dict(seed=51, B=1, T=1),
    "ffgan_b1_t3": dict(seed=52, B=1, T=3),
    "ffgan_b2_t37": dict(seed=53, B=2, T=37),
    "ffgan_b3_t130": dict(seed=54, B=3, T=130),
}
