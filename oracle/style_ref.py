"""CPU oracle for the MelStyleEncoder (TEST INFRASTRUCTURE ONLY): functional restatement of
models/reference_encoder.py:4-92 as StableTTS builds it (models/model.py:38: style_hidden 128, style_vector_dim 256,
kernel 5, 2 heads), eval mode.  Pinned by tests/test_synthesise.py against tests/golden/style_*.npz, which
oracle/make_golden_synth.py writes from the unmodified reference module."""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

HIDDEN, OUT, KERNEL, HEADS = 128, 256, 5, 2


def param_shapes(n_mel=80):
    s = OrderedDict()
    s["spectral.0.weight"], s["spectral.0.bias"] = (HIDDEN, n_mel), (HIDDEN,)
    s["spectral.3.weight"], s["spectral.3.bias"] = (HIDDEN, HIDDEN), (HIDDEN,)
    for i in range(2):
        s[f"temporal.{i}.conv1.weight"], s[f"temporal.{i}.conv1.bias"] = (2 * HIDDEN, HIDDEN, KERNEL), (2 * HIDDEN,)
    s["slf_attn.in_proj_weight"], s["slf_attn.in_proj_bias"] = (3 * HIDDEN, HIDDEN), (3 * HIDDEN,)
    s["slf_attn.out_proj.weight"], s["slf_attn.out_proj.bias"] = (HIDDEN, HIDDEN), (HIDDEN,)
    s["fc.weight"], s["fc.bias"] = (OUT, HIDDEN), (OUT,)
    return s


def make_state(seed=31, n_mel=80):
    """U(+-1/sqrt(fan_in)) for every tensor (the reference's zero in_proj / out_proj biases would leave them untested)."""
    g = torch.Generator().manual_seed(seed)
    shapes = param_shapes(n_mel)
    st = OrderedDict()
    for name, shape in shapes.items():
        wname = name.replace("in_proj_bias", "in_proj_weight").replace(".bias", ".weight")
        st[name] = (torch.rand(shape, generator=g) * 2 - 1) / math.prod(shapes[wname][1:]) ** 0.5
    return st


def mish(x):
    return x * torch.tanh(F.softplus(x))


def style_forward(state, y, x_mask=None):
    """reference_encoder.py:77-92.  y (B, M, T), x_mask (B, 1, T) or None -> (B, 256)."""
    x = y.transpose(1, 2)
    x = mish(F.linear(x, state["spectral.0.weight"], state["spectral.0.bias"]))            # :47-49
    x = mish(F.linear(x, state["spectral.3.weight"], state["spectral.3.bias"]))            # :50-52
    x = x.transpose(1, 2)
    for i in range(2):                                                                      # Conv1dGLU, :16-21 (unmasked)
        h = F.conv1d(x, state[f"temporal.{i}.conv1.weight"], state[f"temporal.{i}.conv1.bias"], padding=KERNEL // 2)
        a, gte = h.split(HIDDEN, dim=1)
        x = x + a * torch.sigmoid(gte)
    x = x.transpose(1, 2)                                                                   # (B, T, H)
    B, T, H = x.shape
    q, k, v = F.linear(x, state["slf_attn.in_proj_weight"], state["slf_attn.in_proj_bias"]).chunk(3, dim=-1)
    heads = lambda z: z.reshape(B, T, HEADS, H // HEADS).transpose(1, 2)                   # noqa: E731
    s = heads(q) @ heads(k).transpose(-1, -2) / (H // HEADS) ** 0.5
    valid = None if x_mask is None else x_mask.reshape(B, T) != 0
    if valid is not None:                                                                   # key_padding_mask = ~x_mask
        s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
    o = (torch.softmax(s, dim=-1) @ heads(v)).transpose(1, 2).reshape(B, T, H)
    o = F.linear(o, state["slf_attn.out_proj.weight"], state["slf_attn.out_proj.bias"])
    o = F.linear(o, state["fc.weight"], state["fc.bias"])                                   # :89
    if valid is None:                                                                       # temporal_avg_pool, :71-75
        return o.mean(dim=1)
    return (o * valid[..., None]).sum(dim=1) / valid.sum(dim=1, keepdim=True)


def make_inputs(seed, B, T, n_mel, lens=None):
    """A log-mel-like reference (N(-4, 2^2)) and, when lens is given, its (B, 1, T) prefix mask."""
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(B, n_mel, T, generator=g) * 2.0 - 4.0
    mask = None if lens is None else (torch.arange(T)[None] < torch.as_tensor(lens)[:, None]).float().unsqueeze(1)
    return y, mask


CASES = {
    "style_t1_m80":      dict(seed=61, B=1, T=1, n_mel=80, lens=None),
    "style_t4_m128":     dict(seed=62, B=2, T=4, n_mel=128, lens=[4, 2]),
    "style_t129_m80":    dict(seed=63, B=3, T=129, n_mel=80, lens=[129, 77, 5]),
    "style_t129_nomask": dict(seed=64, B=2, T=129, n_mel=128, lens=None),
    "style_t700_m128":   dict(seed=65, B=1, T=700, n_mel=128, lens=None),
}
