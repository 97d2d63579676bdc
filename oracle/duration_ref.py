"""CPU oracle for the DurationPredictor (TEST INFRASTRUCTURE ONLY): functional restatement of
models/duration_predictor.py:5-36 as StableTTS builds it (models/model.py:39: in 256, filter 1024, kernel 3), eval mode.
Pinned by tests/test_synthesise.py against tests/golden/dp_*.npz (oracle/make_golden_synth.py, unmodified reference)."""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

IN, FILT, KERNEL, GIN = 256, 1024, 3, 256


def param_shapes():
    s = OrderedDict()
    s["conv1.weight"], s["conv1.bias"] = (FILT, IN, KERNEL), (FILT,)
    s["norm1.weight"], s["norm1.bias"] = (FILT,), (FILT,)
    s["conv2.weight"], s["conv2.bias"] = (FILT, FILT, KERNEL), (FILT,)
    s["norm2.weight"], s["norm2.bias"] = (FILT,), (FILT,)
    s["proj.weight"], s["proj.bias"] = (1, FILT, 1), (1,)
    s["cond.weight"], s["cond.bias"] = (IN, GIN, 1), (IN,)
    return s


def make_state(seed=32):
    """Convs U(+-1/sqrt(fan_in)); LayerNorm affine 1 + 0.1 N(0,1) / 0.1 N(0,1) so it is observable; proj.bias = log 4
    so that durations are a realistic 2-8 frames rather than about 1."""
    g = torch.Generator().manual_seed(seed)
    st = OrderedDict()
    for name, shape in param_shapes().items():
        if name.startswith("norm"):
            r = torch.randn(shape, generator=g) * 0.1
            st[name] = 1.0 + r if name.endswith("weight") else r
            continue
        wshape = param_shapes()[name.rsplit(".", 1)[0] + ".weight"]
        st[name] = (torch.rand(shape, generator=g) * 2 - 1) / math.prod(wshape[1:]) ** 0.5
    st["proj.bias"] = torch.tensor([math.log(4.0)])
    return st


def dp_forward(state, x, x_mask, g):
    """duration_predictor.py:22-36.  x (B, 256, Tx), x_mask (B, 1, Tx), g (B, 256) -> logw (B, 1, Tx)."""
    x = x + F.conv1d(g.unsqueeze(2), state["cond.weight"], state["cond.bias"])
    for i in (1, 2):
        x = torch.relu(F.conv1d(x * x_mask, state[f"conv{i}.weight"], state[f"conv{i}.bias"], padding=KERNEL // 2))
        x = F.layer_norm(x.transpose(1, 2), (FILT,), state[f"norm{i}.weight"], state[f"norm{i}.bias"], 1e-5).transpose(1, 2)
    return F.conv1d(x * x_mask, state["proj.weight"], state["proj.bias"]) * x_mask


def make_inputs(seed, lens, Tx):
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    mask = (torch.arange(Tx)[None] < torch.as_tensor(lens)[:, None]).float().unsqueeze(1)
    x = torch.randn(B, IN, Tx, generator=g) * mask          # a text encoding is masked (models/text_encoder.py:40)
    c = torch.randn(B, GIN, generator=g)
    return x, mask, c


CASES = {
    "dp_t1":   dict(seed=71, lens=[1], Tx=1),
    "dp_t37":  dict(seed=72, lens=[37, 20, 1], Tx=37),
    "dp_t129": dict(seed=73, lens=[129, 100], Tx=129),
}
