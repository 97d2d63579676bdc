"""Drop-in for the reference's ``models.estimator.Decoder`` (models/estimator.py:65-137).

Same constructor signature, same ``forward(t, x, mask, mu, c)``, same parameter names/shapes
(``state_dict()`` carries the reference's 116 ``estimator.*``-relative keys, so checkpoints saved
by the reference load unchanged, api.py:49) — but the computation is one call into the sm_90a
CUDA library through the C ABI (include/stabletts_b200.h).  Parameters live in ordinary
``nn.Parameter`` s (so ``.to()``, ``.eval()``, ``.parameters()`` behave); the library keeps its own
packed copy which is refreshed whenever a parameter's version counter or device changes.

No CPU fallback: tensors must be CUDA fp32; anything else raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from collections import OrderedDict
from typing import Dict, Tuple

import torch
import torch.nn as nn

from . import _lib
from ._native import NativeModule


def _param_shapes(n_mel, hidden, filt, n_layers, kernel, gin) -> "OrderedDict[str, Tuple[int, ...]]":
    """Parameter inventory of Decoder.__init__ (models/estimator.py:66-96) in registration order."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()

    def wb(name, *shape):
        s[name + ".weight"] = tuple(shape)
        s[name + ".bias"] = (shape[0],)

    wb("time_mlp.layer.0", filt, hidden)                       # :55-59
    wb("time_mlp.layer.2", hidden, filt)
    wb("in_proj", hidden, hidden + n_mel, 1)                   # :78
    for i in range(n_layers):                                  # :79
        p = f"blocks.{i}."
        wb(p + "time_fusion.film", 2 * hidden, hidden, 1)      # :28
        for n in "qkv":
            wb(p + f"block.attn.conv_{n}", hidden, hidden, 1)  # diffusion_transformer.py:43-45
        wb(p + "block.attn.conv_o", hidden, hidden, 1)         # :51
        wb(p + "block.mlp.conv_1", filt, hidden, kernel)       # :20
        wb(p + "block.mlp.conv_2", hidden, filt, kernel)       # :21
        wb(p + "block.adaLN_modulation.2", 6 * hidden, hidden)  # :92-96 (0 = Identity, 1 = SiLU)
    wb("final_proj", n_mel, hidden, 1)                         # :80
    wb("cond_proj.0", filt, n_mel, kernel)                     # :83-89
    wb("cond_proj.2", filt, filt, kernel)
    wb("cond_proj.4", hidden, filt, kernel)
    for i in range(n_layers // 2):
        wb(f"lsc_layers.{i}", hidden, 2 * hidden, kernel)      # :94
    return s


class Decoder(NativeModule):
    def __init__(self, noise_channels, cond_channels, hidden_channels, out_channels, filter_channels, dropout=0.1,
                 n_layers=1, n_heads=4, kernel_size=3, gin_channels=0, use_lsc=True):
        super().__init__()
        if not (noise_channels == cond_channels == out_channels):
            raise ValueError("noise/cond/out channels must all equal n_mel (as models/model.py:40 builds it)")
        if not use_lsc:
            raise ValueError("use_lsc=False is not built (the reference never constructs it)")
        if gin_channels != hidden_channels:
            raise ValueError("gin_channels must equal hidden_channels (adaLN_modulation.0 is Identity)")
        self.noise_channels = noise_channels
        self.cond_channels = cond_channels
        self.hidden_channels = hidden_channels
        self.out_channels = out_channels
        self.filter_channels = filter_channels
        self.use_lsc = use_lsc
        self.n_layers, self.n_heads, self.kernel_size, self.gin_channels = n_layers, n_heads, kernel_size, gin_channels
        self.n_lsc_layers = n_layers // 2
        self._shapes = _param_shapes(noise_channels, hidden_channels, filter_channels, n_layers, kernel_size, gin_channels)
        for name, shape in self._shapes.items():
            self._register(name, nn.Parameter(torch.empty(shape)))
        self.initialize_weights()
        self._init_native()                # library state (not part of the module state)

    def _create_handle(self, lib, index):
        dims = _lib.StDims(self.noise_channels, self.hidden_channels, self.filter_channels, self.n_heads,
                           self.n_layers, self.kernel_size, self.gin_channels)
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create(C.byref(dims), index, C.byref(h)), "st_create")
        return h


    def initialize_weights(self):
        """PyTorch default Conv1d/Linear init (U(±1/sqrt(fan_in)) for weight and bias), xavier on the
        q/k/v projections (diffusion_transformer.py:54-56), zero adaLN gates (estimator.py:98-101)."""
        with torch.no_grad():
            for name, shape in self._shapes.items():
                p = self._param(name)
                base = name.rsplit(".", 1)[0]
                wshape = self._shapes[base + ".weight"]
                fan_in = 1
                for d in wshape[1:]:
                    fan_in *= d
                if "adaLN_modulation.2" in name:
                    p.zero_()
                elif name.endswith(".weight") and any(k in name for k in ("conv_q", "conv_k", "conv_v")):
                    nn.init.xavier_uniform_(p)
                else:
                    bound = 1.0 / math.sqrt(fan_in)
                    p.uniform_(-bound, bound)


    # -- the reference's forward ------------------------------------------------------------------
    def forward(self, t, x, mask, mu, c):
        self._refuse_training_graph("Decoder.forward")      # checked BEFORE autograd is switched off below
        with torch.no_grad():
            return self._forward_impl(t, x, mask, mu, c)

    def _forward_impl(self, t, x, mask, mu, c):
        """models/estimator.py:103-137.  t: 0-dim or (B,); x, mu: (B, n_mel, T); mask: (B, 1, T)
        float {0,1}; c: (B, gin).  Returns (B, n_mel, T), exactly 0 at masked frames."""
        B, M, T = x.shape
        x = self._f32c("x", x, (B, self.noise_channels, T))
        mu = self._f32c("mu", mu, (B, self.cond_channels, T))
        mask = self._f32c("mask", mask, (B, 1, T))
        c = self._f32c("c", c, (B, self.gin_channels))
        t = torch.as_tensor(t, dtype=torch.float32, device=x.device).reshape(-1).contiguous()
        if t.numel() not in (1, B) and B > 0:
            raise ValueError("t must be 0-dim or have shape (B,)")
        if B == 0 or T == 0:                    # empty batch / zero frames: the reference returns an empty tensor
            return torch.empty_like(x)
        lib, h, stream = self._prepare(x, B, T, 0)
        out = torch.empty_like(x)
        rc = lib.st_estimator_forward(h, t.data_ptr(), t.numel(), x.data_ptr(), mask.data_ptr(), mu.data_ptr(),
                                      c.data_ptr(), out.data_ptr(), B, T, stream)
        _lib.check(lib, h, rc, "st_estimator_forward")
        return out
