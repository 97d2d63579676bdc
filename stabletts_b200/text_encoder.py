"""Drop-in for the reference's ``models.text_encoder.TextEncoder`` (models/text_encoder.py:8-44) —
SURVEY.md §8 row f2.  Same constructor, same ``forward(x, c, x_lengths) -> (x, mu_x, x_mask)``, same
parameter names (``emb``, ``encoder.{i}.attn.conv_*``, ``encoder.{i}.mlp.conv_*``,
``encoder.{i}.adaLN_modulation.2``, ``proj``); the three DiTConVBlocks run on exactly the kernels of the
CFM estimator (LayerNorm+modulate, wgmma QKV/RoPE, flash attention, O, FFN convs)."""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib
from ._native import NativeModule


def _param_shapes(n_vocab, out_channels, hidden, filt, n_layers, kernel):
    s = OrderedDict()

    def wb(name, *shape):
        s[name + ".weight"] = tuple(shape)
        s[name + ".bias"] = (shape[0],)

    s["emb.weight"] = (n_vocab, hidden)                           # :22
    for i in range(n_layers):                                      # :25
        p = f"encoder.{i}."
        for n in "qkv":
            wb(p + f"attn.conv_{n}", hidden, hidden, 1)
        wb(p + "attn.conv_o", hidden, hidden, 1)
        wb(p + "mlp.conv_1", filt, hidden, kernel)
        wb(p + "mlp.conv_2", hidden, filt, kernel)
        wb(p + "adaLN_modulation.2", 6 * hidden, hidden)
    wb("proj", out_channels, hidden, 1)                           # :26
    return s


class TextEncoder(NativeModule):
    def __init__(self, n_vocab, out_channels, hidden_channels, filter_channels, n_heads, n_layers, kernel_size, p_dropout,
                 gin_channels):
        super().__init__()
        if gin_channels != hidden_channels:
            raise ValueError("gin_channels must equal hidden_channels (adaLN_modulation.0 is Identity)")
        self.n_vocab = n_vocab
        self.out_channels = out_channels
        self.hidden_channels = hidden_channels
        self.filter_channels = filter_channels
        self.n_heads = n_heads
        self.n_layers = n_layers
        self.kernel_size = kernel_size
        self.p_dropout = p_dropout
        self.gin_channels = gin_channels
        self.scale = self.hidden_channels ** 0.5
        self._shapes = _param_shapes(n_vocab, out_channels, hidden_channels, filter_channels, n_layers, kernel_size)
        for name, shape in self._shapes.items():
            self._register(name, nn.Parameter(torch.empty(shape)))
        self.initialize_weights()
        self._init_native()

    def _create_handle(self, lib, index):
        dims = _lib.StDims(self.out_channels, self.hidden_channels, self.filter_channels, self.n_heads, self.n_layers,
                           self.kernel_size, self.gin_channels)
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_text_encoder(C.byref(dims), self.n_vocab, index, C.byref(h)), "st_create_text_encoder")
        return h

    def initialize_weights(self):
        """emb ~ N(0, hidden^-0.5) (:23); PyTorch default conv init; xavier q/k/v; zero adaLN gates (:30-33)."""
        with torch.no_grad():
            for name, shape in self._shapes.items():
                p = self._param(name)
                if name == "emb.weight":
                    nn.init.normal_(p, 0.0, self.hidden_channels ** -0.5)
                    continue
                wshape = self._shapes[name.rsplit(".", 1)[0] + ".weight"]
                fan_in = 1
                for d in wshape[1:]:
                    fan_in *= d
                if "adaLN_modulation.2" in name:
                    p.zero_()
                elif name.endswith(".weight") and any(k in name for k in ("conv_q", "conv_k", "conv_v")):
                    nn.init.xavier_uniform_(p)
                else:
                    p.uniform_(-1.0 / math.sqrt(fan_in), 1.0 / math.sqrt(fan_in))

    def forward(self, x: torch.Tensor, c: torch.Tensor, x_lengths: torch.Tensor):
        self._refuse_training_graph("TextEncoder.forward")      # checked BEFORE autograd is switched off below
        with torch.no_grad():
            return self._forward_impl(x, c, x_lengths)

    def _forward_impl(self, x: torch.Tensor, c: torch.Tensor, x_lengths: torch.Tensor):
        """x: (B, T) int64 token ids; c: (B, gin); x_lengths: (B,).  Returns x (B, hidden, T), mu_x (B, out, T),
        x_mask (B, 1, T) — models/text_encoder.py:34-44."""
        if x.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        B, T = x.shape
        ids = x.detach().to(torch.int64).contiguous()
        lens = x_lengths.detach().to(device=x.device, dtype=torch.int64).contiguous()
        c_ = self._f32c("c", c, (B, self.gin_channels))
        xo = torch.empty(B, self.hidden_channels, T, device=x.device, dtype=torch.float32)
        mu = torch.empty(B, self.out_channels, T, device=x.device, dtype=torch.float32)
        mask = torch.empty(B, 1, T, device=x.device, dtype=torch.float32)
        if B == 0 or T == 0:                    # empty batch / zero tokens: empty tensors, like Decoder / CFMDecoder
            return xo, mu, mask
        # nn.Embedding raises on ids outside [0, n_vocab) (models/text_encoder.py:22,35); a silently clamped id would
        # turn a tokenizer/vocabulary mismatch into plausible-looking output, so validate (one host read per call)
        if bool(((ids < 0) | (ids >= self.n_vocab)).any()):
            raise IndexError(f"token id out of range [0, {self.n_vocab}) in TextEncoder input")
        lib, h, stream = self._prepare(c_, B, T, 0)
        rc = lib.st_text_encoder_forward(h, ids.data_ptr(), c_.data_ptr(), lens.data_ptr(), xo.data_ptr(), mu.data_ptr(),
                                         mask.data_ptr(), B, T, stream)
        _lib.check(lib, h, rc, "st_text_encoder_forward")
        return xo, mu, mask
