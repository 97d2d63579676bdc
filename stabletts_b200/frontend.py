"""Drop-ins for the two small front-end modules of ``StableTTS.synthesise`` (models/model.py:78-80):

* ``MelStyleEncoder`` (models/reference_encoder.py:25-92): reference mel -> speaker vector ``c``;
* ``DurationPredictor`` (models/duration_predictor.py:5-36): text encoding + ``c`` -> ``logw``.

Same constructors, same ``forward`` signatures, same parameter names and default init as the reference; inference only
(eval semantics: dropout is the identity).  Each runs as one call into the CUDA library (``st_style_encoder_forward`` /
``st_duration_predictor_forward``).  Only the configuration ``StableTTS`` builds is implemented; other sizes raise
``ValueError``."""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib
from ._native import NativeModule


def _default_init(module: NativeModule, xavier=(), zeros=(), ones=()):
    """PyTorch's default Linear / Conv1d init, U(+-1/sqrt(fan_in)) for weight and bias, except the listed parameters."""
    with torch.no_grad():
        for name, shape in module._shapes.items():
            p = module._param(name)
            if name in xavier:
                nn.init.xavier_uniform_(p)
            elif name in zeros:
                p.zero_()
            elif name in ones:
                p.fill_(1.0)
            else:
                wshape = module._shapes[name.rsplit(".", 1)[0] + ".weight"]
                fan_in = math.prod(wshape[1:])
                p.uniform_(-1.0 / math.sqrt(fan_in), 1.0 / math.sqrt(fan_in))


class MelStyleEncoder(NativeModule):
    def __init__(self, n_mel_channels=80, style_hidden=128, style_vector_dim=256, style_kernel_size=5, style_head=2, dropout=0.1):
        super().__init__()
        if (style_hidden, style_vector_dim, style_kernel_size, style_head) != (128, 256, 5, 2):
            raise ValueError("MelStyleEncoder is built for style_hidden=128, style_vector_dim=256, style_kernel_size=5, "
                             "style_head=2 (the configuration StableTTS uses, models/model.py:38)")
        if n_mel_channels <= 0 or n_mel_channels % 16:
            raise ValueError("n_mel_channels must be a positive multiple of 16")
        self.in_dim = n_mel_channels
        self.hidden_dim = style_hidden
        self.out_dim = style_vector_dim
        self.kernel_size = style_kernel_size
        self.n_head = style_head
        self.dropout = dropout
        H, K = style_hidden, style_kernel_size
        s = OrderedDict()
        s["spectral.0.weight"], s["spectral.0.bias"] = (H, n_mel_channels), (H,)
        s["spectral.3.weight"], s["spectral.3.bias"] = (H, H), (H,)
        for i in range(2):
            s[f"temporal.{i}.conv1.weight"], s[f"temporal.{i}.conv1.bias"] = (2 * H, H, K), (2 * H,)
        s["slf_attn.in_proj_weight"], s["slf_attn.in_proj_bias"] = (3 * H, H), (3 * H,)
        s["slf_attn.out_proj.weight"], s["slf_attn.out_proj.bias"] = (H, H), (H,)
        s["fc.weight"], s["fc.bias"] = (style_vector_dim, H), (style_vector_dim,)
        self._shapes = s
        for name, shape in s.items():
            self._register(name, nn.Parameter(torch.empty(shape)))
        # nn.MultiheadAttention._reset_parameters: xavier in_proj_weight, zero biases
        _default_init(self, xavier=("slf_attn.in_proj_weight",), zeros=("slf_attn.in_proj_bias", "slf_attn.out_proj.bias"))
        self._init_native()

    def _create_handle(self, lib, index):
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_style_encoder(self.in_dim, index, C.byref(h)), "st_create_style_encoder")
        return h

    def forward(self, x: torch.Tensor, x_mask: torch.Tensor | None = None) -> torch.Tensor:
        """x: (B, n_mel, T) reference mel; x_mask: (B, 1, T) or None -> (B, style_vector_dim) (reference_encoder.py:77-92)."""
        self._refuse_training_graph("MelStyleEncoder.forward")
        with torch.no_grad():
            if not isinstance(x, torch.Tensor) or x.device.type != "cuda":
                raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
            B, M, T = x.shape
            y = self._f32c("x", x, (B, self.in_dim, T))
            out = torch.empty(B, self.out_dim, device=x.device, dtype=torch.float32)
            if B == 0:
                return out
            if T == 0:
                raise ValueError("MelStyleEncoder needs at least one reference frame (the temporal mean of zero frames is undefined)")
            m = None if x_mask is None else (x_mask.detach().reshape(B, T) != 0).to(torch.float32).contiguous()
            lib, h, stream = self._prepare(x)
            rc = lib.st_style_encoder_forward(h, y.data_ptr(), None if m is None else m.data_ptr(), out.data_ptr(), B, T, stream)
            _lib.check(lib, h, rc, "st_style_encoder_forward")
            return out.to(x.dtype)


class DurationPredictor(NativeModule):
    def __init__(self, in_channels, filter_channels, kernel_size, p_dropout, gin_channels=0):
        super().__init__()
        if (in_channels, filter_channels, kernel_size, gin_channels) != (256, 1024, 3, 256):
            raise ValueError("DurationPredictor is built for in_channels=256, filter_channels=1024, kernel_size=3, "
                             "gin_channels=256 (the configuration StableTTS uses, models/model.py:39)")
        self.in_channels = in_channels
        self.filter_channels = filter_channels
        self.kernel_size = kernel_size
        self.p_dropout = p_dropout
        self.gin_channels = gin_channels
        F_, I, K = filter_channels, in_channels, kernel_size
        s = OrderedDict()
        s["conv1.weight"], s["conv1.bias"] = (F_, I, K), (F_,)
        s["norm1.weight"], s["norm1.bias"] = (F_,), (F_,)
        s["conv2.weight"], s["conv2.bias"] = (F_, F_, K), (F_,)
        s["norm2.weight"], s["norm2.bias"] = (F_,), (F_,)
        s["proj.weight"], s["proj.bias"] = (1, F_, 1), (1,)
        s["cond.weight"], s["cond.bias"] = (I, gin_channels, 1), (I,)
        self._shapes = s
        for name, shape in s.items():
            self._register(name, nn.Parameter(torch.empty(shape)))
        _default_init(self, ones=("norm1.weight", "norm2.weight"), zeros=("norm1.bias", "norm2.bias"))
        self._init_native()

    def _create_handle(self, lib, index):
        dims = _lib.StDims(80, self.in_channels, self.filter_channels, 4, 6, self.kernel_size, self.gin_channels)
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_duration_predictor(C.byref(dims), index, C.byref(h)), "st_create_duration_predictor")
        return h

    def forward(self, x: torch.Tensor, x_mask: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
        """x: (B, in_channels, Tx); x_mask: (B, 1, Tx); g: (B, gin_channels) -> logw (B, 1, Tx) (duration_predictor.py:22-36)."""
        self._refuse_training_graph("DurationPredictor.forward")
        with torch.no_grad():
            if not isinstance(x, torch.Tensor) or x.device.type != "cuda":
                raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
            B, _, Tx = x.shape
            x_ = self._f32c("x", x, (B, self.in_channels, Tx))
            m_ = self._f32c("x_mask", x_mask, (B, 1, Tx))
            g_ = self._f32c("g", g, (B, self.gin_channels))
            logw = torch.empty(B, 1, Tx, device=x.device, dtype=torch.float32)
            if B == 0 or Tx == 0:
                return logw
            lib, h, stream = self._prepare(x)
            rc = lib.st_duration_predictor_forward(h, x_.data_ptr(), m_.data_ptr(), g_.data_ptr(), logw.data_ptr(), B, Tx, stream)
            _lib.check(lib, h, rc, "st_duration_predictor_forward")
            return logw.to(x.dtype)
