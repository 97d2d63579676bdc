"""Drop-in for the reference's Vocos vocoder (vocoders/vocos/models/model.py:11-20), the step right after the CFM path
(api.py:76 ``audio_output = self.vocoder_model(mel_output)``; SURVEY.md §8 row f4).

Same ``forward(mel) -> audio`` and the reference's own ``state_dict`` keys (``backbone.embed.*``, ``backbone.norm.*``,
``backbone.convnext.{i}.{gamma, dwconv.*, norm.*, pwconv1.*, pwconv2.*}``, ``backbone.final_layer_norm.*``,
``head.out.*`` and the buffer ``head.istft.window``), so ``load_state_dict(torch.load('vocos.pt'))`` (api.py:54-56) works
unchanged.  The computation is one call into the sm_90a library: conv-GEMMs on the wgmma engine (k = 7 embed conv,
pwconv1 + GELU, pwconv2 + layer scale + residual, the head, and the inverse STFT as ONE windowed inverse-DFT contraction),
row kernels for depthwise-conv + LayerNorm, and a 4-frame overlap-add gather.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib
from ._native import NativeModule, _Node


def _param_shapes(input_channels, dim, intermediate_dim, num_layers, n_fft):
    """Parameter inventory of VocosBackbone / ConvNeXtBlock / ISTFTHead in the reference's registration order."""
    s = OrderedDict()
    s["backbone.embed.weight"] = (dim, input_channels, 7); s["backbone.embed.bias"] = (dim,)            # backbone.py:30
    s["backbone.norm.weight"] = (dim,); s["backbone.norm.bias"] = (dim,)                                 # :31
    for i in range(num_layers):                                                                          # :33-42
        p = f"backbone.convnext.{i}."
        s[p + "gamma"] = (dim,)                                                                          # module.py:27-31
        s[p + "dwconv.weight"] = (dim, 1, 7); s[p + "dwconv.bias"] = (dim,)                              # :22
        s[p + "norm.weight"] = (dim,); s[p + "norm.bias"] = (dim,)                                       # :23
        s[p + "pwconv1.weight"] = (intermediate_dim, dim); s[p + "pwconv1.bias"] = (intermediate_dim,)   # :24
        s[p + "pwconv2.weight"] = (dim, intermediate_dim); s[p + "pwconv2.bias"] = (dim,)                # :26
    s["backbone.final_layer_norm.weight"] = (dim,); s["backbone.final_layer_norm.bias"] = (dim,)         # backbone.py:43
    s["head.out.weight"] = (n_fft + 2, dim); s["head.out.bias"] = (n_fft + 2,)                           # head.py:98-99
    return s


class Vocos(NativeModule):
    """``Vocos(input_channels=128, dim=768, intermediate_dim=2048, num_layers=12, n_fft=2048, hop_length=512)`` — the
    fields of the reference's ``VocosConfig`` / ``MelConfig`` (vocoders/vocos/config.py) as keyword arguments; the
    reference's own call ``Vocos(VocosConfig(), MelConfig())`` is accepted too (dataclass instances are unpacked)."""

    def __init__(self, input_channels=128, dim=768, intermediate_dim=2048, num_layers=12, n_fft=2048, hop_length=512):
        super().__init__()
        if hasattr(input_channels, "__dataclass_fields__"):            # Vocos(vocos_config, mel_config), model.py:12
            vc, mc = input_channels, dim
            input_channels, dim, intermediate_dim, num_layers = vc.input_channels, vc.dim, vc.intermediate_dim, vc.num_layers
            n_fft, hop_length = mc.n_fft, mc.hop_length
        self.input_channels, self.dim, self.intermediate_dim, self.num_layers = input_channels, dim, intermediate_dim, num_layers
        self.n_fft, self.hop_length = n_fft, hop_length
        self._shapes = _param_shapes(input_channels, dim, intermediate_dim, num_layers, n_fft)
        for name, shape in self._shapes.items():
            self._register(name, nn.Parameter(torch.empty(shape)))
        # ISTFT registers its Hann window as a buffer (head.py:28-29): part of the state_dict, not a parameter
        head = self._modules["head"]                                    # created by registering head.out.*
        head.add_module("istft", _Node())
        head._modules["istft"].register_buffer("window", torch.hann_window(n_fft))
        self.initialize_weights()
        self._init_native()

    def initialize_weights(self):
        """backbone.py:46-49: trunc_normal(0.02) conv / linear weights, zero biases; LayerNorm (1, 0); gamma = 1/num_layers
        (:32); the head keeps nn.Linear's default init (it is outside the backbone's ``apply``)."""
        with torch.no_grad():
            for name, shape in self._shapes.items():
                p = self._param(name)
                if name.endswith("gamma"):
                    p.fill_(1.0 / self.num_layers)
                elif ".norm." in name or "final_layer_norm" in name:
                    p.fill_(1.0 if name.endswith("weight") else 0.0)
                elif name.startswith("head.out"):
                    bound = 1.0 / (self.dim ** 0.5)
                    p.uniform_(-bound, bound)
                elif name.endswith(".weight"):
                    nn.init.trunc_normal_(p, std=0.02)
                else:
                    p.zero_()

    def _create_handle(self, lib, index):
        dims = _lib.StVocosDims(self.input_channels, self.dim, self.intermediate_dim, self.num_layers, self.n_fft, self.hop_length)
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_vocos(C.byref(dims), index, C.byref(h)), "st_create_vocos")
        return h

    def _sync_weights(self, lib, h, stream: int, force: bool = False) -> None:
        """Parameters through the base class; the window buffer rides along under its state_dict key."""
        win = self._modules["head"]._modules["istft"]._buffers["window"]
        tag = (win.data_ptr(), win._version)
        if force or self._synced.get("head.istft.window") != tag:
            self._synced.pop(next(iter(self._shapes)), None)            # force the base class to re-finalize
            wc = win.detach().to(torch.float32).contiguous()
            _lib.check(lib, h, lib.st_load_weight(h, b"head.istft.window", wc.data_ptr(), wc.numel(), stream), "st_load_weight(window)")
            self._synced["head.istft.window"] = tag
        super()._sync_weights(lib, h, stream, force)

    def _ensure_workspace(self, lib, h, B, T, cfg, device) -> None:     # the vocoder handle owns its workspace
        return None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """mel (B, input_channels, T) -> audio (B, T * hop_length) — model.py:17-20."""
        self._refuse_training_graph("Vocos.forward")
        with torch.no_grad():
            B, M, T = x.shape
            mel = self._f32c("mel", x, (B, self.input_channels, T))
            audio = torch.empty(B, T * self.hop_length, device=x.device, dtype=torch.float32)
            if B == 0 or T == 0:
                return audio
            lib, h, stream = self._prepare(mel, B, T, 0)
            rc = lib.st_vocos_forward(h, mel.data_ptr(), audio.data_ptr(), B, T, stream)
            _lib.check(lib, h, rc, "st_vocos_forward")
            return audio

