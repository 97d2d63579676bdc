"""Drop-in for the reference's default vocoder, FireflyGAN (vocoders/ffgan/model.py: ``FireflyGANBase`` /
``FireflyGANBaseWrapper``; api.py ``get_vocoder(..., model_name='ffgan')``).

Same ``forward(mel) -> audio`` and the reference's own ``state_dict`` (471 tensors: ``backbone.*`` of the ConvNeXt encoder,
``head.*`` of the HiFiGAN generator with its weight-norm parametrizations ``...parametrizations.weight.original0/1``), so the
published generator checkpoint loads unchanged; checkpoints written with the legacy ``weight_g`` / ``weight_v`` names load
too.  The computation is one call into the sm_90a library (st_ffgan_forward): conv-GEMMs on the wgmma engine for every
convolution — the transposed ones as 3-tap polyphase convs at their input rate, the ResBlock1 convs with dilated taps — and
row kernels for the LayerNorms, the ParralelBlock mean and conv_post + tanh.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import re

import torch
import torch.nn as nn

from . import _lib
from ._native import NativeModule

_G, _V = ".parametrizations.weight.original0", ".parametrizations.weight.original1"
# the encoder's LayerNorm affines: stem, downsample layers 1-3, every block, the final one
_LAYER_NORM = re.compile(r"backbone\.(downsample_layers\.(0\.1|[123]\.0)\.|stages\.\d+\.\d+\.norm\.|norm\.)")


def _param_shapes():
    """The reference's state_dict inventory in its registration order (backbone.py:146-214, head.py:137-223)."""
    from collections import OrderedDict
    dims, depths, mel, c0 = (128, 256, 384, 512), (3, 3, 9, 3), 128, 512
    s = OrderedDict()

    def wn(name, shape):
        s[name + _G] = (shape[0], 1, 1)
        s[name + _V] = shape

    s["backbone.downsample_layers.0.0.weight"] = (dims[0], mel, 7); s["backbone.downsample_layers.0.0.bias"] = (dims[0],)
    s["backbone.downsample_layers.0.1.weight"] = (dims[0],); s["backbone.downsample_layers.0.1.bias"] = (dims[0],)
    for i in range(1, 4):
        p = f"backbone.downsample_layers.{i}."
        s[p + "0.weight"] = (dims[i - 1],); s[p + "0.bias"] = (dims[i - 1],)
        s[p + "1.weight"] = (dims[i], dims[i - 1], 1); s[p + "1.bias"] = (dims[i],)
    for i, (depth, d) in enumerate(zip(depths, dims)):
        for j in range(depth):
            p = f"backbone.stages.{i}.{j}."
            s[p + "gamma"] = (d,)
            s[p + "dwconv.weight"] = (d, 1, 7); s[p + "dwconv.bias"] = (d,)
            s[p + "norm.weight"] = (d,); s[p + "norm.bias"] = (d,)
            s[p + "pwconv1.weight"] = (4 * d, d); s[p + "pwconv1.bias"] = (4 * d,)
            s[p + "pwconv2.weight"] = (d, 4 * d); s[p + "pwconv2.bias"] = (d,)
    s["backbone.norm.weight"] = (dims[-1],); s["backbone.norm.bias"] = (dims[-1],)
    s["head.conv_pre.bias"] = (c0,); wn("head.conv_pre", (c0, c0, 13))
    for i, k in enumerate((16, 16, 4, 4, 4)):
        s[f"head.ups.{i}.bias"] = (c0 >> (i + 1),); wn(f"head.ups.{i}", (c0 >> i, c0 >> (i + 1), k))
    for i in range(5):
        c = c0 >> (i + 1)
        for b, k in enumerate((3, 7, 11)):
            for which in ("convs1", "convs2"):
                for j in range(3):
                    name = f"head.resblocks.{i}.blocks.{b}.{which}.{j}"
                    s[name + ".bias"] = (c,); wn(name, (c, c, k))
    s["head.conv_post.bias"] = (1,); wn("head.conv_post", (1, c0 >> 5, 13))
    return s


def _weight_norm_compat(state_dict, prefix, *args):
    """Legacy torch.nn.utils.weight_norm checkpoints name g / v ``weight_g`` / ``weight_v``; rename them to the
    parametrization keys, as torch's own ``_weight_norm_compat_hook`` does for a parametrized module."""
    for key in [k for k in state_dict if k.startswith(prefix) and (k.endswith(".weight_g") or k.endswith(".weight_v"))]:
        base = key[:-len(".weight_g")]
        state_dict[base + (_G if key.endswith("_g") else _V)] = state_dict.pop(key)


class FireflyGANBase(NativeModule):
    """``FireflyGANBase()`` — the reference's one configuration (model.py:7-29); ``forward(mel (B, 128, T)) -> (B, 512 T)``."""

    n_mel, hop_length = 128, 512

    def __init__(self):
        super().__init__()
        self._shapes = _param_shapes()
        for name, shape in self._shapes.items():
            self._register(name, nn.Parameter(torch.empty(shape)))
        self._register_load_state_dict_pre_hook(_weight_norm_compat)
        self.initialize_weights()
        self._init_native()

    def initialize_weights(self):
        """The reference's init: trunc_normal(0.02) conv / linear weights and zero biases in the backbone
        (backbone.py:201-204), LayerNorm (1, 0), layer scale 1e-6 (:117-121); HiFiGAN convs N(0, 0.01) (head.py:15-18) with
        weight_norm's g = ||v|| and nn.Conv1d's default bias init."""
        with torch.no_grad():
            for name, shape in self._shapes.items():
                p = self._param(name)
                if name.startswith("backbone."):
                    if name.endswith("gamma"):
                        p.fill_(1e-6)
                    elif len(shape) == 1:
                        p.fill_(1.0 if name.endswith("weight") and _LAYER_NORM.match(name) else 0.0)
                    else:
                        nn.init.trunc_normal_(p, std=0.02)
                elif name.endswith(_V):
                    p.normal_(0.0, 0.01)
                    g = self._param(name[:-1] + "0")
                    g.copy_(p.reshape(shape[0], -1).norm(dim=1).reshape(-1, 1, 1))
                elif name.endswith(".bias"):
                    v_shape = self._shapes[name[:-len(".bias")] + _V]
                    bound = 1.0 / (v_shape[1] * v_shape[2]) ** 0.5
                    p.uniform_(-bound, bound)

    def _create_handle(self, lib, index):
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_ffgan(index, C.byref(h)), "st_create_ffgan")
        return h

    def workspace_bytes(self, B: int, T: int) -> int:
        """Device memory st_ffgan_forward holds for a (B, T) call (256 KB per mel frame)."""
        return int(_lib.load_library().st_ffgan_workspace_bytes(None, B, T))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """mel (B, 128, T) -> audio (B, 512 T) — model.py:51-56."""
        self._refuse_training_graph("FireflyGANBase.forward")
        with torch.no_grad():
            B, M, T = x.shape
            mel = self._f32c("mel", x, (B, self.n_mel, T))
            audio = torch.empty(B, T * self.hop_length, device=x.device, dtype=torch.float32)
            if B == 0 or T == 0:
                return audio
            lib, h, stream = self._prepare(mel)
            _lib.check(lib, h, lib.st_ffgan_forward(h, mel.data_ptr(), audio.data_ptr(), B, T, stream), "st_ffgan_forward")
            return audio


class FireflyGANBaseWrapper(nn.Module):
    """model.py:33-43: loads a generator checkpoint (strict) into ``FireflyGANBase`` and switches it to eval mode.  The
    caller moves it to the GPU (``.to('cuda')``), as with the reference's ``get_vocoder``."""

    def __init__(self, model_path):
        super().__init__()
        self.model = FireflyGANBase()
        self.model.load_state_dict(torch.load(model_path, weights_only=True, map_location="cpu"))
        self.model.eval()

    @torch.inference_mode()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.model(x)
