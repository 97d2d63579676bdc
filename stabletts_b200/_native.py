"""Shared plumbing of the drop-in modules: parameters live in ordinary ``nn.Parameter`` s under the
reference's own module paths; the CUDA library keeps a packed copy that is refreshed whenever a
parameter's version counter or storage changes; the workspace is a torch ``uint8`` tensor attached to
the library handle.  No CPU fallback anywhere."""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Tuple

import torch
import torch.nn as nn

from . import _lib


class _Node(nn.Module):
    """Anonymous container: exists only so parameter paths equal the reference's module tree."""


class NativeModule(nn.Module):
    """Base of Decoder / TextEncoder.  Subclasses set ``self._shapes`` (ordered name -> shape) and implement
    ``_create_handle(lib, device_index) -> c_void_p``."""

    def _init_native(self):
        self._handle = None
        self._handle_device = None
        self._synced: Dict[str, Tuple[int, int]] = {}
        self._workspace = None
        # debugging switch between the two CUDA engines (not a backend dispatch; both are this library)
        self._engine = _lib.ST_ENGINE_SIMT if os.environ.get("STABLETTS_B200_ENGINE") == "simt" else _lib.ST_ENGINE_TCGEN05
        self._precision = None                  # None: the library's default (ffn_fp16x2, or STABLETTS_B200_PRECISION)

    # -- module tree ------------------------------------------------------------------------------
    def _register(self, dotted: str, p: nn.Parameter) -> None:
        mod = self
        parts = dotted.split(".")
        for part in parts[:-1]:
            if part not in mod._modules:
                mod.add_module(part, _Node())
            mod = mod._modules[part]
        mod.register_parameter(parts[-1], p)

    def _param(self, dotted: str) -> nn.Parameter:
        mod = self
        parts = dotted.split(".")
        for part in parts[:-1]:
            mod = mod._modules[part]
        return mod._parameters[parts[-1]]


    # -- library plumbing -------------------------------------------------------------------------
    def set_engine(self, name: str) -> None:
        """'tcgen05' (the default product path: the wgmma tensor-core engine, under its historical name) or 'simt' (fp32 cross-check engine) — both CUDA."""
        self._engine = {"tcgen05": _lib.ST_ENGINE_TCGEN05, "simt": _lib.ST_ENGINE_SIMT}[name]
        if self._handle is not None:
            lib = _lib.load_library()
            _lib.check(lib, self._handle, lib.st_set_engine(self._handle, self._engine), "st_set_engine")

    def set_precision(self, name: str) -> None:
        """'ffn_fp16x2' (= 'default': split-bf16 x 3 everywhere except the FFN convs, which take fp16 activations against
        fp16 hi / lo weights in two MMA passes; <= 3e-4 against the reference, -15 % time) or 'bf16x3' (three passes
        everywhere, ~1e-5) — see st_set_precision in the C header."""
        self._precision = {"default": _lib.ST_PRECISION_FFN_FP16X2, "ffn_fp16x2": _lib.ST_PRECISION_FFN_FP16X2,
                           "bf16x3": _lib.ST_PRECISION_BF16X3}[name]
        if self._handle is not None:
            lib = _lib.load_library()
            _lib.check(lib, self._handle, lib.st_set_precision(self._handle, self._precision), "st_set_precision")

    def _ensure_handle(self, device: torch.device):
        lib = _lib.load_library()
        if device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        index = device.index if device.index is not None else torch.cuda.current_device()
        if self._handle is not None and self._handle_device != index:
            self.release()
        if self._handle is None:
            h = self._create_handle(lib, index)
            self._handle, self._handle_device = h, index
            self._synced.clear()
            _lib.check(lib, h, lib.st_set_engine(h, self._engine), "st_set_engine")
            if self._precision is not None:
                _lib.check(lib, h, lib.st_set_precision(h, self._precision), "st_set_precision")
        return lib, self._handle

    def _refuse_training_graph(self, what: str) -> None:
        """The CUDA path is inference-only (no dropout, no autograd graph): in ``train()`` mode with grad enabled the
        reference would return a differentiable, dropout-perturbed output; returning the detached eval output instead
        would silently train nothing, so raise (``compute_loss`` does the same)."""
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError(f"{what} in train() mode with autograd enabled needs dropout + backward kernels, "
                                      "which the inference-only CUDA path does not build; call .eval() / torch.no_grad(), "
                                      "or train with the reference module and load the checkpoint here")

    def invalidate_weights(self) -> None:
        """Force a re-pack of every parameter on the next call.  Needed after in-place updates made THROUGH ``p.data``
        (``p.data.copy_()``, EMA loops, legacy loaders): those do not bump ``p._version``, which is what the automatic
        freshness check keys on together with the storage pointer."""
        self._synced.clear()

    def _sync_weights(self, lib, h, stream: int, force: bool = False) -> None:
        if force:
            self._synced.clear()
        dirty = False
        for name in self._shapes:
            p = self._param(name)
            if p.device.type != "cuda" or p.dtype != torch.float32:
                raise RuntimeError(f"parameter {name} must be CUDA fp32 (got {p.device}, {p.dtype}); call .to('cuda')")
            tag = (p.data_ptr(), p._version)
            if self._synced.get(name) != tag:
                pc = p.detach().contiguous()
                _lib.check(lib, h, lib.st_load_weight(h, name.encode(), pc.data_ptr(), pc.numel(), stream),
                           f"st_load_weight({name})")
                self._synced[name] = tag
                dirty = True
        if dirty:
            _lib.check(lib, h, lib.st_finalize_weights(h, stream), "st_finalize_weights")

    def _prepare(self, ref: torch.Tensor):
        """(lib, handle, stream) for a call on ``ref``'s device: the handle exists and holds the current weights."""
        lib, h = self._ensure_handle(ref.device)
        stream = torch.cuda.current_stream(ref.device).cuda_stream
        self._sync_weights(lib, h, stream)
        return lib, h, stream

    def _attach_workspace(self, lib, h, need: int, device) -> None:
        """Attaches a torch-owned workspace of at least ``need`` bytes (grown, never shrunk) to the handle."""
        if self._workspace is None or self._workspace.numel() < need or self._workspace.device != device:
            self._workspace = None
            self._workspace = torch.empty(need, dtype=torch.uint8, device=device)
            _lib.check(lib, h, lib.st_attach_workspace(h, self._workspace.data_ptr(), self._workspace.numel()),
                       "st_attach_workspace")

    # -- copying / pickling: the library state (ctypes handle, workspace, sync tags) is per-process and per-device;
    #    copies and unpickled modules re-create theirs lazily on first use ---------------------------------------
    _NATIVE_STATE = ("_handle", "_handle_device", "_synced", "_workspace")

    def __getstate__(self):
        state = dict(self.__dict__)
        state["_handle"], state["_handle_device"], state["_synced"], state["_workspace"] = None, None, {}, None
        return state

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in self._NATIVE_STATE:
                continue
            setattr(new, k, copy.deepcopy(v, memo))
        new._handle, new._handle_device, new._synced, new._workspace = None, None, {}, None
        return new

    def release(self) -> None:
        if self._handle is not None:
            _lib.load_library().st_destroy(self._handle)
        self._handle = None
        self._workspace = None
        self._synced.clear()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def launch_count(self) -> int:
        return 0 if self._handle is None else int(_lib.load_library().st_launch_count(self._handle))

    @staticmethod
    def _f32c(name: str, t: torch.Tensor, shape) -> torch.Tensor:
        if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
            raise RuntimeError(f"{name} must be a CUDA tensor (no CPU fallback)")
        if tuple(t.shape) != tuple(shape):
            raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
        return t.detach().to(torch.float32).contiguous()

