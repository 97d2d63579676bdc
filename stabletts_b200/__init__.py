"""stabletts_b200 — CUDA-native (H100, sm_90a) flow-matching DiT mel-denoiser behind StableTTS's
``CFMDecoder`` / ``Decoder`` class surface (reference: models/flow_matching.py,
models/estimator.py, models/diffusion_transformer.py).

Host code is a thin ctypes binding over the C ABI in ``include/stabletts_b200.h``; all compute is
hand-written CUDA in ``libstabletts_b200.so``.  There is no CPU or PyTorch fallback: using the
modules without the built library or without a CUDA device raises.
"""
from .estimator import Decoder                      # noqa: F401
from .flow_matching import CFMDecoder               # noqa: F401
from .text_encoder import TextEncoder               # noqa: F401
from .vocos import Vocos                            # noqa: F401
from .align import expand_by_durations              # noqa: F401
from ._lib import library_path, load_library        # noqa: F401

__all__ = ["Decoder", "CFMDecoder", "TextEncoder", "Vocos", "expand_by_durations", "library_path", "load_library"]
