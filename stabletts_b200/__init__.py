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
from .ffgan import FireflyGANBase, FireflyGANBaseWrapper   # noqa: F401
from .align import expand_by_durations              # noqa: F401
from .frontend import MelStyleEncoder, DurationPredictor   # noqa: F401
from .model import StableTTS                        # noqa: F401
from . import monotonic_align                       # noqa: F401
from .audio import LinearSpectrogram, LogMelSpectrogram   # noqa: F401
from .mel_loss import MultiScaleMelSpectrogramLoss, SingleScaleMelSpectrogramLoss   # noqa: F401
from .resample import Resample, load_and_resample_audio, resample   # noqa: F401
from .discriminator import DiscriminatorP, DiscriminatorR, MultiPeriodDiscriminator, MultiResolutionDiscriminator   # noqa: F401
from ._lib import library_path, load_library        # noqa: F401

__all__ = ["Decoder", "CFMDecoder", "TextEncoder", "Vocos", "FireflyGANBase", "FireflyGANBaseWrapper", "expand_by_durations", "MelStyleEncoder",
           "DurationPredictor", "StableTTS", "monotonic_align", "LinearSpectrogram", "LogMelSpectrogram",
           "MultiScaleMelSpectrogramLoss", "SingleScaleMelSpectrogramLoss", "resample", "Resample", "load_and_resample_audio",
           "DiscriminatorP", "MultiPeriodDiscriminator", "DiscriminatorR", "MultiResolutionDiscriminator",
           "library_path", "load_library"]
