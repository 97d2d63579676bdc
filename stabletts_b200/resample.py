"""Drop-ins for resampling: ``resample`` (``torchaudio.functional.resample``, which the reference calls at
utils/audio.py:73), ``Resample`` (``torchaudio.transforms.Resample``) and ``load_and_resample_audio`` (utils/audio.py:59-74:
the reference audio of every ``StableTTSAPI.inference`` call, api.py:72, and every training clip, preprocess.py:65).

The transform is torchaudio's band-limited sinc interpolation with a Hann window, ``lowpass_filter_width=6`` and
``rolloff=0.99`` (the contract is stated in include/stabletts_b200.h and oracle/resample_ref.py).  ``forward`` is one call
into the CUDA library (``st_resample_forward``: one polyphase kernel that sums only each phase's band of non-zero
coefficients).  Coefficients are evaluated in float64 and rounded once to fp32; torchaudio's ``resample`` evaluates them in
the waveform's dtype, so its fp32 output is up to 1e-4 (at 12345 -> 44.1 kHz) from the float64 result, where this one is
within 1e-6 of max|x|.  A ``Resample`` module uses its ``kernel`` buffer exactly as loaded.

Built: ``sinc_interp_hann`` with the defaults above, integer rates, fp32 CUDA input, no autograd.  Anything else raises;
there is no CPU fallback."""
from __future__ import annotations

import ctypes as C
import functools
import math

import torch

from . import _lib
from ._native import NativeModule

_WIDTH, _ROLLOFF = 6, 0.99


def _check_method(lowpass_filter_width, rolloff, resampling_method, beta) -> None:
    if resampling_method != "sinc_interp_hann":
        raise ValueError(f"resampling_method={resampling_method!r} is not built: only 'sinc_interp_hann' (torchaudio's default)")
    if lowpass_filter_width != _WIDTH or rolloff != _ROLLOFF or beta is not None:
        raise ValueError("only lowpass_filter_width=6, rolloff=0.99 and beta=None are built (torchaudio's defaults, the "
                         "reference's only use)")


def _rates(orig_freq, new_freq):
    for f in (orig_freq, new_freq):
        if isinstance(f, bool) or not isinstance(f, (int, float)) or int(f) != f:
            raise ValueError(f"sample rates must be integers, got {orig_freq!r} -> {new_freq!r}")
        if f <= 0:
            raise ValueError("sample rates must be positive")
        if f >= 2 ** 31:
            raise ValueError("sample rates must be below 2^31")
    return int(orig_freq), int(new_freq)


def pair_dims(orig_freq: int, new_freq: int):
    """(O, N, width, base): the rates over their gcd, the filter half-width in input samples, 0.99 min(O, N)."""
    g = math.gcd(orig_freq, new_freq)
    O, N = orig_freq // g, new_freq // g
    base = min(O, N) * _ROLLOFF
    return O, N, math.ceil(_WIDTH * O / base), base


@functools.lru_cache(maxsize=64)
def band_table(orig_freq: int, new_freq: int):
    """The default table as st_create_resample builds it: (k0 (N,) int64, coef (N, band) fp32 from float64, width).  Phase
    j's coefficient of tap k0[j] + c is coef[j, c]; taps outside the band are exactly 0 in fp32.  Raises ValueError when
    N x band exceeds ST_RESAMPLE_MAX_TABLE."""
    O, N, width, base = pair_dims(orig_freq, new_freq)
    K = 2 * width + O
    limit = _lib.ST_RESAMPLE_MAX_TABLE
    grid = math.ceil(12.0 * O / base) + 3
    # only |t| < 6 is non-zero; every phase has at least 5/8 of its evaluation grid non-zero, so a grid over 4x the bound
    # is a table over the bound
    if N > limit or N * grid > 4 * limit:
        raise ValueError(f"{orig_freq} -> {new_freq}: the coefficient table exceeds {limit} (N x band)")
    j = torch.arange(N, dtype=torch.float64)
    lo = torch.clamp(torch.floor(width + O * j / N - 6.0 * O / base) - 1, min=0).long()
    k = lo[:, None] + torch.arange(grid)[None, :]
    valid = k < K
    t = ((k.double() - width) / O - j[:, None] / N) * base
    t = t.clamp(-_WIDTH, _WIDTH)
    window = torch.cos(t * math.pi / _WIDTH / 2) ** 2
    pt = t * math.pi
    sinc = torch.where(pt == 0, torch.ones_like(pt), torch.sin(pt) / torch.where(pt == 0, torch.ones_like(pt), pt))
    c = (sinc * (window * (base / O))).float() * valid
    nz = c != 0
    first = torch.where(nz.any(1), nz.float().argmax(1), torch.zeros(N, dtype=torch.long))
    last = torch.where(nz.any(1), grid - 1 - nz.flip(1).float().argmax(1), first - 1)
    cnt = last - first + 1
    bw = int(cnt.max())
    if N * bw > limit:
        raise ValueError(f"{orig_freq} -> {new_freq}: the coefficient table exceeds {limit} (N x band = {N * bw})")
    idx = first[:, None] + torch.arange(bw)[None, :]
    coef = torch.gather(c, 1, idx.clamp(max=grid - 1)) * (torch.arange(bw)[None, :] < cnt[:, None])
    return lo + first, coef, width


def default_kernel(orig_freq: int, new_freq: int) -> torch.Tensor:
    """(N, 1, 2 width + O) fp32: torchaudio.transforms.Resample's `kernel` buffer, evaluated in float64 and rounded once."""
    O, N, width, _ = pair_dims(orig_freq, new_freq)
    k0, coef, _ = band_table(orig_freq, new_freq)
    dense = torch.zeros(N, 2 * width + O, dtype=torch.float32)
    cols = (k0[:, None] + torch.arange(coef.shape[1])[None, :]).clamp(max=2 * width + O - 1)
    dense.scatter_add_(1, cols, coef)
    return dense.unsqueeze(1)


def _check_input(x) -> None:
    if not isinstance(x, torch.Tensor):
        raise TypeError("the waveform must be a torch.Tensor")
    if x.dtype != torch.float32:
        raise TypeError(f"the waveform must be float32, got {x.dtype}")
    if x.requires_grad and torch.is_grad_enabled():
        raise RuntimeError("resampling has no backward here: call it under torch.no_grad() / inference_mode, or detach")
    if x.device.type != "cuda":
        raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
    if x.ndim == 0:
        raise ValueError("the waveform must have a time dimension (..., L)")


def _run(lib, h, x: torch.Tensor, out_len: int) -> torch.Tensor:
    shape = x.shape
    L, rows = shape[-1], math.prod(shape[:-1])
    y = torch.empty(*shape[:-1], out_len, device=x.device, dtype=torch.float32)
    if rows == 0 or out_len == 0:
        return y
    xc = x.detach().reshape(rows, L).contiguous()
    stream = torch.cuda.current_stream(x.device).cuda_stream
    _lib.check(lib, h, lib.st_resample_forward(h, xc.data_ptr(), y.data_ptr(), rows, L, stream), "st_resample_forward")
    return y


_HANDLES = {}


def _handle(device: torch.device, O: int, N: int):
    """one library handle per (device, O, N), built once: its table is the pair's default"""
    lib = _lib.load_library()
    index = device.index if device.index is not None else torch.cuda.current_device()
    key = (index, O, N)
    h = _HANDLES.get(key)
    if h is None:
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_resample(O, N, index, C.byref(h)), "st_create_resample")
        _HANDLES[key] = h
    return lib, h


def resample(waveform: torch.Tensor, orig_freq, new_freq, lowpass_filter_width: int = 6, rolloff: float = 0.99,
             resampling_method: str = "sinc_interp_hann", beta=None) -> torch.Tensor:
    """torchaudio.functional.resample: waveform (..., L) fp32 CUDA -> (..., ceil(N L / O)).  orig_freq == new_freq returns
    `waveform` itself.  The table is built once per (device, pair) and cached."""
    _check_method(lowpass_filter_width, rolloff, resampling_method, beta)
    orig, new = _rates(orig_freq, new_freq)
    if orig == new:
        return waveform
    O, N, _, _ = pair_dims(orig, new)
    band_table(O, N)                                               # ValueError over the table bound
    _check_input(waveform)
    lib, h = _handle(waveform.device, O, N)
    return _run(lib, h, waveform, -(-N * waveform.shape[-1] // O))


class Resample(NativeModule):
    """torchaudio.transforms.Resample: the same constructor and state_dict (one persistent buffer, ``kernel``, (N, 1,
    2 width + O), absent when orig_freq == new_freq).  The default ``kernel`` is the float64 formula rounded once
    (torchaudio's own evaluates the j / N term in fp32 and is up to 5.3e-6 from it); a loaded ``kernel`` is used exactly
    as loaded: its non-zero band per phase is packed at the first call after it changes."""

    def __init__(self, orig_freq=16000, new_freq=16000, resampling_method: str = "sinc_interp_hann",
                 lowpass_filter_width: int = 6, rolloff: float = 0.99, beta=None, *, dtype=None):
        super().__init__()
        _check_method(lowpass_filter_width, rolloff, resampling_method, beta)
        if dtype not in (None, torch.float32):
            raise ValueError(f"dtype={dtype} is not built: the kernel buffer is fp32")
        self.orig_freq, self.new_freq = _rates(orig_freq, new_freq)
        self.gcd = math.gcd(self.orig_freq, self.new_freq)
        self.resampling_method = resampling_method
        self.lowpass_filter_width = lowpass_filter_width
        self.rolloff = rolloff
        self.beta = beta
        self._init_native()
        if self.orig_freq != self.new_freq:
            O, N, self.width, _ = pair_dims(self.orig_freq, self.new_freq)
            self.register_buffer("kernel", default_kernel(O, N))

    def _create_handle(self, lib, index):
        h = C.c_void_p()
        _lib.check(lib, None, lib.st_create_resample(self.orig_freq // self.gcd, self.new_freq // self.gcd, index,
                                                     C.byref(h)), "st_create_resample")
        return h

    def _sync_kernel(self, lib, h, stream: int) -> None:
        t = self.kernel
        if t.device.type != "cuda" or t.dtype != torch.float32:
            raise RuntimeError(f"buffer kernel must be CUDA fp32 (got {t.device}, {t.dtype}); call .to('cuda')")
        tag = (t.data_ptr(), t._version)
        if self._synced.get("kernel") != tag:
            tc = t.detach().contiguous()
            _lib.check(lib, h, lib.st_load_weight(h, b"kernel", tc.data_ptr(), tc.numel(), stream), "st_load_weight(kernel)")
            _lib.check(lib, h, lib.st_finalize_weights(h, stream), "st_finalize_weights")
            self._synced["kernel"] = tag

    def set_engine(self, name: str) -> None:
        """Accepted for interface parity with the other modules and ignored: resampling has one engine (fp32 CUDA cores)."""
        if name not in ("tcgen05", "simt"):
            raise KeyError(name)

    def forward(self, waveform: torch.Tensor) -> torch.Tensor:
        if self.orig_freq == self.new_freq:
            return waveform
        _check_input(waveform)
        O, N = self.orig_freq // self.gcd, self.new_freq // self.gcd
        with torch.no_grad():
            lib, h = self._ensure_handle(waveform.device)
            self._sync_kernel(lib, h, torch.cuda.current_stream(waveform.device).cuda_stream)
            return _run(lib, h, waveform, -(-N * waveform.shape[-1] // O))


def load_and_resample_audio(audio_path, target_sr, device="cpu"):
    """utils/audio.py:59-74: decode with torchaudio.load on the host, keep channel 0 as (1, L), resample to target_sr on
    `device` when it is a CUDA device (else on the current CUDA device) and return the result on `device`.  Prints the
    error and returns None when decoding fails, as the reference does."""
    import torchaudio
    try:
        y, sr = torchaudio.load(audio_path)
    except Exception as e:                                         # noqa: BLE001 — the reference's contract
        print(str(e))
        return None
    if y.size(0) > 1:
        y = y[0, :].unsqueeze(0)
    device = torch.device(device)
    if sr != target_sr:
        run_on = device if device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        with torch.no_grad():
            y = resample(y.to(run_on), sr, target_sr)
    return y.to(device)
