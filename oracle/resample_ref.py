"""CPU oracle for resampling (TEST INFRASTRUCTURE ONLY): a float64 statement of the band-limited polyphase contract that
``torchaudio.functional.resample`` implements (utils/audio.py:73, sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99),
plus the seeded test waveforms.  Pinned by tests/test_resample.py against tests/golden/rs_*.npz, which
oracle/make_golden_resample.py writes from torchaudio.

The contract, with g = gcd(orig, new), O = orig / g, N = new / g:
    base  = 0.99 * min(O, N)                       (Python float)
    width = ceil(6 * O / base)                     (Python float arithmetic)
    xpad[m] = x[m - width] for 0 <= m - width < L, else 0
    y[i N + j] = sum_{k = 0}^{2 width + O - 1} coef[j][k] * xpad[i O + k],   output length ceil(N L / O) (integers)
    t = clamp(((k - width) / O - j / N) * base, -6, 6),  window = cos^2(t pi / 12)
    coef[j][k] = sinc(t) * window * base / O,  sinc(t) = sin(pi t) / (pi t), 1 at t = 0
orig == new returns the input unchanged."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.mel_ref import checksum  # noqa: F401  (the fixtures' waveform checksum)

LOWPASS_FILTER_WIDTH = 6
ROLLOFF = 0.99


def dims(orig: int, new: int):
    """(O, N, width, base) of the pair orig -> new."""
    g = math.gcd(int(orig), int(new))
    O, N = int(orig) // g, int(new) // g
    base = min(O, N) * ROLLOFF
    width = math.ceil(LOWPASS_FILTER_WIDTH * O / base)
    return O, N, width, base


def out_length(orig: int, new: int, L: int) -> int:
    O, N, _, _ = dims(orig, new)
    return -(-N * L // O)


def coefficients(orig: int, new: int, phase_dtype=torch.float64) -> torch.Tensor:
    """(N, 2 width + O) float64 coefficients of the contract, in the evaluation order the formula states.  `phase_dtype`
    is the precision of the j / N term (torchaudio.transforms.Resample evaluates it in fp32)."""
    O, N, width, base = dims(orig, new)
    k = torch.arange(2 * width + O, dtype=torch.float64)
    jn = (torch.arange(N, dtype=phase_dtype) / N).to(torch.float64)
    t = ((k[None, :] - width) / O - jn[:, None]) * base
    t = t.clamp(-LOWPASS_FILTER_WIDTH, LOWPASS_FILTER_WIDTH)
    window = torch.cos(t * math.pi / LOWPASS_FILTER_WIDTH / 2) ** 2
    pt = t * math.pi
    sinc = torch.where(pt == 0, torch.ones_like(pt), torch.sin(pt) / torch.where(pt == 0, torch.ones_like(pt), pt))
    return sinc * (window * (base / O))


def resample(x: torch.Tensor, orig: int, new: int, coef: torch.Tensor | None = None) -> torch.Tensor:
    """The contract in float64: x (..., L) -> (..., ceil(N L / O)).  `coef` ((N, 2 width + O) or the module's
    (N, 1, 2 width + O) buffer) replaces the formula's coefficients."""
    if orig == new:
        return x
    O, N, width, _ = dims(orig, new)
    c = coefficients(orig, new) if coef is None else coef.reshape(N, -1).to(torch.float64)
    assert c.shape == (N, 2 * width + O), c.shape
    shape = x.shape
    L = shape[-1]
    xs = x.reshape(-1, L).to(torch.float64)
    xpad = F.pad(xs, (width, width + O))
    n_blocks = L // O + 1                                           # blocks i with i O + 2 width + O <= L + 2 width + O
    frames = xpad.unfold(-1, 2 * width + O, O)[:, :n_blocks]        # (rows, n_blocks, 2 width + O): xpad[i O + k]
    y = torch.einsum("rik,jk->rij", frames, c).reshape(xs.shape[0], -1)[:, :out_length(orig, new, L)]
    return y.reshape(*shape[:-1], y.shape[-1])


def resample_at(x: torch.Tensor, orig: int, new: int, positions) -> torch.Tensor:
    """The contract in float64 at the given output positions only: x (rows, L) -> (rows, len(positions))."""
    O, N, width, _ = dims(orig, new)
    c = coefficients(orig, new)
    L = x.shape[-1]
    cols = []
    for p in positions:
        i, j = divmod(int(p), N)
        m = torch.arange(2 * width + O) + i * O - width             # x index of tap k
        ok = (m >= 0) & (m < L)
        seg = torch.zeros(x.shape[0], 2 * width + O, dtype=torch.float64)
        seg[:, ok] = x[:, m[ok]].to(torch.float64)
        cols.append(seg @ c[j])
    return torch.stack(cols, -1)


def make_wave(kind: str, seed: int, L: int, sample_rate: int) -> torch.Tensor:
    """One seeded fp32 waveform (L,) of the named kind at `sample_rate`."""
    g = torch.Generator().manual_seed(seed)
    n = torch.arange(L, dtype=torch.float64)
    if kind == "noise":                                              # full scale: uniform in [-1, 1)
        return (torch.rand(L, generator=g, dtype=torch.float64) * 2 - 1).float()
    if kind == "sine":
        return (0.9 * torch.sin(2 * math.pi * 440.0 * n / sample_rate)).float()
    if kind == "square":                                            # exactly +-1, 100 Hz
        return ((n * 200 // sample_rate) % 2 * -2.0 + 1.0).float()
    if kind == "silence":
        return torch.zeros(L)
    if kind == "nyquist":                                           # a tone at 0.98 of the source Nyquist frequency
        return (0.8 * torch.sin(2 * math.pi * 0.49 * n + 0.3)).float()
    if kind == "speech":                                            # a decaying harmonic stack + noise
        f0 = 110.0 + 40.0 * torch.rand(1, generator=g, dtype=torch.float64)
        x = sum(0.3 / k * torch.sin(2 * math.pi * k * f0 * n / sample_rate + float(k)) for k in range(1, 16))
        x = x * (0.6 + 0.4 * torch.sin(2 * math.pi * 3.0 * n / sample_rate)) + 0.01 * torch.randn(L, generator=g, dtype=torch.float64)
        return x.float()
    raise ValueError(kind)


def make_batch(kinds, seed: int, L: int, sample_rate: int) -> torch.Tensor:
    return torch.stack([make_wave(k, seed + i, L, sample_rate) for i, k in enumerate(kinds)])


SIGNALS = ["noise", "sine", "square", "silence", "nyquist"]
_TO_44K = [48000, 24000, 16000, 22050, 8000, 96000, 32000]
_PAIRS = [(s, 44100) for s in _TO_44K] + [(44100, 16000), (44100, 22050), (44100, 24000), (12345, 44100), (192000, 16000)]

CASES = {}
for _n, (_o, _w) in enumerate(_PAIRS):
    CASES[f"rs_{_o}_{_w}"] = dict(orig=_o, new=_w, kinds=SIGNALS, seed=500 + 10 * _n, L=_o // 10 + 7)   # 0.1 s + 7
_o48 = dims(48000, 44100)
CASES["rs_48000_44100_L1"] = dict(orig=48000, new=44100, kinds=["noise", "nyquist"], seed=700, L=1)
CASES["rs_48000_44100_short"] = dict(orig=48000, new=44100, kinds=["noise", "sine"], seed=701, L=_o48[2] - 3)   # L < width
CASES["rs_16000_44100_short"] = dict(orig=16000, new=44100, kinds=["noise"], seed=702, L=dims(16000, 44100)[2] - 1)
CASES["rs_192000_16000_short"] = dict(orig=192000, new=16000, kinds=["noise"], seed=703, L=dims(192000, 16000)[2] - 5)
CASES["rs_12345_44100_ragged"] = dict(orig=12345, new=44100, kinds=["noise", "square"], seed=704, L=5 * 823 + 411)  # not a multiple of O

# a 48 kHz clip -> resample -> the reference's LogMelSpectrogram at its default MelConfig
COMPOSED = dict(name="rs_composed_mel", orig=48000, new=44100, kinds=["speech", "noise"], seed=800, L=48000)
