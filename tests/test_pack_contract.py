"""The layout, operand-split and weight-packing kernels against exact statements of their contracts (st_test_pack_ex,
include/stabletts_b200.h), and the inventory that ties every CUDA kernel of the library to a kernel-level test.

Kernels: bct_to_btc_kernel, btc_to_bct_kernel, embed_kernel, split_kernel, split_f16_kernel (elementwise.cu),
pack_conv_kernel (handle.cu), weight_norm_fold_kernel, pack_polyphase_kernel (ffgan.cu), mel_twiddles_kernel and
mel_pack_fb_kernel (mel.cu).  The hook calls the product's own launch_* functions.

These kernels move or re-encode data without arithmetic of their own, so each statement is plain index code on numpy
arrays (fp64 or integers where that applies), and the CPU tests pin it against independent torch code: permute and
slicing, F.embedding, .to(torch.bfloat16) and .half(), the weight_norm parametrization, F.conv_transpose1d through the
oracle's polyphase packing, mpmath and torch.nonzero.

Bars on the GPU: bit for bit, with two exceptions.
  WEIGHT_NORM:  within 2 ulp of fp64 g v / ||v||, and within 2 ulp of torch's own fp32 parametrization beyond that
                parametrization's own distance from fp64 (torch's fp32 norm of a long row is itself a few ulp off);
  MEL_TWIDDLES: the correctly rounded fp32 value; a twiddle within 2^-50 (relative) of a rounding midpoint may be either
                neighbour, and is printed.
Every fp32 output starts as NaN and every integer output as a sentinel; PACK_CONV rows outside the slice it writes, and
the composed packings' unwritten rows, start as a float sentinel that must survive.  `pytest -s` prints the worst
WEIGHT_NORM ratio to its bar and any twiddle-midpoint cases."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ffgan_ref
from kernel_harness import LazyMatrix, NAN, bits, run_ok, set_fields
from kernel_harness import dev, handle  # noqa: F401 (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 7.0                      # float rows a kernel must leave alone
SENT_I32 = -0x5A5A5A5B              # integer outputs start here
FFGAN_UPS = [(512 >> i, 512 >> (i + 1), u) for i, u in enumerate((8, 8, 2, 2, 2))]    # (Cin, Cout, u) of FireflyGAN's ups


# --------------------------------------------------------------------------------------------------------------------
# the statements: plain index code on numpy arrays
# --------------------------------------------------------------------------------------------------------------------
def bf16_rn(x):
    """bf16_rn of fp32 x (numpy) by integer round-to-nearest-even on the bits -> fp32 values (NaN stays NaN)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32)
    out = r.view(np.float32).copy()
    out[np.isnan(x)] = np.nan
    return out


def split_bf16_ref(x):
    """SPLIT_BF16: hi = bf16_rn(x), lo = bf16_rn(x - hi), as fp32 values"""
    x = np.asarray(x, dtype=np.float32)
    hi = bf16_rn(x)
    with np.errstate(invalid="ignore", over="ignore"):
        return hi, bf16_rn((x - hi).astype(np.float32))


def split_f16_ref(x):
    """SPLIT_F16: hi = fp16_rn(x), lo = fp16_rn(x - hi) (numpy's float16 conversion rounds to nearest even), and the
    range flag: 1 when some x is NaN or |x| >= 65520"""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = x.astype(np.float16)
        lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo, int(bool((~(np.abs(x) < 65520.0)).any()))


def bct_to_btc_ref(x, C_, T, bcast=None):
    """out[b, t, c] = x[b, c, t]; with bcast a row B more: out[B, t, c] = bcast[c]"""
    B = x.shape[0]
    b, t, c = np.arange(B)[:, None, None], np.arange(T)[None, :, None], np.arange(C_)[None, None, :]
    out = x[b, c, t]
    if bcast is not None:
        out = np.concatenate([out, np.broadcast_to(bcast[np.arange(C_)][None, None, :], (1, T, C_))], 0)
    return out


def btc_to_bct_ref(x):
    """out[b, c, t] = x[b, t, c]"""
    B, T, C_ = x.shape
    b, c, t = np.arange(B)[:, None, None], np.arange(C_)[None, :, None], np.arange(T)[None, None, :]
    return x[b, t, c]


def embed_ref(ids, lens, emb, scale):
    """x[b, t, :] = (emb[clamp(id)] * scale) * m, m = [t < lens[b]], in fp32 in that order; mask = m"""
    B, T = ids.shape
    m = (np.arange(T)[None, :] < lens[:, None]).astype(np.float32)
    idc = np.clip(ids, 0, emb.shape[0] - 1)
    with np.errstate(invalid="ignore", over="ignore"):
        x = (emb[idc] * np.float32(scale)).astype(np.float32) * m[:, :, None]
    return x.astype(np.float32), m


def pack_conv_ref(w, out, k, n_off, c_off, Cc):
    """out[tap][n_off + n][c] = w[n][c_off + c][tap] for n < Nsrc, c < Cc; the other rows of out keep their values"""
    out = out.copy()
    Nsrc = w.shape[0]
    tap, n, c = np.arange(k)[:, None, None], np.arange(Nsrc)[None, :, None], np.arange(Cc)[None, None, :]
    out[tap, n_off + n, c] = w[n, c_off + c, tap]
    return out


def weight_norm_ref(g, v):
    """W[r, i] = v[r, i] fl32(g[r] / ||v_r||) (the kernel's order) and the fp64 value g v / ||v|| it stands for"""
    v64 = v.astype(np.float64).reshape(v.shape[0], -1)
    norm = np.sqrt((v64 * v64).sum(1))
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (g.astype(np.float64) / norm).astype(np.float32)
        ref64 = g.astype(np.float64)[:, None] * v64 / norm[:, None]
        return (v.reshape(v.shape[0], -1) * s[:, None]).astype(np.float32), ref64


def polyphase_ref(w, u):
    """out[tau][r Cout + c][i] = w[i, c, r + u/2 - (tau - 1) u] where that tap lies in [0, 2u), else 0"""
    Cin, Cout, _ = w.shape
    out = np.zeros((3, u * Cout, Cin), np.float32)
    for tau in range(3):
        for r in range(u):
            kk = r + u // 2 - (tau - 1) * u
            if 0 <= kk < 2 * u:
                out[tau, r * Cout:(r + 1) * Cout, :] = w[:, :, kk].T
    return out


def bands_ref(fb):
    """band[m] = [first, last + 1) of the entries != 0 of column m of fb (n_freqs, n_mels), (0, 0) if none; kband[k] the
    same over row k"""
    def runs(a):                       # a (rows, len): per row
        out = np.zeros((a.shape[0], 2), np.int32)
        for r in range(a.shape[0]):
            first = last = -1
            for i in range(a.shape[1]):
                if a[r, i] != 0:
                    if first < 0:
                        first = i
                    last = i
            if first >= 0:
                out[r] = (first, last + 1)
        return out
    return runs(fb.T), runs(fb)


_TW_CACHE = {}


def twiddles_ref(n_fft):
    """(re, im, ambiguous) fp32: re = fl32(cos 2 pi t / N), im = -fl32(sin 2 pi t / N), t < N/2, each correctly rounded from
    100-bit mpmath values; `ambiguous` lists (t, part) within 2^-50 (relative) of a rounding midpoint, where either
    neighbour is accepted.  N | 4096, so every N's twiddles are a stride of the 4096-point table."""
    if 4096 not in _TW_CACHE:
        import mpmath
        vals = {"re": np.zeros(2048, np.float32), "im": np.zeros(2048, np.float32)}
        amb = set()
        for t in range(2048):
            with mpmath.workprec(100):
                arg = mpmath.mpf(t) / 2048                       # 2 t / 4096
                pair = (("re", mpmath.cospi(arg)), ("im", mpmath.sinpi(arg)))
            for part, exact in pair:
                f = np.float32(float(exact))
                if exact != 0:                                   # the other candidate on the side of the exact value
                    other = np.nextafter(f, np.float32(np.inf if exact > mpmath.mpf(float(f)) else -np.inf))
                    lo_, hi_ = sorted((mpmath.mpf(float(f)), mpmath.mpf(float(other))))
                    mid = (lo_ + hi_) / 2
                    if abs(exact - mpmath.mpf(float(other))) < abs(exact - mpmath.mpf(float(f))):
                        f = other
                    if abs(exact - mid) < abs(exact) * mpmath.mpf(2) ** -50:
                        amb.add((t, part))
                vals[part][t] = f if part == "re" else -f
        _TW_CACHE[4096] = (vals["re"], vals["im"], amb)
    re_, im_, amb = _TW_CACHE[4096]
    step = 4096 // n_fft
    idx = np.arange(n_fft // 2) * step
    return re_[idx].copy(), im_[idx].copy(), sorted((t // step, p) for t, p in amb if t % step == 0 and t // step < n_fft // 2)


# --------------------------------------------------------------------------------------------------------------------
# operands
# --------------------------------------------------------------------------------------------------------------------
def signed(shape, seed, scale=1.0):
    g = np.random.default_rng(seed)
    return (g.standard_normal(shape) * scale).astype(np.float32)


def split_edges():
    """±0, fp32 denormals, values whose fp16 lo plane is subnormal, RNE ties of bf16 and fp16, the fp16 range edge"""
    v = [0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -2.3e-39, 6e-8, -6e-8, 1e-7, 3e-5, -6.1e-5, 65504.0, -65504.0,
         65519.99, -65519.99, 1.0, -1.0, 3.1415927, 1e-3, 2.0 ** -24, 2.0 ** -25, 2.0 ** -14 * 1.5]
    u = []
    for m in range(1, 9):                     # bf16 ties: the 16 dropped bits are exactly 0x8000, kept lsb even and odd
        u += [0x3F800000 | (m << 16) | 0x8000, 0xBF800000 | (m << 17) | 0x8000]
    for m in range(1, 9):                     # fp16 ties: 13 dropped mantissa bits are exactly 0x1000
        u += [0x3F800000 | (m << 13) | 0x1000, 0x47000000 | (m << 14) | 0x1000]
    for m in range(1, 5):                     # x - fp16(x) below the fp16 normal range: subnormal lo planes
        u += [0x3F800000 | m, 0x3C000000 | (m << 2) | 1]
    x = np.concatenate([np.array(v, np.float32), np.array(u, np.uint32).view(np.float32)])
    return np.concatenate([x, signed(1000, 5, 30.0), signed(301, 6, 1e-6)]).astype(np.float32)


def mel_fb(n_fft, n_mels):
    """an HTK triangular filterbank (n_fft/2 + 1, n_mels) in fp32, like torchaudio's melscale_fbanks"""
    n_freqs = n_fft // 2 + 1
    mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)       # noqa: E731
    pts = 700.0 * (10 ** (np.linspace(mel(0.0), mel(8000.0), n_mels + 2) / 2595.0) - 1.0)
    freqs = np.linspace(0, 8000.0, n_freqs)
    down = (freqs[:, None] - pts[None, :-2]) / (pts[1:-1] - pts[:-2])[None, :]
    up = (pts[None, 2:] - freqs[:, None]) / (pts[2:] - pts[1:-1])[None, :]
    return np.maximum(0.0, np.minimum(down, up)).astype(np.float32)


def mel_fb_edges(n_fft, n_mels, seed):
    """a loaded filterbank with the edges: interior zeros, an empty filter, filters at bin 0 and bin n_fft/2, a filter wider
    than 64 bins (when n_fft allows), a denormal weight (non-zero) and -0 entries (zero)"""
    fb = mel_fb(n_fft, n_mels)
    n_freqs = n_fft // 2 + 1
    g = np.random.default_rng(seed)
    fb[:, 1] = 0.0                                               # an empty filter
    fb[:, 0] = 0.0
    fb[0:3, 0] = (0.5, 0.0, 0.25)                                # touches bin 0, interior zero
    fb[:, -1] = 0.0
    fb[-1, -1], fb[-4, -1] = 0.75, 1e-3                          # touches bin n_fft/2
    wide = 2
    fb[:, wide] = 0.0
    w0, w1 = 2, min(n_freqs - 2, 2 + 90)
    fb[w0:w1, wide] = g.uniform(0.1, 1.0, w1 - w0)                # wider than 64 bins where n_freqs allows
    fb[w0 + (w1 - w0) // 2, wide] = 0.0                           # interior zero
    fb[w0 + 1, wide] = -0.0
    col = fb[:, 3]                                               # n_mels >= 5: filter 3 is none of the above
    nz = np.flatnonzero(col)
    col[:] = -0.0                                                # -0 everywhere: empty by value ...
    col[nz[0] if len(nz) else 3] = 1e-40                         # ... but for one denormal weight: a band of one bin
    m3 = n_mels // 2 + 1
    if m3 < n_mels - 1 and m3 > 3:
        nz = np.flatnonzero(fb[:, m3])
        if len(nz) >= 3:
            fb[nz[1], m3] = 0.0                                  # interior zero of an ordinary filter
            fb[nz[-1] + 1 if nz[-1] + 1 < n_freqs else nz[0] - 1, m3] = -0.0   # -0 just outside it
    return fb.astype(np.float32)


# --------------------------------------------------------------------------------------------------------------------
# CPU: the statements against independent torch code
# --------------------------------------------------------------------------------------------------------------------
def test_transposes_match_permute():
    for B, C_, T in ((2, 80, 33), (1, 100, 31), (3, 7, 1)):
        x = signed((B, C_, T), B + C_)
        bc = signed((C_,), 9)
        want = torch.cat([torch.from_numpy(x).permute(0, 2, 1), torch.from_numpy(bc)[None, None, :].expand(1, T, C_)], 0)
        assert torch.equal(torch.from_numpy(np.ascontiguousarray(bct_to_btc_ref(x, C_, T, bc))), want)
        assert torch.equal(torch.from_numpy(np.ascontiguousarray(btc_to_bct_ref(x.transpose(0, 2, 1).copy()))), torch.from_numpy(x))
    assert bct_to_btc_ref(np.zeros((0, 5, 3), np.float32), 5, 3, np.ones(5, np.float32)).shape == (1, 3, 5)


def test_embed_statement_matches_f_embedding():
    ids, lens, emb = embed_operands(3, 9, 16, 11, 1)
    x, m = embed_ref(ids, lens, emb, 13.856406)
    ti = torch.from_numpy(ids).clamp(0, 10)
    mask = (torch.arange(9)[None, :] < torch.from_numpy(lens)[:, None]).float()
    want = F.embedding(ti, torch.from_numpy(emb)) * torch.tensor(13.856406, dtype=torch.float32) * mask[:, :, None]
    got = torch.from_numpy(x)
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(bits(got.nan_to_num(7.0)), bits(want.nan_to_num(7.0)))          # -0 where masked, as torch
    assert torch.equal(torch.from_numpy(m), mask)
    assert (bits(got) == -(2 ** 31)).any()                                             # the operands do reach -0


def test_split_statements_match_torch_casts():
    x = split_edges()
    t = torch.from_numpy(x)
    hi, lo = split_bf16_ref(x)
    th = t.to(torch.bfloat16)
    assert torch.equal(bits(torch.from_numpy(hi).to(torch.bfloat16)), bits(th))
    assert torch.equal(bits(torch.from_numpy(lo).to(torch.bfloat16)), bits((t - th.float()).to(torch.bfloat16)))
    h16, l16, flag = split_f16_ref(x)
    assert flag == 0
    assert torch.equal(bits(torch.from_numpy(h16)), bits(t.half()))
    assert torch.equal(bits(torch.from_numpy(l16)), bits((t - t.half().float()).half()))
    assert (np.abs(l16[l16 != 0]) < 2.0 ** -14).any()                                  # subnormal lo planes occur
    for v, f in ((65520.0, 1), (-65520.0, 1), (np.inf, 1), (np.nan, 1), (65519.99, 0)):
        assert split_f16_ref(np.array([1.0, v], np.float32))[2] == f, v
    assert split_f16_ref(np.array([7e4], np.float32))[:2] == (np.float16(np.inf), np.float16(-np.inf))


def test_pack_conv_statement_matches_permute_and_slicing():
    w = signed((6, 10, 3), 1)
    out = pack_conv_ref(w, np.full((3, 9, 4), SENTINEL, np.float32), 3, 2, 5, 4)
    want = torch.full((3, 9, 4), SENTINEL)
    want[:, 2:8, :] = torch.from_numpy(w)[:, 5:9, :].permute(2, 0, 1)
    assert torch.equal(torch.from_numpy(out), want)


@pytest.mark.parametrize("kind", ["conv", "ups"])
def test_weight_norm_statement_matches_the_parametrization(kind):
    """g per output channel for a Conv1d (dim 0 of (Cout, Cin, k)), per input channel for a ConvTranspose1d (dim 0 of
    (Cin, Cout, 2u)): both are rows of the (dim 0, rest) view the kernel folds"""
    from torch.nn.utils.parametrizations import weight_norm
    torch.manual_seed(3)
    mod = torch.nn.Conv1d(16, 12, 3) if kind == "conv" else torch.nn.ConvTranspose1d(12, 8, 8, stride=4)
    mod = weight_norm(mod)
    with torch.no_grad():
        mod.parametrizations.weight.original0.mul_(torch.linspace(-2, 3, mod.parametrizations.weight.original0.numel()).view_as(mod.parametrizations.weight.original0))
    g = mod.parametrizations.weight.original0.detach().reshape(-1).numpy()
    v = mod.parametrizations.weight.original1.detach().numpy()
    w32, ref64 = weight_norm_ref(g, v)
    want = mod.weight.detach().reshape(v.shape[0], -1).double()
    assert g.shape[0] == v.shape[0]
    assert float((torch.from_numpy(ref64) - want).abs().max()) <= 4 * 2.0 ** -24 * float(want.abs().max())
    assert float((torch.from_numpy(w32).double() - want).abs().max()) <= 4 * 2.0 ** -24 * float(want.abs().max())


def test_weight_norm_statement_is_nan_on_an_all_zero_row_as_torch():
    from torch.nn.utils.parametrizations import weight_norm
    mod = weight_norm(torch.nn.Conv1d(3, 2, 1))
    with torch.no_grad():
        mod.parametrizations.weight.original1[0].zero_()
    assert torch.isnan(mod.weight[0]).all()
    w32, _ = weight_norm_ref(np.array([1.0, 1.0], np.float32), np.array([[0, 0, 0], [1, 2, 3]], np.float32))
    assert np.isnan(w32[0]).all() and np.isfinite(w32[1]).all()


@pytest.mark.parametrize("cin,cout,u", FFGAN_UPS[2:] + [(3, 2, 2), (2, 3, 4), (3, 2, 8)])
def test_polyphase_statement_is_the_transposed_conv(cin, cout, u):
    """the statement is the oracle's packing, and through it F.conv_transpose1d(stride u, padding u/2)"""
    w = torch.from_numpy(signed((cin, cout, 2 * u), u + cin))
    assert torch.equal(torch.from_numpy(polyphase_ref(w.numpy(), u)), ffgan_ref.polyphase_weight(w, u).permute(2, 0, 1))
    x, b = torch.randn(2, cin, 9, dtype=torch.float64), torch.randn(cout, dtype=torch.float64)
    want = F.conv_transpose1d(x, w.double(), b, stride=u, padding=u // 2)
    assert torch.allclose(ffgan_ref.conv_transpose_polyphase(x, w.double(), b, u), want, rtol=1e-12, atol=1e-12)


def test_twiddle_statement_matches_numpy_and_exact_points():
    re_, im_, amb = twiddles_ref(4096)
    t = np.arange(2048)
    assert np.abs(re_ - np.cos(2 * np.pi * t / 4096)).max() < 2 ** -24 and np.abs(im_ + np.sin(2 * np.pi * t / 4096)).max() < 2 ** -24
    assert bits(torch.from_numpy(im_[:1])).item() == -(2 ** 31)                    # -fl32(sin 0) = -0
    assert re_[1024] == 0.0 and im_[1024] == -1.0 and re_[0] == 1.0                # sinpi / cospi: exact at pi/2
    r32, i32, _ = twiddles_ref(32)
    assert np.array_equal(r32, re_[::128]) and np.array_equal(i32, im_[::128])


@pytest.mark.parametrize("n_fft,n_mels", [(32, 5), (64, 20), (512, 80), (1024, 100)])
def test_band_statement_matches_nonzero(n_fft, n_mels):
    fb = mel_fb_edges(n_fft, n_mels, n_fft)
    band, kband = bands_ref(fb)
    t = torch.from_numpy(fb)
    for m in range(n_mels):
        nz = torch.nonzero(t[:, m]).flatten()
        assert tuple(band[m]) == ((int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0)), m
    for k in range(n_fft // 2 + 1):
        nz = torch.nonzero(t[k]).flatten()
        assert tuple(kband[k]) == ((int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0)), k
    # the edges are present: an empty filter, bin 0, bin n_fft/2, interior zeros, -0 outside a band, a denormal
    assert tuple(band[1]) == (0, 0) and band[0][0] == 0 and band[-1][1] == n_fft // 2 + 1
    assert any(((fb[band[m][0]:band[m][1], m] == 0).any()) for m in range(n_mels))
    assert (np.signbit(fb) & (fb == 0)).any() and ((fb != 0) & (np.abs(fb) < 1.1754944e-38)).any()
    if n_fft >= 256:
        assert max(b[1] - b[0] for b in band) > 64


# --------------------------------------------------------------------------------------------------------------------
# the cases
# --------------------------------------------------------------------------------------------------------------------
def embed_operands(B, T, H, n_vocab, seed):
    """ids with values below 0 and at or above n_vocab; lens of 0, T, above T and in between; negative embeddings (so
    masked positions are -0) and one +inf row, used only at masked positions (inf * 0 = NaN, as torch)"""
    g = np.random.default_rng(seed)
    ids = g.integers(-3, n_vocab + 3, (B, T)).astype(np.int64)
    lens = np.array([[0, T, T + 5, max(1, T // 2)][b % 4] for b in range(B)], np.int64)
    emb = (-np.abs(g.standard_normal((n_vocab, H)))).astype(np.float32)
    emb[n_vocab // 2] = np.inf
    for b in range(B):
        ids[b, :min(T, int(lens[b]))][ids[b, :min(T, int(lens[b]))] == n_vocab // 2] = n_vocab // 2 + 1
        if lens[b] < T:
            ids[b, T - 1] = n_vocab // 2
    return ids, lens, emb


def _cases():
    cs = {}
    for C_ in (80, 100, 128, 256, 512):
        for T in (1, 31, 33, 1000):
            cs[f"bct_c{C_}_t{T}"] = dict(kind="BCT_TO_BTC", B=2, C=C_, T=T, bcast=C_ in (80, 100), f32=True, planes=True)
            cs[f"btc_c{C_}_t{T}"] = dict(kind="BTC_TO_BCT", B=2, C=C_, T=T)
    cs["bct_c512_t51000"] = dict(kind="BCT_TO_BTC", B=1, C=512, T=51000, bcast=False, f32=True, planes=False)
    cs["bct_c80_t51000_planes"] = dict(kind="BCT_TO_BTC", B=1, C=80, T=51000, bcast=True, f32=False, planes=True)
    cs["btc_c512_t51000"] = dict(kind="BTC_TO_BCT", B=1, C=512, T=51000)
    cs["bct_c80_t77_planes_only"] = dict(kind="BCT_TO_BTC", B=3, C=80, T=77, bcast=False, f32=False, planes=True)
    cs["bct_c100_t65_f32_only"] = dict(kind="BCT_TO_BTC", B=3, C=100, T=65, bcast=True, f32=True, planes=False)
    cs["bct_b0_bcast"] = dict(kind="BCT_TO_BTC", B=0, C=80, T=45, bcast=True, f32=True, planes=True)
    cs["bct_b0"] = dict(kind="BCT_TO_BTC", B=0, C=80, T=45, bcast=False, f32=True, planes=True)
    for B, T, H, nv, sc in ((4, 37, 256, 100, 16.0), (5, 1, 256, 7, 16.0), (8, 129, 192, 50, 13.856406)):
        cs[f"embed_b{B}_t{T}_h{H}"] = dict(kind="EMBED", B=B, T=T, C=H, n_vocab=nv, scale=sc)
    cs["split_bf16_edges"] = dict(kind="SPLIT_BF16", n="edges")
    cs["split_bf16_inf_nan"] = dict(kind="SPLIT_BF16", n="inf_nan")
    cs["split_bf16_large"] = dict(kind="SPLIT_BF16", n=1 << 20)
    cs["split_f16_edges"] = dict(kind="SPLIT_F16", n="edges")
    cs["split_f16_large"] = dict(kind="SPLIT_F16", n=3 * 1024 * 256 + 5)
    cs["split_f16_out_of_range"] = dict(kind="SPLIT_F16", n="range")
    for k in (1, 3, 5, 7, 11, 13):
        cs[f"pack_k{k}"] = dict(kind="PACK_CONV", parts=[dict(Nsrc=48, Csrc=40, k=k, Ntot=48, n_off=0, c_off=0, Cc=40)])
    cs["pack_offsets"] = dict(kind="PACK_CONV", parts=[dict(Nsrc=17, Csrc=40, k=3, Ntot=64, n_off=29, c_off=11, Cc=23)])
    cs["pack_dw7"] = dict(kind="PACK_CONV", parts=[dict(Nsrc=512, Csrc=1, k=7, Ntot=512, n_off=0, c_off=0, Cc=1)])
    cs["pack_largest"] = dict(kind="PACK_CONV", parts=[dict(Nsrc=1024, Csrc=256, k=3, Ntot=1024, n_off=0, c_off=0, Cc=256)])
    cs["pack_qkv"] = dict(kind="PACK_CONV", compose="qkv", parts=[dict(Nsrc=256, Csrc=256, k=1, Ntot=768, n_off=p * 256, c_off=0, Cc=256)
                                                                  for p in range(3)])
    cs["pack_in_proj_x"] = dict(kind="PACK_CONV", compose="in_x", parts=[dict(Nsrc=256, Csrc=336, k=1, Ntot=256, n_off=0, c_off=0, Cc=80)])
    cs["pack_in_proj_mu"] = dict(kind="PACK_CONV", compose="in_mu", parts=[dict(Nsrc=256, Csrc=336, k=1, Ntot=256, n_off=0, c_off=80, Cc=256)])
    cs["pack_vocos_head"] = dict(kind="PACK_CONV", compose="head", parts=[dict(Nsrc=513, Csrc=512, k=1, Ntot=1280, n_off=o, c_off=0, Cc=512)
                                                                          for o in (0, 640)])
    cs["pack_style_qkv"] = dict(kind="PACK_CONV", compose="style", parts=[dict(Nsrc=384, Csrc=128, k=1, Ntot=384, n_off=0, c_off=0, Cc=128)])
    for name, rows, ln in (("post", 1, 208), ("c16_k3", 16, 48), ("len256", 5, 256), ("pre", 512, 512 * 13), ("ups0", 512, 256 * 16),
                           ("len1", 3, 1), ("len257", 7, 257)):
        cs[f"wn_{name}"] = dict(kind="WEIGHT_NORM", rows=rows, len=ln, edges=name in ("len256", "len257", "c16_k3"))
    for cin, cout, u in FFGAN_UPS + [(6, 5, 2), (5, 6, 4), (3, 7, 8)]:
        cs[f"poly_{cin}x{cout}_u{u}"] = dict(kind="POLYPHASE", Cin=cin, Cout=cout, u=u)
    for n_fft in (32, 64, 128, 256, 512, 1024, 2048, 4096):
        cs[f"tw_{n_fft}"] = dict(kind="MEL_TWIDDLES", n_fft=n_fft)
    for n_fft, n_mels in ((32, 5), (64, 10), (128, 40), (256, 64), (512, 80), (1024, 100), (2048, 128), (4096, 320), (1024, 320)):
        for kb in (True, False):
            cs[f"fb_{n_fft}_{n_mels}" + ("_kband" if kb else "")] = dict(kind="MEL_PACK_FB", n_fft=n_fft, n_mels=n_mels, kband=kb)
    return cs


CASES = _cases()


def make_operands(name, d):
    seed = 4000 + list(CASES).index(name)
    k = d["kind"]
    if k == "BCT_TO_BTC":
        t = dict(x=signed((d["B"], d["C"], d["T"]), seed, 3.0))
        t["x"].reshape(-1)[::97] = -0.0
        if d["bcast"]:
            t["bcast"] = signed((d["C"],), seed + 1)
        return t
    if k == "BTC_TO_BCT":
        return dict(x=signed((d["B"], d["T"], d["C"]), seed))
    if k == "EMBED":
        ids, lens, emb = embed_operands(d["B"], d["T"], d["C"], d["n_vocab"], seed)
        return dict(ids=ids, lens=lens, x=emb)
    if k in ("SPLIT_BF16", "SPLIT_F16"):
        n = d["n"]
        if n == "edges":
            x = split_edges()
        elif n == "inf_nan":
            x = np.concatenate([split_edges()[:40], np.array([np.inf, -np.inf, np.nan, -np.nan, 3.4028235e38, -3.4028235e38], np.float32)])
        elif n == "range":
            x = np.concatenate([split_edges(), np.array([65520.0, -7e4, 1e5], np.float32)])
        else:
            x = signed((n,), seed, 50.0)
        return dict(x=x.astype(np.float32))
    if k == "PACK_CONV":
        p0 = d["parts"][0]
        if d.get("compose") == "head":
            return dict(x=signed((2 * p0["Nsrc"], p0["Csrc"], 1), seed))
        if d.get("compose") == "qkv":
            return dict(x=signed((3 * p0["Nsrc"], p0["Csrc"], 1), seed))
        return dict(x=signed((p0["Nsrc"], p0["Csrc"], p0["k"]), seed))
    if k == "WEIGHT_NORM":
        v = signed((d["rows"], d["len"]), seed)
        g = signed((d["rows"],), seed + 1, 2.0)
        g[::2] = -np.abs(g[::2])                                        # negative g
        if d["edges"]:
            r = 1 % d["rows"]
            g_ = np.random.default_rng(seed)
            v[r] = (10.0 ** g_.uniform(-15, 15, d["len"]) * np.where(np.arange(d["len"]) % 2, -1.0, 1.0)).astype(np.float32)
            v[r, :2] = (1e-15, -1e15)                                    # a dynamic range of 1e30 within the row
            v[0] = 0.0                                                  # an all-zero row: NaN, as torch
        return dict(g=g, x=v)
    if k == "POLYPHASE":
        return dict(x=signed((d["Cin"], d["Cout"], 2 * d["u"]), seed))
    if k == "MEL_TWIDDLES":
        return {}
    if k == "MEL_PACK_FB":
        return dict(x=mel_fb_edges(d["n_fft"], d["n_mels"], seed))
    raise KeyError(k)


# --------------------------------------------------------------------------------------------------------------------
# GPU: the hook's driver
# --------------------------------------------------------------------------------------------------------------------
def run_pack_hook(lib, h, kind, t, dev, fields, outs, desc_edit=None):
    """One st_test_pack_ex call: t = {input: numpy array}, fields = descriptor ints / floats, outs = {output: torch tensor
    on dev} (filled in by the caller).  Returns (rc, error text)."""
    from stabletts_b200 import _lib
    keep = {n: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for n, v in t.items()}
    desc = _lib.StTestPackDesc()
    for n in ("x", "bcast", "g", "ids", "lens"):
        setattr(desc, n, keep[n].data_ptr() if n in keep else None)
    for n in ("out_f32", "out2_f32", "out_hi", "out_lo", "out_i32", "out2_i32"):
        setattr(desc, n, outs[n].data_ptr() if n in outs else None)
    desc.kind = _lib.ST_TEST_PACK_KINDS.index(kind)
    for n, v in fields.items():
        setattr(desc, n, v)
    if desc_edit:
        desc_edit(desc)
    rc = lib.st_test_pack_ex(h, C.byref(desc), torch.cuda.current_stream().cuda_stream)
    return rc, lib.st_last_error(h).decode() if rc else ""


def nan_f32(shape, dev):
    return torch.full(shape, NAN, device=dev)


def sent_i32(shape, dev):
    return torch.full(shape, SENT_I32, dtype=torch.int32, device=dev)


def assert_bits(got, want, what):
    """bit equality of fp32 (or 2-byte) tensors; NaN is compared as NaN (the GPU's NaN payload is its own)"""
    want = torch.as_tensor(np.ascontiguousarray(want)) if isinstance(want, np.ndarray) else want
    got = got.cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan_g, nan_w = torch.isnan(got.float()), torch.isnan(want.float())
    assert torch.equal(nan_g, nan_w), (what, int((nan_g != nan_w).sum()))
    bad = (bits(got) != bits(want)) & ~nan_w
    assert not bad.any(), (what, int(bad.sum()), torch.nonzero(bad)[:5].tolist())


def ulps(got, ref64):
    """|got - ref64| in fp32 ulps of ref64 (subnormal spacing at the bottom)"""
    a = np.abs(ref64)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -126)))
    return np.abs(got.astype(np.float64) - ref64) / 2.0 ** (e - 23)


WN_WORST = {}
TW_MIDPOINTS = []


def run_case(lib, h, name, dev):
    d = CASES[name]
    t = make_operands(name, d)
    k = d["kind"]
    if k == "BCT_TO_BTC":
        B, C_, T = d["B"], d["C"], d["T"]
        rows = B + (1 if d["bcast"] else 0)
        alloc = max(rows, 1)                           # B = 0 without bcast: one row the kernel must not write
        outs = {}
        if d["f32"]:
            outs["out_f32"] = nan_f32((alloc, T, C_), dev)
        if d["planes"]:
            outs["out_hi"] = torch.full((alloc, T, C_), NAN, dtype=torch.bfloat16, device=dev)
            outs["out_lo"] = torch.full((alloc, T, C_), NAN, dtype=torch.bfloat16, device=dev)
        if B == 0:
            t.pop("x")
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(B=B, C=C_, T=T), outs)
        want = bct_to_btc_ref(t["x"] if B else np.zeros((0, C_, T), np.float32), C_, T, t.get("bcast"))
        if rows == 0:
            for n, v in outs.items():
                assert torch.isnan(v.float()).all(), n
            return True
        if d["f32"]:
            assert_bits(outs["out_f32"], want, "out_f32")
        if d["planes"]:
            hi, lo = split_bf16_ref(want)
            assert_bits(outs["out_hi"], torch.from_numpy(hi).to(torch.bfloat16), "hi")
            assert_bits(outs["out_lo"], torch.from_numpy(lo).to(torch.bfloat16), "lo")
    elif k == "BTC_TO_BCT":
        outs = dict(out_f32=nan_f32((d["B"], d["C"], d["T"]), dev))
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(B=d["B"], C=d["C"], T=d["T"]), outs)
        assert_bits(outs["out_f32"], btc_to_bct_ref(t["x"]), "out_f32")
    elif k == "EMBED":
        B, T, H = d["B"], d["T"], d["C"]
        outs = dict(out_f32=nan_f32((B, T, H), dev), out2_f32=nan_f32((B, T), dev))
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(B=B, T=T, C=H, n_vocab=d["n_vocab"], scale=d["scale"]), outs)
        x, m = embed_ref(t["ids"], t["lens"], t["x"], d["scale"])
        assert_bits(outs["out_f32"], x, "x")
        assert_bits(outs["out2_f32"], m, "mask")
    elif k in ("SPLIT_BF16", "SPLIT_F16"):
        x = t["x"]
        f16 = k == "SPLIT_F16"
        dt = torch.float16 if f16 else torch.bfloat16
        outs = dict(out_hi=torch.full(x.shape, NAN, dtype=dt, device=dev), out_lo=torch.full(x.shape, NAN, dtype=dt, device=dev))
        if f16:
            outs["out_i32"] = sent_i32((1,), dev)
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(n=x.size), outs)
        if f16:
            hi, lo, flag = split_f16_ref(x)
            keep = np.abs(x) < 65520.0                 # beyond: only the flag is the contract
            assert_bits(outs["out_hi"][torch.from_numpy(keep)], torch.from_numpy(hi[keep]), "hi")
            assert_bits(outs["out_lo"][torch.from_numpy(keep)], torch.from_numpy(lo[keep]), "lo")
            assert int(outs["out_i32"].item()) == flag
        else:
            hi, lo = split_bf16_ref(x)
            assert_bits(outs["out_hi"], torch.from_numpy(hi).to(torch.bfloat16), "hi")
            assert_bits(outs["out_lo"], torch.from_numpy(lo).to(torch.bfloat16), "lo")
    elif k == "PACK_CONV":
        run_pack_conv_case(lib, h, d, t, dev)
    elif k == "WEIGHT_NORM":
        outs = dict(out_f32=nan_f32((d["rows"], d["len"]), dev))
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(rows=d["rows"], len=d["len"]), outs)
        check_weight_norm(name, t, outs["out_f32"].cpu().numpy())
    elif k == "POLYPHASE":
        cin, cout, u = d["Cin"], d["Cout"], d["u"]
        outs = dict(out_f32=nan_f32((3, u * cout, cin), dev))
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(Cin=cin, Cout=cout, u=u), outs)
        assert_bits(outs["out_f32"], polyphase_ref(t["x"], u), "out_f32")
    elif k == "MEL_TWIDDLES":
        n = d["n_fft"]
        outs = dict(out_f32=nan_f32((n // 2, 2), dev))
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(n_fft=n), outs)
        re_, im_, amb = twiddles_ref(n)
        got = outs["out_f32"].cpu()
        want = torch.from_numpy(np.stack([re_, im_], 1))
        ok = bits(got) == bits(want)
        for tt, part in amb:                           # either neighbour of a near-midpoint value
            j = 0 if part == "re" else 1
            if not ok[tt, j]:
                ok[tt, j] = abs(int(bits(got[tt:tt + 1, j])) - int(bits(want[tt:tt + 1, j]))) == 1
            TW_MIDPOINTS.append((n, tt, part, float(got[tt, j]), float(want[tt, j])))
        assert ok.all(), torch.nonzero(~ok)[:5].tolist()
    elif k == "MEL_PACK_FB":
        n_fft, n_mels = d["n_fft"], d["n_mels"]
        nf = n_fft // 2 + 1
        outs = dict(out_f32=nan_f32((n_mels, nf), dev), out_i32=sent_i32((n_mels, 2), dev))
        if d["kband"]:
            outs["out2_i32"] = sent_i32((nf, 2), dev)
        run_ok(run_pack_hook, lib, h, k, t, dev, dict(n_fft=n_fft, n_mels=n_mels), outs)
        band, kband = bands_ref(t["x"])
        assert_bits(outs["out_f32"], np.ascontiguousarray(t["x"].T), "fbT")
        assert torch.equal(outs["out_i32"].cpu(), torch.from_numpy(band)), "band"
        if d["kband"]:
            assert torch.equal(outs["out2_i32"].cpu(), torch.from_numpy(kband)), "kband"
    return True


def run_pack_conv_case(lib, h, d, t, dev):
    """each part is one call into one sentinel-filled buffer; the result is compared with the statement and with torch"""
    p0 = d["parts"][0]
    out = torch.full((p0["k"], p0["Ntot"], p0["Cc"]), SENTINEL, device=dev)
    want = out.cpu().numpy()
    x = t["x"]
    for i, p in enumerate(d["parts"]):
        src = x[i * p["Nsrc"]:(i + 1) * p["Nsrc"]] if len(d["parts"]) > 1 else x
        run_ok(run_pack_hook, lib, h, "PACK_CONV", dict(x=src), dev, {n: p[n] for n in ("Nsrc", "Csrc", "k", "Ntot", "n_off", "c_off", "Cc")},
               dict(out_f32=out))
        want = pack_conv_ref(src, want, p["k"], p["n_off"], p["c_off"], p["Cc"])
    assert_bits(out, want, "out_f32")
    w = torch.from_numpy(x)
    comp = d.get("compose")
    if comp in ("qkv", "style"):               # cat(w_q, w_k, w_v) (N, C, 1) -> [1][3H][C]
        torch_want = w.permute(2, 0, 1)
    elif comp == "in_x":
        torch_want = w[:, :80, :].permute(2, 0, 1)
    elif comp == "in_mu":
        torch_want = w[:, 80:, :].permute(2, 0, 1)
    elif comp == "head":                       # log-magnitude rows at [0, K), phase rows at [Kp, Kp + K), sentinel between
        torch_want = torch.full((1, 1280, 512), SENTINEL)
        torch_want[0, :513] = w[:513, :, 0]
        torch_want[0, 640:640 + 513] = w[513:, :, 0]
    else:
        torch_want = torch.full(out.shape, SENTINEL)
        torch_want[:, p0["n_off"]:p0["n_off"] + p0["Nsrc"], :] = w[:, p0["c_off"]:p0["c_off"] + p0["Cc"], :].permute(2, 0, 1)
    assert torch.equal(bits(out.cpu()), bits(torch_want.contiguous()))


def check_weight_norm(name, t, got):
    """within 2 ulp of fp64 g v / ||v||, and within 2 ulp of torch's fp32 parametrization (torch._weight_norm, dim 0)
    beyond torch's own distance from fp64: torch's fp32 norm of a long row is itself several ulp off (4.6 ulp at 512 x 13
    taps), so a plain 2-ulp bar against it would measure torch.  NaN exactly on an all-zero row, as torch."""
    g, v = t["g"], t["x"]
    _, ref64 = weight_norm_ref(g, v)
    tw = torch._weight_norm(torch.from_numpy(v), torch.from_numpy(g)[:, None], 0).numpy()
    nan = np.isnan(ref64)
    assert np.array_equal(np.isnan(got), nan) and np.array_equal(np.isnan(tw), nan)
    fin = ~nan
    if not fin.any():
        WN_WORST[name] = (0.0, 0.0)
        return
    e64 = float(ulps(got[fin], ref64[fin]).max())
    e_torch = float(ulps(tw[fin], ref64[fin]).max())
    e32 = float(ulps(got[fin], tw[fin].astype(np.float64)).max())
    WN_WORST[name] = (e64 / 2.0, e32 / (2.0 + e_torch))
    assert e64 <= 2.0 and e32 <= 2.0 + e_torch, (e64, e32, e_torch)


@pytest.fixture(scope="module")
def matrix(dev, handle):
    return LazyMatrix(lambda name: run_case(*handle, name, dev))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_matrix(name, matrix):
    matrix.check(name)


@pytest.mark.gpu
def test_every_kind_ran(matrix):
    """and prints the worst WEIGHT_NORM ratio to its bar and the twiddle-midpoint cases (pytest -s)"""
    from stabletts_b200 import _lib
    for name in CASES:
        matrix[name]
    assert {d["kind"] for d in CASES.values()} == set(_lib.ST_TEST_PACK_KINDS)
    failed = [n for n in CASES if isinstance(matrix[n], Exception)]
    assert not failed, failed
    worst = max(WN_WORST.items(), key=lambda kv: max(kv[1]))
    print(f"\nWEIGHT_NORM worst ratio to its bar: {max(worst[1]):.3f} ({worst[0]}: fp64 {worst[1][0]:.3f}, torch fp32 {worst[1][1]:.3f})")
    print(f"twiddles within 2^-50 of a rounding midpoint: {len(TW_MIDPOINTS)}", *TW_MIDPOINTS[:20], sep="\n  ")


@pytest.mark.gpu
def test_split_f16_flag_clears_on_a_later_in_range_call(dev, handle):
    """the hook reports each call's own range: 0 after an in-range tensor, whatever came before"""
    lib, h = handle
    for x, flag in ((np.array([1e5, 1.0], np.float32), 1), (np.array([65504.0, 1.0], np.float32), 0), (np.array([np.nan], np.float32), 1)):
        outs = dict(out_hi=torch.empty(x.size, dtype=torch.float16, device=dev), out_lo=torch.empty(x.size, dtype=torch.float16, device=dev),
                    out_i32=sent_i32((1,), dev))
        run_ok(run_pack_hook, lib, h, "SPLIT_F16", dict(x=x), dev, dict(n=x.size), outs)
        assert int(outs["out_i32"].item()) == flag, x


@pytest.mark.gpu
def test_refusals(dev, handle):
    """every problem outside the contract is refused with a readable error, and nothing is launched"""
    from stabletts_b200 import _lib
    lib, h = handle
    x = np.ones((2, 8, 3), np.float32)

    def refused(kind, needle, t=None, outs=None, edit=None, **fields):
        o = outs if outs is not None else dict(out_f32=nan_f32((64,), dev))
        rc, err = run_pack_hook(lib, h, kind, dict(x=x) if t is None else t, dev, fields, o, desc_edit=edit)
        assert rc != 0 and needle in err, (kind, needle, err)
        for n, v in o.items():
            assert (torch.isnan(v.float()) | (v == SENT_I32)).all(), (kind, n)

    planes = lambda: dict(out_hi=torch.full((8,), NAN, dtype=torch.bfloat16, device=dev),    # noqa: E731
                          out_lo=torch.full((8,), NAN, dtype=torch.bfloat16, device=dev))
    refused("BCT_TO_BTC", "x is required", t={}, B=1, C=8, T=3)
    refused("BCT_TO_BTC", "0 <= B < 65535", B=-1, C=8, T=3)
    refused("BCT_TO_BTC", "no output requested", outs={}, B=2, C=8, T=3)
    refused("BCT_TO_BTC", "out_hi and out_lo go together", outs=dict(out_hi=planes()["out_hi"]), B=2, C=8, T=3)
    refused("BTC_TO_BCT", "B in [1, 65535]", B=0, C=8, T=3)
    refused("BTC_TO_BCT", "writes out_f32 only", outs=dict(out_f32=nan_f32((64,), dev), **planes()), B=2, C=8, T=3)
    refused("EMBED", "ids, lens and x (emb) are required", B=1, T=2, C=3, n_vocab=4)
    refused("SPLIT_BF16", "writes out_hi and out_lo", n=8)
    refused("SPLIT_BF16", "SPLIT: n >= 0", outs=planes(), n=-1)
    refused("SPLIT_BF16", "belongs to SPLIT_F16", outs=dict(out_i32=sent_i32((1,), dev), **planes()), n=8)
    refused("PACK_CONV", "n_off + Nsrc must be <= Ntot", Nsrc=2, Csrc=8, k=3, Ntot=4, n_off=3, c_off=0, Cc=8)
    refused("PACK_CONV", "c_off + Cc must be <= Csrc", Nsrc=2, Csrc=8, k=3, Ntot=2, n_off=0, c_off=1, Cc=8)
    refused("PACK_CONV", "offsets >= 0", Nsrc=2, Csrc=8, k=3, Ntot=2, n_off=-1, c_off=0, Cc=8)
    refused("PACK_CONV", "x is required", t={}, Nsrc=2, Csrc=8, k=3, Ntot=2, n_off=0, c_off=0, Cc=8)
    refused("WEIGHT_NORM", "g and x (v) are required", rows=2, len=24)
    refused("WEIGHT_NORM", "rows, len >= 1", t=dict(x=x, g=np.ones(2, np.float32)), rows=2, len=0)
    refused("POLYPHASE", "u must be even and >= 2", Cin=2, Cout=1, u=3)
    refused("POLYPHASE", "u must be even and >= 2", Cin=2, Cout=1, u=0)
    refused("POLYPHASE", "Cin, Cout >= 1", Cin=-2, Cout=1, u=2)
    refused("MEL_TWIDDLES", "power of two in [32, 4096]", n_fft=48)
    refused("MEL_TWIDDLES", "power of two in [32, 4096]", n_fft=8192)
    refused("MEL_PACK_FB", "power of two in [32, 4096]", n_fft=16, n_mels=4)
    refused("MEL_PACK_FB", "n_mels in [1, 4096]", n_fft=32, n_mels=0)
    refused("MEL_PACK_FB", "writes out_f32 (fbT) and out_i32 (band)", n_fft=32, n_mels=2)
    refused("SPLIT_F16", "unknown kind", outs=planes(), edit=set_fields(kind=len(_lib.ST_TEST_PACK_KINDS)), n=8)
    rc = lib.st_test_pack_ex(h, None, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and "null descriptor" in lib.st_last_error(h).decode()


# --------------------------------------------------------------------------------------------------------------------
# the binding, and the inventory of kernels and their tests
# --------------------------------------------------------------------------------------------------------------------
def test_kind_numbers_match_the_binding():
    """the binding's st_test_pack_desc.kind names are the enum of include/stabletts_b200.h"""
    from stabletts_b200 import _lib
    header = open(os.path.join(ROOT, "include", "stabletts_b200.h")).read()
    enum = {k: int(v) for k, v in re.findall(r"\bST_TEST_PACK_(\w+)\s*=\s*(\d+)", header)}
    assert enum == {k: i for i, k in enumerate(_lib.ST_TEST_PACK_KINDS)}


# every __global__ kernel of stabletts_b200/csrc -> the kernel-level test that checks it, or why none does
_PACK = "tests/test_pack_contract.py::test_matrix"
_ROW = "tests/test_row_contract.py::test_matrix"
_GLUE = "tests/test_glue_contract.py::test_matrix"
_MPD = "tests/test_mpd_contract.py::test_matrix"
KERNEL_TESTS = {
    # layout, split and packing kernels
    "bct_to_btc_kernel": _PACK, "btc_to_bct_kernel": _PACK, "embed_kernel": _PACK, "split_kernel": _PACK,
    "split_f16_kernel": _PACK, "pack_conv_kernel": _PACK, "weight_norm_fold_kernel": _PACK, "pack_polyphase_kernel": _PACK,
    "mel_twiddles_kernel": _PACK, "mel_pack_fb_kernel": _PACK,
    # conv-GEMM and attention
    "gemm_wgmma_kernel": "tests/test_gemm_contract.py::test_matrix", "gemm_simt_kernel": "tests/test_gemm_contract.py::test_matrix",
    "splitk_reduce_kernel": "tests/test_gemm_contract.py::test_bits_independent_of_sm_count_and_repetition",
    "attention_wgmma_kernel": "tests/test_attention_contract.py::test_matrix",
    "attention_simt_kernel": "tests/test_attention_contract.py::test_matrix",
    "mask_lengths_kernel": "tests/test_attention_contract.py::test_mask_lengths",
    # row kernels
    "film_ln_mod_kernel": _ROW, "dwconv_ln_kernel": _ROW, "spectrum_kernel": _ROW, "idft_basis_kernel": _ROW,
    "overlap_add_kernel": _ROW, "mean3_silu_kernel": _ROW, "post_conv_tanh_kernel": _ROW,
    "glu_residual_kernel": _GLUE, "masked_mean_kernel": _GLUE, "cond_mask_transpose_kernel": _GLUE, "relu_ln_kernel": _GLUE,
    "gemv_kernel": _GLUE, "time_embed_kernel": _GLUE, "time_embed_val_kernel": _GLUE, "rope_table_kernel": _GLUE,
    "lincomb_kernel": _GLUE, "scaled_sumsq_kernel": _GLUE, "cfg_combine_kernel": _GLUE, "cfm_mix_kernel": _GLUE,
    "cfm_loss_kernel": _GLUE, "cfm_loss_final_kernel": _GLUE,
    # the discriminator
    "conv0_fwd_kernel": _MPD, "act_fwd_kernel": _MPD, "nchw_to_rows_kernel": _MPD, "post_fwd_kernel": _MPD, "pack_kernel": _MPD,
    "post_dgrad_kernel": _MPD, "post_wgrad_kernel": _MPD, "act_bwd_kernel": _MPD, "im2col_t_kernel": _MPD,
    "unpack_wgrad_kernel": _MPD, "conv0_wgrad_kernel": _MPD, "conv0_dgrad_kernel": _MPD,
    # alignment, MAS, spectrograms, the mel loss, resampling
    "align_lengths_kernel": "tests/test_align.py::test_align_edges_vs_oracle",
    "align_expand_kernel": "tests/test_align.py::test_align_edges_vs_oracle",
    "mas_scores_kernel": "tests/test_mas.py::test_scores_vs_fp64",
    "mas_dp_kernel": "tests/test_mas.py::test_maximum_path_vs_reference_fixture",
    "mas_path_kernel": "tests/test_mas.py::test_maximum_path_vs_reference_fixture",
    "mas_loss_partial_kernel": "tests/test_mas.py::test_mas_losses_vs_fp64",
    "mas_loss_final_kernel": "tests/test_mas.py::test_mas_losses_vs_fp64",
    "mel_kernel": "tests/test_mel.py::test_gpu_vs_reference_golden",
    "mel_loss_kernel": "tests/test_mel_loss.py::test_gpu_vs_reference_and_oracle",
    "mel_loss_final_kernel": "tests/test_mel_loss.py::test_gpu_vs_reference_and_oracle",
    "mel_loss_gather_kernel": "tests/test_mel_loss.py::test_gpu_finite_differences",
    "resample_kernel": "tests/test_resample.py::test_gpu_vs_torchaudio_golden",
    # exempt
    "fill_pattern_kernel": "exempt: the synthetic operands of st_bench_conv's timing loop; no result depends on its values",
    "fill_kernel": "exempt: writes the constant 1.0 (the style encoder's all-ones pool mask for mask-less calls); checked "
                   "through the style encoder's outputs",
    "scale_kernel": "exempt: one fp32 multiply per element, folding the softmax scale into the style encoder's packed q "
                    "weights; checked through the style encoder's outputs",
}
EXEMPT = {"fill_pattern_kernel", "fill_kernel", "scale_kernel"}


def kernels_in_sources():
    """{kernel name: file} of every __global__ function in stabletts_b200/csrc/*.cu and *.cuh"""
    found = {}
    for path in sorted(glob.glob(os.path.join(ROOT, "stabletts_b200", "csrc", "*.cu*"))):
        src = open(path).read()
        for name in re.findall(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", src):
            found[name] = os.path.basename(path)
    return found


def test_every_kernel_answers_to_a_test():
    """each __global__ kernel has an entry; each entry names a kernel that exists and a test function that exists (or is
    one of the three exemptions, with its reason)"""
    found = kernels_in_sources()
    assert len(found) >= 60, sorted(found)
    missing = sorted(set(found) - set(KERNEL_TESTS))
    assert not missing, f"kernels without a kernel-level test entry: {missing}"
    stale = sorted(set(KERNEL_TESTS) - set(found))
    assert not stale, f"entries for kernels that no longer exist: {stale}"
    for kernel, where in KERNEL_TESTS.items():
        if where.startswith("exempt: "):
            assert kernel in EXEMPT and len(where) > 20, kernel
            continue
        assert kernel not in EXEMPT, kernel
        path, test = where.split("::")
        src = open(os.path.join(ROOT, path)).read()
        assert re.search(rf"^def {test}\(", src, re.M), (kernel, where)
