"""The fp32 row kernels against fp64 statements of their contracts (st_test_row_ex, include/stabletts_b200.h).

Kernels: film_ln_mod_kernel (FiLM·mask -> LayerNorm -> adaLN modulate, the CFM estimator's row kernel), dwconv_ln_kernel<C>
(depthwise k = 7 conv + affine LayerNorm of the vocoders' ConvNeXt blocks), and the Vocos head's spectrum_kernel,
idft_basis_kernel and overlap_add_kernel, and FireflyGAN's mean3_silu_kernel and post_conv_tanh_kernel.  The hook calls the
product's own launchers.

Each kind has an fp64 statement; the CPU tests pin it against independent torch code: gemm_contract_ref's fused LayerNorm
(imported from test_gemm_contract) against F.layer_norm, F.conv1d(groups=C) + F.layer_norm, vocoder_ref.head_spectrum, the
windowed torch.fft.irfft, vocoder_ref.istft_same_reference (F.fold), torch.stack(...).mean(0) + F.silu, F.conv1d + tanh.

Bars, against the fp64 statement on the same fp32 inputs:
  fp32 outputs: max |out - ref64| <= max(4 E32, 8 * 2^-24 * max |ref64|), E32 = max |torch fp32 - ref64| of the same
                operation done by the torch code in fp32 on the CPU;
  split planes: hi = bf16(out_f32) and lo = bf16(out_f32 - hi), bit for bit; the fp16 plane = cvt.rn(clamp(out_f32,
                +-65504)), bit for bit;
  IDFT_BASIS:   every entry within 1 fp32 ulp of the fp64 basis.
`pytest -s` prints the worst ratio to the bar per kind and case group."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import vocoder_ref as V
from kernel_harness import (LazyMatrix, NAN, bar, bits, check_planes, make_mask, report_worst_per_group, run_ok,
                            run_row_hook, set_fields)
from kernel_harness import dev, handle  # noqa: F401 (fixtures)
from test_gemm_contract import gemm_contract_ref, problem as gemm_problem

H = 256                                             # film_ln_mod_kernel's one width
WIDTHS = (128, 256, 384, 512, 768, 1024)            # dwconv_ln_kernel's instances
LN_EPS = 1e-5                                       # film_ln_mod_kernel
VOCOS_EPS = 1e-6                                    # the vocoders' LayerNorms
STFTS = ((2048, 512), (1024, 256), (2048, 128), (1280, 640))


def vocos_shapes(n_fft):
    """the head layout st_create_vocos derives: K bins, phases at Kp (128-aligned), head width Nh, spectrum width K2"""
    K = n_fft // 2 + 1
    Kp = (K + 127) // 128 * 128
    return dict(K=K, Kp=Kp, Nh=2 * Kp, K2=2 * ((K + 63) // 64 * 64))


# --------------------------------------------------------------------------------------------------------------------
# fp64 statements and the independent torch code
# --------------------------------------------------------------------------------------------------------------------
def _table_rows(table, idx, stride, off, n, dtype):
    return table.to(dtype)[idx[:, None] * stride + off + torch.arange(n)[None, :]][:, None, :]


def adaln_ref(d, t):
    """fp64 statement of ADALN: gemm_contract_ref's fused LayerNorm on an identity GEMM of x, with the FiLM table as film2
    (x2 = (gamma x + beta) * mask) and ln_mask_out = mask_out"""
    g = gemm_problem(B=d["B"], BB=d["BB"], T=d["T"], C0=H, N=H, flags=0, ln=1, ln_mask_out=d["mask_out"], mask=True,
                     film2=bool(d["has_film"]), c_clamp=d["c_clamp"], ada_bstride=d["ada_bstride"],
                     film2_bstride=d["film_bstride"])
    gt = {"A0": t["x"], "W": torch.eye(H, dtype=torch.float64)[:, :, None], "mask": t["mask"], "ln_shift": t["shift"],
          "ln_scale": t["scale"]}
    if d["has_film"]:
        gt["film2"] = t["film"]
    r = gemm_contract_ref(g, gt)
    return {"out": r["u"], "xout": r["out2"] if d["has_film"] else None}


def adaln_torch(d, t, dtype):
    """ADALN with F.layer_norm"""
    BB, B = d["BB"], d["B"]
    bb = torch.arange(BB)
    mb, cb = bb % B, bb.clamp(max=d["c_clamp"])
    x = t["x"].to(dtype)
    m = t["mask"].to(dtype)[mb][..., None]
    if d["has_film"]:
        x = (_table_rows(t["film"], mb, d["film_bstride"], 0, H, dtype) * x
             + _table_rows(t["film"], mb, d["film_bstride"], H, H, dtype)) * m
    sh = _table_rows(t["shift"], cb, d["ada_bstride"], 0, H, dtype)
    sc = _table_rows(t["scale"], cb, d["ada_bstride"], 0, H, dtype)
    u = F.layer_norm(x, (H,), eps=LN_EPS) * (1 + sc) + sh
    return {"out": u * m if d["mask_out"] else u, "xout": x if d["has_film"] else None}


def dwconv_ln_ref(d, t):
    """fp64 statement of DWCONV_LN: y[b, t, c] = bias[c] + sum_k w[c, 0, k] x[b, t + k - 3, c] over taps inside [0, T)
    (or y = x), then (y - mean) / sqrt(var + eps) * ln_w + ln_b with the biased variance"""
    x = t["x"].double()
    T = x.shape[1]
    if "w" in t:
        w = t["w"].double()
        y = t["bias"].double().expand_as(x).clone()
        for k in range(7):
            lo, hi = max(0, 3 - k), min(T, T + 3 - k)
            if lo < hi:
                y[:, lo:hi] += w[:, 0, k] * x[:, lo + k - 3:hi + k - 3]
    else:
        y = x
    mean = y.mean(-1, keepdim=True)
    var = ((y - mean) ** 2).mean(-1, keepdim=True)
    return {"out": (y - mean) / torch.sqrt(var + d["eps"]) * t["ln_w"].double() + t["ln_b"].double()}


def dwconv_ln_torch(d, t, dtype):
    """DWCONV_LN with F.conv1d(groups=C) + F.layer_norm"""
    x = t["x"].to(dtype)
    C_ = x.shape[-1]
    if "w" in t:
        x = F.conv1d(x.transpose(1, 2), t["w"].to(dtype), t["bias"].to(dtype), padding=3, groups=C_).transpose(1, 2)
    return {"out": F.layer_norm(x, (C_,), t["ln_w"].to(dtype), t["ln_b"].to(dtype), d["eps"])}


def spectrum_ref(d, t):
    """fp64 statement of SPECTRUM: min(exp(m), 1e2) (cos p | sin p) into the [re | im] halves of K2, zeros elsewhere"""
    K, Kp, K2 = d["K"], d["Kp"], d["K2"]
    x = t["x"].double()
    mag = torch.exp(x[..., :K]).clamp(max=1e2)
    p = x[..., Kp:Kp + K]
    out = torch.zeros(*x.shape[:-1], K2, dtype=torch.float64)
    out[..., :K] = mag * torch.cos(p)
    out[..., K2 // 2:K2 // 2 + K] = mag * torch.sin(p)
    return {"out": out}


def spectrum_torch(d, t, dtype):
    """SPECTRUM through vocoder_ref.head_spectrum (head.py:101-113) with a head Linear that selects the two column groups"""
    K, Kp, K2, Nh = d["K"], d["Kp"], d["K2"], d["Nh"]
    x = t["x"].to(dtype).clone()
    keep = torch.zeros(Nh, dtype=torch.bool)
    keep[:K] = True
    keep[Kp:Kp + K] = True
    x[..., ~keep] = 0.0                              # the NaN the kernel must not read would poison the selection matrix
    sel = torch.zeros(2 * K, Nh, dtype=dtype)
    sel[torch.arange(K), torch.arange(K)] = 1.0
    sel[K + torch.arange(K), Kp + torch.arange(K)] = 1.0
    re, im = V.head_spectrum({"head.out.weight": sel, "head.out.bias": torch.zeros(2 * K, dtype=dtype)}, x)
    out = torch.zeros(*x.shape[:-1], K2, dtype=dtype)
    out[..., :K] = re.transpose(1, 2)
    out[..., K2 // 2:K2 // 2 + K] = im.transpose(1, 2)
    return {"out": out}


def idft_basis_ref(window, n_fft, K2):
    """fp64 statement of IDFT_BASIS, (n_fft, K2).  The angle 2 pi ((k n) mod n_fft) / n_fft is reduced exactly in integers,
    and the quadrant points, where cos or sin is exactly 0 or +-1, take their exact values."""
    K = n_fft // 2 + 1
    k = torch.arange(K, dtype=torch.int64)[:, None]
    n = torch.arange(n_fft, dtype=torch.int64)[None, :]
    r = (k * n) % n_fft
    ang = 2 * math.pi * r.double() / n_fft
    cs, sn = torch.cos(ang), torch.sin(ang)
    quad = (4 * r) % n_fft == 0
    q = (4 * r) // n_fft
    cs = torch.where(quad, torch.tensor([1.0, 0.0, -1.0, 0.0], dtype=torch.float64)[q % 4], cs)
    sn = torch.where(quad, torch.tensor([0.0, 1.0, 0.0, -1.0], dtype=torch.float64)[q % 4], sn)
    c = torch.full((K, 1), 2.0, dtype=torch.float64)
    c[0] = c[-1] = 1.0
    wr = c * cs / n_fft
    wi = -c * sn / n_fft
    wi[0] = wi[-1] = 0.0
    W = torch.zeros(n_fft, K2, dtype=torch.float64)
    w = window.double()[:, None]
    W[:, :K] = wr.T * w
    W[:, K2 // 2:K2 // 2 + K] = wi.T * w
    return W


def overlap_add_ref(frames, window, hop):
    """fp64 statement of OVERLAP_ADD: for each output sample s (position s + pad of the untrimmed signal) the sum of
    frames[b, t, s + pad - t hop] over the frames t in [0, T) that cover it, over the sum of window^2 over the same frames"""
    B, T, n_fft = frames.shape
    pad = (n_fft - hop) // 2
    pos = torch.arange(T * hop) + pad
    acc = torch.zeros(B, T * hop, dtype=torch.float64)
    env = torch.zeros(T * hop, dtype=torch.float64)
    fr, w = frames.double(), window.double()
    for t in range(T):
        n = pos - t * hop
        ok = (n >= 0) & (n < n_fft)
        acc[:, ok] += fr[:, t, n[ok]]
        env[ok] += w[n[ok]] ** 2
    return acc / env


def overlap_add_torch(frames, window, hop, dtype):
    """OVERLAP_ADD as the reference's ISTFT does it after the irfft (head.py:66-81): F.fold, envelope, trim"""
    B, T, n_fft = frames.shape
    pad = (n_fft - hop) // 2
    size = (T - 1) * hop + n_fft
    fold = lambda z: F.fold(z, output_size=(1, size), kernel_size=(1, n_fft), stride=(1, hop))[:, 0, 0]   # noqa: E731
    y = fold(frames.to(dtype).transpose(1, 2))
    env = fold(window.to(dtype).square()[None, :, None].expand(1, n_fft, T))
    return (y / env)[:, pad:size - pad]


def mean3_silu_ref(t):
    """fp64 statement of MEAN3_SILU: v = (r0 + r1 + r2) / 3, v / (1 + exp(-v))"""
    v = (t["x"].double() + t["x1"].double() + t["x2"].double()) / 3.0
    return {"out": v / (1.0 + torch.exp(-v))}


def mean3_silu_torch(t, dtype):
    return {"out": F.silu(torch.stack([t["x"].to(dtype), t["x1"].to(dtype), t["x2"].to(dtype)]).mean(0))}


def post_tanh_ref(t):
    """fp64 statement of POST_TANH: tanh(bias + sum_{k, c} w[0, c, k] x[b, s + k - 6, c]) over taps inside [0, L)"""
    x, w = t["x"].double(), t["w"].double()
    B, L, _ = x.shape
    acc = torch.full((B, L), float(t["bias"].double()[0]), dtype=torch.float64)
    for k in range(13):
        lo, hi = max(0, 6 - k), min(L, L + 6 - k)
        if lo < hi:
            acc[:, lo:hi] += x[:, lo + k - 6:hi + k - 6] @ w[0, :, k]
    return {"out": torch.tanh(acc)}


def post_tanh_torch(t, dtype):
    return {"out": torch.tanh(F.conv1d(t["x"].to(dtype).transpose(1, 2), t["w"].to(dtype), t["bias"].to(dtype), padding=6))[:, 0]}


def reference(d, t):
    """(fp64 statement, torch fp32) of case d on operands t"""
    k = d["kind"]
    if k == "ADALN":
        return adaln_ref(d, t), adaln_torch(d, t, torch.float32)
    if k == "DWCONV_LN":
        return dwconv_ln_ref(d, t), dwconv_ln_torch(d, t, torch.float32)
    if k == "SPECTRUM":
        return spectrum_ref(d, t), spectrum_torch(d, t, torch.float32)
    if k == "OVERLAP_ADD":
        return ({"out": overlap_add_ref(t["x"], t["window"], d["hop"])},
                {"out": overlap_add_torch(t["x"], t["window"], d["hop"], torch.float32)})
    if k == "MEAN3_SILU":
        return mean3_silu_ref(t), mean3_silu_torch(t, torch.float32)
    if k == "POST_TANH":
        return post_tanh_ref(t), post_tanh_torch(t, torch.float32)
    raise KeyError(k)


# --------------------------------------------------------------------------------------------------------------------
# cases and their operands
# --------------------------------------------------------------------------------------------------------------------
def make_operands(d, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)                               # noqa: E731
    ru = lambda *s: torch.rand(*s, generator=g) * 2 - 1                       # noqa: E731
    k = d["kind"]
    if k == "ADALN":
        B, BB, T = d["B"], d["BB"], d["T"]
        x = rn(BB, T, H) * d.get("spread", 1.0) + d.get("offset", 0.0)
        if d.get("const_rows"):                      # every row constant, values that sum exactly in fp32
            x = (torch.randint(-16, 16, (BB, T, 1), generator=g) * 0.375).expand(BB, T, H).contiguous()
        t = {"x": x, "mask": make_mask(B, T, g, d.get("fractional", False))}
        if d["has_film"]:
            t["film"] = 1.0 + 0.5 * rn((B - 1) * d["film_bstride"] + 2 * H)
        rows = min(BB - 1, d["c_clamp"]) + 1
        t["shift"] = 0.5 * rn((rows - 1) * d["ada_bstride"] + H) * d.get("shift_gain", 1.0)
        t["scale"] = 0.5 * rn((rows - 1) * d["ada_bstride"] + H)
        return t
    if k == "DWCONV_LN":
        B, T, C_ = d["B"], d["T"], d["C"]
        gains = torch.tensor([1.0, 30.0, 0.03][:B]) if B > 1 else torch.ones(1)   # ragged content per utterance
        t = {"x": (rn(B, T, C_) * d.get("spread", 1.0) + d.get("offset", 0.0)) * gains[:, None, None]}
        if d["conv"]:
            t["w"] = ru(C_, 1, 7) / math.sqrt(7)
            t["bias"] = 0.1 * ru(C_) * d.get("spread", 1.0)
        t["ln_w"], t["ln_b"] = 1 + 0.1 * rn(C_), 0.1 * rn(C_)
        return t
    if k == "SPECTRUM":
        rows, Nh, K, Kp = d["B"] * d["T"], d["Nh"], d["K"], d["Kp"]
        x = torch.full((d["B"], d["T"], Nh), NAN)                  # the columns outside the two groups must not be read
        m = math.log(100.0) + 1.5 * rn(d["B"], d["T"], K)
        p = 3.0 * rn(d["B"], d["T"], K)
        if d.get("extremes"):
            flat = m.view(-1)
            flat[0::7] = 100.0                                     # exp overflows to inf: the clip must give 100
            flat[1::7] = -200.0                                    # exp underflows to 0
            flat[2::7] = 88.72                                     # exp(m) at the fp32 overflow edge
            flat[3::7] = math.log(100.0)
            p = 1e4 * ru(d["B"], d["T"], K)                        # |phase| up to 1e4
        x[..., :K] = m
        x[..., Kp:Kp + K] = p
        return {"x": x}
    if k == "OVERLAP_ADD":
        win = torch.hann_window(d["n_fft"]) if d["window"] == "hann" else torch.hamming_window(d["n_fft"])
        return {"x": rn(d["B"], d["T"], d["n_fft"]) * win, "window": win}
    if k == "IDFT_BASIS":
        return {"window": torch.hann_window(d["n_fft"]) if d["window"] == "hann" else torch.hamming_window(d["n_fft"])}
    if k == "MEAN3_SILU":
        n, a = d["n"], d.get("amp")
        if a is None:
            return {"x": 2 * rn(n), "x1": 2 * rn(n), "x2": 2 * rn(n)}
        sgn = lambda: torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)   # noqa: E731
        return {"x": a * sgn(), "x1": a * sgn(), "x2": a * sgn() * torch.rand(n, generator=g)}
    if k == "POST_TANH":
        return {"x": 0.5 * rn(d["B"], d["T"], 16), "w": 3 * ru(1, 16, 13) / math.sqrt(16 * 13), "bias": 0.1 * ru(1)}
    raise KeyError(k)


def _cases():
    cs = {}

    def add(name, kind, group, **kw):
        d = dict(kind=kind, group=group, planes=None)
        d.update(kw)
        cs[name] = d

    def adaln(name, group, B, BB, T, film="sample", alias=False, mask_out=1, c_clamp=None, ada_bstride=H, **kw):
        add(name, "ADALN", group, B=B, BB=BB, T=T, C=H, has_film=int(film is not None), alias="xout" if alias else None,
            mask_out=mask_out, film_bstride=2 * H if film == "sample" else 0, c_clamp=BB - 1 if c_clamp is None else c_clamp,
            ada_bstride=ada_bstride, **kw)

    # ADALN: odd row counts (the two-rows-per-warp tail), CFG row mapping, FiLM per sample / shared / off, aliasing, mask_out
    adaln("adaln_t1", "shapes", 1, 1, 1, planes="split")
    adaln("adaln_b3_t37_alias", "shapes", 3, 3, 37, alias=True, planes="split")
    adaln("adaln_t1000_shared_film", "shapes", 2, 2, 1000, film="shared", mask_out=0)
    adaln("adaln_cfg_t37", "cfg", 3, 6, 37, film="shared", mask_out=0, c_clamp=3)
    adaln("adaln_cfg_t1000_alias", "cfg", 2, 4, 1000, alias=True, c_clamp=2, ada_bstride=3 * H, planes="split")
    adaln("adaln_cfg_t1_nofilm_u16", "cfg", 1, 2, 1, film=None, c_clamp=1, planes="u16")
    adaln("adaln_nofilm_t1000_u16", "film", 2, 4, 1000, film=None, mask_out=0, c_clamp=2, planes="u16")
    adaln("adaln_nofilm_maskout_t37", "film", 1, 1, 37, film=None)
    adaln("adaln_fractional_mask", "masks", 2, 2, 37, fractional=True, planes="split")
    adaln("adaln_fractional_mask_cfg", "masks", 2, 4, 37, fractional=True, mask_out=0, c_clamp=2, alias=True)
    adaln("adaln_offset_rows", "values", 1, 1, 37, film=None, offset=100.0, spread=1.0)
    adaln("adaln_offset_rows_cfg", "values", 2, 4, 1000, film=None, offset=-100.0, spread=1.0, c_clamp=2, mask_out=0)
    adaln("adaln_constant_rows", "values", 2, 2, 37, film=None, const_rows=True)
    adaln("adaln_constant_rows_nomask", "values", 1, 1, 37, film=None, const_rows=True, mask_out=0)
    adaln("adaln_fp16_saturates", "values", 1, 2, 37, film=None, mask_out=0, shift_gain=3e5, planes="u16")
    # DWCONV_LN: every width with and without the conv; short T with B = 3 utterances of different scale; variance ~ eps
    for C_ in WIDTHS:
        add(f"dwconv_c{C_}", "DWCONV_LN", "widths", B=2, T=37, C=C_, conv=True, eps=VOCOS_EPS, planes="split")
        add(f"ln_c{C_}", "DWCONV_LN", "widths", B=2, T=37, C=C_, conv=False, eps=VOCOS_EPS)
    for T in (1, 2, 3, 6, 7, 8):
        add(f"dwconv_b3_t{T}", "DWCONV_LN", "short", B=3, T=T, C=512 if T % 2 else 768, conv=True, eps=VOCOS_EPS,
            planes="split" if T == 7 else None)
    add("dwconv_var_near_eps_c512", "DWCONV_LN", "eps", B=2, T=37, C=512, conv=True, eps=VOCOS_EPS, spread=1e-3)
    add("ln_var_near_eps_c768", "DWCONV_LN", "eps", B=2, T=37, C=768, conv=False, eps=VOCOS_EPS, spread=1e-3)
    add("ln_var_near_eps_c128_eps1e-5", "DWCONV_LN", "eps", B=1, T=9, C=128, conv=False, eps=1e-5, spread=3e-3)
    add("ln_offset_rows_c1024", "DWCONV_LN", "eps", B=2, T=37, C=1024, conv=False, eps=VOCOS_EPS, offset=100.0)
    # SPECTRUM
    for n_fft in (1024, 1280, 2048):
        add(f"spectrum_straddle_nfft{n_fft}", "SPECTRUM", "spectrum", B=2, T=37, planes="split", **vocos_shapes(n_fft))
        add(f"spectrum_extremes_nfft{n_fft}", "SPECTRUM", "spectrum", B=1, T=13, extremes=True, **vocos_shapes(n_fft))
    # OVERLAP_ADD (IDFT_BASIS runs in its own test: its bar is in ulps)
    for n_fft, hop in STFTS:
        for win in ("hann", "hamming"):
            for T in (1, 2, 3, 4, 130):
                add(f"ola_{n_fft}_{hop}_{win}_t{T}", "OVERLAP_ADD", "overlap_add", B=3, T=T, n_fft=n_fft, hop=hop, window=win)
    # MEAN3_SILU
    add("mean3_n4", "MEAN3_SILU", "mean3", n=4, planes="split")
    add("mean3_large", "MEAN3_SILU", "mean3", n=3 * 2 ** 18 + 4, planes="split")
    add("mean3_pm1e4", "MEAN3_SILU", "mean3", n=4096, amp=1e4, planes="split")
    add("mean3_pm100", "MEAN3_SILU", "mean3", n=4096, amp=100.0)
    # POST_TANH
    for L in (1, 13, 1000):
        add(f"post_tanh_b3_l{L}", "POST_TANH", "post_tanh", B=3, T=L, C=16)
    return cs


CASES = _cases()


# --------------------------------------------------------------------------------------------------------------------
# CPU: every fp64 statement against independent torch code
# --------------------------------------------------------------------------------------------------------------------
def _close(a, b, tol=1e-10):
    a, b = a.double(), b.double()
    assert torch.allclose(a, b, rtol=tol, atol=tol), float((a - b).abs().max())


@pytest.mark.parametrize("name", ["adaln_b3_t37_alias", "adaln_cfg_t37", "adaln_nofilm_maskout_t37", "adaln_fractional_mask_cfg",
                                  "adaln_cfg_t1000_alias"])
def test_adaln_statement_matches_layer_norm(name):
    d = CASES[name]
    t = make_operands(d, 1)
    r, w = adaln_ref(d, t), adaln_torch(d, t, torch.float64)
    _close(r["out"], w["out"])
    if d["has_film"]:
        _close(r["xout"], w["xout"])


@pytest.mark.parametrize("name", ["dwconv_c128", "ln_c256", "dwconv_b3_t1", "dwconv_b3_t2", "dwconv_b3_t6", "dwconv_var_near_eps_c512"])
def test_dwconv_ln_statement_matches_conv1d_layer_norm(name):
    d = CASES[name]
    t = make_operands(d, 2)
    _close(dwconv_ln_ref(d, t)["out"], dwconv_ln_torch(d, t, torch.float64)["out"])


@pytest.mark.parametrize("name", ["spectrum_straddle_nfft1280", "spectrum_extremes_nfft2048"])
def test_spectrum_statement_matches_head_spectrum(name):
    d = CASES[name]
    t = make_operands(d, 3)
    r, w = spectrum_ref(d, t)["out"], spectrum_torch(d, t, torch.float64)["out"]
    assert torch.equal(r, w)                             # the same elementwise double operations
    assert float(r.abs().max()) <= 100.0 + 1e-12 and torch.isfinite(r).all()


@pytest.mark.parametrize("n_fft", [1024, 1280, 2048])
def test_idft_basis_statements_match_windowed_irfft(n_fft):
    """vocoder_ref.idft_basis against torch.fft.irfft x window on unit spectra, and the exactly reduced statement against it"""
    win = torch.hamming_window(n_fft, dtype=torch.float64)
    K = n_fft // 2 + 1
    Wv = V.idft_basis(win, n_fft)                        # (2K, n_fft)
    eye = torch.eye(K, dtype=torch.complex128)
    want_re = torch.fft.irfft(eye, n_fft, dim=1) * win
    want_im = torch.fft.irfft(1j * eye, n_fft, dim=1) * win
    _close(Wv[:K], want_re, 1e-12)
    _close(Wv[K:], want_im, 1e-12)
    K2 = vocos_shapes(n_fft)["K2"]
    W = idft_basis_ref(win, n_fft, K2)
    _close(W[:, :K], Wv[:K].T, 1e-11)
    _close(W[:, K2 // 2:K2 // 2 + K], Wv[K:].T, 1e-11)
    assert (W[:, K:K2 // 2] == 0).all() and (W[:, K2 // 2 + K:] == 0).all()


@pytest.mark.parametrize("n_fft,hop", STFTS)
@pytest.mark.parametrize("T", [1, 2, 5])
def test_overlap_add_statement_matches_istft_same_reference(n_fft, hop, T):
    """frames = irfft(S) x window through the statement equal the reference ISTFT (F.fold) of S"""
    g = torch.Generator().manual_seed(T)
    K = n_fft // 2 + 1
    re, im = torch.randn(2, K, T, generator=g, dtype=torch.float64), torch.randn(2, K, T, generator=g, dtype=torch.float64)
    win = torch.hann_window(n_fft, dtype=torch.float64)
    frames = (torch.fft.irfft(torch.complex(re, im), n_fft, dim=1) * win[None, :, None]).transpose(1, 2)
    want = V.istft_same_reference(re, im, win, n_fft, hop)
    _close(overlap_add_ref(frames, win, hop), want, 1e-12)
    _close(overlap_add_torch(frames, win, hop, torch.float64), want, 1e-12)


@pytest.mark.parametrize("name", ["mean3_n4", "mean3_pm1e4", "mean3_pm100"])
def test_mean3_silu_statement_matches_silu(name):
    t = make_operands(CASES[name], 4)
    r = mean3_silu_ref(t)["out"]
    assert torch.isfinite(r).all()
    _close(r, mean3_silu_torch(t, torch.float64)["out"], 1e-12)


@pytest.mark.parametrize("L", [1, 13, 40])
def test_post_tanh_statement_matches_conv1d(L):
    d = dict(kind="POST_TANH", B=3, T=L)
    t = make_operands(d, 5)
    _close(post_tanh_ref(t)["out"], post_tanh_torch(t, torch.float64)["out"], 1e-12)


def test_vocos_shapes_match_the_handle_layout():
    assert vocos_shapes(2048) == dict(K=1025, Kp=1152, Nh=2304, K2=2176)
    assert vocos_shapes(1280) == dict(K=641, Kp=768, Nh=1536, K2=1408)


# --------------------------------------------------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------------------------------------------------
def check_case(d, t, o):
    """value checks against the fp64 statement; returns [(output, max |err|, bar)]"""
    ref, f32 = reference(d, t)
    rows = []
    for what in ("out", "xout"):
        if ref.get(what) is None:
            continue
        got = o[what].double()
        assert torch.isfinite(got).all(), what
        e32 = float((f32[what].double() - ref[what]).abs().max())
        err = float((got - ref[what]).abs().max())
        b = bar(ref[what], e32)
        rows.append((what, err, b))
        assert err <= b, (what, err, b, e32)
    check_planes(o, d.get("planes"))
    if d["kind"] == "ADALN":
        # rows whose LayerNorm input is constant (FiLM'd rows with mask 0, or constant x) give exactly shift [* mask]
        BB, B = d["BB"], d["B"]
        bb = torch.arange(BB)
        mb, cb = bb % B, bb.clamp(max=d["c_clamp"])
        m = t["mask"][mb]
        const = (m == 0) if d["has_film"] else torch.ones_like(m, dtype=torch.bool) if d.get("const_rows") else torch.zeros_like(m, dtype=torch.bool)
        sh = t["shift"][cb[:, None] * d["ada_bstride"] + torch.arange(H)[None, :]][:, None, :].expand(BB, d["T"], H)
        want = sh * m[..., None] if d["mask_out"] else sh
        assert torch.equal(o["out"][const], want[const])
        if d["has_film"]:
            assert (o["xout"][m == 0] == 0).all()
    if d["kind"] == "SPECTRUM":
        K, K2 = d["K"], d["K2"]
        assert (o["out"][..., K:K2 // 2] == 0).all() and (o["out"][..., K2 // 2 + K:] == 0).all()
        assert float(o["out"].abs().max()) <= 100.0
    if d["kind"] == "MEAN3_SILU" and d.get("amp"):
        v = (t["x"] + t["x1"] + t["x2"]) / 3.0                               # the kernel's fp32 mean, same order
        assert torch.equal(o["out"][v > 50], v[v > 50])                      # silu(v) = v in fp32 for large v
        assert (o["out"][v < -60].abs() <= 1e-20).all()                      # and -> 0 for large negative v
    return rows


@pytest.fixture(scope="module")
def matrix(dev, handle):
    def run(name):
        d = CASES[name]
        t = make_operands(d, 1000 + list(CASES).index(name))
        return check_case(d, t, run_ok(run_row_hook, *handle, d, t, dev))
    return LazyMatrix(run)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_matrix(name, matrix):
    matrix.check(name)


@pytest.mark.gpu
def test_every_group_ran(matrix):
    """and prints the worst ratio to the bar per kind and case group (pytest -s)"""
    report_worst_per_group(matrix, CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("window", ["hann", "hamming"])
@pytest.mark.parametrize("n_fft,hop", STFTS)
def test_idft_basis_within_one_ulp(n_fft, hop, window, dev, handle):
    """every entry of the basis within 1 fp32 ulp of the fp64 statement (it is evaluated in double and rounded once)"""
    lib, h = handle
    d = dict(kind="IDFT_BASIS", n_fft=n_fft, K2=vocos_shapes(n_fft)["K2"], window=window)
    t = make_operands(d, 7)
    o = run_ok(run_row_hook, lib, h, d, t, dev)
    ref = idft_basis_ref(t["window"], n_fft, d["K2"])
    r32 = ref.float().abs()
    ulp = (torch.nextafter(r32, torch.tensor(math.inf)) - r32).double()
    excess = (o["out"].double() - ref).abs() / ulp
    print(f"IDFT_BASIS {n_fft} {window}: worst |W - ref64| = {float(excess.max()):.3f} ulp")
    assert float(excess.max()) <= 1.0


# ---- properties that need no tolerance -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["adaln_cfg_t1000_alias", "dwconv_c1024", "spectrum_straddle_nfft2048",
                                  "ola_2048_128_hann_t130", "mean3_large", "post_tanh_b3_l1000"])
def test_repeated_runs_are_bit_identical(name, dev, handle):
    lib, h = handle
    d = CASES[name]
    t = make_operands(d, 77)
    first = run_ok(run_row_hook, lib, h, d, t, dev)
    again = run_ok(run_row_hook, lib, h, d, t, dev)
    for k in first:
        assert torch.equal(bits(first[k]), bits(again[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dwconv_b3_t7", "dwconv_b3_t2", "ln_c384", "ola_1024_256_hamming_t130",
                                  "ola_2048_512_hann_t3", "post_tanh_b3_l13"])
def test_utterance_alone_equals_its_batch_row(name, dev, handle):
    """utterance 1 of a B = 3 batch, run alone, gives the bits of its batch row: nothing crosses an utterance edge"""
    lib, h = handle
    d = CASES[name]
    t = make_operands(d, 78)
    whole = run_ok(run_row_hook, lib, h, d, t, dev)
    d1 = dict(d, B=1)
    t1 = {k: (v[1:2].contiguous() if k == "x" else v) for k, v in t.items()}
    one = run_ok(run_row_hook, lib, h, d1, t1, dev)
    assert torch.equal(bits(one["out"][0]), bits(whole["out"][1]))


@pytest.mark.gpu
def test_cfg_uncond_rows_ignore_the_cond_rows_adaln(dev, handle):
    """BB = 2B, c_clamp = B: rows B..2B-1 read adaLN row B; new adaLN rows 0..B-1 leave them bit-identical"""
    lib, h = handle
    d = CASES["adaln_cfg_t37"]
    t = make_operands(d, 79)
    a = run_ok(run_row_hook, lib, h, d, t, dev)
    t2 = dict(t)
    B, s = d["B"], d["ada_bstride"]
    t2["shift"], t2["scale"] = t["shift"].clone(), t["scale"].clone()
    t2["shift"][:B * s] += 1.0
    t2["scale"][:B * s] -= 0.5
    b = run_ok(run_row_hook, lib, h, d, t2, dev)
    assert torch.equal(bits(a["out"][B:]), bits(b["out"][B:]))
    assert not torch.equal(a["out"][:B], b["out"][:B])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["adaln_b3_t37_alias", "adaln_fractional_mask_cfg"])
def test_garbage_in_masked_frames_does_not_reach_unmasked_rows(name, dev, handle):
    """+-1e6 in x at the frames with mask 0 leaves every other row's u (and xout) bit-identical"""
    lib, h = handle
    d = CASES[name]
    t = make_operands(d, 80)
    clean = run_ok(run_row_hook, lib, h, d, t, dev)
    m = t["mask"][torch.arange(d["BB"]) % d["B"]] == 0
    dirty = dict(t)
    dirty["x"] = t["x"].clone()
    junk = (torch.rand(t["x"].shape, generator=torch.Generator().manual_seed(81)) * 2 - 1) * 1e6
    dirty["x"][m] = junk[m]
    o = run_ok(run_row_hook, lib, h, d, dirty, dev)
    assert torch.equal(bits(clean["out"][~m]), bits(o["out"][~m]))
    assert torch.equal(bits(clean["xout"][~m]), bits(o["xout"][~m]))
    assert (o["xout"][m] == 0).all()


@pytest.mark.gpu
def test_refusals(dev, handle):
    """every problem outside the contract is refused with a readable error, and nothing is launched"""
    lib, h = handle

    def refused(name, needle, planes=None, **fields):
        d = CASES[name]
        t = make_operands(d, 90)
        rc, err, o = run_row_hook(lib, h, d, t, dev, planes=planes, desc_edit=set_fields(**fields))
        assert rc != 0 and needle in err, (name, needle, err)
        assert all(torch.isnan(v.float()).all() for k, v in o.items() if k != d.get("alias")), name

    refused("dwconv_c128", "C must be 128, 256, 384, 512, 768 or 1024", C=640)
    refused("dwconv_c128", "C must be 128, 256, 384, 512, 768 or 1024", C=64)
    refused("adaln_t1", "must be 256", C=128)
    refused("adaln_t1", "must be 256", C=512)
    refused("adaln_nofilm_maskout_t37", "out_lo must be NULL", planes="split", u16=1)
    refused("adaln_t1", "out_hi and out_lo go together", planes="split", out_lo=None)
    refused("dwconv_c256", "out_hi and out_lo go together", planes="split", out_hi=None)
    refused("spectrum_straddle_nfft1024", "out_hi and out_lo go together", planes="split", out_lo=None)
    refused("mean3_n4", "out_hi and out_lo go together", planes="split", out_hi=None)
    refused("dwconv_c256", "u16 belongs to ADALN", planes="split", u16=1, out_lo=None)
    refused("ola_2048_512_hann_t2", "multiple of 128 and of hop_length", hop=384)
    refused("ola_2048_512_hann_t2", "multiple of 128 and of hop_length", hop=64)          # 32 overlapping frames
    refused("ola_2048_512_hann_t2", "multiple of 128 and of hop_length", n_fft=2000)
    refused("ola_2048_512_hann_t2", "empty (B, 0)", hop=2048)
    refused("mean3_n4", "positive multiple of 4", n=6)
    refused("mean3_n4", "positive multiple of 4", n=0)
    refused("adaln_t1", "required", mask=None)
    refused("adaln_t1", "required", shift=None)
    refused("adaln_t1", "has_film needs film and xout", xout=None)
    refused("adaln_nofilm_maskout_t37", "belong to has_film", xout=1 << 20)
    refused("dwconv_c256", "required", ln_w=None)
    refused("dwconv_c256", "required", bias=None)
    refused("spectrum_straddle_nfft1024", "required", x=None)
    refused("spectrum_straddle_nfft1024", "K <= Kp", Kp=100)
    refused("ola_2048_512_hann_t2", "required", window=None)
    refused("mean3_n4", "required", x2=None)
    refused("post_tanh_b3_l13", "required", w=None)
    refused("post_tanh_b3_l13", "C must be 16", C=32)
    refused("adaln_t1", "no output requested", planes="", out_f32=None)
    from stabletts_b200 import _lib
    refused("adaln_t1", "unknown kind", kind=len(_lib.ST_TEST_ROW_KINDS))      # the first kind past the last one
    refused("adaln_t1", "unknown kind", kind=-1)
