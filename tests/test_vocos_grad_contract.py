"""The Vocos generator's backward row kernels and packings (vocos_grad.cu) against fp64 statements of their contracts,
through st_test_vocos_grad_ex (include/stabletts_b200.h), one kernel per call.

Bars on the GPU: fp32 outputs within max(4 E32, 8 ulp of max |ref64|) of the fp64 statement, E32 = max |the same
statement in torch fp32 - ref64| (kernel_harness.bar); the layer scale, the transposes and the unpack bit for bit.  The
statements are oracle/vocos_grad_ref.py's adjoints (pinned against torch's float64 autograd by test_vocos_grad_oracle.py).
Shapes cover T = 1, 2, 3, 7 and 40 (every depthwise-conv edge), the three LayerNorm widths, B T not a multiple of 32, the
clip boundary of the spectrum and the head's two column groups.

The module also registers these kernels in the library's kernel inventory (test_pack_contract.KERNEL_TESTS), next to the
test that checks them."""
import math

import pytest
import torch
import torch.nn.functional as F

import test_pack_contract as _inventory
from kernel_harness import LazyMatrix, bar, bits, split_bf16
from kernel_harness import dev, handle  # noqa: F401 (fixtures)
from oracle import vocos_grad_ref as G

_HERE = "tests/test_vocos_grad_contract.py::test_matrix"
_inventory.KERNEL_TESTS.update({k: _HERE for k in (
    "frame_grad_kernel", "spectrum_grad_kernel", "ln_bwd_kernel", "dwconv_adj_kernel", "col_sum_kernel",
    "dwconv_wgrad_kernel", "scale_cols_kernel", "gelu_bwd_kernel", "transpose_rows_kernel", "wgrad_unpack_kernel")})


# --------------------------------------------------------------------------------------------------------------------
# the statements, in a given dtype (fp64: the reference; fp32: its E32)
# --------------------------------------------------------------------------------------------------------------------
def frame_grad_ref(g, win, T, n_fft, hop, dt):
    B = g.shape[0]
    pad = (n_fft - hop) // 2
    s = torch.arange(T * hop) + pad
    env = torch.zeros(T * hop, dtype=dt)
    for j in range(n_fft // hop):
        t = s // hop - j
        ok = (t >= 0) & (t < T)
        env = env + torch.where(ok, win.to(dt)[(s - t * hop).clamp(0, n_fft - 1)].square(), torch.zeros((), dtype=dt))
    ss = torch.arange(T)[:, None] * hop + torch.arange(n_fft)[None, :] - pad
    ok = (ss >= 0) & (ss < T * hop)
    return torch.where(ok[None], (g.to(dt) / env[None])[:, ss.clamp(0, T * hop - 1)], torch.zeros((), dtype=dt))


def dw_ref(x, w, b, dt):
    """z = b + sum_k w[k][c] x[t + k - 3, c] per utterance; x (B, T, C), w [7][C]"""
    C = x.shape[-1]
    return F.conv1d(x.to(dt).transpose(1, 2), w.to(dt).T[:, None, :], b.to(dt), padding=3, groups=C).transpose(1, 2)


def ln_bwd_ref(x, w, b, lnw, g, eps, dt):
    B, T, C = x.shape
    z = dw_ref(x, w, b, dt) if w is not None else x.to(dt)
    z, gg = z.reshape(-1, C), g.to(dt).reshape(-1, C)
    mean = z.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((z - mean) ** 2).mean(-1, keepdim=True) + eps)
    zh = (z - mean) * rstd
    dx, _, _ = G.ln_bwd(z, lnw.to(dt), gg, eps)
    return dx.reshape(B, T, C), zh.reshape(B, T, C)


def gelu_bwd_ref(h, dg, dt):
    h, dg = h.to(dt), dg.to(dt)
    return dg * (0.5 * (1 + torch.erf(h / math.sqrt(2))) + h * torch.exp(-0.5 * h * h) / math.sqrt(2 * math.pi))


# --------------------------------------------------------------------------------------------------------------------
# the hook
# --------------------------------------------------------------------------------------------------------------------
def run_hook(handle, kind, out_shapes, **fields):
    """fields: tensors (moved to the GPU) or ints / floats; out_shapes: {name: shape or (shape, initial tensor)}"""
    from stabletts_b200 import _lib
    lib, h = handle
    d = _lib.StTestVocosGradDesc()
    d.kind = _lib.ST_TEST_VOCOS_GRAD_KINDS.index(kind)
    keep, outs = [], {}
    for k, v in fields.items():
        if isinstance(v, torch.Tensor):
            t = v.contiguous().cuda()
            keep.append(t)
            setattr(d, k, t.data_ptr())
        else:
            setattr(d, k, v)
    for k, spec in out_shapes.items():
        if isinstance(spec, tuple) and len(spec) == 2 and isinstance(spec[1], torch.Tensor):
            t = spec[1].clone().contiguous().cuda()
        else:
            t = torch.full(spec, float("nan"), device="cuda") if k.endswith("f32") else \
                torch.zeros(spec, dtype=torch.bfloat16, device="cuda")
        outs[k] = t
        setattr(d, k, t.data_ptr())
    rc = lib.st_test_vocos_grad_ex(h, C_byref(d), None)
    assert rc == 0, lib.st_last_error(h).decode()
    return {k: v.cpu() for k, v in outs.items()}


def C_byref(d):
    import ctypes
    return ctypes.byref(d)


def within(out, ref64, ref32, what):
    b = bar(ref64, float((ref32.double() - ref64).abs().max()))
    err = float((out.double() - ref64).abs().max())
    assert err <= b, (what, err, b)
    return err / b


# --------------------------------------------------------------------------------------------------------------------
# the cases
# --------------------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def case_frame_grad(handle, B, T, n_fft, hop):
    g = torch.randn(B, T * hop, generator=_gen(T))
    win = torch.hann_window(n_fft)
    o = run_hook(handle, "FRAME_GRAD", {"out_f32": (B * T, n_fft)}, x=g, w=win, B=B, T=T, n_fft=n_fft, hop=hop)
    return within(o["out_f32"].view(B, T, n_fft), frame_grad_ref(g, win, T, n_fft, hop, torch.float64),
                  frame_grad_ref(g, win, T, n_fft, hop, torch.float32), "frame_grad")


def case_spectrum_grad(handle, rows, n_fft):
    K = n_fft // 2 + 1
    Kp = (K + 127) // 128 * 128
    Nh, K2 = 2 * Kp, 2 * ((K + 63) // 64 * 64)
    gen = _gen(rows)
    m = torch.randn(rows, K, generator=gen) * 2 + 3.5
    m = torch.where((m - G.LN_CLIP).abs() < 1e-4, m + 1e-3, m)          # no clip decision at the rounding level
    p = torch.randn(rows, K, generator=gen) * 3
    x = torch.full((rows, Nh), 123.0)
    x[:, :K], x[:, Kp:Kp + K] = m, p
    dS = torch.randn(rows, K2, generator=gen)
    o = run_hook(handle, "SPECTRUM_GRAD", {"out_f32": (rows, Nh)}, x=dS, x1=x, rows=rows, Nh=Nh, Kp=Kp, K=K, K2=K2)

    def ref(dt):
        dm, dp = G.spectrum_grad(dS[:, :K].to(dt), dS[:, K2 // 2:K2 // 2 + K].to(dt), m.to(dt), p.to(dt))
        r = torch.zeros(rows, Nh, dtype=dt)
        r[:, :K], r[:, Kp:Kp + K] = dm, dp
        return r
    assert float((m > G.LN_CLIP).double().mean()) > 0.1
    return within(o["out_f32"], ref(torch.float64), ref(torch.float32), "spectrum_grad")


def case_ln_bwd(handle, B, T, C, dwconv):
    gen = _gen(C + T)
    x = torch.randn(B, T, C, generator=gen) * 1.5 + 0.3
    w = torch.randn(7, C, generator=gen) * 0.3 if dwconv else None
    b = torch.randn(C, generator=gen) * 0.1 if dwconv else None
    lnw = 1 + 0.1 * torch.randn(C, generator=gen)
    g = torch.randn(B, T, C, generator=gen)
    kw = dict(w=w, bias=b) if dwconv else {}
    o = run_hook(handle, "LN_BWD", {"out_f32": (B, T, C), "out2_f32": (B, T, C)}, x=x, x1=lnw, x2=g, B=B, T=T, C=C,
                 eps=1e-6, **kw)
    d64, z64 = ln_bwd_ref(x, w, b, lnw, g, 1e-6, torch.float64)
    d32, z32 = ln_bwd_ref(x, w, b, lnw, g, 1e-6, torch.float32)
    return max(within(o["out_f32"], d64, d32, "ln_bwd dx"), within(o["out2_f32"], z64, z32, "ln_bwd zhat"))


def case_dwconv_adj(handle, B, T, C):
    gen = _gen(10 * T + C)
    dz = torch.randn(B, T, C, generator=gen)
    w = torch.randn(7, C, generator=gen) * 0.3
    res = torch.randn(B, T, C, generator=gen)
    o = run_hook(handle, "DWCONV_ADJ", {"out_f32": ((B, T, C), res)}, x=dz, w=w, B=B, T=T, C=C)

    def ref(dt):
        return res.to(dt) + G.dwconv_bwd(dz.to(dt), w.to(dt).T[:, None, :], dz.to(dt))[0]
    return within(o["out_f32"], ref(torch.float64), ref(torch.float32), "dwconv_adj")


def case_col_sum(handle, rows, C, product):
    gen = _gen(rows + C)
    a = torch.randn(rows, C, generator=gen)
    b = torch.randn(rows, C, generator=gen) if product else None
    kw = dict(x1=b) if product else {}
    o = run_hook(handle, "COL_SUM", {"out_f32": (C,)}, x=a, rows=rows, C=C, **kw)

    def ref(dt):
        return (a.to(dt) * b.to(dt)).sum(0) if product else a.to(dt).sum(0)
    return within(o["out_f32"], ref(torch.float64), ref(torch.float32), "col_sum")


def case_dwconv_wgrad(handle, B, T, C):
    gen = _gen(100 + T + C)
    dz = torch.randn(B, T, C, generator=gen)
    x = torch.randn(B, T, C, generator=gen)
    o = run_hook(handle, "DWCONV_WGRAD", {"out_f32": (C, 1, 7), "out2_f32": (C,)}, x=dz, x1=x, B=B, T=T, C=C)
    r64, r32 = (G.dwconv_bwd(x.to(dt), torch.zeros(C, 1, 7, dtype=dt), dz.to(dt)) for dt in (torch.float64, torch.float32))
    return max(within(o["out_f32"], r64[1], r32[1], "dwconv dw"), within(o["out2_f32"], r64[2], r32[2], "dwconv db"))


def case_scale_cols(handle, rows, C):
    gen = _gen(rows)
    x, gam = torch.randn(rows, C, generator=gen), torch.randn(C, generator=gen)
    o = run_hook(handle, "SCALE_COLS", {"out_f32": (rows, C)}, x=x, w=gam, rows=rows, C=C)
    assert torch.equal(bits(o["out_f32"]), bits(x * gam))
    return 0.0


def case_gelu_bwd(handle, n):
    gen = _gen(n)
    h = torch.randn(n, generator=gen) * 4
    dg = torch.randn(n, generator=gen)
    o = run_hook(handle, "GELU_BWD", {"out_f32": (n,)}, x=dg, x1=h, rows=n)
    return within(o["out_f32"], gelu_bwd_ref(h, dg, torch.float64), gelu_bwd_ref(h, dg, torch.float32), "gelu_bwd")


def case_transpose(handle, B, T, C, taps, ones, planes):
    gen = _gen(B * T + C + taps)
    x = torch.randn(B, T, C, generator=gen)
    Kr = (B * T + 255) // 256 * 256
    Nd = taps * C + 8
    if planes:
        hi, lo = split_bf16(x)
        o = run_hook(handle, "TRANSPOSE_ROWS", {"out_hi": (Nd, Kr), "out_lo": (Nd, Kr)}, x_hi=hi, x_lo=lo, B=B, T=T, C=C,
                     taps=taps, ones=ones, Nd=Nd, Kr=Kr)
        for plane, src in (("out_hi", hi), ("out_lo", lo)):
            ref = G.wgrad_operand(src.float(), taps, Kr)
            if not ones or plane == "out_lo":          # the ones row is the pair (1, 0)
                ref[taps * C] = 0
            assert torch.equal(bits(o[plane]), bits(ref.to(torch.bfloat16))), plane
    else:
        o = run_hook(handle, "TRANSPOSE_ROWS", {"out_f32": (Nd, Kr), "out_hi": (Nd, Kr), "out_lo": (Nd, Kr)}, x=x, B=B, T=T,
                     C=C, taps=taps, ones=ones, Nd=Nd, Kr=Kr)
        ref = G.wgrad_operand(x, taps, Kr)
        if not ones:
            ref[taps * C] = 0
        assert torch.equal(bits(o["out_f32"]), bits(ref))
        rh, rl = split_bf16(ref)
        assert torch.equal(bits(o["out_hi"]), bits(rh)) and torch.equal(bits(o["out_lo"]), bits(rl))
    return 0.0


def case_unpack(handle, Nref, Cx, taps, split, Kp):
    Np = Kp + Nref - split if split else Nref
    dWp = torch.randn(Np, taps * Cx + 8, generator=_gen(Nref + Cx))
    o = run_hook(handle, "WGRAD_UNPACK", {"out_f32": (Nref, Cx, taps), "out2_f32": (Nref,)}, x=dWp, Nref=Nref, C=Cx,
                 taps=taps, split=split, Kp=Kp)
    gw, gb = G.unpack_wgrad(dWp, Nref, Cx, taps, split, Kp)
    assert torch.equal(bits(o["out_f32"]), bits(gw.contiguous())) and torch.equal(bits(o["out2_f32"]), bits(gb.contiguous()))
    return 0.0


CASES = {}
for B, T, n_fft, hop in ((2, 1, 2048, 512), (2, 3, 2048, 512), (1, 40, 2048, 512), (3, 7, 1024, 256), (1, 5, 1280, 640)):
    CASES[f"frame_grad-B{B}-T{T}-n{n_fft}-h{hop}"] = (case_frame_grad, B, T, n_fft, hop)
for rows, n_fft in ((37, 2048), (80, 1024)):
    CASES[f"spectrum_grad-r{rows}-n{n_fft}"] = (case_spectrum_grad, rows, n_fft)
for C in (512, 768, 1024):
    for T in (1, 2, 3, 7, 40):
        for dw in (False, True):
            CASES[f"ln_bwd-C{C}-T{T}-{'dw' if dw else 'ln'}"] = (case_ln_bwd, 2, T, C, dw)
for T in (1, 2, 3, 7, 40):
    CASES[f"dwconv_adj-T{T}"] = (case_dwconv_adj, 3, T, 768)
    CASES[f"dwconv_wgrad-T{T}"] = (case_dwconv_wgrad, 3, T, 96)
for rows, C, prod in ((1, 768, True), (37, 96, False), (1280, 768, True), (1280, 2048, False)):
    CASES[f"col_sum-r{rows}-C{C}-{'prod' if prod else 'sum'}"] = (case_col_sum, rows, C, prod)
CASES["scale_cols"] = (case_scale_cols, 37, 768)
CASES["gelu_bwd"] = (case_gelu_bwd, 100003)
for B, T, C, taps, ones, planes in ((2, 3, 48, 7, 1, False), (2, 3, 48, 7, 1, True), (3, 40, 512, 1, 1, True),
                                    (1, 1, 80, 7, 1, False), (3, 40, 96, 1, 0, False), (2, 7, 16, 7, 1, True)):
    CASES[f"transpose-B{B}-T{T}-C{C}-taps{taps}-ones{ones}-{'planes' if planes else 'f32'}"] = \
        (case_transpose, B, T, C, taps, ones, planes)
for Nref, Cx, taps, split, Kp in ((24, 16, 7, 0, 0), (40, 512, 1, 0, 0), (2 * 513, 64, 1, 513, 640), (2 * 5, 8, 1, 5, 128)):
    CASES[f"unpack-N{Nref}-C{Cx}-taps{taps}-split{split}"] = (case_unpack, Nref, Cx, taps, split, Kp)


@pytest.fixture(scope="module")
def matrix(handle):
    return LazyMatrix(lambda key: CASES[key][0](handle, *CASES[key][1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CASES))
def test_matrix(matrix, key):
    matrix.check(key)
    print(f"{key}: {matrix[key]:.2f} of the bar")


def test_kind_numbers_match_the_binding():
    """the binding's kind names are the enum of include/stabletts_b200.h"""
    import os
    import re
    from stabletts_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "stabletts_b200.h")).read()
    enum = {k: int(v) for k, v in re.findall(r"\bST_TEST_VOCOS_GRAD_(\w+)\s*=\s*(\d+)", header)}
    assert enum == {k: i for i, k in enumerate(_lib.ST_TEST_VOCOS_GRAD_KINDS)}


def test_no_spills_in_the_backward_kernels():
    """-Xptxas -v on vocos_grad.cu: no spill stores or loads in any kernel"""
    import os
    import re
    import subprocess
    import __graft_entry__ as ge
    src = os.path.join(ge.CSRC, "vocos_grad.cu")
    r = subprocess.run([ge._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) >= 10 and all(s == ("0", "0") for s in spills), r.stderr
