"""The conv-GEMM contract (GemmArgs, stabletts_b200/csrc/common.cuh and gemm_epilogue.cuh) against an fp64 restatement of it.

`gemm_contract_ref` states what every engine must compute: the tap sum with (tap - taps//2)·dil offsets and zero rows
outside [0, T), the two-source concat, A row bb % a_bmod, then bias -> SiLU / GELU -> FiLM -> mask -> gate -> residual,
EPI_SILU_OUT, the partial RoPE + q scale of the QKV projection, and the fused FiLM2·mask + LayerNorm + adaLN modulate.
The CPU tests pin that reference against independent torch code (F.conv1d, the oracle's rope_partial, F.layer_norm,
F.gelu, F.silu).  The GPU tests drive every wgmma kernel instance (tile width x epilogue mode x precision), the split-K
path and the SIMT engine through st_test_gemm_ex at product call-site shapes and at the edges where kernels go wrong,
and check the properties that need no tolerance: the bf16 / fp16 planes are the rounding of the fp32 output, results
do not depend on the SM count or on repetition, an utterance alone equals its batch row, and the contract's refusals."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_errs
from kernel_harness import LazyMatrix, bits, check_planes, run_ok
from kernel_harness import dev, handles  # noqa: F401 (fixtures)

EPI = dict(BIAS=1, SILU=2, FILM=4, MASK=8, GATE=16, RESID=32, ROPE=64, GELU=128, SILU_OUT=256)
BIAS, SILU, FILM, MASK, GATE, RESID, ROPE, GELU, SILU_OUT = (EPI[k] for k in EPI)
QSCALE = float(np.float32(0.125 * 1.4426950408889634))     # softmax scale folded into q (fp32 constant of the kernel)
LN_EPS = 1e-5
H = 256                                                     # the estimator's hidden width


# --------------------------------------------------------------------------------------------------------------------
# problems and their operands
# --------------------------------------------------------------------------------------------------------------------
def problem(**kw):
    """One conv-GEMM problem: the st_test_gemm_desc fields plus the test's own knobs: planes (request the 2-byte output
    planes), film2, mask (a mask without EPI_MASK), wstd (weight scale), xscale (scale of A, bias and residual), engines."""
    d = dict(B=1, BB=1, T=65, a_bmod=None, C0=128, C1=0, N=128, taps=1, dil=1, flags=BIAS, c_clamp=0, resid_clamp=None,
             film_H=None, rope_H=0, film_bstride=0, gate_bstride=0, ada_bstride=0, film2_bstride=0, ln=0, ln_mask_out=0,
             prec=0, out16=0, u16=0, ksplit=0, num_sms=0, film2=False, mask=False, planes=False, wstd=None, xscale=1.0,
             engines=("tc", "simt"))
    d.update(kw)
    if d["a_bmod"] is None:
        d["a_bmod"] = d["BB"]
    if d["resid_clamp"] is None:
        d["resid_clamp"] = d["BB"] - 1
    if d["film_H"] is None:
        d["film_H"] = d["N"]
    d["n_src"] = 2 if d["C1"] else 1
    return d


def make_mask(B, T, g):
    """(B, T) prefix masks of different lengths; from T >= 8 on with a hole and two fractional values per row, so a wrong
    mask row or column shows."""
    m = torch.ones(B, T)
    for b in range(B):
        m[b, max(1, T - (b * T) // (B + 1)):] = 0.0
        if T >= 8:
            m[b, (7 * b + 3) % T] = 0.0
            m[b, (5 * b + 1) % T] = 0.5
            m[b, (11 * b + 2) % T] = 0.747
    return m


def make_tensors(d, seed):
    """fp32 CPU operands of problem d.  Per-row tables (FiLM, gate, shift / scale, film2) are random, so all rows differ."""
    g = torch.Generator().manual_seed(seed)
    B, BB, T, N, K, f = d["B"], d["BB"], d["T"], d["N"], d["C0"] + d["C1"], d["flags"]
    rn = lambda *s: torch.randn(*s, generator=g)                                          # noqa: E731
    xs = d["xscale"]
    t = {"A0": rn(d["a_bmod"], T, d["C0"]) * xs}
    if d["C1"]:
        t["A1"] = rn(d["a_bmod"], T, d["C1"]) * xs
    wstd = d["wstd"] if d["wstd"] is not None else 1.0 / math.sqrt(K * d["taps"])
    t["W"] = rn(N, K, d["taps"]) * wstd
    mrows, crows = min(B, BB), min(BB - 1, d["c_clamp"]) + 1
    if f & BIAS:
        t["bias"] = rn(N) * 0.5 * xs
    if (f & MASK) or d["mask"] or d["film2"] or d["ln_mask_out"]:
        t["mask"] = make_mask(B, T, g)
    if f & FILM:
        t["film"] = 1.0 + 0.5 * rn((mrows - 1) * d["film_bstride"] + d["film_H"] + N)
    if f & GATE:
        t["gate"] = rn((crows - 1) * d["gate_bstride"] + N)
    if f & RESID:
        t["resid"] = rn(min(BB - 1, d["resid_clamp"]) + 1, T, N) * xs
    if d["ln"]:
        t["ln_shift"] = 0.5 * rn((crows - 1) * d["ada_bstride"] + N)
        t["ln_scale"] = 0.5 * rn((crows - 1) * d["ada_bstride"] + N)
    if d["film2"]:
        t["film2"] = 1.0 + 0.5 * rn((mrows - 1) * d["film2_bstride"] + d["film_H"] + N)
    return t


# --------------------------------------------------------------------------------------------------------------------
# the fp64 reference of the contract
# --------------------------------------------------------------------------------------------------------------------
def _rows(table, idx, stride, off, N):
    """table[idx * stride + off + n] for every batch row idx and n < N -> (BB, 1, N)"""
    n = torch.arange(N, device=table.device)
    return table.double()[idx[:, None] * stride + off + n[None, :]][:, None, :]


def rope_angles(T, device):
    """the kernel's (T, 16) RoPE angles: fp32 theta_i = 10000^(-2i/32) times the fp32 frame index, rounded to fp32"""
    theta = 1.0 / (10000.0 ** (torch.arange(0, 32, 2, device=device).float() / 32))
    return (torch.arange(T, device=device).float()[:, None] * theta[None, :]).double()


def gemm_contract_ref(d, t):
    """fp64 statement of GemmArgs (common.cuh:23-86, gemm_epilogue.cuh).  Returns the fp32 output `out`, the values of the
    output planes `planes`, `out2` (EPI_SILU_OUT: silu(out); film2: the FiLM2·mask row) and the LayerNorm output `u`."""
    dev = t["A0"].device
    f, B, BB, T, N, taps, dil = d["flags"], d["B"], d["BB"], d["T"], d["N"], d["taps"], d["dil"]
    A = (torch.cat([t["A0"], t["A1"]], -1) if d["C1"] else t["A0"]).double()
    if d["prec"]:                        # the two-pass mode's ONE fp16 A plane (saturated to the finite fp16 range)
        A = A.clamp(-65504.0, 65504.0).half().double()
    W = t["W"].double()
    bb = torch.arange(BB, device=dev)
    Ab = A[bb % d["a_bmod"]]
    tt = torch.arange(T, device=dev)
    v = torch.zeros(BB, T, N, dtype=torch.float64, device=dev)
    for tap in range(taps):
        src = tt + (tap - taps // 2) * dil
        ok = (src >= 0) & (src < T)
        if bool(ok.any()):
            v[:, ok] += Ab[:, src[ok]] @ W[:, :, tap].T
    mb, cb, rb = bb % B, bb.clamp(max=d["c_clamp"]), bb.clamp(max=d["resid_clamp"])
    mrow = t["mask"].double()[mb][..., None] if "mask" in t else torch.ones(BB, T, 1, dtype=torch.float64, device=dev)
    if f & BIAS:
        v = v + t["bias"].double()
    if f & ROPE:                         # pairs (c, c + 16), c < 16, of every 64-wide head of q and k (columns < 2 rope_H)
        ang = rope_angles(T, dev)
        cos, sin = ang.cos(), ang.sin()
        y = v.clone()
        for h0 in range(0, 2 * d["rope_H"], 64):
            x1, x2 = v[..., h0:h0 + 16], v[..., h0 + 16:h0 + 32]
            y[..., h0:h0 + 16] = x1 * cos - x2 * sin
            y[..., h0 + 16:h0 + 32] = x2 * cos + x1 * sin
        y[..., :d["rope_H"]] *= QSCALE
        return {"out": y, "planes": y}
    if f & SILU:
        v = v * torch.sigmoid(v)
    elif f & GELU:
        v = 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    if f & FILM:
        v = _rows(t["film"], mb, d["film_bstride"], 0, N) * v + _rows(t["film"], mb, d["film_bstride"], d["film_H"], N)
    if f & MASK:
        v = v * mrow
    if f & GATE:
        v = v * _rows(t["gate"], cb, d["gate_bstride"], 0, N)
    if f & RESID:
        v = v + t["resid"].double()[rb]
    res = {"out": v, "planes": v}
    if f & SILU_OUT:
        s = v * torch.sigmoid(v)
        res["planes"], res["out2"] = s, s
    if d["ln"]:
        x = v
        if d["film2"]:
            x = (_rows(t["film2"], mb, d["film2_bstride"], 0, N) * x + _rows(t["film2"], mb, d["film2_bstride"], d["film_H"], N)) * mrow
            res["out2"] = x
        mean = x.mean(-1, keepdim=True)
        var = ((x - mean) ** 2).mean(-1, keepdim=True)
        u = (x - mean) / torch.sqrt(var + LN_EPS) * (1.0 + _rows(t["ln_scale"], cb, d["ada_bstride"], 0, N)) \
            + _rows(t["ln_shift"], cb, d["ada_bstride"], 0, N)
        res["u"] = u * mrow if d["ln_mask_out"] else u
    return res


# --------------------------------------------------------------------------------------------------------------------
# CPU: the reference against independent torch code
# --------------------------------------------------------------------------------------------------------------------
def _identity_problem(N, BB, T, B=None, **kw):
    """A GEMM whose contraction is the identity, so the epilogue sees the A values themselves."""
    d = problem(BB=BB, B=B or BB, T=T, C0=N, N=N, flags=0, **kw)
    t = make_tensors(d, 3)
    t["W"] = torch.eye(N)[:, :, None]
    return d, t


@pytest.mark.parametrize("taps,dil,T", [(1, 1, 7), (3, 1, 9), (3, 3, 9), (7, 3, 5), (11, 5, 4), (13, 1, 20), (3, 5, 1)])
@pytest.mark.parametrize("C1", [0, 16])
def test_ref_conv_matches_conv1d(taps, dil, T, C1):
    d = problem(B=2, BB=2, T=T, C0=32, C1=C1, N=24, taps=taps, dil=dil, flags=BIAS)
    t = make_tensors(d, 1)
    x = (torch.cat([t["A0"], t["A1"]], -1) if C1 else t["A0"]).double().transpose(1, 2)
    want = F.conv1d(x, t["W"].double(), t["bias"].double(), padding=dil * (taps - 1) // 2, dilation=dil).transpose(1, 2)
    assert torch.allclose(gemm_contract_ref(d, t)["out"], want, rtol=1e-12, atol=1e-12)


def test_ref_a_bmod_repeats_rows():
    d = problem(B=2, BB=5, a_bmod=2, T=6, C0=16, N=8, taps=3, flags=BIAS)
    t = make_tensors(d, 2)
    out = gemm_contract_ref(d, t)["out"]
    for bb in range(5):
        assert torch.equal(out[bb], out[bb % 2])


def test_ref_rope_matches_oracle():
    from oracle.estimator_ref import rope_partial
    BB, T = 2, 37
    d, t = _identity_problem(3 * H, BB, T, rope_H=H)
    d["flags"] = ROPE
    out = gemm_contract_ref(d, t)["out"]
    x = t["A0"].double()

    def heads(z):                                        # (BB, T, H) -> (BB, nh, T, 64)
        return z.view(BB, T, H // 64, 64).transpose(1, 2)

    q = rope_partial(heads(x[..., :H]), 32).transpose(1, 2).reshape(BB, T, H) * QSCALE
    k = rope_partial(heads(x[..., H:2 * H]), 32).transpose(1, 2).reshape(BB, T, H)
    want = torch.cat([q, k, x[..., 2 * H:]], -1)
    assert max(rel_errs(out, want)) < 1e-6              # rope_partial takes cos / sin in fp32


@pytest.mark.parametrize("film2,mask_out", [(False, False), (True, False), (True, True)])
def test_ref_layernorm_matches_layer_norm(film2, mask_out):
    BB, T = 3, 11
    d, t = _identity_problem(H, BB, T, B=2, ln=1, film2=film2, ln_mask_out=int(mask_out), mask=True, c_clamp=1,
                             ada_bstride=2 * H, film2_bstride=2 * H)
    r = gemm_contract_ref(d, t)
    x = t["A0"].double()
    mb, cb = torch.arange(BB) % 2, torch.arange(BB).clamp(max=1)
    m = t["mask"].double()[mb][..., None]
    if film2:
        f2 = t["film2"].double()
        g2 = torch.stack([f2[b * 2 * H: b * 2 * H + H] for b in mb])[:, None]
        b2 = torch.stack([f2[b * 2 * H + H: b * 2 * H + 2 * H] for b in mb])[:, None]
        x = (g2 * x + b2) * m
        assert torch.allclose(r["out2"], x, rtol=1e-12, atol=1e-12)
    sh = torch.stack([t["ln_shift"].double()[c * 2 * H: c * 2 * H + H] for c in cb])[:, None]
    sc = torch.stack([t["ln_scale"].double()[c * 2 * H: c * 2 * H + H] for c in cb])[:, None]
    u = F.layer_norm(x, (H,), eps=LN_EPS) * (1 + sc) + sh
    if mask_out:
        u = u * m
    assert torch.allclose(r["u"], u, rtol=1e-10, atol=1e-10)
    assert torch.equal(r["out"], t["A0"].double())


@pytest.mark.parametrize("flag,fn", [(SILU, F.silu), (GELU, F.gelu)])
def test_ref_activations(flag, fn):
    d, t = _identity_problem(64, 2, 9)
    d["flags"] = flag
    t["A0"] = t["A0"] * 4
    assert torch.allclose(gemm_contract_ref(d, t)["out"], fn(t["A0"].double()), rtol=1e-12, atol=1e-12)
    d["flags"] = SILU_OUT
    r = gemm_contract_ref(d, t)
    assert torch.equal(r["out"], t["A0"].double()) and torch.allclose(r["out2"], F.silu(t["A0"].double()), rtol=1e-12, atol=1e-12)


def test_ref_epilogue_indexing_elementwise():
    """FiLM (bb % B), mask (bb % B), gate (min(bb, c_clamp)) and residual (min(bb, resid_clamp)) restated one element at a time."""
    B, BB, T, N = 2, 4, 8, 8
    d = problem(B=B, BB=BB, T=T, C0=16, N=N, taps=3, flags=BIAS | FILM | MASK | GATE | RESID, c_clamp=2, resid_clamp=1,
                film_bstride=3 * N, gate_bstride=2 * N, film_H=N + 3)
    t = make_tensors(d, 5)
    r = gemm_contract_ref(d, t)
    conv = gemm_contract_ref(dict(d, flags=0), t)["out"]
    for bb in range(BB):
        for tt in range(T):
            for n in range(N):
                v = float(conv[bb, tt, n]) + float(t["bias"][n])
                fb = (bb % B) * d["film_bstride"]
                v = float(t["film"][fb + n]) * v + float(t["film"][fb + d["film_H"] + n])
                v *= float(t["mask"][bb % B, tt])
                v *= float(t["gate"][min(bb, 2) * d["gate_bstride"] + n])
                v += float(t["resid"][min(bb, 1), tt, n])
                assert abs(float(r["out"][bb, tt, n]) - v) <= 1e-12 * max(1.0, abs(v))


def test_ref_prec_rounds_a_to_fp16_with_saturation():
    d = problem(T=3, C0=8, N=8, flags=0, prec=1)
    t = make_tensors(d, 6)
    t["W"] = torch.eye(8)[:, :, None]
    t["A0"][0, 0, :3] = torch.tensor([1e5, -1e5, 1.0 + 2 ** -12])
    out = gemm_contract_ref(d, t)["out"]
    assert out[0, 0, :3].tolist() == [65504.0, -65504.0, 1.0]


# --------------------------------------------------------------------------------------------------------------------
# GPU: the hook
# --------------------------------------------------------------------------------------------------------------------
# max-rel and l2-rel bars against fp64.  Worst measured on an H100 80GB HBM3 (700 W limit) over this matrix (pytest -s prints
# the table): split-bf16 x3 2.2e-5, two-pass fp16 (against the fp16-rounded A) 8.7e-6, SIMT 2.8e-6.  The split-bf16 worst is
# conv_pre (13 taps x 512 channels) on both tile widths with l2-rel = max-rel: a systematic error of the wgmma accumulation
# that grows with the K loop (the SIMT engine gets 2.8e-6 on the same problem), so the bar keeps 2x room for longer loops.
TOL = {"tc": 5e-5, "simt": 2e-5}
SILU_FAST = 1e-6            # the wgmma epilogue's SiLU runs on the SFU approximations (silu_fast, ~3e-7 relative)
PLANE_Q = {"bf16": 2.0 ** -16, "fp16": 2.0 ** -11}     # + the rounding step of a 2-byte plane (hi + lo, or one fp16 plane)


def run_hook(lib, h, d, t, dev):
    """Runs problem d through st_test_gemm_ex; returns (rc, error text, outputs, plan).  Outputs start as NaN, so an element
    the kernel never wrote fails every comparison."""
    from stabletts_b200 import _lib
    BB, T, N, f = d["BB"], d["T"], d["N"], d["flags"]
    dt = {k: v.to(dev).contiguous() for k, v in t.items()}
    full = lambda dtype: torch.full((BB, T, N), float("nan"), device=dev, dtype=dtype)   # noqa: E731
    o = {"out": full(torch.float32)}
    if d["planes"]:
        if d["out16"]:
            o["hi"] = full(torch.float16)
        else:
            o["hi"], o["lo"] = full(torch.bfloat16), full(torch.bfloat16)
    if (f & SILU_OUT) or d["film2"]:
        o["out2"] = full(torch.float32)
    if d["ln"]:
        if d["u16"]:
            o["u_hi"] = full(torch.float16)
        else:
            o["u_hi"], o["u_lo"] = full(torch.bfloat16), full(torch.bfloat16)
    desc = _lib.StTestGemmDesc()
    for k in ("A0", "A1", "W", "bias", "mask", "film", "gate", "resid", "ln_shift", "ln_scale", "film2"):
        setattr(desc, k, dt[k].data_ptr() if k in dt else None)
    for k, ok in (("out_f32", "out"), ("out_hi", "hi"), ("out_lo", "lo"), ("out2_f32", "out2"), ("u_hi", "u_hi"), ("u_lo", "u_lo")):
        setattr(desc, k, o[ok].data_ptr() if ok in o else None)
    for k in ("film_bstride", "gate_bstride", "ada_bstride", "film2_bstride", "B", "BB", "T", "a_bmod", "n_src", "C0", "C1", "N",
              "taps", "dil", "flags", "c_clamp", "resid_clamp", "film_H", "rope_H", "ln", "ln_mask_out", "prec", "out16", "u16",
              "ksplit", "num_sms"):
        setattr(desc, k, int(d[k]))
    plan = _lib.StTestGemmPlan()
    rc = lib.st_test_gemm_ex(h, C.byref(desc), C.byref(plan), torch.cuda.current_stream().cuda_stream)
    err = lib.st_last_error(h).decode() if rc else ""
    return rc, err, {k: v.cpu() for k, v in o.items()}, plan


def instance_key(plan):
    from stabletts_b200 import _lib
    if plan.engine == 1:
        return "simt"
    if plan.ksplit > 1:
        return "splitk"
    return f"bn{plan.bn}/{_lib.ST_TEST_MODE_NAMES[plan.mode]}/{'fp16x2' if plan.prec else 'bf16x3'}"


def plane_value(o, key_hi, key_lo, f16):
    return o[key_hi].double() if f16 else o[key_hi].double() + o[key_lo].double()


def check_case(d, engine, rc, err, o, plan, ref, dev_sms):
    """value checks against the fp64 reference; returns [(what, max-rel, l2-rel, bar)]"""
    assert rc == 0, err
    tc = engine == "tc"
    fast = tc and bool(d["flags"] & (SILU | SILU_OUT))
    tol = TOL[engine] + (SILU_FAST if fast else 0.0)
    rows = []

    def cmp(what, got, want, bar):
        e = rel_errs(got, want)
        rows.append((what, e[0], e[1], bar))
        assert e[0] < bar and e[1] < bar, (what, e, bar)

    cmp("out", o["out"], ref["out"], tol)
    if "out2" in o:
        cmp("out2", o["out2"], ref["out2"], tol)
    if d["planes"]:
        q = PLANE_Q["fp16" if d["out16"] else "bf16"]
        check_planes(o, "u16" if d["out16"] else "split", o["out2"] if d["flags"] & SILU_OUT else o["out"])
        cmp("planes", plane_value(o, "hi", "lo", d["out16"]), ref["planes"], tol + q)
    if d["ln"]:
        cmp("u", plane_value(o, "u_hi", "u_lo", d["u16"]), ref["u"], tol + PLANE_Q["fp16" if d["u16"] else "bf16"])
    if tc:                               # the persistent grid: min(tiles, SMs), tiles of 128 frames x bn channels
        tiles = d["BB"] * -(-d["T"] // 128) * -(-d["N"] // plan.bn) * max(1, plan.ksplit)
        assert plan.grid == min(tiles, d["num_sms"] or dev_sms), (plan.grid, tiles)
        if d["ksplit"] > 1:
            assert plan.ksplit == d["ksplit"]
    return rows


# ---- the matrix -----------------------------------------------------------------------------------------------------
def _cases():
    cs = {}

    def add(name, **kw):
        assert name not in cs, name
        cs[name] = problem(**kw)

    E = dict(B=2, BB=4, T=129)
    V = dict(ksplit=1)                                             # vocoder GEMMs set batch_invariant: never split-K                                    # estimator with CFG: 2B rows, cond rows 0..B-1
    TC = ("tc",)
    # product call sites (dit_api.cu / vocos_api.cu / ffgan_api.cu) at small T with their real flags, clamps and strides
    for K in (80, 128):
        add(f"cond_k{K}", B=2, BB=3, T=65, C0=K, N=256, flags=BIAS | SILU)
    add("cond_wide", B=2, BB=3, T=65, C0=128, N=256, flags=BIAS | SILU, num_sms=1, engines=TC)
    add("in_proj", B=2, BB=4, a_bmod=2, T=65, C0=80, N=256, flags=RESID, resid_clamp=2, mask=True, planes=True)
    for fbs in (0, 2 * H):
        add(f"in_proj_ln_film2_bs{fbs}", B=2, BB=4, a_bmod=2, T=65, C0=80, N=256, flags=RESID, resid_clamp=2, ln=1, film2=True,
            film2_bstride=fbs, c_clamp=2, ada_bstride=6 * H, out16=int(fbs == 0), planes=True, num_sms=4, engines=TC)
    add("qkv", **E, C0=H, N=3 * H, flags=BIAS | ROPE, rope_H=H, planes=True, engines=TC)
    add("qkv_wide", **E, C0=H, N=3 * H, flags=BIAS | ROPE, rope_H=H, planes=True, num_sms=5, engines=TC)
    add("qkv_simt", **E, C0=H, N=3 * H, flags=BIAS, engines=("simt",))
    O = dict(**E, C0=H, N=H, flags=BIAS | MASK | GATE | RESID, c_clamp=2, gate_bstride=6 * H)
    add("o_proj", **O, planes=True)
    add("o_proj_wide", **O, num_sms=8, planes=True, engines=TC)
    add("o_proj_ln", **O, ln=1, ln_mask_out=1, u16=1, ada_bstride=6 * H, num_sms=8, engines=TC)
    # rows of small variance (~4e-3), where the LayerNorm's eps moves u by ~1e-3
    add("o_proj_ln_small_rows", **O, ln=1, ada_bstride=6 * H, xscale=0.05, num_sms=8, engines=TC)
    C1_ = dict(**E, C0=H, N=1024, taps=3, flags=BIAS | SILU | MASK)
    add("conv_1", **C1_, planes=True)
    add("conv_1_fp16x2", **C1_, prec=1, out16=1, planes=True, num_sms=8, engines=TC)
    C2_ = dict(**E, C0=1024, N=H, taps=3, flags=BIAS | MASK | GATE | RESID, c_clamp=2, gate_bstride=6 * H)
    add("conv_2", **C2_, planes=True)
    add("conv_2_fp16x2", **C2_, prec=1, out16=1, planes=True, num_sms=8, engines=TC)
    add("conv_2_fp16x2_ln_film2", **C2_, prec=1, out16=1, planes=True, ln=1, film2=True, film2_bstride=2 * H, ada_bstride=6 * H,
        num_sms=8, engines=TC)
    # fp16 weight lo plane: subnormal at weights ~1e-2 (the default 1/sqrt(K taps) = 0.018 above), normal at O(1) weights
    add("conv_2_fp16x2_w1", **C2_, prec=1, out16=1, planes=True, wstd=1.0, num_sms=8, engines=TC)
    L = dict(**E, C0=H, C1=H, N=H, taps=3, flags=BIAS | FILM | MASK, film_bstride=2 * H)
    add("long_skip", **L)
    add("long_skip_wide", **L, num_sms=8, engines=TC)
    add("long_skip_fp16x2", **L, prec=1, num_sms=8, engines=TC)
    add("long_skip_fp16x2_ln", **L, prec=1, ln=1, c_clamp=2, ada_bstride=6 * H, num_sms=8, engines=TC)
    add("long_skip_fp16x2_ln_bs0", **dict(L, film_bstride=0), prec=1, ln=1, c_clamp=2, ada_bstride=6 * H, num_sms=8, engines=TC)
    for n in (80, 128):
        add(f"final_proj_n{n}", **E, C0=H, N=n, flags=BIAS | MASK)
    add("pwconv1", **V, B=2, BB=2, T=70, C0=128, N=512, flags=BIAS | GELU, planes=True)
    add("pwconv1_wide", **V, B=2, BB=2, T=70, C0=128, N=512, flags=BIAS | GELU, planes=True, num_sms=2, engines=TC)
    add("pwconv2", **V, B=2, BB=2, T=70, C0=512, N=128, flags=BIAS | GATE | RESID, gate_bstride=0, c_clamp=0)
    for cin, c, u in ((64, 32, 2), (128, 64, 2), (256, 128, 8)):
        add(f"ups_{cin}_u{u}", **V, B=2, BB=2, T=37, C0=cin, N=u * c, taps=3, flags=BIAS | SILU_OUT, planes=True)
    add("ups_wide", **V, B=2, BB=2, T=37, C0=256, N=1024, taps=3, flags=BIAS | SILU_OUT, planes=True, num_sms=2, engines=TC)
    add("conv_pre", **V, B=1, BB=1, T=70, C0=512, N=512, taps=13, flags=BIAS | SILU)
    add("conv_pre_wide", **V, B=1, BB=1, T=70, C0=512, N=512, taps=13, flags=BIAS | SILU, num_sms=1, engines=TC)
    for c in (16, 32, 64):
        R = dict(B=2, BB=2, T=70, C0=c, N=c, ksplit=1)
        for k, dl in ((3, 1), (7, 3), (11, 5)):
            add(f"res_convs1_c{c}_k{k}_d{dl}", **R, taps=k, dil=dl, flags=BIAS | SILU, planes=True)
        add(f"res_convs2_c{c}", **R, taps=7, flags=BIAS | RESID | SILU_OUT, planes=True)
        add(f"res_convs2_last_c{c}", **R, taps=11, flags=BIAS | RESID)
        add(f"narrow_gelu_c{c}", **R, taps=3, flags=BIAS | GELU)
        add(f"narrow_plain_c{c}", **R, taps=3, dil=3, flags=BIAS | MASK)
    # edges: T around the 64-frame consumer half and the 128-frame tile; one CTA walking every tile (num_sms = 1)
    for T in (1, 2, 63, 64, 65, 127, 128, 129, 300):
        P = dict(B=2, BB=2, T=T, C0=H, N=H, taps=3, flags=BIAS | MASK | GATE | RESID, c_clamp=1, gate_bstride=H)
        add(f"T{T}", **P)
        add(f"T{T}_one_sm", **P, num_sms=1, planes=True, engines=TC)
        add(f"T{T}_narrow", B=2, BB=2, T=T, C0=32, N=32, taps=7, dil=5, flags=BIAS | SILU)
    # taps reaching past the whole sequence (T < dil * (taps // 2))
    for T in (1, 4, 9):
        add(f"reach_T{T}", B=1, BB=1, T=T, C0=64, N=128, taps=11, dil=5, flags=BIAS)
    add("C8", B=1, BB=3, T=65, C0=8, N=128, taps=3, flags=BIAS, engines=TC)
    add("concat_80", B=2, BB=2, T=65, C0=H, C1=80, N=H, taps=3, flags=BIAS | MASK)
    for n in (16, 32, 64, 80, 128, 256, 512, 768, 1024):
        add(f"N{n}", B=3, BB=3, T=65, C0=128, N=n, flags=BIAS | MASK)
    for sms in (1, 5):
        add(f"n128_sms{sms}", B=2, BB=4, T=300, C0=128, N=128, flags=BIAS | FILM, film_bstride=2 * 128, num_sms=sms, engines=TC)
        add(f"n256_sms{sms}", B=2, BB=4, T=300, C0=128, N=256, flags=BIAS, num_sms=sms, engines=TC)
    # forced split-K with every epilogue it accepts (K loop of 3 taps x 4 channel blocks: divisible by 2, 3 and 4)
    for ks in (2, 3, 4):
        for nm, fl in (("bias", BIAS), ("silu", BIAS | SILU), ("gelu", BIAS | GELU), ("film_mask", BIAS | FILM | MASK),
                       ("gate_resid", BIAS | MASK | GATE | RESID), ("resid_silu_out", BIAS | RESID | SILU_OUT)):
            add(f"splitk{ks}_{nm}", B=2, BB=2, T=65, C0=H, N=128, taps=3, flags=fl, c_clamp=1, gate_bstride=128, film_bstride=256,
                ksplit=ks, planes=True, engines=TC)
    return cs


CASES = _cases()
RUNS = [(name, e) for name, d in CASES.items() for e in d["engines"]]


@pytest.fixture(scope="module")
def matrix(dev, handles):
    """{(name, engine): (rows, instance key)}"""
    lib, hs = handles
    sms = torch.cuda.get_device_properties(dev).multi_processor_count

    def run(key):
        name, engine = key
        d = CASES[name]
        t = make_tensors(d, 1000 + RUNS.index(key))
        rc, err, o, plan = run_hook(lib, hs[engine], d, t, dev)
        ref = {k: v.cpu() for k, v in gemm_contract_ref(d, {k: v.to(dev) for k, v in t.items()}).items()}
        return check_case(d, engine, rc, err, o, plan, ref, sms), instance_key(plan)
    return LazyMatrix(run)


@pytest.mark.gpu
@pytest.mark.parametrize("name,engine", RUNS, ids=[f"{n}-{e}" for n, e in RUNS])
def test_matrix(name, engine, matrix):
    matrix.check((name, engine))


# every kernel instance launch_bn (gemm_tc.cu) can dispatch, plus the split-K pair and the SIMT engine.  A new instance
# must be added here, and then reached by a case above.
EXPECTED_INSTANCES = (
    [f"bn256/{m}/fp16x2" for m in ("SILU", "LN", "RESID", "PLAIN")]
    + [f"bn256/{m}/bf16x3" for m in ("LN", "ROPE", "SILU", "GELU", "RESID", "SILU_OUT", "PLAIN")]
    + [f"bn128/{m}/bf16x3" for m in ("ROPE", "SILU", "GELU", "RESID", "SILU_OUT", "PLAIN")]
    + [f"bn{b}/{m}/bf16x3" for b in (64, 32, 16) for m in ("SILU", "GELU", "RESID", "SILU_OUT", "PLAIN")]
    + ["splitk", "simt"])


@pytest.mark.gpu
def test_every_instance_reached(matrix):
    """and prints the worst measured error per instance (pytest -s): of the fp32 outputs (out_f32, out2_f32) and of the
    2-byte planes (output and LayerNorm planes, whose bar adds the plane's rounding step)"""
    worst = {}
    for name, engine in RUNS:
        res = matrix[(name, engine)]
        if isinstance(res, Exception):
            continue
        rows, key = res
        w = worst.setdefault(key, {"n": 0, "f32": [0.0, 0.0, 0.0, ""], "planes": [0.0, 0.0, 0.0, ""]})
        w["n"] += 1
        for what, em, el, bar in rows:
            g = w["f32" if what in ("out", "out2") else "planes"]
            if em > g[0]:
                g[3] = f"{name}:{what}"
            g[0], g[1], g[2] = max(g[0], em), max(g[1], el), max(g[2], bar)
    print(f"\n{'instance':22s} {'cases':>5s} | {'fp32 max-rel':>12s} {'l2-rel':>9s} {'bar':>8s} | {'planes max-rel':>14s} {'bar':>8s} | worst fp32 case")
    for k in EXPECTED_INSTANCES + sorted(set(worst) - set(EXPECTED_INSTANCES)):
        if k in worst:
            w = worst[k]
            f, p = w["f32"], w["planes"]
            pl = f"{p[0]:14.2e} {p[2]:8.2e}" if p[2] else f"{'-':>14s} {'-':>8s}"
            print(f"{k:22s} {w['n']:5d} | {f[0]:12.2e} {f[1]:9.2e} {f[2]:8.2e} | {pl} | {f[3]}")
    print("two-pass fp16 weights: the lo plane is subnormal at |w| ~ 1e-2 and normal at O(1) weights")
    for name in ("conv_2_fp16x2", "conv_2_fp16x2_w1"):
        res = matrix[(name, "tc")]
        if not isinstance(res, Exception):
            rows = res[0]
            print(f"  {name:18s} wstd {CASES[name]['wstd'] or 1 / math.sqrt(3 * 1024):.3g}: out_f32 max-rel {rows[0][1]:.2e} l2-rel {rows[0][2]:.2e}")
    assert len(EXPECTED_INSTANCES) == 34
    missing = [k for k in EXPECTED_INSTANCES if k not in worst]
    assert not missing, missing
    assert set(worst) <= set(EXPECTED_INSTANCES), set(worst) - set(EXPECTED_INSTANCES)


# ---- properties that need no tolerance -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,sms", [(128, (0, 1, 5, 7)), (256, (1, 5, 7))])
def test_bits_independent_of_sm_count_and_repetition(N, sms, dev, handles):
    """out_f32 and the planes are bit-identical across SM-count overrides that keep the tile width, and across repeats"""
    lib, hs = handles
    d = problem(B=2, BB=4, T=300, C0=256, N=N, taps=3, flags=BIAS | MASK | GATE | RESID, c_clamp=2, gate_bstride=N, ksplit=1,
                planes=True)
    t = make_tensors(d, 77)
    first = None
    for s in sms:
        for _ in range(2):
            o, plan = run_ok(run_hook, lib, hs["tc"], dict(d, num_sms=s), t, dev)
            if first is None:
                first, bn = o, plan.bn
            assert plan.bn == bn and plan.ksplit == 1
            for k in o:
                assert torch.equal(bits(o[k]), bits(first[k])), (s, k)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_utterance_alone_equals_its_batch_row(engine, dev, handles):
    lib, hs = handles
    B = 3
    d = problem(B=B, BB=B, T=129, C0=256, N=256, taps=3, flags=BIAS | MASK | GATE | RESID | FILM, c_clamp=B - 1, gate_bstride=256,
                film_bstride=512, ksplit=1)
    t = make_tensors(d, 78)
    whole, _ = run_ok(run_hook, lib, hs[engine], d, t, dev)
    for b in range(B):
        one = dict(d, B=1, BB=1, a_bmod=1, c_clamp=0, resid_clamp=0)
        tb = dict(t, A0=t["A0"][b:b + 1], mask=t["mask"][b:b + 1], resid=t["resid"][b:b + 1],
                  gate=t["gate"][b * 256:(b + 1) * 256], film=t["film"][b * 512:b * 512 + 512])
        alone, _ = run_ok(run_hook, lib, hs[engine], one, tb, dev)
        assert torch.equal(bits(alone["out"][0]), bits(whole["out"][b])), b


@pytest.mark.gpu
def test_out16_saturates(dev, handles):
    """|v| = 1e5 overflows fp16: the out16 plane holds +-65504, never inf"""
    lib, hs = handles
    for sms in (0, 1):                   # 128- and 256-channel tiles
        d = problem(B=1, BB=1, T=65, C0=128, N=256, flags=RESID, out16=1, planes=True, num_sms=sms)
        t = make_tensors(d, 79)
        t["resid"][0, :, :8] = 1e5
        t["resid"][0, :, 8:16] = -1e5
        o, _ = run_ok(run_hook, lib, hs["tc"], d, t, dev)
        assert torch.isfinite(o["hi"].float()).all()
        assert (o["hi"][0, :, :8].float() == 65504).all() and (o["hi"][0, :, 8:16].float() == -65504).all()
        check_planes(o, "u16")


def _refused(lib, h, d, dev, *needles):
    rc, err, o, _ = run_hook(lib, h, d, make_tensors(d, 80), dev)
    assert rc != 0, d
    assert any(n in err for n in needles), err
    assert torch.isnan(o["out"]).all()                   # nothing was launched


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_refuses_activation_with_residual_or_silu_out(engine, dev, handles):
    lib, hs = handles
    for fl in (BIAS | SILU | RESID, BIAS | GELU | RESID, BIAS | SILU | SILU_OUT, BIAS | GELU | SILU_OUT):
        _refused(lib, hs[engine], problem(B=2, BB=2, N=128, flags=fl), dev, "does not combine")


@pytest.mark.gpu
def test_refuses_out16_with_split_k(dev, handles):
    lib, hs = handles
    d = problem(B=2, BB=2, T=65, C0=256, N=128, taps=3, flags=BIAS, out16=1, planes=True, ksplit=2)
    _refused(lib, hs["tc"], d, dev, "split-K is not available")
    # and the automatic choice never splits an out16 GEMM (a latency-bound shape that it splits without out16)
    lib_, h = lib, hs["tc"]
    o, plan = run_ok(run_hook, lib_, h, dict(d, ksplit=0, out16=0), make_tensors(d, 81), dev)
    assert plan.ksplit > 1
    o, plan = run_ok(run_hook, lib_, h, dict(d, ksplit=0), make_tensors(d, 81), dev)
    assert plan.ksplit == 1
    check_planes(o, "u16")


@pytest.mark.gpu
def test_refuses_layernorm_unless_n_256(dev, handles):
    lib, hs = handles
    d = problem(B=1, BB=1, T=65, C0=128, N=512, flags=BIAS, ln=1, num_sms=1)        # wide tiles, but two per row
    _refused(lib, hs["tc"], d, dev, "N == 256")
    _refused(lib, hs["tc"], problem(B=1, BB=1, N=256, flags=BIAS | SILU, ln=1, num_sms=1), dev, "fused LayerNorm does not combine")


@pytest.mark.gpu
def test_simt_refuses_what_it_does_not_implement(dev, handles):
    lib, hs = handles
    h = hs["simt"]
    base = dict(B=2, BB=2, T=65, C0=H, N=H, flags=BIAS)
    _refused(lib, h, problem(**base, ln=1), dev, "SIMT")
    _refused(lib, h, problem(**base, prec=1), dev, "SIMT")
    _refused(lib, h, problem(**base, out16=1, planes=True), dev, "SIMT")
    _refused(lib, h, problem(**dict(base, N=3 * H, flags=BIAS | ROPE), rope_H=H), dev, "SIMT")
    _refused(lib, h, problem(**dict(base, C0=8)), dev, "multiple of 16")


@pytest.mark.gpu
def test_refuses_split_factor_that_does_not_divide_k(dev, handles):
    lib, hs = handles
    _refused(lib, hs["tc"], problem(B=2, BB=2, T=65, C0=256, N=128, flags=BIAS, ksplit=3), dev, "does not divide the K loop")
