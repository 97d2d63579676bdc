"""The multi-period discriminator's fp32 row kernels (stabletts_b200/csrc/mpd.cu) against fp64 statements of their contracts
(st_test_mpd_row_ex, include/stabletts_b200.h).

Kernels: conv0_fwd_kernel, act_fwd_kernel, nchw_to_rows_kernel, post_fwd_kernel, pack_kernel, post_dgrad_kernel,
post_wgrad_kernel, act_bwd_kernel, im2col_t_kernel, unpack_wgrad_kernel, conv0_wgrad_kernel and conv0_dgrad_kernel: every
index map and reduction of the discriminator outside the conv-GEMM.  The hook calls the product's own launch_mpd_* functions.

Each kind has a statement written as an explicit index formula; the CPU tests pin it against independent torch code
(F.pad(..., "reflect") + F.conv2d, autograd through them and through F.leaky_relu, F.unfold-style views, the packings of
oracle/mpd_ref.py).

Bars, against the statement on the same fp32 inputs:
  layout and elementwise kinds (ACT_FWD, NCHW_TO_ROWS, ACT_BWD, IM2COL_T, UNPACK_WGRAD, PACK): bit for bit the same
                  operations in torch fp32; padding is +0 by bits;
  arithmetic kinds (CONV0_FWD, POST_FWD, POST_DGRAD, POST_WGRAD, CONV0_WGRAD, CONV0_DGRAD): kernel_harness.bar, i.e.
                  max |out - ref64| <= max(4 E32, 8 * 2^-24 * max |ref64|), E32 = max |torch fp32 - ref64| of the same op or
                  autograd on the CPU;
  split planes:   hi = bf16(v) and lo = bf16(v - hi) of the fp32 value the kernel wrote, bit for bit.
Every output starts as NaN; where a kernel must not write, a sentinel is filled in and must survive.
`pytest -s` prints the worst ratio to the bar per kind and case group."""
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import mpd_ref as R
from kernel_harness import LazyMatrix, NAN, bar, bits, check_planes, report_worst_per_group, run_ok, set_fields
from kernel_harness import dev, handle  # noqa: F401 (fixtures)

SLOPE32 = float(torch.tensor(0.1, dtype=torch.float32))    # f32(0.1): the kernels' leaky slope
CIN, COUT, STRIDE = (1, 32, 128, 512, 1024), (32, 128, 512, 1024, 1024), (3, 3, 3, 3, 1)
SENTINEL = 7.0
EXACT = ("ACT_FWD", "NCHW_TO_ROWS", "ACT_BWD", "IM2COL_T", "UNPACK_WGRAD", "PACK")


def ceil_div(a, b):
    return -(-a // b)


def layer_H(p, L):
    """[Hin, H0 .. H4] of st_mpd_forward for (p, L)"""
    hs = [ceil_div(L, p)]
    for s in STRIDE:
        hs.append(ceil_div(hs[-1], 3) if s == 3 else hs[-1])
    return hs


def kr_of(BBH):
    return ceil_div(BBH, 256) * 256


# --------------------------------------------------------------------------------------------------------------------
# fp64 statements (explicit index formulas; the exact kinds are evaluated in the dtype of their inputs)
# --------------------------------------------------------------------------------------------------------------------
def reflect_view(x, p):
    """(B, L) -> (B, Hin, p): padded sample t >= L is x[2L - 2 - t]"""
    B, L = x.shape
    t = torch.arange(ceil_div(L, p) * p)
    return x[:, torch.where(t >= L, 2 * L - 2 - t, t)].view(B, -1, p)


def conv0_taps(xv, H0):
    """(B, Hin, p) -> (B, H0, 5, p): xv[3h + k - 2], zero outside [0, Hin)"""
    idx = 3 * torch.arange(H0)[:, None] + torch.arange(5)[None, :] - 2
    ok = (idx >= 0) & (idx < xv.shape[1])
    return torch.where(ok[None, :, :, None], xv[:, idx.clamp(0, xv.shape[1] - 1), :], 0.0)


def shift_h(f, s):
    """f[..., h + s, :] along dim -2, zero outside"""
    out = torch.zeros_like(f)
    H = f.shape[-2]
    lo, hi = max(0, -s), min(H, H - s)
    if hi > lo:
        out[..., lo:hi, :] = f[..., lo + s:hi + s, :]
    return out


def nchw_to_rows(f, R_):
    """(B, C, H, p) -> (B p, R, C), rows [H, R) +0"""
    B, C_, H, p = f.shape
    out = torch.zeros(B * p, R_, C_, dtype=f.dtype)
    out[:, :H] = f.permute(0, 3, 2, 1).reshape(B * p, H, C_)
    return out


def rows_to_nchw(r, B, p):
    """(B p, H, C) -> (B, C, H, p)"""
    return r.reshape(B, p, r.shape[1], r.shape[2]).permute(0, 3, 2, 1)


def leaky(v, slope):
    return torch.where(v > 0, v, v * slope)


def conv0_fwd_ref(d, t):
    x, w, b = t["x"].double(), t["w"].double().view(32, 5), t["b"].double()
    Z = torch.einsum("bhkj,ck->bchj", conv0_taps(reflect_view(x, d["p"]), d["H"]), w) + b[None, :, None, None]
    return {"out": leaky(Z, SLOPE32)}


def act_fwd_ref(d, t):
    f = leaky(rows_to_nchw(t["Y"], d["B"], d["p"]), float(torch.tensor(d["slope"], dtype=torch.float32)))
    return {"out": f.contiguous(), "rows": nchw_to_rows(f, d["R"])}


def nchw_to_rows_ref(d, t):
    return {"rows": nchw_to_rows(t["fmap"], d["R"])}


def post_fwd_ref(d, t):
    f, w = t["fmap"].double(), t["w"].double().view(1024, 3)
    post = sum(torch.einsum("bchj,c->bhj", shift_h(f, k - 1), w[:, k]) for k in range(3)) + t["b"].double()[0]
    return {"out": post[:, None]}


def pack_ref(d, t):
    W = t["w"]
    mode = R_PACK[d["mode"]]
    return {"out": mode(W).contiguous()}


R_PACK = {"FWD_S3": R.pack_fwd_s3, "FWD_S1": lambda W: W.permute(2, 0, 1), "DGRAD_S3": R.pack_dgrad_s3, "DGRAD_S1": R.pack_dgrad_s1}


def post_dgrad_ref(d, t):
    gp, w = t["gpost"].double()[:, 0], t["w"].double().view(1024, 3)    # (B, H, p)
    G = sum(shift_h(gp, 1 - k)[:, None] * w[None, :, k, None, None] for k in range(3))   # (B, 1024, H, p)
    return {"out": nchw_to_rows(G, d["H"])}


def post_wgrad_ref(d, t):
    gp, f = t["gpost"].double()[:, 0], t["fmap"].double()
    dw = torch.stack([torch.einsum("bhj,bchj->c", gp, shift_h(f, k - 1)) for k in range(3)], 1)
    return {"out": dw.reshape(-1), "out_b": gp.sum().reshape(1)}


def act_bwd_ref(d, t):
    """v = (G[bb, h + off] + gfmap) (fmap > 0 ? 1 : f32(0.1)), in the inputs' dtype"""
    B, p, H, off = d["B"], d["p"], d["H"], d["off"]
    v = rows_to_nchw(t["G"][:, off:off + H], B, p)
    if "gfmap" in t:
        v = v + t["gfmap"]
    if "fmap" in t:
        v = torch.where(t["fmap"] > 0, v, v * SLOPE32)
    v = v.contiguous()
    out = {"out": v, "rows": nchw_to_rows(v, H + 1)}
    BBH = B * p * H
    tr = torch.zeros(d["C"], BBH, dtype=v.dtype)
    tr[:, :] = v.permute(1, 0, 3, 2).reshape(d["C"], BBH)      # column bb H + h, bb = b p + j
    out["tr"] = tr
    return out


def im2col_t_ref(d, t):
    X, s, H, Kr = t["fmap"], d["stride"], d["H"], d["Kr"]
    B, Cin, Hx, p = X.shape
    idx = s * torch.arange(H)[:, None] + torch.arange(5)[None, :] - 2
    ok = (idx >= 0) & (idx < Hx)
    g = torch.where(ok[None, None, :, :, None], X[:, :, idx.clamp(0, Hx - 1), :], 0.0)      # (B, Cin, H, 5, p), +0 outside
    out = torch.zeros(5 * Cin + 8, Kr, dtype=X.dtype)
    out[:5 * Cin, :B * p * H] = g.permute(3, 1, 0, 4, 2).reshape(5 * Cin, B * p * H)
    out[5 * Cin, :B * p * H] = 1.0
    return {"tr": out}


def unpack_wgrad_ref(d, t):
    dWp, Cout, Cin = t["dWp"], d["Cout"], d["Cin"]
    n, c, k = torch.meshgrid(torch.arange(Cout), torch.arange(Cin), torch.arange(5), indexing="ij")
    return {"out": dWp[n, k * Cin + c], "out_b": dWp[:, 5 * Cin]}


def conv0_wgrad_ref(d, t):
    dz0, x = t["dz0"].double(), t["x"].double()
    taps = conv0_taps(reflect_view(x, d["p"]), d["H"])                   # (B, H0, 5, p)
    return {"out": torch.einsum("bchj,bhkj->ck", dz0, taps), "out_b": dz0.sum((0, 2, 3))}


def conv0_dgrad_ref(d, t):
    """gradient of the padded view: row hin collects w[c, k] dz0[c, h] over 3h + k - 2 = hin; then sample t collects its
    own row and, for t = 2L - 2 - s with s in [L, Hin p), the padded sample s that mirrors it"""
    dz0, w, L, p, H0 = t["dz0"].double(), t["w"].double().view(32, 5), d["L"], d["p"], d["H"]
    B = dz0.shape[0]
    Hin = ceil_div(L, p)
    gv = torch.zeros(B, Hin, p, dtype=torch.float64)
    for k in range(5):
        h = torch.arange(H0)
        hin = 3 * h + k - 2
        ok = (hin >= 0) & (hin < Hin)
        gv.index_add_(1, hin[ok], torch.einsum("bchj,c->bhj", dz0, w[:, k])[:, ok])
    flat = gv.reshape(B, Hin * p)
    gx = flat[:, :L].clone()
    for s in range(L, Hin * p):
        gx[:, 2 * L - 2 - s] += flat[:, s]
    return {"out": gx}


STATEMENTS = dict(CONV0_FWD=conv0_fwd_ref, ACT_FWD=act_fwd_ref, NCHW_TO_ROWS=nchw_to_rows_ref, POST_FWD=post_fwd_ref,
                  PACK=pack_ref, POST_DGRAD=post_dgrad_ref, POST_WGRAD=post_wgrad_ref, ACT_BWD=act_bwd_ref,
                  IM2COL_T=im2col_t_ref, UNPACK_WGRAD=unpack_wgrad_ref, CONV0_WGRAD=conv0_wgrad_ref,
                  CONV0_DGRAD=conv0_dgrad_ref)


# --------------------------------------------------------------------------------------------------------------------
# independent torch code (in fp64 it pins the statement; in fp32 it gives E32, or the bits of the exact kinds)
# --------------------------------------------------------------------------------------------------------------------
def _conv0(x, w, b, p):
    return F.conv2d(R.pad_view(x[:, None], p), w.view(32, 1, 5, 1), b, stride=(3, 1), padding=(2, 0))


def conv0_fwd_torch(d, t, dt):
    return {"out": F.leaky_relu(_conv0(t["x"].to(dt), t["w"].to(dt), t["b"].to(dt), d["p"]), SLOPE32)}


def act_fwd_torch(d, t, dt):
    Y = t["Y"].to(dt)
    f = Y.view(d["B"], d["p"], d["H"], d["C"]).permute(0, 3, 2, 1)
    f = F.leaky_relu(f, float(torch.tensor(d["slope"], dtype=torch.float32))) if d["slope"] != 1.0 else f
    rows = F.pad(f.permute(0, 3, 2, 1).reshape(-1, d["H"], d["C"]), (0, 0, 0, d["R"] - d["H"]))
    return {"out": f.contiguous(), "rows": rows}


def nchw_to_rows_torch(d, t, dt):
    f = t["fmap"].to(dt)
    return {"rows": F.pad(f.permute(0, 3, 2, 1).flatten(0, 1), (0, 0, 0, d["R"] - d["H"]))}


def post_fwd_torch(d, t, dt):
    return {"out": F.conv2d(t["fmap"].to(dt), t["w"].to(dt).view(1, 1024, 3, 1), t["b"].to(dt), padding=(1, 0))}


def pack_torch(d, t, dt):
    """the engine contract: the packed weight applied by mpd_ref.engine_conv is the conv it packs (checked on the CPU in
    test_packings_are_the_conv); here the value placement of FWD_S1 from its definition"""
    W = t["w"].to(dt)
    return {"out": R_PACK[d["mode"]](W).contiguous()}


def _post_autograd(d, t, dt):
    f = t["fmap"].to(dt).clone().requires_grad_(True) if "fmap" in t else torch.zeros(d["B"], 1024, d["H"], d["p"], dtype=dt,
                                                                                      requires_grad=True)
    w = t["w"].to(dt).view(1, 1024, 3, 1).clone().requires_grad_(True) if "w" in t else \
        torch.zeros(1, 1024, 3, 1, dtype=dt, requires_grad=True)
    b = torch.zeros(1, dtype=dt, requires_grad=True)
    F.conv2d(f, w, b, padding=(1, 0)).backward(t["gpost"].to(dt))
    return f.grad, w.grad, b.grad


def post_dgrad_torch(d, t, dt):
    gf, _, _ = _post_autograd(d, t, dt)
    return {"out": gf.permute(0, 3, 2, 1).reshape(-1, d["H"], 1024)}


def post_wgrad_torch(d, t, dt):
    _, gw, gb = _post_autograd(d, t, dt)
    return {"out": gw.reshape(-1), "out_b": gb}


def act_bwd_torch(d, t, dt):
    """autograd of leaky_relu(z, f32(0.1)) at z = the saved fmap (leaky keeps the sign), upstream G's rows + gfmap"""
    B, p, H, C_, off = d["B"], d["p"], d["H"], d["C"], d["off"]
    up = t["G"].to(dt).view(B, p, d["Rg"], C_)[:, :, off:off + H].permute(0, 3, 2, 1)
    if "gfmap" in t:
        up = up + t["gfmap"].to(dt)
    if "fmap" in t:
        z = t["fmap"].to(dt).clone().requires_grad_(True)
        F.leaky_relu(z, SLOPE32).backward(up)
        v = z.grad
    else:
        v = up.contiguous()
    return {"out": v, "rows": F.pad(v.permute(0, 3, 2, 1).reshape(B * p, H, C_), (0, 0, 0, 1)),
            "tr": v.permute(1, 0, 3, 2).reshape(C_, -1)}


def im2col_t_torch(d, t, dt):
    """F.pad + unfold along H of each column's rows; a row of ones; zero padding rows and columns"""
    X, s, H, Kr = t["fmap"].to(dt), d["stride"], d["H"], d["Kr"]
    B, Cin, Hx, p = X.shape
    cols = X.permute(0, 3, 1, 2).reshape(B * p, Cin, Hx)
    need = s * (H - 1) + 5
    cols = F.pad(cols, (2, max(0, need - Hx - 2)))
    u = cols.unfold(2, 5, s)[:, :, :H]                                   # (BB, Cin, H, 5)
    M = u.permute(3, 1, 0, 2).reshape(5 * Cin, B * p * H)
    M = torch.cat([M, torch.ones(1, B * p * H, dtype=dt)])
    return {"tr": F.pad(M, (0, Kr - B * p * H, 0, 7))}


def unpack_wgrad_torch(d, t, dt):
    dWp, Cin = t["dWp"].to(dt), d["Cin"]
    return {"out": dWp[:, :5 * Cin].reshape(-1, 5, Cin).permute(0, 2, 1).contiguous(), "out_b": dWp[:, 5 * Cin]}


def _conv0_autograd(d, t, dt):
    x = t["x"].to(dt).clone().requires_grad_(True) if "x" in t else torch.zeros(d["B"], d["L"], dtype=dt, requires_grad=True)
    w = t["w"].to(dt).clone().requires_grad_(True) if "w" in t else torch.zeros(32, 5, dtype=dt, requires_grad=True)
    b = torch.zeros(32, dtype=dt, requires_grad=True)
    _conv0(x, w, b, d["p"]).backward(t["dz0"].to(dt))
    return x.grad, w.grad, b.grad


def conv0_wgrad_torch(d, t, dt):
    _, gw, gb = _conv0_autograd(d, t, dt)
    return {"out": gw, "out_b": gb}


def conv0_dgrad_torch(d, t, dt):
    gx, _, _ = _conv0_autograd(d, t, dt)
    return {"out": gx}


TORCH = dict(CONV0_FWD=conv0_fwd_torch, ACT_FWD=act_fwd_torch, NCHW_TO_ROWS=nchw_to_rows_torch, POST_FWD=post_fwd_torch,
             PACK=pack_torch, POST_DGRAD=post_dgrad_torch, POST_WGRAD=post_wgrad_torch, ACT_BWD=act_bwd_torch,
             IM2COL_T=im2col_t_torch, UNPACK_WGRAD=unpack_wgrad_torch, CONV0_WGRAD=conv0_wgrad_torch,
             CONV0_DGRAD=conv0_dgrad_torch)


# --------------------------------------------------------------------------------------------------------------------
# cases and their operands
# --------------------------------------------------------------------------------------------------------------------
def with_signed_edges(v, g):
    """v with exact +0, -0 and denormals (both signs) sprinkled in: the `> 0` tests must see them as they are"""
    v = v.clone()
    flat = v.view(-1)
    n = flat.numel()
    specials = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 2.0 ** -149, -(2.0 ** -149), 1.1754942e-38, -1.1754942e-38])
    idx = torch.randperm(n, generator=g)[:max(1, n // 16)]
    flat[idx] = specials[torch.arange(idx.numel()) % specials.numel()]
    return v


def make_operands(d, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)                               # noqa: E731
    k, B, p = d["kind"], d.get("B"), d.get("p")
    if k in ("CONV0_FWD", "CONV0_WGRAD", "CONV0_DGRAD"):
        t = {}
        if k != "CONV0_DGRAD":
            t["x"] = 0.3 * rn(B, d["L"])
        if k != "CONV0_WGRAD":
            t["w"] = rn(32, 1, 5) / 5 ** 0.5
        if k == "CONV0_FWD":
            t["b"] = 0.1 * rn(32)
        else:
            t["dz0"] = rn(B, 32, d["H"], p)
        return t
    if k == "ACT_FWD":
        return {"Y": with_signed_edges(rn(B * p, d["H"], d["C"]), g)}
    if k == "NCHW_TO_ROWS":
        return {"fmap": with_signed_edges(rn(B, d["C"], d["H"], p), g)}
    if k in ("POST_FWD", "POST_DGRAD", "POST_WGRAD"):
        t = {}
        if k != "POST_DGRAD":
            t["fmap"] = leaky(rn(B, 1024, d["H"], p), SLOPE32)
        if k != "POST_WGRAD":
            t["w"] = rn(1, 1024, 3) / (3 * 1024) ** 0.5
        if k == "POST_FWD":
            t["b"] = 0.1 * rn(1)
        else:
            t["gpost"] = rn(B, 1, d["H"], p)
        return t
    if k == "PACK":
        return {"w": rn(d["Cout"], d["Cin"], 5)}
    if k == "ACT_BWD":
        shape = (B, d["C"], d["H"], p)
        t = {"G": rn(B * p, d["Rg"], d["C"])}                    # rows outside [off, off + H) carry values too
        if d.get("gfmap"):
            t["gfmap"] = rn(*shape)
        if d.get("fmap", True):
            t["fmap"] = with_signed_edges(leaky(rn(*shape), SLOPE32), g)
        return t
    if k == "IM2COL_T":
        return {"fmap": with_signed_edges(rn(B, d["Cin"], d["Hx"], p), g)}
    if k == "UNPACK_WGRAD":
        return {"dWp": rn(d["Cout"], 5 * d["Cin"] + 8)}
    raise KeyError(k)


def _cases():
    cs = {}

    def add(name, kind, group, **kw):
        assert name not in cs, name
        cs[name] = dict(kind=kind, group=group, **kw)

    # conv 0 and its gradients: p = 1 .. 11; L a multiple of p, L % p != 0 up to the largest mirror (p - 1 padded samples),
    # the shortest legal L (p = 11, L = 6: H0 = 1), L = 12 at p = 11, L = 4099 at B = 3, B p above one block of positions,
    # the trainer's L = 20480
    geos = [("p1_l300", 2, 1, 300, "mirror"), ("p2_l4096", 2, 2, 4096, "multiple"), ("p2_l3", 1, 2, 3, "shortest"),
            ("p3_l1000_npad2", 3, 3, 1000, "mirror"), ("p5_l4099_b3", 3, 5, 4099, "mirror"), ("p7_l22_npad6", 2, 7, 22, "mirror"),
            ("p7_l700", 2, 7, 700, "multiple"), ("p11_l6", 1, 11, 6, "shortest"), ("p11_l12", 2, 11, 12, "shortest"),
            ("p11_l4099_b8", 8, 11, 4099, "mirror"), ("p2_l20480", 2, 2, 20480, "trainer"),
            ("p11_l20480", 2, 11, 20480, "trainer")]
    for tag, B, p, L, group in geos:
        hs = layer_H(p, L)
        H0 = hs[1]
        add(f"conv0_fwd_{tag}", "CONV0_FWD", group, B=B, p=p, L=L, H=H0, R=3 * hs[2], rows="f" if p % 2 else "split")
        add(f"conv0_wgrad_{tag}", "CONV0_WGRAD", group, B=B, p=p, L=L, H=H0)
        add(f"conv0_dgrad_{tag}", "CONV0_DGRAD", group, B=B, p=p, L=L, H=H0)
    add("conv0_fwd_p5_l4099_r_plus5_both", "CONV0_FWD", "rows", B=3, p=5, L=4099, H=layer_H(5, 4099)[1],
        R=layer_H(5, 4099)[1] + 5, rows="both")
    add("conv0_fwd_p11_l6_r3", "CONV0_FWD", "rows", B=1, p=11, L=6, H=1, R=3, rows="both")
    add("conv0_fwd_p3_l1000_norows", "CONV0_FWD", "rows", B=3, p=3, L=1000, H=layer_H(3, 1000)[1], R=layer_H(3, 1000)[1],
        rows=None)

    # leaky ReLU + NCHW + next-layer rows: H = 1, 2, 3, 7, 29; slopes 0.1 and 1; planes fp32, split, both, none
    for H, C_, R_, B, p, rows in ((1, 32, 3, 2, 3, "f"), (2, 128, 3, 1, 5, "split"), (3, 128, 3, 2, 2, "both"),
                                  (7, 512, 9, 2, 7, "split"), (29, 1024, 29, 1, 11, None), (29, 128, 30, 3, 1, "both")):
        for slope in (0.1, 1.0):
            add(f"act_fwd_h{H}_c{C_}_s{slope:g}", "ACT_FWD", "shapes", B=B, p=p, L=H * p, H=H, C=C_, R=R_, slope=slope, rows=rows)
    for p in (2, 11):
        hs = layer_H(p, 20480)
        for i in range(1, 5):
            R_ = 3 * hs[i + 2] if i < 3 else hs[i + 1]
            add(f"act_fwd_trainer_p{p}_layer{i}", "ACT_FWD", "trainer", B=2, p=p, L=20480, H=hs[i + 1], C=COUT[i], R=R_, slope=0.1,
                rows="split" if i < 4 else None)
    for H, C_, R_, B, p, rows in ((1, 32, 1, 1, 1, "f"), (7, 128, 9, 2, 3, "split"), (29, 1024, 30, 2, 5, "both")):
        add(f"rows_h{H}_c{C_}_r{R_}", "NCHW_TO_ROWS", "shapes", B=B, p=p, L=H * p, H=H, C=C_, R=R_, rows=rows)
    hs = layer_H(11, 20480)
    add("rows_trainer_p11_fmap0", "NCHW_TO_ROWS", "trainer", B=2, p=11, L=20480, H=hs[1], C=32, R=3 * hs[2], rows="both")

    # conv_post forward and gradients: H p below and above one 32-position block, B p up to 88, reductions with fewer
    # elements than the 256 threads and with many per thread
    for B, p, H, group in ((1, 1, 1, "small"), (1, 2, 1, "small"), (2, 3, 2, "small"), (2, 5, 7, "blocks"), (1, 11, 3, "blocks"),
                           (1, 1, 40, "blocks"), (3, 7, 29, "blocks"), (8, 11, 3, "blocks"), (4, 5, 127, "many"), (2, 2, layer_H(2, 20480)[5], "trainer"),
                           (2, 11, layer_H(11, 20480)[5], "trainer")):
        for kind in ("POST_FWD", "POST_DGRAD", "POST_WGRAD"):
            add(f"{kind.lower()}_b{B}_p{p}_h{H}", kind, group, B=B, p=p, L=H * p, H=H, C=1024)

    # the four packings at the layer shapes and an odd one
    for mode in ("FWD_S3", "FWD_S1", "DGRAD_S3", "DGRAD_S1"):
        for Cout, Cin in ((3, 2), (128, 32), (1024, 512)):
            add(f"pack_{mode.lower()}_{Cout}x{Cin}", "PACK", mode.lower(), Cout=Cout, Cin=Cin, mode=mode)

    # dZ = (G + gfmap) leaky'(fmap) in the three (Rg, off) layouts st_mpd_backward builds, written as rows, dZ^T and NCHW
    def act_bwd(name, group, B, p, H, C_, layout, **kw):
        Rg, off = {"post": (H, 0), "s1": (H + 1, 0), "s3": (3 * (ceil_div(H, 3) + 1), 3)}[layout]
        if kw.get("tr"):
            kw.setdefault("Kr", kr_of(B * p * H))
        add(name, "ACT_BWD", group, B=B, p=p, L=H * p, H=H, C=C_, Rg=Rg, off=off, **kw)

    act_bwd("act_bwd_post_b2_p3_h2", "post", 2, 3, 2, 1024, "post", gfmap=True, rows="f", tr="f", nchw=True)
    act_bwd("act_bwd_post_b1_p1_h1", "post", 1, 1, 1, 1024, "post", gfmap=True, rows="split", tr="split")
    act_bwd("act_bwd_post_nogfmap", "post", 2, 5, 7, 1024, "post", rows="both", tr="both", nchw=True)
    act_bwd("act_bwd_s1_b2_p7_h29", "s1", 2, 7, 29, 1024, "s1", gfmap=True, rows="split", tr="split")
    act_bwd("act_bwd_s1_h1", "s1", 1, 2, 1, 1024, "s1", rows="f", tr="both", nchw=True)
    act_bwd("act_bwd_s3_b2_p2_h64_kr256", "s3", 2, 2, 64, 128, "s3", gfmap=True, rows="split", tr="split", Kr=256)
    act_bwd("act_bwd_s3_b3_p5_h7", "s3", 3, 5, 7, 512, "s3", gfmap=True, rows="both", tr="f", nchw=True)
    act_bwd("act_bwd_s3_h3_kr_plus256", "s3", 2, 11, 3, 128, "s3", rows="f", tr="both", Kr=kr_of(66) + 256)
    act_bwd("act_bwd_slope1_nchw", "hook", 2, 3, 7, 128, "s3", fmap=False, nchw=True)
    act_bwd("act_bwd_slope1_gfmap_rows", "hook", 1, 5, 2, 32, "s1", fmap=False, gfmap=True, rows="f")
    act_bwd("act_bwd_conv0_nchw", "conv0", 2, 7, 29, 32, "s3", nchw=True)
    for p in (2, 11):
        hs = layer_H(p, 20480)
        for i in range(0, 5):
            H = hs[i + 1]
            layout = "post" if i == 4 else ("s1" if i == 3 else "s3")
            kw = dict(nchw=True) if i == 0 else dict(rows="split" if p == 2 else "f", tr="split" if p == 2 else "f")
            act_bwd(f"act_bwd_trainer_p{p}_layer{i}", "trainer", 2, p, H, COUT[i], layout, gfmap=i in (1, 3), **kw)

    # the wgrad W operand, stride 3 and 1; Kr = B p H exactly 256 and not a multiple of it
    for B, p, Hx, Cin, s, tr in ((1, 1, 1, 1, 3, "f"), (2, 3, 2, 32, 3, "split"), (2, 5, 7, 32, 3, "both"),
                                 (2, 2, 190, 32, 3, "both"), (2, 7, 29, 128, 3, "split"), (2, 3, 29, 64, 1, "both"),
                                 (1, 2, 128, 32, 1, "f"), (1, 1, 1, 8, 1, "split")):
        H = ceil_div(Hx, 3) if s == 3 else Hx
        add(f"im2col_s{s}_b{B}_p{p}_hx{Hx}_c{Cin}", "IM2COL_T", f"stride{s}", B=B, p=p, L=Hx * p, Hx=Hx, Cin=Cin, H=H, stride=s,
            Kr=kr_of(B * p * H), tr=tr)
    add("im2col_s3_kr_plus256", "IM2COL_T", "stride3", B=2, p=3, L=21, Hx=7, Cin=32, H=3, stride=3, Kr=kr_of(18) + 256, tr="f")
    for p in (2, 11):
        hs = layer_H(p, 20480)
        for i in range(1, 5):
            add(f"im2col_trainer_p{p}_layer{i}", "IM2COL_T", "trainer", B=2, p=p, L=20480, Hx=hs[i], Cin=CIN[i], H=hs[i + 1],
                stride=STRIDE[i], Kr=kr_of(2 * p * hs[i + 1]), tr="split" if p == 2 else "f")

    for Cout, Cin in ((3, 2), (128, 32), (512, 128), (1024, 512), (1024, 1024)):
        add(f"unpack_{Cout}x{Cin}", "UNPACK_WGRAD", "layers", Cout=Cout, Cin=Cin)
    return cs


CASES = _cases()




# --------------------------------------------------------------------------------------------------------------------
# CPU: every statement against independent torch code
# --------------------------------------------------------------------------------------------------------------------
CPU_CASES = ["conv0_fwd_p1_l300", "conv0_fwd_p7_l22_npad6", "conv0_fwd_p11_l6", "conv0_fwd_p11_l12", "conv0_wgrad_p3_l1000_npad2",
             "conv0_wgrad_p11_l6", "conv0_dgrad_p3_l1000_npad2", "conv0_dgrad_p7_l22_npad6", "conv0_dgrad_p11_l12",
             "conv0_dgrad_p2_l4096", "act_fwd_h3_c128_s0.1", "act_fwd_h29_c128_s1", "rows_h7_c128_r9", "post_fwd_b2_p5_h7",
             "post_fwd_b1_p1_h1", "post_dgrad_b2_p5_h7", "post_dgrad_b1_p2_h1", "post_wgrad_b2_p5_h7", "post_wgrad_b1_p1_h1",
             "act_bwd_post_b2_p3_h2", "act_bwd_s1_b2_p7_h29", "act_bwd_s3_b3_p5_h7", "act_bwd_slope1_nchw",
             "act_bwd_slope1_gfmap_rows", "im2col_s3_b2_p5_hx7_c32", "im2col_s1_b2_p3_hx29_c64", "im2col_s3_b1_p1_hx1_c1",
             "unpack_128x32", "pack_fwd_s1_128x32"]


def _compare_statement(d, t, dt):
    r, w = STATEMENTS[d["kind"]](d, {k: v.to(dt) for k, v in t.items()}), TORCH[d["kind"]](d, t, dt)
    for k in r:
        a, b = r[k], w[k].reshape(r[k].shape)
        if d["kind"] in EXACT:
            assert torch.equal(bits(a.float().contiguous()), bits(b.float().contiguous())), k
        else:
            assert torch.allclose(a, b, rtol=1e-10, atol=1e-10 * float(b.abs().max())), (k, float((a - b).abs().max()))


@pytest.mark.parametrize("name", CPU_CASES)
def test_statement_matches_torch(name):
    d = CASES[name]
    t = make_operands(d, 1)
    if d["kind"] in EXACT:
        _compare_statement(d, t, torch.float32)                        # the GPU's bars: the bits of torch fp32
    _compare_statement(d, {k: v.double() for k, v in t.items()}, torch.float64)


def test_reflect_view_is_the_reference_pad():
    """the statement's index formula is F.pad(..., "reflect"), at every mirror length 0 .. p - 1"""
    g = torch.Generator().manual_seed(3)
    for p in (1, 2, 3, 5, 7, 11):
        for L in range(max(2, p), 3 * p + 2):
            if L % p and p - L % p >= L:
                continue
            x = torch.randn(2, L, generator=g, dtype=torch.float64)
            assert torch.equal(reflect_view(x, p), R.pad_view(x[:, None], p)[:, 0]), (p, L)


def test_packings_are_the_conv():
    """each packing, applied as the conv-GEMM engine applies it, is the conv (or its adjoint) it packs"""
    g = torch.Generator().manual_seed(4)
    for H in (1, 2, 7, 29):
        X = torch.randn(H, 6, generator=g, dtype=torch.float64, requires_grad=True)
        W = torch.randn(5, 6, 5, generator=g, dtype=torch.float64)
        for s in (3, 1):
            Y = R.conv_rows(X, W, s)
            dZ = torch.randn(Y.shape, generator=g, dtype=torch.float64)
            (dX,) = torch.autograd.grad((Y * dZ).sum(), X)
            with torch.no_grad():
                if s == 3:
                    Yp, dXp = R.strided_forward(X, W), R.strided_dgrad(dZ, W, H)
                else:
                    Yp, dXp = R.engine_conv(X, R_PACK["FWD_S1"](W)), R.engine_conv(dZ, R_PACK["DGRAD_S1"](W))
            assert torch.allclose(Yp, Y.detach(), rtol=1e-12, atol=1e-12) and torch.allclose(dXp, dX, rtol=1e-12, atol=1e-12)


def test_operands_carry_signed_zeros_and_denormals():
    """the fmaps and pre-activations the slope tests see hold +0, -0 and denormals of both signs"""
    for name in ("act_bwd_post_b2_p3_h2", "act_fwd_h7_c512_s0.1"):
        d = CASES[name]
        v = make_operands(d, 5)["fmap" if d["kind"] == "ACT_BWD" else "Y"]
        b = bits(v)
        assert (b == 0).any() and (b == bits(torch.tensor([-0.0]))[0]).any()
        den = (v != 0) & (v.abs() < 1.1754944e-38)
        assert (den & (v > 0)).any() and (den & (v < 0)).any()


def test_case_geometry_covers_the_edges():
    """p = 1 .. 11 with L % p == 0 and the largest mirror, H0 = 1, R > H0, B p above one 32-position block, reductions
    below and above 256 elements, Kr a multiple of 256 and not, the three (Rg, off) layouts"""
    conv0 = [d for d in CASES.values() if d["kind"] == "CONV0_FWD"]
    assert {d["p"] for d in conv0} >= {1, 2, 3, 5, 7, 11}
    assert any(d["L"] % d["p"] == 0 and d["p"] > 1 for d in conv0)
    assert any(d["L"] % d["p"] == 1 and d["p"] > 2 for d in conv0)                # npad = p - 1
    assert any(d["H"] == 1 for d in conv0) and any(d["R"] > d["H"] for d in conv0)
    post = [d for d in CASES.values() if d["kind"] == "POST_WGRAD"]
    assert min(d["B"] * d["p"] * d["H"] for d in post) < 256 < max(d["B"] * d["p"] * d["H"] for d in post) // 8
    c0 = [d["B"] * d["p"] * d["H"] for d in CASES.values() if d["kind"] == "CONV0_WGRAD"]
    assert min(c0) < 256 < max(c0) // 32
    assert max(d["B"] * d["p"] for d in post) == 88
    kr = [(d["B"] * d["p"] * d["H"], d["Kr"]) for d in CASES.values() if "Kr" in d]
    assert any(n % 256 == 0 and n == k for n, k in kr) and any(n % 256 for n, k in kr) and any(k > kr_of(n) for n, k in kr)
    lay = {(d["Rg"] - d["H"], d["off"]) for d in CASES.values() if d["kind"] == "ACT_BWD"}
    assert (0, 0) in lay and (1, 0) in lay and any(o == 3 for _, o in lay)
    assert {d["H"] for d in CASES.values() if d["kind"] in ("ACT_FWD", "ACT_BWD")} >= {1, 2, 3, 7, 29}


def test_kind_numbers_match_the_binding():
    """the binding's st_test_mpd_row_desc.kind names are the enum of include/stabletts_b200.h, and its pack modes mpd.cuh's"""
    from stabletts_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "stabletts_b200.h")).read()
    enum = {k: int(v) for k, v in re.findall(r"\bST_TEST_MPD_ROW_(\w+)\s*=\s*(\d+)", header)}
    assert enum == {k: i for i, k in enumerate(_lib.ST_TEST_MPD_ROW_KINDS)}
    cuh = open(os.path.join(root, "stabletts_b200", "csrc", "mpd.cuh")).read()
    modes = {k: int(v) for k, v in re.findall(r"\bMPD_PACK_(\w+)\s*=\s*(\d+)", cuh)}
    assert modes == {k: i for i, k in enumerate(_lib.ST_TEST_MPD_PACK_MODES)}


# --------------------------------------------------------------------------------------------------------------------
# GPU: the hook's driver
# --------------------------------------------------------------------------------------------------------------------
def output_shapes(d):
    """{output: shape} of case d: "out", "out_b", and the plane sets "rows" / "tr" it requests"""
    k, B, p, H = d["kind"], d.get("B"), d.get("p"), d.get("H")
    BB = B * p if B else None
    s = {}
    if k == "CONV0_FWD":
        s["out"] = (B, 32, H, p)
    elif k == "ACT_FWD":
        s["out"] = (B, d["C"], H, p)
    elif k == "POST_FWD":
        s["out"] = (B, 1, H, p)
    elif k == "PACK":
        s3 = d["mode"].endswith("S3")
        K3 = 3 * d["Cin"] if s3 else d["Cin"]
        s["out"] = (2 if s3 else 5,) + ((d["Cout"], K3) if d["mode"].startswith("FWD") else (K3, d["Cout"]))
    elif k == "POST_DGRAD":
        s["out"] = (BB, H, 1024)
    elif k == "POST_WGRAD":
        s["out"], s["out_b"] = (1024 * 3,), (1,)
    elif k == "ACT_BWD" and d.get("nchw"):
        s["out"] = (B, d["C"], H, p)
    elif k == "UNPACK_WGRAD":
        s["out"], s["out_b"] = (d["Cout"], d["Cin"], 5), (d["Cout"],)
    elif k == "CONV0_WGRAD":
        s["out"], s["out_b"] = (32, 5), (32,)
    elif k == "CONV0_DGRAD":
        s["out"] = (B, d["L"])
    if d.get("rows"):
        s["rows"] = (BB, d["R"], 32 if k == "CONV0_FWD" else d["C"]) if k != "ACT_BWD" else (BB, H + 1, d["C"])
    if d.get("tr"):
        s["tr"] = (d["C"] if k == "ACT_BWD" else 5 * d["Cin"] + 8, d["Kr"])
    return s


INPUTS = ("x", "w", "b", "Y", "G", "gpost", "fmap", "gfmap", "dz0", "dWp")


def run_mpd_hook(lib, h, d, t, dev, desc_edit=None):
    """Runs case d on operands t through st_test_mpd_row_ex; returns (rc, error text, outputs).  Outputs start as NaN;
    ACT_BWD's dZ^T columns >= B p H start as SENTINEL, which the kernel must leave alone.  A plane set "f", "split" or
    "both" becomes o[set + "_f"], o[set + "_hi"], o[set + "_lo"]."""
    from stabletts_b200 import _lib
    keep = {n: v.to(dev).contiguous() for n, v in t.items()}
    full = lambda s, dtype=torch.float32: torch.full(s, NAN, device=dev, dtype=dtype)    # noqa: E731
    o = {}
    for what, shape in output_shapes(d).items():
        if what in ("rows", "tr"):
            planes = d[what]
            if planes in ("f", "both"):
                o[what + "_f"] = full(shape)
            if planes in ("split", "both"):
                o[what + "_hi"], o[what + "_lo"] = full(shape, torch.bfloat16), full(shape, torch.bfloat16)
        else:
            o[what] = full(shape)
    if d["kind"] == "ACT_BWD" and "tr" in output_shapes(d):
        for n in ("tr_f", "tr_hi", "tr_lo"):
            if n in o:
                o[n][:, d["B"] * d["p"] * d["H"]:] = SENTINEL
    desc = _lib.StTestMpdRowDesc()
    for n in INPUTS:
        setattr(desc, n, keep[n].data_ptr() if n in keep else None)
    for n in ("out", "out_b", "rows_f", "rows_hi", "rows_lo", "tr_f", "tr_hi", "tr_lo"):
        setattr(desc, n, o[n].data_ptr() if n in o else None)
    desc.kind = _lib.ST_TEST_MPD_ROW_KINDS.index(d["kind"])
    for n in ("L", "Kr", "B", "p", "H", "C", "R", "Rg", "off", "Hx", "Cin", "Cout", "stride"):
        if n in d:
            setattr(desc, n, int(d[n]))
    if "mode" in d:
        desc.mode = _lib.ST_TEST_MPD_PACK_MODES.index(d["mode"])
    desc.slope = float(d.get("slope", 0.0))
    if desc_edit:
        desc_edit(desc)
    rc = lib.st_test_mpd_row_ex(h, C.byref(desc), torch.cuda.current_stream().cuda_stream)
    err = lib.st_last_error(h).decode() if rc else ""
    return rc, err, {n: v.cpu() for n, v in o.items()}


def _plane_checks(o, what, want):
    """plane set `what` holds the fp32 values `want` (bits; its hi / lo planes their split)"""
    if what + "_f" in o:
        assert torch.equal(bits(o[what + "_f"]), bits(want.contiguous())), what
    if what + "_hi" in o:
        check_planes({"hi": o[what + "_hi"], "lo": o[what + "_lo"]}, "split", src=want.contiguous())


def check_case(d, t, o):
    """value checks; returns [(output, max |err|, bar)] (exact kinds: (output, 0, 1) once their bits matched)"""
    k = d["kind"]
    ref = STATEMENTS[k](d, t)                           # fp64 for the arithmetic kinds, the fp32 operations for the exact ones
    rows = []
    if k in EXACT:
        for what in ("out", "out_b"):
            if what in o:
                assert torch.equal(bits(o[what]), bits(ref[what].reshape(o[what].shape).contiguous())), what
                rows.append((what, 0.0, 1.0))
        if "rows" in output_shapes(d):
            _plane_checks(o, "rows", ref["rows"])
            rows.append(("rows", 0.0, 1.0))
        if "tr" in output_shapes(d):
            if k == "ACT_BWD":                          # the columns past B p H keep their sentinel in every plane
                BBH = d["B"] * d["p"] * d["H"]
                tr = {n: v for n, v in o.items() if n.startswith("tr_")}
                for n, v in tr.items():
                    assert (v[:, BBH:].float() == SENTINEL).all(), n
                _plane_checks({n: v[:, :BBH] for n, v in tr.items()}, "tr", ref["tr"])
            else:
                _plane_checks(o, "tr", ref["tr"])
            rows.append(("tr", 0.0, 1.0))
        return rows
    f32 = TORCH[k](d, t, torch.float32)
    for what in ("out", "out_b"):
        if what not in ref:
            continue
        r = ref[what].reshape(o[what].shape)
        got = o[what].double()
        assert torch.isfinite(got).all(), what
        e32 = float((f32[what].double().reshape(r.shape) - r).abs().max())
        err = float((got - r).abs().max())
        b = bar(r, e32)
        rows.append((what, err, b))
        assert err <= b, (what, err, b, e32)
    if k == "CONV0_FWD" and "rows" in output_shapes(d):    # the rows hold the bits of fmap0, zero below R
        _plane_checks(o, "rows", nchw_to_rows(o["out"], d["R"]))
    return rows


@pytest.fixture(scope="module")
def matrix(dev, handle):
    def run(name):
        d = CASES[name]
        t = make_operands(d, 3000 + list(CASES).index(name))
        return check_case(d, t, run_ok(run_mpd_hook, *handle, d, t, dev))
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
@pytest.mark.parametrize("name", ["post_wgrad_b3_p7_h29", "conv0_wgrad_p11_l20480", "post_fwd_b8_p11_h3", "conv0_dgrad_p5_l4099_b3"])
def test_repeated_runs_are_bit_identical(name, dev, handle):
    """fixed summation orders: the block reductions and the per-element sums do not depend on scheduling"""
    lib, h = handle
    d = CASES[name]
    t = make_operands(d, 77)
    first, again = run_ok(run_mpd_hook, lib, h, d, t, dev), run_ok(run_mpd_hook, lib, h, d, t, dev)
    for k in first:
        assert torch.equal(bits(first[k]), bits(again[k])), k


@pytest.mark.gpu
def test_refusals(dev, handle):
    """every problem outside the contract is refused with a readable error, and nothing is launched"""
    from stabletts_b200 import _lib
    lib, h = handle

    def refused(name, needle, case=None, **fields):
        """case: fields of the case itself (which outputs the driver allocates); fields: descriptor fields"""
        d = dict(CASES[name], **(case or {}))
        t = make_operands(d, 90)
        rc, err, o = run_mpd_hook(lib, h, d, t, dev, desc_edit=set_fields(**fields))
        assert rc != 0 and needle in err, (name, needle, err)
        for k, v in o.items():
            untouched = torch.isnan(v.float()) | (v.float() == SENTINEL)
            assert untouched.all(), (name, k)

    # geometry st_mpd_forward refuses
    refused("conv0_fwd_p11_l6", "L too short for the reflect pad", L=5)
    refused("conv0_fwd_p2_l4096", "L must be in [1, 2^30]", L=0)
    refused("conv0_fwd_p2_l4096", "B must be in [1, 65535]", B=0)
    refused("post_fwd_b8_p11_h3", "B * period must be at most 65535", B=6000)
    refused("act_fwd_h3_c128_s0.1", "p must be in [1, 4096]", p=0)
    refused("conv0_dgrad_p11_l12", "H must be H0", H=2)
    # rows below the layer's rows, Kr below B p H, Rg below H + off
    refused("conv0_fwd_p5_l4099_b3", "R must be >= H", R=CASES["conv0_fwd_p5_l4099_b3"]["H"] - 1)
    refused("act_fwd_h7_c512_s0.1", "R must be >= H", R=6)
    refused("rows_h7_c128_r9", "R must be >= H", R=6)
    refused("act_bwd_s3_b2_p2_h64_kr256", "Kr must be >= B p H", Kr=255)
    refused("im2col_s3_b2_p2_hx190_c32", "Kr must be >= B p H", Kr=255)
    refused("act_bwd_post_b2_p3_h2", "Rg must be >= H + off", Rg=1)
    refused("act_bwd_s3_b3_p5_h7", "Rg must be >= H + off", off=CASES["act_bwd_s3_b3_p5_h7"]["Rg"] - 6)
    refused("im2col_s3_b2_p5_hx7_c32", "H must be ceil(Hx / 3)", H=4)
    refused("im2col_s3_b2_p5_hx7_c32", "stride must be 1 or 3", stride=2)
    refused("post_dgrad_b2_p5_h7", "C must be 1024", C=512)
    # kinds, pack modes, planes, pointers
    refused("pack_fwd_s3_3x2", "unknown pack mode", mode=4)
    refused("pack_fwd_s3_3x2", "unknown kind", kind=len(_lib.ST_TEST_MPD_ROW_KINDS))
    refused("act_fwd_h2_c128_s0.1", "hi and lo go together", rows_lo=None)
    refused("act_bwd_s1_b2_p7_h29", "hi and lo go together", tr_lo=None)
    refused("conv0_fwd_p2_l4096", "a required input is NULL", x=None)
    refused("post_wgrad_b2_p5_h7", "a required input is NULL", fmap=None)
    refused("act_bwd_post_b2_p3_h2", "a required input is NULL", G=None)
    refused("conv0_wgrad_p2_l4096", "a required output is NULL", out_b=None)
    refused("rows_h1_c32_r1", "a required output is NULL", rows_f=None)
    refused("post_fwd_b2_p5_h7", "does not write", case=dict(rows="f", R=7))
    refused("act_bwd_slope1_nchw", "no output requested", case=dict(nchw=False))
    rc = lib.st_test_mpd_row_ex(h, None, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and "null descriptor" in lib.st_last_error(h).decode()
