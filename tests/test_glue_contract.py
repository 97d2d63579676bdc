"""The front-end row kernels and the CFM conditioning and solver kernels against fp64 statements of their contracts
(st_test_row_ex, include/stabletts_b200.h), and fixed-grid solves deep enough to refill the solver's time tables.

Kernels: the MelStyleEncoder's glu_residual_kernel and masked_mean_kernel, the DurationPredictor's
cond_mask_transpose_kernel and relu_ln_kernel<1024, 0 | 1> (the second writes logw, which becomes durations through
ceil(exp(.))), the CFM conditioning kernels gemv_kernel, time_embed_kernel, time_embed_val_kernel and rope_table_kernel,
and the solver arithmetic lincomb_kernel, scaled_sumsq_kernel (the adaptive controller's error norm), cfg_combine_kernel,
cfm_mix_kernel and cfm_loss_kernel + cfm_loss_final_kernel.  The hook calls the product's own launchers.

Each kind has an fp64 statement; the CPU tests pin it against independent torch code (F.glu, masked_fill + sum, F.layer_norm
after relu, F.linear with F.silu, torch.sin / torch.cos of the reference's embedding code, a plain sum of squares,
F.mse_loss).

Bars, against the fp64 statement on the same fp32 inputs (test_row_contract's, kernel_harness.bar):
  fp32 outputs:   max |out - ref64| <= max(4 E32, 8 * 2^-24 * max |ref64|), E32 = max |torch fp32 - ref64| of the same
                  operation done by the torch code in fp32 on the CPU;
  split planes:   hi = bf16(out_f32) and lo = bf16(out_f32 - hi), bit for bit;
  double outputs: the same rule, E32 taken from the fp32 terms summed in double.
`pytest -s` prints the worst ratio to the bar per kind and case group."""
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_errs
from oracle import cases, weights
from oracle import estimator_ref as R
from kernel_harness import (LazyMatrix, NAN, bar, bits, check_planes, make_mask, report_worst_per_group, run_ok,
                            run_row_hook, set_fields)
from kernel_harness import dev, handle  # noqa: F401 (fixtures)

LN_C = 1024                                     # relu_ln_kernel's one width (DurationPredictor filter_channels)
LN_EPS = 1e-5
SPECIAL_T = (0.0, 1e-7, 0.5, 1.0 - 2.0 ** -24, 1.0)
GRID_ELEMS = 592 * 256                          # scaled_sumsq / cfm_loss run at most 592 blocks of 256 threads
F32 = lambda v: float(torch.tensor(v, dtype=torch.float32))     # noqa: E731  (the value an fp32 descriptor field holds)


# --------------------------------------------------------------------------------------------------------------------
# fp64 statements
# --------------------------------------------------------------------------------------------------------------------
def _silu64(v):
    return v / (1.0 + torch.exp(-v))


def glu_resid_ref(d, t):
    """resid + a sigmoid(g), [a | g] = one 2C row"""
    x, C_ = t["x"].double(), d["C"]
    return {"out": t["x1"].double() + x[..., :C_] / (1.0 + torch.exp(-x[..., C_:]))}


def masked_mean_ref(d, t):
    """sum over the frames with mask != 0 over their count (all frames without a mask); 0 / 0 = NaN when none is valid"""
    x = t["x"].double()
    rows = []
    for b in range(x.shape[0]):
        keep = (t["mask"][b] != 0) if "mask" in t else torch.ones(x.shape[1], dtype=torch.bool)
        rows.append(x[b, keep].sum(0) / float(keep.sum()) if keep.any() else torch.full((x.shape[2],), NAN, dtype=torch.float64))
    return {"out": torch.stack(rows)}


def cond_transpose_ref(d, t):
    """(B, C, T) -> (B, T, C) of (x + cond[b, c]) mask[b, t]"""
    return {"out": ((t["x"].double() + t["bias"].double()[:, :, None]) * t["mask"].double()[:, None, :]).transpose(1, 2)}


def _ln64(t):
    v = t["x"].double().clamp(min=0.0)
    mean = v.mean(-1, keepdim=True)
    var = ((v - mean) ** 2).mean(-1, keepdim=True)
    return (v - mean) / torch.sqrt(var + LN_EPS) * t["ln_w"].double() + t["ln_b"].double()


def relu_ln_ref(d, t):
    """LN(relu(x); ln_w, ln_b, eps 1e-5) m with the biased variance; PROJ: (m sum_c u_c p_c + p_b) m"""
    u, m = _ln64(t), t["mask"].double()
    if d["kind"] == "RELU_LN":
        return {"out": u * m[..., None]}
    return {"out": (m * (u * t["w"].double()).sum(-1) + t["bias"].double()[0]) * m}


def gemv_ref(d, t):
    """y[r, n] = act_out(sum_k act_in(x[r, k]) W[n, k] + bias[n])"""
    x = t["x"].double()
    if d["silu_in"]:
        x = _silu64(x)
    y = (x[:, None, :] * t["w"].double()[None, :, :]).sum(-1)
    if "bias" in t:
        y = y + t["bias"].double()
    return {"out": _silu64(y) if d["silu_out"] else y}


def time_embed_ref(d, t):
    """e_j = 1000 t exp(-j ln(1e4) / (half - 1)) -> [sin e | cos e]"""
    half = d["C"] // 2
    j = torch.arange(half, dtype=torch.float64)
    e = 1000.0 * t["x"].double()[:, None] * torch.exp(-j * math.log(1e4) / (half - 1))[None, :]
    return {"out": torch.cat([torch.sin(e), torch.cos(e)], -1)}


def rope_table_ref(d, t):
    """(cos, sin)(pos 10000^(-2j / 32)), (T, 16, 2)"""
    pos = torch.arange(d["T"], dtype=torch.float64)[:, None]
    ang = pos * 10000.0 ** (-2.0 * torch.arange(16, dtype=torch.float64) / 32.0)[None, :]
    return {"out": torch.stack([torch.cos(ang), torch.sin(ang)], -1)}


def lincomb_ref(d, t):
    """y + sum_{j < n} c_j K_j"""
    y = t["x"].double().clone()
    for j, c in enumerate(d["coef"]):
        y += F32(c) * t["terms"][j].double()
    return {"out": y}


def _sumsq_num_tol(d, t, dtype):
    num = torch.zeros_like(t["x"], dtype=dtype)
    for j, c in enumerate(d["coef"]):
        num = num + torch.tensor(F32(c), dtype=dtype) * t["terms"][j].to(dtype)
    tol = (torch.tensor(F32(d["atol"]), dtype=dtype)
           + torch.tensor(F32(d["rtol"]), dtype=dtype) * torch.maximum(t["x"].to(dtype).abs(), t["x1"].to(dtype).abs()))
    return num, tol


def scaled_sumsq_ref(d, t):
    """sum_e (sum_j c_j K_j[e] / (atol + rtol max(|u[e]|, |v[e]|)))^2"""
    num, tol = _sumsq_num_tol(d, t, torch.float64)
    return {"f64": ((num / tol) ** 2).sum().reshape(1)}


def cfg_combine_ref(d, t):
    """u + s (c - u) with cfg (V = [cond rows | uncond rows]), else c"""
    n = d["B"] * d["n"]
    V = t["x"].double()
    c = V[:n]
    return {"out": V[n:] + F32(d["s_cfg"]) * (c - V[n:]) if d["cfg"] else c}


def cfm_mix_ref(d, t):
    """(1 - (1 - sigma_min) t_b) z + t_b x1"""
    s, tb = F32(d["sigma_min"]), t["x2"].double()[:, None, None]
    return {"out": (1.0 - (1.0 - s) * tb) * t["x1"].double() + tb * t["x"].double()}


def cfm_loss_ref(d, t):
    """sum over every position (padded frames included) of (v - (x1 - (1 - sigma_min) z))^2, sum(mask), and their ratio
    over C"""
    s = F32(d["sigma_min"])
    sq = ((t["x2"].double() - (t["x"].double() - (1.0 - s) * t["x1"].double())) ** 2).sum()
    msum = t["mask"].double().sum()
    return {"out": (sq / (msum * d["C"])).reshape(1), "f64": torch.stack([sq, msum])}


STATEMENTS = dict(GLU_RESID=glu_resid_ref, MASKED_MEAN=masked_mean_ref, COND_TRANSPOSE=cond_transpose_ref, RELU_LN=relu_ln_ref,
                  RELU_LN_PROJ=relu_ln_ref, GEMV=gemv_ref, TIME_EMBED=time_embed_ref, TIME_EMBED_VALS=time_embed_ref,
                  ROPE_TABLE=rope_table_ref, LINCOMB=lincomb_ref, SCALED_SUMSQ=scaled_sumsq_ref, CFG_COMBINE=cfg_combine_ref,
                  CFM_MIX=cfm_mix_ref, CFM_LOSS=cfm_loss_ref)


# --------------------------------------------------------------------------------------------------------------------
# independent torch code (run in fp64 it pins the statement; run in fp32 it gives E32)
# --------------------------------------------------------------------------------------------------------------------
def glu_resid_torch(d, t, dt):
    return {"out": t["x1"].to(dt) + F.glu(t["x"].to(dt), dim=-1)}


def masked_mean_torch(d, t, dt):
    x = t["x"].to(dt)
    valid = (t["mask"] != 0) if "mask" in t else torch.ones(x.shape[:2], dtype=torch.bool)
    return {"out": x.masked_fill(~valid[..., None], 0.0).sum(1) / valid.sum(1, keepdim=True).to(dt)}


def cond_transpose_torch(d, t, dt):
    return {"out": ((t["x"].to(dt) + t["bias"].to(dt).unsqueeze(-1)) * t["mask"].to(dt).unsqueeze(1)).transpose(1, 2)}


def relu_ln_torch(d, t, dt):
    """duration_predictor.py: relu -> norm -> (proj(x * mask) * mask)"""
    u = F.layer_norm(F.relu(t["x"].to(dt)), (LN_C,), t["ln_w"].to(dt), t["ln_b"].to(dt), LN_EPS)
    m = t["mask"].to(dt)[..., None]
    if d["kind"] == "RELU_LN":
        return {"out": u * m}
    return {"out": (F.linear(u * m, t["w"].to(dt)[None, :], t["bias"].to(dt)) * m)[..., 0]}


def gemv_torch(d, t, dt):
    x = t["x"].to(dt)
    y = F.linear(F.silu(x) if d["silu_in"] else x, t["w"].to(dt), t["bias"].to(dt) if "bias" in t else None)
    return {"out": F.silu(y) if d["silu_out"] else y}


def time_embed_torch(d, t, dt):
    """the reference's SinusoidalPosEmb (models/estimator.py)"""
    half = d["C"] // 2
    emb = math.log(10000) / (half - 1)
    emb = torch.exp(torch.arange(half, dtype=dt) * -emb)
    emb = 1000 * t["x"].to(dt).unsqueeze(1) * emb.unsqueeze(0)
    return {"out": torch.cat((emb.sin(), emb.cos()), dim=-1)}


def rope_table_torch(d, t, dt):
    """the reference's rotary table (models/diffusion_transformer.py): theta = 1 / base^(2i / d), outer(pos, theta)"""
    theta = 1.0 / (10000 ** (torch.arange(0, 32, 2, dtype=dt) / 32))
    ang = torch.outer(torch.arange(d["T"], dtype=dt), theta)
    return {"out": torch.stack([ang.cos(), ang.sin()], -1)}


def lincomb_torch(d, t, dt):
    acc = torch.zeros_like(t["x"], dtype=dt)
    for j, c in enumerate(d["coef"]):
        acc = acc + torch.tensor(F32(c), dtype=dt) * t["terms"][j].to(dt)
    return {"out": t["x"].to(dt) + acc}


def scaled_sumsq_torch(d, t, dt):
    """the ratios in dt, their squares summed in double"""
    num, tol = _sumsq_num_tol(d, t, dt)
    return {"f64": ((num / tol).double() ** 2).sum().reshape(1)}


def cfg_combine_torch(d, t, dt):
    """models/flow_matching.py: uncond + cfg_strength (cond - uncond)"""
    cond, uncond = t["x"].to(dt).view(-1, d["B"] * d["n"]).unbind(0) if d["cfg"] else (t["x"].to(dt), None)
    return {"out": uncond + F32(d["s_cfg"]) * (cond - uncond) if d["cfg"] else cond}


def cfm_mix_torch(d, t, dt):
    """models/flow_matching.py: y = (1 - (1 - sigma_min) t) z + t x1"""
    tt = t["x2"].to(dt)[:, None, None]
    return {"out": (1 - (1 - torch.tensor(F32(d["sigma_min"]), dtype=dt)) * tt) * t["x1"].to(dt) + tt * t["x"].to(dt)}


def cfm_loss_torch(d, t, dt):
    """models/flow_matching.py: F.mse_loss(v, u, reduction="sum") / (sum(mask) C); the accumulators from dt terms in double"""
    s = torch.tensor(F32(d["sigma_min"]), dtype=dt)
    u = t["x"].to(dt) - (1 - s) * t["x1"].to(dt)
    v, mask = t["x2"].to(dt), t["mask"].to(dt)
    loss = F.mse_loss(v, u, reduction="sum") / (torch.sum(mask) * d["C"])
    return {"out": loss.reshape(1), "f64": torch.stack([((v - u).double() ** 2).sum(), mask.double().sum()])}


TORCH = dict(GLU_RESID=glu_resid_torch, MASKED_MEAN=masked_mean_torch, COND_TRANSPOSE=cond_transpose_torch, RELU_LN=relu_ln_torch,
             RELU_LN_PROJ=relu_ln_torch, GEMV=gemv_torch, TIME_EMBED=time_embed_torch, TIME_EMBED_VALS=time_embed_torch,
             ROPE_TABLE=rope_table_torch, LINCOMB=lincomb_torch, SCALED_SUMSQ=scaled_sumsq_torch, CFG_COMBINE=cfg_combine_torch,
             CFM_MIX=cfm_mix_torch, CFM_LOSS=cfm_loss_torch)


# --------------------------------------------------------------------------------------------------------------------
# cases and their operands
# --------------------------------------------------------------------------------------------------------------------
def make_operands(d, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)                               # noqa: E731
    ru = lambda *s: torch.rand(*s, generator=g) * 2 - 1                       # noqa: E731
    k = d["kind"]
    if k == "GLU_RESID":
        rows, C_ = (d["B"], d["T"]), d["C"]
        x = rn(*rows, 2 * C_)
        if d.get("extremes"):                      # exp(-g) overflows / underflows: sigmoid must still be 0 or 1
            gg = torch.where(torch.rand(*rows, C_, generator=g) < 0.5, -100.0, 100.0)
            gg.view(-1)[0::5] = 88.72
            gg.view(-1)[1::5] = -88.72
            x[..., C_:] = gg
        return {"x": x, "x1": rn(*rows, C_)}
    if k == "MASKED_MEAN":
        B, T, C_ = d["B"], d["T"], d["C"]
        gains = torch.tensor([1.0, 30.0, 0.03])[:B]                             # rows of different scale
        x = (rn(B, T, C_) + d.get("offset", 0.0)) * gains[:, None, None]
        t = {"x": x}
        if d.get("mask", True):
            m = make_mask(B, T, g)
            for b in d.get("empty_rows", ()):
                m[b] = 0.0
            t["mask"] = m
        return t
    if k == "COND_TRANSPOSE":
        B, C_, T = d["B"], d["C"], d["T"]
        return {"x": rn(B, C_, T), "bias": rn(B, C_), "mask": make_mask(B, T, g, d.get("fractional", False))}
    if k in ("RELU_LN", "RELU_LN_PROJ"):
        B, T = d["B"], d["T"]
        x = rn(B, T, LN_C) * d.get("spread", 1.0) + d.get("offset", 0.0)
        if d.get("nonpositive"):                   # every other frame all <= 0 (one exactly 0): relu gives a zero row
            x[:, ::2] = -x[:, ::2].abs()
            x[0, 0] = 0.0
        t = {"x": x, "ln_w": 1 + 0.1 * rn(LN_C), "ln_b": 0.1 * rn(LN_C), "mask": make_mask(B, T, g, d.get("fractional", False))}
        if k == "RELU_LN_PROJ":
            t["w"], t["bias"] = ru(LN_C) / math.sqrt(LN_C), 0.1 * ru(1)
        return t
    if k == "GEMV":
        B, K, N = d["B"], d["K"], d["N"]
        a = d.get("amp")
        x = rn(B, K) if a is None else a * torch.where(torch.rand(B, K, generator=g) < 0.5, -1.0, 1.0)
        t = {"x": x, "w": ru(N, K) * (d.get("w_gain", 1.0) / math.sqrt(K))}
        if d.get("bias", True):
            t["bias"] = 0.5 * rn(N)
        return t
    if k in ("TIME_EMBED", "TIME_EMBED_VALS"):
        tt = torch.rand(d["n_t"], generator=g)
        sp = d.get("special", SPECIAL_T)
        tt[:len(sp)] = torch.tensor(sp[:d["n_t"]])
        return {"x": tt}
    if k == "ROPE_TABLE":
        return {}
    if k == "LINCOMB":
        n = d["n"]
        return {"x": rn(n), "terms": rn(max(1, len(d["coef"])), n) * 3}
    if k == "SCALED_SUMSQ":
        n, nt = d["n"], len(d["coef"])
        if d.get("accumulate"):
            # the first element of every thread's grid-stride walk has ratio 1, every later one a ratio whose square is below
            # half an fp32 ulp of 1: an fp32 running sum drops all of them, the double sum keeps them
            K = torch.full((1, n), math.sqrt(0.45 * 2.0 ** -23))
            K[0, :GRID_ELEMS] = 1.0
            return {"x": torch.zeros(n), "x1": torch.zeros(n), "terms": K}
        # |u|, |v| spread over 1e-4.5 .. 1e3.5: atol (1e-5) dominates the tolerance in some elements, rtol |u| or rtol |v|
        # in others
        u = rn(n) * 10.0 ** (ru(n) * 4 - 0.5)
        v = u + rn(n) * 10.0 ** (ru(n) * 4 - 0.5)
        return {"x": u, "x1": v, "terms": rn(nt, n) * 10.0 ** (ru(nt, n) - 4)}
    if k == "CFG_COMBINE":
        return {"x": rn((2 if d["cfg"] else 1) * d["B"] * d["n"])}
    if k in ("CFM_MIX", "CFM_LOSS"):
        B, C_, T = d["B"], d["C"], d["T"]
        t = {"x": rn(B, C_, T), "x1": rn(B, C_, T)}                   # padded frames carry values too
        if k == "CFM_MIX":
            tt = torch.rand(B, generator=g)
            tt[:len(d.get("times", ()))] = torch.tensor(d.get("times", ())[:B])
            t["x2"] = tt
        else:
            t["x2"] = rn(B, C_, T)
            t["mask"] = make_mask(B, T, g, d.get("fractional", False))
        return t
    raise KeyError(k)


def _cases():
    cs = {}

    def add(name, kind, group, **kw):
        d = dict(kind=kind, group=group, planes=None)
        d.update(kw)
        cs[name] = d

    # GLU_RESID: C = 128 (the style encoder's width), exp overflow, one frame
    add("glu_b2_t37", "GLU_RESID", "shapes", B=2, T=37, C=128, planes="split")
    add("glu_t1", "GLU_RESID", "shapes", B=1, T=1, C=128)
    add("glu_t1000", "GLU_RESID", "shapes", B=1, T=1000, C=128, planes="split")
    add("glu_c2", "GLU_RESID", "shapes", B=3, T=5, C=2)
    add("glu_g_pm100", "GLU_RESID", "extremes", B=2, T=37, C=128, extremes=True, planes="split")
    # MASKED_MEAN: T around the 8 interleaved partials and long, holes, NULL mask, a row with no valid frame, ragged scale
    for T in (1, 7, 8, 9, 700, 3000):
        add(f"mean_b3_t{T}", "MASKED_MEAN", "lengths", B=3, T=T, C=128)
        add(f"mean_b3_t{T}_nomask", "MASKED_MEAN", "lengths", B=3, T=T, C=128, mask=False)
    add("mean_b3_t3000_offset", "MASKED_MEAN", "offset", B=3, T=3000, C=128, offset=4.0)
    add("mean_b3_t700_offset_nomask", "MASKED_MEAN", "offset", B=3, T=700, C=128, offset=-4.0, mask=False)
    add("mean_b3_t37_empty_row", "MASKED_MEAN", "empty", B=3, T=37, C=128, empty_rows=(1,))
    add("mean_b1_t9_empty", "MASKED_MEAN", "empty", B=1, T=9, C=128, empty_rows=(0,))
    add("mean_b2_t100_c40", "MASKED_MEAN", "widths", B=2, T=100, C=40)
    add("mean_b3_t33_c1", "MASKED_MEAN", "widths", B=3, T=33, C=1)
    # COND_TRANSPOSE: T and C off the 32-tiles, the product's C = 256, T = 1
    add("condT_c256_t37", "COND_TRANSPOSE", "tiles", B=3, C=256, T=37, planes="split")
    add("condT_c256_t1", "COND_TRANSPOSE", "tiles", B=2, C=256, T=1, planes="split")
    add("condT_c40_t33", "COND_TRANSPOSE", "tiles", B=3, C=40, T=33, fractional=True)
    add("condT_c256_t700", "COND_TRANSPOSE", "tiles", B=1, C=256, T=700)
    # RELU_LN and RELU_LN_PROJ: zero rows after relu, offset rows, variance ~ eps, fractional / zero / negative masks,
    # odd row counts, T = 1
    for kind, pre in (("RELU_LN", "relu_ln"), ("RELU_LN_PROJ", "relu_proj")):
        pl = "split" if kind == "RELU_LN" else None
        add(f"{pre}_b3_t37_fractional", kind, "masks", B=3, T=37, C=LN_C, fractional=True, planes=pl)
        add(f"{pre}_t1", kind, "shapes", B=1, T=1, C=LN_C, planes=pl)
        add(f"{pre}_b1_t7", kind, "shapes", B=1, T=7, C=LN_C)
        add(f"{pre}_b2_t700", kind, "shapes", B=2, T=700, C=LN_C, fractional=True)
        add(f"{pre}_nonpositive_rows", kind, "values", B=3, T=37, C=LN_C, nonpositive=True, fractional=True, planes=pl)
        add(f"{pre}_offset100", kind, "values", B=2, T=37, C=LN_C, offset=100.0, fractional=True)
        add(f"{pre}_var_near_eps", kind, "eps", B=2, T=37, C=LN_C, spread=3e-3, fractional=True, planes=pl)
        add(f"{pre}_var_near_eps_offset", kind, "eps", B=1, T=9, C=LN_C, spread=1e-3, offset=1.0)
    # GEMV: K from 1 to 1024, each activation combination, strided rows, N up to the adaLN width 6 x 6 x 256, +-100 inputs
    for K in (1, 31, 80, 256, 1024):
        for si in (0, 1):
            for so in (0, 1):
                add(f"gemv_k{K}_in{si}_out{so}", "GEMV", "K", B=3, K=K, N=37, y_rstride=45, silu_in=si, silu_out=so)
    add("gemv_ada_n9216", "GEMV", "wide", B=3, K=256, N=9216, y_rstride=9216, silu_in=1, silu_out=0)
    add("gemv_ada_layer_stride", "GEMV", "wide", B=2, K=256, N=1536, y_rstride=9216, silu_in=1, silu_out=0)
    add("gemv_tmlp_k1024", "GEMV", "wide", B=5, K=1024, N=256, y_rstride=256, silu_in=0, silu_out=0)
    add("gemv_nobias", "GEMV", "wide", B=2, K=128, N=256, y_rstride=300, silu_in=0, silu_out=1, bias=False)
    for si, so in ((0, 0), (1, 0), (0, 1), (1, 1)):
        add(f"gemv_pm100_in{si}_out{so}", "GEMV", "pm100", B=2, K=1024, N=64, y_rstride=70, silu_in=si, silu_out=so, amp=100.0)
    add("gemv_pm100_outputs", "GEMV", "pm100", B=2, K=256, N=64, y_rstride=64, silu_in=0, silu_out=1, amp=100.0, w_gain=8.0)
    # TIME_EMBED (device times) and TIME_EMBED_VALS (host times in the kernel's arguments): t = 0, 1e-7, 0.5, 1 - 2^-24, 1
    for kind, pre in (("TIME_EMBED", "temb"), ("TIME_EMBED_VALS", "tembv")):
        add(f"{pre}_special", kind, "times", n_t=5, C=256)
        add(f"{pre}_n256", kind, "times", n_t=256, C=256)
        for i, tv in enumerate(SPECIAL_T):
            add(f"{pre}_n1_t{i}", kind, "n1", n_t=1, C=256, special=(tv,))
        add(f"{pre}_c4", kind, "widths", n_t=5, C=4)
    add("temb_n1000", "TIME_EMBED", "times", n_t=1000, C=256)
    # ROPE_TABLE
    for T in (1, 37, 1000, 4096):
        add(f"rope_t{T}", "ROPE_TABLE", "lengths", T=T, C=32)
    # LINCOMB: n = 0 .. 6, zero coefficients, dst aliasing y (the solver's y += dt sum b_j K_j)
    dp_b = [35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84]
    for n_ in range(7):
        add(f"lincomb_n{n_}", "LINCOMB", "terms", n=10007, coef=[0.013 * (j + 1) * (-1) ** j for j in range(n_)])
    add("lincomb_zero_coefs_alias", "LINCOMB", "alias", n=3 * 80 * 1000, coef=[0.02 * c for c in dp_b], alias="out")
    add("lincomb_n2_alias", "LINCOMB", "alias", n=4097, coef=[0.5, -0.25], alias="out")
    add("lincomb_n0_alias", "LINCOMB", "alias", n=33, coef=[], alias="out")
    # SCALED_SUMSQ: n = 1 .. 7 on the grid-stride path, u != v, atol / rtol dominating in turn, one element, fp32 rounding of
    # a running sum
    cerr = [71 / 57600, 0.0, -71 / 16695, 71 / 1920, -17253 / 339200, 22 / 525, -1 / 40]
    for n_ in range(1, 8):
        add(f"sumsq_n{n_}", "SCALED_SUMSQ", "terms", n=3 * GRID_ELEMS + 17, coef=[0.05 * c + 0.01 * (j + 1) for j, c in enumerate(cerr[:n_])],
            atol=1e-5, rtol=1e-5)
    add("sumsq_numel1_n1", "SCALED_SUMSQ", "numel1", n=1, coef=[1.0], atol=1e-5, rtol=1e-5)
    add("sumsq_numel1_n7", "SCALED_SUMSQ", "numel1", n=1, coef=[0.05 * c for c in cerr], atol=1e-5, rtol=1e-5)
    add("sumsq_small_n3", "SCALED_SUMSQ", "numel1", n=300, coef=[1.0, -1.0, 0.5], atol=1e-4, rtol=1e-3)
    add("sumsq_accumulate", "SCALED_SUMSQ", "accumulate", n=32 * GRID_ELEMS, coef=[1.0], atol=1.0, rtol=0.0,
        accumulate=True)
    # CFG_COMBINE
    for B in (1, 3):
        add(f"cfg_off_b{B}", "CFG_COMBINE", "cfg", B=B, n=80 * 37, cfg=0, s_cfg=3.0)
        for s_ in (0.0, 0.7, 3.0):
            add(f"cfg_b{B}_s{s_}", "CFG_COMBINE", "cfg", B=B, n=80 * 37, cfg=1, s_cfg=s_)
    # CFM_MIX and CFM_LOSS: ragged (and fractional) masks, padded frames with values, B = 1 and 3, the grid-stride path
    add("mix_b1", "CFM_MIX", "mix", B=1, C=80, T=37, sigma_min=1e-4)
    add("mix_b3_edges", "CFM_MIX", "mix", B=3, C=80, T=37, sigma_min=1e-4, times=(0.0, 1.0, 0.3))
    add("mix_b3_t1000", "CFM_MIX", "mix", B=3, C=80, T=1000, sigma_min=1e-4)
    add("loss_b1", "CFM_LOSS", "loss", B=1, C=80, T=37, sigma_min=1e-4)
    add("loss_b3_ragged", "CFM_LOSS", "loss", B=3, C=80, T=37, sigma_min=1e-4)
    add("loss_b3_fractional", "CFM_LOSS", "loss", B=3, C=80, T=37, sigma_min=1e-4, fractional=True)
    add("loss_b3_t1000_ragged", "CFM_LOSS", "loss", B=3, C=80, T=1000, sigma_min=1e-4)
    add("loss_b3_t2000_mel128", "CFM_LOSS", "loss", B=3, C=128, T=2000, sigma_min=1e-4)
    return cs


CASES = _cases()


def reference(d, t):
    """(fp64 statement, torch fp32) of case d on operands t"""
    return STATEMENTS[d["kind"]](d, t), TORCH[d["kind"]](d, t, torch.float32)


# --------------------------------------------------------------------------------------------------------------------
# CPU: every fp64 statement against independent torch code
# --------------------------------------------------------------------------------------------------------------------
def _close(a, b, tol=1e-10):
    a, b = a.double(), b.double()
    assert torch.equal(torch.isnan(a), torch.isnan(b))
    ok = ~torch.isnan(a)
    assert torch.allclose(a[ok], b[ok], rtol=tol, atol=tol), float((a[ok] - b[ok]).abs().max())


CPU_CASES = ["glu_b2_t37", "glu_g_pm100", "mean_b3_t9", "mean_b3_t37_empty_row", "mean_b3_t700_offset_nomask", "condT_c40_t33",
             "relu_ln_b3_t37_fractional", "relu_ln_nonpositive_rows", "relu_proj_b3_t37_fractional", "relu_proj_var_near_eps",
             "gemv_k31_in1_out1", "gemv_k1_in0_out0", "gemv_nobias", "gemv_pm100_in1_out1", "temb_special", "tembv_c4",
             "rope_t1000", "lincomb_n0", "lincomb_n6", "sumsq_n7", "sumsq_numel1_n7", "cfg_b3_s0.7", "cfg_off_b1", "mix_b3_edges",
             "loss_b3_fractional"]


@pytest.mark.parametrize("name", CPU_CASES)
def test_statement_matches_torch(name):
    d = CASES[name]
    t = make_operands(d, 1)
    r, w = STATEMENTS[d["kind"]](d, t), TORCH[d["kind"]](d, t, torch.float64)
    for k in r:
        _close(r[k], w[k])


def test_masked_mean_statement_is_nan_exactly_on_empty_rows():
    d = CASES["mean_b3_t37_empty_row"]
    r = masked_mean_ref(d, make_operands(d, 2))["out"]
    assert torch.isnan(r[1]).all() and torch.isfinite(r[[0, 2]]).all()


def test_scaled_sumsq_statement_matches_a_plain_sum_of_squares():
    d = CASES["sumsq_small_n3"]
    t = make_operands(d, 3)
    want = 0.0
    for e in range(d["n"]):
        num = sum(F32(c) * float(t["terms"][j, e]) for j, c in enumerate(d["coef"]))
        tol = F32(d["atol"]) + F32(d["rtol"]) * max(abs(float(t["x"][e])), abs(float(t["x1"][e])))
        want += (num / tol) ** 2
    assert math.isclose(float(scaled_sumsq_ref(d, t)["f64"][0]), want, rel_tol=1e-12)


def test_sumsq_tolerances_are_mixed():
    """the u != v operands really switch the tolerance between atol, rtol |u| and rtol |v|"""
    d = CASES["sumsq_n3"]
    t = make_operands(d, 4)
    u, v = t["x"].abs(), t["x1"].abs()
    big = torch.maximum(u, v) * d["rtol"]
    assert (big < d["atol"] / 10).float().mean() > 0.15 and (big > 10 * d["atol"]).float().mean() > 0.15
    assert (v > u).float().mean() > 0.2 and (u > v).float().mean() > 0.2


def test_time_embedding_is_the_reference_layout():
    """[sin | cos] halves, and at t = 0 exactly (0 | 1)"""
    d = CASES["temb_special"]
    r = time_embed_ref(d, make_operands(d, 5))["out"]
    assert torch.equal(r[0], torch.cat([torch.zeros(128), torch.ones(128)]).double())


def test_kind_numbers_match_the_binding():
    """the binding's st_test_row_desc.kind and st_test_gemm_plan.mode names, and test_gemm_contract's epilogue flags, are
    the enums of include/stabletts_b200.h"""
    from stabletts_b200 import _lib
    from test_gemm_contract import EPI
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "stabletts_b200.h")).read()
    enum = lambda prefix: {k: int(v) for k, v in re.findall(rf"\b{prefix}(\w+)\s*=\s*(\d+)", header)}   # noqa: E731
    for names, prefix in ((_lib.ST_TEST_ROW_KINDS, "ST_TEST_ROW_"), (_lib.ST_TEST_MODE_NAMES, "ST_TEST_MODE_")):
        assert enum(prefix) == {k: i for i, k in enumerate(names)}, prefix
    epi = enum("ST_TEST_EPI_")
    assert {k: epi.get(k) for k in EPI} == EPI


# --------------------------------------------------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------------------------------------------------
def check_case(d, t, o):
    """value checks against the fp64 statement; returns [(output, max |err|, bar)]"""
    ref, f32 = reference(d, t)
    rows = []
    for what in ("out", "f64"):
        if what not in ref:
            continue
        r = ref[what]
        got = o[what].double().reshape(r.shape) if what == "out" and d["kind"] != "GEMV" else o[what].double()
        if d["kind"] == "GEMV":                   # row r at r y_rstride: the columns past N are not written
            assert torch.isnan(got[:, d["N"]:]).all()
            got = got[:, :d["N"]]
        nan = torch.isnan(r)
        assert torch.equal(torch.isnan(got), nan), what         # NaN exactly where the statement is 0 / 0
        assert torch.isfinite(got[~nan]).all(), what
        if (~nan).any():
            e32 = float((f32[what].double() - r)[~nan].abs().max())
            err = float((got - r)[~nan].abs().max())
            b = bar(r[~nan], e32)
            rows.append((what, err, b))
            assert err <= b, (what, err, b, e32)
    if d.get("planes"):
        check_planes(o, d["planes"])
    k = d["kind"]
    if k == "RELU_LN":                            # a row that relu zeroes normalises to exactly ln_b, times the mask
        zero = (t["x"] <= 0).all(-1)
        want = (t["ln_b"][None, None, :] * t["mask"][..., None]).expand(*zero.shape, LN_C)
        assert zero.any() == bool(d.get("nonpositive"))
        assert torch.equal(o["out"][zero], want[zero])
    if k == "COND_TRANSPOSE":                     # two fp32 roundings, the same in any correct kernel
        assert torch.equal(o["out"], f32["out"].contiguous())
    if k == "LINCOMB" and not d["coef"]:
        assert torch.equal(o["out"], t["x"])
    if k == "CFG_COMBINE" and (not d["cfg"] or d["s_cfg"] == 0.0):
        n = d["B"] * d["n"]
        assert torch.equal(o["out"], t["x"][n:] if d["cfg"] else t["x"])
    if k in ("TIME_EMBED", "TIME_EMBED_VALS"):
        zero = t["x"] == 0
        half = d["C"] // 2
        assert (o["out"][zero, :half] == 0).all() and (o["out"][zero, half:] == 1).all()
    return rows


@pytest.fixture(scope="module")
def matrix(dev, handle):
    def run(name):
        d = CASES[name]
        t = make_operands(d, 2000 + list(CASES).index(name))
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


# ---- properties that need no tolerance -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mean_b3_t3000", "mean_b3_t9_nomask", "relu_proj_b2_t700", "glu_t1000", "sumsq_n7", "loss_b3_t1000_ragged"])
def test_repeated_runs_are_bit_identical(name, dev, handle):
    """fixed summation orders: the pool, logw and the GEMV rows do not depend on scheduling.  The norm and the loss add
    up to 592 per-block double partials by atomics, in any order: those agree to the rounding of such a sum (1e-13)."""
    lib, h = handle
    d = CASES[name]
    t = make_operands(d, 77)
    first, again = run_ok(run_row_hook, lib, h, d, t, dev), run_ok(run_row_hook, lib, h, d, t, dev)
    for k in first:
        if k == "f64":
            assert torch.allclose(first[k], again[k], rtol=1e-13, atol=0), k
        elif k == "out" and d["kind"] == "CFM_LOSS":
            assert abs(float(first[k][0]) - float(again[k][0])) <= 1.2e-7 * abs(float(first[k][0])), k
        else:
            assert torch.equal(bits(first[k]), bits(again[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mean_b3_t700", "mean_b3_t3000_offset", "relu_proj_b3_t37_fractional", "relu_ln_b2_t700",
                                  "condT_c256_t37", "glu_b2_t37"])
def test_utterance_alone_equals_its_batch_row(name, dev, handle):
    """utterance 1 of a batch, run alone, gives the bits of its batch row (what lets a batched synthesis equal the
    utterance-by-utterance one)"""
    lib, h = handle
    d = CASES[name]
    t = make_operands(d, 78)
    whole = run_ok(run_row_hook, lib, h, d, t, dev)
    batched = ("x", "x1", "mask") + (("bias",) if d["kind"] == "COND_TRANSPOSE" else ())      # bias: cond (B, C)
    t1 = {k: (v[1:2].contiguous() if k in batched else v) for k, v in t.items()}
    one = run_ok(run_row_hook, lib, h, dict(d, B=1), t1, dev)
    assert torch.equal(bits(one["out"][0]), bits(whole["out"][1]))


@pytest.mark.gpu
def test_masked_frames_do_not_reach_the_pool(dev, handle):
    """+-1e6 at the frames with mask 0 leaves the masked mean bit-identical"""
    lib, h = handle
    d = CASES["mean_b3_t700"]
    t = make_operands(d, 80)
    clean = run_ok(run_row_hook, lib, h, d, t, dev)
    dirty = dict(t, x=t["x"].clone())
    m = t["mask"] == 0
    dirty["x"][m] = 1e6
    assert torch.equal(bits(clean["out"]), bits(run_ok(run_row_hook, lib, h, d, dirty, dev)["out"]))


@pytest.mark.gpu
def test_time_embeddings_from_host_and_device_times_agree(dev, handle):
    """the two launchers run the same arithmetic: bit-identical embeddings of the same 256 times"""
    lib, h = handle
    a, b = CASES["temb_n256"], CASES["tembv_n256"]
    t = make_operands(a, 81)
    assert torch.equal(bits(run_ok(run_row_hook, lib, h, a, t, dev)["out"]), bits(run_ok(run_row_hook, lib, h, b, t, dev)["out"]))


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

    refused("glu_b2_t37", "C must be even", C=127)
    refused("glu_b2_t37", "required", x1=None)
    refused("glu_b2_t37", "out_hi and out_lo go together", out_lo=None)
    refused("mean_b3_t9", "C must be in [1, 128]", C=129)
    refused("mean_b3_t9", "C must be in [1, 128]", C=0)
    refused("mean_b3_t9", "writes out_f32 only", planes="split")
    refused("mean_b3_t9", "B, T >= 1", T=0)
    refused("condT_c256_t37", "required", bias=None)
    refused("condT_c256_t37", "required", mask=None)
    refused("relu_ln_t1", "C must be 1024", C=512)
    refused("relu_ln_t1", "required", mask=None)
    refused("relu_proj_t1", "w (proj weight) and bias (proj bias) are required", w=None)
    refused("relu_proj_t1", "writes out_f32 (logw) only", planes="split")
    refused("gemv_k31_in0_out0", "y_rstride must be >= N", y_rstride=36)
    refused("gemv_k31_in0_out0", "B, K, N >= 1", K=0)
    refused("gemv_k31_in0_out0", "silu_in and silu_out are 0 or 1", silu_in=2)
    refused("gemv_k31_in0_out0", "required", w=None)
    refused("temb_special", "n_t >= 1", n_t=0)
    refused("temb_special", "C must be even and >= 4", C=255)
    refused("tembv_special", "C must be even and >= 4", C=2)
    refused("tembv_special", "required", t_host=None)
    refused("rope_t37", "C must be 32", C=64)
    refused("lincomb_n2_alias", "n_terms in [0, 6]", n_terms=7)
    refused("sumsq_n1", "n_terms in [1, 7]", n_terms=0)
    refused("sumsq_n1", "atol > 0 and rtol >= 0", atol=0.0)
    refused("sumsq_n1", "SCALED_SUMSQ out_f64 only", out_f64=None)
    refused("sumsq_n1", "x (u) and x1 (v) are required", x1=None)
    refused("cfg_b1_s0.7", "cfg is 0 or 1", cfg=2)
    refused("mix_b1", "required", x2=None)
    refused("loss_b1", "and mask", mask=None)
    refused("loss_b1", "CFM_LOSS out_f32 and out_f64", out_f64=None)
    from stabletts_b200 import _lib
    refused("glu_b2_t37", "unknown kind", kind=len(_lib.ST_TEST_ROW_KINDS))


@pytest.mark.gpu
def test_refusals_of_pointer_and_count_edges(dev, handle):
    """a misaligned buffer, a missing term, and launch_time_embed_vals' own bound: n_t = 257 does not fit the 256 times its
    kernel argument holds (refused by the launcher, so nothing is launched)"""
    lib, h = handle
    d = CASES["glu_b2_t37"]
    t = make_operands(d, 91)
    x = t["x"].to(dev)
    rc, err, o = run_row_hook(lib, h, d, t, dev, desc_edit=set_fields(x=x.data_ptr() + 4))
    assert rc != 0 and "8-byte aligned" in err, err
    d = CASES["lincomb_n6"]
    rc, err, o = run_row_hook(lib, h, d, make_operands(d, 92), dev, desc_edit=lambda desc: desc.terms.__setitem__(3, None))
    assert rc != 0 and "terms[0 .. n_terms) are required" in err, err
    assert torch.isnan(o["out"]).all()
    for n_t in (257, 1000):
        d = dict(CASES["tembv_n256"], n_t=n_t)
        rc, err, o = run_row_hook(lib, h, d, make_operands(d, 93), dev)
        assert rc != 0 and "invalid argument" in err, (n_t, err)
        assert torch.isnan(o["out"]).all()
    d = CASES["tembv_n256"]
    rc, err, o = run_row_hook(lib, h, d, make_operands(d, 93), dev, desc_edit=lambda desc: setattr(desc, "n_t", 0))
    assert rc != 0 and "invalid argument" in err, err


# --------------------------------------------------------------------------------------------------------------------
# fixed-grid solves deep enough to cross the time-embedding chunk (256 evaluations) and refill the FiLM table (1024)
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_deep_dopri5_solve_crosses_the_time_table_edges(dev):
    """180 fixed Dormand-Prince steps = 1080 estimator evaluations.  Evaluation 256 (the second 256-time embedding chunk) is
    stage 4 of step 42 and evaluation 1024 (the FiLM table refilled for evaluations 1024 ..) is stage 4 of step 170, both
    mid-step.  B = 1 and a short utterance on the damped vector field of test_adaptive; against the oracle at the cfg2 bar.
    The first call runs directly, the second captures the solve into a CUDA graph and replays it: bit-identical."""
    from stabletts_b200 import CFMDecoder
    steps = 180
    assert 6 * steps > 1024 and (256 // 6, 256 % 6) == (42, 4) and (1024 // 6, 1024 % 6) == (170, 4)
    st = weights.make_state(cases.WEIGHT_SEED, 80)
    for k in list(st):
        if k.startswith("final_proj"):
            st[k] = st[k] * 0.05
    m = CFMDecoder(80, 80, 256, 80, 1024, 4, 6, 3, 0.1, 256).eval()
    m.estimator.load_state_dict(st, strict=True)
    m = m.to(dev)
    inp = weights.make_inputs(211, [20], 20, 80)
    args = [inp[k].to(dev) for k in ("mu", "mask", "c", "x")]
    solve = lambda: m(args[0], args[1], steps, 1.0, args[2], "dopri5_fixed", None, z=args[3]).cpu()   # noqa: E731
    direct, replayed = solve(), solve()
    assert torch.equal(direct, replayed)
    with torch.inference_mode():
        ref = R.cfm_forward(st, inp["mu"], inp["mask"], steps, inp["x"], inp["c"], "dopri5_fixed", None)
    e = rel_errs(direct, ref)
    print(f"dopri5_fixed x {steps} (1080 evaluations): rel errs {e[0]:.2e} / {e[1]:.2e}")
    assert max(e) < 1e-3, e
    assert torch.isfinite(direct).all()
