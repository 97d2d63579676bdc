"""The masked multi-head attention contract (AttnArgs, stabletts_b200/csrc/common.cuh) against an fp64 restatement of it.

`attention_contract_ref` states what each engine must compute from exactly the operands it takes: the wgmma engine a base-2
softmax on split-bf16 planes that are already RoPE'd and q-scaled, the SIMT engine partial RoPE + 1/8 + a natural-exp softmax
on fp32 projections.  Both share the mask rules: row bb uses mask row b = bb % B, key j counts only if j < kvlen[b] and
mask[b, j] != 0, and a row with mask == 0 is written as zero.  The CPU tests pin that reference against the reference model's
own formulations (F.scaled_dot_product_attention with the additive -finfo.max mask of models/diffusion_transformer.py, and the
key_padding_mask of nn.MultiheadAttention in models/reference_encoder.py).  The GPU tests drive both engines through
st_test_attention_ex at the three call sites' shapes (CFM estimator with CFG rows, TextEncoder, MelStyleEncoder), around the
64-key block and the 128-query tile, at long T, with masks that have holes, fractional and -0.0 values, and with logit
distributions where online softmax goes wrong; and check the properties that need no tolerance."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_errs
from kernel_harness import LazyMatrix, bits, check_planes, run_ok, set_fields, split_bf16
from kernel_harness import dev, handles  # noqa: F401 (fixtures)

QSCALE = float(np.float32(0.125 * 1.4426950408889634))     # softmax scale folded into q: 1/8 * log2(e), fp32
ENGINES = ("tc", "simt")
# max-rel and l2-rel bars against fp64.  Worst measured on an H100 80GB HBM3 (700 W limit) over this matrix (pytest -s prints
# the table per engine and case group): wgmma 2.6e-5 (logits_peaked_style; every other group <= 1.5e-5), SIMT 2.5e-6.  The
# wgmma worst is the lo·lo product of S that the split-bf16 x3 MMA drops: q x 8 spreads the base-2 logits over +-61, so the
# dropped term (~2^-18 |q_d k_d| per product) moves them by ~1e-4, and a peaked softmax follows few keys, so it does not
# average out.  The fp64 reference with only that term dropped is 2.63e-5 from the full one; P's split-bf16 rounding and the
# dropped pl·vl term alone give 2.5e-6.
TOL = {"tc": 5e-5, "simt": 2e-5}
PLANE_Q = 2.0 ** -16                                        # + the rounding step of the split-bf16 output planes


# --------------------------------------------------------------------------------------------------------------------
# the fp64 reference of the contract
# --------------------------------------------------------------------------------------------------------------------
def rope_table(T, device="cpu"):
    """restates rope_table_kernel (elementwise.cu): fp32 theta_j = 1 / 10000^(2j / 32) and fp32 angle t * theta_j; cos / sin
    evaluated in double and rounded to fp32.  Returns (cos, sin), each (T, 16) in float64.  Always evaluated on the CPU, so
    the planes the test hands the kernel and the reference's operands come from one table."""
    theta = 1.0 / (10000.0 ** (torch.arange(0, 32, 2).float() / 32))
    ang = (torch.arange(T).float()[:, None] * theta[None, :]).double()
    return ang.cos().float().double().to(device), ang.sin().float().double().to(device)


def rope_apply(x, H, cs):
    """partial RoPE of every 64-wide head of q and k (columns < 2H): pairs (j, j + 16), j < 16, by the frame index"""
    cos, sin = cs
    y = x.clone()
    for h0 in range(0, 2 * H, 64):
        x1, x2 = x[..., h0:h0 + 16], x[..., h0 + 16:h0 + 32]
        y[..., h0:h0 + 16] = x1 * cos - x2 * sin
        y[..., h0 + 16:h0 + 32] = x2 * cos + x1 * sin
    return y


def mask_lengths(mask):
    """kvlen = 1 + the last index with mask != 0 (0 if none), prefix = the first index with mask == 0 (T if none)"""
    B, T = mask.shape
    nz = mask != 0
    t = torch.arange(T, device=mask.device)
    kvlen = torch.where(nz, t + 1, torch.zeros_like(t)).amax(1)
    prefix = torch.where(~nz, t, torch.full_like(t, T)).amin(1)
    return kvlen, prefix


def attention_contract_ref(engine, mask, BB, H, qkv=None, hi=None, lo=None, rope=False):
    """fp64 statement of AttnArgs.  engine "tc": operands hi + lo, base-2 softmax, no RoPE, no scale; "simt": fp32 qkv,
    [RoPE with the restated table], q * 1/8, natural exp.  mask (B, T); row bb uses mask row bb % B.  Returns (BB, T, H)."""
    if engine == "tc":
        x = hi.double() + lo.double()
    else:
        x = qkv.double()
        if rope:
            x = rope_apply(x, H, rope_table(x.shape[1], x.device))
        x = torch.cat([x[..., :H] * 0.125, x[..., H:]], -1)
    B, T = mask.shape
    nh = H // 64
    m = mask.double()[torch.arange(BB, device=mask.device) % B]                     # (BB, T)
    kvlen, _ = mask_lengths(m)
    key_ok = (m != 0) & (torch.arange(T, device=m.device)[None, :] < kvlen[:, None])
    heads = lambda z: z.reshape(BB, T, nh, 64).transpose(1, 2)                      # noqa: E731
    q, k, v = heads(x[..., :H]), heads(x[..., H:2 * H]), heads(x[..., 2 * H:])
    s = q @ k.transpose(-1, -2)
    if engine == "tc":
        s = s * math.log(2.0)                                                       # 2^s = e^(s ln 2)
    s = s.masked_fill(~key_ok[:, None, None, :], -math.inf)
    p = torch.softmax(s, -1).nan_to_num(0.0)                                        # rows without a valid key: no keys
    o = (p @ v).transpose(1, 2).reshape(BB, T, H)
    return torch.where((m != 0)[..., None], o, torch.zeros_like(o))


def plane_source(qkv, H, rope):
    """the fp32 values the producer GEMM writes as planes: fp32(rope(qkv) * QSCALE on q) (EPI_ROPE, the estimator and text
    encoder), or fp32(q * QSCALE | k | v) (the style encoder's pre-scaled q rows)"""
    x = qkv.double()
    if rope:
        x = rope_apply(x, H, rope_table(x.shape[1], x.device))
    return torch.cat([x[..., :H] * QSCALE, x[..., H:]], -1).float()


# --------------------------------------------------------------------------------------------------------------------
# CPU: the reference against the reference model's formulations
# --------------------------------------------------------------------------------------------------------------------
def _cpu_mask(B, T):
    m = (torch.arange(T)[None] < torch.tensor([T, T - 9, 0][:B])[:, None]).float()
    m[0, 3:7] = 0.0
    m[0, 11] = 0.5
    m[0, 12] = -0.25
    m[0, 13] = -0.0
    if B > 1:
        m[1, 0] = 0.0
        m[1, 20] = 1e-3
    return m


def _sdpa(q, k, v, mask, scale=None):
    """F.scaled_dot_product_attention in double with models/diffusion_transformer.py's additive query-and-key mask, then
    the zero rows the block's trailing `* x_mask` gives (a fractional mask value is a valid row: zero only where mask == 0)"""
    am = mask[:, None, :, None] * mask[:, None, None, :]
    am = torch.zeros_like(am).masked_fill(am == 0, -torch.finfo(torch.float32).max).double()
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=am, scale=scale)
    BB, nh, T, _ = o.shape
    return o.transpose(1, 2).reshape(BB, T, nh * 64) * (mask != 0).double()[..., None]


@pytest.mark.parametrize("form", ["estimator", "style"])
def test_ref_simt_form_matches_sdpa(form):
    from oracle.estimator_ref import rope_partial
    H, rope = (256, True) if form == "estimator" else (128, False)
    B, BB, T = 2, 4, 37
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(BB, T, 3 * H, generator=g)
    mask = _cpu_mask(B, T)
    got = attention_contract_ref("simt", mask, BB, H, qkv=qkv, rope=rope)
    mb = mask[torch.arange(BB) % B]
    q, k, v = [t.reshape(BB, T, H // 64, 64).transpose(1, 2).double() for t in qkv.split(H, -1)]
    if rope:
        q, k = rope_partial(q, 32), rope_partial(k, 32)
    want = _sdpa(q, k, v, mb)
    assert max(rel_errs(got, want)) < 1e-6             # rope_partial evaluates cos / sin in fp32
    assert (got[mb == 0] == 0).all()


@pytest.mark.parametrize("form", ["estimator", "style"])
def test_ref_wgmma_form_matches_sdpa(form):
    """base 2 on the planes: softmax(ln 2 * q k^T) v"""
    H, rope = (256, True) if form == "estimator" else (128, False)
    B, BB, T = 2, 4, 37
    g = torch.Generator().manual_seed(2)
    hi, lo = split_bf16(plane_source(torch.randn(BB, T, 3 * H, generator=g), H, rope))
    mask = _cpu_mask(B, T)
    got = attention_contract_ref("tc", mask, BB, H, hi=hi, lo=lo)
    x = hi.double() + lo.double()
    q, k, v = [t.reshape(BB, T, H // 64, 64).transpose(1, 2) for t in x.split(H, -1)]
    want = _sdpa(q, k, v, mask[torch.arange(BB) % B], scale=math.log(2.0))
    assert max(rel_errs(got, want)) < 1e-12


def test_ref_no_rope_form_matches_key_padding_mask():
    """models/reference_encoder.py: nn.MultiheadAttention(128, 2) with key_padding_mask = ~x_mask.bool(); identity
    projections, so the attention core sees q, k, v themselves.  Rows with mask == 0 are compared as the contract's zeros."""
    H, B, T = 128, 3, 41
    g = torch.Generator().manual_seed(3)
    qkv = torch.randn(B, T, 3 * H, generator=g)
    mask = _cpu_mask(B, T)
    got = attention_contract_ref("simt", mask, B, H, qkv=qkv, rope=False)
    q, k, v = [t.double().transpose(0, 1) for t in qkv.split(H, -1)]                 # (T, B, H)
    eye, zero = torch.eye(H, dtype=torch.float64), torch.zeros(3 * H, dtype=torch.float64)
    want, _ = F.multi_head_attention_forward(q, k, v, H, 2, None, zero, None, None, False, 0.0, eye, torch.zeros(H, dtype=torch.float64),
                                             training=False, key_padding_mask=~mask.bool(), need_weights=False,
                                             use_separate_proj_weight=True, q_proj_weight=eye, k_proj_weight=eye, v_proj_weight=eye)
    want = want.transpose(0, 1)
    rows = mask != 0
    assert rows[2].sum() == 0                          # the empty utterance: the module gives NaN there, the contract zeros
    assert torch.allclose(got[rows], want[rows], rtol=1e-12, atol=1e-12)
    assert (got[~rows] == 0).all()


@pytest.mark.parametrize("form", ["estimator", "style"])
def test_ref_base2_on_planes_matches_natural_exp_spec(form):
    """the planes the test makes for the wgmma engine state the same attention as the SIMT form of the fp32 operands, to
    within the planes' representation error (hi + lo keeps ~16 mantissa bits, 2^-17 relative)"""
    H, rope = (256, True) if form == "estimator" else (128, False)
    B, BB, T = 2, 2, 300
    g = torch.Generator().manual_seed(4)
    qkv = torch.randn(BB, T, 3 * H, generator=g)
    mask = _cpu_mask(B, T)
    hi, lo = split_bf16(plane_source(qkv, H, rope))
    a = attention_contract_ref("tc", mask, BB, H, hi=hi, lo=lo)
    b = attention_contract_ref("simt", mask, BB, H, qkv=qkv, rope=rope)
    assert max(rel_errs(a, b)) < 2e-5


def test_ref_rope_table_matches_rope_partial():
    """rope_partial rotates the unit vector e_j (j < 16) at frame t into cos(angle_tj) e_j + sin(angle_tj) e_(j+16)"""
    from oracle.estimator_ref import rope_partial
    T = 2500
    cos, sin = rope_table(T)
    e = torch.zeros(16, 1, T, 64, dtype=torch.float64)
    for j in range(16):
        e[j, 0, :, j] = 1.0
    r = rope_partial(e, 32)
    want_cos = torch.stack([r[j, 0, :, j] for j in range(16)], 1)
    want_sin = torch.stack([r[j, 0, :, j + 16] for j in range(16)], 1)
    assert (cos - want_cos).abs().max() < 1e-6 and (sin - want_sin).abs().max() < 1e-6     # cos / sin of one fp32 angle


def test_ref_mask_lengths_and_row_mapping():
    m = torch.tensor([[1.0, 0.0, 0.5, -0.0], [0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 1.0], [-0.25, 1e-3, 1.0, -0.0]])
    kvlen, prefix = mask_lengths(m)
    assert kvlen.tolist() == [3, 0, 4, 3] and prefix.tolist() == [1, 0, 4, 3]
    # row bb uses mask row bb % B: rows 2, 3 of BB = 4 equal rows 0, 1 when their operands do
    g = torch.Generator().manual_seed(5)
    qkv = torch.randn(2, 4, 3 * 128, generator=g)
    o = attention_contract_ref("simt", m[:2], 4, 128, qkv=torch.cat([qkv, qkv]))
    assert torch.equal(o[2:], o[:2]) and (o[1] == 0).all()


# --------------------------------------------------------------------------------------------------------------------
# GPU: the hook
# --------------------------------------------------------------------------------------------------------------------
def case(group, B, T, lens=None, BB=None, form="est", edits=(), dist="normal", engines=ENGINES):
    """one attention problem.  form "est": H = 256, 4 heads, RoPE (CFM estimator and TextEncoder blocks); "sty": H = 128,
    2 heads, no RoPE (MelStyleEncoder).  lens: prefix lengths of the mask rows; edits: (row, start, stop, value) written into
    the mask afterwards; dist: the logit / value distribution (make_qkv).  The estimator form requests the output planes."""
    H = 256 if form == "est" else 128
    return dict(group=group, B=B, BB=BB or B, T=T, lens=list(lens) if lens is not None else [T] * B, form=form, H=H,
                n_heads=H // 64, rope=form == "est", planes=form == "est", edits=tuple(edits), dist=dist, engines=engines)


def make_mask(d):
    m = (torch.arange(d["T"])[None] < torch.tensor(d["lens"])[:, None]).float()
    for b, s, e, v in d["edits"]:
        m[b, s:e] = v
    return m


def make_qkv(d, seed):
    """(BB, T, 3H) fp32.  The shared components go into dim 63 of each head, which RoPE leaves alone:
    peaked (q x 8: logits spread over tens), offset (+100 on every logit: overflows unless the max is subtracted), rising /
    falling (a ramp of 20 over the keys: the running max moves in every block / never after the first), flat (q = 0: the
    mean of V over the valid keys, V ~ 1 + N(0, 0.25)), vmix (V rows and channels over four and two decades)"""
    g = torch.Generator().manual_seed(seed)
    BB, T, H, dist = d["BB"], d["T"], d["H"], d["dist"]
    x = torch.randn(BB, T, 3 * H, generator=g)
    q, k, v = x[..., :H], x[..., H:2 * H], x[..., 2 * H:]
    last = torch.arange(63, H, 64)                                  # dim 63 of every head
    if dist == "peaked":
        q *= 8.0
    elif dist == "offset":
        q[..., last] = 12.5
        k[..., last] = 64.0                                         # 12.5 * 64 / 8 = 100
    elif dist in ("rising", "falling"):
        ramp = (40.0 * torch.arange(T).float() / max(T - 1, 1)).to(torch.bfloat16).float()   # bf16-exact k: no lo plane
        q[..., last] = 4.0
        k[..., last] = (ramp if dist == "rising" else ramp.flip(0))[None, :, None]
    elif dist == "flat":
        q.zero_()
        v.mul_(0.5).add_(1.0)
    elif dist == "vmix":
        v *= 10.0 ** (4.0 * torch.rand(BB, T, 1, generator=g) - 2.0)
        v *= 10.0 ** (2.0 * torch.rand(1, 1, H, generator=g) - 1.0)
    else:
        assert dist == "normal", dist
    return x


def _cases():
    cs = {}

    def add(name, *a, **kw):
        assert name not in cs, name
        cs[name] = case(*a, **kw)

    # the call sites
    add("estimator_cfg_t1000", "call_site", 2, 1000, [1000, 640], BB=4)
    add("text_encoder_t37", "call_site", 3, 37, [37, 1, 20])
    add("style_t700_ones", "call_site", 2, 700, form="sty")
    add("style_t129", "call_site", 2, 129, [129, 77], form="sty")
    add("style_t1", "call_site", 2, 1, [1, 0], form="sty")
    # the shapes of the earlier kernel test
    for i, (lens, T) in enumerate([([300, 211], 300), ([1], 1), ([33, 0, 40], 40), ([129], 129), ([1000, 517], 1000),
                                   ([64, 63, 65], 70)]):
        add(f"old{i}_t{T}", "old_shapes", len(lens), T, lens)
    # T and kvlen around the 64-key block and the 128-query tile
    for T in (1, 2, 63, 64, 65, 127, 128, 129, 192, 193, 300):
        lens = sorted({L for L in (T, T - 1, 64, 65, 128, 129) if 1 <= L <= T}, reverse=True)
        add(f"edge_t{T}", "edges", len(lens), T, lens)
    # 40 key blocks: every ring slot reused 20 times
    add("long_t2500", "long", 1, 2500)
    add("long_t2500_cfg", "long", 1, 2500, [2437], BB=2, edits=((0, 1000, 1030, 0.0),))
    # masks (estimator form; CFG rows where the mapping matters)
    M = dict(B=2, T=300)
    add("mask_hole_first_block", "masks", **M, lens=[300, 260], BB=4, edits=((0, 5, 12, 0.0), (1, 20, 21, 0.0)))
    add("mask_hole_60_70", "masks", **M, lens=[300, 280], edits=((0, 60, 70, 0.0), (1, 60, 70, 0.0)))
    add("mask_hole_key0", "masks", **M, lens=[300, 250], BB=4, edits=((0, 0, 1, 0.0), (1, 0, 3, 0.0)))
    add("mask_hole_at_block", "masks", **M, lens=[300, 300], edits=((0, 128, 140, 0.0), (1, 64, 70, 0.0)))
    add("mask_single_key", "masks", **M, lens=[0, 0], edits=((0, 100, 101, 1.0), (1, 299, 300, 1.0)))
    add("mask_fractional", "masks", **M, lens=[300, 240], BB=4,
        edits=((0, 10, 11, 0.5), (0, 70, 71, 1e-3), (0, 150, 151, -0.25), (1, 3, 4, 0.5), (1, 64, 65, -0.25), (1, 200, 201, 1e-3)))
    add("mask_neg_zero", "masks", **M, lens=[300, 300], edits=((0, 30, 40, -0.0), (1, 64, 65, -0.0), (1, 250, 300, -0.0)))
    add("mask_empty_mid_batch", "masks", 3, 300, [300, 0, 293])
    add("mask_holes_t200", "masks", 2, 200, [200, 150], edits=((0, 37, 49, 0.0), (0, 130, 131, 0.0), (1, 0, 5, 0.0)))
    add("mask_style_holes", "masks", 2, 193, [193, 150], form="sty", edits=((0, 0, 2, 0.0), (0, 60, 70, 0.0), (1, 64, 65, 0.0)))
    # logit / value distributions
    for dist in ("normal", "peaked", "offset", "rising", "falling", "flat", "vmix"):
        add(f"logits_{dist}", "logits", 2, 193, [193, 150], dist=dist, edits=((0, 60, 70, 0.0),))
    for dist in ("peaked", "offset", "rising", "flat"):
        add(f"logits_{dist}_style", "logits", 2, 700, [700, 389], form="sty", dist=dist)
    return cs


CASES = _cases()
RUNS = [(name, e) for name, d in CASES.items() for e in d["engines"]]
GROUPS = ("call_site", "old_shapes", "edges", "long", "masks", "logits")


def run_hook(lib, h, engine, d, qkv, mask, dev, planes=None, lengths=False, desc_edit=None):
    """Runs problem d through st_test_attention_ex; returns (rc, error text, outputs).  The wgmma engine gets the planes the
    producer GEMM would write (plane_source), the SIMT engine the fp32 qkv.  Outputs start as NaN (lengths as -7), so an
    element the kernel never wrote fails every comparison."""
    from stabletts_b200 import _lib
    BB, T, H = d["BB"], d["T"], d["H"]
    want_planes = d["planes"] if planes is None else planes
    full = lambda dtype: torch.full((BB, T, H), float("nan"), device=dev, dtype=dtype)   # noqa: E731
    o = {"out": full(torch.float32)}
    if want_planes:
        o["hi"], o["lo"] = full(torch.bfloat16), full(torch.bfloat16)
    if lengths:
        o["kvlen"] = torch.full((d["B"],), -7, dtype=torch.int32, device=dev)
        o["prefix"] = torch.full((d["B"],), -7, dtype=torch.int32, device=dev)
    keep = {"mask": mask.to(dev).contiguous()}
    if engine == "tc":
        hi, lo = split_bf16(plane_source(qkv, H, d["rope"]))
        keep["qkv_hi"], keep["qkv_lo"] = hi.to(dev).contiguous(), lo.to(dev).contiguous()
    else:
        keep["qkv"] = qkv.to(dev).contiguous()
    desc = _lib.StTestAttnDesc()
    for k in ("qkv", "qkv_hi", "qkv_lo", "mask"):
        setattr(desc, k, keep[k].data_ptr() if k in keep else None)
    for k, ok in (("out_f32", "out"), ("out_hi", "hi"), ("out_lo", "lo"), ("kvlen_out", "kvlen"), ("prefix_out", "prefix")):
        setattr(desc, k, o[ok].data_ptr() if ok in o else None)
    for k in ("BB", "B", "T", "H", "n_heads"):
        setattr(desc, k, int(d[k]))
    desc.rope = int(d["rope"] and engine == "simt")
    if desc_edit:
        desc_edit(desc)
    rc = lib.st_test_attention_ex(h, C.byref(desc), torch.cuda.current_stream().cuda_stream)
    err = lib.st_last_error(h).decode() if rc else ""
    return rc, err, {k: v.cpu() for k, v in o.items()}


def reference(engine, d, qkv, mask, dev):
    """the fp64 reference on the device, from the operands run_hook handed the engine"""
    if engine == "tc":
        hi, lo = split_bf16(plane_source(qkv, d["H"], d["rope"]))
        r = attention_contract_ref("tc", mask.to(dev), d["BB"], d["H"], hi=hi.to(dev), lo=lo.to(dev))
    else:
        r = attention_contract_ref("simt", mask.to(dev), d["BB"], d["H"], qkv=qkv.to(dev), rope=d["rope"])
    return r.cpu()


def zero_rows(d, mask):
    """(BB, T) rows that must be exactly zero: mask == 0, which includes every row at or beyond kvlen"""
    return (mask[torch.arange(d["BB"]) % d["B"]] == 0)


def check_case(d, engine, o, ref, mask):
    """value checks against the fp64 reference; returns [(what, max-rel, l2-rel, bar)]"""
    rows = []

    def cmp(what, got, want, bar):
        e = rel_errs(got, want)
        rows.append((what, e[0], e[1], bar))
        assert e[0] < bar and e[1] < bar, (what, e, bar)

    z = zero_rows(d, mask)
    assert (o["out"][z] == 0).all()                   # == 0: the sign of a masked row is not part of the contract
    cmp("out", o["out"], ref, TOL[engine])
    if "hi" in o:
        check_planes(o, "split")                      # the output planes are the split of out_f32, bit for bit
        cmp("planes", o["hi"].double() + o["lo"].double(), ref, TOL[engine] + PLANE_Q)
    return rows


@pytest.fixture(scope="module")
def matrix(dev, handles):
    """{(name, engine): rows}"""
    lib, hs = handles

    def run(key):
        name, engine = key
        d = CASES[name]
        qkv, mask = make_qkv(d, 2000 + list(CASES).index(name)), make_mask(d)
        o = run_ok(run_hook, lib, hs[engine], engine, d, qkv, mask, dev)
        return check_case(d, engine, o, reference(engine, d, qkv, mask, dev), mask)
    return LazyMatrix(run)


@pytest.mark.gpu
@pytest.mark.parametrize("name,engine", RUNS, ids=[f"{n}-{e}" for n, e in RUNS])
def test_matrix(name, engine, matrix):
    matrix.check((name, engine))


@pytest.mark.gpu
def test_every_group_ran(matrix):
    """and prints the worst measured error per engine and case group (pytest -s)"""
    worst = {}
    for name, engine in RUNS:
        rows = matrix[(name, engine)]
        if isinstance(rows, Exception):
            continue
        w = worst.setdefault((engine, CASES[name]["group"]), {"n": 0, "out": [0.0, 0.0, ""], "planes": [0.0, 0.0, ""]})
        w["n"] += 1
        for what, em, el, bar in rows:
            g = w[what]
            if em > g[0]:
                g[2] = name
            g[0], g[1] = max(g[0], em), max(g[1], el)
    print(f"\n{'engine':6s} {'group':11s} {'cases':>5s} | {'max-rel':>9s} {'l2-rel':>9s} {'bar':>8s} | {'planes':>9s} | worst case")
    for engine in ENGINES:
        for group in GROUPS:
            w = worst.get((engine, group))
            if w:
                f, p = w["out"], w["planes"]
                pl = f"{p[0]:9.2e}" if p[2] else f"{'-':>9s}"
                print(f"{engine:6s} {group:11s} {w['n']:5d} | {f[0]:9.2e} {f[1]:9.2e} {TOL[engine]:8.2e} | {pl} | {f[2]}")
    missing = [(e, g) for e in ENGINES for g in GROUPS if (e, g) not in worst]
    assert not missing, missing
    failed = [k for k in RUNS if isinstance(matrix[k], Exception)]
    assert not failed, failed


# ---- properties that need no tolerance -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_utterance_alone_equals_its_batch_row(engine, dev, handles):
    """an utterance alone (B = 1, T = L) gives the bits of its row in a padded batch with other neighbours"""
    lib, hs = handles
    Tb = 720
    for L in (63, 64, 65, 129, 700):
        batch = case("p", 3, Tb, [Tb, L, 300])
        qkv, mask = make_qkv(batch, L), make_mask(batch)
        whole = run_ok(run_hook, lib, hs[engine], engine, batch, qkv, mask, dev, planes=True)
        alone = case("p", 1, L)
        one = run_ok(run_hook, lib, hs[engine], engine, alone, qkv[1:2, :L].contiguous(), mask[1:2, :L].contiguous(), dev, planes=True)
        assert torch.equal(bits(one["out"][0]), bits(whole["out"][1, :L])), (L, engine)
        assert torch.equal(bits(one["hi"][0]), bits(whole["hi"][1, :L]))
        assert (whole["out"][1, L:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_cfg_rows_do_not_depend_on_the_unconditional_rows(engine, dev, handles):
    lib, hs = handles
    d = case("p", 2, 300, [300, 211], BB=4, edits=((0, 40, 50, 0.0),))
    qkv, mask = make_qkv(d, 11), make_mask(d)
    a = run_ok(run_hook, lib, hs[engine], engine, d, qkv, mask, dev)
    qkv2 = qkv.clone()
    qkv2[2:] = torch.randn(2, 300, 768, generator=torch.Generator().manual_seed(12)) * 3.0
    b = run_ok(run_hook, lib, hs[engine], engine, d, qkv2, mask, dev)
    assert torch.equal(bits(a["out"][:2]), bits(b["out"][:2]))
    assert not torch.equal(a["out"][2:], b["out"][2:])
    assert torch.equal(bits(a["hi"][:2]), bits(b["hi"][:2]))


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("form", ["est", "sty"])
def test_garbage_in_masked_frames_changes_nothing(engine, form, dev, handles):
    """finite garbage up to +-1e6 in q / k / v of masked frames (holes and [kvlen, T)) leaves the valid rows bit-identical
    and the masked rows zero"""
    lib, hs = handles
    d = case("p", 3, 321, [321, 250, 64], form=form, edits=((0, 0, 3, 0.0), (0, 60, 70, 0.0), (1, 128, 140, 0.0), (2, 5, 6, 0.0)))
    qkv, mask = make_qkv(d, 21), make_mask(d)
    clean = run_ok(run_hook, lib, hs[engine], engine, d, qkv, mask, dev, planes=True)
    dirty_qkv = qkv.clone()
    bad = mask == 0
    g = torch.Generator().manual_seed(22)
    junk = (torch.rand(dirty_qkv.shape, generator=g) * 2.0 - 1.0) * 1e6
    dirty_qkv[bad] = junk[bad]
    dirty = run_ok(run_hook, lib, hs[engine], engine, d, dirty_qkv, mask, dev, planes=True)
    assert torch.equal(bits(clean["out"][~bad]), bits(dirty["out"][~bad]))
    assert torch.equal(bits(clean["hi"][~bad]), bits(dirty["hi"][~bad]))
    assert (dirty["out"][bad] == 0).all() and (dirty["hi"][bad].float() == 0).all() and (dirty["lo"][bad].float() == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_repeated_runs_are_bit_identical(engine, dev, handles):
    lib, hs = handles
    d = case("p", 2, 1000, [1000, 517], BB=4, edits=((0, 100, 120, 0.0),))
    qkv, mask = make_qkv(d, 31), make_mask(d)
    first = run_ok(run_hook, lib, hs[engine], engine, d, qkv, mask, dev)
    for _ in range(2):
        again = run_ok(run_hook, lib, hs[engine], engine, d, qkv, mask, dev)
        for k in first:
            assert torch.equal(bits(first[k]), bits(again[k])), k


@pytest.mark.gpu
def test_mask_lengths(dev, handles):
    """kvlen_out / prefix_out are 1 + the last nonzero index and the first zero index"""
    lib, hs = handles
    g = torch.Generator().manual_seed(41)
    masks = {"t1": torch.tensor([[1.0], [0.0], [-0.0], [0.5]])}
    for T in (300, 1000):
        m = torch.ones(8, T)
        m[1] = 0.0                                                    # all zeros
        m[2] = -0.0                                                   # all -0.0
        m[3, 257:] = 0.0                                              # a length past the block stride
        m[4, T - 1] = -0.0
        m[4, 260] = 0.0
        m[5] = (torch.rand(T, generator=g) > 0.5).float() * (torch.rand(T, generator=g) - 0.5)   # fractional, both signs
        m[6, :] = 0.0
        m[6, T - 1] = 1e-3
        m[7, 0] = -0.0
        masks[f"t{T}"] = m
    for name, m in masks.items():
        B, T = m.shape
        d = case("p", B, T)
        o = run_ok(run_hook, lib, hs["simt"], "simt", d, torch.zeros(B, T, 768), m, dev, lengths=True)
        kvlen, prefix = mask_lengths(m)
        assert o["kvlen"].tolist() == kvlen.tolist(), name
        assert o["prefix"].tolist() == prefix.tolist(), name
    assert mask_lengths(masks["t300"])[0].tolist()[:4] == [300, 0, 0, 257]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_refusals(engine, dev, handles):
    """every problem outside the contract is refused with a readable error, and nothing is launched"""
    lib, hs = handles
    d = case("p", 2, 65, [65, 40], BB=4)
    qkv, mask = make_qkv(d, 51), make_mask(d)

    def refused(needle, **kw):
        rc, err, o = run_hook(lib, hs[engine], engine, d, qkv, mask, dev, planes=True, **kw)
        assert rc != 0 and needle in err, (needle, err)
        assert torch.isnan(o["out"]).all() and torch.isnan(o["hi"].float()).all()

    refused("H must be 64 n_heads", desc_edit=set_fields(H=192))
    refused("H must be 64 n_heads", desc_edit=set_fields(n_heads=0, H=0))
    refused("positive multiple of B", desc_edit=set_fields(BB=3))
    refused("positive multiple of B", desc_edit=set_fields(BB=0))
    refused("mask is required", desc_edit=set_fields(mask=None))
    rc, err, _ = run_hook(lib, hs[engine], engine, d, qkv, mask, dev, planes=False, desc_edit=set_fields(out_f32=None))
    assert rc != 0 and "no output requested" in err, err
    refused("out_hi and out_lo go together", desc_edit=set_fields(out_lo=None))
    refused("out_hi and out_lo go together", desc_edit=set_fields(out_hi=None))
    if engine == "tc":
        refused("qkv_hi and qkv_lo", desc_edit=set_fields(qkv_lo=None))
        refused("qkv_hi and qkv_lo", desc_edit=set_fields(qkv_hi=None))
        refused("rope must be 0", desc_edit=set_fields(rope=1))
    else:
        refused("needs the fp32 qkv", desc_edit=set_fields(qkv=None))
