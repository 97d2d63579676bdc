"""The GPU-side harness of the kernel-contract tests (test_gemm_contract, test_attention_contract, test_row_contract,
test_glue_contract), and the `dev` fixture of every GPU test module.

pytest finds a fixture in a test module's namespace, so a module imports the fixtures it uses by name:
    from kernel_harness import dev, handle          # noqa: F401 (fixtures)
`handle` and `handles` need `dev` imported next to them."""
import ctypes as C

import pytest
import torch

NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


# --------------------------------------------------------------------------------------------------------------------
# handles of the test hooks
# --------------------------------------------------------------------------------------------------------------------
def hook_handle(engine=None):
    """(lib, h): a FireflyGAN handle, which is all a test hook needs (the device, and the engine: "tc", "simt" or None for
    the default).  The caller destroys it with lib.st_destroy."""
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    h = C.c_void_p()
    _lib.check(lib, None, lib.st_create_ffgan(0, C.byref(h)), "st_create_ffgan")
    if engine is not None:
        eid = {"tc": _lib.ST_ENGINE_TCGEN05, "simt": _lib.ST_ENGINE_SIMT}[engine]
        _lib.check(lib, h, lib.st_set_engine(h, eid), "st_set_engine")
    return lib, h


@pytest.fixture(scope="module")
def handle(dev):
    """(lib, one handle on the default engine)"""
    lib, h = hook_handle()
    yield lib, h
    lib.st_destroy(h)


@pytest.fixture(scope="module")
def handles(dev):
    """(lib, {"tc": handle on the wgmma engine, "simt": handle on the SIMT engine})"""
    hs = {}
    for engine in ("tc", "simt"):
        lib, hs[engine] = hook_handle(engine)
    yield lib, hs
    for h in hs.values():
        lib.st_destroy(h)


def run_ok(hook, *args, **kw):
    """hook(*args, **kw) on a problem inside the contract: asserts rc == 0 and returns what the hook returns after
    (rc, error text)"""
    rc, err, *rest = hook(*args, **kw)
    assert rc == 0, err
    return rest[0] if len(rest) == 1 else tuple(rest)


def set_fields(**fields):
    """a desc_edit for the drivers: overwrites these descriptor fields after the driver has filled the descriptor in"""
    def edit(desc):
        for k, v in fields.items():
            setattr(desc, k, v)
    return edit


# --------------------------------------------------------------------------------------------------------------------
# the case matrix: each case runs once, on first use, so -k selects what runs
# --------------------------------------------------------------------------------------------------------------------
class LazyMatrix(dict):
    """{key: what run(key) returned | the exception it raised}"""
    def __init__(self, run):
        super().__init__()
        self.run = run

    def __missing__(self, key):
        try:
            res = self.run(key)
        except Exception as e:           # noqa: BLE001 — reported by that case's test
            res = e
        self[key] = res
        return res

    def check(self, key):
        """the body of a case's test: re-raises the exception its run stored"""
        res = self[key]
        if isinstance(res, Exception):
            raise res


# --------------------------------------------------------------------------------------------------------------------
# bits and the 2-byte output planes
# --------------------------------------------------------------------------------------------------------------------
def bits(x):
    """the bit patterns of x: int32 of an fp32 tensor, int16 of a 2-byte one"""
    return x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int16)


def split_bf16(x):
    """the split-bf16 planes of fp32 x: hi = bf16(x), lo = bf16(x - hi)"""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def fp16_plane(x):
    """the fp16 plane of fp32 x: cvt.rn(clamp(x, +-65504))"""
    return x.clamp(-65504.0, 65504.0).half()


def check_planes(o, planes, src=None):
    """the 2-byte planes o["hi"] (and o["lo"]) are the rounding of the fp32 values they stand for (src, by default
    o["out"]), bit for bit: planes "split" is split_bf16, "u16" fp16_plane, None none.  This pins pair order and packing."""
    x = o["out"] if src is None else src
    if planes == "split":
        hi, lo = split_bf16(x)
        assert torch.equal(bits(o["hi"]), bits(hi))
        assert torch.equal(bits(o["lo"]), bits(lo))
    elif planes == "u16":
        assert torch.equal(bits(o["hi"]), bits(fp16_plane(x)))


# --------------------------------------------------------------------------------------------------------------------
# st_test_row_ex (test_row_contract, test_glue_contract)
# --------------------------------------------------------------------------------------------------------------------
def bar(ref64, e32):
    """the row kernels' bar: max(4 E32, 8 ulp of max |ref64|)"""
    return max(4.0 * e32, 8.0 * 2.0 ** -24 * float(ref64.abs().max()))


def make_mask(B, T, g, fractional=False):
    """prefix masks of different lengths with holes (and fractional values: 0.5, 0.747, 1e-3, -0.25)"""
    m = torch.ones(B, T)
    for b in range(B):
        m[b, max(1, T - (b * T) // (B + 1)):] = 0.0
        if T >= 8:
            m[b, (7 * b + 3) % T] = 0.0
            m[b, (3 * b + 5) % T] = 0.0
            if fractional:
                m[b, (5 * b + 1) % T] = 0.5
                m[b, (11 * b + 2) % T] = 0.747
                m[b, (13 * b + 4) % T] = 1e-3
                m[b, (2 * b + 6) % T] = -0.25
    return m


# the fp32 output's shape per kind (None: no fp32 output), and the length of the double output of the kinds that have one
ROW_OUT_SHAPE = dict(
    ADALN=lambda d: (d["BB"], d["T"], d["C"]), DWCONV_LN=lambda d: (d["B"], d["T"], d["C"]),
    SPECTRUM=lambda d: (d["B"], d["T"], d["K2"]), IDFT_BASIS=lambda d: (d["n_fft"], d["K2"]),
    OVERLAP_ADD=lambda d: (d["B"], d["T"] * d["hop"]), MEAN3_SILU=lambda d: (d["n"],), POST_TANH=lambda d: (d["B"], d["T"]),
    GLU_RESID=lambda d: (d["B"], d["T"], d["C"]), MASKED_MEAN=lambda d: (d["B"], d["C"]),
    COND_TRANSPOSE=lambda d: (d["B"], d["T"], d["C"]), RELU_LN=lambda d: (d["B"], d["T"], d["C"]),
    RELU_LN_PROJ=lambda d: (d["B"], d["T"]), GEMV=lambda d: (d["B"], d["y_rstride"]), TIME_EMBED=lambda d: (d["n_t"], d["C"]),
    TIME_EMBED_VALS=lambda d: (d["n_t"], d["C"]), ROPE_TABLE=lambda d: (d["T"], 16, 2), LINCOMB=lambda d: (d["n"],),
    SCALED_SUMSQ=lambda d: None, CFG_COMBINE=lambda d: (d["B"] * d["n"],), CFM_MIX=lambda d: (d["B"], d["C"], d["T"]),
    CFM_LOSS=lambda d: (1,))
ROW_OUT_F64 = dict(SCALED_SUMSQ=1, CFM_LOSS=2)


def run_row_hook(lib, h, d, t, dev, planes=None, desc_edit=None):
    """Runs case d on operands t through st_test_row_ex; returns (rc, error text, outputs).  Outputs start as NaN, so an
    element the kernel never wrote fails every comparison.  d["alias"] names the output that is x itself (ADALN's xout,
    LINCOMB's out); TIME_EMBED_VALS takes its times x from the host.  The descriptor fields d names are copied."""
    from stabletts_b200 import _lib
    k = d["kind"]
    planes = d.get("planes") if planes is None else planes
    shape = ROW_OUT_SHAPE[k](d)
    keep = {n: v.to(dev).contiguous() for n, v in t.items()}
    full = lambda s, dtype=torch.float32: torch.full(s, NAN, device=dev, dtype=dtype)    # noqa: E731
    o = {}
    if shape is not None:
        o["out"] = full(shape)
    if k in ROW_OUT_F64:
        o["f64"] = full((ROW_OUT_F64[k],), torch.float64)
    if planes == "split":
        o["hi"], o["lo"] = full(shape, torch.bfloat16), full(shape, torch.bfloat16)
    elif planes == "u16":
        o["hi"] = full(shape, torch.float16)
    if k == "ADALN" and d["has_film"]:
        o["xout"] = full(shape)
    if d.get("alias"):
        o[d["alias"]] = keep["x"]
    desc = _lib.StTestRowDesc()
    for n in ("x", "x1", "x2", "w", "bias", "ln_w", "ln_b", "film", "shift", "scale", "mask", "window"):
        setattr(desc, n, keep[n].data_ptr() if n in keep else None)
    host_t = None                                 # keeps TIME_EMBED_VALS' host times alive through the call
    if k == "TIME_EMBED_VALS":
        desc.x = None
        host_t = (C.c_float * d["n_t"])(*t["x"].tolist())
        desc.t_host = C.cast(host_t, C.c_void_p)
    for n, on in (("xout", "xout"), ("out_f32", "out"), ("out_hi", "hi"), ("out_lo", "lo"), ("out_f64", "f64")):
        setattr(desc, n, o[on].data_ptr() if on in o else None)
    desc.kind = _lib.ST_TEST_ROW_KINDS.index(k)
    for n in ("B", "BB", "T", "C", "c_clamp", "has_film", "mask_out", "Nh", "Kp", "K", "K2", "n_fft", "hop", "n", "film_bstride",
              "ada_bstride", "N", "y_rstride", "silu_in", "silu_out", "n_t", "cfg"):
        if n in d:
            setattr(desc, n, int(d[n]))
    for n in ("eps", "atol", "rtol", "sigma_min", "s_cfg"):
        if n in d:
            setattr(desc, n, float(d[n]))
    if "coef" in d:
        desc.n_terms = len(d["coef"])
        for j, c in enumerate(d["coef"]):
            desc.terms[j] = keep["terms"][j].data_ptr()
            desc.coef[j] = c
    desc.u16 = int(planes == "u16")
    if desc_edit:
        desc_edit(desc)
    rc = lib.st_test_row_ex(h, C.byref(desc), torch.cuda.current_stream().cuda_stream)
    err = lib.st_last_error(h).decode() if rc else ""
    return rc, err, {n: v.cpu() for n, v in o.items()}


def report_worst_per_group(matrix, cases):
    """prints the worst ratio to the bar per kind and case group (pytest -s) of a matrix of row-hook cases, whose runs
    return [(output, max |err|, bar)]; asserts that every group ran and that no case failed"""
    groups = sorted({(d["kind"], d["group"]) for d in cases.values()})
    worst = {}
    for name, d in cases.items():
        rows = matrix[name]
        if isinstance(rows, Exception):
            continue
        w = worst.setdefault((d["kind"], d["group"]), [0, 0.0, ""])
        w[0] += 1
        for what, err, b in rows:
            if err / b >= w[1]:
                w[1], w[2] = err / b, f"{name} ({what}: {err:.2e} / {b:.2e})"
    kw = max(len(kind) for kind, _ in groups) + 1
    gw = max(len(group) for _, group in groups) + 1
    print(f"\n{'kind':{kw}s} {'group':{gw}s} {'cases':>5s} | {'err/bar':>8s} | worst case")
    for kind, group in groups:
        w = worst.get((kind, group))
        if w:
            print(f"{kind:{kw}s} {group:{gw}s} {w[0]:5d} | {w[1]:8.3f} | {w[2]}")
    missing = [k for k in groups if k not in worst]
    assert not missing, missing
    failed = [n for n in cases if isinstance(matrix[n], Exception)]
    assert not failed, failed
