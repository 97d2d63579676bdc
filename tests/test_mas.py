"""Monotonic alignment search (``stabletts_b200.monotonic_align.maximum_path``) and ``StableTTS.compute_losses``.

CPU: the oracle (oracle/mas_ref.py) against the fixtures of the unmodified reference (tests/golden/mas_*.npz: numba's
``maximum_path``; fwd_*.npz: ``StableTTS.forward`` in eval mode; recipe oracle/make_golden_mas.py), the fixtures' margins,
and the refusals.
GPU: the path bit for bit against the fixtures and against the oracle on a sweep (the trainer's B = 32 at 1000 x 400,
every degenerate length, ties, scales 1e-3 to 1e5, decision bits that overflow shared memory, strided input), batch
independence and CUDA-graph capture; st_mas_scores against fp64; compute_losses against fwd_* on both engines."""
import os

import numpy as np
import pytest
import torch

from kernel_harness import dev  # noqa: F401 (a fixture)
from oracle import mas_ref, synth_ref, weights
from oracle.make_golden_mas import FWD_CASES, MAS_CASES, MARGIN_FACTOR, inject_by_shape, margin

ENGINES = ["tcgen05", "simt"]
DIFF_BAR = {"tcgen05": 1e-3, "simt": 5e-5}         # test_gpu_parity's compute_loss bars
SCORE_ULPS = 16                                     # st_mas_scores: |err| <= 16 * 2^-24 * (Σ_d (y² / 2 + |y mu| + mu² / 2) + |c0|)


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _fwd_inputs(g):
    keys = ("ids", "x_lengths", "y", "y_lengths", "z", "z_lengths")
    return {k: torch.from_numpy(g[k]) for k in keys}


def _draws(g):
    u_cfg, u_t, noise = (torch.from_numpy(g[k]) for k in ("u_cfg", "u_t", "noise"))
    return {("rand",) + tuple(u_cfg.shape): u_cfg, ("rand",) + tuple(u_t.shape): u_t, ("randn",) + tuple(noise.shape): noise}


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


# ------------------------------------------------------------------ CPU ------------------------------------------------------

@pytest.mark.parametrize("name", list(MAS_CASES))
def test_oracle_path_equals_reference_fixture(name, golden_dir):
    g = _golden(golden_dir, name)
    assert np.array_equal(mas_ref.maximum_path(g["neg_cent"], g["mask"]), g["path"].astype(np.int32))


@pytest.mark.parametrize("name", list(FWD_CASES))
def test_oracle_losses_match_forward_fixture(name, golden_dir):
    cs, g = FWD_CASES[name], _golden(golden_dir, name)
    st = synth_ref.make_state(n_mel=cs["n_mel"])
    assert float(g["weight_checksum"]) == pytest.approx(weights.checksum(st), rel=1e-12)
    inp = _fwd_inputs(g)
    (dur, diff, prior, attn), _ = mas_ref.forward_losses(st, inp["ids"], inp["x_lengths"], inp["y"], inp["y_lengths"], inp["z"],
                                                         inp["z_lengths"], torch.from_numpy(g["u_cfg"]), torch.from_numpy(g["u_t"]),
                                                         torch.from_numpy(g["noise"]))
    assert torch.equal(attn.to(torch.uint8), torch.from_numpy(g["attn"]))
    for got, key in ((dur, "dur_loss"), (diff, "diff_loss"), (prior, "prior_loss")):
        assert _rel(got, g[key]) <= 2e-5, (key, got, float(g[key]))


def test_fixture_margins_hold(golden_dir):
    """each fwd_* target has a backtrack gap above MARGIN_FACTOR x t_y x SCORE_BAR x max|neg_cent|, recomputed here from the
    oracle's own encoders (so a GPU mu_x within the bar cannot move the path), and it used both cfg branches"""
    for name, cs in FWD_CASES.items():
        g = _golden(golden_dir, name)
        assert float(g["margin"]) > MARGIN_FACTOR
        st = synth_ref.make_state(n_mel=cs["n_mel"])
        inp = _fwd_inputs(g)
        _, (nc, mask) = mas_ref.forward_losses(st, inp["ids"], inp["x_lengths"], inp["y"], inp["y_lengths"], inp["z"], inp["z_lengths"],
                                               torch.from_numpy(g["u_cfg"]), torch.from_numpy(g["u_t"]), torch.from_numpy(g["noise"]))
        assert margin(nc.numpy(), mask.numpy()) > MARGIN_FACTOR, name
        keep = g["u_cfg"] > 0.2
        assert keep.any() and (~keep).any(), name


def test_refusals():
    from stabletts_b200 import StableTTS, monotonic_align
    with pytest.raises(RuntimeError, match="CUDA"):
        monotonic_align.maximum_path(torch.zeros(1, 4, 3), torch.ones(1, 4, 3))
    with pytest.raises(ValueError):
        monotonic_align.maximum_path(torch.zeros(1, 4, 3), torch.ones(1, 4, 2))
    with pytest.raises(ValueError):
        monotonic_align.maximum_path(torch.zeros(4, 3), torch.ones(4, 3))
    m = StableTTS(401, 80, 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
    args = (torch.zeros(1, 5, dtype=torch.long), torch.tensor([5]), torch.zeros(1, 80, 8), torch.tensor([8]), torch.zeros(1, 80, 8),
            torch.tensor([8]))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.compute_losses(*args)
    with pytest.raises(NotImplementedError, match="compute_losses"):
        m(*args)
    with pytest.raises(NotImplementedError):
        m.train().compute_losses(*args)


# ------------------------------------------------------------------ GPU ------------------------------------------------------

def _gpu_path(nc, mask, dev):
    from stabletts_b200 import monotonic_align
    return monotonic_align.maximum_path(torch.as_tensor(nc).to(dev), torch.as_tensor(mask).to(dev))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=str)
@pytest.mark.parametrize("name", list(MAS_CASES))
def test_maximum_path_vs_reference_fixture(name, dtype, dev, golden_dir):
    g = _golden(golden_dir, name)
    nc = torch.from_numpy(g["neg_cent"]).to(dtype)
    mask = torch.from_numpy(g["mask"]).to(dtype)
    out = _gpu_path(nc, mask, dev)
    assert out.dtype == dtype and out.device == dev
    want = g["path"].astype(np.int32) if dtype == torch.float32 else mas_ref.maximum_path(nc.float().numpy(), g["mask"])
    assert np.array_equal(out.float().cpu().numpy().astype(np.int32), want)


def _lengths_mask(t_y, t_x, Ty, Tx):
    t_y, t_x = torch.as_tensor(t_y), torch.as_tensor(t_x)
    return ((torch.arange(Ty)[None, :, None] < t_y[:, None, None]) & (torch.arange(Tx)[None, None, :] < t_x[:, None, None])).float()


def _train_scores(gen, B, Ty, Tx, D=80):
    mu = torch.randn(B, D, Tx, generator=gen)
    tok = torch.sort(torch.randint(0, Tx, (B, Ty), generator=gen), dim=1).values
    y = torch.gather(mu, 2, tok[:, None, :].expand(B, D, Ty)) + torch.randn(B, D, Ty, generator=gen)
    return mas_ref.neg_cent64(y, mu).float()


def _sweep_cases():
    gen = torch.Generator().manual_seed(2024)
    cases = []
    # the trainer's shape: B = 32, the sampler's largest bucket (1000 frames), a few hundred interspersed tokens
    B, Ty, Tx = 32, 1000, 400
    t_y = torch.randint(700, 1001, (B,), generator=gen)
    t_y[0] = 1000
    t_x = torch.minimum(torch.randint(100, 401, (B,), generator=gen), t_y)
    t_x[0] = 400
    cases.append(("b32_1000x400_buckets", _train_scores(gen, B, Ty, Tx), _lengths_mask(t_y, t_x, Ty, Tx)))
    cases.append(("b32_1000x400_full", _train_scores(gen, B, Ty, Tx), torch.ones(B, Ty, Tx)))
    # t_x = t_y, t_x = 1, t_x > t_y, t_y = 1, t_y = 0, at every scale; then ties
    t_y, t_x = [64, 64, 20, 1, 0, 64, 33, 7], [64, 1, 50, 1, 10, 40, 33, 64]
    for scale in (1e-3, 1.0, 1e2, 1e5):
        cases.append((f"edges_scale{scale:g}", torch.randn(8, 64, 64, generator=gen) * scale, _lengths_mask(t_y, t_x, 64, 64)))
    cases.append(("ties", torch.randint(-1, 2, (8, 64, 64), generator=gen).float(), _lengths_mask(t_y, t_x, 64, 64)))
    cases.append(("ties_scale1e5", torch.randint(-3, 4, (8, 64, 64), generator=gen).float() * 1e5, _lengths_mask(t_y, t_x, 64, 64)))
    # decision bits beyond shared memory: 6000 x ⌈2000/32⌉ words = 1.5 MB
    cases.append(("bits_in_workspace_6000x2000", _train_scores(gen, 1, 6000, 2000, D=16), torch.ones(1, 6000, 2000)))
    return cases


@pytest.mark.gpu
def test_maximum_path_sweep_vs_oracle(dev):
    for name, nc, mask in _sweep_cases():
        out = _gpu_path(nc, mask, dev)
        want = mas_ref.maximum_path(nc.numpy(), mask.numpy())
        assert np.array_equal(out.cpu().numpy().astype(np.int32), want), name
    # a strided view: neg_cent built as (B, T_x, T_y) and transposed
    gen = torch.Generator().manual_seed(7)
    base = torch.randn(4, 90, 200, generator=gen).to(dev)
    nc = base.transpose(1, 2)
    mask = _lengths_mask([200, 150, 99, 91], [90, 77, 90, 13], 200, 90).to(dev)
    out = _gpu_path(nc, mask, dev)
    assert np.array_equal(out.cpu().numpy().astype(np.int32), mas_ref.maximum_path(nc.cpu().numpy(), mask.cpu().numpy()))


@pytest.mark.gpu
def test_utterance_alone_equals_its_batch_row_and_graph_capture(dev):
    from stabletts_b200 import monotonic_align
    gen = torch.Generator().manual_seed(11)
    B, Ty, Tx = 6, 300, 120
    nc = _train_scores(gen, B, Ty, Tx).to(dev)
    mask = _lengths_mask([300, 211, 120, 57, 300, 90], [120, 80, 120, 57, 3, 100], Ty, Tx).to(dev)
    full = monotonic_align.maximum_path(nc, mask)
    for b in range(B):
        assert torch.equal(monotonic_align.maximum_path(nc[b:b + 1], mask[b:b + 1]), full[b:b + 1]), b
    static_nc, static_mask = nc.clone(), mask.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        monotonic_align.maximum_path(static_nc, static_mask)                  # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = monotonic_align.maximum_path(static_nc, static_mask)
    nc2 = _train_scores(gen, B, Ty, Tx).to(dev)
    static_nc.copy_(nc2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_out, monotonic_align.maximum_path(nc2, mask))
    assert not torch.equal(static_out, full)


@pytest.mark.gpu
@pytest.mark.parametrize("D,B,Ty,Tx", [(80, 3, 257, 97), (128, 2, 130, 64), (80, 1, 1, 1), (80, 32, 1000, 400)])
def test_scores_vs_fp64(D, B, Ty, Tx, dev):
    from stabletts_b200 import monotonic_align
    gen = torch.Generator().manual_seed(D + Ty)
    y = torch.randn(B, D, Ty, generator=gen) * 2.0 - 4.0
    mu = torch.randn(B, D, Tx, generator=gen) * 1.5 - 3.0
    out = monotonic_align.scores(y.to(dev), mu.to(dev)).cpu().double()
    ref = mas_ref.neg_cent64(y, mu)
    y64, mu64 = y.double(), mu.double()
    scale = (0.5 * (y64 ** 2).sum(1)[:, :, None] + torch.einsum("bdt,bds->bts", y64.abs(), mu64.abs())
             + 0.5 * (mu64 ** 2).sum(1)[:, None, :] + 0.5 * np.log(2 * np.pi) * D)
    ratio = float(((out - ref).abs() / (SCORE_ULPS * 2.0 ** -24 * scale)).max())
    print(f"st_mas_scores D={D} ({B},{Ty},{Tx}): worst error / bar = {ratio:.3f}")
    assert ratio <= 1.0


def _set_engine(model, engine):
    for mod in (model.encoder, model.ref_encoder, model.dp, model.decoder.estimator):
        mod.set_engine(engine)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(FWD_CASES))
def test_compute_losses_vs_forward_fixture(name, engine, dev, golden_dir):
    from stabletts_b200 import StableTTS
    cs, g = FWD_CASES[name], _golden(golden_dir, name)
    m = StableTTS(synth_ref.N_VOCAB, cs["n_mel"], 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
    m.load_state_dict(synth_ref.make_state(n_mel=cs["n_mel"]), strict=True)
    m = m.to(dev)
    _set_engine(m, engine)
    inp = {k: v.to(dev) for k, v in _fwd_inputs(g).items()}
    with inject_by_shape(_draws(g)):
        dur, diff, prior, attn = m.compute_losses(inp["ids"], inp["x_lengths"], inp["y"], inp["y_lengths"], inp["z"], inp["z_lengths"])
    assert attn.shape == g["attn"].shape
    assert torch.equal(attn.cpu().to(torch.uint8), torch.from_numpy(g["attn"]))
    errs = {"dur": _rel(dur, g["dur_loss"]), "prior": _rel(prior, g["prior_loss"]), "diff": _rel(diff, g["diff_loss"])}
    print(name, engine, errs)
    assert errs["dur"] <= 1e-4 and errs["prior"] <= 1e-4 and errs["diff"] <= DIFF_BAR[engine], errs
    with pytest.raises(NotImplementedError):
        m.train().compute_losses(inp["ids"], inp["x_lengths"], inp["y"], inp["y_lengths"], inp["z"], inp["z_lengths"])


# ---- st_mas_losses against the fp64 statement of the header; st_maximum_path's dur and cum against its own path ----------
LOG_2PI = float(np.log(2 * np.pi))


def _loss_operands(seed, B, M, Ty, Tx, y_len, x_len):
    """ragged y_mask / x_mask from the lengths; durations 0 .. 5 at valid tokens (0 included: log 1e-8 is in play) and
    values at padded tokens too; logw non-zero everywhere, padded tokens included (the formula counts them)"""
    gen = torch.Generator().manual_seed(seed)
    y_len, x_len = torch.as_tensor(y_len, dtype=torch.int64), torch.as_tensor(x_len, dtype=torch.int64)
    y_mask = (torch.arange(Ty)[None, :] < y_len[:, None]).float()
    x_mask = (torch.arange(Tx)[None, :] < x_len[:, None]).float()
    dur = torch.randint(0, 6, (B, Tx), generator=gen).float()
    dur[:, 0] = 0.0
    return {"y": torch.randn(B, M, Ty, generator=gen), "mu_y": torch.randn(B, M, Ty, generator=gen) * 0.7 + 0.2, "y_mask": y_mask,
            "logw": torch.randn(B, Tx, generator=gen) * 1.5, "x_mask": x_mask, "dur": dur, "x_lengths": x_len}


def mas_losses_ref(t, M):
    """(prior_loss, dur_loss) of the header's statement in fp64 on the fp32 inputs"""
    y, mu, ym = t["y"].double(), t["mu_y"].double(), t["y_mask"].double()
    prior = (0.5 * ((y - mu) ** 2 + LOG_2PI) * ym[:, None, :]).sum() / (ym.sum() * M)
    e = t["logw"].double() - torch.log(1e-8 + t["dur"].double()) * t["x_mask"].double()
    return prior, (e ** 2).sum() / float(t["x_lengths"].sum())


def mas_losses_terms32(t, M):
    """the fp32 terms as models/model.py and duration_predictor.py form them, summed in double: E32's reference"""
    prior_t = 0.5 * ((t["y"] - t["mu_y"]) ** 2 + LOG_2PI) * t["y_mask"][:, None, :]
    dur_t = (t["logw"] - torch.log(1e-8 + t["dur"]) * t["x_mask"]) ** 2
    return (prior_t.double().sum() / (t["y_mask"].double().sum() * M), dur_t.double().sum() / float(t["x_lengths"].sum()))


def _run_mas_losses(t, dev, B, M, Ty, Tx, ws_bytes=None, **null):
    """st_mas_losses through _lib; outputs start as NaN.  null: argument names passed as NULL.  -> (rc, error, prior, dur)"""
    import ctypes as C
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    g = {k: v.to(dev).contiguous() for k, v in t.items()}
    out = torch.full((2,), float("nan"), device=dev)
    need = int(lib.st_mas_workspace_bytes(max(B, 1), Ty, Tx))
    ws = torch.empty(max(need, 1), device=dev, dtype=torch.uint8)
    ptr = lambda k: None if null.get(k) else g[k].data_ptr()                   # noqa: E731
    rc = lib.st_mas_losses(ptr("y"), ptr("mu_y"), ptr("y_mask"), ptr("logw"), ptr("x_mask"), ptr("dur"), ptr("x_lengths"), ws.data_ptr(),
                           need if ws_bytes is None else ws_bytes, B, M, Ty, Tx, out.data_ptr(), C.c_void_p(out.data_ptr() + 4),
                           torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize(dev)
    err = lib.st_last_error(None).decode() if rc else ""
    o = out.cpu()
    return rc, err, float(o[0]), float(o[1])


def _loss_cases():
    gen = torch.Generator().manual_seed(31)
    y_len = torch.randint(700, 1001, (32,), generator=gen)
    x_len = torch.minimum(torch.randint(100, 401, (32,), generator=gen), y_len)
    y_len[0], x_len[0] = 1000, 400
    y_len[5] = 0                                                   # an utterance whose y_mask is all zero
    return {"b32_m80_1000x400": (32, 80, 1000, 400, y_len, x_len), "b32_m128_1000x400": (32, 128, 1000, 400, y_len, x_len),
            "b1_m1_1x1": (1, 1, 1, 1, [1], [1]), "b3_m80_37x11": (3, 80, 37, 11, [37, 20, 1], [11, 4, 1])}


LOSS_CASES = _loss_cases()


def test_loss_statement_matches_the_reference_formulas():
    """the fp64 statement is torch's fp64 of the reference's own expressions (mse-style sums over masks)"""
    for name, (B, M, Ty, Tx, yl, xl) in LOSS_CASES.items():
        if B > 3:
            continue
        t = _loss_operands(1, B, M, Ty, Tx, yl, xl)
        prior, dur = mas_losses_ref(t, M)
        t64 = {k: v.double() if v.is_floating_point() else v for k, v in t.items()}
        y_mask = t64["y_mask"][:, None, :]
        want_prior = torch.sum(0.5 * ((t64["y"] - t64["mu_y"]) ** 2 + np.log(2 * np.pi)) * y_mask) / (torch.sum(y_mask) * M)
        logw_ = torch.log(1e-8 + t64["dur"]) * t64["x_mask"]
        want_dur = torch.sum((t64["logw"] - logw_) ** 2) / torch.sum(t64["x_lengths"])
        assert abs(float(prior - want_prior)) <= 1e-12 * abs(float(want_prior)), name
        assert abs(float(dur - want_dur)) <= 1e-12 * abs(float(want_dur)), name
        if Tx > 1:                                 # a valid token with dur = 0, and logw at every padded token
            assert (t["dur"][t["x_mask"] > 0] == 0).any() and (t["logw"][t["x_mask"] == 0] != 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LOSS_CASES))
def test_mas_losses_vs_fp64(name, dev):
    """st_mas_losses against the header's statement: max(4 E32, 8 ulp), E32 from the fp32 terms summed in double"""
    from kernel_harness import bar
    B, M, Ty, Tx, yl, xl = LOSS_CASES[name]
    t = _loss_operands(7, B, M, Ty, Tx, yl, xl)
    rc, err, prior, dur = _run_mas_losses(t, dev, B, M, Ty, Tx)
    assert rc == 0, err
    for what, got, r64, r32 in zip(("prior", "dur"), (prior, dur), mas_losses_ref(t, M), mas_losses_terms32(t, M)):
        e32, e = abs(float(r32 - r64)), abs(got - float(r64))
        b = bar(r64.reshape(1), e32)
        print(f"{name} {what}: err {e:.2e} / bar {b:.2e} = {e / b:.3f}")
        assert e <= b, (what, got, float(r64), e32)


@pytest.mark.gpu
def test_mas_losses_refusals(dev):
    """a workspace below st_mas_workspace_bytes, B <= 0, a NULL pointer: refused, nothing written"""
    B, M, Ty, Tx, yl, xl = LOSS_CASES["b3_m80_37x11"]
    t = _loss_operands(8, B, M, Ty, Tx, yl, xl)
    from stabletts_b200 import _lib
    need = int(_lib.load_library().st_mas_workspace_bytes(B, Ty, Tx))
    for kw, needle, b_ in ((dict(ws_bytes=need - 1), "workspace smaller", B), ({}, "bad argument", 0), ({}, "bad argument", -1),
                           (dict(y=True), "bad argument", B), (dict(x_lengths=True), "bad argument", B), (dict(dur=True), "bad argument", B)):
        rc, err, prior, dur = _run_mas_losses(t, dev, b_, M, Ty, Tx, **kw)
        assert rc != 0 and needle in err, (kw, b_, err)
        assert np.isnan(prior) and np.isnan(dur), kw


def _path_dur_cum(nc, dev, mask=None, x_lengths=None, y_lengths=None):
    """st_maximum_path with every output starting as NaN -> (path, dur, cum) on the CPU"""
    from stabletts_b200 import _lib
    from stabletts_b200.monotonic_align import workspace
    lib = _lib.load_library()
    B, Ty, Tx = nc.shape
    ncd = nc.to(dev).contiguous()
    outs = [torch.full(s, float("nan"), device=dev) for s in ((B, Ty, Tx), (B, Tx), (B, Tx))]
    keep = [None if v is None else v.to(dev).contiguous() for v in (mask, x_lengths, y_lengths)]
    ws = workspace(B, Ty, Tx, dev)
    _lib.check(lib, None, lib.st_maximum_path(ncd.data_ptr(), *[None if v is None else v.data_ptr() for v in keep],
                                              *[o.data_ptr() for o in outs], ws.data_ptr(), ws.numel(), B, Ty, Tx,
                                              torch.cuda.current_stream(dev).cuda_stream), "st_maximum_path")
    return [o.cpu() for o in outs]


def _check_dur_cum(path, dur, cum, what):
    """dur = path summed over frames, cum its inclusive prefix sums, bit for bit"""
    assert torch.equal(dur, path.sum(1)), what
    assert torch.equal(cum, torch.cumsum(path.sum(1).double(), 1).float()), what


@pytest.mark.gpu
def test_durations_and_prefix_sums_are_the_path(dev):
    """dur and cum of st_maximum_path against its own path, with lengths from the mask and from x_lengths / y_lengths (the
    same path either way), on the sweep of test_maximum_path_sweep_vs_oracle (t_x > t_y, t_y = 0, bits in the workspace)
    and at Tx = 511, 512, 513 (the 512-thread chunked scan) and the 9632-token limit"""
    for name, nc, mask in _sweep_cases():
        path, dur, cum = _path_dur_cum(nc, dev, mask=mask)
        _check_dur_cum(path, dur, cum, name)
        xl, yl = mask[:, 0, :].sum(1).long(), mask[:, :, 0].sum(1).long()
        p2, d2, c2 = _path_dur_cum(nc, dev, x_lengths=xl, y_lengths=yl)
        assert torch.equal(p2, path) and torch.equal(d2, dur) and torch.equal(c2, cum), name
    gen = torch.Generator().manual_seed(12)
    for Tx in (511, 512, 513, 9632):
        Ty = Tx + 37
        nc = torch.randn(2, Ty, Tx, generator=gen)
        yl, xl = torch.tensor([Ty, Ty - 40]), torch.tensor([Tx, Tx - 2])
        path, dur, cum = _path_dur_cum(nc, dev, x_lengths=xl, y_lengths=yl)
        _check_dur_cum(path, dur, cum, Tx)
        assert torch.equal(dur.sum(1), yl.float()) and (dur[1, Tx - 2:] == 0).all(), Tx
        if Tx < 1000:
            p2, d2, c2 = _path_dur_cum(nc, dev, mask=_lengths_mask(yl, xl, Ty, Tx))
            assert torch.equal(p2, path) and torch.equal(d2, dur) and torch.equal(c2, cum), Tx
