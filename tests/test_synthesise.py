"""StableTTS.synthesise on the CUDA path: the MelStyleEncoder, the DurationPredictor and the drop-in StableTTS.

CPU: the oracles (oracle/style_ref.py, duration_ref.py, synth_ref.py) against the fixtures of the unmodified reference
(tests/golden/style_*.npz, dp_*.npz, synth_*.npz; recipe oracle/make_golden_synth.py), the drop-in's state_dict
inventory and strict loading, and the refusals (CPU tensors, training, unsupported configurations).
GPU: both engines against the fixtures (c, logw, the whole synthesise in both precision modes), the DurationPredictor's
batch independence, and the Mish GEMM epilogue (EPI_MISH) against an fp64 statement through st_test_gemm_ex."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_errs
from kernel_harness import dev  # noqa: F401 (a fixture)
from oracle import duration_ref as D, style_ref as S, synth_ref as Y, weights

MISH = 512


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _durations(logw, mask):
    return torch.ceil(torch.exp(logw.double()) * mask.double())


# ------------------------------------------------------------------ CPU ------------------------------------------------------

@pytest.mark.parametrize("name", list(S.CASES))
def test_style_oracle_vs_reference_golden(name, golden_dir):
    cs = S.CASES[name]
    g = _golden(golden_dir, name)
    st = S.make_state(n_mel=cs["n_mel"])
    assert float(g["weight_checksum"]) == pytest.approx(weights.checksum(st), rel=1e-12)
    y, mask = S.make_inputs(cs["seed"], cs["B"], cs["T"], cs["n_mel"], cs["lens"])
    with torch.inference_mode():
        c = S.style_forward(st, y, mask)
    assert max(rel_errs(c, torch.from_numpy(g["c"]))) <= 2e-5


@pytest.mark.parametrize("name", list(D.CASES))
def test_duration_oracle_vs_reference_golden(name, golden_dir):
    cs = D.CASES[name]
    g = _golden(golden_dir, name)
    st = D.make_state()
    assert float(g["weight_checksum"]) == pytest.approx(weights.checksum(st), rel=1e-12)
    x, mask, c = D.make_inputs(int(g["seed"]), cs["lens"], cs["Tx"])
    with torch.inference_mode():
        logw = D.dp_forward(st, x, mask, c)
    ref = torch.from_numpy(g["logw"])
    assert max(rel_errs(logw, ref)) <= 2e-5
    assert torch.equal(_durations(logw, mask), _durations(ref, mask))


@pytest.mark.parametrize("name", list(Y.CASES))
def test_synthesise_oracle_vs_reference_golden(name, golden_dir):
    cs = Y.CASES[name]
    g = _golden(golden_dir, name)
    st = Y.make_state(n_mel=cs["n_mel"])
    assert float(g["weight_checksum"]) == pytest.approx(weights.checksum(st), rel=1e-12)
    ids, lens, y = Y.make_inputs(int(g["seed"]), cs["lens"], cs["T_ref"], cs["n_mel"])
    out = Y.synthesise(st, ids, lens, cs["n_timesteps"], y, torch.from_numpy(g["z"]), cs["length_scale"], cs["solver"], cs["cfg"])
    assert torch.equal(out["attn"].to(torch.uint8), torch.from_numpy(g["attn"]))
    for k in ("encoder_outputs", "decoder_outputs"):
        assert max(rel_errs(out[k], torch.from_numpy(g[k]))) <= 2e-5, k


def test_fixture_durations_are_realistic_and_clear_of_integers(golden_dir):
    """the fixture weights give 2-8 frame durations on average, and every valid w = exp(logw) is at least 5e-4 w from an
    integer, so that a logw within the 5e-5 bar of the GPU tests cannot move a duration"""
    for name, cs in Y.CASES.items():
        g = _golden(golden_dir, name)
        logw = torch.from_numpy(g["logw"]).double()
        mask = (torch.arange(logw.shape[-1])[None] < torch.as_tensor(cs["lens"])[:, None]).double().unsqueeze(1)
        w = torch.exp(logw)[mask > 0]
        assert 2.0 <= float(w.mean()) <= 8.0, (name, float(w.mean()))
        assert bool(((w - w.round()).abs() >= 5e-4 * w).all()), name


def test_drop_in_inventory_and_strict_load(golden_dir):
    from stabletts_b200 import StableTTS
    m = StableTTS(401, 80, 256, 1024, 4, 3, 6, 3, 0.1, 256)
    got = [[k, list(v.shape)] for k, v in m.state_dict().items()]
    inv = json.loads(str(np.load(os.path.join(golden_dir, "reference_inventory.npz"))["stabletts"]))
    assert len(got) == 189 and got == inv
    st = Y.make_state(n_mel=80)
    m.load_state_dict(st, strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in st.items())


def test_default_init_matches_reference_conventions():
    from stabletts_b200 import DurationPredictor, MelStyleEncoder
    torch.manual_seed(0)
    s = MelStyleEncoder(80)
    assert torch.count_nonzero(s.slf_attn.in_proj_bias) == 0 and torch.count_nonzero(s.slf_attn.out_proj.bias) == 0
    assert float(s._param("spectral.0.weight").abs().max()) <= 80 ** -0.5
    d = DurationPredictor(256, 1024, 3, 0.5, 256)
    assert torch.equal(d.norm1.weight, torch.ones(1024)) and torch.count_nonzero(d.norm2.bias) == 0
    assert float(d.conv2.weight.abs().max()) <= (1024 * 3) ** -0.5


def test_cpu_tensors_training_and_unsupported_configurations_raise():
    from stabletts_b200 import DurationPredictor, MelStyleEncoder, StableTTS
    s, d = MelStyleEncoder(80).eval(), DurationPredictor(256, 1024, 3, 0.5, 256).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        s(torch.zeros(1, 80, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        d(torch.zeros(1, 256, 3), torch.ones(1, 1, 3), torch.zeros(1, 256))
    m = StableTTS(401, 80, 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.synthesise(torch.zeros(1, 5, dtype=torch.long), torch.tensor([5]), 2, y=torch.zeros(1, 80, 4))
    with pytest.raises(NotImplementedError, match="reference"):
        m(None, None, None, None, None, None)
    with pytest.raises(NotImplementedError):
        m.train().synthesise(torch.zeros(1, 5, dtype=torch.long), torch.tensor([5]), 2, y=torch.zeros(1, 80, 4))
    with pytest.raises(NotImplementedError):
        s.train()(torch.zeros(1, 80, 4))
    with pytest.raises(NotImplementedError):
        d.train()(torch.zeros(1, 256, 3), torch.ones(1, 1, 3), torch.zeros(1, 256))
    for kw in (dict(style_hidden=256), dict(style_head=4), dict(style_kernel_size=3), dict(style_vector_dim=192)):
        with pytest.raises(ValueError):
            MelStyleEncoder(80, **kw)
    with pytest.raises(ValueError):
        MelStyleEncoder(72)
    for args in ((192, 1024, 3, 0.5, 256), (256, 768, 3, 0.5, 256), (256, 1024, 5, 0.5, 256)):
        with pytest.raises(ValueError):
            DurationPredictor(*args)


def test_mish_reference_statement():
    """the fp64 Mish of the epilogue tests is nn.Mish (softplus threshold 20)"""
    x = torch.linspace(-30, 30, 2001, dtype=torch.float64)
    assert torch.allclose(_mish64(x), torch.nn.Mish()(x), rtol=1e-15, atol=1e-300)


def _mish64(v):
    return v * torch.tanh(F.softplus(v))


# ------------------------------------------------------------------ GPU ------------------------------------------------------

ENGINES = ["tcgen05", "simt"]
C_BAR = {"tcgen05": 1e-4, "simt": 2e-5}


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(S.CASES))
def test_style_encoder_vs_reference_golden(name, engine, dev, golden_dir):
    from stabletts_b200 import MelStyleEncoder
    cs = S.CASES[name]
    m = MelStyleEncoder(cs["n_mel"]).eval()
    m.load_state_dict(S.make_state(n_mel=cs["n_mel"]), strict=True)
    m = m.to(dev)
    m.set_engine(engine)
    y, mask = S.make_inputs(cs["seed"], cs["B"], cs["T"], cs["n_mel"], cs["lens"])
    c = m(y.to(dev), None if mask is None else mask.to(dev)).cpu()
    e = rel_errs(c, torch.from_numpy(_golden(golden_dir, name)["c"]))
    assert e[0] <= C_BAR[engine], (name, engine, e)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(D.CASES))
def test_duration_predictor_vs_reference_golden(name, engine, dev, golden_dir):
    from stabletts_b200 import DurationPredictor
    cs = D.CASES[name]
    g = _golden(golden_dir, name)
    m = DurationPredictor(256, 1024, 3, 0.5, 256).eval()
    m.load_state_dict(D.make_state(), strict=True)
    m = m.to(dev)
    m.set_engine(engine)
    x, mask, c = D.make_inputs(int(g["seed"]), cs["lens"], cs["Tx"])
    logw = m(x.to(dev), mask.to(dev), c.to(dev)).cpu()
    ref = torch.from_numpy(g["logw"])
    e = rel_errs(logw, ref)
    assert e[0] <= 5e-5, (name, engine, e)
    assert torch.equal(_durations(logw, mask), _durations(ref, mask))


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("lens", [[129, 70, 3], [129] * 6 + [100, 57, 3] + [120] * 11], ids=["B3", "B20"])
def test_duration_predictor_utterance_alone_is_bit_identical_to_its_batch_row(engine, lens, dev):
    """B = 20 at Tx = 129 gives the convs enough tiles for 256-channel tiles on 132 SMs, while one utterance runs on
    128-channel tiles: the identity then also rests on both tile widths summing every element in the same order"""
    from stabletts_b200 import DurationPredictor
    m = DurationPredictor(256, 1024, 3, 0.5, 256).eval()
    m.load_state_dict(D.make_state(), strict=True)
    m = m.to(dev)
    m.set_engine(engine)
    x, mask, c = D.make_inputs(5, lens, 129)
    x, mask, c = x.to(dev), mask.to(dev), c.to(dev)
    batch = m(x, mask, c)
    for b in sorted({0, len(lens) // 2, len(lens) - 2, len(lens) - 1}):
        alone = m(x[b:b + 1], mask[b:b + 1], c[b:b + 1])
        assert torch.equal(alone, batch[b:b + 1]), b


@pytest.mark.gpu
@pytest.mark.parametrize("taps,C0", [(3, 256), (3, 1024)])
def test_wide_and_128_channel_tiles_give_identical_rows(taps, C0, dev):
    """the DurationPredictor conv shapes through st_test_gemm_ex without split-K: a batch of 20 runs on 256-channel tiles,
    one utterance on 128-channel tiles, and every output element is bit-identical"""
    import ctypes as C
    from stabletts_b200 import _lib
    from test_gemm_contract import make_tensors, problem, run_hook
    lib = _lib.load_library()
    h = C.c_void_p()
    _lib.check(lib, None, lib.st_create_ffgan(0, C.byref(h)), "st_create_ffgan")
    try:
        d = problem(B=20, BB=20, T=129, C0=C0, N=1024, taps=taps, flags=BIAS_, ksplit=1, num_sms=132)
        t = make_tensors(d, 29)
        rc, err, big, plan = run_hook(lib, h, d, t, dev)
        assert rc == 0 and plan.bn == 256, (err, plan.bn)
        for b in (0, 19):
            d1 = problem(B=1, BB=1, T=129, C0=C0, N=1024, taps=taps, flags=BIAS_, ksplit=1, num_sms=132)
            t1 = dict(t, A0=t["A0"][b:b + 1])
            rc, err, one, plan1 = run_hook(lib, h, d1, t1, dev)
            assert rc == 0 and plan1.bn == 128, (err, plan1.bn)
            assert torch.equal(one["out"].view(torch.int32), big["out"][b:b + 1].view(torch.int32)), b
    finally:
        lib.st_destroy(h)


@pytest.mark.gpu
@pytest.mark.parametrize("length_scale", [1.15, 0.9, 1.0])
def test_alignment_matches_torch_cumsum_at_fractional_length_scale(length_scale, dev):
    """expand_by_durations against the reference's generate_path (oracle/align_ref.py, torch's CPU cumsum) on 200 random
    61-token utterances with 2-8 frame durations: identical alignment and output length.  Utterances whose exact total
    is an integer are left out: there y_lengths depends on the order in which the reference's fp32 torch.sum adds."""
    from oracle import align_ref
    from stabletts_b200 import expand_by_durations
    g = torch.Generator().manual_seed(11)
    checked = 0
    for i in range(200):
        d = torch.randint(2, 9, (1, 1, 61), generator=g).float()
        logw = torch.log(d - 0.5)                                   # ceil(exp(logw)) = d
        x_mask = torch.ones(1, 1, 61)
        total = (d * length_scale).double().sum()
        if length_scale != 1.0 and abs(float(total - total.round())) < 1e-3:
            continue
        mu_x = torch.randn(1, 8, 61, generator=g)
        _, _, y_len, attn = align_ref.expand_by_durations(logw, x_mask, mu_x, length_scale)
        _, _, y_len_d, attn_d = expand_by_durations(logw.to(dev), x_mask.to(dev), mu_x.to(dev), length_scale, return_attn=True)
        assert torch.equal(y_len_d.cpu(), y_len), i
        assert torch.equal(attn_d.cpu(), attn), i
        checked += 1
    assert checked >= 180


def _set_engine(model, engine, precision):
    for mod in (model.encoder, model.ref_encoder, model.dp, model.decoder.estimator):
        mod.set_engine(engine)
    for mod in (model.encoder, model.decoder.estimator):
        mod.set_precision(precision)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [("tcgen05", "bf16x3"), ("tcgen05", "ffn_fp16x2"), ("simt", "bf16x3")], ids="-".join)
@pytest.mark.parametrize("name", list(Y.CASES))
def test_synthesise_vs_reference_golden(name, mode, dev, golden_dir):
    from stabletts_b200 import StableTTS
    cs = Y.CASES[name]
    g = _golden(golden_dir, name)
    m = StableTTS(Y.N_VOCAB, cs["n_mel"], 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
    m.load_state_dict(Y.make_state(n_mel=cs["n_mel"]), strict=True)
    m = m.to(dev)
    _set_engine(m, *mode)
    ids, lens, y = Y.make_inputs(int(g["seed"]), cs["lens"], cs["T_ref"], cs["n_mel"])
    out = m.synthesise(ids.to(dev), lens.to(dev), cs["n_timesteps"], 1.0, y.to(dev), cs["length_scale"], cs["solver"], cs["cfg"],
                       z=torch.from_numpy(g["z"]).to(dev))
    attn = out["attn"].cpu()
    assert attn.shape == g["attn"].shape, (attn.shape, g["attn"].shape)          # the output length
    assert torch.equal(attn.to(torch.uint8), torch.from_numpy(g["attn"]))
    for k in ("encoder_outputs", "decoder_outputs"):
        e = rel_errs(out[k].cpu(), torch.from_numpy(g[k]))
        assert e[0] <= 1e-3, (name, mode, k, e)


# ---- the Mish epilogue (EPI_MISH) through the conv-GEMM contract hook ------------------------------------------------------

def _mish_cases():
    from test_gemm_contract import problem
    return {
        "linear_m80": problem(B=1, BB=1, T=300, C0=80, N=128, flags=BIAS_ | MISH, planes=True),      # spectral.0 at M = 80
        "linear_128": problem(B=2, BB=2, T=129, C0=128, N=128, flags=BIAS_ | MISH, planes=True),     # spectral.3
        "masked_t1": problem(B=3, BB=3, T=1, C0=128, N=128, flags=BIAS_ | MISH | MASK_),
        "conv5_n256": problem(B=2, BB=2, T=65, C0=128, N=256, taps=5, flags=BIAS_ | MISH, num_sms=2),  # would take wide tiles
        "narrow_n64": problem(B=1, BB=1, T=70, C0=64, N=64, flags=BIAS_ | MISH),                       # would take narrow tiles
        "splitk2": problem(B=1, BB=1, T=100, C0=128, N=128, taps=5, flags=BIAS_ | MISH, ksplit=2, planes=True, engines=("tc",)),
        "splitk4": problem(B=2, BB=2, T=33, C0=256, N=128, flags=BIAS_ | MISH | MASK_, ksplit=4, engines=("tc",)),
        "no_split": problem(B=1, BB=1, T=100, C0=128, N=128, taps=5, flags=BIAS_ | MISH, ksplit=1),
        "big_args": problem(B=1, BB=1, T=64, C0=128, N=128, flags=BIAS_ | MISH, xscale=12.0),           # past the threshold 20
    }


BIAS_, MASK_ = 1, 8


def _mish_ref(d, t):
    from test_gemm_contract import gemm_contract_ref
    v = gemm_contract_ref(dict(d, flags=d["flags"] & BIAS_), t)["out"]
    v = _mish64(v)
    if d["flags"] & MASK_:
        v = v * t["mask"].double()[torch.arange(d["BB"]) % d["B"]][..., None]
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "simt"])
@pytest.mark.parametrize("name", list(_mish_cases()))
def test_mish_epilogue_vs_fp64(name, engine, dev):
    import ctypes as C
    from stabletts_b200 import _lib
    from test_gemm_contract import make_tensors, run_hook
    d = _mish_cases()[name]
    if engine not in d["engines"]:
        pytest.skip("split-K runs on the wgmma engine only")
    lib = _lib.load_library()
    h = C.c_void_p()
    _lib.check(lib, None, lib.st_create_ffgan(0, C.byref(h)), "st_create_ffgan")
    try:
        _lib.check(lib, h, lib.st_set_engine(h, {"tc": 0, "simt": 1}[engine]), "st_set_engine")
        t = make_tensors(d, 17)
        rc, err, o, plan = run_hook(lib, h, d, t, dev)
        assert rc == 0, err
        ref = _mish_ref(d, t)
        bar = 5e-5 if engine == "tc" else 2e-5
        e = rel_errs(o["out"], ref)
        assert e[0] < bar and e[1] < bar, (name, engine, e)
        if d["planes"]:
            assert torch.equal(o["hi"].view(torch.int16), o["out"].to(torch.bfloat16).view(torch.int16))
            assert torch.equal(o["lo"].view(torch.int16), (o["out"] - o["hi"].float()).to(torch.bfloat16).view(torch.int16))
        if engine == "tc":
            if d["ksplit"] > 1:
                assert plan.ksplit == d["ksplit"]
            else:
                assert (plan.bn, _lib.ST_TEST_MODE_NAMES[plan.mode], plan.ksplit) == (128, "MISH", 1), (plan.bn, plan.mode)
        else:
            assert plan.engine == 1
    finally:
        lib.st_destroy(h)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_mish_refuses_second_activation_residual_and_layernorm(engine, dev):
    import ctypes as C
    from stabletts_b200 import _lib
    from test_gemm_contract import make_tensors, problem, run_hook
    lib = _lib.load_library()
    h = C.c_void_p()
    _lib.check(lib, None, lib.st_create_ffgan(0, C.byref(h)), "st_create_ffgan")
    try:
        _lib.check(lib, h, lib.st_set_engine(h, {"tc": 0, "simt": 1}[engine]), "st_set_engine")
        for fl, needle in ((BIAS_ | MISH | 2, "alternatives"), (BIAS_ | MISH | 128, "alternatives"), (BIAS_ | MISH | 32, "EPI_RESID"),
                           (BIAS_ | MISH | 256, "EPI_SILU_OUT")):
            d = problem(B=1, BB=1, T=16, C0=128, N=128, flags=fl)
            rc, err, _, _ = run_hook(lib, h, d, make_tensors(d, 1), dev)
            assert rc != 0 and needle in err, (fl, err)
    finally:
        lib.st_destroy(h)
