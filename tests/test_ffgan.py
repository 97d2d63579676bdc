"""The FireflyGAN vocoder (vocoders/ffgan/, the reference's default vocoder).  CPU: the oracle against the fixtures of the
unmodified reference (tests/golden/ffgan_*.npz), the polyphase form of the transposed convs, the weight-norm fold, the
fixture weights' liveness, the drop-in's state_dict inventory and checkpoint loading.  GPU: the CUDA path against the
fixtures and the oracle, batch independence, the empty batch, and the conv-GEMM hook for every conv shape the model uses."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from conftest import rel_errs
from kernel_harness import dev  # noqa: F401 (a fixture)
from oracle import ffgan_ref as R


@pytest.fixture(scope="module")
def state():
    return R.make_state()


@pytest.mark.parametrize("name", list(R.CASES))
def test_oracle_vs_reference_golden(name, state, golden_dir):
    cs = R.CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    assert float(g["weight_checksum"]) == pytest.approx(R.weight_checksum(state), rel=1e-12)
    with torch.inference_mode():
        out = R.ffgan_forward(state, R.make_mel(cs["seed"], cs["B"], cs["T"]), polyphase=True)
    ref = torch.from_numpy(g["audio"])
    assert out.shape == ref.shape == (cs["B"], cs["T"] * 512)
    mx, l2 = rel_errs(out, ref)
    assert max(mx, l2) <= 2e-5, (mx, l2)


@pytest.mark.parametrize("u,k", [(8, 16), (2, 4)])
def test_polyphase_equals_conv_transpose(u, k):
    g = torch.Generator().manual_seed(u)
    x = torch.randn(2, 24, 19, generator=g, dtype=torch.float64)
    w = torch.randn(24, 12, k, generator=g, dtype=torch.float64)
    b = torch.randn(12, generator=g, dtype=torch.float64)
    ref = F.conv_transpose1d(x, w, b, stride=u, padding=(k - u) // 2)
    out = R.conv_transpose_polyphase(x, w, b, u)
    assert out.shape == ref.shape == (2, 12, 19 * u)
    assert float((out - ref).abs().max()) <= 1e-12


@pytest.mark.parametrize("transposed", [False, True])
def test_weight_norm_fold_matches_torch_parametrization(transposed):
    """dim 0 is C_out for Conv1d and C_in for ConvTranspose1d: g is (C_out, 1, 1) resp. (C_in, 1, 1)."""
    torch.manual_seed(3)
    conv = (nn.ConvTranspose1d(16, 8, 4, 2, padding=1) if transposed else nn.Conv1d(16, 8, 5, padding=2))
    conv = torch.nn.utils.parametrizations.weight_norm(conv)
    par = conv.parametrizations.weight
    with torch.no_grad():
        par.original0.copy_(torch.rand_like(par.original0) + 0.5)
    assert par.original0.shape == ((16 if transposed else 8), 1, 1)
    got = R.fold_weight_norm(par.original0.detach(), par.original1.detach())
    assert torch.allclose(got, conv.weight.detach(), rtol=1e-6, atol=1e-7)


def test_fixture_weights_are_live(state, golden_dir):
    """The reference's own init is nearly inert (audio std ~0.002); the fixture weights must exercise every layer."""
    audio = np.load(os.path.join(golden_dir, "ffgan_b3_t130.npz"))["audio"]
    assert audio.std() > 0.1 and np.abs(audio).max() > 0.9
    mel = R.make_mel(5, 1, 6)
    with torch.inference_mode():
        ref = R.ffgan_forward(state, mel)
        for i, depth in enumerate(R.DEPTHS):
            for j in range(depth):
                assert float((R.ffgan_forward(state, mel, skip_block=(i, j)) - ref).norm() / ref.norm()) > 1e-3, (i, j)
        for i in range(len(R.UPS)):
            for b in range(len(R.RES_K)):
                assert float((R.ffgan_forward(state, mel, skip_resblock=(i, b)) - ref).norm() / ref.norm()) > 1e-3, (i, b)


def test_drop_in_inventory_matches_reference(golden_dir, state):
    from stabletts_b200 import FireflyGANBase
    m = FireflyGANBase()
    got = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    inv = np.load(os.path.join(golden_dir, "ffgan_inventory.npz"))                   # oracle/make_golden_ffgan.py
    assert got == [(k, tuple(s)) for k, s in json.loads(str(inv["inventory"]))]
    assert len(got) == 471 and sum(int(np.prod(s)) for _, s in got) == int(inv["n_params"]) == 36511330
    m.load_state_dict(state, strict=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(torch.zeros(1, 128, 4))


@pytest.mark.parametrize("legacy", [False, True])
def test_wrapper_loads_checkpoint(tmp_path, state, legacy):
    """FireflyGANBaseWrapper(path): strict load + eval(), from the parametrization keys or the legacy weight_g / weight_v."""
    from stabletts_b200 import FireflyGANBaseWrapper
    sd = dict(state)
    if legacy:
        sd = {k.replace(".parametrizations.weight.original0", ".weight_g").replace(".parametrizations.weight.original1", ".weight_v"): v
              for k, v in sd.items()}
        assert any(k.endswith(".weight_g") for k in sd)
    path = tmp_path / "generator.pt"
    torch.save(sd, path)
    w = FireflyGANBaseWrapper(str(path))
    assert not w.model.training
    got = w.model.state_dict()
    assert list(got) == list(state) and all(torch.equal(got[k], state[k]) for k in state)


# ------------------------------------------------------------------ GPU ------------------------------------------------------

def _model(dev, state, engine="tcgen05"):
    from stabletts_b200 import FireflyGANBase
    m = FireflyGANBase().eval()
    m.load_state_dict(state, strict=True)
    m = m.to(dev)
    m.set_engine(engine)
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("name", list(R.CASES))
def test_ffgan_vs_reference_golden(name, engine, dev, state, golden_dir):
    cs = R.CASES[name]
    m = _model(dev, state, engine)
    audio = m(R.make_mel(cs["seed"], cs["B"], cs["T"]).to(dev))
    ref = torch.from_numpy(np.load(os.path.join(golden_dir, name + ".npz"))["audio"])
    assert audio.shape == ref.shape
    e = rel_errs(audio, ref)
    assert max(e) <= (1e-3 if engine == "tcgen05" else 2e-4), (name, engine, e)
    assert torch.isfinite(audio).all()


@pytest.mark.gpu
def test_ffgan_large_vs_oracle_and_properties(dev, state):
    """B = 8, T = 600 (4800 frames: the backbone's pwconv GEMMs and the first ups reach the 256-channel tiles) against the
    oracle on two rows; an utterance alone equals its row of the batch; the empty batch."""
    m = _model(dev, state)
    mel = R.make_mel(61, 8, 600)
    audio = m(mel.to(dev)).cpu()
    with torch.inference_mode():
        ref = R.ffgan_forward(state, mel[[0, 7]])
    e = rel_errs(audio[[0, 7]], ref)
    assert max(e) <= 1e-3, e
    alone = m(mel[3:4].to(dev)).cpu()
    assert rel_errs(alone, audio[3:4])[0] <= 1e-5
    assert m(torch.zeros(0, 128, 5, device=dev)).shape == (0, 2560)


def _conv_cases():
    cases = [(512, 13, 1, False)]                                                      # conv_pre
    for i in range(5):
        c = 256 >> i
        cases += [(c, k, d, False) for k in R.RES_K for d in R.RES_D]                  # convs1 (dilated) / convs2 (d = 1)
        cases.append((c, 2 * R.UPS[i][0], R.UPS[i][0], True))                         # ups[i] (C_in = 2c -> c)
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_conv_hook_every_model_shape(engine, dev):
    """st_test_conv_ex (the head's conv-GEMM: dilated taps, polyphase transposed conv) against F.conv1d /
    F.conv_transpose1d for every (C, k, dilation) and every (u, k) of the model."""
    import ctypes as C
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    h = C.c_void_p()
    _lib.check(lib, None, lib.st_create_ffgan(0, C.byref(h)), "st_create_ffgan")
    try:
        _lib.check(lib, h, lib.st_set_engine(h, {"simt": 1, "tcgen05": 0}[engine]), "st_set_engine")
        g = torch.Generator().manual_seed(9)
        B, T = 2, 70
        for c, k, d, tr in _conv_cases():
            cin = 2 * c if tr else c
            x = torch.randn(B, cin, T, generator=g)
            w = torch.randn((cin, c, k) if tr else (c, c, k), generator=g) / (cin * k) ** 0.5
            b = torch.randn(c, generator=g)
            ref = F.conv_transpose1d(x, w, b, stride=d, padding=d // 2) if tr else F.conv1d(x, w, b, padding=d * (k - 1) // 2, dilation=d)
            xd, wd, bd = x.to(dev), w.to(dev), b.to(dev)
            out = torch.empty(ref.shape, device=dev)
            rc = lib.st_test_conv_ex(h, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), out.data_ptr(), B, cin, c, T, k, d, int(tr),
                                     torch.cuda.current_stream().cuda_stream)
            _lib.check(lib, h, rc, "st_test_conv_ex")
            e = rel_errs(out, ref)
            assert max(e) <= (1e-4 if engine == "tcgen05" else 1e-5), (c, k, d, tr, e)
    finally:
        lib.st_destroy(h)
