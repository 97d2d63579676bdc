"""Row f4 (SURVEY.md §8f): the vocoder hand-off.  CPU: state_dict inventory of the drop-in against the oracle's restated
inventory and the stored parameter inventory of the unmodified reference Vocos, also for api.py's Vocos(VocosConfig(),
MelConfig()) from the top-level config.py (512 / 1536 / 8); st_create_vocos's refusals.  GPU: the CUDA path through the C ABI
against the fixtures generated from the unmodified reference (tests/golden/vocos_*.npz: the vocos training config and api.py's
config, one of them with 16 % of the magnitudes on the 1e2 clip) and against the oracle at sizes that reach the 256-channel
GEMM tiles, at T = 1, 2, 3, and across the dims and STFT shapes st_create_vocos accepts; size-independent properties (batch
independence, frame-count scaling of the output)."""
import ctypes as C
import dataclasses
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import rel_errs
from kernel_harness import dev  # noqa: F401 (a fixture)
from oracle import vocoder_ref as V


def test_drop_in_inventory_matches_reference_keys(golden_dir):
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200 import Vocos
    m = Vocos()
    want = V.param_shapes()
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert list(got) == list(want) and got == dict(want)
    m.load_state_dict(V.make_state(), strict=True)
    inv = np.load(os.path.join(golden_dir, "reference_inventory.npz"))          # oracle/make_golden_inventory.py
    assert [(k, tuple(s)) for k, s in json.loads(str(inv["vocos"]))] == list(got.items())
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(torch.zeros(1, 128, 4))


@dataclasses.dataclass
class RootVocosConfig:                 # the reference's top-level config.py VocosConfig, the one api.py imports
    input_channels: int = 128
    dim: int = 512
    intermediate_dim: int = 1536
    num_layers: int = 8


@dataclasses.dataclass
class RootMelConfig:                   # the fields of the top-level MelConfig that Vocos reads
    n_fft: int = 2048
    hop_length: int = 512


def test_api_py_vocos_inventory():
    """Vocos(VocosConfig(), MelConfig()) as api.py's get_vocoder builds it has the 512 / 1536 / 8 inventory of the oracle and
    loads its state strictly"""
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200 import Vocos
    m = Vocos(RootVocosConfig(), RootMelConfig())
    assert (m.dim, m.intermediate_dim, m.num_layers, m.n_fft, m.hop_length) == (512, 1536, 8, 2048, 512)
    want = V.param_shapes(**V.API_DIMS)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert list(got) == list(want) and got == dict(want)
    assert len([k for k in got if k.endswith("dwconv.weight")]) == 8
    m.load_state_dict(V.make_state(**V.API_DIMS), strict=True)


@pytest.mark.parametrize("n_fft,hop", [(1024, 1024), (2048, 2048), (2048, 4096)])
def test_create_refuses_hop_not_below_n_fft(n_fft, hop):
    """hop_length == n_fft: the reference's "same" ISTFT returns a (B, 0) signal, the overlap-add would divide by a zero
    envelope; st_create_vocos refuses it before touching the device"""
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    h = C.c_void_p()
    assert lib.st_create_vocos(C.byref(_lib.StVocosDims(128, 512, 1536, 8, n_fft, hop)), 0, C.byref(h)) != 0
    err = lib.st_last_error(None).decode()
    assert ("empty (B, 0)" in err) if n_fft % hop == 0 else ("multiple of 128 and of hop_length" in err), err


def _model(dev, engine="tcgen05", head_gain=0.5, **dims):
    from stabletts_b200 import Vocos
    d = dict(V.DIMS); d.update(dims)
    m = Vocos(**d).eval()
    m.load_state_dict(V.make_state(head_gain=head_gain, **dims), strict=True)
    m = m.to(dev)
    m.set_engine(engine)
    return m


ALL_CASES = {**V.CASES, **V.API_CASES}
BAR = {"tcgen05": 1e-3, "simt": 2e-4}


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("name", list(ALL_CASES))
def test_vocos_vs_reference_golden(name, engine, dev, golden_dir):
    cs = ALL_CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    m = _model(dev, engine, **cs.get("state", {}))
    mel = V.make_mel(cs["seed"], cs["B"], cs["T"])
    audio = m(mel.to(dev))
    ref = torch.from_numpy(g["audio"])
    assert audio.shape == ref.shape == (cs["B"], cs["T"] * 512)
    e = rel_errs(audio, ref)
    print(f"{name} {engine}: max-rel {e[0]:.2e} l2-rel {e[1]:.2e}")
    assert max(e) < BAR[engine], (name, engine, e)
    assert torch.isfinite(audio).all()


def _vs_oracle(dev, engine, mel, head_gain=0.5, **dims):
    d = dict(V.DIMS); d.update(dims)
    m = _model(dev, engine, head_gain=head_gain, **dims)
    st = V.make_state(head_gain=head_gain, **dims)
    with torch.inference_mode():
        ref = V.vocos_forward(st, mel, d["n_fft"], d["hop_length"])
    audio = m(mel.to(dev)).cpu()
    assert audio.shape == ref.shape == (mel.shape[0], mel.shape[2] * d["hop_length"])
    assert torch.isfinite(audio).all()
    return rel_errs(audio, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("T", [1, 2, 3])
def test_api_config_short_inputs_vs_oracle(T, engine, dev):
    """api.py's 512 / 1536 / 8 Vocos at one to three frames: dwconv taps off both edges, an ISTFT of one to three frames"""
    e = _vs_oracle(dev, engine, V.make_mel(60 + T, 2, T), **V.API_DIMS)
    print(f"api T={T} {engine}: max-rel {e[0]:.2e} l2-rel {e[1]:.2e}")
    assert max(e) < BAR[engine], (T, engine, e)


SWEEP = [(dim, n_fft, hop) for dim in (512, 1024) for n_fft, hop in ((1024, 256), (2048, 128), (1280, 640))]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("dim,n_fft,hop", SWEEP, ids=[f"dim{d}-nfft{n}-hop{h}" for d, n, h in SWEEP])
def test_accepted_configurations_vs_oracle(dim, n_fft, hop, engine, dev):
    """two-layer Vocos across what st_create_vocos accepts: dim 1024 (dwconv_ln_kernel<1024>), 16 overlapping frames
    (2048 / 128), an n_fft that is not a power of two (1280: K = 641, K2 = 1408) and two-frame overlap (1280 / 640)"""
    e = _vs_oracle(dev, engine, V.make_mel(70 + dim // 512, 2, 37), dim=dim, intermediate_dim=2 * dim, num_layers=2,
                   n_fft=n_fft, hop_length=hop)
    print(f"dim {dim} n_fft {n_fft} hop {hop} {engine}: max-rel {e[0]:.2e} l2-rel {e[1]:.2e}")
    assert max(e) < BAR[engine], (dim, n_fft, hop, engine, e)


@pytest.mark.gpu
def test_drop_in_refuses_hop_equal_to_n_fft(dev):
    from stabletts_b200 import Vocos
    m = Vocos(dim=512, intermediate_dim=1536, num_layers=1, n_fft=1024, hop_length=1024).eval().to(dev)
    with pytest.raises(RuntimeError, match=r"empty \(B, 0\)"):
        m(torch.zeros(1, 128, 4, device=dev))


@pytest.mark.gpu
def test_vocos_large_vs_oracle_and_properties(dev):
    """B = 6, T = 700 (4200 frames: the pwconv GEMMs reach the 256-channel GEMM tiles) against the oracle on the host; an utterance's
    audio does not depend on its batch neighbours; n_mel = 80 (the CFM path's BASELINE width) works as input width."""
    st = V.make_state()
    m = _model(dev)
    mel = V.make_mel(77, 6, 700)
    audio = m(mel.to(dev)).cpu()
    with torch.inference_mode():
        ref = V.vocos_forward(st, mel[[0, 5]])
    e = rel_errs(audio[[0, 5]], ref)
    assert max(e) < 1e-3, e
    alone = m(mel[2:3].to(dev)).cpu()
    assert rel_errs(alone, audio[2:3])[0] < 1e-5
    m80 = _model(dev, input_channels=80)
    st80 = V.make_state(input_channels=80)
    mel80 = V.make_mel(78, 2, 130, n_mel=80)
    with torch.inference_mode():
        ref80 = V.vocos_forward(st80, mel80)
    assert max(rel_errs(m80(mel80.to(dev)), ref80)) < 1e-3
    assert m(torch.zeros(0, 128, 5, device=dev)).shape == (0, 2560)
