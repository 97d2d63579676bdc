"""Resampling: the drop-in `resample`, `Resample` and `load_and_resample_audio` on the polyphase kernel (resample.cu).

CPU: the float64 oracle (oracle/resample_ref.py) against fixtures from torchaudio (tests/golden/rs_*.npz; recipe
oracle/make_golden_resample.py), the package's default table against torchaudio's coefficients, the state_dict, the
refusals and load_and_resample_audio through a fake decoder.
GPU: every fixture within 1e-6 max|x| of the float64 result (the default table and torchaudio's loaded buffer), a 10-minute
clip, input shapes and strides, exact properties (determinism, batch independence, CUDA-graph replay, devices) and the
composition 48 kHz -> resample -> LogMelSpectrogram against the float64 chain."""
import os

import numpy as np
import pytest
import torch

from oracle import mel_ref, resample_ref as R


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _wave(cs):
    return R.make_batch(cs["kinds"], cs["seed"], cs["L"], cs["orig"])


_PAIR_CASES = [n for n in R.CASES if n.count("_") == 2]                    # one full-length case per rate pair
# the rates api.py and preprocess.py meet (corpora at 48 / 24 / 16 / 22.05 / 8 / 96 kHz, and 44.1 kHz down)
_COMMON = ["rs_48000_44100", "rs_24000_44100", "rs_16000_44100", "rs_22050_44100", "rs_8000_44100", "rs_96000_44100",
           "rs_44100_16000", "rs_44100_22050", "rs_44100_24000", "rs_192000_16000"]


# ------------------------------------------------------------------ CPU ------------------------------------------------------

@pytest.mark.parametrize("name", list(R.CASES))
def test_oracle_vs_torchaudio_golden(name, golden_dir):
    cs, g = R.CASES[name], _golden(golden_dir, name)
    x = _wave(cs)
    np.testing.assert_allclose(R.checksum(x), g["wave_checksum"], rtol=1e-12)
    out = R.resample(x, cs["orig"], cs["new"])
    ref = torch.from_numpy(g["out64"])
    assert out.shape == ref.shape and out.shape[-1] == R.out_length(cs["orig"], cs["new"], cs["L"])
    assert float((out - ref).abs().max()) <= 1e-12


@pytest.mark.parametrize("name", _PAIR_CASES)
def test_default_table_is_the_float64_kernel_rounded_once(name, golden_dir):
    from stabletts_b200 import Resample
    from stabletts_b200.resample import band_table, default_kernel
    cs, g = R.CASES[name], _golden(golden_dir, name)
    k64 = torch.from_numpy(g["kernel64"])
    assert torch.equal(default_kernel(cs["orig"], cs["new"]), k64)
    assert torch.equal(Resample(cs["orig"], cs["new"]).kernel, k64)
    k0, coef, width = band_table(cs["orig"], cs["new"])                     # every non-zero tap lies in its phase's band
    O, N, w, _ = R.dims(cs["orig"], cs["new"])
    assert width == w and coef.shape[0] == N and N * coef.shape[1] <= 1 << 18
    outside = k64[:, 0].clone()
    outside.scatter_(1, (k0[:, None] + torch.arange(coef.shape[1])[None]).clamp(max=2 * w + O - 1), 0.0)
    assert not outside.any()


@pytest.mark.parametrize("name", _PAIR_CASES)
def test_default_kernel_vs_torchaudio_buffer(name, golden_dir):
    """torchaudio.transforms.Resample evaluates j / N in fp32: the formula with that one term in fp32 gives its buffer bit
    for bit, and at the common rates the float64 default is within 1e-5 of it (more where base = 0.99 min(O, N) is large
    and amplifies the fp32 rounding of j / N: 1.3e-5 at 32 -> 44.1 kHz, 3.3e-5 at 12345 -> 44.1 kHz)."""
    from stabletts_b200 import Resample
    cs, g = R.CASES[name], _golden(golden_dir, name)
    ta = torch.from_numpy(g["kernel"])
    assert torch.equal(R.coefficients(cs["orig"], cs["new"], torch.float32).float().unsqueeze(1), ta)
    d = float((Resample(cs["orig"], cs["new"]).kernel - ta).abs().max())
    O, N, _, base = R.dims(cs["orig"], cs["new"])
    assert d <= (1e-5 if name in _COMMON else max(1e-5, base * 2.0 ** -23)), d


def test_state_dict_matches_torchaudio(golden_dir):
    import torchaudio
    from stabletts_b200 import Resample
    m = Resample(48000, 44100)
    ta = torchaudio.transforms.Resample(48000, 44100)
    sd = m.state_dict()
    assert list(sd) == list(ta.state_dict()) == ["kernel"]
    assert sd["kernel"].shape == ta.state_dict()["kernel"].shape == (147, 1, 2 * 7 + 160)
    assert sd["kernel"].dtype == torch.float32 and list(m.parameters()) == []
    assert (m.orig_freq, m.new_freq, m.gcd, m.width) == (ta.orig_freq, ta.new_freq, ta.gcd, ta.width)
    m.load_state_dict(ta.state_dict(), strict=True)
    assert torch.equal(m.kernel, ta.kernel)
    ta.load_state_dict(Resample(48000, 44100).state_dict(), strict=True)
    assert list(Resample(44100, 44100).state_dict()) == list(torchaudio.transforms.Resample(44100, 44100).state_dict()) == []


@pytest.mark.parametrize("kw", [dict(resampling_method="sinc_interp_kaiser"), dict(lowpass_filter_width=16),
                                dict(rolloff=0.95), dict(beta=8.0)])
def test_refused_methods(kw):
    from stabletts_b200 import Resample, resample
    with pytest.raises(ValueError):
        resample(torch.zeros(1, 100), 48000, 44100, **kw)
    with pytest.raises(ValueError):
        Resample(48000, 44100, **kw)


@pytest.mark.parametrize("pair", [(44100.5, 16000), (48000, 44100.25), (0, 16000), (16000, -1), ("48000", 44100),
                                  (44101, 44100), (1, 999999937)])
def test_refused_rates(pair):
    """non-integer or non-positive rates, and pairs whose table exceeds ST_RESAMPLE_MAX_TABLE (N x band)"""
    from stabletts_b200 import Resample, resample
    with pytest.raises(ValueError):
        resample(torch.zeros(1, 100), *pair)
    with pytest.raises(ValueError):
        Resample(*pair)


def test_refused_inputs():
    from stabletts_b200 import Resample, resample
    m = Resample(48000, 44100)
    for fn in (lambda x: resample(x, 48000, 44100), m):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(torch.zeros(1, 100))
        with pytest.raises(TypeError):
            fn(torch.zeros(1, 100, dtype=torch.float64))
        with pytest.raises(TypeError):
            fn(torch.zeros(1, 100, dtype=torch.float16))
        with pytest.raises(RuntimeError, match="backward"):
            fn(torch.zeros(1, 100, requires_grad=True))


def test_same_rate_returns_the_input():
    from stabletts_b200 import Resample, resample
    x = torch.randn(2, 50)
    assert resample(x, 44100, 44100) is x
    assert resample(x, 44100.0, 44100) is x
    assert Resample(22050, 22050)(x) is x


def test_load_and_resample_audio_with_a_fake_decoder(monkeypatch, capsys):
    import torchaudio
    from stabletts_b200 import load_and_resample_audio
    stereo = torch.randn(2, 300)

    def fake_load(path):
        if path == "broken.wav":
            raise RuntimeError("cannot decode broken.wav")
        return (stereo if path == "stereo.wav" else stereo[:1]), 44100

    monkeypatch.setattr(torchaudio, "load", fake_load)
    y = load_and_resample_audio("stereo.wav", 44100)
    assert y.shape == (1, 300) and y.device.type == "cpu" and torch.equal(y, stereo[:1])
    assert torch.equal(load_and_resample_audio("mono.wav", 44100, device="cpu"), stereo[:1])
    assert load_and_resample_audio("broken.wav", 44100) is None
    assert "cannot decode broken.wav" in capsys.readouterr().out
    if not torch.cuda.is_available():                                       # resampling needs the GPU: no CPU fallback
        with pytest.raises((RuntimeError, AssertionError)):
            load_and_resample_audio("stereo.wav", 16000)


# ------------------------------------------------------------------ GPU ------------------------------------------------------

def _bar(x):
    return 1e-6 * float(x.abs().max())


@pytest.mark.gpu
def test_gpu_vs_torchaudio_golden(golden_dir):
    from stabletts_b200 import resample
    worst = []
    for name, cs in R.CASES.items():
        g = _golden(golden_dir, name)
        x = _wave(cs)
        out = resample(x.cuda(), cs["orig"], cs["new"])
        ref = torch.from_numpy(g["out64"])
        assert out.shape == ref.shape and out.dtype == torch.float32
        err = float((out.double().cpu() - ref).abs().max())
        bar = _bar(x)
        worst.append((err / bar, name, err, float(g["E32"])))
        assert err <= bar, (name, err, bar)
    r, name, err, e32 = max(worst)
    print(f"[resample] worst ratio to the bar {r:.3f} ({name}: {err:.3e}; torchaudio's fp32 error there {e32:.3e})")


@pytest.mark.gpu
def test_gpu_module_with_torchaudio_buffer(golden_dir):
    """Resample with torchaudio's loaded buffer, against the float64 result over that buffer; the default module equals the
    function bit for bit (the module packs the same table from its dense buffer)."""
    from stabletts_b200 import Resample, resample
    worst = []
    for name in _PAIR_CASES:
        cs, g = R.CASES[name], _golden(golden_dir, name)
        x = _wave(cs)
        m = Resample(cs["orig"], cs["new"])
        assert torch.equal(m.cuda()(x.cuda()), resample(x.cuda(), cs["orig"], cs["new"]))
        m.load_state_dict({"kernel": torch.from_numpy(g["kernel"])})
        out = m.cuda()(x.cuda())
        ref = R.resample(x, cs["orig"], cs["new"], coef=torch.from_numpy(g["kernel"]))
        err = float((out.double().cpu() - ref).abs().max())
        worst.append((err / _bar(x), name, err))
        assert err <= _bar(x), (name, err)
        m.kernel.mul_(2.0)                                                  # an in-place update is re-packed (and
        assert torch.equal(m(x.cuda()), 2 * out)                            # doubling every tap is exact in fp32)
    r, name, err = max(worst)
    print(f"[Resample, torchaudio's buffer] worst ratio to the bar {r:.3f} ({name}: {err:.3e})")


@pytest.mark.gpu
def test_gpu_ten_minute_clip_and_shapes():
    from stabletts_b200 import resample
    L = 600 * 48000
    x = R.make_batch(["speech"], 900, L, 48000)
    y = resample(x.cuda(), 48000, 44100)
    n = R.out_length(48000, 44100, L)
    assert y.shape == (1, n)
    pos = [0, 1, 146, 147, 5000, 12_345_677, n // 2 + 3, n - 148, n - 2, n - 1]
    err = float((y[:, pos].double().cpu() - R.resample_at(x, 48000, 44100, pos)).abs().max())
    print(f"[resample 10 min] {L} -> {n}, sampled outputs max abs {err:.3e}")
    assert err <= _bar(x)
    base = R.make_batch(["noise", "sine", "square", "nyquist", "noise", "sine"], 901, 7001, 24000)
    for shape in [(7001,), (6, 1, 7001), (2, 3, 7001)]:
        xs = base.reshape(shape) if len(shape) > 1 else base[0]
        out = resample(xs.cuda(), 24000, 44100)
        ref = R.resample(xs, 24000, 44100)
        assert out.shape == ref.shape == (*shape[:-1], R.out_length(24000, 44100, 7001))
        assert float((out.double().cpu() - ref).abs().max()) <= _bar(xs)
    wide = R.make_batch(["noise", "sine"], 902, 2 * 9000, 16000).cuda()
    strided = wide[:, ::2]                                                  # a non-contiguous view
    assert not strided.is_contiguous()
    out = resample(strided, 16000, 44100)
    assert torch.equal(out, resample(strided.contiguous(), 16000, 44100))
    assert float((out.double().cpu() - R.resample(strided.cpu(), 16000, 44100)).abs().max()) <= _bar(strided)
    assert resample(wide[:0], 16000, 44100).shape == (0, R.out_length(16000, 44100, 18000))
    assert resample(wide[:, :0], 16000, 44100).shape == (2, 0)


@pytest.mark.gpu
def test_gpu_exact_properties():
    from stabletts_b200 import resample
    for o, n in [(48000, 44100), (16000, 44100), (192000, 16000), (12345, 44100)]:
        x = R.make_batch(["noise", "sine", "square", "silence"], 903, 20011, o).cuda()
        full = resample(x, o, n)
        assert torch.equal(resample(x, o, n), full)                         # a repeated call is bitwise identical
        for b in range(x.shape[0]):                                         # an utterance alone equals its batch row
            assert torch.equal(resample(x[b], o, n), full[b])
        assert not full[3].any()
    x = R.make_batch(["noise", "speech"], 904, 48000, 48000).cuda()
    y = resample(x, 48000, 44100)
    static = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        resample(static, 48000, 44100)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gy = resample(static, 48000, 44100)
    x2 = R.make_batch(["sine", "noise"], 905, 48000, 48000).cuda()
    static.copy_(x2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gy, resample(x2, 48000, 44100))
    static.copy_(x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gy, y)


@pytest.mark.gpu
def test_gpu_devices_and_refusals(monkeypatch):
    import torchaudio
    from stabletts_b200 import Resample, load_and_resample_audio, resample
    last = torch.cuda.device_count() - 1
    torch.cuda.set_device(0)
    x = R.make_batch(["noise"], 906, 4807, 48000)
    y = resample(x.to(f"cuda:{last}"), 48000, 44100)
    assert y.device == torch.device(f"cuda:{last}") and torch.cuda.current_device() == 0
    assert float((y.double().cpu() - R.resample(x, 48000, 44100)).abs().max()) <= _bar(x)
    m = Resample(48000, 44100).to(f"cuda:{last}")
    assert torch.equal(m(x.to(f"cuda:{last}")), y) and torch.cuda.current_device() == 0
    with pytest.raises(TypeError):
        resample(x.cuda().double(), 48000, 44100)
    with pytest.raises(RuntimeError, match="backward"):
        resample(x.cuda().requires_grad_(), 48000, 44100)
    with torch.no_grad():
        assert torch.equal(resample(x.cuda().requires_grad_(), 48000, 44100), resample(x.cuda(), 48000, 44100))
    stereo = torch.cat([x, -x])
    monkeypatch.setattr(torchaudio, "load", lambda path: (stereo, 48000))
    ref = resample(x.cuda(), 48000, 44100)
    a = load_and_resample_audio("clip.wav", 44100)                          # api.py: no device, then .to(device)
    assert a.device.type == "cpu" and torch.equal(a, ref.cpu())
    b = load_and_resample_audio("clip.wav", 44100, device=torch.device("cuda"))   # preprocess.py
    assert b.device.type == "cuda" and torch.equal(b, ref)


@pytest.mark.gpu
def test_gpu_composed_with_log_mel(golden_dir):
    """48 kHz -> resample -> LogMelSpectrogram (preprocess.py:65 then :73), both this library's, against the float64 chain
    of torchaudio and the reference module: within max(1e-4, 4 E32), the rule of tests/test_mel.py"""
    from stabletts_b200 import LogMelSpectrogram, resample
    cs = R.COMPOSED
    g = _golden(golden_dir, cs["name"])
    x = _wave(cs)
    np.testing.assert_allclose(R.checksum(x), g["wave_checksum"], rtol=1e-12)
    mel = LogMelSpectrogram(**mel_ref.CONFIGS["default"])
    mel.mel_scale.fb.copy_(torch.from_numpy(g["fb"]))
    out = mel.cuda()(resample(x.cuda(), cs["orig"], cs["new"]))
    ref = torch.from_numpy(g["out64"])
    err = float((out.double().cpu() - ref).abs().max())
    bar = max(1e-4, 4 * float(g["E32"]))
    print(f"[resample -> log-mel] max abs {err:.3e}, bar {bar:.3e} (E32 {float(g['E32']):.3e})")
    assert out.shape == ref.shape and err <= bar
