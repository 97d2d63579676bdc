"""The multi-scale mel loss of the Vocos trainer: MultiScaleMelSpectrogramLoss / SingleScaleMelSpectrogramLoss on the
mel_loss.cu kernels, forward and waveform gradient.

CPU: the float64 oracle with its explicit adjoint (oracle/mel_loss_ref.py) against the fixtures of the unmodified reference
module (tests/golden/mlw_*.npz; recipe oracle/make_golden_mel_loss.py) and against torch autograd, the state_dict
inventory, the refusals.
GPU: the loss against the reference's float64 loss, the gradient against the oracle with the sign and clamp masks taken from
the drop-in LogMelSpectrogram and against the reference's float64 autograd, the small-FFT log-mels, exact properties
(x = y, determinism, batch rows, finite differences, no gradient work under no_grad) and a small generator trained through
the loss.  Bars: E32 is the reference module's own fp32 error on the same case."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_errs
from oracle import mel_loss_ref as R, mel_ref as M


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _fbs(g):
    return [torch.from_numpy(g[f"fb{i}"]) for i in range(int(g["n_scales"]))]


def _case(name, golden_dir):
    cs, g = R.CASES[name], _golden(golden_dir, name)
    cfgs = R.scale_configs(cs)
    x, y = R.make_pair(cs)
    np.testing.assert_allclose(np.concatenate([M.checksum(x), M.checksum(y)]), g["wave_checksum"], rtol=1e-12)
    return cs, g, cfgs, x, y


# ------------------------------------------------------------------ CPU ------------------------------------------------------

@pytest.mark.parametrize("name", list(R.CASES))
def test_oracle_vs_reference_golden(name, golden_dir):
    cs, g, cfgs, x, y = _case(name, golden_dir)
    loss, gx, gy = R.gradients(x, y, R.hann_windows(cfgs), _fbs(g), cfgs)
    assert abs(float(loss) - float(g["loss64"])) <= 1e-9
    ref = torch.from_numpy(g["gy64"])
    assert float((gy - ref).abs().max()) <= 1e-9 * float(ref.abs().max())
    if "gx64" in g:
        refx = torch.from_numpy(g["gx64"])
        assert float((gx - refx).abs().max()) <= 1e-9 * float(refx.abs().max())
        assert float((gx + gy)[0].abs().max()) == 0.0                        # the x = y row: Δ ≡ 0, no gradient


def test_oracle_adjoint_vs_autograd():
    """The explicit adjoint against torch autograd of the same float64 forward, with pad > 0 at every scale (a short input:
    both reflect pads fold into the frames of the largest scale)."""
    cfgs = R.MULTI
    fbs = [M.slaney_fb(c) for c in cfgs]
    wins = R.hann_windows(cfgs)
    x, y = R.make_pair(dict(B=2, L=1500, kind="noise", seed=7, noise=0.05))
    xd, yd = x.double().requires_grad_(), y.double().requires_grad_()
    R.loss(xd, yd, wins, fbs, cfgs).backward()
    loss, gx, gy = R.gradients(x, y, wins, fbs, cfgs)
    assert abs(float(loss) - float(R.loss(x, y, wins, fbs, cfgs))) <= 1e-12
    for a, b in ((gx, xd.grad), (gy, yd.grad)):
        assert float((a - b).abs().max()) <= 1e-12 * float(b.abs().max())


def test_oracle_masks_are_honoured():
    """Injected signs and clamp masks replace the oracle's own: all-zero signs give zero gradients, flipped signs negate."""
    cfgs = R.MULTI[:3]
    fbs = [M.slaney_fb(c) for c in cfgs]
    wins = R.hann_windows(cfgs)
    x, y = R.make_pair(dict(B=1, L=600, kind="noise", seed=8, noise=0.05))
    _, gx, gy = R.gradients(x, y, wins, fbs, cfgs)
    deltas = [(a - b).transpose(1, 2) for a, b in zip(R.log_mels(x, wins, fbs, cfgs), R.log_mels(y, wins, fbs, cfgs))]
    _, fx, fy = R.gradients(x, y, wins, fbs, cfgs, signs=[-torch.sign(d) for d in deltas])
    assert torch.allclose(fx, -gx, rtol=0, atol=1e-15) and torch.allclose(fy, -gy, rtol=0, atol=1e-15)
    _, zx, zy = R.gradients(x, y, wins, fbs, cfgs, signs=[torch.zeros_like(d) for d in deltas])
    assert float(zx.abs().max()) == 0 and float(zy.abs().max()) == 0


def test_state_dict_matches_reference_inventory(golden_dir):
    from stabletts_b200 import LogMelSpectrogram, MultiScaleMelSpectrogramLoss, SingleScaleMelSpectrogramLoss
    g = _golden(golden_dir, "mlw_b2_segment")
    m = MultiScaleMelSpectrogramLoss()
    sd = m.state_dict()
    keys = [f"mel_transforms.{i}.{k}" for i in range(7) for k in ("spectrogram.window", "mel_scale.fb")]
    assert list(sd) == keys
    assert isinstance(m.mel_transforms, torch.nn.ModuleList) and all(isinstance(t, LogMelSpectrogram) for t in m.mel_transforms)
    assert list(m.parameters()) == []
    for i, (nm, w) in enumerate(zip(R.N_MELS, R.WINDOWS)):
        ref = torch.from_numpy(g[f"fb{i}"])
        assert tuple(sd[f"mel_transforms.{i}.mel_scale.fb"].shape) == (w // 2 + 1, nm)
        assert rel_errs(sd[f"mel_transforms.{i}.mel_scale.fb"], ref)[0] <= 1e-5         # float64 formulas vs torchaudio's fp32
        assert torch.equal(sd[f"mel_transforms.{i}.spectrogram.window"], torch.hann_window(w))
        t = m.mel_transforms[i]
        assert (t.n_fft, t.hop_length, t.pad) == (w, w // 4, (w - w // 4) // 2)
    m.load_state_dict({k: (torch.from_numpy(g[f"fb{int(k.split('.')[1])}"]) if k.endswith("fb") else v) for k, v in sd.items()},
                      strict=True)
    assert torch.equal(m.mel_transforms[0].mel_scale.fb, torch.from_numpy(g["fb0"]))
    s = SingleScaleMelSpectrogramLoss()
    assert list(s.state_dict()) == ["mel_transform.spectrogram.window", "mel_transform.mel_scale.fb"]
    assert tuple(s.state_dict()["mel_transform.mel_scale.fb"].shape) == (1025, 128)


def test_refusals():
    from stabletts_b200 import MultiScaleMelSpectrogramLoss
    with pytest.raises(AssertionError):
        MultiScaleMelSpectrogramLoss(n_mels=[5, 10], window_lengths=[32])
    with pytest.raises(ValueError):
        MultiScaleMelSpectrogramLoss(n_mels=[5], window_lengths=[16])                   # n_fft below 32
    with pytest.raises(ValueError):
        MultiScaleMelSpectrogramLoss(n_mels=[5], window_lengths=[48])                   # not a power of two
    m = MultiScaleMelSpectrogramLoss()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 4096), torch.randn(1, 4096))


# ------------------------------------------------------------------ GPU ------------------------------------------------------

def _module(cs, g):
    from stabletts_b200 import MultiScaleMelSpectrogramLoss, SingleScaleMelSpectrogramLoss
    m = MultiScaleMelSpectrogramLoss() if cs["scales"] == "multi" else SingleScaleMelSpectrogramLoss()
    ts = list(m.mel_transforms) if cs["scales"] == "multi" else [m.mel_transform]
    for t, fb in zip(ts, _fbs(g)):
        t.mel_scale.fb.copy_(fb)
    return m.cuda(), ts


def _masks(ts, x, y):
    """sgn(Δ) and the clamp masks [mel >= 1e-5] from the drop-in LogMelSpectrogram's fp32 outputs, (B, T, m) per scale"""
    floor = float(torch.tensor(1e-5, dtype=torch.float32).log())
    signs, cx, cy = [], [], []
    with torch.no_grad():
        for t in ts:
            lx, ly = t(x).transpose(1, 2).double().cpu(), t(y).transpose(1, 2).double().cpu()
            signs.append(torch.sign(lx - ly))
            cx.append(lx > floor)
            cy.append(ly > floor)
    return signs, cx, cy


def _run(m, x, y, grad_x=False):
    xd = x.detach().cuda().clone().requires_grad_(grad_x)
    yd = y.detach().cuda().clone().requires_grad_(True)
    loss = m(xd, yd)
    loss.backward()
    return loss.detach(), (xd.grad if grad_x else None), yd.grad


# bars: the first H100 run measured the ratios printed by these tests; the floors keep more than a 2x margin (DESIGN.md §8 f9)
GRAD_FLOOR_L2, GRAD_FLOOR_MAX = 1e-5, 3e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(R.CASES))
def test_gpu_vs_reference_and_oracle(name, golden_dir):
    cs, g, cfgs, x, y = _case(name, golden_dir)
    m, ts = _module(cs, g)
    gx_on = "gx64" in g
    loss, gx, gy = _run(m, x, y, gx_on)
    # loss against the reference's float64 loss
    l64 = float(g["loss64"])
    el, bl = abs(float(loss) - l64), max(1e-6 * l64, 4 * float(g["E32_loss"]))
    # gradient against the reference's float64 autograd: its own fp32 error plus what sign ties can move
    ref = torch.from_numpy(g["gy64"])
    e_ref = float((gy.double().cpu() - ref).norm())
    b_ref = 4 * float(g["E32_grad_l2"]) * float(ref.norm()) + float(g["flip_bound"])
    # gradient against the oracle with the drop-in's own signs and clamp masks
    signs, cx, cy = _masks(ts, x.cuda(), y.cuda())
    _, ox, oy = R.gradients(x, y, R.hann_windows(cfgs), _fbs(g), cfgs, signs=signs, clamps_x=cx, clamps_y=cy)
    e_max, e_l2 = rel_errs(gy, oy)
    b_l2, b_max = max(GRAD_FLOOR_L2, 4 * float(g["E32_grad_l2"])), max(GRAD_FLOOR_MAX, 4 * float(g["E32_grad_max"]))
    print(f"[mel loss {name}] loss |d| {el:.2e} / bar {bl:.2e} ({el / bl:.3f}); grad vs ref64 L2 {e_ref:.2e} / {b_ref:.2e} "
          f"({e_ref / b_ref:.3f}); grad vs oracle L2 rel {e_l2:.2e} / {b_l2:.2e} ({e_l2 / b_l2:.3f}), max rel {e_max:.2e} / "
          f"{b_max:.2e} ({e_max / b_max:.3f})")
    assert el <= bl
    assert e_ref <= b_ref
    assert e_l2 <= b_l2 and e_max <= b_max
    if gx_on:
        ex_max, ex_l2 = rel_errs(gx, ox)
        bx_l2, bx_max = max(GRAD_FLOOR_L2, 4 * float(g["E32_gradx_l2"])), max(GRAD_FLOOR_MAX, 4 * float(g["E32_gradx_max"]))
        print(f"[mel loss {name}] grad x vs oracle L2 rel {ex_l2:.2e} / {bx_l2:.2e}, max rel {ex_max:.2e} / {bx_max:.2e}")
        assert ex_l2 <= bx_l2 and ex_max <= bx_max
        assert float((gx + gy)[0].abs().max()) == 0.0                        # the x = y row


@pytest.mark.gpu
@pytest.mark.parametrize("n_fft,n_mels", [(32, 5), (64, 10), (128, 20)])
def test_gpu_small_fft_log_mel(n_fft, n_mels):
    """The new small sizes of LogMelSpectrogram against the float64 oracle under test_mel.py's max(1e-4, 4 E32) rule."""
    from stabletts_b200 import LogMelSpectrogram
    cfg = R.scale_config(n_mels, n_fft)
    fb = M.slaney_fb(cfg).float()
    win = torch.hann_window(n_fft)
    x = M.make_batch(["noise", "speech", "quiet", "lowpass"], 501, 5000)
    m = LogMelSpectrogram(**cfg)
    m.mel_scale.fb.copy_(fb)
    out = m.cuda()(x.cuda()).double().cpu()
    ref = M.log_mel(x, win, fb, cfg)
    e32 = float((M.log_mel(x, win, fb, cfg, torch.float32).double() - ref).abs().max())
    err, bar = float((out - ref).abs().max()), max(1e-4, 4 * e32)
    print(f"[mel n_fft {n_fft}] max abs {err:.3e}, bar {bar:.3e}")
    assert out.shape == ref.shape and err <= bar
    for b in range(x.shape[0]):                                              # an utterance alone equals its batch row
        assert torch.equal(m(x[b:b + 1].cuda())[0].double().cpu(), out[b])
    x1 = M.make_batch(["noise"], 502, cfg["pad"] + 1)                        # the shortest legal input
    err1 = float((m(x1.cuda()).double().cpu() - M.log_mel(x1, win, fb, cfg)).abs().max())
    assert err1 <= max(1e-4, 4 * float((M.log_mel(x1, win, fb, cfg, torch.float32).double() - M.log_mel(x1, win, fb, cfg)).abs().max()))


@pytest.mark.gpu
def test_gpu_loss_log_mels_are_the_modules():
    """sgn(Δ) of the loss is decided on LogMelSpectrogram's own log-mels: a loss over one scale equals the mean |Δ| of the
    module's outputs (summed in double)."""
    from stabletts_b200 import MultiScaleMelSpectrogramLoss
    x, y = R.make_pair(dict(B=3, L=6000, kind="speech", seed=9, noise=0.01))
    x, y = x.cuda(), y.cuda()
    for nm, w in zip(R.N_MELS, R.WINDOWS):
        m = MultiScaleMelSpectrogramLoss([nm], [w]).cuda()
        t = m.mel_transforms[0]
        with torch.no_grad():
            want = float((t(x) - t(y)).abs().double().mean())
            got = float(m(x, y))
        assert got == float(torch.tensor(want, dtype=torch.float32)), (w, got, want)


@pytest.mark.gpu
def test_gpu_exact_properties():
    from stabletts_b200 import MultiScaleMelSpectrogramLoss
    m = MultiScaleMelSpectrogramLoss().cuda().train()
    x, y = R.make_pair(dict(B=4, L=9000, kind="speech", seed=11, noise=0.03))
    x, y = x.cuda(), y.cuda()
    # loss(x, x) == 0 and its gradient is zero
    l0, gx0, gy0 = _run(m, x, x.clone(), True)
    assert float(l0) == 0.0 and float(gx0.abs().max()) == 0.0 and float(gy0.abs().max()) == 0.0
    # bitwise repeatable
    l1, gx1, gy1 = _run(m, x, y, True)
    l2, gx2, gy2 = _run(m, x, y, True)
    assert torch.equal(l1, l2) and torch.equal(gx1, gx2) and torch.equal(gy1, gy2)
    assert torch.equal(gx1, _run(m, x, y, True)[1])
    # B = 4, a power of two: each row's gradient is 1/4 of that row's gradient alone, bit for bit
    for b in range(4):
        _, gxb, gyb = _run(m, x[b:b + 1], y[b:b + 1], True)
        assert torch.equal(gy1[b:b + 1] * 4, gyb) and torch.equal(gx1[b:b + 1] * 4, gxb)
    # (B, 1, L) in, gradients in that shape; the scalar is 0-dim
    _, gx3, gy3 = _run(m, x.unsqueeze(1), y.unsqueeze(1), True)
    assert gy3.shape == (4, 1, 9000) and torch.equal(gy3[:, 0], gy1) and l1.shape == ()
    # grad_output scales the saved gradient
    yd = y.clone().requires_grad_()
    (m(x, yd) * 15).backward()
    assert torch.equal(yd.grad, gy1 * 15)
    # no gradient work under no_grad: one launch per scale and the reduction, no gather
    n0 = m.launch_count()
    with torch.no_grad():
        ln = m(x, y.clone().requires_grad_())
    assert m.launch_count() - n0 == 8 and torch.equal(ln, l1)
    n0 = m.launch_count()
    _run(m, x, y, False)
    assert m.launch_count() - n0 == 9                                       # only y's gradient: one gather
    with pytest.raises(TypeError):
        m(x.double(), y.double())
    with pytest.raises(ValueError):
        m(x[:, :768], y[:, :768])                                           # pad = 768 at n_fft 2048: pad < L needed
    with pytest.raises(ValueError):
        m(x, y[:, :-1])


@pytest.mark.gpu
def test_gpu_finite_differences():
    """Central differences of the fp32 loss along two directions against <grad, v>, on a small input away from ties."""
    from stabletts_b200 import MultiScaleMelSpectrogramLoss
    m = MultiScaleMelSpectrogramLoss().cuda()
    x, y = R.make_pair(dict(B=1, L=3000, kind="speech", seed=13, noise=0.05))
    x, y = x.cuda(), y.cuda()
    _, _, gy = _run(m, x, y)
    gen = torch.Generator().manual_seed(14)
    for v in (gy / gy.norm(), torch.randn(y.shape, generator=gen).cuda()):
        v = v / v.norm()
        eps = 1e-3
        with torch.no_grad():
            fd = (float(m(x, y + eps * v)) - float(m(x, y - eps * v))) / (2 * eps)
        an = float((gy.double() * v.double()).sum())
        print(f"[mel loss fd] finite difference {fd:.6e}, analytic {an:.6e}")
        assert abs(fd - an) <= 2e-2 * float(gy.norm())


@pytest.mark.gpu
def test_gpu_trains_a_generator():
    """A seeded Conv1d generator makes y; loss.backward() through the drop-in fills its parameter gradients as the same
    graph does with the float64 oracle's gradient (signs and clamps from the drop-in's log-mels)."""
    from stabletts_b200 import MultiScaleMelSpectrogramLoss
    torch.manual_seed(21)
    gen = torch.nn.Sequential(torch.nn.Conv1d(4, 16, 7, padding=3), torch.nn.Tanh(), torch.nn.Conv1d(16, 1, 7, padding=3)).cuda()
    z = torch.randn(2, 4, 4096, generator=torch.Generator().manual_seed(22)).cuda()
    x = M.make_batch(["speech", "noise"], 23, 4096).cuda().unsqueeze(1)
    m = MultiScaleMelSpectrogramLoss().cuda()
    y = gen(z)
    m(x, y).backward()
    ours = [p.grad.clone() for p in gen.parameters()]
    gen.zero_grad()
    y = gen(z)
    cfgs = R.MULTI
    fbs = [t.mel_scale.fb.cpu() for t in m.mel_transforms]
    signs, cx, cy = _masks(list(m.mel_transforms), x, y.detach())
    _, _, gy = R.gradients(x.cpu(), y.detach().cpu(), R.hann_windows(cfgs), fbs, cfgs, signs=signs, clamps_x=cx, clamps_y=cy)
    y.backward(gy.view(y.shape).float().cuda())
    worst = 0.0
    for a, p in zip(ours, gen.parameters()):
        e_max, e_l2 = rel_errs(a, p.grad)
        worst = max(worst, e_l2)
        assert e_l2 <= 4 * GRAD_FLOOR_L2, e_l2
    print(f"[mel loss generator] worst parameter-gradient L2 rel {worst:.2e}")
