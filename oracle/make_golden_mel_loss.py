"""Fixtures of the multi-scale mel loss from the UNMODIFIED reference module vocoders/vocos/models/loss.py, imported as
vocoders/vocos/train.py imports it (sys.path at vocoders/vocos):

    STABLETTS_REFERENCE_DIR=<checkout> python oracle/make_golden_mel_loss.py      # writes tests/golden/mlw_*.npz

For each case of oracle/mel_loss_ref.py: the loss and d loss / dy (and d loss / dx where the case asks) from the module in
fp32 and in float64 (the module and inputs cast with .double()), `E32_*` = the reference's own fp32 error (loss: absolute;
gradient: L2 and max-norm relative), every scale's fb, the waveform checksum, and `flip_bound` (oracle.mel_loss_ref.flip_bound
of the float64 Δ).  Needs torchaudio."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
from oracle import mel_loss_ref as R, mel_ref as M        # noqa: E402
from oracle.stage_reference import REF                     # noqa: E402


def _import_reference():
    if not REF or not os.path.isdir(REF):
        raise SystemExit("set STABLETTS_REFERENCE_DIR to a checkout of the reference")
    for mod in [k for k in sys.modules if k in ("config", "utils", "models") or k.startswith(("utils.", "models."))]:
        del sys.modules[mod]
    sys.path.insert(0, os.path.join(REF, "vocoders", "vocos"))
    from models.loss import MultiScaleMelSpectrogramLoss, SingleScaleMelSpectrogramLoss
    return MultiScaleMelSpectrogramLoss, SingleScaleMelSpectrogramLoss


def _run(module, x, y, grad_x, dtype):
    xd, yd = x.detach().to(dtype).clone().requires_grad_(grad_x), y.detach().to(dtype).clone().requires_grad_(True)
    loss = module.to(dtype)(xd, yd)
    loss.backward()
    return loss.detach(), (xd.grad if grad_x else None), yd.grad


def _errs(g32, g64):
    d = g32.double() - g64
    return float(d.norm() / g64.norm()), float(d.abs().max() / g64.abs().max())


def main():
    Multi, Single = _import_reference()
    for name, cs in R.CASES.items():
        m = Multi() if cs["scales"] == "multi" else Single()
        transforms = list(m.mel_transforms) if cs["scales"] == "multi" else [m.mel_transform]
        cfgs = R.scale_configs(cs)
        for t, c in zip(transforms, cfgs):                  # the oracle's configs are the module's
            assert (t.n_fft, t.hop_length, t.pad, t.n_mels) == (c["n_fft"], c["hop_length"], c["pad"], c["n_mels"]), name
        fbs = [t.mel_scale.fb.detach().float().clone() for t in transforms]
        assert all(float(fb.abs().sum(0).min()) > 0 for fb in fbs), "an all-zero filter"
        x, y = R.make_pair(cs)
        gx_on = cs.get("grad_x", False)
        l32, gx32, gy32 = _run(m, x, y, gx_on, torch.float32)
        l64, gx64, gy64 = _run(m, x, y, gx_on, torch.float64)
        wins = R.hann_windows(cfgs)
        deltas = [(a - b).transpose(1, 2) for a, b in zip(R.log_mels(x, wins, fbs, cfgs), R.log_mels(y, wins, fbs, cfgs))]
        if "half_rows" in cs:       # y = x / 2: Δ near log 2 where neither side clamps, 0 where both do, in (0, log 2] between
            mx = [R._scale_forward(x.double(), w.double(), fb.double(), c)[2] for w, fb, c in zip(wins, fbs, cfgs)]
            my = [R._scale_forward(y.double(), w.double(), fb.double(), c)[2] for w, fb, c in zip(wins, fbs, cfgs)]
            for r in cs["half_rows"]:
                for d, a, b in zip(deltas, mx, my):
                    ca, cb = a[r] < 1e-5, b[r] < 1e-5
                    assert bool(((d[r] - np.log(2)).abs() < 0.05)[~ca & ~cb].all()), name
                    assert bool((d[r][ca & cb] == 0).all()), name
                    only = d[r][~ca & cb]
                    assert bool(((only > 0) & (only <= np.log(2) + 1e-12)).all()), name
        if "equal_rows" in cs:
            for r in cs["equal_rows"]:
                assert all(bool((d[r] == 0).all()) for d in deltas)
        fb_bound = R.flip_bound(y, deltas, wins, fbs, cfgs)
        e_l2, e_max = _errs(gy32, gy64)
        small = sum(int((d.abs() <= 1e-4).sum()) for d in deltas)
        zero = sum(int((d == 0).sum()) for d in deltas)
        print(f"{name}: loss {float(l64):.6f}, E32 loss {abs(float(l32) - float(l64)):.2e}, grad L2 {e_l2:.2e} max {e_max:.2e}, "
              f"|Δ| <= 1e-4: {small} (== 0: {zero}), flip_bound {fb_bound:.3e} (||gy|| {float(gy64.norm()):.3e})")
        out = dict(loss32=float(l32), loss64=float(l64), gy32=gy32.numpy(), gy64=gy64.numpy(),
                   E32_loss=abs(float(l32) - float(l64)), E32_grad_l2=e_l2, E32_grad_max=e_max, flip_bound=fb_bound,
                   wave_checksum=np.concatenate([M.checksum(x), M.checksum(y)]), n_scales=len(fbs))
        if gx_on:
            out.update(gx32=gx32.numpy(), gx64=gx64.numpy(), E32_gradx_l2=_errs(gx32, gx64)[0], E32_gradx_max=_errs(gx32, gx64)[1])
        for i, fb in enumerate(fbs):
            out[f"fb{i}"] = fb.numpy()
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)


if __name__ == "__main__":
    main()
