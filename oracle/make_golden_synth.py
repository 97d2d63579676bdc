"""Fixtures of StableTTS.synthesise and of its two front-end modules from the UNMODIFIED reference modules:

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_synth

writes tests/golden/style_*.npz (MelStyleEncoder), dp_*.npz (DurationPredictor) and synth_*.npz (the whole synthesise).
torchdiffeq is absent: the fixed-grid stand-in of make_golden_inventory.py is registered; `monotonic_align` (imported by
models/model.py, used only by the training forward) is a stub.  The CFM's initial noise is drawn from a seeded generator
in place of torch.randn_like and recorded in each fixture as `z`.

Durations are discontinuous: ceil(exp(logw)) flips when w = exp(logw) crosses an integer.  Every case asserts that each
valid token's w is at least 5e-4 w away from the nearest integer; a seed that fails is skipped for the next one, and the
seed used is recorded.  With that margin a logw within 5e-5 relative of the fixture gives the same durations.
With a fractional length_scale the output length y_lengths = (long) sum(ceil(w) * length_scale) has the same kind of
edge: when the exact total is an integer, whether an fp32 sum lands on it or just below depends on the summation order
(torch.sum's is platform-dependent).  The synthesise cases with a fractional length_scale also require every utterance's
total to be at least 1e-3 from an integer."""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import duration_ref, estimator_ref as R, style_ref, synth_ref, weights   # noqa: E402
from oracle.stage_reference import REF                                            # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
MARGIN = 5e-4


def _import_reference():
    if not os.path.isdir(REF):
        raise SystemExit("set STABLETTS_REFERENCE_DIR to a checkout of the reference")
    sys.path.insert(0, REF)
    stub = types.ModuleType("torchdiffeq")
    stub.odeint = lambda f, y0, t, method=None, rtol=None, atol=None: R.odeint_fixed(f, y0, t, method)[None]
    sys.modules.setdefault("torchdiffeq", stub)
    ma = types.ModuleType("monotonic_align")
    ma.maximum_path = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("monotonic_align is not used by synthesise"))
    sys.modules["monotonic_align"] = ma
    from models.model import StableTTS
    from models.reference_encoder import MelStyleEncoder
    from models.duration_predictor import DurationPredictor
    return StableTTS, MelStyleEncoder, DurationPredictor


def margin_ok(logw, x_mask):
    w = (torch.exp(logw) * x_mask).double()
    d = (w - torch.round(w)).abs()
    return bool(((d >= MARGIN * w) | (x_mask == 0)).all())


def total_margin_ok(logw, x_mask, length_scale):
    if float(length_scale).is_integer():               # integer frame counts: every fp32 summation order is exact
        return True
    total = (torch.ceil(torch.exp(logw) * x_mask) * length_scale).double().sum([1, 2])
    return bool(((total - total.round()).abs() >= 1e-3).all())


class SeededRandnLike:
    """torch.randn_like replaced by draws from a seeded generator, recorded (the CFM's z, models/flow_matching.py:45)."""
    def __init__(self, seed):
        self.g, self.drawn = torch.Generator().manual_seed(seed), []

    def __enter__(self):
        self.orig = torch.randn_like
        torch.randn_like = lambda t, **kw: self.drawn.append(torch.randn(t.shape, generator=self.g, dtype=t.dtype)) or self.drawn[-1].clone()
        return self

    def __exit__(self, *exc):
        torch.randn_like = self.orig


def main():
    StableTTS, MelStyleEncoder, DurationPredictor = _import_reference()
    torch.set_grad_enabled(False)
    for name, cs in style_ref.CASES.items():
        st = style_ref.make_state(n_mel=cs["n_mel"])
        m = MelStyleEncoder(cs["n_mel"], style_vector_dim=256, style_kernel_size=5, dropout=0.25).eval()
        m.load_state_dict(st, strict=True)
        y, mask = style_ref.make_inputs(cs["seed"], cs["B"], cs["T"], cs["n_mel"], cs["lens"])
        c = m(y, mask)
        assert torch.isfinite(c).all()
        np.savez_compressed(os.path.join(OUT, name + ".npz"), c=c.numpy(), weight_checksum=weights.checksum(st))
    st = duration_ref.make_state()
    dp = DurationPredictor(256, 1024, 3, 0.5, 256).eval()
    dp.load_state_dict(st, strict=True)
    for name, cs in duration_ref.CASES.items():
        seed = cs["seed"]
        while True:
            x, mask, c = duration_ref.make_inputs(seed, cs["lens"], cs["Tx"])
            logw = dp(x, mask, c)
            if margin_ok(logw, mask):
                break
            seed += 1000
        np.savez_compressed(os.path.join(OUT, name + ".npz"), logw=logw.numpy(), seed=seed, weight_checksum=weights.checksum(st))
    for name, cs in synth_ref.CASES.items():
        st = synth_ref.make_state(n_mel=cs["n_mel"])
        model = StableTTS(synth_ref.N_VOCAB, cs["n_mel"], 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
        model.load_state_dict(st, strict=True)
        seed = cs["seed"]
        while True:
            ids, lens, y = synth_ref.make_inputs(seed, cs["lens"], cs["T_ref"], cs["n_mel"])
            c = model.ref_encoder(y, None)
            x, mu_x, x_mask = model.encoder(ids, c, lens)
            logw = model.dp(x, x_mask, c)
            if margin_ok(logw, x_mask) and total_margin_ok(logw, x_mask, cs["length_scale"]):
                break
            seed += 1000
        with SeededRandnLike(seed) as rnd:
            out = model.synthesise(ids, lens, cs["n_timesteps"], 1.0, y, cs["length_scale"], cs["solver"], cs["cfg"])
        assert len(rnd.drawn) == 1
        w = torch.exp(logw) * x_mask
        print(name, "seed", seed, "T_y", out["attn"].shape[-1], "durations", float(w[x_mask > 0].min()), float(w.max()))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), seed=seed, z=rnd.drawn[0].numpy(), c=c.numpy(), logw=logw.numpy(),
                            encoder_outputs=out["encoder_outputs"].numpy(), decoder_outputs=out["decoder_outputs"].numpy(),
                            attn=out["attn"].numpy().astype(np.uint8), weight_checksum=weights.checksum(st))


if __name__ == "__main__":
    main()
