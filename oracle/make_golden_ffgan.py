"""tests/golden/ffgan_*.npz and tests/golden/ffgan_inventory.npz from the UNMODIFIED reference FireflyGANBase
(vocoders/ffgan/model.py; it imports with torch and numpy only).  Authoring container only:

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_ffgan

The weights are oracle/ffgan_ref.make_state (O(1) gain per layer: the reference's own init gives audio std ~0.002).  Before
writing anything the recipe asserts that the fixtures exercise the model: audio std > 0.1, max |audio| inside tanh's
nonlinear range, and removing any single ConvNeXt block or ResBlock1 changes the audio by more than 1e-3 relative."""
import json
import os
import sys

import numpy as np
import torch

from oracle import ffgan_ref as R

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def check_liveness(st):
    mel = R.make_mel(50, 2, 40)
    with torch.inference_mode():
        ref = R.ffgan_forward(st, mel)
        std, peak = float(ref.std()), float(ref.abs().max())
        print(f"audio std {std:.3f}, max |audio| {peak:.3f}")
        assert std > 0.1 and peak > 0.9, (std, peak)
        for i, depth in enumerate(R.DEPTHS):
            for j in range(depth):
                d = float((R.ffgan_forward(st, mel, skip_block=(i, j)) - ref).norm() / ref.norm())
                assert d > 1e-3, ("ConvNeXt block", i, j, d)
        for i in range(len(R.UPS)):
            for b in range(len(R.RES_K)):
                d = float((R.ffgan_forward(st, mel, skip_resblock=(i, b)) - ref).norm() / ref.norm())
                assert d > 1e-3, ("ResBlock1", i, b, d)


def main():
    sys.path.insert(0, os.environ.get("STABLETTS_REFERENCE_DIR", ""))
    from vocoders.ffgan.model import FireflyGANBase        # vocoders/ffgan/model.py:45
    m = FireflyGANBase().eval()
    inv = [(k, list(v.shape)) for k, v in m.state_dict().items()]
    assert [(k, tuple(s)) for k, s in inv] == list(R.param_shapes().items())
    st = R.make_state()
    print("load_state_dict:", m.load_state_dict(st, strict=True))
    check_liveness(st)
    n_params = sum(int(np.prod(s)) for _, s in inv)
    np.savez_compressed(os.path.join(OUT, "ffgan_inventory.npz"), inventory=json.dumps(inv), n_params=n_params)
    for name, cs in R.CASES.items():
        mel = R.make_mel(cs["seed"], cs["B"], cs["T"])
        with torch.inference_mode():
            audio = m(mel)
            ora = R.ffgan_forward(st, mel)
        print(name, tuple(audio.shape), f"std {float(audio.std()):.3f}", "oracle max-abs diff", float((ora - audio).abs().max()))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), audio=audio.numpy().astype(np.float32),
                            weight_checksum=R.weight_checksum(st))


if __name__ == "__main__":
    main()
