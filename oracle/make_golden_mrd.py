"""Writes tests/golden/mrd_*.npz from the UNMODIFIED reference MultiResolutionDiscriminator (vocoders/vocos/models/
discriminator.py, staged by oracle/stage_mel_loss.py and imported through its load_reference()), run in float64 on the CPU.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_mel_loss && python -m oracle.make_golden_mrd

Per case (oracle/mrd_ref.py::CASES): the weights are the reference's own init right after torch.manual_seed(weight_seed),
stored only as (sum, sum of squares) checksums per state_dict tensor, so a test regenerates them and checks them.  Each
DiscriminatorR runs on the same input; the loss is Σ <score, g> + Σ <fmap_i, g_i> over every window with seeded N(0, 1)
upstream gradients; the fixture holds every score and the input gradient in full, and (norm, dot with a seeded probe) of
every fmap and of every original0 / original1 / bias gradient (mpd_ref.fixture_quantities)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import mrd_ref as R, stage_mel_loss  # noqa: E402


def main():
    _, _, disc, _ = stage_mel_loss.load_reference()
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name, cs in R.CASES.items():
        torch.manual_seed(cs["weight_seed"])
        mrd = disc.MultiResolutionDiscriminator().double()
        x = R.make_wave(cs).requires_grad_(True)
        sf = [d(x) for d in mrd.discriminators]
        R.upstream_loss(sf, cs["seed"]).backward()
        q = R.fixture_quantities(sf, x.grad, [p.grad for p in mrd.parameters()], cs["seed"])
        q = {k: v.numpy() for k, v in q.items()}
        q["checksums"] = R.checksums(mrd.state_dict()).numpy()
        q["keys"] = np.array(list(mrd.state_dict().keys()))
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **q)
        print(name, os.path.getsize(os.path.join(out_dir, name + ".npz")), "bytes")


if __name__ == "__main__":
    main()
