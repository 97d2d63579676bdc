"""Writes tests/golden/vocos_grad_*.npz from the UNMODIFIED reference Vocos (vocoders/vocos/models/model.py, staged by
oracle/stage_mel_loss.py and imported through its load_reference()), run in float64 on the CPU.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_mel_loss && python -m oracle.make_golden_vocos_grad

Per case (oracle/vocos_grad_ref.py::FIXTURES): the seeded weights of vocoder_ref.make_state, stored only as (sum, sum of
squares) checksums per state_dict tensor, so a test regenerates them and checks them; a mel whose log-magnitudes all stay
1e-3 away from ln 100 (no clip decision can flip); a seeded N(0, 1) upstream gradient on the audio.  The fixture holds the
audio in full and (norm, dot with a seeded probe) of every parameter gradient in state_dict order."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import stage_mel_loss, vocos_grad_ref as G  # noqa: E402


def main():
    _, model, _, config = stage_mel_loss.load_reference()
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name, cs in G.FIXTURES.items():
        d = G.case_dims(cs)
        vc = config.VocosConfig(input_channels=d["input_channels"], dim=d["dim"], intermediate_dim=d["intermediate_dim"],
                                num_layers=d["num_layers"])
        mc = config.MelConfig(n_fft=d["n_fft"], hop_length=d["hop_length"])
        m = model.Vocos(vc, mc).double()
        state = G.case_state(cs)
        m.load_state_dict({k: v.double() for k, v in state.items()}, strict=True)
        mel = G.case_mel(cs)
        audio = m(mel)
        (audio * G.seeded(audio.shape, cs["seed"], 1)).sum().backward()
        q = {"audio": audio.detach().numpy(), "checksums": G.checksums(state),
             "grad_stats": G.grad_stats([p.grad for p in m.parameters()], cs["seed"]).numpy(),
             "keys": np.array([k for k, _ in m.named_parameters()])}
        assert list(q["keys"]) == G.param_names(d)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **q)
        print(name, os.path.getsize(os.path.join(out_dir, name + ".npz")), "bytes")


if __name__ == "__main__":
    main()
