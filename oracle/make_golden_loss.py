"""Generate tests/golden/loss_*.npz from the UNMODIFIED reference ``CFMDecoder.compute_loss``
(models/flow_matching.py:69-100), eval mode, no autograd (authoring container only).

    python -m oracle.make_golden_loss       # needs STABLETTS_REFERENCE_DIR=<reference checkout>

The reference draws ``t`` and ``z`` from the global generator, whose stream differs between CPU and CUDA;
both sides therefore consume the same INJECTED draws (``loss_draws`` below, seeded CPU generator): here
``torch.rand`` / ``torch.randn_like`` are patched around the reference call, in tests/test_gpu_parity.py
around the drop-in's call.  Everything else is the reference's own code.  TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import os
from unittest import mock

import numpy as np
import torch

from oracle import cases, weights
from oracle.make_golden import OUT, _import_reference

LOSS_CASES = {
    "loss_b3_ragged": dict(seed=31, lengths=[60, 45, 33], T=60, n_mel=80),
    "loss_b1": dict(seed=32, lengths=[50], T=50, n_mel=80),
    "loss_b2_mel128": dict(seed=33, lengths=[40, 37], T=41, n_mel=128),
}


def loss_draws(seed: int, B: int, n_mel: int, T: int):
    """the uniform draw behind t (:92) and the noise z (:96), in the order the reference draws them"""
    g = torch.Generator().manual_seed(seed + 7000)
    return torch.rand(B, 1, 1, generator=g), torch.randn(B, n_mel, T, generator=g)


class inject_draws:
    """patches torch.rand / torch.randn_like to return the given draws (moved to the requested device)"""

    def __init__(self, u, z):
        self.u, self.z = u, z

    def __enter__(self):
        u, z = self.u, self.z
        self.p = [mock.patch("torch.rand", lambda *a, device=None, dtype=None, **k: u.to(device=device, dtype=dtype)),
                  mock.patch("torch.randn_like", lambda x, **k: z.to(device=x.device, dtype=x.dtype))]
        for p in self.p:
            p.start()
        return self

    def __exit__(self, *exc):
        for p in self.p:
            p.stop()


def main():
    _, CFMDecoder = _import_reference()
    for name, cs in LOSS_CASES.items():
        m = CFMDecoder(cs["n_mel"], cs["n_mel"], 256, cs["n_mel"], 1024, 4, 6, 3, 0.1, 256).eval()
        st = weights.make_state(cases.WEIGHT_SEED, cs["n_mel"])
        m.estimator.load_state_dict(st, strict=True)
        inp = weights.make_inputs(cs["seed"], cs["lengths"], cs["T"], cs["n_mel"])
        x1 = inp["x"] * inp["mask"]                          # a masked target mel, as the training collate produces
        u, z = loss_draws(cs["seed"], len(cs["lengths"]), cs["n_mel"], cs["T"])
        with torch.no_grad(), inject_draws(u, z):
            loss, y = m.compute_loss(x1, inp["mask"], inp["mu"], inp["c"])
        np.savez_compressed(os.path.join(OUT, name + ".npz"), loss=loss.numpy(), y=y.numpy(),
                            weight_checksum=weights.checksum(st), input_checksum=weights.checksum([x1, inp["mu"], inp["c"], u, z]))
        print(name, float(loss), tuple(y.shape))


if __name__ == "__main__":
    main()
