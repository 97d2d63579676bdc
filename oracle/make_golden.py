"""Generate tests/golden/*.npz from the UNMODIFIED reference (authoring container only).

    python -m oracle.make_golden            # needs STABLETTS_REFERENCE_DIR=<reference checkout>

Imports the reference's own ``models.estimator.Decoder`` and
``models.flow_matching.CFMDecoder`` (the latter with a stand-in ``torchdiffeq`` module, because
the real package is absent — so the *stepping* in SOLVE fixtures is the restated fixed-grid
driver while every estimator evaluation, ``cfg_wrapper`` and the ``randn_like`` draw are the
reference's own code).  Weights/inputs come from ``oracle.weights`` seeds; only outputs,
lengths and drift checksums are stored.  TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

from oracle import cases, weights
from oracle.estimator_ref import odeint_fixed

REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _import_reference():
    if not os.path.isdir(REF):
        raise SystemExit("reference checkout not present; goldens can only be made in the authoring container")
    sys.path.insert(0, REF)
    stub = types.ModuleType("torchdiffeq")

    def odeint(f, y0, t, method=None, rtol=None, atol=None):
        return odeint_fixed(f, y0, t, method)[None]          # [-1] is the final state
    stub.odeint = odeint
    sys.modules["torchdiffeq"] = stub
    from models.estimator import Decoder                     # noqa: E402
    from models.flow_matching import CFMDecoder              # noqa: E402
    return Decoder, CFMDecoder


def main():
    torch.set_num_threads(os.cpu_count())
    Decoder, CFMDecoder = _import_reference()
    os.makedirs(OUT, exist_ok=True)
    models = {}

    def get_cfm(n_mel):
        if n_mel not in models:
            m = CFMDecoder(n_mel, n_mel, 256, n_mel, 1024, 4, 6, 3, 0.1, 256).eval()   # models/model.py:40
            st = weights.make_state(cases.WEIGHT_SEED, n_mel)
            m.estimator.load_state_dict(st, strict=True)     # validates the 116 names/shapes
            models[n_mel] = (m, weights.checksum(st))
        return models[n_mel]

    for name, cs in cases.ESTIMATOR_CASES.items():
        m, wsum = get_cfm(cs["n_mel"])
        inp = weights.make_inputs(cs["seed"], cs["lengths"], cs["T"], cs["n_mel"],
                                  t_per_sample=cs.get("t_per_sample", False), t_value=cs.get("t_value", 0.37))
        with torch.inference_mode():
            out = m.estimator(inp["t"], inp["x"], inp["mask"], inp["mu"], inp["c"])
        np.savez_compressed(os.path.join(OUT, name + ".npz"), out=out.numpy(), lengths=np.array(cs["lengths"]),
                            weight_checksum=wsum,
                            input_checksum=weights.checksum([inp["x"], inp["mu"], inp["c"]]))
        print(name, tuple(out.shape), float(out.abs().max()))

    for name, cs in cases.SOLVE_CASES.items():
        m, wsum = get_cfm(cs["n_mel"])
        inp = weights.make_inputs(cs["seed"], cs["lengths"], cs["T"], cs["n_mel"])
        fs, fc = weights.make_cfg_params(cases.CFG_SEED, cs["n_mel"])
        kw = None if cs["cfg"] is None else dict(fake_speaker=fs, fake_content=fc, cfg_strength=cs["cfg"])
        torch.manual_seed(cs["seed"] + 1000)                 # CFMDecoder.forward draws randn_like(mu) from the global RNG
        out = m(inp["mu"], inp["mask"], cs["steps"], 1.0, inp["c"], cs["method"], kw)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), out=out.numpy(), lengths=np.array(cs["lengths"]),
                            weight_checksum=wsum, input_checksum=weights.checksum([inp["mu"], inp["c"]]))
        print(name, tuple(out.shape), float(out.abs().max()))


if __name__ == "__main__":
    main()
