"""Fixtures that let the suite compare with the unmodified reference without a checkout of it:

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_inventory

writes tests/golden/reference_inventory.npz (one JSON string per module: parameter names and shapes of the reference's Decoder, StableTTS,
TextEncoder and Vocos, as their state_dict lists them) and tests/golden/live_estimator.npz (the reference Decoder's
output on one seeded ragged call, and its RotaryPositionalEmbeddings on a seeded q)."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import cases, weights                      # noqa: E402
from oracle import estimator_ref as R                  # noqa: E402
from oracle.stage_reference import REF                 # noqa: E402


def main():
    if not os.path.isdir(REF):
        raise SystemExit("set STABLETTS_REFERENCE_DIR to a checkout of the reference")
    sys.path.insert(0, REF)
    stub = types.ModuleType("torchdiffeq")
    stub.odeint = lambda f, y0, t, method=None, rtol=None, atol=None: R.odeint_fixed(f, y0, t, method)[None]
    sys.modules.setdefault("torchdiffeq", stub)
    from models.estimator import Decoder
    from models.diffusion_transformer import RotaryPositionalEmbeddings
    from models.model import StableTTS
    from models.text_encoder import TextEncoder

    def inv(m):
        return [[k, list(v.shape)] for k, v in m.state_dict().items()]
    code = ("import sys, json; sys.path.insert(0, sys.argv[1]);"
            "from config import MelConfig, VocosConfig; from models.model import Vocos;"
            "print(json.dumps([[k, list(v.shape)] for k, v in Vocos(VocosConfig(), MelConfig()).state_dict().items()]))")
    vocos = json.loads(subprocess.run([sys.executable, "-c", code, os.path.join(REF, "vocoders", "vocos")],
                                      capture_output=True, text=True, check=True).stdout)
    dec = Decoder(80, 80, 256, 80, 1024, 0.1, 6, 4, 3, 256).eval()
    out = {"decoder": inv(dec), "stabletts": inv(StableTTS(401, 80, 256, 1024, 4, 3, 6, 3, 0.1, 256)),
           "text_encoder": inv(TextEncoder(401, 80, 256, 1024, 4, 3, 3, 0.1, 256)), "vocos": vocos}
    gold = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gold, "reference_inventory.npz"), **{k: np.array(json.dumps(v)) for k, v in out.items()})
    dec.load_state_dict(weights.make_state(cases.WEIGHT_SEED, 80), strict=True)
    inp = weights.make_inputs(99, [70, 45], 70, 80, t_per_sample=True)
    q = torch.randn(2, 4, 37, 64, generator=torch.Generator().manual_seed(5))
    with torch.inference_mode():
        ref = dec(inp["t"], inp["x"], inp["mask"], inp["mu"], inp["c"])
        rope = RotaryPositionalEmbeddings(32)(q)
    np.savez_compressed(os.path.join(gold, "live_estimator.npz"), out=ref.numpy(), rope=rope.numpy())


if __name__ == "__main__":
    main()
