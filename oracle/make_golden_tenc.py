"""tests/golden/tenc_*.npz from the UNMODIFIED reference TextEncoder (authoring container only):
python -m oracle.make_golden_tenc"""
import os, sys
import numpy as np
import torch
from oracle import text_encoder_ref as T

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    sys.path.insert(0, os.environ.get("STABLETTS_REFERENCE_DIR", ""))
    from models.text_encoder import TextEncoder
    for name, cs in T.CASES.items():
        enc = TextEncoder(401, cs["out_channels"], 256, 1024, 4, 3, 3, 0.1, 256).eval()
        st = T.make_state(3, out_channels=cs["out_channels"])
        enc.load_state_dict(st, strict=True)
        ids, c, lens = T.make_inputs(cs["seed"], cs["lens"], cs["T"])
        with torch.inference_mode():
            x, mu, m = enc(ids, c, lens)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), x=x.numpy(), mu=mu.numpy(), mask=m.numpy())
        print(name, tuple(x.shape), tuple(mu.shape), float(mu.abs().max()))


if __name__ == "__main__":
    main()
