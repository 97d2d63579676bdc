"""tests/golden/align_*.npz from the UNMODIFIED reference's generate_path / sequence_mask (authoring
container only):  python -m oracle.make_golden_align"""
import os, sys, types
import numpy as np
import torch
from oracle import align_ref as A

REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    sys.path.insert(0, REF)
    stub = types.ModuleType("torchdiffeq"); stub.odeint = lambda *a, **k: None
    sys.modules.setdefault("torchdiffeq", stub)
    from models.model import generate_path
    from utils.mask import sequence_mask
    for name, cs in A.ALIGN_CASES.items():
        logw, x_mask, mu_x = A.make_align_inputs(cs["seed"], cs["B"], cs["Tx"], cs["M"], cs["lens"])
        # models/model.py:83-95 executed with the reference's own helpers
        w = torch.exp(logw) * x_mask
        w_ceil = torch.ceil(w) * cs["length_scale"]
        y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()
        y_max_length = y_lengths.max()
        y_mask = sequence_mask(y_lengths, y_max_length).unsqueeze(1).to(x_mask.dtype)
        attn_mask = x_mask.unsqueeze(-1) * y_mask.unsqueeze(2)
        attn = generate_path(w_ceil.squeeze(1), attn_mask.squeeze(1)).unsqueeze(1)
        mu_y = torch.matmul(attn.squeeze(1).transpose(1, 2), mu_x.transpose(1, 2)).transpose(1, 2)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), mu_y=mu_y.numpy(), y_mask=y_mask.numpy(),
                            y_lengths=y_lengths.numpy(), attn=attn.numpy())
        print(name, tuple(mu_y.shape), y_lengths.tolist())


if __name__ == "__main__":
    main()
