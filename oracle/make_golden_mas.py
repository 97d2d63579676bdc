"""Fixtures of monotonic alignment search and of StableTTS's training forward from the UNMODIFIED reference:

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_mas          # needs numba

mas_*.npz: neg_cent, mask and the path of the reference's own ``monotonic_align.maximum_path`` (numba).
fwd_*.npz: the value of ``StableTTS.forward`` (models/model.py:114-178) in eval mode under no_grad with the real
``maximum_path``.  Its three random draws are injected by shape: ``torch.rand(B, 1)`` behind the cfg dropout mask (:138),
``torch.rand([B, 1, 1])`` behind compute_loss's t and ``torch.randn_like`` behind its noise.

Margin.  The alignment is discontinuous in the scores, and a GPU's mu_x and neg_cent differ from the reference's in the last
bits.  So the target mel is built from the reference encoder's own mu_x, expanded by drawn durations, plus noise: the optimum
then has a clear gap.  The smallest backtrack gap |value[y-1,i] - value[y-1,i-1]| along the chosen path must exceed
MARGIN_FACTOR x t_y x SCORE_BAR x max|neg_cent|; SCORE_BAR bounds the relative score error an engine's mu_x can cause, and
t_y rows of it can accumulate in a value.  A seed that fails is skipped for the next one and the seed used is recorded."""
import os
import sys
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mas_ref, synth_ref, weights                                    # noqa: E402
from oracle.make_golden_synth import _import_reference                            # noqa: E402
from oracle.stage_reference import REF                                            # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SCORE_BAR = 1e-4
MARGIN_FACTOR = 4.0

MAS_CASES = {
    # training-like: scores of a target built from token means, ragged lengths
    "mas_ragged":  dict(seed=1, B=4, Ty=160, Tx=64, t_y=[160, 131, 97, 40], t_x=[64, 50, 33, 40], kind="train"),
    # t_x = t_y, t_x = 1, t_y = 1, two rows with t_x > t_y, a zero-length row
    "mas_edges":   dict(seed=2, B=6, Ty=40, Tx=30, t_y=[30, 40, 1, 12, 3, 0], t_x=[30, 1, 1, 29, 30, 17], kind="normal"),
    "mas_ties":    dict(seed=3, B=3, Ty=90, Tx=40, t_y=[90, 77, 50], t_x=[40, 31, 25], kind="ties"),
    "mas_scale1e5": dict(seed=4, B=3, Ty=120, Tx=48, t_y=[120, 100, 64], t_x=[48, 45, 64], kind="scale1e5"),
}

FWD_CASES = {
    "fwd_b3_mel80":  dict(seed=11, lens=[23, 15, 9], z_T=40, z_lens=[40, 31, 22], u_cfg=[0.9, 0.1, 0.6], n_mel=80),
    "fwd_b2_mel128": dict(seed=12, lens=[17, 11], z_T=36, z_lens=[29, 36], u_cfg=[0.05, 0.8], n_mel=128),
}


def prefix_mask(t_y, t_x, Ty, Tx):
    ty, tx = np.asarray(t_y), np.asarray(t_x)
    return ((np.arange(Ty)[None, :, None] < ty[:, None, None]) & (np.arange(Tx)[None, None, :] < tx[:, None, None])).astype(np.float32)


def mas_inputs(cs):
    g = torch.Generator().manual_seed(cs["seed"])
    B, Ty, Tx = cs["B"], cs["Ty"], cs["Tx"]
    if cs["kind"] == "train":
        mu = torch.randn(B, 80, Tx, generator=g)
        tok = torch.sort(torch.randint(0, Tx, (B, Ty), generator=g), dim=1).values
        y = torch.gather(mu, 2, tok[:, None, :].expand(B, 80, Ty)) + 0.5 * torch.randn(B, 80, Ty, generator=g)
        nc = mas_ref.neg_cent64(y, mu).float()
    elif cs["kind"] == "ties":
        nc = torch.randint(-2, 3, (B, Ty, Tx), generator=g).float()
    elif cs["kind"] == "scale1e5":
        nc = torch.randn(B, Ty, Tx, generator=g) * 1e5
    else:
        nc = torch.randn(B, Ty, Tx, generator=g) * 3.0
    return nc.numpy(), prefix_mask(cs["t_y"], cs["t_x"], Ty, Tx)


class inject_by_shape:
    """torch.rand / torch.randn_like return the given draws, chosen by the requested shape (moved to the device asked for)."""

    def __init__(self, draws):
        self.draws = {tuple(k): v for k, v in draws.items()}

    def __enter__(self):
        def rand(*size, device=None, dtype=None, **kw):
            shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (list, tuple, torch.Size)) else tuple(size)
            return self.draws[("rand",) + shape].to(device=device, dtype=dtype or torch.float32)
        self.p = [mock.patch("torch.rand", rand),
                  mock.patch("torch.randn_like", lambda t, **kw: self.draws[("randn",) + tuple(t.shape)].to(t.device, t.dtype))]
        for p in self.p:
            p.start()
        return self

    def __exit__(self, *exc):
        for p in self.p:
            p.stop()


def fwd_inputs(cs, seed, model):
    """ids, lengths, z, the draws, and a target mel y built from the reference encoder's own mu_x (see the margin above)."""
    B, n_mel = len(cs["lens"]), cs["n_mel"]
    ids, x_lengths, z = synth_ref.make_inputs(seed, cs["lens"], cs["z_T"], n_mel)
    g = torch.Generator().manual_seed(seed + 500)
    z_lengths = torch.as_tensor(cs["z_lens"])
    u_cfg = torch.as_tensor(cs["u_cfg"], dtype=torch.float32)[:, None]
    keep = u_cfg > model.cfg_dropout
    z_mask = mas_ref.sequence_mask(z_lengths, z.shape[2]).unsqueeze(1)
    c = model.ref_encoder(z, z_mask) * keep + ~keep * model.fake_speaker.repeat(B, 1)
    _, mu_x, _ = model.encoder(ids, c, x_lengths)
    d = torch.randint(1, 6, (B, ids.shape[1]), generator=g) * mas_ref.sequence_mask(x_lengths, ids.shape[1]).long()
    y_lengths = d.sum(1)
    Ty = int(y_lengths.max())
    y = torch.zeros(B, n_mel, Ty)
    for b in range(B):
        tok = torch.repeat_interleave(torch.arange(ids.shape[1]), d[b])
        y[b, :, :len(tok)] = mu_x[b][:, tok] + 0.3 * torch.randn(n_mel, len(tok), generator=g)
    draws = {("rand", B, 1): u_cfg, ("rand", B, 1, 1): torch.rand(B, 1, 1, generator=g),
             ("randn", B, n_mel, Ty): torch.randn(B, n_mel, Ty, generator=g)}
    return dict(ids=ids, x_lengths=x_lengths, y=y, y_lengths=y_lengths, z=z, z_lengths=z_lengths), draws, mu_x


def margin(nc, mask):
    """(smallest backtrack gap / (t_y · SCORE_BAR · max|neg_cent|)) over the utterances: must exceed MARGIN_FACTOR"""
    path, value = mas_ref.maximum_path(nc, mask, return_value=True)
    t_y, _ = mas_ref.lengths_from_mask(mask)
    gaps = mas_ref.backtrack_gap(value, path, t_y)
    scale = np.abs(np.where(mask > 0, nc, 0)).max()
    return float(min(gaps[b] / (max(int(t_y[b]), 1) * SCORE_BAR * scale) for b in range(len(gaps))))


def main():
    StableTTS, _, _ = _import_reference()
    sys.modules.pop("monotonic_align", None)                 # the stub of make_golden_synth: use the real package here
    sys.path.insert(0, REF)
    import monotonic_align
    import models.model as ref_model
    ref_model.monotonic_align = monotonic_align
    torch.set_grad_enabled(False)
    for name, cs in MAS_CASES.items():
        nc, mask = mas_inputs(cs)
        path = monotonic_align.maximum_path(torch.from_numpy(nc), torch.from_numpy(mask)).numpy()
        assert np.array_equal(path.astype(np.int32), mas_ref.maximum_path(nc, mask)), name
        np.savez_compressed(os.path.join(OUT, name + ".npz"), neg_cent=nc, mask=mask.astype(np.uint8), path=path.astype(np.uint8))
        print(name, nc.shape, "ones", int(path.sum()))
    for name, cs in FWD_CASES.items():
        st = synth_ref.make_state(n_mel=cs["n_mel"])
        model = StableTTS(synth_ref.N_VOCAB, cs["n_mel"], 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
        model.load_state_dict(st, strict=True)
        seed = cs["seed"]
        while True:
            inp, draws, mu_x = fwd_inputs(cs, seed, model)
            nc = mas_ref.neg_cent64(inp["y"], mu_x).float().numpy()
            x_mask = mas_ref.sequence_mask(inp["x_lengths"], mu_x.shape[2])
            y_mask = mas_ref.sequence_mask(inp["y_lengths"], inp["y"].shape[2])
            mask = (y_mask[:, :, None] * x_mask[:, None, :]).numpy()
            m = margin(nc, mask)
            if m > MARGIN_FACTOR:
                break
            print(name, "seed", seed, "margin", m, "too small")
            seed += 1000
        with inject_by_shape(draws):
            dur_loss, diff_loss, prior_loss, attn = model(inp["ids"], inp["x_lengths"], inp["y"], inp["y_lengths"], inp["z"],
                                                          inp["z_lengths"])
        print(name, "seed", seed, "margin", round(m, 1), "T_y", inp["y"].shape[2], float(dur_loss), float(diff_loss), float(prior_loss))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), seed=seed, margin=m, **{k: v.numpy() for k, v in inp.items()},
                            u_cfg=draws[("rand", len(cs["lens"]), 1)].numpy(), u_t=draws[("rand", len(cs["lens"]), 1, 1)].numpy(),
                            noise=draws[("randn",) + tuple(inp["y"].shape)].numpy(), dur_loss=dur_loss.numpy(),
                            diff_loss=diff_loss.numpy(), prior_loss=prior_loss.numpy(), attn=attn.numpy().astype(np.uint8),
                            weight_checksum=weights.checksum(st))


if __name__ == "__main__":
    main()
