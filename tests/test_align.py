"""Row f1 (SURVEY.md §8f): duration -> alignment -> mu_y glue.  CPU: oracle restatement vs the
reference-generated fixtures.  GPU: the CUDA kernels
through the C ABI vs the same fixtures — a gather, so the bar is bit-exact."""
import os

import numpy as np
import pytest
import torch

from oracle import align_ref as A


@pytest.mark.parametrize("name", list(A.ALIGN_CASES))
def test_oracle_vs_golden(name, golden_dir):
    cs = A.ALIGN_CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    logw, x_mask, mu_x = A.make_align_inputs(cs["seed"], cs["B"], cs["Tx"], cs["M"], cs["lens"])
    mu_y, y_mask, y_len, attn = A.expand_by_durations(logw, x_mask, mu_x, cs["length_scale"])
    assert torch.equal(y_len, torch.from_numpy(g["y_lengths"]))
    assert torch.equal(mu_y, torch.from_numpy(g["mu_y"])) and torch.equal(y_mask, torch.from_numpy(g["y_mask"]))
    assert torch.equal(attn, torch.from_numpy(g["attn"]))
    # every valid output frame is covered by exactly one token
    cover = attn.sum(dim=2).squeeze(1)
    assert torch.equal(cover, y_mask.squeeze(1) * (cover > 0).float())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(A.ALIGN_CASES))
def test_cuda_vs_golden(name, golden_dir):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200.align import expand_by_durations
    dev = torch.device("cuda:0")
    cs = A.ALIGN_CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    logw, x_mask, mu_x = A.make_align_inputs(cs["seed"], cs["B"], cs["Tx"], cs["M"], cs["lens"])
    mu_y, y_mask, y_len, attn = expand_by_durations(logw.to(dev), x_mask.to(dev), mu_x.to(dev), cs["length_scale"], return_attn=True)
    assert torch.equal(y_len.cpu(), torch.from_numpy(g["y_lengths"]))
    assert torch.equal(mu_y.cpu(), torch.from_numpy(g["mu_y"]))
    assert torch.equal(y_mask.cpu(), torch.from_numpy(g["y_mask"]))
    assert torch.equal(attn.cpu(), torch.from_numpy(g["attn"]))
    # device-resident form: caller-provided cap, no host read; the extra frames are zero / masked out
    cap = int(g["y_lengths"].max()) + 7
    mu2, m2, _, _ = expand_by_durations(logw.to(dev), x_mask.to(dev), mu_x.to(dev), cs["length_scale"], max_length=cap)
    assert torch.equal(mu2[:, :, :mu_y.shape[2]].cpu(), torch.from_numpy(g["mu_y"])) and float(mu2[:, :, mu_y.shape[2]:].abs().max()) == 0.0
    assert float(m2[:, :, mu_y.shape[2]:].abs().max()) == 0.0


def test_no_cpu_fallback():
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200.align import expand_by_durations
    logw, x_mask, mu_x = A.make_align_inputs(1, 1, 4, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        expand_by_durations(logw, x_mask, mu_x)


# --------------------------------------------------------------------------------------------------------------------
# the edges of st_align_lengths / st_align_expand against the oracle, bit for bit.  The reference runs synthesise on
# CUDA, so the oracle's exp is torch's on the same device; the rest of it runs as written.
# --------------------------------------------------------------------------------------------------------------------
def _edge_inputs(name):
    """(logw, x_mask, mu_x, length_scale) of an edge case; logw (B, 1, Tx) may hold -inf (a valid token of duration 0)"""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if name.startswith("ulp_"):                 # logw = fp32(ln k) and its two neighbours: the ceil decides the frame
        k = torch.arange(1, 61, dtype=torch.float64)
        ln = torch.log(k).float()
        logw = torch.stack([torch.nextafter(ln, torch.tensor(-1.0)), ln, torch.nextafter(ln, torch.tensor(99.0))], 1).reshape(1, 1, -1)
        Tx = logw.shape[2]
        x_mask = torch.ones(1, 1, Tx)
        return logw, x_mask, torch.randn(1, 80, Tx, generator=g), float(name.split("_")[1])
    B, Tx, M = {"tx1": (2, 1, 80), "all_zero": (2, 7, 16)}.get(name, (3, 100, 80))
    x_mask = torch.ones(B, 1, Tx)
    logw = torch.randn(B, 1, Tx, generator=g) * 0.8 + 0.6
    ls = 1.0
    if name.startswith("scale_"):
        ls = float(name.split("_")[1])
        x_mask[1, :, 71:] = 0.0
    elif name == "zero_dur":
        logw[:, :, 3::7] = -float("inf")        # valid tokens that take no frame
        logw[0, :, 0] = -float("inf")
        logw[1, :, -1] = -float("inf")
    elif name == "holes":
        x_mask[0, :, 10:13] = 0.0               # holes inside the utterance
        x_mask[1, :, 50] = 0.0
        x_mask[2, :, 1::2] = 0.0
        x_mask[2, :, 90:] = 0.0
    elif name == "all_zero":
        logw[:] = -float("inf")                 # y_len clamps to 1 and no token covers the frame
        x_mask[1, :, 3:] = 0.0
    elif name == "tx1":
        logw[1] = -2.0
    mu_x = torch.randn(B, M, Tx, generator=g) * x_mask
    return logw * x_mask if name != "zero_dur" and name != "all_zero" else logw, x_mask, mu_x, ls


ALIGN_EDGES = ["zero_dur", "holes", "scale_0.5", "scale_1.15", "scale_2", "tx1", "all_zero", "ulp_1.0", "ulp_1.15"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ALIGN_EDGES)
def test_align_edges_vs_oracle(name):
    """y_lengths, mu_y, y_mask and attn equal the oracle's bit for bit, with max_length both below and above y_len"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200.align import expand_by_durations
    dev = torch.device("cuda:0")
    logw, x_mask, mu_x, ls = _edge_inputs(name)
    dev_exp = lambda v: torch.exp(v.to(dev)).cpu()        # noqa: E731
    mu_r, ym_r, yl_r, attn_r = A.expand_by_durations(logw, x_mask, mu_x, ls, exp=dev_exp)
    args = (logw.to(dev), x_mask.to(dev), mu_x.to(dev), ls)
    mu_y, y_mask, y_len, attn = expand_by_durations(*args, return_attn=True)
    assert torch.equal(y_len.cpu(), yl_r), (y_len.cpu(), yl_r)
    assert torch.equal(bits(mu_y.cpu()), bits(mu_r)) and torch.equal(y_mask.cpu(), ym_r) and torch.equal(attn.cpu(), attn_r)
    if name == "all_zero":
        assert yl_r.tolist() == [1, 1] and float(attn_r.abs().max()) == 0.0 and float(mu_r.abs().max()) == 0.0
    Ty = mu_r.shape[2]
    for cap in sorted({max(1, Ty // 2), max(1, Ty - 1), Ty + 37}):
        mu2, m2, yl2, attn2 = expand_by_durations(*args, max_length=cap, return_attn=True)
        n = min(cap, Ty)
        assert torch.equal(yl2.cpu(), yl_r)
        assert torch.equal(bits(mu2[:, :, :n].cpu()), bits(mu_r[:, :, :n])) and torch.equal(m2[:, :, :n].cpu(), ym_r[:, :, :n])
        assert torch.equal(attn2[..., :n].cpu(), attn_r[..., :n])
        if cap > Ty:
            assert float(mu2[:, :, Ty:].abs().max()) == 0.0 and float(m2[:, :, Ty:].abs().max()) == 0.0
            assert float(attn2[..., Ty:].abs().max()) == 0.0
    if name.startswith("ulp_"):
        w_dev, w_cpu = torch.ceil(dev_exp(logw)), torch.ceil(torch.exp(logw))
        print(f"\n{name}: {int((w_dev != w_cpu).sum())} of {logw.numel()} durations at fp32(ln k) +- 1 ulp would fall on the other "
              f"side of the ceil with the CPU's exp")


def bits(x):
    return x.contiguous().view(torch.int32)
