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
