"""Row f12 (DESIGN.md §8), CPU: the fp64 oracle of the Vocos generator's backward.  Its autograd against the fixtures of
the unmodified reference Vocos (tests/golden/vocos_grad_*.npz, oracle/make_golden_vocos_grad.py) to 1e-9, and each
explicit adjoint of oracle/vocos_grad_ref.py (what st_vocos_backward's row kernels and packings compute) against torch's
float64 autograd to 1e-12, at T = 1, 2, 3 and 7 for the depthwise conv's utterance edges."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vocos_grad_ref as G
from oracle import vocoder_ref as V


def _rel(a, b):
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


@pytest.mark.parametrize("name", sorted(G.FIXTURES))
def test_oracle_autograd_vs_reference_golden(name, golden_dir):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cs = G.FIXTURES[name]
    d = G.case_dims(cs)
    state = G.case_state(cs)
    assert np.allclose(G.checksums(state), z["checksums"], rtol=1e-12, atol=0)
    assert list(z["keys"]) == G.param_names(d)
    mel = G.case_mel(cs)
    g = G.seeded((cs["B"], cs["T"] * d["hop_length"]), cs["seed"], 1)
    audio, grads = G.oracle_grads(state, mel, g, d["n_fft"], d["hop_length"])
    assert _rel(audio, torch.from_numpy(z["audio"])) <= 1e-9
    stats = G.grad_stats([grads[n] for n in G.param_names(d)], cs["seed"])
    ref = torch.from_numpy(z["grad_stats"])
    assert float(((stats[:, 0] - ref[:, 0]).abs() / ref[:, 0]).max()) <= 1e-9
    probe = torch.tensor([math.sqrt(s) for s in G.param_sizes(d)], dtype=torch.float64)
    assert float(((stats[:, 1] - ref[:, 1]).abs() / (ref[:, 0] * probe)).max()) <= 1e-9


def test_clip_fixture_reaches_the_clip():
    cs = G.FIXTURES["vocos_grad_api_b2_t16_clip"]
    st = {k: v.double() for k, v in G.case_state(cs).items()}
    lm = V.head_log_magnitudes(st, G.case_mel(cs))
    frac = float((lm > G.LN_CLIP).double().mean())
    assert 0.02 < frac < 0.5 and G.clip_margin(st, G.case_mel(cs)) >= 1e-3


@pytest.mark.parametrize("T", [1, 2, 3, 7])
def test_frame_grad_is_the_istft_adjoint(T):
    n_fft, hop, B = 256, 64, 2
    K = n_fft // 2 + 1
    win = torch.hann_window(n_fft, dtype=torch.float64)
    frames = torch.randn(B, T, n_fft, dtype=torch.float64, requires_grad=True)
    W = V.idft_basis(win, n_fft)
    # the overlap-add of the frames, as istft_same_as_gemm computes it from [re | im] = frames · W^+ (here: frames directly)
    pad = (n_fft - hop) // 2
    L = T * hop
    s = torch.arange(L) + pad
    out = torch.zeros(B, L, dtype=torch.float64)
    for j in range(n_fft // hop):
        t = s // hop - j
        ok = (t >= 0) & (t < T)
        out = out + torch.where(ok[None], frames[:, t.clamp(0, T - 1), s - t.clamp(0, T - 1) * hop], torch.zeros((), dtype=torch.float64))
    y = out / G.envelope(win, T, n_fft, hop)
    g = torch.randn(B, L, dtype=torch.float64)
    (y * g).sum().backward()
    assert _rel(G.frame_grad(g, win, T, n_fft, hop), frames.grad) <= 1e-12
    # and through the basis: d[re | im] = dF W^T, with the imaginary DC / Nyquist gradients exactly 0, as irfft's backward
    re = torch.randn(B, K, T, dtype=torch.float64, requires_grad=True)
    im = torch.randn(B, K, T, dtype=torch.float64, requires_grad=True)
    a = V.istft_same_reference(re, im, win, n_fft, hop)
    (a * g).sum().backward()
    dS = G.frame_grad(g, win, T, n_fft, hop) @ W.T
    assert _rel(dS[..., :K].transpose(1, 2), re.grad) <= 1e-12
    assert _rel(dS[..., K:].transpose(1, 2), im.grad) <= 1e-12
    assert torch.all(dS[..., K] == 0) and torch.all(dS[..., 2 * K - 1] == 0)
    assert float(im.grad[:, 0].abs().max()) <= 1e-12 and float(im.grad[:, K - 1].abs().max()) <= 1e-12


def test_spectrum_grad_with_the_clip():
    gen = torch.Generator().manual_seed(3)
    m = (torch.randn(64, 40, generator=gen, dtype=torch.float64) * 3 + 3).requires_grad_()
    p = torch.randn(64, 40, generator=gen, dtype=torch.float64, requires_grad=True)
    with torch.no_grad():
        m[0, 0] = G.LN_CLIP                                      # exp(m) rounds to the bound or next to it
    a = torch.clip(torch.exp(m), max=1e2)
    re, im = a * torch.cos(p), a * torch.sin(p)
    dre, dim = torch.randn_like(re), torch.randn_like(im)
    (re * dre + im * dim).sum().backward()
    dm, dp = G.spectrum_grad(dre, dim, m.detach(), p.detach())
    assert float((m.detach() > G.LN_CLIP + 1e-9).double().mean()) > 0.1
    assert _rel(dm, m.grad) <= 1e-12 and _rel(dp, p.grad) <= 1e-12


@pytest.mark.parametrize("C", [512, 768])
def test_layernorm_bwd(C):
    gen = torch.Generator().manual_seed(C)
    x = (torch.randn(37, C, generator=gen, dtype=torch.float64) * 2 + 0.5).requires_grad_()
    w = (1 + 0.1 * torch.randn(C, generator=gen, dtype=torch.float64)).requires_grad_()
    b = (0.1 * torch.randn(C, generator=gen, dtype=torch.float64)).requires_grad_()
    g = torch.randn(37, C, generator=gen, dtype=torch.float64)
    (F.layer_norm(x, (C,), w, b, 1e-6) * g).sum().backward()
    dx, dw, db = G.ln_bwd(x.detach(), w.detach(), g)
    assert _rel(dx, x.grad) <= 1e-12 and _rel(dw, w.grad) <= 1e-12 and _rel(db, b.grad) <= 1e-12


@pytest.mark.parametrize("T", [1, 2, 3, 7])
def test_dwconv_bwd_at_utterance_edges(T):
    B, C = 3, 16
    gen = torch.Generator().manual_seed(T)
    x = torch.randn(B, T, C, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(C, 1, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    b = torch.randn(C, generator=gen, dtype=torch.float64, requires_grad=True)
    dz = torch.randn(B, T, C, generator=gen, dtype=torch.float64)
    y = F.conv1d(x.transpose(1, 2), w, b, padding=3, groups=C).transpose(1, 2)
    (y * dz).sum().backward()
    dx, dw, db = G.dwconv_bwd(x.detach(), w.detach(), dz)
    assert _rel(dx, x.grad) <= 1e-12 and _rel(dw, w.grad) <= 1e-12 and _rel(db, b.grad) <= 1e-12


def test_gelu_bwd():
    h = torch.linspace(-8, 8, 1001, dtype=torch.float64, requires_grad=True)
    dg = torch.randn(1001, dtype=torch.float64)
    (F.gelu(h) * dg).sum().backward()
    assert _rel(G.gelu_bwd(h.detach(), dg), h.grad) <= 1e-12


@pytest.mark.parametrize("T", [1, 2, 3, 7])
def test_embed_wgrad_packing(T):
    """dW of the k = 7 embed conv = dY^T · [X^T; 1]^T with the 7-tap shifted transpose, unpacked to (dim, n_mel, 7)"""
    B, Cin, Cout = 2, 16, 24
    gen = torch.Generator().manual_seed(10 + T)
    x = torch.randn(B, Cin, T, generator=gen, dtype=torch.float64)
    w = torch.randn(Cout, Cin, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    b = torch.randn(Cout, generator=gen, dtype=torch.float64, requires_grad=True)
    dy = torch.randn(B, Cout, T, generator=gen, dtype=torch.float64)
    (F.conv1d(x, w, b, padding=3) * dy).sum().backward()
    Kr = (B * T + 255) // 256 * 256
    Xt = G.wgrad_operand(x.transpose(1, 2), 7, Kr)
    dYt = torch.zeros(Cout, Kr, dtype=torch.float64)
    dYt[:, :B * T] = dy.transpose(1, 2).reshape(B * T, Cout).T
    gw, gb = G.unpack_wgrad(dYt @ Xt.T, Cout, Cin, 7)
    assert _rel(gw, w.grad) <= 1e-12 and _rel(gb, b.grad) <= 1e-12


def test_head_wgrad_unpack_undoes_the_column_groups():
    K, Kp, C = 5, 128, 8
    gen = torch.Generator().manual_seed(1)
    dWp = torch.randn(2 * Kp, C + 8, generator=gen, dtype=torch.float64)
    gw, gb = G.unpack_wgrad(dWp, 2 * K, C, 1, K, Kp)
    assert torch.equal(gw[:K, :, 0], dWp[:K, :C]) and torch.equal(gw[K:, :, 0], dWp[Kp:Kp + K, :C])
    assert torch.equal(gb[:K], dWp[:K, C]) and torch.equal(gb[K:], dWp[Kp:Kp + K, C])
