"""Row f12 (DESIGN.md §8): training the Vocos generator.  ``Vocos.forward`` in train() mode with grad enabled runs
st_vocos_forward_train and st_vocos_backward; every parameter gradient is checked against the fp64 autograd of the oracle
(oracle/vocoder_ref.py, the reference's ISTFT path) at the trainer's config, api.py's config, T = 1, 2, 3, dim 1024 with
(n_fft, hop) = (1024, 256) and a case with 16 % of the magnitudes on the 1e2 clip; against the fixtures of the unmodified
reference (tests/golden/vocos_grad_*.npz); bitwise properties (train audio = eval audio, repeated calls, interleaved
forwards and backwards); an AdamW step between calls; the refusals; and two AdamW steps of train.py's generator half-step
against the staged reference module.  Bars per parameter tensor, L2-relative: 1e-3 on the wgmma engine, 1e-4 on SIMT."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import rel_errs
from oracle import vocos_grad_ref as G
from oracle import vocoder_ref as V

BARS = {"tcgen05": 1e-3, "simt": 1e-4}
TRAIN = dict(V.DIMS)
API = dict(V.DIMS, **V.API_DIMS)
BIG = dict(V.DIMS, dim=1024, intermediate_dim=2048, num_layers=4, n_fft=1024, hop_length=256)


def _kw(dims):
    return dict(input_channels=dims["input_channels"], dim=dims["dim"], intermediate_dim=dims["intermediate_dim"],
                num_layers=dims["num_layers"], n_fft=dims["n_fft"], hop_length=dims["hop_length"])


def _module(dims, state, engine):
    from stabletts_b200 import Vocos
    m = Vocos(**_kw(dims))
    m.load_state_dict(state, strict=True)
    m = m.cuda().train()
    m.set_engine(engine)
    return m


def _grads(m, mel, g):
    m.zero_grad(set_to_none=True)
    audio = m(mel.cuda())
    (audio * g.cuda()).sum().backward()
    return audio.detach(), {n: m._param(n).grad.detach().clone() for n in m._shapes}


def _check_grads(got, ref, bar, what):
    worst = max(((n, rel_errs(got[n], ref[n])[1]) for n in ref), key=lambda t: t[1])
    bad = {n: rel_errs(got[n], ref[n])[1] for n in ref if rel_errs(got[n], ref[n])[1] > bar}
    print(f"{what}: worst L2-rel {worst[1]:.2e} ({worst[0]})")
    assert not bad, (what, bad)


CASES = {   # name -> dims, B, T, state / input seeds, head gain
    "train_b1_t40": (TRAIN, 1, 40, 1, 0.5),
    "train_b4_t40": (TRAIN, 4, 40, 2, 0.5),
    "api_b3_t40": (API, 3, 40, 3, 0.5),
    "api_b2_t1": (API, 2, 1, 4, 0.5),
    "api_b2_t2": (API, 2, 2, 5, 0.5),
    "api_b1_t3": (API, 1, 3, 6, 0.5),
    "dim1024_nfft1024_b2_t24": (BIG, 2, 24, 7, 0.5),
    "api_b2_t16_clip": (API, 2, 16, 8, V.HEAD_GAIN_CLIP),
}


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tcgen05", "simt"])
@pytest.mark.parametrize("case", list(CASES))
def test_gradients_vs_oracle(case, engine):
    dims, B, T, seed, gain = CASES[case]
    state = V.make_state(seed, head_gain=gain, **{k: dims[k] for k in ("input_channels", "dim", "intermediate_dim",
                                                                        "num_layers", "n_fft", "hop_length")})
    mel = G.make_clean_mel(state, seed, B, T, dims)
    g = G.seeded((B, T * dims["hop_length"]), seed, 1).float()
    ref_audio, ref = G.oracle_grads(state, mel, g.double(), dims["n_fft"], dims["hop_length"])
    m = _module(dims, state, engine)
    audio, got = _grads(m, mel, g)
    assert rel_errs(audio, ref_audio)[1] <= BARS[engine]
    _check_grads(got, ref, BARS[engine], f"{case} {engine}")


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tcgen05", "simt"])
@pytest.mark.parametrize("name", sorted(G.FIXTURES))
def test_gradients_vs_reference_golden(name, engine, golden_dir):
    """(norm, probe dot) of every parameter gradient of the unmodified reference Vocos in float64 (make_golden_vocos_grad.py)"""
    path = os.path.join(golden_dir, name + ".npz")
    z = np.load(path)
    cs = G.FIXTURES[name]
    dims = G.case_dims(cs)
    state = G.case_state(cs)
    assert np.allclose(G.checksums(state), z["checksums"], rtol=1e-12, atol=0)
    mel = G.case_mel(cs)
    g = G.seeded((cs["B"], cs["T"] * dims["hop_length"]), cs["seed"], 1)
    m = _module(dims, state, engine)
    audio, got = _grads(m, mel.float(), g.float())
    assert rel_errs(audio, torch.from_numpy(z["audio"]))[1] <= BARS[engine]
    stats = G.grad_stats([got[n].cpu().double() for n in m._shapes], cs["seed"])
    ref = torch.from_numpy(z["grad_stats"])
    norm_err = ((stats[:, 0] - ref[:, 0]).abs() / ref[:, 0]).max()
    # the probe dot of a tensor: its error is at most ||d|| ||probe||, so bound it relative to ||grad|| ||probe||
    probe = torch.tensor([float(np.sqrt(np.prod(s))) for s in G.param_sizes(dims)], dtype=torch.float64)
    dot_err = ((stats[:, 1] - ref[:, 1]).abs() / (ref[:, 0] * probe)).max()
    print(f"{name} {engine}: gradient norms max rel {float(norm_err):.2e}, probe dots {float(dot_err):.2e}")
    assert norm_err <= BARS[engine] and dot_err <= BARS[engine]


def _small(engine="tcgen05", seed=9):
    state = V.make_state(seed, **API)
    m = _module(API, state, engine)
    mel = V.make_mel(seed, 2, 12)
    g = G.seeded((2, 12 * 512), seed, 1).float()
    return state, m, mel, g


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tcgen05", "simt"])
def test_train_audio_bitwise_equals_eval_and_repeats(engine):
    _, m, mel, g = _small(engine)
    a1, g1 = _grads(m, mel, g)
    a2, g2 = _grads(m, mel, g)
    with torch.no_grad():
        a_eval = m.eval()(mel.cuda())
    m.train()
    assert a1.requires_grad is False and torch.equal(a1, a_eval) and torch.equal(a1, a2)
    assert all(torch.equal(g1[n], g2[n]) for n in g1)


@pytest.mark.gpu
def test_two_forwards_then_two_backwards():
    _, m, mel, g = _small()
    mel2 = V.make_mel(10, 2, 12)
    _, ga = _grads(m, mel, g)
    _, gb = _grads(m, mel2, 2 * g)
    m.zero_grad(set_to_none=True)
    a1 = m(mel.cuda())
    a2 = m(mel2.cuda())
    (a2 * (2 * g).cuda()).sum().backward(retain_graph=False)
    first = {n: m._param(n).grad.clone() for n in m._shapes}
    m.zero_grad(set_to_none=True)
    (a1 * g.cuda()).sum().backward()
    assert all(torch.equal(first[n], gb[n]) for n in gb)
    assert all(torch.equal(m._param(n).grad, ga[n]) for n in ga)


@pytest.mark.gpu
def test_adamw_step_between_calls_matches_oracle_at_new_weights():
    state, m, mel, g = _small()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    _grads(m, mel, g)
    opt.step()
    new = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    _, got = _grads(m, mel, g)
    _, ref = G.oracle_grads(new, mel, g.double(), 2048, 512)
    _check_grads(got, ref, BARS["tcgen05"], "after one AdamW step")


@pytest.mark.gpu
def test_refusals_and_eval_path():
    _, m, mel, g = _small()
    with pytest.raises(NotImplementedError, match="mel gradient"):
        m(mel.cuda().requires_grad_())
    audio = m(mel.cuda())
    s = (audio * g.cuda()).sum()
    gp = torch.autograd.grad(s, [m._param("head.out.bias")], create_graph=True)[0]
    with pytest.raises(RuntimeError):
        gp.sum().backward()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(mel)
    out = m.eval()(mel.cuda())
    assert not out.requires_grad
    m.train()
    with torch.no_grad():
        assert not m(mel.cuda()).requires_grad
    for p in m.parameters():
        p.requires_grad_(False)
    assert not m(mel.cuda()).requires_grad


@pytest.mark.gpu
def test_wrong_handle_kind_refused():
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    h = C.c_void_p()
    assert lib.st_create_mpd(2, 0, C.byref(h)) == 0
    try:
        buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
        f = torch.zeros(4096, device="cuda")
        assert lib.st_vocos_saved_bytes(h, 1, 4) == 0
        assert lib.st_vocos_forward_train(h, f.data_ptr(), f.data_ptr(), 1, 4, buf.data_ptr(), None) != 0
        assert b"handle is not a Vocos vocoder" in lib.st_last_error(h)
        ptrs = (C.c_void_p * 1)(f.data_ptr())
        assert lib.st_vocos_backward(h, buf.data_ptr(), f.data_ptr(), 1, 4, ptrs, None) != 0
        assert b"handle is not a Vocos vocoder" in lib.st_last_error(h)
    finally:
        lib.st_destroy(h)


@pytest.mark.gpu
def test_two_adamw_generator_half_steps_vs_staged_reference():
    """train.py's generator half-step with the Vocos swapped (mel loss on the generated audio; the discriminators' terms
    are a seeded linear functional here), two AdamW steps against the staged reference Vocos with TF32 off.  Bars of
    test_two_adamw_half_steps_vs_staged_reference (test_mpd.py): losses 1e-3 relative; at most 1 % of the parameter
    elements end more than lr / 2 from the reference's, none more than 6 lr."""
    from oracle import stage_mel_loss
    if not stage_mel_loss.available():
        pytest.skip("oracle/_ref/vocos was not staged by build() (no reference checkout where it ran)")
    from stabletts_b200 import Vocos
    ref_loss, ref_model, _, ref_cfg = stage_mel_loss.load_reference()
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        torch.manual_seed(0)
        ref = ref_model.Vocos(ref_cfg.VocosConfig(), ref_cfg.MelConfig()).cuda().train()
        ours = Vocos(ref_cfg.VocosConfig(), ref_cfg.MelConfig()).cuda().train()
        ours.load_state_dict(ref.state_dict(), strict=True)
        mels = V.make_mel(3, 2, 40).cuda()
        audios = 0.1 * G.seeded((2, 40 * 512), 3, 2).float().cuda()
        w = G.seeded((2, 40 * 512), 3, 3).float().cuda()
        loss_fn = ref_loss.MultiScaleMelSpectrogramLoss().cuda()
        runs = {}
        for name, m in (("ours", ours), ("ref", ref)):
            opt = torch.optim.AdamW(m.parameters(), lr=1e-4, betas=(0.8, 0.99))
            losses = []
            for _ in range(2):
                opt.zero_grad()
                fake = m(mels)
                loss = loss_fn(fake, audios) * 45 + 1e-3 * (fake * w).sum()
                loss.backward()
                torch.nn.utils.clip_grad_norm_(m.parameters(), 1000)
                opt.step()
                losses.append(float(loss.detach()))
            runs[name] = (losses, {k: v.detach().clone() for k, v in m.state_dict().items()})
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    (lo, so), (lr_, sr) = runs["ours"], runs["ref"]
    lr = 1e-4
    loss_err = max(abs(a - b) / abs(b) for a, b in zip(lo, lr_))
    diffs = torch.cat([(so[k] - sr[k]).abs().flatten() for k in sr])
    frac, mx = float((diffs > lr / 2).double().mean()), float(diffs.max()) / lr
    print(f"losses {lo} vs {lr_}: max rel {loss_err:.2e}; parameter elements > lr/2 apart {frac:.2e}, max {mx:.2f} lr")
    assert loss_err <= 1e-3 and frac <= 1e-2 and mx <= 6
