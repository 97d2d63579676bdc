"""Groundwork for SURVEY.md §8 row f4 (vocoder hand-off): the CPU oracle of the reference's Vocos, pinned against
fixtures generated from the unmodified reference (oracle/make_golden_vocoder.py), in BOTH formulations of the inverse
STFT — the reference's irfft + fold, and the single windowed-inverse-DFT GEMM + overlap-add gather the tensor-core
path will run.  There is no CUDA path for this row yet; nothing here touches the product."""
import os

import numpy as np
import pytest
import torch

from oracle import vocoder_ref as V


ALL_CASES = {**V.CASES, **V.API_CASES}


@pytest.mark.parametrize("name", list(ALL_CASES))
@pytest.mark.parametrize("gemm_istft", [False, True])
def test_vocos_restatement_vs_reference_golden(name, gemm_istft, golden_dir):
    """both configurations: the vocos training config (vocos_b*) and api.py's 512 / 1536 / 8 Vocos (vocos_api_*), whose
    fixtures come from the reference imported exactly as api.py imports it"""
    cs = ALL_CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    st = V.make_state(**cs.get("state", {}))
    assert abs(float(sum(float(v.double().sum()) for v in st.values())) - float(g["weight_checksum"])) < 1e-6 * abs(float(g["weight_checksum"]))
    mel = V.make_mel(cs["seed"], cs["B"], cs["T"])
    with torch.inference_mode():
        audio = V.vocos_forward(st, mel, gemm_istft=gemm_istft)
    ref = torch.from_numpy(g["audio"])
    assert audio.shape == ref.shape == (cs["B"], cs["T"] * 512)
    err = float((audio - ref).abs().max() / ref.abs().max())
    assert err < (2e-4 if gemm_istft else 2e-5), err          # fp32 GEMM over K = 2050 vs the FFT: rounding only


def test_istft_gemm_formulation_is_exact_in_float64():
    """[re | im] · W followed by the 4-frame gather equals irfft + fold + envelope to float64 rounding, including the
    DC / Nyquist imaginary parts irfft ignores and the trimmed 'same' padding."""
    g = torch.Generator().manual_seed(5)
    B, T, n_fft, hop = 2, 9, 2048, 512
    re = torch.randn(B, n_fft // 2 + 1, T, generator=g, dtype=torch.float64)
    im = torch.randn(B, n_fft // 2 + 1, T, generator=g, dtype=torch.float64)
    w = torch.hann_window(n_fft, dtype=torch.float64)
    a = V.istft_same_reference(re, im, w, n_fft, hop)
    b = V.istft_same_as_gemm(re, im, w, n_fft, hop)
    assert a.shape == b.shape == (B, T * hop)
    assert float((a - b).abs().max()) < 1e-11 * float(a.abs().max() + 1)


def test_default_head_gain_keeps_the_training_config_states():
    """head_gain's default is the scale the committed vocos_b* fixtures were made with"""
    a, b = V.make_state(), V.make_state(head_gain=0.5)
    assert all(torch.equal(a[k], b[k]) for k in a)


def test_clip_fixture_drives_a_share_of_magnitudes_onto_the_clip():
    """vocos_api_b2_t64_clip's head gain puts 5 % to 30 % of its (frame, bin) magnitudes above 1e2, so the
    min(exp(m), 1e2) of head.py:106 decides part of the audio; the other fixtures stay below it"""
    for name, cs in V.API_CASES.items():
        st = V.make_state(**cs["state"])
        with torch.inference_mode():
            m = V.head_log_magnitudes(st, V.make_mel(cs["seed"], cs["B"], cs["T"]))
        frac = float((m.exp() > 1e2).double().mean())
        if name.endswith("_clip"):
            assert 0.05 <= frac <= 0.30, frac
        else:
            assert frac == 0.0, (name, frac)
