"""CPU oracle of ``StableTTS.synthesise`` (TEST INFRASTRUCTURE ONLY): models/model.py:49-112 composed from the oracles
of its stages — style_ref (MelStyleEncoder), text_encoder_ref (TextEncoder), duration_ref (DurationPredictor), align_ref
(durations -> alignment -> mu_y) and estimator_ref (the CFM solve, with the initial noise z passed in).  Pinned by
tests/test_synthesise.py against tests/golden/synth_*.npz (oracle/make_golden_synth.py, unmodified reference)."""
from __future__ import annotations

from collections import OrderedDict

import torch

from oracle import align_ref, duration_ref, estimator_ref, style_ref, text_encoder_ref, weights

N_VOCAB = 401


def sub(state, prefix):
    return OrderedDict((k[len(prefix):], v) for k, v in state.items() if k.startswith(prefix))


def make_state(seed=81, n_mel=80):
    """The 189 tensors of StableTTS(401, n_mel, 256, 1024, 4, 3, 6, 3, 0.1, 256) in the reference's state_dict order:
    both adaLN gate sets re-randomised (the reference zeroes them, which would hide every DiT block), dp.proj.bias = log 4,
    and non-zero fake_speaker / fake_content."""
    fs, fc = weights.make_cfg_params(seed, n_mel)
    st = OrderedDict([("fake_speaker", fs), ("fake_content", fc)])
    for prefix, part in (("encoder.", text_encoder_ref.make_state(seed + 1, out_channels=n_mel)),
                         ("ref_encoder.", style_ref.make_state(seed + 2, n_mel)),
                         ("dp.", duration_ref.make_state(seed + 3)),
                         ("decoder.estimator.", weights.make_state(seed + 4, n_mel))):
        st.update((prefix + k, v) for k, v in part.items())
    return st


def make_inputs(seed, lens, T_ref, n_mel):
    """Interspersed token ids (blank 0 between symbols, datas/dataset.py intersperse), their lengths, a reference mel."""
    g = torch.Generator().manual_seed(seed)
    B, Tx = len(lens), max(lens)
    ids = torch.randint(1, N_VOCAB, (B, Tx), generator=g)
    ids[:, 0::2] = 0
    ids = ids * (torch.arange(Tx)[None] < torch.as_tensor(lens)[:, None])
    y = torch.randn(B, n_mel, T_ref, generator=g) * 2.0 - 4.0
    return ids, torch.as_tensor(lens), y


def front(state, ids, lens, y):
    """c, (x, mu_x, x_mask), logw: models/model.py:79-81."""
    c = style_ref.style_forward(sub(state, "ref_encoder."), y, None)
    x, mu_x, x_mask = text_encoder_ref.text_encoder_forward(sub(state, "encoder."), ids, c, lens)
    logw = duration_ref.dp_forward(sub(state, "dp."), x, x_mask, c)
    return c, mu_x, x_mask, logw


def synthesise(state, ids, lens, n_timesteps, y, z, length_scale=1.0, solver="euler", cfg=1.0):
    """models/model.py:49-112 with the CFM's noise z (B, n_mel, T_y) passed in.  Returns the reference's dict."""
    with torch.inference_mode():
        c, mu_x, x_mask, logw = front(state, ids, lens, y)
        mu_y, y_mask, _, attn = align_ref.expand_by_durations(logw, x_mask, mu_x, length_scale)
        guide = None if cfg == 1.0 else dict(fake_speaker=state["fake_speaker"], fake_content=state["fake_content"], cfg_strength=cfg)
        dec = estimator_ref.cfm_forward(sub(state, "decoder.estimator."), mu_y, y_mask, n_timesteps, z, c, solver, guide)
    return {"encoder_outputs": mu_y, "decoder_outputs": dec, "attn": attn}


CASES = {
    # the shape api.py uses: one utterance of 129 interspersed tokens, a 5 s reference (430 frames at 44.1 kHz / hop 512),
    # 128 mel channels, CFG 3.0, 10-step Euler
    "synth_api":   dict(seed=91, lens=[129], T_ref=430, n_mel=128, n_timesteps=10, solver="euler", cfg=3.0, length_scale=1.0),
    "synth_b3":    dict(seed=92, lens=[61, 37, 15], T_ref=120, n_mel=80, n_timesteps=4, solver="midpoint", cfg=1.0,
                        length_scale=1.15),
    "synth_mel80": dict(seed=93, lens=[33, 21], T_ref=64, n_mel=80, n_timesteps=3, solver="euler", cfg=2.0, length_scale=1.0),
}
