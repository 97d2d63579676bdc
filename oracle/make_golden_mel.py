"""Fixtures of the log-mel front end from the UNMODIFIED reference module utils/audio.py::LogMelSpectrogram:

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_mel

writes tests/golden/mel_*.npz.  Each mel case stores the module's output in float64 (the module and input .double()) and
in fp32, `E32` = max |fp32 - float64| (the reference's own fp32 error), the module's `fb`, and the waveform's checksum (the
waveforms are regenerated from oracle/mel_ref.py's seeds).  The LinearSpectrogram cases store the float64 magnitude.  The
composed case runs the fp32 module into the reference's MelStyleEncoder (oracle/style_ref.py's seeded weights, 128 mels,
no mask: api.py:72-73 then models/model.py:79) and stores c."""
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mel_ref as M, style_ref, weights            # noqa: E402
from oracle.stage_reference import REF                         # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _import_reference():
    if not REF or not os.path.isdir(REF):
        raise SystemExit("set STABLETTS_REFERENCE_DIR to a checkout of the reference")
    sys.path.insert(0, REF)
    from config import MelConfig
    from utils.audio import LogMelSpectrogram
    from models.reference_encoder import MelStyleEncoder
    return MelConfig, LogMelSpectrogram, MelStyleEncoder


def _wave(cs, cfg):
    return M.make_batch(cs["kinds"], cs["seed"], cs["L"], cfg["sample_rate"])


def main():
    MelConfig, LogMelSpectrogram, MelStyleEncoder = _import_reference()
    torch.set_grad_enabled(False)
    for name, cfg in M.CONFIGS.items():                        # the oracle's configs are the reference's MelConfig
        kw = {k: v for k, v in cfg.items() if k in ("sample_rate", "n_fft", "win_length", "hop_length", "n_mels")}
        assert asdict(MelConfig(**kw)) == cfg, name
    for name, cs in M.CASES.items():
        cfg = M.CONFIGS[cs["cfg"]]
        m = LogMelSpectrogram(**cfg).eval()
        x = _wave(cs, cfg)
        out32 = m(x)
        out64 = m.double()(x.double())
        e32 = float((out32.double() - out64).abs().max())
        print(f"{name}: T {out64.shape[-1]}, E32 {e32:.3e}, range [{float(out64.min()):.2f}, {float(out64.max()):.2f}]")
        np.savez_compressed(os.path.join(OUT, name + ".npz"), out64=out64.numpy(), out32=out32.numpy(), E32=e32,
                            fb=m.mel_scale.fb.float().numpy(), wave_checksum=M.checksum(x))
    for name, cs in M.LINEAR_CASES.items():
        cfg = M.CONFIGS[cs["cfg"]]
        m = LogMelSpectrogram(**cfg).eval().double()
        x = _wave(cs, cfg)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), linear64=m.spectrogram(x.double()).numpy(),
                            wave_checksum=M.checksum(x))
    cs = M.COMPOSED
    cfg = M.CONFIGS[cs["cfg"]]
    x = _wave(cs, cfg)
    mel = LogMelSpectrogram(**cfg).eval()(x)
    st = style_ref.make_state(n_mel=cfg["n_mels"])
    enc = MelStyleEncoder(cfg["n_mels"], style_vector_dim=256, style_kernel_size=5).eval()
    enc.load_state_dict(st, strict=True)
    c = enc(mel, None)
    assert torch.isfinite(c).all()
    np.savez_compressed(os.path.join(OUT, cs["name"] + ".npz"), c=c.numpy(), wave_checksum=M.checksum(x),
                        weight_checksum=weights.checksum(st))


if __name__ == "__main__":
    main()
