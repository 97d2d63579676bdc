"""Fixtures of resampling from torchaudio, the function the reference calls at utils/audio.py:73 (and
vocoders/vocos/dataset.py):

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_resample

writes tests/golden/rs_*.npz.  Each case stores torchaudio.functional.resample's output in float64 (the waveform .double(),
so the coefficients are float64 too) and in fp32, `E32` = max |fp32 - float64|, the fp32 `kernel` buffer of
torchaudio.transforms.Resample, that kernel evaluated in float64 and rounded once (`kernel64`), and the waveform's checksum
(the waveforms are regenerated from oracle/resample_ref.py's seeds).  The composed case resamples a 48 kHz clip to 44.1 kHz
and runs the reference's LogMelSpectrogram at its default MelConfig, in float64 and in fp32 (needs the reference checkout)."""
import math
import os
import sys
from dataclasses import asdict

import numpy as np
import torch
import torchaudio
from torchaudio.functional.functional import _get_sinc_resample_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import resample_ref as R                           # noqa: E402
from oracle.stage_reference import REF                         # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    torch.set_grad_enabled(False)
    for name, cs in R.CASES.items():
        o, n = cs["orig"], cs["new"]
        x = R.make_batch(cs["kinds"], cs["seed"], cs["L"], o)
        out64 = torchaudio.functional.resample(x.double(), o, n)
        out32 = torchaudio.functional.resample(x, o, n)
        e32 = float((out32.double() - out64).abs().max())
        kernel = torchaudio.transforms.Resample(o, n).kernel
        kernel64 = _get_sinc_resample_kernel(o, n, math.gcd(o, n), dtype=torch.float64)[0].float()
        print(f"{name}: L {cs['L']} -> {out64.shape[-1]}, E32 {e32:.3e}, "
              f"|kernel - kernel64| {float((kernel - kernel64).abs().max()):.2e}")
        np.savez_compressed(os.path.join(OUT, name + ".npz"), out64=out64.numpy(), out32=out32.numpy(), E32=e32,
                            kernel=kernel.numpy(), kernel64=kernel64.numpy(), wave_checksum=R.checksum(x))
    if not REF or not os.path.isdir(REF):
        raise SystemExit("set STABLETTS_REFERENCE_DIR to a checkout of the reference for the composed case")
    sys.path.insert(0, REF)
    from config import MelConfig
    from utils.audio import LogMelSpectrogram
    cs = R.COMPOSED
    x = R.make_batch(cs["kinds"], cs["seed"], cs["L"], cs["orig"])
    mel = LogMelSpectrogram(**asdict(MelConfig())).eval()
    mel32 = mel(torchaudio.functional.resample(x, cs["orig"], cs["new"]))
    mel64 = mel.double()(torchaudio.functional.resample(x.double(), cs["orig"], cs["new"]))
    e32 = float((mel32.double() - mel64).abs().max())
    print(f"{cs['name']}: mel {tuple(mel64.shape)}, E32 {e32:.3e}")
    np.savez_compressed(os.path.join(OUT, cs["name"] + ".npz"), out64=mel64.numpy(), out32=mel32.numpy(), E32=e32,
                        fb=mel.mel_scale.fb.float().numpy(), wave_checksum=R.checksum(x))


if __name__ == "__main__":
    main()
