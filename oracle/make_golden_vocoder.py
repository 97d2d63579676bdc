"""tests/golden/vocos_*.npz from the UNMODIFIED reference Vocos (authoring container only; each configuration runs in its own
process because the vocoder's ``models`` / ``config`` packages shadow the TTS ones):

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_vocoder          # vocos_b*  (vocoders/vocos/config.py)
    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.make_golden_vocoder --api    # vocos_api_*  (api.py's Vocos)
"""
import os
import sys

import numpy as np
import torch

from oracle import vocoder_ref as V

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")


def write(m, cases):
    for name, cs in cases.items():
        st = V.make_state(**cs.get("state", {}))
        print("load_state_dict:", m.load_state_dict(st, strict=True))
        mel = V.make_mel(cs["seed"], cs["B"], cs["T"])
        with torch.inference_mode():
            audio = m(mel)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), audio=audio.numpy().astype(np.float32),
                            weight_checksum=float(sum(float(v.double().sum()) for v in st.values())))
        print(name, tuple(audio.shape), float(audio.abs().max()))


def main():
    """the vocos training configuration: vocoders/vocos first on sys.path, so `config` is vocoders/vocos/config.py"""
    sys.path.insert(0, os.path.join(REF, "vocoders", "vocos"))
    from config import MelConfig, VocosConfig            # vocoders/vocos/config.py
    from models.model import Vocos                       # vocoders/vocos/models/model.py
    write(Vocos(VocosConfig(), MelConfig()).eval(), V.CASES)


def main_api():
    """api.py's get_vocoder(..., 'vocos'), imported as api.py imports it: the reference root on sys.path, so `config` (in
    api.py and in vocoders/vocos/models/model.py alike) is the top-level config.py"""
    if not REF:
        raise SystemExit("set STABLETTS_REFERENCE_DIR to a checkout of the reference")
    sys.path.insert(0, REF)
    from vocoders.vocos.models.model import Vocos        # api.py:27
    from config import MelConfig, VocosConfig            # api.py:28
    assert os.path.samefile(sys.modules["config"].__file__, os.path.join(REF, "config.py")), sys.modules["config"].__file__
    vc = VocosConfig()
    got = dict(dim=vc.dim, intermediate_dim=vc.intermediate_dim, num_layers=vc.num_layers)
    assert got == V.API_DIMS, got
    write(Vocos(vc, MelConfig()).eval(), V.API_CASES)


if __name__ == "__main__":
    main_api() if "--api" in sys.argv else main()
