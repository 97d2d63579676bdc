"""tests/golden/vocos_*.npz from the UNMODIFIED reference Vocos (authoring container only; run in its own process
because the vocoder's ``models`` / ``config`` packages shadow the TTS ones):  python -m oracle.make_golden_vocoder"""
import os
import sys

import numpy as np
import torch

from oracle import vocoder_ref as V

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    sys.path.insert(0, os.path.join(os.environ.get("STABLETTS_REFERENCE_DIR", ""), "vocoders", "vocos"))
    from config import MelConfig, VocosConfig            # vocoders/vocos/config.py
    from models.model import Vocos                       # vocoders/vocos/models/model.py
    m = Vocos(VocosConfig(), MelConfig()).eval()
    st = V.make_state()
    missing = m.load_state_dict(st, strict=True)
    print("load_state_dict:", missing)
    for name, cs in V.CASES.items():
        mel = V.make_mel(cs["seed"], cs["B"], cs["T"])
        with torch.inference_mode():
            audio = m(mel)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), audio=audio.numpy().astype(np.float32),
                            weight_checksum=float(sum(float(v.double().sum()) for v in st.values())))
        print(name, tuple(audio.shape), float(audio.abs().max()))


if __name__ == "__main__":
    main()
