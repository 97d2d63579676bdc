"""Stage the reference's OWN ``utils/audio.py`` under the git-ignored ``oracle/_ref/`` (BASELINE INFRASTRUCTURE ONLY —
nothing under ``stabletts_b200/`` ever imports it), for the reference arm of ``bench_mel.py``.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_mel

The file is copied UNMODIFIED, byte for byte, next to the modules ``oracle/stage_reference.py`` stages, with its SHA-256
digest in ``oracle/_ref/MEL_MANIFEST.json``; ``load_reference()`` verifies it before importing.  It needs torchaudio (its
MelScale).  Without a reference checkout nothing is staged and ``bench_mel.py`` reports the oracle's parity only.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")
DST = os.path.join(ROOT, "oracle", "_ref")
MANIFEST = os.path.join(DST, "MEL_MANIFEST.json")
FILES = ["utils/audio.py"]


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(force: bool = False) -> bool:
    """Copies the file (if the reference checkout is present).  Returns True when the staged copy is usable."""
    if not REF or not os.path.isdir(REF):
        return available()
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(REF, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if force or not os.path.exists(dst) or _sha(dst) != _sha(src):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    init = os.path.join(DST, "utils", "__init__.py")          # the reference's package marker is an empty file
    if not os.path.exists(init):
        open(init, "w").close()
    with open(MANIFEST, "w") as f:
        json.dump({"source": "KdaiP/StableTTS utils/audio.py, copied unmodified", "sha256": manifest}, f, indent=1)
    return True


def available() -> bool:
    return os.path.exists(MANIFEST)


def load_reference():
    """Imports the staged, checksum-verified utils/audio.py and returns the reference LogMelSpectrogram class."""
    if not available():
        raise RuntimeError("the reference utils/audio.py is not staged (run `python -m oracle.stage_mel` where a checkout exists)")
    for rel, digest in json.load(open(MANIFEST))["sha256"].items():
        if _sha(os.path.join(DST, rel)) != digest:
            raise RuntimeError(f"oracle/_ref/{rel} does not match its manifest digest")
    if DST not in sys.path:
        sys.path.insert(0, DST)
    for name in ("utils", "utils.audio"):
        mod = sys.modules.get(name)
        if mod is not None and not getattr(mod, "__file__", "").startswith(tuple(p for p in (DST, REF) if p)):
            del sys.modules[name]                              # an unrelated `utils` package shadows the staged one
    from utils.audio import LogMelSpectrogram                  # noqa: E402
    return LogMelSpectrogram


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "reference checkout not present and nothing staged", DST)
