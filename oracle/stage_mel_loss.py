"""Stage the reference's OWN Vocos training modules under the git-ignored ``oracle/_ref/vocos/`` (BASELINE INFRASTRUCTURE
ONLY — nothing under ``stabletts_b200/`` ever imports them), for the reference arms of ``bench_mel_loss.py``.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_mel_loss

``vocoders/vocos/{config.py, models/*.py, utils/audio.py}`` are copied UNMODIFIED, byte for byte, with their SHA-256 digests
in ``oracle/_ref/vocos/MANIFEST.json``; ``load_reference()`` verifies them before importing.  They get a directory of their
own because their module names (config, models, utils) are also the main reference's.  They need torchaudio.
"""
from __future__ import annotations

import glob
import hashlib
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")
DST = os.path.join(ROOT, "oracle", "_ref", "vocos")
MANIFEST = os.path.join(DST, "MANIFEST.json")


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(force: bool = False) -> bool:
    """Copies the files (if the reference checkout is present).  Returns True when the staged copy is usable."""
    src_root = os.path.join(REF, "vocoders", "vocos") if REF else ""
    if not src_root or not os.path.isdir(src_root):
        return available()
    rels = ["config.py", "utils/audio.py"] + sorted(os.path.relpath(p, src_root) for p in glob.glob(os.path.join(src_root, "models", "*.py")))
    manifest = {}
    for rel in rels:
        src, dst = os.path.join(src_root, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if force or not os.path.exists(dst) or _sha(dst) != _sha(src):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    init = os.path.join(DST, "utils", "__init__.py")          # the reference's package marker is an empty file
    if not os.path.exists(init):
        open(init, "w").close()
    with open(MANIFEST, "w") as f:
        json.dump({"source": "KdaiP/StableTTS vocoders/vocos, copied unmodified", "sha256": manifest}, f, indent=1)
    return True


def available() -> bool:
    return os.path.exists(MANIFEST)


def load_reference():
    """Imports the staged, checksum-verified modules; returns the reference's ``models.loss``, ``models.model``,
    ``models.discriminator`` and ``config`` modules."""
    if not available():
        raise RuntimeError("the reference vocoders/vocos is not staged (run `python -m oracle.stage_mel_loss` where a checkout exists)")
    for rel, digest in json.load(open(MANIFEST))["sha256"].items():
        if _sha(os.path.join(DST, rel)) != digest:
            raise RuntimeError(f"oracle/_ref/vocos/{rel} does not match its manifest digest")
    for name in [k for k in sys.modules if k in ("config", "utils", "models") or k.startswith(("utils.", "models."))]:
        del sys.modules[name]                                 # the main reference's modules of the same names
    sys.path.insert(0, DST)
    try:
        import config
        from models import discriminator, loss, model
    finally:
        sys.path.remove(DST)
    return loss, model, discriminator, config


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "reference checkout not present and nothing staged", DST)
