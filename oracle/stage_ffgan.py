"""Stage the reference's OWN FireflyGAN modules under the git-ignored ``oracle/_ref/`` (BASELINE INFRASTRUCTURE ONLY —
nothing under ``stabletts_b200/`` ever imports them), for the PyTorch arm of ``bench_vocoder.py``.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_ffgan

``vocoders/ffgan/{backbone,head,model}.py`` (and the empty package markers) are copied UNMODIFIED, byte for byte, next to
the modules ``oracle/stage_reference.py`` stages, with their SHA-256 digests in ``oracle/_ref/FFGAN_MANIFEST.json``;
``load_reference()`` verifies them before importing.  Without a reference checkout nothing is staged and
``bench_vocoder.py`` times the oracle restatement instead (labelled ``kind: "port"``).
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
MANIFEST = os.path.join(DST, "FFGAN_MANIFEST.json")
FILES = ["vocoders/__init__.py", "vocoders/ffgan/__init__.py", "vocoders/ffgan/backbone.py", "vocoders/ffgan/head.py",
         "vocoders/ffgan/model.py"]


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(force: bool = False) -> bool:
    """Copies the files (if the reference checkout is present).  Returns True when the staged copy is usable."""
    if not REF or not os.path.isdir(REF):
        return available()
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(REF, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if force or not os.path.exists(dst) or _sha(dst) != _sha(src):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    with open(MANIFEST, "w") as f:
        json.dump({"source": "KdaiP/StableTTS vocoders/ffgan, copied unmodified", "sha256": manifest}, f, indent=1)
    return True


def available() -> bool:
    return os.path.exists(MANIFEST)


def load_reference():
    """Imports the staged, checksum-verified reference module and returns its FireflyGANBase class."""
    if not available():
        raise RuntimeError("the reference FireflyGAN is not staged (run `python -m oracle.stage_ffgan` where a checkout exists)")
    for rel, digest in json.load(open(MANIFEST))["sha256"].items():
        if _sha(os.path.join(DST, rel)) != digest:
            raise RuntimeError(f"oracle/_ref/{rel} does not match its manifest digest")
    if DST not in sys.path:
        sys.path.insert(0, DST)
    from vocoders.ffgan.model import FireflyGANBase           # noqa: E402
    return FireflyGANBase


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "reference checkout not present and nothing staged", DST)
