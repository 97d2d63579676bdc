"""Stage the reference's OWN ``monotonic_align/`` package under the git-ignored ``oracle/_ref/`` (BASELINE INFRASTRUCTURE
ONLY — nothing under ``stabletts_b200/`` ever imports it), for the reference arms of ``bench_mas.py``.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_mas

``monotonic_align/__init__.py`` and ``core.py`` are copied UNMODIFIED, byte for byte, with their SHA-256 digests in
``oracle/_ref/MAS_MANIFEST.json``; ``load_reference()`` verifies them before importing.  The package needs numba.  Without
a reference checkout nothing is staged and ``bench_mas.py`` reports the reference's time as not measured.
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
MANIFEST = os.path.join(DST, "MAS_MANIFEST.json")
FILES = ["monotonic_align/__init__.py", "monotonic_align/core.py"]


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(force: bool = False) -> bool:
    """Copies the package (if the reference checkout is present).  Returns True when the staged copy is usable."""
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
        json.dump({"source": "KdaiP/StableTTS monotonic_align/, copied unmodified", "sha256": manifest}, f, indent=1)
    return True


def available() -> bool:
    return os.path.exists(MANIFEST)


def load_reference():
    """Imports the staged, checksum-verified package and returns the module (its ``maximum_path``).  Raises ImportError
    when numba is missing."""
    if not available():
        raise RuntimeError("the reference monotonic_align is not staged (run `python -m oracle.stage_mas` where a checkout exists)")
    for rel, digest in json.load(open(MANIFEST))["sha256"].items():
        if _sha(os.path.join(DST, rel)) != digest:
            raise RuntimeError(f"oracle/_ref/{rel} does not match its manifest digest")
    mod = sys.modules.get("monotonic_align")
    if mod is not None and not getattr(mod, "__file__", "").startswith(DST):
        del sys.modules["monotonic_align"]                     # e.g. the stub stage_synth registers for synthesise-only use
    if DST not in sys.path:
        sys.path.insert(0, DST)
    import monotonic_align                                     # noqa: E402
    return monotonic_align


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "reference checkout not present and nothing staged", DST)
