"""Stage the reference's OWN StableTTS front-end modules under the git-ignored ``oracle/_ref/`` (BASELINE INFRASTRUCTURE
ONLY — nothing under ``stabletts_b200/`` ever imports them), for the PyTorch arm of ``bench_synthesise.py``.

    STABLETTS_REFERENCE_DIR=<checkout> python -m oracle.stage_synth

``models/{model,text_encoder,reference_encoder,duration_predictor}.py`` are copied UNMODIFIED, byte for byte, next to the
modules ``oracle/stage_reference.py`` stages (estimator, DiT blocks, flow matching, utils/mask.py), with their SHA-256
digests in ``oracle/_ref/SYNTH_MANIFEST.json``; ``load_reference()`` verifies both manifests before importing.
``monotonic_align`` (imported by models/model.py, used only by the training forward) is replaced by a stub.  Without a
reference checkout nothing is staged and ``bench_synthesise.py`` times the oracle restatement instead (``kind: "port"``).
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import sys
import types

from oracle import stage_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")
DST = os.path.join(ROOT, "oracle", "_ref")
MANIFEST = os.path.join(DST, "SYNTH_MANIFEST.json")
FILES = ["models/model.py", "models/text_encoder.py", "models/reference_encoder.py", "models/duration_predictor.py"]


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(force: bool = False) -> bool:
    """Copies the files (if the reference checkout is present).  Returns True when the staged copy is usable."""
    if not REF or not os.path.isdir(REF):
        return available()
    if not stage_reference.stage(force):
        return False
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(REF, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if force or not os.path.exists(dst) or _sha(dst) != _sha(src):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    with open(MANIFEST, "w") as f:
        json.dump({"source": "KdaiP/StableTTS models/, copied unmodified", "sha256": manifest}, f, indent=1)
    return True


def available() -> bool:
    return os.path.exists(MANIFEST) and stage_reference.available()


def load_reference():
    """Imports the staged, checksum-verified reference modules and returns the reference StableTTS class."""
    if not available():
        raise RuntimeError("the reference StableTTS is not staged (run `python -m oracle.stage_synth` where a checkout exists)")
    for rel, digest in json.load(open(MANIFEST))["sha256"].items():
        if _sha(os.path.join(DST, rel)) != digest:
            raise RuntimeError(f"oracle/_ref/{rel} does not match its manifest digest")
    stage_reference.load_reference()                     # verifies its own manifest, registers the torchdiffeq stand-in
    if "monotonic_align" not in sys.modules:
        stub = types.ModuleType("monotonic_align")

        def maximum_path(*args, **kwargs):
            raise RuntimeError("monotonic_align is not staged: StableTTS.forward (training) is not part of the baseline")
        stub.maximum_path = maximum_path
        sys.modules["monotonic_align"] = stub
    from models.model import StableTTS                    # noqa: E402
    return StableTTS


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "reference checkout not present and nothing staged", DST)
