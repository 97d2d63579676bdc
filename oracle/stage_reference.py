"""Stage the reference's OWN modules for the hot path under the git-ignored ``oracle/_ref/`` (TEST / BASELINE
INFRASTRUCTURE ONLY — nothing under ``stabletts_b200/`` ever imports them).

    python -m oracle.stage_reference          # needs a checkout of the reference (STABLETTS_REFERENCE_DIR)

A machine that only has this repository has no reference checkout, so the files the CPU baseline needs —
``models/estimator.py``, ``models/diffusion_transformer.py``, ``models/flow_matching.py``, ``utils/mask.py`` (BASELINE.md
§4, SURVEY.md appendix) — are copied UNMODIFIED, byte for byte, into ``oracle/_ref/`` which is listed in ``.gitignore``
(never enters history; it travels with the built tree like the ``.so``).  A manifest with the
SHA-256 of every staged file is written next to them; ``load_reference()`` verifies it before importing, so what
``bench.py --impl reference`` times is provably the genuine module.  ``torchdiffeq`` is absent: a stand-in module
supplying only the fixed-grid stepping (``oracle.estimator_ref.odeint_fixed``) is registered before the import, exactly as
``oracle/make_golden.py`` does.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("STABLETTS_REFERENCE_DIR", "")        # a checkout of KdaiP/StableTTS @ 71dfa41; unset: nothing is staged
DST = os.path.join(ROOT, "oracle", "_ref")
FILES = ["models/estimator.py", "models/diffusion_transformer.py", "models/flow_matching.py", "utils/mask.py"]
PACKAGES = ["models", "utils"]


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(force: bool = False) -> bool:
    """Copies the files (if the reference checkout is present).  Returns True when oracle/_ref is usable."""
    if not REF or not os.path.isdir(REF):
        return os.path.exists(os.path.join(DST, "MANIFEST.json"))
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(REF, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if force or not os.path.exists(dst) or _sha(dst) != _sha(src):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    for pkg in PACKAGES:                       # the reference's package markers are empty files
        init = os.path.join(DST, pkg, "__init__.py")
        if not os.path.exists(init):
            open(init, "w").close()
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump({"source": "KdaiP/StableTTS @ 71dfa41, copied unmodified", "sha256": manifest}, f, indent=1)
    return True


def available() -> bool:
    return os.path.exists(os.path.join(DST, "MANIFEST.json"))


def load_reference():
    """Imports the staged, checksum-verified reference modules and returns (Decoder, CFMDecoder)."""
    if not available():
        raise RuntimeError("oracle/_ref is not staged (run `python -m oracle.stage_reference` where a reference checkout exists)")
    manifest = json.load(open(os.path.join(DST, "MANIFEST.json")))["sha256"]
    for rel, digest in manifest.items():
        if _sha(os.path.join(DST, rel)) != digest:
            raise RuntimeError(f"oracle/_ref/{rel} does not match its manifest digest")
    from oracle.estimator_ref import odeint_fixed
    stub = types.ModuleType("torchdiffeq")

    def odeint(f, y0, t, method=None, rtol=None, atol=None):
        return odeint_fixed(f, y0, t, method)[None]            # trajectory[-1] is the final state
    stub.odeint = odeint
    sys.modules.setdefault("torchdiffeq", stub)
    if DST not in sys.path:
        sys.path.insert(0, DST)
    for name in ("models", "models.estimator", "models.diffusion_transformer", "models.flow_matching", "utils", "utils.mask"):
        mod = sys.modules.get(name)
        if mod is not None and not getattr(mod, "__file__", "").startswith(tuple(p for p in (DST, REF) if p)):
            del sys.modules[name]                              # an unrelated `models` / `utils` package shadows the staged one
    from models.estimator import Decoder                       # noqa: E402
    from models.flow_matching import CFMDecoder                # noqa: E402
    return Decoder, CFMDecoder


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "reference checkout not present and nothing staged", DST)
