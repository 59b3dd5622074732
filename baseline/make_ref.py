"""Place the UNMODIFIED reference package next to the bench so that `bench.py --impl reference` and the
`cpu_baseline` leg can time the reference itself on the GPU box's host cores.

    python baseline/make_ref.py            # build container only: /root/reference must exist

`pip install --no-index --no-build-isolation --target baseline/_ref /root/reference` (the contract's recipe) fails here:
the reference's build backend is `pdm-backend`, which is not installed and cannot be fetched (no network).  The
package is pure Python, so this recipe copies `src/ptwt` byte for byte into the git-ignored `baseline/_ref/ptwt`
(never into history; it travels to the GPU box with the snapshot) and records the file hashes.  PyWavelets is absent
from the image as well: the reference is imported with the `pywt` / `more_itertools` shims of `oracle/shims`
(filter taps and level formulas only).  Nothing in the product imports `baseline/`.
"""
from __future__ import annotations

import hashlib
import json
import shutil
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
SRC = Path("/root/reference/src/ptwt")
DST = HERE / "_ref" / "ptwt"


def make(force: bool = False) -> Path | None:
    if DST.exists() and not force:
        return DST
    try:
        present = SRC.is_dir()
    except OSError:          # a reference checkout the building user may not read counts as absent
        present = False
    if not present:
        return None
    if DST.exists():
        shutil.rmtree(DST)
    DST.parent.mkdir(parents=True, exist_ok=True)
    shutil.copytree(SRC, DST, ignore=shutil.ignore_patterns("__pycache__"))
    manifest = {str(p.relative_to(DST)): hashlib.sha256(p.read_bytes()).hexdigest() for p in sorted(DST.rglob("*.py"))}
    (DST.parent / "MANIFEST.json").write_text(json.dumps({"source": str(SRC), "files": manifest}, indent=1))
    return DST


def import_ref():
    """The reference `ptwt` module from baseline/_ref (None when it was never placed there)."""
    import importlib

    if not (DST / "__init__.py").exists():
        return None
    shims = HERE.parent / "oracle" / "shims"
    for mod in ("pywt", "more_itertools"):
        try:
            importlib.import_module(mod)
        except Exception:  # noqa: BLE001
            if str(shims) not in sys.path:
                sys.path.insert(0, str(shims))
    if str(DST.parent) not in sys.path:
        sys.path.insert(0, str(DST.parent))
    return importlib.import_module("ptwt")


if __name__ == "__main__":
    out = make(force="--force" in sys.argv)
    print(out if out else "reference not present: nothing copied")
