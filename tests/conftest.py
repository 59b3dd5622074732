"""pytest configuration: `gpu` marker, repo root on sys.path, shared helpers."""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = ROOT / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")
    config.addinivalue_line("markers", "slow: long-running")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    manifest = json.loads((GOLDEN / "reference_vectors.json").read_text())
    arrays = np.load(GOLDEN / "reference_vectors.npz")
    return manifest, arrays


@pytest.fixture(scope="session")
def reference_api():
    """What the unmodified reference computed beyond the transform vectors (oracle/make_golden_api.py)."""
    manifest = json.loads((GOLDEN / "reference_api.json").read_text())
    arrays = np.load(GOLDEN / "reference_api.npz")
    return manifest, arrays


@pytest.fixture
def knob():
    """Set tuning / test switches of libwtb200 for one test: ``knob("NO_WPAIR", 1)`` (restored afterwards)."""
    from pytorch_wavelet_toolbox_b200 import _native

    saved = {}

    def _set(name, value):
        if name not in saved:
            saved[name] = _native.get_knob(name)
        _native.set_knob(name, value)

    yield _set
    for name, value in saved.items():
        _native.set_knob(name, value)


def flatten_coeffs(coeffs):
    """Coefficient pytree -> flat tensor list in the order the golden fixtures use."""
    out = []
    for el in coeffs:
        if isinstance(el, torch.Tensor):
            out.append(el)
        elif isinstance(el, dict):
            out.extend(el[k] for k in ("aad", "ada", "add", "daa", "dad", "dda", "ddd"))
        else:
            out.extend(el)
    return out


#: stated tolerances of the parity gate (SURVEY.md section 8d): |delta| <= TOL[dtype] * max|coefficient| -- the scale
#: is always max|reference value| of the compared tensor (or of the coefficient tree it belongs to), never a looser
#: constant (round 1 used 10.0 / 10 * max|x| in places)
TOL = {torch.float32: 1e-5, torch.float64: 1e-11}


def assert_close_rel(got: torch.Tensor, want: torch.Tensor, dtype=None, scale=None, what=""):
    got = got.detach().cpu()
    want = want.detach().cpu()
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    assert got.dtype == want.dtype, f"{what}: dtype {got.dtype} != {want.dtype}"
    dtype = dtype or want.dtype
    if want.numel() == 0:
        return
    s = scale if scale is not None else max(float(want.abs().max()), 1e-30)
    err = float((got.double() - want.double()).abs().max())
    assert err <= TOL[dtype] * s, f"{what}: max abs err {err:.3e} > {TOL[dtype]:.0e} * {s:.3e}"
