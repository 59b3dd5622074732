"""Every kernel instantiation compiled into libwtb200.so is either mapped to a case that launches it or recorded as
unreachable with a reason (tests/kernel_cases.py).  Adding or removing an instantiation without updating the
inventory fails here; no GPU needed."""
from __future__ import annotations

import shutil
import subprocess
from pathlib import Path

import pytest

from kernel_cases import CASES, UNREACHABLE


def normalise(name: str) -> str:
    """``void wtb::k<float, 2>(wtb::P<float>)`` -> ``k<float, 2>``: no ``void``, no namespace, no argument list."""
    name = name.strip()
    if name.startswith("void "):
        name = name[len("void "):]
    name = name.replace("wtb::", "")
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i].strip()
    return name


def _tool(name: str, cuda_name: str | None = None) -> str | None:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    bindir = Path(nvcc).resolve().parent
    for cand in (bindir / name, shutil.which(name), bindir / cuda_name if cuda_name else None):
        if cand and Path(cand).exists():
            return str(cand)
    return None


def compiled_kernels() -> set[str]:
    from pytorch_wavelet_toolbox_b200 import _native

    _native.load()          # raises if the library was not built
    lib = Path(_native.LIB_PATH)
    cuobjdump = _tool("cuobjdump")
    cxxfilt = _tool("c++filt", "cu++filt")
    if not cuobjdump or not cxxfilt:
        pytest.skip(f"needs cuobjdump and c++filt from the CUDA toolkit (found {cuobjdump}, {cxxfilt})")
    out = subprocess.run([cuobjdump, "-symbols", str(lib)], capture_output=True, text=True, check=True).stdout
    mangled = [ln.split()[-1] for ln in out.splitlines() if "STO_ENTRY" in ln]
    assert mangled, f"cuobjdump lists no kernel entry in {lib}"
    dem = subprocess.run([cxxfilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
    names = [normalise(n) for n in dem.splitlines() if n.strip()]
    assert len(names) == len(mangled)
    return set(names)


def test_normalise():
    assert normalise("void wtb::axis1d_fast_kernel<float, 4, 2, false>(wtb::Fast1dParams<float>)") == \
        "axis1d_fast_kernel<float, 4, 2, false>"
    assert normalise("wtb::cwt_filter_spectra_kernel(double2 const*, double2 const*, double2*, int)") == \
        "cwt_filter_spectra_kernel"


def test_every_instantiation_is_mapped_or_unreachable():
    compiled = compiled_kernels()
    assert not set(CASES) & set(UNREACHABLE), sorted(set(CASES) & set(UNREACHABLE))
    missing = sorted(compiled - set(CASES) - set(UNREACHABLE))
    stale = sorted((set(CASES) | set(UNREACHABLE)) - compiled)
    assert not missing, f"{len(missing)} compiled instantiations have no case and no reason: {missing}"
    assert not stale, f"{len(stale)} inventory entries are not compiled: {stale}"
    print(f"{len(compiled)} instantiations: {len(CASES)} with a case, {len(UNREACHABLE)} unreachable")


def test_unreachable_reasons_are_given():
    for name, reason in UNREACHABLE.items():
        assert isinstance(reason, str) and reason.strip(), name


def test_cases_are_well_formed():
    entries = {"wavedec", "waverec", "wavedec2", "waverec2", "wavedec3", "waverec3", "MatrixWavedec", "MatrixWaverec",
               "MatrixWavedec2", "MatrixWaverec2", "swt", "iswt", "cwt", "cwt_grad", "wavedec_tap_grad"}
    layouts = {"packed", "offset", "pitch", "pitch16", "own", "views", "contiguous"}
    for name, c in CASES.items():
        assert c["entry"] in entries, name
        assert c["dtype"] in ("float32", "float64"), name
        assert c["layout"] in layouts, name
        assert c["modes"], name
