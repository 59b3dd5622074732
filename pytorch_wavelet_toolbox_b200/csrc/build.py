"""Build libwtb200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m pytorch_wavelet_toolbox_b200.csrc.build [--force] [--verbose]

The shared object is plain C ABI (include/wtb200.h): no torch / pybind dependency, the
CUDA runtime is linked statically, so the file runs on any machine with an H100 and a recent driver.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
LIB = HERE / "libwtb200.so"
SOURCES = [HERE / "wtb200.cu"]
HEADERS = sorted(HERE.glob("*.cuh")) + [ROOT / "include" / "wtb200.h"]
# traffic twin of fwd2d_wpair_kernel for tools/time_wpair_ceiling.py: a separate object, never part of the library
TWIN = ROOT / "tools" / "wpair_twin" / "libwpair_twin.so"
TWIN_SOURCES = [ROOT / "tools" / "wpair_twin" / "wpair_twin.cu"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: cannot build libwtb200.so")


def needs_build(out: Path = LIB, sources: list[Path] = SOURCES) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(p.stat().st_mtime > t for p in sources + HEADERS + [Path(__file__)])


def build(force: bool = False, verbose: bool = False, extra: list[str] | None = None) -> Path:
    """Build libwtb200.so and the wpair traffic twin; returns the library's path."""
    _build_one(TWIN, TWIN_SOURCES, force, verbose, extra)
    return _build_one(LIB, SOURCES, force, verbose, extra)


def _build_one(out: Path, sources: list[Path], force: bool, verbose: bool, extra: list[str] | None) -> Path:
    if not force and not needs_build(out, sources):
        return out
    cmd = [
        _nvcc(), "-O3", "-std=c++17",
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-lineinfo",
        "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
        "--expt-relaxed-constexpr",
        "-shared", "-cudart", "static",
        "-o", str(out),
    ] + [str(s) for s in sources]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    if extra:
        cmd += extra
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if verbose:
        sys.stderr.write(proc.stdout + proc.stderr)
    return out


if __name__ == "__main__":
    out = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(out)
