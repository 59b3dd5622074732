"""pytorch_wavelet_toolbox_b200 -- H100-native backend for ptwt's fast wavelet transforms.

The eight names below are drop-ins for the functions / classes of the same name in
``ptwt`` (v0lta/PyTorch-Wavelet-Toolbox): identical signatures, return containers and
errors; the arithmetic runs in hand-written sm_90a CUDA kernels behind the C ABI declared
in ``include/wtb200.h``.

    import pytorch_wavelet_toolbox_b200 as ptwt_b200
    coeffs = ptwt_b200.wavedec2(images, "db4", level=4)      # CUDA or CPU tensors
    ptwt_b200.install()                                      # make ``ptwt.wavedec2`` etc. use it
"""
from __future__ import annotations

from . import constants
from .constants import (
    Wavelet,
    WaveletCoeff1d,
    WaveletCoeff2d,
    WaveletCoeffNd,
    WaveletDetailDict,
    WaveletDetailTuple2d,
    WaveletTensorTuple,
)
from .fwt import host_staging, wavedec, wavedec2, wavedec3, waverec, waverec2, waverec3
from .matrix_fwt import MatrixWavedec, MatrixWaverec, construct_boundary_a, construct_boundary_s
from .matrix_fwt_nd import MatrixWavedec2, MatrixWavedec3, MatrixWaverec2, MatrixWaverec3
from .separable import fswavedec2, fswavedec3, fswaverec2, fswaverec3
from .packets import WaveletPacket, WaveletPacket2D, WaveletPacket3D
from .stationary import iswt, iswt2, swt, swt2
from .continuous import cwt

__version__ = "0.1.0"

HOT_PATH_NAMES = (
    "wavedec", "waverec", "wavedec2", "waverec2", "wavedec3", "waverec3", "MatrixWavedec", "MatrixWaverec",
)
#: "next" rows of SURVEY.md section 8(f) that ride on the same kernels
NEXT_ROW_NAMES = (
    "fswavedec2", "fswavedec3", "fswaverec2", "fswaverec3",
    "MatrixWavedec2", "MatrixWaverec2", "MatrixWavedec3", "MatrixWaverec3",  # separable mode only
    "WaveletPacket", "WaveletPacket2D",                                      # level-wise batched node expansion
    "swt", "iswt",                                                           # stationary transform, csrc/swt.cuh
    "cwt",                                                                   # continuous transform, csrc/cwt.cuh
)

#: additions beyond the ptwt API: ptwt has no such names, so install() has nothing to rebind for them
BEYOND_PTWT_NAMES = ("WaveletPacket3D", "swt2", "iswt2")

__all__ = list(HOT_PATH_NAMES) + list(NEXT_ROW_NAMES) + list(BEYOND_PTWT_NAMES) + [
    "Wavelet", "WaveletTensorTuple", "WaveletDetailTuple2d", "WaveletDetailDict", "WaveletCoeff1d",
    "WaveletCoeff2d", "WaveletCoeffNd", "construct_boundary_a", "construct_boundary_s", "install", "uninstall", "host_staging",
]

_saved: dict = {}


def install() -> list[str]:
    """Rebind the hot-path names inside an importable ``ptwt`` to this backend.

    ptwt has no backend registry (SURVEY.md section 8b), so the switch is a rebinding of the eight
    names in ``ptwt``, in the defining modules and in the modules that imported them by value
    (``ptwt.packets``, ``ptwt.separable_conv_transform``; reference packets.py:34-37,
    separable_conv_transform.py:33).  Returns the list of ``module.name`` bindings replaced.
    """
    import importlib
    import sys
    import warnings

    import torch

    from . import _native

    # This backend has no CPU compute path: on a machine without a usable CUDA device (or without the built library)
    # rebinding would turn a working CPU ptwt into a failing one, so nothing is touched there.
    try:
        usable = torch.cuda.is_available() and _native.load() is not None
    except Exception:  # noqa: BLE001
        usable = False
    if not usable:
        warnings.warn("pytorch_wavelet_toolbox_b200.install(): no CUDA device / libwtb200.so -- ptwt left untouched",
                      RuntimeWarning, stacklevel=2)
        return []
    ptwt = importlib.import_module("ptwt")
    mine = {name: globals()[name] for name in HOT_PATH_NAMES + NEXT_ROW_NAMES}
    replaced = []
    for modname, mod in list(sys.modules.items()):
        if mod is None or not (modname == "ptwt" or modname.startswith("ptwt.")):
            continue
        for name, obj in mine.items():
            cur = getattr(mod, name, None)
            if cur is not None and cur is not obj:
                _saved.setdefault((modname, name), cur)
                setattr(mod, name, obj)
                replaced.append(f"{modname}.{name}")
    del ptwt
    return replaced


def uninstall() -> None:
    """Undo :func:`install`."""
    import sys

    for (modname, name), obj in list(_saved.items()):
        mod = sys.modules.get(modname)
        if mod is not None:
            setattr(mod, name, obj)
    _saved.clear()
