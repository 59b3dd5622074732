"""A stand-in ``ptwt`` package for the install() tests: the module layout of the reference (the eight hot-path names
in ``ptwt`` and in their defining modules, and the copies ``ptwt.packets`` / ``ptwt.separable_conv_transform`` took by
value, reference packets.py:34-37, separable_conv_transform.py:33), bound to the oracle port, i.e. a working CPU ptwt."""
from __future__ import annotations

import contextlib
import sys
import types

from oracle import ptwt_port as P

LAYOUT = {
    "ptwt.conv_transform": ("wavedec", "waverec"),
    "ptwt.conv_transform_2": ("wavedec2", "waverec2"),
    "ptwt.conv_transform_3": ("wavedec3", "waverec3"),
    "ptwt.matmul_transform": ("MatrixWavedec", "MatrixWaverec"),
    "ptwt.packets": ("wavedec", "waverec", "wavedec2", "waverec2", "WaveletPacket", "WaveletPacket2D"),
    "ptwt.separable_conv_transform": ("wavedec", "waverec", "wavedec2", "wavedec3"),
}


class WaveletPacket:
    """Placeholder for the reference's packet class (only its binding is exercised)."""


class WaveletPacket2D:
    """Placeholder for the reference's 2-D packet class (only its binding is exercised)."""


def _binding(name):
    return {"WaveletPacket": WaveletPacket, "WaveletPacket2D": WaveletPacket2D}.get(name) or getattr(P, name)


@contextlib.contextmanager
def stand_in_ptwt():
    """Register the stand-in as ``ptwt`` for the duration of the block; undo install() and the registration after."""
    import pytorch_wavelet_toolbox_b200 as wt

    saved = {k: v for k, v in sys.modules.items() if k == "ptwt" or k.startswith("ptwt.")}
    for k in saved:
        del sys.modules[k]
    top = types.ModuleType("ptwt")
    sys.modules["ptwt"] = top
    for modname, names in LAYOUT.items():
        mod = types.ModuleType(modname)
        for name in names:
            setattr(mod, name, _binding(name))
            setattr(top, name, _binding(name))
        setattr(top, modname.split(".", 1)[1], mod)
        sys.modules[modname] = mod
    try:
        yield top
    finally:
        wt.uninstall()
        for k in [k for k in sys.modules if k == "ptwt" or k.startswith("ptwt.")]:
            del sys.modules[k]
        sys.modules.update(saved)
