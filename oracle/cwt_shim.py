"""Continuous wavelets for the PyWavelets stand-in -- TEST INFRASTRUCTURE ONLY.

The reference's cwt module imports ``ContinuousWavelet``, ``DiscreteContinuousWavelet`` and
``pywt._functions.scale2frequency`` (src/ptwt/continuous_transform.py:10-11) and subclasses ``ContinuousWavelet`` for
its learnable wavelets, so these must be in place BEFORE the reference is imported.  When PyWavelets itself is
absent, :func:`import_reference` adds them to the stand-in in ``oracle/shims/pywt`` and then imports the reference:
  * ``ContinuousWavelet`` is the package's built-in table (mexh, morl, cmorB-C, shanB-C), the same provenance rule
    the stand-in already follows for filter taps.  Its attributes are set in ``__new__``, as pywt sets them in
    ``__cinit__``; the reference's ``_DifferentiableContinuousWavelet.__init__`` relies on that.
  * ``DiscreteContinuousWavelet`` dispatches continuous names to it and everything else to the discrete stand-in.
  * ``_functions.central_frequency`` / ``scale2frequency`` restate pywt's (argmax of ``|fft(psi)[1:]|``, folded to
    the lower half, over the support's length).
The discrete part of the stand-in is untouched, so the existing fixtures are generated exactly as before.
"""
from __future__ import annotations

import importlib
import sys

import numpy as np

from pytorch_wavelet_toolbox_b200._wavelets import CONTINUOUS_BOUNDS, BuiltinContinuousWavelet

from . import ref_import


def _is_continuous_name(name) -> bool:
    return isinstance(name, str) and (name in CONTINUOUS_BOUNDS or name.startswith(("cmor", "shan")))


def _extend(pywt) -> None:
    if getattr(pywt, "ContinuousWavelet", None) is BuiltinContinuousWavelet:
        return
    discrete = pywt.Wavelet

    def DiscreteContinuousWavelet(name, filter_bank=None):
        if _is_continuous_name(name):
            return BuiltinContinuousWavelet(name)
        return discrete(name, filter_bank)

    def central_frequency(wavelet, precision=8):
        if not isinstance(wavelet, (discrete, BuiltinContinuousWavelet)):
            wavelet = DiscreteContinuousWavelet(wavelet)
        approx = wavelet.wavefun(precision)
        psi, x = (approx[0], approx[1]) if len(approx) == 2 else (approx[1], approx[-1])
        domain = float(x[-1] - x[0])
        index = np.argmax(abs(np.fft.fft(np.asarray(psi))[1:])) + 2
        if index > len(psi) / 2:
            index = len(psi) - index + 2
        return 1.0 / (domain / (index - 1))

    def scale2frequency(wavelet, scale, precision=8):
        return central_frequency(wavelet, precision=precision) / scale

    pywt.ContinuousWavelet = BuiltinContinuousWavelet
    pywt.DiscreteContinuousWavelet = DiscreteContinuousWavelet
    pywt._functions.central_frequency = central_frequency
    pywt._functions.scale2frequency = scale2frequency
    pywt.central_frequency, pywt.scale2frequency = central_frequency, scale2frequency


def import_reference():
    """The unmodified reference ``ptwt``, with continuous wavelets in the PyWavelets stand-in if that is in use."""
    if not ref_import.reference_available():
        raise RuntimeError("the reference checkout is not present on this machine")
    try:
        pywt = importlib.import_module("pywt")
    except Exception:  # noqa: BLE001
        if str(ref_import.SHIMS) not in sys.path:
            sys.path.insert(0, str(ref_import.SHIMS))
        pywt = importlib.import_module("pywt")
    if getattr(pywt, "__version__", "") == "0.0-shim":
        if "ptwt.continuous_transform" in sys.modules and \
                sys.modules["ptwt.continuous_transform"].ContinuousWavelet is not BuiltinContinuousWavelet:
            raise RuntimeError("the reference was imported before its continuous wavelets were provided; "
                               "import it through oracle.cwt_shim.import_reference in a fresh process")
        _extend(pywt)
    return ref_import.import_reference()
