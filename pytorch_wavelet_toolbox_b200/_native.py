"""ctypes binding of libwtb200.so (the C ABI in include/wtb200.h).

There is NO CPU or PyTorch fallback behind these calls: if the shared object is missing
or no CUDA device is usable, the public transforms raise ``RuntimeError``.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
import contextlib
from typing import Iterator, Optional, Sequence

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "csrc" / "libwtb200.so"

WT_F32, WT_F64 = 0, 1
MODES = {"zero": 0, "constant": 1, "reflect": 2, "periodic": 3, "symmetric": 4}
WT_MAX_FILT_LEN = 128
WT_EWORKSPACE = -3

_i64 = C.c_int64
_i64p = C.POINTER(C.c_int64)
_i32p = C.POINTER(C.c_int32)
_f64p = C.POINTER(C.c_double)
_vp = C.c_void_p


class WtLevel(C.Structure):
    """``struct wt_level`` (include/wtb200.h)."""

    _fields_ = [
        ("details", _vp),
        ("approx", _vp),
        ("dims", _i64 * 3),
        ("strides", _i64 * 3),
        ("approx_strides", _i64 * 3),
        ("details_batch_stride", _i64),
        ("band_stride", _i64),
        ("approx_batch_stride", _i64),
    ]


#: every symbol include/wtb200.h declares -> (restype, argtypes)
SIGNATURES = {
    "wt_version": (C.c_int, []),
    "wt_last_error": (C.c_char_p, []),
    "wt_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "wt_coeff_len": (_i64, [_i64, C.c_int]),
    "wt_dwt_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, _i64, _i64p, C.c_int]),
    "wt_dwt_fwd": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f64p, _f64p, _vp, _i64, _i64p,
                             _i64p, _i64, C.POINTER(WtLevel), _vp, C.c_size_t, _vp]),
    "wt_dwt_inv": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _f64p, _f64p, _vp, _i64, _i64p, _i64p, _i64,
                             C.POINTER(WtLevel), _vp, C.c_size_t, _vp]),
    "wt_matrix_fwd": (C.c_int, [C.c_int, C.c_int, C.c_int, _f64p, _f64p, _i64p, _i32p, C.c_int, _i32p, _i32p,
                                _i32p, _i32p, _vp, _vp, _i64, _i64, C.POINTER(_vp), _i64p, _vp, _i64, _vp,
                                C.c_size_t, C.c_int, _vp]),
    "wt_matrix_inv": (C.c_int, [C.c_int, C.c_int, C.c_int, _f64p, _f64p, _i64p, _i64p, _i32p, _i32p, _i32p,
                                _i32p, _vp, _vp, _i64, C.POINTER(_vp), _i64p, _i64, _vp, _i64, _vp, C.c_size_t,
                                C.c_int, _vp]),
    "wt_matrix_axis_fwd": (C.c_int, [C.c_int, C.c_int, _f64p, _f64p, _i64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, _vp, _vp, _i64, _i64, _i64, _i64, _vp, _i64, _i64, _vp]),
    "wt_matrix_axis_inv": (C.c_int, [C.c_int, C.c_int, _f64p, _f64p, _i64, _i64, C.c_int, C.c_int, C.c_int, C.c_int,
                                     _vp, _vp, _i64, _i64, _i64, _i64, _vp, _i64, _i64, _vp]),
    "wt_tap_corr": (C.c_int, [C.c_int, C.c_int, _vp, _vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp]),
    "wt_swt_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, _i64, _i64, C.POINTER(_vp), C.c_int]),
    "wt_swt_fwd": (C.c_int, [C.c_int, C.c_int, C.c_int, _f64p, _f64p, _vp, _i64, _i64, _i64, _vp, _i64, _i64,
                             C.POINTER(_vp), _vp, C.c_size_t, _vp]),
    "wt_swt_inv": (C.c_int, [C.c_int, C.c_int, C.c_int, _f64p, _f64p, _vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp,
                             _i64, C.POINTER(_vp), _vp, C.c_size_t, _vp]),
    "wt_swt_pass_plan": (C.c_int, [C.c_int, C.c_int, C.c_int, _i64, _i64, _i64p]),
    "wt_swt2_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, _i64, _i64, _i64]),
    "wt_swt_pass_fwd": (C.c_int, [C.c_int, C.c_int, _f64p, _f64p, _i64, C.c_int, C.POINTER(_vp), _i64p,
                                  C.POINTER(_vp), _i64p, C.POINTER(_vp), _i64p, _i64, _i64, _vp]),
    "wt_swt_pass_inv": (C.c_int, [C.c_int, C.c_int, _f64p, _f64p, _i64, C.c_int, C.POINTER(_vp), _i64p,
                                  C.POINTER(_vp), _i64p, C.POINTER(_vp), _i64p, _i64, _i64, _vp]),
    "wt_cwt_workspace_bytes": (C.c_size_t, [C.c_int, _i64, _i64, _i64, C.c_int]),
    "wt_cwt_filter_spectra": (C.c_int, [C.c_int, _i64, _vp, _vp, _vp, _vp]),
    "wt_cwt_fwd": (C.c_int, [C.c_int, C.c_int, _i64, _vp, _vp, _vp, C.c_int, _vp, _i64, _i64, _i64, _vp, _i64, _i64,
                             _vp, C.c_size_t, _vp]),
    "wt_cwt_adj": (C.c_int, [C.c_int, C.c_int, _i64, _vp, _vp, _vp, C.c_int, _vp, _i64, _i64, _i64, _i64, _vp, _i64,
                             _vp, C.c_size_t, _vp]),
    "wt_launch_count": (C.c_uint64, []),
    "wt_launch_count_reset": (None, []),
    "wt_set_knob": (C.c_int, [C.c_char_p, C.c_longlong]),
    "wt_unset_knob": (C.c_int, [C.c_char_p]),
    "wt_get_knob": (C.c_int, [C.c_char_p, C.POINTER(C.c_longlong)]),
}

_lib: Optional[C.CDLL] = None


class NativeError(RuntimeError):
    """A libwtb200 call failed (bad argument or CUDA error)."""


def load() -> C.CDLL:
    """Load the in-tree shared object; raise loudly if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("WTB200_LIB", LIB_PATH))
    if not path.exists():
        raise RuntimeError(
            f"libwtb200.so not found at {path}. Build it with "
            "`python -m pytorch_wavelet_toolbox_b200.csrc.build` (needs nvcc); there is no CPU fallback."
        )
    lib = C.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the .so disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().wt_last_error().decode("utf-8", "replace")
        kind = "CUDA error" if rc > 0 else "invalid argument"
        raise NativeError(f"{what} failed ({kind} {rc}): {msg}")


def f64_array(a: Sequence[float]):
    arr = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
    return arr, arr.ctypes.data_as(_f64p)


def i64_array(a: Sequence[int]):
    arr = np.ascontiguousarray(np.asarray(a, dtype=np.int64))
    return arr, arr.ctypes.data_as(_i64p)


def i32_array(a: Sequence[int]):
    arr = np.ascontiguousarray(np.asarray(a, dtype=np.int32))
    return arr, arr.ctypes.data_as(_i32p)


def coeff_len(n: int, filt_len: int) -> int:
    """Per-level output extent: pad (2L-3)//2 left, that + n%2 right, stride-2 valid conv
    (reference src/ptwt/_util.py:198-228)."""
    padl = (2 * filt_len - 3) // 2
    return (n + 2 * padl + (n % 2) - filt_len) // 2 + 1


def launch_count() -> int:
    return int(load().wt_launch_count())


def launch_count_reset() -> None:
    load().wt_launch_count_reset()


def set_knob(name: str, value: Optional[int]) -> None:
    """Set (or with ``None`` unset) a tuning / test switch of the library (include/wtb200.h, csrc/knobs.cuh)."""
    lib = load()
    rc = lib.wt_unset_knob(name.encode()) if value is None else lib.wt_set_knob(name.encode(), int(value))
    check(rc, f"wt_set_knob({name})")


def get_knob(name: str) -> Optional[int]:
    v = C.c_longlong(0)
    rc = load().wt_get_knob(name.encode(), C.byref(v))
    if rc < 0:
        check(rc, f"wt_get_knob({name})")
    return int(v.value) if rc == 1 else None


@contextlib.contextmanager
def knobs(**values: Optional[int]) -> Iterator[None]:
    """``with knobs(NO_WPAIR=1): ...`` -- switches restored on exit."""
    old = {k: get_knob(k) for k in values}
    try:
        for k, v in values.items():
            set_knob(k, v)
        yield
    finally:
        for k, v in old.items():
            set_knob(k, v)
