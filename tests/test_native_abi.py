"""The C-ABI library loads and exports every symbol include/wtb200.h declares (no GPU needed)."""
from __future__ import annotations

import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _declared_symbols():
    text = (ROOT / "include" / "wtb200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(wt_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_expected_surface():
    names = _declared_symbols()
    for must in ("wt_dwt_fwd", "wt_dwt_inv", "wt_matrix_fwd", "wt_matrix_inv", "wt_last_error", "wt_version"):
        assert must in names


def test_library_exports_every_declared_symbol():
    from pytorch_wavelet_toolbox_b200 import _native

    lib = _native.load()
    for name in _declared_symbols():
        assert hasattr(lib, name), f"libwtb200.so does not export {name}"
    assert set(_native.SIGNATURES) == set(_declared_symbols())
    assert lib.wt_version() == 100


def test_struct_layout_matches_header():
    from pytorch_wavelet_toolbox_b200 import _native

    # 2 pointers + (3 + 3 + 3) int64 + 3 int64
    assert ctypes.sizeof(_native.WtLevel) == 2 * 8 + 9 * 8 + 3 * 8


def test_coeff_len_matches_reference_formula():
    from pytorch_wavelet_toolbox_b200 import _native

    lib = _native.load()
    for L in (2, 4, 8, 12, 16, 5, 7):
        for n in (1, 2, 7, 16, 31, 64, 65, 4096, 2051):
            padl = (2 * L - 3) // 2
            want = (n + 2 * padl + n % 2 - L) // 2 + 1
            assert lib.wt_coeff_len(n, L) == want == _native.coeff_len(n, L)
    # the sizes SURVEY.md quotes for BASELINE config 2 and 5
    sizes = [4096]
    for _ in range(4):
        sizes.append(_native.coeff_len(sizes[-1], 8))
    assert sizes == [4096, 2051, 1029, 518, 262]
    sizes = [2048]
    for _ in range(5):
        sizes.append(_native.coeff_len(sizes[-1], 16))
    assert sizes == [2048, 1031, 523, 269, 142, 78]


def test_bad_arguments_are_rejected_without_a_gpu():
    from pytorch_wavelet_toolbox_b200 import _native

    lib = _native.load()
    dims, dims_p = _native.i64_array([16])
    lo, lo_p = _native.f64_array([0.7, 0.7])
    rc = lib.wt_dwt_fwd(4, 0, 0, 1, 2, lo_p, lo_p, None, 1, dims_p, dims_p, 16, None, None, 0, None)
    assert rc == -1 and b"ndim" in lib.wt_last_error()
    rc = lib.wt_dwt_fwd(1, 0, 9, 1, 2, lo_p, lo_p, None, 1, dims_p, dims_p, 16, None, None, 0, None)
    assert rc == -1 and b"mode" in lib.wt_last_error()
    rc = lib.wt_dwt_fwd(1, 0, 0, 1, 500, lo_p, lo_p, None, 1, dims_p, dims_p, 16, None, None, 0, None)
    assert rc == -4
    with pytest.raises(_native.NativeError):
        _native.check(rc, "wt_dwt_fwd")


KNOB_NAMES = (
    "DISABLE_FUSED", "NO_FFMA2", "CHUNK", "STREAMS", "FWD3D_TILE", "CONVF_CHUNK", "CONVF_K", "MATF_CHUNK",
    "MATI_CHUNK", "MATF_K", "MATI_K", "MATI_NT", "MATI_MINCTAS", "MATI_MERGE_N", "MATF_KCOARSE", "NO_WPAIR",
    "WPAIR_SEG", "WPAIR_MIN", "WPAIR_DEEP", "NO_AUX_STREAM", "WPAIR_VAR", "WPAIR", "MATF_NT", "MATF_MINB", "MATF_CPC",
    "NO_DMMA", "FUSE2",
)
# switches of matrix-FWT kernels that have been removed: unknown names now
RETIRED_KNOB_NAMES = ("MATF_VARIANT", "DMMA_PERM", "MATF_MINCTAS", "MATI_ROWS")


def test_knob_registry_lists_exactly_the_live_switches_and_rejects_retired_ones():
    """The tuning / test switches (csrc/knobs.cuh) are process state of the library, set through the C ABI: exactly
    the names listed here are accepted, set / get / unset round-trip, negative values survive, unknown and retired
    names fail with WT_EINVAL instead of being silently ignored."""
    from pytorch_wavelet_toolbox_b200 import _native

    text = (ROOT / "pytorch_wavelet_toolbox_b200" / "csrc" / "knobs.cuh").read_text()
    body = text[text.index("#define WTB_KNOB_LIST(X)"):text.index("enum KnobId")]
    names = re.findall(r"X\(([A-Z0-9_]+)\)", body)
    assert len(KNOB_NAMES) == 27
    assert tuple(names) == KNOB_NAMES
    for must in ("NO_DMMA", "MATI_K", "MATF_K", "WPAIR", "DISABLE_FUSED"):
        assert must in names
    lib = _native.load()
    for name in RETIRED_KNOB_NAMES:
        assert name not in names
        value = ctypes.c_longlong(0)
        assert lib.wt_set_knob(name.encode(), 1) == -1 and b"unknown knob" in lib.wt_last_error()  # WT_EINVAL
        assert lib.wt_get_knob(name.encode(), ctypes.byref(value)) == -1
        with pytest.raises(_native.NativeError):
            _native.set_knob(name, 1)
        with pytest.raises(_native.NativeError):
            _native.get_knob(name)
    for name in names:
        before = _native.get_knob(name)
        with _native.knobs(**{name: -3}):
            assert _native.get_knob(name) == -3
            with _native.knobs(**{name: None}):
                assert _native.get_knob(name) is None
            assert _native.get_knob(name) == -3
        assert _native.get_knob(name) == before
    with pytest.raises(Exception):
        _native.set_knob("NOT_A_KNOB", 1)
    with pytest.raises(Exception):
        _native.get_knob("NOT_A_KNOB")
