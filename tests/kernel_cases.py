"""Inventory of the kernel instantiations compiled into libwtb200.so.

``CASES`` maps the normalised name of every instantiation some input can reach (``fwd2d_strip_f32_kernel<12, 64,
false>``: no ``void``, no ``wtb::``, no argument list) to one case that launches it.  ``UNREACHABLE`` maps the
name of every other instantiation to the reason no input reaches it.  tests/test_kernel_inventory.py checks that the
two together are exactly what the library holds; tests/test_gpu_kernel_inventory.py runs every case, checks with the
profiler that the instantiation ran and compares its outputs with the float64 oracle.

A case is a dict:

``entry``
    the public call whose launches are checked: ``wavedec``, ``waverec``, ``wavedec2``, ``waverec2``, ``wavedec3``,
    ``waverec3``, ``MatrixWavedec``, ``MatrixWaverec``, ``MatrixWavedec2``, ``MatrixWaverec2``, ``swt``, ``iswt``,
    ``cwt``, ``cwt_grad`` (the gradient of ``cwt`` with respect to its input) or ``wavedec_tap_grad`` (the
    gradient of ``wavedec`` with respect to learnable filter taps).  A synthesis case first runs the matching
    analysis and compares both with the oracle.
``wavelet``, ``dtype``, ``shape`` (batch first), ``level``
``modes``
    boundary modes (``odd_coeff_padding_mode`` for the matrix transforms) to run, one call each.
``layout``
    of the input of an analysis case: ``packed`` (a contiguous tensor), ``offset`` (storage offset of one element,
    so the base is not on a 16-byte boundary), ``pitch`` (rows of a slightly wider tensor of an odd pitch: never a
    multiple of 16 bytes) or ``pitch16`` (rows of a wider tensor whose pitch is a multiple of 16 elements).
    Of the coefficients of a synthesis case: ``own`` (what this package's analysis returned), ``views`` (the
    oracle's coefficients as it returns them, channel slices of one tensor), ``contiguous`` (each oracle band a
    contiguous tensor of its own) or ``offset`` (each oracle band at a storage offset of one element).
``knobs``
    library switches (include/wtb200.h) set for the call.
``scales``
    the scales of a ``cwt`` case.
``orthogonalization``
    of the boundary rows of a matrix case (``qr`` unless given).
"""
from __future__ import annotations

MODES = ("zero", "constant", "reflect", "periodic", "symmetric")
NON_PERIODIC = ("zero", "constant", "reflect", "symmetric")
FILTER_LENGTHS = (2, 4, 6, 8, 10, 12, 14, 16)
_DB = {2: "haar", 4: "db2", 6: "db3", 8: "db4", 10: "db5", 12: "db6", 14: "db7", 16: "db8"}
_SYM = {8: "sym4", 10: "sym5", 12: "sym6", 14: "sym7", 16: "sym8"}
_TNAME = {"float32": "float", "float64": "double"}
#: elements per 16 bytes
_VEC = {"float32": 4, "float64": 2}


def coeff_len(n: int, filt_len: int) -> int:
    """Extent of one analysis level along an axis of n samples (non-periodic modes)."""
    padl = (2 * filt_len - 3) // 2
    return (n + 2 * padl + (n % 2) - filt_len) // 2 + 1


def wavelet(filt_len: int, alt: bool = False) -> str:
    return _SYM[filt_len] if alt and filt_len in _SYM else _DB[filt_len]


def odd_coarsest(start: int, filt_len: int, level: int) -> int:
    """The first extent >= start whose coarsest approximation (level `level`) has an odd extent: a contiguous band
    of that width has a row pitch that is not a multiple of 16 bytes."""
    n = start
    while True:
        m = n
        for _ in range(level):
            m = coeff_len(m, filt_len)
        if m % 2:
            return n
        n += 1


def case(entry, wavelet, dtype, shape, level=1, modes=("reflect",), layout="packed", knobs=None, **extra):
    c = {"entry": entry, "wavelet": wavelet, "dtype": dtype, "shape": tuple(shape), "level": level,
         "modes": tuple(modes), "layout": layout, "knobs": dict(knobs or {})}
    c.update(extra)
    return c


CASES: dict[str, dict] = {}
UNREACHABLE: dict[str, str] = {}


def _add(name: str, c: dict) -> None:
    assert name not in CASES, name
    CASES[name] = c


# ---- 1-D analysis along a contiguous axis -----------------------------------------------------------------------
# axis1d_fast_kernel<T, L, OFF, MATRIX>: OFF = (first input index of an output) mod (elements per 16 bytes).  The
# convolution path starts at -pad_left(L) = 2 - L, the matrix path at shift - (L - 1) = 1 - L / 2, so OFF is fixed
# by L and the dtype; every other OFF is compiled but never launched.
for dt in ("float32", "float64"):
    T, V = _TNAME[dt], _VEC[dt]
    for L in FILTER_LENGTHS:
        conv_off = (2 - L) % V
        mat_off = (1 - L // 2) % V
        for off in range(V):
            for matrix in (False, True):
                name = f"axis1d_fast_kernel<{T}, {L}, {off}, {str(matrix).lower()}>"
                want = mat_off if matrix else conv_off
                if off != want:
                    path = "matrix path (base = 1 - L/2)" if matrix else "convolution path (base = 2 - L)"
                    UNREACHABLE[name] = f"the {path} fixes OFF = {want} for L = {L} in {T}; OFF {off} is never launched"
                elif matrix:
                    # one level of MatrixWavedec along rows whose pitch is a multiple of 16 bytes; the odd length
                    # pads the level with one sample (odd_coeff_padding_mode)
                    _add(name, case("MatrixWavedec", wavelet(L, dt == "float64"), dt, (3, 2047), 1, MODES, "pitch16"))
                else:
                    # one level (a group of one: the fused multi-level kernel needs two); odd length, rows of a
                    # 16-byte pitch; the periodic mode too
                    _add(name, case("wavedec", wavelet(L, dt == "float64"), dt, (3, 4501), 1, MODES, "pitch16"))

# conv1d_fused_kernel<T, L>: groups of 2..5 levels, not periodic, 16-byte aligned rows
for dt in ("float32", "float64"):
    for L in FILTER_LENGTHS:
        _add(f"conv1d_fused_kernel<{_TNAME[dt]}, {L}>",
             case("wavedec", wavelet(L, dt == "float32"), dt, (3, 4501), 3, NON_PERIODIC, "pitch16"))

# axis1d_inv_fast_kernel<T, L>: every level of waverec whose bands and output rows are 16-byte aligned (all but the
# last level, whose output rows are the caller's)
for dt in ("float32", "float64"):
    for L in FILTER_LENGTHS:
        _add(f"axis1d_inv_fast_kernel<{_TNAME[dt]}, {L}>",
             case("waverec", wavelet(L, dt == "float64"), dt, (3, 4501), 3, ("zero", "periodic"), "own"))

# the general single-axis kernels: rows that are not 16-byte aligned (1-D), float64 3-D
_add("axis_fwd_kernel<float>", case("wavedec", "db3", "float32", (3, 301), 2, MODES, "packed"))
_add("axis_fwd_kernel<double>", case("wavedec3", "db2", "float64", (2, 9, 11, 13), 2, MODES, "packed"))
_add("axis_inv_kernel<float>", case("waverec", "db3", "float32", (3, 301), 1, ("zero", "periodic"), "contiguous"))
_add("axis_inv_kernel<double>", case("waverec3", "db2", "float64", (2, 9, 11, 13), 2, ("zero", "periodic"), "own"))

# ---- 2-D analysis -------------------------------------------------------------------------------------------------
# fwd2d_strip*_kernel<.., TMA>: TMA when the input's base, row pitch and batch stride are multiples of 16 bytes (the
# second level reads this package's own aligned buffer, so it always takes TMA).  203 x 263: three strips of 64
# (float32) or five of 32 (float64) columns with a ragged last one, three row segments, odd extents.
_NO_TMA_LAYOUTS = ("packed", "offset", "pitch")


def _fwd2d_case(dt, L, tma, knobs=None):
    layout = "pitch16" if tma else _NO_TMA_LAYOUTS[(L // 2) % 3]
    return case("wavedec2", wavelet(L, L % 4 == 0), dt, (2, 203, 263), 2, MODES, layout, knobs)


for L in FILTER_LENGTHS:
    for tma in (False, True):
        b = str(tma).lower()
        _add(f"fwd2d_strip_f32_kernel<{L}, 64, {b}>", _fwd2d_case("float32", L, tma))
        _add(f"fwd2d_strip_kernel<float, {L}, 64, {b}>", _fwd2d_case("float32", L, tma, {"NO_FFMA2": 1}))
        _add(f"fwd2d_strip_kernel<double, {L}, 32, {b}>", _fwd2d_case("float64", L, tma))

# levels 1-2 in one launch: the kernel of independent warps (WPAIR, default only for images of >= 2^24 samples;
# WPAIR_VAR picks the variant for L = 8) and the opt-in strip kernel (FUSE2).  Neither accepts the periodic mode.
_WPAIR = {"WPAIR": 1, "WPAIR_MIN": 1}
for L, stages, minb, var in ((2, 3, 12, None), (4, 3, 12, None), (6, 3, 12, None), (8, 2, 12, None), (8, 2, 15, 1),
                             (8, 3, 12, 3)):
    knobs = dict(_WPAIR, **({"WPAIR_VAR": var} if var else {}))
    _add(f"fwd2d_wpair_kernel<{L}, {stages}, {minb}>",
         case("wavedec2", wavelet(L), "float32", (3, 132, 260), 3, NON_PERIODIC, "packed", knobs))
for L in (2, 4, 6, 8):
    _add(f"fwd2d_fuse2_f32_kernel<{L}>",
         case("wavedec2", wavelet(L, L == 8), "float32", (2, 203, 263), 3, NON_PERIODIC, "pitch16",
              {"WPAIR": 0, "FUSE2": 1}))

# ---- 2-D synthesis (float32) --------------------------------------------------------------------------------------
# inv2d_strip_kernel<L, TMA>: TMA when every band of a level has 16-byte aligned rows; coefficients this package did
# not produce (odd widths, offsets, the oracle's channel slices) take the other instantiation
_FOREIGN = ("views", "contiguous", "offset")
for i, L in enumerate(FILTER_LENGTHS):
    _add(f"inv2d_strip_kernel<{L}, true>",
         case("waverec2", wavelet(L), "float32", (2, 203, 263), 2, ("zero", "periodic"), "own"))
    _add(f"inv2d_strip_kernel<{L}, false>",
         case("waverec2", wavelet(L, True), "float32", (2, 201, odd_coarsest(261, L, 2)), 2, ("zero", "periodic"),
              _FOREIGN[i % 3]))

# ---- 3-D (float32, L <= 8) ----------------------------------------------------------------------------------------
# fwd3d_tile_kernel<L, TH, TW, TMA>: FWD3D_TILE 0 / 1 / 2 = 16 x 32, 11 x 44, 8 x 64 output tiles.  7 x 35 x 135:
# two or more tiles along H and W for every shape, odd extents; 136 columns give TMA rows.
_TILES = ((16, 32), (11, 44), (8, 64))
for L in (2, 4, 6, 8):
    for t, (th, tw) in enumerate(_TILES):
        for tma in (False, True):
            layout = "pitch16" if tma else ("packed", "offset", "pitch")[t]
            _add(f"fwd3d_tile_kernel<{L}, {th}, {tw}, {str(tma).lower()}>",
                 case("wavedec3", wavelet(L, t == 1), "float32", (2, 9, 35, 135), 2, MODES, layout,
                      {"FWD3D_TILE": t}))
    _add(f"inv3d_tile_kernel<{L}, true>",
         case("waverec3", wavelet(L), "float32", (2, 7, 35, 135), 2, ("zero", "periodic"), "own"))
    _add(f"inv3d_tile_kernel<{L}, false>",
         case("waverec3", wavelet(L, True), "float32", (2, 7, 33, odd_coarsest(133, L, 2)), 2, ("zero", "periodic"),
              ("views", "contiguous", "offset", "views")[L // 2 - 1]))

# ---- matrix FWT ---------------------------------------------------------------------------------------------------
# Rows of 32767 samples: level 1 pads one sample and runs alone, levels 2-3 (16384 -> 8192 -> 4096 samples) run as one
# fused group over several chunks.  The fused analysis runs only when the entries of the boundary rows in the opposite
# corner are round-off of at most 1e-13: float32 QR leaves ~1e-7 there, Gram-Schmidt exact zeros.
for L in FILTER_LENGTHS:
    for nt in (128, 256):
        _add(f"mat_fwd_dmma2_kernel<{L}, {nt}>",
             case("MatrixWavedec", wavelet(L, nt == 256), "float64", (2, 32767), 3, MODES, "packed", {"MATF_NT": nt}))
        _add(f"mat_inv_dmma_kernel<{L}, {nt}>",
             case("MatrixWaverec", wavelet(L, nt == 128), "float64", (2, 32767), 3, ("zero",), "own", {"MATI_NT": nt}))
    for dt in ("float32", "float64"):
        T = _TNAME[dt]
        for nt, minb in ((128, 1), (128, 6), (256, 1), (256, 3)):
            knobs = {"MATF_NT": nt, "MATF_MINB": 1 if minb == 1 else 2}
            if dt == "float64":
                knobs["NO_DMMA"] = 1
            _add(f"mat_fwd_fused_kernel<{T}, {L}, {nt}, {minb}>",
                 case("MatrixWavedec", wavelet(L, minb > 1), dt, (2, 32767), 3, ("zero", "reflect"), "packed", knobs,
                      orthogonalization="gramschmidt" if dt == "float32" else "qr"))
        _add(f"mat_inv_fast_kernel<{T}, {L}>",
             case("MatrixWaverec", wavelet(L, dt == "float32"), dt, (3, 4095), 2, ("zero",), "own",
                  {"NO_DMMA": 1} if dt == "float64" else {}))
        # separable 2-D: the axis that is not contiguous runs the register-blocked axis kernels
        _add(f"mat_axis_fwd_blk_kernel<{T}, {L}>",
             case("MatrixWavedec2", wavelet(L), dt, (2, 75, 68), 2, ("zero", "reflect"), "packed"))
        _add(f"mat_axis_inv_blk_kernel<{T}, {L}>",
             case("MatrixWaverec2", wavelet(L, True), dt, (2, 75, 68), 2, ("zero",), "own"))
for dt in ("float32", "float64"):
    T = _TNAME[dt]
    # rows whose pitch is not a multiple of 16 bytes: the general kernels
    _add(f"mat_fwd_kernel<{T}>", case("MatrixWavedec", "db3", dt, (3, 1001), 2, MODES, "packed"))
    _add(f"mat_inv_kernel<{T}>", case("MatrixWaverec", "db3", dt, (3, 1001), 2, ("zero",), "own"))
    _add(f"mat_axis_fwd_kernel<{T}>", case("MatrixWavedec2", "db2", dt, (2, 33, 45), 1, ("zero", "reflect"), "packed"))
    _add(f"mat_axis_inv_kernel<{T}>", case("MatrixWaverec2", "db2", dt, (2, 33, 45), 1, ("zero",), "own"))

# ---- stationary transform -----------------------------------------------------------------------------------------
# swt_*_kernel<T, LT>: LT = L for the unrolled lengths, 0 for any other (db10: L = 20).  Odd length: rows of one
# sample, halo tiles.
for dt in ("float32", "float64"):
    T = _TNAME[dt]
    for L in FILTER_LENGTHS + (20,):
        wav = "db10" if L == 20 else wavelet(L, dt == "float64")
        lt = 0 if L == 20 else L
        _add(f"swt_fwd_kernel<{T}, {lt}>", case("swt", wav, dt, (3, 4099), 4, ("periodic",), "packed"))
        _add(f"swt_inv_kernel<{T}, {lt}>", case("iswt", wav, dt, (3, 4099), 4, ("periodic",), "own"))
    # a level whose extension is longer than the signal and not periodic: one level per launch from an index table
    _add(f"swt_level_kernel<{T}, false>", case("swt", "db4", dt, (4, 14), 3, ("periodic",), "packed"))
    _add(f"swt_level_kernel<{T}, true>", case("iswt", "db4", dt, (4, 14), 3, ("periodic",), "own"))

# ---- gradients with respect to learnable filter taps --------------------------------------------------------------
for dt in ("float32", "float64"):
    _add(f"tap_corr_kernel<{_TNAME[dt]}>", case("wavedec_tap_grad", "db3", dt, (3, 301), 2, MODES, "packed"))

# ---- continuous transform -----------------------------------------------------------------------------------------
_SCALES = (1.0, 2.5, 6.0, 17.0, 40.0)
# the filter spectra are cached per (wavelet, scales, FFT size): scales no other case uses
_add("cwt_filter_spectra_kernel", case("cwt", "morl", "float32", (3, 1500), scales=(1.25, 3.5, 9.0, 21.0, 33.0)))
_add("cwt_data_spectra_kernel<float>", case("cwt", "morl", "float32", (3, 1500), scales=_SCALES))
_add("cwt_data_spectra_kernel<double>", case("cwt", "cmor1.5-1.0", "float64", (3, 1500), scales=_SCALES))
_add("cwt_main_kernel<false>", case("cwt", "mexh", "float64", (3, 1501), scales=_SCALES))
_add("cwt_main_kernel<true>", case("cwt", "cmor1.5-1.0", "float32", (3, 1501), scales=_SCALES))
_add("cwt_adj_spectra_kernel<false>", case("cwt_grad", "morl", "float64", (3, 1500), scales=_SCALES))
_add("cwt_adj_spectra_kernel<true>", case("cwt_grad", "cmor1.5-1.0", "float32", (3, 1500), scales=_SCALES))
_add("cwt_adj_main_kernel<float>", case("cwt_grad", "morl", "float32", (3, 1501), scales=_SCALES))
_add("cwt_adj_main_kernel<double>", case("cwt_grad", "cmor1.5-1.0", "float64", (3, 1501), scales=_SCALES))
