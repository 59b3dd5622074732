"""Inputs whose memory layout reaches the kernels without a copy.

The host code copies an input only when its innermost stride is not 1, and passes equally strided detail bands a
constant element step apart without a copy (fwt._pack_bands), so every other layout user code produces reaches the
kernels as it is: broadcast batches, rows and planes (stride 0), interleaved batches (batch stride smaller than the
row stride), overlapping frames, crops of a taller canvas, every third item, size-1 axes of any stride, detail bands
shared between arguments (band step 0) or stored in reverse order (negative band step).  For every case:

1. the outputs match the float64 oracle (oracle/ptwt_port.py, swt_port.py, cwt_port.py) run on the same values made
   contiguous: |delta| <= conftest.TOL[dtype] * max|oracle tree|;
2. the same call on a contiguous copy launches the same kernels and then returns the same bits; where the two kernel
   lists differ, the difference is the one the case pins (TMA against no TMA, a fast path against the general one);
3. only libwtb200 kernels ran: no torch copy or elementwise kernel slipped in before them (where the host code is
   meant to copy -- gradients of expanded loss gradients, the separable matrix transform -- the copy is asserted);
4. the whole storage under the input is bit-identical afterwards and no output shares it;
5. the instantiation that read the input is pinned (``_readers``), so that a change to a gate fails here instead of
   quietly testing another kernel.

On an H100 80GB HBM3 (700 W limit) ``cuTensorMapEncodeTiled`` accepts a batch or row stride of 0 and batch strides
smaller than the row stride (``ZERO_STRIDE_TMA``, ``NON_MONOTONE_TMA``), and the TMA kernels read such maps
correctly.  The float64 DMMA matrix analysis takes frames of any hop.  The layout builders are checked on the CPU by
tests/test_layouts.py.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL, assert_close_rel, flatten_coeffs
from kernel_cases import CASES as KERNEL_CASES
from kernel_cases import UNREACHABLE, coeff_len
from oracle import cwt_port as CP
from oracle import ptwt_port as P
from oracle import swt_port as SP
from pytorch_wavelet_toolbox_b200 import _native
from pytorch_wavelet_toolbox_b200.constants import DETAIL_KEYS_3D

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
_T = {F32: "float", F64: "double"}
#: elements per 16 bytes
_VEC = {F32: 4, F64: 2}
#: every kernel instantiation compiled into libwtb200 (tests/kernel_cases.py)
LIBRARY = set(KERNEL_CASES) | set(UNREACHABLE)

#: what the H100's driver does with a tensor map whose batch or row stride is 0, or whose batch stride is smaller than
#: its row stride: it encodes the map, and the TMA instantiations serve such inputs
ZERO_STRIDE_TMA = True
NON_MONOTONE_TMA = True


# ---- layout builders --------------------------------------------------------------------------------------------------
def _dense_strides(dims):
    st, acc = [], 1
    for d in reversed(dims):
        st.append(acc)
        acc *= d
    return tuple(reversed(st))


def _rand(gen, dtype, device, *shape):
    return torch.randn(shape, generator=gen, dtype=F64).to(dtype).to(device)


#: input layouts of an analysis call [B, *dims]
LAYOUTS = ("packed", "bcast", "bcast_rows", "interleaved", "frames", "canvas", "every3", "unit_last")


def build(layout: str, shape, dtype, gen, device=DEV, hop=None):
    """(view, base): a tensor of `shape` = (B, *dims) in `layout` over the storage of the contiguous tensor `base`.

    ``bcast``        ``item.expand(B, ...)``: batch stride 0
    ``bcast_rows``   the first transformed axis broadcast (rows in 2-D, planes in 3-D): its stride is 0
    ``interleaved``  ``x[dims[0], B, ...]`` with the batch moved to the front (what ``axes=(0, 2)`` does to
                     time-major data): batch stride prod(dims[1:]), smaller than the stride of dims[0]
    ``frames``       overlapping items ``hop`` elements apart (1-D: ``signal.unfold(-1, N, hop)``)
    ``canvas``       the top-left ``dims`` of a canvas 3 rows taller and 16 elements wider: batch stride is not
                     rows x pitch
    ``every3``       ``x[::3]``
    ``unit_last``    2-D ``[B, H, 1]``: column 3 of a transposed ``[B, 5, H]`` (last axis of size 1 and stride H)
    """
    B, dims = shape[0], tuple(shape[1:])
    if layout == "packed":
        base = _rand(gen, dtype, device, *shape)
        return base, base
    if layout == "bcast":
        base = _rand(gen, dtype, device, 1, *dims)
        return base.expand(shape), base
    if layout == "bcast_rows":
        base = _rand(gen, dtype, device, B, 1, *dims[1:])
        return base.expand(shape), base
    if layout == "interleaved":
        base = _rand(gen, dtype, device, dims[0], B, *dims[1:])
        return base.movedim(1, 0), base
    if layout == "frames":
        base = _rand(gen, dtype, device, (B - 1) * hop + math.prod(dims))
        if len(dims) == 1:
            return base.unfold(-1, dims[0], hop), base
        return base.as_strided(shape, (hop,) + _dense_strides(dims)), base
    if layout == "canvas":
        canvas = (dims[0] + 3,) + dims[1:-1] + (dims[-1] + 16,) if len(dims) > 1 else (dims[0] + 16,)
        base = _rand(gen, dtype, device, B, *canvas)
        return base[(slice(None),) + tuple(slice(0, d) for d in dims)], base
    if layout == "every3":
        base = _rand(gen, dtype, device, 3 * B, *dims)
        return base[::3], base
    if layout == "unit_last":
        assert dims[1:] == (1,), dims
        base = _rand(gen, dtype, device, B, 5, dims[0])
        return base.transpose(1, 2)[..., 3:4], base
    raise ValueError(layout)


#: layouts of the detail bands of one synthesis level
BAND_LAYOUTS = ("shared", "reversed", "bcast", "zeros")


def band_set(layout: str, shape, nbands: int, dtype, gen, device=DEV):
    """(bands, bases): `nbands` detail bands of `shape` in the order the synthesis kernels take them (band k = 1, 2..).

    ``shared``    one tensor for every band: band step 0
    ``reversed``  slices of one [B, nbands, ...] buffer in reverse memory order: band step -(one band)
    ``bcast``     slices of one [1, nbands, ...] buffer, each expanded over the batch: batch stride 0
    ``zeros``     one ``torch.zeros(1, ...).expand(B, ...)`` for every band: band step 0 and batch stride 0
    """
    B, dims = shape[0], tuple(shape[1:])
    if layout == "shared":
        z = _rand(gen, dtype, device, *shape)
        return [z] * nbands, [z]
    if layout == "reversed":
        buf = _rand(gen, dtype, device, B, nbands, *dims)
        return [buf[:, nbands - 1 - k] for k in range(nbands)], [buf]
    if layout == "bcast":
        buf = _rand(gen, dtype, device, 1, nbands, *dims)
        return [buf[:, k].expand(shape) for k in range(nbands)], [buf]
    if layout == "zeros":
        z = torch.zeros((1,) + dims, dtype=dtype, device=device)
        return [z.expand(shape)] * nbands, [z]
    raise ValueError(layout)


def coefficients(entry: str, layout: str, like, dtype, gen, device=DEV):
    """(container, bases): coefficients shaped like the oracle container `like`, with fresh values, their detail
    bands in `layout` (approximation too for ``bcast`` / ``zeros``: an expanded batch of one)."""
    bases = []

    def approx(t):
        if layout in ("bcast", "zeros"):
            a = _rand(gen, dtype, device, 1, *t.shape[1:])
            bases.append(a)
            return a.expand(t.shape)
        a = _rand(gen, dtype, device, *t.shape)
        bases.append(a)
        return a

    def bands(shape, n):
        bs, b = band_set(layout, tuple(shape), n, dtype, gen, device)
        bases.extend(b)
        return bs

    if entry == "iswt":
        # every level's detail has the same shape: the details of one iswt call are one band set
        return [approx(like[0])] + bands(like[1].shape, len(like) - 1), bases
    if entry in ("waverec", "MatrixWaverec"):
        # one band per level: broadcast batches only
        return [approx(like[0])] + [bands(t.shape, 1)[0] if layout != "zeros" else approx(t) for t in like[1:]], bases
    out = [approx(like[0])]
    for lv in like[1:]:
        if entry == "waverec2":
            v, h, d = bands(lv[0].shape, 3)       # band order k = 1 (vertical), 2 (horizontal), 3 (diagonal)
            out.append(type(lv)(h, v, d))
        else:
            bs = bands(lv["aad"].shape, 7)
            out.append(dict(zip(DETAIL_KEYS_3D, bs)))
    return tuple(out), bases


# ---- tree helpers -------------------------------------------------------------------------------------------------------
def _map_tree(c, fn):
    if isinstance(c, torch.Tensor):
        return fn(c)
    if isinstance(c, dict):
        return {k: fn(v) for k, v in c.items()}
    if isinstance(c, tuple) and hasattr(c, "_fields"):
        return type(c)(*[fn(t) for t in c])
    return type(c)(_map_tree(t, fn) for t in c)


def _flat(c):
    if isinstance(c, torch.Tensor):
        return [c]
    return flatten_coeffs(c)


def _oracle_input(c):
    return _map_tree(c, lambda t: t.detach().cpu().contiguous().to(F64))


def _contiguous(c):
    return _map_tree(c, lambda t: t.contiguous())


def _packed_like_own(entry, c):
    """The coefficients of a synthesis case as this package's analysis lays them out: the bands of a level slices of
    one contiguous buffer (gathered before the call, so that the call itself copies nothing)."""
    if entry == "iswt":
        return [c[0].contiguous()] + list(torch.stack(list(c[1:]), 1).unbind(1))
    if entry == "waverec2":
        return (c[0].contiguous(),) + tuple(
            type(lv)(*(lambda v, h, d: (h, v, d))(*torch.stack([lv[1], lv[0], lv[2]], 1).unbind(1))) for lv in c[1:])
    if entry == "waverec3":
        return (c[0].contiguous(),) + tuple(
            dict(zip(DETAIL_KEYS_3D, torch.stack([lv[k] for k in DETAIL_KEYS_3D], 1).unbind(1))) for lv in c[1:])
    return _contiguous(c)


def _close_tree(got, want, dtype, what, same_dtype=True):
    """|got - want| <= TOL[dtype] * max|want tree|; the outputs are in `dtype` unless not `same_dtype` (cwt returns
    float64 or complex128 for every input dtype)."""
    fg, fw = _flat(got), _flat(want)
    assert len(fg) == len(fw), f"{what}: {len(fg)} tensors, oracle {len(fw)}"
    scale = max([float(t.abs().max()) for t in fw if t.numel()] + [1e-30])
    for j, (a, b) in enumerate(zip(fg, fw)):
        assert a.dtype == dtype or not same_dtype, f"{what} tensor {j}: dtype {a.dtype}"
        if b.is_complex():
            a, b = a.detach().cpu().to(b.dtype), b.contiguous()
            assert a.shape == b.shape, f"{what} tensor {j}: shape {tuple(a.shape)} != {tuple(b.shape)}"
            err = float((a - b).abs().max())
            assert err <= TOL[dtype] * scale, f"{what} tensor {j}: max abs err {err:.3e} > {TOL[dtype]:.0e} * {scale:.3e}"
        else:
            assert_close_rel(a.double(), b.contiguous().double(), dtype=dtype, scale=scale, what=f"{what} tensor {j}")


def _bits(bases):
    return [b.detach().reshape(-1).clone() for b in bases]


def _assert_untouched(bases, snaps, outs, what):
    for j, (b, s) in enumerate(zip(bases, snaps)):
        nb, ns = b.detach().reshape(-1), s
        assert torch.equal(nb.view(torch.uint8), ns.view(torch.uint8)), f"{what}: the storage of input {j} changed"
    mine = {b.untyped_storage().data_ptr() for b in bases}
    for j, t in enumerate(_flat(outs)):
        assert t.untyped_storage().data_ptr() not in mine, f"{what}: output {j} shares storage with the input"


def _same_bits(a, b, what):
    fa, fb = _flat(a), _flat(b)
    assert len(fa) == len(fb)
    for j, (x, y) in enumerate(zip(fa, fb)):
        assert x.dtype == y.dtype and x.shape == y.shape, what
        xv = torch.view_as_real(x) if x.is_complex() else x
        yv = torch.view_as_real(y) if y.is_complex() else y
        assert torch.equal(xv, yv), f"{what}: output {j} differs from the contiguous call's in the same kernels"


def _lib_only(names, what):
    foreign = sorted({n for n in names if n not in LIBRARY})
    assert not foreign, f"{what}: kernels that are not this library's ran: {foreign}"


# ---- cases --------------------------------------------------------------------------------------------------------------
_DB = {2: "haar", 4: "db2", 6: "db3", 8: "db4", 16: "db8"}
_LEN = {w: L for L, w in _DB.items()}
_WPAIR = {2: 3, 4: 3, 6: 3, 8: 2}      # fwd2d_wpair_kernel<L, STAGES, 12> at the default variant
CASES: dict[str, dict] = {}


def _add(c):
    cid = "-".join(str(c[k]) for k in ("entry", "layout", "dtype", "wavelet")) + "-" + "x".join(map(str, c["shape"]))
    cid += f"-level{c['level']}"
    for k in ("hop", "tag"):
        if c.get(k) is not None:
            cid += f"-{k}{c[k]}"
    assert cid not in CASES, cid
    c.setdefault("knobs", {})
    CASES[cid] = c


def _case(entry, layout, dtype, wavelet, shape, level, modes, **kw):
    _add(dict(entry=entry, layout=layout, dtype=dtype, wavelet=wavelet, shape=tuple(shape), level=level,
              modes=tuple(modes), **kw))


def _coeff_widths(c):
    """Widths of the coefficients of every level of a synthesis case, finest first."""
    L, ws = _LEN[c["wavelet"]], [c["shape"][-1]]
    for _ in range(c["level"]):
        ws.append(coeff_len(ws[-1], L))
    return ws[1:]


_M3 = ("reflect", "periodic", "zero")
for dt in ("float32", "float64"):
    for L in (2, 8, 16):
        for W in (132, 131):      # rows of 16-byte multiples (TMA) or not
            for lay in LAYOUTS[1:-1]:
                _case("wavedec2", lay, dt, _DB[L], (3, 203, W), 2, _M3, hop=7 * W if lay == "frames" else None)
        _case("wavedec2", "unit_last", dt, _DB[L], (3, 203, 1), 2, ("zero",))
        for W in (132, 135):       # coefficient rows of 16-byte multiples at one level, at both or at neither
            for lay in BAND_LAYOUTS:
                _case("waverec2", lay, dt, _DB[L], (3, 203, W), 2, ("reflect",))

# the levels-1-2 kernels and the two-stream chunked branch (float32; the knobs of tests/kernel_cases.py)
for L in (4, 8):
    for lay in ("interleaved", "bcast"):
        _case("wavedec2", lay, "float32", _DB[L], (3, 132, 260), 3, ("reflect", "zero"),
              knobs={"WPAIR": 1, "WPAIR_MIN": 1}, tag="wpair")
        _case("wavedec2", lay, "float32", _DB[L], (2, 203, 264), 3, ("symmetric", "zero"),
              knobs={"WPAIR": 0, "FUSE2": 1}, tag="fuse2")
_case("wavedec2", "interleaved", "float32", "db4", (3, 203, 132), 2, ("reflect",), knobs={"CHUNK": 1}, tag="chunk")

# 3-D: 136 columns give TMA rows, 135 do not
for W in (136, 135):
    for lay in ("interleaved", "bcast", "bcast_rows"):
        _case("wavedec3", lay, "float32", "db2", (2, 9, 35, W), 2, _M3)
for lay in ("interleaved", "bcast", "bcast_rows"):
    _case("wavedec3", lay, "float64", "db2", (2, 9, 11, 13), 2, _M3)
for dt in ("float32", "float64"):
    for W in (42, 41):
        for lay in BAND_LAYOUTS:
            _case("waverec3", lay, dt, "db2", (2, 9, 13, W), 2, ("zero",))

# 1-D: frames hop = 0 (mod 4) and not, broadcast and sliced batches; one level (axis1d_fast_kernel / axis_fwd_kernel)
# and three (conv1d_fused_kernel for the levels that read 16-byte rows)
for dt in ("float32", "float64"):
    for level in (1, 3):
        for lay, hop in (("frames", 200), ("frames", 202), ("frames", 133), ("bcast", None), ("every3", None)):
            _case("wavedec", lay, dt, "db4", (4, 517), level, _M3, hop=hop)
        for lay in ("canvas", "every3"):       # 516 samples: rows 16-byte aligned
            _case("wavedec", lay, dt, "db4", (4, 516), level, _M3)
    _case("waverec", "bcast", dt, "db4", (4, 517), 3, ("zero",))

# matrix transforms: float32 frames of even hop reach the fused analysis, of odd hop the general one; the float64 DMMA
# analysis takes frames of any hop
for dt in ("float32", "float64"):
    orth = "gramschmidt" if dt == "float32" else "qr"
    for lay, hop in (("frames", 200), ("frames", 131), ("bcast", None)):
        _case("MatrixWavedec", lay, dt, "db3", (4, 1024), 3, ("zero",), hop=hop, orthogonalization=orth)
    _case("MatrixWaverec", "bcast", dt, "db3", (4, 1024), 3, ("zero",), orthogonalization=orth)
_case("MatrixWavedec2", "bcast", "float32", "db2", (3, 40, 36), 1, ("zero",), copy=True)

# stationary and continuous transforms
for dt in ("float32", "float64"):
    for lay, hop in (("frames", 200), ("frames", 131), ("bcast", None)):
        _case("swt", lay, dt, "db2", (4, 515), 3, ("periodic",), hop=hop)
    for lay in ("shared", "reversed", "bcast"):
        _case("iswt", lay, dt, "db2", (4, 515), 3, ("periodic",))
for wav, dt in (("morl", "float32"), ("cmor1.5-1.0", "float64")):
    for lay, hop in (("frames", 500), ("frames", 333), ("bcast", None)):
        _case("cwt", lay, dt, wav, (3, 1500), 0, ("-",), hop=hop)

_SCALES = np.asarray((1.0, 2.5, 6.0, 17.0))


def _tma(c, layout, W=None) -> bool:
    """Whether the input of `c` in `layout` (rows of W elements) passes the 16-byte gates of the TMA kernels and the
    driver maps it."""
    dtype = getattr(torch, c["dtype"])
    W = c["shape"][-1] if W is None else W
    if layout in BAND_LAYOUTS:
        # bands of one level: contiguous tensors or slices of one buffer, rows of W elements
        if W % _VEC[dtype]:
            return False
        return ZERO_STRIDE_TMA if layout in ("bcast", "zeros") else True
    if layout == "unit_last" or W % _VEC[dtype]:
        return False
    if layout in ("bcast", "bcast_rows"):
        return ZERO_STRIDE_TMA
    if layout == "interleaved":
        return NON_MONOTONE_TMA
    return True


def _readers(c, layout, mode) -> list[str]:
    """The instantiations the call on `c`'s input in `layout` must launch (the ones that read the caller's tensors)."""
    e, dtype, L = c["entry"], getattr(torch, c["dtype"]), _LEN.get(c["wavelet"], 0)
    T, tma = _T[dtype], str(_tma(c, layout)).lower()
    hop = c.get("hop") if layout == "frames" else None
    xs = {"bcast": 0, "every3": 3 * c["shape"][-1], "canvas": c["shape"][-1] + 16}.get(
        layout, hop if hop is not None else c["shape"][-1])
    if e == "wavedec2":
        tag = c.get("tag")
        if tag == "wpair" and tma == "true":
            return [f"fwd2d_wpair_kernel<{L}, {_WPAIR[L]}, 12>"]
        if tag == "fuse2" and tma == "true":
            return [f"fwd2d_fuse2_f32_kernel<{L}>"]
        return [f"fwd2d_strip_f32_kernel<{L}, 64, {tma}>" if dtype == F32 else f"fwd2d_strip_kernel<double, {L}, 32, {tma}>"]
    if e in ("waverec2", "waverec3") and dtype == F32:
        # one launch per level: TMA where all four (eight) inputs of the level have 16-byte rows
        k = "inv2d_strip_kernel" if e == "waverec2" else "inv3d_tile_kernel"
        return sorted({f"{k}<{L}, {str(_tma(c, layout, w)).lower()}>" for w in _coeff_widths(c)})
    if e == "waverec2":
        return ["axis_inv_kernel<double>"]
    if e == "wavedec3":
        return [f"fwd3d_tile_kernel<{L}, *, {tma}>" if dtype == F32 else "axis_fwd_kernel<double>"]
    if e == "waverec3":
        return ["axis_inv_kernel<double>"]
    if e == "wavedec":
        if c["level"] > 1 and mode != "periodic" and xs % 4 == 0:
            return [f"conv1d_fused_kernel<{T}, {L}>"]
        if xs % _VEC[dtype] == 0:
            return [f"axis1d_fast_kernel<{T}, {L}, {(2 - L) % _VEC[dtype]}, false>"]
        return [f"axis_fwd_kernel<{T}>"]
    if e == "waverec":
        return [f"axis1d_inv_fast_kernel<{T}, {L}>"]
    if e == "MatrixWavedec":
        if dtype == F64:     # the DMMA analysis loads rows of any stride
            return [f"mat_fwd_dmma2_kernel<{L}, *>"]
        return [f"mat_fwd_kernel<float>"] if xs % 2 else [f"mat_fwd_fused_kernel<float, {L}, *>"]
    if e == "MatrixWaverec":
        return [f"mat_inv_fast_kernel<float, {L}>" if dtype == F32 else f"mat_inv_dmma_kernel<{L}, *>"]
    if e == "MatrixWavedec2":
        # rows of 36 samples: the general kernel along the rows, the register-blocked one along the columns
        return ["mat_axis_fwd_kernel<float>", f"mat_axis_fwd_blk_kernel<float, {L}>"]
    if e == "swt":
        return [f"swt_fwd_kernel<{T}, {L}>"]
    if e == "iswt":
        return [f"swt_inv_kernel<{T}, {L}>"]
    if e == "cwt":
        return [f"cwt_data_spectra_kernel<{T}>", f"cwt_main_kernel<{str(c['wavelet'].startswith('cmor')).lower()}>"]
    raise ValueError(e)


def _launched_pattern(pattern: str, names) -> bool:
    """`pattern` with ``*`` standing for the remaining template arguments (tile shapes, thread counts)."""
    if "*" not in pattern:
        return pattern in names
    head, tail = pattern.split("*")
    return any(n.startswith(head) and n.endswith(tail) for n in names)


# ---- running a case -------------------------------------------------------------------------------------------------------
def _call(c, mode):
    """(function of the input, oracle of the float64 input) of case `c` in `mode`."""
    e, wav, level = c["entry"], c["wavelet"], c["level"]
    dtype = getattr(torch, c["dtype"])
    if e in ("wavedec", "wavedec2", "wavedec3"):
        dec, pdec = getattr(wt, e), getattr(P, e)
        return lambda x: dec(x, wav, mode=mode, level=level), lambda x: pdec(x, wav, mode=mode, level=level)
    if e in ("waverec", "waverec2", "waverec3"):
        return lambda c_: getattr(wt, e)(c_, wav), lambda c_: getattr(P, e)(c_, wav)
    if e.startswith("Matrix"):
        orth = c.get("orthogonalization", "qr")
        kw = dict(orthogonalization=orth, odd_coeff_padding_mode=mode) if "dec" in e else dict(orthogonalization=orth)
        args = (wav, level) if "dec" in e else (wav,)
        obj = getattr(wt, e)(*args, **kw)        # one object: its operators are built once, by the first call

        def oracle(x):
            from test_gpu_kernel_inventory import _operators_built_in

            with _operators_built_in(dtype):
                return getattr(P, e)(*args, **kw)(x)

        return obj, oracle
    if e == "swt":
        return lambda x: wt.swt(x, wav, level), lambda x: SP.swt(x, wav, level)
    if e == "iswt":
        return lambda c_: wt.iswt(c_, wav), lambda c_: SP.iswt(list(c_), wav)
    if e == "cwt":
        return lambda x: wt.cwt(x, _SCALES, wav)[0], lambda x: CP.cwt(x, _SCALES, wav, index_dtype=dtype)[0]
    raise ValueError(e)


def _synthesis_like(c, gen):
    """The oracle's analysis of a random input of the case's shape: the container a synthesis case fills."""
    e = c["entry"]
    x64 = torch.randn(c["shape"], generator=gen, dtype=F64)
    if e == "iswt":
        return SP.swt(x64, c["wavelet"], c["level"])
    if e == "MatrixWaverec":
        return P.MatrixWavedec(c["wavelet"], c["level"])(x64)
    return getattr(P, e.replace("rec", "dec"))(x64, c["wavelet"], mode="zero", level=c["level"])


def run_case(c, seed=0, pin=True):
    """Run every mode of case `c` with checks 1-4 (and 5 when `pin`); returns {mode: (names strided, names contiguous)}."""
    dtype = getattr(torch, c["dtype"])
    g = torch.Generator().manual_seed(seed)
    from test_gpu_kernel_inventory import launched

    seen = {}
    with _native.knobs(**c["knobs"]):
        for mode in c["modes"]:
            what = f"{c['entry']} {c['layout']} {c['dtype']} {c['wavelet']} {c['shape']} {mode}"
            fn, oracle = _call(c, mode)
            if c["entry"] in ("waverec", "waverec2", "waverec3", "MatrixWaverec", "iswt"):
                arg, bases = coefficients(c["entry"], c["layout"], _synthesis_like(c, g), dtype, g)
            else:
                arg, base = build(c["layout"], c["shape"], dtype, g, hop=c.get("hop"))
                bases = [base]
            contig = _packed_like_own(c["entry"], arg) if c["layout"] in BAND_LAYOUTS else _contiguous(arg)
            snaps = _bits(bases)
            # the contiguous call first: it builds what later calls reuse (operators, filter spectra), so that the
            # profile of the strided call holds its own launches only
            ref, ref_names = launched(lambda: fn(contig))
            got, names = launched(lambda: fn(arg))
            torch.cuda.synchronize()
            _assert_untouched(bases, snaps, got, what)
            assert names, f"{what}: no kernel launch recorded"
            if c.get("copy"):
                assert any(n not in LIBRARY for n in names), f"{what}: the host copy did not run: {names}"
            else:
                _lib_only(names, what)
            _close_tree(got, oracle(_oracle_input(arg)), dtype, what, same_dtype=c["entry"] != "cwt")
            readers = _readers(c, c["layout"], mode)
            # the same instantiations (a layout may change how often one runs: the general 3-D path loops over
            # planes that cannot be folded into rows) must compute the same bits; different ones only where the
            # instantiation that reads the input differs
            lib, ref_lib = {n for n in names if n in LIBRARY}, {n for n in ref_names if n in LIBRARY}
            if lib == ref_lib:
                _same_bits(got, ref, what)
            elif c["layout"] not in BAND_LAYOUTS:
                assert readers != _readers(c, "packed", mode), f"{what}: kernels {names} != contiguous call's {ref_names}"
            if pin:
                for r in readers:
                    assert _launched_pattern(r, names), f"{what}: {r} was not launched; launched {sorted(set(names))}"
                    if r.endswith("true>") and "*" not in r and r[:-5] + "false>" not in readers:
                        assert r[:-5] + "false>" not in names, f"{what}: the non-TMA twin of {r} ran too"
            seen[mode] = (names, ref_names)
    return seen


@pytest.mark.parametrize("cid", sorted(CASES))
def test_layout_reaches_the_kernel_and_matches_the_oracle(cid):
    c = CASES[cid]
    seen = run_case(c)
    if c.get("tag") == "chunk":
        # three chunks of one image, two levels each, alternating between two streams
        for names, _ in seen.values():
            assert sum(n.startswith("fwd2d_strip_f32_kernel<8, 64,") for n in names) == 6, names


# ---- gradients ---------------------------------------------------------------------------------------------------------------
def _grad_names_ok(names, what):
    assert names, f"{what}: no kernel launch recorded"
    assert any(n in LIBRARY for n in names), f"{what}: no library kernel in the backward pass: {names}"


@pytest.mark.parametrize("mode", ["reflect", "zero"])
@pytest.mark.parametrize("dtype", [F32, F64])
def test_sum_loss_gradient(dtype, mode):
    """``wavedec2(x).sum()``: every band's gradient is one expanded scalar (stride 0 in every axis).  The backward
    pass makes it contiguous (a torch copy) before the synthesis kernels run."""
    from test_gpu_kernel_inventory import launched

    g = torch.Generator().manual_seed(3)
    x = torch.randn((3, 45, 53), generator=g, dtype=F64).to(dtype)
    xg = x.to(DEV).requires_grad_(True)
    coeffs = wt.wavedec2(xg, "db4", mode=mode, level=2)
    loss = sum(t.sum() for t in _flat(coeffs))
    _, names = launched(lambda: loss.backward(), repeatable=False)
    _grad_names_ok(names, "sum loss")
    assert any(n not in LIBRARY for n in names), f"the expanded gradient was not copied: {names}"
    xw = x.to(F64).requires_grad_(True)
    sum(t.sum() for t in _flat(P.wavedec2(xw, "db4", mode=mode, level=2))).backward()
    assert_close_rel(xg.grad.double(), xw.grad, dtype=dtype, scale=float(xw.grad.abs().max()), what="sum-loss gradient")


@pytest.mark.parametrize("mode", ["reflect", "periodic", "zero"])
@pytest.mark.parametrize("dtype", [F32, F64])
def test_gradient_of_interleaved_and_framed_leaves(dtype, mode):
    """Gradients with respect to a time-major leaf ``[H, B, W]`` transformed with ``axes=(0, 2)``, and to a signal
    cut into overlapping frames (the frames' gradients add up where they overlap)."""
    g = torch.Generator().manual_seed(4)
    leaf64 = torch.randn((45, 3, 53), generator=g, dtype=F64)
    leaf = leaf64.to(dtype).to(DEV).requires_grad_(True)
    got = wt.wavedec2(leaf, "db3", mode=mode, level=2, axes=(0, 2))
    ref = leaf64.to(dtype).to(F64).requires_grad_(True)
    want = P.wavedec2(ref.movedim(1, 0), "db3", mode=mode, level=2)
    _close_tree([t.movedim(1, 0) for t in _flat(got)], _flat(want), dtype, "interleaved wavedec2")
    ws = [torch.randn(t.shape, generator=g, dtype=F64) for t in _flat(want)]
    sum((t.movedim(1, 0) * w.to(DEV, dtype)).sum() for t, w in zip(_flat(got), ws)).backward()
    sum((t * w).sum() for t, w in zip(_flat(want), ws)).backward()
    assert_close_rel(leaf.grad.double(), ref.grad, dtype=dtype, scale=float(ref.grad.abs().max()),
                     what="interleaved leaf gradient")

    sig64 = torch.randn((3 * 131 + 400,), generator=g, dtype=F64)
    sig = sig64.to(dtype).to(DEV).requires_grad_(True)
    got = wt.wavedec(sig.unfold(-1, 400, 131), "db4", mode=mode, level=3)
    sref = sig64.to(dtype).to(F64).requires_grad_(True)
    want = P.wavedec(sref.unfold(-1, 400, 131), "db4", mode=mode, level=3)
    _close_tree(got, want, dtype, "framed wavedec")
    ws = [torch.randn(t.shape, generator=g, dtype=F64) for t in want]
    sum((t * w.to(DEV, dtype)).sum() for t, w in zip(got, ws)).backward()
    sum((t * w).sum() for t, w in zip(want, ws)).backward()
    assert_close_rel(sig.grad.double(), sref.grad, dtype=dtype, scale=float(sref.grad.abs().max()),
                     what="framed leaf gradient")
