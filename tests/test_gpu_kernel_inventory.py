"""Every reachable kernel instantiation of libwtb200 (tests/kernel_cases.py) runs and matches the float64 oracle.

For each case the profiler lists the kernels the entry call launched, the test asserts that the case's instantiation
is among them, and every output is compared with the oracle (oracle/ptwt_port.py, swt_port.py, cwt_port.py) run in
float64 on the same input rounded to the case's dtype: |delta| <= conftest.TOL[dtype] * max|oracle coefficient tree|.
Where the transform itself depends on the dtype (the orthogonalised boundary rows of the matrix transforms, the taps
the continuous transform picks), the oracle takes those from a run in the case's dtype and computes in float64.
Synthesis cases also compare the reconstruction.  Batches that cross the 65535 limit of a CUDA grid dimension and
inputs at the 16-byte alignment edges get their own tests, which also check with the profiler which kernel served
each call.
"""
from __future__ import annotations

import contextlib
import time

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL, assert_close_rel, flatten_coeffs
from kernel_cases import CASES, case, odd_coarsest
from oracle import cwt_port as CP
from oracle import ptwt_port as P
from oracle import swt_port as SP
from pytorch_wavelet_toolbox_b200 import _native
from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet
from test_kernel_inventory import normalise

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64


def launched(fn, repeatable=True):
    """(fn(), normalised names of the CUDA kernels it launched, in launch order).

    A profiling session only a few hundred microseconds long now and then delivers no kernel record at all, so the
    session is padded by a few milliseconds on both sides; should it still record nothing although the library
    counted launches, a call that can be repeated (not a backward pass) is profiled once more."""
    for attempt in range(2 if repeatable else 1):
        torch.cuda.synchronize()
        before = _native.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.005 * (1 + 10 * attempt))
            out = fn()
            torch.cuda.synchronize()
            time.sleep(0.005 * (1 + 10 * attempt))
        names = [normalise(e.name) for e in prof.events() if e.device_type == DeviceType.CUDA]
        if names or _native.launch_count() == before:
            break
    return out, names


def test_profiler_lists_this_librarys_kernels():
    """The profiler sees libwtb200's kernels under the names the inventory uses (bools print as true / false)."""
    x = torch.randn(2, 64, 64, device=DEV)
    _, names = launched(lambda: wt.wavedec2(x, "db2", level=1))
    assert "fwd2d_strip_f32_kernel<4, 64, true>" in names, names


# ---- inputs and coefficient containers ------------------------------------------------------------------------------
def _place(x: torch.Tensor, layout: str) -> torch.Tensor:
    """x on the device in the requested memory layout (same values)."""
    shape, W = tuple(x.shape), x.shape[-1]
    if layout in ("packed", "own", "contiguous"):
        return x.to(DEV).contiguous()
    if layout == "offset":
        buf = torch.zeros(x.numel() + 1, dtype=x.dtype, device=DEV)
        out = buf[1:].view(shape)
    elif layout in ("pitch", "pitch16"):
        # "pitch": an odd number of elements, never a multiple of 16 bytes
        pitch = W + (4 if W % 2 else 5) if layout == "pitch" else (W + 15) // 16 * 16 + 16
        out = torch.zeros(shape[:-1] + (pitch,), dtype=x.dtype, device=DEV)[..., :W]
    else:
        raise ValueError(layout)
    out.copy_(x)
    return out


def _map_tree(c, fn):
    if isinstance(c, torch.Tensor):
        return fn(c)
    if isinstance(c, dict):
        return {k: fn(v) for k, v in c.items()}
    if isinstance(c, tuple) and hasattr(c, "_fields"):
        return type(c)(*[fn(t) for t in c])
    return type(c)(_map_tree(t, fn) for t in c)


def _foreign(want64, dtype, layout):
    """The oracle's float64 coefficients as a container this package did not produce, rounded to dtype."""
    if layout == "views":
        # keep the oracle's channel-slice views: re-create every view on a device copy of its base
        bases = {}

        def view(t):
            base = t._base if t._base is not None else t
            if id(base) not in bases:
                nb = torch.empty_like(base, dtype=dtype, device=DEV)
                nb.copy_(base)
                assert nb.stride() == base.stride()
                bases[id(base)] = (base, nb)
            base, nb = bases[id(base)]
            return nb.as_strided(t.shape, t.stride(), nb.storage_offset() + t.storage_offset() - base.storage_offset())

        return _map_tree(want64, view)
    return _map_tree(want64, lambda t: _place(t.to(dtype), layout))


def _rounded(tree, dtype):
    return _map_tree(tree, lambda t: t.to(dtype).to(F64))


def _close_tree(got, want, dtype, what):
    fg, fw = flatten_coeffs(got), flatten_coeffs(want)
    assert len(fg) == len(fw), f"{what}: {len(fg)} tensors, oracle {len(fw)}"
    scale = max([float(t.abs().max()) for t in fw if t.numel()] + [1e-30])
    for j, (a, b) in enumerate(zip(fg, fw)):
        assert a.dtype == dtype, f"{what} tensor {j}: dtype {a.dtype}"
        assert_close_rel(a.double(), b.contiguous(), dtype=dtype, scale=scale, what=f"{what} tensor {j}")


def _close(got, want, dtype, what):
    """Complex-aware |got - want| <= TOL * max|want|."""
    got = got.detach().cpu()
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    err = float((got.to(want.dtype) - want).abs().max())
    scale = float(want.abs().max())
    assert err <= TOL[dtype] * scale, f"{what}: max abs err {err:.3e} > {TOL[dtype]:.0e} * {scale:.3e}"


_DEC = {"wavedec": (wt.wavedec, P.wavedec, wt.waverec, P.waverec),
        "wavedec2": (wt.wavedec2, P.wavedec2, wt.waverec2, P.waverec2),
        "wavedec3": (wt.wavedec3, P.wavedec3, wt.waverec3, P.waverec3)}
_MAT = {1: (wt.MatrixWavedec, P.MatrixWavedec, wt.MatrixWaverec, P.MatrixWaverec),
        2: (wt.MatrixWavedec2, P.MatrixWavedec2, wt.MatrixWaverec2, P.MatrixWaverec2)}


@contextlib.contextmanager
def _operators_built_in(dtype):
    """The matrix oracle builds its boundary operators in `dtype` and applies them in float64.  Which orthonormal
    basis of the boundary rows QR returns depends on the precision it runs in (float32 and float64 differ by O(1) in
    the last boundary row), and this package, like the reference, builds the operator in the data's dtype."""
    if dtype == F64:
        yield
        return
    dense, sparse = P.boundary_matrix, P.boundary_matrix_sparse
    P.boundary_matrix = lambda lo, hi, n, method="qr": dense(lo.to(dtype), hi.to(dtype), n, method).to(F64)
    P.boundary_matrix_sparse = lambda lo, hi, n, method="qr": sparse(lo.to(dtype), hi.to(dtype), n, method).to(F64)
    try:
        yield
    finally:
        P.boundary_matrix, P.boundary_matrix_sparse = dense, sparse


def _weights(tree, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(t.shape, generator=g, dtype=F64) for t in flatten_coeffs(tree)]


def _weighted(tree, ws):
    return sum((t * w.to(t.device, t.dtype)).sum() for t, w in zip(flatten_coeffs(tree), ws))


def _learnable(name, dtype, device):
    tt = wt.WaveletTensorTuple.from_wavelet(as_wavelet(name), dtype)
    return wt.WaveletTensorTuple(*[t.clone().to(device).requires_grad_(True) for t in tt])


def run_case(c: dict, seed: int = 0) -> list[str]:
    """Run one inventory case, compare everything with the oracle, return the kernels the entry call launched."""
    entry, wav, level, layout = c["entry"], c["wavelet"], c["level"], c["layout"]
    dtype = getattr(torch, c["dtype"])
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["shape"], generator=g, dtype=F64).to(dtype)
    x64 = x.to(F64)
    names: list[str] = []
    with _native.knobs(**c["knobs"]):
        if entry in ("cwt", "cwt_grad"):
            scales = np.asarray(c["scales"])
            want, _ = CP.cwt(x64, scales, wav, index_dtype=dtype)
            if entry == "cwt":
                (got, _), names = launched(lambda: wt.cwt(_place(x, layout), scales, wav))
                _close(got, want, dtype, f"cwt {wav}")
                return names
            wr = torch.randn(want.shape, generator=g, dtype=F64)

            def loss(coef):
                w = wr.to(coef.device)
                if coef.is_complex():
                    return (coef.real * w).sum() + (coef.imag * w.flip(-1)).sum()
                return (coef * w).sum()

            xg = _place(x, layout).requires_grad_(True)
            coef, _ = wt.cwt(xg, scales, wav)
            _close(coef, want, dtype, f"cwt {wav}")
            _, names = launched(lambda: loss(coef).backward(), repeatable=False)
            xw = x64.clone().requires_grad_(True)
            loss(CP.cwt(xw, scales, wav, index_dtype=dtype)[0]).backward()
            assert xg.grad.dtype == dtype
            _close(xg.grad, xw.grad, dtype, f"cwt gradient {wav}")
            return names

        for mode in c["modes"]:
            what = f"{entry} {wav} {c['dtype']} {c['shape']} level {level} {mode} {layout}"
            if entry in ("swt", "iswt"):
                want = SP.swt(x64, wav, level)
                if entry == "swt":
                    got, n = launched(lambda: wt.swt(_place(x, layout), wav, level))
                    names += n
                else:
                    got = wt.swt(x.to(DEV), wav, level)
                _close_tree(got, want, dtype, what)
                rec, n = launched(lambda: wt.iswt(got, wav))
                if entry == "iswt":
                    names += n
                _close_tree([rec], [SP.iswt(_rounded(list(want), dtype), wav)], dtype, what + " iswt")
                continue
            if entry == "wavedec_tap_grad":
                ws = _weights(P.wavedec(x64, wav, mode=mode, level=level), 7)
                wa, wb = _learnable(wav, dtype, DEV), _learnable(wav, F64, "cpu")
                got = wt.wavedec(_place(x, layout), wa, mode=mode, level=level)
                want = P.wavedec(x64, wb, mode=mode, level=level)
                _close_tree([t.detach() for t in got], [t.detach() for t in want], dtype, what)
                _, n = launched(lambda: _weighted(got, ws).backward(), repeatable=False)
                names += n
                _weighted(want, ws).backward()
                scale = max(float(t.grad.abs().max()) for t in wb[:2])
                for tname, ta, tb in zip(("dec_lo", "dec_hi"), wa[:2], wb[:2]):
                    assert ta.grad is not None, f"{what}: no gradient for {tname}"
                    assert_close_rel(ta.grad.double(), tb.grad, dtype=dtype, scale=scale, what=f"{what} {tname} grad")
                continue
            if entry.startswith("Matrix"):
                nd = 2 if entry.endswith("2") else 1
                dec, pdec, rec, prec = _MAT[nd]
                orth = c.get("orthogonalization", "qr")
                with _operators_built_in(dtype):
                    want = pdec(wav, level, orthogonalization=orth, odd_coeff_padding_mode=mode)(x64)
                    want_rec = prec(wav, orthogonalization=orth)(_rounded(want, dtype))
                if entry.startswith("MatrixWavedec"):
                    got, n = launched(lambda: dec(wav, level, orthogonalization=orth,
                                                  odd_coeff_padding_mode=mode)(_place(x, layout)))
                    names += n
                else:
                    got = dec(wav, level, orthogonalization=orth, odd_coeff_padding_mode=mode)(x.to(DEV))
                _close_tree(got, want, dtype, what)
                y, n = launched(lambda: rec(wav, orthogonalization=orth)(got))
                if entry.startswith("MatrixWaverec"):
                    names += n
                _close_tree([y], [want_rec], dtype, what + " reconstruction")
                continue
            fam = entry.replace("waverec", "wavedec")
            dec, pdec, rec, prec = _DEC[fam]
            want = pdec(x64, wav, mode=mode, level=level)
            if entry.startswith("wavedec"):
                got, n = launched(lambda: dec(_place(x, layout), wav, mode=mode, level=level))
                names += n
                _close_tree(got, want, dtype, what)
            elif layout == "own":
                got = dec(x.to(DEV), wav, mode=mode, level=level)
                _close_tree(got, want, dtype, what)
            else:
                got = _foreign(want, dtype, layout)
            y, n = launched(lambda: rec(got, wav))
            if entry.startswith("waverec"):
                names += n
            _close_tree([y], [prec(_rounded(want, dtype), wav)], dtype, what + " reconstruction")
    return names


@pytest.mark.parametrize("name", sorted(CASES))
def test_instantiation_runs_and_matches_the_oracle(name):
    names = run_case(CASES[name])
    assert name in names, f"{name} was not launched by {CASES[name]}; launched: {sorted(set(names))}"


# ---- batches that cross the 65535 limit of gridDim.y / gridDim.z ----------------------------------------------------
BIG = 65600
PICK = [0, 65534, 65535, 65536, BIG - 1]


def _big(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((BIG,) + tuple(shape), generator=g, dtype=F64).to(dtype)


def _pick_tree(tree):
    return _map_tree(tree, lambda t: t[PICK])


def _count(names, prefix):
    return sum(1 for n in names if n.startswith(prefix))


def _no(names, *prefixes):
    bad = [n for n in set(names) if n.startswith(prefixes)]
    assert not bad, f"kernels that decline batches above 65535 were launched: {bad}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_big_batch_wavedec_waverec(dtype):
    T = "float" if dtype == torch.float32 else "double"
    x = _big((64,), dtype, 1)
    c, names = launched(lambda: wt.wavedec(x.to(DEV), "db3", mode="reflect", level=2))
    assert _count(names, f"axis_fwd_kernel<{T}>") == 2, names
    _no(names, "axis1d_fast_kernel", "conv1d_fused_kernel")
    want = P.wavedec(x[PICK].to(F64), "db3", mode="reflect", level=2)
    _close_tree(_pick_tree(c), want, dtype, "wavedec")
    y, names = launched(lambda: wt.waverec(c, "db3"))
    assert _count(names, f"axis_inv_kernel<{T}>") == 2, names
    _no(names, "axis1d_inv_fast_kernel")
    _close_tree([y[PICK]], [P.waverec(_rounded(want, dtype), "db3")], dtype, "waverec")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_big_batch_wavedec2_waverec2(dtype):
    x = _big((10, 12), dtype, 2)
    c, names = launched(lambda: wt.wavedec2(x.to(DEV), "db2", mode="symmetric", level=2))
    # two launches per level: images [0, 65535) and [65535, 65600)
    prefix = "fwd2d_strip_f32_kernel<4, 64," if dtype == torch.float32 else "fwd2d_strip_kernel<double, 4, 32,"
    assert _count(names, prefix) == 4, names
    want = P.wavedec2(x[PICK].to(F64), "db2", mode="symmetric", level=2)
    _close_tree(_pick_tree(c), want, dtype, "wavedec2")
    y, names = launched(lambda: wt.waverec2(c, "db2"))
    if dtype == torch.float32:
        assert _count(names, "inv2d_strip_kernel<4,") == 4, names
    else:
        assert _count(names, "axis_inv_kernel<double>") > 0, names
    _close_tree([y[PICK]], [P.waverec2(_rounded(want, dtype), "db2")], dtype, "waverec2")


def test_big_batch_wavedec3_waverec3():
    x = _big((5, 6, 7), torch.float32, 3)
    c, names = launched(lambda: wt.wavedec3(x.to(DEV), "db2", mode="zero", level=1))
    # the tiled kernel declines more than 65535 volumes: the general per-axis kernels serve the call
    assert _count(names, "axis_fwd_kernel<float>") > 0, names
    _no(names, "fwd3d_tile_kernel")
    want = P.wavedec3(x[PICK].to(F64), "db2", mode="zero", level=1)
    _close_tree(_pick_tree(c), want, torch.float32, "wavedec3")
    y, names = launched(lambda: wt.waverec3(c, "db2"))
    assert _count(names, "axis_inv_kernel<float>") > 0, names
    _no(names, "inv3d_tile_kernel")
    _close_tree([y[PICK]], [P.waverec3(_rounded(want, torch.float32), "db2")], torch.float32, "waverec3")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_big_batch_matrix_wavedec_waverec(dtype):
    T = "float" if dtype == torch.float32 else "double"
    x = _big((64,), dtype, 4)
    c, names = launched(lambda: wt.MatrixWavedec("db2", 2)(x.to(DEV)))
    assert _count(names, f"mat_fwd_kernel<{T}>") == 2, names
    _no(names, "axis1d_fast_kernel", "mat_fwd_fused_kernel", "mat_fwd_dmma2_kernel")
    with _operators_built_in(dtype):
        want = P.MatrixWavedec("db2", 2)(x[PICK].to(F64))
        want_rec = P.MatrixWaverec("db2")(_rounded(want, dtype))
    _close_tree(_pick_tree(c), want, dtype, "MatrixWavedec")
    y, names = launched(lambda: wt.MatrixWaverec("db2")(c))
    assert _count(names, f"mat_inv_kernel<{T}>") == 2, names
    _no(names, "mat_inv_fast_kernel", "mat_inv_dmma_kernel")
    _close_tree([y[PICK]], [want_rec], dtype, "MatrixWaverec")


def test_big_batch_matrix_wavedec2_row_chunks():
    x = _big((8, 8), torch.float32, 5)
    c, names = launched(lambda: wt.MatrixWavedec2("db2", 1)(x.to(DEV)))
    # the contiguous axis has 8 * 65600 rows: launches of at most 65535 rows each
    assert _count(names, "axis1d_fast_kernel<float, 4, 3, true>") >= 8, names
    with _operators_built_in(torch.float32):
        want = P.MatrixWavedec2("db2", 1)(x[PICK].to(F64))
        want_rec = P.MatrixWaverec2("db2")(_rounded(want, torch.float32))
    _close_tree(_pick_tree(c), want, torch.float32, "MatrixWavedec2")
    y, names = launched(lambda: wt.MatrixWaverec2("db2")(c))
    assert _count(names, "mat_inv_fast_kernel<float, 4>") >= 8, names
    _close_tree([y[PICK]], [want_rec], torch.float32, "MatrixWaverec2")


def test_big_batch_swt_iswt():
    x = _big((32,), torch.float32, 6)
    c, names = launched(lambda: wt.swt(x.to(DEV), "db2", 2))
    assert _count(names, "swt_fwd_kernel<float, 4>") > 0, names
    want = SP.swt(x[PICK].to(F64), "db2", 2)
    _close_tree(_pick_tree(c), want, torch.float32, "swt")
    y, names = launched(lambda: wt.iswt(c, "db2"))
    assert _count(names, "swt_inv_kernel<float, 4>") > 0, names
    _close_tree([y[PICK]], [SP.iswt(_rounded(list(want), torch.float32), "db2")], torch.float32, "iswt")


def test_big_batch_tap_gradient():
    """The gradient with respect to learnable taps sums over all rows; tap_corr cuts them into chunks of 65535."""
    x = _big((40,), F64, 7)
    wa, wb = _learnable("db2", F64, DEV), _learnable("db2", F64, "cpu")
    got = wt.wavedec(x.to(DEV), wa, mode="reflect", level=1)
    want = P.wavedec(x, wb, mode="reflect", level=1)
    ws = _weights(want, 8)
    _, names = launched(lambda: _weighted(got, ws).backward(), repeatable=False)
    assert _count(names, "tap_corr_kernel<double>") >= 2, names
    _weighted(want, ws).backward()
    scale = max(float(t.grad.abs().max()) for t in wb[:2])
    for tname, ta, tb in zip(("dec_lo", "dec_hi"), wa[:2], wb[:2]):
        assert_close_rel(ta.grad, tb.grad, dtype=F64, scale=scale, what=f"{tname} gradient")


# ---- layouts at the 16-byte alignment edges --------------------------------------------------------------------------
def _expected(ndim, dtype, synthesis, L=6):
    f32 = dtype == "float32"
    if ndim == 1:
        return f"axis_{'inv' if synthesis else 'fwd'}_kernel<{'float' if f32 else 'double'}>"
    if ndim == 2:
        if synthesis:
            return f"inv2d_strip_kernel<{L}, false>" if f32 else "axis_inv_kernel<double>"
        return f"fwd2d_strip_f32_kernel<{L}, 64, false>" if f32 else f"fwd2d_strip_kernel<double, {L}, 32, false>"
    if synthesis:
        return f"inv3d_tile_kernel<{L}, false>" if f32 else "axis_inv_kernel<double>"
    return f"fwd3d_tile_kernel<{L}," if f32 else "axis_fwd_kernel<double>"


_SHAPES = {1: (3, 301), 2: (2, 45, 53), 3: (2, 9, 13, 17)}


@pytest.mark.parametrize("layout", ["offset", "pitch"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_misaligned_input(ndim, dtype, layout):
    """Input whose base is one element past a 16-byte boundary, or whose row pitch is wider than the row and not a
    multiple of 16 bytes: the kernels that stage through TMA or 128-bit loads step aside."""
    entry = {1: "wavedec", 2: "wavedec2", 3: "wavedec3"}[ndim]
    names = run_case(case(entry, "db3", dtype, _SHAPES[ndim], 2, ("zero", "periodic", "symmetric"), layout))
    want = _expected(ndim, dtype, False)
    if want.endswith(","):     # any tile shape of the 3-D kernel, without TMA
        assert any(n.startswith(want) and n.endswith("false>") for n in names), (want, sorted(set(names)))
    else:
        assert want in names, (want, sorted(set(names)))


@pytest.mark.parametrize("layout", ["views", "contiguous", "offset"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("ndim", [2, 3])
def test_foreign_coefficients(ndim, dtype, layout):
    """Coefficients this package did not produce -- the oracle's channel-slice views, contiguous bands of odd width,
    bands one element past a 16-byte boundary -- reach the synthesis kernels that do not use TMA."""
    shape = (2, 41, odd_coarsest(51, 6, 2)) if ndim == 2 else (2, 9, 13, odd_coarsest(15, 6, 2))
    entry = "waverec2" if ndim == 2 else "waverec3"
    names = run_case(case(entry, "db3", dtype, shape, 2, ("zero", "reflect"), layout))
    want = _expected(ndim, dtype, True)
    assert want in names, (want, sorted(set(names)))
