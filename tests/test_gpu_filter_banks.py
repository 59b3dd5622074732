"""The convolution-path kernels and their gradients with filter banks that are not orthogonal.

Every db / sym / haar bank has ``rec = reversed dec`` and ``dec_hi = alternating flip of dec_lo``, so a kernel tap
table, a host routine or an autograd adjoint that takes the bank's other filter, or a filter in the wrong direction,
passes every test that uses one.  The banks of tests/filter_banks.py break both identities:

* every kernel instantiation of wavedec*, waverec* and the tap gradient (tests/kernel_cases.py) runs again with an
  unstructured bank of its length (CDF 9/7 or a second unstructured bank where the inventory uses its alternative
  wavelet), matches the float64 oracle and launches the same instantiation;
* the package reproduces what the unmodified reference computed with these banks (tests/golden/bank_vectors.*), for
  CUDA inputs and for CPU inputs staged through the device, packets and gradients included;
* odd lengths and L = 18 / 20 in every mode and dimension, or the oracle's exception;
* bior2.2 and CDF 9/7 reconstruct to the stated tolerance on the fused 2-D paths (the default two-level launch of
  images of 2^24 samples included) and the 3-D tile kernels;
* gradients with respect to the data through all six transforms, and with respect to all four filters, match the
  oracle under autograd; the profiler shows which kernels served the backward passes.

Comparisons follow tests/test_gpu_kernel_inventory.py: |delta| <= conftest.TOL[dtype] * max|oracle tree|, the oracle
run in float64 on the input rounded to the case dtype.
"""
from __future__ import annotations

import json

import numpy as np
import pytest
import torch

import filter_banks as FB
import pytorch_wavelet_toolbox_b200 as wt
from conftest import GOLDEN, TOL, assert_close_rel, flatten_coeffs
from kernel_cases import CASES, MODES
from oracle import ptwt_port as P
from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet
from test_gpu_kernel_inventory import DEV, F64, _close_tree, _map_tree, _rounded, _weighted, _weights, launched, run_case

pytestmark = pytest.mark.gpu

_TRANSFORMS = {1: (wt.wavedec, P.wavedec, wt.waverec, P.waverec, "axis"),
               2: (wt.wavedec2, P.wavedec2, wt.waverec2, P.waverec2, "axes"),
               3: (wt.wavedec3, P.wavedec3, wt.waverec3, P.waverec3, "axes")}
_DTYPES = [torch.float32, torch.float64]


def _rand(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=F64).to(dtype)


def _crop(y, shape):
    return y[(Ellipsis,) + tuple(slice(0, n) for n in shape[1:])]


# ---- every convolution-path instantiation, again with a non-orthogonal bank ------------------------------------------
_CONV_ENTRIES = ("wavedec", "waverec", "wavedec2", "waverec2", "wavedec3", "waverec3", "wavedec_tap_grad")
BANK_CASES = sorted(n for n, c in CASES.items() if c["entry"] in _CONV_ENTRIES)


def with_bank(c: dict) -> dict:
    """The inventory case with the bank of its filter length in place of its orthogonal wavelet."""
    alt = c["wavelet"].startswith("sym")
    return dict(c, wavelet=FB.bank_for_length(len(as_wavelet(c["wavelet"])), alt))


def test_bank_cases_cover_the_convolution_path():
    assert len(BANK_CASES) >= 150, len(BANK_CASES)
    assert any(isinstance(with_bank(CASES[n])["wavelet"], FB.FilterBank) and with_bank(CASES[n])["wavelet"].name
               == "cdf9/7" for n in BANK_CASES)


@pytest.mark.parametrize("name", BANK_CASES)
def test_instantiation_with_a_non_orthogonal_bank(name):
    """The kernel is chosen by L, dtype and layout, never by the taps: the same instantiation runs and matches."""
    c = with_bank(CASES[name])
    names = run_case(c)
    assert name in names, f"{name} was not launched with {c['wavelet']}; launched: {sorted(set(names))}"


# ---- the unmodified reference's numbers (tests/golden/bank_vectors.*) -------------------------------------------------
@pytest.fixture(scope="module")
def bank_vectors():
    manifest = json.loads((GOLDEN / "bank_vectors.json").read_text())
    return manifest, np.load(GOLDEN / "bank_vectors.npz")


def _fixture_bank(manifest, arrays, name):
    return FB.FilterBank(name, *arrays[manifest["banks"][name]])


def _split(flat, shapes):
    out, at = [], 0
    for s in shapes:
        n = int(np.prod(s))
        out.append(torch.from_numpy(flat[at: at + n].reshape(s)).to(F64))
        at += n
    return out


@pytest.mark.parametrize("device", ["cuda", "cpu"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_matches_the_reference_fixture(bank_vectors, ndim, device):
    manifest, arrays = bank_vectors
    dec, _, rec, _, axkw = _TRANSFORMS[ndim]
    cases = [c for c in manifest["cases"] if c["ndim"] == ndim]
    assert cases
    for case in cases:
        key, dtype = case["key"], getattr(torch, case["dtype"])
        b = _fixture_bank(manifest, arrays, case["bank"])
        axes = tuple(case["axes"]) if isinstance(case["axes"], list) else case["axes"]
        kw = {} if axes is None else {axkw: axes}
        want = _split(arrays[f"{key}_o"], case["shapes"])
        x = torch.from_numpy(arrays[f"{key}_x"]).to(device)
        what = f"{key}: {case['bank']} {case['mode']} {case['dtype']} {case['shape']} level {case['level']} {device}"
        c = dec(x, b, mode=case["mode"], level=case["level"], **kw)
        got = flatten_coeffs(c)
        assert all(t.device.type == device for t in got), what
        _close_tree(got, want[:-1], dtype, what)
        y = rec(c, b, **kw)
        assert y.device.type == device, what
        _close_tree([y], want[-1:], dtype, what + " waverec")


@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_packets_match_the_reference_fixture(bank_vectors, device):
    manifest, arrays = bank_vectors
    for case in manifest["packets"]:
        key = case["key"]
        b = _fixture_bank(manifest, arrays, case["bank"])
        x = torch.from_numpy(arrays[f"{key}_x"]).to(device)
        cls = wt.WaveletPacket if case["ndim"] == 1 else wt.WaveletPacket2D
        wp = cls(x, b, mode=case["mode"], maxlevel=case["maxlevel"])
        want = _split(arrays[f"{key}_o"], case["shapes"])
        what = f"{key}: {cls.__name__} {case['bank']} {case['mode']} {device}"
        _close_tree([wp[k] for k in case["keys"]], want[:-1], F64, what)
        _close_tree([wp.reconstruct()[""]], want[-1:], F64, what + " reconstruct")


def test_gradients_match_the_reference_fixture(bank_vectors):
    """Data and all four filters, through wavedec* and waverec*, float64."""
    manifest, arrays = bank_vectors
    for case in manifest["grads"]:
        key = case["key"]
        dec, _, rec, _, _ = _TRANSFORMS[case["ndim"]]
        taps = [t.to(DEV).requires_grad_(True) for t in torch.from_numpy(arrays[manifest["banks"][case["bank"]]])]
        bank = wt.WaveletTensorTuple(*taps)
        x = torch.from_numpy(arrays[f"{key}_x"]).to(DEV).requires_grad_(True)
        c = dec(x, bank, mode=case["mode"], level=case["level"])
        outs = flatten_coeffs(c) + [rec(c, bank)]
        ws = _split(arrays[f"{key}_w"], case["shapes"])
        sum((w.to(DEV) * t).sum() for w, t in zip(ws, outs)).backward()
        what = f"{key}: {case['bank']} {case['mode']} {case['ndim']}-D"
        assert_close_rel(x.grad, torch.from_numpy(arrays[f"{key}_gx"]), what=what + " data gradient")
        want = torch.from_numpy(arrays[f"{key}_gtaps"])
        assert_close_rel(torch.stack([t.grad for t in taps]), want, what=what + " tap gradients")


# ---- odd lengths and the lengths past the unrolled kernels -----------------------------------------------------------
_ODD_SHAPES = {1: ((3, 301), 2), 2: ((2, 45, 53), 2), 3: ((2, 9, 13, 17), 1)}


def _same_outcome(fn_ours, fn_oracle):
    """Run the oracle; where it raises, the package must raise the same exception type.  Returns the oracle's
    result, or None after checking the exception."""
    try:
        return fn_oracle()
    except Exception as ex:  # noqa: BLE001
        with pytest.raises(type(ex)):
            fn_ours()
        return None


@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("filt_len", FB.ODD_LENGTHS + FB.LONG_LENGTHS)
def test_odd_and_long_banks(filt_len, ndim):
    b = FB.unstructured(filt_len)
    dec, pdec, rec, prec, _ = _TRANSFORMS[ndim]
    shape, level = _ODD_SHAPES[ndim]
    ran = {"analysis": 0, "synthesis": 0}
    for dtype in _DTYPES:
        x = _rand(shape, dtype, filt_len)
        x64 = x.to(F64)
        for mode in MODES:
            what = f"{b} {ndim}-D {dtype} {mode}"
            want = _same_outcome(lambda: dec(x.to(DEV), b, mode=mode, level=level),
                                 lambda: pdec(x64, b, mode=mode, level=level))
            if want is None:
                continue
            got = dec(x.to(DEV), b, mode=mode, level=level)
            _close_tree(flatten_coeffs(got), flatten_coeffs(want), dtype, what)
            ran["analysis"] += 1
            want_rec = _same_outcome(lambda: rec(got, b), lambda: prec(_rounded(want, dtype), b))
            if want_rec is None:
                # the reference's crop rejects the levels of some odd lengths ("padding error"): one level it takes
                want = pdec(x64, b, mode=mode, level=1)
                got = dec(x.to(DEV), b, mode=mode, level=1)
                want_rec = prec(_rounded(want, dtype), b)
            _close_tree([rec(got, b)], [want_rec], dtype, what + " reconstruction")
            ran["synthesis"] += 1
    assert min(ran.values()) >= 4, f"{b} {ndim}-D: only {ran} mode / dtype pairs ran"


# ---- perfect reconstruction ---------------------------------------------------------------------------------------
def _assert_reconstructs(y, x, what):
    err = float((_crop(y, x.shape).to(x.device) - x).abs().max())
    scale = float(x.abs().max())
    assert err <= TOL[x.dtype] * scale, f"{what}: max abs err {err:.3e} > {TOL[x.dtype]:.0e} * {scale:.3e}"


@pytest.mark.parametrize("dtype", _DTYPES)
@pytest.mark.parametrize("bank", sorted(FB.PR_BANKS))
def test_pr_banks_reconstruct_2d(bank, dtype):
    b = FB.PR_BANKS[bank]()
    x = _rand((2, 203, 263), dtype, 11).to(DEV)
    for mode in MODES:
        c, names = launched(lambda: wt.wavedec2(x, b, mode=mode, level=3))
        if dtype == torch.float32:
            assert any(n.startswith(f"fwd2d_strip_f32_kernel<{len(b)}, 64,") for n in names), names
        y, names = launched(lambda: wt.waverec2(c, b))
        if dtype == torch.float32:
            assert any(n.startswith(f"inv2d_strip_kernel<{len(b)},") for n in names), names
        _assert_reconstructs(y, x, f"{bank} {dtype} {mode}")


@pytest.mark.parametrize("bank", sorted(FB.PR_BANKS))
def test_pr_banks_reconstruct_large_images(bank):
    """8 float32 images of 4096 x 4096 (the least input the kernel of independent warps serves by default): levels
    1-2 of bior2.2 run in one launch of it."""
    b = FB.PR_BANKS[bank]()
    x = torch.randn((8, 4096, 4096), generator=torch.Generator(device=DEV).manual_seed(12), device=DEV)
    for mode in MODES:
        c, names = launched(lambda: wt.wavedec2(x, b, mode=mode))
        if len(b) == 6 and mode != "periodic":
            assert any(n.startswith("fwd2d_wpair_kernel<6,") for n in names), (mode, sorted(set(names)))
        _assert_reconstructs(wt.waverec2(c, b), x, f"{bank} 4096^2 {mode}")


@pytest.mark.parametrize("dtype", _DTYPES)
@pytest.mark.parametrize("bank", sorted(FB.PR_BANKS))
def test_pr_banks_reconstruct_3d(bank, dtype):
    b = FB.PR_BANKS[bank]()
    x = _rand((2, 14, 35, 135), dtype, 13).to(DEV)
    tiles = dtype == torch.float32 and len(b) <= 8
    for mode in MODES:
        c, names = launched(lambda: wt.wavedec3(x, b, mode=mode, level=2))
        if tiles:
            assert any(n.startswith(f"fwd3d_tile_kernel<{len(b)},") for n in names), (mode, sorted(set(names)))
        y, names = launched(lambda: wt.waverec3(c, b))
        if tiles:
            assert any(n.startswith(f"inv3d_tile_kernel<{len(b)},") for n in names), (mode, sorted(set(names)))
        _assert_reconstructs(y, x, f"{bank} {dtype} {mode}")


@pytest.mark.parametrize("bank", sorted(FB.PR_BANKS))
def test_pr_banks_reconstruct_1d(bank):
    b = FB.PR_BANKS[bank]()
    for dtype in _DTYPES:
        x = _rand((3, 4501), dtype, 14).to(DEV)
        for mode in MODES:
            _assert_reconstructs(wt.waverec(wt.wavedec(x, b, mode=mode, level=4), b), x, f"{bank} {dtype} {mode}")


# ---- gradients with respect to the data ----------------------------------------------------------------------------
#: odd extents, level 3; 2-D: widths whose bands give both 16-byte aligned and unaligned rows over the levels (L = 2
#: halves 203 into 102, 51, 26: never a multiple of 4 floats); 3-D: float32 L <= 8 runs on the tile kernels
_GRAD_SHAPES = {1: (3, 301), 2: (2, 61, 203), 3: (1, 33, 35, 41)}
_GRAD_SHAPES_L2 = {1: (3, 301), 2: (2, 61, 199), 3: (1, 33, 35, 41)}
_GRAD_LEVEL = 3
GRAD_LENGTHS = (2, 6, 8, 16)


def _expected_backward(entry, L, dtype):
    """Instantiation prefixes the backward pass of `entry` must launch (float32 only)."""
    if dtype != torch.float32:
        return ()
    return {"wavedec2": (f"inv2d_strip_kernel<{L}, true>", f"inv2d_strip_kernel<{L}, false>"),
            "waverec2": (f"fwd2d_strip_f32_kernel<{L}, 64,",),
            "wavedec3": (f"inv3d_tile_kernel<{L},",) if L <= 8 else (),
            "waverec3": (f"fwd3d_tile_kernel<{L},",) if L <= 8 else ()}.get(entry, ())


def _analysis_grad(ndim, b, x, mode, level, seed):
    """(package gradient, oracle gradient, kernels of the backward pass) of a weighted loss of the coefficients."""
    dec, pdec, _, _, _ = _TRANSFORMS[ndim]
    x64 = x.to(F64, copy=True).requires_grad_(True)
    want = pdec(x64, b, mode=mode, level=level)
    ws = _weights(want, seed)
    _weighted(want, ws).backward()
    xg = x.to(DEV).requires_grad_(True)
    got = dec(xg, b, mode=mode, level=level)
    _close_tree([t.detach() for t in flatten_coeffs(got)], [t.detach() for t in flatten_coeffs(want)], x.dtype,
                f"{b} {mode}")
    _, names = launched(lambda: _weighted(got, ws).backward(), repeatable=False)
    return xg.grad, x64.grad, names


def _synthesis_grad(ndim, b, x, mode, level, seed):
    """The same for a weighted loss of the reconstruction from coefficients given as leaves."""
    _, pdec, rec, prec, _ = _TRANSFORMS[ndim]
    coeffs = _rounded(pdec(x.to(F64), b, mode=mode, level=level), x.dtype)
    leaves64 = _map_tree(coeffs, lambda t: t.clone().requires_grad_(True))
    leaves = _map_tree(coeffs, lambda t: t.to(x.dtype).to(DEV).requires_grad_(True))
    y64 = prec(leaves64, b)
    wy = torch.randn(y64.shape, generator=torch.Generator().manual_seed(seed), dtype=F64)
    (y64 * wy).sum().backward()
    y = rec(leaves, b)
    _close_tree([y.detach()], [y64.detach()], x.dtype, f"{b} {mode} reconstruction")
    _, names = launched(lambda: (y * wy.to(DEV, x.dtype)).sum().backward(), repeatable=False)
    got = [t.grad for t in flatten_coeffs(leaves)]
    want = [t.grad for t in flatten_coeffs(leaves64)]
    return got, want, names


@pytest.mark.parametrize("dtype", _DTYPES)
@pytest.mark.parametrize("filt_len", GRAD_LENGTHS)
@pytest.mark.parametrize("entry", ["wavedec", "waverec", "wavedec2", "waverec2", "wavedec3", "waverec3"])
def test_data_gradient(entry, filt_len, dtype):
    ndim = {"wavedec": 1, "waverec": 1}.get(entry) or int(entry[-1])
    b = FB.unstructured(filt_len)
    x = _rand((_GRAD_SHAPES_L2 if filt_len == 2 else _GRAD_SHAPES)[ndim], dtype, 100 + filt_len)
    names: list[str] = []
    for mode in MODES:
        what = f"{entry} {b} {dtype} {mode}"
        if entry.startswith("wavedec"):
            got, want, n = _analysis_grad(ndim, b, x, mode, _GRAD_LEVEL, 7)
            assert got.dtype == dtype, what
            assert_close_rel(got.double(), want, dtype=dtype, what=what + " data gradient")
        else:
            got, want, n = _synthesis_grad(ndim, b, x, mode, _GRAD_LEVEL, 8)
            _close_tree(got, want, dtype, what + " coefficient gradients")
        names += n
    for prefix in _expected_backward(entry, filt_len, dtype):
        assert any(n.startswith(prefix) for n in names), f"{entry} {b} {dtype}: no {prefix} in {sorted(set(names))}"


_SHORT_SHAPES = {1: (3, 5), 2: (2, 5, 7), 3: (1, 5, 6, 7)}


@pytest.mark.parametrize("dtype", _DTYPES)
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_data_gradient_of_short_signals(ndim, dtype):
    """Signals shorter than the extension of every level (L = 16): fold_extension adds each halo sample back onto
    the sample it copies, several times over.  Modes the oracle rejects at this length raise the same type here."""
    b = FB.unstructured(16)
    dec, pdec, _, _, _ = _TRANSFORMS[ndim]
    x = _rand(_SHORT_SHAPES[ndim], dtype, 21)
    ran = 0
    for mode in MODES:
        what = f"{b} {ndim}-D {dtype} {mode}"
        if _same_outcome(lambda: dec(x.to(DEV), b, mode=mode, level=2),
                         lambda: pdec(x.to(F64), b, mode=mode, level=2)) is None:
            continue
        got, want, _ = _analysis_grad(ndim, b, x, mode, 2, 9)
        assert_close_rel(got.double(), want, dtype=dtype, what=what + " data gradient")
        ran += 1
    assert ran >= 3, ran


# ---- gradients with respect to all four filters ---------------------------------------------------------------------
_TAP_SHAPES = {1: (3, 157), 2: (2, 37, 45), 3: (2, 11, 13, 17)}


@pytest.mark.parametrize("dtype", _DTYPES)
@pytest.mark.parametrize("filt_len", [6, 8])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_tap_gradients(ndim, filt_len, dtype):
    b = FB.unstructured(filt_len)
    dec, pdec, rec, prec, _ = _TRANSFORMS[ndim]
    x = _rand(_TAP_SHAPES[ndim], dtype, 30 + ndim)
    level = 2
    for mode in MODES:
        what = f"{b} {ndim}-D {dtype} {mode}"
        t64 = [torch.tensor(f, dtype=F64, requires_grad=True) for f in b.filter_bank]
        c64 = pdec(x.to(F64), wt.WaveletTensorTuple(*t64), mode=mode, level=level)
        y64 = prec(c64, wt.WaveletTensorTuple(*t64))
        ws = _weights(c64, 40)
        wy = torch.randn(y64.shape, generator=torch.Generator().manual_seed(41), dtype=F64)
        (_weighted(c64, ws) + (y64 * wy).sum()).backward()
        taps = [torch.tensor(f, dtype=dtype, device=DEV, requires_grad=True) for f in b.filter_bank]
        c = dec(x.to(DEV), wt.WaveletTensorTuple(*taps), mode=mode, level=level)
        y = rec(c, wt.WaveletTensorTuple(*taps))
        _close_tree([t.detach() for t in flatten_coeffs(c)], [t.detach() for t in flatten_coeffs(c64)], dtype, what)
        (_weighted(c, ws) + (y * wy.to(DEV, dtype)).sum()).backward()
        scale = max(float(t.grad.abs().max()) for t in t64)
        for tname, ta, tb in zip(("dec_lo", "dec_hi", "rec_lo", "rec_hi"), taps, t64):
            assert ta.grad is not None, f"{what}: no gradient for {tname}"
            assert_close_rel(ta.grad.double(), tb.grad, dtype=dtype, scale=scale, what=f"{what} {tname} gradient")
