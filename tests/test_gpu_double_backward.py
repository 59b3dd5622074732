"""Gradients of gradients: gradient penalties and Hessian-vector products through the transforms.

Under ``create_graph=True`` every backward pass of the package runs as a chain of its own autograd Functions (each
kernel's adjoint is another kernel of the library), so the results of a backward pass carry a graph and can be
differentiated again, as the reference's chain of torch operators can.  This file checks:

* ``gradgradcheck`` in float64 at small odd and even extents, two levels: wavedec / waverec in 1, 2 and 3 dimensions in
  every mode, with haar, db2 and a bank that is not orthogonal, with respect to the data and with respect to the data
  and all four filters; swt / iswt; cwt with a real and a complex wavelet;
* an R1 penalty ``D + gamma * |dD/dx|^2`` (``D`` a weighted sum of the coefficients) at sizes users train at: the
  gradients of the weights (and of the filters, where they are learnable) match the float64 oracle ports
  (oracle/ptwt_port.py, swt_port.py, cwt_port.py), which are torch operators and can be differentiated twice;
* a Hessian-vector product of a reconstruction loss with respect to learnable filters matches the oracle's;
* first-order gradients taken with ``create_graph=False`` (taps as floats, no graph) and ``create_graph=True`` (taps as
  tensors, recorded) agree: one backward path serves both;
* the profiler shows what the second-order pass runs: the library's analysis, synthesis, tap-correlation, swt and cwt
  kernels, and otherwise only PyTorch's elementwise, copy, fill, pad and index kernels; never cuDNN, cuFFT, cuBLAS or
  CUTLASS.

Comparisons: |delta| <= conftest.TOL[dtype] * max|oracle tree|, the oracle run in float64 on the input rounded to the
case's dtype.
"""
from __future__ import annotations

import itertools
import re
import time

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType, gradgradcheck
from torch.profiler import ProfilerActivity, profile

import filter_banks as FB
import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL, flatten_coeffs
from kernel_cases import CASES, MODES, UNREACHABLE
from oracle import cwt_port as CP
from oracle import ptwt_port as P
from oracle import swt_port as SP
from test_gpu_kernel_inventory import DEV, F64
from test_kernel_inventory import normalise

pytestmark = pytest.mark.gpu

_TRANSFORMS = {1: (wt.wavedec, wt.waverec, P.wavedec, P.waverec),
               2: (wt.wavedec2, wt.waverec2, P.wavedec2, P.waverec2),
               3: (wt.wavedec3, wt.waverec3, P.wavedec3, P.waverec3)}


def _rand(shape, dtype=F64, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=F64).to(dtype).to(device)


def _bank(name):
    return FB.unstructured(6) if name == "unstructured6" else name


def _taps(wavelet, device, dtype=F64):
    """The wavelet's four filters as leaves that require grad."""
    from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet

    return [torch.tensor(list(f), dtype=dtype, device=device, requires_grad=True)
            for f in as_wavelet(wavelet).filter_bank]


# ---- gradgradcheck --------------------------------------------------------------------------------------------------
#: odd and even extents; every mode can pad both levels of a six-tap filter
_SMALL = {1: (2, 13), 2: (1, 9, 8), 3: (1, 8, 9, 7)}


@pytest.mark.parametrize("wrt", ["data", "data+filters"])
@pytest.mark.parametrize("wavelet", ["haar", "db2", "unstructured6"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_gradgradcheck_wavedec_waverec(ndim, wavelet, wrt):
    dec, rec, _, _ = _TRANSFORMS[ndim]
    x = _rand(_SMALL[ndim], seed=ndim, device=DEV).requires_grad_(True)
    for mode in MODES:
        if wrt == "data":
            def fn(x):
                c = dec(x, _bank(wavelet), mode=mode, level=2)
                return tuple(flatten_coeffs(c)) + (rec(c, _bank(wavelet)),)

            inputs = (x,)
        else:
            def fn(x, *taps):
                w = wt.WaveletTensorTuple(*taps)
                c = dec(x, w, mode=mode, level=2)
                return tuple(flatten_coeffs(c)) + (rec(c, w),)

            inputs = (x,) + tuple(_taps(_bank(wavelet), DEV))
        # the tap correlation sums in float64 with one atomicAdd per warp and tap: repeated backward passes agree to
        # round-off, not bit for bit
        nondet_tol = 0.0 if wrt == "data" else 1e-12
        assert gradgradcheck(fn, inputs, fast_mode=True, nondet_tol=nondet_tol), f"{ndim}-D {wavelet} {mode} {wrt}"


def test_gradgradcheck_swt_iswt():
    x = _rand((3, 24), seed=5, device=DEV).requires_grad_(True)

    def fn(x):
        c = wt.swt(x, "db2", 3)
        return tuple(c) + (wt.iswt(c, "db2"),)

    assert gradgradcheck(fn, (x,), fast_mode=True)


@pytest.mark.parametrize("wavelet", ["morl", "cmor1.5-1.0"])
def test_gradgradcheck_cwt(wavelet):
    x = _rand((2, 45), seed=6, device=DEV).requires_grad_(True)
    scales = np.arange(1, 7)
    assert gradgradcheck(lambda x: wt.cwt(x, scales, wavelet)[0], (x,), fast_mode=True)


# ---- the same first-order gradients with and without a graph ---------------------------------------------------------
#: odd and even extents, two levels of db3 in every mode
_AGREE = {1: (3, 67), 2: (2, 33, 40), 3: (1, 17, 20, 15)}


@pytest.mark.parametrize("dtype", [torch.float32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("learnable", [False, True], ids=["data", "learnable"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_gradients_agree_with_and_without_create_graph(ndim, learnable, dtype):
    """A backward pass without grad mode runs on the filters as floats, one in grad mode on the filters as tensors;
    both give the same gradients: the data gradient bit for bit, the filter gradients to the round-off of the tap
    correlation's float64 atomics."""
    dec, rec, _, _ = _TRANSFORMS[ndim]
    x0 = _rand(_AGREE[ndim], dtype, seed=30 + ndim, device=DEV)
    tol = 1e-12 if dtype == F64 else TOL[dtype]
    for mode in MODES:
        results = []
        for create_graph in (False, True):
            x = x0.clone().requires_grad_(True)
            taps = _taps("db3", DEV, dtype) if learnable else []
            w = wt.WaveletTensorTuple(*taps) if learnable else "db3"
            c = dec(x, w, mode=mode, level=2)
            outs = flatten_coeffs(c) + [rec(c, w)]
            # weights that require grad: under create_graph=True every gradient then carries a graph
            weights = [_rand(t.shape, dtype, seed=40 + j, device=DEV).requires_grad_(True) for j, t in enumerate(outs)]
            loss = sum((t * u).sum() for t, u in zip(outs, weights))
            grads = torch.autograd.grad(loss, [x] + taps, create_graph=create_graph)
            assert all(g.requires_grad == create_graph for g in grads), f"{mode}: create_graph={create_graph}"
            results.append([g.detach() for g in grads])
        (gx1, *gt1), (gx2, *gt2) = results
        assert torch.equal(gx1, gx2), f"{ndim}-D {mode}: data gradients differ"
        for k, (a, b) in enumerate(zip(gt1, gt2)):
            err, scale = float((a - b).abs().max()), float(a.abs().max())
            assert err <= tol * scale, f"{ndim}-D {mode}: filter {k} gradients differ by {err:.3e} > {tol:.0e} * {scale:.3e}"


# ---- R1 penalty at user sizes ----------------------------------------------------------------------------------------
_ANALYSIS = {n for n, c in CASES.items() if c["entry"] in ("wavedec", "wavedec2", "wavedec3")} | set(UNREACHABLE)
_SYNTHESIS = {n for n, c in CASES.items() if c["entry"] in ("waverec", "waverec2", "waverec3")}
_TAP_CORR = {n for n, c in CASES.items() if c["entry"] == "wavedec_tap_grad"}
_SWT = {n for n, c in CASES.items() if c["entry"] in ("swt", "iswt")}
_CWT = {n for n, c in CASES.items() if c["entry"] in ("cwt", "cwt_grad")}
_LIBRARY = set(CASES) | set(UNREACHABLE)
#: PyTorch's glue: elementwise arithmetic and casts, copies (cat, memcpy), fills, pads, index_add / index_select / flip
_TORCH_GLUE = re.compile(r"elementwise|fill|copy|memcpy|memset|pad|index|flip", re.IGNORECASE)
_VENDOR = re.compile(r"cudnn|cufft|fft|gemm|gemv|cublas|cutlass|xmma|im2col|col2im", re.IGNORECASE)


def kernels_of(fn):
    """(fn(), full names of the CUDA kernels and copies it ran).  Full names: the inventory's normalised form cuts
    PyTorch's ``at::native::(anonymous namespace)::...`` kernels down to ``at::native::``."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        out = fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    return out, [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]


def check_second_order_kernels(names, required: dict, what: str) -> None:
    """Every kernel is the library's or PyTorch glue, and each family in `required` ran at least once."""
    assert names, f"{what}: the profiler recorded no kernel"
    ours = {normalise(n) for n in names} & _LIBRARY
    foreign = sorted({n for n in names if normalise(n) not in _LIBRARY})
    assert not [n for n in foreign if _VENDOR.search(n)], f"{what}: vendor kernels ran: {foreign}"
    assert all(_TORCH_GLUE.search(n) for n in foreign), \
        f"{what}: kernels outside the library and glue: {[n for n in foreign if not _TORCH_GLUE.search(n)]}"
    for family, members in required.items():
        assert ours & members, f"{what}: no {family} kernel in {sorted(ours)}"


def _real_view(t):
    return torch.view_as_real(t) if t.is_complex() else t


def _r1_step(transform, x, weights, gamma, profiled):
    """loss = D + gamma * |dD/dx|^2 with D = sum_j <W_j, c_j>; backward; returns the kernels of that backward."""
    coeffs = transform(x)
    d = sum((_real_view(c) * w).sum() for c, w in zip(coeffs, weights))
    gx, = torch.autograd.grad(d, x, create_graph=True)
    assert gx.requires_grad, "the gradient carries no graph"
    loss = d.sum() + gamma * (gx ** 2).sum()
    if profiled:
        return kernels_of(loss.backward)[1]
    loss.backward()
    return []


def _compare(got, want, dtype, what):
    scale = max(float(t.abs().max()) for t in want)
    for j, (a, b) in enumerate(zip(got, want)):
        assert a is not None, f"{what} {j}: no gradient"
        err = float((a.detach().cpu().double() - b).abs().max())
        assert err <= TOL[dtype] * scale, f"{what} {j}: max abs err {err:.3e} > {TOL[dtype]:.0e} * {scale:.3e}"


def _packet_leaves(data, wavelet, mode, transform):
    """The 16 nodes of a two-level 2-D packet tree built from one-level wavedec2 calls (how the reference expands a
    WaveletPacket2D node: children a, h, v, d)."""
    nodes = {"": data}
    for path in ("",) + tuple("ahvd"):
        a, (h, v, d) = transform(nodes[path], wavelet, mode=mode, level=1)
        nodes.update({path + "a": a, path + "h": h, path + "v": v, path + "d": d})
    return [nodes[p + q] for p, q in itertools.product("ahvd", repeat=2)]


def _pair(kind, wavelet, mode, level, dtype, scales=None):
    """(package transform, oracle transform) as functions of (x, taps) returning a flat coefficient list."""
    if kind in ("wavedec", "wavedec2", "wavedec3"):
        ndim = {"wavedec": 1}.get(kind) or int(kind[-1])
        dec, _, pdec, _ = _TRANSFORMS[ndim]
        return (lambda x, w: flatten_coeffs(dec(x, w, mode=mode, level=level)),
                lambda x, w: flatten_coeffs(pdec(x, w, mode=mode, level=level)))
    if kind == "fswavedec2":
        # fswavedec2's pyramid is wavedec2's; its dict keys map da/ad/dd to horizontal/vertical/diagonal
        def pkg(x, w):
            c = wt.fswavedec2(x, w, mode=mode, level=level)
            return [c[0]] + [t for lv in c[1:] for t in (lv["da"], lv["ad"], lv["dd"])]

        return pkg, lambda x, w: flatten_coeffs(P.wavedec2(x, w, mode=mode, level=level))
    if kind == "packets2d":
        def pkg(x, w):
            wp = wt.WaveletPacket2D(x, w, mode=mode, maxlevel=2)
            return [wp["".join(k)] for k in itertools.product("ahvd", repeat=2)]

        return pkg, lambda x, w: _packet_leaves(x, w, mode, P.wavedec2)
    if kind == "swt":
        return (lambda x, w: list(wt.swt(x, w, level)), lambda x, w: list(SP.swt(x, w, level)))
    if kind == "cwt":
        return (lambda x, w: [wt.cwt(x, scales, wavelet)[0]],
                lambda x, w: [CP.cwt(x, scales, wavelet, index_dtype=dtype)[0]])
    raise ValueError(kind)


_R1_CASES = {
    # name: (kind, shape, dtype, wavelet, mode, level, learnable filters, device of the leaf)
    "wavedec2-db4-reflect-f32": ("wavedec2", (8, 256, 256), torch.float32, "db4", "reflect", 3, False, DEV),
    "wavedec3-sym4-zero-learnable": ("wavedec3", (2, 48, 48, 48), F64, "sym4", "zero", 2, True, DEV),
    "wavedec-db6-symmetric-cpu-learnable": ("wavedec", (16, 8192), F64, "db6", "symmetric", 4, True, "cpu"),
    "fswavedec2-bank-periodic-learnable": ("fswavedec2", (4, 96, 130), F64, "unstructured6", "periodic", 2, True, DEV),
    "waveletpacket2d-db3-reflect": ("packets2d", (4, 64, 72), F64, "db3", "reflect", 2, False, DEV),
    "swt-db4-f32": ("swt", (4, 4096), torch.float32, "db4", None, 4, False, DEV),
    "cwt-morl": ("cwt", (4, 3000), F64, "morl", None, None, False, DEV),
    "cwt-cmor-f32": ("cwt", (4, 3000), torch.float32, "cmor1.5-1.0", None, None, False, DEV),
}


def _required(kind, learnable):
    if kind == "swt":
        return {"swt": _SWT}
    if kind == "cwt":
        return {"cwt": _CWT}
    req = {"analysis": _ANALYSIS, "synthesis": _SYNTHESIS}
    if learnable:
        req["tap_corr"] = _TAP_CORR
    return req


@pytest.mark.parametrize("name", sorted(_R1_CASES))
def test_r1_penalty_matches_the_oracle(name):
    kind, shape, dtype, wavelet, mode, level, learnable, device = _R1_CASES[name]
    scales = np.arange(1, 41) if wavelet == "morl" else np.geomspace(1, 64, 24)
    pkg, ora = _pair(kind, _bank(wavelet), mode, level, dtype, scales)
    gamma = 0.5
    x0 = _rand(shape, dtype, seed=11)
    out_dtype = F64 if kind == "cwt" else dtype    # cwt returns float64 / complex128 for every input dtype

    # the oracle in float64 on the same input and weights
    taps64 = _taps(_bank(wavelet), "cpu") if learnable else None
    w64 = wt.WaveletTensorTuple(*taps64) if learnable else _bank(wavelet)
    x64 = x0.to(F64).requires_grad_(True)
    c64 = ora(x64, w64)
    g = torch.Generator().manual_seed(12)
    ws64 = [torch.randn(_real_view(c).shape, generator=g, dtype=F64).to(out_dtype).to(F64).requires_grad_(True)
            for c in c64]
    _r1_step(lambda x: ora(x, w64), x64, ws64, gamma, profiled=False)

    # the package: the filters live where the data lives
    taps = _taps(_bank(wavelet), device) if learnable else None
    w = wt.WaveletTensorTuple(*taps) if learnable else _bank(wavelet)
    x = x0.to(device).requires_grad_(True)
    ws = [t.detach().to(device, out_dtype).requires_grad_(True) for t in ws64]
    names = _r1_step(lambda x: pkg(x, w), x, ws, gamma, profiled=True)

    _compare([t.grad for t in ws], [t.grad for t in ws64], dtype, f"{name}: weight gradient")
    if learnable:   # analysis only: the reconstruction filters get no gradient
        assert all(t.grad is None for t in taps[2:] + taps64[2:])
        _compare([t.grad for t in taps[:2]], [t.grad for t in taps64[:2]], dtype, f"{name}: filter gradient")
    check_second_order_kernels(names, _required(kind, learnable), name)


# ---- Hessian-vector product with respect to the filters ---------------------------------------------------------------
def _reconstruction_loss(dec, rec, x):
    def loss(*taps):
        w = wt.WaveletTensorTuple(*taps)
        y = rec(dec(x, w, mode="periodic", level=2), w)
        return ((y[..., : x.shape[-2], : x.shape[-1]] - x) ** 2).sum()

    return loss


def test_tap_hessian_vector_product():
    bank = FB.unstructured(6)
    x64 = _rand((2, 32, 40), seed=21)
    v64 = tuple(_rand((6,), seed=22 + k) for k in range(4))
    taps64 = tuple(t.detach() for t in _taps(bank, "cpu"))
    _, want = torch.autograd.functional.hvp(_reconstruction_loss(P.wavedec2, P.waverec2, x64), taps64, v64)

    taps = tuple(t.detach().to(DEV) for t in taps64)
    v = tuple(t.to(DEV) for t in v64)
    loss = _reconstruction_loss(wt.wavedec2, wt.waverec2, x64.to(DEV))
    _, got = torch.autograd.functional.hvp(loss, taps, v)
    _compare(list(got), list(want), F64, "tap Hessian-vector product")

    # the same product by one double backward (the Hessian is symmetric), profiled
    leaves = tuple(t.clone().requires_grad_(True) for t in taps)
    grads = torch.autograd.grad(loss(*leaves), leaves, create_graph=True)
    hv, names = kernels_of(lambda: torch.autograd.grad(grads, leaves, v))
    _compare(list(hv), list(want), F64, "tap Hessian-vector product by double backward")
    check_second_order_kernels(names, _required("wavedec2", True), "tap Hessian-vector product")
