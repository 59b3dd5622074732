"""Parity of the CUDA path (through the public API -> ctypes -> C ABI -> kernels) with the oracle.

Tolerances (stated, SURVEY.md section 8d): |delta| <= 1e-5 * max|c| in float32 and 1e-11 * max|c| in
float64, where c is the oracle's coefficient tensor; round-trip errors are reported against the
input's max.  The oracle (oracle/ptwt_port.py) runs the reference's own torch-CPU operator sequence.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from pytorch_wavelet_toolbox_b200 import _native
from conftest import TOL, assert_close_rel, flatten_coeffs
from oracle import ptwt_port as P

pytestmark = pytest.mark.gpu

MODES = ("zero", "constant", "reflect", "periodic", "symmetric")
DEV = "cuda"


def _cmp_tree(got, want, what):
    fg, fw = flatten_coeffs(got), flatten_coeffs(want)
    assert len(fg) == len(fw), what
    assert type(got) is type(want), what
    scale = max(float(t.abs().max()) for t in fw if t.numel())
    for j, (a, b) in enumerate(zip(fg, fw)):
        assert a.is_cuda
        assert_close_rel(a, b, scale=scale, what=f"{what} tensor {j}")


def _run(case, x, mod):
    fam, wav, mode, level, axes = case["family"], case["wavelet"], case["mode"], case["level"], case["axes"]
    if isinstance(axes, list):
        axes = tuple(axes)
    if fam == "wavedec":
        kw = {} if axes is None else {"axis": axes}
        c = mod.wavedec(x, wav, mode=mode, level=level, **kw)
        return c, mod.waverec(c, wav, **kw)
    if fam == "wavedec2":
        kw = {} if axes is None else {"axes": axes}
        c = mod.wavedec2(x, wav, mode=mode, level=level, **kw)
        return c, mod.waverec2(c, wav, **kw)
    if fam == "wavedec3":
        kw = {} if axes is None else {"axes": axes}
        c = mod.wavedec3(x, wav, mode=mode, level=level, **kw)
        return c, mod.waverec3(c, wav, **kw)
    if fam in ("matrix2", "matrix3"):
        kw = {} if axes is None else {"axes": axes}
        dec, rec = ((mod.MatrixWavedec2, mod.MatrixWaverec2) if fam == "matrix2" else (mod.MatrixWavedec3, mod.MatrixWaverec3))
        c = dec(wav, level, odd_coeff_padding_mode=mode, **kw)(x)
        return c, rec(wav, **kw)(c)
    meth = "gramschmidt" if fam == "matrix_gs" else "qr"
    c = mod.MatrixWavedec(wav, level, orthogonalization=meth, odd_coeff_padding_mode=mode)(x)
    return c, mod.MatrixWaverec(wav, orthogonalization=meth)(c)


def test_native_library_is_the_one_running():
    from pytorch_wavelet_toolbox_b200 import _native

    _native.launch_count_reset()
    wt.wavedec(torch.randn(4, 64, device=DEV), "db2", level=2)
    assert _native.launch_count() >= 1


@pytest.mark.parametrize("on_host", [False, True])
def test_golden_vectors_from_the_reference(golden, on_host):
    """Every committed fixture the unmodified reference produced, through the CUDA path; CUDA tensors
    and CPU tensors (staged through the device) give the same numbers."""
    manifest, arrays = golden
    for case in manifest["cases"]:
        i = case["id"]
        x = torch.from_numpy(arrays[f"c{i}_x"])
        xin = x if on_host else x.to(DEV)
        c, rec = _run(case, xin, wt)
        flat = flatten_coeffs(c)
        assert len(flat) == case["n_out"]
        want = [torch.from_numpy(arrays[f"c{i}_o{j}"]) for j in range(case["n_out"])]
        scale = max(float(t.abs().max()) for t in want)
        for j, t in enumerate(flat):
            assert t.device.type == ("cpu" if on_host else "cuda")
            assert_close_rel(t, want[j], scale=scale, what=f"case {i} ({case['family']} {case['wavelet']}) out {j}")
        wrec = torch.from_numpy(arrays[f"c{i}_rec"])
        assert_close_rel(rec, wrec, scale=float(wrec.abs().max()), what=f"case {i} reconstruction")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mode", MODES)
def test_wavedec_1d_sweep(dtype, mode):
    g = torch.Generator().manual_seed(11)
    for wav in ("haar", "db2", "db3", "db4", "db5", "sym5", "db8"):
        for n in (64, 65, 31, 257):
            for level in (1, 2, None):
                x = torch.randn(3, n, generator=g, dtype=torch.float64).to(dtype)
                try:
                    want = P.wavedec(x, wav, mode=mode, level=level)
                except RuntimeError:
                    with pytest.raises(RuntimeError):
                        wt.wavedec(x.to(DEV), wav, mode=mode, level=level)
                    continue
                got = wt.wavedec(x.to(DEV), wav, mode=mode, level=level)
                _cmp_tree(got, want, f"wavedec {wav} {mode} n={n} level={level}")
                rec = wt.waverec(got, wav)
                assert_close_rel(rec, P.waverec(want, wav), scale=float(x.abs().max()), what="waverec")
                assert_close_rel(rec[..., :n], x, scale=float(x.abs().max()), what="round trip")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mode", MODES)
def test_wavedec2_sweep(dtype, mode):
    g = torch.Generator().manual_seed(12)
    for wav in ("haar", "db2", "db4", "sym4", "db6", "db8"):
        for shape in ((64, 64), (33, 40), (31, 31), (65, 128), (130, 47)):
            for level in (1, 2, None):
                x = torch.randn((2,) + shape, generator=g, dtype=torch.float64).to(dtype)
                try:
                    want = P.wavedec2(x, wav, mode=mode, level=level)
                except RuntimeError:
                    with pytest.raises(RuntimeError):
                        wt.wavedec2(x.to(DEV), wav, mode=mode, level=level)
                    continue
                got = wt.wavedec2(x.to(DEV), wav, mode=mode, level=level)
                _cmp_tree(got, want, f"wavedec2 {wav} {mode} {shape} level={level}")
                if len(got) > 1:
                    assert isinstance(got[1], tuple) and got[1]._fields == ("horizontal", "vertical", "diagonal")
                rec = wt.waverec2(got, wav)
                assert_close_rel(rec, P.waverec2(want, wav), scale=float(x.abs().max()), what="waverec2")
                assert_close_rel(rec[..., : shape[0], : shape[1]], x, scale=float(x.abs().max()), what="round trip")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mode", MODES)
def test_wavedec3_sweep(dtype, mode):
    g = torch.Generator().manual_seed(13)
    for wav in ("haar", "db2", "sym4"):
        for shape in ((16, 16, 16), (17, 18, 19), (31, 32, 33), (8, 40, 21)):
            for level in (1, 2, None):
                x = torch.randn((2,) + shape, generator=g, dtype=torch.float64).to(dtype)
                try:
                    want = P.wavedec3(x, wav, mode=mode, level=level)
                except RuntimeError:
                    with pytest.raises(RuntimeError):
                        wt.wavedec3(x.to(DEV), wav, mode=mode, level=level)
                    continue
                got = wt.wavedec3(x.to(DEV), wav, mode=mode, level=level)
                _cmp_tree(got, want, f"wavedec3 {wav} {mode} {shape} level={level}")
                rec = wt.waverec3(got, wav)
                assert_close_rel(rec, P.waverec3(want, wav), scale=float(x.abs().max()), what="waverec3")
                sl = tuple(slice(0, s) for s in shape)
                assert_close_rel(rec[(Ellipsis,) + sl], x, scale=float(x.abs().max()), what="round trip")


def test_axes_batch_folding_and_missing_batch_dim():
    """tests/test_convolution_fwt.py:270-388 and tests/test_convolution_fwt_3.py:100-164 of the reference."""
    g = torch.Generator().manual_seed(14)
    x = torch.randn(2, 20, 22, 24, 26, generator=g, dtype=torch.float64)
    xd = x.to(DEV)
    _cmp_tree(wt.wavedec(xd, "db2", level=2, axis=2), P.wavedec(x, "db2", level=2, axis=2), "axis=2")
    _cmp_tree(wt.wavedec2(xd, "db2", level=2, axes=(1, 3)), P.wavedec2(x, "db2", level=2, axes=(1, 3)), "axes=(1,3)")
    _cmp_tree(wt.wavedec2(xd, "db3", level=1, axes=(-1, 1)), P.wavedec2(x, "db3", level=1, axes=(-1, 1)), "axes=(-1,1)")
    _cmp_tree(wt.wavedec3(xd, "db2", level=1, axes=(4, 1, 2)), P.wavedec3(x, "db2", level=1, axes=(4, 1, 2)), "axes3")
    c = wt.wavedec2(xd, "db2", level=2, axes=(1, 3))
    assert_close_rel(wt.waverec2(c, "db2", axes=(1, 3)), x, what="axes round trip")
    c = wt.wavedec3(xd, "db2", level=1, axes=(4, 1, 2))
    assert_close_rel(wt.waverec3(c, "db2", axes=(4, 1, 2)), x, what="axes3 round trip")
    c = wt.wavedec(xd, "db2", level=2, axis=2)
    assert_close_rel(wt.waverec(c, "db2", axis=2), x, what="axis round trip")
    # no batch dimension
    v = torch.randn(50, generator=g, dtype=torch.float64)
    _cmp_tree(wt.wavedec(v.to(DEV), "db3", level=2), P.wavedec(v, "db3", level=2), "no batch 1d")
    m = torch.randn(33, 35, generator=g)
    _cmp_tree(wt.wavedec2(m.to(DEV), "db2", level=2), P.wavedec2(m, "db2", level=2), "no batch 2d")
    vol = torch.randn(12, 13, 14, generator=g)
    _cmp_tree(wt.wavedec3(vol.to(DEV), "haar", level=1), P.wavedec3(vol, "haar", level=1), "no batch 3d")
    # non-contiguous input
    xt = torch.randn(40, 6, generator=g, dtype=torch.float64)
    _cmp_tree(wt.wavedec(xt.to(DEV).T, "db2", level=2), P.wavedec(xt.T, "db2", level=2), "transposed input")


def test_waverec_accepts_foreign_layouts():
    """Coefficients that did not come from this package (contiguous tensors, the oracle's channel-slice
    views) go through the gather path; ours go through zero-copy. Both must agree."""
    g = torch.Generator().manual_seed(15)
    x = torch.randn(3, 45, 52, generator=g, dtype=torch.float64)
    want = P.wavedec2(x, "db3", level=2)
    foreign = tuple([want[0].to(DEV)] + [wt.WaveletDetailTuple2d(*[t.to(DEV).contiguous() for t in lv]) for lv in want[1:]])
    rec_f = wt.waverec2(foreign, "db3")
    rec_o = wt.waverec2(wt.wavedec2(x.to(DEV), "db3", level=2), "db3")
    ref = P.waverec2(want, "db3")
    assert_close_rel(rec_f, ref, what="foreign layout")
    assert_close_rel(rec_o, ref, what="own layout")
    # plain tuples instead of the named tuple, lists for 1-D
    c1 = P.wavedec(x, "db2", level=3)
    assert_close_rel(wt.waverec(tuple(t.to(DEV) for t in c1), "db2"), P.waverec(c1, "db2"), what="tuple in")


def test_custom_filter_bank_objects_and_tensor_tuples():
    g = torch.Generator().manual_seed(16)

    class MyHaar:
        name = "unscaled Haar"
        filter_bank = ([0.5, 0.5], [-0.5, 0.5], [0.5, 0.5], [0.5, -0.5])
        dec_lo, dec_hi, rec_lo, rec_hi = filter_bank
        dec_len = rec_len = 2

        def __len__(self):
            return 2

    x = torch.tensor([56.0, 40.0, 8.0, 24.0, 48.0, 48.0, 40.0, 16.0], device=DEV)
    c = wt.wavedec(x, MyHaar(), level=3)  # Ripples in Mathematics p.7 (reference test_convolution_fwt.py:98-118)
    for got, w in zip(c, ([35.0], [-3.0], [16.0, 10.0], [8.0, -8.0, 0.0, 12.0])):
        assert torch.equal(got.reshape(-1).cpu(), torch.tensor(w))
    from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet

    w = as_wavelet("db3")
    tt = wt.WaveletTensorTuple.from_wavelet(w, torch.float64)
    xx = torch.randn(2, 40, generator=g, dtype=torch.float64)
    _cmp_tree(wt.wavedec(xx.to(DEV), tt, level=2), P.wavedec(xx, "db3", level=2), "tensor tuple wavelet")


def test_readme_example_config0():
    """BASELINE.json configs[0]: haar, zero, level 2, len 16, float32, CPU tensor in -> CPU tensors out."""
    x = torch.tensor([0, 1, 2, 3, 4, 5, 6, 7, 7, 6, 5, 4, 3, 2, 1, 0], dtype=torch.float32)
    c = wt.wavedec(x, "haar", mode="zero", level=2)
    assert all(t.device.type == "cpu" for t in c)
    s = 0.5 ** 0.5
    assert torch.allclose(c[0], torch.tensor([3.0, 11.0, 11.0, 3.0]), atol=1e-6)
    assert torch.allclose(c[1], torch.tensor([-2.0, -2.0, 2.0, 2.0]), atol=1e-6)
    assert torch.allclose(c[2], torch.tensor([-s] * 4 + [s] * 4), atol=1e-6)
    assert (wt.waverec(c, "haar") - x).abs().max() < 1e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_matrix_fwt_sweep(dtype):
    g = torch.Generator().manual_seed(17)
    for wav in ("haar", "db2", "db3", "db4", "db6", "sym5", "db8"):
        for n in (32, 33, 64, 100, 127, 256):
            for level in (1, 2, 3, None):
                for meth in ("qr", "gramschmidt"):
                    for odd_mode in ("zero", "reflect"):
                        x = torch.randn(4, n, generator=g, dtype=torch.float64).to(dtype)
                        ref_fw = P.MatrixWavedec(wav, level, orthogonalization=meth, odd_coeff_padding_mode=odd_mode)
                        want = ref_fw(x)
                        fw = wt.MatrixWavedec(wav, level, orthogonalization=meth, odd_coeff_padding_mode=odd_mode)
                        got = fw(x.to(DEV))
                        assert len(got) == len(want)
                        scale = max(float(t.abs().max()) for t in want)
                        tag = f"matrix {wav} n={n} level={level} {meth} {odd_mode}"
                        for a, b in zip(got, want):
                            assert_close_rel(a, b.contiguous(), scale=scale, what=tag)
                        if len(want) == 1:
                            continue
                        rec = wt.MatrixWaverec(wav, orthogonalization=meth)(got)
                        wrec = P.MatrixWaverec(wav, orthogonalization=meth)(want)
                        assert_close_rel(rec, wrec.contiguous(), scale=float(x.abs().max()), what=tag + " inverse")


def test_matrix_round_trip_and_orthogonality_config4_shape():
    """BASELINE.json configs[3] geometry at a reduced batch: db6, len 65536, float64, level None -> 12."""
    g = torch.Generator().manual_seed(18)
    x = torch.randn(8, 65536, generator=g, dtype=torch.float64)
    fw = wt.MatrixWavedec("db6")
    c = fw(x.to(DEV))
    assert fw.level == 12 and [t.shape[-1] for t in c] == [16] + [16 * 2 ** k for k in range(12)]
    want = P.MatrixWavedec("db6")(x)
    scale = max(float(t.abs().max()) for t in want)
    for a, b in zip(c, want):
        assert_close_rel(a, b.contiguous(), scale=scale, what="cfg4 coefficients")
    rec = wt.MatrixWaverec("db6")(c)
    assert float((rec.cpu() - x).abs().max()) < 1e-11      # reference: 1.8e-14
    # orthogonal transform: energy is preserved
    e_in = float((x ** 2).sum())
    e_out = sum(float((t.double() ** 2).sum()) for t in c)
    assert abs(e_in - e_out) / e_in < 1e-12
    # operator property agrees with applying the transform
    small = wt.MatrixWavedec("db4", 3)
    xs = torch.randn(5, 64, generator=g, dtype=torch.float64)
    cs = small(xs.to(DEV))
    op = small.sparse_fwt_operator.to_dense()
    assert_close_rel(torch.cat([t.cpu() for t in cs], -1), (op @ xs.T).T.contiguous(), what="operator")
    inv = wt.MatrixWaverec("db4")
    inv(cs)
    eye = inv.sparse_ifwt_operator.to_dense() @ op
    assert (eye - torch.eye(64, dtype=torch.float64)).abs().max() < 1e-8


@pytest.mark.parametrize("dtype,n,batch", [(torch.float64, 65536, 640), (torch.float32, 262144, 96)])
def test_matrix_level_groups_never_run_in_place(dtype, n, batch):
    """Long rows are analysed in several fused launches whose intermediate approximations ping-pong between the two
    halves of the scratch buffer.  Regression: a group of even depth in the middle of the chain used to get its own
    source half as destination (float64 with 2 levels per launch; float32 from 262144 samples on), which only shows
    with enough rows in flight.  The fused chain must agree with the per-level kernels, preserve energy and invert."""
    g = torch.Generator(device=DEV).manual_seed(19)
    x = torch.randn(batch, n, generator=g, device=DEV, dtype=dtype)
    fw = wt.MatrixWavedec("db6")
    c = fw(x)
    with _native.knobs(DISABLE_FUSED=1):
        want = wt.MatrixWavedec("db6")(x)
    scale = max(float(t.abs().max()) for t in want)
    for a, b in zip(c, want):
        assert_close_rel(a, b, scale=scale, what=f"fused groups vs per-level kernels, n={n} {dtype}")
    e_in = float((x.double() ** 2).sum())
    e_out = sum(float((t.double() ** 2).sum()) for t in c)
    assert abs(e_in - e_out) / e_in < (1e-12 if dtype == torch.float64 else 1e-5)
    rec = wt.MatrixWaverec("db6")(c)
    assert float((rec - x).abs().max()) < (1e-10 if dtype == torch.float64 else 2e-4)


def test_full_size_properties_config2():
    """BASELINE.json configs[1] geometry (4096x4096 float32, db4, level 4, reflect) on 2 images:
    extents, parity against the oracle on one image, round trip, linearity."""
    g = torch.Generator(device=DEV).manual_seed(1234)
    x = torch.randn(2, 4096, 4096, generator=g, device=DEV, dtype=torch.float32)
    c = wt.wavedec2(x, "db4", level=4)
    assert c[0].shape == (2, 262, 262)
    assert [lv.horizontal.shape[-1] for lv in c[1:]] == [262, 518, 1029, 2051]
    want = P.wavedec2(x[:1].cpu(), "db4", level=4)
    scale = max(float(t.abs().max()) for t in flatten_coeffs(want))
    for a, b in zip(flatten_coeffs(c), flatten_coeffs(want)):
        assert_close_rel(a[:1], b, scale=scale, what="cfg2 coefficients")
    rec = wt.waverec2(c, "db4")
    err = float((rec - x).abs().max())
    assert err < 2e-5, err          # reference itself: 1.9e-6
    y = torch.randn(2, 4096, 4096, generator=g, device=DEV, dtype=torch.float32)
    cy = wt.wavedec2(y, "db4", level=4)
    cz = wt.wavedec2(2.0 * x - y, "db4", level=4)
    for a, b, z in zip(flatten_coeffs(c), flatten_coeffs(cy), flatten_coeffs(cz)):
        assert float((2.0 * a - b - z).abs().max()) < 2e-4


def test_full_size_properties_config3():
    """BASELINE.json configs[2] geometry (256^3 float32, sym4, level 3, zero) on 1 volume."""
    g = torch.Generator(device=DEV).manual_seed(99)
    x = torch.randn(1, 256, 256, 256, generator=g, device=DEV, dtype=torch.float32)
    c = wt.wavedec3(x, "sym4", level=3)
    assert c[0].shape == (1, 38, 38, 38)
    assert [lv["aad"].shape[-1] for lv in c[1:]] == [38, 69, 131]
    want = P.wavedec3(x.cpu(), "sym4", level=3)
    scale = max(float(t.abs().max()) for t in flatten_coeffs(want))
    for a, b in zip(flatten_coeffs(c), flatten_coeffs(want)):
        assert_close_rel(a, b, scale=scale, what="cfg3 coefficients")
    rec = wt.waverec3(c, "sym4")
    assert float((rec - x).abs().max()) < 2e-5


def test_empty_batch_and_single_sample():
    x = torch.zeros(0, 32, device=DEV)
    c = wt.wavedec(x, "db2", level=2)
    assert [t.shape for t in c] == [torch.Size([0, 10]), torch.Size([0, 10]), torch.Size([0, 17])]
    one = torch.randn(1, 1, 2, dtype=torch.float64)
    _cmp_tree(wt.wavedec(one.to(DEV), "haar", mode="zero", level=1), P.wavedec(one, "haar", mode="zero", level=1), "len 2")


def _weighted_sum(coeffs, seed):
    g = torch.Generator().manual_seed(seed)
    tot = 0.0
    for t in flatten_coeffs(coeffs):
        w = torch.randn(t.shape, generator=g, dtype=torch.float64).to(t.device, t.dtype)
        tot = tot + (t * w).sum()
    return tot


@pytest.mark.parametrize("mode", ["zero", "reflect", "constant", "periodic", "symmetric"])
def test_autograd_matches_the_reference_operators(mode):
    """SURVEY 8f row 3: gradients w.r.t. the data through wavedec*/waverec* equal those of the
    reference's torch-operator chain (the oracle port under torch autograd, float64)."""
    g = torch.Generator().manual_seed(31)
    cases = [
        (wt.wavedec, P.wavedec, wt.waverec, P.waverec, torch.randn(3, 41, generator=g, dtype=torch.float64), "db3", 2),
        (wt.wavedec2, P.wavedec2, wt.waverec2, P.waverec2, torch.randn(2, 30, 37, generator=g, dtype=torch.float64), "db2", 2),
        (wt.wavedec3, P.wavedec3, wt.waverec3, P.waverec3, torch.randn(2, 12, 15, 14, generator=g, dtype=torch.float64), "db2", 1),
    ]
    for fwd, pfwd, inv, pinv, x, wav, level in cases:
        xa = x.clone().requires_grad_(True)
        xb = x.clone().requires_grad_(True)
        ca = fwd(xa.to(DEV), wav, mode=mode, level=level)
        cb = pfwd(xb, wav, mode=mode, level=level)
        for a, b in zip(flatten_coeffs(ca), flatten_coeffs(cb)):
            assert_close_rel(a, b, what=f"forward under grad {mode}")
        _weighted_sum(ca, 5).backward()
        _weighted_sum(cb, 5).backward()
        assert_close_rel(xa.grad, xb.grad, what=f"grad of {fwd.__name__} {mode}")
        # synthesis: gradients w.r.t. every coefficient tensor
        la = [t.detach().clone().requires_grad_(True) for t in flatten_coeffs(cb)]
        lb = [t.detach().clone().requires_grad_(True) for t in flatten_coeffs(cb)]

        def rebuild(flat, like):
            out, i = [flat[0]], 1
            for el in like[1:]:
                if isinstance(el, torch.Tensor):
                    out.append(flat[i]); i += 1
                elif isinstance(el, dict):
                    out.append(dict(zip(el.keys(), flat[i:i + 7]))); i += 7
                else:
                    out.append(type(el)(*flat[i:i + 3])); i += 3
            return out if isinstance(like, list) else tuple(out)

        ya = inv(rebuild([t.to(DEV) for t in la], cb), wav)
        yb = pinv(rebuild(lb, cb), wav)
        assert_close_rel(ya, yb, what="inverse under grad")
        w = torch.randn(yb.shape, generator=g, dtype=torch.float64)
        (ya * w.to(DEV)).sum().backward()
        (yb * w).sum().backward()
        for a, b in zip(la, lb):
            assert_close_rel(a.grad, b.grad, what=f"grad of {inv.__name__}")


def test_autograd_cpu_leaf_and_matrix_grads_rejected():
    x = torch.randn(2, 64, requires_grad=True)
    c = wt.wavedec(x, "db2", level=2)            # CPU leaf: staged to the GPU, gradients come back on the CPU
    sum(t.sum() for t in c).backward()
    xr = x.detach().clone().requires_grad_(True)
    sum(t.sum() for t in P.wavedec(xr, "db2", level=2)).backward()
    assert x.grad.device.type == "cpu" and torch.allclose(x.grad, xr.grad, atol=1e-5)
    with pytest.raises(NotImplementedError):
        wt.MatrixWavedec("haar", 2)(torch.randn(2, 32, device=DEV, requires_grad=True))


def _learnable(name, dtype=torch.float64, device="cpu"):
    from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet

    tt = wt.WaveletTensorTuple.from_wavelet(as_wavelet(name), dtype)
    return wt.WaveletTensorTuple(*[t.clone().to(device).requires_grad_(True) for t in tt])


@pytest.mark.parametrize("mode", ["zero", "reflect", "constant", "periodic", "symmetric"])
def test_filter_tap_gradients_match_the_reference_operators(mode):
    """SURVEY 8f row 3, second half: learnable wavelets.  Gradients w.r.t. the four filters (and the data) through
    wavedec* / waverec* equal those of the reference's torch-operator chain (the oracle port under autograd, float64;
    the reference builds its conv kernels from the filter tensors, _util.py:129-141)."""
    g = torch.Generator().manual_seed(41)
    cases = [
        (wt.wavedec, P.wavedec, wt.waverec, P.waverec, torch.randn(3, 41, generator=g, dtype=torch.float64), "db3", 2),
        (wt.wavedec2, P.wavedec2, wt.waverec2, P.waverec2, torch.randn(2, 30, 37, generator=g, dtype=torch.float64), "db2", 2),
        (wt.wavedec3, P.wavedec3, wt.waverec3, P.waverec3, torch.randn(2, 12, 15, 14, generator=g, dtype=torch.float64), "db2", 1),
    ]
    for fwd, pfwd, inv, pinv, x, wav, level in cases:
        wa, wb = _learnable(wav), _learnable(wav)
        xa = x.clone().requires_grad_(True)
        xb = x.clone().requires_grad_(True)
        ca = fwd(xa.to(DEV), wa, mode=mode, level=level)
        cb = pfwd(xb, wb, mode=mode, level=level)
        for a, b in zip(flatten_coeffs(ca), flatten_coeffs(cb)):
            assert_close_rel(a, b, scale=float(b.abs().max()) + 1.0, what=f"forward with learnable filters {mode}")
        ya = inv(ca, wa)
        yb = pinv(cb, wb)
        w = torch.randn(yb.shape, generator=g, dtype=torch.float64)
        (_weighted_sum(ca, 7) + (ya * w.to(DEV)).sum()).backward()
        (_weighted_sum(cb, 7) + (yb * w).sum()).backward()
        assert_close_rel(xa.grad, xb.grad, scale=float(xb.grad.abs().max()), what=f"data grad {fwd.__name__} {mode}")
        for name, ta, tb in zip(("dec_lo", "dec_hi", "rec_lo", "rec_hi"), wa, wb):
            assert ta.grad is not None, f"{name} got no gradient ({fwd.__name__} {mode})"
            scale = max(float(t.grad.abs().max()) for t in wb)
            assert_close_rel(ta.grad, tb.grad, scale=scale, what=f"{name} grad of {fwd.__name__} {mode}")


@pytest.mark.parametrize("mode", ["constant", "symmetric", "periodic", "reflect"])
def test_autograd_extension_longer_than_the_signal(mode):
    """Under grad the boundary extension runs inside the analysis kernel and the backward pass folds the gradient of
    the extended signal (LevelAnalysis outside zero mode): short signals whose extension wraps more than once, odd lengths, all the
    levels the signal allows -- data and filter gradients against the oracle's torch-operator chain."""
    g = torch.Generator().manual_seed(47)
    for n, wav, level in ((9, "db4", 1), (11, "db3", 2), (6, "db2", 1), (23, "db5", 1)):
        x = torch.randn(3, n, generator=g, dtype=torch.float64)
        wa, wb = _learnable(wav), _learnable(wav)
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        try:
            cb = P.wavedec(xb, wb, mode=mode, level=level)
        except (RuntimeError, ValueError):    # torch's pad refuses this mode at this length: so does the reference
            with pytest.raises((RuntimeError, ValueError)):
                wt.wavedec(xa.to(DEV), wa, mode=mode, level=level)
            continue
        ca = wt.wavedec(xa.to(DEV), wa, mode=mode, level=level)
        for a, b in zip(ca, cb):
            assert_close_rel(a, b, scale=float(b.abs().max()) + 1.0, what=f"short signal forward {mode} n={n}")
        _weighted_sum(ca, 5).backward()
        _weighted_sum(cb, 5).backward()
        assert_close_rel(xa.grad, xb.grad, scale=float(xb.grad.abs().max()), what=f"short signal data grad {mode} n={n}")
        for ta, tb in zip(wa[:2], wb[:2]):
            assert_close_rel(ta.grad, tb.grad, scale=float(tb.grad.abs().max()), what=f"short signal tap grad {mode} n={n}")


def test_filter_tap_gradients_first_layer_and_float32():
    """Data without grad, filters with grad (the usual first-layer case): the filters still get their gradient; float32
    filters on the GPU get float32 gradients on the GPU."""
    g = torch.Generator().manual_seed(43)
    x = torch.randn(4, 200, generator=g)
    wa, wb = _learnable("db4", torch.float32, DEV), _learnable("db4", torch.float32)
    ca = wt.wavedec(x.to(DEV), wa, level=3)
    cb = P.wavedec(x, wb, level=3)
    _weighted_sum(ca, 3).backward()
    _weighted_sum(cb, 3).backward()
    for ta, tb in zip(wa[:2], wb[:2]):
        assert ta.grad.is_cuda and ta.grad.dtype == torch.float32
        assert float((ta.grad.cpu() - tb.grad).abs().max()) <= 2e-4 * float(tb.grad.abs().max())
    assert wa[2].grad is None and wa[3].grad is None   # the reconstruction filters were not used


def test_host_pipeline_equals_device_path(monkeypatch):
    """CPU tensors large enough for the chunked H2D / transform / D2H pipeline give exactly what the
    device path gives (chunk size forced down so that several chunks and a ragged tail occur)."""
    from pytorch_wavelet_toolbox_b200 import fwt as F

    monkeypatch.setattr(F, "HOST_PIPELINE_MIN_BYTES", 1)
    monkeypatch.setattr(F, "HOST_PIPELINE_CHUNK_BYTES", 3 * 96 * 100 * 4)
    g = torch.Generator().manual_seed(21)
    x = torch.randn(11, 96, 100, generator=g)
    host = wt.wavedec2(x, "db4", level=2)
    dev = wt.wavedec2(x.to(DEV), "db4", level=2)
    for a, b in zip(flatten_coeffs(host), flatten_coeffs(dev)):
        assert a.device.type == "cpu" and torch.equal(a, b.cpu())
    x1 = torch.randn(9, 4, 300, generator=g, dtype=torch.float64)
    h1 = wt.wavedec(x1, "db3", level=3, mode="symmetric")
    d1 = wt.wavedec(x1.to(DEV), "db3", level=3, mode="symmetric")
    for a, b in zip(h1, d1):
        assert torch.equal(a, b.cpu())


def test_separable_front_ends():
    """fswavedec2/3 + fswaverec2/3 (SURVEY 8f row 1): dict containers over the fused kernels."""
    g = torch.Generator().manual_seed(23)
    x = torch.randn(2, 45, 52, generator=g, dtype=torch.float64)
    for mode in ("zero", "reflect", "periodic"):
        fs = wt.fswavedec2(x.to(DEV), "db3", mode=mode, level=2)
        wd = P.wavedec2(x, "db3", mode=mode, level=2)
        assert list(fs[1].keys()) == ["da", "ad", "dd"]
        assert_close_rel(fs[0], wd[0], what="fs approx")
        for d, t in zip(fs[1:], wd[1:]):
            assert_close_rel(d["da"], t.horizontal, what="da")
            assert_close_rel(d["ad"], t.vertical, what="ad")
            assert_close_rel(d["dd"], t.diagonal, what="dd")
        rec = wt.fswaverec2(fs, "db3")
        assert_close_rel(rec[..., :45, :52], x, what="fs round trip")
    x3 = torch.randn(2, 20, 22, 24, generator=g)
    fs = wt.fswavedec3(x3.to(DEV), "haar", level=2)
    wd = P.wavedec3(x3, "haar", mode="reflect", level=2)
    assert list(fs[1].keys()) == ["daa", "ada", "dda", "aad", "dad", "add", "ddd"]
    for d, t in zip(fs[1:], wd[1:]):
        for k in d:
            assert_close_rel(d[k], t[k], what=k)
    assert_close_rel(wt.fswaverec3(fs, "haar"), x3, what="fs3 round trip")
    assert wt.fswavedec2(x.to(DEV), "db3")[0].shape[-1] == P.wavedec2(x, "db3", level=3)[0].shape[-1]
    with pytest.raises(ValueError):
        wt.fswaverec2((x, (x, x, x)), "db3")


def test_long_and_odd_filters_take_the_general_kernels():
    """Filters the fused kernels do not cover (L > 16, odd L) run on the general kernels and still match."""
    g = torch.Generator().manual_seed(41)
    x1 = torch.randn(3, 300, generator=g, dtype=torch.float64)
    for wav in ("db10", "db20"):
        _cmp_tree(wt.wavedec(x1.to(DEV), wav, level=2, mode="symmetric"), P.wavedec(x1, wav, level=2, mode="symmetric"), wav)
        c = wt.wavedec(x1.to(DEV), wav, level=2, mode="zero")
        assert_close_rel(wt.waverec(c, wav)[..., :300], x1, what=f"{wav} round trip")
    x2 = torch.randn(2, 90, 100, generator=g)
    _cmp_tree(wt.wavedec2(x2.to(DEV), "db10", level=2), P.wavedec2(x2, "db10", level=2), "db10 2d")
    assert_close_rel(wt.waverec2(wt.wavedec2(x2.to(DEV), "db10", level=2), "db10"), P.waverec2(P.wavedec2(x2, "db10", level=2), "db10"),
                     scale=10.0, what="db10 2d inverse")

    class Odd5:  # odd-length custom filter bank (padding amounts follow the reference's formula for any L)
        name = "odd5"
        filter_bank = ([0.1, 0.2, 0.4, 0.2, 0.1], [-0.1, 0.3, -0.4, 0.3, -0.1], [0.1, 0.2, 0.4, 0.2, 0.1], [0.1, -0.3, 0.4, -0.3, 0.1])
        dec_lo, dec_hi, rec_lo, rec_hi = filter_bank
        dec_len = rec_len = 5

        def __len__(self):
            return 5

    _cmp_tree(wt.wavedec(x1.to(DEV), Odd5(), level=2, mode="zero"), P.wavedec(x1, Odd5(), level=2, mode="zero"), "odd filter")
    _cmp_tree(wt.wavedec2(x2.to(DEV), Odd5(), level=1, mode="constant"), P.wavedec2(x2, Odd5(), level=1, mode="constant"), "odd filter 2d")


def test_config5_geometry_db8_level5():
    """BASELINE.json configs[4] per-sample geometry (2048x2048 float32, db8, level 5) on 2 images."""
    g = torch.Generator(device=DEV).manual_seed(55)
    x = torch.randn(2, 2048, 2048, generator=g, device=DEV)
    c = wt.wavedec2(x, "db8", level=5)
    assert [lv.horizontal.shape[-1] for lv in c[1:]] == [78, 142, 269, 523, 1031] and c[0].shape[-1] == 78
    want = P.wavedec2(x[:1].cpu(), "db8", level=5)
    scale = max(float(t.abs().max()) for t in flatten_coeffs(want))
    for a, b in zip(flatten_coeffs(c), flatten_coeffs(want)):
        assert_close_rel(a[:1], b, scale=scale, what="cfg5 coefficients")
    assert float((wt.waverec2(c, "db8") - x).abs().max()) < 5e-5


def test_tiny_and_ragged_shapes():
    g = torch.Generator().manual_seed(43)
    for shape in ((1, 8, 9), (3, 9, 8), (2, 7, 130), (1, 131, 6)):
        x = torch.randn(shape, generator=g, dtype=torch.float64)
        for mode in ("zero", "symmetric", "constant"):
            _cmp_tree(wt.wavedec2(x.to(DEV), "db2", level=1, mode=mode), P.wavedec2(x, "db2", level=1, mode=mode), f"tiny {shape} {mode}")
            _cmp_tree(wt.wavedec2(x.float().to(DEV), "db2", level=1, mode=mode), P.wavedec2(x.float(), "db2", level=1, mode=mode), f"tiny f32 {shape}")
    v = torch.randn(2, 5, 6, 70, generator=g)
    _cmp_tree(wt.wavedec3(v.to(DEV), "haar", level=1, mode="symmetric"), P.wavedec3(v, "haar", level=1, mode="symmetric"), "thin volume")


def test_calls_can_be_captured_in_a_cuda_graph():
    """No allocation, synchronisation or host round trip inside the native entry points: a whole transform
    can be captured once and replayed (the way to run the small configurations without per-call host cost)."""
    g = torch.Generator().manual_seed(71)
    x2 = torch.randn((3, 200, 136), generator=g).to(DEV)
    x1 = torch.randn((4, 1000), generator=g).to(DEV)
    xm = torch.randn((4, 512), generator=g, dtype=torch.float64).to(DEV)
    fw = wt.MatrixWavedec("db3", level=3)
    iv = wt.MatrixWaverec("db3")
    fw(xm)  # operator construction (QR on the host) happens outside the capture
    iv(fw(xm))

    def run():
        c2 = wt.wavedec2(x2, "db4", level=3)
        c1 = wt.wavedec(x1, "sym5", mode="symmetric", level=4)
        cm = fw(xm)
        return c2, wt.waverec2(c2, "db4"), c1, wt.waverec(c1, "sym5"), cm, iv(cm)

    eager = run()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            captured = run()
    # new input values, same buffers: the replay must recompute everything
    x2.mul_(-2.0); x1.add_(1.0); xm.mul_(0.5)
    graph.replay()
    torch.cuda.synchronize()
    fresh = run()
    torch.cuda.synchronize()
    def leaves(t):
        if isinstance(t, torch.Tensor):
            return [t]
        if isinstance(t, dict):
            return [v for k in sorted(t) for v in leaves(t[k])]
        return [v for el in t for v in leaves(el)]

    got, want = leaves(captured), leaves(fresh)
    assert len(got) == len(want) and len(got) > 20
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert not torch.equal(leaves(eager)[0], want[0])


def test_deep_matrix_synthesis_groups_on_the_fp64_tensor_cores(knob):
    """WTB200_MATI_K=4 runs float64 MatrixWaverec as 4-level groups of the DMMA synthesis cascade (mat_inv_dmma_kernel,
    intermediate approximations stay in shared memory) instead of the default 2; it must agree with the oracle."""
    knob("MATI_K", 4)
    g = torch.Generator().manual_seed(83)
    for wav, n, level in (("db2", 64, 3), ("db4", 256, 4), ("db6", 4096, 6), ("sym5", 1000, 5), ("haar", 48, 3),
                          ("db3", 202, 4)):
        x = torch.randn((5, n), generator=g, dtype=torch.float64)
        want_c = P.MatrixWavedec(wav, level)(x)
        want = P.MatrixWaverec(wav)(want_c)
        got = wt.MatrixWaverec(wav)([t.to(DEV) for t in want_c])
        assert_close_rel(got, want, scale=float(want.abs().max()), what=f"fused synthesis {wav} n={n} L{level}")


@pytest.mark.parametrize("nt", [128, 256])
def test_matrix_analysis_on_the_fp64_tensor_cores(knob, nt):
    """float64 MatrixWavedec runs groups of levels as one DMMA cascade (mat_fwd_dmma2_kernel, the polyphase kernel in
    matrix_dmma.cuh) with 128 or 256 threads per CTA.  It must agree with the oracle where its dense operators fit and
    with the per-level kernels (DISABLE_FUSED) everywhere, for every filter length, odd lengths and unaligned rows."""
    knob("MATF_NT", nt)
    g = torch.Generator().manual_seed(85 + 2)
    for wav, n, level, bs in (("haar", 64, 3, 5), ("db2", 96, None, 7), ("db3", 250, 4, 7), ("db4", 1000, None, 4),
                              ("sym5", 4096, 7, 7), ("db6", 5001, None, 3), ("db7", 20000, 5, 7), ("db8", 8192, None, 7),
                              ("db6", 65536, None, 7), ("db5", 40000, 3, 9)):
        x = torch.randn((bs, n), generator=g, dtype=torch.float64)
        got = wt.MatrixWavedec(wav, level)(x.to(DEV))
        with _native.knobs(DISABLE_FUSED=1):
            per_level = wt.MatrixWavedec(wav, level)(x.to(DEV))
        tag = f"dmma analysis nt={nt} {wav} n={n} level={level}"
        scale = max(float(t.abs().max()) for t in per_level)
        assert len(got) == len(per_level)
        for a, b in zip(got, per_level):
            assert_close_rel(a, b, scale=scale, what=tag + " vs per-level kernels")
        if n <= 4096:
            want = P.MatrixWavedec(wav, level)(x)
            for a, b in zip(got, want):
                assert_close_rel(a, b.contiguous(), scale=scale, what=tag + " vs oracle")
    # rows that are not 16-byte aligned (a strided view): scalar detail stores
    x = torch.randn((6, 1025), generator=g, dtype=torch.float64).to(DEV)[:, 1:]
    got = wt.MatrixWavedec("db4", 4)(x)
    want = P.MatrixWavedec("db4", 4)(x.cpu().contiguous())
    for a, b in zip(got, want):
        assert_close_rel(a, b.contiguous(), scale=float(want[0].abs().max()), what="unaligned rows")


def test_matrix_synthesis_on_the_fp64_tensor_cores():
    """float64 MatrixWaverec runs groups of levels as one DMMA cascade (mat_inv_dmma_kernel in matrix_dmma.cuh, one
    chunk of the finest output per CTA).  It must agree with the oracle where the oracle's dense operators fit, with
    the per-level kernels (NO_DMMA) everywhere, and invert MatrixWavedec, on aligned and unaligned rows."""
    g = torch.Generator().manual_seed(84)
    for wav, n, level, bs in (("haar", 64, 3, 5), ("db2", 96, None, 7), ("db3", 250, 4, 7), ("db4", 1000, None, 4),
                              ("sym5", 4096, 7, 7), ("db6", 5001, None, 3), ("db7", 20000, 5, 7), ("db8", 8192, None, 7),
                              ("db6", 65536, None, 7), ("db4", 65536, 2, 5)):
        x = torch.randn((bs, n), generator=g, dtype=torch.float64)
        co = wt.MatrixWavedec(wav, level)(x.to(DEV))
        got = wt.MatrixWaverec(wav)(co)
        with _native.knobs(NO_DMMA=1):
            per_level = wt.MatrixWaverec(wav)(co)
        tag = f"dmma synthesis {wav} n={n} level={level}"
        assert_close_rel(got, per_level, scale=float(per_level.abs().max()), what=tag + " vs per-level kernels")
        assert float((got[..., :n].cpu() - x).abs().max()) < 1e-9, tag + " round trip"
        if n <= 4096:
            want = P.MatrixWaverec(wav)([t.cpu() for t in co])
            assert_close_rel(got, want.contiguous(), scale=float(want.abs().max()), what=tag + " vs oracle")
    # strided views of a packed buffer (rows not 16-byte aligned -> 8-byte copies)
    x = torch.randn((6, 1024), generator=g, dtype=torch.float64)
    co = wt.MatrixWavedec("db4", 4)(x.to(DEV))
    odd = [torch.empty(6, t.shape[-1] + 1, device=DEV, dtype=torch.float64)[:, 1:].copy_(t) for t in co]
    assert float((wt.MatrixWaverec("db4")(odd).cpu() - x).abs().max()) < 1e-10


@pytest.mark.parametrize("tile", ["0", "1", "2"])
def test_wavedec3_every_tile_shape(knob, tile):
    """The 3-D analysis kernel is instantiated for three tile shapes (16x32, 11x44, 8x64); the host picks by
    waste, WTB200_FWD3D_TILE forces one.  All must agree with the oracle on ragged extents and every mode."""
    knob("FWD3D_TILE", int(tile))
    g = torch.Generator().manual_seed(97 + int(tile))
    for mode in MODES:
        for shape, wav, lev in (((2, 37, 50, 91), "sym4", 2), ((1, 20, 131, 45), "db2", 2), ((3, 16, 18, 140), "haar", 1)):
            x = torch.randn(shape, generator=g)
            try:
                want = P.wavedec3(x, wav, mode=mode, level=lev)
            except RuntimeError:
                continue
            got = wt.wavedec3(x.to(DEV), wav, mode=mode, level=lev)
            _cmp_tree(got, want, f"tile {tile} {mode} {shape} {wav}")


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_separable_matrix_2d_3d_sweep(dtype):
    """MatrixWavedec2/3 + MatrixWaverec2/3 (separable boundary-wavelet transforms, SURVEY 8f row 2) against the
    oracle: even and odd extents (every padding mode of the odd sample), moved axes, extra batch dimensions."""
    g = torch.Generator().manual_seed(113)
    cases2 = [("db2", (3, 24, 40), 2, None), ("db3", (2, 31, 45), 2, None), ("haar", (17, 19), 3, None),
              ("sym4", (2, 3, 36, 33), 2, None), ("db2", (21, 2, 26), 2, (0, 2))]
    cases3 = [("haar", (2, 8, 12, 16), 2, None), ("db2", (11, 13, 15), 2, None), ("db2", (2, 14, 3, 12, 16), 1, (1, 3, 4))]
    for odd_mode in MODES:
        for wav, shape, level, axes in cases2:
            x = torch.randn(shape, generator=g, dtype=torch.float64).to(dtype)
            kw = {} if axes is None else {"axes": axes}
            want = P.MatrixWavedec2(wav, level, odd_coeff_padding_mode=odd_mode, **kw)(x)
            got = wt.MatrixWavedec2(wav, level, odd_coeff_padding_mode=odd_mode, **kw)(x.to(DEV))
            _cmp_tree(got, want, f"MatrixWavedec2 {wav} {shape} {odd_mode}")
            rec = wt.MatrixWaverec2(wav, **kw)(got)
            wrec = P.MatrixWaverec2(wav, **kw)(want)
            assert_close_rel(rec, wrec, scale=float(wrec.abs().max()), what=f"MatrixWaverec2 {wav} {shape}")
        for wav, shape, level, axes in cases3:
            x = torch.randn(shape, generator=g, dtype=torch.float64).to(dtype)
            kw = {} if axes is None else {"axes": axes}
            want = P.MatrixWavedec3(wav, level, odd_coeff_padding_mode=odd_mode, **kw)(x)
            got = wt.MatrixWavedec3(wav, level, odd_coeff_padding_mode=odd_mode, **kw)(x.to(DEV))
            _cmp_tree(got, want, f"MatrixWavedec3 {wav} {shape} {odd_mode}")
            rec = wt.MatrixWaverec3(wav, **kw)(got)
            wrec = P.MatrixWaverec3(wav, **kw)(want)
            assert_close_rel(rec, wrec, scale=float(wrec.abs().max()), what=f"MatrixWaverec3 {wav} {shape}")


def test_separable_matrix_2d_is_orthogonal_and_inverts():
    """Even extents: the separable operator is orthogonal (energy preserved) and the synthesis inverts it."""
    x = torch.randn(4, 256, 192, device=DEV, dtype=torch.float64)
    c = wt.MatrixWavedec2("db4", 3)(x)
    energy = float(c[0].pow(2).sum()) + sum(float(t.pow(2).sum()) for lv in c[1:] for t in lv)
    assert abs(energy - float(x.pow(2).sum())) <= 1e-9 * energy
    rec = wt.MatrixWaverec2("db4")(c)
    assert float((rec - x).abs().max()) <= 1e-10


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_wavedec_1d_fused_multilevel_kernel_long_signals(dtype):
    """Long 1-D signals take the fused multi-level kernel (several CTAs per signal, halos between chunks,
    boundary extension at both ends); periodic mode and short levels fall back to the per-level kernels."""
    g = torch.Generator().manual_seed(131)
    for wav, n, level in (("db4", 100_003, 7), ("haar", 65_536, 9), ("sym5", 40_000, 6), ("db8", 70_001, 5), ("db2", 33_333, 11)):
        x = torch.randn((3, n), generator=g, dtype=torch.float64).to(dtype)
        for mode in MODES:
            want = P.wavedec(x, wav, mode=mode, level=level)
            got = wt.wavedec(x.to(DEV), wav, mode=mode, level=level)
            _cmp_tree(got, want, f"wavedec fused {wav} n={n} L{level} {mode}")
            rec = wt.waverec(got, wav)
            assert_close_rel(rec[..., :n], x, scale=float(x.abs().max()), what=f"round trip {wav} {mode}")
