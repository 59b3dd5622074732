"""cwt on the GPU: parity with the reference's stored outputs and with the oracle port at sizes users run, every
partition regime of csrc/cwt.cuh, host staging, gradients, learnable-parameter refusal, launch count and install()."""
from __future__ import annotations

import sys
import types

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL
from oracle import cwt_fixture as FX
from oracle import cwt_port as P
from pytorch_wavelet_toolbox_b200 import _native
from pytorch_wavelet_toolbox_b200 import _wavelets
from pytorch_wavelet_toolbox_b200 import continuous as CW

pytestmark = pytest.mark.gpu
META, ARR = FX.load()


def close(got: torch.Tensor, want: torch.Tensor, in_dtype: torch.dtype, what=""):
    """|got - want| <= TOL[input dtype] * max|want| (float32 input: the reference's data FFT runs in complex64)."""
    assert got.shape == want.shape and got.dtype == want.dtype, f"{what}: {got.shape} {got.dtype} vs {want.shape} {want.dtype}"
    scale = max(float(want.abs().max()), 1e-300)
    err = float((got.detach().cpu() - want.detach().cpu()).abs().max())
    assert err <= TOL[in_dtype] * scale, f"{what}: {err:.3e} > {TOL[in_dtype]:.0e} * {scale:.3e}"


def _filters(wavelet, scales, dtype, precision=12):
    smp = CW.sample_wavelet(_wavelets.as_continuous_wavelet(wavelet), precision)
    return CW._Filters(smp, CW._scales_array(scales), dtype)


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["id"])
def test_fixture_parity(case):
    x = FX.data(case).cuda()
    coef, freqs = wt.cwt(x, FX.scales(case), FX.wavelet(case), sampling_period=case["sampling_period"],
                         precision=case["precision"])
    assert coef.is_cuda
    close(coef, torch.from_numpy(ARR[case["id"] + "_coef"]), x.dtype, case["id"])
    want_f = ARR[case["id"] + "_freqs"]
    assert freqs.dtype == want_f.dtype
    np.testing.assert_array_equal(freqs, want_f)


@pytest.mark.parametrize("case", META["errors"], ids=lambda c: c["case"])
def test_errors_match_the_reference(case):
    exc = {"IndexError": IndexError, "RuntimeError": RuntimeError, "ValueError": ValueError}[case["raises"]]
    with pytest.raises(exc):
        wt.cwt(torch.zeros(16, dtype=torch.float64, device="cuda"), np.array(case["scales"]), "morl")


#: (wavelet, scales, shape, dtype, precision): one per partition regime of csrc/cwt.cuh
PORT_CASES = {
    # H = 2048; 129 real scales: 64 pairs and one single; P = 1 up to scale 127 (K = 2033), P = 2 from scale 128
    "pairs_odd_P1_P2": ("morl", np.arange(1, 130), (4, 16384), torch.float32, 12),
    # K up to 16385 > F = 4096 and > n; n = 5000 not a multiple of H
    "long_filters_K_gt_F_gt_n": ("cmor1.5-1.0", np.geomspace(1, 1024, 24), (2, 5000), torch.float64, 12),
    # n = 100 < H = 128; unsorted and duplicate scales
    "unsorted_duplicates_n_lt_H": ("mexh", np.array([7.0, 3.0, 3.0, 12.5, 1.0, 40.0, 0.5]), (3, 100), torch.float64, 12),
    "n_1": ("shan0.1-0.4", np.arange(1, 31), (1,), torch.float64, 12),
    "n_2_real": ("morl", np.arange(1, 12), (2, 3, 2), torch.float64, 12),
    "lead_dims_prec10": ("morl", np.arange(1, 9), (2, 3, 777), torch.float32, 10),
    "shan_reference_benchmark_shape": ("shan0.1-0.4", np.arange(1, 31), (32, 10_000), torch.float32, 12),
    "float32_scales_prec8": ("cmor1.5-1.0", np.array([0.75, 1.5, 33.0, 90.0], dtype=np.float32), (5, 3001),
                             torch.float64, 8),
}


@pytest.mark.parametrize("name", list(PORT_CASES))
def test_port_parity_at_size(name):
    w, scales, shape, dtype, prec = PORT_CASES[name]
    g = torch.Generator().manual_seed(list(PORT_CASES).index(name))
    x = torch.randn(shape, generator=g, dtype=torch.float64).to(dtype).cuda()
    got, fg = wt.cwt(x, scales, w, precision=prec)
    want, fw = P.cwt(x, scales, w, precision=prec)
    close(got, want, dtype, name)
    np.testing.assert_allclose(fg, fw, rtol=1e-14)


def test_partition_regimes_are_exercised():
    """The port cases above reach P = 1 and P > 1, filters longer than F and than n, n < H and n % H != 0."""
    f = _filters("morl", np.arange(1, 130), torch.float32)
    lg = CW.fft_log2(16384, f.kmax)
    meta, _ = CW.channel_layout(f, lg)
    assert lg == 12 and (meta[:, 1] == 1).any() and (meta[:, 1] > 1).any() and meta[-1, 4] == -1
    f = _filters("cmor1.5-1.0", np.geomspace(1, 1024, 24), torch.float64)
    lg = CW.fft_log2(5000, f.kmax)
    assert f.kmax > (1 << lg) and f.kmax > 5000 and 5000 % (1 << (lg - 1))
    f = _filters("mexh", np.array([7.0, 3.0, 3.0, 12.5, 1.0, 40.0, 0.5]), torch.float64)
    assert 100 < (1 << (CW.fft_log2(100, f.kmax) - 1))


def test_non_contiguous_input():
    g = torch.Generator().manual_seed(5)
    base = torch.randn(700, 6, generator=g, dtype=torch.float64).cuda()
    x = base.T                                     # [6, 700], inner stride 6
    assert not x.is_contiguous()
    got, _ = wt.cwt(x, np.arange(1, 20), "morl")
    want, _ = P.cwt(x.contiguous(), np.arange(1, 20), "morl")
    close(got, want, torch.float64, "non-contiguous")
    got, _ = wt.cwt(base[::2, 1], np.arange(1, 5), "cmor1.5-1.0")
    want, _ = P.cwt(base[::2, 1].contiguous(), np.arange(1, 5), "cmor1.5-1.0")
    close(got, want, torch.float64, "strided 1-D")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cpu_input_is_staged_and_returned_on_the_cpu(dtype):
    g = torch.Generator().manual_seed(9)
    x = torch.randn(3, 1500, generator=g, dtype=torch.float64).to(dtype)
    got, _ = wt.cwt(x, np.arange(1, 17), "cmor1.5-1.0")
    assert got.device.type == "cpu"
    want, _ = P.cwt(x, np.arange(1, 17), "cmor1.5-1.0")
    close(got, want, dtype, "cpu staging")


@pytest.mark.parametrize("w", ["morl", "cmor1.5-1.0"])
def test_gradcheck(w):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 40, generator=g, dtype=torch.float64).cuda().requires_grad_(True)
    scales = np.array([1.0, 2.5, 6.0])                 # an odd number of real scales; K = 97 > n at scale 6
    assert torch.autograd.gradcheck(lambda t: wt.cwt(t, scales, w)[0], (x,), eps=1e-6, atol=1e-7)


@pytest.mark.parametrize("w,scales", [("morl", np.arange(1, 40)), ("cmor1.5-1.0", np.geomspace(0.5, 300, 17))])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_gradients_match_the_port_at_size(w, scales, dtype):
    g = torch.Generator().manual_seed(13)
    x0 = torch.randn(3, 3000, generator=g, dtype=torch.float64).to(dtype).cuda()
    grads = []
    for fn in (wt.cwt, P.cwt):
        x = x0.clone().requires_grad_(True)
        coef, _ = fn(x, scales, w)
        wr = torch.randn(coef.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64).cuda()
        if coef.is_complex():
            loss = (coef.real * wr).sum() + (coef.imag * wr.flip(-1)).sum()
        else:
            loss = (coef * wr).sum()
        loss.backward()
        grads.append(x.grad)
    assert grads[0].dtype == dtype
    close(grads[0], grads[1], dtype, "grad")


@pytest.mark.parametrize("case", META["grads"], ids=lambda c: c["id"])
def test_fixture_gradients(case):
    x = torch.from_numpy(ARR[case["x"]]).to(getattr(torch, case["dtype"])).cuda().requires_grad_(True)
    coef, _ = wt.cwt(x, np.arange(1, 8), case["wavelet"])
    if case["complex"]:
        loss = (torch.view_as_real(coef) * FX.loss_weights(coef.shape + (2,)).cuda()).sum()
    else:
        loss = (coef * FX.loss_weights(coef.shape).cuda()).sum()
    loss.backward()
    close(x.grad, torch.from_numpy(ARR[case["id"] + "_grad"]), x.dtype, case["id"])


class _LearnableMorlet(torch.nn.Module):
    complex_cwt = True
    lower_bound, upper_bound = -8.0, 8.0

    def __init__(self):
        super().__init__()
        self.bandwidth = torch.nn.Parameter(torch.tensor(1.5, dtype=torch.float64))

    def wavefun(self, precision, dtype=torch.float64):
        grid = torch.linspace(-8.0, 8.0, 2 ** precision, dtype=dtype, device=self.bandwidth.device)
        psi = torch.exp(-(grid ** 2) / self.bandwidth) * torch.exp(2j * torch.pi * grid) / torch.sqrt(
            torch.pi * self.bandwidth)
        return psi, grid


def test_learnable_wavelet_parameters_raise_not_implemented():
    m = _LearnableMorlet()
    x = torch.randn(2, 64, dtype=torch.float64, device="cuda")
    with pytest.raises(NotImplementedError, match="no_grad"):
        wt.cwt(x, np.arange(1, 4), m)
    with torch.no_grad():
        got, _ = wt.cwt(x, np.arange(1, 4), m)
        want, _ = P.cwt(x, np.arange(1, 4), m)
    assert m.bandwidth.device == x.device
    close(got, want, torch.float64, "learnable module under no_grad")
    m.requires_grad_(False)
    got, _ = wt.cwt(x, np.arange(1, 4), m)
    close(got, want, torch.float64, "frozen module")


def test_launch_count():
    x = torch.randn(4, 3000, dtype=torch.float32, device="cuda")
    scales = np.array([1.2345, 2.5, 7.75])             # a filter set no other test uses: the spectra cache misses
    _native.launch_count_reset()
    wt.cwt(x, scales, "morl")
    torch.cuda.synchronize()
    assert _native.launch_count() == 3                 # filter spectra, data spectra, main
    _native.launch_count_reset()
    wt.cwt(x, scales, "morl")
    torch.cuda.synchronize()
    assert _native.launch_count() == 2


def test_install_rebinds_ptwt_cwt(monkeypatch):
    """install() reaches ``ptwt.cwt`` and ``ptwt.continuous_transform.cwt`` (the reference's two bindings)."""
    pkg = types.ModuleType("ptwt")
    mod = types.ModuleType("ptwt.continuous_transform")
    pkg.cwt = mod.cwt = P.cwt
    pkg.continuous_transform = mod
    monkeypatch.setitem(sys.modules, "ptwt", pkg)
    monkeypatch.setitem(sys.modules, "ptwt.continuous_transform", mod)
    try:
        replaced = wt.install()
        assert "ptwt.cwt" in replaced and "ptwt.continuous_transform.cwt" in replaced
        assert pkg.cwt is wt.cwt and mod.cwt is wt.cwt
        x = torch.randn(2, 800, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
        got, _ = pkg.cwt(x.cuda(), np.arange(1, 31), "morl")
        want, _ = P.cwt(x, np.arange(1, 31), "morl")
        close(got, want, torch.float64, "installed ptwt.cwt")
    finally:
        wt.uninstall()
    assert pkg.cwt is P.cwt and mod.cwt is P.cwt
