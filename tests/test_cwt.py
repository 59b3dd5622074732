"""cwt host logic without a GPU: signature, built-in wavelets, frequencies, index tables, the per-scale FIR and the
port, against tests/golden/cwt_vectors.* (written from the unmodified reference by oracle/make_golden_cwt.py)."""
from __future__ import annotations

import inspect
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from oracle import cwt_fixture as FX
from oracle import cwt_port as P
from oracle.ref_import import reference_available
from pytorch_wavelet_toolbox_b200 import _wavelets
from pytorch_wavelet_toolbox_b200 import continuous as CW

ROOT = Path(__file__).resolve().parent.parent
META, ARR = FX.load()


def _tol(want: np.ndarray, dtype: str) -> float:
    return (1e-11 if dtype == "float64" else 1e-5) * max(float(np.abs(want).max()), 1e-300)


def test_signature_matches_the_reference():
    params = list(inspect.signature(wt.cwt).parameters.values())
    assert [p.name for p in params] == [s["name"] for s in META["signature"]]
    for p, s in zip(params, META["signature"]):
        assert p.kind.name == s["kind"]
        assert (None if p.default is inspect.Parameter.empty else repr(p.default)) == s["default"]


def test_cwt_is_exported_and_installed_with_the_other_rows():
    assert "cwt" in wt.__all__ and "cwt" in wt.NEXT_ROW_NAMES
    assert wt.cwt is CW.cwt


@pytest.mark.parametrize("name", sorted(META["modules"]))
@pytest.mark.parametrize("precision", [8, 10])
def test_builtin_families_match_the_reference_modules(name, precision):
    psi, x = CW.BuiltinContinuousWavelet(name).wavefun(precision)
    want_psi = ARR[f"module_{name}_p{precision}_psi"]
    want_x = FX.StoredWavelet(name).wavefun(precision)[1].numpy()
    assert META["modules"][name]["bounds"] == [x[0], x[-1]]
    np.testing.assert_allclose(x, want_x, rtol=0, atol=1e-13)
    np.testing.assert_allclose(psi, want_psi, rtol=0, atol=1e-12 * np.abs(want_psi).max())


def test_builtin_sets_pywt_attributes_in_new():
    w = _wavelets.BuiltinContinuousWavelet.__new__(_wavelets.BuiltinContinuousWavelet, "cmor1.5-1.0")
    assert (w.lower_bound, w.upper_bound, w.complex_cwt) == (-8.0, 8.0, True)
    assert (w.bandwidth_frequency, w.center_frequency) == (1.5, 1.0)
    s = _wavelets.BuiltinContinuousWavelet("shan0.1-0.4")
    assert (s.lower_bound, s.upper_bound, s.bandwidth_frequency, s.center_frequency) == (-20.0, 20.0, 0.1, 0.4)
    m = _wavelets.BuiltinContinuousWavelet("morl")
    assert not m.complex_cwt and m.bandwidth_frequency is None


@pytest.mark.parametrize("precision", [8, 10, 12])
@pytest.mark.parametrize("name,freq", [("mexh", 0.25), ("morl", 0.8125), ("cmor1.5-1.0", 1.0)])
def test_central_frequency_known_answers(name, freq, precision):
    smp = CW.sample_wavelet(CW.BuiltinContinuousWavelet(name), precision)
    assert CW.central_frequency(smp.psi, smp.x) == freq


def _frequencies(case):
    """cwt's frequency path without the transform (it needs no GPU)."""
    wav = _wavelets.as_continuous_wavelet(FX.wavelet(case))
    smp = CW.sample_wavelet(wav, case["precision"])
    f = CW.central_frequency(smp.psi, smp.x) / CW._scales_array(FX.scales(case))
    f /= case["sampling_period"]
    return f


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["id"])
def test_frequencies_match_the_fixture(case):
    f = _frequencies(case)
    want = ARR[case["id"] + "_freqs"]
    assert str(f.dtype) == case["freqs_dtype"]
    np.testing.assert_array_equal(f, want)


def test_float32_index_tables_differ_from_float64_as_in_the_reference():
    smp = CW.sample_wavelet(CW.BuiltinContinuousWavelet("morl"), 12)
    scales = np.concatenate([np.arange(1, 129), np.geomspace(1, 1024, 64)])
    differ = 0
    for s in scales:
        t32 = CW.index_table(s, smp.x, 4096, torch.float32)
        t64 = CW.index_table(s, smp.x, 4096, torch.float64)
        assert int(t64.max()) < 4096 and int(t32.max()) < 4096
        differ += not torch.equal(t32, t64)
    assert differ == 54
    assert len(CW.index_table(1.0, smp.x, 4096, torch.float64)) == 17
    assert len(CW.index_table(1024.0, smp.x, 4096, torch.float64)) == 16385


@pytest.mark.parametrize("case", [c for c in META["cases"] if np.prod(c["shape"]) <= 600], ids=lambda c: c["id"])
def test_per_scale_fir_reproduces_the_fixture(case):
    """y_s[t] = sum_k g_s[k] x[t + f_s + 1 - k], evaluated directly: the fold of diff, -sqrt(s) and crop."""
    x = FX.data(case)
    wav = _wavelets.as_continuous_wavelet(FX.wavelet(case))
    smp = CW.sample_wavelet(wav, case["precision"])
    filters = CW._Filters(smp, CW._scales_array(FX.scales(case)), x.dtype)
    xs = x.double().reshape(-1, x.shape[-1]).numpy()
    n = xs.shape[-1]
    want = ARR[case["id"] + "_coef"].reshape(len(filters.taps), -1, n)
    for s, (g, f) in enumerate(filters.taps):
        full = np.stack([np.convolve(row, g) for row in xs])          # full[i] = sum_k g[k] x[i - k]
        got = full[:, f + 1: f + 1 + n]
        if not filters.complex_out:
            got = got.real
        assert np.abs(got - want[s]).max() <= _tol(want, case["dtype"]), s


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["id"])
def test_port_matches_the_fixture(case):
    x = FX.data(case)
    coef, freqs = P.cwt(x, FX.scales(case), FX.wavelet(case), sampling_period=case["sampling_period"],
                        precision=case["precision"])
    want = ARR[case["id"] + "_coef"]
    assert str(coef.dtype).replace("torch.", "") == case["coef_dtype"]
    assert tuple(coef.shape) == want.shape
    assert float(np.abs(coef.numpy() - want).max()) <= _tol(want, case["dtype"])
    np.testing.assert_array_equal(freqs, ARR[case["id"] + "_freqs"])


@pytest.mark.parametrize("case", META["errors"], ids=lambda c: c["case"])
def test_port_and_host_raise_the_reference_errors(case):
    x = torch.zeros(16, dtype=torch.float64)
    exc = {"IndexError": IndexError, "RuntimeError": RuntimeError, "ValueError": ValueError}[case["raises"]]
    with pytest.raises(exc):
        P.cwt(x, np.array(case["scales"]), "morl")
    smp = CW.sample_wavelet(CW.BuiltinContinuousWavelet("morl"), 12)
    with pytest.raises(exc):
        CW._Filters(smp, np.array(case["scales"]), torch.float64)


def test_channel_layout_pairs_real_scales_and_folds_the_crop():
    smp = CW.sample_wavelet(CW.BuiltinContinuousWavelet("morl"), 12)
    filters = CW._Filters(smp, np.array([1.0, 2.0, 9.0, 3.0, 5.0]), torch.float64)
    meta, rows = CW.channel_layout(filters, 7)
    H = 64
    assert meta.shape == (3, 6) and rows.shape[1] == H
    assert meta[:, 3].tolist() == [0, 2, 4] and meta[:, 4].tolist() == [1, 3, -1]
    for part0, parts, d, s1, s2, e in meta:
        D = d * H + e
        assert D == max(filters.taps[s][1] + 1 for s in (s1, s2) if s >= 0)
        taps = rows[part0: part0 + parts].reshape(-1)
        need = 0
        for s, part in ((s1, taps.real), (s2, taps.imag)):
            if s < 0:
                assert not part.any()
                continue
            g, f = filters.taps[s]
            need = max(need, -(-(D - f - 1 + len(g)) // H))
            np.testing.assert_array_equal(part[D - f - 1: D - f - 1 + len(g)], g)
            assert not part[: D - f - 1].any() and not part[D - f - 1 + len(g):].any()
        assert parts == need
    cplx = CW._Filters(CW.sample_wavelet(CW.BuiltinContinuousWavelet("cmor1.5-1.0"), 12), np.arange(1, 4),
                       torch.float64)
    meta_c, _ = CW.channel_layout(cplx, 8)
    assert meta_c[:, 3].tolist() == [0, 1, 2] and (meta_c[:, 4] == -1).all()


@pytest.mark.parametrize("n,kmax,lg", [(1, 17, 6), (200, 241, 9), (200, 17, 6), (10_000, 1201, 12),
                                       (16384, 2049, 12), (1 << 18, 16385, 12), (1000, 100, 8)])
def test_fft_size_rule(n, kmax, lg):
    assert CW.fft_log2(n, kmax) == lg


def test_names_outside_the_builtin_table_raise_without_pywavelets(monkeypatch):
    monkeypatch.setattr(_wavelets, "_pywt", None)
    for name in ("gaus1", "cgau2", "fbsp1-1.5-1.0", "db4", "nonsense"):
        with pytest.raises(ValueError, match="mexh, morl, cmorB-C, shanB-C"):
            wt.cwt(torch.zeros(8), np.array([1.0]), name)
    with pytest.raises(ValueError):
        _wavelets.as_continuous_wavelet("cmor")


def test_unsupported_dtype_raises_value_error():
    with pytest.raises(ValueError):
        wt.cwt(torch.zeros(8, dtype=torch.float16), np.array([1.0]), "morl")


@pytest.mark.skipif(not reference_available(), reason="the reference checkout is not present")
def test_port_equals_the_reference():
    """In a fresh interpreter: the reference's continuous wavelets must be provided before it is imported."""
    code = """
import numpy as np, torch
from oracle.cwt_shim import import_reference
from oracle import cwt_port as P
ptwt = import_reference()
g = torch.Generator().manual_seed(3)
for w in ("mexh", "morl", "cmor1.5-1.0", "shan0.1-0.4"):
    for dt in (torch.float64, torch.float32):
        x = torch.randn(2, 300, generator=g, dtype=torch.float64).to(dt)
        for scales in (np.arange(1, 40), np.geomspace(0.3, 90, 9), np.array([2.5, 1.5], dtype=np.float32)):
            r, fr = ptwt.cwt(x, scales, w, sampling_period=0.1)
            p, fp = P.cwt(x, scales, w, sampling_period=0.1)
            assert r.dtype == p.dtype and torch.equal(r, p), (w, dt)
            assert fr.dtype == fp.dtype and np.array_equal(fr, fp), (w, dt, fr, fp)
print("ok")
"""
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stderr[-2000:]


def test_native_cwt_entry_points_check_their_arguments_without_a_gpu():
    from pytorch_wavelet_toolbox_b200 import _native as N

    lib = N.load()
    # F = 4096, n = 1000: one block plus the overhang window / block -> 2 x 4096 complex128 per signal (and channel)
    assert lib.wt_cwt_workspace_bytes(12, 4, 1000, 3, 0) == 4 * 2 * 4096 * 16
    assert lib.wt_cwt_workspace_bytes(12, 4, 1000, 3, 1) == 4 * 3 * 2 * 4096 * 16
    assert lib.wt_cwt_workspace_bytes(13, 4, 1000, 3, 0) == 0
    assert lib.wt_cwt_filter_spectra(5, 1, None, None, None, None) == -4          # WT_EUNSUPPORTED
    args = (None, None, None, 0, None, 4, 1000, 1000, None, 4000, 1000, None, 0, None)
    assert lib.wt_cwt_fwd(2, 12, 3, *args) == -1                                  # WT_EINVAL: dtype
    assert lib.wt_cwt_fwd(0, 13, 3, *args) == -4
    assert lib.wt_cwt_fwd(0, 12, 0, *args) == -2                                  # WT_ESHAPE: no channel
    assert lib.wt_cwt_fwd(0, 12, 3, *args) == -1                                  # NULL buffers
    assert lib.wt_cwt_adj(1, 12, 3, None, None, None, 0, None, 4000, 1000, 4, 0, None, 1000, None, 0, None) == -2
