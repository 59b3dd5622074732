"""Stationary transform without a GPU: the oracle port and the closed form against the reference's stored outputs
(oracle/make_golden_swt.py), swt_max_level, the source tables of the non-periodic levels, signatures, the level-0
case and the error types."""
from __future__ import annotations

import inspect
import json

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import GOLDEN, TOL
from oracle import swt_closed_form as CF
from oracle import swt_port as P
from oracle.make_golden_swt import custom_bank
from pytorch_wavelet_toolbox_b200 import stationary
from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet, filter_bank, swt_max_level


@pytest.fixture(scope="module")
def swt_golden():
    return json.loads((GOLDEN / "swt_vectors.json").read_text()), np.load(GOLDEN / "swt_vectors.npz")


def wavelet_arg(name, dtype):
    return custom_bank(dtype) if name == "custom" else name


def test_port_equals_the_reference(swt_golden):
    man, arr = swt_golden
    for case in man["cases"]:
        k, dt = case["key"], getattr(torch, case["dtype"])
        x = torch.from_numpy(arr[case["x"]]).to(dt)
        c = P.swt(x, wavelet_arg(case["wavelet"], dt), case["level"], axis=case["axis"])
        want = torch.from_numpy(arr[f"{k}_c"])
        assert len(c) == want.shape[0], k
        rec = P.iswt(c, wavelet_arg(case["wavelet"], dt), axis=case["axis"])
        if dt == torch.float64:   # same torch operators on the same values: bit for bit
            assert all(torch.equal(a, b) for a, b in zip(c, want)), k
            assert torch.equal(rec, torch.from_numpy(arr[f"{k}_r"])), k
        else:
            scale = float(want.abs().max()) if want.numel() else 1.0
            assert float((torch.stack(c) - want).abs().max()) <= TOL[dt] * scale, k


def test_closed_form_equals_the_reference(swt_golden):
    man, arr = swt_golden
    for case in man["cases"]:
        if case["dtype"] != "float64" or case["axis"] is not None or len(case["shape"]) != 2:
            continue
        k = case["key"]
        fb = custom_bank(torch.float64) if case["wavelet"] == "custom" else filter_bank(as_wavelet(case["wavelet"]))
        fb = [np.asarray(f, dtype=np.float64) for f in fb]
        want = arr[f"{k}_c"]
        level = want.shape[0] - 1
        c = CF.swt(arr[case["x"]], fb[0], fb[1], level)
        scale = max(float(np.abs(want).max()), 1e-30)
        assert max(float(np.abs(a - b).max()) for a, b in zip(c, want)) <= 1e-12 * scale, k
        r = CF.iswt(list(want), fb[2], fb[3])
        assert float(np.abs(r - arr[f"{k}_r"]).max()) <= 1e-12 * max(float(np.abs(r).max()), 1.0), k


def test_the_fixtures_cover_the_non_periodic_extension(swt_golden):
    man, _ = swt_golden
    quirk = [c for c in man["cases"] if c["quirk"]]
    assert len(quirk) >= 20
    assert {c["n"] for c in quirk} >= {14, 37}


def test_swt_max_level_matches_pywt(swt_golden):
    man, _ = swt_golden
    for n, want in man["swt_max_level"].items():
        assert swt_max_level(int(n)) == want


def test_tables_reproduce_the_reference_extension():
    """The host tables of the kernels give the port's (reference-verified) extension on every level, and are
    absent exactly where that extension is periodic."""
    for n in (1, 3, 14, 37, 48, 96):
        for L in (2, 4, 8, 10, 16):
            for level in range(1, 8):
                d = 2 ** (level - 1)
                for inverse in (False, True):
                    hl, hr = d * (L // 2 - 1), d * (L // 2)
                    pl, pr = (hr, hl) if inverse else (hl, hr)
                    ext = P.extension_index(n, pl, pr).numpy()
                    i, m = np.arange(n)[:, None], np.arange(L)[None, :]
                    pos = i + (pl + pr) - d * m if inverse else i + d * m
                    src = stationary._level_sources(n, L, level, inverse)
                    if src is None:
                        assert np.array_equal(ext, CF.periodic(n, pl, pr))
                    else:
                        assert np.array_equal(src, ext[pos])


def test_transposed_table_is_the_transpose():
    src = stationary._level_sources(14, 8, 3, False)
    fwd, tr = stationary._csr(src, False), stationary._csr(src, True)
    n, L = src.shape
    off = 2 * ((n + 2) // 2)

    # forward rows hold (source, tap) for i*L + tap; transposed rows k hold (i, tap) with src[i, tap] == k
    pairs = fwd[off:].reshape(n, L, 2)
    assert np.array_equal(pairs[..., 0], src) and np.array_equal(pairs[..., 1], np.tile(np.arange(L), (n, 1)))
    tp = tr[off:].reshape(-1, 2)
    for k in range(n):
        got = sorted(map(tuple, tp[tr[k]:tr[k + 1]]))
        want = sorted((i, t) for i in range(n) for t in range(L) if src[i, t] == k)
        assert got == want


def test_signatures_match_the_reference(swt_golden):
    man, _ = swt_golden
    for name in ("swt", "iswt"):
        got = [[n, p.kind.name, repr(p.default)] for n, p in inspect.signature(getattr(wt, name)).parameters.items()]
        assert [g[:2] for g in got] == [w[:2] for w in man["signatures"][name]], name
        assert [g[2] for g in got] == [w[2] for w in man["signatures"][name]], name


def test_level_zero_returns_the_input_without_a_device():
    x = torch.randn(3, 15)
    out = wt.swt(x, "db4")
    assert len(out) == 1 and torch.equal(out[0], x)
    out = wt.swt(x, "db4", 0)
    assert len(out) == 1 and torch.equal(out[0], x)
    y = torch.randn(16)
    assert torch.equal(wt.iswt([y], "db2"), y) and torch.equal(wt.iswt((y,), "db2"), y)


def test_errors_have_the_reference_types(swt_golden):
    man, _ = swt_golden
    err = man["errors"]
    x = torch.randn(2, 16)
    c = P.swt(x, "db2", 2)
    calls = {
        "swt_int": lambda: wt.swt(x.to(torch.int32), "db2", 1),
        "swt_half": lambda: wt.swt(x.half(), "db2", 1),
        "swt_axis_out_of_range": lambda: wt.swt(x, "db2", 1, axis=5),
        "swt_axis_tuple": lambda: wt.swt(x, "db2", 1, axis=(0, 1)),
        "iswt_int": lambda: wt.iswt([t.to(torch.int32) for t in c], "db2"),
        "iswt_axis_out_of_range": lambda: wt.iswt(c, "db2", axis=5),
        "iswt_mixed_dtype": lambda: wt.iswt([c[0], c[1].double(), c[2]], "db2"),
        "iswt_unequal_length": lambda: wt.iswt([c[0], c[1][..., :8], c[2]], "db2"),
        "iswt_unequal_batch": lambda: wt.iswt([c[0], c[1][:1], c[2]], "db2"),
    }
    assert set(calls) == set(err)
    for name, call in calls.items():
        with pytest.raises(Exception) as info:
            call()
        assert type(info.value).__name__ == err[name], name


def test_odd_filter_lengths_are_rejected():
    bank = tuple(torch.ones(3, dtype=torch.float64) for _ in range(4))
    with pytest.raises(ValueError, match="even filter length"):
        wt.swt(torch.randn(2, 16, dtype=torch.float64), bank, 1)


def test_install_rebinds_the_stationary_names():
    assert "swt" in wt.NEXT_ROW_NAMES and "iswt" in wt.NEXT_ROW_NAMES
    assert wt.swt is stationary.swt and wt.iswt is stationary.iswt
