"""The non-orthogonal filter banks of tests/filter_banks.py and the oracle on them (no GPU needed).

* every unstructured bank is far from the structure of an orthogonal bank, so a kernel, tap table or adjoint that
  takes the other filter of a pair, or a filter in the wrong direction, computes other numbers;
* bior2.2 and CDF 9/7 reconstruct to round-off through the oracle in every mode and dimension;
* the oracle port reproduces the unmodified reference's outputs on these banks bit for bit, and its gradients to
  round-off (tests/golden/bank_vectors.*, oracle/make_golden_banks.py): the port shares ``filter_bank`` /
  ``as_wavelet`` with the package, so a mistake there would otherwise show up in neither.
"""
from __future__ import annotations

import json
import math

import numpy as np
import pytest
import torch

import filter_banks as FB
from conftest import GOLDEN, flatten_coeffs
from oracle import ptwt_port as P

MODES = ("zero", "constant", "reflect", "periodic", "symmetric")
F64 = torch.float64
_DEC = {1: (P.wavedec, P.waverec, "axis"), 2: (P.wavedec2, P.waverec2, "axes"), 3: (P.wavedec3, P.waverec3, "axes")}


@pytest.fixture(scope="module")
def bank_vectors():
    manifest = json.loads((GOLDEN / "bank_vectors.json").read_text())
    return manifest, np.load(GOLDEN / "bank_vectors.npz")


def fixture_bank(manifest, arrays, name: str) -> FB.FilterBank:
    """A bank as the fixture stores it (its taps, not tests/filter_banks.py's)."""
    return FB.FilterBank(name, *arrays[manifest["banks"][name]])


@pytest.mark.parametrize("filt_len", FB.ALL_LENGTHS)
def test_unstructured_bank_is_far_from_orthogonal_structure(filt_len):
    for variant in (0, 1):
        b = FB.unstructured(filt_len, variant)
        assert len(b) == b.dec_len == b.rec_len == filt_len
        assert FB.orthogonal_structure(b) == [], (b, FB.structure_distances(b))
        assert math.isclose(sum(b.dec_lo), math.sqrt(2), rel_tol=1e-14)
        assert np.linalg.norm(b.dec_lo) <= 1.5
        for f in (b.dec_hi, b.rec_lo, b.rec_hi):
            assert math.isclose(np.linalg.norm(f), 1.0, rel_tol=1e-14)
        assert all((f[0] == 0.0) == (filt_len in FB.ZERO_FIRST) for f in b.filter_bank)
    # seeded: the same taps every time, and the two variants differ
    assert FB.unstructured(filt_len).filter_bank != FB.unstructured(filt_len, 1).filter_bank


def test_orthogonal_banks_have_the_structure_the_check_looks_for():
    """The structure check is not vacuous: it finds both identities in every db / sym bank."""
    from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet

    for name in ("haar", "db2", "db3", "db8", "sym4", "sym8"):
        w = as_wavelet(name)
        found = FB.orthogonal_structure(FB.FilterBank(name, *w.filter_bank))
        assert "rec_lo = reversed dec_lo" in found and "rec_hi = reversed dec_hi" in found, (name, found)
        assert "dec_hi = alternating flip of dec_lo" in found, (name, found)


def test_cdf97_agrees_with_the_quoted_taps():
    b = FB.cdf97()
    assert np.abs(np.array(b.dec_lo) - FB.CDF97_QUOTED_DEC_LO).max() < 1e-12
    assert np.abs(np.array(b.rec_lo) - FB.CDF97_QUOTED_REC_LO).max() < 1e-12


@pytest.mark.parametrize("bank", sorted(FB.PR_BANKS))
@pytest.mark.parametrize("mode", MODES)
def test_pr_bank_reconstructs_through_the_oracle(bank, mode):
    b = FB.PR_BANKS[bank]()
    g = torch.Generator().manual_seed(3)
    for ndim, shape, level in ((1, (2, 77), 3), (2, (2, 23, 31), 2), (3, (1, 12, 13, 15), 1)):
        dec, rec, _ = _DEC[ndim]
        x = torch.randn(shape, generator=g, dtype=F64)
        y = rec(dec(x, b, mode=mode, level=level), b)
        y = y[(Ellipsis,) + tuple(slice(0, n) for n in shape[1:])]
        err = float((y - x).abs().max())
        assert err < 1e-13 * float(x.abs().max()), (bank, mode, ndim, err)


def test_fixture_taps_are_the_banks_of_this_suite(bank_vectors):
    manifest, arrays = bank_vectors
    mine = {"bior2.2": FB.bior22(), "cdf9/7": FB.cdf97(), "unstructured6": FB.unstructured(6),
            "unstructured8": FB.unstructured(8)}
    assert sorted(manifest["banks"]) == sorted(mine)
    for name, b in mine.items():
        assert np.array_equal(arrays[manifest["banks"][name]], np.array(b.filter_bank)), name


def _split(flat: torch.Tensor, shapes):
    out, at = [], 0
    for s in shapes:
        n = math.prod(s)
        out.append(flat[at: at + n].reshape(s))
        at += n
    assert at == flat.numel()
    return out


def test_port_reproduces_bank_fixture(bank_vectors):
    """Coefficients and reconstructions of wavedec / waverec in 1-, 2- and 3-D: bit for bit, float32 and float64."""
    manifest, arrays = bank_vectors
    for case in manifest["cases"]:
        key, ndim = case["key"], case["ndim"]
        b = fixture_bank(manifest, arrays, case["bank"])
        dec, rec, axkw = _DEC[ndim]
        axes = tuple(case["axes"]) if isinstance(case["axes"], list) else case["axes"]
        kw = {} if axes is None else {axkw: axes}
        x = torch.from_numpy(arrays[f"{key}_x"])
        c = dec(x, b, mode=case["mode"], level=case["level"], **kw)
        got = flatten_coeffs(c) + [rec(c, b, **kw)]
        want = _split(torch.from_numpy(arrays[f"{key}_o"]), case["shapes"])
        assert [list(t.shape) for t in got] == case["shapes"], key
        for j, (a, w) in enumerate(zip(got, want)):
            assert a.dtype == w.dtype and torch.equal(a.contiguous(), w), (case, j)


def test_port_reproduces_bank_gradients(bank_vectors):
    """Gradients with respect to the data and to all four filters of a weighted loss of wavedec* and waverec*.  The
    loss is bit for bit the reference's; the port builds its padding and n-D filters with other torch ops than the
    reference, so autograd may sum the same products in another order: 1e-13 of the largest gradient."""
    manifest, arrays = bank_vectors
    for case in manifest["grads"]:
        key, ndim = case["key"], case["ndim"]
        dec, rec, _ = _DEC[ndim]
        taps = [t.clone().requires_grad_(True) for t in torch.from_numpy(arrays[manifest["banks"][case["bank"]]])]
        x = torch.from_numpy(arrays[f"{key}_x"]).requires_grad_(True)
        c = dec(x, tuple(taps), mode=case["mode"], level=case["level"])
        outs = flatten_coeffs(c) + [rec(c, tuple(taps))]
        ws = _split(torch.from_numpy(arrays[f"{key}_w"]), case["shapes"])
        loss = sum((w * t).sum() for w, t in zip(ws, outs))
        loss.backward()
        assert float(loss.detach()) == case["loss"], key
        for what, got, want in (("data", x.grad, arrays[f"{key}_gx"]),
                                ("taps", torch.stack([t.grad for t in taps]), arrays[f"{key}_gtaps"])):
            want = torch.from_numpy(want)
            err = float((got - want).abs().max())
            assert err <= 1e-13 * float(want.abs().max()), (key, what, err)
