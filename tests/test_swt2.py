"""2-D stationary transform without a GPU: the oracle port against the closed form and against the pinned 1-D swt
port, round trips, band orientation, the tile regimes the library plans for the pass along axes[0], default levels,
signatures and errors."""
from __future__ import annotations

import inspect

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from filter_banks import bior22, cdf97
from oracle import swt2_closed_form as CF
from oracle import swt2_port as P
from oracle import swt_port as P1
from pytorch_wavelet_toolbox_b200 import _native, stationary
from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet, filter_bank, swt_max_level


def _taps(wavelet):
    return [np.asarray(f, dtype=np.float64) for f in filter_bank(as_wavelet(wavelet))]


def _flat(coeffs):
    out = [coeffs[0]]
    for el in coeffs[1:]:
        out.extend(el)
    return out


def _max_err(got, want):
    return max(float(np.abs(np.asarray(g, dtype=np.float64) - np.asarray(w, dtype=np.float64)).max())
               for g, w in zip(_flat(got), _flat(want)))


@pytest.mark.parametrize("H, W, wavelet, level", [
    (5, 7, "db2", 2),       # odd extents
    (8, 12, "db4", 3),      # non-square; pads longer than H at level 3
    (1, 9, "haar", 3),      # 1 x W
    (6, 1, "sym4", 2),      # H x 1
    (3, 4, "db3", 3),       # both extents shorter than the dilated filter
    (12, 10, "db5", 2),
])
def test_port_equals_the_closed_form(H, W, wavelet, level):
    x = torch.randn(2, H, W, dtype=torch.float64, generator=torch.Generator().manual_seed(H * 31 + W))
    dec_lo, dec_hi, rec_lo, rec_hi = _taps(wavelet)
    c = P.swt2(x, wavelet, level)
    want = CF.swt2(x.numpy(), dec_lo, dec_hi, level)
    assert len(c) == level + 1 and all(isinstance(el, wt.WaveletDetailTuple2d) for el in c[1:])
    assert _max_err(c, want) <= 1e-12 * max(float(np.abs(want[0]).max()), 1.0)
    r = P.iswt2(c, wavelet)
    assert float(np.abs(r.numpy() - CF.iswt2(want, rec_lo, rec_hi)).max()) <= 1e-12 * float(x.abs().max())


@pytest.mark.parametrize("H, W, wavelet, level", [(16, 32, "db2", 2), (32, 24, "db4", 2), (64, 64, "sym3", 3)])
def test_rank_one_images_factor_into_the_1d_swt(H, W, wavelet, level):
    """For x = u (x) v and pads that fit the extents (so the pinned 1-D port is periodic): A_j = a_j(u) (x) a_j(v),
    cH_j = d_j(u) (x) a_j(v), cV_j = a_j(u) (x) d_j(v), cD_j = d_j(u) (x) d_j(v)."""
    L = len(_taps(wavelet)[0])
    assert (2 ** (level - 1)) * (L // 2) <= min(H, W)
    g = torch.Generator().manual_seed(7)
    u, v = torch.randn(H, dtype=torch.float64, generator=g), torch.randn(W, dtype=torch.float64, generator=g)
    c = P.swt2(torch.outer(u, v), wavelet, level)
    for j in range(1, level + 1):
        cu, cv = P1.swt(u[None], wavelet, j), P1.swt(v[None], wavelet, j)
        au, du, av, dv = cu[0][0], cu[1][0], cv[0][0], cv[1][0]
        h, vv, d = c[1 + level - j]
        for got, want in ((h, torch.outer(du, av)), (vv, torch.outer(au, dv)), (d, torch.outer(du, dv))):
            assert torch.allclose(got, want, rtol=0, atol=1e-12), j
        if j == level:
            assert torch.allclose(c[0], torch.outer(au, av), rtol=0, atol=1e-12)


@pytest.mark.parametrize("bank", ["haar", "db4", "sym6", "db8", bior22(), cdf97()], ids=str)
def test_port_round_trip(bank):
    x = torch.randn(3, 24, 20, dtype=torch.float64)
    for level in (1, 2, 3):
        r = P.iswt2(P.swt2(x, bank, level), bank)
        assert float((r - x).abs().max()) <= 1e-12, level


def test_band_orientation():
    """An input constant along axes[1] has no high-pass content along it: cV = cD = 0, while cH is not."""
    col = torch.randn(16, 1, dtype=torch.float64)
    x = col.expand(16, 12).clone()
    cA, (cH, cV, cD) = P.swt2(x, "db2", 1)
    assert float(cV.abs().max()) < 1e-13 and float(cD.abs().max()) < 1e-13
    assert float(cH.abs().max()) > 1e-3
    # the same with axes swapped: constant along axes[1] of (-1, -2), i.e. along the rows
    cA, (cH, cV, cD) = P.swt2(x.T.contiguous(), "db2", 1, axes=(-1, -2))
    assert float(cV.abs().max()) < 1e-13 and float(cH.abs().max()) > 1e-3


def _plan(dtype, inverse, L, H, W, level):
    tile = (np.zeros(4, dtype=np.int64))
    rc = _native.load().wt_swt_pass_plan(dtype, int(inverse), L, H * W, (1 << (level - 1)) * W,
                                         tile.ctypes.data_as(_native._i64p))
    assert rc in (0, 1), rc
    if rc == 0:
        return "level"
    D, M, C, R = (int(v) for v in tile)
    assert D % R == 0 and R & (R - 1) == 0 and D * M == H * W
    return "whole" if C == M else "halo"


# (H, W, filter length, level) -> the regime of the axes[0] pass (float32 analysis / synthesis, float64 analysis)
COLUMN_REGIMES = [
    (256, 256, 8, 1, "whole"),      # 256 rows of 256 samples per plane: whole columns
    (2048, 8, 8, 1, "halo"),        # 2048 rows of 8: too tall for one tile
    (1601, 8, 8, 5, "halo"),        # odd H: D = W, d0 = 16 rows
    (1601, 8, 8, 7, "level"),       # halo of 7 * 64 rows exceeds a quarter tile: per-level kernel
    (1024, 24, 4, 3, "whole"),      # D = 24 * 4 is not a power of two: R = 32 columns
]


@pytest.mark.parametrize("H, W, L, level, regime", COLUMN_REGIMES)
def test_column_pass_plans_reach_every_regime(H, W, L, level, regime):
    for dtype in (_native.WT_F32, _native.WT_F64):
        for inverse in (False, True):
            got = _plan(dtype, inverse, L, H, W, level)
            if dtype == _native.WT_F32 and not inverse:
                assert got == regime, (dtype, inverse)
    assert {r for *_, r in COLUMN_REGIMES} == {"whole", "halo", "level"}


def test_one_d_plans_are_unchanged():
    """With a first dilation of 1 the planner is the 1-D one: D = min(2^(j-1), n & -n), power-of-two tiles."""
    for n in (4096, 4099, 12288, 65536, 3 << 16):
        for level in (1, 3, 7):
            tile = np.zeros(4, dtype=np.int64)
            rc = _native.load().wt_swt_pass_plan(_native.WT_F32, 0, 8, n, 1 << (level - 1),
                                                 tile.ctypes.data_as(_native._i64p))
            if rc == 1:
                assert tile[0] == min(1 << (level - 1), n & -n)


def test_workspace_query():
    lib = _native.load()
    assert lib.wt_swt2_workspace_bytes(_native.WT_F32, 1, 4, 8, 16) == 2 * 4 * 8 * 16 * 4
    assert lib.wt_swt2_workspace_bytes(_native.WT_F64, 3, 4, 8, 16) == 3 * 4 * 8 * 16 * 8
    assert lib.wt_swt2_workspace_bytes(_native.WT_F32, 0, 4, 8, 16) == 0


def test_default_level_and_level_zero():
    assert min(swt_max_level(48), swt_max_level(40)) == 3
    x = torch.randn(2, 48, 40, dtype=torch.float64)
    assert len(P.swt2(x, "haar")) == 4
    for level in (None, 0, -1):
        x = torch.randn(3, 15, 8)
        out = wt.swt2(x, "db4", level)
        assert isinstance(out, tuple) and len(out) == 1 and torch.equal(out[0], x)
    y = torch.randn(2, 16, 16)
    assert torch.equal(wt.iswt2((y,), "db2"), y)


def test_signatures_and_exports():
    sig = inspect.signature(wt.swt2).parameters
    assert list(sig) == ["data", "wavelet", "level", "axes"]
    assert sig["level"].default is None and sig["axes"].default == (-2, -1)
    assert sig["axes"].kind is inspect.Parameter.KEYWORD_ONLY
    sig = inspect.signature(wt.iswt2).parameters
    assert list(sig) == ["coeffs", "wavelet", "axes"]
    assert sig["axes"].default == inspect.signature(wt.waverec2).parameters["axes"].default
    assert {"swt2", "iswt2"} <= set(wt.BEYOND_PTWT_NAMES) and {"swt2", "iswt2"} <= set(wt.__all__)
    assert "swt2" not in wt.NEXT_ROW_NAMES + wt.HOT_PATH_NAMES
    assert wt.swt2 is stationary.swt2 and wt.iswt2 is stationary.iswt2


def test_errors_are_raised_on_the_host():
    x = torch.randn(2, 16, 16)
    c = P.swt2(x, "db2", 2)
    cases = [
        (lambda: wt.swt2(x.to(torch.int32), "db2", 1), ValueError),
        (lambda: wt.swt2(x.half(), "db2", 1), ValueError),
        (lambda: wt.swt2(torch.randn(16), "db2", 1), ValueError),
        (lambda: wt.swt2(x, "db2", 1, axes=(1, 1)), ValueError),
        (lambda: wt.swt2(x, "db2", 1, axes=(0, 5)), ValueError),
        (lambda: wt.swt2(x, tuple(torch.ones(3, dtype=torch.float64) for _ in range(4)), 1), ValueError),
        (lambda: wt.iswt2((c[0].to(torch.int32),) + c[1:], "db2"), ValueError),
        (lambda: wt.iswt2(c, "db2", axes=(-1, -1)), ValueError),
        (lambda: wt.iswt2((c[0], [c[1][0], c[1][1], c[1][2]]), "db2"), ValueError),
        (lambda: wt.iswt2((c[0], c[1], c[2]._replace(horizontal=c[2][0][:, :8])), "db2"), RuntimeError),
        (lambda: wt.iswt2((c[0][:, :8],) + c[1:], "db2"), RuntimeError),
        (lambda: wt.iswt2((c[0],) + c[1:], tuple(torch.ones(3, dtype=torch.float64) for _ in range(4))), ValueError),
    ]
    for k, (call, exc) in enumerate(cases):
        with pytest.raises(exc):
            call()
    bank = tuple(torch.nn.Parameter(torch.tensor(f, dtype=torch.float64)) for f in _taps("db2"))
    with pytest.raises(NotImplementedError):
        wt.swt2(x.double(), bank, 1)
    with pytest.raises(NotImplementedError):
        wt.iswt2(tuple([c[0].double()] + [tuple(t.double() for t in el) for el in c[1:]]), bank)
