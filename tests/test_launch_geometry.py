"""The batch construction and trace reading of tests/launch_geometry.py (no GPU): every item is exact in float32, no
two items are proportional, the per-item check tells items apart, and grids are read from a chrome trace."""
from __future__ import annotations

import itertools
import math

import pytest
import torch

from launch_geometry import bits_needed, coeff_len, combine, item_errors, kernel_launches, pairs, quantised


@pytest.mark.parametrize("n", [1, 2, 3, 96, 129, 528, 2400, 60000])
def test_pairs_are_distinct_primitive_and_non_proportional(n):
    pq = pairs(n)
    assert pq.shape == (n, 2)
    assert len({tuple(r) for r in pq.tolist()}) == n
    assert bool((pq[:, 0] > 0).all()) and bool((pq[:, 1] != 0).all())
    assert all(math.gcd(p, abs(q)) == 1 for p, q in pq.tolist())
    assert bits_needed(pq) < 24
    if n <= 600:
        # p_b q_c - q_b p_c != 0 for every b != c
        det = pq[:, 0, None] * pq[None, :, 1] - pq[:, 1, None] * pq[None, :, 0]
        assert int((det == 0).sum()) == n


@pytest.mark.parametrize("n", [96, 2400, 60000])
def test_every_item_is_exact_in_float32(n):
    g = torch.Generator().manual_seed(n)
    u, v = quantised((257,), g), quantised((257,), g)
    assert bool(((u * 256).round() == u * 256).all()) and float(u.abs().max()) <= 4
    pq = pairs(n)
    x32 = combine(u.float(), v.float(), pq, torch.float32)
    x64 = combine(u, v, pq, torch.float64)
    exact = pq[:, :1].double() * u + pq[:, 1:].double() * v
    assert torch.equal(x64, exact)
    assert torch.equal(x32.double(), exact)


def test_item_errors_tell_items_apart():
    """An item computed from another item's data, or written at another item's offset, exceeds the tolerance."""
    g = torch.Generator().manual_seed(3)
    u, v = quantised((2, 40), g), quantised((2, 40), g)
    cu, cv = [2 * u[0], u[1]], [v[0] - v[1], 3 * v[1]]
    pq = pairs(50)
    got = [combine(a, b, pq, torch.float64) for a, b in zip(cu, cv)]
    err, scale = item_errors(got, cu, cv, pq)
    assert float(err.max()) == 0.0
    assert torch.allclose(scale, pq[:, 0].abs().double() * 8 + pq[:, 1].abs().double() * 8, rtol=0.5)
    for b, c in itertools.permutations(range(0, 50, 7), 2):
        bad = [t.clone() for t in got]
        bad[1][b] = got[1][c]
        err, scale = item_errors(bad, cu, cv, pq)
        assert float(err[b]) > 1e-3 * float(scale[b]), (b, c)
        assert float(err.max()) == float(err[b])


def test_kernel_launches_from_a_chrome_trace():
    trace = {"traceEvents": [
        {"cat": "kernel", "name": "void wtb::axis_fwd_kernel<double>(wtb::AxisFwdParams<double>)", "ts": 20,
         "args": {"grid": [8448, 1, 1], "block": [256, 1, 1], "stream": 7, "correlation": 41}},
        {"cat": "cuda_runtime", "name": "cudaLaunchKernel", "ts": 5, "args": {}},
        {"cat": "kernel", "name": "void wtb::fwd2d_strip_f32_kernel<8, 64, true>(wtb::Fwd2dParams<float>, CUtensorMap)",
         "ts": 10, "args": {"grid": [9, 3, 96], "block": [256, 1, 1], "stream": 13, "correlation": 40}},
        {"cat": "kernel", "name": "void wtb::axis_inv_kernel<double>(wtb::AxisInvParams<double>)", "ts": 5,
         "args": {"grid": [8448, 1, 1], "block": [256, 1, 1], "stream": 13, "correlation": 42}},
    ]}
    # host launch order (correlation id), not device start time: the last launch started first on another stream
    ks = kernel_launches(trace)
    assert [k.name for k in ks] == ["fwd2d_strip_f32_kernel<8, 64, true>", "axis_fwd_kernel<double>",
                                    "axis_inv_kernel<double>"]
    assert ks[0].grid == (9, 3, 96) and ks[0].stream == 13 and ks[1].block == (256, 1, 1)
    with pytest.raises(AssertionError, match="no grid"):
        kernel_launches({"traceEvents": [{"cat": "kernel", "name": "k", "args": {}}]})


def test_coeff_len_matches_the_oracle():
    from oracle import ptwt_port as P

    for n, wav, L in ((1024, "db4", 8), (1023, "db3", 6), (96, "db2", 4), (4001, "db3", 6), (7, "haar", 2)):
        assert P.wavedec(torch.zeros(1, n, dtype=torch.float64), wav, level=1)[0].shape[-1] == coeff_len(n, L)
