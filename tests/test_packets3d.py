"""WaveletPacket3D without a device: keys and their errors, orders, the default depth, constructor errors.

Nothing here reaches a transform, so every test runs on a machine without a GPU; the numbers are checked against the
node-by-node oracle in tests/test_gpu_packets3d.py.
"""
from __future__ import annotations

import itertools

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt

WP3 = wt.WaveletPacket3D
SUBBANDS = ["aaa", "aad", "ada", "add", "daa", "dad", "dda", "ddd"]


def test_exported_but_not_rebound_by_install():
    assert "WaveletPacket3D" in wt.__all__
    assert "WaveletPacket3D" not in wt.HOT_PATH_NAMES + wt.NEXT_ROW_NAMES


def test_key_errors_in_the_order_of_the_other_packet_classes():
    with pytest.raises(ValueError, match="initialized via 'transform'"):
        WP3(None, "haar")["aaa"]                     # before transform: even a bad key gives this error first
    wp = WP3(torch.zeros(2, 16, 16, 16), "haar", maxlevel=2)
    with pytest.raises(KeyError, match="level 3"):
        wp["aaaaaaaaa"]
    with pytest.raises(KeyError, match="level 3"):
        wp["aaaaaax"]                                  # too deep comes before invalid, as in 1-D and 2-D
    for bad in ("a", "aa", "aaaa", "aadd", "aax", "xaa", "aahaaa", "qqqaad", "AAA"):
        with pytest.raises(ValueError, match="Invalid key"):
            wp[bad]
    with pytest.raises(ValueError, match="Invalid key"):
        wp.initialize(["aad", "aaddx"])
    # a rejected key expands nothing
    assert list(wp.keys()) == [""]
    assert wp[""].shape == (2, 16, 16, 16)


def test_natural_order():
    assert WP3.get_natural_order(0) == [""]
    assert WP3.get_natural_order(1) == SUBBANDS
    two = WP3.get_natural_order(2)
    assert two == [a + b for a, b in itertools.product(SUBBANDS, repeat=2)]
    assert len(two) == 64 and len(set(two)) == 64
    assert WP3.get_level(2, "natural") == two
    assert len(WP3.get_natural_order(3)) == 512


def _axis_path(key: str, axis: int) -> str:
    return "".join({"a": "l", "d": "h"}[c] for c in key[axis::3])


@pytest.mark.parametrize("level", [1, 2, 3])
def test_freq_order_is_the_gray_code_along_every_axis(level):
    from pytorch_wavelet_toolbox_b200.packets import _graycode_order

    cube = WP3.get_freq_order(level)
    assert WP3.get_level(level) == cube and WP3.get_level(level, "freq") == cube
    n = 2 ** level
    assert len(cube) == n and all(len(r) == n and all(len(c) == n for c in r) for r in cube)
    flat = [k for plane in cube for row in plane for k in row]
    assert sorted(flat) == sorted(WP3.get_natural_order(level))        # every key exactly once
    gray = _graycode_order(level, "l", "h")
    for d, r, c in itertools.product(range(n), repeat=3):
        key = cube[d][r][c]
        assert (_axis_path(key, 0), _axis_path(key, 1), _axis_path(key, 2)) == (gray[d], gray[r], gray[c])
    # neighbours along any axis differ in one letter of that axis's path: one step in frequency
    for i in range(n - 1):
        assert sum(p != q for p, q in zip(gray[i], gray[i + 1])) == 1


def test_freq_order_of_depth_one_and_bad_orders():
    assert WP3.get_freq_order(1) == [[["aaa", "aad"], ["ada", "add"]], [["daa", "dad"], ["dda", "ddd"]]]
    assert WP3.get_freq_order(0) == [[[""]]]
    with pytest.raises(ValueError, match="Unsupported order"):
        WP3.get_level(1, "nope")


def test_maxlevel_default_is_that_of_the_smallest_transformed_extent():
    assert WP3(torch.zeros(2, 64, 40, 50), "db2").maxlevel == 3                   # floor(log2(40 / 3))
    assert WP3(torch.zeros(64, 9, 64, 64), "haar", axes=(0, 2, 3)).maxlevel == 6  # axis 1 (9) is not transformed
    assert WP3(torch.zeros(8, 8, 8), "db4").maxlevel == 0
    assert WP3(torch.zeros(2, 32, 32, 32), "db1", maxlevel=1).maxlevel == 1
    wp = WP3(None, "db2")
    assert wp.maxlevel is None and wp.transform(torch.zeros(1, 20, 30, 40)).maxlevel == 2


def test_constructor_errors_and_deprecation():
    with pytest.raises(NotImplementedError):
        WP3(None, "haar", orthogonalization="cholesky")
    with pytest.raises(TypeError, match="unexpected keyword"):
        WP3(None, "haar", boundary="qr")
    with pytest.raises(ValueError):
        WP3(None, "haar", axes=(-2, -1))
    with pytest.raises(ValueError):
        WP3(None, "haar", axes=(1, 1, 2))
    with pytest.warns(DeprecationWarning):
        wp = WP3(None, "haar", boundary_orthogonalization="gramschmidt")
    assert wp.orthogonalization == "gramschmidt"


def test_past_maxlevel_and_unexpanded_leaves():
    wp = WP3(torch.zeros(2, 32, 32, 32), "db2", maxlevel=1)
    with pytest.raises(KeyError):
        wp["aadaad"]
    with pytest.raises(KeyError):
        wp.reconstruct()                          # the depth-1 leaves were never expanded
