"""The layout builders of tests/test_gpu_layouts.py produce the strides they are named for, fold() hands them on as
views of the same storage, and _pack_bands passes shared and reversed band sets without a copy, so the GPU cases
cannot quietly turn into the contiguous case.  No GPU needed."""
from __future__ import annotations

import pytest
import torch

from pytorch_wavelet_toolbox_b200 import fwt
from pytorch_wavelet_toolbox_b200._shape import fold
from test_gpu_layouts import BAND_LAYOUTS, LAYOUTS, band_set, build

F32 = torch.float32
_SHAPES = {1: (4, 517), 2: (3, 23, 12), 3: (2, 9, 7, 8)}


def _strides_as_named(layout, t, ndim):
    B, dims = t.shape[0], t.shape[1:]
    s = t.stride()
    if layout == "packed":
        assert t.is_contiguous()
    elif layout == "bcast":
        assert s[0] == 0 and B > 1
    elif layout == "bcast_rows":
        assert s[1] == 0 and s[0] > 0
    elif layout == "interleaved":
        assert 0 < s[0] < s[1], s
        assert s[0] == t[0].numel() // dims[0]
    elif layout == "frames":
        assert 0 < s[0] < t[0].numel(), s          # consecutive items overlap
    elif layout == "canvas":
        assert s[0] != dims[0] * s[1] if ndim > 1 else s[0] != dims[0]
        assert ndim == 1 or s[-2] != dims[-1]      # rows of a wider pitch
    elif layout == "every3":
        assert s[0] == 3 * t[0].numel()
    elif layout == "unit_last":
        assert dims[-1] == 1 and s[-1] != 1 and s[-2] == 1, s


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_builder_strides_and_fold(layout, ndim):
    if layout == "unit_last":
        if ndim != 2:
            pytest.skip("a 2-D layout")
        shape = (3, 23, 1)
    elif (layout == "interleaved" or layout == "bcast_rows") and ndim == 1:
        pytest.skip("needs a second transformed axis")
    else:
        shape = _SHAPES[ndim]
    g = torch.Generator().manual_seed(0)
    hop = {1: 131, 2: 7 * shape[-1], 3: 3 * shape[-1]}[ndim] if layout == "frames" else None
    t, base = build(layout, shape, F32, g, device="cpu", hop=hop)
    assert tuple(t.shape) == shape and t.stride(-1) == (1 if layout != "unit_last" else t.stride(-1))
    assert t.untyped_storage().data_ptr() == base.untyped_storage().data_ptr()
    assert base.is_contiguous()
    _strides_as_named(layout, t, ndim)
    x, _ = fold(t, ndim, None)
    # a view of the caller's storage, unit inner stride (or a last axis of one element, which _unit_strides rewrites)
    assert x.untyped_storage().data_ptr() == base.untyped_storage().data_ptr()
    assert x.data_ptr() == t.data_ptr() and x.stride() == t.stride()
    assert x.stride(-1) == 1 or x.shape[-1] == 1
    if layout == "unit_last":
        assert fwt._unit_strides(x)[-1] == 1
    assert torch.equal(x, t)


def test_interleaved_is_what_axes_fold_produces():
    """``wavedec2(x[H, B, W], axes=(0, 2))`` folds to the interleaved layout the GPU cases build directly."""
    x = torch.randn(23, 3, 12)
    f, _ = fold(x, 2, (0, 2))
    assert f.stride() == (12, 36, 1) and f.data_ptr() == x.data_ptr()
    v, _ = build("interleaved", (3, 23, 12), F32, torch.Generator().manual_seed(0), device="cpu")
    assert v.stride() == f.stride()


@pytest.mark.parametrize("layout", BAND_LAYOUTS)
@pytest.mark.parametrize("nbands", [3, 7])
def test_band_sets_take_the_zero_copy_branch(layout, nbands):
    shape = (3, 11, 12) if nbands == 3 else (2, 5, 6, 8)
    bands, bases = band_set(layout, shape, nbands, F32, torch.Generator().manual_seed(1), device="cpu")
    base, band_stride, st, bs = fwt._pack_bands(bands, 4)
    assert base.data_ptr() == bands[0].data_ptr(), "the bands were gathered into a new buffer"
    plane = bands[0][0].numel()
    want = {"shared": 0, "zeros": 0, "reversed": -plane, "bcast": plane}[layout]
    assert band_stride == want
    assert bs == (0 if layout in ("bcast", "zeros") else bands[0].stride(0))
    assert st == tuple(bands[0].stride()[1:])
    for k, t in enumerate(bands):   # what the kernels address as band k + 1 is the k-th argument
        assert t.data_ptr() == base.data_ptr() + k * band_stride * t.element_size()


def test_iswt_detail_lists_take_the_zero_copy_branch():
    """One tensor for every level, and levels stored in reverse order, reach the iswt kernels as one band set."""
    for layout, want in (("shared", 0), ("reversed", -517)):
        details, _ = band_set(layout, (4, 517), 3, F32, torch.Generator().manual_seed(2), device="cpu")
        base, band_stride, _, _ = fwt._pack_bands(details, 4)
        assert base.data_ptr() == details[0].data_ptr() and band_stride == want
