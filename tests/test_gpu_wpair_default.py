"""The kernel of independent warps (csrc/fused2d_wpair.cuh) is the default for levels 1-2 of float32 2-D analyses of
at least 8 images of >= 2^24 samples; other inputs keep one strip-kernel launch per level (WPAIR=0).  Its row pass is
the strip kernel's and its column pass adds the rows of an output in the same order, so its coefficients equal one
launch per level bit for bit."""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import flatten_coeffs
from pytorch_wavelet_toolbox_b200 import _native

pytestmark = pytest.mark.gpu


def _run(x, wav, mode, level, **knobs):
    with _native.knobs(**knobs):
        _native.launch_count_reset()
        got = flatten_coeffs(wt.wavedec2(x, wav, mode=mode, level=level))
        torch.cuda.synchronize()
        return got, _native.launch_count()


def _assert_equal(a_list, b_list, what):
    for j, (a, b) in enumerate(zip(a_list, b_list)):
        assert a.shape == b.shape and torch.equal(a, b), f"{what}: tensor {j} differs"


def test_two_levels_in_one_launch_by_default():
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.randn(8, 4096, 4096, generator=g, device="cuda")   # the smallest input it is used for
    for level in (2, 3):
        fused, n_fused = _run(x, "db4", "reflect", level)
        assert n_fused == level - 1, f"level {level}: {n_fused} launches by default"
        for off in ({"WPAIR": 0}, {"NO_WPAIR": 1}):
            plain, n_plain = _run(x, "db4", "reflect", level, **off)
            assert n_plain == level, f"{off}: {n_plain} launches for {level} levels"
            _assert_equal(fused, plain, f"{off} level {level}")


def test_smaller_images_keep_one_launch_per_level():
    """One 4096^2 image, and images of 2048^2 and smaller, measured faster with one launch per level."""
    for shape in ((1, 4096, 4096), (4, 2048, 2048), (64, 512, 512)):
        x = torch.randn(shape, device="cuda")
        _, n = _run(x, "db4", "reflect", 3)
        assert n == 3, f"{shape}: {n} launches for 3 levels"


@pytest.mark.parametrize("mode", ["zero", "constant", "reflect", "symmetric"])
@pytest.mark.parametrize("wav", ["haar", "db3", "db4"])
def test_wpair_equals_one_launch_per_level(mode, wav):
    """WPAIR_MIN=1 puts smaller images through the two-level kernel (rows must be 16-byte aligned for its TMA map)."""
    g = torch.Generator(device="cuda").manual_seed(22)
    x = torch.randn(2, 1030, 2052, generator=g, device="cuda")
    fused, n_fused = _run(x, wav, mode, 3, WPAIR_MIN=1)
    plain, n_plain = _run(x, wav, mode, 3, WPAIR=0)
    assert (n_fused, n_plain) == (2, 3), f"launches {n_fused} (wpair) and {n_plain} (per level) for 3 levels"
    for j, (a, b) in enumerate(zip(fused, plain)):
        assert torch.equal(a, b), f"{wav} {mode} tensor {j}: max |delta| {float((a - b).abs().max()):.3e}"


def test_headline_shape_equals_one_launch_per_level():
    """8 images of the config-2 size (4096^2, db4, level 4, reflect): the default path against one launch per level."""
    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.randn(8, 4096, 4096, generator=g, device="cuda")
    fused, n_fused = _run(x, "db4", "reflect", 4)
    plain, n_plain = _run(x, "db4", "reflect", 4, WPAIR=0)
    assert n_fused < n_plain == 4
    _assert_equal(fused, plain, "8 x 4096^2 db4 L4")
