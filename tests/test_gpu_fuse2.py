"""GPU tests of the two-level 2-D analysis strip kernel (csrc/fused2d_fuse2.cuh).

The kernel forms every coefficient with the same FMA sequence as one strip-kernel launch per level, from the same
float32 approximation values, so it is compared BIT FOR BIT (torch.equal) with one launch per level, and against the
oracle within |delta| <= 1e-5 * max|c| on a few cases.  The kernel is opt-in (FUSE2=1); WPAIR=0 keeps the kernel of
independent warps (fused2d_wpair.cuh), which takes levels 1-2 of large images first, out of the way.
"""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import assert_close_rel, flatten_coeffs
from oracle import ptwt_port as P
from pytorch_wavelet_toolbox_b200 import _native

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _run(x, wav, mode, level, fuse2=True, **knobs):
    with _native.knobs(WPAIR=0, FUSE2=1 if fuse2 else 0, **knobs):
        _native.launch_count_reset()
        got = flatten_coeffs(wt.wavedec2(x, wav, mode=mode, level=level))
        torch.cuda.synchronize()
        return got, _native.launch_count()


def _assert_bit_identical(x, wav, mode, level, what, **knobs):
    fused, n_fused = _run(x, wav, mode, level, **knobs)
    plain, n_plain = _run(x, wav, mode, level, fuse2=False, **knobs)
    assert len(fused) == len(plain)
    for j, (a, b) in enumerate(zip(fused, plain)):
        assert a.shape == b.shape, f"{what}: tensor {j} shape {tuple(a.shape)} != {tuple(b.shape)}"
        if not torch.equal(a, b):
            err = float((a - b).abs().max())
            raise AssertionError(f"{what}: tensor {j} differs from one launch per level (max |delta| {err:.3e})")
    return n_fused, n_plain


# (shape, level): one strip (64 x 64: approximation band 35, just above the decline limit of 32), two strips,
# a ragged / shifted last strip, one and several row segments, odd sizes, levels 2 to 5
SHAPES = [
    ((2, 64, 64), 2),
    ((2, 66, 70), 3),
    ((1, 96, 160), 2),
    ((3, 132, 260), 4),
    ((2, 200, 264), 5),
    ((1, 130, 1030), 2),
    ((2, 517, 136), 3),
    ((1, 1100, 120), 2),
    ((2, 71, 333), 4),
]


@pytest.mark.parametrize("mode", ["zero", "constant", "reflect", "symmetric", "periodic"])
@pytest.mark.parametrize("wav", ["haar", "db2", "db3", "db4", "sym4"])
def test_fuse2_bit_identical_to_one_launch_per_level(mode, wav):
    g = torch.Generator().manual_seed(11)
    for shape, level in SHAPES:
        x = torch.randn(shape, generator=g).to(DEV)
        n_fused, n_plain = _assert_bit_identical(x, wav, mode, level, f"{wav} {mode} {shape} L{level}")
        if mode == "periodic":
            assert n_fused == n_plain, f"periodic must decline: {n_fused} vs {n_plain} launches"


def test_fuse2_launches_fewer_kernels_than_levels():
    x = torch.randn(2, 512, 512, device=DEV)
    for level in (2, 3, 4, 5):
        _, n_fused = _run(x, "db4", "reflect", level)
        _, n_plain = _run(x, "db4", "reflect", level, fuse2=False)
        assert n_fused < level <= n_plain, f"level {level}: {n_fused} fused vs {n_plain} per-level launches"


def test_fuse2_declines_below_the_size_limit():
    """An approximation band under 32 rows or columns stays on one launch per level, and still agrees."""
    g = torch.Generator().manual_seed(12)
    for shape in ((1, 56, 200), (1, 200, 56), (2, 40, 40)):
        x = torch.randn(shape, generator=g).to(DEV)
        for level in (2, 3):
            n_fused, n_plain = _assert_bit_identical(x, "db4", "reflect", level, f"{shape} L{level}")
            if level == 2:
                assert n_fused == n_plain == 2, (shape, n_fused, n_plain)


@pytest.mark.parametrize("mode", ["zero", "reflect", "symmetric", "periodic"])
def test_fuse2_chunked_two_stream_branch(mode):
    """The batch cut into chunks on the caller's and the auxiliary stream (CHUNK), with the two-level kernel."""
    g = torch.Generator().manual_seed(13)
    for level in (2, 3, 4):
        x = torch.randn(7, 200, 264, generator=g).to(DEV)
        _assert_bit_identical(x, "db4", mode, level, f"chunked {mode} L{level}", CHUNK=3)


@pytest.mark.parametrize("wav,mode", [("db4", "reflect"), ("haar", "zero"), ("db3", "symmetric"), ("sym4", "constant")])
def test_fuse2_matches_the_oracle(wav, mode):
    g = torch.Generator().manual_seed(14)
    x = torch.randn(2, 300, 452, generator=g)
    got, _ = _run(x.to(DEV), wav, mode, 4)
    for i in range(x.shape[0]):
        want = flatten_coeffs(P.wavedec2(x[i:i + 1], wav, mode=mode, level=4))
        scale = max(float(t.abs().max()) for t in want)
        for j, (a, b) in enumerate(zip(got, want)):
            assert_close_rel(a[i:i + 1], b, scale=scale, what=f"{wav} {mode} image {i} tensor {j}")


def test_fuse2_full_size_bit_identical():
    """4 images at the headline shape (4096^2, db4, level 4, reflect)."""
    g = torch.Generator(device=DEV).manual_seed(15)
    x = torch.randn(4, 4096, 4096, generator=g, device=DEV)
    n_fused, n_plain = _assert_bit_identical(x, "db4", "reflect", 4, "4 x 4096^2 db4 L4")
    assert n_fused < n_plain
