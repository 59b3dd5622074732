"""Which kernels run a 2-D / 3-D DWT call is decided before its first launch.

Tall shapes on either side of a launch-grid limit of the fused kernels: below it the fused kernels run, past it the
general per-axis kernels, and both match the float64 oracle.  A call refused for too small a workspace returns
WT_EWORKSPACE without launching anything, and with the full workspace computes what the normal API call computes.
"""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import flatten_coeffs
from oracle import ptwt_port as P
from pytorch_wavelet_toolbox_b200 import _native as N
from test_gpu_kernel_inventory import _close_tree, _map_tree, _rounded, launched

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, F64 = torch.float32, torch.float64

# (entry, extents of one analysis input, prefix of every kernel of this library the call launches).  Each pair
# straddles a limit on the grid of the fused kernel: past it, one dimension would need 65536 blocks.
TALL = [
    ("wavedec3", (2, 2**21, 4), "axis_fwd_kernel<float>"),       # 2^20 output rows, tiles of 16
    ("wavedec3", (2, 2**20, 4), "fwd3d_tile_kernel<2,"),
    ("waverec3", (2, 2**20, 4), "axis_inv_kernel<float>"),       # 2^20 output rows, tiles of 16
    ("waverec3", (2, 2**20 - 16, 4), "inv3d_tile_kernel<2,"),
    ("wavedec2", (2**25, 2), "axis_fwd_kernel<float>"),          # 2^24 output rows, segments of 256
    ("wavedec2", (2**24, 2), "fwd2d_strip_f32_kernel<2,"),
    ("waverec2", (2**25, 2), "axis_inv_kernel<float>"),          # 2^25 output rows, segments of 512
    ("waverec2", (2**24, 2), "inv2d_strip_kernel<2,"),
]

_API = {"wavedec2": (wt.wavedec2, P.wavedec2), "wavedec3": (wt.wavedec3, P.wavedec3),
        "waverec2": (wt.waverec2, P.waverec2), "waverec3": (wt.waverec3, P.waverec3)}
_DEC = {"waverec2": P.wavedec2, "waverec3": P.wavedec3}


@pytest.mark.parametrize("entry,shape,kernel", TALL, ids=[f"{e}-{'x'.join(map(str, s))}" for e, s, _ in TALL])
def test_tall_shapes_run_on_the_kernels_their_grid_fits(entry, shape, kernel):
    fn, oracle = _API[entry]
    g = torch.Generator().manual_seed(len(shape) + shape[1])
    x = torch.randn((1,) + shape, generator=g, dtype=F64).to(F32).to(F64)
    if entry.startswith("wavedec"):
        xd = x.to(DEV, F32)
        got, names = launched(lambda: fn(xd, "haar", mode="symmetric", level=1))
        want = oracle(x, "haar", mode="symmetric", level=1)
        _close_tree(_map_tree(got, torch.Tensor.cpu), want, F32, entry)
    else:
        coeffs = _rounded(_DEC[entry](x, "haar", mode="symmetric", level=1), F32)
        cd = _map_tree(coeffs, lambda t: t.to(DEV, F32))
        got, names = launched(lambda: fn(cd, "haar"))
        _close_tree([got.cpu()], [oracle(coeffs, "haar")], F32, entry)
    ours = [n for n in names if not n.startswith("at::")]   # synthesis gathers separately allocated bands first
    assert ours and all(n.startswith(kernel) for n in ours), names


class _ShortWorkspaceFirst:
    """The library, except that wt_dwt_fwd / wt_dwt_inv are first called with a workspace one element short of what
    the caller passes, then as passed.  Records (return code, launches made) of each short call."""

    def __init__(self, lib, itemsize):
        self._lib = lib
        self._itemsize = itemsize
        self.short = []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def _twice(self, name, args):
        fn = getattr(self._lib, name)
        *head, ws, ws_bytes, stream = args
        assert ws_bytes > self._itemsize, f"{name}: the shape needs no workspace"
        before = self._lib.wt_launch_count()
        rc = fn(*head, ws, ws_bytes - self._itemsize, stream)
        self.short.append((rc, self._lib.wt_launch_count() - before))
        return fn(*args)

    def wt_dwt_fwd(self, *args):
        return self._twice("wt_dwt_fwd", args)

    def wt_dwt_inv(self, *args):
        return self._twice("wt_dwt_inv", args)


# general-routed: filters longer than the 2-D (16) and 3-D (8) fused kernels take
@pytest.mark.parametrize("ndim,wavelet,shape", [(2, "db9", (3, 96, 100)), (3, "db5", (2, 40, 44, 48))])
def test_a_refused_call_launches_nothing(ndim, wavelet, shape, monkeypatch):
    dec, rec = (wt.wavedec2, wt.waverec2) if ndim == 2 else (wt.wavedec3, wt.waverec3)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(shape, generator=g, dtype=F32).to(DEV)
    want_c = dec(x, wavelet, mode="reflect", level=2)
    want_y = rec(want_c, wavelet)
    torch.cuda.synchronize()

    lib = _ShortWorkspaceFirst(N.load(), 4)
    monkeypatch.setattr(N, "load", lambda: lib)
    got_c = dec(x, wavelet, mode="reflect", level=2)
    got_y = rec(got_c, wavelet)
    torch.cuda.synchronize()
    monkeypatch.undo()

    assert lib.short == [(N.WT_EWORKSPACE, 0), (N.WT_EWORKSPACE, 0)]
    for a, b in zip(flatten_coeffs(got_c), flatten_coeffs(want_c), strict=True):
        assert torch.equal(a, b)
    assert torch.equal(got_y, want_y)
