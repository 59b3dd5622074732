"""wt_dwt_workspace_bytes: 0 for calls the fused 2-D / 3-D kernels run, the general path's exact requirement for the
rest.  DISABLE_FUSED=1 sends every call to the general path, so the expected amount comes from the library itself."""
from __future__ import annotations

import pytest

from pytorch_wavelet_toolbox_b200 import _native as N

F32, F64 = 0, 1
FWD, INV = 0, 1


def _bytes(ndim, dtype, levels, L, batch, dims, inverse):
    dims_arr, dims_p = N.i64_array(dims)
    return int(N.load().wt_dwt_workspace_bytes(ndim, dtype, levels, L, batch, dims_p, inverse))


def _general(knob, *args):
    knob("DISABLE_FUSED", 1)
    want = _bytes(*args)
    knob("DISABLE_FUSED", 0)
    assert want > 0
    return want


# (ndim, dtype, levels, filter length, batch, dims of x or y, direction): the fused kernels take these
FUSED = [
    (2, F32, 1, 8, 1, (2, 2**30 - 2), FWD),       # widest level input of the 2-D strip kernel
    (2, F64, 3, 8, 4, (256, 256), FWD),
    (2, F32, 3, 16, 4, (256, 256), INV),
    (3, F32, 1, 2, 1, (2, 2**20, 4), FWD),        # 32768 tile rows of 16
    (3, F32, 1, 2, 1, (2, 2**20 - 16, 4), INV),   # 65535 tile rows of 16 output rows
    (3, F32, 2, 8, 65535, (16, 16, 16), FWD),
    (2, F32, 1, 2, 1, (2**24, 2), FWD),           # 32768 segments of 256 rows
    (2, F32, 1, 2, 1, (2**24, 2), INV),           # 32768 segments of 512 rows
]

# ... and the general path these
GENERAL = [
    (2, F32, 1, 8, 1, (2, 2**30), FWD),           # level input of 2^30 columns
    (3, F32, 1, 2, 1, (2, 2**21, 4), FWD),        # 65536 tile rows
    (3, F32, 1, 2, 1, (2, 2**20, 4), INV),        # 65536 tile rows
    (2, F32, 1, 2, 1, (2**25, 2), FWD),           # 65536 segments
    (2, F32, 1, 2, 1, (2**25, 2), INV),           # 65536 segments
    (2, F32, 2, 3, 2, (64, 64), FWD),             # odd filter length
    (2, F32, 2, 3, 2, (64, 64), INV),
    (3, F32, 1, 5, 2, (16, 16, 16), INV),
    (2, F32, 2, 18, 2, (64, 64), FWD),            # longer than the 2-D kernels take
    (3, F32, 1, 10, 2, (16, 16, 16), FWD),        # longer than the 3-D kernels take
    (2, F64, 2, 8, 2, (64, 64), INV),             # float64 2-D synthesis
    (3, F64, 2, 4, 2, (16, 16, 16), FWD),         # float64 3-D
    (3, F64, 2, 4, 2, (16, 16, 16), INV),
    (3, F32, 1, 4, 65536, (8, 8, 8), FWD),        # batch past gridDim.z
    (3, F32, 1, 4, 65536, (8, 8, 8), INV),
]


@pytest.mark.parametrize("args", FUSED)
def test_fused_route_needs_no_workspace(args, knob):
    assert _bytes(*args) == 0
    assert _general(knob, *args) > 0


@pytest.mark.parametrize("args", GENERAL)
def test_general_route_gets_the_general_requirement(args, knob):
    assert _bytes(*args) == _general(knob, *args)


@pytest.mark.parametrize("args", FUSED + GENERAL)
def test_retired_bit_1_of_inverse_is_ignored(args, knob):
    *head, inverse = args
    assert _bytes(*head, inverse | 2) == _bytes(*args)
    knob("DISABLE_FUSED", 1)
    assert _bytes(*head, inverse | 2) == _bytes(*args)


def test_one_dimensional_transform_needs_no_workspace():
    assert _bytes(1, F32, 5, 8, 4, (4096,), FWD) == 0
    assert _bytes(1, F64, 5, 7, 4, (4096,), INV) == 0


@pytest.mark.parametrize("args", [
    (4, F32, 1, 8, 1, (8, 8, 8), FWD),            # ndim
    (2, 7, 1, 8, 1, (8, 8), FWD),                 # dtype
    (2, F32, 1, 1, 1, (8, 8), FWD),               # filter length
    (2, F32, 1, 8, -1, (8, 8), FWD),              # batch
    (2, F32, 1, 8, 1, (0, 8), INV),               # extent
])
def test_arguments_the_transform_rejects_need_no_workspace(args):
    assert _bytes(*args) == 0
