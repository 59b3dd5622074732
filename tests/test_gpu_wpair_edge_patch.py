"""The edge strips of fwd2d_wpair_kernel extend their staged input rows past the left and right borders by copying
in-range samples of the same rows within shared memory.  Every instantiation, in every non-periodic mode, at even and
odd widths (an odd width is patched in zero mode too; it is a view with a 16-byte row pitch, as the kernel's TMA map
needs), must equal one launch per level bit for bit."""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import flatten_coeffs
from pytorch_wavelet_toolbox_b200 import _native

pytestmark = pytest.mark.gpu

# (wavelet, WPAIR_VAR): the six instantiations <2, 3, 12> <4, 3, 12> <6, 3, 12> <8, 2, 12> <8, 2, 15> <8, 3, 12>
_CASES = [("haar", None), ("db2", None), ("db3", None), ("db4", None), ("db4", 1), ("db4", 3)]


def _run(x, wav, mode, **knobs):
    with _native.knobs(**knobs):
        _native.launch_count_reset()
        got = flatten_coeffs(wt.wavedec2(x, wav, mode=mode, level=2))
        torch.cuda.synchronize()
        return got, _native.launch_count()


@pytest.mark.parametrize("width", [1000, 1001, 1023])
@pytest.mark.parametrize("mode", ["zero", "constant", "reflect", "symmetric"])
@pytest.mark.parametrize("wav,var", _CASES, ids=[f"{w}-var{v}" for w, v in _CASES])
def test_edge_patch_equals_one_launch_per_level(wav, var, mode, width):
    g = torch.Generator(device="cuda").manual_seed(width)
    x = torch.randn(2, 72, 1024, generator=g, device="cuda")[:, :, :width]
    knobs = {"WPAIR": 1, "WPAIR_MIN": 1}
    if var is not None:
        knobs["WPAIR_VAR"] = var
    fused, n_fused = _run(x, wav, mode, **knobs)
    plain, n_plain = _run(x, wav, mode, WPAIR=0)
    assert (n_fused, n_plain) == (1, 2), f"launches {n_fused} (wpair) and {n_plain} (per level) for 2 levels"
    for j, (a, b) in enumerate(zip(fused, plain)):
        assert a.shape == b.shape and torch.equal(a, b), \
            f"{wav} var {var} {mode} width {width} tensor {j}: max |delta| {float((a - b).abs().max()):.3e}"
