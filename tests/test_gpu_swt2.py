"""swt2 / iswt2 on the GPU: parity with the float64 oracle port (oracle/swt2_port.py) across filter lengths, the tile
regimes of the pass along axes[0] (whole columns, halo tiles, the per-level kernel), awkward extents and levels,
moved axes, layouts and host tensors; zero-copy inverse, gradients, training-size batches, which kernels run and how
many launches a level takes."""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL
from filter_banks import bior22
from oracle import swt2_port as P
from pytorch_wavelet_toolbox_b200 import _native, stationary
from test_gpu_kernel_inventory import launched

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def flat(coeffs):
    out = [coeffs[0]]
    for el in coeffs[1:]:
        assert isinstance(el, wt.WaveletDetailTuple2d)
        out.extend(el)
    return out


def close(got, want, dtype, what=""):
    """|got - want| <= TOL[dtype] * max|want| over the whole list (want: float64 oracle values)."""
    got, want = (flat(t) if isinstance(t, tuple) else list(t) if isinstance(t, list) else [t] for t in (got, want))
    assert len(got) == len(want), what
    scale = max([float(w.abs().max()) for w in want] + [1e-30])
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == dtype, (what, g.shape, w.shape, g.dtype)
        err = float((g.detach().cpu().double() - w.detach().cpu().double()).abs().max())
        assert err <= TOL[dtype] * scale, f"{what}: {err:.3e} > {TOL[dtype]:.0e} * {scale:.3e}"


def rand(shape, dtype, seed=0):
    return torch.randn(shape, dtype=F64, generator=torch.Generator().manual_seed(seed)).to(dtype)


def check(x, wavelet, level, what="", axes=(-2, -1)):
    """swt2 and iswt2 of x (any device / layout) against the port on the float64 copy of x."""
    dtype = x.dtype
    c = wt.swt2(x, wavelet, level, axes=axes)
    want = P.swt2(x.detach().cpu().double(), wavelet, level, axes=axes)
    close(c, want, dtype, f"swt2 {what}")
    y = wt.iswt2(c, wavelet, axes=axes)
    c64 = (c[0].detach().cpu().double(),) + tuple(tuple(t.detach().cpu().double() for t in el) for el in c[1:])
    close(y, P.iswt2(c64, wavelet, axes=axes), dtype, f"iswt2 {what}")
    return c, y


@pytest.mark.parametrize("dtype", [torch.float32, F64])
@pytest.mark.parametrize("wavelet", ["haar", "db2", "db3", "db4", "db5", "db6", "db7", "db8", "db10"])
def test_every_filter_length(dtype, wavelet):
    """The eight unrolled lengths and db10 (L = 20: the generic instantiation)."""
    check(rand((2, 48, 40), dtype, 1).to(DEV), wavelet, 3, wavelet)


# the regimes tests/test_swt2.py proves the planner reaches for the pass along axes[0]
@pytest.mark.parametrize("dtype", [torch.float32, F64])
@pytest.mark.parametrize("B, H, W, wavelet, level", [
    (3, 256, 256, "db4", 2),        # whole columns
    (2, 2048, 8, "db4", 1),         # halo tiles
    (2, 1601, 8, "db4", 5),         # halo tiles, odd H, levels past swt_max_level
    (2, 1601, 8, "db4", 7),         # per-level kernel (level 7 of the pass along axes[0])
    (2, 1024, 24, "db2", 3),        # D = 24 gcd(H, d): not a power of two
])
def test_tile_regimes(dtype, B, H, W, wavelet, level):
    check(rand((B, H, W), dtype, H + W).to(DEV), wavelet, level, f"{H}x{W}")


@pytest.mark.parametrize("dtype", [torch.float32, F64])
@pytest.mark.parametrize("H, W, wavelet, level", [
    (33, 47, "db2", 3),        # odd extents
    (20, 12, "sym4", 4),       # not divisible by 2^J; dilations past both extents
    (1, 64, "haar", 4),        # 1 x W
    (64, 1, "db3", 3),         # H x 1
    (5, 3, "db8", 5),          # extents far shorter than the dilated filter
])
def test_awkward_extents_and_levels(dtype, H, W, wavelet, level):
    check(rand((3, H, W), dtype, H * W).to(DEV), wavelet, level, f"{H}x{W}")


def test_default_level_and_non_orthogonal_bank():
    x = rand((2, 48, 40), F64, 3).to(DEV)
    c = wt.swt2(x, "db2")
    assert len(c) == 4
    check(x, bior22(), 2, "bior2.2")


def test_moved_axes_non_contiguous_and_cpu_input():
    x = rand((2, 20, 3, 24), torch.float32, 4).to(DEV)
    check(x, "db2", 2, "4-D axes (1, 3)", axes=(1, 3))
    check(rand((2, 3, 16, 4, 12), F64, 5).to(DEV), "db3", 2, "5-D axes (3, 1)", axes=(3, 1))
    check(rand((2, 3, 16, 4, 12), F64, 6).to(DEV), "db2", 2, "5-D axes (-1, 1)", axes=(-1, 1))
    wide = rand((3, 40, 70), torch.float32, 7).to(DEV)
    check(wide[:, :, 3:51], "db4", 2, "row pitch 70")
    check(wide[:, ::2, ::2], "db4", 2, "every other sample")
    check(wide.transpose(1, 2), "haar", 3, "transposed")
    xc = rand((2, 32, 24), F64, 8)
    c, y = check(xc, "sym4", 2, "cpu")
    assert all(t.device.type == "cpu" for t in flat(c)) and y.device.type == "cpu"
    assert float((y - xc).abs().max()) <= 1e-12


def test_round_trip():
    for dtype, tol in ((torch.float32, 1e-5), (F64, 1e-12)):
        x = rand((3, 96, 80), dtype, 10).to(DEV)
        for wavelet, level in (("haar", 4), ("db4", 3), ("sym6", 2)):
            y = wt.iswt2(wt.swt2(x, wavelet, level), wavelet)
            assert float((y - x).abs().max()) <= tol * float(x.abs().max()), (dtype, wavelet)


def test_gradcheck_and_gradgradcheck():
    for H, W, wavelet, level in ((8, 6, "db2", 2), (5, 4, "haar", 2), (6, 8, "db3", 1)):
        x = rand((2, H, W), F64, H).to(DEV).requires_grad_(True)
        fwd = lambda t: tuple(flat(wt.swt2(t, wavelet, level)))     # noqa: E731
        assert torch.autograd.gradcheck(fwd, (x,))
        assert torch.autograd.gradgradcheck(fwd, (x,))
        cs = [t.detach().requires_grad_(True) for t in flat(wt.swt2(x.detach(), wavelet, level))]

        def inv(*ts):
            return wt.iswt2((ts[0],) + tuple(wt.WaveletDetailTuple2d(*ts[1 + 3 * k: 4 + 3 * k])
                                             for k in range(level)), wavelet)
        assert torch.autograd.gradcheck(inv, tuple(cs))
        assert torch.autograd.gradgradcheck(inv, tuple(cs))


def test_gradients_match_the_port_at_training_size():
    x = rand((8, 256, 256), torch.float32, 11)
    w = [rand((8, 256, 256), torch.float32, 20 + k) for k in range(10)]
    xg = x.to(DEV).requires_grad_(True)
    sum((a.to(DEV) * b).sum() for a, b in zip(w, flat(wt.swt2(xg, "db4", 3)))).backward()
    xp = x.double().requires_grad_(True)
    sum((a.double() * b).sum() for a, b in zip(w, flat(P.swt2(xp, "db4", 3)))).backward()
    close(xg.grad, xp.grad, torch.float32, "swt2 grad")
    c = [t.detach().requires_grad_(True) for t in flat(wt.swt2(x.to(DEV), "db4", 3))]
    wy = rand((8, 256, 256), torch.float32, 30)
    (wt.iswt2((c[0],) + tuple(wt.WaveletDetailTuple2d(*c[1 + 3 * k: 4 + 3 * k]) for k in range(3)), "db4")
     * wy.to(DEV)).sum().backward()
    cp = [t.detach().cpu().double().requires_grad_(True) for t in c]
    (P.iswt2((cp[0],) + tuple(wt.WaveletDetailTuple2d(*cp[1 + 3 * k: 4 + 3 * k]) for k in range(3)), "db4")
     * wy.double()).sum().backward()
    close([t.grad for t in c], [t.grad for t in cp], torch.float32, "iswt2 grad")


def test_training_size_batch_items():
    x = rand((64, 256, 256), torch.float32, 12).to(DEV)
    c = wt.swt2(x, "db4", 3)
    y = wt.iswt2(c, "db4")
    pick = [0, 31, 32, 63]
    want = P.swt2(x[pick].double().cpu(), "db4", 3)
    close(tuple([c[0][pick]] + [wt.WaveletDetailTuple2d(*(t[pick] for t in el)) for el in c[1:]]), want,
          torch.float32, "swt2 items")
    close(y[pick], x[pick].double().cpu(), torch.float32, "iswt2 items")


@pytest.mark.parametrize("dtype", [torch.float32, F64])
def test_two_launches_per_level(dtype):
    """Analysis: one launch along axes[1], one along axes[0] for both of its bands; synthesis the same."""
    x = rand((4, 128, 96), dtype, 14).to(DEV)
    for level in (1, 2, 5):
        _native.launch_count_reset()
        c = wt.swt2(x, "db4", level)
        assert _native.launch_count() == 2 * level
        _native.launch_count_reset()
        wt.iswt2(c, "db4")
        assert _native.launch_count() == 2 * level
    # the per-level kernel takes the two bands of the pass along axes[0] in one launch each
    _native.launch_count_reset()
    wt.swt2(rand((2, 1601, 8), dtype, 15).to(DEV), "db4", 7)
    assert _native.launch_count() == 2 * 7 + 1


def test_learnable_taps_and_odd_lengths_are_refused():
    x = rand((2, 16, 16), F64, 16).to(DEV)
    bank = tuple(torch.nn.Parameter(torch.tensor(f, dtype=F64)) for f in bior22().filter_bank)
    with pytest.raises(NotImplementedError):
        wt.swt2(x, bank, 2)
    c = wt.swt2(x, tuple(t.detach() for t in bank), 2)
    with pytest.raises(NotImplementedError):
        wt.iswt2(c, bank)
    with torch.no_grad():
        close(wt.swt2(x, bank, 2), P.swt2(x.cpu(), tuple(t.detach() for t in bank), 2), F64, "no_grad")
    odd = tuple(torch.ones(3, dtype=F64) for _ in range(4))
    _native.launch_count_reset()
    with pytest.raises(ValueError, match="even filter length"):
        wt.swt2(x, odd, 1)
    with pytest.raises(ValueError, match="even filter length"):
        wt.iswt2(c, odd)
    assert _native.launch_count() == 0


def test_iswt2_reads_its_own_views_without_a_copy():
    x = rand((4, 64, 48), torch.float32, 9).to(DEV)
    c = wt.swt2(x, "db4", 3)
    base = c[0].untyped_storage().data_ptr()
    assert all(t.untyped_storage().data_ptr() == base for t in flat(c))
    assert all(t.data_ptr() % 128 == 0 for t in flat(c))
    y, names = launched(lambda: wt.iswt2(c, "db4"))
    assert names and all(n.startswith("swt_") for n in names), names      # no gather copy
    close(y, x.double().cpu(), torch.float32, "round trip")

    def wide(t):        # a band in rows of a wider tensor (row pitch W + 1): a foreign layout, gathered once
        out = torch.zeros(t.shape[:-1] + (t.shape[-1] + 1,), dtype=t.dtype, device=t.device)[..., :-1]
        return out.copy_(t)
    own = (wide(c[0]),) + tuple(wt.WaveletDetailTuple2d(*(wide(t) for t in el)) for el in c[1:])
    base, _, _ = stationary._pack_planes(flat(c)[1:])
    assert base.data_ptr() == c[1][0].data_ptr()                            # the bands themselves
    base, _, _ = stationary._pack_planes(flat(own)[1:])
    assert base.untyped_storage().data_ptr() not in {t.untyped_storage().data_ptr() for t in flat(own)}
    assert torch.equal(wt.iswt2(own, "db4"), y)
    tr = (c[0].transpose(1, 2).contiguous().transpose(1, 2),) + c[1:]
    assert torch.equal(wt.iswt2(tr, "db4"), y)


def test_only_the_stationary_kernels_run():
    allowed = {f"swt_{k}_kernel<{T}, {L}>" for k in ("fwd", "inv") for T in ("float", "double")
               for L in (0, 2, 4, 6, 8, 10, 12, 14, 16)}
    allowed |= {f"swt_level_kernel<{T}, {b}>" for T in ("float", "double") for b in ("false", "true")}
    seen = set()
    for shape, wavelet, level in (((2, 64, 48), "db4", 3), ((2, 1601, 8), "db4", 7), ((2, 40, 36), "db10", 2)):
        for dtype in (torch.float32, F64):
            x = rand(shape, dtype, 13).to(DEV)
            c, names = launched(lambda: wt.swt2(x, wavelet, level))
            _, inames = launched(lambda: wt.iswt2(c, wavelet))
            assert names and inames and set(names + inames) <= allowed, (names, inames)
            seen |= set(names + inames)
    assert "swt_level_kernel<float, false>" in seen and "swt_fwd_kernel<float, 0>" in seen, seen
