"""swt / iswt on the GPU: parity with the reference's stored outputs and with the oracle port, the tile structures
of csrc/swt.cuh (halo chunks, whole residue classes, the switch between them, per-level table launches), host
staging, round trips, gradients and the launch count of the fused path."""
from __future__ import annotations

import json

import numpy as np
import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import GOLDEN, TOL
from oracle import swt_port as P
from oracle.make_golden_swt import custom_bank
from pytorch_wavelet_toolbox_b200 import _native

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def swt_golden():
    return json.loads((GOLDEN / "swt_vectors.json").read_text()), np.load(GOLDEN / "swt_vectors.npz")


def wavelet_arg(name, dtype):
    return custom_bank(dtype) if name == "custom" else name


def close(got, want, what=""):
    """|got - want| <= TOL * max|want| over the whole coefficient list (conftest.TOL)."""
    if isinstance(want, torch.Tensor):
        got, want = [got], [want]
    assert len(got) == len(want), what
    scale = max([float(w.abs().max()) for w in want if w.numel()] + [1e-30])
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == w.dtype, what
        err = float((g.detach().cpu().double() - w.detach().cpu().double()).abs().max()) if w.numel() else 0.0
        assert err <= TOL[w.dtype] * scale, f"{what}: {err:.3e} > {TOL[w.dtype]:.0e} * {scale:.3e}"


def test_parity_with_the_reference_fixtures(swt_golden):
    man, arr = swt_golden
    for case in man["cases"]:
        k, dt = case["key"], getattr(torch, case["dtype"])
        wav = wavelet_arg(case["wavelet"], dt)
        x = torch.from_numpy(arr[case["x"]]).to(dt).cuda()
        c = wt.swt(x, wav, case["level"], axis=case["axis"])
        want = list(torch.from_numpy(arr[f"{k}_c"]))
        close(c, want, f"swt {case}")
        assert all(t.is_cuda for t in c)
        close(wt.iswt(c, wav, axis=case["axis"]), torch.from_numpy(arr[f"{k}_r"]), f"iswt {case}")
        close(wt.iswt([t.cuda() for t in want], wav, axis=case["axis"]), torch.from_numpy(arr[f"{k}_r"]),
              f"iswt of the reference coefficients {case}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n, wavelet, level", [
    (1 << 20, "db4", 8),            # one halo group over many chunks
    ((1 << 20) + 6, "db2", 6),      # levels past swt_max_level: rows of 2 samples, dilations that do not divide n
    (3 << 16, "db8", 10),           # halo group, then whole residue classes of a non-power-of-two length
    (65536, "haar", None),          # 16 levels: halo group, then whole columns
    (4096, "sym5", 6),              # one signal per CTA
    (12288, "db3", 5),              # exactly one float32 tile of whole columns
    (12289, "db3", 3),              # odd length past the tile: halo chunks of one-sample rows
    (6 * 1024, "db10", 7),          # generic filter length (no unrolled instantiation)
    (100000, "db4", 4),             # the last chunk is partial
])
def test_parity_with_the_port_across_tile_structures(dtype, n, wavelet, level):
    g = torch.Generator().manual_seed(n % 997)
    batch = 3 if n < (1 << 19) else 2
    x = torch.randn(batch, n, generator=g, dtype=torch.float64).to(dtype)
    c = wt.swt(x.cuda(), wavelet, level)
    want = P.swt(x, wavelet, level)        # on the CPU: cuDNN may run float32 convolutions in TF32
    close(c, want, f"swt n={n}")
    close(wt.iswt(c, wavelet), P.iswt(want, wavelet), f"iswt n={n}")


@pytest.mark.parametrize("n, wavelet, level", [(14, "db4", 3), (14, "db8", 5), (37, "db3", 4), (5, "sym5", 3),
                                               (24, "db4", 6), (1, "db2", 2)])
def test_non_periodic_levels_match_the_port(n, wavelet, level):
    x = torch.randn(4, n, dtype=torch.float64)
    c = wt.swt(x.cuda(), wavelet, level)
    want = P.swt(x, wavelet, level)
    close(c, want, "swt")
    close(wt.iswt(c, wavelet), P.iswt(want, wavelet), "iswt")


def test_cpu_tensors_and_non_contiguous_input():
    x = torch.randn(64, 5, dtype=torch.float64)
    c = wt.swt(x, "db3", 3, axis=0)
    assert all(t.device.type == "cpu" for t in c)
    close(c, P.swt(x, "db3", 3, axis=0), "cpu swt")
    y = wt.iswt(c, "db3", axis=0)
    assert y.device.type == "cpu"
    close(y, x, "cpu round trip")
    xs = torch.randn(3, 256, dtype=torch.float32, device="cuda")[:, ::2]
    close(wt.swt(xs, "db2", 4), P.swt(xs.cpu(), "db2", 4), "strided input")


def test_round_trip_and_zero_copy_views():
    x = torch.randn(8, 4096, dtype=torch.float64, device="cuda")
    c = wt.swt(x, "sym4", 5)
    base = c[0].untyped_storage().data_ptr()
    assert all(t.untyped_storage().data_ptr() == base for t in c)
    assert all(t.data_ptr() % 16 == 0 for t in c[0].unbind(0))
    close(wt.iswt(c, "sym4"), x, "round trip")


def test_gradcheck_small_shapes():
    for n, wavelet, level in ((16, "db2", 2), (14, "db4", 3), (12, "haar", 2)):
        x = torch.randn(2, n, dtype=torch.float64, device="cuda", requires_grad=True)
        assert torch.autograd.gradcheck(lambda t: tuple(wt.swt(t, wavelet, level)), (x,))
        cs = [t.detach().requires_grad_(True) for t in wt.swt(x.detach(), wavelet, level)]
        assert torch.autograd.gradcheck(lambda *ts: wt.iswt(list(ts), wavelet), tuple(cs))


def test_gradients_match_the_reference_and_the_port(swt_golden):
    man, arr = swt_golden
    for case in man["grads"]:
        k = case["key"]
        wav = wavelet_arg(case["wavelet"], torch.float64)
        x = torch.from_numpy(arr[f"{k}_x"]).cuda().requires_grad_(True)
        w = torch.from_numpy(arr[f"{k}_w"]).cuda()
        sum((wk * ck).sum() for wk, ck in zip(w, wt.swt(x, wav, case["level"]))).backward()
        close(x.grad, torch.from_numpy(arr[f"{k}_gx"]), f"swt grad {k}")
        cin = [t.detach().requires_grad_(True) for t in wt.swt(x.detach(), wav, case["level"])]
        (wt.iswt(cin, wav) * torch.from_numpy(arr[f"{k}_wy"]).cuda()).sum().backward()
        close([t.grad for t in cin], list(torch.from_numpy(arr[f"{k}_gc"])), f"iswt grad {k}")
    x = torch.randn(4, 65536, dtype=torch.float64)
    w = torch.randn(9, 4, 65536, dtype=torch.float64)
    xg, xp = x.cuda().requires_grad_(True), x.clone().requires_grad_(True)
    sum((a * b).sum() for a, b in zip(w.cuda(), wt.swt(xg, "db6", 8))).backward()
    sum((a * b).sum() for a, b in zip(w, P.swt(xp, "db6", 8))).backward()
    close(xg.grad, xp.grad, "large swt grad")


def test_learnable_taps_raise():
    bank = tuple(torch.nn.Parameter(t.clone()) for t in custom_bank(torch.float64))
    x = torch.randn(2, 32, dtype=torch.float64, device="cuda")
    with pytest.raises(NotImplementedError):
        wt.swt(x, bank, 2)
    c = wt.swt(x, tuple(t.detach() for t in bank), 2)
    with pytest.raises(NotImplementedError):
        wt.iswt(c, bank)


def test_levels_are_fused_into_fewer_launches():
    x = torch.randn(16, 1 << 20, device="cuda")
    _native.launch_count_reset()
    c = wt.swt(x, "db4", 8)
    fwd = _native.launch_count()
    _native.launch_count_reset()
    wt.iswt(c, "db4")
    inv = _native.launch_count()
    assert 1 <= fwd < 8 and 1 <= inv < 8, (fwd, inv)
    _native.launch_count_reset()
    wt.swt(torch.randn(256, 65536, dtype=torch.float64, device="cuda"), "haar")
    assert _native.launch_count() <= 3
