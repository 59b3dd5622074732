"""WaveletPacket3D on the H100 against the node-by-node float64 oracle (oracle/packets3d.py).

Every node, the reconstruction, the round trip, the number of transform calls and kernel launches per tree level,
lazy partial expansion, gradients and CPU inputs.  Tolerances are those of tests/conftest.py, relative to the largest
oracle value of the tree.
"""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL, assert_close_rel
from oracle import packets3d as O
from pytorch_wavelet_toolbox_b200 import _native
from pytorch_wavelet_toolbox_b200 import packets as packets_mod

SUBBANDS = O.SUBBANDS

# dtype, wavelet, mode, separable, shape, axes, maxlevel
CASES = [
    ("float32", "db2", "reflect", False, (2, 16, 18, 20), None, 2),
    ("float64", "db1", "zero", False, (3, 15, 17, 19), None, 2),
    ("float64", "db4", "constant", False, (2, 20, 21, 22), None, 2),
    ("float32", "db4", "periodic", False, (1, 24, 23, 25), None, 2),
    ("float64", "db2", "symmetric", False, (2, 13, 16, 11), None, 2),
    ("float32", "db1", "zero", False, (2, 17, 9, 12), None, 2),
    ("float32", "db2", "symmetric", True, (2, 14, 15, 16), None, 2),
    ("float64", "db4", "reflect", True, (1, 19, 20, 21), None, 2),
    ("float64", "db2", "boundary", False, (2, 16, 18, 20), None, 2),
    ("float64", "db1", "boundary", False, (2, 15, 9, 13), None, 2),
    ("float32", "db4", "boundary", True, (1, 32, 34, 36), None, 2),
    ("float32", "db4", "reflect", False, (2, 19, 3, 26, 24), (1, 3, 4), 2),
    ("float64", "db2", "zero", True, (13, 2, 14, 3, 15), (0, 2, 4), 2),
    ("float64", "db1", "boundary", False, (2, 12, 3, 10, 14), (-4, -1, -2), 2),
    ("float32", "db2", "reflect", False, (2, 32, 30, 34), None, 3),
]


def _ids(case):
    dtype, wav, mode, sep, shape, axes, lev = case
    return f"{dtype}-{wav}-{mode}{'-sep' if sep else ''}-{'x'.join(map(str, shape))}-{axes}-L{lev}"


def _input(shape, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64).to(getattr(torch, dtype))


def _kw(mode, sep, axes):
    kw = {"mode": mode, "separable": sep}
    if axes is not None:
        kw["axes"] = axes
    return kw


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_every_node_and_the_reconstruction_match_the_node_by_node_oracle(case):
    dtype, wav, mode, sep, shape, axes, lev = case
    x = _input(shape, dtype)
    kw = _kw(mode, sep, axes)
    want = O.packet_tree(x, wav, lev, **kw)
    wp = wt.WaveletPacket3D(x.cuda(), wav, maxlevel=lev, **kw)
    wp.initialize(wp.get_natural_order(lev))
    assert set(wp.keys()) == set(want.keys())
    scale = max(float(t.abs().max()) for t in want.values())
    for k, t in want.items():
        assert_close_rel(wp[k], t.to(x.dtype), scale=scale, what=f"node {k!r}")
    want_rec = O.reconstruct(want, wav, lev, **kw)
    rec = wp.reconstruct()[""]
    assert rec.is_cuda
    assert_close_rel(rec, want_rec.to(x.dtype), scale=scale, what="reconstruction")
    # the round trip returns the input (on odd extents the root comes back one sample longer, as in 2-D)
    sl = tuple(slice(0, n) for n in x.shape)
    assert_close_rel(rec[sl], x, scale=float(x.abs().max()), what="round trip")


class _Counter:
    """Counts the calls of one transform entry point the packet class uses."""

    def __init__(self, monkeypatch, owner, name):
        self.calls = 0
        fn = getattr(owner, name)

        def spy(*args, **kwargs):
            self.calls += 1
            return fn(*args, **kwargs)

        monkeypatch.setattr(owner, name, spy)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_fused_float32_path_is_one_call_and_one_launch_per_tree_level(monkeypatch, depth):
    dec = _Counter(monkeypatch, packets_mod, "wavedec3")
    rec = _Counter(monkeypatch, packets_mod, "waverec3")
    x = _input((2, 40, 36, 44), "float32").cuda()
    wp = wt.WaveletPacket3D(x, "db2", mode="reflect", maxlevel=depth)
    _native.launch_count_reset()
    wp.initialize(wp.get_natural_order(depth))
    torch.cuda.synchronize()
    assert (dec.calls, _native.launch_count()) == (depth, depth)      # node by node: 1 + 8 + ... + 8^(depth-1)
    assert len(wp) == 1 + sum(8 ** j for j in range(1, depth + 1))
    _native.launch_count_reset()
    out = wp.reconstruct()[""]
    torch.cuda.synchronize()
    assert (rec.calls, _native.launch_count()) == (depth, depth)
    assert float((out - x).abs().max()) <= 2 * TOL[torch.float32] * float(x.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("mode,separable,dtype", [("zero", False, "float64"), ("periodic", True, "float32"),
                                                  ("boundary", False, "float64")])
def test_one_transform_call_per_tree_level_on_every_path(monkeypatch, mode, separable, dtype):
    if mode == "boundary":
        dec = _Counter(monkeypatch, packets_mod.MatrixWavedec3, "__call__")
        rec = _Counter(monkeypatch, packets_mod.MatrixWaverec3, "__call__")
    elif separable:
        dec = _Counter(monkeypatch, packets_mod, "fswavedec3")
        rec = _Counter(monkeypatch, packets_mod, "fswaverec3")
    else:
        dec = _Counter(monkeypatch, packets_mod, "wavedec3")
        rec = _Counter(monkeypatch, packets_mod, "waverec3")
    x = _input((2, 24, 20, 22), dtype).cuda()
    wp = wt.WaveletPacket3D(x, "db2", mode=mode, separable=separable, maxlevel=2)
    wp.initialize(wp.get_natural_order(2))
    assert dec.calls == 2
    wp.reconstruct()
    assert rec.calls == 2
    if separable:
        # fswavedec3 is the fused pyramid in the separable container: still one launch per level on float32
        _native.launch_count_reset()
        wt.WaveletPacket3D(x, "db2", mode=mode, separable=True, maxlevel=2).initialize(wp.get_natural_order(2))
        torch.cuda.synchronize()
        assert _native.launch_count() == 2


def _walk_nodes(keys):
    """The nodes a node-by-node walk creates for the requested keys: every child of every proper prefix."""
    made = {""}
    for k in keys:
        for j in range(0, len(k), 3):
            made.update(k[:j] + c for c in SUBBANDS)
    return made


@pytest.mark.gpu
def test_partial_initialize_creates_exactly_the_nodes_of_a_node_by_node_walk(monkeypatch):
    dec = _Counter(monkeypatch, packets_mod, "wavedec3")
    x = _input((2, 32, 28, 30), "float64")
    want = O.packet_tree(x, "db2", 3, mode="reflect")
    wp = wt.WaveletPacket3D(x.cuda(), "db2", mode="reflect", maxlevel=3)
    keys = ["aadddaaaa", "aad", "dddada", "aadadd"]
    wp.initialize(keys)
    assert set(wp.keys()) == _walk_nodes(keys)
    assert "aaa" in wp and "aadaaa" in wp and "adaaaa" not in wp and "dddaaaaaa" not in wp
    assert dec.calls == 3                                     # one call per tree level, however many parents
    scale = max(float(t.abs().max()) for t in want.values())
    for k in wp.keys():
        assert_close_rel(wp[k], want[k], scale=scale, what=f"node {k!r}")
    calls = dec.calls
    wp["daddddaad"]                                           # one more branch: two calls, one per missing level
    assert dec.calls == calls + 2
    assert set(wp.keys()) == _walk_nodes(keys + ["daddddaad"])
    wp.initialize(keys)                                       # nothing left to expand
    assert dec.calls == calls + 2


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["reflect", "zero"])
def test_gradients_of_the_depth_two_nodes_and_of_the_reconstruction_match_the_oracle(mode):
    shape = (2, 13, 12, 14)
    x = _input(shape, "float64")
    keys = wt.WaveletPacket3D.get_natural_order(2)
    tree = O.packet_tree(x, "db2", 2, mode=mode)
    g = torch.Generator().manual_seed(1)
    weights = {k: torch.randn(tree[k].shape, generator=g, dtype=torch.float64) for k in keys}

    def loss_of(nodes, dev):
        return sum((nodes[k] * weights[k].to(dev)).sum() for k in keys)

    xr = x.clone().requires_grad_(True)
    (want,) = torch.autograd.grad(loss_of(O.packet_tree(xr, "db2", 2, mode=mode), "cpu"), xr)
    xg = x.cuda().requires_grad_(True)
    wp = wt.WaveletPacket3D(xg, "db2", mode=mode, maxlevel=2)
    wp.initialize(keys)
    (got,) = torch.autograd.grad(loss_of(wp, "cuda"), xg)
    assert_close_rel(got, want, what=f"{mode}: gradient of the depth-2 nodes")

    # through reconstruct: the leaves are scaled first so the gradient is not the identity's
    w_rec = torch.randn((2, 14, 12, 14), generator=g, dtype=torch.float64)   # the root comes back one longer on 13
    xr = x.clone().requires_grad_(True)
    t = O.packet_tree(xr, "db2", 2, mode=mode)
    t = {k: (v * 1.5 if k == "aaaaad" else v) for k, v in t.items()}
    (want,) = torch.autograd.grad((O.reconstruct(t, "db2", 2, mode=mode) * w_rec).sum(), xr)
    xg = x.cuda().requires_grad_(True)
    wp = wt.WaveletPacket3D(xg, "db2", mode=mode, maxlevel=2)
    wp.initialize(keys)
    wp["aaaaad"] = wp["aaaaad"] * 1.5
    (got,) = torch.autograd.grad((wp.reconstruct()[""] * w_rec.cuda()).sum(), xg)
    assert_close_rel(got, want, what=f"{mode}: gradient through reconstruct")


@pytest.mark.gpu
def test_boundary_mode_under_grad_raises_the_matrix_path_error():
    x = _input((1, 16, 16, 16), "float64").cuda().requires_grad_(True)
    wp = wt.WaveletPacket3D(x, "db2", mode="boundary", maxlevel=1)
    with pytest.raises(NotImplementedError, match="matrix"):
        wp["aad"]
    with torch.no_grad():
        assert wp["aad"].shape == (1, 8, 8, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["reflect", "boundary"])
def test_cpu_input_comes_back_on_the_cpu(mode):
    x = _input((2, 12, 14, 10), "float32")
    wp = wt.WaveletPacket3D(x, "db2", mode=mode, maxlevel=2)
    wp.initialize(wp.get_natural_order(2))
    want = O.packet_tree(x, "db2", 2, mode=mode)
    scale = max(float(t.abs().max()) for t in want.values())
    for k in want:
        assert wp[k].device.type == "cpu", k
        assert_close_rel(wp[k], want[k].float(), scale=scale, what=f"node {k!r}")
    rec = wp.reconstruct()[""]
    assert rec.device.type == "cpu"
    assert_close_rel(rec[:, :12, :14, :10], x, scale=float(x.abs().max()), what="round trip")
