"""The kernels at the launch geometries that training-size batches select, every batch item against the float64 oracle.

The host code picks most launch geometries from the batch size, the extents and the SM count: row segments per strip
and chunks per segment (2-D strips), planes per CTA (3-D tiles), chunks per CTA (fused matrix analysis), grid-stride
iterations (general per-axis and swt level kernels), the two-stream batch chunks of the 2-D analysis and the cluster
size of the levels-1-2 kernel.  Each case here targets one regime of those rules, reads the grid the profiler recorded
(``args["grid"]`` of the chrome trace), derives the regime from it and asserts that the case reached it, so a retuned
heuristic that moves a case fails here by name instead of quietly testing the easy end.

Every item of every batch is checked: item b is ``p_b * u + q_b * v`` (tests/launch_geometry.py), the oracle
(oracle/ptwt_port.py, swt_port.py) runs on ``u`` and ``v`` only, and item b must match ``p_b C(u) + q_b C(v)`` to
``TOL[dtype] * (|p_b| max|C(u)| + |q_b| max|C(v)|)``, the maxima taken over the coefficient tree.  Synthesis cases
feed ``p_b a + q_b b`` for random coefficient trees ``a``, ``b`` and check the reconstruction the same way.
"""
from __future__ import annotations

import gc
import math
import os
import tempfile
import time

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import pytorch_wavelet_toolbox_b200 as wt
from conftest import TOL, flatten_coeffs
from launch_geometry import coeff_len, combine, item_errors, load_trace, pairs, quantised
from oracle import ptwt_port as P
from oracle import swt_port as SP
from pytorch_wavelet_toolbox_b200 import _native
from test_gpu_kernel_inventory import _map_tree, _operators_built_in, _place

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
TNAME = {F32: "float", F64: "double"}


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def traced(fn):
    """(fn(), the kernels it launched as launch_geometry.Launch records, in launch order)."""
    for attempt in range(2):
        torch.cuda.synchronize()
        before = _native.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.005 * (1 + 10 * attempt))
            out = fn()
            torch.cuda.synchronize()
            time.sleep(0.005 * (1 + 10 * attempt))
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            launches = load_trace(path)
        if launches or _native.launch_count() == before:
            return out, launches
    return out, launches


def of(launches, prefix):
    """The launches whose kernel name starts with prefix, with a message listing all names when there are none."""
    got = [k for k in launches if k.name.startswith(prefix)]
    assert got, f"{prefix} was not launched; launched: {sorted({k.name for k in launches})}"
    return got


def cdiv(a, b):
    return -(-a // b)


# ---- oracle runs on u and v, cached per module ----------------------------------------------------------------------
_ORACLE: dict = {}


def oracle_uv(item_shape, seed, fn, *args, **kwargs):
    """(u, v, C(u), C(v), C([u, v])): u, v quantised float64 of item_shape from seed, C = fn(., *args, **kwargs) run
    once on the batch [u, v].  Cached under the oracle call itself: function, arguments, shape and seed."""
    key = (fn.__module__, fn.__qualname__, args, tuple(sorted(kwargs.items())), tuple(item_shape), seed)
    if key not in _ORACLE:
        g = torch.Generator().manual_seed(seed)
        uv = quantised((2,) + tuple(item_shape), g)
        tree = fn(uv, *args, **kwargs)
        flat = flatten_coeffs(tree)
        _ORACLE[key] = (uv[0], uv[1], [t[0] for t in flat], [t[1] for t in flat], tree)
    return _ORACLE[key]


def random_tree_uv(tree2, seed, fn, *args):
    """(a2, R(a), R(b)): a2 a tree of quantised random coefficients with the shapes of tree2 (batch of 2: a and b),
    R = the oracle's synthesis fn(., *args), run once on a2.  tree2 is a cached oracle_uv tree, so its id is unique
    for the module's lifetime."""
    key = ("synthesis", id(tree2), seed, fn.__module__, fn.__qualname__, args)
    if key not in _ORACLE:
        g = torch.Generator().manual_seed(seed)
        a2 = _map_tree(tree2, lambda t: quantised(t.shape, g))
        y = fn(a2, *args)
        _ORACLE[key] = (a2, y[0], y[1])
    return _ORACLE[key]


def check_items(got, cu, cv, pq, dtype, what):
    flat = flatten_coeffs(got) if not isinstance(got, torch.Tensor) else [got]
    for j, t in enumerate(flat):
        assert t.dtype == dtype, f"{what} tensor {j}: dtype {t.dtype}"
    err, scale = item_errors(flat, cu, cv, pq)
    tol = TOL[dtype] * scale
    bad = (err > tol).nonzero().flatten().tolist()
    assert not bad, (f"{what}: {len(bad)} of {len(pq)} items off, first items {bad[:8]}: max abs err "
                     f"{[f'{float(err[i]):.3e}' for i in bad[:8]]} > tol {[f'{float(tol[i]):.3e}' for i in bad[:8]]}")


def batch_of(u, v, pq, dtype, layout="packed"):
    x = combine(u.to(DEV, dtype), v.to(DEV, dtype), pq, dtype)
    return x if layout == "packed" else _place(x, layout)


def coefficient_batch(a2, pq, dtype, layout):
    """The tree a2 (batch [a, b]) as a batch of p_b a + q_b b on the device, each tensor in `layout`."""
    return _map_tree(a2, lambda t: batch_of(t[0], t[1], pq, dtype, layout))


# ---- 2-D analysis strips: fwd2d_strip_f32_kernel / fwd2d_strip_kernel<double> ---------------------------------------
def _strip_name(dtype, L):
    return f"fwd2d_strip_f32_kernel<{L}, 64," if dtype == F32 else f"fwd2d_strip_kernel<double, {L}, 32,"


def _strip_width(name):
    return int(name.split("<")[1].split(",")[2 if name.startswith("fwd2d_strip_kernel") else 1])


def _strip_segments(Mh, nseg, step=16, lead=3):
    """Segment lengths that cut Mh rows into nseg segments.  The 2-D analysis kernel works a segment in chunks of
    16 rows with HALO / 2 = 3 rows of lead-in (db4), so its segments are 16 k - 3 rows; the synthesis kernel's are
    32 k - 2 (L / 2 - 1) = 32 k - 6 rows (db4)."""
    return [s for s in range(step - lead, Mh + step, step) if cdiv(Mh, s) == nseg]


@pytest.mark.parametrize("dtype,B,regime", [(F32, 96, "long"), (F32, 2, "short"), (F64, 48, "long"), (F64, 2, "short")],
                         ids=["f32-long", "f32-short", "f64-long", "f64-short"])
def test_fwd2d_strip_segments(dtype, B, regime):
    """1024^2 db4 level 3: level 1 in segments of >= 10 chunks of 16 rows (training batches) or <= 4 (two images)."""
    u, v, cu, cv, _ = oracle_uv((1024, 1024), 11, P.wavedec2, "db4", mode="reflect", level=3)
    pq = pairs(B)
    x = batch_of(u, v, pq, dtype)
    got, launches = traced(lambda: wt.wavedec2(x, "db4", mode="reflect", level=3))
    check_items(got, cu, cv, pq, dtype, f"wavedec2 {dtype} B={B}")
    ks = of(launches, _strip_name(dtype, 8))
    assert len(ks) == 3, [k.name for k in ks]
    k1 = ks[0]                                            # level 1
    Mh, Mw = got[-1][0].shape[-2:]
    TW = _strip_width(k1.name)
    assert k1.grid[0] == cdiv(Mw, TW) and k1.grid[2] == B, (k1.grid, Mh, Mw)
    chunks = {(s + 3) // 16 for s in _strip_segments(Mh, k1.grid[1])}
    msg = f"{k1.grid[1]} segments of {Mh} rows, {chunks} chunks of 16 rows per segment"
    if regime == "long":
        assert chunks and min(chunks) >= 10, f"long-segment regime not reached: {msg}"
    else:
        assert chunks and max(chunks) <= 4, f"short-segment regime not reached: {msg}"


_RAGGED = {F32: (55, (449, 511, 512)), F64: (29, (449, 479, 480))}


@pytest.mark.parametrize("last", ["1", "TW-1", "TW"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_fwd2d_strip_ragged_edges(dtype, last):
    """A last segment of one row, and a last strip of 1, TW - 1 or TW columns (db4, level 1, 306 output rows)."""
    B, widths = _RAGGED[dtype]
    Mw_want = widths[["1", "TW-1", "TW"].index(last)]
    H, W = 2 * (306 - 3), 2 * (Mw_want - 3)
    u, v, cu, cv, _ = oracle_uv((H, W), 12 + W, P.wavedec2, "db4", mode="symmetric", level=1)
    pq = pairs(B)
    x = batch_of(u, v, pq, dtype)
    got, launches = traced(lambda: wt.wavedec2(x, "db4", mode="symmetric", level=1))
    check_items(got, cu, cv, pq, dtype, f"wavedec2 {dtype} {H}x{W} B={B}")
    (k,) = of(launches, _strip_name(dtype, 8))
    Mh, Mw = got[-1][0].shape[-2:]
    assert (Mh, Mw) == (306, Mw_want)
    TW = _strip_width(k.name)
    nstrip, nseg = k.grid[0], k.grid[1]
    assert nstrip == cdiv(Mw, TW)
    cols = Mw - (nstrip - 1) * TW
    assert cols == {"1": 1, "TW-1": TW - 1, "TW": TW}[last], f"last strip has {cols} columns"
    lasts = {Mh - (nseg - 1) * s for s in _strip_segments(Mh, nseg)}
    assert lasts == {1}, f"ragged-segment regime not reached: {nseg} segments of {Mh} rows, last segment {lasts}"


# ---- 2-D synthesis strips: inv2d_strip_kernel<L, TMA> ---------------------------------------------------------------
@pytest.mark.parametrize("B,regime", [(96, "long"), (2, "short")])
@pytest.mark.parametrize("tma", [True, False], ids=["tma", "plain"])
def test_inv2d_strip_segments(tma, B, regime):
    """1024^2 db4 synthesis: the level writing the image in segments of >= 8 chunks of 32 rows, or <= 4.

    Rows padded to 16 elements stage through TMA (three levels).  A level whose approximation has rows of odd width
    (515) cannot; the library's own intermediate approximations are aligned, so that case runs one level."""
    level = 3 if tma else 1
    *_, tree2 = oracle_uv((1024, 1024), 11, P.wavedec2, "db4", mode="reflect", level=level)
    a2, ra, rb = random_tree_uv(tree2, 21, P.waverec2, "db4")
    pq = pairs(B)
    c = coefficient_batch(a2, pq, F32, "pitch16" if tma else "contiguous")
    y, launches = traced(lambda: wt.waverec2(c, "db4"))
    check_items(y, [ra], [rb], pq, F32, f"waverec2 B={B} tma={tma}")
    ks = of(launches, f"inv2d_strip_kernel<8, {str(tma).lower()}>")
    assert len(ks) == level, [k.name for k in ks]
    k1 = ks[-1]                                           # the level that writes the image
    OH, OW = y.shape[-2:]
    assert k1.grid[0] == cdiv(OW, 128) and k1.grid[2] == B, k1.grid
    chunks = {(s + 6) // 32 for s in _strip_segments(OH, k1.grid[1], 32, 6)}
    msg = f"{k1.grid[1]} segments of {OH} rows, {chunks} chunks of 32 rows per segment"
    if regime == "long":
        assert chunks and min(chunks) >= 8, f"long-segment regime not reached: {msg}"
    else:
        assert chunks and max(chunks) <= 4, f"short-segment regime not reached: {msg}"


# ---- 3-D tiles: fwd3d_tile_kernel / inv3d_tile_kernel ---------------------------------------------------------------
_TILES = ((16, 32), (11, 44), (8, 64))


def _oracle3():
    return oracle_uv((128, 128, 128), 31, P.wavedec3, "sym4", mode="zero", level=1)


@pytest.mark.parametrize("B,regime", [(88, "whole depth"), (2, "depth segments")])
@pytest.mark.parametrize("tile", [0, 1, 2])
def test_fwd3d_tile_depth(tile, B, regime):
    """128^3 sym4: 67 output planes, in one CTA per tile column for training batches, in segments of <= 24 for two."""
    u, v, cu, cv, _ = _oracle3()
    pq = pairs(B)
    x = batch_of(u, v, pq, F32)
    with _native.knobs(FWD3D_TILE=tile):
        got, launches = traced(lambda: wt.wavedec3(x, "sym4", mode="zero", level=1))
    del x
    check_items(got, cu, cv, pq, F32, f"wavedec3 tile {tile} B={B}")
    th, tw = _TILES[tile]
    (k,) = of(launches, f"fwd3d_tile_kernel<8, {th}, {tw},")
    Md, Mh, Mw = got[0].shape[-3:]
    nty = cdiv(Mh, th)
    assert k.grid[0] == cdiv(Mw, tw) and k.grid[1] % nty == 0 and k.grid[2] == B, k.grid
    nseg = k.grid[1] // nty
    planes = cdiv(Md, nseg)
    if regime == "whole depth":
        assert nseg == 1, f"whole-depth regime not reached: {Md} planes in {nseg} segments"
    else:
        assert planes <= 24, f"depth-segment regime not reached: {Md} planes in {nseg} segments"


@pytest.mark.parametrize("B,regime", [(88, "whole depth"), (2, "depth segments")])
def test_inv3d_tile_depth(B, regime):
    """128^3 sym4 synthesis: all 64 output plane pairs in one CTA per tile column, or segments of <= 16 pairs."""
    *_, tree2 = _oracle3()
    a2, ra, rb = random_tree_uv(tree2, 32, P.waverec3, "sym4")
    pq = pairs(B)
    c = coefficient_batch(a2, pq, F32, "pitch16")
    y, launches = traced(lambda: wt.waverec3(c, "sym4"))
    del c
    check_items(y, [ra], [rb], pq, F32, f"waverec3 B={B}")
    (k,) = of(launches, "inv3d_tile_kernel<8,")
    OD, OH, OW = y.shape[-3:]
    nty = cdiv(OH, 16)                                    # output tiles of 16 x 64 (inv3d.cuh)
    assert k.grid[0] == cdiv(OW, 64) and k.grid[1] % nty == 0 and k.grid[2] == B, k.grid
    nseg = k.grid[1] // nty
    if regime == "whole depth":
        assert nseg == 1, f"whole-depth regime not reached: {cdiv(OD, 2)} plane pairs in {nseg} segments"
    else:
        assert cdiv(cdiv(OD, 2), nseg) <= 16, f"depth-segment regime not reached: {OD} planes in {nseg} segments"


# ---- fused matrix analysis: mat_fwd_fused_kernel, chunks per CTA ----------------------------------------------------
def _mat_dec(t):
    return wt.MatrixWavedec("db4", 3, orthogonalization="gramschmidt")(t)


def _mat_ref(t):
    """The oracle's Gram-Schmidt analysis with boundary operators built in float32 and applied in float64."""
    with _operators_built_in(F32):
        return P.MatrixWavedec("db4", 3, orthogonalization="gramschmidt")(t)


_MAT_CHUNKS = {32768: 8, 49152: 12}


@pytest.mark.parametrize("n,B,cpc", [(32768, 528, 8), (32768, 264, 4), (32768, 132, 2), (32768, 66, 1), (49152, 264, 8)],
                         ids=["8-chunks-cpc8", "8-chunks-cpc4", "8-chunks-cpc2", "8-chunks-cpc1", "12-chunks-cpc8"])
def test_matrix_fused_chunks_per_cta(n, B, cpc):
    """float32 Gram-Schmidt, 3 levels in one fused launch: rows of 32768 (8 chunks) through CTAs that take 8, 4, 2 or 1
    chunks, and rows of 49152 (12 chunks) at 8 per CTA, whose second CTA starts at chunk 8 and stops at the row's end
    after 4."""
    u, v, cu, cv, _ = oracle_uv((n,), 41, _mat_ref)
    # chunks per row: the grid of a launch that takes one chunk per CTA
    with _native.knobs(MATF_CPC=1):
        _, one = traced(lambda: _mat_dec(batch_of(u, v, pairs(2), F32)))
    nchunks = of(one, "mat_fwd_fused_kernel<float,")[0].grid[0]
    assert nchunks == _MAT_CHUNKS[n], f"{nchunks} chunks per row of {n}: the cases below no longer tell cpc apart"
    pq = pairs(B)
    x = batch_of(u, v, pq, F32)
    got, launches = traced(lambda: _mat_dec(x))
    check_items(got, cu, cv, pq, F32, f"MatrixWavedec rows of {n}, B={B}")
    k = of(launches, "mat_fwd_fused_kernel<float,")[0]
    assert k.grid[1] == B, k.grid
    # chunks per CTA start at 8 and halve; with 8 or 12 chunks per row each choice gives its own grid
    seen = [c for c in (8, 4, 2, 1) if cdiv(nchunks, c) == k.grid[0]]
    last = nchunks - (k.grid[0] - 1) * cpc
    assert seen == [cpc], (f"regime of {cpc} chunks per CTA not reached: {nchunks} chunks per row in {k.grid[0]} CTAs "
                           f"fit {seen} chunks per CTA")
    if nchunks % cpc:
        assert 0 < last < cpc and k.grid[0] > 1, f"no CTA past the first is cut at the row's end: last takes {last}"


# ---- grid-stride loops: axis_fwd_kernel / axis_inv_kernel / swt_level_kernel ----------------------------------------
def _iterations(k, total):
    per_pass = k.grid[0] * k.grid[1] * k.grid[2] * k.block[0]
    return cdiv(total, per_pass), total % per_pass != 0


def test_axis_grid_stride_wavedec3_float64():
    """40 x 96^3 float64 db2: every thread of the first analysis pass and of the last synthesis pass runs several
    grid-stride iterations, the last one ragged."""
    B, n = 40, 96
    u, v, cu, cv, tree2 = oracle_uv((n, n, n), 51, P.wavedec3, "db2", mode="reflect", level=2)
    pq = pairs(B)
    x = batch_of(u, v, pq, F64)
    got, launches = traced(lambda: wt.wavedec3(x, "db2", mode="reflect", level=2))
    del x
    check_items(got, cu, cv, pq, F64, "wavedec3 float64")
    k = of(launches, "axis_fwd_kernel<double>")[0]
    m = coeff_len(n, 4)
    it, ragged = _iterations(k, B * n * n * m)           # the first pass filters one axis of the whole volume
    assert it >= 2 and ragged, f"grid-stride regime not reached: grid {k.grid}, {it} iterations, ragged {ragged}"
    del got
    a2, ra, rb = random_tree_uv(tree2, 52, P.waverec3, "db2")
    c = coefficient_batch(a2, pq, F64, "packed")
    y, launches = traced(lambda: wt.waverec3(c, "db2"))
    check_items(y, [ra], [rb], pq, F64, "waverec3 float64")
    k = of(launches, "axis_inv_kernel<double>")[-1]
    it, ragged = _iterations(k, y.numel())               # the last pass writes the whole output
    assert it >= 2 and ragged, f"grid-stride regime not reached: grid {k.grid}, {it} iterations, ragged {ragged}"


def test_axis_grid_stride_rows_float32():
    """2400 float32 rows of 4001 samples whose pitch is no multiple of 16 bytes, db3, one level, and the synthesis of
    odd-width coefficient rows: several grid-stride iterations, the last one ragged."""
    R, n = 2400, 4001
    u, v, cu, cv, tree2 = oracle_uv((n,), 61, P.wavedec, "db3", mode="reflect", level=1)
    pq = pairs(R)
    x = batch_of(u, v, pq, F32, "pitch")
    got, launches = traced(lambda: wt.wavedec(x, "db3", mode="reflect", level=1))
    check_items(got, cu, cv, pq, F32, "wavedec float32 rows")
    k = of(launches, "axis_fwd_kernel<float>")[0]
    it, ragged = _iterations(k, R * got[0].shape[-1])
    assert it >= 2 and ragged, f"grid-stride regime not reached: grid {k.grid}, {it} iterations, ragged {ragged}"
    a2, ra, rb = random_tree_uv(tree2, 62, P.waverec, "db3")
    c = coefficient_batch(a2, pq, F32, "contiguous")
    assert c[0].shape[-1] % 2 == 1                       # rows of odd width: not 16-byte aligned
    y, launches = traced(lambda: wt.waverec(c, "db3"))
    check_items(y, [ra], [rb], pq, F32, "waverec float32 rows")
    k = of(launches, "axis_inv_kernel<float>")[-1]
    it, ragged = _iterations(k, y.numel())
    assert it >= 2, f"grid-stride regime not reached: grid {k.grid}, {it} iterations"


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_swt_level_grid_stride(dtype):
    """60000 rows of 14 samples, db4, 3 levels (a level's extension is longer than the row): swt_level_kernel threads
    run two grid-stride iterations, the second ragged, in both directions."""
    R, n = 60000, 14
    u, v, cu, cv, _ = oracle_uv((n,), 71, SP.swt, "db4", 3)
    pq = pairs(R)
    x = batch_of(u, v, pq, dtype)
    got, launches = traced(lambda: wt.swt(x, "db4", 3))
    check_items(got, cu, cv, pq, dtype, f"swt {dtype}")
    for k in of(launches, f"swt_level_kernel<{TNAME[dtype]}, false>"):
        it, ragged = _iterations(k, R * n)
        assert it >= 2 and ragged, f"grid-stride regime not reached: grid {k.grid}, {it} iterations, ragged {ragged}"
    ru, rv = [SP.iswt([t.unsqueeze(0) for t in c], "db4")[0] for c in (cu, cv)]
    y, launches = traced(lambda: wt.iswt(got, "db4"))
    check_items(y, [ru], [rv], pq, dtype, f"iswt {dtype}")
    for k in of(launches, f"swt_level_kernel<{TNAME[dtype]}, true>"):
        it, ragged = _iterations(k, R * n)
        assert it >= 2 and ragged, f"grid-stride regime not reached: grid {k.grid}, {it} iterations, ragged {ragged}"


# ---- the two-stream chunked 2-D analysis ----------------------------------------------------------------------------
def _level1_chunks(launches, prefix, Mw1, TW):
    """(images, stream) of every level-1 launch of the kernel prefix, in launch order."""
    return [(k.grid[2], k.stream) for k in of(launches, prefix) if k.grid[0] == cdiv(Mw1, TW)]


def test_two_stream_default_trigger_odd_batch():
    """129 x 1024^2 float32 (>= 2^27 samples): halves of 65 and 64 images on two streams, default switches."""
    B = 129
    u, v, cu, cv, _ = oracle_uv((1024, 1024), 11, P.wavedec2, "db4", mode="reflect", level=3)
    pq = pairs(B)
    x = batch_of(u, v, pq, F32)
    got, launches = traced(lambda: wt.wavedec2(x, "db4", mode="reflect", level=3))
    del x
    check_items(got, cu, cv, pq, F32, "wavedec2 129 images")
    chunks = _level1_chunks(launches, _strip_name(F32, 8), got[-1][0].shape[-1], 64)
    assert [c for c, _ in chunks] == [65, 64] and chunks[0][1] != chunks[1][1], \
        f"two-stream regime with uneven halves not reached: level-1 launches (images, stream) {chunks}"


def test_two_stream_forced_chunks_reuse_scratch():
    """CHUNK=5 over 16 images of 512^2: chunks 5, 5, 5, 1 alternating between two streams, so each stream reuses its
    scratch slots for the intermediate approximations."""
    B = 16
    u, v, cu, cv, _ = oracle_uv((512, 512), 81, P.wavedec2, "db4", mode="zero", level=3)
    pq = pairs(B)
    x = batch_of(u, v, pq, F32)
    with _native.knobs(CHUNK=5):
        got, launches = traced(lambda: wt.wavedec2(x, "db4", mode="zero", level=3))
    check_items(got, cu, cv, pq, F32, "wavedec2 CHUNK=5")
    chunks = _level1_chunks(launches, _strip_name(F32, 8), got[-1][0].shape[-1], 64)
    streams = [s for _, s in chunks]
    assert [c for c, _ in chunks] == [5, 5, 5, 1] and len(set(streams)) == 2 and \
        streams[0] == streams[2] != streams[1] == streams[3], \
        f"regime of 4 chunks on 2 streams not reached: level-1 launches (images, stream) {chunks}"


def test_two_stream_split_between_pair_and_strip_kernels():
    """CHUNK=8 over 9 images of 2^16 samples with WPAIR_MIN=2^16: the chunk of 8 images takes the levels-1-2 kernel,
    the chunk of one image (fewer than 8 images) the per-level strip kernel."""
    B, H, W = 9, 256, 256
    u, v, cu, cv, _ = oracle_uv((H, W), 91, P.wavedec2, "db4", mode="reflect", level=3)
    pq = pairs(B)
    x = batch_of(u, v, pq, F32)
    with _native.knobs(CHUNK=8, WPAIR_MIN=H * W):
        got, launches = traced(lambda: wt.wavedec2(x, "db4", mode="reflect", level=3))
    check_items(got, cu, cv, pq, F32, "wavedec2 CHUNK=8 WPAIR_MIN=2^16")
    pair = [(k.grid[1], k.stream) for k in of(launches, "fwd2d_wpair_kernel<8,")]
    strip = _level1_chunks(launches, _strip_name(F32, 8), got[-1][0].shape[-1], 64)
    assert [c for c, _ in pair] == [8] and [c for c, _ in strip] == [1] and pair[0][1] != strip[0][1], \
        f"split regime not reached: levels-1-2 launches (images, stream) {pair}, strip launches {strip}"


# ---- fwd2d_wpair_kernel cluster sizes -------------------------------------------------------------------------------
# level-2 columns a strip owns: 128 level-1 columns less the 16-byte aligned left halo, halved (WPairGeom::TW2)
_TW2 = {2: 64, 4: 62, 6: 62, 8: 60}
_WPAIR = [("haar", 2, None, "fwd2d_wpair_kernel<2, 3, 12>"), ("db2", 4, None, "fwd2d_wpair_kernel<4, 3, 12>"),
          ("db3", 6, None, "fwd2d_wpair_kernel<6, 3, 12>"), ("db4", 8, None, "fwd2d_wpair_kernel<8, 2, 12>"),
          ("db4", 8, 1, "fwd2d_wpair_kernel<8, 2, 15>"), ("db4", 8, 3, "fwd2d_wpair_kernel<8, 3, 12>")]
# strip counts for clusters of 6 (two clusters), 3 (three), 2 (two) and 1
_NSTRIP = {6: 12, 3: 9, 2: 4, 1: 7}


def _width_for(Mw2, L):
    """The smallest width whose level-2 coefficients are Mw2 wide among those whose rows are a multiple of 16 bytes
    (the kernel stages its input through TMA)."""
    W = 4
    while coeff_len(coeff_len(W, L), L) < Mw2:
        W += 4
    assert coeff_len(coeff_len(W, L), L) == Mw2
    return W


@pytest.mark.parametrize("cluster", [6, 3, 2, 1])
@pytest.mark.parametrize("wav,L,var,name", _WPAIR, ids=[w[3] for w in _WPAIR])
def test_wpair_cluster_sizes(wav, L, var, name, cluster):
    """Each levels-1-2 kernel instantiation at strip counts whose largest divisor among 6, 3, 2 is the cluster size."""
    nstrip = _NSTRIP[cluster]
    Mw2 = nstrip * _TW2[L] - 5                           # a ragged last strip
    H, W, B = 72, _width_for(Mw2, L), 3
    u, v, cu, cv, _ = oracle_uv((H, W), 100 + W + L, P.wavedec2, wav, mode="reflect", level=2)
    pq = pairs(B)
    x = batch_of(u, v, pq, F32)
    knobs = {"WPAIR": 1, "WPAIR_MIN": 1}
    if var is not None:
        knobs["WPAIR_VAR"] = var
    with _native.knobs(**knobs):
        got, launches = traced(lambda: wt.wavedec2(x, wav, mode="reflect", level=2))
    check_items(got, cu, cv, pq, F32, f"wavedec2 {wav} {name} width {W}")
    (k,) = of(launches, name)
    assert k.grid[1] == B and got[1][0].shape[-1] == Mw2, (k.grid, got[1][0].shape)
    # clusters of adjacent strips: the largest of 6, 3, 2 that divides the strip count
    seen = next(c for c in (6, 3, 2, 1) if k.grid[0] % c == 0)
    assert seen == cluster, f"cluster-of-{cluster} regime not reached: {k.grid[0]} strips give clusters of {seen}"
    assert math.gcd(k.grid[0], 6) == {6: 6, 3: 3, 2: 2, 1: 1}[cluster]
