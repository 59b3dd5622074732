"""Padded multi-level fast wavelet transform in 1, 2 and 3 dimensions on the H100.

Drop-in for ``ptwt.wavedec / waverec`` (``/root/reference/src/ptwt/conv_transform.py:69,146``),
``ptwt.wavedec2 / waverec2`` (``conv_transform_2.py:74,160``) and ``ptwt.wavedec3 / waverec3``
(``conv_transform_3.py:76,148``): same signatures, defaults, return containers and errors.
The reference's per-level ``F.pad -> conv*d(stride=2) -> split`` and
``stack -> conv_transpose*d -> crop`` bodies are replaced by ONE call into libwtb200
(``wt_dwt_fwd`` / ``wt_dwt_inv``, include/wtb200.h) that runs every level on the GPU with the
boundary extension evaluated inside the kernels (no padded copy, no stacked copy).

Host responsibilities kept here: argument validation, extents per level, output allocation
(one packed coefficient buffer per call), building the reference's containers from views.
CPU tensors are staged to the current CUDA device and the results are copied back, so the
call is a drop-in for CPU callers too; there is no CPU compute path.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
from dataclasses import dataclass, field
from typing import Any, Optional, Sequence, Union

import torch

from . import _native as N
from ._shape import (
    AxisHint,
    Fold,
    check_dtype,
    check_mode,
    check_pad_feasible,
    check_tensor,
    ensure_axes,
    fold,
    round_up,
    unfold,
)
from ._wavelets import any_requires_grad, as_wavelet, dwt_max_level, dwtn_max_level, filter_bank, taps_in_dtype
from .constants import DETAIL_KEYS_3D, WaveletDetailTuple2d

__all__ = ["wavedec", "waverec", "wavedec2", "waverec2", "wavedec3", "waverec3"]

#: byte alignment of every coefficient row / band start in the packed output buffer.
ROW_ALIGN_BYTES = 16
BAND_ALIGN_BYTES = 128


# --------------------------------------------------------------------------------------
# device plumbing
# --------------------------------------------------------------------------------------
def _compute_device(t: torch.Tensor) -> torch.device:
    if t.is_cuda:
        return t.device
    if t.device.type != "cpu":
        raise RuntimeError(f"unsupported device {t.device}; expected a CUDA or CPU tensor")
    if not torch.cuda.is_available():
        raise RuntimeError(
            "pytorch_wavelet_toolbox_b200 needs a CUDA device (H100, sm_90a): the transforms have "
            "no CPU implementation. Got a CPU tensor and torch.cuda.is_available() is False."
        )
    return torch.device("cuda", torch.cuda.current_device())


def _dtype_code(dt: torch.dtype) -> int:
    return N.WT_F32 if dt == torch.float32 else N.WT_F64


def _no_autograd(*tensors: torch.Tensor, wavelet: Any = None) -> None:
    if torch.is_grad_enabled() and (
        any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors) or any_requires_grad(wavelet)
    ):
        raise NotImplementedError(
            "gradients are implemented for the data path of wavedec/waverec, wavedec2/waverec2 and "
            "wavedec3/waverec3 only (not for learnable filter taps, not through the matrix transforms); "
            "call under torch.no_grad() or detach the inputs."
        )


# --------------------------------------------------------------------------------------
# extents and packed layout
# --------------------------------------------------------------------------------------
@dataclass
class _Level:
    dims: tuple[int, ...]          # coefficient extents of this level
    pitch: int                     # row pitch in elements (>= dims[-1])
    plane: int                     # elements reserved per band
    strides: tuple[int, ...]       # element strides inside a band
    det_off: int = 0               # offset of band 1 inside one batch item of the packed buffer


@dataclass
class _Plan:
    ndim: int
    filt_len: int
    in_dims: tuple[int, ...]
    levels: list[_Level] = field(default_factory=list)   # finest first
    approx_off: int = 0
    item_elems: int = 0
    itemsize: int = 4
    dims_c: Any = None           # (array, pointer) of in_dims as int64, built once
    levels_c: Any = None         # (bytes of the wt_level[] template, per-level offsets), built on first use

    @property
    def nbands(self) -> int:
        return 1 << self.ndim


def _band_strides(dims: Sequence[int], pitch: int) -> tuple[int, ...]:
    st = [1] * len(dims)
    acc = pitch
    for a in range(len(dims) - 2, -1, -1):
        st[a] = acc
        acc *= dims[a]
    return tuple(st)


def _make_plan(in_dims: Sequence[int], filt_len: int, levels: int, itemsize: int) -> _Plan:
    """Cached: the layout depends only on (extents, filter length, level count, element size)."""
    return _make_plan_cached(tuple(int(d) for d in in_dims), int(filt_len), int(levels), int(itemsize))


@functools.lru_cache(maxsize=512)
def _make_plan_cached(in_dims: tuple, filt_len: int, levels: int, itemsize: int) -> _Plan:
    ndim = len(in_dims)
    plan = _Plan(ndim, filt_len, tuple(int(d) for d in in_dims))
    row_al = max(ROW_ALIGN_BYTES // itemsize, 1)
    band_al = max(BAND_ALIGN_BYTES // itemsize, 1)
    cur = plan.in_dims
    for _ in range(levels):
        cur = tuple(N.coeff_len(n, filt_len) for n in cur)
        pitch = round_up(cur[-1], row_al)
        rows = math.prod(cur[:-1]) if ndim > 1 else 1
        plane = round_up(rows * pitch, band_al)
        plan.levels.append(_Level(cur, pitch, plane, _band_strides(cur, pitch)))
    # packed item: [cA_n | details_n | ... | details_1]
    off = plan.levels[-1].plane if levels else 0
    plan.approx_off = 0
    for lv in reversed(plan.levels):
        lv.det_off = off
        off += (plan.nbands - 1) * lv.plane
    plan.item_elems = off
    plan.itemsize = itemsize
    plan.dims_c = N.i64_array(plan.in_dims)
    return plan


@functools.lru_cache(maxsize=1024)
def _pads_ok(dims: tuple, filt_len: int, level: int, mode: str, itemsize: int):
    """None when every level can be padded in this mode, else the exception the reference's F.pad raises."""
    plan = _make_plan_cached(dims, filt_len, level, itemsize)
    cur = dims
    try:
        for lv in plan.levels:
            check_pad_feasible(mode, cur, filt_len)
            cur = lv.dims
    except RuntimeError as ex:
        return str(ex)
    return None


def _check_pads(dims: tuple, filt_len: int, level: int, mode: str, plan: "_Plan") -> None:
    msg = _pads_ok(dims, filt_len, level, mode, plan.itemsize)
    if msg is not None:
        raise RuntimeError(msg)


def _view_band(buf: torch.Tensor, off: int, lv: _Level) -> torch.Tensor:
    """View of one band [batch, *dims] inside the packed buffer [batch, item_elems]."""
    b = buf.shape[0]
    return buf.as_strided((b,) + lv.dims, (buf.stride(0),) + lv.strides, buf.storage_offset() + off)


def _view_details(buf: torch.Tensor, lv: _Level, nbands: int) -> list[torch.Tensor]:
    """The detail bands k = 1 .. nbands-1 of one level as views [batch, *dims]: one strided view
    [batch, nbands-1, *dims] split along the band axis (two dispatcher calls instead of nbands-1)."""
    if nbands == 2:
        return [_view_band(buf, lv.det_off, lv)]
    b = buf.shape[0]
    allb = buf.as_strided((b, nbands - 1) + lv.dims, (buf.stride(0), lv.plane) + lv.strides, buf.storage_offset() + lv.det_off)
    return list(allb.unbind(1))


def _result_views(buf: torch.Tensor, plan: "_Plan"):
    approx = _view_band(buf, plan.approx_off, plan.levels[-1])
    details = [_view_details(buf, lv, plan.nbands) for lv in reversed(plan.levels)]
    return approx, details


# --------------------------------------------------------------------------------------
# analysis
# --------------------------------------------------------------------------------------
def _analysis(data: torch.Tensor, wavelet: Any, mode: Optional[str], level: Optional[int], axes: AxisHint,
              ndim: int):
    """Returns (approx [B,*], [per level coarsest-first: list of bands k=1..], Fold)."""
    check_tensor(data)
    check_dtype(data)
    x, f = fold(data, ndim, axes)
    wav = as_wavelet(wavelet)
    dec_lo, dec_hi, _, _ = filter_bank(wav)
    filt_len = len(dec_lo)
    dims = tuple(int(d) for d in x.shape[1:])
    if level is None:
        level = dwt_max_level(dims[0], filt_len) if ndim == 1 else dwtn_max_level(dims, filt_len)
    if level <= 0:
        return x, [], f
    mode = check_mode(mode)
    if len(dec_hi) != filt_len:
        raise ValueError("dec_lo and dec_hi must have the same length")
    if filt_len < 2 or filt_len > N.WT_MAX_FILT_LEN:
        raise ValueError(f"filter length {filt_len} not supported (2..{N.WT_MAX_FILT_LEN})")
    plan = _make_plan(dims, filt_len, level, x.element_size())
    _check_pads(dims, filt_len, level, mode, plan)
    if torch.is_grad_enabled() and (x.requires_grad or any_requires_grad(wav)):
        from ._autograd import analysis_with_grad

        approx, details = analysis_with_grad(x, dec_lo, dec_hi, mode, level, ndim, _compute_device(x))
        return approx, details, f

    dev = _compute_device(x)
    on_host = not x.is_cuda
    batch = x.shape[0]
    if on_host and batch > 1 and x[0].numel() * x.element_size() * batch >= HOST_PIPELINE_MIN_BYTES:
        buf = _analysis_host_pipeline(x, plan, mode, dec_lo, dec_hi, dev)
        approx, details = _result_views(buf, plan)
        return approx, details, f
    with torch.cuda.device(dev):
        xd = x.to(dev, non_blocking=True) if on_host else x
        if xd.stride(-1) != 1 and xd.shape[-1] != 1:
            xd = xd.contiguous()
        if batch > 0 and any(s < 0 for s in xd.stride()):
            xd = xd.contiguous()
        buf = torch.empty((batch, plan.item_elems), dtype=x.dtype, device=dev)
        scratch_elems = sum(lv.plane for lv in plan.levels[:-1])
        scratch = torch.empty((batch, max(scratch_elems, 1)), dtype=x.dtype, device=dev)
        _run_fwd(xd, plan, mode, dec_lo, dec_hi, buf, scratch)
        if on_host:
            host = pinned_empty(buf.shape, buf.dtype)
            host.copy_(buf, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            buf = host
    approx, details = _result_views(buf, plan)
    return approx, details, f


# --------------------------------------------------------------------------------------
# host staging: CPU tensors in -> pinned result out
# --------------------------------------------------------------------------------------
_host_reuse = False
_host_cache: dict = {}


class host_staging:
    """``with host_staging(reuse=True): ...`` -- results of transforms of CPU tensors are written into ONE pinned host
    buffer per (shape, dtype) that is REUSED by the next call of the same shape (page-locking 4 GB per call costs more
    than the transform).  The tensors returned by a call are then only valid until the next call of that shape; the
    default (``reuse=False``) gives every call a fresh pinned buffer like round 1.  The cache is dropped on exit."""

    def __init__(self, reuse: bool = True):
        self.reuse = reuse

    def __enter__(self):
        global _host_reuse
        self._old = _host_reuse
        _host_reuse = self.reuse
        return self

    def __exit__(self, *exc):
        global _host_reuse
        _host_reuse = self._old
        if not _host_reuse:
            _host_cache.clear()
        return False


def pinned_empty(shape, dtype: torch.dtype) -> torch.Tensor:
    """Pinned host buffer for a result (fresh, or the cached one inside ``host_staging(reuse=True)``)."""
    if not _host_reuse:
        return torch.empty(shape, dtype=dtype, pin_memory=True)
    key = (tuple(shape), dtype)
    buf = _host_cache.get(key)
    if buf is None:
        buf = _host_cache[key] = torch.empty(shape, dtype=dtype, pin_memory=True)
    return buf


#: host inputs at least this large are transformed through the chunked copy/compute/copy pipeline
HOST_PIPELINE_MIN_BYTES = 64 << 20
#: bytes of input per pipeline chunk (PCIe transfers of this size run at full rate)
HOST_PIPELINE_CHUNK_BYTES = 256 << 20
#: smallest chunk the pipeline cuts mid-size inputs into
HOST_PIPELINE_MIN_CHUNK_BYTES = 32 << 20
_pipe_streams: dict = {}


def _analysis_host_pipeline(x: torch.Tensor, plan: _Plan, mode: str, dec_lo, dec_hi, dev: torch.device) -> torch.Tensor:
    """Host tensor in, packed host buffer out, with H2D / transform / D2H of consecutive batch chunks
    overlapped on three streams (PCIe is full duplex, so the copies in both directions run
    concurrently; the transform itself is ~2 % of the time).  Double-buffered device staging."""
    batch = x.shape[0]
    item_bytes = x[0].numel() * x.element_size()
    # chunk: 256 MB for large inputs (PCIe transfers of this size run at full rate), at least ~8 chunks for mid-size
    # inputs so that the copy-in of chunk k+1, the transform of chunk k and the copy-out of chunk k-1 really overlap
    # (with 2-3 chunks the pipeline is mostly fill and drain: BASELINE config 3, 537 MB, 16.5 ms vs 10.7 ms of copies)
    chunk_bytes = min(HOST_PIPELINE_CHUNK_BYTES, max(HOST_PIPELINE_MIN_CHUNK_BYTES, item_bytes * batch // 8))
    bc = max(1, min(batch, chunk_bytes // max(item_bytes, 1)))
    with torch.cuda.device(dev):
        if dev not in _pipe_streams:
            _pipe_streams[dev] = tuple(torch.cuda.Stream(device=dev) for _ in range(3))
        s_in, s_cmp, s_out = _pipe_streams[dev]
        xs = x if x.is_contiguous() else x.contiguous()
        host = pinned_empty((batch, plan.item_elems), x.dtype)
        d_in = [torch.empty((bc,) + tuple(x.shape[1:]), dtype=x.dtype, device=dev) for _ in range(2)]
        d_out = [torch.empty((bc, plan.item_elems), dtype=x.dtype, device=dev) for _ in range(2)]
        scratch = torch.empty((bc, max(sum(lv.plane for lv in plan.levels[:-1]), 1)), dtype=x.dtype, device=dev)
        cur = torch.cuda.current_stream(dev)
        for st in (s_in, s_cmp, s_out):
            st.wait_stream(cur)
        ev_cmp: list = []
        ev_out: list = []
        for i, lo in enumerate(range(0, batch, bc)):
            hi = min(lo + bc, batch)
            n, k = hi - lo, i % 2
            with torch.cuda.stream(s_in):
                if i >= 2:
                    s_in.wait_event(ev_cmp[i - 2])      # the transform that read d_in[k] is done
                d_in[k][:n].copy_(xs[lo:hi], non_blocking=True)
                e_in = torch.cuda.Event()
                e_in.record(s_in)
            with torch.cuda.stream(s_cmp):
                s_cmp.wait_event(e_in)
                if i >= 2:
                    s_cmp.wait_event(ev_out[i - 2])     # the copy-out that read d_out[k] is done
                _run_fwd(d_in[k][:n], plan, mode, dec_lo, dec_hi, d_out[k][:n], scratch[:n])
                e = torch.cuda.Event()
                e.record(s_cmp)
                ev_cmp.append(e)
            with torch.cuda.stream(s_out):
                s_out.wait_event(ev_cmp[i])
                host[lo:hi].copy_(d_out[k][:n], non_blocking=True)
                e = torch.cuda.Event()
                e.record(s_out)
                ev_out.append(e)
        s_out.synchronize()
        for t in d_in + d_out + [scratch]:
            t.record_stream(s_cmp)
    return host


def _fill_levels(plan: _Plan, buf: torch.Tensor, scratch: torch.Tensor):
    """``wt_level[levels]`` for this call: the shape part is a per-plan template (copied with one memcpy),
    only the pointers and batch strides are written per call."""
    nl = len(plan.levels)
    tmpl = plan.levels_c
    if tmpl is None:
        arr0 = (N.WtLevel * nl)()
        offs = []
        soff = 0
        for i, lv in enumerate(plan.levels):
            d = arr0[i]
            d.band_stride = lv.plane
            for a in range(plan.ndim):
                d.dims[a] = lv.dims[a]
                d.strides[a] = lv.strides[a]
                d.approx_strides[a] = lv.strides[a]
            if i == nl - 1:
                offs.append((lv.det_off, plan.approx_off, True))
            else:
                offs.append((lv.det_off, soff, False))
                soff += lv.plane
        tmpl = plan.levels_c = (bytes(arr0), tuple(offs))
    raw, offs = tmpl
    arr = (N.WtLevel * nl).from_buffer_copy(raw)
    es = buf.element_size()
    bptr, sptr = buf.data_ptr(), scratch.data_ptr()
    bstride, sstride = buf.stride(0), scratch.stride(0)
    for i, (det_off, a_off, in_buf) in enumerate(offs):
        d = arr[i]
        d.details = bptr + det_off * es
        d.details_batch_stride = bstride
        if in_buf:
            d.approx = bptr + a_off * es
            d.approx_batch_stride = bstride
        else:
            d.approx = sptr + a_off * es
            d.approx_batch_stride = sstride
    return arr


@functools.lru_cache(maxsize=256)
def _taps_c_cached(values: tuple, dt: torch.dtype):
    arr = taps_in_dtype(list(values), dt)
    return arr, arr.ctypes.data_as(N._f64p)


def _taps_c(seq, dt: torch.dtype):
    """Filter taps as a ctypes double array (rounded to the compute dtype first); cached for plain
    Python sequences, rebuilt for tensors (learnable filters)."""
    if isinstance(seq, torch.Tensor):
        return N.f64_array(taps_in_dtype(seq, dt))
    return _taps_c_cached(tuple(float(v) for v in seq), dt)


def _unit_strides(t: torch.Tensor) -> list[int]:
    """Element strides with the (arbitrary) strides of size-1 axes replaced by the contiguous value, so that a
    size-1 last axis never looks like a strided innermost axis to the native code."""
    st = list(t.stride())
    nxt = 1
    for a in range(t.dim() - 1, -1, -1):
        if t.shape[a] == 1:
            st[a] = nxt
        nxt = st[a] * t.shape[a] if t.shape[a] > 1 else nxt
    return st


def _run_fwd(xd: torch.Tensor, plan: _Plan, mode: str, dec_lo, dec_hi, buf: torch.Tensor,
             scratch: torch.Tensor) -> None:
    lib = N.load()
    dt = xd.dtype
    batch = xd.shape[0]
    lo_arr, lo_p = _taps_c(dec_lo, dt)
    hi_arr, hi_p = _taps_c(dec_hi, dt)
    dims_arr, dims_p = plan.dims_c
    xs_arr, xs_p = N.i64_array(_unit_strides(xd)[1:])
    levels = _fill_levels(plan, buf, scratch)
    code = _dtype_code(dt)
    stream = torch.cuda.current_stream(xd.device).cuda_stream
    ws_bytes = int(lib.wt_dwt_workspace_bytes(plan.ndim, code, len(plan.levels), plan.filt_len, batch, dims_p, 0))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=xd.device) if ws_bytes else None
    rc = lib.wt_dwt_fwd(
        plan.ndim, code, N.MODES[mode], len(plan.levels), plan.filt_len, lo_p, hi_p,
        xd.data_ptr(), batch, dims_p, xs_p, xd.stride(0), levels,
        ws.data_ptr() if ws is not None else None, ws_bytes, stream,
    )
    N.check(rc, "wt_dwt_fwd")


# --------------------------------------------------------------------------------------
# synthesis
# --------------------------------------------------------------------------------------
def _same_device_dtype(tensors: Sequence[torch.Tensor]) -> None:
    dev, dt = tensors[0].device, tensors[0].dtype
    for t in tensors:  # reference _util.py:307-348: device first, then dtype
        if t.device != dev:
            raise ValueError("coefficients must be on the same device")
    for t in tensors:
        if t.dtype != dt:
            raise ValueError("coefficients must have the same dtype")


def _pack_bands(bands: list[torch.Tensor], row_al: int):
    """(base tensor, band_stride, strides, batch_stride) for equally shaped bands [B, *dims].

    Zero-copy when the bands are equally strided slices of one buffer with unit inner stride
    (what :func:`_analysis` and the reference's own ``torch.split`` views are); otherwise the
    bands are gathered into one fresh buffer (the reference always pays this copy:
    ``torch.stack``, conv_transform_2.py:224).
    """
    b0 = bands[0]
    es = b0.element_size()
    ok = b0.dim() >= 2 and (b0.stride(-1) == 1 or b0.shape[-1] == 1) and all(s >= 0 for s in b0.stride())
    step = None
    if ok:
        for k, t in enumerate(bands[1:], start=1):
            if t.stride() != b0.stride():
                ok = False
                break
            delta = t.data_ptr() - bands[k - 1].data_ptr()
            if delta % es:
                ok = False
                break
            if step is None:
                step = delta // es
            elif delta // es != step:
                ok = False
                break
    if ok:
        st = list(b0.stride()[1:])
        st[-1] = 1
        return b0, (step or 0), tuple(st), b0.stride(0)
    dims = tuple(b0.shape[1:])
    pitch = round_up(dims[-1], row_al)
    packed = torch.empty((b0.shape[0], len(bands)) + dims[:-1] + (pitch,), dtype=b0.dtype, device=b0.device)
    for k, t in enumerate(bands):
        packed[:, k][..., : dims[-1]].copy_(t)
    inner = packed[:, 0][..., : dims[-1]]
    return inner, packed.stride(1), tuple(inner.stride()[1:]), packed.stride(0)


def _synthesis(approx: torch.Tensor, levels_in: list[list[torch.Tensor]], probes: list[torch.Tensor],
               wavelet: Any, ndim: int, f: Fold) -> torch.Tensor:
    """approx [B,*]; levels_in coarsest-first, each the bands k=1..2^ndim-1 as [B,*] tensors;
    probes[i] is the tensor of level i whose extents the reference compares the running
    reconstruction with (1-D: the detail; 2-D: horizontal; 3-D: "aad")."""
    wav = as_wavelet(wavelet)
    _, _, rec_lo, rec_hi = filter_bank(wav)
    filt_len = len(rec_lo)
    if not levels_in:
        return approx
    padl = (2 * filt_len - 3) // 2
    # Walk the levels exactly in the reference's order of checks: band shapes against the running
    # approximation (ValueError; conv_transform_2.py:217-221, conv_transform_3.py:200-204; in 1-D
    # torch.stack raises RuntimeError, conv_transform.py:186), then the crop (conv_transform.py:
    # 190-199, _util.py:231-244): full = 2(c-1) + L - 2 padl, one more sample is dropped when the
    # next finer detail is one shorter; anything else is an AssertionError.
    cur = tuple(approx.shape[1:])
    out_dims_per_level = []
    nl = len(levels_in)
    for i in range(nl):
        for t in levels_in[i]:
            if tuple(t.shape[1:]) != cur or t.shape[0] != approx.shape[0]:
                if ndim == 1:
                    raise RuntimeError(
                        f"stack expects each tensor to be equal size, but got {[approx.shape[0], *cur]} "
                        f"and {list(t.shape)}")
                raise ValueError("All coefficients on each level must have the same shape")
        full = tuple(2 * (c - 1) + filt_len - 2 * padl for c in cur)
        if i + 1 < nl:
            nxt = tuple(probes[i + 1].shape[1:])
            got = []
            for a in range(ndim - 1, -1, -1):  # the reference adjusts the last axis first
                if nxt[a] == full[a]:
                    got.append(full[a])
                elif nxt[a] == full[a] - 1:
                    got.append(full[a] - 1)
                else:
                    raise AssertionError("padding error, please check if dec and rec wavelets are identical.")
            full = tuple(reversed(got))
        if any(v < 1 for v in full):
            raise ValueError("coefficient tensors are too small for this wavelet")
        out_dims_per_level.append(full)
        cur = full
    if filt_len < 2 or filt_len > N.WT_MAX_FILT_LEN or len(rec_hi) != filt_len:
        raise ValueError(f"filter length {filt_len} not supported (2..{N.WT_MAX_FILT_LEN})")
    if torch.is_grad_enabled() and (
        approx.requires_grad or any(t.requires_grad for lv in levels_in for t in lv) or any_requires_grad(wav)
    ):
        from ._autograd import synthesis_with_grad

        return synthesis_with_grad(approx, levels_in, probes, rec_lo, rec_hi, ndim, _compute_device(approx))

    dev = _compute_device(approx)
    on_host = not approx.is_cuda
    batch = approx.shape[0]
    dt = approx.dtype
    es = approx.element_size()
    row_al = max(ROW_ALIGN_BYTES // es, 1)
    with torch.cuda.device(dev):
        if on_host:
            approx = approx.to(dev, non_blocking=True)
            levels_in = [[t.to(dev, non_blocking=True) for t in lv] for lv in levels_in]
        keep = []  # keep packed buffers alive until the launch is enqueued
        arr = (N.WtLevel * nl)()
        # arr[0] = finest level
        for i, bands in enumerate(levels_in):
            li = nl - 1 - i
            d = arr[li]
            base, band_stride, st, bstride = _pack_bands(bands, row_al)
            keep.append(base)
            d.details = base.data_ptr()
            d.band_stride = band_stride
            d.details_batch_stride = bstride
            cdims = tuple(bands[0].shape[1:])
            for a in range(ndim):
                d.dims[a] = cdims[a]
                d.strides[a] = st[a]
            if i == 0:
                ap = approx
                if (ap.stride(-1) != 1 and ap.shape[-1] != 1) or any(s < 0 for s in ap.stride()):
                    ap = ap.contiguous()
                keep.append(ap)
                d.approx = ap.data_ptr()
                d.approx_batch_stride = ap.stride(0)
                for a in range(ndim):
                    d.approx_strides[a] = ap.stride(1 + a) if a < ndim - 1 else 1
            else:
                # scratch for the reconstruction coming from the coarser level
                pitch = round_up(cdims[-1], row_al)
                sc = torch.empty((batch,) + cdims[:-1] + (pitch,), dtype=dt, device=dev)
                keep.append(sc)
                d.approx = sc.data_ptr()
                d.approx_batch_stride = sc.stride(0)
                for a in range(ndim):
                    d.approx_strides[a] = sc.stride(1 + a)
        out_dims = out_dims_per_level[-1]
        y = torch.empty((batch,) + out_dims, dtype=dt, device=dev)
        lib = N.load()
        lo_arr, lo_p = _taps_c(rec_lo, dt)
        hi_arr, hi_p = _taps_c(rec_hi, dt)
        od_arr, od_p = N.i64_array(out_dims)
        ys_arr, ys_p = N.i64_array(y.stride()[1:])
        code = _dtype_code(dt)
        stream = torch.cuda.current_stream(dev).cuda_stream
        ws_bytes = int(lib.wt_dwt_workspace_bytes(ndim, code, nl, filt_len, batch, od_p, 1))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
        rc = lib.wt_dwt_inv(ndim, code, nl, filt_len, lo_p, hi_p, y.data_ptr(), batch, od_p, ys_p, y.stride(0),
                            arr, ws.data_ptr() if ws is not None else None, ws_bytes, stream)
        N.check(rc, "wt_dwt_inv")
        if on_host:
            host = pinned_empty(y.shape, dt)
            host.copy_(y, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            y = host
        del keep
    return y


def _fold_coeff_tensors(tensors: list[torch.Tensor], ndim: int, axes: AxisHint):
    lead = check_tensor(tensors[0])
    check_dtype(lead)
    folded = []
    f: Optional[Fold] = None
    for t in tensors:
        ft, f = fold(t, ndim, axes, lead=f)
        folded.append(ft)
    return folded, f


# --------------------------------------------------------------------------------------
# public API -- 1-D
# --------------------------------------------------------------------------------------
def wavedec(data: torch.Tensor, wavelet: Any, *, mode: str = "reflect", level: Optional[int] = None,
            axis: int = -1) -> list[torch.Tensor]:
    """1-D analysis FWT, ``[cA_n, cD_n, ..., cD_1]`` (reference conv_transform.py:69-143)."""
    approx, details, f = _analysis(data, wavelet, mode, level, axis, 1)
    result = [approx] + [bands[0] for bands in details]
    return [unfold(t, f) for t in result]


def waverec(coeffs: Sequence[torch.Tensor], wavelet: Any, *, axis: AxisHint = None) -> torch.Tensor:
    """1-D synthesis FWT (reference conv_transform.py:146-204)."""
    if not isinstance(coeffs, list):
        coeffs = list(coeffs)
    for c in coeffs[1:]:
        if not isinstance(c, torch.Tensor):
            raise ValueError(f"Unexpected input type {type(c)}")
    folded, f = _fold_coeff_tensors(list(coeffs), 1, axis)
    _same_device_dtype(folded)
    levels_in = [[t] for t in folded[1:]]
    y = _synthesis(folded[0], levels_in, [lv[0] for lv in levels_in], wavelet, 1, f)
    return unfold(y, f)


# --------------------------------------------------------------------------------------
# public API -- 2-D
# --------------------------------------------------------------------------------------
def wavedec2(data: torch.Tensor, wavelet: Any, *, mode: str = "reflect", level: Optional[int] = None,
             axes: tuple[int, int] = (-2, -1)):
    """2-D analysis FWT, ``(cA_n, (cH_n, cV_n, cD_n), ..., (cH_1, cV_1, cD_1))``
    (reference conv_transform_2.py:74-157).  Band k=2 (hi along axis -2, lo along -1) is the
    reference's ``lh`` = horizontal, k=1 its ``hl`` = vertical (reference _util.py:901-905)."""
    approx, details, f = _analysis(data, wavelet, mode, level, axes, 2)
    out: list[Any] = [unfold(approx, f)]
    for bands in details:
        out.append(WaveletDetailTuple2d(unfold(bands[1], f), unfold(bands[0], f), unfold(bands[2], f)))
    return tuple(out)


def waverec2(coeffs, wavelet: Any, *, axes: AxisHint = None) -> torch.Tensor:
    """2-D synthesis FWT (reference conv_transform_2.py:160-253)."""
    lead = check_tensor(coeffs[0])
    check_dtype(lead)
    ensure_axes(axes, 2)
    for el in coeffs[1:]:
        if not isinstance(el, tuple) or len(el) != 3:
            raise ValueError(
                f"Unexpected detail coefficient type: {type(el)}. Detail coefficients must be a 3-tuple of "
                "tensors as returned by wavedec2."
            )
    flat: list[torch.Tensor] = [lead]
    for el in coeffs[1:]:
        flat.extend(el)
    folded, f = _fold_coeff_tensors(flat, 2, axes)
    _same_device_dtype(folded)
    levels_in = []
    probes = []
    for i in range(len(coeffs) - 1):
        h, v, d = folded[1 + 3 * i: 4 + 3 * i]
        levels_in.append([v, h, d])  # band order k = 1 (lo_H hi_W), 2 (hi_H lo_W), 3
        probes.append(h)             # the reference probes coeffs[c_pos + 2][0] = horizontal
    y = _synthesis(folded[0], levels_in, probes, wavelet, 2, f)
    return unfold(y, f)


# --------------------------------------------------------------------------------------
# public API -- 3-D
# --------------------------------------------------------------------------------------
def wavedec3(data: torch.Tensor, wavelet: Any, *, mode: str = "zero", level: Optional[int] = None,
             axes: tuple[int, int, int] = (-3, -2, -1)):
    """3-D analysis FWT, ``(cA_n, {aad..ddd}_n, ..., {aad..ddd}_1)``
    (reference conv_transform_3.py:76-145; default mode is "zero")."""
    approx, details, f = _analysis(data, wavelet, mode, level, axes, 3)
    out: list[Any] = [unfold(approx, f)]
    for bands in details:
        out.append({key: unfold(bands[k], f) for k, key in enumerate(DETAIL_KEYS_3D)})
    return tuple(out)


def waverec3(coeffs, wavelet: Any, *, axes: AxisHint = None) -> torch.Tensor:
    """3-D synthesis FWT (reference conv_transform_3.py:148-251)."""
    lead = check_tensor(coeffs[0])
    check_dtype(lead)
    ensure_axes(axes, 3)
    for el in coeffs[1:]:
        if not isinstance(el, dict) or len(el) != 7:
            raise ValueError(
                f"Unexpected detail coefficient type: {type(el)}. Detail coefficients must be a dict containing "
                "7 tensors as returned by wavedec3."
            )
    flat: list[torch.Tensor] = [lead]
    for el in coeffs[1:]:
        flat.extend(el[key] for key in DETAIL_KEYS_3D)
    folded, f = _fold_coeff_tensors(flat, 3, axes)
    _same_device_dtype(folded)
    levels_in = []
    probes = []
    for i in range(len(coeffs) - 1):
        bands = folded[1 + 7 * i: 8 + 7 * i]
        levels_in.append(list(bands))
        probes.append(bands[0])  # "aad"
    y = _synthesis(folded[0], levels_in, probes, wavelet, 3, f)
    return unfold(y, f)
