"""Stationary (undecimated, "a trous") wavelet transform on the H100.

Drop-in for ``ptwt.swt`` / ``ptwt.iswt`` (reference ``src/ptwt/stationary_transform.py:56-108`` and ``:111-156``):
same signatures, return containers and errors.  The reference's per-level ``_circular_pad -> conv1d(dilation) ->
split`` and ``stack -> _circular_pad -> conv_transpose1d -> mean`` bodies are replaced by ONE call into libwtb200
(``wt_swt_fwd`` / ``wt_swt_inv``, include/wtb200.h, csrc/swt.cuh) that runs groups of levels with the intermediate
approximations on chip and the periodic extension evaluated as an index modulo n (no padded copy).

Where a pad is longer than the signal the reference pads in rounds of at most n samples (``_circular_pad``), which
is not the periodic extension whenever a round other than the last adds a total that is not a multiple of n.  That
quirk is kept: for such a level the host builds the source index of every tap from the reference's rounds, and the
kernels read it from a table (only short signals with an explicit ``level`` get there).

Outputs are views of one packed ``[batch, level + 1, pitch]`` buffer (rows 16-byte aligned); ``iswt`` consumes such
views without a copy.  CPU tensors are staged to the current CUDA device and back, as in :func:`wavedec`.

``swt2`` / ``iswt2`` are the 2-D transform (PyWavelets' ``swt2`` with ``trim_approx=True``, ``norm=False``; the
reference has none).  Each level is two one-axis passes on the same kernels (``wt_swt_pass_fwd`` / ``wt_swt_pass_inv``):
rows of W samples along ``axes[1]``, then each H x W plane as one periodic signal of H W samples at dilation d W along
``axes[0]``.  The extension is exactly periodic at every level, including dilations longer than the extent: there is
no reference ``swt2`` whose multi-round padding could be copied.
"""
from __future__ import annotations

import ctypes as C
import functools
from typing import Any, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import _native as N
from ._shape import AxisHint, check_dtype, check_tensor, ensure_axes, fold, round_up, unfold
from ._wavelets import any_requires_grad, as_wavelet, filter_bank, swt_max_level, taps_in_dtype
from .constants import WaveletDetailTuple2d
from .fwt import (BAND_ALIGN_BYTES, ROW_ALIGN_BYTES, _compute_device, _dtype_code, _fold_coeff_tensors, _pack_bands,
                  _same_device_dtype, pinned_empty)

__all__ = ["swt", "iswt", "swt2", "iswt2"]


# --------------------------------------------------------------------------------------
# the reference's extension and the tables of the levels where it is not periodic
# --------------------------------------------------------------------------------------
def circular_pad_sources(n: int, pl: int, pr: int, pos: np.ndarray) -> np.ndarray:
    """Index in ``[0, n)`` of the sample the reference's ``_circular_pad(x, [pl, pr])`` puts at positions ``pos``.

    Each round is ``F.pad(mode="circular")`` by at most n on either side (stationary_transform.py:24-53); a circular
    pad by (a, b) of a length-l tensor puts ``in[(q - a) mod l]`` at position q, so the rounds are undone backwards."""
    rounds = []
    if pl <= n and pr <= n:
        rounds.append((pl, pr))
    else:
        while pl > 0 or pr > 0:
            rounds.append((min(n, pl), min(n, pr)))
            pl, pr = max(pl - n, 0), max(pr - n, 0)
    lengths = [n]
    for a, b in rounds:
        lengths.append(lengths[-1] + a + b)
    p = np.asarray(pos, dtype=np.int64)
    for (a, _), ln in zip(reversed(rounds), reversed(lengths[:-1])):
        p = (p - a) % ln
    return p


MAX_PADDED_LEN = 1 << 31


def _level_sources(n: int, filt_len: int, level: int, inverse: bool) -> Optional[np.ndarray]:
    """``[n, L]`` source indices of the taps of one level, or None where they are the periodic ``(i + d(m - hl)) mod n``
    (analysis) / ``(i + d(hl - m)) mod n`` (synthesis)."""
    d = 1 << (level - 1)
    hl, hr = d * (filt_len // 2 - 1), d * (filt_len // 2)
    pl, pr = (hr, hl) if inverse else (hl, hr)
    if max(pl, pr) <= n:
        return None
    if n + pl + pr >= MAX_PADDED_LEN:
        raise RuntimeError(f"swt level {level} pads a signal of {n} samples to {n + pl + pr}: too long")
    i = np.arange(n, dtype=np.int64)[:, None]
    m = np.arange(filt_len, dtype=np.int64)[None, :]
    pos = i + (pl + pr) - d * m if inverse else i + d * m
    src = circular_pad_sources(n, pl, pr, pos)
    periodic = (pos - pl) % n
    return None if np.array_equal(src, periodic) else src


def _csr(src: np.ndarray, transpose: bool) -> np.ndarray:
    """Table layout of include/wtb200.h: rowptr[n + 1], padded to even length, then (column, tap) pairs."""
    n, L = src.shape
    if transpose:
        flat = src.reshape(-1)
        order = np.argsort(flat, kind="stable")
        rowptr = np.concatenate([[0], np.cumsum(np.bincount(flat, minlength=n))])
        pairs = np.stack([order // L, order % L], 1)
    else:
        rowptr = np.arange(n + 1, dtype=np.int64) * L
        pairs = np.stack([src.reshape(-1), np.tile(np.arange(L), n)], 1)
    head = np.zeros(2 * ((n + 2) // 2), dtype=np.int64)
    head[: n + 1] = rowptr
    return np.concatenate([head, pairs.reshape(-1)]).astype(np.int32)


_TABLE_CACHE: dict = {}


@functools.lru_cache(maxsize=256)
def _quirk_levels(n: int, filt_len: int, levels: int, inverse: bool) -> tuple:
    return tuple(j for j in range(1, levels + 1) if _level_sources(n, filt_len, j, inverse) is not None)


def _tables(n: int, filt_len: int, levels: int, inverse: bool, transpose: bool, device: torch.device):
    """(ctypes array of per-level table pointers or None, tensors to keep alive).  ``inverse``: which of the
    reference's two extensions; ``transpose``: the adjoint of it (the backward pass)."""
    quirk = _quirk_levels(n, filt_len, levels, inverse)
    if not quirk:
        return None, []
    ptrs = (C.c_void_p * levels)()
    keep = []
    for j in quirk:
        key = (n, filt_len, j, inverse, transpose, str(device))
        t = _TABLE_CACHE.get(key)
        if t is None:
            t = _TABLE_CACHE[key] = torch.from_numpy(_csr(_level_sources(n, filt_len, j, inverse), transpose)).to(device)
        ptrs[j - 1] = t.data_ptr()
        keep.append(t)
    return ptrs, keep


# --------------------------------------------------------------------------------------
# launches
# --------------------------------------------------------------------------------------
def _window_taps(fb, dtype: torch.dtype, inverse: bool):
    """Window-order taps of wt_swt_fwd (analysis: dec[::-1]) or wt_swt_inv (synthesis: 0.5 rec), rounded to the
    compute dtype first like the reference's filter tensors (_util.py:129-141)."""
    dec_lo, dec_hi, rec_lo, rec_hi = fb
    if inverse:
        return 0.5 * taps_in_dtype(rec_lo, dtype), 0.5 * taps_in_dtype(rec_hi, dtype)
    return taps_in_dtype(dec_lo, dtype)[::-1].copy(), taps_in_dtype(dec_hi, dtype)[::-1].copy()


def _workspace(code: int, levels: int, L: int, batch: int, n: int, tables, inverse: bool, device) -> tuple:
    lib = N.load()
    ws_bytes = int(lib.wt_swt_workspace_bytes(code, levels, L, batch, n, tables, int(inverse)))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=device) if ws_bytes else None
    return ws, ws_bytes


def _packed_empty(batch: int, levels: int, n: int, dtype: torch.dtype, device) -> torch.Tensor:
    es = torch.empty((), dtype=dtype).element_size()
    return torch.empty((batch, levels + 1, round_up(n, max(ROW_ALIGN_BYTES // es, 1))), dtype=dtype, device=device)


def run_analysis(x: torch.Tensor, f_lo, f_hi, levels: int, L: int, tables_inverse: bool, transpose: bool) -> torch.Tensor:
    """wt_swt_fwd on ``x [B, n]`` (CUDA, unit inner stride) -> packed ``[B, levels + 1, pitch]``."""
    batch, n = x.shape
    out = _packed_empty(batch, levels, n, x.dtype, x.device)
    if batch == 0:
        return out
    tables, keep = _tables(n, L, levels, tables_inverse, transpose, x.device)
    code = _dtype_code(x.dtype)
    ws, ws_bytes = _workspace(code, levels, L, batch, n, tables, False, x.device)
    lo_arr, lo_p = N.f64_array(f_lo)
    hi_arr, hi_p = N.f64_array(f_hi)
    rc = N.load().wt_swt_fwd(code, levels, L, lo_p, hi_p, x.data_ptr(), batch, n, x.stride(0), out.data_ptr(),
                             out.stride(0), out.stride(1), tables, ws.data_ptr() if ws is not None else None, ws_bytes,
                             torch.cuda.current_stream(x.device).cuda_stream)
    N.check(rc, "wt_swt_fwd")
    del keep
    return out


def run_synthesis(approx: torch.Tensor, details: Sequence[torch.Tensor], g_lo, g_hi, L: int, tables_inverse: bool,
                  transpose: bool) -> torch.Tensor:
    """wt_swt_inv: ``approx [B, n]`` and ``details`` = [cD_J, ..., cD_1] (CUDA) -> ``[B, n]``."""
    levels = len(details)
    batch, n = approx.shape
    y = torch.empty((batch, n), dtype=approx.dtype, device=approx.device)
    if batch == 0:
        return y
    es = approx.element_size()
    base, band, _, dbs = _pack_bands(list(details), max(ROW_ALIGN_BYTES // es, 1))
    ap = approx if approx.stride(-1) == 1 or n == 1 else approx.contiguous()
    tables, keep = _tables(n, L, levels, tables_inverse, transpose, approx.device)
    code = _dtype_code(approx.dtype)
    ws, ws_bytes = _workspace(code, levels, L, batch, n, tables, True, approx.device)
    lo_arr, lo_p = N.f64_array(g_lo)
    hi_arr, hi_p = N.f64_array(g_hi)
    rc = N.load().wt_swt_inv(code, levels, L, lo_p, hi_p, ap.data_ptr(), ap.stride(0), base.data_ptr(), dbs, band,
                             batch, n, y.data_ptr(), y.stride(0), tables, ws.data_ptr() if ws is not None else None,
                             ws_bytes, torch.cuda.current_stream(approx.device).cuda_stream)
    N.check(rc, "wt_swt_inv")
    del keep, base
    return y


# --------------------------------------------------------------------------------------
# autograd: each direction's backward is the other kernel with the adjoint taps and the transposed tables, run as a
# Function of its own whose backward is the forward kernel again, so in grad mode (create_graph=True) gradients of any
# order reach the data.
# --------------------------------------------------------------------------------------
def _swt_adjoint(g: torch.Tensor, fb, levels: int, L: int, n: int) -> torch.Tensor:
    """Adjoint of swt: packed ``[B, levels + 1, pitch]`` gradient -> ``[B, n]`` (the pitch padding is not read)."""
    g = g.contiguous()
    f_lo, f_hi = _window_taps(fb, g.dtype, inverse=False)
    details = [g[:, k, :n] for k in range(1, levels + 1)]
    return run_synthesis(g[:, 0, :n], details, f_lo, f_hi, L, tables_inverse=False, transpose=True)


def _iswt_adjoint(gy: torch.Tensor, fb, levels: int, L: int) -> tuple:
    """Adjoint of iswt: ``[B, n]`` gradient -> the gradients of approx and the ``levels`` details."""
    f_lo, f_hi = _window_taps(fb, gy.dtype, inverse=True)
    n = gy.shape[-1]
    packed = run_analysis(gy.contiguous(), f_lo, f_hi, levels, L, tables_inverse=True, transpose=True)
    return tuple(packed[:, k, :n] for k in range(levels + 1))


class _SwtFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fb, levels, L):
        ctx.fb, ctx.levels, ctx.L, ctx.n = fb, levels, L, x.shape[-1]
        f_lo, f_hi = _window_taps(fb, x.dtype, inverse=False)
        return run_analysis(x.contiguous(), f_lo, f_hi, levels, L, tables_inverse=False, transpose=False)

    @staticmethod
    def backward(ctx, g):
        return _SwtAdjointFunction.apply(g, ctx.fb, ctx.levels, ctx.L, ctx.n), None, None, None


class _SwtAdjointFunction(torch.autograd.Function):
    """The backward pass of swt as a differentiable map; its own adjoint is swt, written into the packed layout
    with zeros in the pitch padding (those entries never reach the data gradient)."""

    @staticmethod
    def forward(ctx, g, fb, levels, L, n):
        ctx.fb, ctx.levels, ctx.L, ctx.n, ctx.pitch = fb, levels, L, n, g.shape[-1]
        return _swt_adjoint(g, fb, levels, L, n)

    @staticmethod
    def backward(ctx, u):
        packed = _SwtFunction.apply(u, ctx.fb, ctx.levels, ctx.L)
        return F.pad(packed[..., :ctx.n], (0, ctx.pitch - ctx.n)), None, None, None, None


class _IswtFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fb, L, approx, *details):
        ctx.fb, ctx.L, ctx.levels = fb, L, len(details)
        g_lo, g_hi = _window_taps(fb, approx.dtype, inverse=True)
        return run_synthesis(approx, details, g_lo, g_hi, L, tables_inverse=True, transpose=False)

    @staticmethod
    def backward(ctx, gy):
        return (None, None) + _IswtAdjointFunction.apply(gy, ctx.fb, ctx.levels, ctx.L)


class _IswtAdjointFunction(torch.autograd.Function):
    """The backward pass of iswt as a differentiable map; its own adjoint is iswt."""

    @staticmethod
    def forward(ctx, gy, fb, levels, L):
        ctx.fb, ctx.L = fb, L
        return _iswt_adjoint(gy, fb, levels, L)

    @staticmethod
    def backward(ctx, *us):
        return _IswtFunction.apply(ctx.fb, ctx.L, *[u.contiguous() for u in us]), None, None, None


def _check_taps_without_grad(wav: Any, what: str = "swt/iswt") -> None:
    if torch.is_grad_enabled() and any_requires_grad(wav):
        raise NotImplementedError(
            f"{what} compute gradients with respect to the data only, not with respect to learnable filter taps; "
            "pass plain filters or call under torch.no_grad()."
        )


def _filter_bank(wavelet: Any, what: str = "swt/iswt"):
    wav = as_wavelet(wavelet)
    fb = filter_bank(wav)
    L = len(fb[0])
    if any(len(f) != L for f in fb):
        raise ValueError("all four filters of the wavelet must have the same length")
    if L < 2 or L > N.WT_MAX_FILT_LEN or L % 2:
        raise ValueError(f"{what} need an even filter length in 2..{N.WT_MAX_FILT_LEN}, got {L}")
    return wav, fb, L


def _check_axis(t: torch.Tensor, axis: AxisHint) -> None:
    """The reference moves ``axis`` last with ``permute``, which raises RuntimeError for an axis out of range."""
    if isinstance(axis, int) and not -t.dim() <= axis < t.dim():
        raise RuntimeError(f"axis {axis} is out of range for a tensor with {t.dim()} dimensions")


# --------------------------------------------------------------------------------------
# public API
# --------------------------------------------------------------------------------------
def swt(data: torch.Tensor, wavelet: Any, level: Optional[int] = None, *, axis: AxisHint = None) -> list[torch.Tensor]:
    """1-D stationary wavelet transform, ``[cA_J, cD_J, ..., cD_1]``, each as long as the input
    (reference stationary_transform.py:56-108; pywt.swt with trim_approx=True, norm=False)."""
    check_tensor(data)
    check_dtype(data)
    _check_axis(data, axis)
    x, f = fold(data, 1, axis)
    n = int(x.shape[-1])
    if level is None:
        level = swt_max_level(n)
    if level <= 0:
        return [unfold(x, f)]
    wav, fb, L = _filter_bank(wavelet)
    _check_taps_without_grad(wav)
    dev = _compute_device(x)
    on_host = not x.is_cuda
    with torch.cuda.device(dev):
        if torch.is_grad_enabled() and x.requires_grad:
            xd = x.to(dev)
            packed = _SwtFunction.apply(xd, fb, level, L)
            out = [packed[:, k, :n] for k in range(level + 1)]
            if on_host:
                out = [t.cpu() for t in out]
            return [unfold(t, f) for t in out]
        xd = x.to(dev, non_blocking=True) if on_host else x
        if xd.stride(-1) != 1 and n != 1:
            xd = xd.contiguous()
        f_lo, f_hi = _window_taps(fb, x.dtype, inverse=False)
        packed = run_analysis(xd, f_lo, f_hi, level, L, tables_inverse=False, transpose=False)
        if on_host:
            host = pinned_empty(packed.shape, packed.dtype)
            host.copy_(packed, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            packed = host
    return [unfold(packed[:, k, :n], f) for k in range(level + 1)]


def iswt(coeffs: Sequence[torch.Tensor], wavelet: Any, *, axis: AxisHint = None) -> torch.Tensor:
    """Inverse of :func:`swt` (reference stationary_transform.py:111-156)."""
    if not isinstance(coeffs, list):
        coeffs = list(coeffs)
    lead = check_tensor(coeffs[0])
    check_dtype(lead)
    _check_axis(lead, axis)
    folded = []
    f = None
    for t in coeffs:
        ft, f = fold(t, 1, axis, lead=f)
        folded.append(ft)
    _same_device_dtype(folded)
    approx, details = folded[0], folded[1:]
    if not details:
        return unfold(approx, f)
    for t in details:   # the reference stacks the running approximation with each detail (stationary_transform.py:142)
        if t.shape != approx.shape:
            raise RuntimeError(f"stack expects each tensor to be equal size, but got {list(approx.shape)} at entry 0 "
                               f"and {list(t.shape)} at entry 1")
    wav, fb, L = _filter_bank(wavelet)
    _check_taps_without_grad(wav)
    dev = _compute_device(approx)
    on_host = not approx.is_cuda
    with torch.cuda.device(dev):
        if torch.is_grad_enabled() and any(t.requires_grad for t in folded):
            y = _IswtFunction.apply(fb, L, *[t.to(dev) for t in folded])
            return unfold(y.cpu() if on_host else y, f)
        if on_host:
            approx = approx.to(dev, non_blocking=True)
            details = [t.to(dev, non_blocking=True) for t in details]
        g_lo, g_hi = _window_taps(fb, approx.dtype, inverse=True)
        y = run_synthesis(approx, details, g_lo, g_hi, L, tables_inverse=True, transpose=False)
        if on_host:
            host = pinned_empty(y.shape, y.dtype)
            host.copy_(y, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            y = host
    return unfold(y, f)


# --------------------------------------------------------------------------------------
# 2-D: one launch per axis pass, two passes per level
# --------------------------------------------------------------------------------------
def _dense_planes(t: torch.Tensor) -> torch.Tensor:
    """``t [B, H, W]`` itself when every plane is dense with row pitch W (what the pass along axes[0] reads as one
    signal of H W samples), else a contiguous copy."""
    _, H, W = t.shape
    if (W == 1 or t.stride(2) == 1) and (H == 1 or t.stride(1) == W):
        return t
    return t.contiguous()


def _rows(t: torch.Tensor) -> tuple[torch.Tensor, int]:
    """``t [B, H, W]`` as B H rows of W samples one stride apart (the pass along axes[1]): (tensor, row stride)."""
    B, H, W = t.shape
    if W == 1 or t.stride(2) == 1:
        if H == 1:
            return t, t.stride(0)
        if B == 1 or t.stride(0) == H * t.stride(1):
            return t, t.stride(1)
    return t.contiguous(), W


def _pack_planes(bands: list[torch.Tensor]) -> tuple[torch.Tensor, int, int]:
    """(tensor at band 0, band stride, batch stride) of equally shaped ``[B, H, W]`` bands with dense planes: the bands
    themselves when they are equally strided planes of one buffer (what :func:`swt2` returns), else one gather."""
    _, H, W = bands[0].shape
    base, step, st, bs = _pack_bands(bands, 1)
    if H > 1 and st[0] != W:
        base = torch.stack(bands, 1)
        step, bs = base.stride(1), base.stride(0)
    return base, step, bs


def _ptrs(*addrs: int):
    return (C.c_void_p * len(addrs))(*addrs)


def _i64s(*vals: int):
    return (C.c_int64 * len(vals))(*vals)


def _pass(inverse: bool, code: int, taps, L: int, dilation: int, in0, in0_bs, in1, in1_bs, out0, out0_bs, batch: int,
          n: int, stream) -> None:
    """One wt_swt_pass_fwd / wt_swt_pass_inv call; in* / out* are tuples of addresses and batch strides, one per band
    set.  Analysis: in0 -> out0 (low), in1 (high, an output).  Synthesis: in0 (low), in1 (high) -> out0."""
    lo_arr, lo_p = N.f64_array(taps[0])
    hi_arr, hi_p = N.f64_array(taps[1])
    sets = len(in0)
    lib = N.load()
    if inverse:
        rc = lib.wt_swt_pass_inv(code, L, lo_p, hi_p, dilation, sets, _ptrs(*in0), _i64s(*in0_bs), _ptrs(*in1),
                                 _i64s(*in1_bs), _ptrs(*out0), _i64s(*out0_bs), batch, n, stream)
    else:
        rc = lib.wt_swt_pass_fwd(code, L, lo_p, hi_p, dilation, sets, _ptrs(*in0), _i64s(*in0_bs), _ptrs(*out0),
                                 _i64s(*out0_bs), _ptrs(*in1), _i64s(*in1_bs), batch, n, stream)
    N.check(rc, "wt_swt_pass_inv" if inverse else "wt_swt_pass_fwd")


def _workspace2(code: int, levels: int, B: int, H: int, W: int, dtype, device) -> tuple[int, int, int]:
    """Addresses of the workspace planes: the two bands of the pass along axes[1] and the running approximation."""
    ws_bytes = int(N.load().wt_swt2_workspace_bytes(code, levels, B, H, W))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=device)
    plane = B * H * W * torch.empty((), dtype=dtype).element_size()
    base = ws.data_ptr()
    return ws, base, base + plane, base + 2 * plane


def band_pitch(n: int, dtype: torch.dtype) -> int:
    """Elements between the planes of one item of :func:`swt2`'s packed buffer: H W rounded up to 128 bytes."""
    es = torch.empty((), dtype=dtype).element_size()
    return round_up(n, BAND_ALIGN_BYTES // es)


def run_analysis2(x: torch.Tensor, f_lo, f_hi, levels: int, L: int) -> torch.Tensor:
    """``x [B, H, W]`` (CUDA) -> packed ``[B, 3 levels + 1, pitch]``: cA_J, then (cH_j, cV_j, cD_j) for j = J..1, each
    band a dense H x W plane at the start of its row."""
    B, H, W = x.shape
    n = H * W
    out = torch.empty((B, 3 * levels + 1, band_pitch(n, x.dtype)), dtype=x.dtype, device=x.device)
    if out.numel() == 0 or n == 0:
        return out
    code, es = _dtype_code(x.dtype), x.element_size()
    stream = torch.cuda.current_stream(x.device).cuda_stream
    x, rs = _rows(x)
    ws, lo_w, hi_w, a_ws = _workspace2(code, levels, B, H, W, x.dtype, x.device)
    obs, band = out.stride(0), out.stride(1) * es
    src, src_rs = x.data_ptr(), rs
    for j in range(1, levels + 1):
        d = 1 << (j - 1)
        _pass(False, code, (f_lo, f_hi), L, d, (src,), (src_rs,), (hi_w,), (W,), (lo_w,), (W,), B * H, W, stream)
        k = out.data_ptr() + (1 + 3 * (levels - j)) * band        # cH_j; cV_j and cD_j follow
        a_dst, a_bs = (out.data_ptr(), obs) if j == levels else (a_ws, n)
        # set 0: lo_W -> (cA_j, cH_j); set 1: hi_W -> (cV_j, cD_j)
        _pass(False, code, (f_lo, f_hi), L, d * W, (lo_w, hi_w), (n, n), (k, k + 2 * band), (obs, obs),
              (a_dst, k + band), (a_bs, obs), B, n, stream)
        src, src_rs = a_ws, W
    del ws, x
    return out


def run_synthesis2(approx: torch.Tensor, details: Sequence[torch.Tensor], g_lo, g_hi, L: int) -> torch.Tensor:
    """``approx [B, H, W]`` and ``details`` = [cH_J, cV_J, cD_J, ..., cH_1, cV_1, cD_1] (CUDA) -> ``[B, H, W]``."""
    levels = len(details) // 3
    B, H, W = approx.shape
    n = H * W
    y = torch.empty((B, H, W), dtype=approx.dtype, device=approx.device)
    if y.numel() == 0:
        return y
    code, es = _dtype_code(approx.dtype), approx.element_size()
    stream = torch.cuda.current_stream(approx.device).cuda_stream
    a = _dense_planes(approx)
    base, step, dbs = _pack_planes(list(details))
    ws, lo_w, hi_w, a_ws = _workspace2(code, levels, B, H, W, approx.dtype, approx.device)
    cur, cur_bs = a.data_ptr(), a.stride(0)
    for j in range(levels, 0, -1):
        d = 1 << (j - 1)
        k = base.data_ptr() + 3 * (levels - j) * step * es       # cH_j; cV_j and cD_j follow
        kv, kd = k + step * es, k + 2 * step * es
        # set 0: (cA_j, cH_j) -> lo_W; set 1: (cV_j, cD_j) -> hi_W
        _pass(True, code, (g_lo, g_hi), L, d * W, (cur, kv), (cur_bs, dbs), (k, kd), (dbs, dbs), (lo_w, hi_w),
              (n, n), B, n, stream)
        dst = y.data_ptr() if j == 1 else a_ws
        _pass(True, code, (g_lo, g_hi), L, d, (lo_w,), (W,), (hi_w,), (W,), (dst,), (W,), B * H, W, stream)
        cur, cur_bs = a_ws, n
    del ws, a, base
    return y


def _bands2(packed: torch.Tensor, levels: int, H: int, W: int) -> list[torch.Tensor]:
    """The 3 levels + 1 ``[B, H, W]`` views of a packed buffer."""
    B = packed.shape[0]
    return [packed[:, k, :H * W].view(B, H, W) for k in range(3 * levels + 1)]


def _swt2_adjoint(g: torch.Tensor, fb, levels: int, L: int, H: int, W: int) -> torch.Tensor:
    """Adjoint of swt2: packed gradient -> ``[B, H, W]`` (the pitch padding is not read)."""
    f_lo, f_hi = _window_taps(fb, g.dtype, inverse=False)
    bands = _bands2(g.contiguous(), levels, H, W)
    return run_synthesis2(bands[0], bands[1:], f_lo, f_hi, L)


def _iswt2_adjoint(gy: torch.Tensor, fb, levels: int, L: int) -> tuple:
    """Adjoint of iswt2: ``[B, H, W]`` gradient -> the gradients of approx and the 3 levels details."""
    f_lo, f_hi = _window_taps(fb, gy.dtype, inverse=True)
    _, H, W = gy.shape
    return tuple(_bands2(run_analysis2(gy, f_lo, f_hi, levels, L), levels, H, W))


class _Swt2Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fb, levels, L):
        ctx.fb, ctx.levels, ctx.L, ctx.hw = fb, levels, L, tuple(x.shape[-2:])
        f_lo, f_hi = _window_taps(fb, x.dtype, inverse=False)
        return run_analysis2(x, f_lo, f_hi, levels, L)

    @staticmethod
    def backward(ctx, g):
        return _Swt2AdjointFunction.apply(g, ctx.fb, ctx.levels, ctx.L, *ctx.hw), None, None, None


class _Swt2AdjointFunction(torch.autograd.Function):
    """The backward pass of swt2 as a differentiable map; its own adjoint is swt2, written into the packed layout
    with zeros in the pitch padding."""

    @staticmethod
    def forward(ctx, g, fb, levels, L, H, W):
        ctx.fb, ctx.levels, ctx.L, ctx.n, ctx.pitch = fb, levels, L, H * W, g.shape[-1]
        return _swt2_adjoint(g, fb, levels, L, H, W)

    @staticmethod
    def backward(ctx, u):
        packed = _Swt2Function.apply(u, ctx.fb, ctx.levels, ctx.L)
        return F.pad(packed[..., :ctx.n], (0, ctx.pitch - ctx.n)), None, None, None, None, None


class _Iswt2Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fb, L, approx, *details):
        ctx.fb, ctx.L, ctx.levels = fb, L, len(details) // 3
        g_lo, g_hi = _window_taps(fb, approx.dtype, inverse=True)
        return run_synthesis2(approx, details, g_lo, g_hi, L)

    @staticmethod
    def backward(ctx, gy):
        return (None, None) + _Iswt2AdjointFunction.apply(gy, ctx.fb, ctx.levels, ctx.L)


class _Iswt2AdjointFunction(torch.autograd.Function):
    """The backward pass of iswt2 as a differentiable map; its own adjoint is iswt2."""

    @staticmethod
    def forward(ctx, gy, fb, levels, L):
        ctx.fb, ctx.L = fb, L
        return _iswt2_adjoint(gy, fb, levels, L)

    @staticmethod
    def backward(ctx, *us):
        return _Iswt2Function.apply(ctx.fb, ctx.L, *us), None, None, None


def swt2(data: torch.Tensor, wavelet: Any, level: Optional[int] = None, *, axes: tuple[int, int] = (-2, -1)):
    """2-D stationary wavelet transform, ``(cA_J, (cH_J, cV_J, cD_J), ..., (cH_1, cV_1, cD_1))`` with the details as
    :class:`WaveletDetailTuple2d`, every band shaped like the input: PyWavelets' ``swt2`` with ``trim_approx=True``
    and ``norm=False``, in the container of :func:`wavedec2`.

    Level j (dilation d = 2^(j-1), hl = L/2 - 1, window taps f = dec[::-1]) computes, with a the filter along
    ``axes[0]`` and b the one along ``axes[1]``:

        c_ab[r, s] = sum_m sum_k f_a[m] f_b[k] A_{j-1}[(r + d (m - hl)) mod H, (s + d (k - hl)) mod W]

    cA = (lo, lo), cH = (hi, lo), cV = (lo, hi), cD = (hi, hi): the orientation of :func:`wavedec2`'s bands.  The
    extension is periodic at every level, also where d (L - 1) exceeds an extent (the reference has no ``swt2``, and
    its 1-D ``swt``'s multi-round padding is not copied here).  The default level is the largest that
    ``swt_max_level`` allows along both axes; a level <= 0 returns ``(data,)``.
    """
    check_tensor(data)
    check_dtype(data)
    x, f = fold(data, 2, axes)
    H, W = int(x.shape[-2]), int(x.shape[-1])
    if level is None:
        level = min(swt_max_level(H), swt_max_level(W))
    if level <= 0:
        return (unfold(x, f),)
    wav, fb, L = _filter_bank(wavelet, "swt2/iswt2")
    _check_taps_without_grad(wav, "swt2/iswt2")
    dev = _compute_device(x)
    on_host = not x.is_cuda
    with torch.cuda.device(dev):
        if torch.is_grad_enabled() and x.requires_grad:
            packed = _Swt2Function.apply(x.to(dev), fb, level, L)
            bands = _bands2(packed, level, H, W)
            if on_host:
                bands = [t.cpu() for t in bands]
        else:
            xd = x.to(dev, non_blocking=True) if on_host else x
            f_lo, f_hi = _window_taps(fb, x.dtype, inverse=False)
            packed = run_analysis2(xd, f_lo, f_hi, level, L)
            if on_host:
                host = pinned_empty(packed.shape, packed.dtype)
                host.copy_(packed, non_blocking=True)
                torch.cuda.current_stream(dev).synchronize()
                packed = host
            bands = _bands2(packed, level, H, W)
    out: list[Any] = [unfold(bands[0], f)]
    for k in range(level):
        h, v, d = bands[1 + 3 * k: 4 + 3 * k]
        out.append(WaveletDetailTuple2d(unfold(h, f), unfold(v, f), unfold(d, f)))
    return tuple(out)


def iswt2(coeffs, wavelet: Any, *, axes: AxisHint = None) -> torch.Tensor:
    """Inverse of :func:`swt2`: per level and axis the synthesis of include/wtb200.h with g = 0.5 rec, i.e. the mean
    of the four branches.  Reads :func:`swt2`'s own views without a copy; other layouts are gathered once."""
    lead = check_tensor(coeffs[0])
    check_dtype(lead)
    ensure_axes(axes, 2)
    for el in coeffs[1:]:
        if not isinstance(el, tuple) or len(el) != 3:
            raise ValueError(
                f"Unexpected detail coefficient type: {type(el)}. Detail coefficients must be a 3-tuple of "
                "tensors as returned by swt2."
            )
    flat: list[torch.Tensor] = [lead]
    for el in coeffs[1:]:
        flat.extend(el)
    folded, f = _fold_coeff_tensors(flat, 2, axes)
    _same_device_dtype(folded)
    approx, details = folded[0], folded[1:]
    if not details:
        return unfold(approx, f)
    for t in details:
        if t.shape != approx.shape:
            raise RuntimeError(f"all swt2 bands must have the same shape, got {list(approx.shape)} for the "
                               f"approximation and {list(t.shape)} for a detail")
    wav, fb, L = _filter_bank(wavelet, "swt2/iswt2")
    _check_taps_without_grad(wav, "swt2/iswt2")
    dev = _compute_device(approx)
    on_host = not approx.is_cuda
    with torch.cuda.device(dev):
        if torch.is_grad_enabled() and any(t.requires_grad for t in folded):
            y = _Iswt2Function.apply(fb, L, *[t.to(dev) for t in folded])
            return unfold(y.cpu() if on_host else y, f)
        if on_host:
            approx = approx.to(dev, non_blocking=True)
            details = [t.to(dev, non_blocking=True) for t in details]
        g_lo, g_hi = _window_taps(fb, approx.dtype, inverse=True)
        y = run_synthesis2(approx, details, g_lo, g_hi, L)
        if on_host:
            host = pinned_empty(y.shape, y.dtype)
            host.copy_(y, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            y = host
    return unfold(y, f)
