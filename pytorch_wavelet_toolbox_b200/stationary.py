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
"""
from __future__ import annotations

import ctypes as C
import functools
from typing import Any, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import _native as N
from ._shape import AxisHint, check_dtype, check_tensor, fold, round_up, unfold
from ._wavelets import any_requires_grad, as_wavelet, filter_bank, swt_max_level, taps_in_dtype
from .fwt import ROW_ALIGN_BYTES, _compute_device, _dtype_code, _pack_bands, _same_device_dtype, pinned_empty

__all__ = ["swt", "iswt"]


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


def _check_taps_without_grad(wav: Any) -> None:
    if torch.is_grad_enabled() and any_requires_grad(wav):
        raise NotImplementedError(
            "swt/iswt compute gradients with respect to the data only, not with respect to learnable filter taps; "
            "pass plain filters or call under torch.no_grad()."
        )


def _filter_bank(wavelet: Any):
    wav = as_wavelet(wavelet)
    fb = filter_bank(wav)
    L = len(fb[0])
    if any(len(f) != L for f in fb):
        raise ValueError("all four filters of the wavelet must have the same length")
    if L < 2 or L > N.WT_MAX_FILT_LEN or L % 2:
        raise ValueError(f"swt/iswt need an even filter length in 2..{N.WT_MAX_FILT_LEN}, got {L}")
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
