"""Differentiable path of the padded transforms (SURVEY.md section 8f, row 3).

The reference is differentiable by construction (it is a chain of torch operators); users train
through it (e.g. ``examples/network_compression/wavelet_linear.py:118,150``).  Under grad mode the
transforms therefore switch from the fused multi-level launch to a level-by-level chain whose only
non-torch nodes are ``torch.autograd.Function`` s around the CUDA kernels:

* ``LevelAnalysis``, one analysis level; with ZERO extension its adjoint is exactly one synthesis level with the
  flipped decomposition filters (the crop of the transposed convolution removes the zero padding);
* ``LevelSynthesis``, one synthesis level, whose adjoint is one zero-extension analysis level with the flipped
  reconstruction filters.

The boundary extension (reflect / constant / periodic / symmetric) happens INSIDE the analysis kernel on the forward
pass (no padded copy of the level input is made).  Because ``pad_left = L - 2`` is even, the
level outputs are the slice ``[pad_left/2 : pad_left/2 + M]`` of the zero-extension transform ``A0`` of the extended
signal ``E x``, so the backward pass is ``E^T A0^T S^T``: the band gradients are placed in a zero field (``S^T``), one
synthesis launch with the flipped decomposition filters gives the gradient of the extended signal (``A0^T``), and
``fold_extension`` adds every halo sample back onto the sample it was copied from (``E^T``; the source-index map is taken
from the forward extension itself, so every mode, including extensions longer than the signal, folds consistently).

Gradients with respect to the filter taps (learnable wavelets: the reference's filters are ``nn.Parameter`` s,
``src/ptwt/wavelets_learnable.py:167-189``, used by ``examples/network_compression/wavelet_linear.py:118,150``):
the filters enter the two Functions as tensor inputs.  Per axis the tap gradient is the correlation
``sum_i c[i] * s[2 i + t + 2 - L]`` of the band gradients -- carried through the ADJOINT of the other axes' passes
with the same single-axis kernels -- with the level input (analysis), or of the bands -- carried through the other
axes' synthesis passes -- with the output gradient (synthesis); ``TapCorrelation`` (``wt_tap_corr``,
csrc/tap_grad.cuh) evaluates it.

Every order of gradient runs through one backward path; only the origin of the taps differs.  Without grad mode
(``create_graph=False``) a backward pass takes the taps as the Python floats its forward pass kept: it launches exactly
the kernels it always launched and never reads device-resident taps back to the host.  In grad mode
(``create_graph=True``: gradient penalties, Hessian-vector products) it takes the saved tap TENSORS instead, so every
pass runs through the other Function's ``apply`` and autograd records it.  The Functions are each other's adjoints,
and ``TapCorrelation`` is bilinear: its backward is one synthesis pass (signal side) and one zero-extension analysis
pass (coefficient side) with the cotangent as taps.  Every node of such a graph is again one of these three Functions
or differentiable index / pad / slice glue, so gradients of any order reach the data and the filters.
"""
from __future__ import annotations

import itertools
from typing import Sequence

import torch
import torch.nn.functional as F

_TORCH_MODE = {"constant": "replicate", "zero": "constant", "reflect": "reflect", "periodic": "circular"}


def _floats(seq) -> tuple:
    if isinstance(seq, torch.Tensor):
        return tuple(float(v) for v in seq.detach().cpu().reshape(-1))
    return tuple(float(v) for v in seq)


def _sym_pad_axis(x: torch.Tensor, axis: int, left: int, right: int) -> torch.Tensor:
    n = x.shape[axis]
    if left > n or right > n:  # longer than the signal: extend in steps (reference _util.py:163-173)
        if left > n:
            x = _sym_pad_axis(x, axis, n, 0)
            left -= n
        if right > n:
            x = _sym_pad_axis(x, axis, 0, n)
            right -= n
        return _sym_pad_axis(x, axis, left, right)
    parts = [x]
    if left:
        parts.insert(0, x.narrow(axis, 0, left).flip(axis))
    if right:
        parts.append(x.narrow(axis, n - right, right).flip(axis))
    return torch.cat(parts, axis)


def extend(x: torch.Tensor, ndim: int, filt_len: int, mode: str) -> torch.Tensor:
    """Boundary extension of ``[B, d1..dN]`` by (L-2, L-2 + n%2) per axis with torch ops."""
    base = (2 * filt_len - 3) // 2
    pads = [(base, base + x.shape[1 + a] % 2) for a in range(ndim)]
    if mode == "symmetric":
        for a, (l, r) in enumerate(pads):
            x = _sym_pad_axis(x, 1 + a, l, r)
        return x
    flat: list[int] = []
    for l, r in reversed(pads):
        flat += [l, r]
    return F.pad(x.unsqueeze(1), flat, mode=_TORCH_MODE[mode]).squeeze(1)


_EXT_INDEX_CACHE: dict = {}


def _ext_source_index(n: int, filt_len: int, mode: str, device: torch.device) -> torch.Tensor:
    """For every position of the extended axis, the index of the sample of ``[0, n)`` it is a copy of."""
    key = (n, filt_len, mode, str(device))
    idx = _EXT_INDEX_CACHE.get(key)
    if idx is None:
        src = torch.arange(n, dtype=torch.float64).unsqueeze(0)
        idx = extend(src, 1, filt_len, mode)[0].round().to(torch.long).to(device)
        if len(_EXT_INDEX_CACHE) > 256:
            _EXT_INDEX_CACHE.clear()
        _EXT_INDEX_CACHE[key] = idx
    return idx


def fold_extension(gxp: torch.Tensor, dims: Sequence[int], filt_len: int, mode: str) -> torch.Tensor:
    """Adjoint of :func:`extend`: gradient of the extended ``[B, P1..PN]`` -> gradient of ``[B, d1..dN]``.

    The extension is separable, so the fold runs axis by axis: the interior is taken as is, every halo sample is
    added onto its source sample (``index_add_``)."""
    base = (2 * filt_len - 3) // 2
    g = gxp
    for a, n in enumerate(dims):
        left, right = base, base + n % 2
        ax = 1 + a
        if g.shape[ax] != n + left + right:
            raise AssertionError("fold_extension: unexpected extended length")
        idx = _ext_source_index(n, filt_len, mode, g.device)
        out = g.narrow(ax, left, n).clone()
        if left:
            out.index_add_(ax, idx[:left], g.narrow(ax, 0, left))
        if right:
            out.index_add_(ax, idx[left + n:], g.narrow(ax, left + n, right))
        g = out
    return g


def _as_tap_tensor(seq) -> torch.Tensor:
    if isinstance(seq, torch.Tensor):
        return seq
    return torch.tensor([float(v) for v in seq], dtype=torch.float64)


def _flip(taps):
    """A filter reversed: a tuple of floats, or a 1-D tensor (autograd records the flip)."""
    return taps.flip(0) if isinstance(taps, torch.Tensor) else tuple(taps)[::-1]


def _backward_taps(ctx) -> tuple:
    """The two filters a backward pass runs with.  In grad mode (``create_graph=True``) the tap tensors the forward
    pass saved first, so that autograd records their use; otherwise the floats it kept in ``ctx.taps``, which launch
    the kernels without reading device-resident taps back to the host."""
    if torch.is_grad_enabled():
        return tuple(t.reshape(-1) for t in ctx.saved_tensors[:2])
    return ctx.taps


def _tap_grad_inputs(ctx, d: torch.Tensor, needs: Sequence[bool]) -> tuple:
    """Rows 0 and 1 of the ``[2, L]`` float64 tap gradient ``d`` as the gradients of the two filter inputs (the first
    two saved tensors): in their dtype, on their device, in their shape; None where none is needed."""
    return tuple(d[k].to(device=t.device, dtype=t.dtype).reshape(t.shape) if needs[k] else None
                 for k, t in enumerate(ctx.saved_tensors[:2]))


def _analysis_level(x: torch.Tensor, dec_lo, dec_hi, ndim: int, mode: str) -> tuple:
    """One analysis level ``x [B, d..] -> (approx, *details)``.  Float taps launch the kernel directly; tensor taps
    go through :class:`LevelAnalysis`, which autograd records in grad mode."""
    if isinstance(dec_lo, torch.Tensor):
        return LevelAnalysis.apply(x, dec_lo, dec_hi, ndim, mode)
    from . import fwt

    approx, details, _ = fwt._analysis(x, (list(dec_lo), list(dec_hi), None, None), mode, 1, None, ndim)
    return (approx,) + tuple(details[0])


def _synthesis_level(rec_lo, rec_hi, ndim: int, bands: Sequence[torch.Tensor]) -> torch.Tensor:
    """One synthesis level of the 2^ndim ``bands``, uncropped.  Float taps launch the kernel directly; tensor taps go
    through :class:`LevelSynthesis`, which autograd records in grad mode."""
    if isinstance(rec_lo, torch.Tensor):
        return LevelSynthesis.apply(rec_lo, rec_hi, ndim, *bands)
    from . import fwt

    wav = (None, None, list(rec_lo), list(rec_hi))
    return fwt._synthesis(bands[0], [list(bands[1:])], [bands[1]], wav, ndim, None)


def _axis_rows(t: torch.Tensor, axis: int) -> torch.Tensor:
    """[B, d1..dN] -> contiguous [rows, d_axis] with `axis` (0-based among the d's) last."""
    return t.movedim(1 + axis, -1).reshape(-1, t.shape[1 + axis]).contiguous()


def _rows_back(rows: torch.Tensor, like_shape: Sequence[int], axis: int, new_len: int) -> torch.Tensor:
    shp = list(like_shape)
    moved = [shp[0]] + [d for i, d in enumerate(shp[1:]) if i != axis] + [new_len]
    return rows.reshape(moved).movedim(-1, 1 + axis)


def _axis_pass(lo_band: torch.Tensor, hi_band: torch.Tensor, axis: int, out_len: int, rec_lo, rec_hi):
    """One synthesis pass along one axis, cropped to `out_len` samples; with ``rec := flipped dec`` it is the adjoint
    of the zero-extension analysis pass."""
    rl, rh = _axis_rows(lo_band, axis), _axis_rows(hi_band, axis)
    y = _synthesis_level(rec_lo, rec_hi, 1, (rl, rh))[:, :out_len]
    return _rows_back(y, lo_band.shape, axis, out_len)


def _band_index(bits: Sequence[int]) -> int:
    k = 0
    for b in bits:
        k = 2 * k + b
    return k


def _tap_grads(bands: Sequence[torch.Tensor], sig: torch.Tensor, ndim: int, rec_lo, rec_hi) -> torch.Tensor:
    """Sum over the axes of the tap correlations.  `bands` are the 2^ndim band tensors (gradients for analysis,
    coefficients for synthesis) in the order k = sum_a hi(a) << (ndim-1-a); `sig` is the level input (analysis) or
    the gradient of the cropped level output (synthesis); `rec_lo, rec_hi` are the taps of the synthesis passes that
    carry the bands across the other axes (the flipped decomposition filters for analysis).  Returns [2, L] float64:
    row 0 lo taps, row 1 hi taps."""
    L = len(rec_lo)
    total = torch.zeros(2, L, dtype=torch.float64, device=sig.device)
    for a in range(ndim):
        cur = {bits: bands[_band_index(bits)] for bits in itertools.product((0, 1), repeat=ndim)}
        for a2 in range(ndim):
            if a2 == a:
                continue
            nxt = {}
            for bits, t in cur.items():
                if bits[a2] != 0:
                    continue
                other = cur[bits[:a2] + (1,) + bits[a2 + 1:]]
                nxt[bits[:a2] + (None,) + bits[a2 + 1:]] = _axis_pass(t, other, a2, sig.shape[1 + a2], rec_lo, rec_hi)
            cur = nxt
        q_lo = next(t for bits, t in cur.items() if bits[a] == 0)
        q_hi = next(t for bits, t in cur.items() if bits[a] == 1)
        total += TapCorrelation.apply(_axis_rows(q_lo, a), _axis_rows(q_hi, a), _axis_rows(sig, a), L)
    return total


class TapCorrelation(torch.autograd.Function):
    """``out[k, t] = sum_{r, i} c_k[r, i] * s[r, 2 i + t + 2 - L]`` of coefficient rows ``c_lo, c_hi [R, m]`` and
    signal rows ``s [R, n]`` (one wt_tap_corr launch) -> ``[2, L]`` float64.  It is bilinear; for the cotangent
    ``v [2, L]`` ``d s[j] = sum_k sum_i c_k[i] v[k, j - 2 i + L - 2]`` is one synthesis pass of the coefficients with
    ``rec := v`` (its crop of L - 2 samples gives exactly this index), and ``d c_k[i] = sum_t v[k, t] s[2 i + t + 2 - L]``
    one zero-extension analysis pass of the signal with ``dec := flipped v``."""

    @staticmethod
    def forward(ctx, c_lo, c_hi, s, filt_len: int):
        from . import _native as N
        from .fwt import _dtype_code

        c_lo, c_hi, s = c_lo.contiguous(), c_hi.contiguous(), s.contiguous()
        ctx.save_for_backward(c_lo, c_hi, s)
        out = torch.empty(2 * filt_len, dtype=torch.float64, device=s.device)
        with torch.cuda.device(s.device):
            rc = N.load().wt_tap_corr(_dtype_code(s.dtype), filt_len, c_lo.data_ptr(), c_hi.data_ptr(), c_lo.stride(0),
                                      s.data_ptr(), s.stride(0), c_lo.shape[0], c_lo.shape[1], s.shape[1],
                                      out.data_ptr(), torch.cuda.current_stream(s.device).cuda_stream)
        N.check(rc, "wt_tap_corr")
        return out.view(2, filt_len)

    @staticmethod
    def backward(ctx, v):
        c_lo, c_hi, s = ctx.saved_tensors
        g_lo = g_hi = g_s = None
        if ctx.needs_input_grad[2]:
            g_s = LevelSynthesis.apply(v[0], v[1], 1, c_lo, c_hi)[:, :s.shape[1]]
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            g_lo, g_hi = LevelAnalysis.apply(s, v[0].flip(0), v[1].flip(0), 1, "zero")
            if g_lo.shape != c_lo.shape:
                raise AssertionError("TapCorrelation: unexpected coefficient extents")
        return g_lo, g_hi, g_s, None


def _zero_analysis_backward(ctx, bands, in_shape, x, dec_lo, dec_hi):
    """Backward of one zero-extension analysis level of a signal `x` of shape ``in_shape``: (gx, g_dec_lo, g_dec_hi).
    `x` is needed (and given) only when a filter needs its gradient."""
    needs = ctx.needs_input_grad
    rec_lo, rec_hi = _flip(dec_lo), _flip(dec_hi)
    gx = g_lo = g_hi = None
    if needs[0]:
        # adjoint of (zero pad -> stride-2 correlation) = transposed convolution with the same kernel,
        # cropped by the pad: the synthesis kernel with rec := flipped dec
        gx = _synthesis_level(rec_lo, rec_hi, ctx.ndim, bands)
        gx = gx[(slice(None),) + tuple(slice(0, n) for n in in_shape[1:])]
    if needs[1] or needs[2]:
        d = _tap_grads(bands, x, ctx.ndim, rec_lo, rec_hi).flip(1)   # d dec[m] = out[L - 1 - m]
        g_lo, g_hi = _tap_grad_inputs(ctx, d, needs[1:3])
    return gx, g_lo, g_hi


class LevelAnalysis(torch.autograd.Function):
    """One analysis level ``x [B, d..] -> 2^ndim bands`` with the boundary extension of ``mode`` evaluated inside the
    kernel (no padded copy of the input); the filters are tensor inputs.  Backward: zero mode synthesises and crops;
    the other modes pad, synthesise and fold, see the module docstring."""

    @staticmethod
    def forward(ctx, x, dec_lo_t, dec_hi_t, ndim: int, mode: str):
        ctx.taps = (_floats(dec_lo_t), _floats(dec_hi_t))
        ctx.ndim, ctx.mode, ctx.in_shape = ndim, mode, tuple(x.shape)
        ctx.save_for_backward(dec_lo_t, dec_hi_t, x if (dec_lo_t.requires_grad or dec_hi_t.requires_grad) else None)
        return _analysis_level(x, *ctx.taps, ndim, mode)

    @staticmethod
    def backward(ctx, *grads):
        from . import _native as N

        ndim, mode = ctx.ndim, ctx.mode
        dec_lo, dec_hi = _backward_taps(ctx)
        x = ctx.saved_tensors[2] if ctx.needs_input_grad[1] or ctx.needs_input_grad[2] else None
        ref = next(g for g in grads if g is not None)
        if mode == "zero":
            bands = [g.contiguous() if g is not None else torch.zeros_like(ref) for g in grads]
            return _zero_analysis_backward(ctx, bands, ctx.in_shape, x, dec_lo, dec_hi) + (None, None)
        L = len(ctx.taps[0])
        dims = ctx.in_shape[1:]
        base = (2 * L - 3) // 2
        shift = base // 2
        ext_dims = tuple(n + 2 * base + n % 2 for n in dims)
        m = tuple(ref.shape[1:])
        # S^T: the band gradients inside the zero field of the zero-extension transform of the extended signal
        flat: list[int] = []
        for a in reversed(range(ndim)):
            mp = N.coeff_len(ext_dims[a], L)
            flat += [shift, mp - m[a] - shift]
        bands = [F.pad(g if g is not None else torch.zeros_like(ref), flat) for g in grads]
        xp = extend(x, ndim, L, mode) if x is not None else None   # recomputed here instead of kept from the forward
        gxp, g_lo, g_hi = _zero_analysis_backward(ctx, bands, (ctx.in_shape[0],) + ext_dims, xp, dec_lo, dec_hi)
        gx = fold_extension(gxp, dims, L, mode) if gxp is not None else None
        return gx, g_lo, g_hi, None, None


class LevelSynthesis(torch.autograd.Function):
    """One synthesis level: ``2^ndim bands -> y [B, 2c - L + 2 ..]``; the filters are tensor inputs."""

    @staticmethod
    def forward(ctx, rec_lo_t, rec_hi_t, ndim: int, *bands):
        ctx.taps = (_floats(rec_lo_t), _floats(rec_hi_t))
        ctx.ndim, ctx.coeff_shape = ndim, tuple(bands[0].shape)
        if rec_lo_t.requires_grad or rec_hi_t.requires_grad:
            ctx.save_for_backward(rec_lo_t, rec_hi_t, *bands)
        else:
            ctx.save_for_backward(rec_lo_t, rec_hi_t)
        return _synthesis_level(*ctx.taps, ndim, bands)

    @staticmethod
    def backward(ctx, gy):
        rec_lo, rec_hi = _backward_taps(ctx)
        gy = gy.contiguous()
        out_bands = (None,) * (2 ** ctx.ndim)
        if any(ctx.needs_input_grad[3:]):
            # adjoint of (transposed convolution -> crop) = zero-extension analysis with dec := flipped rec
            out = _analysis_level(gy, _flip(rec_lo), _flip(rec_hi), ctx.ndim, "zero")
            sl = (slice(None),) + tuple(slice(0, n) for n in ctx.coeff_shape[1:])
            out_bands = tuple(t[sl] for t in out)
        g_lo = g_hi = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            bands = [b.contiguous() for b in ctx.saved_tensors[2:]]
            d = _tap_grads(bands, gy, ctx.ndim, rec_lo, rec_hi)       # d rec[t] = out[t]
            g_lo, g_hi = _tap_grad_inputs(ctx, d, ctx.needs_input_grad[:2])
        return (g_lo, g_hi, None) + out_bands


def analysis_with_grad(x: torch.Tensor, dec_lo, dec_hi, mode: str, level: int, ndim: int, dev: torch.device):
    """Level-by-level differentiable analysis of folded data ``[B, d1..dN]``; returns
    (approx, [coarsest-first lists of bands k = 1..])."""
    from . import _native as N
    from ._shape import check_pad_feasible

    lo_t, hi_t = _as_tap_tensor(dec_lo), _as_tap_tensor(dec_hi)
    L = int(lo_t.numel())
    if L % 2:
        raise NotImplementedError("the differentiable path needs an even filter length")
    home = x.device
    cur = x.to(dev)
    details = []
    for _ in range(level):
        dims = tuple(cur.shape[1:])
        check_pad_feasible(mode, dims, L)
        m = tuple(N.coeff_len(n, L) for n in dims)
        bands = LevelAnalysis.apply(cur, lo_t, hi_t, ndim, mode)
        if tuple(bands[0].shape[1:]) != m:
            raise AssertionError("unexpected coefficient extents")
        details.append([b.to(home) for b in bands[1:]])
        cur = bands[0]
    details.reverse()
    return cur.to(home), details


def synthesis_with_grad(approx: torch.Tensor, levels_in, probes, rec_lo, rec_hi, ndim: int, dev: torch.device):
    """Level-by-level differentiable synthesis; arguments as fwt._synthesis (already validated)."""
    lo_t, hi_t = _as_tap_tensor(rec_lo), _as_tap_tensor(rec_hi)
    home = approx.device
    cur = approx.to(dev)
    for i, bands in enumerate(levels_in):
        want = tuple(bands[0].shape[1:])
        if tuple(cur.shape[1:]) != want:
            raise ValueError("All coefficients on each level must have the same shape")
        y = LevelSynthesis.apply(lo_t, hi_t, ndim, cur, *[b.to(dev) for b in bands])
        if i + 1 < len(levels_in):
            nxt = tuple(probes[i + 1].shape[1:])
            sl = [slice(None)]
            for a in range(ndim):
                if nxt[a] == y.shape[1 + a]:
                    sl.append(slice(None))
                elif nxt[a] == y.shape[1 + a] - 1:
                    sl.append(slice(0, nxt[a]))
                else:
                    raise AssertionError("padding error, please check if dec and rec wavelets are identical.")
            y = y[tuple(sl)]
        cur = y
    return cur.to(home)
