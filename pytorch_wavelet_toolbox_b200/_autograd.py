"""Differentiable path of the padded transforms (SURVEY.md section 8f, row 3).

The reference is differentiable by construction (it is a chain of torch operators); users train
through it (e.g. ``examples/network_compression/wavelet_linear.py:118,150``).  Under grad mode the
transforms therefore switch from the fused multi-level launch to a level-by-level chain whose only
non-torch nodes are two ``torch.autograd.Function`` s around the CUDA kernels:

* one analysis level with ZERO extension, whose adjoint is exactly one synthesis level with the
  flipped decomposition filters (the crop of the transposed convolution removes the zero padding);
* one synthesis level, whose adjoint is one zero-extension analysis level with the flipped
  reconstruction filters.

The boundary extension (reflect / constant / periodic / symmetric) happens INSIDE the analysis kernel on the forward
pass (``ModeLevelAnalysis``: no padded copy of the level input is made).  Because ``pad_left = L - 2`` is even, the
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
axes' synthesis passes -- with the output gradient (synthesis); ``wt_tap_corr`` (csrc/tap_grad.cuh) evaluates it.

Higher-order gradients (``create_graph=True``: gradient penalties, Hessian-vector products): the three Functions are
each other's adjoints, so when a backward pass runs in grad mode it computes the same quantities through the other
Function's ``apply`` with the flipped tap TENSORS (saved by every Function) instead of a raw launch, and the tap
correlation runs through ``TapCorrelation``, whose backward is one synthesis pass (signal side) and one zero-extension
analysis pass (coefficient side) with the cotangent as taps.  Every node of such a graph is again one of these four
Functions or differentiable index / pad / slice glue, so gradients of any order reach the data and the filters.  With
``create_graph=False`` the backward passes launch the kernels directly, as they always have.
"""
from __future__ import annotations

from typing import Any, Sequence

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


def _as_tap_tensor(seq, like: torch.Tensor) -> torch.Tensor:
    if isinstance(seq, torch.Tensor):
        return seq
    return torch.tensor([float(v) for v in seq], dtype=torch.float64)


def _axis_rows(t: torch.Tensor, axis: int) -> torch.Tensor:
    """[B, d1..dN] -> contiguous [rows, d_axis] with `axis` (0-based among the d's) last."""
    return t.movedim(1 + axis, -1).reshape(-1, t.shape[1 + axis]).contiguous()


def _rows_back(rows: torch.Tensor, like_shape: Sequence[int], axis: int, new_len: int) -> torch.Tensor:
    shp = list(like_shape)
    moved = [shp[0]] + [d for i, d in enumerate(shp[1:]) if i != axis] + [new_len]
    return rows.reshape(moved).movedim(-1, 1 + axis)


def _axis_adjoint_analysis(lo_band: torch.Tensor, hi_band: torch.Tensor, axis: int, out_len: int, dec_lo, dec_hi):
    """Adjoint of the zero-extension analysis pass along one axis: (lo, hi) bands -> signal of `out_len` samples."""
    from . import fwt

    rl, rh = _axis_rows(lo_band, axis), _axis_rows(hi_band, axis)
    wav = (None, None, list(dec_lo)[::-1], list(dec_hi)[::-1])
    f = fwt.Fold(1, (-1,), list(rl.shape))
    y = fwt._synthesis(rl, [[rh]], [rh], wav, 1, f)[:, :out_len]
    return _rows_back(y, lo_band.shape, axis, out_len)


def _axis_synthesis(lo_band: torch.Tensor, hi_band: torch.Tensor, axis: int, out_len: int, rec_lo, rec_hi):
    """One synthesis pass along one axis, cropped to `out_len` samples."""
    from . import fwt

    rl, rh = _axis_rows(lo_band, axis), _axis_rows(hi_band, axis)
    wav = (None, None, list(rec_lo), list(rec_hi))
    f = fwt.Fold(1, (-1,), list(rl.shape))
    y = fwt._synthesis(rl, [[rh]], [rh], wav, 1, f)[:, :out_len]
    return _rows_back(y, lo_band.shape, axis, out_len)


def _axis_pass_graph(lo_band: torch.Tensor, hi_band: torch.Tensor, axis: int, out_len: int, rec_lo_t: torch.Tensor,
                     rec_hi_t: torch.Tensor) -> torch.Tensor:
    """One synthesis pass along one axis through :class:`LevelSynthesis` (recorded by autograd), cropped to
    `out_len` samples; with ``rec := flipped dec`` it is the adjoint of the zero-extension analysis pass."""
    rl, rh = _axis_rows(lo_band, axis), _axis_rows(hi_band, axis)
    y = LevelSynthesis.apply(rec_lo_t, rec_hi_t, 1, rl, rh)[:, :out_len]
    return _rows_back(y, lo_band.shape, axis, out_len)


def _tap_corr(c_lo: torch.Tensor, c_hi: torch.Tensor, sig: torch.Tensor, axis: int, filt_len: int) -> torch.Tensor:
    """out[k, t] = sum c_k[.., i, ..] * sig[.., 2 i + t + 2 - L, ..] along `axis` (float64, on the device)."""
    rl, rh, rs = _axis_rows(c_lo, axis), _axis_rows(c_hi, axis), _axis_rows(sig, axis)
    return _tap_corr_rows(rl, rh, rs, filt_len)


def _tap_corr_rows(rl: torch.Tensor, rh: torch.Tensor, rs: torch.Tensor, filt_len: int) -> torch.Tensor:
    """:func:`_tap_corr` of contiguous rows ``[R, m]`` (coefficients) and ``[R, n]`` (signal): one wt_tap_corr launch."""
    from . import _native as N
    from .fwt import _dtype_code

    out = torch.empty(2 * filt_len, dtype=torch.float64, device=rs.device)
    with torch.cuda.device(rs.device):
        rc = N.load().wt_tap_corr(_dtype_code(rs.dtype), filt_len, rl.data_ptr(), rh.data_ptr(), rl.stride(0),
                                  rs.data_ptr(), rs.stride(0), rl.shape[0], rl.shape[1], rs.shape[1], out.data_ptr(),
                                  torch.cuda.current_stream(rs.device).cuda_stream)
    N.check(rc, "wt_tap_corr")
    return out.view(2, filt_len)


def _band_index(bits: Sequence[int]) -> int:
    k = 0
    for b in bits:
        k = 2 * k + b
    return k


def _tap_grads(bands: Sequence[torch.Tensor], sig: torch.Tensor, ndim: int, lo, hi, synthesis: bool) -> torch.Tensor:
    """Sum over the axes of the tap correlations.  `bands` are the 2^ndim band tensors (gradients for analysis,
    coefficients for synthesis) in the order k = sum_a hi(a) << (ndim-1-a); `sig` is the level input (analysis) or
    the gradient of the cropped level output (synthesis).  Returns [2, L] float64: row 0 lo taps, row 1 hi taps.

    Given the taps as tensors (grad mode), every pass and correlation is recorded by autograd."""
    import itertools

    if isinstance(lo, torch.Tensor):
        return _tap_grads_graph(bands, sig, ndim, lo, hi, synthesis)
    L = len(lo)
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
                key = bits[:a2] + (None,) + bits[a2 + 1:]
                n_out = sig.shape[1 + a2]
                nxt[key] = (_axis_synthesis(t, other, a2, n_out, lo, hi) if synthesis
                            else _axis_adjoint_analysis(t, other, a2, n_out, lo, hi))
            cur = nxt
        q_lo = next(t for bits, t in cur.items() if bits[a] == 0)
        q_hi = next(t for bits, t in cur.items() if bits[a] == 1)
        total += _tap_corr(q_lo, q_hi, sig, a, L)
    return total


def _tap_grads_graph(bands, sig: torch.Tensor, ndim: int, lo_t: torch.Tensor, hi_t: torch.Tensor,
                     synthesis: bool) -> torch.Tensor:
    """:func:`_tap_grads` with the passes through :class:`LevelSynthesis` and the correlations through
    :class:`TapCorrelation`, so that the result is differentiable in the bands, the signal and the taps."""
    import itertools

    rec_lo, rec_hi = (lo_t, hi_t) if synthesis else (_flipped(lo_t), _flipped(hi_t))
    L = lo_t.numel()
    terms = []
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
                nxt[bits[:a2] + (None,) + bits[a2 + 1:]] = _axis_pass_graph(t, other, a2, sig.shape[1 + a2], rec_lo,
                                                                            rec_hi)
            cur = nxt
        q_lo = next(t for bits, t in cur.items() if bits[a] == 0)
        q_hi = next(t for bits, t in cur.items() if bits[a] == 1)
        terms.append(TapCorrelation.apply(_axis_rows(q_lo, a), _axis_rows(q_hi, a), _axis_rows(sig, a), L))
    return sum(terms[1:], terms[0])


def _flipped(taps: torch.Tensor) -> torch.Tensor:
    return taps.reshape(-1).flip(0)


class TapCorrelation(torch.autograd.Function):
    """``out[k, t] = sum_{r, i} c_k[r, i] * s[r, 2 i + t + 2 - L]`` of coefficient rows ``c_lo, c_hi [R, m]`` and
    signal rows ``s [R, n]`` (wt_tap_corr) -> ``[2, L]`` float64.  It is bilinear; for the cotangent ``v [2, L]``
    ``d s[j] = sum_k sum_i c_k[i] v[k, j - 2 i + L - 2]`` is one synthesis pass of the coefficients with ``rec := v``
    (its crop of L - 2 samples gives exactly this index), and ``d c_k[i] = sum_t v[k, t] s[2 i + t + 2 - L]`` one
    zero-extension analysis pass of the signal with ``dec := flipped v``."""

    @staticmethod
    def forward(ctx, c_lo, c_hi, s, filt_len: int):
        c_lo, c_hi, s = c_lo.contiguous(), c_hi.contiguous(), s.contiguous()
        ctx.save_for_backward(c_lo, c_hi, s)
        return _tap_corr_rows(c_lo, c_hi, s, filt_len)

    @staticmethod
    def backward(ctx, v):
        c_lo, c_hi, s = ctx.saved_tensors
        g_lo = g_hi = g_s = None
        if ctx.needs_input_grad[2]:
            g_s = LevelSynthesis.apply(v[0], v[1], 1, c_lo, c_hi)[:, :s.shape[1]]
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            g_lo, g_hi = ZeroLevelAnalysis.apply(s, v[0].flip(0), v[1].flip(0), 1)
            if g_lo.shape != c_lo.shape:
                raise AssertionError("TapCorrelation: unexpected coefficient extents")
        return g_lo, g_hi, g_s, None


class ZeroLevelAnalysis(torch.autograd.Function):
    """One analysis level with zero extension: ``x [B, d..] -> 2^ndim bands``; the filters are tensor inputs."""

    @staticmethod
    def forward(ctx, x, dec_lo_t, dec_hi_t, ndim: int):
        from . import fwt

        dec_lo, dec_hi = _floats(dec_lo_t), _floats(dec_hi_t)
        wav = (list(dec_lo), list(dec_hi), list(dec_lo), list(dec_hi))
        approx, details, _ = fwt._analysis(x, wav, "zero", 1, None, ndim)
        ctx.taps = (dec_lo, dec_hi)
        ctx.ndim = ndim
        ctx.in_shape = tuple(x.shape)
        ctx.tap_meta = (dec_lo_t.dtype, dec_lo_t.device, tuple(dec_lo_t.shape), dec_hi_t.dtype, dec_hi_t.device,
                        tuple(dec_hi_t.shape))
        ctx.save_for_backward(x if (dec_lo_t.requires_grad or dec_hi_t.requires_grad) else None, dec_lo_t, dec_hi_t)
        return (approx,) + tuple(details[0])

    @staticmethod
    def backward(ctx, *grads):
        ref = next(g for g in grads if g is not None)
        bands = [g.contiguous() if g is not None else torch.zeros_like(ref) for g in grads]
        graph = torch.is_grad_enabled()   # create_graph=True: the tap tensors go through the other Functions
        x = tap_tensors = None
        if graph or ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            x, *taps = ctx.saved_tensors
            tap_tensors = tuple(taps) if graph else None
        gx, g_lo, g_hi = _zero_analysis_backward(bands, ctx.in_shape, ctx.taps, ctx.ndim, ctx.tap_meta, x,
                                                 ctx.needs_input_grad[:3], tap_tensors)
        return gx, g_lo, g_hi, None


def _zero_analysis_backward(bands, in_shape, taps, ndim: int, tap_meta, x, needs, tap_tensors=None):
    """Backward of one zero-extension analysis level of a signal of shape ``in_shape``: (gx, g_dec_lo, g_dec_hi).

    ``tap_tensors`` (grad mode only): the filters as tensors; the result is then recorded by autograd."""
    from . import fwt

    dec_lo, dec_hi = taps
    if tap_tensors is not None:
        dec_lo, dec_hi = tap_tensors
    gx = None
    if needs[0] and tap_tensors is not None:
        gx = LevelSynthesis.apply(_flipped(dec_lo), _flipped(dec_hi), ndim, *bands)
        gx = gx[(slice(None),) + tuple(slice(0, n) for n in in_shape[1:])]
    elif needs[0]:
        # adjoint of (zero pad -> stride-2 correlation) = transposed convolution with the same kernel,
        # cropped by the pad: the synthesis kernel with rec := flipped dec
        wav = (None, None, list(dec_lo)[::-1], list(dec_hi)[::-1])
        f = fwt.Fold(ndim, tuple(range(-ndim, 0)), list(in_shape))
        gx = fwt._synthesis(bands[0], [list(bands[1:])], [bands[1]], wav, ndim, f)
        sl = (slice(None),) + tuple(slice(0, n) for n in in_shape[1:])
        gx = gx[sl]
    g_lo = g_hi = None
    if needs[1] or needs[2]:
        d = _tap_grads(bands, x, ndim, dec_lo, dec_hi, synthesis=False).flip(1)   # d dec[m] = out[L - 1 - m]
        ldt, ldev, lshape, hdt, hdev, hshape = tap_meta
        if needs[1]:
            g_lo = d[0].to(device=ldev, dtype=ldt).reshape(lshape)
        if needs[2]:
            g_hi = d[1].to(device=hdev, dtype=hdt).reshape(hshape)
    return gx, g_lo, g_hi


class ModeLevelAnalysis(torch.autograd.Function):
    """One analysis level with the boundary extension of ``mode`` evaluated inside the kernel (no padded copy of the
    input); backward = fold(synthesis(band gradients in a zero field)), see the module docstring."""

    @staticmethod
    def forward(ctx, x, dec_lo_t, dec_hi_t, ndim: int, mode: str):
        from . import fwt

        dec_lo, dec_hi = _floats(dec_lo_t), _floats(dec_hi_t)
        wav = (list(dec_lo), list(dec_hi), list(dec_lo), list(dec_hi))
        approx, details, _ = fwt._analysis(x, wav, mode, 1, None, ndim)
        ctx.taps = (dec_lo, dec_hi)
        ctx.ndim = ndim
        ctx.mode = mode
        ctx.in_shape = tuple(x.shape)
        ctx.tap_meta = (dec_lo_t.dtype, dec_lo_t.device, tuple(dec_lo_t.shape), dec_hi_t.dtype, dec_hi_t.device,
                        tuple(dec_hi_t.shape))
        ctx.save_for_backward(x if (dec_lo_t.requires_grad or dec_hi_t.requires_grad) else None, dec_lo_t, dec_hi_t)
        return (approx,) + tuple(details[0])

    @staticmethod
    def backward(ctx, *grads):
        from . import _native as N

        ndim, mode = ctx.ndim, ctx.mode
        L = len(ctx.taps[0])
        dims = ctx.in_shape[1:]
        base = (2 * L - 3) // 2
        shift = base // 2
        ext_dims = tuple(n + 2 * base + n % 2 for n in dims)
        ref = next(g for g in grads if g is not None)
        m = tuple(ref.shape[1:])
        # S^T: the band gradients inside the zero field of the zero-extension transform of the extended signal
        flat: list[int] = []
        for a in reversed(range(ndim)):
            mp = N.coeff_len(ext_dims[a], L)
            flat += [shift, mp - m[a] - shift]
        bands = [F.pad(g if g is not None else torch.zeros_like(ref), flat) for g in grads]
        xp = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            xp = extend(ctx.saved_tensors[0], ndim, L, mode)   # recomputed here instead of kept from the forward pass
        tap_tensors = tuple(ctx.saved_tensors[1:]) if torch.is_grad_enabled() else None   # create_graph=True
        gxp, g_lo, g_hi = _zero_analysis_backward(bands, (ctx.in_shape[0],) + ext_dims, ctx.taps, ndim, ctx.tap_meta, xp,
                                                  ctx.needs_input_grad[:3], tap_tensors)
        gx = fold_extension(gxp, dims, L, mode) if gxp is not None else None
        return gx, g_lo, g_hi, None, None


class LevelSynthesis(torch.autograd.Function):
    """One synthesis level: ``2^ndim bands -> y [B, 2c - L + 2 ..]``; the filters are tensor inputs."""

    @staticmethod
    def forward(ctx, rec_lo_t, rec_hi_t, ndim: int, *bands):
        from . import fwt

        rec_lo, rec_hi = _floats(rec_lo_t), _floats(rec_hi_t)
        wav = (None, None, list(rec_lo), list(rec_hi))
        f = fwt.Fold(ndim, tuple(range(-ndim, 0)), list(bands[0].shape))
        y = fwt._synthesis(bands[0], [list(bands[1:])], [bands[1]], wav, ndim, f)
        ctx.taps = (rec_lo, rec_hi)
        ctx.ndim = ndim
        ctx.coeff_shape = tuple(bands[0].shape)
        ctx.tap_meta = (rec_lo_t.dtype, rec_lo_t.device, tuple(rec_lo_t.shape), rec_hi_t.dtype, rec_hi_t.device,
                        tuple(rec_hi_t.shape))
        if rec_lo_t.requires_grad or rec_hi_t.requires_grad:
            ctx.save_for_backward(rec_lo_t, rec_hi_t, *bands)
        else:
            ctx.save_for_backward(rec_lo_t, rec_hi_t)
        return y

    @staticmethod
    def backward(ctx, gy):
        from . import fwt

        graph = torch.is_grad_enabled()   # create_graph=True: the tap tensors go through the other Functions
        rec_lo, rec_hi = ctx.saved_tensors[:2] if graph else ctx.taps
        gy = gy.contiguous()
        out_bands = (None,) * (2 ** ctx.ndim)
        if any(ctx.needs_input_grad[3:]):
            # adjoint of (transposed convolution -> crop) = zero-extension analysis with dec := flipped rec
            if graph:
                out = ZeroLevelAnalysis.apply(gy, _flipped(rec_lo), _flipped(rec_hi), ctx.ndim)
            else:
                wav = (list(rec_lo)[::-1], list(rec_hi)[::-1], None, None)
                approx, details, _ = fwt._analysis(gy, wav, "zero", 1, None, ctx.ndim)
                out = [approx] + list(details[0])
            sl = (slice(None),) + tuple(slice(0, n) for n in ctx.coeff_shape[1:])
            out_bands = tuple(t[sl] for t in out)
        g_lo = g_hi = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            bands = [b.contiguous() for b in ctx.saved_tensors[2:]]
            d = _tap_grads(bands, gy, ctx.ndim, rec_lo, rec_hi, synthesis=True)       # d rec[t] = out[t]
            ldt, ldev, lshape, hdt, hdev, hshape = ctx.tap_meta
            if ctx.needs_input_grad[0]:
                g_lo = d[0].to(device=ldev, dtype=ldt).reshape(lshape)
            if ctx.needs_input_grad[1]:
                g_hi = d[1].to(device=hdev, dtype=hdt).reshape(hshape)
        return (g_lo, g_hi, None) + out_bands


def analysis_with_grad(x: torch.Tensor, dec_lo, dec_hi, mode: str, level: int, ndim: int, dev: torch.device):
    """Level-by-level differentiable analysis of folded data ``[B, d1..dN]``; returns
    (approx, [coarsest-first lists of bands k = 1..])."""
    from . import _native as N
    from ._shape import check_pad_feasible

    lo_t, hi_t = _as_tap_tensor(dec_lo, x), _as_tap_tensor(dec_hi, x)
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
        if mode == "zero":
            bands = ZeroLevelAnalysis.apply(cur, lo_t, hi_t, ndim)
        else:
            bands = ModeLevelAnalysis.apply(cur, lo_t, hi_t, ndim, mode)
        if tuple(bands[0].shape[1:]) != m:
            raise AssertionError("unexpected coefficient extents")
        details.append([b.to(home) for b in bands[1:]])
        cur = bands[0]
    details.reverse()
    return cur.to(home), details


def synthesis_with_grad(approx: torch.Tensor, levels_in, probes, rec_lo, rec_hi, ndim: int, dev: torch.device):
    """Level-by-level differentiable synthesis; arguments as fwt._synthesis (already validated)."""
    lo_t, hi_t = _as_tap_tensor(rec_lo, approx), _as_tap_tensor(rec_hi, approx)
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
