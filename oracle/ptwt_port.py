"""CPU restatement ("port") of the reference's hot path -- TEST INFRASTRUCTURE ONLY.

This file is the oracle the CUDA path is checked against and the ``cpu_baseline`` / ``--impl
reference`` arm of bench.py (kind "port").  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s CPU-baseline legs may import it; the product package never does.

It follows the reference's algorithm step by step, with the same torch CPU operators the reference
calls (so its speed is representative of ptwt on the host cores), written as one N-dimensional code
path instead of the reference's three per-dimension modules:

  analysis  level loop   pad -> conv{1,2,3}d(stride=2) with outer-product filters -> split
                         /root/reference/src/ptwt/conv_transform.py:133-141
                         /root/reference/src/ptwt/conv_transform_2.py:142-149
                         /root/reference/src/ptwt/conv_transform_3.py:122-141
  synthesis level loop   stack -> conv_transpose{1,2,3}d(stride=2) -> crop (+1 when the next detail is shorter)
                         conv_transform.py:184-199, conv_transform_2.py:208-249, conv_transform_3.py:191-249
  padding amounts        (2L-3)//2 left, that + n%2 right                     _util.py:198-228
  symmetric padding      cat of flipped slices, recursive when pad > length   _util.py:163-195
  filters                analysis: flipped dec_*, synthesis: un-flipped rec_* _util.py:95-141
                         N-d filters: outer products, first letter = slowest  _util.py:881-936
  folding                move axes last, add / fold batch dims                _util.py:493-570, 613-676
  matrix FWT             sameshift strided conv matrix, rows with nnz != L replaced by a dense QR
                         matmul_transform.py:47-165, 310-430, 603-703; sparse_math.py:253-311, 350-405, 482-516

Parity is PINNED: tests/test_oracle.py compares every function here with the committed golden fixtures
under tests/golden/ that oracle/make_golden*.py generated from the unmodified reference.
"""
from __future__ import annotations

import itertools
import math
import sys
from typing import Any, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet, dwt_max_level, dwtn_max_level, filter_bank
from pytorch_wavelet_toolbox_b200.constants import DETAIL_KEYS_3D, WaveletDetailTuple2d

_TORCH_MODE = {"constant": "replicate", "zero": "constant", "reflect": "reflect", "periodic": "circular",
               "symmetric": "symmetric"}
_CONV = {1: F.conv1d, 2: F.conv2d, 3: F.conv3d}
_CONVT = {1: F.conv_transpose1d, 2: F.conv_transpose2d, 3: F.conv_transpose3d}


# ---------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------
def _taps(wavelet: Any, dtype: torch.dtype, flip: bool):
    bank = filter_bank(as_wavelet(wavelet))
    out = []
    for f in bank:
        # tensors keep their autograd graph (the reference differentiates through learnable filters, _util.py:129-141)
        t = (f.cpu() if isinstance(f, torch.Tensor) else torch.tensor(list(map(float, f)), dtype=torch.float64)).to(dtype)
        out.append(t.flip(-1) if flip else t)
    return out  # dec_lo, dec_hi, rec_lo, rec_hi


def _nd_filters(lo: torch.Tensor, hi: torch.Tensor, ndim: int) -> torch.Tensor:
    """[2^ndim, 1, L, ..] outer-product filters in the reference's order (_util.py:881-936):
    1-D (lo, hi); 2-D ll, lh, hl, hh with lh = outer(hi, lo); 3-D lll, llh, ..., hhh."""
    if ndim == 1:
        return torch.stack([lo, hi], 0).unsqueeze(1)
    if ndim == 2:
        pairs = [(lo, lo), (hi, lo), (lo, hi), (hi, hi)]
        return torch.stack([torch.outer(a, b) for a, b in pairs], 0).unsqueeze(1)
    combos = itertools.product([lo, hi], repeat=3)
    # a (x) (b (x) c): the same association as the reference's _outer(a, _outer(b, c)) so that the
    # products round identically
    return torch.stack([a.reshape(-1, 1, 1) * torch.outer(b, c).unsqueeze(0) for a, b, c in combos], 0).unsqueeze(1)


def _sym_pad_axis(x: torch.Tensor, axis: int, left: int, right: int) -> torch.Tensor:
    n = x.shape[axis]
    if left > n or right > n:
        if left > n:
            x = _sym_pad_axis(x, axis, n, 0)
            left -= n
        if right > n:
            x = _sym_pad_axis(x, axis, 0, n)
            right -= n
        return _sym_pad_axis(x, axis, left, right)
    parts = [x]
    if left > 0:
        parts.insert(0, x.narrow(axis, 0, left).flip(axis))
    if right > 0:
        parts.append(x.narrow(axis, n - right, right).flip(axis))
    return torch.cat(parts, axis)


def _pad(x: torch.Tensor, ndim: int, filt_len: int, mode: str) -> torch.Tensor:
    """x [B, 1, d1..dN] -> padded copy."""
    if mode not in _TORCH_MODE:
        raise ValueError(f"Padding mode not supported: {mode}")
    base = (2 * filt_len - 3) // 2
    pads = [(base, base + x.shape[2 + a] % 2) for a in range(ndim)]
    if mode == "symmetric":
        for a, (l, r) in enumerate(pads):
            x = _sym_pad_axis(x, 2 + a, l, r)
        return x
    flat: list[int] = []
    for l, r in reversed(pads):
        flat += [l, r]
    return F.pad(x, flat, mode=_TORCH_MODE[mode])


def _fold(t: torch.Tensor, ndim: int, axes: Sequence[int], lead_rank: Optional[int] = None):
    if t.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"Input dtype {t.dtype} not supported")
    default = tuple(range(-ndim, 0))
    if tuple(axes) != default:
        if len(set(axes)) != len(axes):
            raise ValueError("Cant transform the same axis twice.")
        t = torch.movedim(t, tuple(axes), default)
    shape = list(t.shape)
    rank = lead_rank if lead_rank is not None else len(shape)
    if rank < ndim:
        raise ValueError(f"At least {ndim} input dimensions required.")
    if rank == ndim:
        t = t.unsqueeze(0)
    elif rank > ndim + 1:
        t = t.reshape([math.prod(t.shape[:-ndim])] + list(t.shape[-ndim:]))
    return t, shape


def _unfold(t: torch.Tensor, ndim: int, axes: Sequence[int], lead_shape: Sequence[int]) -> torch.Tensor:
    rank = len(lead_shape)
    if rank == ndim:
        t = t.squeeze(0)
    elif rank > ndim + 1:
        t = t.reshape(list(lead_shape[:-ndim]) + list(t.shape[-ndim:]))
    default = tuple(range(-ndim, 0))
    if tuple(axes) != default:
        t = torch.movedim(t, default, tuple(axes))
    return t


def _axes(axes, ndim):
    if axes is None:
        return tuple(range(-ndim, 0))
    if isinstance(axes, int):
        if ndim != 1:
            raise ValueError(f"tried passing single axis to {ndim}D transform")
        return (axes,)
    if len(axes) != ndim:
        raise ValueError(f"tried passing {len(axes)}D axes {axes} to {ndim}D transform")
    if len(set(axes)) != len(axes):
        raise ValueError("Cant transform the same axis twice.")
    return tuple(axes)


# ---------------------------------------------------------------------------------------------
# level loops on folded data
# ---------------------------------------------------------------------------------------------
def analysis_levels(x: torch.Tensor, wavelet: Any, mode: str, level: int, ndim: int):
    """x [B, d1..dN] -> (approx [B,..], [finest..coarsest: tensor [B, 2^ndim, ..] incl. band 0])."""
    dec_lo, dec_hi, _, _ = _taps(wavelet, x.dtype, flip=True)
    filt = _nd_filters(dec_lo, dec_hi, ndim).to(x.device)  # the reference builds its filters on data.device
    cur = x.unsqueeze(1)
    outs = []
    for _ in range(level):
        cur = _pad(cur, ndim, dec_lo.shape[0], mode)
        res = _CONV[ndim](cur, filt, stride=2)
        outs.append(res)
        cur = res[:, 0:1]
    return cur.squeeze(1), outs


def synthesis_levels(approx: torch.Tensor, levels: Sequence[Sequence[torch.Tensor]], wavelet: Any, ndim: int):
    """approx [B,..]; levels coarsest-first, each the 2^ndim - 1 detail bands in the reference's order."""
    _, _, rec_lo, rec_hi = _taps(wavelet, approx.dtype, flip=False)
    L = rec_lo.shape[0]
    filt = _nd_filters(rec_lo, rec_hi, ndim).to(approx.device)
    cur = approx
    base = (2 * L - 3) // 2
    for i, bands in enumerate(levels):
        if ndim > 1:
            for b in bands:
                if b.shape != cur.shape:
                    raise ValueError("All coefficients on each level must have the same shape")
        stacked = torch.stack([cur] + list(bands), 1)
        cur = _CONVT[ndim](stacked, filt, stride=2).squeeze(1)
        for a in range(ndim):
            left, right = base, base
            if i + 1 < len(levels):
                pred = cur.shape[1 + a] - (left + right)
                nxt = levels[i + 1][0].shape[1 + a]
                if nxt == pred - 1:
                    right += 1
                elif nxt != pred:
                    raise AssertionError("padding error, please check if dec and rec wavelets are identical.")
            cur = cur.narrow(1 + a, left, cur.shape[1 + a] - left - right)
    return cur


# ---------------------------------------------------------------------------------------------
# reference-shaped API
# ---------------------------------------------------------------------------------------------
def _filt_len(wavelet: Any) -> int:
    return len(filter_bank(as_wavelet(wavelet))[0])


def wavedec(data, wavelet, *, mode="reflect", level=None, axis=-1):
    ax = _axes(axis, 1)
    x, shape = _fold(data, 1, ax)
    if level is None:
        level = dwt_max_level(x.shape[-1], _filt_len(wavelet))
    approx, outs = analysis_levels(x, wavelet, mode, level, 1)
    res = [approx] + [o[:, 1] for o in reversed(outs)]
    return [_unfold(t, 1, ax, shape) for t in res]


def waverec(coeffs, wavelet, *, axis=None):
    ax = _axes(axis, 1)
    coeffs = list(coeffs)
    lead, shape = _fold(coeffs[0], 1, ax)
    rest = [_fold(c, 1, ax, len(shape))[0] for c in coeffs[1:]]
    y = synthesis_levels(lead, [[c] for c in rest], wavelet, 1)
    return _unfold(y, 1, ax, shape)


def wavedec2(data, wavelet, *, mode="reflect", level=None, axes=(-2, -1)):
    ax = _axes(axes, 2)
    x, shape = _fold(data, 2, ax)
    if level is None:
        level = dwtn_max_level(x.shape[-2:], _filt_len(wavelet))
    approx, outs = analysis_levels(x, wavelet, mode, level, 2)
    res: list[Any] = [_unfold(approx, 2, ax, shape)]
    for o in reversed(outs):
        res.append(WaveletDetailTuple2d(*[_unfold(o[:, k], 2, ax, shape) for k in (1, 2, 3)]))
    return tuple(res)


def waverec2(coeffs, wavelet, *, axes=None):
    ax = _axes(axes, 2)
    lead, shape = _fold(coeffs[0], 2, ax)
    levels = []
    for el in coeffs[1:]:
        if not isinstance(el, tuple) or len(el) != 3:
            raise ValueError(f"Unexpected detail coefficient type: {type(el)}.")
        levels.append([_fold(t, 2, ax, len(shape))[0] for t in el])
    return _unfold(synthesis_levels(lead, levels, wavelet, 2), 2, ax, shape)


def wavedec3(data, wavelet, *, mode="zero", level=None, axes=(-3, -2, -1)):
    ax = _axes(axes, 3)
    x, shape = _fold(data, 3, ax)
    if level is None:
        level = dwtn_max_level(x.shape[-3:], _filt_len(wavelet))
    approx, outs = analysis_levels(x, wavelet, mode, level, 3)
    res: list[Any] = [_unfold(approx, 3, ax, shape)]
    for o in reversed(outs):
        res.append({key: _unfold(o[:, k + 1], 3, ax, shape) for k, key in enumerate(DETAIL_KEYS_3D)})
    return tuple(res)


def waverec3(coeffs, wavelet, *, axes=None):
    ax = _axes(axes, 3)
    lead, shape = _fold(coeffs[0], 3, ax)
    levels = []
    for el in coeffs[1:]:
        if not isinstance(el, dict) or len(el) != 7:
            raise ValueError(f"Unexpected detail coefficient type: {type(el)}.")
        levels.append([_fold(el[k], 3, ax, len(shape))[0] for k in DETAIL_KEYS_3D])
    return _unfold(synthesis_levels(lead, levels, wavelet, 3), 3, ax, shape)


# ---------------------------------------------------------------------------------------------
# boundary-filter matrix FWT
# ---------------------------------------------------------------------------------------------
def strided_conv_matrix(filt: torch.Tensor, n: int) -> torch.Tensor:
    """Dense "sameshift" stride-2 convolution matrix [n/2.., n] (sparse_math.py:350-405, 482-516):
    full[r, c] = filt[r - c]; keep rows start .. start + n - 1 with start = L//2 - 1 + L%2; of those
    every second one beginning with the second (rows 1::2)."""
    L = filt.shape[0]
    start = L // 2 - 1 + L % 2
    rows = torch.arange(1, n, 2) + start
    cols = torch.arange(n)
    k = rows.reshape(-1, 1) - cols.reshape(1, -1)
    valid = (k >= 0) & (k < L)
    mat = torch.zeros((rows.shape[0], n), dtype=filt.dtype)
    mat[valid] = filt[k[valid]]
    return mat, valid.sum(1)


def boundary_matrix(lo: torch.Tensor, hi: torch.Tensor, n: int, method: str = "qr") -> torch.Tensor:
    """Dense orthogonalised level operator [n, n] (matmul_transform.py:74-81, 121-165;
    sparse_math.py:269-311 / 314-347)."""
    a_lo, nnz_lo = strided_conv_matrix(lo, n)
    a_hi, nnz_hi = strided_conv_matrix(hi, n)
    mat = torch.cat([a_lo, a_hi], 0)
    nnz = torch.cat([nnz_lo, nnz_hi])
    rows = (nnz != lo.shape[0]).nonzero().reshape(-1)
    if rows.numel() == 0:
        return mat
    sel = mat[rows]
    if method == "qr":
        q, _ = torch.linalg.qr(sel.T)
        new = q.T
    elif method == "gramschmidt":
        new = sel.clone()
        for p in range(new.shape[0]):
            cur = new[p].clone()
            acc = torch.zeros_like(cur)
            for d in range(p):
                acc += torch.dot(cur, new[d]) * new[d]
            cur = cur - acc
            new[p] = cur / torch.linalg.vector_norm(cur)
    else:
        raise ValueError(f"Invalid orthogonalization method: {method}")
    mat = mat.clone()
    mat[rows] = new
    return mat


def boundary_matrix_sparse(lo: torch.Tensor, hi: torch.Tensor, n: int, method: str = "qr") -> torch.Tensor:
    """``boundary_matrix(lo, hi, n, method).to_sparse()`` assembled from its O(n L) entries: the same values, the same
    orthogonalised boundary rows, without the dense [n, n] operator (34 GB of float64 at n = 65536)."""
    L = lo.shape[0]
    start = L // 2 - 1 + L % 2
    r = torch.arange(1, n, 2) + start
    m = r.shape[0]
    cols = r.reshape(-1, 1) - torch.arange(L).reshape(1, -1)          # column of tap k in conv row i
    valid = (cols >= 0) & (cols < n)
    inner = valid.sum(1) == L
    idx_i, idx_j, vals, sel = [], [], [], []
    for b, filt in enumerate((lo, hi)):
        taps = filt.reshape(1, -1).expand(m, L)
        keep = valid & inner.reshape(-1, 1)
        idx_i.append((torch.arange(m).reshape(-1, 1) + b * m).expand(m, L)[keep])
        idx_j.append(cols[keep])
        vals.append(taps[keep])
        for i in (~inner).nonzero().reshape(-1).tolist():
            row = torch.zeros(n, dtype=filt.dtype)
            row[cols[i][valid[i]]] = filt[valid[i]]
            sel.append((b * m + i, row))
    if sel:
        rows = torch.stack([row for _, row in sel])
        if method == "qr":
            q, _ = torch.linalg.qr(rows.T)
            new = q.T
        elif method == "gramschmidt":
            new = rows.clone()
            for p in range(new.shape[0]):
                cur = new[p].clone()
                acc = torch.zeros_like(cur)
                for d in range(p):
                    acc += torch.dot(cur, new[d]) * new[d]
                cur = cur - acc
                new[p] = cur / torch.linalg.vector_norm(cur)
        else:
            raise ValueError(f"Invalid orthogonalization method: {method}")
        for (i, _), row in zip(sel, new):
            nz = (row != 0).nonzero().reshape(-1)
            idx_i.append(torch.full_like(nz, i))
            idx_j.append(nz)
            vals.append(row[nz])
    i, j, v = torch.cat(idx_i), torch.cat(idx_j), torch.cat(vals)
    nz = v != 0
    return torch.sparse_coo_tensor(torch.stack([i[nz], j[nz]]), v[nz], (2 * m, n)).coalesce()


def _odd_pad(x: torch.Tensor, mode: str) -> torch.Tensor:
    """One sample appended on the right of [B, n] (matmul_transform.py:381-388, 412-421)."""
    if mode not in _TORCH_MODE:
        raise ValueError(f"Padding mode not supported: {mode}")
    if mode == "symmetric":
        return torch.cat([x, x[:, -1:]], 1)
    return F.pad(x.unsqueeze(1), (0, 1), mode=_TORCH_MODE[mode]).squeeze(1)


class MatrixWavedec:
    def __init__(self, wavelet, level=None, *, axis=None, orthogonalization="qr", odd_coeff_padding_mode="zero"):
        self.wavelet = as_wavelet(wavelet)
        self.level = level
        self.axis = _axes(axis, 1)
        self.method = orthogonalization
        self.odd_mode = odd_coeff_padding_mode
        self.ops: list[torch.Tensor] = []
        self.pads: list[bool] = []
        self.key = None

    def _build(self, length: int, dtype):
        dec_lo, dec_hi, _, _ = _taps(self.wavelet, dtype, flip=False)
        L = dec_lo.shape[0]
        self.ops, self.pads = [], []
        cur = length
        for _ in range(self.level):
            if cur < L:
                break
            pad = cur % 2 != 0
            cur += 1 if pad else 0
            self.pads.append(pad)
            self.ops.append(boundary_matrix_sparse(dec_lo, dec_hi, cur, self.method))
            cur //= 2

    def __call__(self, data):
        x, shape = _fold(data, 1, self.axis)
        if x.shape[-1] % 2:
            x = _odd_pad(x, self.odd_mode)
        length = x.shape[-1]
        if self.level is None:
            self.level = int(np.log2(length / (len(filter_bank(self.wavelet)[0]) - 1)))
        elif self.level <= 0:
            raise ValueError("level must be a positive integer.")
        if self.key != (length, x.dtype, self.level):
            self._build(length, x.dtype)
            self.key = (length, x.dtype, self.level)
        lo = x.T
        his = []
        for op, pad in zip(self.ops, self.pads):
            if pad:
                lo = _odd_pad(lo.T, self.odd_mode).T
            c = torch.sparse.mm(op, lo)
            lo, hi = c[: c.shape[0] // 2], c[c.shape[0] // 2:]
            his.append(hi)
        res = [lo.T] + [h.T for h in reversed(his)]
        return [_unfold(t, 1, self.axis, shape) for t in res]


class MatrixWaverec:
    def __init__(self, wavelet, *, axis=None, orthogonalization="qr"):
        self.wavelet = as_wavelet(wavelet)
        self.axis = _axes(axis, 1)
        self.method = orthogonalization
        self.ops: list[torch.Tensor] = []
        self.key = None

    def _build(self, length: int, level: int, dtype):
        _, _, rec_lo, rec_hi = _taps(self.wavelet, dtype, flip=True)
        L = rec_lo.shape[0]
        self.ops = []
        cur = length
        for _ in range(level):
            if cur < L:
                break
            cur += cur % 2
            self.ops.append(boundary_matrix_sparse(rec_lo, rec_hi, cur, self.method).t().coalesce())
            cur //= 2

    def __call__(self, coeffs):
        coeffs = list(coeffs)
        lead, shape = _fold(coeffs[0], 1, self.axis)
        rest = [_fold(c, 1, self.axis, len(shape))[0] for c in coeffs[1:]]
        level = len(rest)
        if level == 0:
            return _unfold(lead, 1, self.axis, shape)
        length = rest[-1].shape[-1] * 2
        if self.key != (length, level, lead.dtype):
            self._build(length, level, lead.dtype)
            self.key = (length, level, lead.dtype)
        lo = lead.T
        for i, hi in enumerate(rest):
            hi = hi.T
            if lo.shape != hi.shape:
                raise ValueError("coefficients must have the same shape")
            lo = torch.sparse.mm(self.ops[::-1][i], torch.cat([lo, hi], 0))
            if i + 1 < level and rest[i + 1].shape[-1] != lo.shape[0]:
                lo = lo[:-1]
                assert lo.shape[0] == rest[i + 1].shape[-1], "padding error"
        return _unfold(lo.T, 1, self.axis, shape)


# ---------------------------------------------------------------------------------------------
# separable 2-D / 3-D boundary-filter matrix FWT (SURVEY.md section 8f row 2)
#   matmul_transform_2.py:368-531 (analysis), :740-856 (synthesis); matmul_transform_3.py:131-300, :303-480
# the 1-D level operator is applied along every axis as a dense matmul
# ---------------------------------------------------------------------------------------------
def _apply_along(mat: torch.Tensor, x: torch.Tensor, dim: int) -> torch.Tensor:
    return torch.movedim(torch.tensordot(mat, x, dims=([1], [dim])), 0, dim)


def _odd_pad_axis(x: torch.Tensor, dim: int, mode: str) -> torch.Tensor:
    moved = torch.movedim(x, dim, -1)
    flat = moved.reshape(-1, moved.shape[-1])
    return torch.movedim(_odd_pad(flat, mode).reshape(*moved.shape[:-1], moved.shape[-1] + 1), -1, dim)


_KEYS_ND = {2: ("ad", "da", "dd"), 3: ("aad", "ada", "add", "daa", "dad", "dda", "ddd")}


class _MatrixWavedecNd:
    ndim = 2

    def __init__(self, wavelet, level=None, *, axes=None, orthogonalization="qr", odd_coeff_padding_mode="zero"):
        self.wavelet = as_wavelet(wavelet)
        self.level = level
        self.axes = _axes(axes, self.ndim)
        self.method = orthogonalization
        self.odd_mode = odd_coeff_padding_mode

    def __call__(self, data):
        nd = self.ndim
        x, shape = _fold(data, nd, self.axes)
        dec_lo, dec_hi, _, _ = _taps(self.wavelet, x.dtype, flip=False)
        L = dec_lo.shape[0]
        if self.level is None:
            self.level = int(np.min([np.log2(s / (L - 1)) for s in x.shape[1:]]))
        elif self.level <= 0:
            raise ValueError("level must be a positive integer.")
        cur = x
        out = []
        for _ in range(self.level):
            if any(s < L for s in cur.shape[1:]):
                break
            for a in range(nd, 0, -1):
                if cur.shape[a] % 2:
                    cur = _odd_pad_axis(cur, a, self.odd_mode)
            for a in range(nd, 0, -1):
                cur = _apply_along(boundary_matrix(dec_lo, dec_hi, cur.shape[a], self.method), cur, a)
            half = [s // 2 for s in cur.shape[1:]]
            bands = {}
            for key in _KEYS_ND[nd]:
                sl = tuple(slice(half[a], None) if key[a] == "d" else slice(0, half[a]) for a in range(nd))
                bands[key] = cur[(slice(None),) + sl]
            out.append(bands)
            cur = cur[(slice(None),) + tuple(slice(0, h) for h in half)]
        res = [_unfold(cur, nd, self.axes, shape)]
        for bands in reversed(out):
            un = {k: _unfold(v, nd, self.axes, shape) for k, v in bands.items()}
            res.append((un["ad"], un["da"], un["dd"]) if nd == 2 else un)
        return tuple(res)


class MatrixWavedec2(_MatrixWavedecNd):
    ndim = 2

    def __init__(self, wavelet, level=None, *, axes=None, orthogonalization="qr", separable=True,
                 odd_coeff_padding_mode="zero"):
        if not separable:
            raise NotImplementedError("port covers the separable operator only")
        super().__init__(wavelet, level, axes=axes, orthogonalization=orthogonalization,
                         odd_coeff_padding_mode=odd_coeff_padding_mode)


class MatrixWavedec3(_MatrixWavedecNd):
    ndim = 3


class _MatrixWaverecNd:
    ndim = 2

    def __init__(self, wavelet, *, axes=None, orthogonalization="qr", separable=True):
        if not separable:
            raise NotImplementedError("port covers the separable operator only")
        self.wavelet = as_wavelet(wavelet)
        self.axes = _axes(axes, self.ndim)
        self.method = orthogonalization

    def __call__(self, coeffs):
        nd = self.ndim
        lead, shape = _fold(coeffs[0], nd, self.axes)
        _, _, rec_lo, rec_hi = _taps(self.wavelet, lead.dtype, flip=True)
        cur = lead
        for el in coeffs[1:]:
            if nd == 2:
                el = {"ad": el[0], "da": el[1], "dd": el[2]}
            bands = {k: _fold(v, nd, self.axes, len(shape))[0] for k, v in el.items()}
            dshape = tuple(bands["d" * nd].shape[1:])
            full = torch.zeros((cur.shape[0],) + tuple(2 * c for c in dshape), dtype=cur.dtype)
            full[(slice(None),) + tuple(slice(0, c) for c in dshape)] = cur[(slice(None),) + tuple(slice(0, c) for c in dshape)]
            for key, t in bands.items():
                sl = tuple(slice(dshape[a], None) if key[a] == "d" else slice(0, dshape[a]) for a in range(nd))
                full[(slice(None),) + sl] = t
            cur = full
            for a in range(nd, 0, -1):
                cur = _apply_along(boundary_matrix(rec_lo, rec_hi, cur.shape[a], self.method).T, cur, a)
        return _unfold(cur, nd, self.axes, shape)


class MatrixWaverec2(_MatrixWaverecNd):
    ndim = 2


class MatrixWaverec3(_MatrixWaverecNd):
    ndim = 3

    def __init__(self, wavelet, *, axes=None, orthogonalization="qr"):
        super().__init__(wavelet, axes=axes, orthogonalization=orthogonalization)
