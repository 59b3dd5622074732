"""Boundary-filter ("matrix") fast wavelet transform on the H100.

Drop-in for ``ptwt.MatrixWavedec`` / ``ptwt.MatrixWaverec``
(``/root/reference/src/ptwt/matmul_transform.py:172,502``).  The reference materialises one
sparse ``n x n`` operator per level (seconds of pure-Python COO construction,
``sparse_math.py:390-401``) and applies it with ``torch.sparse.mm``.  Here the operator is never
built for the transform itself: its interior is a stride-2 filter band, applied as a filter, and
its orthogonalised boundary rows are four small dense blocks per level, computed on the host
with the reference's own recipe (same ``torch.linalg.qr`` call on the same dense slab, in the
input dtype) and applied by the kernels in ``csrc/matrix_generic.cuh``.

``sparse_fwt_operator`` / ``sparse_ifwt_operator`` / ``construct_boundary_a`` /
``construct_boundary_s`` still return the explicit sparse operators (built vectorised from the
band + blocks) for transparency and for the parity tests.
"""
from __future__ import annotations

import ctypes as C
import functools
import sys
import warnings
from typing import Any, Optional, Sequence

import numpy as np
import torch

from . import _native as N
from ._shape import AxisHint, Fold, check_dtype, check_mode, check_tensor, ensure_axes, fold, unfold
from ._wavelets import as_wavelet, filter_bank, taps_in_dtype
from .fwt import _compute_device, _dtype_code, _no_autograd, _same_device_dtype, pinned_empty

__all__ = ["MatrixWavedec", "MatrixWaverec", "construct_boundary_a", "construct_boundary_s", "orthogonalize_rows"]

_ORTH_METHODS = ("qr", "gramschmidt")


def _deprecated_alias(**aliases: str):
    """``boundary=`` -> ``orthogonalization=`` with a DeprecationWarning (reference _util.py:750-799)."""

    def deco(fn):
        @functools.wraps(fn)
        def wrapper(*args, **kwargs):
            for old, new in aliases.items():
                if old in kwargs:
                    if new in kwargs:
                        raise TypeError(
                            f"{fn.__name__} received both {old} and {new} as arguments! {old} is deprecated, "
                            f"use {new} instead."
                        )
                    warnings.warn(
                        f"`{old}` is deprecated as an argument to `{fn.__name__}`; use `{new}` instead.",
                        DeprecationWarning,
                        stacklevel=2,
                    )
                    kwargs[new] = kwargs.pop(old)
            return fn(*args, **kwargs)

        return wrapper

    return deco


# --------------------------------------------------------------------------------------
# boundary rows of one level operator
# --------------------------------------------------------------------------------------
def _shift(filt_len: int) -> int:
    # row i of the "sameshift" strided convolution matrix puts tap m on column 2 i + shift - m
    # (reference sparse_math.py:371-377 start_row, :503-505 rows 1::2)
    return filt_len // 2 + filt_len % 2


def _raw_rows(filt: torch.Tensor, n: int, rows: Sequence[int]) -> torch.Tensor:
    """Dense truncated rows of the strided convolution matrix for the given row indices."""
    L = filt.shape[0]
    out = torch.zeros((len(rows), n), dtype=filt.dtype)
    sh = _shift(L)
    for r, i in enumerate(rows):
        for m in range(L):
            c = 2 * i + sh - m
            if 0 <= c < n:
                out[r, c] = filt[m]
    return out


def _boundary_row_ids(n: int, filt_len: int) -> tuple[list[int], list[int]]:
    """Rows (per half) whose filter support overhangs the signal: (top, bottom)."""
    sh = _shift(filt_len)
    half = n // 2
    top = [i for i in range(half) if 2 * i + sh - (filt_len - 1) < 0]
    bot = [i for i in range(half) if 2 * i + sh >= n and i not in top]
    return top, bot


def orthogonalize_rows(sel: torch.Tensor, method: str) -> torch.Tensor:
    """Orthonormalise the rows of ``sel`` the way the reference does.

    ``qr``: ``q, _ = torch.linalg.qr(sel.T)``; rows of ``q.T`` (reference sparse_math.py:283-285).
    ``gramschmidt``: classical Gram-Schmidt in row order, then normalisation
    (reference sparse_math.py:314-347).
    """
    if method == "qr":
        q, _ = torch.linalg.qr(sel.T)
        return q.T.contiguous()
    if method == "gramschmidt":
        rows = sel.clone()
        for p in range(rows.shape[0]):
            cur = rows[p].clone()
            acc = torch.zeros_like(cur)
            for d in range(p):
                acc += torch.dot(cur, rows[d]) * rows[d]
            cur = cur - acc
            rows[p] = cur / torch.linalg.vector_norm(cur)
        return rows
    raise ValueError(f"Invalid orthogonalization method: {method}")


class _LevelBlocks:
    """Boundary rows of one level operator, ready for the kernels.

    ``nb_top + nb_bot`` rows per half (top rows first).  Every row is stored as a left window (first
    ``w_left`` columns) and a right window (last ``w_right`` columns): the orthogonalisation leaves
    round-off sized entries of a top row in the right corner and vice versa, and they are kept
    because the reference keeps them (``q.T.to_sparse()``, sparse_math.py:285).
    """

    __slots__ = ("n", "nb_top", "nb_bot", "w_left", "w_right", "lo_left", "lo_right", "hi_left", "hi_right")

    def flat(self) -> torch.Tensor:
        return torch.cat([self.lo_left.reshape(-1), self.lo_right.reshape(-1), self.hi_left.reshape(-1),
                          self.hi_right.reshape(-1)])


@functools.lru_cache(maxsize=256)
def _level_blocks_cached(lo_key: bytes, hi_key: bytes, dtype_name: str, n: int, method: str) -> _LevelBlocks:
    dtype = getattr(torch, dtype_name)
    lo = torch.from_numpy(np.frombuffer(lo_key, dtype=np.float64).copy()).to(dtype)
    hi = torch.from_numpy(np.frombuffer(hi_key, dtype=np.float64).copy()).to(dtype)
    L = lo.shape[0]
    top, bot = _boundary_row_ids(n, L)
    ids = top + bot
    blk = _LevelBlocks()
    blk.n = n
    blk.nb_top, blk.nb_bot = len(top), len(bot)
    if not ids:
        z = torch.zeros((0, 0), dtype=dtype)
        blk.w_left = blk.w_right = 0
        blk.lo_left = blk.lo_right = blk.hi_left = blk.hi_right = z
        return blk
    # one slab, rows in the reference's order: boundary rows of the lo half (ascending), then of
    # the hi half (reference matmul_transform.py:121-136: unique row indices of cat([A_lo, A_hi]))
    sel = torch.cat([_raw_rows(lo, n, ids), _raw_rows(hi, n, ids)], 0)
    q = orthogonalize_rows(sel, method)
    nb = len(ids)
    nz = (q != 0).any(0).nonzero().reshape(-1)
    half = n // 2
    left = nz[nz < half]
    right = nz[nz >= half]
    blk.w_left = int(left.max()) + 1 if left.numel() else 0
    blk.w_right = n - int(right.min()) if right.numel() else 0
    blk.lo_left = q[:nb, : blk.w_left].contiguous()
    blk.hi_left = q[nb:, : blk.w_left].contiguous()
    blk.lo_right = q[:nb, n - blk.w_right:].contiguous()
    blk.hi_right = q[nb:, n - blk.w_right:].contiguous()
    return blk


#: the multi-level fused kernel cannot reach a boundary row's entries in the opposite corner window;
#: it is used only when all of them are at most this large (round-off of the float64 QR: ~1e-16)
FUSED_CROSS_CORNER_MAX = 1e-13


def _cross_corner_max(blocks: Sequence["_LevelBlocks"]) -> float:
    worst = 0.0
    for b in blocks:
        nt = b.nb_top
        for top_part, bot_part in ((b.lo_right[:nt], b.lo_left[nt:]), (b.hi_right[:nt], b.hi_left[nt:])):
            for t in (top_part, bot_part):
                if t.numel():
                    worst = max(worst, float(t.abs().max()))
    return worst


def _level_blocks(lo_taps: np.ndarray, hi_taps: np.ndarray, dtype: torch.dtype, n: int, method: str) -> _LevelBlocks:
    return _level_blocks_cached(lo_taps.tobytes(), hi_taps.tobytes(), str(dtype).split(".")[-1], int(n), method)


def _level_operator_sparse(lo_taps: np.ndarray, hi_taps: np.ndarray, dtype: torch.dtype, n: int,
                           method: Optional[str], device="cpu") -> torch.Tensor:
    """Explicit sparse [n, n] operator of one level: band rows + orthogonalised boundary rows."""
    L = lo_taps.shape[0]
    half = n // 2
    sh = _shift(L)
    lo = torch.from_numpy(lo_taps).to(dtype)
    hi = torch.from_numpy(hi_taps).to(dtype)
    i = torch.arange(half).reshape(-1, 1)
    m = torch.arange(L).reshape(1, -1)
    cols = 2 * i + sh - m
    valid = (cols >= 0) & (cols < n)
    rows_idx = i.expand_as(cols)
    if method is not None:
        blk = _level_blocks(lo_taps, hi_taps, dtype, n, method)
        interior = (rows_idx >= blk.nb_top) & (rows_idx < half - blk.nb_bot)
        valid = valid & interior
    r = rows_idx[valid]
    c = cols[valid]
    v_lo = lo.reshape(1, -1).expand(half, L)[valid]
    v_hi = hi.reshape(1, -1).expand(half, L)[valid]
    idx = [torch.stack([r, c]), torch.stack([r + half, c])]
    vals = [v_lo, v_hi]
    if method is not None:
        def add(block: torch.Tensor, row0: int, col0: int):
            if block.numel() == 0:
                return
            rr, cc = torch.meshgrid(torch.arange(block.shape[0]), torch.arange(block.shape[1]), indexing="ij")
            keep = block != 0
            idx.append(torch.stack([rr[keep] + row0, cc[keep] + col0]))
            vals.append(block[keep])
        nt = blk.nb_top
        for band, (bl, br) in enumerate(((blk.lo_left, blk.lo_right), (blk.hi_left, blk.hi_right))):
            base = band * half
            add(bl[:nt], base, 0)
            add(br[:nt], base, n - blk.w_right)
            add(bl[nt:], base + half - blk.nb_bot, 0)
            add(br[nt:], base + half - blk.nb_bot, n - blk.w_right)
    mat = torch.sparse_coo_tensor(torch.cat(idx, 1), torch.cat(vals), size=(n, n), dtype=dtype)
    return mat.coalesce().to(device)


def _analysis_taps(wavelet: Any, dtype: torch.dtype) -> tuple[np.ndarray, np.ndarray]:
    dec_lo, dec_hi, _, _ = filter_bank(as_wavelet(wavelet))
    return taps_in_dtype(dec_lo, dtype), taps_in_dtype(dec_hi, dtype)


def _synthesis_taps(wavelet: Any, dtype: torch.dtype) -> tuple[np.ndarray, np.ndarray]:
    """Rows of S^T carry the FLIPPED reconstruction filters (reference matmul_transform.py:110-116)."""
    _, _, rec_lo, rec_hi = filter_bank(as_wavelet(wavelet))
    return (np.ascontiguousarray(taps_in_dtype(rec_lo, dtype)[::-1]),
            np.ascontiguousarray(taps_in_dtype(rec_hi, dtype)[::-1]))


@_deprecated_alias(boundary="orthogonalization")
def construct_boundary_a(wavelet: Any, length: int, device="cpu", orthogonalization: str = "qr",
                         dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """Sparse boundary-wavelet analysis matrix (reference matmul_transform.py:434-463)."""
    lo, hi = _analysis_taps(wavelet, dtype)
    return _level_operator_sparse(lo, hi, dtype, length, orthogonalization, device)


@_deprecated_alias(boundary="orthogonalization")
def construct_boundary_s(wavelet: Any, length: int, device="cpu", orthogonalization: str = "qr",
                         dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """Sparse boundary-wavelet synthesis matrix (reference matmul_transform.py:467-499)."""
    lo, hi = _synthesis_taps(wavelet, dtype)
    return _level_operator_sparse(lo, hi, dtype, length, orthogonalization, device).transpose(0, 1)


def _cat_identity(mat: torch.Tensor, new_length: int) -> torch.Tensor:
    """blockdiag(mat, I) of size new_length (reference sparse_math.py cat_sparse_identity_matrix)."""
    mat = mat.coalesce()
    k = mat.shape[0]
    extra = torch.arange(k, new_length, device=mat.device)
    idx = torch.cat([mat.indices(), torch.stack([extra, extra])], 1)
    val = torch.cat([mat.values(), torch.ones(extra.shape[0], dtype=mat.dtype, device=mat.device)])
    return torch.sparse_coo_tensor(idx, val, size=(new_length, new_length)).coalesce()


def _level_sizes(input_length: int, level: int, filt_len: int):
    """size_list / pad_list bookkeeping of the reference (matmul_transform.py:310-354)."""
    sizes: list[int] = []
    pads: list[bool] = []
    cur = input_length
    for lvl in range(1, level + 1):
        if cur < filt_len:
            sys.stderr.write(
                f"Warning: The selected number of decomposition levels {level}"
                f" is too large for the given input size {input_length}. At "
                f"level {lvl}, the current signal length {cur} is "
                f"smaller than the filter length {filt_len}. Therefore, the "
                "transformation is only computed up to the decomposition level "
                f"{lvl-1}.\n"
            )
            break
        if cur % 2 != 0:
            cur += 1
            pads.append(True)
        else:
            pads.append(False)
        sizes.append(cur)
        cur //= 2
    return sizes, pads, cur


class _BlockStore:
    """Per-object cache of the device-resident boundary blocks of all levels."""

    def __init__(self):
        self.key = None
        self.levels: list[_LevelBlocks] = []
        self.device_flat: Optional[torch.Tensor] = None
        self._fused_ok: Optional[int] = None

    def get(self, lo: np.ndarray, hi: np.ndarray, dtype, sizes: Sequence[int], method: str, dev: torch.device):
        key = (lo.tobytes(), hi.tobytes(), dtype, tuple(sizes), method, str(dev))
        if key != self.key:
            self.levels = [_level_blocks(lo, hi, dtype, n, method) for n in sizes]
            flat = torch.cat([b.flat() for b in self.levels]) if self.levels else torch.zeros(0, dtype=dtype)
            if flat.numel() == 0:
                flat = torch.zeros(1, dtype=dtype)
            self.device_flat = flat.to(dev)
            self.key = key
            self._fused_ok = None
        return self.levels, self.device_flat

    def allow_fused(self) -> int:
        """1 when the cross-corner entries of every level are round-off (see FUSED_CROSS_CORNER_MAX)."""
        if self._fused_ok is None:
            self._fused_ok = 1 if _cross_corner_max(self.levels) <= FUSED_CROSS_CORNER_MAX else 0
        return self._fused_ok


class MatrixWavedec:
    """1-D boundary-wavelet FWT, ``[cA_n, cD_n, ..., cD_1]`` (reference matmul_transform.py:172-430)."""

    @_deprecated_alias(boundary="orthogonalization")
    def __init__(self, wavelet: Any, level: Optional[int] = None, *, axis: AxisHint = None,
                 orthogonalization: str = "qr", odd_coeff_padding_mode: str = "zero") -> None:
        self.wavelet = as_wavelet(wavelet)
        self.level = level
        self.odd_coeff_padding_mode = odd_coeff_padding_mode
        self.orthogonalization = orthogonalization
        self.axis = ensure_axes(axis, 1)[0]
        self.input_length: Optional[int] = None
        self.pad_list: list[bool] = []
        self.padded = False
        self.size_list: list[int] = []
        self._built = False
        self._dtype: Optional[torch.dtype] = None
        self._store = _BlockStore()
        self._call_cache: Optional[dict] = None
        self._sparse_cache: Optional[list[torch.Tensor]] = None
        if self.orthogonalization not in _ORTH_METHODS:
            raise NotImplementedError
        if self.wavelet.dec_len != self.wavelet.rec_len:
            raise ValueError("All filters must have the same length")

    # -- explicit operators (transparency; not used by __call__) ---------------------------
    @property
    def fwt_matrix_list(self) -> list[torch.Tensor]:
        if not self._built:
            return []
        if self._sparse_cache is None:
            lo, hi = _analysis_taps(self.wavelet, self._dtype)
            self._sparse_cache = [
                _level_operator_sparse(lo, hi, self._dtype, n, self.orthogonalization) for n in self.size_list[:-1]
            ]
        return self._sparse_cache

    @property
    def sparse_fwt_operator(self) -> torch.Tensor:
        """Product of the level operators (reference matmul_transform.py:268-308)."""
        mats = self.fwt_matrix_list
        if len(mats) == 1:
            return mats[0]
        if len(mats) > 1:
            if self.padded:
                raise NotImplementedError
            fwt = mats[0]
            for m in mats[1:]:
                fwt = torch.sparse.mm(_cat_identity(m, fwt.shape[0]), fwt)
            return fwt
        raise ValueError("Call this object first to create the transformation matrices for each level.")

    def _plan(self, length: int, dtype: torch.dtype) -> None:
        sizes, pads, last = _level_sizes(length, self.level, self.wavelet.dec_len)
        self.size_list = sizes + [last]
        self.pad_list = pads
        self.padded = any(pads)
        self._dtype = dtype
        self._built = True
        self._sparse_cache = None

    def __call__(self, input_signal: torch.Tensor) -> list[torch.Tensor]:
        check_tensor(input_signal)
        check_dtype(input_signal)
        x, f = fold(input_signal, 1, self.axis)
        n_in = x.shape[-1]
        first_pad = n_in % 2 != 0
        if first_pad:
            check_mode(self.odd_coeff_padding_mode)
        length = n_in + (1 if first_pad else 0)

        rebuild = False
        if self.input_length != length:
            self.input_length = length
            rebuild = True
        if self.level is None:
            wlen = len(self.wavelet)
            self.level = int(np.log2(length / (wlen - 1)))
            rebuild = True
        elif self.level <= 0:
            raise ValueError("level must be a positive integer.")
        if not self._built or rebuild or self._dtype != x.dtype:
            self._plan(length, x.dtype)
        sizes = self.size_list[:-1]
        nl = len(sizes)
        if nl == 0:
            return [unfold(x, f)]
        if self.padded:
            check_mode(self.odd_coeff_padding_mode)
        _no_autograd(input_signal, wavelet=self.wavelet)

        dev = _compute_device(x)
        on_host = not x.is_cuda
        batch = x.shape[0]
        dt = x.dtype
        lo_t, hi_t = _analysis_taps(self.wavelet, dt)
        with torch.cuda.device(dev):
            xd = x.to(dev, non_blocking=True) if on_host else x
            if xd.stride(-1) != 1 and xd.shape[-1] != 1:
                xd = xd.contiguous()
            blocks, flat = self._store.get(lo_t, hi_t, dt, sizes, self.orthogonalization, dev)
            # everything that depends only on (length, dtype, device) is prepared once per object
            ck = (length, dt, str(dev), first_pad, self.odd_coeff_padding_mode, tuple(sizes))
            cc = self._call_cache
            if cc is None or cc["key"] != ck:
                lens = [n // 2 for n in sizes]
                offs = {}
                o = lens[-1]
                for l in range(nl - 1, -1, -1):
                    offs[l] = o
                    o += lens[l]
                padded = [1 if p else 0 for p in self.pad_list]
                padded[0] = 1 if first_pad else 0
                cc = {
                    "key": ck, "lens": lens, "offs": offs, "total": lens[-1] + sum(lens),
                    "n": N.i64_array(sizes), "pd": N.i32_array(padded),
                    "nbt": N.i32_array([b.nb_top for b in blocks]), "nbb": N.i32_array([b.nb_bot for b in blocks]),
                    "wl": N.i32_array([b.w_left for b in blocks]), "wr": N.i32_array([b.w_right for b in blocks]),
                    "lo": N.f64_array(lo_t), "hi": N.f64_array(hi_t),
                    "mode": N.MODES[self.odd_coeff_padding_mode if (self.padded or first_pad) else "zero"],
                    "fused": self._store.allow_fused(),
                    "hi_ptrs": (C.c_void_p * nl)(), "hi_strides": (C.c_int64 * nl)(),
                }
                self._call_cache = cc
            lens, offs = cc["lens"], cc["offs"]
            # packed output [batch, total]: [cA | cD_n | ... | cD_1]
            out = torch.empty((batch, cc["total"]), dtype=dt, device=dev)
            es = out.element_size()
            base, ostride = out.data_ptr(), out.stride(0)
            hi_ptrs, hi_strides = cc["hi_ptrs"], cc["hi_strides"]
            for l in range(nl):
                hi_ptrs[l] = base + offs[l] * es
                hi_strides[l] = ostride
            scratch_elems = 2 * batch * (sizes[0] // 2) if nl > 1 else 0
            scratch = torch.empty((max(scratch_elems, 1),), dtype=dt, device=dev)
            lib = N.load()
            rc = lib.wt_matrix_fwd(
                _dtype_code(dt), nl, len(lo_t), cc["lo"][1], cc["hi"][1], cc["n"][1], cc["pd"][1], cc["mode"],
                cc["nbt"][1], cc["nbb"][1], cc["wl"][1], cc["wr"][1], flat.data_ptr(), xd.data_ptr(), batch, xd.stride(0),
                hi_ptrs, hi_strides, base, ostride,
                scratch.data_ptr(), scratch_elems * es, cc["fused"],
                torch.cuda.current_stream(dev).cuda_stream,
            )
            N.check(rc, "wt_matrix_fwd")
            if on_host:
                host = pinned_empty(out.shape, dt)
                host.copy_(out, non_blocking=True)
                torch.cuda.current_stream(dev).synchronize()
                out = host
        result = [out[:, : lens[-1]]]
        for l in range(nl - 1, -1, -1):
            result.append(out[:, offs[l]: offs[l] + lens[l]])
        return [unfold(t, f) for t in result]


class MatrixWaverec:
    """Inverse boundary-wavelet FWT (reference matmul_transform.py:502-703)."""

    @_deprecated_alias(boundary="orthogonalization")
    def __init__(self, wavelet: Any, *, axis: AxisHint = None, orthogonalization: str = "qr") -> None:
        self.wavelet = as_wavelet(wavelet)
        self.orthogonalization = orthogonalization
        self.axis = ensure_axes(axis, 1)
        self.level: Optional[int] = None
        self.input_length: Optional[int] = None
        self.padded = False
        self.size_list: list[int] = []
        self._built = False
        self._dtype: Optional[torch.dtype] = None
        self._store = _BlockStore()
        self._sparse_cache: Optional[list[torch.Tensor]] = None
        if self.orthogonalization not in _ORTH_METHODS:
            raise NotImplementedError
        if self.wavelet.dec_len != self.wavelet.rec_len:
            raise ValueError("All filters must have the same length")

    @property
    def ifwt_matrix_list(self) -> list[torch.Tensor]:
        if not self._built:
            return []
        if self._sparse_cache is None:
            lo, hi = _synthesis_taps(self.wavelet, self._dtype)
            self._sparse_cache = [
                _level_operator_sparse(lo, hi, self._dtype, n, self.orthogonalization).transpose(0, 1).coalesce()
                for n in self.size_list
            ]
        return self._sparse_cache

    @property
    def sparse_ifwt_operator(self) -> torch.Tensor:
        """Product of the level operators (reference matmul_transform.py:559-601)."""
        mats = self.ifwt_matrix_list
        if len(mats) == 1:
            return mats[0]
        if len(mats) > 1:
            if self.padded:
                raise NotImplementedError
            ifwt = mats[-1]
            for m in mats[:-1][::-1]:
                ifwt = torch.sparse.mm(m, _cat_identity(ifwt, m.shape[0]))
            return ifwt
        raise ValueError("Call this object first to create the transformation matrices for each level.")

    def _plan(self, dtype: torch.dtype) -> None:
        sizes, pads, _ = _level_sizes(self.input_length, self.level, self.wavelet.rec_len)
        self.size_list = sizes
        self.padded = any(pads)
        self._dtype = dtype
        self._built = True
        self._sparse_cache = None

    def __call__(self, coefficients: Sequence[torch.Tensor]) -> torch.Tensor:
        if not isinstance(coefficients, list):
            coefficients = list(coefficients)
        lead = check_tensor(coefficients[0])
        check_dtype(lead)
        for c in coefficients[1:]:
            if not isinstance(c, torch.Tensor):
                raise ValueError(f"Unexpected input type {type(c)}")
        folded = []
        f: Optional[Fold] = None
        for t in coefficients:
            ft, f = fold(t, 1, self.axis, lead=f)
            folded.append(ft)
        _same_device_dtype(folded)
        dt = folded[0].dtype
        level = len(folded) - 1
        input_length = folded[-1].shape[-1] * 2
        rebuild = False
        if self.level != level or self.input_length != input_length:
            self.level = level
            self.input_length = input_length
            rebuild = True
        if not self._built or rebuild or self._dtype != dt:
            self._plan(dt)
        if level == 0:
            return unfold(folded[0], f)
        sizes = self.size_list
        nl = len(sizes)
        if nl < level:
            raise IndexError("list index out of range")  # the reference indexes past its operator list
        # shape walk (reference matmul_transform.py:682-699)
        cur_len = folded[0].shape[-1]
        keep = [0] * nl
        for c_pos in range(level):
            l = level - 1 - c_pos
            hi = folded[1 + c_pos]
            if hi.shape[-1] != cur_len or hi.shape[0] != folded[0].shape[0]:
                raise ValueError("coefficients must have the same shape")
            if 2 * cur_len != sizes[l]:
                raise RuntimeError(
                    f"size mismatch: level operator is {sizes[l]}x{sizes[l]} but got {2 * cur_len} coefficients")
            cur_len = sizes[l]
            if c_pos < level - 1:
                nxt = folded[c_pos + 2].shape[-1]
                if nxt != cur_len:
                    cur_len -= 1
                    assert cur_len == nxt, "padding error, please open an issue on github"
            keep[l] = cur_len
        _no_autograd(*folded, wavelet=self.wavelet)

        dev = _compute_device(folded[0])
        on_host = not folded[0].is_cuda
        batch = folded[0].shape[0]
        lo_t, hi_t = _synthesis_taps(self.wavelet, dt)
        _, _, rec_lo, rec_hi = filter_bank(self.wavelet)
        with torch.cuda.device(dev):
            if on_host:
                folded = [t.to(dev, non_blocking=True) for t in folded]
            folded = [t if (t.stride(-1) == 1 or t.shape[-1] == 1) else t.contiguous() for t in folded]
            blocks, flat = self._store.get(lo_t, hi_t, dt, sizes, self.orthogonalization, dev)
            y = torch.empty((batch, keep[0]), dtype=dt, device=dev)
            es = y.element_size()
            his = [folded[level - l] for l in range(nl)]  # his[l] = detail of level l (0 = finest)
            hi_ptrs = (C.c_void_p * nl)(*[t.data_ptr() for t in his])
            hi_strides = (C.c_int64 * nl)(*[t.stride(0) for t in his])
            n_arr, n_p = N.i64_array(sizes)
            k_arr, k_p = N.i64_array(keep)
            nbt_arr, nbt_p = N.i32_array([b.nb_top for b in blocks])
            nbb_arr, nbb_p = N.i32_array([b.nb_bot for b in blocks])
            wt_arr, wt_p = N.i32_array([b.w_left for b in blocks])
            wb_arr, wb_p = N.i32_array([b.w_right for b in blocks])
            lo_arr, lo_p = N.f64_array(taps_in_dtype(rec_lo, dt))
            hi_arr, hi_p = N.f64_array(taps_in_dtype(rec_hi, dt))
            scratch_elems = 2 * batch * sizes[0] if nl > 1 else 0
            scratch = torch.empty((max(scratch_elems, 1),), dtype=dt, device=dev)
            lib = N.load()
            rc = lib.wt_matrix_inv(
                _dtype_code(dt), nl, len(lo_t), lo_p, hi_p, n_p, k_p, nbt_p, nbb_p, wt_p, wb_p, flat.data_ptr(),
                folded[0].data_ptr(), folded[0].stride(0), hi_ptrs, hi_strides, batch, y.data_ptr(), y.stride(0),
                scratch.data_ptr(), scratch_elems * es, self._store.allow_fused(),
                torch.cuda.current_stream(dev).cuda_stream,
            )
            N.check(rc, "wt_matrix_inv")
            if on_host:
                host = pinned_empty(y.shape, dt)
                host.copy_(y, non_blocking=True)
                torch.cuda.current_stream(dev).synchronize()
                y = host
        return unfold(y, f)
