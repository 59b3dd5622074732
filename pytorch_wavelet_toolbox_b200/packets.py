"""Wavelet packets with level-wise BATCHED node expansion (SURVEY.md section 8f, row 4).

Drop-ins for ``ptwt.WaveletPacket`` / ``ptwt.WaveletPacket2D`` (reference ``src/ptwt/packets.py``): the same lazy
dictionary semantics (a node exists once one of its siblings was requested; ``initialize`` / ``reconstruct`` /
``get_level`` / ``get_natural_order`` / ``get_freq_order``; the same errors), the same numbers -- every node is one
level-1 transform of its parent (``packets.py:312-316``, ``:528-539``) -- but the reference expands node by node, i.e.
``2^d`` / ``4^d`` tiny launches at depth ``d``.  Here all equally shaped parents of one tree level that a request
needs are stacked along a new leading dimension and expanded by ONE call into the hot path (one kernel launch per
tree level instead of one per node); ``reconstruct`` runs one synthesis call per tree level.

The reference's quirk in separable mode is kept: ``fsdict["ad"] -> horizontal, fsdict["da"] -> vertical``
(``packets.py:603-606``), although ``"ad"`` (low-pass on axis -2, high-pass on axis -1) is the VERTICAL band of
``wavedec2`` (SURVEY.md appendix A, quirk 10).

``WaveletPacket3D`` goes beyond the ``ptwt`` API, which stops at 2-D packets: the same semantics for volumes and clips,
one level-1 ``wavedec3`` / ``fswavedec3`` / ``MatrixWavedec3`` call on the stacked parents per tree level.  A node key
is one 3-letter subband key (``wavedec3``'s ``"aad"`` .. ``"ddd"`` plus ``"aaa"``) per level.
"""
from __future__ import annotations

import collections
from itertools import product
from typing import Any, Iterable, Optional, Sequence

import torch

from ._shape import ensure_axes
from ._wavelets import as_wavelet, dwt_max_level
from .constants import WaveletDetailTuple2d
from .fwt import wavedec, wavedec2, wavedec3, waverec, waverec2, waverec3
from .matrix_fwt import MatrixWavedec, MatrixWaverec, _ORTH_METHODS
from .matrix_fwt_nd import MatrixWavedec2, MatrixWavedec3, MatrixWaverec2, MatrixWaverec3
from .separable import fswavedec2, fswavedec3, fswaverec2, fswaverec3

__all__ = ["WaveletPacket", "WaveletPacket2D", "WaveletPacket3D"]

#: the eight children of a 3-D packet node in natural order; letter i is the filter along axes[i]
SUBBANDS_3D = tuple("".join(p) for p in product("ad", repeat=3))


def _graycode_order(level: int, x: str = "a", y: str = "d") -> list[str]:
    """Frequency (Gray code) order of the paths of one tree level (reference packets.py:296-305)."""
    if level == 0:
        return [""]
    order = [x, y]
    for _ in range(level - 1):
        order = [x + p for p in order] + [y + p for p in order[::-1]]
    return order


def _neg_axes(axes: Sequence[int], ndim: int) -> tuple[int, ...]:
    """Axes counted from the end: stacking nodes along a NEW leading dimension then leaves them unchanged."""
    return tuple(a if a < 0 else a - ndim for a in axes)


class _PacketBase(collections.UserDict):
    _filter_keys: frozenset = frozenset()   # a node's children, as suffixes of its key
    _key_chars: frozenset = frozenset()     # the letters a key may contain
    _key_width = 1                          # letters per tree level
    _ndim = 1

    def _invalid_key(self, key: str) -> ValueError:
        rule = f"All chars in the key must be of the set {set(self._key_chars)}."
        if self._key_width > 1:
            rule += f" Its length must be a multiple of {self._key_width}, one subband key per level."
        return ValueError(f"Invalid key '{key}'. {rule}")

    def _check_access(self, key: str) -> None:
        """The reference's access checks (packets.py:332-359, 642-665), in its order."""
        if self.maxlevel is None:
            raise ValueError("The wavelet packet tree must be initialized via 'transform' before "
                             "its values can be accessed!")
        w = self._key_width
        level = -(-len(key) // w)
        if key not in self and level > self.maxlevel:
            raise KeyError(f"The requested level {level} with key '{key}' is too large and cannot be accessed! "
                           f"This wavelet packet tree is initialized with maximum level {self.maxlevel}.")
        if key not in self:
            if key == "":
                raise ValueError("The requested root of the packet tree cannot be accessed! The wavelet packet tree is "
                                 "not properly initialized. Run `transform` before accessing tree values.")
            if len(key) % w or key[-w:] not in self._filter_keys:
                raise self._invalid_key(key)

    def __getitem__(self, key: str) -> torch.Tensor:
        self._check_access(key)
        if key not in self:
            # a single request: the chain of missing ancestors, one node per tree level
            self._require([key])
        return super().__getitem__(key)

    def initialize(self, keys: Iterable[str]) -> None:
        """Initialize the tree partially (reference packets.py:179-189): exactly the nodes the reference would create
        (all children of every proper prefix of a requested key), but one batched expansion per tree level."""
        keys = list(keys)
        for key in keys:
            self._check_access(key)
        self._require(keys)

    def _require(self, keys: Sequence[str]) -> None:
        w = self._key_width
        depth = max((len(k) // w for k in keys), default=0)
        for level in range(depth):
            start = level * w
            parents: list[str] = []
            for k in keys:
                if len(k) > start and k not in self.data:
                    par = k[:start]
                    if par not in parents and not self._expanded(par):
                        parents.append(par)
            # validate the requests of this level like a node-by-node walk would
            for k in keys:
                if len(k) > start and k[start:start + w] not in self._filter_keys:
                    raise self._invalid_key(k)
            if parents:
                self._expand_nodes(parents)

    def _expanded(self, path: str) -> bool:
        return all(path + c in self.data for c in self._filter_keys)

    def _stack(self, paths: Sequence[str]) -> torch.Tensor:
        nodes = [self.data[p] for p in paths]
        return nodes[0].unsqueeze(0) if len(nodes) == 1 else torch.stack(nodes, 0)


class WaveletPacket(_PacketBase):
    """One-dimensional wavelet packets (reference packets.py:68-360), level-wise batched."""

    _filter_keys = frozenset({"a", "d"})
    _key_chars = _filter_keys

    def __init__(self, data: Optional[torch.Tensor], wavelet: Any, *, mode: str = "reflect",
                 maxlevel: Optional[int] = None, axis: Optional[int] = None, orthogonalization: str = "qr",
                 **deprecated: Any) -> None:
        if "boundary_orthogonalization" in deprecated:
            import warnings

            warnings.warn("boundary_orthogonalization is deprecated; use orthogonalization", DeprecationWarning, stacklevel=2)
            orthogonalization = deprecated.pop("boundary_orthogonalization")
        if deprecated:
            raise TypeError(f"unexpected keyword arguments {sorted(deprecated)}")
        super().__init__()
        self.wavelet = as_wavelet(wavelet)
        self.mode = mode
        self.orthogonalization = orthogonalization
        self._matrix_wavedec_dict: dict[int, MatrixWavedec] = {}
        self._matrix_waverec_dict: dict[int, MatrixWaverec] = {}
        self.maxlevel: Optional[int] = None
        self.axis = ensure_axes(axis, 1)[0]
        if self.orthogonalization not in _ORTH_METHODS:
            raise NotImplementedError
        if data is not None:
            self.transform(data, maxlevel)
        else:
            self.data = {}

    def transform(self, data: torch.Tensor, maxlevel: Optional[int] = None) -> "WaveletPacket":
        self.data = {"": data}
        if maxlevel is None:
            maxlevel = dwt_max_level(data.shape[self.axis], self.wavelet.dec_len)
        self.maxlevel = maxlevel
        return self

    # -- level-1 transforms of a stack of equally shaped nodes ----------------------------------------
    def _ax(self, t: torch.Tensor) -> int:
        return _neg_axes((self.axis,), t.dim())[0]

    def _wavedec(self, stacked: torch.Tensor, axis: int):
        if self.mode == "boundary":
            length = stacked.shape[axis]
            if length not in self._matrix_wavedec_dict:
                self._matrix_wavedec_dict[length] = MatrixWavedec(self.wavelet, level=1, axis=axis,
                                                                  orthogonalization=self.orthogonalization)
            return self._matrix_wavedec_dict[length](stacked)
        return wavedec(stacked, self.wavelet, level=1, mode=self.mode, axis=axis)

    def _waverec(self, lo: torch.Tensor, hi: torch.Tensor, axis: int) -> torch.Tensor:
        if self.mode == "boundary":
            length = lo.shape[axis]
            if length not in self._matrix_waverec_dict:
                self._matrix_waverec_dict[length] = MatrixWaverec(self.wavelet, axis=axis,
                                                                  orthogonalization=self.orthogonalization)
            return self._matrix_waverec_dict[length]([lo, hi])
        return waverec([lo, hi], self.wavelet, axis=axis)

    def _expand_nodes(self, paths: Sequence[str]) -> None:
        axis = self._ax(self.data[paths[0]])
        lo, hi = self._wavedec(self._stack(paths), axis)
        for i, p in enumerate(paths):
            self.data[p + "a"] = lo[i]
            self.data[p + "d"] = hi[i]

    def reconstruct(self) -> "WaveletPacket":
        """Reconstruct the input from the leaves (reference packets.py:191-243), one synthesis call per tree level."""
        if self.maxlevel is None:
            self.maxlevel = dwt_max_level(self[""].shape[-1], self.wavelet.dec_len)
        for level in reversed(range(self.maxlevel)):
            nodes = self.get_level(level)
            for node in nodes:
                for child in ("a", "d"):
                    if node + child not in self:
                        raise KeyError(f"Key {node + child} not found")
            lo = self._stack([n + "a" for n in nodes])
            hi = self._stack([n + "d" for n in nodes])
            axis = self._ax(self.data[nodes[0] + "a"])
            rec = self._waverec(lo, hi, axis)
            for i, node in enumerate(nodes):
                r = rec[i]
                if level > 0 and r.shape[axis] != self[node].shape[axis]:
                    assert r.shape[axis] == self[node].shape[axis] + 1, "padding error, please open an issue on github"
                    r = r.narrow(axis, 0, r.shape[axis] - 1)
                self[node] = r
        return self

    @staticmethod
    def get_level(level: int, order: str = "freq") -> list[str]:
        if order == "freq":
            return _graycode_order(level)
        if order == "natural":
            return ["".join(p) for p in product(["a", "d"], repeat=level)]
        raise ValueError(f"Unsupported order '{order}'. Choose from 'freq' and 'natural'.")

    _get_graycode_order = staticmethod(_graycode_order)


class WaveletPacket2D(_PacketBase):
    """Two-dimensional wavelet packets (reference packets.py:362-771), level-wise batched."""

    _filter_keys = frozenset({"a", "h", "v", "d"})
    _key_chars = _filter_keys
    _ndim = 2

    def __init__(self, data: Optional[torch.Tensor], wavelet: Any, *, mode: str = "reflect",
                 maxlevel: Optional[int] = None, axes: Optional[tuple[int, int]] = None, orthogonalization: str = "qr",
                 separable: bool = False, **deprecated: Any) -> None:
        if "boundary_orthogonalization" in deprecated:
            import warnings

            warnings.warn("boundary_orthogonalization is deprecated; use orthogonalization", DeprecationWarning, stacklevel=2)
            orthogonalization = deprecated.pop("boundary_orthogonalization")
        if deprecated:
            raise TypeError(f"unexpected keyword arguments {sorted(deprecated)}")
        super().__init__()
        self.wavelet = as_wavelet(wavelet)
        self.mode = mode
        self.orthogonalization = orthogonalization
        self.separable = separable
        self.matrix_wavedec2_dict: dict[tuple[int, ...], MatrixWavedec2] = {}
        self.matrix_waverec2_dict: dict[tuple[int, ...], MatrixWaverec2] = {}
        self.axes = tuple(ensure_axes(axes, 2))
        if self.orthogonalization not in _ORTH_METHODS:
            raise NotImplementedError
        self.maxlevel: Optional[int] = None
        if data is not None:
            self.transform(data, maxlevel)
        else:
            self.data = {}

    def _sizes(self, t: torch.Tensor) -> tuple[int, int]:
        return t.shape[self.axes[0]], t.shape[self.axes[1]]

    def transform(self, data: torch.Tensor, maxlevel: Optional[int] = None) -> "WaveletPacket2D":
        self.data = {"": data}
        if maxlevel is None:
            maxlevel = dwt_max_level(min(self._sizes(data)), self.wavelet.dec_len)
        self.maxlevel = maxlevel
        return self

    def _wavedec(self, stacked: torch.Tensor, axes: tuple[int, int]):
        """(a, h, v, d) of a stack of nodes."""
        if self.mode == "boundary":
            shape = (stacked.shape[axes[0]], stacked.shape[axes[1]])
            if shape not in self.matrix_wavedec2_dict:
                self.matrix_wavedec2_dict[shape] = MatrixWavedec2(self.wavelet, level=1, axes=axes,
                                                                  orthogonalization=self.orthogonalization,
                                                                  separable=self.separable)
            a, (h, v, d) = self.matrix_wavedec2_dict[shape](stacked)
            return a, h, v, d
        if self.separable:
            a, fs = fswavedec2(stacked, self.wavelet, level=1, mode=self.mode, axes=axes)
            return a, fs["ad"], fs["da"], fs["dd"]        # the reference's mapping (packets.py:603-606)
        a, (h, v, d) = wavedec2(stacked, self.wavelet, level=1, mode=self.mode, axes=axes)
        return a, h, v, d

    def _waverec(self, a, h, v, d, axes: tuple[int, int]) -> torch.Tensor:
        if self.mode == "boundary":
            shape = (a.shape[axes[0]], a.shape[axes[1]])
            if shape not in self.matrix_waverec2_dict:
                self.matrix_waverec2_dict[shape] = MatrixWaverec2(self.wavelet, axes=axes,
                                                                  orthogonalization=self.orthogonalization,
                                                                  separable=self.separable)
            return self.matrix_waverec2_dict[shape]((a, WaveletDetailTuple2d(h, v, d)))
        if self.separable:
            return fswaverec2((a, {"ad": h, "da": v, "dd": d}), self.wavelet, axes=axes)
        return waverec2((a, WaveletDetailTuple2d(h, v, d)), self.wavelet, axes=axes)

    def _expand_nodes(self, paths: Sequence[str]) -> None:
        axes = _neg_axes(self.axes, self.data[paths[0]].dim())
        a, h, v, d = self._wavedec(self._stack(paths), axes)
        for i, p in enumerate(paths):
            self.data[p + "a"] = a[i]
            self.data[p + "h"] = h[i]
            self.data[p + "v"] = v[i]
            self.data[p + "d"] = d[i]

    def reconstruct(self) -> "WaveletPacket2D":
        """Reconstruct the input from the leaves (reference packets.py:466-517), one synthesis call per tree level."""
        if self.maxlevel is None:
            self.maxlevel = dwt_max_level(min(self._sizes(self[""])), self.wavelet.dec_len)
        for level in reversed(range(self.maxlevel)):
            nodes = self.get_natural_order(level)
            for node in nodes:
                for child in ("a", "h", "v", "d"):
                    if node + child not in self:
                        raise KeyError(f"Key {node + child} not found")
            axes = _neg_axes(self.axes, self.data[nodes[0] + "a"].dim())
            rec = self._waverec(*[self._stack([n + c for n in nodes]) for c in ("a", "h", "v", "d")], axes)
            for i, node in enumerate(nodes):
                r = rec[i]
                if level > 0:
                    for ax in axes:
                        want = self[node].shape[ax]
                        if r.shape[ax] != want:
                            assert r.shape[ax] == want + 1, "padding error, please open an issue on GitHub"
                            r = r.narrow(ax, 0, want)
                self[node] = r
        return self

    @staticmethod
    def get_level(level: int, order: str = "freq"):
        if order == "freq":
            return WaveletPacket2D.get_freq_order(level)
        if order == "natural":
            return WaveletPacket2D.get_natural_order(level)
        raise ValueError(f"Unsupported order '{order}'. Choose from 'freq' and 'natural'.")

    @staticmethod
    def get_natural_order(level: int) -> list[str]:
        return ["".join(p) for p in product(["a", "h", "v", "d"], repeat=level)]

    @staticmethod
    def get_freq_order(level: int) -> list[list[str]]:
        """2-D frequency order: rows and columns of the node grid in Gray-code order of their 1-D paths
        (reference packets.py:716-771, after pywt's ``_wavelet_packets.py``)."""
        split = {"a": "ll", "h": "hl", "v": "lh", "d": "hh"}
        grid: dict[str, dict[str, str]] = {}
        for node in product(["a", "h", "v", "d"], repeat=level):
            row = "".join(split[c][0] for c in node)
            col = "".join(split[c][1] for c in node)
            grid.setdefault(row, {})[col] = "".join(node)
        order = _graycode_order(level, x="l", y="h") if level > 0 else ["l", "h"]
        return [[grid[r][c] for c in order if c in grid[r]] for r in order if r in grid]


class WaveletPacket3D(_PacketBase):
    """Three-dimensional wavelet packets, level-wise batched (an addition beyond the ``ptwt`` API).

    Every node is one level-1 ``wavedec3`` of its parent (``fswavedec3`` with ``separable=True``, ``MatrixWavedec3``
    in mode ``"boundary"``); its key appends the subband key (``"aaa"`` .. ``"ddd"``, first letter along ``axes[0]``)
    to the parent's, so ``"aad"`` lies at depth 1 and ``"aaddda"`` at depth 2.
    """

    _filter_keys = frozenset(SUBBANDS_3D)
    _key_chars = frozenset({"a", "d"})
    _key_width = 3
    _ndim = 3

    def __init__(self, data: Optional[torch.Tensor], wavelet: Any, *, mode: str = "reflect",
                 maxlevel: Optional[int] = None, axes: tuple[int, int, int] = (-3, -2, -1),
                 orthogonalization: str = "qr", separable: bool = False, **deprecated: Any) -> None:
        if "boundary_orthogonalization" in deprecated:
            import warnings

            warnings.warn("boundary_orthogonalization is deprecated; use orthogonalization", DeprecationWarning, stacklevel=2)
            orthogonalization = deprecated.pop("boundary_orthogonalization")
        if deprecated:
            raise TypeError(f"unexpected keyword arguments {sorted(deprecated)}")
        super().__init__()
        self.wavelet = as_wavelet(wavelet)
        self.mode = mode
        self.orthogonalization = orthogonalization
        self.separable = separable
        self.matrix_wavedec3_dict: dict[tuple[int, ...], MatrixWavedec3] = {}
        self.matrix_waverec3_dict: dict[tuple[int, ...], MatrixWaverec3] = {}
        self.axes = tuple(ensure_axes(axes, 3))
        if self.orthogonalization not in _ORTH_METHODS:
            raise NotImplementedError
        self.maxlevel: Optional[int] = None
        if data is not None:
            self.transform(data, maxlevel)
        else:
            self.data = {}

    def _check_access(self, key: str) -> None:
        super()._check_access(key)
        # every level's letters, not only the last level's: a bad key fails before any node is expanded
        if key not in self and not set(key) <= self._key_chars:
            raise self._invalid_key(key)

    def _sizes(self, t: torch.Tensor) -> tuple[int, int, int]:
        return t.shape[self.axes[0]], t.shape[self.axes[1]], t.shape[self.axes[2]]

    def transform(self, data: torch.Tensor, maxlevel: Optional[int] = None) -> "WaveletPacket3D":
        self.data = {"": data}
        if maxlevel is None:
            maxlevel = dwt_max_level(min(self._sizes(data)), self.wavelet.dec_len)
        self.maxlevel = maxlevel
        return self

    def _wavedec(self, stacked: torch.Tensor, axes: tuple[int, ...]) -> dict[str, torch.Tensor]:
        """The eight subbands of a stack of nodes, keyed like the children."""
        if self.mode == "boundary":
            shape = tuple(stacked.shape[a] for a in axes)
            if shape not in self.matrix_wavedec3_dict:
                self.matrix_wavedec3_dict[shape] = MatrixWavedec3(self.wavelet, level=1, axes=axes,
                                                                  orthogonalization=self.orthogonalization)
            a, det = self.matrix_wavedec3_dict[shape](stacked)
        elif self.separable:
            a, det = fswavedec3(stacked, self.wavelet, level=1, mode=self.mode, axes=axes)
        else:
            a, det = wavedec3(stacked, self.wavelet, level=1, mode=self.mode, axes=axes)
        return {"aaa": a, **det}

    def _waverec(self, bands: dict[str, torch.Tensor], axes: tuple[int, ...]) -> torch.Tensor:
        coeffs = (bands["aaa"], {k: bands[k] for k in SUBBANDS_3D[1:]})
        if self.mode == "boundary":
            shape = tuple(bands["aaa"].shape[a] for a in axes)
            if shape not in self.matrix_waverec3_dict:
                self.matrix_waverec3_dict[shape] = MatrixWaverec3(self.wavelet, axes=axes,
                                                                  orthogonalization=self.orthogonalization)
            return self.matrix_waverec3_dict[shape](coeffs)
        if self.separable:
            return fswaverec3(coeffs, self.wavelet, axes=axes)
        return waverec3(coeffs, self.wavelet, axes=axes)

    def _expand_nodes(self, paths: Sequence[str]) -> None:
        axes = _neg_axes(self.axes, self.data[paths[0]].dim())
        bands = self._wavedec(self._stack(paths), axes)
        for i, p in enumerate(paths):
            for c in SUBBANDS_3D:
                self.data[p + c] = bands[c][i]

    def reconstruct(self) -> "WaveletPacket3D":
        """Reconstruct the input from the leaves, one synthesis call per tree level."""
        if self.maxlevel is None:
            self.maxlevel = dwt_max_level(min(self._sizes(self[""])), self.wavelet.dec_len)
        for level in reversed(range(self.maxlevel)):
            nodes = self.get_natural_order(level)
            for node in nodes:
                for child in SUBBANDS_3D:
                    if node + child not in self:
                        raise KeyError(f"Key {node + child} not found")
            axes = _neg_axes(self.axes, self.data[nodes[0] + "aaa"].dim())
            # all children of the level in one stack [8, nodes, ...]: the seven detail bands reach the synthesis
            # kernel as equally strided slices of one buffer, without a second copy
            kids = torch.stack([self.data[n + c] for c in SUBBANDS_3D for n in nodes], 0)
            kids = kids.reshape((len(SUBBANDS_3D), len(nodes)) + kids.shape[1:])
            rec = self._waverec(dict(zip(SUBBANDS_3D, kids.unbind(0))), axes)
            for i, node in enumerate(nodes):
                r = rec[i]
                if level > 0:
                    for ax in axes:
                        want = self[node].shape[ax]
                        if r.shape[ax] != want:
                            assert r.shape[ax] == want + 1, "padding error, please open an issue on GitHub"
                            r = r.narrow(ax, 0, want)
                self[node] = r
        return self

    @staticmethod
    def get_level(level: int, order: str = "freq"):
        if order == "freq":
            return WaveletPacket3D.get_freq_order(level)
        if order == "natural":
            return WaveletPacket3D.get_natural_order(level)
        raise ValueError(f"Unsupported order '{order}'. Choose from 'freq' and 'natural'.")

    @staticmethod
    def get_natural_order(level: int) -> list[str]:
        return ["".join(p) for p in product(SUBBANDS_3D, repeat=level)]

    @staticmethod
    def get_freq_order(level: int) -> list[list[list[str]]]:
        """3-D frequency order ``[depth][row][col]``: the node grid indexed by the 1-D filter path along each of the
        three axes, every axis in Gray-code order of its paths (the 3-D form of ``WaveletPacket2D.get_freq_order``)."""
        to_lh = {"a": "l", "d": "h"}
        grid: dict[tuple[str, str, str], str] = {}
        for node in WaveletPacket3D.get_natural_order(level):
            grid[tuple("".join(to_lh[c] for c in node[a::3]) for a in range(3))] = node
        order = _graycode_order(level, x="l", y="h")
        return [[[grid[d, r, c] for c in order] for r in order] for d in order]
