"""Node-by-node restatement of 3-D wavelet packets (float64 in the conv modes) -- TEST INFRASTRUCTURE ONLY.

The oracle of ``pytorch_wavelet_toolbox_b200.WaveletPacket3D``.  The reference has no 3-D packets, so there is no
fixture: the tree is a plain recursive dict in which every node is ONE level-1 transform of its parent, computed by the
port's pinned building blocks (``tests/test_oracle.py``) without any batching of nodes:

  conv modes        ``ptwt_port.wavedec3(level=1)`` / ``ptwt_port.waverec3``
  separable=True    three passes of the port's level-1 1-D ``wavedec`` per node, last axis first, and ``waverec`` in the
                    opposite order (reference ``separable_conv_transform.py:39-112``)
  mode "boundary"   ``ptwt_port.MatrixWavedec3(level=1)`` / ``ptwt_port.MatrixWaverec3``

A node key is one 3-letter subband key per level, letter i the filter along ``axes[i]``.  Everything runs on the CPU
and keeps the autograd graph, so it is the oracle of the gradients too.  The conv modes compute in float64.  Mode
"boundary" computes in the input's dtype, because its operator depends on that dtype, as in the reference: the
orthogonalised boundary rows come from a QR in the input's dtype, and for filters longer than 4 taps the float32 and
float64 QR return some boundary rows with opposite signs (a pivot that is zero in exact arithmetic takes its sign from
round-off).
"""
from __future__ import annotations

from itertools import product
from typing import Any, Sequence

import torch

from oracle import ptwt_port as P

SUBBANDS = tuple("".join(p) for p in product("ad", repeat=3))


def _level1(x: torch.Tensor, wavelet: Any, mode: str, axes: Sequence[int], separable: bool,
            orthogonalization: str) -> dict[str, torch.Tensor]:
    if mode == "boundary":
        a, det = P.MatrixWavedec3(wavelet, 1, axes=axes, orthogonalization=orthogonalization)(x)
        return {"aaa": a, **det}
    if separable:
        # the reference's _separable_conv_dwtn_: split along axes[2], then each half along axes[1], then axes[0];
        # every split prepends its letter, so letter i ends up belonging to axes[i]
        parts = {"": x}
        for ax in reversed(axes):
            nxt = {}
            for key, t in parts.items():
                lo, hi = P.wavedec(t, wavelet, mode=mode, level=1, axis=ax)
                nxt["a" + key], nxt["d" + key] = lo, hi
            parts = nxt
        return parts
    a, det = P.wavedec3(x, wavelet, mode=mode, level=1, axes=axes)
    return {"aaa": a, **det}


def _synthesis1(bands: dict[str, torch.Tensor], wavelet: Any, mode: str, axes: Sequence[int], separable: bool,
                orthogonalization: str) -> torch.Tensor:
    if mode == "boundary":
        return P.MatrixWaverec3(wavelet, axes=axes, orthogonalization=orthogonalization)(
            (bands["aaa"], {k: bands[k] for k in SUBBANDS[1:]}))
    if separable:
        # the reference's _separable_conv_idwtn: merge the first letter (axes[0]) first
        parts = dict(bands)
        for ax in axes:
            parts = {key[1:]: P.waverec([parts[key], parts["d" + key[1:]]], wavelet, axis=ax)
                     for key in parts if key[0] == "a"}
        return parts[""]
    return P.waverec3((bands["aaa"], {k: bands[k] for k in SUBBANDS[1:]}), wavelet, axes=axes)


def _neg(axes: Sequence[int], ndim: int) -> tuple[int, ...]:
    return tuple(a if a < 0 else a - ndim for a in axes)


def packet_tree(x: torch.Tensor, wavelet: Any, maxlevel: int, *, mode: str = "reflect",
                axes: Sequence[int] = (-3, -2, -1), separable: bool = False,
                orthogonalization: str = "qr") -> dict[str, torch.Tensor]:
    """Every node down to ``maxlevel``: {key: tensor}, the root under ``""``; on the CPU, in float64 except in mode
    "boundary" (see the module docstring)."""
    axes = _neg(axes, x.dim())
    tree = {"": x.cpu() if mode == "boundary" else x.cpu().double()}

    def walk(key: str, depth: int) -> None:
        if depth == maxlevel:
            return
        for sub, t in _level1(tree[key], wavelet, mode, axes, separable, orthogonalization).items():
            tree[key + sub] = t
            walk(key + sub, depth + 1)

    walk("", 0)
    return tree


def reconstruct(tree: dict[str, torch.Tensor], wavelet: Any, maxlevel: int, *, mode: str = "reflect",
                axes: Sequence[int] = (-3, -2, -1), separable: bool = False,
                orthogonalization: str = "qr") -> torch.Tensor:
    """The root rebuilt from the leaves at ``maxlevel``, node by node: a node rebuilt one sample longer than the one
    stored is cut back on that axis; the root is not."""
    tree = dict(tree)
    axes = _neg(axes, tree[""].dim())

    def rebuild(key: str, depth: int) -> torch.Tensor:
        if depth == maxlevel:
            return tree[key]
        r = _synthesis1({sub: rebuild(key + sub, depth + 1) for sub in SUBBANDS}, wavelet, mode, axes, separable,
                        orthogonalization)
        if depth > 0:
            for ax in axes:
                r = r.narrow(ax, 0, tree[key].shape[ax])
        return r

    return rebuild("", 0)
