"""Closed-form float64 restatement of the 2-D stationary transform -- TEST INFRASTRUCTURE ONLY.

Plain index arithmetic in numpy, independent of torch's convolutions (oracle/swt2_port.py uses those).  Level j,
d = 2^(j-1), hl = L/2 - 1, f = dec[::-1], a the filter along the first of the two axes, b along the second:

  analysis   c_ab[r, s] = sum_m sum_k f_a[m] f_b[k] A[(r + d (m - hl)) mod H, (s + d (k - hl)) mod W]
  synthesis  A[r, s] = sum_ab sum_m sum_k g_a[m] g_b[k] c_ab[(r + d (hl - m)) mod H, (s + d (hl - k)) mod W],
             g = 0.5 rec

Bands in the order cA (lo, lo), cH (hi, lo), cV (lo, hi), cD (hi, hi).
"""
from __future__ import annotations

import numpy as np

_PAIRS = ((0, 0), (1, 0), (0, 1), (1, 1))


def swt2(x: np.ndarray, dec_lo, dec_hi, level: int) -> list:
    """``x [..., H, W]`` -> ``[cA_J, (cH_J, cV_J, cD_J), ..., (cH_1, cV_1, cD_1)]``."""
    a = np.asarray(x, dtype=np.float64)
    H, W = a.shape[-2:]
    L = len(dec_lo)
    hl = L // 2 - 1
    f = (np.asarray(dec_lo, dtype=np.float64)[::-1], np.asarray(dec_hi, dtype=np.float64)[::-1])
    r, s = np.arange(H), np.arange(W)
    details = []
    for j in range(1, level + 1):
        d = 2 ** (j - 1)
        bands = []
        for pa, pb in _PAIRS:
            c = np.zeros_like(a)
            for m in range(L):
                rows = (r + d * (m - hl)) % H
                for k in range(L):
                    cols = (s + d * (k - hl)) % W
                    c += f[pa][m] * f[pb][k] * a[..., rows[:, None], cols[None, :]]
            bands.append(c)
        a = bands[0]
        details.append(tuple(bands[1:]))
    return [a] + details[::-1]


def iswt2(coeffs, rec_lo, rec_hi) -> np.ndarray:
    y = np.asarray(coeffs[0], dtype=np.float64)
    H, W = y.shape[-2:]
    L = len(rec_lo)
    hl = L // 2 - 1
    g = (0.5 * np.asarray(rec_lo, dtype=np.float64), 0.5 * np.asarray(rec_hi, dtype=np.float64))
    r, s = np.arange(H), np.arange(W)
    J = len(coeffs) - 1
    for lv, det in enumerate(coeffs[1:]):
        d = 2 ** (J - 1 - lv)
        bands = [y] + [np.asarray(t, dtype=np.float64) for t in det]
        out = np.zeros_like(y)
        for (pa, pb), c in zip(_PAIRS, bands):
            for m in range(L):
                rows = (r + d * (hl - m)) % H
                for k in range(L):
                    cols = (s + d * (hl - k)) % W
                    out += g[pa][m] * g[pb][k] * c[..., rows[:, None], cols[None, :]]
        y = out
    return y
