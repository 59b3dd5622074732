"""Closed-form float64 restatement of the stationary transform -- TEST INFRASTRUCTURE ONLY.

Plain index arithmetic in numpy, independent of torch's convolutions (oracle/swt_port.py uses those):

  analysis   level j, d = 2^(j-1), hl = L/2 - 1:   c_k[i] = sum_m dec_k[L-1-m] * a[src(i + d m)]
             with src = the extension by (d hl, d L/2); periodic: src(i + d m) = (i + d (m - hl)) mod n
  synthesis  y[i] = 0.5 * sum_m (rec_lo[m] a[src'(i + P - d m)] + rec_hi[m] c_j[src'(i + P - d m)])
             with src' = the extension by (d L/2, d hl), P = d (L - 1); periodic: (i + d (hl - m)) mod n
"""
from __future__ import annotations

import numpy as np

from oracle.swt_port import extension_index


def swt(x: np.ndarray, dec_lo, dec_hi, level: int) -> list[np.ndarray]:
    """``x [..., n]`` -> ``[cA_J, cD_J, ..., cD_1]``."""
    a = np.asarray(x, dtype=np.float64)
    n, L = a.shape[-1], len(dec_lo)
    hl = L // 2 - 1
    i = np.arange(n)
    details = []
    for j in range(1, level + 1):
        d = 2 ** (j - 1)
        src = extension_index(n, d * hl, d * (L // 2)).numpy()
        lo = np.zeros_like(a)
        hi = np.zeros_like(a)
        for m in range(L):
            s = src[i + d * m]
            lo += dec_lo[L - 1 - m] * a[..., s]
            hi += dec_hi[L - 1 - m] * a[..., s]
        details.append(hi)
        a = lo
    return [a] + details[::-1]


def iswt(coeffs, rec_lo, rec_hi) -> np.ndarray:
    y = np.asarray(coeffs[0], dtype=np.float64)
    n, L = y.shape[-1], len(rec_lo)
    hl = L // 2 - 1
    i = np.arange(n)
    J = len(coeffs) - 1
    for k, c in enumerate(coeffs[1:]):
        d = 2 ** (J - 1 - k)
        src = extension_index(n, d * (L // 2), d * hl).numpy()
        c = np.asarray(c, dtype=np.float64)
        out = np.zeros_like(y)
        for m in range(L):
            s = src[i + d * (L - 1) - d * m]
            out += rec_lo[m] * y[..., s] + rec_hi[m] * c[..., s]
        y = 0.5 * out
    return y


def periodic(n: int, pl: int, pr: int) -> np.ndarray:
    """The periodic extension's source indices, for comparison with :func:`extension_index`."""
    return (np.arange(n + pl + pr) - pl) % n
