"""Filter banks that are not orthogonal, given as taps (no PyWavelets needed).

Every orthogonal bank has ``rec = reversed dec`` and ``dec_hi = alternating flip of dec_lo``, so a kernel, a tap table
or an autograd adjoint that takes the other filter of the bank, or the right filter in the wrong direction, computes
the same numbers as the correct code on every db / sym / haar bank.  The banks here break both identities:

* ``unstructured(L)``: four independent seeded random filters of any length (``dec_lo`` sums to sqrt(2), the other
  three have unit norm, so that deep levels neither blow up nor vanish; for half of the lengths the first tap is zero,
  the way PyWavelets pads its biorthogonal banks).  They reconstruct nothing: synthesis is compared with the
  oracle's synthesis of the same coefficients.
* ``bior22()`` and ``cdf97()``: perfect-reconstruction biorthogonal banks in PyWavelets' bior2.2 / bior4.4 layout.

A bank is an object with ``name``, ``filter_bank``, ``dec_lo`` / ``dec_hi`` / ``rec_lo`` / ``rec_hi``, ``dec_len`` /
``rec_len`` and ``__len__``: what ``WaveletTensorTuple.from_wavelet``, this package and the oracle read.
"""
from __future__ import annotations

import functools
import math

import numpy as np

SQRT2 = math.sqrt(2.0)
#: lengths of the unrolled fused / TMA kernels, of the general kernels (longer), and odd lengths (general kernels)
EVEN_LENGTHS = (2, 4, 6, 8, 10, 12, 14, 16)
LONG_LENGTHS = (18, 20)
ODD_LENGTHS = (3, 5, 7)
ALL_LENGTHS = EVEN_LENGTHS + LONG_LENGTHS + ODD_LENGTHS
#: lengths whose unstructured bank starts with a zero tap (half of them)
ZERO_FIRST = (4, 8, 12, 16, 20, 5)


class FilterBank:
    """A wavelet given by its four filters (plain float lists)."""

    def __init__(self, name: str, dec_lo, dec_hi, rec_lo, rec_hi):
        self.name = name
        self.dec_lo, self.dec_hi, self.rec_lo, self.rec_hi = ([float(v) for v in f]
                                                              for f in (dec_lo, dec_hi, rec_lo, rec_hi))
        assert len({len(self.dec_lo), len(self.dec_hi), len(self.rec_lo), len(self.rec_hi)}) == 1, name
        self.dec_len = self.rec_len = len(self.dec_lo)

    @property
    def filter_bank(self):
        return (self.dec_lo, self.dec_hi, self.rec_lo, self.rec_hi)

    def __len__(self) -> int:
        return self.dec_len

    def __repr__(self) -> str:
        return self.name


def _unit(v: np.ndarray) -> np.ndarray:
    return v / np.linalg.norm(v)


@functools.lru_cache(maxsize=None)
def unstructured(filt_len: int, variant: int = 0) -> FilterBank:
    """Four independent random filters of `filt_len` taps (seeded by length and variant)."""
    rng = np.random.default_rng(1000 * variant + filt_len)
    zero_first = filt_len in ZERO_FIRST
    while True:
        f = rng.standard_normal((4, filt_len))
        if zero_first:
            f[:, 0] = 0.0
        lo = f[0] * (SQRT2 / f[0].sum())
        # a low-pass whose taps nearly cancel needs a large gain to sum to sqrt(2), and that gain compounds over the
        # levels (an orthogonal low-pass has norm 1): draw again
        if np.linalg.norm(lo) > 1.5:
            continue
        bank = FilterBank(f"unstructured{filt_len}" + (f"v{variant}" if variant else ""),
                          lo, _unit(f[1]), _unit(f[2]), _unit(f[3]))
        if not orthogonal_structure(bank):
            return bank


def bior22() -> FilterBank:
    """bior2.2 (CDF 5/3): reconstructs to round-off in every mode."""
    return FilterBank("bior2.2",
                      [SQRT2 * v for v in (0, -1 / 8, 1 / 4, 3 / 4, 1 / 4, -1 / 8)],
                      [SQRT2 * v for v in (0, 1 / 4, -1 / 2, 1 / 4, 0, 0)],
                      [SQRT2 * v for v in (0, 1 / 4, 1 / 2, 1 / 4, 0, 0)],
                      [SQRT2 * v for v in (0, 1 / 8, 1 / 4, -3 / 4, 1 / 4, 1 / 8)])


#: lifting factors of the CDF 9/7 wavelet (Daubechies & Sweldens, "Factoring wavelet transforms into lifting steps")
_ALPHA = -1.586134342059924
_BETA = -0.05298011857296141
_GAMMA = 0.8829110755309333
_DELTA = 0.4435068520439712


def _lifting_matrix(n: int) -> np.ndarray:
    """The 9/7 lifting analysis on periodic signals of n samples as a matrix: rows [0, n/2) give the low-pass
    outputs, rows [n/2, n) the high-pass outputs (no final scaling: the filters are normalised afterwards)."""
    out = np.empty((n, n))
    for j in range(n):
        x = np.zeros(n)
        x[j] = 1.0
        s, d = x[0::2].copy(), x[1::2].copy()
        d += _ALPHA * (s + np.roll(s, -1))
        s += _BETA * (d + np.roll(d, 1))
        d += _GAMMA * (s + np.roll(s, -1))
        s += _DELTA * (d + np.roll(d, 1))
        out[:, j] = np.concatenate([s, d])
    return out


@functools.lru_cache(maxsize=None)
def cdf97() -> FilterBank:
    """CDF 9/7 in the bior4.4 layout (10 taps): derived in float64 from the lifting factors, so the bank reconstructs
    exactly up to round-off (the 16-digit taps usually quoted reconstruct only to ~4e-12).

    Lifting is invertible for any factors, so the analysis low-pass (a row of the lifting matrix, 9 taps) and the
    synthesis low-pass (a column of its inverse, 7 taps) form a biorthogonal pair; each is scaled to sum sqrt(2),
    and the two high-pass filters follow by alternating the signs of the other bank's low-pass."""
    n, c = 32, 8
    a = _lifting_matrix(n)
    h = a[c, 2 * c - 4: 2 * c + 5]                   # analysis low-pass around input 2c, symmetric
    g = np.linalg.inv(a)[2 * c - 3: 2 * c + 4, c]    # synthesis low-pass of output c, symmetric
    h = h * (SQRT2 / h.sum())
    g = g * (SQRT2 / g.sum())
    dec_lo = np.concatenate([[0.0], h])
    rec_lo = np.concatenate([[0.0], g, [0.0, 0.0]])
    sign = np.array([(-1.0) ** k for k in range(10)])
    return FilterBank("cdf9/7", dec_lo, -sign * rec_lo, rec_lo, sign * dec_lo)


#: CDF 9/7 as usually quoted (PyWavelets' bior4.4, 16 digits): the derived bank agrees with it to ~1e-12
CDF97_QUOTED_DEC_LO = (0.0, 0.03782845550726404, -0.023849465019556843, -0.11062440441843718, 0.37740285561283066,
                       0.8526986790088938, 0.37740285561283066, -0.11062440441843718, -0.023849465019556843,
                       0.03782845550726404)
CDF97_QUOTED_REC_LO = (0.0, -0.06453888262869706, -0.04068941760916406, 0.41809227322161724, 0.7884856164055829,
                       0.41809227322161724, -0.04068941760916406, -0.06453888262869706, 0.0, 0.0)

PR_BANKS = {"bior2.2": bior22, "cdf9/7": cdf97}


def pr_bank(filt_len: int):
    """The perfect-reconstruction bank of this length, or None."""
    return {6: bior22, 10: cdf97}.get(filt_len, lambda: None)()


# ---- how far a bank is from the structure of an orthogonal one ------------------------------------------------------
#: a filter counts as (anti-)palindromic / a bank as orthogonally structured within this distance (unit-scaled taps)
STRUCTURE_TOL = 0.1


def _dist(a, b) -> float:
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(np.abs(a).max(), np.abs(b).max()))


def alternating_flip(f) -> np.ndarray:
    """g[k] = (-1)^k f[L-1-k]: the high-pass an orthogonal bank derives from its low-pass (up to a global sign)."""
    f = np.asarray(f, dtype=np.float64)
    return np.array([(-1.0) ** k for k in range(len(f))]) * f[::-1]


def structure_distances(bank: FilterBank) -> dict[str, float]:
    """Distances (relative max-abs) of the identities an orthogonal bank satisfies; all > STRUCTURE_TOL for a bank
    that tells the filters and their directions apart."""
    d = {}
    for name in ("dec_lo", "dec_hi", "rec_lo", "rec_hi"):
        f = np.asarray(getattr(bank, name))
        d[f"{name} palindrome"] = _dist(f, f[::-1])
        d[f"{name} anti-palindrome"] = _dist(f, -f[::-1])
    d["rec_lo = reversed dec_lo"] = _dist(bank.rec_lo, bank.dec_lo[::-1])
    d["rec_hi = reversed dec_hi"] = _dist(bank.rec_hi, bank.dec_hi[::-1])
    flip = alternating_flip(bank.dec_lo)
    d["dec_hi = alternating flip of dec_lo"] = min(_dist(bank.dec_hi, flip), _dist(bank.dec_hi, -flip))
    return d


def orthogonal_structure(bank: FilterBank) -> list[str]:
    """The identities of an orthogonal bank that `bank` satisfies to within STRUCTURE_TOL."""
    return [k for k, v in structure_distances(bank).items() if v <= STRUCTURE_TOL]


def bank_for_length(filt_len: int, alt: bool = False) -> FilterBank:
    """The bank a kernel case of `filt_len` taps runs with: where the case uses its alternative wavelet, the
    perfect-reconstruction bank of that length if there is one, else a second unstructured bank."""
    if alt:
        return pr_bank(filt_len) or unstructured(filt_len, 1)
    return unstructured(filt_len)
