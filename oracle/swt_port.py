"""CPU restatement ("port") of ptwt.swt / ptwt.iswt -- TEST INFRASTRUCTURE ONLY.

Written from the closed form of the reference's stationary transform (src/ptwt/stationary_transform.py), with the
same torch CPU operators it calls so that float64 results agree bit for bit:

  analysis   level j, d = 2^(j-1):  E(a) = extension by (d (L/2 - 1), d L/2), then conv1d(dilation d) with the
             flipped dec_lo / dec_hi; keep [cA_J, cD_J, ..., cD_1]
  synthesis  level j from J down:   E(stack[a, cD_j]) by (d L/2, d (L/2 - 1)), conv_transpose1d(dilation d,
             groups 2, padding = both pads) with rec_lo / rec_hi, mean of the two channels
  E          periodic while both pads fit in n; a longer pad is applied in rounds of at most n samples per side,
             each wrapping the tensor built so far (not periodic when a round before the last adds a total that is
             not a multiple of n)

Only tests/ and __graft_entry__.smoke() import it; the product package never does.
"""
from __future__ import annotations

from typing import Any, Optional

import torch
import torch.nn.functional as F

from oracle.ptwt_port import _axes, _fold, _taps, _unfold
from pytorch_wavelet_toolbox_b200._wavelets import swt_max_level


def extension_index(n: int, pl: int, pr: int) -> torch.Tensor:
    """Source sample in [0, n) of every position of the reference's extension of a length-n signal by (pl, pr)."""
    idx = torch.arange(n)
    while True:
        a, b = min(n, pl), min(n, pr)
        ln = idx.numel()
        idx = torch.cat([idx[ln - a:], idx, idx[:b]])
        pl, pr = pl - a, pr - b
        if pl <= 0 and pr <= 0:
            return idx


def swt(data: torch.Tensor, wavelet: Any, level: Optional[int] = None, *, axis=None) -> list[torch.Tensor]:
    ax = _axes(axis, 1)
    x, shape = _fold(data, 1, ax)
    n = x.shape[-1]
    if level is None:
        level = swt_max_level(n)
    dec_lo, dec_hi, _, _ = _taps(wavelet, x.dtype, flip=True)
    L = dec_lo.shape[0]
    filt = torch.stack([dec_lo, dec_hi], 0).unsqueeze(1).to(x.device)
    lo = x.unsqueeze(1)
    details = []
    for j in range(level):
        d = 2 ** j
        ext = lo[..., extension_index(n, d * (L // 2 - 1), d * (L // 2)).to(x.device)]
        res = F.conv1d(ext, filt, dilation=d)
        lo = res[:, :1]
        details.append(res[:, 1])
    out = [lo.squeeze(1)] + details[::-1]
    return [_unfold(t, 1, ax, shape) for t in out]


def iswt(coeffs, wavelet: Any, *, axis=None) -> torch.Tensor:
    ax = _axes(axis, 1)
    coeffs = list(coeffs)
    y, shape = _fold(coeffs[0], 1, ax)
    details = [_fold(c, 1, ax, len(shape))[0] for c in coeffs[1:]]
    _, _, rec_lo, rec_hi = _taps(wavelet, y.dtype, flip=False)
    L = rec_lo.shape[0]
    filt = torch.stack([rec_lo, rec_hi], 0).unsqueeze(1).to(y.device)
    n = y.shape[-1]
    for k, hi in enumerate(details):
        d = 2 ** (len(details) - 1 - k)
        pl, pr = d * (L // 2), d * (L // 2 - 1)
        z = torch.stack([y, hi], 1)[..., extension_index(n, pl, pr).to(y.device)]
        y = F.conv_transpose1d(z, filt, dilation=d, groups=2, padding=pl + pr).mean(1)
    return _unfold(y, 1, ax, shape)
