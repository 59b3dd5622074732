"""CPU restatement ("port") of the 2-D stationary transform swt2 / iswt2 -- TEST INFRASTRUCTURE ONLY.

The reference has no swt2, so this is written from the definition (PyWavelets' swt2 with trim_approx=True,
norm=False) in the reference's own style for the 1-D swt and for wavedec2:

  analysis   level j, d = 2^(j-1): periodic index padding by (d (L/2 - 1), d L/2) along both axes, conv2d(dilation d)
             with the four outer-product filters of the flipped dec_lo / dec_hi that the port builds for wavedec2
             (outer(lo, lo), outer(hi, lo), outer(lo, hi), outer(hi, hi); the first factor along axes[0]), split
             into cA, cH, cV, cD
  synthesis  level j from J down: stack [cA, cH, cV, cD], periodic padding by (d L/2, d (L/2 - 1)) along both axes,
             conv_transpose2d(dilation d, groups 4) with the outer products of rec_lo / rec_hi, mean of the four

Unlike oracle/swt_port.py the extension is periodic at every level, also where a pad exceeds the extent.
Only tests/ and tools/ import it; the product package never does.
"""
from __future__ import annotations

from typing import Any, Optional

import torch
import torch.nn.functional as F

from oracle.ptwt_port import _axes, _fold, _nd_filters, _taps, _unfold
from pytorch_wavelet_toolbox_b200._wavelets import swt_max_level
from pytorch_wavelet_toolbox_b200.constants import WaveletDetailTuple2d


def periodic_index(n: int, pl: int, pr: int, device=None) -> torch.Tensor:
    """Source sample in [0, n) of every position of the periodic extension of a length-n axis by (pl, pr)."""
    return (torch.arange(n + pl + pr, device=device) - pl) % n


def _pad2(t: torch.Tensor, pl: int, pr: int) -> torch.Tensor:
    """Periodic padding of the last two axes of ``t`` by (pl, pr) each."""
    H, W = t.shape[-2:]
    t = t[..., periodic_index(H, pl, pr, t.device), :]
    return t[..., periodic_index(W, pl, pr, t.device)]


def swt2(data: torch.Tensor, wavelet: Any, level: Optional[int] = None, *, axes=(-2, -1)):
    ax = _axes(axes, 2)
    x, shape = _fold(data, 2, ax)
    H, W = x.shape[-2:]
    if level is None:
        level = min(swt_max_level(H), swt_max_level(W))
    dec_lo, dec_hi, _, _ = _taps(wavelet, x.dtype, flip=True)
    L = dec_lo.shape[0]
    filt = _nd_filters(dec_lo, dec_hi, 2).to(x.device)
    a = x.unsqueeze(1)
    details = []
    for j in range(level):
        d = 2 ** j
        res = F.conv2d(_pad2(a, d * (L // 2 - 1), d * (L // 2)), filt, dilation=d)
        a = res[:, :1]
        details.append((res[:, 1], res[:, 2], res[:, 3]))
    out: list[Any] = [_unfold(a.squeeze(1), 2, ax, shape)]
    for h, v, dd in reversed(details):
        out.append(WaveletDetailTuple2d(*[_unfold(t, 2, ax, shape) for t in (h, v, dd)]))
    return tuple(out)


def iswt2(coeffs, wavelet: Any, *, axes=None) -> torch.Tensor:
    ax = _axes(axes, 2)
    y, shape = _fold(coeffs[0], 2, ax)
    levels = [[_fold(t, 2, ax, len(shape))[0] for t in el] for el in coeffs[1:]]
    _, _, rec_lo, rec_hi = _taps(wavelet, y.dtype, flip=False)
    L = rec_lo.shape[0]
    filt = _nd_filters(rec_lo, rec_hi, 2).to(y.device)
    for k, (h, v, dd) in enumerate(levels):
        d = 2 ** (len(levels) - 1 - k)
        pl, pr = d * (L // 2), d * (L // 2 - 1)
        z = _pad2(torch.stack([y, h, v, dd], 1), pl, pr)
        y = F.conv_transpose2d(z, filt, dilation=d, groups=4, padding=pl + pr).mean(1)
    return _unfold(y, 2, ax, shape)
