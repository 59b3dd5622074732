"""Torch restatement of the reference's per-scale FFT continuous wavelet transform -- TEST INFRASTRUCTURE ONLY.

It follows the algorithm of ``ptwt.cwt`` (src/ptwt/continuous_transform.py:27-156) step by step, on whatever device
the data is on: integrate the sampled wavelet, pick the filter taps at each scale from an index table computed in
the data's dtype on the CPU, convolve through a zero-padded FFT of power-of-two size, take ``-sqrt(scale)`` times the first
difference, crop the centre, and stack the scales.  The data spectrum is taken in the data's precision (complex64
for float32 input) and promoted by the complex128 filter spectrum, as in the reference.  Written independently of
the product's overlap-save kernels; it is what the GPU tests and tools/time_cwt.py compare ``cwt`` against.
"""
from __future__ import annotations

from typing import Any

import numpy as np
import torch

from pytorch_wavelet_toolbox_b200._wavelets import BuiltinContinuousWavelet, _pywt, as_continuous_wavelet


def _samples(wavelet: Any, precision: int, device: torch.device):
    if isinstance(wavelet, torch.nn.Module):
        with torch.no_grad():
            psi, grid = wavelet.wavefun(precision)
        psi, grid = psi.cpu(), grid.cpu()
        conj = bool(wavelet.complex_cwt)
    else:
        out = wavelet.wavefun(precision)
        psi, grid = (out[0], out[1]) if len(out) == 2 else (out[1], out[2])
        psi, grid = torch.as_tensor(np.asarray(psi)), torch.as_tensor(np.asarray(grid))
        exact = (BuiltinContinuousWavelet,) + ((_pywt.ContinuousWavelet,) if _pywt is not None else ())
        conj = type(wavelet) in exact and bool(wavelet.complex_cwt)
    integral = torch.cumsum(psi, 0) * (grid[1] - grid[0])
    if conj:
        integral = integral.conj().resolve_conj()
    return integral.to(device), grid.to(torch.float64)


def cwt(data: torch.Tensor, scales: Any, wavelet: Any, sampling_period: float = 1.0, precision: int = 12,
        index_dtype: Any = None):
    """``index_dtype``: the dtype in which the sample positions of the scaled wavelet are computed (default: the
    data's, as the reference does).  A float32 transform picks its taps in float32; checking it with float64
    arithmetic needs the same taps."""
    wav = as_continuous_wavelet(wavelet)
    if isinstance(scales, torch.Tensor):
        scales = scales.cpu().numpy()
    elif np.isscalar(scales):
        scales = np.array([scales])
    int_psi, grid = _samples(wav, precision, data.device)
    lo, hi, dx = float(grid[0]), float(grid[-1]), float(grid[1] - grid[0])
    n = data.shape[-1]
    coefs = []
    cached_len, data_hat = None, None
    for s in scales:
        # on the CPU whatever the data's device: CUDA divides a float32 tensor by a scalar as a multiplication by the
        # reciprocal, which picks other taps at some scales than the reference's CPU tables (the fixtures) do
        pos = torch.arange(float(s) * (hi - lo) + 1, dtype=index_dtype or data.dtype) / (float(s) * dx)
        pos = torch.floor(pos).long()
        pos = pos[pos < int_psi.shape[0]]
        taps = torch.flip(int_psi.cpu()[pos], (0,)).to(data.device)
        K = taps.shape[0]
        size = 1 << int(np.ceil(np.log2(n + K - 1)))
        if size != cached_len:
            data_hat, cached_len = torch.fft.fft(data, size, dim=-1), size
        full = torch.fft.ifft(data_hat * torch.fft.fft(taps, size), dim=-1)[..., : n + K - 1]
        if K < 2:
            raise ValueError(f"Selected scale of {s} too small.")
        step = -np.sqrt(s) * (full[..., 1:] - full[..., :-1])
        left = (K - 2) // 2
        coefs.append(step[..., left: left + n])
    out = torch.stack(coefs)
    complex_out = bool(getattr(wav, "complex_cwt", False)) and not (_pywt is not None and type(wav) is _pywt.Wavelet)
    if not complex_out:
        out = out.real
    if isinstance(wav, torch.nn.Module):
        with torch.no_grad():
            psi = wav.wavefun(precision)[0].cpu().numpy()
    else:
        approx = wav.wavefun(precision)
        psi = np.asarray(approx[0] if len(approx) == 2 else approx[1])
    index = np.argmax(np.abs(np.fft.fft(psi)[1:])) + 2
    if index > len(psi) / 2:
        index = len(psi) - index + 2
    freqs = np.float64(index - 1) / (hi - lo) / scales
    if np.isscalar(freqs):
        freqs = np.array([freqs])
    return out, freqs / sampling_period
