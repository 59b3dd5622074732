"""Continuous wavelet transform on the H100.

Drop-in for ``ptwt.cwt`` (reference ``src/ptwt/continuous_transform.py:27-156``): same signature, output dtype
(float64, or complex128 for complex wavelets, whatever the input precision) and shape ``[S, *data.shape]``, same
frequencies and error types.  The reference's per-scale loop (FFT of filter and data, product, inverse FFT, ``diff``,
crop, and finally ``torch.stack``) is replaced by uniformly partitioned overlap-save in float64 on libwtb200
(``wt_cwt_*``, include/wtb200.h, csrc/cwt.cuh): one launch computes the spectra of the data blocks, shared by every
scale, and one launch produces every scale's output blocks straight into the result.  Real-wavelet scales run in
pairs through one complex inverse FFT.

The per-scale filter is built on the host exactly as the reference builds it, including the index table computed in
the data's dtype (for float32 input it differs from the float64 table at many scales), then folded with the diff,
the ``-sqrt(scale)`` factor and the crop into one FIR per scale:
    y_s[t] = sum_{k=0..K} g_s[k] x[t + f_s + 1 - k],   g_s[k] = -sqrt(s) (h_s[k] - h_s[k-1]),  f_s = (K - 2) // 2.
Index tables, taps and their spectra are cached per (wavelet samples, scales, precision, dtype, FFT size, device).

CPU tensors are staged to the current CUDA device and back, as in :func:`swt`.  Gradients flow to the data through
the adjoint kernels; gradients with respect to a wavelet's own parameters are not supported.
"""
from __future__ import annotations

import collections
import functools
import hashlib
from typing import Any, Union

import numpy as np
import torch

from . import _native as N
from ._shape import check_dtype
from ._wavelets import BuiltinContinuousWavelet, _pywt, as_continuous_wavelet
from .fwt import _compute_device, _dtype_code, pinned_empty

__all__ = ["cwt"]

MIN_HOP_LOG2, MAX_HOP_LOG2 = 5, 11     # H = 32 .. 2048, F = 2H (csrc/cwt.cuh: 2^6 .. 2^12)
_META = 6
_CACHE_SIZE = 16


# --------------------------------------------------------------------------------------
# the wavelet, sampled and integrated (reference _integrate_wavelet, continuous_transform.py:159-226)
# --------------------------------------------------------------------------------------
class _Sampled:
    """``int_psi`` and the grid of one wavelet at one precision, plus what the reference derives from its type."""

    def __init__(self, int_psi: np.ndarray, psi: np.ndarray, x: np.ndarray, complex_out: bool):
        self.int_psi, self.psi, self.x, self.complex_out = int_psi, psi, x, complex_out
        h = hashlib.blake2b(digest_size=16)
        for a in (int_psi, x):
            h.update(str(a.dtype).encode())
            h.update(np.ascontiguousarray(a).tobytes())
        self.key = (h.hexdigest(), bool(complex_out))

    @functools.cached_property
    def central_frequency(self) -> np.float64:
        return central_frequency(self.psi, self.x)


def _as_numpy(a: Any) -> np.ndarray:
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def _is_module_wavelet(wav: Any) -> bool:
    return isinstance(wav, torch.nn.Module) and hasattr(wav, "complex_cwt")


def _check_params_without_grad(wav: Any) -> None:
    if isinstance(wav, torch.nn.Module) and torch.is_grad_enabled() and any(p.requires_grad for p in wav.parameters()):
        raise NotImplementedError(
            "cwt computes gradients with respect to the data only, not with respect to the wavelet's learnable "
            "parameters; call it under torch.no_grad() or freeze the parameters (requires_grad_(False))."
        )


def _conjugates(wav: Any) -> bool:
    """The reference conjugates ``int_psi`` only for an object whose type is exactly ``ContinuousWavelet`` and for its
    own learnable modules, when the wavelet is complex (continuous_transform.py:87-91)."""
    exact = (BuiltinContinuousWavelet,) + ((_pywt.ContinuousWavelet,) if _pywt is not None else ())
    if type(wav) in exact or _is_module_wavelet(wav):
        return bool(getattr(wav, "complex_cwt", False))
    return False


def _complex_out(wav: Any) -> bool:
    """pywt's ``Wavelet`` gives a real result; everything else follows ``complex_cwt`` (continuous_transform.py:138-144)."""
    if _pywt is not None and type(wav) is _pywt.Wavelet:
        return False
    return bool(getattr(wav, "complex_cwt", False))


def sample_wavelet(wav: Any, precision: int) -> _Sampled:
    """``int_psi = cumsum(psi) * step`` over the wavelet's grid, conjugated where the reference conjugates it."""
    if isinstance(wav, torch.nn.Module):
        with torch.no_grad():
            approx = wav.wavefun(precision)
    else:
        approx = wav.wavefun(precision)
    if len(approx) == 2:
        psi, x = approx
    elif len(approx) == 3:
        _, psi, x = approx
    else:   # the reference unpacks (int_psi_d, int_psi_r, x) into two names here
        raise ValueError("too many values to unpack (expected 2)")
    if isinstance(psi, torch.Tensor) and psi.requires_grad and torch.is_grad_enabled():
        raise NotImplementedError("cwt computes gradients with respect to the data only; the wavelet's samples "
                                  "require grad. Call it under torch.no_grad().")
    psi, x = _as_numpy(psi), _as_numpy(x)
    step = x[1] - x[0]
    int_psi = np.cumsum(psi)
    int_psi *= step
    if _conjugates(wav):
        int_psi = np.conj(int_psi)
    return _Sampled(int_psi, psi, x, _complex_out(wav))


@functools.lru_cache(maxsize=64)
def _sample_named(name: str, precision: int) -> _Sampled:
    """Names resolve to immutable wavelets, so their samples are computed once per precision."""
    return sample_wavelet(as_continuous_wavelet(name), precision)


def central_frequency(psi: np.ndarray, x: np.ndarray) -> np.float64:
    """pywt's ``central_frequency``: the largest non-DC bin of ``|fft(psi)|``, folded to the lower half.  A numpy
    float64, as in pywt, so that dividing float32 scales by it gives float64 frequencies."""
    domain = float(x[-1] - x[0])
    index = np.argmax(np.abs(np.fft.fft(psi)[1:])) + 2
    if index > len(psi) / 2:
        index = len(psi) - index + 2
    return 1.0 / (domain / (index - 1))


# --------------------------------------------------------------------------------------
# per-scale filters
# --------------------------------------------------------------------------------------
def index_table(scale: Any, x: np.ndarray, n_psi: int, dtype: torch.dtype) -> torch.Tensor:
    """Indices into ``int_psi`` of the filter at ``scale``: the reference's expression, evaluated in the data's
    dtype (continuous_transform.py:104-111) on the CPU for data on any device.  (The reference evaluates it on the
    data's device, and CUDA divides a float32 tensor by a scalar as a multiplication by the reciprocal, which picks
    other taps at about a third of the scales; the CPU tables keep the result independent of where the data lives.)"""
    span, step = float(x[-1] - x[0]), float(x[1] - x[0])
    s = float(scale)
    j = torch.floor(torch.arange(s * span + 1, dtype=dtype) / (s * step)).type(torch.long)
    if j[-1] >= n_psi:
        j = torch.masked_select(j, j < n_psi)
    return j


def scale_filter(scale: Any, sampled: _Sampled, dtype: torch.dtype) -> tuple[np.ndarray, int]:
    """(g_s, f_s): the FIR taps ``-sqrt(s) (h[k] - h[k-1])``, k = 0..K, and the crop offset ``(K - 2) // 2``."""
    int_psi = torch.from_numpy(np.ascontiguousarray(sampled.int_psi))
    h = int_psi[index_table(scale, sampled.x, len(int_psi), dtype)].flip(0).numpy()
    K = len(h)
    if K < 2:   # the reference's coefficients would be shorter than the signal
        raise ValueError("Selected scale of {} too small.".format(scale))
    g = np.zeros(K + 1, dtype=h.dtype)
    g[:K] = h
    g[1:] -= h
    g *= -np.sqrt(scale)
    return g, (K - 2) // 2


def _scales_array(scales: Any) -> np.ndarray:
    if isinstance(scales, torch.Tensor):
        return scales.detach().cpu().numpy()
    if np.isscalar(scales):
        return np.array([scales])
    return np.asarray(scales)


class _Filters:
    """Every scale's (g_s, f_s) for one (wavelet samples, scales, data dtype)."""

    def __init__(self, sampled: _Sampled, scales: np.ndarray, dtype: torch.dtype):
        self.taps = [scale_filter(s, sampled, dtype) for s in scales.reshape(-1)]
        self.complex_out = sampled.complex_out
        self.kmax = max(len(g) for g, _ in self.taps)


def fft_log2(n: int, kmax: int) -> int:
    """FFT size F = 2H: the hop H is the power of two covering the shorter of the signal and the longest filter,
    clamped to 32..2048 (64 KB of complex128 per CTA at F = 4096)."""
    m = max(1, min(int(n), int(kmax)))
    return min(max((m - 1).bit_length(), MIN_HOP_LOG2), MAX_HOP_LOG2) + 1


def channel_layout(filters: _Filters, lg: int) -> tuple[np.ndarray, np.ndarray]:
    """(meta ``[channels, 6]`` int32, taps ``[parts, H]`` complex128) of include/wtb200.h for FFT size 2^lg.

    A channel's FIR is ``y[t] = sum_j c[j] x[t + D - j]`` with ``D = max(f_s + 1)`` over its scales, and scale s's
    taps g_s start at ``j = D - f_s - 1``; ``D = d H + e``.  A real-wavelet channel holds two consecutive scales as
    real and imaginary part."""
    H = 1 << (lg - 1)
    taps = filters.taps
    if filters.complex_out:
        groups = [[s] for s in range(len(taps))]
    else:
        groups = [list(range(s, min(s + 2, len(taps)))) for s in range(0, len(taps), 2)]
    meta = np.zeros((len(groups), _META), dtype=np.int32)
    rows = []
    part0 = 0
    for c, members in enumerate(groups):
        D = max(taps[s][1] + 1 for s in members)
        P = -(-max(D - taps[s][1] - 1 + len(taps[s][0]) for s in members) // H)
        row = np.zeros(P * H, dtype=np.complex128)
        for slot, s in enumerate(members):
            g, f = taps[s]
            seg = row[D - f - 1: D - f - 1 + len(g)]
            if filters.complex_out:
                seg += g
            elif slot == 0:
                seg.real += np.real(g)
            else:
                seg.imag += np.real(g)
        rows.append(row.reshape(P, H))
        meta[c] = (part0, P, D // H, members[0], members[1] if len(members) > 1 else -1, D % H)
        part0 += P
    return meta, np.concatenate(rows)


class _Plan:
    """Channels, their filter-part spectra on the device, and the twiddles, for one FFT size."""

    def __init__(self, filters: _Filters, lg: int, device: torch.device):
        meta, rows = channel_layout(filters, lg)
        self.lg, self.channels, self.scales = lg, len(meta), len(filters.taps)
        self.complex_out = filters.complex_out
        self.meta = torch.from_numpy(meta).to(device)
        self.twiddles = _twiddles(lg, device)
        parts = torch.from_numpy(rows).to(device)
        self.spectra = torch.empty((len(rows), 1 << lg), dtype=torch.complex128, device=device)
        rc = N.load().wt_cwt_filter_spectra(lg, len(rows), parts.data_ptr(), self.twiddles.data_ptr(),
                                            self.spectra.data_ptr(), torch.cuda.current_stream(device).cuda_stream)
        N.check(rc, "wt_cwt_filter_spectra")
        # once per cache miss: the plan may be used from any stream afterwards, and `parts` may be freed
        torch.cuda.current_stream(device).synchronize()


_TWIDDLES: dict = {}


def _twiddles(lg: int, device: torch.device) -> torch.Tensor:
    key = (lg, str(device))
    t = _TWIDDLES.get(key)
    if t is None:
        F = 1 << lg
        t = _TWIDDLES[key] = torch.from_numpy(np.exp(-2j * np.pi * np.arange(F // 2) / F)).to(device)
    return t


class _LRU(collections.OrderedDict):
    def get_or(self, key, make):
        if key in self:
            self.move_to_end(key)
            return self[key]
        value = self[key] = make()
        while len(self) > _CACHE_SIZE:
            self.popitem(last=False)
        return value


_FILTERS = _LRU()
_PLANS = _LRU()


def _plan(sampled: _Sampled, scales: np.ndarray, precision: int, dtype: torch.dtype, n: int,
          device: torch.device) -> _Plan:
    fkey = (sampled.key, scales.dtype.str, scales.tobytes(), int(precision), dtype)
    filters = _FILTERS.get_or(fkey, lambda: _Filters(sampled, scales, dtype))
    lg = fft_log2(n, filters.kmax)
    return _PLANS.get_or((fkey, lg, str(device)), lambda: _Plan(filters, lg, device))


# --------------------------------------------------------------------------------------
# launches
# --------------------------------------------------------------------------------------
def _workspace(plan: _Plan, batch: int, n: int, adjoint: bool, device) -> tuple:
    nbytes = int(N.load().wt_cwt_workspace_bytes(plan.lg, batch, n, plan.channels, int(adjoint)))
    return torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=device), nbytes


def run_forward(x: torch.Tensor, plan: _Plan) -> torch.Tensor:
    """wt_cwt_fwd on ``x [B, n]`` (CUDA, unit inner stride) -> ``[S, B, n]`` float64 or complex128."""
    batch, n = x.shape
    out = torch.empty((plan.scales, batch, n), dtype=torch.complex128 if plan.complex_out else torch.float64,
                      device=x.device)
    if batch == 0:
        return out
    ws, nbytes = _workspace(plan, batch, n, False, x.device)
    rc = N.load().wt_cwt_fwd(_dtype_code(x.dtype), plan.lg, plan.channels, plan.meta.data_ptr(),
                             plan.spectra.data_ptr(), plan.twiddles.data_ptr(), int(plan.complex_out), x.data_ptr(),
                             batch, n, x.stride(0), out.data_ptr(), batch * n, n, ws.data_ptr(), nbytes,
                             torch.cuda.current_stream(x.device).cuda_stream)
    N.check(rc, "wt_cwt_fwd")
    return out


def run_adjoint(gy: torch.Tensor, plan: _Plan, dtype: torch.dtype) -> torch.Tensor:
    """wt_cwt_adj: ``gy [S, B, n]`` -> ``[B, n]`` in ``dtype``."""
    _, batch, n = gy.shape
    gx = torch.empty((batch, n), dtype=dtype, device=gy.device)
    if batch == 0:
        return gx
    gy = gy.to(torch.complex128 if plan.complex_out else torch.float64).contiguous()
    ws, nbytes = _workspace(plan, batch, n, True, gy.device)
    rc = N.load().wt_cwt_adj(_dtype_code(dtype), plan.lg, plan.channels, plan.meta.data_ptr(), plan.spectra.data_ptr(),
                             plan.twiddles.data_ptr(), int(plan.complex_out), gy.data_ptr(), batch * n, n, batch, n,
                             gx.data_ptr(), n, ws.data_ptr(), nbytes, torch.cuda.current_stream(gy.device).cuda_stream)
    N.check(rc, "wt_cwt_adj")
    return gx


class _CwtFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan):
        ctx.plan, ctx.dtype = plan, x.dtype
        return run_forward(x.contiguous(), plan)

    @staticmethod
    def backward(ctx, gy):
        return _CwtAdjointFunction.apply(gy, ctx.plan, ctx.dtype), None


class _CwtAdjointFunction(torch.autograd.Function):
    """``gy -> Re(A^H gy)`` in the data's dtype.  Under torch's convention for complex gradients the adjoint of this
    real-linear map is ``u -> A u``: the forward transform again, in float64 or complex128 like ``gy``."""

    @staticmethod
    def forward(ctx, gy, plan, dtype):
        ctx.plan = plan
        return run_adjoint(gy, plan, dtype)

    @staticmethod
    def backward(ctx, u):
        return _CwtFunction.apply(u, ctx.plan), None, None


# --------------------------------------------------------------------------------------
# public API
# --------------------------------------------------------------------------------------
def cwt(
    data: torch.Tensor,
    scales: Union[np.ndarray, torch.Tensor],
    wavelet: Any,
    sampling_period: float = 1.0,
    precision: int = 12,
) -> tuple[torch.Tensor, np.ndarray]:
    """Continuous wavelet transform along the last axis -> (coefficients ``[S, *data.shape]``, frequencies)
    (reference continuous_transform.py:27-156)."""
    check_dtype(data)
    wav = as_continuous_wavelet(wavelet)
    scales = _scales_array(scales)
    _check_params_without_grad(wav)
    dev = _compute_device(data)
    if isinstance(wav, torch.nn.Module) and data.is_cuda:
        wav.to(data.device)   # the reference leaves its learnable wavelets on the data's device
    sampled = _sample_named(wavelet, int(precision)) if isinstance(wavelet, str) else sample_wavelet(wav, precision)
    n = int(data.shape[-1])
    lead = tuple(data.shape[:-1])
    if scales.size == 0:
        raise RuntimeError("stack expects a non-empty TensorList")
    x = data.reshape(-1, n)
    on_host = not data.is_cuda
    with torch.cuda.device(dev):
        plan = _plan(sampled, scales, precision, data.dtype, n, dev)
        if torch.is_grad_enabled() and data.requires_grad:
            out = _CwtFunction.apply(x.to(dev), plan)
            if on_host:
                out = out.cpu()
        else:
            xd = x.to(dev, non_blocking=True) if on_host else x
            if xd.stride(-1) != 1 and n != 1:
                xd = xd.contiguous()
            out = run_forward(xd, plan)
            if on_host:
                host = pinned_empty(out.shape, out.dtype)
                host.copy_(out, non_blocking=True)
                torch.cuda.current_stream(dev).synchronize()
                out = host
    frequencies = sampled.central_frequency / scales
    if np.isscalar(frequencies):
        frequencies = np.array([frequencies])
    frequencies /= sampling_period
    return out.reshape((plan.scales,) + lead + (n,)), frequencies
