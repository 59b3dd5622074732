"""Helpers for tests/test_gpu_launch_geometry.py: batches whose every item is checked against two oracle runs, and the
launch grids the profiler recorded.

Batches.  Item b of a batch is ``x_b = p_b * u + q_b * v``.  ``u`` and ``v`` are random multiples of 2^-8 in [-4, 4]
and the ``(p_b, q_b)`` are distinct primitive integer pairs with ``p_b > 0`` and ``q_b != 0``, so no two of them are
proportional.  Every transform here is linear, so the oracle runs on ``u`` and ``v`` once each and item b must equal
``p_b * C(u) + q_b * C(v)``.  An item that reads another item's input, or is written at another item's offset, gives
``p_c * C(u) + q_c * C(v)`` for some ``c != b`` and cannot pass.  ``|x_b| * 2^8`` stays below 2^24, so every ``x_b`` is
exact in float32 as well as in float64.

Grids.  ``kernel_launches`` reads a ``torch.profiler`` chrome trace: the name, grid, block and stream of every kernel,
in host launch order.
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass

import torch

from test_kernel_inventory import normalise

FRACTION_BITS = 8      # u, v are multiples of 2^-8
MAGNITUDE = 4          # ... in [-4, 4]
MANTISSA_BITS = 24     # float32 significand


def pairs(n: int) -> torch.Tensor:
    """[n, 2] int64: n distinct primitive (p, q) with p > 0 and q != 0, smallest max(|p|, |q|) first."""
    out: list[tuple[int, int]] = []
    r = 1
    while len(out) < n:
        # the ring max(|p|, |q|) == r: p == r with any q, or |q| == r with p < r
        ring = [(r, q) for q in range(-r, r + 1)] + [(p, s * r) for p in range(1, r) for s in (-1, 1)]
        out.extend((p, q) for p, q in ring if q != 0 and math.gcd(p, abs(q)) == 1)
        r += 1
    return torch.tensor(out[:n], dtype=torch.int64)


def bits_needed(pq: torch.Tensor) -> int:
    """Significand bits a combination p * u + q * v can need: integer part of (|p| + |q|) * 4 plus 8 fraction bits."""
    top = int((pq[:, 0].abs() + pq[:, 1].abs()).max()) * MAGNITUDE * (1 << FRACTION_BITS)
    return top.bit_length()


def quantised(shape, generator: torch.Generator) -> torch.Tensor:
    """float64 multiples of 2^-8 in [-4, 4]."""
    q = 1 << FRACTION_BITS
    n = torch.randint(-MAGNITUDE * q, MAGNITUDE * q + 1, tuple(shape), generator=generator, dtype=torch.int64)
    return n.to(torch.float64) / q


def combine(u: torch.Tensor, v: torch.Tensor, pq: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """[len(pq), *u.shape] in dtype on u's device: item b is p_b * u + q_b * v, exact in float32 and float64.

    ``u`` and ``v`` are already in ``dtype``: products and the sum are exact there (bits_needed < 24)."""
    assert bits_needed(pq) < MANTISSA_BITS, "the combination would not be exact in float32"
    shape = (-1,) + (1,) * u.dim()
    p = pq[:, 0].to(u.device, dtype).view(shape)
    q = pq[:, 1].to(u.device, dtype).view(shape)
    return p * u.unsqueeze(0) + q * v.unsqueeze(0)


def item_errors(got: list[torch.Tensor], cu: list[torch.Tensor], cv: list[torch.Tensor], pq: torch.Tensor):
    """(err, scale): per item, max |got_b - (p_b cu + q_b cv)| over every tensor of the tree, and
    |p_b| max|cu| + |q_b| max|cv| with the maxima taken over the whole tree.  got tensors are [B, ...], cu / cv are
    the oracle's float64 tensors without the batch dimension."""
    assert len(got) == len(cu) == len(cv), (len(got), len(cu), len(cv))
    dev = got[0].device
    p = pq[:, 0].to(dev, torch.float64)
    q = pq[:, 1].to(dev, torch.float64)
    su = max(float(t.abs().max()) for t in cu if t.numel())
    sv = max(float(t.abs().max()) for t in cv if t.numel())
    err = torch.zeros(len(pq), dtype=torch.float64, device=dev)
    for j, (g, a, b) in enumerate(zip(got, cu, cv)):
        assert tuple(g.shape) == (len(pq),) + tuple(a.shape), f"tensor {j}: shape {tuple(g.shape)}, oracle {tuple(a.shape)}"
        if not a.numel():
            continue
        shape = (-1,) + (1,) * a.dim()
        a, b = a.to(dev), b.to(dev)
        d = g.double() - (p.view(shape) * a + q.view(shape) * b)
        err = torch.maximum(err, d.abs().flatten(1).amax(1))
        del d
    return err.cpu(), (p.abs() * su + q.abs() * sv).cpu()


@dataclass(frozen=True)
class Launch:
    name: str             # normalised as in test_kernel_inventory: "fwd2d_strip_f32_kernel<8, 64, true>"
    grid: tuple           # (x, y, z)
    block: tuple
    stream: int | None
    ts: float
    correlation: int          # id of the host-side launch call: increases in host launch order


def kernel_launches(trace: dict) -> list[Launch]:
    """Every kernel of a chrome trace exported by torch.profiler, in host launch order (the correlation id of the
    launch call; kernels on different streams may start on the device in another order)."""
    out = []
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") != "kernel":
            continue
        args = ev.get("args", {})
        for key in ("grid", "correlation"):
            if key not in args:
                raise AssertionError(f"the profiler trace carries no {key} for kernel {ev.get('name')!r}: "
                                     f"args {sorted(args)}")
        out.append(Launch(normalise(ev["name"]), tuple(args["grid"]), tuple(args.get("block", ())), args.get("stream"),
                          float(ev.get("ts", 0.0)), int(args["correlation"])))
    out.sort(key=lambda k: k.correlation)
    return out


def load_trace(path) -> list[Launch]:
    with open(path) as f:
        return kernel_launches(json.load(f))


def coeff_len(n: int, L: int) -> int:
    """Coefficients along one axis for n samples and L taps in the non-periodic modes (ptwt's padding)."""
    padl = (2 * L - 3) // 2
    return (n + 2 * padl + n % 2 - L) // 2 + 1
