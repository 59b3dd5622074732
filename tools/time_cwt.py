"""Time cwt on one GPU with CUDA events, against the oracle port (the reference's per-scale FFT algorithm) on the
same GPU.

    python tools/time_cwt.py [--reps 20]

Workloads: the reference's own benchmark (examples/speed_tests/timeitcwt_1d.py: 32 x 10^4 float32, shan0.1-0.4,
scales 1..30, sampling_period 4 pi / 800), a float32 scalogram with a real wavelet (morl, 128 scales: pairs of scales
share an inverse FFT), and long float64 signals with a complex wavelet over 64 geometric scales up to 2^10 (filters of
up to ~16 k taps, several filter parts per scale).  For each it prints one JSON line: the median / min / max ms per
call of cwt (filter spectra cached, as in steady use) and of the port, the rate over the algorithmic bytes (the input
read once, S * n * (8 | 16) bytes written once) and that rate as a share of the H100 SXM data-sheet 3.35 TB/s, and
the max error of the timed outputs against the port relative to max |coefficient|.  The first line names the card,
its power limit and max SM clock.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pytorch_wavelet_toolbox_b200 as wt  # noqa: E402
from oracle import cwt_port as P  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# (label, batch, n, dtype, wavelet, scales, sampling_period)
CASES = [
    ("reference_benchmark", 32, 10_000, torch.float32, "shan0.1-0.4", np.arange(1, 31), 4 * np.pi / 800),
    ("morl_128_scales", 64, 16384, torch.float32, "morl", np.arange(1, 129), 1.0),
    ("cmor_geometric_long", 8, 1 << 18, torch.float64, "cmor1.5-1.0", np.geomspace(1, 1024, 64), 1.0),
]


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (out[0].split(", ") + ["?", "?", "?"])[:3] if out else ("?", "?", "?")
    return {"card": name, "power_limit": power, "max_sm_clock": clock, "torch_name": torch.cuda.get_device_name()}


def timed(fn, reps: int) -> list[float]:
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def stats(ms: list[float]) -> dict:
    return {"median_ms": round(statistics.median(ms), 4), "min_ms": round(min(ms), 4), "max_ms": round(max(ms), 4)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_cwt.py needs a CUDA device")
    print(json.dumps(card()), flush=True)
    for label, batch, n, dtype, wavelet, scales, period in CASES:
        x = torch.randn(batch, n, device="cuda", dtype=dtype, generator=torch.Generator("cuda").manual_seed(1))
        with torch.no_grad():
            got, _ = wt.cwt(x, scales, wavelet, sampling_period=period)
            ms = timed(lambda: wt.cwt(x, scales, wavelet, sampling_period=period), args.reps)
            want, _ = P.cwt(x, scales, wavelet, sampling_period=period)
            port = timed(lambda: P.cwt(x, scales, wavelet, sampling_period=period), max(3, args.reps // 4))
            err = float((got - want).abs().max()) / float(want.abs().max())
        nbytes = x.numel() * x.element_size() + got.numel() * got.element_size()
        med = statistics.median(ms)
        row = {"workload": label, "batch": batch, "n": n, "dtype": str(dtype).replace("torch.", ""),
               "wavelet": wavelet, "scales": len(scales), "out_dtype": str(got.dtype).replace("torch.", ""),
               "algorithmic_bytes": nbytes, "cwt": stats(ms), "GB_per_s": round(nbytes / med / 1e6, 1),
               "share_of_3_35_TBps": round(nbytes / med / 1e-3 / HBM_BYTES_PER_S, 3), "port": stats(port),
               "speedup_vs_port": round(statistics.median(port) / med, 2), "max_rel_err_vs_port": err}
        print(json.dumps(row), flush=True)
        del x, got, want
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
