"""Time swt and iswt on one GPU with CUDA events, against the oracle port's torch path on the same GPU.

    python tools/time_swt.py [--reps 20]

Cases are shapes a user of the stationary transform runs: long float32 signals, a float32 image's worth of rows,
and float64 rows at the default (maximal) level.  For each case it prints one JSON line: the median / min / max ms
per call of swt and iswt, the rate over the algorithmic bytes (es * n * (J + 2) per signal: the input read once and
J + 1 bands written once, or the reverse) and that rate as a share of the H100 SXM data-sheet 3.35 TB/s, the
port's (the reference algorithm's) median ms on the same GPU, and the max error of the timed outputs against the
port, relative to max |coefficient|.  The first line names the card and its power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pytorch_wavelet_toolbox_b200 as wt  # noqa: E402
from oracle import swt_port as P  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# (batch, n, dtype, wavelet, level)
CASES = [
    (64, 1 << 20, torch.float32, "db4", 8),
    (4096, 4096, torch.float32, "db8", 6),
    (256, 65536, torch.float64, "haar", None),
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
        raise SystemExit("time_swt.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False    # the port's float32 convolutions in float32, like the kernels
    print(json.dumps(card()))
    for batch, n, dtype, wavelet, level in CASES:
        x = torch.randn(batch, n, device="cuda", dtype=dtype, generator=torch.Generator("cuda").manual_seed(1))
        J = level if level is not None else wt._wavelets.swt_max_level(n)
        nbytes = x.element_size() * n * (J + 2) * batch
        with torch.no_grad():
            c = wt.swt(x, wavelet, level)
            fwd = timed(lambda: wt.swt(x, wavelet, level), args.reps)
            inv = timed(lambda: wt.iswt(c, wavelet), args.reps)
            c_port = P.swt(x, wavelet, level)
            port_fwd = timed(lambda: P.swt(x, wavelet, level), max(3, args.reps // 4))
            port_inv = timed(lambda: P.iswt(c_port, wavelet), max(3, args.reps // 4))
            y, y_port = wt.iswt(c, wavelet), P.iswt(c_port, wavelet)
            scale = max(float(t.abs().max()) for t in c_port)
            err_fwd = max(float((a - b).abs().max()) for a, b in zip(c, c_port)) / scale
            err_inv = float((y - y_port).abs().max()) / float(y_port.abs().max())
        row = {"batch": batch, "n": n, "dtype": str(dtype).replace("torch.", ""), "wavelet": wavelet, "level": J,
               "algorithmic_bytes": nbytes}
        for name, ms, port in (("swt", fwd, port_fwd), ("iswt", inv, port_inv)):
            med = statistics.median(ms)
            row[name] = dict(stats(ms), GB_per_s=round(nbytes / med / 1e6, 1),
                             share_of_3_35_TBps=round(nbytes / med / 1e-3 / HBM_BYTES_PER_S, 3),
                             port_median_ms=round(statistics.median(port), 3),
                             speedup_vs_port=round(statistics.median(port) / med, 2))
        row["swt"]["max_rel_err_vs_port"] = err_fwd
        row["iswt"]["max_rel_err_vs_port"] = err_inv
        print(json.dumps(row), flush=True)
        del x, c, c_port, y, y_port
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
