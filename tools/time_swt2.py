"""Time swt2 and iswt2 on one GPU with CUDA events, alternating with the oracle port's torch path on the same GPU.

    python tools/time_swt2.py [--reps 20]

Each level runs as two one-axis passes on the 1-D stationary kernels (stationary.py), so a level moves 9 planes
(the pass along axes[1] reads 1 and writes 2, the pass along axes[0] reads 2 and writes 4) where a fused 2-D level
would move 5.  For each case it prints one JSON line: the median / min / max ms per call of swt2 and iswt2, the rate
over the algorithmic bytes (es H W (3J + 2) per image: the input read once and 3J + 1 bands written once, or the
reverse) and that rate as a share of the H100 SXM data-sheet 3.35 TB/s, the same for the design's own traffic
(es H W (9J) per image), the port's (cuDNN, TF32 off) median ms, and the max error of the timed outputs against the
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
from oracle import swt2_port as P  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# (batch, H, W, dtype, wavelet, level)
CASES = [
    (16, 1024, 1024, torch.float32, "db4", 4),
    (64, 256, 256, torch.float32, "haar", 6),
    (4, 2048, 2048, torch.float64, "sym4", 3),
]


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (out[0].split(", ") + ["?", "?", "?"])[:3] if out else ("?", "?", "?")
    return {"card": name, "power_limit": power, "max_sm_clock": clock, "torch_name": torch.cuda.get_device_name()}


def time_once(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def stats(ms: list[float]) -> dict:
    return {"median_ms": round(statistics.median(ms), 4), "min_ms": round(min(ms), 4), "max_ms": round(max(ms), 4)}


def flat(coeffs) -> list[torch.Tensor]:
    out = [coeffs[0]]
    for el in coeffs[1:]:
        out.extend(el)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_swt2.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False    # the port's float32 convolutions in float32, like the kernels
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(card()))
    for batch, H, W, dtype, wavelet, level in CASES:
        x = torch.randn(batch, H, W, device="cuda", dtype=dtype, generator=torch.Generator("cuda").manual_seed(1))
        es = x.element_size()
        alg = es * H * W * (3 * level + 2) * batch
        own = es * H * W * 9 * level * batch
        with torch.no_grad():
            c = wt.swt2(x, wavelet, level)
            c_port = P.swt2(x, wavelet, level)
            fns = {"swt2": lambda: wt.swt2(x, wavelet, level), "iswt2": lambda: wt.iswt2(c, wavelet),
                   "port_swt2": lambda: P.swt2(x, wavelet, level), "port_iswt2": lambda: P.iswt2(c_port, wavelet)}
            for fn in fns.values():
                fn()
            torch.cuda.synchronize()
            ms: dict = {k: [] for k in fns}
            for r in range(args.reps):            # alternate the four calls so that drift hits all of them alike
                for k, fn in fns.items():
                    if k.startswith("port") and r % 4:
                        continue
                    ms[k].append(time_once(fn))
            c = wt.swt2(x, wavelet, level)
            y, y_port = wt.iswt2(c, wavelet), P.iswt2(c_port, wavelet)
            scale = max(float(t.abs().max()) for t in flat(c_port))
            err_fwd = max(float((a - b).abs().max()) for a, b in zip(flat(c), flat(c_port))) / scale
            err_inv = float((y - y_port).abs().max()) / float(y_port.abs().max())
        row = {"batch": batch, "H": H, "W": W, "dtype": str(dtype).replace("torch.", ""), "wavelet": wavelet,
               "level": level, "algorithmic_bytes": alg, "design_bytes": own}
        for name in ("swt2", "iswt2"):
            med = statistics.median(ms[name])
            port = statistics.median(ms["port_" + name])
            row[name] = dict(stats(ms[name]), GB_per_s=round(alg / med / 1e6, 1),
                             share_of_3_35_TBps=round(alg / med / 1e-3 / HBM_BYTES_PER_S, 3),
                             design_GB_per_s=round(own / med / 1e6, 1),
                             design_share_of_3_35_TBps=round(own / med / 1e-3 / HBM_BYTES_PER_S, 3),
                             port_median_ms=round(port, 3), speedup_vs_port=round(port / med, 2))
        row["swt2"]["max_rel_err_vs_port"] = err_fwd
        row["iswt2"]["max_rel_err_vs_port"] = err_inv
        print(json.dumps(row), flush=True)
        del x, c, c_port, y, y_port
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
