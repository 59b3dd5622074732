"""Time the 2-D analysis with each way of running two levels per launch, on one GPU, with CUDA events.

    python tools/time_fwd2d_pairs.py [--reps 20]

Variants (knobs of csrc/knobs.cuh, set through the C ABI in this process; the order alternates per repetition):
  default      -- levels 1-2 by fwd2d_wpair_kernel for images of >= 2^24 samples, one strip-kernel launch per level
                  otherwise
  wpair_fuse2  -- FUSE2=1: as the default, every other level pair by fwd2d_fuse2_f32_kernel
  fuse2        -- WPAIR=0 FUSE2=1: every level pair by fwd2d_fuse2_f32_kernel
  per_level    -- WPAIR=0: one strip-kernel launch per level
  *_one_chunk  -- the same with CHUNK=batch (no split of the batch over two streams)

For each case it prints one JSON line: the median / min / max ms per call of every variant and, for level 2, the
rate over the call's algorithmic bytes (input read once, level-1 details and level-2 bands written once).
Needs a CUDA device; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pytorch_wavelet_toolbox_b200 as wt  # noqa: E402
from pytorch_wavelet_toolbox_b200 import _native  # noqa: E402

VARIANTS = {
    "default": {},
    "wpair_fuse2": {"FUSE2": 1},
    "fuse2": {"WPAIR": 0, "FUSE2": 1},
    "per_level": {"WPAIR": 0},
}
# (batch, side, wavelet, level, with one-chunk variants)
CASES = [
    (64, 4096, "db4", 2, True),
    (64, 4096, "db4", 4, True),
    (8, 4096, "db4", 4, False),
    (1, 4096, "db4", 4, False),
    (1024, 128, "db4", 3, False),
    (256, 256, "db4", 3, False),
    (64, 512, "db4", 3, False),
    (16, 1024, "db4", 3, False),
    (4, 2048, "db4", 3, False),
    (16, 2048, "db8", 5, False),   # not covered by either kernel: a control
]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    for batch, n, wav, level, chunk_variants in CASES:
        x = torch.randn(batch, n, n, device="cuda")
        variants = dict(VARIANTS)
        if chunk_variants:
            variants.update({k + "_one_chunk": dict(v, CHUNK=batch) for k, v in VARIANTS.items()})
        times = {k: [] for k in variants}
        for name, kn in variants.items():   # warm-up: module load, dynamic shared memory opt-in, allocator
            with _native.knobs(**kn):
                for _ in range(3):
                    wt.wavedec2(x, wav, mode="reflect", level=level)
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for name, kn in variants.items():
                with _native.knobs(**kn):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    wt.wavedec2(x, wav, mode="reflect", level=level)
                    b.record()
                    b.synchronize()
                    times[name].append(a.elapsed_time(b))
        res = {"case": f"{batch}x{n}^2 {wav} L{level}"}
        L = 8 if wav == "db4" else 16
        m1 = (n + L - 1) // 2
        m2 = (m1 + L - 1) // 2
        for name, ts in times.items():
            ts.sort()
            r = {"ms_median": round(ts[len(ts) // 2], 4), "ms_min": round(ts[0], 4), "ms_max": round(ts[-1], 4)}
            if level == 2:
                alg = 4 * batch * (n * n + 3 * m1 * m1 + 4 * m2 * m2)
                r["alg_TB_per_s"] = round(alg / (r["ms_median"] * 1e-3) / 1e12, 3)
            res[name] = r
        print(json.dumps(res), flush=True)
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
