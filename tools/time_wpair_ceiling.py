"""How close the levels-1-2 wavedec2 launch (fwd2d_wpair_kernel) comes to what the card can stream, on one GPU.

    python tools/time_wpair_ceiling.py [--batch 64] [--side 4096] [--reps 10]

In one process, alternating per repetition, CUDA events around each call (db4, reflect, float32 [batch, side, side]):
  copy            -- torch copy_ of the input into a tensor of the same size: the copy ceiling (read + write bytes)
  twin_s2_c12 ... -- the traffic twin of fwd2d_wpair_kernel<8, S, *> (tools/wpair_twin): same grid, segments,
                     one-warp CTAs, TMA boxes, ring, mbarriers and stores, no filtering; at most C CTAs per SM
                     (c0: as many as its shared memory allows); one launch over the whole batch; _stcs: streaming
                     stores, _ldef: evict-first input boxes, _lockN: N adjacent strips as warps of one CTA kept in
                     step by a named barrier after every group; _clN: one-warp CTAs launched as clusters of N
                     adjacent strips kept in step by the kernel's split cluster barrier, _clN_join: the same barrier
                     with the wait right after the arrive
  kernel_cC_clN   -- the real fwd2d_wpair_kernel<8, 2, 12> launched from the twin's object at the twin's settings:
                     at most C CTAs per SM, clusters of N strips, one launch over the whole batch; _s3: <8, 3, 12>,
                     _m15: <8, 2, 15>
  wpair_l2_segN   -- levels 1-2 with segments of N level-2 rows (WPAIR_SEG)
  wpair_l2        -- wavedec2(level=2) as the library runs it (levels 1-2 in one launch per half batch)
  wpair_l2_one    -- the same with CHUNK=batch (one launch over the whole batch, like the twin)
  per_level_l2    -- WPAIR=0: one strip-kernel launch per level
  wpair_l4, per_level_l4 -- the full level-4 transform, by default and with WPAIR=0

Every rate is given over two byte counts computed from the shapes: `alg` = input read once and every band written
once; `dram` = `alg` plus the approximation bands that one launch per level writes and reads back.  The TMA boxes'
re-read halo columns (10 % of the input at db4) are in neither: most of them hit L2.
Prints one JSON line per variant and one with the card.  Needs a CUDA device; writes nothing.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import subprocess
import sys
from itertools import product
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import pytorch_wavelet_toolbox_b200 as wt  # noqa: E402
from pytorch_wavelet_toolbox_b200 import _native, fwt  # noqa: E402
from pytorch_wavelet_toolbox_b200._wavelets import as_wavelet, filter_bank  # noqa: E402
from pytorch_wavelet_toolbox_b200.csrc.build import TWIN  # noqa: E402

L = 8   # db4


def coeff_len(n: int) -> int:
    return (n + L - 1) // 2


def level_bytes(batch: int, side: int, level: int, fused_pairs: bool) -> tuple[int, int]:
    """(alg, dram) bytes of a `level`-level float32 transform; fused_pairs: levels 1-2 keep cA1 on chip."""
    n, alg, inter = side, batch * side * side, 0
    for lv in range(1, level + 1):
        m = coeff_len(n)
        alg += batch * (3 if lv < level else 4) * m * m
        if lv < level and not (fused_pairs and lv == 1):
            inter += 2 * batch * m * m   # cA_lv written by one launch, read by the next
        n = m
    return 4 * alg, 4 * (alg + inter)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--side", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)

    B, n = args.batch, args.side
    x = torch.randn(B, n, n, device="cuda")
    y = torch.empty_like(x)
    wav = "db4"

    twin = ctypes.CDLL(str(TWIN))
    twin.wpair_twin_fwd.restype = ctypes.c_int
    twin.wpair_twin_fwd.argtypes = [ctypes.c_int] * 6 + [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                                         ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int,
                                                         ctypes.c_void_p]
    twin.wpair_kernel_fwd.restype = ctypes.c_int
    twin.wpair_kernel_fwd.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                                           ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int,
                                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    dec_lo, dec_hi, _, _ = filter_bank(as_wavelet(wav))
    taps_lo, taps_hi = (ctypes.c_double * L)(*dec_lo), (ctypes.c_double * L)(*dec_hi)
    plan = fwt._make_plan((n, n), L, 2, 4)
    buf = torch.empty((B, plan.item_elems), device="cuda")
    scratch = torch.empty((B, max(sum(lv.plane for lv in plan.levels[:-1]), 1)), device="cuda")
    lv = fwt._fill_levels(plan, buf, scratch)

    def run_twin(nstg: int, ctas: int, hint: int = 0, wpc: int = 1, cluster: int = 1, csync: int = 0):
        rc = twin.wpair_twin_fwd(nstg, ctas, hint, wpc, cluster, csync, x.data_ptr(), B, n, n, x.stride(0), x.stride(1),
                                 ctypes.addressof(lv), _native.MODES["reflect"], torch.cuda.current_stream().cuda_stream)
        if rc != 0:
            raise RuntimeError(f"wpair_twin_fwd returned {rc}")

    def run_kernel(ctas: int, cluster: int, var: int = 0):
        rc = twin.wpair_kernel_fwd(var, ctas, cluster, x.data_ptr(), B, n, n, x.stride(0), x.stride(1), ctypes.addressof(lv),
                                   _native.MODES["reflect"], taps_lo, taps_hi, torch.cuda.current_stream().cuda_stream)
        if rc != 0:
            raise RuntimeError(f"wpair_kernel_fwd returned {rc}")

    def call(level: int, **kn):
        def f():
            with _native.knobs(**kn):
                wt.wavedec2(x, wav, mode="reflect", level=level)
        return f

    l2f, l2p, l4f, l4p = (level_bytes(B, n, 2, True), level_bytes(B, n, 2, False), level_bytes(B, n, 4, True),
                          level_bytes(B, n, 4, False))
    copy_bytes = 2 * x.numel() * 4
    variants = {
        "copy": (lambda: y.copy_(x), (copy_bytes, copy_bytes)),
        "twin_s2_c12": (lambda: run_twin(2, 12), l2f),
        "twin_s2_c0": (lambda: run_twin(2, 0), l2f),
        "twin_s3_c12": (lambda: run_twin(3, 12), l2f),
        "twin_s2_c8": (lambda: run_twin(2, 8), l2f),
        "twin_s2_c10": (lambda: run_twin(2, 10), l2f),
        "twin_s2_c12_stcs": (lambda: run_twin(2, 12, 1), l2f),
        "twin_s2_c12_ldef": (lambda: run_twin(2, 12, 2), l2f),
        "twin_s2_c12_both": (lambda: run_twin(2, 12, 3), l2f),
        "twin_s2_c12_lock2": (lambda: run_twin(2, 12, 0, 2), l2f),
        "twin_s2_c12_lock3": (lambda: run_twin(2, 12, 0, 3), l2f),
        "twin_s2_c12_lock6": (lambda: run_twin(2, 12, 0, 6), l2f),
    }
    # the kernel's lockstep scheme on the twin, and the kernel itself, at the same cluster sizes and CTAs per SM
    # (18 strips per 4096^2 image: 9 is the largest divisor within the limit of 16 CTAs per cluster, a non-portable size)
    for ctas, cl in product((12, 8), (1, 2, 3, 6, 9)):
        if ctas != 12 and cl not in (6, 9):
            continue
        variants[f"twin_s2_c{ctas}_cl{cl}"] = (lambda c=ctas, k=cl: run_twin(2, c, 0, 1, k, 1), l2f)
        if cl in (3, 6, 9):
            variants[f"twin_s2_c{ctas}_cl{cl}_join"] = (lambda c=ctas, k=cl: run_twin(2, c, 0, 1, k, 2), l2f)
        variants[f"kernel_c{ctas}_cl{cl}"] = (lambda c=ctas, k=cl: run_kernel(c, k), l2f)
    for cl in (2, 3, 6, 9):   # the other db4 instantiations: a 3-stage ring; 15 CTAs per SM
        variants[f"kernel_s3_c12_cl{cl}"] = (lambda k=cl: run_kernel(12, k, 3), l2f)
        variants[f"kernel_m15_c0_cl{cl}"] = (lambda k=cl: run_kernel(0, k, 1), l2f)
    variants |= {
        "wpair_l2": (call(2), l2f),
        "wpair_l2_one": (call(2, CHUNK=B), l2f),
        "wpair_l2_seg48": (call(2, WPAIR_SEG=48), l2f),
        "wpair_l2_seg96": (call(2, WPAIR_SEG=96), l2f),
        "wpair_l2_seg288": (call(2, WPAIR_SEG=288), l2f),
        "per_level_l2": (call(2, WPAIR=0), l2p),
        "wpair_l4": (call(4), l4f),
        "per_level_l4": (call(4, WPAIR=0), l4p),
    }
    for name in list(variants):   # warm-up: module load, shared-memory opt-in, allocator
        try:
            for _ in range(3):
                variants[name][0]()
        except RuntimeError as e:   # a launch configuration this card does not take (e.g. a cluster size)
            print(json.dumps({"variant": name, "error": str(e)}), flush=True)
            del variants[name]
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.reps):
        for name, (f, _) in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    for name, (_, (alg, dram)) in variants.items():
        ts = sorted(times[name])
        med = ts[len(ts) // 2]
        print(json.dumps({"variant": name, "ms_median": round(med, 4), "ms_min": round(ts[0], 4),
                          "ms_max": round(ts[-1], 4), "alg_GB": round(alg / 1e9, 3), "dram_GB": round(dram / 1e9, 3),
                          "alg_TB_per_s": round(alg / (med * 1e-3) / 1e12, 3),
                          "dram_TB_per_s": round(dram / (med * 1e-3) / 1e12, 3)}), flush=True)


if __name__ == "__main__":
    main()
