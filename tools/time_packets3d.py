"""Time a full depth-3 WaveletPacket3D expansion and reconstruction against a node-by-node walk, on one GPU.

    python tools/time_packets3d.py [--reps 20]

Input: 8 x 128^3 float32, db2, mode "reflect", depth 3 (512 leaves).  Two ways on the same GPU:

* ``WaveletPacket3D``: one level-1 ``wavedec3`` call on the stacked parents per tree level (3 calls), and one
  ``waverec3`` call per level for ``reconstruct``;
* a node-by-node walk: one level-1 ``wavedec3`` call per node (1 + 8 + 64 = 73), and one ``waverec3`` call per node to
  rebuild the root, which is what a user without 3-D packets writes by hand.

Each time is the CUDA-event time from before the first call is enqueued until the last kernel ends, so host-side
cost that keeps the GPU waiting is included; median / min / max over ``--reps`` runs after one warm-up run.  The
first line names the card and its power limit; the last checks that both ways give the same nodes and root.
Writes nothing.
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
from pytorch_wavelet_toolbox_b200.packets import SUBBANDS_3D  # noqa: E402

SHAPE, WAVELET, MODE, DEPTH = (8, 128, 128, 128), "db2", "reflect", 3


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
    return {"median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3)}


def packet_expand(x: torch.Tensor) -> wt.WaveletPacket3D:
    wp = wt.WaveletPacket3D(x, WAVELET, mode=MODE, maxlevel=DEPTH)
    wp.initialize(wp.get_natural_order(DEPTH))
    return wp


def packet_reconstruct(wp: wt.WaveletPacket3D) -> torch.Tensor:
    return wp.reconstruct()[""]


def walk_expand(x: torch.Tensor) -> dict:
    tree = {"": x}
    for level in range(DEPTH):
        for key in wt.WaveletPacket3D.get_natural_order(level):
            a, det = wt.wavedec3(tree[key], WAVELET, mode=MODE, level=1)
            tree[key + "aaa"] = a
            tree.update({key + k: v for k, v in det.items()})
    return tree


def walk_reconstruct(tree: dict) -> torch.Tensor:
    tree = dict(tree)
    for level in reversed(range(DEPTH)):
        for key in wt.WaveletPacket3D.get_natural_order(level):
            r = wt.waverec3((tree[key + "aaa"], {k: tree[key + k] for k in SUBBANDS_3D[1:]}), WAVELET)
            if level > 0:
                r = r[(..., *(slice(0, n) for n in tree[key].shape[-3:]))]
            tree[key] = r
    return tree[""]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_packets3d.py needs a CUDA device")
    print(json.dumps(card()), flush=True)
    x = torch.randn(SHAPE, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    with torch.no_grad():
        wp = packet_expand(x)
        tree = walk_expand(x)
        # compared before timing: reconstruct overwrites the inner nodes of the packet tree with their reconstructions
        node_err = max(float((wp[k] - tree[k]).abs().max()) for k in tree)
        root_err = float((packet_reconstruct(wp) - walk_reconstruct(tree)).abs().max())
        # reconstruct reads only the leaves, so repeating it on one tree repeats the same work
        rows = {
            "WaveletPacket3D": {"expand": timed(lambda: packet_expand(x), args.reps),
                                "reconstruct": timed(lambda: packet_reconstruct(wp), args.reps)},
            "node_by_node": {"expand": timed(lambda: walk_expand(x), args.reps),
                             "reconstruct": timed(lambda: walk_reconstruct(tree), args.reps)},
        }
    for name, parts in rows.items():
        print(json.dumps({"way": name, "shape": list(SHAPE), "dtype": "float32", "wavelet": WAVELET, "mode": MODE,
                          "depth": DEPTH, **{k: stats(v) for k, v in parts.items()}}), flush=True)
    speedup = {k: round(statistics.median(rows["node_by_node"][k]) / statistics.median(rows["WaveletPacket3D"][k]), 2)
               for k in ("expand", "reconstruct")}
    print(json.dumps({"speedup_over_node_by_node": speedup, "nodes_compared": len(tree),
                      "max_abs_node_diff": node_err, "max_abs_root_diff": root_err,
                      "max_abs_input": float(x.abs().max())}), flush=True)


if __name__ == "__main__":
    main()
