"""Model set-up on the GPU: the exact mean neighbour distance (csrc/gsb_knn.cu), the initial scale of
init_model_from_pointcloud, at 100 k (the random initialisation's default), 1 M and 6 M points on uniform, SfM-like
(surfaces of very different density) and outlier-laden clouds (tests/knn_restatement.py builds all three).

Each call is timed between CUDA events, the operator's host work and its one status read-back included, after warm-up;
the script reports the median, p10 and p90.  Where oracle/_ref holds the reference's nanoflann harness
(oracle/build_ref_knn.py), the reference's own search (tree build and queries, OpenMP over the host's cores) is timed
on the same clouds with a host clock, and the host's core count is reported with it.

Prints one JSON line per case and a last one with the card's name and power limit, read in the same run.  Writes
nothing to the tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
        p, c = q.splitlines()[0].split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(p), float(c)
    except Exception:
        info["power_limit_w"] = None
    return info


def _stats(ts) -> dict:
    ts = np.sort(np.asarray(ts))
    return {"median_ms": float(np.median(ts)), "p10_ms": float(np.percentile(ts, 10)),
            "p90_ms": float(np.percentile(ts, 90)), "n": len(ts)}


def _gpu_times(fn, iters: int, warmup: int) -> list:
    ts = []
    for i in range(warmup + iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        if i >= warmup:
            ts.append(a.elapsed_time(b))
    return ts


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sizes", default="100000,1000000,6000000")
    ap.add_argument("--shapes", default="uniform,sfm,outliers")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-max", type=int, default=6_000_000, help="largest cloud the reference's search is timed on")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_init.py needs a CUDA device")
    import __graft_entry__ as ge
    import knn_restatement as kr
    from oracle import build_ref_knn

    pkg = ge.load_package()
    pkg.load()
    ops = torch.ops.gsplat_b200
    ref = build_ref_knn.load()
    dev = torch.device("cuda:0")
    for n in [int(s) for s in a.sizes.split(",")]:
        for shape in a.shapes.split(","):
            pts_np = kr.CLOUDS[shape](n, seed=1)
            pts = torch.from_numpy(pts_np).to(dev)
            out = ops.mean_neighbor_distances(pts)
            row = {"case": f"{shape}_{n}", "points": n,
                   "kernel": _stats(_gpu_times(lambda: ops.mean_neighbor_distances(pts), a.iters, a.warmup))}
            if ref is not None and n <= a.ref_max:
                reps = 3 if n <= 1_000_000 else 1
                ts, r = [], None
                for _ in range(reps):
                    t0 = time.perf_counter()
                    r = build_ref_knn.mean_dist(ref, pts_np)
                    ts.append(1e3 * (time.perf_counter() - t0))
                g = out.cpu().numpy()
                row["reference_host"] = dict(_stats(ts), nproc=os.cpu_count())
                row["exact_le_reference"] = bool((g <= r).all())
                row["differs_from_reference_frac"] = float((g != r).mean())
            else:
                row["reference_host"] = "not measured (harness not built)" if ref is None else "not measured"
            print(json.dumps(row), flush=True)
    print(json.dumps({"card": _card()}), flush=True)


if __name__ == "__main__":
    main()
