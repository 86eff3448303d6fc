"""Evaluation (metrics.py, csrc/gsb_metrics.cu) on the GPU.

  metrics   PSNR and SSIM of one 1920x1080 view: the kernel (one launch) beside the reference's float32 torch composition
            (metrics.cpp:40-116 restated in tests/metrics_restatement.py: five grouped conv2d, the element-wise maps and
            the .item() reads) on the same device and inputs.  Medians of K calls between CUDA events after warm-up;
            both results are compared in the same run.
  evaluate  MetricsEvaluator.evaluate over 8 views of the config-B scene (1 M Gaussians, 1920x1080, SH degree 3):
            wall-clock seconds per view, render included (what the reference reports as time_per_image), through the
            fastgs rasterizer (the reference's evaluation path) and through the from-world path (gut=True).

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing to the tree (the
evaluator's CSV goes to a temporary directory)."""
from __future__ import annotations

import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(q.splitlines()[0])
    except Exception:
        info["power_limit_w"] = None
    return info


def _time(fn, iters: int, warmup: int) -> float:
    ts = []
    for i in range(warmup + iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        if i >= warmup:
            ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def bench_metrics(M, iters: int, warmup: int, dev) -> dict:
    import metrics_restatement as R
    g = torch.Generator(device=dev).manual_seed(0)
    H, W = 1080, 1920
    image = torch.rand((3, H, W), device=dev, generator=g) * 1.4 - 0.2
    target = (0.7 * image.clamp(0, 1) + 0.3 * torch.rand((3, H, W), device=dev, generator=g)).contiguous()
    out = torch.empty(2, device=dev)
    kernel_ms = _time(lambda: M.image_metrics(image, target, out), iters, warmup)
    torch_ms = _time(lambda: R.metrics_torch(image, target), iters, warmup)
    mine = M.image_metrics(image, target).cpu().tolist()
    ref = R.metrics_torch(image, target)
    return {"size": [H, W], "kernel_ms": kernel_ms, "torch_composition_ms": torch_ms, "speedup": torch_ms / kernel_ms,
            "kernel": {"psnr": mine[0], "ssim": mine[1]}, "torch_composition": {"psnr": ref[0], "ssim": ref[1]},
            "abs_diff": {"psnr": abs(mine[0] - ref[0]), "ssim": abs(mine[1] - ref[1])}}


def bench_evaluate(pkg, M, repeats: int, dev) -> dict:
    import numpy as np

    import scenes
    sc = scenes.scene_b()
    t = {k: torch.from_numpy(v).to(dev) for k, v in sc.items() if isinstance(v, np.ndarray)}
    raw = pkg.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    g = torch.Generator(device=dev).manual_seed(1)
    P = {k: (v + 0.02 * torch.randn(v.shape, device=dev, generator=g)).contiguous() for k, v in raw.items()}
    res = {"scene": {"N": int(sc["means"].shape[0]), "width": sc["width"], "height": sc["height"],
                     "sh_degree": sc["sh_degree"], "views": 8}}
    with tempfile.TemporaryDirectory() as tmp:
        for name, gut in (("fastgs", False), ("gut", True)):
            ev = M.MetricsEvaluator(True, [1], os.path.join(tmp, name), gut=gut)
            views = []
            for v in range(8):
                V = torch.from_numpy(scenes.scene_b(N=1, view=v)["viewmats"][0]).to(dev)
                K = t["Ks"][0]
                img = ev.render(raw, 3, (V, K, sc["width"], sc["height"]), t["background"])
                img = img[0].permute(2, 0, 1) if gut else img
                views.append((V, K, sc["width"], sc["height"], img.clamp(0, 1).contiguous()))
            ev.evaluate(0, P, 3, views, t["background"])  # warm-up
            per_view = sorted(ev.evaluate(1, P, 3, views, t["background"]).elapsed_time for _ in range(repeats))
            r = ev.reporter.all_metrics[-1]
            res[name] = {"s_per_view_median": per_view[len(per_view) // 2], "psnr": r.psnr, "ssim": r.ssim}
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=200, help="timed kernel / composition calls")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5, help="timed evaluations per renderer")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.load_package()
    pkg.load()
    M = importlib.import_module(pkg.__name__ + ".metrics")
    dev = torch.device("cuda:0")
    out = {"card": _card(), "metrics": bench_metrics(M, args.iters, args.warmup, dev),
           "evaluate": bench_evaluate(pkg, M, args.repeats, dev)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
