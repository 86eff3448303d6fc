"""Bilateral-grid benchmark (SURVEY.md 8 f5): kernel times at 1920x1080 with a 16x16x8 grid and 200 images -- this
library's and, where oracle/build_ref_bilagrid.py built them into oracle/_ref, the reference's own kernels in the same
run -- and the graphed config-B training iteration (1 M Gaussians, 1920x1080) with and without the grid on both
rasterizer paths.

  python bench_bilateral_grid.py [--iters K] [--images N]

Prints one JSON line.  Kernel times are the median of K launches timed with CUDA events; iteration times are the
median over K graph replays.  Writes nothing to the tree."""
from __future__ import annotations

import argparse
import importlib
import json
import os
import subprocess
import sys

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


def _time(fn, iters: int) -> float:
    ts = []
    for _ in range(3):
        fn()
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def kernels(iters: int, n_images: int) -> dict:
    ns = torch.ops.gsplat_b200
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    H, W = 1080, 1920
    grids = torch.randn((n_images, 12, 8, 16, 16), device=dev, generator=g) * 0.1
    grids[:, 0] += 1.0
    grids[:, 5] += 1.0
    grids[:, 10] += 1.0
    img = torch.rand((H, W, 3), device=dev, generator=g) * 1.2 - 0.1
    v_out = torch.randn((H, W, 3), device=dev, generator=g)
    idx = torch.tensor([n_images // 2], dtype=torch.int32, device=dev)
    v_grids = torch.zeros_like(grids)
    w = torch.ones(1, device=dev)
    res = {"this_library": {
        "slice_fwd_ms": _time(lambda: ns.bilagrid_slice(grids, img, idx, False), iters),
        "slice_bwd_ms": _time(lambda: ns.bilagrid_slice_backward(grids, img, idx, v_out, v_grids, False), iters),
        "tv_loss_and_grad_ms": _time(lambda: ns.bilagrid_tv(grids, w, True), iters),
    }}
    so = os.path.join(ROOT, "oracle", "_ref", "libbilagrid_ref.so")
    if os.path.exists(so):
        # the reference's kernels as its BilateralGrid component drives them: one image's grid, the clamped image
        torch.ops.load_library(so)
        ref = torch.ops.bilagrid_ref
        g1, x = grids[n_images // 2].contiguous(), img.clamp(0, 1).contiguous()
        w0 = torch.ones((), device=dev)
        res["reference"] = {
            "slice_fwd_ms": _time(lambda: ref.slice_forward(g1, x), iters),
            "slice_bwd_ms": _time(lambda: ref.slice_backward(g1, x, v_out), iters),
            # forward and backward are two launches there (and the backward reads its weight with .item())
            "tv_loss_and_grad_ms": _time(lambda: (ref.tv_forward(grids), ref.tv_backward(grids, w0)), iters),
        }
        res["slice_bwd_speedup"] = res["reference"]["slice_bwd_ms"] / res["this_library"]["slice_bwd_ms"]
    else:
        res["reference"] = None
    return res


def iterations(iters: int, n_images: int) -> dict:
    import __graft_entry__ as ge
    import scenes
    from parity import to_dev

    pkg = ge.load_package()
    pkg.load()
    training = importlib.import_module(pkg.__name__ + ".training")
    bil = importlib.import_module(pkg.__name__ + ".bilateral")
    fg = importlib.import_module(pkg.__name__ + ".fastgs")
    dev = torch.device("cuda:0")
    sc = scenes.scene_b()
    t = to_dev(sc, dev)
    raw = pkg.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    g = torch.Generator(device=dev).manual_seed(1)
    target = torch.rand((3, 1080, 1920), device=dev, generator=g)
    res = {}

    def run(make, call):
        step = make()
        call(step, 0)
        k = [0]

        def one():
            k[0] += 1
            call(step, k[0] % n_images)
        return _time(one, iters)

    for grid in (False, True):
        P = {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}
        bg = bil.BilateralGrid(n_images, device=dev) if grid else None
        res[f"gsplat_graphed_{'grid' if grid else 'nogrid'}_ms"] = run(
            lambda: training.GraphedTrainStep(P, 3, 1920, 1080, bilateral_grid=bg),
            lambda s, i: s(t["viewmats"], t["Ks"], target, t["background"], **({"image_idx": i} if grid else {})))
        del P
    inp = scenes.fastgs_inputs(sc)
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw", "opacity_raw": "opacities_raw",
             "sh0": "sh0", "shN": "shN"}
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(dev), active_sh_bases=inp["active_sh_bases"],
                          width=inp["width"], height=inp["height"], focal_x=inp["fx"], focal_y=inp["fy"], center_x=inp["cx"],
                          center_y=inp["cy"], near_plane=inp["near_plane"], far_plane=inp["far_plane"])
    w2c = torch.from_numpy(inp["w2c"]).to(dev)
    bgc = torch.tensor([0.3, 0.2, 0.1], device=dev)
    for grid in (False, True):
        P = {k: torch.from_numpy(inp[v]).to(dev).requires_grad_(True) for k, v in names.items()}
        bg = bil.BilateralGrid(n_images, device=dev) if grid else None
        res[f"fastgs_graphed_{'grid' if grid else 'nogrid'}_ms"] = run(
            lambda: training.GraphedFastGsTrainStep(P, 3, s, bilateral_grid=bg),
            lambda st, i: st(w2c, s.cam_position, target, bgc, **({"image_idx": i} if grid else {})))
        del P
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--images", type=int, default=200)
    ap.add_argument("--skip-iterations", action="store_true")
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.load_package().load()
    out = {"card": _card(), "image": "1920x1080", "grid": "16x16x8", "images": args.images}
    out["kernels"] = kernels(args.iters, args.images)
    if not args.skip_iterations:
        out["iteration_config_b"] = iterations(args.iters, args.images)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
