"""Time the five render modes (RGB, D, ED, RGB_D, RGB_ED) at config B -- 1 M Gaussians, 1920x1080, SH degree 3 --
on the operator path (rasterize(): the gsplat:: operators + autograd) and on the fused path (rasterize_fused()),
forward alone and forward + backward.

    python bench_render_modes.py [--gaussians N] [--iters K] [--warmup W]

One call is timed by CUDA events around it (the backward included for "fwd+bwd"); each row gives the median, p10
and p90 over K calls after W warm-up calls.  The card's name and power limit are read in the same run and printed
with the numbers.  Prints one JSON line per (path, mode, pass) and a table; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

MODES = ("RGB", "D", "ED", "RGB_D", "RGB_ED")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unavailable"
    return name, q


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts = np.asarray(ts)
    return dict(median_ms=float(np.median(ts)), p10_ms=float(np.percentile(ts, 10)), p90_ms=float(np.percentile(ts, 90)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render_modes.py needs a CUDA device")
    import __graft_entry__ as ge
    import scenes

    pkg = ge.load_package()
    pkg.load()
    dev = torch.device("cuda:0")
    sc = scenes.scene_b(N=args.gaussians)  # config B: 1920x1080, SH degree 3
    t = {k: (torch.from_numpy(np.ascontiguousarray(v)).to(dev) if isinstance(v, np.ndarray) else v)
         for k, v in sc.items()}
    W, H, deg = sc["width"], sc["height"], sc["sh_degree"]
    bg = t.get("background")
    act = {k: t[k].clone().requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh_coeffs")}
    raw = {k: v.detach().clone().requires_grad_(True) for k, v in
           pkg.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"]).items()}
    g = torch.Generator(device=dev).manual_seed(0)
    cot = {"image": torch.randn((3, H, W), device=dev, generator=g),
           "depth": torch.randn((1, H, W), device=dev, generator=g),
           "alpha": torch.randn((1, H, W), device=dev, generator=g)}

    def operator(mode):
        return pkg.rasterize(act["means"], act["quats"], act["scales"], act["opacities"], act["sh_coeffs"], deg,
                             t["viewmats"], t["Ks"], W, H, bg_color=bg, render_mode=mode)

    def fused(mode):
        o = pkg.rasterize_fused(raw["means"], raw["sh0"], raw["shN"], raw["scaling_raw"], raw["rotation_raw"],
                                raw["opacity_raw"], deg, t["viewmats"], t["Ks"], W, H, bg_color=bg, render_mode=mode)
        return o

    def loss(o):
        alpha = o.alpha if o.alpha.dim() == 3 else o.alpha.permute(0, 3, 1, 2)[0]
        s = (alpha * cot["alpha"]).sum()
        if o.image is not None:
            s = s + (o.image * cot["image"]).sum()
        if o.depth is not None:
            s = s + (o.depth * cot["depth"]).sum()
        return s

    name, power = card()
    print(f"# device: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    print(f"# config B: {args.gaussians} Gaussians, {W}x{H}, SH degree {deg}; {args.iters} timed calls after "
          f"{args.warmup} warm-up calls", flush=True)
    rows = []
    for path, run in (("operator", operator), ("fused", fused)):
        for mode in MODES:
            def fwd():
                with torch.no_grad():
                    run(mode)

            def fwd_bwd():
                for p in list(act.values()) + list(raw.values()):
                    p.grad = None
                loss(run(mode)).backward()

            for pas, fn in (("fwd", fwd), ("fwd+bwd", fwd_bwd)):
                r = dict(path=path, mode=mode, pass_=pas, **timed(fn, args.iters, args.warmup), device=name,
                         power_limit=power)
                rows.append(r)
                print(json.dumps(r), flush=True)
    print(f"\n{'path':9s} {'mode':7s} {'pass':8s} {'median ms':>10s} {'p10':>8s} {'p90':>8s}")
    for r in rows:
        print(f"{r['path']:9s} {r['mode']:7s} {r['pass_']:8s} {r['median_ms']:10.3f} {r['p10_ms']:8.3f} {r['p90_ms']:8.3f}")


if __name__ == "__main__":
    main()
