"""Default-strategy (adaptive density control) refine benchmark: one refine -- grow_gs (duplicate, split) then
prune_gs -- at 1 M and 6 M Gaussians (SH degree 3) with seeded statistics giving about 5 % duplicated, 5 % split and 2 %
pruned rows.  This library's strategy (adc.py over csrc/gsb_adc.cu) and, where oracle/build_ref.py built the
reference's gsplat kernels into oracle/_ref, the reference's composition (the torch ops of default_strategy.cpp
grow_gs / prune_gs, as tests/adc_restatement.py restates them, around the reference's own quats_to_rotmats) in the same
run, from the same state and the same normals.

  python bench_adc.py [--iters K] [--sizes 1000000,6000000] [--window W]

Then the graphed fastgs training iteration at 1 M Gaussians, 1920x1080, with the strategy refining every 100 iterations
(re-captures included) beside the same iteration without a strategy.

Every timed refine starts from the same restored state (the restore is outside the timed window); times are the median
of K runs between CUDA events after warm-up, and include the refine's one count read-back and the normals' draw.  At
each timed size the two outputs are compared: counts and every group and moment bit for bit, except the split copies'
means, which agree to 1e-5 relative (the composition forms the offset with einsum).  Prints one JSON line.  Writes
nothing to the tree."""
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

GROUPS = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(q.splitlines()[0])
    except Exception:
        info["power_limit_w"] = None
    return info


def _time(restore, fn, iters: int, warmup: int = 3) -> float:
    ts = []
    for i in range(warmup + iters):
        restore()
        torch.manual_seed(5)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        if i >= warmup:
            ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def _scene(N: int, dev):
    """Raw parameters, moments and statistics: 10 % of the rows have a high gradient signal, half of them small
    (duplicated) and half large (split); 2 % of the rest are below the opacity threshold (pruned)."""
    g = torch.Generator(device=dev).manual_seed(0)
    u = lambda *s: torch.rand(*s, device=dev, generator=g)
    r = u(N)
    high, dead = r < 0.10, (r >= 0.10) & (r < 0.12)
    small = u(N) < 0.5
    base = torch.where(high & small, 0.004, 0.04)
    P = {"means": torch.randn(N, 3, device=dev, generator=g), "sh0": torch.randn(N, 1, 3, device=dev, generator=g),
         "shN": torch.randn(N, 15, 3, device=dev, generator=g),
         "scaling_raw": torch.log(base[:, None] * (0.6 + 0.4 * u(N, 3))),
         "rotation_raw": torch.randn(N, 4, device=dev, generator=g),
         "opacity_raw": torch.logit(0.05 + 0.9 * u(N, 1))}
    P["opacity_raw"][dead] = -7.0
    count = torch.randint(1, 5, (N,), device=dev, generator=g).float()
    sig = torch.where(high, 5e-4 + 1e-2 * u(N), 1e-4 * u(N))
    info = torch.stack([count, sig * count])
    M1 = {k: torch.randn(v.shape, device=dev, generator=g) for k, v in P.items()}
    M2 = {k: torch.rand(v.shape, device=dev, generator=g) for k, v in P.items()}
    return P, M1, M2, info


def _same(P, M1, M2, WP, WM1, WM2, n_plain) -> bool:
    ok = all(torch.equal(P[k], WP[k]) for k in GROUPS if k != "means")
    ok &= all(torch.equal(M1[k], WM1[k]) and torch.equal(M2[k], WM2[k]) for k in GROUPS)
    ok &= torch.equal(P["means"][:n_plain], WP["means"][:n_plain])
    ok &= torch.allclose(P["means"][n_plain:], WP["means"][n_plain:], rtol=1e-5, atol=1e-5)
    return bool(ok)


def run(sizes, iters: int) -> dict:
    import __graft_entry__ as ge
    import adc_restatement as R
    pkg = ge.load_package()
    pkg.load()
    adc = importlib.import_module(pkg.__name__ + ".adc")
    training = importlib.import_module(pkg.__name__ + ".training")
    from oracle import ref_ops
    ref = ref_ops._ns() if ref_ops.available() else None
    dev = torch.device("cuda:0")
    cfg = adc.DefaultConfig()
    it = cfg.start_refine + cfg.refine_every  # <= reset_every: no too-big pruning
    out = {"card": _card(), "iters": iters, "results": []}
    for N in sizes:
        base, m1_0, m2_0, info0 = _scene(N, dev)
        P = {k: v.clone().requires_grad_(True) for k, v in base.items()}
        opt = training.FusedAdam(P)
        strat = adc.DefaultStrategy(P, opt, cfg)

        def restore_lib():
            for k in GROUPS:
                P[k] = base[k].clone().requires_grad_(True)
                opt.exp_avg[k], opt.exp_avg_sq[k] = m1_0[k].clone(), m2_0[k].clone()
            strat.densification_info = info0.clone()
        t_lib = _time(restore_lib, lambda: strat.grow_and_prune(it), iters)
        restore_lib()
        torch.manual_seed(5)
        strat.grow_and_prune(it)
        counts, z = strat.last_counts, strat.last_z
        row = {"N": N, "op": "refine", "duplicated": counts[0], "split": counts[1], "pruned": counts[2],
               "n_final": counts[3], "this_library_ms": t_lib}
        lib_out = ({k: P[k].detach() for k in GROUPS}, dict(opt.exp_avg), dict(opt.exp_avg_sq))
        n_plain = counts[3] - 2 * strat.last_kept_split
        if ref is not None:
            with torch.no_grad():
                q2r = ref.quats_to_rotmats
                row["reference_ms"] = _time(lambda: None, lambda: R.refine(base, m1_0, m2_0, info0, it, cfg, 1.0, q2r),
                                            iters)
                torch.manual_seed(5)
                WP, WM1, WM2, wc, wz = R.refine(base, m1_0, m2_0, info0, it, cfg, 1.0, q2r)
                row["same_normals"] = bool(torch.equal(wz, z))
                row["outputs_equal"] = bool(wc == counts and _same(*lib_out, WP, WM1, WM2, n_plain))
                del WP, WM1, WM2
        out["results"].append(row)
        del strat, opt, P, lib_out, base, m1_0, m2_0, info0
        torch.cuda.empty_cache()
    if ref is None:
        out["reference"] = "skipped: oracle/_ref/libgsplat_ref.so not built"
    return out


def iteration_fastgs(iters: int) -> dict:
    """The graphed fastgs iteration (1 M Gaussians, 1920x1080, SH degree 3) with the strategy refining every 100
    iterations -- part A captured, the refine eager, Adam captured, a re-capture after every refine that replaced the
    tensors -- beside the same iteration without a strategy.  Per-iteration times over one window of `iters`
    iterations (CUDA events around the window), so the refines and re-captures are amortised."""
    import __graft_entry__ as ge
    import scenes
    pkg = ge.load_package()
    adc = importlib.import_module(pkg.__name__ + ".adc")
    fg = importlib.import_module(pkg.__name__ + ".fastgs")
    training = importlib.import_module(pkg.__name__ + ".training")
    dev = torch.device("cuda:0")
    inp = scenes.fastgs_inputs(scenes.scene_b(N=1_000_000))
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw",
             "opacity_raw": "opacities_raw", "sh0": "sh0", "shN": "shN"}
    raw = {k: torch.from_numpy(inp[v]).to(dev).contiguous() for k, v in names.items()}
    cam = torch.from_numpy(inp["cam_position"]).to(dev)
    s = fg.FastGSSettings(cam_position=cam, active_sh_bases=16, width=inp["width"], height=inp["height"],
                          focal_x=inp["fx"], focal_y=inp["fy"], center_x=inp["cx"], center_y=inp["cy"],
                          near_plane=inp["near_plane"], far_plane=inp["far_plane"])
    w2c = torch.from_numpy(inp["w2c"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(3)
    target = torch.rand((3, inp["height"], inp["width"]), device=dev, generator=g)
    res = {"gaussians": raw["means"].shape[0], "iters": iters, "refine_every": 100}

    def window(step):
        for _ in range(5):
            step(w2c, cam, target)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            step(w2c, cam, target)
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / iters

    P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    res["graphed_no_strategy_ms"] = window(training.GraphedFastGsTrainStep(P, 3, s))
    del P
    torch.cuda.empty_cache()
    P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    st = adc.DefaultStrategy(P, training.FusedAdam(P), adc.DefaultConfig(start_refine=0, refine_every=100), sh_degree=3)
    step = training.GraphedFastGsTrainStep(P, 3, s, strategy=st)
    res["graphed_with_strategy_ms"] = window(step)
    res["refines_in_window"] = st.refines
    res["captures"] = step.captures
    res["n_after"] = st.n
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--sizes", default="1000000,6000000")
    ap.add_argument("--window", type=int, default=300, help="iterations of the graphed fastgs window")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adc.py needs a CUDA device")
    out = run([int(s) for s in a.sizes.split(",")], a.iters)
    torch.cuda.empty_cache()
    out["iteration_fastgs"] = iteration_fastgs(a.window) if a.window > 0 else None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
