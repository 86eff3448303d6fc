"""ADMM sparsification (sparsity.py, csrc/gsb_sparsity.cu, gsb_adc.cu) on the GPU.

Kernel parts at 1 M and 6 M Gaussians, each beside the reference's torch composition (restated line by line in
tests/sparsity_restatement.py) from the same state:
  update  update_state: the device select of the prune_z threshold and the elementwise z / u pass, against sort + ops
  loss    the loss and its gradient added into opacity_raw.grad, against sigmoid / norm / pow and autograd
  prune   the final prune at SH degree 3 with both Adam moments, against topk + index_select of 6 tensors x 3
Times are medians of K runs between CUDA events after warm-up.  At each size the outputs are compared in the same run:
z and u bit for bit, the loss to 1e-5 relative and the gradient to 1e-5 of its largest entry, the pruned rows and
moments bit for bit (when no row is tied at the boundary).

Then the graphed fastgs iteration at 1 M Gaussians, 1920x1080, with the MCMC strategy, inside the sparsity phase
(loss in the captured part, an update every 50 iterations), beside the same iteration without sparsity.  Prints one
JSON line with the card's name and power limit.  Writes nothing to the tree."""
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
    g = torch.Generator(device=dev).manual_seed(0)
    P = {"means": torch.randn(N, 3, device=dev, generator=g), "sh0": torch.randn(N, 1, 3, device=dev, generator=g),
         "shN": torch.randn(N, 15, 3, device=dev, generator=g), "scaling_raw": torch.randn(N, 3, device=dev, generator=g),
         "rotation_raw": torch.randn(N, 4, device=dev, generator=g),
         "opacity_raw": torch.randn(N, 1, device=dev, generator=g) * 3}
    M1 = {k: torch.randn(v.shape, device=dev, generator=g) for k, v in P.items()}
    M2 = {k: torch.rand(v.shape, device=dev, generator=g) for k, v in P.items()}
    return P, M1, M2


def run(sizes, iters: int) -> dict:
    import __graft_entry__ as ge
    import sparsity_restatement as R
    pkg = ge.load_package()
    pkg.load()
    sp = importlib.import_module(pkg.__name__ + ".sparsity")
    adc = importlib.import_module(pkg.__name__ + ".adc")
    ns = torch.ops.gsplat_b200
    dev = torch.device("cuda:0")
    out = {"card": _card(), "iters": iters, "results": []}
    for N in sizes:
        P, M1, M2 = _scene(N, dev)
        o = P["opacity_raw"]
        k = sp.prune_count(0.6, N)
        # ---- update: a state after one update, then one more update timed from it
        z0, u0 = torch.empty(N, device=dev), torch.empty(N, device=dev)
        ns.sparsity_update(o, z0, u0, k, True)
        o1 = (o + 0.1 * torch.randn_like(o)).contiguous()
        ns.sparsity_update(o1, z0, u0, k, False)
        z, u = z0.clone(), u0.clone()
        restore = lambda: (z.copy_(z0), u.copy_(u0))
        row = {"N": N, "update_this_library_ms": _time(restore, lambda: ns.sparsity_update(o, z, u, k, False), iters)}
        rz, ru = z0.view(-1, 1).clone(), u0.view(-1, 1).clone()

        def ref_update():
            R.update_state(o, rz.clone(), ru.clone(), 0.6)
        row["update_reference_ms"] = _time(lambda: None, ref_update, iters)
        restore()
        ns.sparsity_update(o, z, u, k, False)
        wz, wu = R.update_state(o, z0.view(-1, 1).clone(), u0.view(-1, 1).clone(), 0.6)
        row["update_equal"] = bool(torch.equal(z, wz.flatten()) and torch.equal(u, wu.flatten()))
        # ---- loss and gradient, added into an existing gradient
        rho = torch.full((1,), 5e-4, device=dev)
        g0 = torch.randn(N, device=dev) * 1e-6
        g = g0.clone()
        row["loss_this_library_ms"] = _time(lambda: g.copy_(g0), lambda: ns.sparsity_loss(o.view(-1), z0, u0, rho, g),
                                            iters)
        oo = o.detach().clone().requires_grad_(True)
        gz, gu = z0.view(-1, 1), u0.view(-1, 1)

        def ref_loss():
            oo.grad = g0.view(-1, 1).clone()
            R.loss(oo, gz, gu, 5e-4).backward()
        row["loss_reference_ms"] = _time(lambda: None, ref_loss, iters)
        g.copy_(g0)
        lv = ns.sparsity_loss(o.view(-1), z0, u0, rho, g)
        ref_loss()
        want = R.loss(oo.detach(), gz, gu, 5e-4)
        scale = float((oo.grad - g0.view(-1, 1)).abs().max())
        row["loss_equal"] = bool(abs(float(lv) - float(want)) <= 1e-5 * abs(float(want))
                                 and float((g.view(-1, 1) - oo.grad).abs().max()) <= 1e-5 * scale)
        del oo, g, g0
        # ---- prune at SH degree 3, both moments
        lists = ([P[k_] for k_ in GROUPS], [M1[k_] for k_ in GROUPS], [M2[k_] for k_ in GROUPS])
        row["prune_this_library_ms"] = _time(lambda: None, lambda: adc.lowest_opacity_removed(*lists, k), iters)
        row["prune_reference_ms"] = _time(lambda: None,
                                          lambda: R.remove_gaussians(P, M1, M2, R.prune_mask(o, 0.6)), iters)
        gp, g1, g2, _ = adc.lowest_opacity_removed(*lists, k)
        WP, WM1, WM2 = R.remove_gaussians(P, M1, M2, R.prune_mask(o, 0.6))
        s = torch.sigmoid(o.flatten())
        v = torch.sort(s).values[k - 1]
        tied = int((s == v).sum()) > 1
        row["prune_rows"] = [N, N - k]
        row["prune_equal"] = "tie at the boundary" if tied else bool(
            all(torch.equal(a, WP[n]) and torch.equal(b, WM1[n]) and torch.equal(c, WM2[n])
                for n, a, b, c in zip(GROUPS, gp, g1, g2)))
        out["results"].append(row)
        del P, M1, M2, lists, gp, g1, g2, WP, WM1, WM2, z, u, z0, u0, o1
        torch.cuda.empty_cache()
    return out


def iteration_fastgs(iters: int) -> dict:
    """The graphed fastgs iteration (1 M Gaussians, 1920x1080, SH degree 3, MCMC) inside the sparsity phase -- the
    loss in the captured part A, an eager update every 50 iterations -- beside the same iteration without sparsity.
    Per-iteration times over one window of `iters` iterations after the phase entry's re-capture."""
    import __graft_entry__ as ge
    import scenes
    pkg = ge.load_package()
    mc = importlib.import_module(pkg.__name__ + ".mcmc")
    sp = importlib.import_module(pkg.__name__ + ".sparsity")
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
    res = {"gaussians": raw["means"].shape[0], "width": inp["width"], "height": inp["height"], "iters": iters,
           "update_every": 50}
    cfg = mc.MCMCConfig(start_refine=10 ** 9, max_cap=raw["means"].shape[0])

    def window(sparsity):
        P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
        st = mc.MCMC(P, training.FusedAdam(P), cfg, sh_degree=3)
        step = training.GraphedFastGsTrainStep(P, 3, s, strategy=st, sparsity=sparsity)
        for _ in range(10):  # enters the phase at 5 (with sparsity): the re-capture is outside the window
            step(w2c, cam, target)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            step(w2c, cam, target)
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / iters, step.captures

    res["graphed_mcmc_ms"], _ = window(None)
    torch.cuda.empty_cache()
    cfg_s = sp.SparsityConfig(start_iteration=5, sparsify_steps=10 ** 6)
    res["graphed_mcmc_sparsity_ms"], res["captures_with_sparsity"] = window(sp.ADMMSparsity(cfg_s))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--sizes", default="1000000,6000000")
    ap.add_argument("--window", type=int, default=300, help="iterations of the graphed fastgs window")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparsity.py needs a CUDA device")
    out = run([int(x) for x in a.sizes.split(",")], a.iters)
    torch.cuda.empty_cache()
    out["iteration_fastgs"] = iteration_fastgs(a.window) if a.window > 0 else None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
