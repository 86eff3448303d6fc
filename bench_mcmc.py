"""MCMC refine benchmark (SURVEY.md 8 f6): a relocation refine with 1 % and 5 % dead Gaussians and a 5 % growth step at
1 M and 6 M Gaussians (SH degree 3) -- this library's strategy (mcmc.py over csrc/gsb_mcmc.cu) and, where
oracle/build_ref.py built the reference's gsplat kernels into oracle/_ref, the reference's composition (the torch ops of
mcmc.cpp relocate_gs / add_new_gs around the reference's own relocation kernel) in the same run.

  python bench_mcmc.py [--iters K] [--sizes 1000000,6000000] [--window W]

Then the graphed config-D iteration with the strategy at the cap (refine amortised) beside the same iteration without
a strategy (iteration_config_d).

Dead Gaussians are a seeded subset pushed below logit(0.005).  Every timed run starts from the same restored state
(the restore is outside the timed window); times are the median of K runs between CUDA events after warm-up.  Each
timed size's outputs are checked against the strategy's invariants: every dead row is a copy of an alive row, that
row's Adam moments are zero and the dead rows' moments are kept (relocation); the new rows copy their samples and
start with zero moments (growth).  Prints one JSON line.  Writes nothing to the tree."""
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


def _scene(N: int, dead_frac: float, dev) -> dict:
    g = torch.Generator(device=dev).manual_seed(0)
    P = {"means": torch.randn(N, 3, device=dev, generator=g), "sh0": torch.randn(N, 1, 3, device=dev, generator=g),
         "shN": torch.randn(N, 15, 3, device=dev, generator=g),
         "scaling_raw": torch.randn(N, 3, device=dev, generator=g) - 4,
         "rotation_raw": torch.randn(N, 4, device=dev, generator=g),
         "opacity_raw": torch.randn(N, 1, device=dev, generator=g)}
    P["opacity_raw"].clamp_(min=-5.0)  # sigmoid >= 0.0067: alive unless pushed below
    dead = torch.randperm(N, device=dev, generator=g)[:int(dead_frac * N)]
    P["opacity_raw"][dead] = -5.3 - torch.rand(dead.numel(), 1, device=dev, generator=g)  # below logit(0.005) = -5.293
    return P


# ---- the reference's composition: mcmc.cpp:112-190 and :192-347 as torch ops around its relocation kernel ----------
def ref_relocate(ref, P, M1, M2, binoms, min_opacity=0.005):
    op = torch.sigmoid(P["opacity_raw"]).squeeze(-1)
    dead_mask = (op <= min_opacity) | ((P["rotation_raw"] * P["rotation_raw"]).sum(-1) < 1e-8)
    dead = dead_mask.nonzero().squeeze(-1)
    alive = (~dead_mask).nonzero().squeeze(-1)
    s = alive.index_select(0, torch.multinomial(op.index_select(0, alive), dead.numel(), True))
    ratios = torch.ones_like(op, dtype=torch.int32)
    ratios.index_add_(0, s, torch.ones_like(s, dtype=torch.int32))
    ratios = ratios.index_select(0, s).clamp_max_(51).contiguous()
    no, nsc = ref.relocation(op.index_select(0, s), torch.exp(P["scaling_raw"]).index_select(0, s), ratios, binoms, 51)
    no = no.clamp_(min_opacity, 1.0 - 1e-7)
    P["opacity_raw"][s] = torch.logit(no).unsqueeze(-1)
    P["scaling_raw"].index_put_((s,), torch.log(nsc))
    for k in GROUPS:
        P[k].index_put_((dead,), P[k].index_select(0, s))
    for k in GROUPS:
        M1[k].index_put_((s,), torch.zeros((), device=s.device))
        M2[k].index_put_((s,), torch.zeros((), device=s.device))
    return dead, s


def ref_grow(ref, P, M1, M2, binoms, n_new, min_opacity=0.005):
    op = torch.sigmoid(P["opacity_raw"]).squeeze(-1)
    s = torch.multinomial(op, n_new, True)
    counts = torch.zeros(op.shape[0], dtype=torch.float32, device=op.device)
    counts.index_add_(0, s, torch.ones_like(s, dtype=torch.float32))
    ratios = torch.clamp(counts.index_select(0, s) + 1, 1, 51).to(torch.int32).contiguous()
    no, nsc = ref.relocation(op.index_select(0, s), torch.exp(P["scaling_raw"]).index_select(0, s), ratios, binoms, 51)
    no = torch.clamp(no, min_opacity, 1.0 - 1e-7)
    P["opacity_raw"][s] = torch.logit(no).unsqueeze(-1)
    P["scaling_raw"].index_put_((s,), torch.log(nsc))
    nP = {k: torch.cat([P[k], P[k].index_select(0, s)], 0) for k in GROUPS}
    nM1 = {k: torch.cat([M1[k], torch.zeros_like(P[k].index_select(0, s))], 0) for k in GROUPS}
    nM2 = {k: torch.cat([M2[k], torch.zeros_like(P[k].index_select(0, s))], 0) for k in GROUPS}
    return nP, nM1, nM2, s


def _check_relocation(P0, M10, P, M1, dead, s) -> bool:
    ok = all(torch.equal(P[k][dead], P[k][s]) for k in ("means", "sh0", "shN", "rotation_raw"))
    ok &= all(not bool(M1[k][s].any()) for k in GROUPS)
    ok &= all(torch.equal(M1[k][dead[~torch.isin(dead, s)]], M10[k][dead[~torch.isin(dead, s)]]) for k in GROUPS)
    ok &= not bool((torch.sigmoid(P0["opacity_raw"]).squeeze(-1)[s] <= 0.005).any())
    return bool(ok)


def _check_growth(P, M1, N, s) -> bool:
    ok = all(torch.equal(P[k][N:], P[k][s]) for k in GROUPS)
    ok &= all(not bool(M1[k][N:].any()) for k in GROUPS)
    return bool(ok)


def run(sizes, iters: int) -> dict:
    import __graft_entry__ as ge
    pkg = ge.load_package()
    pkg.load()
    mc = importlib.import_module(pkg.__name__ + ".mcmc")
    training = importlib.import_module(pkg.__name__ + ".training")
    from oracle import ref_ops
    ref = ref_ops._ns() if ref_ops.available() else None
    dev = torch.device("cuda:0")
    binoms = mc.binomial_table().to(dev)
    out = {"card": _card(), "iters": iters, "results": []}
    for N in sizes:
        for dead_frac in (0.01, 0.05):
            base = _scene(N, dead_frac, dev)
            g = torch.Generator(device=dev).manual_seed(1)
            m1_0 = {k: torch.randn(v.shape, device=dev, generator=g) for k, v in base.items()}
            m2_0 = {k: torch.rand(v.shape, device=dev, generator=g) for k, v in base.items()}
            # this library: capacity-resident strategy at the cap (no growth)
            P = {k: v.clone().requires_grad_(True) for k, v in base.items()}
            opt = training.FusedAdam(P)
            strat = mc.MCMC(P, opt, mc.MCMCConfig(max_cap=N))

            def restore_lib():
                with torch.no_grad():
                    for k in GROUPS:
                        strat.store[k][:N].copy_(base[k])
                        strat.store_m1[k][:N].copy_(m1_0[k])
                        strat.store_m2[k][:N].copy_(m2_0[k])
            t_lib = _time(restore_lib, strat.relocate, iters)
            restore_lib()
            strat.relocate()
            dead, n_dead = strat.last_dead
            nd = int(n_dead.item())
            ok_lib = _check_relocation(base, m1_0, {k: strat.store[k][:N] for k in GROUPS},
                                       {k: strat.store_m1[k][:N] for k in GROUPS}, dead[:nd].long(),
                                       strat.last_samples[:nd].long())
            row = {"N": N, "op": f"relocate_{int(dead_frac * 100)}pct_dead", "n_dead": nd,
                   "this_library_ms": t_lib, "this_library_verified": ok_lib}
            del strat, opt, P
            if ref is not None:
                RP = {k: v.clone() for k, v in base.items()}
                RM1 = {k: v.clone() for k, v in m1_0.items()}
                RM2 = {k: v.clone() for k, v in m2_0.items()}

                def restore_ref():
                    for k in GROUPS:
                        RP[k].copy_(base[k])
                        RM1[k].copy_(m1_0[k])
                        RM2[k].copy_(m2_0[k])
                with torch.no_grad():
                    row["reference_ms"] = _time(restore_ref, lambda: ref_relocate(ref, RP, RM1, RM2, binoms), iters)
                    restore_ref()
                    d, s = ref_relocate(ref, RP, RM1, RM2, binoms)
                    row["reference_verified"] = _check_relocation(base, m1_0, RP, RM1, d, s)
                del RP, RM1, RM2
            out["results"].append(row)
            torch.cuda.empty_cache()
        # 5 % growth from N
        base = _scene(N, 0.0, dev)
        n_new = mc.growth_count(N, 10 ** 9)
        g = torch.Generator(device=dev).manual_seed(2)
        m1_0 = {k: torch.randn(v.shape, device=dev, generator=g) for k, v in base.items()}
        m2_0 = {k: torch.rand(v.shape, device=dev, generator=g) for k, v in base.items()}
        P = {k: v.clone().requires_grad_(True) for k, v in base.items()}
        opt = training.FusedAdam(P)
        strat = mc.MCMC(P, opt, mc.MCMCConfig(max_cap=N + n_new))
        for k in GROUPS:
            opt.exp_avg[k].copy_(m1_0[k])
            opt.exp_avg_sq[k].copy_(m2_0[k])

        def restore_grow():
            strat.n = N
            with torch.no_grad():
                for k in ("opacity_raw", "scaling_raw"):
                    strat.store[k][:N].copy_(base[k])
        t_lib = _time(restore_grow, strat.grow, iters)
        restore_grow()
        strat.grow()
        ok_lib = _check_growth(strat.store, strat.store_m1, N, strat.last_grow_samples.long())
        row = {"N": N, "op": "grow_5pct", "n_new": n_new, "this_library_ms": t_lib, "this_library_verified": ok_lib}
        del strat, opt, P
        torch.cuda.empty_cache()
        if ref is not None:
            with torch.no_grad():
                RP = {k: v.clone() for k, v in base.items()}

                def restore_ref():
                    for k in ("opacity_raw", "scaling_raw"):
                        RP[k].copy_(base[k])
                row["reference_ms"] = _time(restore_ref, lambda: ref_grow(ref, RP, m1_0, m2_0, binoms, n_new), iters)
                restore_ref()
                nP, nM1, _, s = ref_grow(ref, RP, m1_0, m2_0, binoms, n_new)
                row["reference_verified"] = _check_growth(nP, nM1, N, s)
                del nP, nM1, RP
        out["results"].append(row)
        del base, m1_0, m2_0
        torch.cuda.empty_cache()
    if ref is None:
        out["reference"] = "skipped: oracle/_ref/libgsplat_ref.so not built"
    return out


def iteration_config_d(iters: int) -> dict:
    """The graphed config-D iteration (6 M Gaussians, 1920x1080, SH degree 3) with the strategy at the cap -- noise and
    regularisers in the graph, a relocation refine every 100 iterations run eagerly between the two captured parts --
    beside the same iteration without a strategy.  Times are per iteration over one window of `iters` iterations
    (CUDA events around the window), so the refines are amortised."""
    import __graft_entry__ as ge
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import scenes
    from parity import to_dev
    pkg = ge.load_package()
    mc = importlib.import_module(pkg.__name__ + ".mcmc")
    training = importlib.import_module(pkg.__name__ + ".training")
    dev = torch.device("cuda:0")
    sc = scenes.scene_b(N=6_000_000)
    t = to_dev(sc, dev)
    raw = pkg.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    raw = {k: v.detach().clone() for k, v in raw.items()}
    N = raw["means"].shape[0]
    g = torch.Generator(device=dev).manual_seed(3)
    with torch.no_grad():  # 1 % dead, so that every refine relocates
        raw["opacity_raw"].view(-1)[torch.randperm(N, device=dev, generator=g)[:N // 100]] = -6.0
    target = torch.rand((3, 1080, 1920), device=dev, generator=g)
    del sc, t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"]
    res = {"gaussians": N, "iters": iters, "refine_every": 100}

    def window(step):
        for _ in range(5):
            step(t["viewmats"], t["Ks"], target, t["background"])
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            step(t["viewmats"], t["Ks"], target, t["background"])
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / iters

    P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    res["graphed_no_strategy_ms"] = window(training.GraphedTrainStep(P, 3, 1920, 1080))
    del P
    torch.cuda.empty_cache()
    P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    st = mc.MCMC(P, training.FusedAdam(P), mc.MCMCConfig(max_cap=N, start_refine=0, refine_every=100), sh_degree=3)
    step = training.GraphedTrainStep(P, 3, 1920, 1080, strategy=st)
    res["graphed_with_strategy_ms"] = window(step)
    res["refines_in_window"] = st.refines
    res["captures"] = step.captures
    res["n_after"] = st.n
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--sizes", default="1000000,6000000")
    ap.add_argument("--window", type=int, default=200, help="iterations of the graphed config-D window")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mcmc.py needs a CUDA device")
    out = run([int(s) for s in a.sizes.split(",")], a.iters)
    torch.cuda.empty_cache()
    out["iteration_config_d"] = iteration_config_d(a.window) if a.window > 0 else None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
