"""GPU: the MCMC strategy (SURVEY.md 8 f6) -- dead mask, weighted sampler, relocation and growth against the torch
restatement (tests/mcmc_restatement.py), the refine without host read-back, and training on both rasterizer paths
against the restatement fed the strategy's own draws and noise."""
import importlib

import numpy as np
import pytest
import torch

import mcmc_restatement as R
import scenes
from parity import rel, to_dev

pytestmark = pytest.mark.gpu


def _mc(native):
    return importlib.import_module(native.__name__ + ".mcmc")


def _ns():
    return torch.ops.gsplat_b200


def _native_relocation(native):
    return lambda op, sc, ratios, binoms, n_max: native.relocation(op, sc, ratios, binoms.to(op.device), n_max)


def _params(N, K, dev, seed=0, dead_frac=0.0):
    """Raw parameters with opacities and quaternion norms on both sides of the thresholds, away from the last ulp."""
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(N, generator=g) * 2
    if dead_frac:
        pick = torch.randperm(N, generator=g)[:int(dead_frac * N)]
        o[pick[: len(pick) // 2]] = -6.0 - torch.rand(len(pick) // 2, generator=g)  # sigmoid < 0.0025
    # exactly at the threshold's neighbourhood, but a clear margin from it
    o[::97] = -5.3  # sigmoid 0.00497 <= 0.005: dead
    o[1::97] = -5.28  # sigmoid 0.00506: alive
    q = torch.randn(N, 4, generator=g)
    if dead_frac:
        q[pick[len(pick) // 2:]] *= 1e-5  # |q|^2 ~ 4e-10 < 1e-8: dead
    q[2::89] *= 0.02  # |q|^2 ~ 1.6e-3: alive
    P = {"means": torch.randn(N, 3, generator=g), "sh0": torch.randn(N, 1, 3, generator=g),
         "shN": torch.randn(N, K, 3, generator=g), "scaling_raw": torch.randn(N, 3, generator=g) - 4,
         "rotation_raw": q, "opacity_raw": o}
    M1 = {k: torch.randn(v.shape, generator=g) for k, v in P.items()}
    M2 = {k: torch.rand(v.shape, generator=g) for k, v in P.items()}
    dv = lambda d: {k: v.to(dev).contiguous() for k, v in d.items()}
    return dv(P), dv(M1), dv(M2)


@pytest.mark.parametrize("case", ["mixed", "all_dead", "none_dead", "one_alive", "large"])
def test_dead_mask_and_order(native, cuda_device, case):
    N = {"large": 3_000_017}.get(case, 50_000)
    P, _, _ = _params(N, 0, cuda_device, seed=1, dead_frac=0.1)
    if case == "all_dead":
        P["opacity_raw"].fill_(-7.0)
    elif case == "none_dead":
        P["opacity_raw"].fill_(1.0)
        P["rotation_raw"][:, 0] = 1.0
    elif case == "one_alive":
        P["opacity_raw"].fill_(-7.0)
        P["opacity_raw"][N // 3] = 0.5
    dead, n_dead, w = _ns().mcmc_dead(P["opacity_raw"], P["rotation_raw"], 0.005)
    want = R.dead_mask(P, 0.005).nonzero().squeeze(-1)
    n = int(n_dead.item())
    assert n == want.numel()
    assert torch.equal(dead[:n].long(), want)
    op = torch.sigmoid(P["opacity_raw"])
    assert torch.equal(w, torch.where(R.dead_mask(P, 0.005), torch.zeros_like(op), op))
    if case == "one_alive":
        assert n == N - 1


def _searchsorted(w, u):
    C = np.cumsum(w.astype(np.float64))
    return np.searchsorted(C, u * C[-1], side="right")


@pytest.mark.parametrize("N", [1, 7, 100_003, 2_000_000])
def test_sampler_injected_uniforms_match_numpy(native, cuda_device, N):
    """Index for index: the first i with C[i] > u * C[N-1]; weights in [2^-8, 1) keep the float64 prefix exact in any
    summation order, and a quarter of them are zero."""
    rng = np.random.default_rng(N)
    w = rng.uniform(2 ** -8, 1.0, N).astype(np.float32)
    w[rng.random(N) < 0.25] = 0.0
    w[0 if N == 1 else N - 1] = 0.5
    u = rng.random(max(N, 4096))
    u[:4] = [0.0, np.nextafter(1.0, 0.0), 0.5, 1e-12]
    got = _ns().mcmc_sample(torch.from_numpy(w).to(cuda_device), u.size, None, torch.from_numpy(u).to(cuda_device), False)
    want = _searchsorted(w, u)
    want = np.minimum(want, N - 1)  # u = 1 - 2^-53 may round u * total up to total: the last positive weight
    got = got.cpu().numpy()
    assert np.array_equal(got, want)
    assert np.all(w[got] > 0)


def test_sampler_philox_seeded_chi_square(native, cuda_device):
    """10^6 draws from torch's generator: deterministic under a seed, different under another, zero weights never
    drawn, and the counts fit the weights (chi-square at the 1e-4 level)."""
    from scipy import stats
    N = 1000
    rng = np.random.default_rng(3)
    w = rng.uniform(0.01, 1.0, N).astype(np.float32)
    w[::10] = 0.0
    wt = torch.from_numpy(w).to(cuda_device)
    draws = []
    for seed in (7, 7, 8):
        torch.manual_seed(seed)
        draws.append(_ns().mcmc_sample(wt, 1_000_000, None, None, False).cpu().numpy())
    assert np.array_equal(draws[0], draws[1])
    assert not np.array_equal(draws[0], draws[2])
    counts = np.bincount(draws[0], minlength=N)
    assert counts[::10].sum() == 0
    nz = w > 0
    expected = w[nz].astype(np.float64) / w[nz].sum() * 1_000_000
    chi2, p = stats.chisquare(counts[nz], expected)
    print(f"chi2 {chi2:.1f} over {nz.sum() - 1} dof, p = {p:.4f}")
    assert p > 1e-4


def test_sampler_above_2_pow_24(native, cuda_device):
    """The reference's host loop takes over above 2^24 Gaussians; here the same kernel runs."""
    N = (1 << 24) + 1000
    torch.manual_seed(0)
    logits = torch.randn(N, device=cuda_device)
    logits[-1000:] = 30.0  # the tail past 2^24 carries ~ sigmoid(30) = 1 each
    s = _ns().mcmc_sample(logits, 200_000, None, None, True)
    assert int(s.min()) >= 0 and int(s.max()) < N
    assert int((s >= (1 << 24)).sum()) > 0  # the tail is drawn (expected ~ 200000 * 1000 / 8.4e6 = 24)
    u = torch.tensor([np.nextafter(1.0, 0.0), 0.0], dtype=torch.float64, device=cuda_device)
    e = _ns().mcmc_sample(logits, 2, None, u, True).cpu().tolist()
    assert e == [N - 1, 0]


def _lists(P, M1, M2):
    return [P[k] for k in R.GROUPS], [M1[k] for k in R.GROUPS], [M2[k] for k in R.GROUPS]


def _ulp_close(a, b, ulps=1):
    a, b = a.float().contiguous(), b.float().contiguous()
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    return bool(((ia - ib).abs() <= ulps).all())


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_relocate_injected_matches_restatement(native, cuda_device, deg):
    K = (deg + 1) ** 2 - 1
    N = 20_000
    P, M1, M2 = _params(N, K, cuda_device, seed=10 + deg, dead_frac=0.05)
    P["opacity_raw"] = P["opacity_raw"].reshape(N, 1).contiguous()
    dead, n_dead, w = _ns().mcmc_dead(P["opacity_raw"].reshape(-1), P["rotation_raw"], 0.005)
    n = int(n_dead.item())
    # injected samples: alive indices with many duplicates (one index drawn 60 times: ratio clamped to 51)
    alive = (~R.dead_mask(P, 0.005)).nonzero().squeeze(-1)
    g = torch.Generator(device=cuda_device).manual_seed(deg)
    samples = alive[torch.randint(0, 50, (n,), device=cuda_device, generator=g)]
    samples[:60] = alive[3]
    Q = {k: v.clone() for k, v in P.items()}
    Q1 = {k: v.clone() for k, v in M1.items()}
    Q2 = {k: v.clone() for k, v in M2.items()}
    s32 = torch.zeros(N, dtype=torch.int32, device=cuda_device)
    s32[:n] = samples.int()
    _ns().mcmc_relocate(*_lists(P, M1, M2), s32, dead, n_dead, _mc(native).binomial_table().to(cuda_device), 0.005)
    R.relocate_gs(Q, Q1, Q2, samples, _native_relocation(native), _mc(native).binomial_table().to(cuda_device), 0.005)
    for k in R.GROUPS:
        if k in ("opacity_raw", "scaling_raw"):
            assert _ulp_close(P[k], Q[k]), k
        else:
            assert torch.equal(P[k], Q[k]), k
        assert torch.equal(M1[k], Q1[k]) and torch.equal(M2[k], Q2[k]), k


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_grow_injected_matches_restatement(native, cuda_device, deg):
    K = (deg + 1) ** 2 - 1
    N, cap = 30_000, 40_000
    P, M1, M2 = _params(N, K, cuda_device, seed=20 + deg)
    n_new = R.growth_count(N, cap)
    g = torch.Generator(device=cuda_device).manual_seed(deg)
    samples = torch.randint(0, 200, (n_new,), device=cuda_device, generator=g)
    store = {k: torch.full((cap,) + tuple(v.shape[1:]), 7.0, device=cuda_device) for k, v in P.items()}
    s1 = {k: torch.full_like(store[k], 7.0) for k in P}
    s2 = {k: torch.full_like(store[k], 7.0) for k in P}
    for k in P:
        store[k][:N], s1[k][:N], s2[k][:N] = P[k], M1[k], M2[k]
    b = _mc(native).binomial_table().to(cuda_device)
    _ns().mcmc_grow(*_lists(store, s1, s2), N, samples.int(), b, 0.005)
    Q, Q1, Q2 = R.add_new_gs({k: v.clone() for k, v in P.items()}, M1, M2, samples, _native_relocation(native), b, 0.005)
    M = N + n_new
    for k in R.GROUPS:
        got = store[k][:M]
        if k in ("opacity_raw", "scaling_raw"):
            assert _ulp_close(got, Q[k]), k
        else:
            assert torch.equal(got, Q[k]), k
        assert torch.equal(s1[k][:M], Q1[k]) and torch.equal(s2[k][:M], Q2[k]), k
        assert bool((store[k][M:] == 7.0).all()), k  # rows past the new ones untouched


def test_relocate_own_draws_invariants_without_host_sync(native, cuda_device):
    """The strategy's own refine under set_sync_debug_mode("error"): every dead row becomes a copy of an alive row s,
    s carries relocation(op_s, min(copies + 1, 51)), its moments are zero and the dead rows keep theirs."""
    mc, training = _mc(native), importlib.import_module(native.__name__ + ".training")
    N = 100_000
    P, _, _ = _params(N, 15, cuda_device, seed=5, dead_frac=0.05)
    P = {k: v.requires_grad_(True) for k, v in P.items()}
    opt = training.FusedAdam(P)
    with torch.no_grad():
        for k in P:
            opt.exp_avg[k].normal_()
            opt.exp_avg_sq[k].uniform_()
    strat = mc.MCMC(P, opt, mc.MCMCConfig(max_cap=N + 3000))
    before = {k: v.detach().clone() for k, v in P.items()}
    m1 = {k: v.clone() for k, v in opt.exp_avg.items()}
    dead_want = R.dead_mask(before, 0.005).nonzero().squeeze(-1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        strat.relocate()
        strat.grow()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert strat.n == N + 3000 and P["means"].shape[0] == N + 3000 and P["means"].grad is None
    dead, n_dead = strat.last_dead
    n = int(n_dead.item())
    assert torch.equal(dead[:n].long(), dead_want)
    s = strat.last_samples[:n].long()
    assert not bool(R.dead_mask(before, 0.005)[s].any())
    counts = torch.bincount(s, minlength=N)
    ratio = (counts[s] + 1).clamp_max(51).int()
    o, sc = native.relocation(torch.sigmoid(before["opacity_raw"][s]), torch.exp(before["scaling_raw"][s]), ratio,
                              strat.binoms, 51)
    gs = strat.last_grow_samples.long()
    regrown = torch.zeros(N, dtype=torch.bool, device=cuda_device)
    regrown[gs] = True  # growth rewrote these rows' opacity and scale again
    keep = ~regrown[s]
    want_o = torch.logit(o.clamp(0.005, 1 - 1e-7))
    assert _ulp_close(P["opacity_raw"].detach()[:N][s][keep], want_o[keep])
    assert _ulp_close(P["scaling_raw"].detach()[:N][s][keep], torch.log(sc)[keep])
    for k in R.GROUPS:
        assert torch.equal(P[k].detach()[dead_want][keep], P[k].detach()[s][keep]) or k in ("opacity_raw", "scaling_raw")
        assert not bool(opt.exp_avg[k][s].any()), k
        assert torch.equal(opt.exp_avg[k][dead_want], m1[k][dead_want]), k
        assert not bool(opt.exp_avg[k][N:].any()), k
    for k in ("means", "sh0", "shN", "rotation_raw"):
        assert torch.equal(P[k].detach()[dead_want], P[k].detach()[s]), k


def _gsplat_problem(native, dev):
    sc = scenes.scene_b(N=6000, width=160, height=112, view=2, scale_mul=2.0)
    t = to_dev(sc, dev)
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    raw = {k: v.detach().clone() for k, v in raw.items()}
    with torch.no_grad():
        raw["opacity_raw"].view(-1)[::40] = -7.0  # dead rows for the first relocations
    g = torch.Generator(device=dev).manual_seed(3)
    target = torch.rand((3, 112, 160), device=dev, generator=g)
    return t, raw, target


def _fastgs_problem(native, dev):
    fg = importlib.import_module(native.__name__ + ".fastgs")
    inp = scenes.fastgs_inputs(scenes.scene_small(N=3000, width=160, height=112, sh_degree=3, seed=6, view=2))
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw",
             "opacity_raw": "opacities_raw", "sh0": "sh0", "shN": "shN"}
    raw = {k: torch.from_numpy(inp[v]).to(dev).contiguous() for k, v in names.items()}
    with torch.no_grad():
        raw["opacity_raw"].view(-1)[::40] = -7.0
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(dev), active_sh_bases=16,
                          width=inp["width"], height=inp["height"], focal_x=inp["fx"], focal_y=inp["fy"],
                          center_x=inp["cx"], center_y=inp["cy"], near_plane=inp["near_plane"],
                          far_plane=inp["far_plane"])
    g = torch.Generator(device=dev).manual_seed(2)
    target = torch.rand((3, inp["height"], inp["width"]), device=dev, generator=g)
    return fg, s, torch.from_numpy(inp["w2c"]).to(dev), raw, target


@pytest.mark.parametrize("path", ["gsplat", "fastgs"])
def test_training_with_strategy_matches_restatement(native, cuda_device, path):
    """60 iterations, refine every 10 from 10 on, cap 1.12 N: growth at 10, 20 and 30 (the third reaches the cap), the
    refines at 40 and 50 only relocate; the SH degree rises every 20 iterations.  The restatement is fed the step's
    photometric gradients (taken before the regularisers are added), the strategy's own draws and its noise, so the two
    differ only by rounding -- separate renders would let Adam amplify gradient differences where gradients are tiny."""
    mc, training = _mc(native), importlib.import_module(native.__name__ + ".training")
    cfg_a = training.AdamConfig(means_lr=1.6e-4, iterations=30000)
    if path == "gsplat":
        t, raw, target = _gsplat_problem(native, cuda_device)
    else:
        fg, settings, w2c, raw, target = _fastgs_problem(native, cuda_device)
    N0 = raw["means"].shape[0]
    cfg = mc.MCMCConfig(start_refine=5, refine_every=10, stop_refine=1000, max_cap=int(1.12 * N0),
                        sh_degree_interval=20)
    P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    opt = training.FusedAdam(P, cfg_a)
    strat = mc.MCMC(P, opt, cfg)
    if path == "gsplat":
        step = training.TrainStep(P, 0, 160, 112, optimizer=opt, strategy=strat)
        run = lambda: step(t["viewmats"], t["Ks"], target, t["background"])
    else:
        step = training.FastGsTrainStep(P, 0, settings.width, settings.height, optimizer=opt, strategy=strat)
        run = lambda: step(w2c, settings, target)
    seen = {}
    regularize = strat.regularize

    def snapshot_then_regularize(params=None):
        seen["G"] = {k: P[k].grad.detach().clone() for k in R.GROUPS}
        seen["deg"] = step.sh_degree if path == "gsplat" else strat.sh_degree
        return regularize(params)
    strat.regularize = snapshot_then_regularize
    rs = R.Strategy(raw, cfg_a.lrs(), cfg, _native_relocation(native), strat.binoms,
                    lambda Q, noise, lr: native.add_noise(Q["opacity_raw"].reshape(-1), Q["scaling_raw"],
                                                          Q["rotation_raw"], noise, Q["means"], lr))
    ns, grew_at = [], []
    for it in range(1, 61):
        refines = strat.refines
        run()
        assert seen["deg"] == rs.sh_degree  # the degree the step rendered with
        reloc = strat.last_samples[:int(strat.last_dead[1].item())] if strat.refines > refines else None
        grew = rs.iteration(it, seen["G"], reloc, strat.last_grow_samples, strat.last_noise)
        if grew:
            grew_at.append(it)
        ns.append(strat.n)
        assert strat.sh_degree == rs.sh_degree
        assert all(P[k].shape == rs.P[k].shape for k in R.GROUPS)
    print(path, "N:", sorted(set(ns)), "growth at", grew_at)
    assert ns == rs.ns
    assert grew_at == [10, 20, 30]
    assert ns[-1] == cfg.max_cap
    for k in R.GROUPS:
        if P[k].numel():
            e = rel(P[k].detach(), rs.P[k])
            e1, e2 = rel(opt.exp_avg[k], rs.M1[k]), rel(opt.exp_avg_sq[k], rs.M2[k])
            print(f"  {k}: params {e:.2e} exp_avg {e1:.2e} exp_avg_sq {e2:.2e}")
            assert e < 1e-5 and e1 < 1e-4 and e2 < 1e-4, k
    assert opt.steps["means"] == 60 - 3 and rs.steps["means"] == 57  # Adam skipped on the growth iterations


def test_regularizer_losses_and_gradients(native, cuda_device):
    """200 Gaussians (one CTA) and ~1 M (the grid-stride loop and the last-CTA reduction over the 128-CTA cap): the two
    loss terms against scale_reg * mean(exp(s)) and opacity_reg * mean(sigmoid(o)) in float64, bit-equal across two
    runs; the gradients against autograd added onto existing ones."""
    for N in (200, 1_000_003):
        P, _, _ = _params(N, 0, cuda_device, seed=9)
        s, o = P["scaling_raw"], P["opacity_raw"]
        # existing gradients of the regularisers' own magnitude, so that the added part keeps its precision
        v_s0, v_o0 = torch.randn_like(s) * 1e-10, torch.randn_like(o) * 1e-9
        runs = []
        for _ in range(2):
            v_s, v_o = v_s0.clone(), v_o0.clone()
            loss = _ns().mcmc_regularize(s, o, 0.01, 0.02, v_s, v_o)
            runs.append((loss.clone(), v_s, v_o))
        assert torch.equal(runs[0][0], runs[1][0]), N
        assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2]), N
        want = torch.stack([0.01 * torch.exp(s.double()).mean(), 0.02 * torch.sigmoid(o.double()).mean()])
        assert torch.allclose(runs[0][0].double(), want, rtol=1e-6, atol=0), N
        g, _, _ = R.regularizer_grads({"scaling_raw": s, "opacity_raw": o}, 0.01, 0.02)
        assert rel(runs[0][1] - v_s0, g["scaling_raw"]) < 1e-5, N
        assert rel(runs[0][2] - v_o0, g["opacity_raw"]) < 1e-5, N


@pytest.mark.parametrize("path", ["gsplat", "fastgs"])
def test_graphed_with_strategy_equals_eager(native, cuda_device, path):
    """The compressed schedule of the eager test: the graphed step (noise and regularisers captured, the refine eager
    between the two captured parts) against the eager step from the same seed.  Re-captures happen after the growth
    steps (10, 20, 30) and the SH bump at 40 only -- not after the relocation-only refine at 50 -- and the warm-up
    moves nothing."""
    mc, training = _mc(native), importlib.import_module(native.__name__ + ".training")
    cfg_a = training.AdamConfig(means_lr=1.6e-4, iterations=30000)
    if path == "gsplat":
        t, raw, target = _gsplat_problem(native, cuda_device)
    else:
        fg, settings, w2c, raw, target = _fastgs_problem(native, cuda_device)
    N0 = raw["means"].shape[0]
    cfg = mc.MCMCConfig(start_refine=5, refine_every=10, stop_refine=1000, max_cap=int(1.12 * N0),
                        sh_degree_interval=20)
    A = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    B = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    C = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    sa = mc.MCMC(A, training.FusedAdam(A, cfg_a), cfg)
    sb = mc.MCMC(B, training.FusedAdam(B, cfg_a), cfg)
    sc = mc.MCMC(C, training.FusedAdam(C, cfg_a), cfg)  # a second eager run: the floor of run-to-run differences

    def eager_step(Q, s):
        if path == "gsplat":
            e = training.TrainStep(Q, 0, 160, 112, optimizer=s.optimizer, strategy=s)
            return lambda: e(t["viewmats"], t["Ks"], target, t["background"])
        e = training.FastGsTrainStep(Q, 0, settings.width, settings.height, optimizer=s.optimizer, strategy=s)
        return lambda: e(w2c, settings, target)
    run_a, run_c = eager_step(A, sa), eager_step(C, sc)
    if path == "gsplat":
        graphed = training.GraphedTrainStep(B, 0, 160, 112, strategy=sb)
        run_b = lambda: graphed(t["viewmats"], t["Ks"], target, t["background"])
    else:
        graphed = training.GraphedFastGsTrainStep(B, 0, settings, strategy=sb)
        run_b = lambda: graphed(w2c, settings.cam_position, target)
    before = {k: v.detach().clone() for k, v in B.items()}
    graphed.capture(*((t["viewmats"], t["Ks"], target, t["background"]) if path == "gsplat"
                      else (w2c, settings.cam_position, target)))
    for k in B:
        assert torch.equal(B[k].detach(), before[k]), k  # warm-up and capture moved nothing
    ns_a, ns_b, la, lb = [], [], [], []
    captures_at = []
    for it in range(1, 61):
        torch.manual_seed(1000 + it)  # both runs draw from the same generator state
        la.append(float(run_a()))
        torch.manual_seed(1000 + it)
        c = graphed.captures
        lb.append(float(run_b()))
        torch.manual_seed(1000 + it)
        run_c()
        if graphed.captures != c:
            captures_at.append(it)
        ns_a.append(sa.n)
        ns_b.append(sb.n)
    print(path, "re-captured at", captures_at, "N", sorted(set(ns_b)))
    assert ns_a == ns_b and ns_b[-1] == cfg.max_cap
    assert captures_at == [11, 21, 31, 41]
    assert graphed.captures == 5
    for a, b in zip(la, lb):
        assert abs(a - b) <= 1e-4 * max(1.0, abs(a))
    assert sc.n == sa.n
    for k in R.GROUPS:
        if A[k].numel():
            e = rel(B[k].detach(), A[k].detach())
            e1 = rel(sb.optimizer.exp_avg[k], sa.optimizer.exp_avg[k])
            floor = rel(C[k].detach(), A[k].detach())  # the backward's atomics make two eager runs differ too
            print(f"  {k}: params {e:.2e} (eager vs eager {floor:.2e}) exp_avg {e1:.2e}")
            assert e < max(1e-4, 5 * floor) and e1 < 1e-2, k
    assert sa.optimizer.steps == sb.optimizer.steps
    assert sb.sh_degree == 3
