"""GPU: ADMM sparsification -- the state update bit for bit against the torch restatement
(tests/sparsity_restatement.py) over sizes and input kinds, the loss and its gradient, the final prune for both
strategies, the phase without host synchronisation, a short schedule through the eager training steps on both
rasterizer paths and strategies, and the graphed steps against the eager ones."""
import importlib

import pytest
import torch

import scenes
import sparsity_restatement as R
from parity import to_dev

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -23


def _ns():
    return torch.ops.gsplat_b200


def _mods(native):
    return tuple(importlib.import_module(native.__name__ + "." + m) for m in ("sparsity", "training", "mcmc", "adc"))


def _opacity(N, kind, dev, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        o = torch.randn(N, generator=g) * 3
    elif kind == "quantised":  # heavy ties: 7 distinct values
        o = (torch.randint(0, 7, (N,), generator=g).float() - 3.0) * 0.5
    else:  # all equal
        o = torch.full((N,), 0.25)
    return o.to(dev).contiguous()


@pytest.mark.parametrize("kind", ["random", "quantised", "equal"])
@pytest.mark.parametrize("N", [1, 4, 1000, 1_000_003, 2 ** 24 + 3])
def test_update_matches_restatement_bitwise(native, cuda_device, N, kind):
    o = _opacity(N, kind, cuda_device, seed=N)
    k = R.prune_index(0.6, N)
    z, u = torch.empty_like(o), torch.empty_like(o)
    _ns().sparsity_update(o, z, u, k, True)
    wz, wu = R.initialize(o[:, None], 0.6)
    assert torch.equal(z, wz.flatten()) and torch.equal(u, wu.flatten()), "initialize"
    for step in range(2):
        o2 = (o + 0.3 * _opacity(N, "random", cuda_device, seed=N + 1 + step)).contiguous()
        if kind != "random":
            o2 = o2.round()  # keep the ties
        _ns().sparsity_update(o2, z, u, k, False)
        wz, wu = R.update_state(o2[:, None], wz, wu, 0.6)
        assert torch.equal(z, wz.flatten()) and torch.equal(u, wu.flatten()), ("update", step)
    if N >= 1000:
        assert int((z == 0).sum()) >= k


def test_loss_and_gradient(native, cuda_device):
    N = 1_000_003
    o = _opacity(N, "random", cuda_device, seed=5)
    z, u = R.initialize(o[:, None], 0.6)
    z, u = R.update_state((o + 0.2)[:, None], z, u, 0.6)
    z, u = z.flatten().contiguous(), u.flatten().contiguous()
    rho = torch.full((1,), 5e-4, device=cuda_device)
    g0 = torch.randn(N, device=cuda_device) * 1e-6
    runs = []
    for _ in range(2):
        g = g0.clone()
        loss = _ns().sparsity_loss(o, z, u, rho, g)
        runs.append((loss.clone(), g))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])  # deterministic
    oo = o.clone().requires_grad_(True)
    want = R.loss(oo, z, u, 5e-4)
    want.backward()
    assert abs(float(runs[0][0]) - float(want)) <= 1e-5 * abs(float(want))
    w = g0 + oo.grad
    d = (runs[0][1] - w).abs()
    tol = 8 * EPS * (w.abs() + oo.grad.abs()) + 1e-30
    assert bool((d <= tol).all()), float((d / tol).max())
    # rho == 0: zero loss, gradient untouched
    g = g0.clone()
    loss = _ns().sparsity_loss(o, z, u, torch.zeros(1, device=cuda_device), g)
    assert float(loss) == 0.0 and torch.equal(g, g0)


def _params(N, K, dev, seed, quantised):
    g = torch.Generator().manual_seed(seed)
    o = ((torch.randint(0, 9, (N,), generator=g).float() - 4.0) * 0.5 if quantised else torch.randn(N, generator=g))
    means = torch.randn(N, 3, generator=g)
    means[:, 0] = torch.arange(N, dtype=torch.float32)  # the row's identity
    P = {"means": means, "sh0": torch.randn(N, 1, 3, generator=g), "shN": torch.randn(N, K, 3, generator=g),
         "scaling_raw": torch.randn(N, 3, generator=g), "rotation_raw": torch.randn(N, 4, generator=g),
         "opacity_raw": o[:, None]}
    P = {k: v.to(dev).contiguous() for k, v in P.items()}
    return P


def _strategy(native, kind, P, dev):
    sp, training, mc, adc = _mods(native)
    Q = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    opt = training.FusedAdam(Q)
    g = torch.Generator(device=dev).manual_seed(1)
    for k in R.GROUPS:
        opt.exp_avg[k].copy_(torch.randn(Q[k].shape, device=dev, generator=g))
        opt.exp_avg_sq[k].copy_(torch.rand(Q[k].shape, device=dev, generator=g))
        opt.steps[k] = 7
    if kind == "mcmc":
        return mc.MCMC(Q, opt, mc.MCMCConfig(max_cap=P["means"].shape[0] + 100)), Q, opt
    return adc.DefaultStrategy(Q, opt), Q, opt


@pytest.mark.parametrize("quantised", [False, True])
@pytest.mark.parametrize("K", [0, 15])
@pytest.mark.parametrize("kind", ["mcmc", "default"])
def test_prune_removes_exactly_n_prune(native, cuda_device, kind, K, quantised):
    N = 200_003
    P = _params(N, K, cuda_device, seed=K + 3 * quantised, quantised=quantised)
    strat, Q, opt = _strategy(native, kind, P, cuda_device)
    sp = _mods(native)[0].ADMMSparsity(_mods(native)[0].SparsityConfig(sparsify_steps=10, start_iteration=5))
    M1 = {k: opt.exp_avg[k].clone() for k in R.GROUPS}
    M2 = {k: opt.exp_avg_sq[k].clone() for k in R.GROUPS}
    n_prune = sp.prune(strat)
    assert n_prune == R.prune_index(0.6, N) and strat.n == N - n_prune
    kept = Q["means"].detach()[:, 0].long()
    assert bool((kept[1:] > kept[:-1]).all())  # in order
    s = torch.sigmoid(P["opacity_raw"].flatten())
    want = ~R.prune_mask(P["opacity_raw"], 0.6)
    got = torch.zeros(N, dtype=torch.bool, device=cuda_device)
    got[kept] = True
    v = torch.sort(s).values[n_prune - 1]
    assert torch.equal(got[s != v], want[s != v])  # equal except rows tied at the boundary
    assert int(got[s == v].sum()) == int(want[s == v].sum())
    if quantised:  # ties: the first in index order are removed
        tied = (s == v).nonzero().flatten()
        n_tie_pruned = n_prune - int((s < v).sum())
        assert not bool(got[tied[:n_tie_pruned]].any()) and bool(got[tied[n_tie_pruned:]].all())
    for k in R.GROUPS:
        assert torch.equal(Q[k].detach(), P[k].index_select(0, kept)), k
        assert torch.equal(opt.exp_avg[k], M1[k].index_select(0, kept)), k
        assert torch.equal(opt.exp_avg_sq[k], M2[k].index_select(0, kept)), k
        assert opt.steps[k] == 7
    if kind == "default":
        assert strat.densification_info.shape == (2, N - n_prune) and not bool(strat.densification_info.any())


def test_phase_does_not_synchronise(native, cuda_device):
    """Loss iterations, an update iteration and the prune iteration, as the training step orders them."""
    sp_mod, training, mc, adc = _mods(native)
    P = _params(300_001, 15, cuda_device, seed=4, quantised=False)
    for kind in ("mcmc", "default"):
        strat, Q, opt = _strategy(native, kind, P, cuda_device)
        sp = sp_mod.ADMMSparsity(sp_mod.SparsityConfig(sparsify_steps=8, start_iteration=10, update_every=4))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for it in range(10, 19):
                for k in R.GROUPS:
                    Q[k].grad = torch.ones_like(Q[k])
                with torch.no_grad():
                    sp.loss_step(Q["opacity_raw"], it)
                sp.after_step(strat, it)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert sp.done and strat.n == 300_001 - R.prune_index(0.6, 300_001), kind


def _fastgs_problem(native, dev):
    fg = importlib.import_module(native.__name__ + ".fastgs")
    inp = scenes.fastgs_inputs(scenes.scene_small(N=3000, width=160, height=112, sh_degree=3, seed=6, view=2))
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw",
             "opacity_raw": "opacities_raw", "sh0": "sh0", "shN": "shN"}
    raw = {k: torch.from_numpy(inp[v]).to(dev).contiguous() for k, v in names.items()}
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(dev), active_sh_bases=1,
                          width=inp["width"], height=inp["height"], focal_x=inp["fx"], focal_y=inp["fy"],
                          center_x=inp["cx"], center_y=inp["cy"], near_plane=inp["near_plane"],
                          far_plane=inp["far_plane"])
    g = torch.Generator(device=dev).manual_seed(2)
    target = torch.rand((3, inp["height"], inp["width"]), device=dev, generator=g)
    return s, torch.from_numpy(inp["w2c"]).to(dev), raw, target


def _gsplat_problem(native, dev):
    sc = scenes.scene_b(N=6000, width=160, height=112, view=2, scale_mul=2.0)
    t = to_dev(sc, dev)
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    raw = {k: v.detach().clone() for k, v in raw.items()}
    g = torch.Generator(device=dev).manual_seed(3)
    target = torch.rand((3, 112, 160), device=dev, generator=g)
    return t, raw, target


def _make_strategy(native, kind, raw, refine: bool):
    sp_mod, training, mc, adc = _mods(native)
    Q = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    opt = training.FusedAdam(Q, training.AdamConfig(iterations=20))
    n = raw["means"].shape[0]
    if kind == "mcmc":
        cfg = mc.MCMCConfig(start_refine=5 if refine else 10 ** 6, refine_every=10, stop_refine=15,
                            max_cap=int(1.1 * n))
        return mc.MCMC(Q, opt, cfg), Q
    # without refines, stop_refine lies beyond the run too: reaching it re-captures the graphed step
    cfg = adc.DefaultConfig(start_refine=5 if refine else 10 ** 6, refine_every=10,
                            stop_refine=15 if refine else 10 ** 6, reset_every=10 ** 6)
    return adc.DefaultStrategy(Q, opt, cfg), Q


def _runner(native, path, prob, Q, strat, sp, graphed=False):
    training = _mods(native)[1]
    if path == "gsplat":
        t, _, target = prob
        if graphed:
            g = training.GraphedTrainStep(Q, 0, 160, 112, strategy=strat, sparsity=sp)
            return g, lambda: g(t["viewmats"], t["Ks"], target, t["background"])
        e = training.TrainStep(Q, 0, 160, 112, optimizer=strat.optimizer, strategy=strat, sparsity=sp)
        return e, lambda: e(t["viewmats"], t["Ks"], target, t["background"])
    settings, w2c, _, target = prob
    if graphed:
        g = training.GraphedFastGsTrainStep(Q, 0, settings, strategy=strat, sparsity=sp, capacity_slack=2.0)
        return g, lambda: g(w2c, settings.cam_position, target)
    e = training.FastGsTrainStep(Q, 0, settings.width, settings.height, optimizer=strat.optimizer, strategy=strat,
                                 sparsity=sp)
    return e, lambda: e(w2c, settings, target)


def _problem(native, path, dev):
    if path == "gsplat":
        prob = _gsplat_problem(native, dev)
        return prob, prob[1]
    prob = _fastgs_problem(native, dev)
    return prob, prob[2]


@pytest.mark.parametrize("kind", ["mcmc", "default"])
@pytest.mark.parametrize("path", ["gsplat", "fastgs"])
def test_short_schedule_matches_restatement(native, cuda_device, path, kind):
    """Base 20 (a refine at 10), 120 sparsity steps: loss from 20, updates at 70 and 120, prune at 140.  Every
    initialisation, update, loss, gradient and the prune go through the restatement from the state the step had."""
    sp_mod = _mods(native)[0]
    prob, raw = _problem(native, path, cuda_device)
    strat, Q = _make_strategy(native, kind, raw, refine=True)
    sp = sp_mod.ADMMSparsity(sp_mod.SparsityConfig(sparsify_steps=120, start_iteration=20))
    _, run = _runner(native, path, prob, Q, strat, sp)
    post_at, updates, losses, prunes = [], [], [], []
    post_backward = strat.post_backward

    def post(it, *a):
        post_at.append(it)
        return post_backward(it, *a)
    strat.post_backward = post
    init, upd, add, remove = sp.initialize, sp.update_state, sp.add_loss_gradient, strat.remove_lowest_opacity

    def initialize(o):
        init(o)
        wz, wu = R.initialize(o.detach(), 0.6)
        updates.append(torch.equal(sp.z, wz.flatten()) and torch.equal(sp.u, wu.flatten()))

    def update_state(o):
        wz, wu = R.update_state(o.detach(), sp.z.view(-1, 1).clone(), sp.u.view(-1, 1).clone(), 0.6)
        upd(o)
        updates.append(torch.equal(sp.z, wz.flatten()) and torch.equal(sp.u, wu.flatten()))

    def add_loss_gradient(o):
        g0, z, u = o.grad.clone(), sp.z.clone(), sp.u.clone()
        loss = add(o)
        with torch.enable_grad():  # the step calls this under no_grad
            oo = o.detach().clone().requires_grad_(True)
            want = R.loss(oo, z.view(-1, 1), u.view(-1, 1), 5e-4)
            want.backward()
        e = float(((o.grad - g0) - oo.grad).abs().max() / oo.grad.abs().max().clamp_min(1e-30))
        losses.append((abs(float(loss) - float(want)) / max(1e-30, abs(float(want))), e))
        return loss

    def remove_lowest_opacity(n_prune):
        S = {k: Q[k].detach().clone() for k in R.GROUPS}
        opt = strat.optimizer
        M1 = {k: opt.exp_avg[k].clone() for k in R.GROUPS}
        M2 = {k: opt.exp_avg_sq[k].clone() for k in R.GROUPS}
        remove(n_prune)
        mask = R.prune_mask(S["opacity_raw"], 0.6)
        WP, WM1, WM2 = R.remove_gaussians(S, M1, M2, mask)
        s = torch.sigmoid(S["opacity_raw"].flatten())
        v = torch.sort(s).values[n_prune - 1]
        if int((s == v).sum()) == 1:  # no tie at the boundary: the kept set is determined
            prunes.append(all(torch.equal(Q[k].detach(), WP[k]) and torch.equal(opt.exp_avg[k], WM1[k])
                              and torch.equal(opt.exp_avg_sq[k], WM2[k]) for k in R.GROUPS))
        else:
            prunes.append(all(Q[k].shape == WP[k].shape for k in R.GROUPS))
    sp.initialize, sp.update_state, sp.add_loss_gradient = initialize, update_state, add_loss_gradient
    strat.remove_lowest_opacity = remove_lowest_opacity
    ns = []
    for it in range(1, 146):
        ns.append(strat.n)
        run()
    print(path, kind, "N", ns[0], "->", ns[19], "->", strat.n, "worst loss / gradient", max(losses))
    assert post_at == list(range(1, 21))
    assert updates == [True, True, True] and len(losses) == 120 and prunes == [True]
    assert all(l <= 1e-5 and e <= 1e-5 for l, e in losses)
    assert strat.n == ns[139] - R.prune_index(0.6, ns[139]) and sp.done
    assert ns[139] == ns[20]  # no refine in the phase


def test_refine_at_the_base_iteration_raises(native, cuda_device):
    sp_mod, training, mc, adc = _mods(native)
    prob, raw = _problem(native, "fastgs", cuda_device)
    with torch.no_grad():
        raw["opacity_raw"].view(-1)[::40] = -7.0  # pruned by the refine at 20
    Q = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    opt = training.FusedAdam(Q)
    strat = adc.DefaultStrategy(Q, opt, adc.DefaultConfig(start_refine=10, refine_every=20, grad_threshold=1e9))
    sp = sp_mod.ADMMSparsity(sp_mod.SparsityConfig(sparsify_steps=10, start_iteration=20))
    _, run = _runner(native, "fastgs", prob, Q, strat, sp)
    for _ in range(20):
        run()
    assert strat.n < raw["means"].shape[0]
    with pytest.raises(ValueError, match="base iteration"):
        run()


@pytest.mark.parametrize("kind", ["mcmc", "default"])
@pytest.mark.parametrize("path", ["gsplat", "fastgs"])
def test_graphed_equals_eager(native, cuda_device, path, kind):
    """The graphed step against the eager one from the same seeds, base 20, 120 steps, and two iterations after the
    prune.  Captures: the first, one at phase entry (20) and one after the prune (141) -- no others.  After the base
    iteration neither step runs post_backward, so MCMC injects no noise: not in the re-capture at 141 either."""
    sp_mod = _mods(native)[0]
    prob, raw = _problem(native, path, cuda_device)
    runs = []
    for graphed in (False, True, False):  # the second eager run is the floor of run-to-run differences
        strat, Q = _make_strategy(native, kind, raw, refine=False)
        sp = sp_mod.ADMMSparsity(sp_mod.SparsityConfig(sparsify_steps=120, start_iteration=20))
        step, run = _runner(native, path, prob, Q, strat, sp, graphed)
        runs.append((strat, Q, step, run, [], []))
    _, _, g, _, _, captures_at = runs[1]
    for it in range(1, 143):
        if it == 141 and kind == "mcmc":
            noise = [r[0].last_noise for r in runs]
        for strat, Q, step, run, losses, caps in runs:
            torch.manual_seed(1000 + it)
            c = getattr(step, "captures", 0)
            losses.append(float(run()))
            if getattr(step, "captures", 0) != c:
                caps.append(it)
    (sa, A, _, _, la, _), (sb, B, _, _, lb, _), (sc, C, _, _, lc, _) = runs
    print(path, kind, "captures at", captures_at, "N", sa.n)
    assert captures_at == [1, 20, 141] and g.captures == 3
    if kind == "mcmc":
        assert all(n is not None and r[0].last_noise is n for r, n in zip(runs, noise))
    assert sa.n == sb.n == sc.n == 3000 - R.prune_index(0.6, 3000) if path == "fastgs" else sa.n == sb.n
    for a, b, c in zip(la, lb, lc):
        assert abs(a - b) <= max(1e-3 * max(1.0, abs(a)), 5 * abs(a - c))
    rel = lambda X, Y: float((X - Y).abs().max() / X.abs().max().clamp_min(1e-12))
    for k in R.GROUPS:
        if A[k].numel():
            e, floor = rel(A[k].detach(), B[k].detach()), rel(A[k].detach(), C[k].detach())
            print(f"  {k}: graphed vs eager {e:.2e} (eager vs eager {floor:.2e})")
            assert e < max(1e-3, 5 * floor), k
    assert sa.optimizer.steps == sb.optimizer.steps
