"""GPU: the default densification strategy (adaptive density control) -- classify and apply against the torch
restatement (tests/adc_restatement.py), the reset kernel, the iterations that must not synchronise, and training on the
fastgs path (eager and graphed) and the 3DGUT path against the restatement fed the strategy's own state and normals.

Bitwise equality everywhere except the means of split copies: the restatement forms the offset R(q) (s * z) with
torch's einsum (a batched matrix product whose reduction order is cuBLAS's) and F.normalize, the kernel with a
fixed-order sum and sqrtf.  Each of R's entries may differ by a few ulp of 1 and each of the sum's three products is
rounded differently, so an offset component may differ by a few ulp of A = sum_j |R_ij| s_j |z_j|, and the added mean
by half an ulp of the result: the bound used is 16 eps (|result| + 2A), eps = 2^-23."""
import importlib

import pytest
import torch

import adc_restatement as R
import scenes
from parity import to_dev

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -23


def _adc(native):
    return importlib.import_module(native.__name__ + ".adc")


def _ns():
    return torch.ops.gsplat_b200


def _params(N, K, dev, case, seed=0):
    """Raw parameters whose every compared quantity keeps a clear margin from its threshold (defaults, scene scale 1):
    max scale 0.0024-0.004 (small), 0.024-0.04 (large, copies 0.015-0.025) or 0.24-0.4 (huge, copies 0.15-0.25);
    gradient signal <= 1e-4 (low) or >= 5e-4 (high); opacity >= 0.047, <= 0.0025 (dead) or 0.007-0.009 (faint: its
    revised split copies fall to 0.0035-0.0045); |q|^2 >= 1e-2 or <= 1e-8 / 25."""
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g)
    size = torch.randint(0, 2, (N,), generator=g)  # 0 small, 1 large, 2 huge
    high = u(N) < 0.1
    dead = torch.zeros(N, dtype=torch.bool)
    faint = torch.zeros(N, dtype=torch.bool)
    bad_rot = torch.zeros(N, dtype=torch.bool)
    if case == "none":
        high[:] = False
    elif case == "all_pruned":
        dead[:] = True
    elif case == "only_dup":
        size[:] = 0
    elif case == "only_split":
        size[:] = 1
    else:  # mixed
        size[u(N) < 0.05] = 2
        dead = u(N) < 0.02
        faint = (u(N) < 0.03) & ~dead
        bad_rot = u(N) < 0.01
    base = torch.tensor([0.004, 0.04, 0.4])[size]
    scaling = torch.log(base[:, None] * (0.6 + 0.4 * u(N, 3)))
    count = torch.randint(0, 5, (N,), generator=g).float()
    sig = torch.where(high, 5e-4 + 1e-2 * u(N), 1e-4 * u(N))
    info = torch.stack([count, sig * count.clamp_min(1.0)])
    o = torch.logit(0.05 + 0.9 * u(N))
    o[dead] = -6.0 - 3.0 * u(int(dead.sum()))
    o[faint] = torch.logit(0.007 + 0.002 * u(int(faint.sum())))
    q = torch.randn(N, 4, generator=g)
    q = q / q.norm(dim=-1, keepdim=True) * (0.1 + u(N, 1))
    q[bad_rot] *= 1e-5
    P = {"means": torch.randn(N, 3, generator=g), "sh0": torch.randn(N, 1, 3, generator=g),
         "shN": torch.randn(N, K, 3, generator=g), "scaling_raw": scaling, "rotation_raw": q,
         "opacity_raw": o[:, None]}
    M1 = {k: torch.randn(v.shape, generator=g) for k, v in P.items()}
    M2 = {k: torch.rand(v.shape, generator=g) for k, v in P.items()}
    dv = lambda d: {k: v.to(dev).contiguous() for k, v in d.items()}
    return dv(P), dv(M1), dv(M2), info.to(dev).contiguous()


def _assert_rows_equal(got, want, n_plain, what):
    """Bitwise, except the means of rows >= n_plain (split copies), within the bound of the module docstring."""
    P, M1, M2, A = got
    WP, WM1, WM2 = want
    for k in R.GROUPS:
        assert P[k].shape == WP[k].shape, (what, k)
        if k == "means":
            assert torch.equal(P[k][:n_plain], WP[k][:n_plain]), (what, k)
            d = (P[k][n_plain:] - WP[k][n_plain:]).abs()
            tol = 16 * EPS * (WP[k][n_plain:].abs() + 2 * A)
            assert bool((d <= tol).all()), (what, float((d / tol.clamp_min(1e-30)).max()))
        else:
            assert torch.equal(P[k], WP[k]), (what, k)
        assert torch.equal(M1[k], WM1[k]) and torch.equal(M2[k], WM2[k]), (what, k)


def _offset_magnitude(native, P, M1, M2, info, it, cfg, z):
    """A = sum_j |R_ij| s_j |z_j| per output row: the restatement with zero means, |R| and |z|."""
    Q = dict(P)
    Q["means"] = torch.zeros_like(P["means"])
    out = R.refine(Q, M1, M2, info, it, cfg, 1.0, lambda q: native.quats_to_rotmats(q).abs(),
                   z.abs() if z is not None else None)
    return out[0]["means"]


@pytest.mark.parametrize("K", [0, 15])
@pytest.mark.parametrize("N", [50_000, 3_000_017])
@pytest.mark.parametrize("case", ["none", "all_pruned", "only_dup", "only_split", "mixed", "mixed_revised"])
def test_classify_apply_match_restatement(native, cuda_device, case, N, K):
    adc = _adc(native)
    revised = case == "mixed_revised"
    it = 40 if revised else 20  # 40 > reset_every 30: too-big rows are pruned as well
    P, M1, M2, info = _params(N, K, cuda_device, case.replace("_revised", ""), seed=N + K)
    cfg = adc.DefaultConfig(reset_every=30, revised_opacity=revised)
    counts, ws = _ns().adc_classify(info, P["scaling_raw"], P["rotation_raw"], P["opacity_raw"], cfg.grad_threshold,
                                    cfg.grow_scale3d, cfg.prune_scale3d, 1.0, cfg.prune_opacity, it > cfg.reset_every,
                                    revised)
    c = counts.tolist()
    torch.manual_seed(N)
    z = torch.randn((2, c[1], 3), device=cuda_device) if c[1] else None
    gp, g1, g2, ginfo = _ns().adc_apply([P[k] for k in R.GROUPS], [M1[k] for k in R.GROUPS], [M2[k] for k in R.GROUPS],
                                        ws, counts, c[1], c[3], z, revised)
    WP, WM1, WM2, wc, _ = R.refine(P, M1, M2, info, it, cfg, 1.0, native.quats_to_rotmats, z)
    print(case, N, K, "counts", c)
    assert tuple(c[:4]) == wc
    assert c[4] + c[5] + 2 * c[6] == c[3] and c[7] == 0
    expect = {"none": lambda: c[:3] == [0, 0, 0], "all_pruned": lambda: c[3] == 0,
              "only_dup": lambda: c[0] > 0 and c[1] == 0 and c[2] == 0,
              "only_split": lambda: c[1] > 0 and c[0] == 0 and c[2] == 0,
              "mixed": lambda: min(c[:3]) > 0, "mixed_revised": lambda: min(c[:3]) > 0}[case]
    assert expect()
    A = _offset_magnitude(native, P, M1, M2, info, it, cfg, z)[c[4] + c[5]:]
    _assert_rows_equal(({k: v for k, v in zip(R.GROUPS, gp)}, dict(zip(R.GROUPS, g1)), dict(zip(R.GROUPS, g2)), A),
                       (WP, WM1, WM2), c[4] + c[5], case)
    assert ginfo.shape == (2, c[3]) and not bool(ginfo.any())


def test_reset_opacity_matches_restatement(native, cuda_device):
    adc = _adc(native)
    P, M1, M2, _ = _params(1_000_003, 0, cuda_device, "mixed", seed=4)
    P["opacity_raw"][::7] = float("nan")
    cfg = adc.DefaultConfig()
    WP, WM1, WM2 = dict(P), dict(M1), dict(M2)
    R.reset_opacity(WP, WM1, WM2, cfg)
    o, m1, m2 = P["opacity_raw"].clone(), M1["opacity_raw"].clone(), M2["opacity_raw"].clone()
    _ns().adc_reset_opacity(o, m1, m2, cfg.prune_opacity)
    assert torch.equal(o.nan_to_num(7.0), WP["opacity_raw"].nan_to_num(7.0))
    assert not bool(m1.any()) and not bool(m2.any())


def _strategy_for(native, P, cfg, M1=None, M2=None):
    adc, training = _adc(native), importlib.import_module(native.__name__ + ".training")
    P = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    opt = training.FusedAdam(P)
    if M1 is not None:
        for k in R.GROUPS:
            opt.exp_avg[k].copy_(M1[k])
            opt.exp_avg_sq[k].copy_(M2[k])
    return adc.DefaultStrategy(P, opt, cfg), P, opt


def test_non_refine_and_reset_iterations_do_not_synchronise(native, cuda_device):
    adc = _adc(native)
    P, M1, M2, info = _params(200_000, 15, cuda_device, "mixed", seed=8)
    cfg = adc.DefaultConfig(start_refine=10, refine_every=10, reset_every=30, pause_refine_after_reset=5,
                            stop_refine=55)
    strat, Q, opt = _strategy_for(native, P, cfg, M1, M2)
    strat.densification_info.copy_(info)
    for k in R.GROUPS:
        Q[k].grad = torch.ones_like(Q[k])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        skips = [strat.post_backward(it) for it in (11, 29, 30, 31)]  # 30 resets only (paused refine)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert skips == [(), (), ("opacity_raw",), ()]
    assert strat.refines == 0 and strat.resets == 1 and Q["opacity_raw"].grad is None and Q["means"].grad is not None
    WP, WM1, WM2 = dict(P), dict(M1), dict(M2)
    R.reset_opacity(WP, WM1, WM2, cfg)
    assert torch.equal(Q["opacity_raw"].detach(), WP["opacity_raw"]) and not bool(opt.exp_avg["opacity_raw"].any())
    assert torch.equal(strat.densification_info, info)  # only a refine consumes the statistics


def _fastgs_problem(native, dev):
    fg = importlib.import_module(native.__name__ + ".fastgs")
    inp = scenes.fastgs_inputs(scenes.scene_small(N=3000, width=160, height=112, sh_degree=3, seed=6, view=2))
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw",
             "opacity_raw": "opacities_raw", "sh0": "sh0", "shN": "shN"}
    raw = {k: torch.from_numpy(inp[v]).to(dev).contiguous() for k, v in names.items()}
    with torch.no_grad():
        raw["opacity_raw"].view(-1)[::40] = -7.0  # rows for the first prune
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(dev), active_sh_bases=1,
                          width=inp["width"], height=inp["height"], focal_x=inp["fx"], focal_y=inp["fy"],
                          center_x=inp["cx"], center_y=inp["cy"], near_plane=inp["near_plane"],
                          far_plane=inp["far_plane"])
    g = torch.Generator(device=dev).manual_seed(2)
    target = torch.rand((3, inp["height"], inp["width"]), device=dev, generator=g)
    return s, torch.from_numpy(inp["w2c"]).to(dev), raw, target


def _thresholds(native, dev, settings, w2c, raw, target, its=10):
    """A gradient threshold in a wide gap of the signal after `its` eager iterations near its 85th percentile, and a
    grow scale at the median maximum scale, so that refines both duplicate and split."""
    adc, training = _adc(native), importlib.import_module(native.__name__ + ".training")
    strat, P, opt = _strategy_for(native, raw, adc.DefaultConfig(start_refine=10 ** 6))
    step = training.FastGsTrainStep(P, 0, settings.width, settings.height, optimizer=opt, strategy=strat)
    for _ in range(its):
        step(w2c, settings, target)
    info = strat.densification_info
    g = torch.sort((info[1] / info[0].clamp_min(1.0))).values
    g = g[g > 0]
    k0 = int(0.85 * g.numel())
    k = next(k for k in range(k0, g.numel() - 1) if g[k + 1] > g[k] * 1.01)
    smax = torch.exp(raw["scaling_raw"]).max(-1).values
    return float((g[k] + g[k + 1]) / 2), float(smax.median())


def test_fastgs_training_matches_restatement(native, cuda_device):
    """60 eager iterations, refine every 10 from 20, reset at 30, stop at 55.  At every refine the state before it
    (parameters, moments, statistics) goes through the restatement with the strategy's own normals: counts, rows and
    moments must match, and so must N and every group's Adam step count over the run."""
    adc, training = _adc(native), importlib.import_module(native.__name__ + ".training")
    settings, w2c, raw, target = _fastgs_problem(native, cuda_device)
    thr, grow = _thresholds(native, cuda_device, settings, w2c, raw, target)
    cfg = adc.DefaultConfig(start_refine=10, refine_every=10, reset_every=30, stop_refine=55, grad_threshold=thr,
                            grow_scale3d=grow, prune_scale3d=4 * grow)
    strat, P, opt = _strategy_for(native, raw, cfg)
    step = training.FastGsTrainStep(P, 0, settings.width, settings.height, optimizer=opt, strategy=strat)
    seen = {}

    def snapshot():
        seen["P"] = {k: P[k].detach().clone() for k in R.GROUPS}
        seen["M1"] = {k: opt.exp_avg[k].clone() for k in R.GROUPS}
        seen["M2"] = {k: opt.exp_avg_sq[k].clone() for k in R.GROUPS}
        seen["info"] = strat.densification_info.clone()
        return None
    strat.regularize = lambda params=None: snapshot()
    rs = R.Strategy(raw, opt.exp_avg, opt.exp_avg_sq, cfg, 1.0, native.quats_to_rotmats)
    ns, changed_at = [], []
    for it in range(1, 61):
        refines = strat.refines
        step(w2c, settings, target)
        rs.P, rs.M1, rs.M2, rs.info = seen["P"], seen["M1"], seen["M2"], seen["info"]
        skip = rs.post_backward(it, strat.last_z if strat.refines > refines else None)
        rs.adam_bookkeeping(skip)
        if strat.refines > refines:
            assert strat.last_counts == rs.counts, it
            assert strat.replaced == (skip == R.GROUPS), it
        if strat.replaced:  # Adam skipped every group: the state is the refine's (and the reset's) output
            changed_at.append((it, rs.counts))
            n_plain = rs.counts[3] - 2 * strat.last_kept_split
            A = _offset_magnitude(native, seen["P"], seen["M1"], seen["M2"], seen["info"], it, cfg, strat.last_z)
            _assert_rows_equal(({k: P[k].detach() for k in R.GROUPS}, opt.exp_avg, opt.exp_avg_sq, A[n_plain:]),
                               (rs.P, rs.M1, rs.M2), n_plain, it)
            assert strat.densification_info.shape == (2, strat.n) and P["means"].grad is None
        ns.append(strat.n)
        assert strat.n == rs.P["means"].shape[0]
        assert opt.steps == rs.steps, it
    print("refines that changed the set (iteration, counts):", changed_at, "N:", ns[0], "->", ns[-1])
    assert len(changed_at) >= 3
    assert any(c[0] > 0 for _, c in changed_at) and any(c[1] > 0 for _, c in changed_at)
    assert any(c[2] > 0 for _, c in changed_at)
    assert strat.densification_info.numel() == 0 and strat.resets == 1
    assert opt.steps["means"] == 60 - len(changed_at)


def test_graphed_fastgs_with_strategy_equals_eager(native, cuda_device):
    """The graphed step against the eager one from the same seed: same N after every iteration, losses and parameters
    close.  Re-captures follow the refine at 20, which replaces the tensors, and stop_refine (35) only; the reset-only
    iteration (30, refining paused after the reset) keeps the graphs, and the warm-up moves nothing.  One refine only:
    the two runs' statistics differ in the last bits (the backward's atomics), and once a refine has grown the set a
    row may sit within those bits of the gradient threshold at the next one."""
    adc, training = _adc(native), importlib.import_module(native.__name__ + ".training")
    settings, w2c, raw, target = _fastgs_problem(native, cuda_device)
    thr, grow = _thresholds(native, cuda_device, settings, w2c, raw, target)
    cfg = adc.DefaultConfig(start_refine=10, refine_every=10, reset_every=30, pause_refine_after_reset=5,
                            stop_refine=35, grad_threshold=thr, grow_scale3d=grow, prune_scale3d=4 * grow)
    sa, A, _ = _strategy_for(native, raw, cfg)
    sb, B, _ = _strategy_for(native, raw, cfg)
    sc, C, _ = _strategy_for(native, raw, cfg)  # a second eager run: the floor of run-to-run differences
    eager = training.FastGsTrainStep(A, 0, settings.width, settings.height, optimizer=sa.optimizer, strategy=sa)
    eager_c = training.FastGsTrainStep(C, 0, settings.width, settings.height, optimizer=sc.optimizer, strategy=sc)
    # the reset at 30 halves the instances and they grow back past the re-capture at 36: room for that
    graphed = training.GraphedFastGsTrainStep(B, 0, settings, strategy=sb, capacity_slack=3.0)
    before = {k: v.detach().clone() for k, v in B.items()}
    graphed.capture(w2c, settings.cam_position, target)
    for k in B:
        assert torch.equal(B[k].detach(), before[k]), k
    assert not bool(sb.densification_info.any())  # the warm-up's statistics were undone
    captures_at, want_at, la, lb, lc = [], [], [], [], []
    for it in range(1, 61):
        torch.manual_seed(1000 + it)
        la.append(float(eager(w2c, settings, target)))
        if sa.replaced or it == cfg.stop_refine:
            want_at.append(it + 1)
        torch.manual_seed(1000 + it)
        c = graphed.captures
        lb.append(float(graphed(w2c, settings.cam_position, target)))
        if graphed.captures != c:
            captures_at.append(it)
        torch.manual_seed(1000 + it)
        lc.append(float(eager_c(w2c, settings, target)))
        assert not graphed.overflowed(), it
        assert sa.n == sb.n, it
    print("re-captured at", captures_at, "N", sa.n)
    assert 30 not in want_at and 31 not in captures_at
    assert captures_at == want_at == [21, 36]
    # the backward's atomics make two eager runs differ too, and densification compounds the differences
    for a, b, c in zip(la, lb, lc):
        assert abs(a - b) <= max(1e-3 * max(1.0, abs(a)), 5 * abs(a - c))
    assert sa.optimizer.steps == sb.optimizer.steps
    rel = lambda X, Y: float((X - Y).abs().max() / X.abs().max().clamp_min(1e-12))
    for k in R.GROUPS:
        if A[k].numel():
            floor = rel(A[k].detach(), C[k].detach()) if C[k].shape == A[k].shape else float("inf")
            e = rel(A[k].detach(), B[k].detach())
            print(f"  {k}: graphed vs eager {e:.2e} (eager vs eager {floor:.2e})")
            assert e < max(1e-3, 5 * floor), k


def test_3dgut_training_prunes_and_resets_without_growth(native, cuda_device):
    """TrainStep (3DGUT) produces no statistics: refines never grow, but the faint rows are pruned at the first refine
    and the opacities are reset at 30, matching the restatement."""
    adc, training = _adc(native), importlib.import_module(native.__name__ + ".training")
    sc = scenes.scene_b(N=6000, width=160, height=112, view=2, scale_mul=2.0)
    t = to_dev(sc, cuda_device)
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    raw = {k: v.detach().clone() for k, v in raw.items()}
    with torch.no_grad():
        raw["opacity_raw"].view(-1)[::40] = -7.0
    g = torch.Generator(device=cuda_device).manual_seed(3)
    target = torch.rand((3, 112, 160), device=cuda_device, generator=g)
    cfg = adc.DefaultConfig(start_refine=10, refine_every=10, reset_every=30, stop_refine=55, grad_threshold=0.0,
                            prune_scale3d=1e3)
    strat, P, opt = _strategy_for(native, raw, cfg)
    step = training.TrainStep(P, 0, 160, 112, optimizer=opt, strategy=strat)
    counts = []
    for it in range(1, 61):
        refines = strat.refines
        step(t["viewmats"], t["Ks"], target, t["background"])
        if strat.refines > refines:
            counts.append(strat.last_counts)
        if it == 30:  # the reset's iteration skips the opacity group's Adam step
            assert float(P["opacity_raw"].detach().max()) <= R.reset_threshold(cfg.prune_opacity)
    print("3DGUT refines:", counts)
    assert all(c[0] == 0 and c[1] == 0 for c in counts)
    assert counts[0][2] >= len(range(0, 6000, 40)) and strat.n == 6000 - sum(c[2] for c in counts)
    assert strat.resets == 1
