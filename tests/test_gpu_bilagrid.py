"""GPU: the bilateral grid (SURVEY.md 8 f5) -- slice forward / backward and the TV loss against the float64
restatement (tests/bilagrid_restatement.py), the Python mirror of the reference's BilateralGrid, and the training
iteration with the grid on both rasterizer paths, eager and graphed."""
import importlib

import pytest
import torch

import bilagrid_restatement as R
import scenes
from parity import rel, to_dev

pytestmark = pytest.mark.gpu


def _mods(native):
    return (importlib.import_module(native.__name__ + ".bilateral"), importlib.import_module(native.__name__ + ".training"))


def _grids(n, X, Y, L, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return (R.identity_grids(n, X, Y, L) + 0.2 * torch.randn(n, 12, L, Y, X, generator=g, dtype=torch.float64)).float().to(dev)


@pytest.mark.parametrize("h,w", [(1080, 1920), (97, 173), (23, 40)])
@pytest.mark.parametrize("chw,X,Y,L", [(False, 16, 16, 8), (True, 12, 9, 4)])
def test_slice_vs_float64_restatement(native, cuda_device, h, w, chw, X, Y, L):
    """Inputs in [-0.2, 1.2], random non-identity grids, image 3 of 5; 23x40 has grid cells smaller than a CTA's pixel
    block.  The other images' grids get exactly zero gradient."""
    ns = torch.ops.gsplat_b200
    grids = _grids(5, X, Y, L, h + w, cuda_device)
    g = torch.Generator().manual_seed(h * w)
    img = (torch.rand(h, w, 3, generator=g) * 1.4 - 0.2)
    v_out = torch.randn(h, w, 3, generator=g)
    idx = torch.tensor([3], dtype=torch.int32, device=cuda_device)
    dev_img = (img.permute(2, 0, 1) if chw else img).contiguous().to(cuda_device)
    dev_v = (v_out.permute(2, 0, 1) if chw else v_out).contiguous().to(cuda_device)
    out = ns.bilagrid_slice(grids, dev_img, idx, chw)
    v_grids = torch.zeros_like(grids)
    v_img = ns.bilagrid_slice_backward(grids, dev_img, idx, dev_v, v_grids, chw)
    torch.cuda.synchronize()
    if chw:
        out, v_img = out.permute(1, 2, 0), v_img.permute(1, 2, 0)
    g3 = grids[3].double().cpu()
    want = R.slice_fwd(g3, img.double())
    want_vg, want_vi = R.slice_bwd(g3, img.double(), v_out.double())
    # the same restatement with float32 inputs rounded through float32 outputs: the error floor of a float32 kernel
    f32_err = float((want.float().double() - want).abs().max())
    err = float((out.double().cpu() - want).abs().max())
    e_vi, e_vg = rel(v_img.cpu(), want_vi), rel(v_grids[3].cpu(), want_vg)
    print(f"[{h}x{w} chw={chw} grid {X}x{Y}x{L}] fwd max|err| {err:.2e} (float32 rounding {f32_err:.1e}), "
          f"v_input rel_l2 {e_vi:.2e}, v_grid rel_l2 {e_vg:.2e}")
    assert err <= 1e-5
    assert e_vi <= 1e-5
    assert e_vg <= 1e-4
    others = torch.cat([v_grids[:3].flatten(), v_grids[4:].flatten()])
    assert int((others != 0).sum()) == 0


def test_slice_identity_reproduces_clamped_input(native, cuda_device):
    bil, _ = _mods(native)
    bg = bil.BilateralGrid(2, device=cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(0)
    img = torch.rand((3, 97, 173), device=cuda_device, generator=g) * 1.4 - 0.2
    out = bg.apply(img, 1)
    assert float((out - img.clamp(0, 1)).abs().max()) <= 1e-6


@pytest.mark.parametrize("N,X,Y,L", [(200, 16, 16, 8), (3, 12, 9, 4), (2, 5, 1, 3)])
def test_tv_vs_float64_restatement(native, cuda_device, N, X, Y, L):
    ns = torch.ops.gsplat_b200
    grids = _grids(N, X, Y, L, N, cuda_device)
    w = torch.tensor([2.5], device=cuda_device)
    loss, grad = ns.bilagrid_tv(grids, w, True)
    loss_only, _ = ns.bilagrid_tv(grids, None, False)
    want = R.tv_loss(grids.double().cpu())
    want_g = R.tv_grad(grids.double().cpu()) * 2.5
    e_l = abs(float(loss) - float(want)) / abs(float(want))
    e_g = rel(grad.cpu(), want_g)
    print(f"[N={N} {X}x{Y}x{L}] tv {float(loss):.8e} vs {float(want):.8e}: rel {e_l:.2e}; grad rel_l2 {e_g:.2e}")
    assert e_l <= 1e-6 and e_g <= 1e-6
    assert float(loss_only) == float(loss)  # deterministic
    ident = R.identity_grids(N, X, Y, L).float().to(cuda_device)
    assert float(ns.bilagrid_tv(ident, None, False)[0]) == 0.0


def test_python_mirror_autograd_matches_restatement(native, cuda_device):
    """BilateralGrid.apply ([C,H,W] and [1,C,H,W]) and tv_loss through autograd."""
    bil, _ = _mods(native)
    bg = bil.BilateralGrid(4, grid_X=12, grid_Y=9, grid_L=4, device=cuda_device)
    with torch.no_grad():
        bg.grids.copy_(_grids(4, 12, 9, 4, 7, cuda_device))
    g = torch.Generator().manual_seed(9)
    img = (torch.rand(3, 57, 81, generator=g) * 1.4 - 0.2)
    v = torch.randn(1, 3, 57, 81, generator=g)
    x = img[None].to(cuda_device).requires_grad_(True)
    out = bg.apply(x, 2)
    assert out.shape == (1, 3, 57, 81)
    ((out * v.to(cuda_device)).sum() + 3.0 * bg.tv_loss()).backward()
    wv_g, wv_i = R.slice_bwd(bg.grids.detach()[2].double().cpu(), img.permute(1, 2, 0).double(),
                             v[0].permute(1, 2, 0).double())
    want_g = R.tv_grad(bg.grids.detach().double().cpu()) * 3.0
    want_g[2] += wv_g
    assert rel(x.grad[0].permute(1, 2, 0).cpu(), wv_i) <= 1e-5
    assert rel(bg.grids.grad.cpu(), want_g) <= 1e-4


def _gsplat_setup(native, dev, W=320, H=192):
    sc = scenes.scene_b(N=8000, width=W, height=H, view=2, scale_mul=2.0)
    t = to_dev(sc, dev)
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    g = torch.Generator(device=dev).manual_seed(3)
    targets = [torch.rand((3, H, W), device=dev, generator=g) for _ in range(3)]
    return t, raw, targets


def _clone(raw):
    return {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}


def test_identity_grid_first_iteration_equals_no_grid_loss(native, cuda_device):
    """With identity grids the slice is the clamp, so the first loss equals the plain loss (TV = 0)."""
    bil, training = _mods(native)
    t, raw, tg = _gsplat_setup(native, cuda_device)
    a = training.TrainStep(_clone(raw), 3, 320, 192, optimizer=None)
    b = training.TrainStep(_clone(raw), 3, 320, 192, optimizer=None, bilateral_grid=bil.BilateralGrid(3, device=cuda_device))
    la = float(a(t["viewmats"], t["Ks"], tg[0], t["background"]))
    lb = float(b(t["viewmats"], t["Ks"], tg[0], t["background"], image_idx=1))
    print(f"gsplat path: no grid {la:.8f}, identity grid {lb:.8f}")
    assert abs(la - lb) <= 1e-6


def test_gsplat_training_with_grid_matches_autograd_composition(native, cuda_device):
    """Five iterations cycling the image: TrainStep with the grid vs rasterize_fused -> BilateralGrid.apply ->
    unclamped loss -> + weight * tv_loss -> backward -> FusedAdam for the Gaussians and torch.optim.Adam(eps=1e-15) with
    the restated schedule for the grids.  Then the graphed step against the eager one."""
    bil, training = _mods(native)
    t, raw, tg = _gsplat_setup(native, cuda_device)
    cfg = training.AdamConfig(means_lr=1.6e-3, iterations=30000)
    PA, PB = _clone(raw), _clone(raw)
    gA = bil.BilateralGrid(3, device=cuda_device)
    gB = bil.BilateralGrid(3, device=cuda_device)
    with torch.no_grad():
        init = _grids(3, 16, 16, 8, 11, cuda_device)
        gA.grids.copy_(init)
        gB.grids.copy_(init)
    step = training.TrainStep(PA, 3, 320, 192, optimizer=training.FusedAdam(PA, cfg), bilateral_grid=gA, tv_loss_weight=10.0)
    optB = training.FusedAdam(PB, cfg)
    adam = torch.optim.Adam([gB.grids], lr=2e-3, eps=1e-15)
    sched = bil.WarmupExponentialLR(2e-3, cfg.iterations)
    for it in range(5):
        idx = it % 3
        la = float(step(t["viewmats"], t["Ks"], tg[idx], t["background"], image_idx=idx))
        out = native.rasterize_fused(PB["means"], PB["sh0"], PB["shN"], PB["scaling_raw"], PB["rotation_raw"],
                                     PB["opacity_raw"], 3, t["viewmats"], t["Ks"], 320, 192, bg_color=t["background"])
        img = gB.apply(out.render_colors[0].permute(2, 0, 1), idx)
        loss, _ = training.photometric_loss_unclamped(img, tg[idx], 0.2)
        total = loss + 10.0 * gB.tv_loss()
        total.backward()
        optB.step(it + 1)
        optB.zero_grad()
        adam.step()
        adam.zero_grad()
        for grp in adam.param_groups:
            grp["lr"] = sched.step()
        print(f"it {it}: fused {la:.7f} composition {float(total):.7f}")
        assert abs(la - float(total)) <= 2e-5 * max(1.0, abs(la))
    for k in PA:
        if PA[k].numel():
            assert rel(PA[k].detach(), PB[k].detach()) < 1e-4, k
    assert rel(gA.grids.detach(), gB.grids.detach()) <= 1e-4
    assert rel(gA.grids.detach() - init, gB.grids.detach() - init) <= 1e-3  # the updates themselves agree


@pytest.mark.parametrize("path", ["gsplat", "fastgs"])
def test_graphed_with_grid_equals_eager(native, cuda_device, path):
    """One captured graph serves every image: the index changes between replays."""
    bil, training = _mods(native)
    cfg = training.AdamConfig(means_lr=1.6e-3)
    init = _grids(3, 16, 16, 8, 5, cuda_device)
    gA, gB = bil.BilateralGrid(3, device=cuda_device), bil.BilateralGrid(3, device=cuda_device)
    with torch.no_grad():
        gA.grids.copy_(init)
        gB.grids.copy_(init)
    if path == "gsplat":
        t, raw, tg = _gsplat_setup(native, cuda_device)
        A, B = _clone(raw), _clone(raw)
        eager = training.TrainStep(A, 3, 320, 192, optimizer=training.FusedAdam(A, cfg), bilateral_grid=gA)
        eager.size_capacity(t["viewmats"], t["Ks"], tg[0], t["background"])
        graphed = training.GraphedTrainStep(B, 3, 320, 192, cfg, bilateral_grid=gB)
        run_a = lambda i: eager(t["viewmats"], t["Ks"], tg[i], t["background"], image_idx=i)
        run_b = lambda i: graphed(t["viewmats"], t["Ks"], tg[i], t["background"], image_idx=i)
    else:
        fg = importlib.import_module(native.__name__ + ".fastgs")
        inp = scenes.fastgs_inputs(scenes.scene_small(N=2500, width=160, height=112, sh_degree=3, seed=6, view=2))
        names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw",
                 "opacity_raw": "opacities_raw", "sh0": "sh0", "shN": "shN"}
        A = {k: torch.from_numpy(inp[v]).to(cuda_device).requires_grad_(True) for k, v in names.items()}
        B = {k: torch.from_numpy(inp[v]).to(cuda_device).requires_grad_(True) for k, v in names.items()}
        s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(cuda_device),
                              active_sh_bases=inp["active_sh_bases"], width=inp["width"], height=inp["height"],
                              focal_x=inp["fx"], focal_y=inp["fy"], center_x=inp["cx"], center_y=inp["cy"],
                              near_plane=inp["near_plane"], far_plane=inp["far_plane"])
        w2c = torch.from_numpy(inp["w2c"]).to(cuda_device)
        g = torch.Generator(device=cuda_device).manual_seed(2)
        tg = [torch.rand((3, inp["height"], inp["width"]), device=cuda_device, generator=g) for _ in range(3)]
        bgc = torch.tensor([0.3, 0.2, 0.1], device=cuda_device)
        eager = training.FastGsTrainStep(A, 3, inp["width"], inp["height"], optimizer=training.FusedAdam(A, cfg),
                                         bilateral_grid=gA)
        graphed = training.GraphedFastGsTrainStep(B, 3, s, cfg, bilateral_grid=gB)
        run_a = lambda i: eager(w2c, s, tg[i], bgc, image_idx=i)
        run_b = lambda i: graphed(w2c, s.cam_position, tg[i], bgc, image_idx=i)
    la, lb = [], []
    for it in range(5):
        i = (2 * it) % 3
        la.append(float(run_a(i)))
        lb.append(float(run_b(i)))
    print(path, "eager ", [f"{v:.6f}" for v in la])
    print(path, "graph ", [f"{v:.6f}" for v in lb])
    for a, b in zip(la, lb):
        assert abs(a - b) < 2e-5 * max(1.0, abs(a))
    for k in A:
        if A[k].numel():
            assert rel(B[k].detach(), A[k].detach()) < 1e-4, k
    assert rel(gB.grids.detach() - init, gA.grids.detach() - init) < 1e-4
    assert not torch.equal(gB.grids.detach(), init)


def test_fastgs_identity_grid_first_iteration_equals_no_grid_loss(native, cuda_device):
    bil, training = _mods(native)
    fg = importlib.import_module(native.__name__ + ".fastgs")
    inp = scenes.fastgs_inputs(scenes.scene_small(N=2500, width=160, height=112, sh_degree=3, seed=6, view=2))
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw", "opacity_raw": "opacities_raw",
             "sh0": "sh0", "shN": "shN"}
    mk = lambda: {k: torch.from_numpy(inp[v]).to(cuda_device).requires_grad_(True) for k, v in names.items()}
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(cuda_device),
                          active_sh_bases=inp["active_sh_bases"], width=inp["width"], height=inp["height"], focal_x=inp["fx"],
                          focal_y=inp["fy"], center_x=inp["cx"], center_y=inp["cy"], near_plane=inp["near_plane"],
                          far_plane=inp["far_plane"])
    w2c = torch.from_numpy(inp["w2c"]).to(cuda_device)
    tgt = torch.rand((3, inp["height"], inp["width"]), device=cuda_device, generator=torch.Generator(device=cuda_device).manual_seed(4))
    bgc = torch.tensor([0.3, 0.2, 0.1], device=cuda_device)
    a = training.FastGsTrainStep(mk(), 3, inp["width"], inp["height"], optimizer=None)
    b = training.FastGsTrainStep(mk(), 3, inp["width"], inp["height"], optimizer=None,
                                 bilateral_grid=bil.BilateralGrid(2, device=cuda_device))
    la, lb = float(a(w2c, s, tgt, bgc)), float(b(w2c, s, tgt, bgc, image_idx=1))
    print(f"fastgs path: no grid {la:.8f}, identity grid {lb:.8f}")
    assert abs(la - lb) <= 1e-6


def test_fastgs_training_with_grid_matches_autograd_composition(native, cuda_device):
    """Five iterations cycling the image on the fastgs path: FastGsTrainStep with the grid vs fast_rasterize (autograd,
    background composite) -> BilateralGrid.apply -> unclamped loss -> + weight * tv_loss -> backward -> FusedAdam for the
    Gaussians and torch.optim.Adam(eps=1e-15) with the restated schedule for the grids."""
    bil, training = _mods(native)
    fg = importlib.import_module(native.__name__ + ".fastgs")
    inp = scenes.fastgs_inputs(scenes.scene_small(N=2500, width=160, height=112, sh_degree=3, seed=6, view=2))
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw", "opacity_raw": "opacities_raw",
             "sh0": "sh0", "shN": "shN"}
    mk = lambda: {k: torch.from_numpy(inp[v]).to(cuda_device).requires_grad_(True) for k, v in names.items()}
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(cuda_device),
                          active_sh_bases=inp["active_sh_bases"], width=inp["width"], height=inp["height"], focal_x=inp["fx"],
                          focal_y=inp["fy"], center_x=inp["cx"], center_y=inp["cy"], near_plane=inp["near_plane"],
                          far_plane=inp["far_plane"])
    w2c = torch.from_numpy(inp["w2c"]).to(cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(8)
    tg = [torch.rand((3, inp["height"], inp["width"]), device=cuda_device, generator=g) for _ in range(3)]
    bgc = torch.tensor([0.3, 0.2, 0.1], device=cuda_device)
    cfg = training.AdamConfig(iterations=30000)
    PA, PB = mk(), mk()
    init = _grids(3, 16, 16, 8, 13, cuda_device)
    gA, gB = bil.BilateralGrid(3, device=cuda_device), bil.BilateralGrid(3, device=cuda_device)
    with torch.no_grad():
        gA.grids.copy_(init)
        gB.grids.copy_(init)
    step = training.FastGsTrainStep(PA, 3, inp["width"], inp["height"], optimizer=training.FusedAdam(PA, cfg),
                                    bilateral_grid=gA, tv_loss_weight=10.0)
    with pytest.raises(ValueError):
        step(w2c, s, tg[0], bgc)  # a step with a grid needs the image index
    step.iteration = 0
    optB = training.FusedAdam(PB, cfg)
    adam = torch.optim.Adam([gB.grids], lr=2e-3, eps=1e-15)
    sched = bil.WarmupExponentialLR(2e-3, cfg.iterations)
    be = fg.default_backend()
    for it in range(5):
        idx = (it * 2) % 3
        la = float(step(w2c, s, tg[idx], bgc, image_idx=idx))
        img, _ = fg.fast_rasterize(be, PB["means"], PB["scaling_raw"], PB["rotation_raw"], PB["opacity_raw"], PB["sh0"],
                                   PB["shN"], w2c, s, bg_color=bgc)
        sliced = gB.apply(img, idx)
        loss, _ = training.photometric_loss_unclamped(sliced, tg[idx], 0.2)
        total = loss + 10.0 * gB.tv_loss()
        total.backward()
        optB.step(it + 1)
        optB.zero_grad()
        adam.step()
        adam.zero_grad()
        for grp in adam.param_groups:
            grp["lr"] = sched.step()
        print(f"fastgs it {it}: fused {la:.7f} composition {float(total):.7f}")
        assert abs(la - float(total)) <= 2e-5 * max(1.0, abs(la))
    for k in PA:
        if PA[k].numel():
            assert rel(PA[k].detach(), PB[k].detach()) < 1e-4, k
    assert rel(gA.grids.detach(), gB.grids.detach()) <= 1e-4
    assert rel(gA.grids.detach() - init, gB.grids.detach() - init) <= 1e-3
