"""GPU: the fastgs (EWA) rasterizer, SURVEY.md 8 f4 -- this backend (include/fastgs/rasterization_api.h ->
shim/FastGs.cpp -> gsb_fastgs_*) against
  * the reference's own fastgs kernels compiled unmodified (oracle/_ref/libfastgs_ref.so; oracle/build_ref.py), driven
    through the same torch binding, and
  * the CPU restatement oracle/fastgs_oracle.c (float32 and float64),
on the same raw parameters.  The reference has no tests for this path (SURVEY.md 4); the bar is BASELINE.json's
north_star: 1e-4 relative on the image, 1e-3 on gradients, plus the per-Gaussian bounds of tests/parity.py."""
import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel

pytestmark = pytest.mark.gpu
PARAMS = ("means", "scales_raw", "rotations_raw", "opacities_raw", "sh0", "shN")


def _fg(native):
    import importlib
    return importlib.import_module(native.__name__ + ".fastgs")


def _ref_backend(native):
    from oracle import ref_fastgs
    if not ref_fastgs.available():
        pytest.skip("oracle/_ref/libfastgs_ref.so not built (build() makes it where the reference's sources are present); "
                    "test_gpu_vs_reference_golden.py compares against its stored outputs")
    return ref_fastgs.backend(_fg(native))


def reference(native, inp, dev, gi, ga, w2c_grad=False, dens=None):
    """What the reference computes on these inputs: its own fastgs kernels where oracle/build_ref.py built them
    (oracle/_ref), else the float64 CPU restatement, which tests/golden/ref_fastgs_small.npz pins to those kernels."""
    from oracle import ref_fastgs
    if ref_fastgs.available():
        return run(_fg(native), ref_fastgs.backend(_fg(native)), inp, dev, gi, ga, w2c_grad=w2c_grad, dens=dens)
    from oracle import fastgs_oracle as fgo
    d = None if dens is None else dens.cpu().numpy()
    o = fgo.render(**inp, grad_image=gi.cpu().numpy(), grad_alpha=ga.cpu().numpy(), want_w2c_grad=w2c_grad,
                   densification_info=d, precision="f64")
    if dens is not None:
        dens.copy_(torch.from_numpy(o["densification_info"]).to(dens))
    grads = {k: torch.from_numpy(o["grad_" + k]).float().to(dev) for k in PARAMS}
    return dict(image=torch.from_numpy(o["image"]).float().to(dev), alpha=torch.from_numpy(o["alpha"]).float().to(dev),
                grads=grads, w2c_grad=torch.from_numpy(o["grad_w2c"]).float().to(dev) if w2c_grad else None)


def _leaves(inp, dev, requires_grad=True):
    return {k: torch.from_numpy(inp[k]).to(dev).requires_grad_(requires_grad) for k in PARAMS}


def _settings(fg, inp, dev):
    return fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(dev), active_sh_bases=inp["active_sh_bases"],
                             width=inp["width"], height=inp["height"], focal_x=inp["fx"], focal_y=inp["fy"],
                             center_x=inp["cx"], center_y=inp["cy"], near_plane=inp["near_plane"], far_plane=inp["far_plane"])


def run(fg, backend, inp, dev, gi, ga, w2c_grad=False, dens=None):
    P = _leaves(inp, dev)
    w2c = torch.from_numpy(inp["w2c"]).to(dev).requires_grad_(w2c_grad)
    s = _settings(fg, inp, dev)
    image, alpha = fg.fast_rasterize(backend, P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"],
                                     P["shN"], w2c, s, densification_info=dens)
    ((image * gi).sum() + (alpha * ga).sum()).backward()
    torch.cuda.synchronize()
    grads = {k: (P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])) for k in PARAMS}
    return dict(image=image.detach(), alpha=alpha.detach(), grads=grads, w2c_grad=w2c.grad)


def image_close(a, b, tag, rel_tol=1e-4):
    e, ea = rel(a["image"], b["image"]), rel(a["alpha"], b["alpha"])
    d = (a["image"] - b["image"]).abs()
    frac = float((d > 1e-3).double().mean())
    print(f"[{tag}] image rel_l2 {e:.2e}, alpha rel_l2 {ea:.2e}, max |d| {float(d.max()):.2e}, pixels off by > 1e-3: {frac:.2e}")
    assert e < rel_tol and ea < rel_tol, (tag, e, ea)
    # a pixel at a decision boundary (alpha >= 1/255, T < 1e-4, tile test) may gain or lose one contribution
    assert frac < 1e-3 and float(d.max()) < 2e-2, (tag, frac, float(d.max()))


def grads_close(a, b, n, tag, **kw):
    for k in PARAMS:
        assert_grad_close(a["grads"][k], b["grads"][k], k, n, tag=tag, **kw)


def _weights(inp, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn((3, inp["height"], inp["width"]), device=dev, generator=g),
            torch.randn((1, inp["height"], inp["width"]), device=dev, generator=g))


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_fastgs_b200_vs_reference_kernels_and_oracle(native, cuda_device, deg):
    fg = _fg(native)
    sc = scenes.scene_small(N=3000, width=200, height=120, sh_degree=deg, seed=11 + deg, view=1, )
    inp = scenes.fastgs_inputs(sc)
    gi, ga = _weights(inp, cuda_device)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga)
    ref = reference(native, inp, cuda_device, gi, ga)
    n = inp["means"].shape[0]
    image_close(mine, ref, f"deg{deg} b200 vs reference kernels")
    grads_close(mine, ref, n, f"deg{deg} b200 vs reference kernels")
    # the CPU restatement, float64: pins the oracle to the reference kernels and this library's path to both
    from oracle import fastgs_oracle as fgo
    o = fgo.render(**{k: inp[k] for k in inp}, grad_image=gi.cpu().numpy(), grad_alpha=ga.cpu().numpy(), precision="f64")
    oracle = dict(image=torch.from_numpy(o["image"]).to(cuda_device), alpha=torch.from_numpy(o["alpha"]).to(cuda_device),
                  grads={"means": o["grad_means"], "scales_raw": o["grad_scales_raw"], "rotations_raw": o["grad_rotations_raw"],
                         "opacities_raw": o["grad_opacities_raw"], "sh0": o["grad_sh0"], "shN": o["grad_shN"]})
    image_close(ref, oracle, f"deg{deg} reference kernels vs f64 oracle")
    image_close(mine, oracle, f"deg{deg} b200 vs f64 oracle")
    grads_close(ref, oracle, n, f"deg{deg} reference kernels vs f64 oracle")
    grads_close(mine, oracle, n, f"deg{deg} b200 vs f64 oracle")


def test_fastgs_config_a(native, cuda_device):
    """BASELINE.json configs[0]: 10k Gaussians, 256x256, SH degree 0."""
    fg = _fg(native)
    inp = scenes.fastgs_inputs(scenes.scene_a())
    gi, ga = _weights(inp, cuda_device, 1)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga)
    ref = reference(native, inp, cuda_device, gi, ga)
    image_close(mine, ref, "config A b200 vs reference kernels")
    grads_close(mine, ref, inp["means"].shape[0], "config A b200 vs reference kernels")


def test_fastgs_w2c_gradient_and_densification(native, cuda_device):
    fg = _fg(native)
    inp = scenes.fastgs_inputs(scenes.scene_small(N=2500, width=176, height=144, sh_degree=2, seed=3, view=2))
    gi, ga = _weights(inp, cuda_device, 2)
    n = inp["means"].shape[0]
    d1 = torch.zeros((2, n), device=cuda_device)
    d2 = torch.zeros((2, n), device=cuda_device)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga, w2c_grad=True, dens=d1)
    ref = reference(native, inp, cuda_device, gi, ga, w2c_grad=True, dens=d2)
    assert mine["w2c_grad"] is not None and ref["w2c_grad"] is not None
    e = rel(mine["w2c_grad"][:3], ref["w2c_grad"][:3])
    print(f"w2c gradient rel_l2 {e:.2e}")
    assert e < 1e-3
    assert torch.equal(d1[0], d2[0])  # the same primitives are visible
    assert rel(d1[1], d2[1]) < 1e-3
    # a second backward call accumulates
    mine2 = run(fg, fg.default_backend(), inp, cuda_device, gi, ga, dens=d1)
    assert torch.equal(d1[0], 2 * d2[0])


def test_fastgs_edge_cases(native, cuda_device):
    fg = _fg(native)
    be = fg.default_backend()
    inp = scenes.fastgs_inputs(scenes.scene_small(N=500, width=100, height=70, sh_degree=1, seed=5))
    gi, ga = _weights(inp, cuda_device, 3)
    # everything culled: image and alpha are zero, gradients are zero
    far = dict(inp)
    far["opacities_raw"] = np.full_like(inp["opacities_raw"], -12.0)
    r = run(fg, be, far, cuda_device, gi, ga)
    assert not r["image"].any() and not r["alpha"].any()
    assert all(not g.any() for g in r["grads"].values())
    # N == 0
    empty = {k: (v[:0] if k in PARAMS else v) for k, v in inp.items()}
    r0 = run(fg, be, empty, cuda_device, gi, ga)
    assert not r0["image"].any() and r0["image"].shape == (3, 70, 100)
    # a primitive covering the whole frame (the warp-cooperative tile count / big-run paths) plus the ordinary ones
    big = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    big["scales_raw"][:3] = np.log(1.5)
    big["means"][:3] = [[0.0, 0.0, 3.0], [0.3, 0.1, 3.5], [-0.2, 0.0, 2.5]]
    mine = run(fg, be, big, cuda_device, gi, ga)
    ref = reference(native, big, cuda_device, gi, ga)
    image_close(mine, ref, "frame-filling primitives, b200 vs reference kernels")
    grads_close(mine, ref, big["means"].shape[0], "frame-filling primitives", frac_tol=5e-3)
    # rejected inputs fail loudly
    with pytest.raises(RuntimeError):
        bad = dict(inp)
        bad["active_sh_bases"] = 9  # the tensors hold 4 bases
        run(fg, be, bad, cuda_device, gi, ga)


def test_fastgs_forward_context_is_self_contained(native, cuda_device):
    """Forward's opaque buffers carry what the backward needs; nothing depends on Python-side or library state."""
    fg = _fg(native)
    be = fg.default_backend()
    inp = scenes.fastgs_inputs(scenes.scene_small(N=800, width=96, height=64, sh_degree=3, seed=9))
    P = _leaves(inp, cuda_device, requires_grad=False)
    w2c = torch.from_numpy(inp["w2c"]).to(cuda_device)
    s = _settings(fg, inp, cuda_device)
    img1, al1, c1 = be.forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"], P["shN"], w2c, s)
    img2, al2, c2 = be.forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"], P["shN"], w2c, s)
    assert torch.equal(img1, img2) and torch.equal(al1, al2)  # deterministic
    assert int(c1["ints"][1]) == int(c2["ints"][1]) > 0
    gi, ga = _weights(inp, cuda_device, 4)
    g1 = be.backward(c1, gi, ga, img1, al1, P["means"], P["scales_raw"], P["rotations_raw"], P["shN"], w2c, s)
    g2 = be.backward(c2, gi, ga, img2, al2, P["means"], P["scales_raw"], P["rotations_raw"], P["shN"], w2c, s)
    for a, b in zip(g1[:6], g2[:6]):
        assert rel(a, b) < 1e-5  # float atomics: order-dependent in the last bits only


@pytest.mark.parametrize("deg", [0, 3])
def test_reference_fastgs_caller_runs_on_the_b200_backend(native, cuda_device, deg):
    """The reference's OWN caller of its default rasterizer -- FastGSRasterize of fast_rasterizer_autograd.cpp, compiled
    unmodified against include/fastgs/rasterization_api.h and linked against libgsplat_b200.so
    (oracle/_ref/libref_fastgs_l3_b200.so, oracle/ref_fastgs_l3_harness.cpp) -- executes forward and backward on the GPU
    through this backend and agrees with the package's Python mirror of the same sequence."""
    import os
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_fastgs_l3_b200.so")
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/libref_fastgs_l3_b200.so not built (build() makes it where the reference's sources are present)")
    torch.ops.load_library(so)
    fg = _fg(native)
    inp = scenes.fastgs_inputs(scenes.scene_small(N=3000, width=200, height=120, sh_degree=deg, seed=21, view=3))
    gi, ga = _weights(inp, cuda_device, 5)
    bg = torch.tensor([0.2, 0.5, 0.7], device=cuda_device)
    n = inp["means"].shape[0]
    res = {}
    for tag in ("reference_cpp", "python_mirror"):
        P = _leaves(inp, cuda_device)
        w2c = torch.from_numpy(inp["w2c"]).to(cuda_device)
        dens = torch.zeros((2, n), device=cuda_device)
        s = _settings(fg, inp, cuda_device)
        if tag == "reference_cpp":
            img, alpha = torch.ops.ref_fastgs_l3_b200.fast_render(
                P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"], P["shN"], w2c, s.cam_position,
                deg, inp["width"], inp["height"], inp["fx"], inp["fy"], inp["cx"], inp["cy"], bg, dens)
        else:
            img, alpha = fg.fast_rasterize(fg.default_backend(), P["means"], P["scales_raw"], P["rotations_raw"],
                                           P["opacities_raw"], P["sh0"], P["shN"], w2c, s, bg_color=bg, densification_info=dens)
        ((img * gi).sum() + (alpha * ga).sum()).backward()
        torch.cuda.synchronize()
        res[tag] = (img.detach(), alpha.detach(), {k: (P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])) for k in PARAMS}, dens)
    assert torch.equal(res["reference_cpp"][0], res["python_mirror"][0])  # same kernels, same inputs, same order
    assert torch.equal(res["reference_cpp"][1], res["python_mirror"][1])
    assert float(res["python_mirror"][1].mean()) > 0.05
    for k in PARAMS:
        assert_grad_close(res["reference_cpp"][2][k], res["python_mirror"][2][k], k, n, rel_tol=2e-5,
                          tag=f"reference C++ fastgs caller vs Python mirror (deg {deg})")
    assert torch.equal(res["reference_cpp"][3][0], res["python_mirror"][3][0]) and float(res["python_mirror"][3][0].sum()) > 100


@pytest.mark.parametrize("cfg,n_gauss", [("B", 1_000_000), ("D", 6_000_000)], ids=["configB_1M", "configD_6M"])
def test_fastgs_full_size_against_reference_kernels(native, cuda_device, cfg, n_gauss):
    """BASELINE.json configs[1] / [3] at full size (1080p, SH degree 3) through the fastgs path: this backend against the
    reference's own kernels on the same raw parameters, plus size-independent properties."""
    fg = _fg(native)
    inp = scenes.fastgs_inputs(scenes.scene_b(N=n_gauss))
    gi, ga = _weights(inp, cuda_device, 7)
    gi, ga = gi / gi.numel(), ga / ga.numel()
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga)
    assert 0.0 <= float(mine["alpha"].min()) and float(mine["alpha"].max()) <= 1.0 - 1e-4 + 1e-6
    assert float(mine["image"].min()) >= 0.0
    assert float(mine["alpha"].mean()) > 0.9  # the slab is opaque at this density
    # culled primitives receive exactly zero gradient; visible ones almost always a non-zero one
    P = _leaves(inp, cuda_device, requires_grad=False)
    s = _settings(fg, inp, cuda_device)
    _, _, ctx = fg.default_backend().forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"],
                                             P["shN"], torch.from_numpy(inp["w2c"]).to(cuda_device), s)
    n_inst = int(ctx["ints"][1])
    print(f"[config {cfg} fastgs] instances {n_inst}")
    assert n_inst > 5 * n_gauss // 2
    del ctx, P
    ref = run(fg, _ref_backend(native), inp, cuda_device, gi, ga)
    image_close(mine, ref, f"config {cfg} fastgs, b200 vs reference kernels")
    grads_close(mine, ref, n_gauss, f"config {cfg} fastgs, b200 vs reference kernels")
    zero_mine = (mine["grads"]["means"].abs().sum(-1) == 0)
    zero_ref = (ref["grads"]["means"].abs().sum(-1) == 0)
    assert float((zero_mine != zero_ref).double().mean()) < 1e-3


def test_fastgs_training_iteration(native, cuda_device):
    """FastGsTrainStep (fastgs forward -> background -> fused loss-and-gradient -> fastgs backward -> one-launch Adam)
    against the same iteration composed with autograd and torch.optim-free reference formulas: the gradients that reach
    the optimizer equal those of loss.backward() through FastGSRasterize, and the parameters move alike."""
    import importlib
    fg = _fg(native)
    training = importlib.import_module(native.__name__ + ".training")
    sc = scenes.scene_small(N=2500, width=160, height=112, sh_degree=3, seed=4, view=1)
    inp = scenes.fastgs_inputs(sc)
    dev = cuda_device
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw", "opacity_raw": "opacities_raw",
             "sh0": "sh0", "shN": "shN"}
    s = _settings(fg, inp, dev)
    w2c = torch.from_numpy(inp["w2c"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    target = torch.rand((3, inp["height"], inp["width"]), device=dev, generator=g)
    bg = torch.tensor([0.1, 0.3, 0.6], device=dev)
    # (1) the fused iteration
    P1 = {k: torch.from_numpy(inp[v]).to(dev).requires_grad_(True) for k, v in names.items()}
    ts = training.FastGsTrainStep(P1, 3, inp["width"], inp["height"], optimizer=None)
    loss1 = ts(w2c, s, target, bg)
    g1 = {k: P1[k].grad.clone() for k in P1}
    # (2) autograd through the Python mirror of the reference's caller + the loss function
    P2 = {k: torch.from_numpy(inp[v]).to(dev).requires_grad_(True) for k, v in names.items()}
    img, _ = fg.fast_rasterize(fg.default_backend(), P2["means"], P2["scaling_raw"], P2["rotation_raw"], P2["opacity_raw"],
                               P2["sh0"], P2["shN"], w2c, s, bg_color=bg)
    loss2, _ = training.photometric_loss(img, target, 0.2)
    loss2.backward()
    assert abs(float(loss1) - float(loss2)) < 1e-6
    for k in P1:
        assert_grad_close(g1[k], P2[k].grad, k, inp["means"].shape[0], rel_tol=2e-5, tag="fastgs train step vs autograd")
    # (3) with the optimizer: three iterations lower the loss and every group moves
    P3 = {k: torch.from_numpy(inp[v]).to(dev).requires_grad_(True) for k, v in names.items()}
    before = {k: v.detach().clone() for k, v in P3.items()}
    ts3 = training.FastGsTrainStep(P3, 3, inp["width"], inp["height"], optimizer=training.FusedAdam(P3))
    losses = [float(ts3(w2c, s, target, bg)) for _ in range(1002)][::500]
    print("fastgs training losses (iterations 1, 501, 1001):", losses)
    assert losses[-1] < losses[0]
    assert all(not torch.equal(P3[k].detach(), before[k]) for k in P3)


def test_fastgs_capacity_mode_and_graphed_iteration(native, cuda_device):
    """include/fastgs/rasterization_ext.h: forward_capacity (no host read-back) renders what forward_wrapper renders when
    the capacity suffices, clips when it does not, and lets the whole training iteration replay from one CUDA graph with the
    same parameter updates as the eager iteration."""
    import importlib
    fg = _fg(native)
    training = importlib.import_module(native.__name__ + ".training")
    be = fg.default_backend()
    inp = scenes.fastgs_inputs(scenes.scene_small(N=2500, width=160, height=112, sh_degree=3, seed=6, view=2))
    dev = cuda_device
    P = _leaves(inp, dev, requires_grad=False)
    w2c = torch.from_numpy(inp["w2c"]).to(dev)
    s = _settings(fg, inp, dev)
    img, al, c = be.forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"], P["shN"], w2c, s)
    n = int(c["ints"][1])
    img2, al2, c2 = be.forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"], P["shN"], w2c, s,
                               capacity=n + 100)
    assert torch.equal(img, img2) and torch.equal(al, al2) and int(c2["n_instances_dev"].item()) == n
    gi, ga = _weights(inp, dev, 8)
    g1 = be.backward(c, gi, ga, img, al, P["means"], P["scales_raw"], P["rotations_raw"], P["shN"], w2c, s)
    g2 = be.backward(c2, gi, ga, img2, al2, P["means"], P["scales_raw"], P["rotations_raw"], P["shN"], w2c, s)
    for a, b in zip(g1[:6], g2[:6]):
        assert rel(a, b) < 1e-5
    # too small a capacity: reported through the device-side count, no out-of-bounds access, still a finite image
    img3, _, c3 = be.forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"], P["shN"], w2c, s,
                             capacity=n // 2)
    assert int(c3["n_instances_dev"].item()) == n > n // 2 and bool(torch.isfinite(img3).all())
    be.backward(c3, gi, ga, img3, al, P["means"], P["scales_raw"], P["rotations_raw"], P["shN"], w2c, s)
    torch.cuda.synchronize()
    # graph == eager over a few iterations (Adam included; the shN group is frozen for the first 1000 iterations in both)
    names = {"means": "means", "scaling_raw": "scales_raw", "rotation_raw": "rotations_raw", "opacity_raw": "opacities_raw",
             "sh0": "sh0", "shN": "shN"}
    g = torch.Generator(device=dev).manual_seed(1)
    target = torch.rand((3, inp["height"], inp["width"]), device=dev, generator=g)
    bg = torch.tensor([0.3, 0.2, 0.1], device=dev)
    PA = {k: torch.from_numpy(inp[v]).to(dev).requires_grad_(True) for k, v in names.items()}
    PB = {k: torch.from_numpy(inp[v]).to(dev).requires_grad_(True) for k, v in names.items()}
    eager = training.FastGsTrainStep(PA, 3, inp["width"], inp["height"], optimizer=training.FusedAdam(PA))
    graphed = training.GraphedFastGsTrainStep(PB, 3, s)
    la, lb = [], []
    for _ in range(5):
        la.append(float(eager(w2c, s, target, bg)))
        lb.append(float(graphed(w2c, s.cam_position, target, bg)))
    assert not graphed.overflowed()
    print("eager losses", la, "graph losses", lb)
    assert max(abs(a - b) for a, b in zip(la, lb)) < 1e-5
    for k in PA:
        assert rel(PB[k].detach(), PA[k].detach()) < 1e-5, k


@pytest.mark.parametrize("active", [1, 4, 9])
def test_fastgs_partially_active_sh(native, cuda_device, active):
    """Training raises the active SH degree every 1000 iterations while shN always holds 15 bases
    (fast_rasterizer.cpp:33-34): fewer active bases than stored ones -- the inactive rows get zero gradient."""
    fg = _fg(native)
    inp = scenes.fastgs_inputs(scenes.scene_small(N=2000, width=150, height=90, sh_degree=3, seed=31, view=1))
    inp["active_sh_bases"] = active
    gi, ga = _weights(inp, cuda_device, 9)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga)
    ref = reference(native, inp, cuda_device, gi, ga)
    image_close(mine, ref, f"active {active} of 16 bases, b200 vs reference kernels")
    grads_close(mine, ref, inp["means"].shape[0], f"active {active} of 16 bases")
    assert not mine["grads"]["shN"][:, active - 1:].any()
    if active > 1:
        assert mine["grads"]["shN"][:, :active - 1].any()


def test_dump_reference_fastgs_golden(native, cuda_device, tmp_path):
    """Writes ref_fastgs_small.npz (into $GSB_GOLDEN_OUT, else a temporary directory): outputs of the reference's own fastgs kernels (oracle/_ref/libfastgs_ref.so) on
    a small scene.  The file is committed as tests/golden/ref_fastgs_small.npz and pins oracle/fastgs_oracle.c in the no-GPU
    suite (tests/test_oracle_fastgs.py::test_oracle_vs_reference_fastgs_golden)."""
    import os
    fg = _fg(native)
    inp = scenes.fastgs_inputs(scenes.scene_small(N=1500, width=176, height=112, sh_degree=3, seed=13, view=2))
    rng = np.random.default_rng(17)
    gi = torch.from_numpy(rng.standard_normal((3, inp["height"], inp["width"])).astype(np.float32)).to(cuda_device)
    ga = torch.from_numpy(rng.standard_normal((1, inp["height"], inp["width"])).astype(np.float32)).to(cuda_device)
    n = inp["means"].shape[0]
    dens = torch.zeros((2, n), device=cuda_device)
    ref = run(fg, _ref_backend(native), inp, cuda_device, gi, ga, w2c_grad=True, dens=dens)
    out = os.environ.get("GSB_GOLDEN_OUT") or str(tmp_path)
    os.makedirs(out, exist_ok=True)
    np.savez_compressed(os.path.join(out, "ref_fastgs_small.npz"), image=ref["image"].cpu().numpy(), alpha=ref["alpha"].cpu().numpy(),
                        grad_image=gi.cpu().numpy(), grad_alpha=ga.cpu().numpy(), grad_w2c=ref["w2c_grad"].cpu().numpy(),
                        densification_info=dens.cpu().numpy(),
                        **{"grad_" + k: v.cpu().numpy() for k, v in ref["grads"].items()})
    assert float(ref["alpha"].mean()) > 0.05
