"""GPU: the rows around the hot path (SURVEY.md 8 f2 / f3): fused SSIM + L1 loss with its gradient, fused Adam, and a
few whole training iterations -- against plain torch restatements of the reference's formulas
(src/training/trainer.cpp:103-126, src/training/kernels/ssim.cu, fastgs/optimizer/include/adam_kernels.cuh:13-36)."""
import math

import numpy as np
import pytest
import torch

import loss_restatement as lr
import scenes
from parity import rel, to_dev

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H,W", [(64, 80), (70, 150), (9, 40), (270, 480)])
def test_photometric_loss_and_gradient_vs_torch(native, cuda_device, H, W):
    from gsplat_b200 import training
    g = torch.Generator(device=cuda_device).manual_seed(H * 1000 + W)
    renders = (torch.rand((1, H, W, 3), device=cuda_device, generator=g) * 1.4 - 0.2).requires_grad_(True)  # some clamp
    target = torch.rand((3, H, W), device=cuda_device, generator=g)
    loss, stats = training.photometric_loss(renders, target, 0.2)
    (loss * 1.7).backward()
    want, l1, ssim, g64 = lr.photometric_loss_f64(renders, target, 0.2)
    g64 = 1.7 * g64
    print(f"[{H}x{W}] loss {float(loss):.6f} vs torch f64 {want:.6f}; grad rel_l2 {rel(renders.grad, g64):.2e}")
    assert abs(float(loss) - want) < 2e-6 * max(1.0, abs(want))
    assert abs(float(stats[1]) - l1) < 2e-6 and abs(float(stats[2]) - ssim) < 2e-6
    assert rel(renders.grad, g64) < 2e-5
    assert float((renders.grad - g64.float()).abs().max()) < 1e-4 * float(g64.abs().max())
    # the same target in the blend's own layout
    loss2, _ = training.photometric_loss(renders.detach(), target.permute(1, 2, 0)[None].contiguous(), 0.2)
    assert abs(float(loss2) - float(loss)) < 1e-7
    # renders (and their gradient) as [3,H,W] planes: the fastgs path's image layout
    planes = renders.detach()[0].permute(2, 0, 1).contiguous().requires_grad_(True)
    loss3, _ = training.photometric_loss(planes, target, 0.2)
    (loss3 * 1.7).backward()
    assert abs(float(loss3) - float(loss)) < 1e-7
    assert torch.equal(planes.grad, renders.grad[0].permute(2, 0, 1))


def test_fused_adam_matches_reference_formula(native, cuda_device):
    from gsplat_b200 import training
    g = torch.Generator(device=cuda_device).manual_seed(5)
    shapes = {"means": (1001, 3), "sh0": (1001, 1, 3), "shN": (1001, 15, 3), "scaling_raw": (1001, 3),
              "rotation_raw": (1001, 4), "opacity_raw": (1001, 1)}
    P = {k: torch.randn(s, device=cuda_device, generator=g).requires_grad_(True) for k, s in shapes.items()}
    ref = {k: v.detach().double().clone() for k, v in P.items()}
    m = {k: torch.zeros_like(v) for k, v in ref.items()}
    v2 = {k: torch.zeros_like(v) for k, v in ref.items()}
    cfg = training.AdamConfig(iterations=100)
    opt = training.FusedAdam(P, cfg)
    lr = cfg.lrs()
    steps = {k: 0 for k in P}
    for it in (1, 2, 1500, 1501):  # shN is frozen while iteration <= 1000 (its step count still advances)
        for k in P:
            P[k].grad = torch.randn(shapes[k], device=cuda_device, generator=g)
        grads = {k: P[k].grad.double().clone() for k in P}
        opt.step(it)
        for i, k in enumerate(training.PARAM_GROUPS):
            steps[k] += 1
            if k == "shN" and it <= 1000:
                continue
            gr = grads[k]
            # the kernel's coefficients are float32: beta = fl(0.9), 1 - beta = fl(1 - fl(0.9)) (adam_kernels.cuh:28-29)
            b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
            ob1, ob2 = float(np.float32(1) - np.float32(0.9)), float(np.float32(1) - np.float32(0.999))
            m[k] = b1 * m[k] + ob1 * gr
            v2[k] = b2 * v2[k] + ob2 * gr * gr
            bc1 = float(np.float32(1.0 / (1.0 - 0.9 ** steps[k])))
            bc2 = float(np.float32(1.0 / math.sqrt(1.0 - 0.999 ** steps[k])))
            ref[k] = ref[k] - float(np.float32(lr[i])) * bc1 * m[k] / (v2[k].sqrt() * bc2 + 1e-15)
        lr[0] *= 0.01 ** (1.0 / 100)
    for k in P:
        assert rel(P[k].detach(), ref[k]) < 1e-6, k
        assert rel(opt.exp_avg[k], m[k]) < 1e-6 and rel(opt.exp_avg_sq[k], v2[k]) < 1e-6, k


def test_training_iterations_reduce_the_loss_without_host_readback(native, cuda_device):
    """Five iterations of the whole step (fused render -> fused loss -> backward -> fused Adam) on a small scene: the loss
    falls, and with a capacity the step never reads anything back (n_isects stays on the device)."""
    from gsplat_b200 import training
    sc = scenes.scene_b(N=20000, width=640, height=360, view=2, scale_mul=2.0)
    t = to_dev(sc, cuda_device)
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    with torch.no_grad():
        tgt = native.rasterize_fused(raw["means"], raw["sh0"], raw["shN"], raw["scaling_raw"], raw["rotation_raw"],
                                     raw["opacity_raw"], 3, t["viewmats"], t["Ks"], 640, 360,
                                     bg_color=t["background"]).image.contiguous()
    g = torch.Generator(device=cuda_device).manual_seed(1)
    P = {k: (v + 0.05 * torch.randn(v.shape, device=cuda_device, generator=g)).detach().requires_grad_(True)
         for k, v in raw.items()}
    step = training.TrainStep(P, 3, 640, 360, optimizer=training.FusedAdam(P, training.AdamConfig(means_lr=1.6e-3)))
    n = step.size_capacity(t["viewmats"], t["Ks"], tgt, t["background"])
    assert step.capacity > n > 10000
    losses = [step(t["viewmats"], t["Ks"], tgt, t["background"]) for _ in range(6)]
    vals = [float(l) for l in losses]
    print("losses", [f"{v:.5f}" for v in vals], "intersections", int(step.last["n_isects"].item()))
    assert vals[-1] < vals[0] and all(math.isfinite(v) for v in vals)
    assert int(step.last["n_isects"].item()) <= step.capacity


def test_graphed_iteration_equals_eager_iteration(native, cuda_device):
    """GraphedTrainStep (one CUDA-graph launch per iteration) moves the parameters exactly like the eager TrainStep."""
    from gsplat_b200 import training
    sc = scenes.scene_b(N=20000, width=640, height=360, view=2, scale_mul=2.0)
    t = to_dev(sc, cuda_device)
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    g = torch.Generator(device=cuda_device).manual_seed(3)
    tgt = torch.rand((3, 360, 640), device=cuda_device, generator=g)
    cfg = training.AdamConfig(means_lr=1.6e-3)
    A = {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}
    B = {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}
    eager = training.TrainStep(A, 3, 640, 360, optimizer=training.FusedAdam(A, cfg))
    eager.size_capacity(t["viewmats"], t["Ks"], tgt, t["background"])
    graphed = training.GraphedTrainStep(B, 3, 640, 360, cfg)
    la, lb = [], []
    for it in range(4):
        la.append(float(eager(t["viewmats"], t["Ks"], tgt, t["background"])))
        lb.append(float(graphed(t["viewmats"], t["Ks"], tgt, t["background"])))
    assert not graphed.overflowed()
    print("eager ", [f"{v:.6f}" for v in la])
    print("graph ", [f"{v:.6f}" for v in lb])
    for a, b in zip(la, lb):
        assert abs(a - b) < 2e-5 * max(1.0, abs(a))
    for k in A:  # blend gradients are accumulated with float atomics: equal up to summation order, then through Adam
        if A[k].numel():
            assert rel(B[k].detach(), A[k].detach()) < 1e-4, k


# ------------------------------------------------------------------------------------------
# the same rows against the REFERENCE's own kernels (oracle/_ref: ssim.cu and adam_kernels.cuh compiled unmodified)
# ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_train(native):
    from oracle import ref_ops
    if not ref_ops.available():
        pytest.skip("oracle/_ref/libgsplat_ref.so not built")
    from oracle import ref_train as rt
    try:
        ref_ops._ns().fusedssim
    except (AttributeError, RuntimeError):
        pytest.skip("oracle/_ref was built without the training kernels")
    return rt


@pytest.mark.parametrize("H,W", [(11, 11), (17, 33), (70, 150), (540, 960), (1080, 1920)])
def test_photometric_loss_vs_reference_kernels(native, ref_train, cuda_device, H, W):
    from gsplat_b200 import training
    g = torch.Generator(device=cuda_device).manual_seed(7)
    renders = (torch.rand((1, H, W, 3), device=cuda_device, generator=g) * 1.4 - 0.2)
    target = torch.rand((3, H, W), device=cuda_device, generator=g)
    a = renders.clone().requires_grad_(True)
    loss, _ = training.photometric_loss(a, target, 0.2)
    loss.backward()
    b = renders.clone().requires_grad_(True)
    image = torch.clamp(b[0].permute(2, 0, 1), 0.0, 1.0)  # rasterizer.cpp:401
    want = ref_train.ref_photometric_loss(image, target, 0.2)
    want.backward()
    print(f"[{H}x{W}] loss {float(loss):.7f} vs reference kernels {float(want):.7f}; grad rel_l2 {rel(a.grad, b.grad):.2e}")
    assert abs(float(loss) - float(want)) < 5e-6 * max(1.0, abs(float(want)))
    assert rel(a.grad, b.grad) < 1e-4


def test_fused_adam_vs_reference_kernel(native, ref_train, cuda_device):
    from gsplat_b200 import training
    g = torch.Generator(device=cuda_device).manual_seed(9)
    shapes = {"means": (5003, 3), "sh0": (5003, 1, 3), "shN": (5003, 15, 3), "scaling_raw": (5003, 3),
              "rotation_raw": (5003, 4), "opacity_raw": (5003, 1)}
    init = {k: torch.randn(s, device=cuda_device, generator=g) for k, s in shapes.items()}
    A = {k: v.clone().requires_grad_(True) for k, v in init.items()}
    B = {k: v.clone().requires_grad_(True) for k, v in init.items()}
    cfg = training.AdamConfig(iterations=50)
    mine, theirs = training.FusedAdam(A, cfg), ref_train.RefFusedAdam(B, cfg.lrs(), iterations=50)
    for it in (1, 2, 3, 1200, 1201):
        for k in shapes:
            gr = torch.randn(shapes[k], device=cuda_device, generator=g)
            A[k].grad, B[k].grad = gr.clone(), gr.clone()
        mine.step(it)
        theirs.step(it, training.PARAM_GROUPS)
    for k in shapes:  # same float32 formula; the reference build is --use_fast_math (approximate sqrt / division)
        assert rel(A[k].detach(), B[k].detach()) < 2e-6, k
        assert rel(mine.exp_avg[k], theirs.m[k]) < 2e-6 and rel(mine.exp_avg_sq[k], theirs.v[k]) < 2e-6, k
