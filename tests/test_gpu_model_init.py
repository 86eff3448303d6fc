"""GPU: the exact mean neighbour distance (csrc/gsb_knn.cu) and the model set-up and export built on it (model.py).

  * bitwise equal to the float32 restatement (knn_restatement.py) on the hand-made clouds and on 1e5 and 1e6 points of
    the uniform, SfM-like and outlier-laden shapes; at most the reference's approximate distances on the stored fixture;
  * repeatable bit for bit, and capturable in a CUDA graph; non-finite coordinates raise;
  * init_model_from_pointcloud against the reference's torch composition on the same device, both branches;
  * end to end: set-up from points of a scenes.py model, 50 MCMC training iterations, save_ply / load_ply, and the
    loaded model renders the image of the trained one."""
import importlib
import os
import time

import numpy as np
import pytest
import torch

import knn_restatement as kr
import scenes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


@pytest.fixture(scope="module")
def model(native):
    return importlib.import_module(native.__name__ + ".model")


@pytest.fixture(scope="module")
def ops(native):
    return torch.ops.gsplat_b200


def gpu_dist(ops, pts, dev):
    out = ops.mean_neighbor_distances(torch.from_numpy(np.ascontiguousarray(pts, F32)).to(dev))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def assert_bitwise(got, want, label):
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert len(bad) == 0, f"{label}: {len(bad)} of {len(want)} differ, e.g. {[(int(i), got[i], want[i]) for i in bad[:5]]}"


@pytest.mark.parametrize("case", sorted(kr.hand_cases()))
def test_kernel_equals_restatement_on_hand_made_clouds(ops, cuda_device, case):
    pts = kr.hand_cases()[case]
    assert_bitwise(gpu_dist(ops, pts, cuda_device), kr.mean_neighbor_distances(pts), case)


@pytest.mark.parametrize("n", [100_000, 1_000_000])
@pytest.mark.parametrize("shape", sorted(kr.CLOUDS))
def test_kernel_equals_restatement_on_large_clouds(ops, cuda_device, shape, n):
    pts = kr.CLOUDS[shape](n, seed=21)
    got = gpu_dist(ops, pts, cuda_device)
    assert_bitwise(got, kr.mean_neighbor_distances(pts), f"{shape} {n}")


def test_kernel_is_at_most_the_stored_reference(ops, cuda_device):
    z = np.load(os.path.join(ROOT, "tests", "golden", "knn_ref_small.npz"))
    got = gpu_dist(ops, z["points"], cuda_device)
    assert (got <= z["ref"]).all()
    print(f"the reference's approximate distances differ from the exact ones at {100 * float((got != z['ref']).mean()):.2f}%"
          f" of {len(got)} points")


def test_repeatable_and_graph_capturable(ops, cuda_device):
    pts = torch.from_numpy(kr.cloud_outliers(200_000, seed=5)).to(cuda_device)
    a = ops.mean_neighbor_distances(pts)
    b = ops.mean_neighbor_distances(pts)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    out = torch.full_like(a, -1.0)
    status = torch.full((1,), -1, dtype=torch.int32, device=cuda_device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside the capture
        ops.mean_neighbor_distances_out(pts, out, status)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.mean_neighbor_distances_out(pts, out, status)
    out.fill_(-1.0)
    status.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(out.view(torch.int32), a.view(torch.int32))
    # the same graph on moved points: the statistics and the grid are recomputed on the device
    pts.mul_(3.0).add_(1.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), ops.mean_neighbor_distances(pts).view(torch.int32))


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_points_raise(ops, cuda_device, bad):
    pts = torch.rand(1000, 3, device=cuda_device)
    pts[517, 1] = bad
    with pytest.raises(RuntimeError, match="finite"):
        ops.mean_neighbor_distances(pts)
    with pytest.raises(RuntimeError):
        ops.mean_neighbor_distances(pts[517:518].clone())  # a single non-finite point as well
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    ops.mean_neighbor_distances_out(pts, torch.empty(1000, device=cuda_device), status)
    assert int(status.item()) == 1  # GSB_KNN_NONFINITE


def test_bad_arguments_raise(ops, cuda_device):
    with pytest.raises(RuntimeError):
        ops.mean_neighbor_distances(torch.rand(10, 3))  # CPU
    with pytest.raises(RuntimeError):
        ops.mean_neighbor_distances(torch.rand(10, 3, device=cuda_device, dtype=torch.float64))
    with pytest.raises(RuntimeError):
        ops.mean_neighbor_distances(torch.rand(10, 4, device=cuda_device))
    assert ops.mean_neighbor_distances(torch.empty(0, 3, device=cuda_device)).shape == (0,)
    # a strided view is taken as its contiguous copy
    p = torch.rand(500, 6, device=cuda_device)[:, ::2]
    assert torch.equal(ops.mean_neighbor_distances(p), ops.mean_neighbor_distances(p.contiguous()))


def test_outlier_cloud_of_a_million_points_finishes(ops, cuda_device):
    pts = torch.from_numpy(kr.cloud_outliers(1_000_000, seed=8, frac=1e-2)).to(cuda_device)
    ops.mean_neighbor_distances(pts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ops.mean_neighbor_distances(pts)
    torch.cuda.synchronize()
    print(f"1e6 points, 1% far outliers: {1e3 * (time.perf_counter() - t0):.2f} ms "
          f"({torch.cuda.get_device_name()})")


# ---- set-up ------------------------------------------------------------------------------------------------------------
def reference_composition(positions, colors, center, cfg, dists_fn):
    """splat_data.cpp:516-591 written out with torch, as a second statement of the order of operations."""
    dists = torch.norm(positions - center, 2, 1)
    scale = dists.median().item()
    means = positions * scale if cfg.random else positions
    nn = torch.clamp_min(dists_fn(means), 1e-7)
    scaling = torch.log(torch.sqrt(nn) * float(np.float32(cfg.init_scaling))).unsqueeze(-1).repeat(1, 3)
    N = means.shape[0]
    rot = torch.zeros(N, 4, device=means.device)
    rot[:, 0] = 1
    opac = torch.logit(float(np.float32(cfg.init_opacity)) * torch.ones(N, 1, device=means.device))
    fused = (colors - 0.5) / float(np.float32(0.28209479177387814))
    shs = torch.zeros(N, 3, (cfg.sh_degree + 1) ** 2, device=means.device)
    shs[:, :, 0] = fused
    return dict(means=means, sh0=shs[:, :, :1].transpose(1, 2), shN=shs[:, :, 1:].transpose(1, 2),
                scaling_raw=scaling, rotation_raw=rot, opacity_raw=opac), scale


@pytest.mark.parametrize("random_init", [False, True])
def test_init_equals_the_reference_composition(model, ops, cuda_device, random_init):
    cfg = model.InitConfig(sh_degree=3, random=random_init, init_num_pts=20000)
    center = torch.tensor([0.1, -0.2, 0.3])
    if random_init:
        torch.manual_seed(77)
        P, scale, deg = model.init_model_from_pointcloud(None, None, center, cfg)
        torch.manual_seed(77)
        positions = (torch.rand((20000, 3), device=cuda_device) * 2.0 - 1.0) * float(np.float32(3.0))
        colors = torch.rand((20000, 3), device=cuda_device)
    else:
        pos, col = model.random_point_cloud(30000)
        positions = pos.to(cuda_device)
        P, scale, deg = model.init_model_from_pointcloud(positions, col.to(cuda_device), center, cfg)
        colors = col.to(cuda_device) / 255.0
    ref, ref_scale = reference_composition(positions, colors, center.to(cuda_device), cfg, ops.mean_neighbor_distances)
    assert deg == 3 and scale == ref_scale
    for k, v in ref.items():
        assert P[k].is_cuda and P[k].requires_grad and P[k].is_contiguous(), k
        assert P[k].shape == v.shape and torch.equal(P[k].detach(), v), k


def test_train_save_load_renders_the_same_image(model, native, cuda_device, tmp_path):
    training = importlib.import_module(native.__name__ + ".training")
    mc = importlib.import_module(native.__name__ + ".mcmc")
    sc = scenes.scene_b(N=20000, width=320, height=180, view=2, scale_mul=2.0)
    t = {k: torch.from_numpy(v).to(cuda_device) for k, v in sc.items() if isinstance(v, np.ndarray)}
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    with torch.no_grad():
        target = native.rasterize_fused(raw["means"], raw["sh0"], raw["shN"], raw["scaling_raw"], raw["rotation_raw"],
                                        raw["opacity_raw"], 3, t["viewmats"], t["Ks"], 320, 180,
                                        bg_color=t["background"]).image.contiguous()
    g = torch.Generator().manual_seed(4)
    pick = torch.randperm(20000, generator=g)[:6000]
    points = t["means"][pick].cpu()
    colors = torch.randint(0, 256, (6000, 3), dtype=torch.uint8, generator=g)
    P, scene_scale, deg = model.init_model_from_pointcloud(points, colors, points.mean(0), model.InitConfig(sh_degree=3))
    assert np.isfinite(P["scaling_raw"].detach().cpu().numpy()).all()
    opt = training.FusedAdam(P, training.AdamConfig(means_lr=1.6e-4 * scene_scale))
    strat = mc.MCMC(P, opt, mc.MCMCConfig(start_refine=10, refine_every=10, max_cap=7000), sh_degree=3)
    step = training.TrainStep(P, deg, 320, 180, optimizer=opt, strategy=strat)
    losses = [float(step(t["viewmats"], t["Ks"], target, t["background"])) for _ in range(50)]
    print(f"loss {losses[0]:.4f} -> {losses[-1]:.4f}, {step.params['means'].shape[0]} Gaussians")
    assert losses[-1] < losses[0]

    trained = {k: v.detach() for k, v in step.params.items()}
    path = tmp_path / "trained.ply"
    model.save_ply(trained, path)
    Q, q_scale, q_deg = model.load_ply(path)
    assert q_deg == 3 and q_scale == 0.5
    mem = dict(trained, rotation_raw=torch.nn.functional.normalize(trained["rotation_raw"], dim=-1))
    for k in mem:
        assert torch.equal(Q[k].detach(), mem[k].reshape(Q[k].shape)), k

    def render(p):
        with torch.no_grad():
            return native.rasterize_fused(p["means"], p["sh0"], p["shN"], p["scaling_raw"], p["rotation_raw"],
                                          p["opacity_raw"], 3, t["viewmats"], t["Ks"], 320, 180,
                                          bg_color=t["background"]).image
    a, b = render(mem), render({k: v.detach() for k, v in Q.items()})
    err = float((a - b).abs().max())
    print(f"max |image(loaded) - image(in memory)| = {err:.3g}")
    assert err <= 1e-6
