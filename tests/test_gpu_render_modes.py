"""GPU: the depth render modes (RenderMode D / ED / RGB_D / RGB_ED, rasterizer.cpp:272-420) -- the blend operators at 1
and 4 channels against the float64 oracle, and the fused operator's RenderMode overloads against the unfused mirror.

The blend is independent per channel: the forward is  render_k = sum_i c_ik alpha_i T_i + T_final bg_k,  and alpha /
last_ids do not depend on colour; for fixed geometry the backward's geometry gradient is a sum of one term per channel
plus the alpha term.  So the 3-channel oracle gives exact 1- and 4-channel references: one call with channels 0..2 and
the alpha cotangent, one with (c3, 0, 0), (v3, 0, 0), background (bg3, 0, 0) and a zero alpha cotangent; geometry
gradients add, colour gradients are read per call.  NC = 1 is the second call alone, with the alpha cotangent."""
import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel, to_dev
from test_gpu_parity import DISTORTED

pytestmark = pytest.mark.gpu
RAW = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")
MODES = ("RGB", "D", "ED", "RGB_D", "RGB_ED")


def _pad3(x):
    """[..., 1] -> [..., 3] with two zero channels."""
    return np.concatenate([x, np.zeros(x.shape[:-1] + (2,), x.dtype)], -1)


def oracle_nc(orc, sc, colors, bg, masks, off, flat, vrc, vra, okw):
    """Forward (f32) and backward (f64) of the NC-channel blend by the decomposition above."""
    W, H = sc["width"], sc["height"]
    nc = colors.shape[-1]
    geo = (sc["means"], sc["quats"], sc["scales"])
    common = dict(masks=masks, width=W, height=H, tile_size=16, viewmats=sc["viewmats"], Ks=sc["Ks"], tile_offsets=off,
                  flatten_ids=flat, **okw)
    op = sc["opacities"][None]
    calls = []  # (colors [1,N,3], bg [1,3] | None, v colours, v alpha)
    if nc == 4:
        calls.append((colors[..., :3], None if bg is None else bg[..., :3], vrc[..., :3], vra))
    last = lambda x: _pad3(x[..., -1:])
    calls.append((last(colors), None if bg is None else last(bg), last(vrc), vra if nc == 1 else np.zeros_like(vra)))
    fw = [orc.raster_fwd(*geo, np.ascontiguousarray(c), op, b, **common) for c, b, _, _ in calls]
    renders = np.concatenate([fw[0][0]] + ([fw[1][0][..., :1]] if nc == 4 else []), -1) if nc == 4 else fw[0][0][..., :1]
    alphas, last_ids = fw[0][1], fw[0][2]
    grads = None
    for (c, b, v, va) in calls:
        g = orc.raster_bwd(*geo, np.ascontiguousarray(c), op, b, render_alphas=alphas, last_ids=last_ids,
                           v_render_colors=np.ascontiguousarray(v), v_render_alphas=va, precision="f64", **common)
        if grads is None:
            grads = [g[0], g[1], g[2], [g[3]], g[4]]
        else:
            for k in (0, 1, 2, 4):
                grads[k] = grads[k] + g[k]
            grads[3].append(g[3])
    vc = grads[3]
    grads[3] = np.concatenate([vc[0], vc[1][..., :1]], -1) if nc == 4 else vc[0][..., :1]
    return renders, alphas, last_ids, grads


def _scene(name):
    if name == "a":
        return scenes.scene_a(background=False)
    if name == "small_rot":
        return scenes.scene_small(N=3000, width=200, height=120, view=1)
    if name == "b30k":  # 640x360: the two-pixel backward
        return scenes.scene_b(N=30000, width=640, height=360, view=3, scale_mul=2.0)
    if name == "b30k_wide":  # 1284x723: 81 x 46 tiles, enough for the four-pixel backward on any H100
        return scenes.scene_b(N=30000, width=1284, height=723, view=3, scale_mul=2.0)
    raise KeyError(name)


def _camera(model, dev):
    if model == "pinhole":
        return {}, {}
    cfg = DISTORTED[model]
    okw = dict(camera_model=cfg["camera_model"], radial=cfg["radial"], tangential=cfg["tangential"],
               thin_prism=cfg["thin_prism"])
    d = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    nkw = dict(camera_model=cfg["camera_model"], radial_coeffs=d(cfg["radial"]), tangential_coeffs=d(cfg["tangential"]),
               thin_prism_coeffs=d(cfg["thin_prism"]))
    return okw, nkw


def _lists(orc, sc, okw):
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    radii, m2d, depths, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"],
                                                 sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **okw)
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, tw, th)
    return depths, orc.isect_offsets(ids, 1, tw, th), flat


CASES = [  # (scene, camera, channels, background, masks)
    ("a", "pinhole", 1, False, False), ("a", "pinhole", 4, True, False),
    ("small_rot", "pinhole", 1, True, True), ("small_rot", "pinhole", 4, False, True),
    ("small_rot", "opencv", 4, True, False), ("small_rot", "fisheye", 1, True, False),
    ("small_rot", "fisheye", 4, False, False), ("small_rot", "opencv", 1, False, False),
    ("b30k", "pinhole", 4, True, False), ("b30k", "pinhole", 1, False, False),
    ("b30k_wide", "pinhole", 4, True, False), ("b30k_wide", "opencv", 1, True, False),
]


@pytest.mark.parametrize("name,model,nc,with_bg,with_masks", CASES)
def test_blend_nc_vs_oracle(native, orc, cuda_device, name, model, nc, with_bg, with_masks):
    sc = _scene(name)
    W, H = sc["width"], sc["height"]
    n_g = sc["means"].shape[0]
    okw, nkw = _camera(model, cuda_device)
    depths, off, flat = _lists(orc, sc, okw)
    rng = np.random.default_rng(5)
    rgb = rng.random((1, n_g, 3), dtype=np.float32)
    colors = np.ascontiguousarray(depths[..., None] if nc == 1 else np.concatenate([rgb, depths[..., None]], -1))
    bg = rng.random((1, nc), dtype=np.float32) if with_bg else None
    masks = None
    if with_masks:
        tw, th = (W + 15) // 16, (H + 15) // 16
        masks = np.ones((1, th, tw), bool)
        masks[0, 1, 2] = masks[0, th - 1, 0] = False
    vrc = rng.standard_normal((1, H, W, nc)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    r_ref, a_ref, l_ref, g_ref = oracle_nc(orc, sc, colors, bg, masks, off, flat, vrc, vra, okw)

    t = to_dev(sc, cuda_device)
    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    args = (t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], d(bg), d(masks), W, H, 16,
            t["viewmats"], t["Ks"], d(off), d(flat))
    r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(*args, **nkw)
    r, a, li = r.cpu().numpy(), a.cpu().numpy(), li.cpu().numpy()
    assert r.shape == (1, H, W, nc)
    # a masked tile gets the background; its alphas / last_ids are left as they were (Fwd.cu:143-150)
    live = np.ones((H, W), bool) if masks is None else np.repeat(np.repeat(masks[0], 16, 0), 16, 1)[:H, :W]
    e_img, e_alpha = rel(r, r_ref), rel(a[0][live], a_ref[0][live])
    print(f"[{name} {model} NC={nc} bg={with_bg} masks={with_masks}] rel_l2 render {e_img:.2e} alpha {e_alpha:.2e}")
    assert e_img < 1e-4 and e_alpha < 1e-4
    assert (li[0][live] != l_ref[0][live]).mean() < 2e-3

    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*args, d(a_ref), d(l_ref), d(vrc), d(vra), **nkw)
    # Depth alone (NC = 1): camera-space depths are an order of magnitude larger than colours, and the float32
    # cancellation in the blend's v_alpha (colour in front against colour behind) grows with them.  On the b30k scenes
    # the geometry gradients come out ~1.2e-3 from the float64 oracle; the 3-channel kernel, fed (depth, 0, 0), gives
    # the same gradients (checked below), so the bound is the blend's float32 arithmetic on these inputs.
    rel_tol = 2e-3 if nc == 1 else 1e-3
    for nm, got, want in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g, g_ref):
        got = got.cpu().numpy().reshape(want.shape)
        assert_grad_close(got, want, nm, n_g, rel_tol=rel_tol, tag=f"{name} {model} NC={nc} vs f64 oracle")
        untouched = np.abs(want).reshape(n_g, -1).sum(-1) == 0
        assert np.all(got.reshape(n_g, -1)[untouched] == 0)
    if nc == 1:  # the same blend through the 3-channel kernels, colours (depth, 0, 0)
        pad = lambda x: None if x is None else np.concatenate([x, np.zeros(x.shape[:-1] + (2,), np.float32)], -1)
        args3 = (t["means"], t["quats"], t["scales"], d(pad(colors)), t["opacities"][None], d(pad(bg)), d(masks), W, H,
                 16, t["viewmats"], t["Ks"], d(off), d(flat))
        r3, _, _ = native.rasterize_to_pixels_from_world_3dgs_fwd(*args3, **nkw)
        assert np.array_equal(r3.cpu().numpy()[..., :1], r)
        g3 = native.rasterize_to_pixels_from_world_3dgs_bwd(*args3, d(a_ref), d(l_ref), d(pad(vrc)), d(vra), **nkw)
        for nm, x1, x3 in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g, g3):
            x3 = x3[..., :1] if nm == "v_colors" else x3
            assert rel(x1.cpu().numpy(), x3.cpu().numpy()) < 1e-5, nm


@pytest.mark.parametrize("name,model", [("small_rot", "pinhole"), ("b30k_wide", "pinhole"), ("small_rot", "fisheye")])
def test_four_channels_extend_the_rgb_blend(native, orc, cuda_device, name, model):
    """At NC = 4 the first three channels, alphas and last_ids are the 3-channel call's bit for bit; with a zero
    cotangent on the fourth channel the gradients are the 3-channel backward's up to float32 round-off."""
    sc = _scene(name)
    W, H = sc["width"], sc["height"]
    okw, nkw = _camera(model, cuda_device)
    depths, off, flat = _lists(orc, sc, okw)
    t = to_dev(sc, cuda_device)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    rgb = np.random.default_rng(8).random((1, sc["means"].shape[0], 3), dtype=np.float32)
    bg3 = np.array([[0.2, 0.5, 0.7]], np.float32)
    out = {}
    for nc in (3, 4):
        colors = rgb if nc == 3 else np.concatenate([rgb, depths[..., None]], -1)
        bg = bg3 if nc == 3 else np.concatenate([bg3, [[0.0]]], -1).astype(np.float32)
        args = (t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], d(bg), None, W, H, 16,
                t["viewmats"], t["Ks"], d(off), d(flat))
        r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(*args, **nkw)
        g = torch.Generator(device=cuda_device).manual_seed(1)
        v3 = torch.randn((1, H, W, 3), device=cuda_device, generator=g)
        va = torch.randn((1, H, W, 1), device=cuda_device, generator=g)
        v = v3 if nc == 3 else torch.cat([v3, torch.zeros_like(v3[..., :1])], -1)
        grads = native.rasterize_to_pixels_from_world_3dgs_bwd(*args, a, li, v.contiguous(), va, **nkw)
        out[nc] = (r, a, li, grads)
    r3, a3, l3, g3 = out[3]
    r4, a4, l4, g4 = out[4]
    assert torch.equal(r4[..., :3], r3) and torch.equal(a4, a3) and torch.equal(l4, l3)
    for nm, x3, x4 in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g3, g4):
        if nm == "v_colors":
            x4 = x4[..., :3]
        e = rel(x4.cpu().numpy(), x3.cpu().numpy())
        print(f"[{name} {model}] {nm}: NC=4 with a zero depth cotangent vs NC=3: rel_l2 {e:.2e}")
        assert e < 1e-5, (nm, e)


def _run_mode(native, t, sc, dev, mode, fused, seed=0):
    W, H = sc["width"], sc["height"]
    raw = native.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    g = torch.Generator(device=dev).manual_seed(seed)
    raw["rotation_raw"] = raw["rotation_raw"] * (torch.rand((raw["means"].shape[0], 1), device=dev, generator=g) + 0.5)
    P = {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}
    kw = dict(bg_color=t.get("background"), render_mode=mode)
    if fused:
        o = native.rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"],
                                   P["opacity_raw"], sc["sh_degree"], t["viewmats"], t["Ks"], W, H, **kw)
        image, depth, alpha = o.image, o.depth, o.alpha.permute(0, 3, 1, 2)[0]
    else:
        o = native.rasterize_from_raw(P, sc["sh_degree"], t["viewmats"], t["Ks"], W, H, **kw)
        image, depth, alpha = o.image, o.depth, o.alpha
    loss = (alpha * torch.randn(alpha.shape, device=dev, generator=g)).sum()
    for x in (image, depth):
        if x is not None:
            loss = loss + (x * torch.randn(x.shape, device=dev, generator=g)).sum()
    loss.backward()
    grads = {k: (P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])) for k in RAW}
    return image, depth, alpha, grads


@pytest.mark.parametrize("mode", MODES)
def test_fused_modes_match_unfused(native, cuda_device, mode):
    sc = scenes.scene_small(N=3000, width=200, height=120, view=1)
    n_g = sc["means"].shape[0]
    t = to_dev(sc, cuda_device)
    fi, fd, fa, fg = _run_mode(native, t, sc, cuda_device, mode, fused=True)
    ui, ud, ua, ug = _run_mode(native, t, sc, cuda_device, mode, fused=False)
    assert (fi is None) == (ui is None) == (mode in ("D", "ED"))
    assert (fd is None) == (ud is None) == (mode == "RGB")
    assert rel(fa, ua) < 1e-5
    if fi is not None:
        assert fi.shape == (3, 120, 200) and rel(fi, ui) < 1e-5
    if fd is not None:
        assert fd.shape == (1, 120, 200) and rel(fd, ud) < 1e-5
    for k in RAW:
        assert_grad_close(fg[k], ug[k], k, n_g, rel_tol=2e-4, tag=f"{mode} fused vs unfused")
    if mode in ("D", "ED"):  # the depth is not differentiable: no colour gradient reaches the SH coefficients
        assert torch.count_nonzero(fg["sh0"]) == 0 and torch.count_nonzero(fg["shN"]) == 0
        assert torch.count_nonzero(ug["sh0"]) == 0 and torch.count_nonzero(ug["shN"]) == 0


@pytest.mark.parametrize("mode", ["ED", "RGB_ED"])
def test_expected_depth_chain_rule(native, orc, cuda_device, mode):
    """ED = acc / max(alpha, 1e-10): the mirror's gradients equal the operator backward fed with the chain-rule
    cotangents, computed in float64 from the oracle forward."""
    sc = scenes.scene_small(N=3000, width=200, height=120, view=1)
    W, H = sc["width"], sc["height"]
    t = to_dev(sc, cuda_device)
    nc = 1 if mode == "ED" else 4
    # the mirror, on activated parameters
    # both sides get the oracle's projection, so that their intersection lists are the same
    ref = orc.render_pipeline(sc, "f32")
    proj = tuple(torch.from_numpy(ref[k]).to(cuda_device) for k in ("radii", "means2d", "depths"))
    P = {k: t[k].detach().clone().requires_grad_(True) for k in ("means", "quats", "scales", "opacities")}
    o = native.rasterize(P["means"], P["quats"], P["scales"], P["opacities"], t["sh_coeffs"], sc["sh_degree"],
                         t["viewmats"], t["Ks"], W, H, bg_color=t.get("background"), render_mode=mode, projection=proj)
    g = torch.Generator(device=cuda_device).manual_seed(3)
    v_ed = torch.randn((1, H, W), device=cuda_device, generator=g)
    v_al = torch.randn((1, H, W), device=cuda_device, generator=g)
    v_im = torch.randn((3, H, W), device=cuda_device, generator=g) if nc == 4 else None
    loss = (o.depth * v_ed).sum() + (o.alpha * v_al).sum()
    if v_im is not None:
        loss = loss + (o.image * v_im).sum()
    loss.backward()
    # the operator backward with cotangents from the oracle forward, chain rule in float64
    depths = ref["depths"]
    colors = depths[..., None] if nc == 1 else np.concatenate([ref["colors"], depths[..., None]], -1)
    colors = np.ascontiguousarray(colors.astype(np.float32))
    bg = sc.get("background")
    bgn = None if bg is None else (np.zeros((1, 1), np.float32) if nc == 1 else
                                   np.concatenate([bg, np.zeros((1, 1), np.float32)], -1))
    zero = np.zeros((1, H, W, nc), np.float32)
    r, a, li, _ = oracle_nc(orc, sc, colors, bgn, None, ref["tile_offsets"], ref["flatten_ids"], zero, zero[..., :1], {})
    acc, al = r[..., -1].astype(np.float64), a[..., 0].astype(np.float64)
    ved, val = v_ed.cpu().numpy().astype(np.float64), v_al.cpu().numpy().astype(np.float64)
    v_acc = ved / np.maximum(al, 1e-10)
    v_alpha = val - ved * acc / np.maximum(al, 1e-10) ** 2 * (al > 1e-10)
    vrc = v_acc[..., None]
    if nc == 4:  # clamp(image, 0, 1) backward
        img = r[0, ..., :3].transpose(2, 0, 1)
        vi = v_im.cpu().numpy() * ((img >= 0) & (img <= 1))
        vrc = np.concatenate([vi.transpose(1, 2, 0)[None], vrc], -1)
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(cuda_device)
    di = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.int32)).to(cuda_device)
    gk = native.rasterize_to_pixels_from_world_3dgs_bwd(
        t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], None if bgn is None else d(bgn), None,
        W, H, 16, t["viewmats"], t["Ks"], di(ref["tile_offsets"]), di(ref["flatten_ids"]), d(a), di(li), d(vrc),
        d(v_alpha[..., None]))
    n_g = sc["means"].shape[0]
    for nm, key, want in (("v_means", "means", gk[0]), ("v_quats", "quats", gk[1]), ("v_scales", "scales", gk[2]),
                          ("v_opacities", "opacities", gk[4][0])):
        got = P[key].grad
        if nc == 4 and nm == "v_means":  # the SH direction gradient reaches the means too: compare blend-only terms
            continue
        assert_grad_close(got.cpu().numpy(), want.cpu().numpy().reshape(got.shape), nm, n_g, rel_tol=2e-4,
                          tag=f"{mode} mirror vs operator with chain-rule cotangents")


@pytest.mark.parametrize("nc", [1, 4])
@pytest.mark.parametrize("n", [5, 0])
def test_blend_nc_empty_inputs(native, cuda_device, nc, n):
    dev = cuda_device
    W, H = 64, 48
    vm = torch.eye(4, device=dev)[None]
    K = torch.tensor([[[50.0, 0, 32], [0, 50.0, 24], [0, 0, 1]]], device=dev)
    means = torch.zeros(n, 3, device=dev); means[:, 2] = 3
    quats = torch.tensor([[1.0, 0, 0, 0]], device=dev).repeat(n, 1)
    scales = torch.full((n, 3), 0.1, device=dev)
    colors = torch.rand(1, n, nc, device=dev)
    opac = torch.full((1, n), 0.5, device=dev)
    off = torch.zeros(1, 3, 4, dtype=torch.int32, device=dev)
    flat = torch.zeros(0, dtype=torch.int32, device=dev)
    bg = torch.rand(1, nc, device=dev)
    r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(means, quats, scales, colors, opac, bg, None, W, H, 16, vm,
                                                              K, off, flat)
    assert r.shape == (1, H, W, nc)
    assert torch.equal(r, bg.view(1, 1, 1, nc).expand(1, H, W, nc)) and float(a.abs().max()) == 0
    assert int(li.abs().max()) == 0
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(means, quats, scales, colors, opac, bg, None, W, H, 16, vm, K, off,
                                                       flat, a, li, torch.ones_like(r), torch.ones_like(a))
    assert g[3].shape == (1, n, nc)
    assert all(x.numel() == 0 or float(x.abs().max()) == 0 for x in g)


@pytest.mark.parametrize("mode", MODES)
def test_modes_zero_intersections(native, cuda_device, mode):
    """Every Gaussian behind the camera: no intersection; the background and zero gradients in every mode, fused and
    unfused alike."""
    dev = cuda_device
    W, H, n = 64, 48, 5
    vm = torch.eye(4, device=dev)[None]
    K = torch.tensor([[[50.0, 0, 32], [0, 50.0, 24], [0, 0, 1]]], device=dev)
    bg = torch.tensor([[0.1, 0.2, 0.3]], device=dev)
    nc = {"RGB": 3, "D": 1, "ED": 1, "RGB_D": 4, "RGB_ED": 4}[mode]
    raw = dict(means=torch.tensor([[0.0, 0.0, -3.0]], device=dev).repeat(n, 1), sh0=torch.rand(n, 1, 3, device=dev),
               shN=torch.zeros(n, 15, 3, device=dev), scaling_raw=torch.full((n, 3), -2.3, device=dev),
               rotation_raw=torch.tensor([[1.0, 0, 0, 0]], device=dev).repeat(n, 1),
               opacity_raw=torch.zeros(n, 1, device=dev))
    for fused in (True, False):
        P = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
        if fused:
            o = native.rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"],
                                       P["opacity_raw"], 3, vm, K, W, H, bg_color=bg, render_mode=mode)
            assert int(o.n_isects.item()) == 0
        else:
            o = native.rasterize_from_raw(P, 3, vm, K, W, H, bg_color=bg, render_mode=mode)
            assert o.n_isects == 0
        assert o.render_colors.shape == (1, H, W, nc)
        want = bg if nc == 3 else (torch.zeros(1, 1, device=dev) if nc == 1 else torch.cat([bg, bg[:, :1] * 0], -1))
        assert torch.equal(o.render_colors.detach(), want.view(1, 1, 1, nc).expand(1, H, W, nc))
        (o.render_colors.sum() + o.alpha.sum()).backward()
        assert all(P[k].grad is None or torch.count_nonzero(P[k].grad) == 0 for k in RAW)
        assert (o.image is None) == (mode in ("D", "ED")) and (o.depth is None) == (mode == "RGB")
