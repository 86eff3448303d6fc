"""CPU tests of the fastgs (EWA) oracle, SURVEY.md 8 f4 (oracle/fastgs_oracle.c).

The reference holds no test vectors for this path; the oracle is pinned to the reference's own kernels on the GPU box
(tests/test_gpu_fastgs.py).  Here: self-consistency -- the analytic backward against central differences of the smooth
float64 build, float32 against float64, and the structural properties of the forward."""
import numpy as np
import pytest

import scenes
from oracle import fastgs_oracle as fgo


def _scene(n=60, w=72, h=56, deg=3, view=1, seed=5):
    sc = scenes.scene_small(N=n, width=w, height=h, sh_degree=deg, seed=seed, view=view)
    return scenes.fastgs_inputs(sc)


def _loss_weights(inp, seed=0):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((3, inp["height"], inp["width"])).astype(np.float32),
            rng.standard_normal((1, inp["height"], inp["width"])).astype(np.float32))


def _render(inp, precision, **kw):
    args = {k: inp[k] for k in ("means", "scales_raw", "rotations_raw", "opacities_raw", "sh0", "shN", "w2c",
                                 "cam_position", "active_sh_bases", "width", "height", "fx", "fy", "cx", "cy",
                                 "near_plane", "far_plane")}
    return fgo.render(**args, precision=precision, **kw)


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_backward_matches_central_differences(deg):
    inp = _scene(n=40, deg=deg)
    gi, ga = _loss_weights(inp)
    out = _render(inp, "f64s", grad_image=gi, grad_alpha=ga, want_w2c_grad=True)

    def loss(x):
        o = _render(x, "f64s")
        return float((o["image"].astype(np.float64) * gi).sum() + (o["alpha"].astype(np.float64) * ga).sum())

    rng = np.random.default_rng(1)
    eps = 2.0 ** -9  # exactly representable steps: the interface arrays are float32, outputs float32
    for key, gkey in (("means", "grad_means"), ("scales_raw", "grad_scales_raw"), ("rotations_raw", "grad_rotations_raw"),
                      ("opacities_raw", "grad_opacities_raw"), ("sh0", "grad_sh0"), ("shN", "grad_shN"), ("w2c", "grad_w2c")):
        if inp[key].size == 0:
            continue
        d = rng.standard_normal(inp[key].shape).astype(np.float32)
        if key == "w2c":
            d[3] = 0  # the last row is not a parameter
            d[:3, :3] *= 0.05
        d = (np.round(d * 64) / 64).astype(np.float32)
        step = np.float32(eps * (0.05 if key in ("means", "w2c") else 1.0))
        plus, minus = dict(inp), dict(inp)
        plus[key] = (inp[key] + step * d).astype(np.float32)
        minus[key] = (inp[key] - step * d).astype(np.float32)
        if key == "w2c":  # the camera position is not tied to w2c in this API: keep it fixed
            pass
        actual = (plus[key].astype(np.float64) - minus[key].astype(np.float64))
        fd = (loss(plus) - loss(minus))
        an = float((out[gkey].reshape(actual.shape) * actual).sum())
        # the rendered outputs are float32: the difference of two losses carries ~1e-7 * |loss| of rounding
        scale = max(abs(an), 1e-3)
        assert abs(fd - an) <= 2e-2 * scale + 2e-4, (key, fd, an)


def test_float32_agrees_with_float64():
    inp = _scene(n=300, w=120, h=88)
    gi, ga = _loss_weights(inp)
    a = _render(inp, "f32", grad_image=gi, grad_alpha=ga)
    b = _render(inp, "f64", grad_image=gi, grad_alpha=ga)
    assert np.abs(a["image"] - b["image"]).max() < 5e-3  # a threshold may flip a single contribution (<= 1/255 * colour)
    assert np.mean(np.abs(a["image"] - b["image"]) > 1e-4) < 5e-3
    for k in ("grad_means", "grad_scales_raw", "grad_rotations_raw", "grad_opacities_raw", "grad_sh0", "grad_shN"):
        den = np.linalg.norm(b[k]) + 1e-12
        assert np.linalg.norm(a[k] - b[k]) / den < 2e-2, k


def test_forward_properties():
    inp = _scene(n=200, w=100, h=70)
    out = _render(inp, "f32")
    img, al = out["image"], out["alpha"][0]
    assert img.shape == (3, 70, 100) and al.shape == (70, 100)
    assert (al >= 0).all() and (al <= 1 - 1e-4 + 1e-6).all()  # transmittance never drops below 1e-4
    assert (img >= 0).all()  # colours are clamped at zero before blending
    assert out["n_instances"] == int(out["n_touched"].sum())
    # a primitive behind the near plane or with negligible opacity is culled
    far = dict(inp)
    far["opacities_raw"] = np.full_like(inp["opacities_raw"], -12.0)
    o2 = _render(far, "f32")
    assert o2["n_instances"] == 0 and not o2["image"].any() and not o2["alpha"].any()
    # permuting the primitives does not change the picture (order is by depth)
    perm = np.random.default_rng(0).permutation(inp["means"].shape[0])
    p = dict(inp)
    for k in ("means", "scales_raw", "rotations_raw", "opacities_raw", "sh0", "shN"):
        p[k] = np.ascontiguousarray(inp[k][perm])
    o3 = _render(p, "f32")
    assert np.abs(o3["image"] - img).max() < 1e-5


def test_densification_info_accumulates():
    inp = _scene(n=50)
    gi, ga = _loss_weights(inp)
    dens = np.zeros((2, inp["means"].shape[0]), np.float32)
    out = _render(inp, "f32", grad_image=gi, grad_alpha=ga, densification_info=dens)
    d = out["densification_info"]
    vis = out["n_touched"] > 0
    assert (d[0][vis] == 1).all() and (d[0][~vis] == 0).all() and (d[1] >= 0).all()


def test_oracle_vs_reference_fastgs_golden():
    """Pins the oracle to the REFERENCE'S OWN fastgs kernels without a GPU: tests/golden/ref_fastgs_small.npz was produced on
    the GPU by tests/test_gpu_fastgs.py::test_dump_reference_fastgs_golden from oracle/_ref/libfastgs_ref.so, i.e.
    /root/reference/fastgs/rasterization/src/*.cu compiled unmodified (oracle/build_ref.py).  Scene:
    scenes.scene_small(N=1500, 176x112, SH degree 3, seed 13, view 2) -> scenes.fastgs_inputs; cotangents from numpy
    default_rng(17)."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_fastgs_small.npz"))
    inp = scenes.fastgs_inputs(scenes.scene_small(N=1500, width=176, height=112, sh_degree=3, seed=13, view=2))
    n = inp["means"].shape[0]
    dens = np.zeros((2, n), np.float32)
    for precision, tol_img, tol_grad in (("f32", 1e-4, 1e-3), ("f64", 1e-4, 1e-3)):
        o = fgo.render(**inp, grad_image=g["grad_image"], grad_alpha=g["grad_alpha"], want_w2c_grad=True,
                       densification_info=dens.copy(), precision=precision)

        def rel(a, b):
            a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
            return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
        assert rel(o["image"], g["image"]) < tol_img and rel(o["alpha"], g["alpha"]) < tol_img
        assert np.abs(o["image"] - g["image"]).max() < 2e-2  # a pixel at a threshold may gain / lose one contribution
        for k, gk in (("grad_means", "grad_means"), ("grad_scales_raw", "grad_scales_raw"), ("grad_rotations_raw", "grad_rotations_raw"),
                      ("grad_opacities_raw", "grad_opacities_raw"), ("grad_sh0", "grad_sh0"), ("grad_shN", "grad_shN")):
            e = rel(o[k].reshape(g[gk].shape), g[gk])
            assert e < tol_grad, (precision, k, e)
        assert rel(o["grad_w2c"][:3], g["grad_w2c"][:3]) < tol_grad
        assert np.array_equal(o["densification_info"][0], g["densification_info"][0])  # the same primitives are visible
        assert rel(o["densification_info"][1], g["densification_info"][1]) < tol_grad


def test_python_mirror_of_the_fastgs_caller_routes_gradients(pkg):
    """Host logic, no GPU: the package's mirror of FastGSRasterize / fast_rasterize (fastgs.py; reference:
    fast_rasterizer_autograd.cpp:10-160, fast_rasterizer.cpp:12-74) driven by a stand-in backend that calls the CPU oracle --
    gradient order, densification_info pass-through, w2c gradient on request, background composite."""
    import importlib

    import torch
    fg = importlib.import_module(pkg.__name__ + ".fastgs")
    inp = _scene(n=80, w=64, h=48, deg=2)
    keys = ("means", "scales_raw", "rotations_raw", "opacities_raw", "sh0", "shN")

    class OracleBackend:
        def forward(self, means, scales_raw, rotations_raw, opacities_raw, sh0, shN, w2c, s, capacity=0):
            self.args = dict(means=means.detach().numpy(), scales_raw=scales_raw.detach().numpy(),
                             rotations_raw=rotations_raw.detach().numpy(), opacities_raw=opacities_raw.detach().numpy(),
                             sh0=sh0.detach().numpy(), shN=shN.detach().numpy(), w2c=w2c.detach().numpy(),
                             cam_position=s.cam_position.numpy(), active_sh_bases=s.active_sh_bases, width=s.width,
                             height=s.height, fx=s.focal_x, fy=s.focal_y, cx=s.center_x, cy=s.center_y,
                             near_plane=s.near_plane, far_plane=s.far_plane)
            o = fgo.render(**self.args, precision="f64")
            return torch.from_numpy(o["image"]), torch.from_numpy(o["alpha"]), {"n": o["n_instances"]}

        def backward(self, ctx, grad_image, grad_alpha, image, alpha, means, scales_raw, rotations_raw, shN, w2c, s,
                     densification_info=None, want_w2c_grad=False):
            o = fgo.render(**self.args, grad_image=grad_image.numpy(), grad_alpha=grad_alpha.numpy(), precision="f64",
                           want_w2c_grad=want_w2c_grad,
                           densification_info=None if densification_info is None else densification_info.numpy())
            if densification_info is not None:
                densification_info.copy_(torch.from_numpy(o["densification_info"]))
            g = [torch.from_numpy(o[k]).float() for k in ("grad_means", "grad_scales_raw", "grad_rotations_raw",
                                                           "grad_opacities_raw", "grad_sh0", "grad_shN")]
            return (*g, torch.from_numpy(o["grad_w2c"]).float() if want_w2c_grad else None)

    P = {k: torch.from_numpy(inp[k]).requires_grad_(True) for k in keys}
    w2c = torch.from_numpy(inp["w2c"]).requires_grad_(True)
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]), active_sh_bases=inp["active_sh_bases"],
                          width=inp["width"], height=inp["height"], focal_x=inp["fx"], focal_y=inp["fy"], center_x=inp["cx"],
                          center_y=inp["cy"])
    bg = torch.tensor([0.2, 0.4, 0.6])
    dens = torch.zeros((2, inp["means"].shape[0]))
    gi, ga = _loss_weights(inp, 3)
    image, alpha = fg.fast_rasterize(OracleBackend(), P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"],
                                     P["shN"], w2c, s, bg_color=bg, densification_info=dens)
    ((image * torch.from_numpy(gi)).sum() + (alpha * torch.from_numpy(ga)).sum()).backward()
    # what the caller's sequence must amount to: image = raw + (1 - alpha) bg, so the rasterizer sees grad_alpha - bg . grad_image
    raw = _render(inp, "f64")
    assert np.allclose(image.detach().numpy(), raw["image"] + (1 - raw["alpha"]) * bg.numpy()[:, None, None], atol=1e-6)
    ga_eff = ga - (gi * bg.numpy()[:, None, None]).sum(0, keepdims=True)
    want = _render(inp, "f64", grad_image=gi, grad_alpha=ga_eff, want_w2c_grad=True)
    for k, wk in zip(keys, ("grad_means", "grad_scales_raw", "grad_rotations_raw", "grad_opacities_raw", "grad_sh0", "grad_shN")):
        assert P[k].grad.shape == P[k].shape
        assert np.allclose(P[k].grad.numpy().reshape(want[wk].shape), want[wk], rtol=1e-4, atol=1e-7), k
    assert np.allclose(w2c.grad.numpy()[:3], want["grad_w2c"][:3], rtol=1e-4, atol=1e-6)
    assert float(dens[0].sum()) == float((raw["n_touched"] > 0).sum())
