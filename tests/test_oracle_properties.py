"""CPU: self-consistency of the oracle on the rows the reference's tests do not pin
(UT projection, from-world blend fwd/bwd): float32 vs float64 builds, finite differences of the
forward against the analytic backward, and structural properties of the blend."""
import numpy as np
import pytest

import scenes


@pytest.fixture(scope="module")
def small(orc):
    sc = scenes.scene_small(N=600, width=96, height=64, sh_degree=2, view=3)
    rng = np.random.default_rng(1)
    vrc = rng.standard_normal((1, sc["height"], sc["width"], 3)).astype(np.float32)
    vra = rng.standard_normal((1, sc["height"], sc["width"], 1)).astype(np.float32)
    o32 = orc.render_pipeline(sc, "f32", True, vrc, vra)
    o64 = orc.render_pipeline(sc, "f64", True, vrc, vra)
    return sc, vrc, vra, o32, o64


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def test_f32_vs_f64(small):
    sc, _, _, o32, o64 = small
    assert (o32["radii"] != o64["radii"]).sum() <= 2  # ceil() borderline flips only
    if np.array_equal(o32["flatten_ids"], o64["flatten_ids"]):
        assert rel(o32["renders"], o64["renders"]) < 1e-5
        for k in ("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"):
            assert rel(o32[k], o64[k]) < 1e-3, k


def test_blend_properties(small):
    sc, _, _, o32, _ = small
    a = o32["alphas"]
    assert np.all(a >= 0) and np.all(a <= 1.0)
    # transmittance never drops below the 1e-4 stop threshold by more than one max-alpha step
    assert np.all(1 - a > 1e-4 * (1 - 0.999) - 1e-9)
    off = o32["tile_offsets"].reshape(-1)
    li = o32["last_ids"][0]
    ts = 16
    tw = (sc["width"] + ts - 1) // ts
    n = len(o32["flatten_ids"])
    for ty in range((sc["height"] + ts - 1) // ts):
        for tx in range(tw):
            t = ty * tw + tx
            lo, hi = off[t], (off[t + 1] if t + 1 < len(off) else n)
            blk = li[ty * ts:(ty + 1) * ts, tx * ts:(tx + 1) * ts]
            touched = blk[blk != 0]
            assert np.all((touched >= lo) & (touched < hi))


def test_backward_matches_finite_differences(orc, small):
    """d(sum(render * vrc) + sum(alpha * vra)) / d(param) by central differences in float64."""
    sc, vrc, vra, _, o64 = small
    base = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in sc.items()}

    def loss(scn):
        # keep the isect lists fixed (projection / binning is not differentiated, Ops.h:67)
        r, a, _ = orc.raster_fwd(scn["means"], scn["quats"], scn["scales"], o64["colors"], scn["opacities"][None],
                                 scn["background"], None, scn["width"], scn["height"], 16, scn["viewmats"], scn["Ks"],
                                 o64["tile_offsets"], o64["flatten_ids"], precision="f64")
        return float((r.astype(np.float64) * vrc).sum() + (a.astype(np.float64) * vra).sum())

    vis = np.nonzero(np.abs(o64["v_means"]).sum(-1) > 1e-3)[0][:6]
    checked = 0
    for g in vis:
        for name, key, dim in (("means", "v_means", 0), ("scales", "v_scales", 1), ("opacities", "v_opacities", None),
                               ("quats", "v_quats", 2)):
            ana = o64[key][0, g] if dim is None else o64[key][g, dim]
            if abs(ana) <= 0.05:
                continue
            ok = False
            nums = []
            # the forward is only piecewise smooth (1/255 cut, T <= 1e-4 stop): accept if any step size agrees
            for eps in (1e-4, 5e-5, 2e-4):
                p = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in base.items()}
                m = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in base.items()}
                if dim is None:
                    p[name][g] += eps; m[name][g] -= eps
                    h = float(p[name][g]) - float(m[name][g])
                else:
                    p[name][g, dim] += eps; m[name][g, dim] -= eps
                    h = float(p[name][g, dim]) - float(m[name][g, dim])
                num = (loss(p) - loss(m)) / h
                nums.append(num)
                if abs(num - ana) <= 0.03 * abs(ana) + 0.02:
                    ok = True
                    break
            assert ok, (name, g, nums, ana)
            checked += 1
    assert checked >= 6


# ------------------------------------------------------------------------------------------
# a2: camera models of the oracle (the checker of the GPU's distorted-camera tests)
# ------------------------------------------------------------------------------------------
OPENCV = dict(camera_model=0, radial=np.array([[-0.12, 0.05, 0.002, 0.01, -0.003, 0.0005]], np.float32),
              tangential=np.array([[0.002, -0.001]], np.float32),
              thin_prism=np.array([[0.001, 0.0002, -0.0005, 0.0001]], np.float32))
FISHEYE = dict(camera_model=2, radial=np.array([[0.03, -0.004, 0.0007, -0.0001]], np.float32), tangential=None,
               thin_prism=None)


def _project_and_blend(orc, sc, colors, **cam):
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    radii, m2d, depths, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"],
                                                 sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **cam)
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, tw, th)
    off = orc.isect_offsets(ids, 1, tw, th)
    img, alp, _ = orc.raster_fwd(sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], None, None, W, H,
                                 16, sc["viewmats"], sc["Ks"], off, flat, **cam)
    return radii, m2d, img, alp


def test_zero_distortion_is_the_perfect_pinhole(orc):
    """All-zero OpenCV coefficients go through the general camera code (Newton undistortion included) and must
    reproduce the perfect-pinhole results."""
    sc = scenes.scene_small(N=400, width=96, height=64, sh_degree=0, view=2)
    colors = np.random.default_rng(5).random((1, 400, 3), dtype=np.float32)
    zero = dict(camera_model=0, radial=np.zeros((1, 6), np.float32), tangential=np.zeros((1, 2), np.float32),
                thin_prism=np.zeros((1, 4), np.float32))
    r0, m0, i0, a0 = _project_and_blend(orc, sc, colors, camera_model=0)
    r1, m1, i1, a1 = _project_and_blend(orc, sc, colors, **zero)
    assert np.array_equal(r0, r1)
    assert rel(m1, m0) < 1e-6 and rel(i1, i0) < 1e-5 and rel(a1, a0) < 1e-5


@pytest.mark.parametrize("cam", [OPENCV, FISHEYE], ids=["opencv", "fisheye"])
def test_blend_unprojection_inverts_the_projection(orc, cam):
    """The UT projection maps world -> distorted image, the blend maps pixel -> ray by undistorting; for a small
    isotropic Gaussian the alpha image must peak at the projected centre under every camera model."""
    W, H = 160, 112
    Ks = np.array([[[140.0, 0, 80.0], [0, 150.0, 56.0], [0, 0, 1]]], np.float32)
    viewmats = np.eye(4, dtype=np.float32)[None]
    pts = np.array([[0.9, 0.5, 3.0], [-1.0, -0.55, 2.5], [0.2, -0.6, 4.0], [-0.7, 0.6, 3.5]], np.float32)
    moved = 0.0
    for pt in pts:
        sc = dict(means=pt[None].copy(), quats=np.array([[1, 0, 0, 0]], np.float32),
                  scales=np.full((1, 3), 0.03, np.float32), opacities=np.array([0.9], np.float32), viewmats=viewmats,
                  Ks=Ks, width=W, height=H)
        radii, m2d, _, alp = _project_and_blend(orc, sc, np.ones((1, 1, 3), np.float32), **cam)
        assert (radii > 0).all(), "test point must be visible"
        a = alp[0, :, :, 0]
        ys, xs = np.mgrid[0:H, 0:W]
        wsum = a.sum()
        assert wsum > 0
        cx, cy = ((xs + 0.5) * a).sum() / wsum, ((ys + 0.5) * a).sum() / wsum  # alpha-weighted centroid
        assert abs(cx - m2d[0, 0, 0]) < 0.35 and abs(cy - m2d[0, 0, 1]) < 0.35, (pt, (cx, cy), m2d[0, 0])
        ideal = np.array([Ks[0, 0, 0] * pt[0] / pt[2] + Ks[0, 0, 2], Ks[0, 1, 1] * pt[1] / pt[2] + Ks[0, 1, 2]])
        moved = max(moved, float(np.linalg.norm(ideal - m2d[0, 0])))
    assert moved > 1.0  # the distortion is not a no-op: off-centre points land more than a pixel from the ideal pinhole


# (camera, rolling-shutter direction or None for the global shutter); the ids of the global cases are the camera's
FD_CASES = [(dict(camera_model=0), None), (OPENCV, None), (FISHEYE, None), (dict(camera_model=0), 0), (OPENCV, 1),
            (FISHEYE, 2), (dict(camera_model=0), 3)]
FD_IDS = ["pinhole", "opencv", "fisheye", "pinhole-rolling_top_to_bottom", "opencv-rolling_left_to_right",
          "fisheye-rolling_bottom_to_top", "pinhole-rolling_right_to_left"]


@pytest.mark.parametrize("cam,rs_type", FD_CASES, ids=FD_IDS)
def test_backward_matches_finite_differences_without_cutoffs(orc, cam, rs_type):
    """The analytic backward against central differences of the forward, camera model by camera model, on the
    test-only ORC_SMOOTH float64 build of the oracle (no 1/255 cut, no T <= 1e-4 stop): with fixed intersection
    lists the forward is then smooth, so the comparison is tight (1 %) on EVERY checked component instead of
    "some step size agrees up to a threshold crossing".  The cut-offs themselves only gate which pairs contribute.
    The rolling-shutter cases give every pixel its own pose, between the start pose and one turned by 3 degrees."""
    sc = scenes.scene_small(N=300, width=80, height=64, sh_degree=0, view=2)
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    if rs_type is not None:
        from test_oracle_rolling_shutter import end_pose
        cam = dict(cam, viewmats1=end_pose(sc["viewmats"], deg=3.0), rs_type=rs_type)
    rng = np.random.default_rng(8)
    colors = rng.random((1, 300, 3), dtype=np.float32)
    vrc = rng.standard_normal((1, H, W, 3))
    vra = rng.standard_normal((1, H, W, 1))
    radii, m2d, depths, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"],
                                                 sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, precision="f64", **cam)
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, tw, th)
    off = orc.isect_offsets(ids, 1, tw, th)

    def fwd(P):
        return orc.raster_fwd(P["means"], P["quats"], P["scales"], colors, P["opacities"][None], sc["background"], None, W,
                              H, 16, sc["viewmats"], sc["Ks"], off, flat, precision="f64s", **cam)

    base = {k: sc[k].copy() for k in ("means", "quats", "scales", "opacities")}
    img, alp, li = fwd(base)
    g = orc.raster_bwd(base["means"], base["quats"], base["scales"], colors, base["opacities"][None], sc["background"],
                       None, W, H, 16, sc["viewmats"], sc["Ks"], off, flat, alp, li, vrc.astype(np.float32),
                       vra.astype(np.float32), precision="f64s", **cam)
    ana = dict(means=g[0], quats=g[1], scales=g[2], opacities=g[4][0])

    def loss(P):
        r, a, _ = fwd(P)
        return float((r.astype(np.float64) * vrc).sum() + (a.astype(np.float64) * vra).sum())

    cand = np.argsort(-np.abs(ana["means"]).sum(-1))[:10]
    checked = 0
    for gi in cand:
        for name, dim in (("means", 0), ("means", 1), ("means", 2), ("scales", 0), ("scales", 1), ("scales", 2),
                          ("quats", 0), ("quats", 1), ("quats", 2), ("quats", 3), ("opacities", None)):
            a_ = float(ana[name][gi] if dim is None else ana[name][gi, dim])
            eps = 1e-3 if name != "opacities" else 2e-3
            p = {k: v.copy() for k, v in base.items()}
            m = {k: v.copy() for k, v in base.items()}
            if dim is None:
                p[name][gi] += eps; m[name][gi] -= eps
                h = float(p[name][gi]) - float(m[name][gi])
            else:
                p[name][gi, dim] += eps; m[name][gi, dim] -= eps
                h = float(p[name][gi, dim]) - float(m[name][gi, dim])
            num = (loss(p) - loss(m)) / h
            assert abs(num - a_) <= 0.01 * abs(a_) + 2e-3, (name, int(gi), dim, num, a_)
            checked += 1
    assert checked == 110


def test_ut_projection_tends_to_the_linearised_projection_for_small_gaussians(orc):
    """Independent check of the unscented transform (sigma points, weights lambda/(D+lambda) and 1/(2(D+lambda)),
    ProjectionUT3DGSFused.cu:84-150): for a Gaussian that is small compared with its depth the UT mean is the
    projected centre and the UT covariance is J Sigma J^T of the pinhole Jacobian, up to O((sigma/z)^2)."""
    rng = np.random.default_rng(12)
    N, W, H = 200, 320, 240
    fx, fy, cx, cy = 260.0, 250.0, 160.0, 120.0
    Ks = np.array([[[fx, 0, cx], [0, fy, cy], [0, 0, 1]]], np.float32)
    vm = scenes.look_at(np.array([0.4, -0.3, -0.5]), (0.0, 0.0, 3.0)).astype(np.float32)[None]
    means = np.stack([rng.uniform(-1, 1, N), rng.uniform(-0.7, 0.7, N), rng.uniform(2.5, 4.0, N)], -1).astype(np.float32)
    quats = rng.standard_normal((N, 4)).astype(np.float32)
    quats /= np.linalg.norm(quats, axis=-1, keepdims=True)
    scales = rng.uniform(0.004, 0.012, (N, 3)).astype(np.float32)
    eps2d = 1e-4
    radii, m2d, depths, conics, _ = orc.projection_ut(means, quats, scales, np.full(N, 0.9, np.float32), vm, Ks, W, H,
                                                      eps2d, 0.01, 1e4, 0.0, precision="f64")
    vis = (radii[0] > 0).all(-1)
    assert vis.sum() > 100
    R, t = vm[0, :3, :3].astype(np.float64), vm[0, :3, 3].astype(np.float64)
    for i in np.nonzero(vis)[0][:60]:
        pc = R @ means[i].astype(np.float64) + t
        uv = np.array([fx * pc[0] / pc[2] + cx, fy * pc[1] / pc[2] + cy])
        w, x, y, z = quats[i].astype(np.float64)
        Rg = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                       [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                       [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        S3 = Rg @ np.diag(scales[i].astype(np.float64) ** 2) @ Rg.T
        J = np.array([[fx / pc[2], 0, -fx * pc[0] / pc[2] ** 2], [0, fy / pc[2], -fy * pc[1] / pc[2] ** 2]])
        S2 = J @ (R @ S3 @ R.T) @ J.T + eps2d * np.eye(2)
        inv = np.linalg.inv(S2)
        assert np.abs(m2d[0, i] - uv).max() < 2e-3, (i, m2d[0, i], uv)
        assert abs(depths[0, i] - pc[2]) < 1e-5
        got = conics[0, i].astype(np.float64)
        want = np.array([inv[0, 0], inv[0, 1], inv[1, 1]])
        assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max(), (i, got, want)
