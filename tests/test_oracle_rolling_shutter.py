"""CPU: the oracle's restatement of the rolling shutter (gsplat/Cameras.cuh:268-413).

A rolling-shutter camera reads its image out row by row (or column by column) while it moves from the start-of-frame
pose (viewmats0) to the end-of-frame pose (viewmats1).  The projection iterates each sigma point to the pose of the
row or column it lands on, and the blend casts every pixel's ray from the pose of its own read-out time.  These tests
check the restatement against itself (end pose = start pose is the global shutter; the reversed direction with
swapped poses is the same camera at pixel centres; the backward is the derivative of the forward) and against stored
outputs of the reference's own kernels (tests/golden/ref_rolling_small.npz, written by
tests/test_gpu_rolling_shutter.py::test_dump_reference_rolling_golden from the reference's build without
--use_fast_math)."""
import os

import numpy as np
import pytest

import scenes

RS_TYPES = [0, 1, 2, 3]  # gsplat/Common.h ShutterType: top-to-bottom, left-to-right, bottom-to-top, right-to-left
RS_IDS = ["top_to_bottom", "left_to_right", "bottom_to_top", "right_to_left"]
GLOBAL = 4
GRADS = ("v_means", "v_quats", "v_scales", "v_colors", "v_opacities")

# camera models as oracle keyword arguments: OpenCV pinhole with all 6 + 2 + 4 coefficients, the 4-coefficient fisheye
CAMERAS = {
    "pinhole": dict(camera_model=0),
    "opencv": dict(camera_model=0, radial=np.array([[-0.12, 0.05, 0.002, 0.01, -0.003, 0.0005]], np.float32),
                   tangential=np.array([[0.002, -0.001]], np.float32),
                   thin_prism=np.array([[0.001, 0.0002, -0.0005, 0.0001]], np.float32)),
    "fisheye": dict(camera_model=2, radial=np.array([[0.03, -0.004, 0.0007, -0.0001]], np.float32)),
}

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_rolling_small.npz")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def within_one_ulp(a, b):
    """float32 interface arrays of a float64 computation that differ only by rounding below 1e-12: the stored values
    are at most one float32 ulp apart."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all(np.abs(a.astype(np.float64) - b) <= np.spacing(np.abs(b)).astype(np.float64)))


def end_pose(viewmats, deg=2.5, axis=1, shift=(0.04, -0.02, 0.03)):
    """The end-of-frame pose: the start pose turned by `deg` degrees about camera axis `axis` (0 = x, pitch: image
    points move vertically; 1 = y, yaw: they move horizontally) and moved by `shift`."""
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [k for k in range(3) if k != axis]
    dR = np.eye(3)
    dR[i, i], dR[i, j], dR[j, i], dR[j, j] = c, -s, s, c
    V1 = np.asarray(viewmats, np.float64).copy()
    V1[0, :3, :3] = dR @ V1[0, :3, :3]
    V1[0, :3, 3] = dR @ V1[0, :3, 3] + np.asarray(shift)
    return V1.astype(np.float32)


# ------------------------------------------------------------------------------------------
# the golden scene: small, ragged on both axes (70 % 16 = 6, 45 % 16 = 13)
# ------------------------------------------------------------------------------------------
def golden_scene():
    return scenes.scene_small(N=500, width=70, height=45, sh_degree=0, view=2)


# (camera, rolling direction) of each stored case
GOLDEN_CASES = [("pinhole", 0), ("pinhole", 1), ("pinhole", 2), ("pinhole", 3), ("fisheye", 3)]


def golden_end_pose(sc):
    return end_pose(sc["viewmats"], deg=4.0)


def golden_colors(sc):
    return np.random.default_rng(11).random((1, sc["means"].shape[0], 3), dtype=np.float32)


def golden_cotangents(sc):
    rng = np.random.default_rng(12)
    H, W = sc["height"], sc["width"]
    return (rng.standard_normal((1, H, W, 3)).astype(np.float32), rng.standard_normal((1, H, W, 1)).astype(np.float32))


# ------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------
def project(orc, sc, cam, precision="f32", **rs):
    W, H = sc["width"], sc["height"]
    return orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"], sc["Ks"], W, H,
                             0.3, 0.01, 1e4, 0.0, precision=precision, **cam, **rs)


def lists(orc, sc, proj):
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    radii, m2d, depths = proj[:3]
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, tw, th)
    return orc.isect_offsets(ids, 1, tw, th), flat


def blend(orc, sc, colors, off, flat, vrc, vra, cam, precision, bg=True, **rs):
    W, H = sc["width"], sc["height"]
    b = sc["background"] if bg else None
    a = (sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], b, None, W, H, 16, sc["viewmats"],
         sc["Ks"], off, flat)
    r, alp, li = orc.raster_fwd(*a, precision=precision, **cam, **rs)
    g = orc.raster_bwd(*a, alp, li, vrc, vra, precision=precision, **cam, **rs)
    return r, alp, li, g


@pytest.fixture(scope="module")
def small():
    sc = scenes.scene_small(N=800, width=90, height=70, sh_degree=0, view=3)  # 90 % 16 = 10, 70 % 16 = 6
    rng = np.random.default_rng(3)
    colors = rng.random((1, 800, 3), dtype=np.float32)
    vrc = rng.standard_normal((1, 70, 90, 3)).astype(np.float32)
    vra = rng.standard_normal((1, 70, 90, 1)).astype(np.float32)
    return sc, colors, vrc, vra


# ------------------------------------------------------------------------------------------
# end pose = start pose: every rolling direction is the global shutter
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", list(CAMERAS), ids=list(CAMERAS))
@pytest.mark.parametrize("rs_type", RS_TYPES, ids=RS_IDS)
def test_static_camera_equals_global_shutter(orc, small, rs_type, cam):
    """With viewmats1 = viewmats0 the pose interpolation returns the start pose, so the iteration of the projection and
    the per-pixel rays reproduce the global shutter in float64: radii and last_ids exactly, the float64 gradients to
    1e-12, and the float32 outputs (means2d, depths, conics, image, alpha) to their last bit.

    That needs a start pose whose quaternion is exactly unit, here a half turn about x (the camera at z = 6 looking
    back at the scene): GLM's slerp of a quaternion q with itself takes its acos branch when |q|^2 is further than one
    epsilon from 1, and then returns q scaled by 1 + O(tau (1 - tau) (1 - |q|^2)).  A pose read from a generic float32
    rotation matrix (|q|^2 - 1 ~ 1e-7) therefore moves points by ~1e-8 relative under a static rolling shutter, in the
    reference as here: checked to 1e-6 on the scene's own rotated camera."""
    sc, colors, vrc, vra = small
    c = CAMERAS[cam]
    flip = np.array([[[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 6], [0, 0, 0, 1]]], np.float32)
    generic = sc
    sc = dict(sc, viewmats=flip)
    rs = dict(viewmats1=sc["viewmats"].copy(), rs_type=rs_type)
    pg = project(orc, sc, c, "f64")
    pr = project(orc, sc, c, "f64", **rs)
    assert np.array_equal(pr[0], pg[0])
    vis = (pg[0] > 0).all(-1)
    assert vis.sum() > 300
    for k in (1, 2, 3):
        assert within_one_ulp(pr[k][vis], pg[k][vis]), k
    off, flat = lists(orc, sc, pg)
    rg, ag, lg, gg = blend(orc, sc, colors, off, flat, vrc, vra, c, "f64")
    rr, ar, lr, gr = blend(orc, sc, colors, off, flat, vrc, vra, c, "f64", **rs)
    assert float(ag.mean()) > 0.3
    assert np.array_equal(lr, lg)
    assert within_one_ulp(rr, rg) and within_one_ulp(ar, ag)
    for nm, a, b in zip(GRADS, gr, gg):
        assert rel(a, b) < 1e-12, nm
    pg = project(orc, generic, c, "f64")
    pr = project(orc, generic, c, "f64", viewmats1=generic["viewmats"].copy(), rs_type=rs_type)
    vis = (pg[0] > 0).all(-1) & (pr[0] > 0).all(-1)
    assert vis.sum() > 300 and rel(pr[1][vis], pg[1][vis]) < 1e-6


# ------------------------------------------------------------------------------------------
# reversal: top-to-bottom from A to B is bottom-to-top from B to A at pixel centres
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [(0, 2), (1, 3)], ids=["vertical", "horizontal"])
def test_reversed_direction_with_swapped_poses_is_the_same_camera(orc, small, pair):
    """At a pixel centre (j + 0.5, i + 0.5) top-to-bottom reads row i at tau = i / (H - 1) and bottom-to-top reads it at
    (H - ceil(i + 0.5)) / (H - 1) = 1 - tau; with the poses swapped both interpolate to the same pose (slerp(A, B, t)
    = slerp(B, A, 1 - t) up to the sign of the quaternion).  The same holds for left-to-right and right-to-left."""
    sc, colors, vrc, vra = small
    A, B = sc["viewmats"], end_pose(sc["viewmats"], deg=3.0)
    fwd_t, rev_t = pair
    off, flat = lists(orc, sc, project(orc, sc, {}, "f64", viewmats1=B, rs_type=fwd_t))
    for cam in ("pinhole", "fisheye"):
        c = CAMERAS[cam]
        r1, a1, l1, g1 = blend(orc, sc, colors, off, flat, vrc, vra, c, "f64", viewmats1=B, rs_type=fwd_t)
        scr = dict(sc, viewmats=B)
        r2, a2, l2, g2 = blend(orc, scr, colors, off, flat, vrc, vra, c, "f64", viewmats1=A, rs_type=rev_t)
        assert float(a1.mean()) > 0.3
        assert np.array_equal(l1, l2), cam
        assert rel(r2, r1) < 1e-10 and rel(a2, a1) < 1e-10, cam
        for nm, x, y in zip(GRADS, g2, g1):
            assert rel(x, y) < 1e-9, (cam, nm, rel(x, y))
        # and the motion matters: the global shutter at either pose renders a different image
        rg = blend(orc, sc, colors, off, flat, vrc, vra, c, "f64")[0]
        assert rel(rg, r1) > 1e-2, cam


def test_rolling_projection_moves_the_gaussians_and_follows_the_rows(orc, small):
    """The iteration lands each centre on the pose of its own row: a Gaussian projected by the rolling camera sits
    where the global camera at that row's pose puts it (for the Gaussian's centre, to the rounding of the last of ten
    fixed-point steps), and the motion moves the median Gaussian by more than a pixel."""
    sc = small[0]
    H = sc["height"]
    V1 = end_pose(sc["viewmats"], deg=3.0)
    pg = project(orc, sc, {}, "f64")
    pr = project(orc, sc, {}, "f64", viewmats1=V1, rs_type=0)
    vis = (pg[0] > 0).all(-1)[0] & (pr[0] > 0).all(-1)[0]
    assert np.median(np.abs(pr[1][0][vis] - pg[1][0][vis]).max(-1)) > 1.0
    # a single point (a tiny isotropic Gaussian) against the global shutter at the pose of its row
    from scipy.spatial.transform import Rotation, Slerp
    V0 = sc["viewmats"][0].astype(np.float64)
    V1d = V1[0].astype(np.float64)
    slerp = Slerp([0, 1], Rotation.from_matrix([V0[:3, :3], V1d[:3, :3]]))
    pt = dict(sc, means=np.array([[0.2, -0.3, 3.0]], np.float32), quats=np.array([[1, 0, 0, 0]], np.float32),
              scales=np.full((1, 3), 1e-3, np.float32), opacities=np.array([0.9], np.float32))
    _, m2d, _, _, _ = project(orc, pt, {}, "f64", viewmats1=V1, rs_type=0)
    u, v = m2d[0, 0]
    tau = np.floor(v) / (H - 1)
    Vt = np.eye(4)
    Vt[:3, :3] = slerp([tau]).as_matrix()[0]
    Vt[:3, 3] = (1 - tau) * V0[:3, 3] + tau * V1d[:3, 3]
    c = Vt[:3, :3] @ pt["means"][0].astype(np.float64) + Vt[:3, 3]
    K = sc["Ks"][0].astype(np.float64)
    assert abs(K[0, 0] * c[0] / c[2] + K[0, 2] - u) < 1e-3 and abs(K[1, 1] * c[1] / c[2] + K[1, 2] - v) < 1e-3


# ------------------------------------------------------------------------------------------
# the reference's kernels (precise build), stored
# ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold():
    return np.load(G)


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("case", range(len(GOLDEN_CASES)), ids=[f"{c}-{RS_IDS[r]}" for c, r in GOLDEN_CASES])
def test_oracle_matches_reference_rolling_golden(orc, gold, case, precision):
    """Projection, intersection lists, blend forward and blend backward of the rolling shutter against the
    reference's kernels built without --use_fast_math.  A sigma point whose row estimate sits on a floor() boundary may
    settle one row apart between two float implementations: a few Gaussians may move by more than 0.02 px."""
    cam, rs_type = GOLDEN_CASES[case]
    p = f"c{case}_"
    sc = golden_scene()
    W, H = sc["width"], sc["height"]
    assert W % 16 and H % 16
    c = CAMERAS[cam]
    rs = dict(viewmats1=golden_end_pose(sc), rs_type=rs_type)
    radii, m2d, depths, conics, _ = project(orc, sc, c, precision, **rs)
    g_r = gold[p + "radii"]
    mism = int((radii != g_r).any(-1).sum())
    both = (radii > 0).all(-1) & (g_r > 0).all(-1)
    dm = np.abs(m2d - gold[p + "means2d"]).max(-1)
    ok = both & (dm <= 0.02)
    print(f"[{cam} {RS_IDS[rs_type]} {precision}] radii differ {mism}, visible {int(both.sum())}, off by > 0.02 px "
          f"{int((both & ~ok).sum())}; means2d rel {rel(m2d[ok], gold[p + 'means2d'][ok]):.2e}")
    assert both.sum() > 180 and mism <= 3 and (both & ~ok).sum() <= 3
    assert rel(m2d[ok], gold[p + "means2d"][ok]) < 5e-5
    assert rel(depths[both], gold[p + "depths"][both]) < 1e-6
    assert rel(conics[ok], gold[p + "conics"][ok]) < 1e-3
    # the stored lists are the reference's intersection of its own projection: the oracle's intersection agrees
    tw, th = (W + 15) // 16, (H + 15) // 16
    _, ids, flat = orc.isect_tiles(gold[p + "means2d"], g_r, gold[p + "depths"], 1, 16, tw, th)
    assert np.array_equal(flat, gold[p + "flatten_ids"])
    assert np.array_equal(orc.isect_offsets(ids, 1, tw, th), gold[p + "tile_offsets"])
    colors = golden_colors(sc)
    a = (sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], sc["background"], None, W, H, 16,
         sc["viewmats"], sc["Ks"], gold[p + "tile_offsets"], gold[p + "flatten_ids"])
    r, alp, li = orc.raster_fwd(*a, precision=precision, **c, **rs)
    print(f"[{cam} {RS_IDS[rs_type]} {precision}] image rel {rel(r, gold[p + 'renders']):.2e}, last_ids differ "
          f"{float((li != gold[p + 'last_ids']).mean()):.2e}")
    # measured 1.1e-6 .. 1.8e-6, and 5.8e-5 where one pixel's 1/255 decision flips; a flip moves a pixel by <= 2e-2
    assert rel(r, gold[p + "renders"]) < 1e-4 and rel(alp, gold[p + "alphas"]) < 1e-4
    assert np.abs(r - gold[p + "renders"]).max() < 2e-2
    assert (li != gold[p + "last_ids"]).mean() < 2e-3
    g = orc.raster_bwd(*a, gold[p + "alphas"], gold[p + "last_ids"], gold["v_render_colors"], gold["v_render_alphas"],
                       precision=precision, **c, **rs)
    for nm, got in zip(GRADS, g):
        e = rel(got.reshape(gold[p + nm].shape), gold[p + nm])
        print(f"[{cam} {RS_IDS[rs_type]} {precision}] {nm} rel {e:.2e}")
        assert e < 1e-3, (nm, e)
