"""CPU: the intersect fixtures take the depth-sort branches they are named for, and the oracle's tie order.

The GPU tests of tests/test_gpu_isect_edges.py compare the planned intersect path with the oracle on these inputs.
They only test the branch a fixture is named for while the fixture still selects it, which is checked here with a
numpy restatement of the sort's pass-skip rule (gsb_devsort.cuh radix_pass_skipped)."""
import numpy as np
import pytest

import isect_fixtures as fx
import scenes


def test_skip_rule_restatement():
    # the rule on hand-made keys: a byte is skipped when it agrees over the active keys, inactive keys do not count
    d = np.uint32([0x40A15A37, 0x40A15A00, 0x12345678]).view(np.float32)
    act = np.array([True, True, False])
    assert fx.skip_pattern(d, act) == (1, 2, 3)
    assert fx.skip_pattern(d, np.ones(3, bool)) == ()
    assert fx.skip_pattern(np.float32([7.5]), [True]) == (0, 1, 2, 3)
    assert fx.skip_pattern(np.float32([1.0, 2.0]), [False, False]) == ()


@pytest.mark.parametrize("name", sorted(fx.DEPTHS))
@pytest.mark.parametrize("C,N", [(1, 3000), (3, 3000), (1, 200_000), (3, 1)])
def test_fixture_selects_its_skip_pattern(orc, name, C, N):
    W, H = 1280, 720
    m2d, radii, depths, active = fx.intersect_inputs(name, C, N, W, H, seed=C * 7 + N)
    tpg, _, _ = orc.isect_tiles(m2d, radii, depths, C, 16, (W + 15) // 16, (H + 15) // 16)
    # "active" is exactly "has at least one tile": every inactive kind (zero radii, box past the edge) has no tile
    assert np.array_equal(tpg > 0, active)
    if N > 1:
        assert (radii[~active] == 0).all(-1).any() and (radii[~active] > 0).all(-1).any()
    want = fx.DEPTHS[name][1]
    assert fx.skip_pattern(depths, active) == want
    if N > 1:  # the inactive Gaussians' depths would change the pattern if the sort did not ignore them
        assert fx.skip_pattern(depths, np.ones_like(active)) == ()


def test_single_gaussian_skips_every_pass():
    for name in fx.DEPTHS:
        m2d, radii, depths, active = fx.intersect_inputs(name, 1, 1, 640, 480)
        assert active.all() and fx.skip_pattern(depths, active) == (0, 1, 2, 3)


@pytest.mark.parametrize("scene", ["one_visible", "wall"])
def test_scene_depths_skip_every_pass(orc, scene):
    """The two whole-path scenes: with the oracle's projection, the Gaussians that have tiles share every depth byte."""
    sc = {"one_visible": scenes.scene_one_visible, "wall": scenes.scene_wall}[scene]()
    W, H = sc["width"], sc["height"]
    radii, m2d, depths, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"],
                                                 sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    tpg, ids, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, (W + 15) // 16, (H + 15) // 16)
    active = tpg > 0
    n_act = int(active.sum())
    print(f"{scene}: {n_act} Gaussians with tiles, {len(flat)} intersections, skipped passes "
          f"{fx.skip_pattern(depths, active)}")
    assert fx.skip_pattern(depths, active) == (0, 1, 2, 3)
    if scene == "one_visible":
        assert n_act == 1 and len(flat) > 20
    else:
        assert n_act > 1000
        # overlapping footprints: most tiles hold many equal-depth Gaussians, so their order decides the image
        assert np.median(np.bincount((ids >> 32).astype(np.int64))) > 30


def test_oracle_orders_depth_ties_by_index(orc):
    """orc.isect_tiles sorts stably, like the reference's CUB radix sort: equal (camera, tile, depth) keys keep
    ascending flattened index.  The GPU tests expect exactly this order."""
    C, N, W, H = 3, 5000, 320, 240
    m2d, radii, depths, active = fx.intersect_inputs("skip_all", C, N, W, H, max_radius=60)
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, C, 16, W // 16, H // 16)
    head = ids >> 32
    same = head[1:] == head[:-1]
    assert same.sum() > 10 * C * (W // 16) * (H // 16) // 2  # long runs of ties
    assert (np.diff(flat)[same] > 0).all()
    # and across tiles the order is ascending (camera, tile)
    assert (np.diff(head) >= 0).all()
    # mixed depths: within a tile ascending (depth bits, index)
    m2d, radii, depths, _ = fx.intersect_inputs("skip_013", C, N, W, H, max_radius=60)
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, C, 16, W // 16, H // 16)
    key = ((ids & 0xFFFFFFFF).astype(np.uint64) << np.uint64(32)) | flat.astype(np.uint64)
    same = (ids >> 32)[1:] == (ids >> 32)[:-1]
    assert (np.diff(key.astype(np.int64))[same] > 0).all()
    assert (np.diff(ids & 0xFFFFFFFF)[same] == 0).sum() > 1000  # 128 distinct depths: many ties broken by index
