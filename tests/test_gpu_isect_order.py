"""GPU: the planned intersection path places every (chunk, tile) group in depth order directly.

A camera on the slab's diagonal correlates depth with screen position, so consecutive Gaussians in depth order pile
onto the same tiles: (chunk, tile) groups of more than 16 members, and with enlarged Gaussians boxes of more than 32
tiles.  flatten_ids, isect_ids and the tile offsets must equal the CPU oracle's element for element."""
import numpy as np
import pytest
import torch

import scenes
from isect_fixtures import WINDOW_TILES

pytestmark = pytest.mark.gpu


def _project(native, sc, dev):
    t = {k: torch.from_numpy(sc[k]).to(dev) for k in ("means", "quats", "scales", "opacities", "viewmats", "Ks")}
    radii, means2d, depths, _, _ = native.projection_ut_3dgs_fused(
        t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], sc["width"], sc["height"],
        0.3, 0.01, 1e4, 0.0)
    return radii, means2d, depths


# five 1080p cameras: 40 800 (camera, tile) pairs, more than one window of the histogram and placement
WINDOWED_VIEWS = (0, 1, 2, 3, 5)


@pytest.mark.parametrize("n_gauss,views,scale_mul", [(200_000, (1,), 1.0), (50_000, (1,), 4.0), (100_000, (1, 3), 2.0),
                                                     (50_000, WINDOWED_VIEWS, 2.0)])
def test_diagonal_view_lists_equal_oracle(native, orc, cuda_device, n_gauss, views, scale_mul):
    per_view = [_project(native, scenes.scene_b(N=n_gauss, view=v, scale_mul=scale_mul), cuda_device) for v in views]
    radii, means2d, depths = (torch.cat([pv[i] for pv in per_view], 0).contiguous() for i in range(3))
    C, W, H = len(views), 1920, 1080
    tw, th = (W + 15) // 16, (H + 15) // 16
    tpg, ids, flat = native.intersect_tile(means2d, radii, depths, C, 16, tw, th, True)
    off = native.intersect_offset(ids, C, tw, th)
    m_h, r_h, d_h = means2d.cpu().numpy(), radii.cpu().numpy(), depths.cpu().numpy()
    tpg_ref, ids_ref, flat_ref = orc.isect_tiles(m_h, r_h, d_h, C, 16, tw, th)
    off_ref = orc.isect_offsets(ids_ref, C, tw, th)

    # the scene exercises what the placement has to keep in order
    tiles = (ids_ref >> 32).astype(np.int64)
    n = tpg_ref.reshape(-1)
    glob = (tiles >> (tw * th).bit_length()) * (tw * th) + (tiles & ((1 << (tw * th).bit_length()) - 1))
    windows = -(-C * tw * th // WINDOW_TILES)
    print(f"views {views} x{scale_mul}: {len(ids_ref)} intersections, largest tile list {np.bincount(tiles).max()}, "
          f"largest box {n.max()} tiles, {C * tw * th} tiles in {windows} windows "
          f"({int((glob >= WINDOW_TILES).sum())} intersections past the first)")
    if scale_mul > 1.0:
        assert n.max() > 32
    if views == WINDOWED_VIEWS:
        assert C * tw * th > WINDOW_TILES and (glob >= WINDOW_TILES).sum() > 1000
    assert np.array_equal(tpg.cpu().numpy(), tpg_ref)
    assert np.array_equal(off.cpu().numpy(), off_ref)
    assert np.array_equal(ids.cpu().numpy(), ids_ref)
    assert np.array_equal(flat.cpu().numpy(), flat_ref)


def test_diagonal_view_ewa_instances_in_order(native, cuda_device):
    """The fastgs (EWA) path places with the per-tile ellipse test: every tile's instances must be ordered by (depth bits,
    index), and every primitive must sit in exactly the tiles of its box that pass the test -- the front kernel's mask
    for boxes of up to 32 tiles, as many tiles as its exact count for the larger ones (those re-evaluate the test)."""
    _check_ewa_instances(native, cuda_device, scenes.scene_b(N=50_000, view=1, scale_mul=4.0))


def test_windowed_ewa_instances_in_order(native, cuda_device):
    """The same at 4112x2320: 37 265 tiles, two windows of the histogram and placement.  The longer focal length
    spreads the slab over the whole frame, so the second window (the last tile row) receives instances too."""
    sc = scenes.scene_b(N=50_000, width=4112, height=2320, view=1, scale_mul=2.0)
    sc["Ks"][0, 0, 0] = sc["Ks"][0, 1, 1] = 2400.0
    tile = _check_ewa_instances(native, cuda_device, sc)
    n_tiles = ((4112 + 15) // 16) * ((2320 + 15) // 16)
    past = int((tile >= WINDOW_TILES).sum())
    print(f"{n_tiles} tiles in {-(-n_tiles // WINDOW_TILES)} windows, {past} instances past the first")
    assert n_tiles > WINDOW_TILES and past > 100


def _check_ewa_instances(native, cuda_device, scene):
    import importlib
    fg = importlib.import_module(native.__name__ + ".fastgs")
    inp = scenes.fastgs_inputs(scene)
    P = {k: torch.from_numpy(inp[k]).to(cuda_device) for k in
         ("means", "scales_raw", "rotations_raw", "opacities_raw", "sh0", "shN")}
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(cuda_device),
                          active_sh_bases=inp["active_sh_bases"], width=inp["width"], height=inp["height"],
                          focal_x=inp["fx"], focal_y=inp["fy"], center_x=inp["cx"], center_y=inp["cy"],
                          near_plane=inp["near_plane"], far_plane=inp["far_plane"])
    _, _, ctx = fg.default_backend().forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"], P["sh0"],
                                             P["shN"], torch.from_numpy(inp["w2c"]).to(cuda_device), s)
    torch.cuda.synchronize()

    def aligned(buf):  # the shim places its workspaces at the first 256-byte boundary of each byte tensor
        return buf[(-buf.data_ptr()) % 256:].cpu().numpy()

    a256 = lambda v: (v + 255) // 256 * 256
    N = inp["means"].shape[0]
    gw, gh = (inp["width"] + 15) // 16, (inp["height"] + 15) // 16
    prim = aligned(ctx["buffers"][0])
    o = 2 * a256(64 * N)  # gsb_fastgs.cu prim_layout: records, moments, counts, boxes, masks, depths
    counts = prim[o:o + 4 * N].view(np.int32)
    o += a256(4 * N)
    boxes = prim[o:o + 8 * N].view(np.uint32).reshape(N, 2)
    o += a256(8 * N)
    masks = prim[o:o + 4 * N].view(np.uint32)
    o += a256(4 * N)
    dbits = prim[o:o + 4 * N].view(np.uint32)
    toff = aligned(ctx["buffers"][1])[:4 * (gw * gh + 1)].view(np.int32)
    inst = ctx["buffers"][2].cpu().numpy().view(np.int32)
    assert toff[-1] == len(inst) > 0

    tile = np.repeat(np.arange(gw * gh), np.diff(toff))
    key = (dbits[inst].astype(np.uint64) << np.uint64(32)) | inst.astype(np.uint64)
    same = tile[1:] == tile[:-1]
    assert np.all(key[1:][same] > key[:-1][same])

    x0, y0 = boxes[inst, 0] & 0xFFFF, boxes[inst, 0] >> 16
    w, h = (boxes[inst, 1] & 0xFFFF).astype(np.int64), (boxes[inst, 1] >> 16).astype(np.int64)
    dx, dy = tile % gw - x0.astype(np.int64), tile // gw - y0.astype(np.int64)
    assert np.all((dx >= 0) & (dx < w) & (dy >= 0) & (dy < h))
    assert np.unique(inst.astype(np.int64) * (gw * gh) + tile).size == len(inst)
    assert np.array_equal(np.bincount(inst, minlength=N), np.maximum(counts, 0))
    small = w * h <= 32
    assert np.all((masks[inst[small]] >> (dy * w + dx)[small].astype(np.uint32)) & 1)
    print(f"{len(inst)} instances, largest box {int((w * h).max())} tiles, {int((~small).sum())} instances of boxes "
          f"larger than 32 tiles, largest tile list {int(np.diff(toff).max())}")
    assert (~small).sum() > 0
    return tile
