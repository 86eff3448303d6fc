"""Synthetic scenes for parity tests and the bench (numpy, seeded, float32).

Recipes follow SURVEY.md section 8(d), which itself follows the reference's test scene in
tests/test_rasterization.cpp:456-469 (all paths relative to /root/reference).
Quaternions are (w, x, y, z) and normalised; scales are post-exp, opacities post-sigmoid,
exactly what gs::training::rasterize hands to the gsplat:: ops (rasterizer.cpp:72-80).
"""
from __future__ import annotations

import numpy as np


def _finish(rng, N, sh_degree, means, scales, width, height, fx, fy, viewmat=None, background=True,
            sh_K=None):
    quats = rng.standard_normal((N, 4)).astype(np.float32)
    quats /= np.linalg.norm(quats, axis=-1, keepdims=True)
    opac = (rng.random(N, dtype=np.float32) * 0.5 + 0.3).astype(np.float32)
    K = sh_K if sh_K is not None else (sh_degree + 1) ** 2
    sh = ((rng.random((N, K, 3), dtype=np.float32) - 0.5) * 0.3).astype(np.float32)
    Ks = np.array([[[fx, 0, width / 2.0], [0, fy, height / 2.0], [0, 0, 1]]], np.float32)
    if viewmat is None:
        viewmat = np.eye(4, dtype=np.float32)
    bg = rng.random((1, 3), dtype=np.float32) if background else None
    return dict(means=means.astype(np.float32), quats=quats, scales=scales.astype(np.float32),
                opacities=opac, sh_coeffs=sh, sh_degree=sh_degree, viewmats=viewmat[None].astype(np.float32),
                Ks=Ks, width=width, height=height, tile_size=16, background=bg)


def scene_a(N=10_000, width=256, height=256, sh_degree=0, seed=42, background=False):
    """Config A: 10k Gaussians, 256x256, SH deg 0, identity view (BASELINE.json configs[0])."""
    rng = np.random.default_rng(seed)
    means = rng.random((N, 3), dtype=np.float32) * 2 - 1
    means[:, 2] = np.abs(means[:, 2]) + 2
    scales = rng.random((N, 3), dtype=np.float32) * 0.05 + 0.01
    return _finish(rng, N, sh_degree, means, scales, width, height, 300.0, 300.0, background=background)


def look_at(eye, target, up=(0.0, -1.0, 0.0)):
    """World->camera [4,4] (OpenCV convention: +z forward, +y down)."""
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    f = target - eye
    f /= np.linalg.norm(f)
    r = np.cross(f, -up)
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    R = np.stack([r, d, f])  # rows
    V = np.eye(4)
    V[:3, :3] = R
    V[:3, 3] = -R @ eye
    return V.astype(np.float32)


def scene_b(N=1_000_000, width=1920, height=1080, sh_degree=3, seed=42, view=None, scale_mul=None,
            background=True):
    """Config B/D: N Gaussians in a frustum-shaped slab, 1080p, SH deg 3 (BASELINE.json
    configs[1], [3]).  `view` = None (identity) or an index 0..7 on the config-E camera ring
    (radius 3 about (0,0,3), looking at it)."""
    rng = np.random.default_rng(seed)
    means = np.empty((N, 3), np.float32)
    means[:, 0] = rng.random(N, dtype=np.float32) * 3.0 - 1.5
    means[:, 1] = rng.random(N, dtype=np.float32) * 1.7 - 0.85
    means[:, 2] = rng.random(N, dtype=np.float32) * 2.0 + 2.0
    lo, hi = np.log(0.003), np.log(0.02)
    scales = np.exp(rng.random((N, 3), dtype=np.float32) * (hi - lo) + lo)
    if scale_mul is None:
        scale_mul = (1_000_000 / N) ** (1.0 / 3.0) if N > 1_000_000 else 1.0
    scales = scales * np.float32(scale_mul)
    viewmat = None
    if view is not None:
        ang = 2 * np.pi * (view % 8) / 8.0
        # ring of radius 3 about the slab centre (0,0,3); view 0 is the identity camera at the origin
        eye = np.array([3.0 * np.sin(ang), 0.0, 3.0 - 3.0 * np.cos(ang)])
        viewmat = look_at(eye, (0.0, 0.0, 3.0))
    return _finish(rng, N, sh_degree, means, scales, width, height, 1600.0, 1600.0, viewmat=viewmat,
                   background=background)


def scene_small(N=2000, width=200, height=120, sh_degree=3, seed=7, view=None):
    """A small 1080p-like scene (non-multiple-of-16 size, rotated camera) for CPU-sized parity."""
    rng = np.random.default_rng(seed)
    means = np.empty((N, 3), np.float32)
    means[:, 0] = rng.random(N, dtype=np.float32) * 3.0 - 1.5
    means[:, 1] = rng.random(N, dtype=np.float32) * 1.8 - 0.9
    means[:, 2] = rng.random(N, dtype=np.float32) * 2.0 + 2.0
    scales = np.exp(rng.random((N, 3), dtype=np.float32) * (np.log(0.15) - np.log(0.02)) + np.log(0.02))
    viewmat = None
    if view is not None:
        ang = 2 * np.pi * (view % 8) / 8.0
        eye = np.array([3.0 * np.sin(ang), 0.2, 3.0 - 3.0 * np.cos(ang)])
        viewmat = look_at(eye, (0.0, 0.0, 3.0))
    return _finish(rng, N, sh_degree, means, scales, width, height, 160.0, 170.0, viewmat=viewmat)


def scene_one_visible(N=2000, width=200, height=120, sh_degree=3, seed=13):
    """One Gaussian in view, every other one culled: behind the camera, or far outside the frustum.  With a single
    Gaussian that has tiles, the intersect stage's depth sort skips all four of its radix passes."""
    rng = np.random.default_rng(seed)
    means = np.empty((N, 3), np.float32)
    means[:, 0] = rng.random(N, dtype=np.float32) * 3.0 - 1.5
    means[:, 1] = rng.random(N, dtype=np.float32) * 1.8 - 0.9
    means[:, 2] = -(rng.random(N, dtype=np.float32) * 2.0 + 1.0)  # behind the camera
    side = rng.random(N) < 0.3
    means[side, 0] = np.where(rng.random(int(side.sum())) < 0.5, -60.0, 60.0)  # in front, 20x the frustum's width away
    means[side, 2] = rng.random(int(side.sum()), dtype=np.float32) * 2.0 + 2.0
    k = N // 2
    means[k] = (0.05, -0.03, 2.5)
    scales = np.exp(rng.random((N, 3), dtype=np.float32) * (np.log(0.15) - np.log(0.02)) + np.log(0.02))
    scales[k] = (0.4, 0.25, 0.3)  # covers most of the frame
    return _finish(rng, N, sh_degree, means, scales, width, height, 160.0, 170.0)


def scene_wall(N=1500, width=200, height=120, sh_degree=3, seed=17, depth=3.0):
    """A fronto-parallel wall: identity view and every Gaussian at camera depth `depth` exactly, with footprints large
    enough to overlap many times, so the order of equal-depth Gaussians (ascending index, the reference's stable sort)
    decides the image.  The intersect stage's depth sort skips all four of its radix passes."""
    rng = np.random.default_rng(seed)
    means = np.empty((N, 3), np.float32)
    means[:, 0] = rng.random(N, dtype=np.float32) * 4.4 - 2.2
    means[:, 1] = rng.random(N, dtype=np.float32) * 2.6 - 1.3
    means[:, 2] = depth
    scales = np.exp(rng.random((N, 3), dtype=np.float32) * (np.log(0.12) - np.log(0.04)) + np.log(0.04))
    return _finish(rng, N, sh_degree, means, scales, width, height, 160.0, 170.0)


def fastgs_inputs(scene: dict, seed: int = 3) -> dict:
    """The RAW parameters the reference's fastgs rasterizer takes (fast_rasterizer.cpp:24-54) for a scene dict:
    log-scales, un-normalised quaternions, logit opacities, sh0 / shN split, w2c and the camera position."""
    rng = np.random.default_rng(seed)
    n = scene["means"].shape[0]
    sh = scene["sh_coeffs"]
    V = scene["viewmats"][0].astype(np.float64)
    Ks = scene["Ks"][0]
    qscale = (rng.random((n, 1), dtype=np.float32) * 1.5 + 0.5).astype(np.float32)
    o = scene["opacities"].astype(np.float64)
    return dict(
        means=scene["means"], scales_raw=np.log(scene["scales"]).astype(np.float32),
        rotations_raw=(scene["quats"] * qscale).astype(np.float32),
        opacities_raw=np.log(o / (1.0 - o)).astype(np.float32).reshape(n, 1),
        sh0=np.ascontiguousarray(sh[:, :1, :]), shN=np.ascontiguousarray(sh[:, 1:, :]),
        w2c=scene["viewmats"][0].copy(), cam_position=(-V[:3, :3].T @ V[:3, 3]).astype(np.float32),
        active_sh_bases=(scene["sh_degree"] + 1) ** 2, width=scene["width"], height=scene["height"],
        fx=float(Ks[0, 0]), fy=float(Ks[1, 1]), cx=float(Ks[0, 2]), cy=float(Ks[1, 2]), near_plane=0.01, far_plane=1e10)
