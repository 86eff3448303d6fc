"""Float32 CPU restatement of the exact mean neighbour distance (csrc/gsb_knn.cu, include/gsb200.h
gsb_knn_mean_dist), the exact version of the reference's compute_mean_neighbor_distances
(src/core/splat_data.cpp:63-111):

  for each point, the k = min(4, N) smallest squared distances over all points (itself and its duplicates included),
  each ((dx*dx) + (dy*dy)) + (dz*dz) in float32 with dx = q.x - p.x; walked in ascending order, the first (at most 3)
  with d2 > 1e-8f are averaged as sqrtf values summed in float32 in that order; 0.01f when none qualifies.

best_sq_brute computes the k smallest by brute force (small N).  best_sq_tree takes candidates from scipy's cKDTree
(float64, k >= 16), re-ranks them in float32, and re-checks by brute force every point whose float32 k-th best is
not safely below the float64 distance of its last candidate (so the candidates may miss nothing)."""
from __future__ import annotations

import numpy as np

F32 = np.float32
THRESH = F32(1e-8)


def sq_dist(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    """float32 squared distances of queries q [M,3] to points p [P,3] -> [M,P], no contraction."""
    dx = q[:, None, 0] - p[None, :, 0]
    dy = q[:, None, 1] - p[None, :, 1]
    dz = q[:, None, 2] - p[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def best_sq_brute(pts: np.ndarray, rows: np.ndarray | None = None, chunk: int = 512) -> np.ndarray:
    """The k = min(4, N) smallest squared distances of pts[rows] (all points by default), ascending, [M,k]."""
    pts = np.ascontiguousarray(pts, F32)
    n = pts.shape[0]
    k = min(4, n)
    rows = np.arange(n) if rows is None else rows
    out = np.empty((len(rows), k), F32)
    for s in range(0, len(rows), chunk):
        d = sq_dist(pts[rows[s:s + chunk]], pts)
        part = np.partition(d, k - 1, axis=1)[:, :k] if k < n else d
        out[s:s + chunk] = np.sort(part, axis=1)
    return out


def best_sq_tree(pts: np.ndarray, kc: int = 16) -> np.ndarray:
    from scipy.spatial import cKDTree

    pts = np.ascontiguousarray(pts, F32)
    n = pts.shape[0]
    k = min(4, n)
    if n <= kc:
        return best_sq_brute(pts)
    d64, idx = cKDTree(pts.astype(np.float64)).query(pts.astype(np.float64), k=kc)
    q = pts[:, None, :]
    c = pts[idx]
    dx, dy, dz = q[..., 0] - c[..., 0], q[..., 1] - c[..., 1], q[..., 2] - c[..., 2]
    d32 = np.sort((dx * dx + dy * dy) + dz * dz, axis=1)[:, :k]
    # a point outside the candidates is at float64 distance >= d64[:, -1]; its float32 square is within a relative
    # 2^-21 of the float64 one.  Where that bound does not clear the k-th best, fall back to brute force.
    safe = d32[:, k - 1].astype(np.float64) < (d64[:, -1] ** 2) * (1.0 - 1e-5)
    bad = np.nonzero(~safe)[0]
    if len(bad):
        d32[bad] = best_sq_brute(pts, bad)
    return d32


def mean_from_best(best: np.ndarray) -> np.ndarray:
    """compute_mean_neighbor_distances' loop over the ascending [M,k] squared distances."""
    m = best.shape[0]
    s = np.zeros(m, F32)
    valid = np.zeros(m, np.int32)
    for j in range(best.shape[1]):
        take = (best[:, j] > THRESH) & (valid < 3)
        s = np.where(take, s + np.sqrt(best[:, j]), s).astype(F32)
        valid += take
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = (s / valid.astype(F32)).astype(F32)
    return np.where(valid > 0, mean, F32(0.01)).astype(F32)


def mean_neighbor_distances(pts: np.ndarray, brute_max: int = 4096) -> np.ndarray:
    """The exact mean neighbour distances of float32 points [N,3] -> [N] float32."""
    pts = np.ascontiguousarray(pts, F32).reshape(-1, 3)
    n = pts.shape[0]
    if n == 0:
        return np.zeros(0, F32)
    best = best_sq_brute(pts) if n <= brute_max else best_sq_tree(pts)
    return mean_from_best(best)


# ---- the cloud shapes of the tests and bench_init.py -------------------------------------------------------------------
def cloud_uniform(n: int, seed: int = 0) -> np.ndarray:
    return np.random.default_rng(seed).uniform(-1.0, 1.0, (n, 3)).astype(F32)


def cloud_sfm(n: int, seed: int = 0) -> np.ndarray:
    """SfM-like: points on a few noisy planes and spheres (surfaces), in clusters of very different density."""
    rng = np.random.default_rng(seed)
    parts = []
    sizes = rng.multinomial(n, [0.35, 0.25, 0.2, 0.2])
    # a ground plane, a wall, two spheres
    g = sizes[0]
    parts.append(np.stack([rng.uniform(-5, 5, g), rng.normal(0, 0.01, g), rng.uniform(-5, 5, g)], 1))
    w = sizes[1]
    parts.append(np.stack([rng.uniform(-5, 5, w), rng.uniform(0, 3, w), 5 + rng.normal(0, 0.01, w)], 1))
    for c, r, m in (((1.0, 1.0, 0.0), 0.8, sizes[2]), ((-2.0, 0.5, 2.0), 0.3, sizes[3])):
        v = rng.normal(size=(m, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        parts.append(np.asarray(c) + r * v * (1 + rng.normal(0, 0.005, (m, 1))))
    pts = np.concatenate(parts).astype(F32)
    return pts[rng.permutation(n)]


def cloud_outliers(n: int, seed: int = 0, frac: float = 1e-3) -> np.ndarray:
    """The SfM-like cloud with a fraction of its points moved far out (up to 1e4 away), a few of them as pairs."""
    rng = np.random.default_rng(seed + 1)
    pts = cloud_sfm(n, seed)
    m = max(2, int(n * frac))
    sel = rng.choice(n, m, replace=False)
    far = rng.normal(size=(m, 3))
    far = far / np.linalg.norm(far, axis=1, keepdims=True) * rng.uniform(50, 1e4, (m, 1))
    far[1::2] = far[0::2][: len(far[1::2])] + rng.normal(0, 0.5, (len(far[1::2]), 3))  # outlier pairs
    pts[sel] = far.astype(F32)
    return pts


CLOUDS = {"uniform": cloud_uniform, "sfm": cloud_sfm, "outliers": cloud_outliers}


def hand_cases() -> dict:
    """The small hand-made clouds both the restatement and the kernel are checked on."""
    rng = np.random.default_rng(5)
    lat = np.stack(np.meshgrid(np.arange(6), np.arange(5), np.arange(4), indexing="ij"), -1).reshape(-1, 3)
    plane = rng.uniform(-1, 1, (300, 3)).astype(F32)
    plane[:, 2] = 0.5
    far = rng.uniform(0, 1, (200, 3)).astype(F32)
    far[7] = (1e5, -3e4, 2e4)
    dup = np.repeat(rng.uniform(-1, 1, (40, 3)), 3, axis=0)  # clusters of three duplicates
    cases = {f"n{n}": rng.uniform(-1, 1, (n, 3)).astype(F32) for n in range(0, 6)}
    cases.update({
        "all_equal": np.full((9, 3), 0.25, F32),
        "five_dup_one": np.concatenate([np.full((5, 3), -0.5, F32), np.asarray([[0.5, 0.25, 1.0]], F32)]),
        "lattice": lat.astype(F32) * F32(0.5),
        "planar": plane,
        "far_outlier": far,
        "dup_clusters": dup.astype(F32),
        "tiny_dist": np.asarray([[0, 0, 0], [5e-5, 0, 0], [0, 2e-4, 0], [1, 1, 1]], F32),  # d2 near 1e-8
    })
    return cases
