"""Generate the model set-up fixtures from the reference's own third-party code (oracle/build_ref_knn.py):

  knn_ref_small.npz   points (SfM-like, outlier-laden, lattice) and the reference's approximate mean neighbour
                      distances (nanoflann, leaf size 10, KNNResultSet(4), SearchParameters(10))
  ply_tinyply.npz     small models at SH degree 0 and 3 in SplatData layout
  ply_tinyply_sh{0,3}.ply   those models as write_ply_impl writes them through tinyply, after to_point_cloud's
                      transpose of sh0 / shN, zero normals and normalised rotation (splat_data.cpp:484-506)

Runs where the reference's sources are present: python tests/golden/make_knn_ply_golden.py"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import build_ref_knn  # noqa: E402
import knn_restatement as kr  # noqa: E402


def model(n, degree, seed):
    g = torch.Generator().manual_seed(seed)
    K = (degree + 1) ** 2
    return {"means": torch.randn(n, 3, generator=g), "sh0": torch.randn(n, 1, 3, generator=g),
            "shN": torch.randn(n, K - 1, 3, generator=g), "scaling_raw": torch.randn(n, 3, generator=g) - 3,
            "rotation_raw": torch.randn(n, 4, generator=g) * 2, "opacity_raw": torch.randn(n, 1, generator=g)}


def main():
    build_ref_knn.build()
    lib = build_ref_knn.load()
    pts = np.concatenate([kr.cloud_sfm(2500, seed=3), kr.cloud_outliers(1500, seed=4),
                          kr.hand_cases()["lattice"] + np.float32(7.0)]).astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "knn_ref_small.npz"), points=pts, ref=build_ref_knn.mean_dist(lib, pts))

    arrays = {}
    for degree, n in ((0, 5), (3, 7)):
        P = model(n, degree, seed=11 + degree)
        arrays.update({f"sh{degree}_{k}": v.numpy() for k, v in P.items()})
        names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + \
            [f"f_rest_{i}" for i in range(P["shN"].shape[1] * 3)] + ["opacity"] + \
            [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)]
        groups = [P["means"], torch.zeros_like(P["means"]), P["sh0"].transpose(1, 2).flatten(1),
                  P["shN"].transpose(1, 2).flatten(1), P["opacity_raw"], P["scaling_raw"],
                  torch.nn.functional.normalize(P["rotation_raw"], dim=-1)]
        build_ref_knn.write_ply(lib, os.path.join(HERE, f"ply_tinyply_sh{degree}.ply"),
                                [g.contiguous().numpy() for g in groups], names)
    np.savez_compressed(os.path.join(HERE, "ply_tinyply.npz"), **arrays)


if __name__ == "__main__":
    main()
