"""CPU: the model set-up and export without a device.

  * the float32 restatement of the exact mean neighbour distance (knn_restatement.py) against a scalar brute force on
    hand-made clouds, and its candidate path against its brute-force path;
  * the exact distances are at most the reference's approximate ones (nanoflann, eps = 10) on the stored fixture, and
    live where oracle/_ref holds the harness;
  * save_ply byte for byte against files tinyply wrote, load_ply(save_ply(x)) == x, property order and defaults, and
    the files load_ply refuses;
  * a caller compiled against the FusedOps.h declaration links against the shim."""
import os
import subprocess

import numpy as np
import pytest
import torch

import knn_restatement as kr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
F32 = np.float32


def scalar_oracle(pts):
    """compute_mean_neighbor_distances with an exact search, one point at a time in float32 scalars."""
    pts = np.asarray(pts, F32)
    n = len(pts)
    out = np.empty(n, F32)
    for i in range(n):
        q = pts[i]
        d = []
        for p in pts:
            dx, dy, dz = F32(q[0] - p[0]), F32(q[1] - p[1]), F32(q[2] - p[2])
            d.append(F32(F32(F32(dx * dx) + F32(dy * dy)) + F32(dz * dz)))
        d.sort()
        s, valid = F32(0.0), 0
        for j in range(min(4, n)):
            if valid < 3 and d[j] > F32(1e-8):
                s = F32(s + np.sqrt(d[j]))
                valid += 1
        out[i] = F32(s / F32(valid)) if valid else F32(0.01)
    return out


@pytest.mark.parametrize("case", sorted(kr.hand_cases()))
def test_restatement_equals_scalar_brute_force(case):
    pts = kr.hand_cases()[case]
    want = scalar_oracle(pts)
    got = kr.mean_neighbor_distances(pts)
    assert got.dtype == F32 and got.shape == (len(pts),)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


def test_restatement_edge_values():
    c = kr.hand_cases()
    assert (kr.mean_neighbor_distances(c["n1"]) == F32(0.01)).all()
    assert (kr.mean_neighbor_distances(c["all_equal"]) == F32(0.01)).all()
    five = kr.mean_neighbor_distances(c["five_dup_one"])
    d = F32(np.sqrt(F32(F32(F32(1.0) + F32(0.5625)) + F32(2.25))))
    # the four nearest of a duplicate are all at distance 0 (KNNResultSet(4)); the distinct point's first three
    # qualifying distances are its distances to the duplicates
    assert (five[:5] == F32(0.01)).all() and five[5] == d
    assert kr.mean_neighbor_distances(np.zeros((0, 3), F32)).shape == (0,)


@pytest.mark.parametrize("shape", sorted(kr.CLOUDS))
def test_candidate_path_equals_brute_force(shape):
    pts = kr.CLOUDS[shape](3000, seed=2)
    np.testing.assert_array_equal(kr.mean_from_best(kr.best_sq_tree(pts)), kr.mean_from_best(kr.best_sq_brute(pts)))


def _compare_with_reference(pts, ref, label):
    exact = kr.mean_neighbor_distances(pts)
    if len(pts) == 0:
        return 0.0
    assert (exact <= ref).all(), f"{label}: the exact mean exceeds the reference's at {np.nonzero(exact > ref)[0][:10]}"
    frac = float((exact != ref).mean())
    print(f"{label}: {len(pts)} points, the reference's approximate search differs at {100 * frac:.2f}% of them, "
          f"by at most {float(np.max(ref / exact - 1)):.3g} relative")
    return frac


def test_exact_is_at_most_the_stored_reference():
    z = np.load(os.path.join(GOLDEN, "knn_ref_small.npz"))
    _compare_with_reference(z["points"], z["ref"], "stored fixture")


def test_exact_is_at_most_the_live_reference():
    from oracle import build_ref_knn

    lib = build_ref_knn.load()
    if lib is None:
        pytest.skip("the reference's nanoflann harness is not built (oracle/_ref)")
    for shape, fn in kr.CLOUDS.items():
        pts = fn(20000, seed=9)
        _compare_with_reference(pts, build_ref_knn.mean_dist(lib, pts), f"live {shape}")
    for name, pts in kr.hand_cases().items():
        _compare_with_reference(pts, build_ref_knn.mean_dist(lib, pts), f"live {name}")


# ---- PLY ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model(pkg):
    import importlib
    return importlib.import_module(pkg.__name__ + ".model")


def golden_params(degree):
    z = np.load(os.path.join(GOLDEN, "ply_tinyply.npz"))
    keys = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")
    return {k: torch.from_numpy(z[f"sh{degree}_{k}"]) for k in keys}


@pytest.mark.parametrize("degree", [0, 3])
def test_save_ply_is_byte_identical_to_tinyply(model, tmp_path, degree):
    P = golden_params(degree)
    path = tmp_path / "m.ply"
    model.save_ply(P, path)
    assert path.read_bytes() == open(os.path.join(GOLDEN, f"ply_tinyply_sh{degree}.ply"), "rb").read()


@pytest.mark.parametrize("degree", [0, 3])
def test_load_of_save_roundtrips(model, tmp_path, degree):
    P = golden_params(degree)
    P["opacity_raw"] = P["opacity_raw"].reshape(-1, 1)
    path = tmp_path / "m.ply"
    model.save_ply(P, path)
    Q, scene_scale, sh = model.load_ply(path, device="cpu")
    assert scene_scale == 0.5
    # a file without f_rest_* columns gets the reference's 15 zero rows, hence degree 3
    assert sh == (degree if degree else 3)
    for k, v in P.items():
        w = torch.nn.functional.normalize(v, dim=-1) if k == "rotation_raw" else v
        if k == "shN" and degree == 0:
            w = torch.zeros(v.shape[0], 15, 3)
        assert Q[k].shape == w.shape and Q[k].dtype == torch.float32, k
        assert torch.equal(Q[k].detach(), w), k
    assert Q["opacity_raw"].shape == (P["means"].shape[0], 1)


def write_ply(path, names, table, fmt="binary_little_endian", types=None, endian="<"):
    types = types or ["float"] * len(names)
    head = ["ply", f"format {fmt} 1.0", "comment written by a test", f"element vertex {len(table)}"]
    head += [f"property {t} {n}" for t, n in zip(types, names)] + ["end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        f.write(np.asarray(table, endian + "f4").tobytes())


def test_load_ply_reads_any_property_order(model, tmp_path):
    P = golden_params(3)
    names = model.ply_attribute_names(P)
    table = np.frombuffer(model.ply_bytes(P)[len(model.ply_header(names, 7)):], "<f4").reshape(7, -1)
    perm = np.random.default_rng(0).permutation(len(names))
    path = tmp_path / "shuffled.ply"
    write_ply(path, [names[i] for i in perm], table[:, perm])
    Q, _, sh = model.load_ply(path, device="cpu")
    model.save_ply(P, tmp_path / "ordered.ply")
    R, _, _ = model.load_ply(tmp_path / "ordered.ply", device="cpu")
    assert sh == 3
    for k in Q:
        assert torch.equal(Q[k], R[k]), k


def test_load_ply_defaults_for_missing_properties(model, tmp_path):
    pts = np.asarray([[1, 2, 3], [4, 5, 6]], F32)
    path = tmp_path / "xyz.ply"
    write_ply(path, ["z", "x", "y"], pts[:, [2, 0, 1]])
    Q, scene_scale, sh = model.load_ply(path, device="cpu")
    assert torch.equal(Q["means"], torch.from_numpy(pts))
    assert torch.equal(Q["scaling_raw"], torch.full((2, 3), -5.0))
    assert torch.equal(Q["rotation_raw"], torch.tensor([[1.0, 0, 0, 0]] * 2))
    assert torch.equal(Q["opacity_raw"], torch.zeros(2, 1))
    assert torch.equal(Q["sh0"], torch.zeros(2, 1, 3)) and torch.equal(Q["shN"], torch.zeros(2, 15, 3))
    assert sh == 3 and scene_scale == 0.5
    # degree 1: nine f_rest columns
    names = ["x", "y", "z"] + [f"f_rest_{i}" for i in range(9)]
    table = np.arange(2 * 12, dtype=F32).reshape(2, 12)
    write_ply(tmp_path / "d1.ply", names, table)
    Q, _, sh = model.load_ply(tmp_path / "d1.ply", device="cpu")
    assert sh == 1 and Q["shN"].shape == (2, 3, 3)
    assert torch.equal(Q["shN"][1], torch.from_numpy(table[1, 3:].reshape(3, 3).T.copy()))


@pytest.mark.parametrize("kind", ["ascii", "big_endian", "double", "uchar"])
def test_load_ply_rejects_unsupported_files(model, tmp_path, kind):
    path = tmp_path / f"{kind}.ply"
    if kind == "ascii":
        with open(path, "w") as f:
            f.write("ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\n"
                    "property float z\nend_header\n1 2 3\n")
    elif kind == "big_endian":
        write_ply(path, ["x", "y", "z"], [[1, 2, 3]], fmt="binary_big_endian", endian=">")
    else:
        t = "double" if kind == "double" else "uchar"
        write_ply(path, ["x", "y", "z"], [[1, 2, 3]], types=["float", "float", t])
    with pytest.raises(ValueError):
        model.load_ply(path, device="cpu")


def test_random_point_cloud_matches_the_loader_fallback(model):
    pos, col = model.random_point_cloud()
    torch.manual_seed(8128)
    want = torch.rand((10000, 3)) * 2.0 - 1.0
    assert torch.equal(pos, want) and col.dtype == torch.uint8 and col.shape == (10000, 3)
    assert torch.equal(col, torch.randint(0, 256, (10000, 3), dtype=torch.uint8))


def test_init_model_on_the_cpu_with_a_stand_in_search(model):
    """The torch composition of init_model_from_pointcloud, with the restatement standing in for the kernel."""
    pts = torch.from_numpy(kr.cloud_sfm(500, seed=1))
    col = torch.randint(0, 256, (500, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    search = lambda m: torch.from_numpy(kr.mean_neighbor_distances(m.detach().numpy()))  # noqa: E731
    P, scale, deg = model.init_model_from_pointcloud(pts, col, torch.zeros(3), model.InitConfig(sh_degree=2),
                                                     device="cpu", neighbor_distances=search)
    assert deg == 2 and list(P) == ["means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw"]
    assert P["shN"].shape == (500, 8, 3) and P["opacity_raw"].shape == (500, 1)
    d = np.maximum(kr.mean_neighbor_distances(pts.numpy()), 1e-7)
    np.testing.assert_allclose(P["scaling_raw"][:, 0].detach().numpy(), np.log(np.sqrt(d) * 0.1), rtol=1e-6)
    assert scale == float(torch.norm(pts, 2, 1).median())
    assert torch.all(P["shN"] == 0) and torch.all(P["rotation_raw"][:, 0] == 1)
    np.testing.assert_allclose(P["opacity_raw"].detach().numpy(), 0.0, atol=1e-7)


def test_fusedops_declaration_links_against_the_shim(pkg, tmp_path):
    """A caller of gsplat::mean_neighbor_distances[_out] compiles against FusedOps.h and links with --no-undefined."""
    from torch.utils import cpp_extension as ce

    pkg.build()
    src = tmp_path / "caller.cpp"
    src.write_text('#include "FusedOps.h"\n'
                   "at::Tensor init_scales(const at::Tensor &p) { return gsplat::mean_neighbor_distances(p); }\n"
                   "void init_scales_into(const at::Tensor &p, at::Tensor o, at::Tensor s) {\n"
                   "    gsplat::mean_neighbor_distances_out(p, o, s);\n}\n")
    inc = []
    for i in [os.path.join(ROOT, "include", "gsplat"), os.path.join(ROOT, "include")] + ce.include_paths() + \
            ["/usr/local/cuda/include"]:
        inc += ["-I", i]
    obj = str(tmp_path / "caller.o")
    subprocess.run(["g++", "-std=c++17", "-O0", "-fPIC", "-DGSB_NO_GLM", "-c", str(src), "-o", obj] + inc, check=True)
    lib_dir = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib")
    tl = ce.library_paths()[0]
    so = str(tmp_path / "libcaller.so")
    subprocess.run(["g++", "-shared", "-o", so, obj, "-L", lib_dir, "-lgsplat_b200", "-lgsb200", "-L", tl, "-ltorch",
                    "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Wl,--no-undefined",
                    "-Wl,-rpath," + lib_dir, "-Wl,-rpath," + tl], check=True)
    out = subprocess.run(["nm", "-D", "--undefined-only", "-C", so], capture_output=True, text=True).stdout
    assert "gsplat::mean_neighbor_distances(at::Tensor)" in out
    assert "gsplat::mean_neighbor_distances_out(at::Tensor, at::Tensor, at::Tensor)" in out


def test_knn_c_abi_validation(pkg):
    """gsb_knn_mean_dist's argument checks, before anything reaches the device."""
    import ctypes as C

    path = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsb200.so")
    if not os.path.exists(path):
        pkg.build()
    L = C.CDLL(path)
    L.gsb_knn_mean_dist_workspace.restype = C.c_size_t
    buf = np.zeros(1 << 20, np.uint8)
    base = (buf.ctypes.data + 255) & ~255
    ptr, null = C.c_void_p(base), C.c_void_p(None)
    u32, sz = C.c_uint32, C.c_size_t
    need = L.gsb_knn_mean_dist_workspace(u32(100))
    assert need < (1 << 20) - 256
    assert L.gsb_knn_mean_dist_workspace(u32(1000)) > need

    def call(N=100, pts=ptr, out=ptr, ws=ptr, nb=None, status=ptr):
        return L.gsb_knn_mean_dist(u32(N), pts, out, ws, sz(need if nb is None else nb), status, null)

    assert call(N=(1 << 28) + 1) == -1
    assert call(pts=null) == -1 and call(out=null) == -1 and call(status=null) == -1
    assert call(ws=null) == -3 and call(ws=C.c_void_p(base + 4)) == -3 and call(nb=need - 1) == -3
