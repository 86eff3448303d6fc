"""Python mirror of the reference's model set-up and PLY I/O (src/core/splat_data.cpp, src/loader/formats/ply.cpp,
src/training/training_setup.cpp), on this library's nearest-neighbour kernel:

  mean_neighbor_distances     compute_mean_neighbor_distances (splat_data.cpp:63-111) as one sm_90a call
                              (csrc/gsb_knn.cu): exact, where the reference's nanoflann query (eps = 10) is approximate
  InitConfig                  the optimization parameters the set-up reads (parameters.hpp:30-34, 72-74)
  init_model_from_pointcloud  SplatData::init_model_from_pointcloud (splat_data.cpp:508-614): the six raw parameter
                              tensors in strategy.PARAM_GROUPS order, the scene scale and the SH degree
  random_point_cloud          the loader's fallback cloud (training_setup.cpp:82-91)
  save_ply                    SplatData::save_ply -> to_point_cloud + write_ply_impl (splat_data.cpp:113-169, 402-418,
                              484-506), byte for byte what tinyply writes
  load_ply                    load_ply (ply.cpp:497-636)

Deviations from the reference, on purpose:
  * The neighbour search is exact (DESIGN.md 4.17): every initial scale is at most the reference's, and equal where its
    approximate search happens to find the true neighbours.
  * load_ply locates every property by name, so the f_dc_* / f_rest_* columns need not be contiguous, and it rejects
    non-float32 properties (the reference skips them without advancing its offsets and so misreads the file).
  * save_ply is synchronous; the reference's asynchronous save only moves the same write to a thread."""
from __future__ import annotations

import math
import re
from dataclasses import dataclass

import numpy as np
import torch

from . import _product_ns, load
from .strategy import PARAM_GROUPS

SH_C0 = 0.28209479177387814  # splat_data.cpp:538 (kInvSH, a float there)


def _f32(v: float) -> float:
    """A C++ float parameter as the double torch receives it."""
    return float(np.float32(v))


def mean_neighbor_distances(points: torch.Tensor) -> torch.Tensor:
    """[N] float32 on the device: for each point of points [N,3] (float32, CUDA) the mean distance to its (up to three)
    nearest neighbours at a squared distance above 1e-8, searched exactly; 0.01 where none qualifies.  Raises on
    non-finite coordinates (one read-back)."""
    load()
    return _product_ns().mean_neighbor_distances(points)


@dataclass
class InitConfig:
    """The optimization parameters init_model_from_pointcloud reads (include/core/parameters.hpp)."""
    sh_degree: int = 3
    init_scaling: float = 0.1
    init_opacity: float = 0.5
    random: bool = False          # random initialisation instead of the point cloud
    init_num_pts: int = 100_000
    init_extent: float = 3.0


def init_model_from_pointcloud(points: torch.Tensor | None, colors: torch.Tensor | None, scene_center: torch.Tensor,
                               cfg: InitConfig | None = None, device: torch.device | str = "cuda",
                               neighbor_distances=mean_neighbor_distances):
    """(params, scene_scale, sh_degree) of a new model: params holds means, sh0 [N,1,3], shN [N,K-1,3], scaling_raw,
    rotation_raw [N,4] and opacity_raw [N,1] (strategy.PARAM_GROUPS), contiguous, float32, requiring grad, ready for
    training.FusedAdam and the densification strategies.  points [N,3] float32 and colors [N,3] (0..255, usually
    uint8) are the point cloud (unused when cfg.random); scene_center [3].  The torch operations are the reference's,
    in its order; `neighbor_distances` is the exact search (a stand-in may be passed for tests)."""
    cfg = cfg or InitConfig()
    dev = torch.device(device)
    f32 = dict(dtype=torch.float32, device=dev)
    with torch.no_grad():
        if cfg.random:
            n = int(cfg.init_num_pts)
            positions = (torch.rand((n, 3), **f32) * 2.0 - 1.0) * _f32(cfg.init_extent)
            colors = torch.rand((n, 3), **f32)
        else:
            positions = points
            colors = colors / 255.0
        scene_center = scene_center.to(positions.device)
        dists = torch.norm(positions - scene_center, 2, 1)
        scene_scale = dists.median().item()

        if cfg.random:
            means = (positions * scene_scale).to(dev)
        else:
            means = positions.to(dev, copy=True)  # the caller's tensor does not become a parameter
        nn_dist = torch.clamp_min(neighbor_distances(means.contiguous()), 1e-7)
        scaling = torch.log(torch.sqrt(nn_dist) * _f32(cfg.init_scaling)).unsqueeze(-1).repeat(1, 3).to(**f32)
        rotation = torch.zeros((means.shape[0], 4), **f32)
        rotation[:, 0] = 1
        opacity = torch.logit(_f32(cfg.init_opacity) * torch.ones((means.shape[0], 1), **f32))
        fused_color = (colors.to(dev) - 0.5) / _f32(SH_C0)
        feature_shape = int((cfg.sh_degree + 1) ** 2)
        shs = torch.zeros((fused_color.shape[0], 3, feature_shape), **f32)
        shs[:, :, 0] = fused_color
        sh0 = shs[:, :, 0:1].transpose(1, 2).contiguous()
        shN = shs[:, :, 1:].transpose(1, 2).contiguous()
    tensors = (means, sh0, shN, scaling, rotation, opacity)
    params = {k: t.contiguous().requires_grad_(True) for k, t in zip(PARAM_GROUPS, tensors)}
    return params, scene_scale, int(cfg.sh_degree)


def random_point_cloud(n: int = 10_000, seed: int = 8128):
    """(positions [n,3] float32 in [-1, 1], colors [n,3] uint8) on the CPU, the loader's fallback when a dataset has no
    point cloud: torch.manual_seed(seed), rand, then randint(0, 256) (training_setup.cpp:82-91)."""
    torch.manual_seed(seed)
    positions = torch.rand((n, 3))
    positions = positions * 2.0 - 1.0
    colors = torch.randint(0, 256, (n, 3), dtype=torch.uint8)
    return positions, colors


# ---- PLY ---------------------------------------------------------------------------------------------------------------
def ply_attribute_names(params: dict) -> list:
    """SplatData::get_attribute_names (splat_data.cpp:402-418)."""
    names = ["x", "y", "z", "nx", "ny", "nz"]
    names += [f"f_dc_{i}" for i in range(params["sh0"].shape[1] * params["sh0"].shape[2])]
    names += [f"f_rest_{i}" for i in range(params["shN"].shape[1] * params["shN"].shape[2])]
    names.append("opacity")
    names += [f"scale_{i}" for i in range(params["scaling_raw"].shape[1])]
    names += [f"rot_{i}" for i in range(params["rotation_raw"].shape[1])]
    return names


def ply_header(names: list, n: int) -> bytes:
    """tinyply's binary header (tinyply.hpp:673-707): no comments, every property float."""
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    lines += [f"property float {a}" for a in names]
    lines.append("end_header")
    return ("\n".join(lines) + "\n").encode("ascii")


def ply_bytes(params: dict) -> bytes:
    """The bytes save_ply writes.  The vertex rows are gathered on the device, as to_point_cloud lays them out
    (sh0 / shN channel-major, zero normals, normalised rotation), and copied to the host once."""
    with torch.no_grad():
        means = params["means"].detach().float()
        n = means.shape[0]
        cols = [means, torch.zeros_like(means),
                params["sh0"].detach().transpose(1, 2).flatten(1),
                params["shN"].detach().transpose(1, 2).flatten(1),
                params["opacity_raw"].detach().reshape(n, -1),
                params["scaling_raw"].detach(),
                torch.nn.functional.normalize(params["rotation_raw"].detach(), dim=-1)]
        rows = torch.cat([c.reshape(n, -1).float() for c in cols], 1).contiguous().cpu().numpy()
    names = ply_attribute_names(params)
    assert rows.shape[1] == len(names), (rows.shape, len(names))
    return ply_header(names, n) + rows.astype("<f4", copy=False).tobytes()


def save_ply(params: dict, path) -> None:
    """SplatData::save_ply with join_threads: the model as a binary little-endian float32 PLY at `path`."""
    data = ply_bytes(params)
    with open(path, "wb") as f:
        f.write(data)


_HEADER_LIMIT = 10000  # lines (ply.cpp MAX_HEADER_LINES)


def _parse_header(buf: bytes):
    if not (buf.startswith(b"ply\n") or buf.startswith(b"ply\r\n")):
        raise ValueError("not a PLY file (missing the 'ply' magic line)")
    pos, fmt, n, props, in_vertex = 0, None, None, [], False
    for _ in range(_HEADER_LIMIT):
        end = buf.find(b"\n", pos)
        if end < 0:
            raise ValueError("PLY header has no end_header line")
        line = buf[pos:end].rstrip(b"\r").decode("ascii", "replace").strip()
        pos = end + 1
        if not line or line.startswith("#") or line.startswith("comment") or line.startswith("obj_info"):
            continue
        tok = line.split()
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            in_vertex = tok[1] == "vertex"
            if in_vertex:
                n = int(tok[2])
            elif n is not None:
                raise ValueError(f"PLY element '{tok[1]}' after vertex is not supported")
        elif tok[0] == "property" and in_vertex:
            if tok[1] == "list":
                raise ValueError(f"PLY list property '{tok[-1]}' is not supported")
            if tok[1] not in ("float", "float32"):
                raise ValueError(f"PLY property '{tok[2]}' is {tok[1]}; only float32 properties are supported")
            props.append(tok[2])
        elif tok[0] == "end_header":
            if fmt != "binary_little_endian":
                raise ValueError(f"only binary_little_endian PLY is supported (the file is {fmt})")
            if n is None:
                raise ValueError("PLY file has no vertex element")
            return pos, n, props
        elif tok[0] != "ply":
            continue
    raise ValueError("PLY header too long")


def load_ply(path, device: torch.device | str = "cuda"):
    """(params, scene_scale, sh_degree) of a saved model, as the reference's load_ply reads it: x y z, f_dc_*, f_rest_*,
    opacity, scale_*, rot_* in any order.  Missing ones take its defaults: zero means, opacity and SH, scale -5,
    identity rotation, 15 shN rows; sh_degree = int(sqrt(Bn + 1)) - 1, scene_scale = 0.5.  Raises ValueError on ASCII
    or big-endian files and on properties that are not float32."""
    with open(path, "rb") as f:
        buf = f.read()
    off, n, props = _parse_header(buf)
    ncol = len(props)
    if len(buf) - off < n * ncol * 4:
        raise ValueError(f"PLY file holds fewer than the {n} vertices its header declares")
    table = np.frombuffer(buf, "<f4", count=n * ncol, offset=off).reshape(n, ncol)
    col = {name: i for i, name in enumerate(props)}

    def numbered(prefix):
        idx = {int(m.group(1)): i for name, i in col.items() if (m := re.fullmatch(re.escape(prefix) + r"(\d+)", name))}
        count = max(idx) + 1 if idx else 0
        return count, idx

    def gather(names, default):
        out = np.full((n, len(names)), default, np.float32)
        for j, name in enumerate(names):
            if name in col:
                out[:, j] = table[:, col[name]]
        return out

    means = gather(["x", "y", "z"], 0.0)

    def sh(prefix, default_rows):
        count, idx = numbered(prefix)
        if count > 0 and count % 3 == 0:
            b = count // 3
            flat = np.zeros((n, count), np.float32)
            for j, i in idx.items():
                flat[:, j] = table[:, i]
            return flat.reshape(n, 3, b).transpose(0, 2, 1)  # channel-major on file -> [N, B, 3]
        return np.zeros((n, default_rows, 3), np.float32)

    sh0 = sh("f_dc_", 1)
    shN = sh("f_rest_", 15)
    opacity = gather(["opacity"], 0.0)
    scaling = gather(["scale_0", "scale_1", "scale_2"], 0.0) if "scale_0" in col else np.full((n, 3), -5.0, np.float32)
    if "rot_0" in col:
        rotation = gather(["rot_0", "rot_1", "rot_2", "rot_3"], 0.0)
    else:
        rotation = np.zeros((n, 4), np.float32)
        rotation[:, 0] = 1.0
    dev = torch.device(device)
    tensors = [means, sh0, shN, scaling, rotation, opacity]
    params = {k: torch.from_numpy(np.ascontiguousarray(t)).to(dev).requires_grad_(True)
              for k, t in zip(PARAM_GROUPS, tensors)}
    sh_degree = int(math.sqrt(shN.shape[1] + 1)) - 1
    return params, 0.5, sh_degree
