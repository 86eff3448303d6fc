"""Float64 restatement of the bilateral grid (src/training/components/bilateral_grid.cpp:94-127 and
src/training/kernels/bilateral_grid_{forward,backward,tv}.cu), the yardstick of tests/test_bilagrid*.py.

Cell indices, fractions and the luminance mask come from float32 coordinates computed with the reference's operations
(forward.cu:34-50; the luminance as the multiply and two fused multiply-adds nvcc makes of it, each FMA here an exact
float64 product-sum rounded to float32); everything after that is float64."""
from __future__ import annotations

import numpy as np
import torch

LUM = (0.299, 0.587, 0.114)


def identity_grids(n, X=16, Y=16, L=8, dtype=torch.float64):
    eye = torch.eye(4, dtype=dtype)[:3]
    g = eye.repeat(L * Y * X, 1).reshape(1, L, Y, X, 12).permute(0, 4, 1, 2, 3)
    return g.repeat(n, 1, 1, 1, 1).contiguous()


def coords(x_hwc, L, H, W):
    """x_hwc: clamped image [h, w, 3] (any float dtype).  Returns int corners, float64 fractions and the z mask."""
    h, w = x_hwc.shape[0], x_hwc.shape[1]
    xf = np.asarray(x_hwc.detach().cpu().numpy(), dtype=np.float32)
    j = np.arange(w, dtype=np.float32)
    i = np.arange(h, dtype=np.float32)
    gx = (j / np.float32(w - 1)).astype(np.float32) * np.float32(W - 1)
    gy = (i / np.float32(h - 1)).astype(np.float32) * np.float32(H - 1)
    k = [np.float64(np.float32(v)) for v in LUM]
    t = (np.float32(LUM[0]) * xf[..., 0]).astype(np.float32)
    u = (k[1] * xf[..., 1].astype(np.float64) + t.astype(np.float64)).astype(np.float32)
    lum = (k[2] * xf[..., 2].astype(np.float64) + u.astype(np.float64)).astype(np.float32)
    gz = (lum * np.float32(L - 1)).astype(np.float32)
    x0 = np.floor(gx).astype(np.int64)
    y0 = np.floor(gy).astype(np.int64)
    zf = np.floor(gz).astype(np.int64)
    x1 = np.minimum(x0 + 1, W - 1)
    y1 = np.minimum(y0 + 1, H - 1)
    z1 = np.minimum(np.maximum(zf + 1, 0), L - 1)
    z0 = np.maximum(zf, 0)
    fx = (gx - x0.astype(np.float32)).astype(np.float64)
    fy = (gy - y0.astype(np.float32)).astype(np.float64)
    fz = (gz - z0.astype(np.float32)).astype(np.float64)
    zpass = (z0.astype(np.float32) != gz) & (z1.astype(np.float32) != gz)
    X0, X1 = np.broadcast_to(x0[None, :], (h, w)), np.broadcast_to(x1[None, :], (h, w))
    Y0, Y1 = np.broadcast_to(y0[:, None], (h, w)), np.broadcast_to(y1[:, None], (h, w))
    FX, FY = np.broadcast_to(fx[None, :], (h, w)), np.broadcast_to(fy[:, None], (h, w))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    return dict(x0=t(X0), x1=t(X1), y0=t(Y0), y1=t(Y1), z0=t(z0), z1=t(z1), fx=t(FX), fy=t(FY), fz=t(fz),
                zpass=t(zpass))


def _corners(c):
    """(weight, z, y, x) of the 8 corners, weights [h, w]."""
    out = []
    for zz, wz in ((c["z0"], 1 - c["fz"]), (c["z1"], c["fz"])):
        for yy, wy in ((c["y0"], 1 - c["fy"]), (c["y1"], c["fy"])):
            for xx, wx in ((c["x0"], 1 - c["fx"]), (c["x1"], c["fx"])):
                out.append((wx * wy * wz, zz, yy, xx))
    return out


def slice_fwd(grid, img_hwc):
    """grid [12, L, H, W], img_hwc [h, w, 3] (unclamped) -> [h, w, 3], float64."""
    grid = grid.double()
    x = img_hwc.double().clamp(0, 1)
    L, H, W = grid.shape[1:]
    c = coords(x, L, H, W)
    A = torch.zeros(x.shape[0], x.shape[1], 12, dtype=torch.float64)
    for wgt, zz, yy, xx in _corners(c):
        A += wgt[..., None] * grid[:, zz, yy, xx].permute(1, 2, 0)
    xs = torch.cat([x, torch.ones_like(x[..., :1])], -1)
    return torch.stack([(A[..., 4 * d:4 * d + 4] * xs).sum(-1) for d in range(3)], -1)


def slice_bwd(grid, img_hwc, v_out):
    """(v_grid [12, L, H, W], v_img [h, w, 3] with respect to the UNCLAMPED image), float64."""
    grid = grid.double()
    raw = img_hwc.double()
    x = raw.clamp(0, 1)
    g = v_out.double()
    L, H, W = grid.shape[1:]
    c = coords(x, L, H, W)
    xs = torch.cat([x, torch.ones_like(x[..., :1])], -1)
    outer = torch.stack([xs[..., s] * g[..., d] for d in range(3) for s in range(4)], -1)  # [h, w, 12], c = 4d+s
    v_grid = torch.zeros(12, L * H * W, dtype=torch.float64)
    A = torch.zeros(x.shape[0], x.shape[1], 12, dtype=torch.float64)
    dA = torch.zeros_like(A)
    for wgt, zz, yy, xx in _corners(c):
        flat = ((zz * H + yy) * W + xx).reshape(-1)
        v_grid.index_add_(1, flat, (wgt[..., None] * outer).reshape(-1, 12).T)
        A += wgt[..., None] * grid[:, zz, yy, xx].permute(1, 2, 0)
    # d A / d z: bilinear planes at z1 minus z0
    for zz, sign in ((c["z0"], -1.0), (c["z1"], 1.0)):
        for yy, wy in ((c["y0"], 1 - c["fy"]), (c["y1"], c["fy"])):
            for xx, wx in ((c["x0"], 1 - c["fx"]), (c["x1"], c["fx"])):
                dA += sign * (wx * wy)[..., None] * grid[:, zz, yy, xx].permute(1, 2, 0)
    v_x = torch.stack([sum(g[..., d] * A[..., 4 * d + s] for d in range(3)) for s in range(3)], -1)
    gz = (dA * outer).sum(-1) * (L - 1) * c["zpass"].double()
    v_x = v_x + gz[..., None] * torch.tensor(LUM, dtype=torch.float64)
    inside = (raw >= 0) & (raw <= 1)
    return v_grid.reshape(12, L, H, W), torch.where(inside, v_x, torch.zeros_like(v_x))


def tv_loss(grids):
    """(1 / (12 N)) * sum over (n, c) of the three means of squared neighbour differences, float64, differentiable."""
    g = grids.double()
    N = g.shape[0]
    total = torch.zeros((), dtype=torch.float64)
    for dim in (4, 3, 2):  # x, y, z
        if g.shape[dim] > 1:
            d = torch.diff(g, dim=dim)
            total = total + (d * d).mean(dim=(2, 3, 4)).sum()
    return total / (12 * N)


def tv_grad(grids):
    g = grids.double().detach().requires_grad_(True)
    tv_loss(g).backward()
    return g.grad


def rel_l2(a, b):
    a = torch.as_tensor(a).double().flatten()
    b = torch.as_tensor(b).double().flatten()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))
