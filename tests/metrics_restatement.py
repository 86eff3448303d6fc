"""Restatements of the reference's evaluation metrics (src/training/metrics/metrics.cpp:17-116), the yardsticks of
csrc/gsb_metrics.cu:

  window_1d      gaussian(11, 1.5) in float32, quirk included: inv_denom = 1.0f / 2.0f * sigma * sigma = 1.125, so the
                 taps are exp(-d^2 * 1.125) normalised (an effective sigma of ~0.67, not 1.5)
  metrics_f64    float64 NumPy: PSNR::compute and SSIM::compute of clamp(image, 0, 1) against the target, the 2-D window
                 the outer product of the float32 taps, "same" zero padding, the mean over the whole map
  metrics_torch  the reference's formula transcribed to float32 torch ops (five grouped conv2d and the maps, with the
                 .item() reads), on whatever device its inputs are

Images are [3,H,W]; the rendered image is clamped, the target is used as given."""
from __future__ import annotations

import numpy as np

WINDOW, PAD = 11, 5
C1, C2 = np.float32(0.01) * np.float32(0.01), np.float32(0.03) * np.float32(0.03)  # metrics.hpp:50-51, float


def window_1d() -> np.ndarray:
    """metrics.cpp:17-31 for (11, 1.5): float32 taps, summed in index order and divided."""
    sigma = np.float32(1.5)
    inv_denom = np.float32(1.0) / np.float32(2.0) * sigma * sigma  # C++ precedence: (1 / 2) * sigma * sigma
    g = np.empty(WINDOW, np.float32)
    for x in range(WINDOW):
        d = x - WINDOW // 2
        g[x] = np.exp(-np.float32(d * d) * inv_denom)
    s = np.float32(0.0)
    for v in g:
        s = np.float32(s + v)
    return (g / s).astype(np.float32)


def _filter_same(a: np.ndarray, w: np.ndarray) -> np.ndarray:
    """Separable 'same' correlation of each [H,W] plane of `a` with w x w, zero padding PAD."""
    C, H, W = a.shape
    p = np.zeros((C, H + 2 * PAD, W + 2 * PAD), np.float64)
    p[:, PAD:PAD + H, PAD:PAD + W] = a
    rows = sum(w[j] * p[:, :, j:j + W] for j in range(WINDOW))
    return sum(w[j] * rows[:, j:j + H, :] for j in range(WINDOW))


def ssim_map_f64(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    w = window_1d().astype(np.float64)
    f = lambda t: _filter_same(t, w)
    mu1, mu2 = f(x), f(y)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = f(x * x) - mu1_sq, f(y * y) - mu2_sq, f(x * y) - mu1_mu2
    c1, c2 = float(C1), float(C2)
    return ((2 * mu1_mu2 + c1) * (2 * s12 + c2)) / ((mu1_sq + mu2_sq + c1) * (s1 + s2 + c2))


def psnr_f64(x: np.ndarray, y: np.ndarray) -> float:
    mse = max(float(np.mean((x - y) ** 2)), 1e-10)
    return 20.0 * np.log10(1.0 / np.sqrt(mse))


def metrics_f64(image, target) -> tuple[float, float]:
    """(psnr, ssim) of clamp(image, 0, 1) against target, both [3,H,W], in float64."""
    x = np.clip(np.asarray(image, np.float64), 0.0, 1.0)
    y = np.asarray(target, np.float64)
    assert x.shape == y.shape and x.ndim == 3 and x.shape[0] == 3
    return psnr_f64(x, y), float(np.mean(ssim_map_f64(x, y)))


def metrics_torch(image, target) -> tuple[float, float]:
    """metrics.cpp:40-116 after the clamp at :441, op for op in float32 torch (inputs [3,H,W] torch tensors)."""
    import torch
    import torch.nn.functional as F

    pred = torch.clamp(image.float()[None], 0.0, 1.0)
    gt = target.float()[None]
    # PSNR::compute
    mse = (pred - gt).pow(2).reshape(pred.size(0), -1).mean(1, keepdim=True)
    mse = torch.clamp_min(mse, 1e-10)
    psnr = (20.0 * torch.log10(1.0 / mse.sqrt())).mean().item()
    # SSIM::compute with create_window(11, 3)
    g = torch.from_numpy(window_1d()).unsqueeze(1)
    win = g.mm(g.t()).unsqueeze(0).unsqueeze(0).expand(3, 1, WINDOW, WINDOW).contiguous().to(pred.device)
    conv = lambda t: F.conv2d(t, win, padding=PAD, groups=3)
    mu1, mu2 = conv(pred), conv(gt)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = conv(pred * pred) - mu1_sq
    sigma2_sq = conv(gt * gt) - mu2_sq
    sigma12 = conv(pred * gt) - mu1_mu2
    c1, c2 = float(C1), float(C2)
    ssim_map = ((2.0 * mu1_mu2 + c1) * (2.0 * sigma12 + c2)) / ((mu1_sq + mu2_sq + c1) * (sigma1_sq + sigma2_sq + c2))
    return psnr, ssim_map.mean().item()
