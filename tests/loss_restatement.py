"""Float64 restatement of the reference's photometric loss (src/training/trainer.cpp:103-126 with
fused_ssim(..., "valid") of include/kernels/fused_ssim.cuh:27-117), the yardstick of csrc/gsb_loss.cu:

  x     = clamp(render, 0, 1) (rasterizer.cpp:401), or the render as it is for the loss of a bilateral-grid output
  L1    = mean |x - target| over all 3 H W values
  SSIM  = mean of the 11x11, sigma = 1.5 Gaussian-window SSIM map with zero padding, C1 = 0.01^2, C2 = 0.03^2, the map
          cropped by 5 pixels per side only when H > 10 and W > 10 ("valid")
  loss  = (1 - lambda) L1 + lambda (1 - SSIM)

Plain torch autograd in float64 gives dLoss/d(render): the clamp passes the gradient where 0 <= render <= 1 (torch's
inclusive mask, zero at NaN), and |.| has subgradient 0 where render == target.  When a side is 10 or less the
reference's fused_ssim backward hands its kernel an all-zero map gradient (fused_ssim.cuh:87-95 fills the zero map
only when it cropped); this restatement, like csrc/gsb_loss.cu, differentiates the uncropped mean it computes.

Renders are [1,H,W,3] (the blend's output) or [3,H,W] (the fastgs path's planes); the target is [3,H,W], [1,3,H,W] or
[1,H,W,3], the layouts csrc/gsb_loss.cu accepts."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

WINDOW, PAD, SIGMA = 11, 5, 1.5
C1, C2 = 0.01 ** 2, 0.03 ** 2


def window_1d() -> list[float]:
    g = [math.exp(-((j - PAD) ** 2) / (2.0 * SIGMA * SIGMA)) for j in range(WINDOW)]
    s = math.fsum(g)
    return [v / s for v in g]


def renders_chw(renders: torch.Tensor) -> torch.Tensor:
    """[3,H,W] view of renders given as [1,H,W,3] or [3,H,W]."""
    if renders.dim() == 4 and renders.shape[0] == 1 and renders.shape[3] == 3:
        return renders[0].permute(2, 0, 1)
    assert renders.dim() == 3 and renders.shape[0] == 3, tuple(renders.shape)
    return renders


def target_chw(target: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """[3,H,W] view of a target given as [3,H,W], [1,3,H,W] or [1,H,W,3] ([1,H,W,3] wins when both fit, as in the
    kernel's shim)."""
    if tuple(target.shape) == (1, H, W, 3):
        return target[0].permute(2, 0, 1)
    if tuple(target.shape) == (1, 3, H, W):
        return target[0]
    assert tuple(target.shape) == (3, H, W), (tuple(target.shape), H, W)
    return target


def _filter(t: torch.Tensor) -> torch.Tensor:
    """Separable 11x11 window over each [H,W] plane of t [3,H,W], zero padding: the map has t's size."""
    w = window_1d()
    H, W = t.shape[-2:]
    p = F.pad(t, (PAD, PAD, PAD, PAD))
    rows = sum(w[j] * p[:, :, j:j + W] for j in range(WINDOW))
    return sum(w[j] * rows[:, j:j + H, :] for j in range(WINDOW))


def ssim_map(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """The uncropped SSIM map of [3,H,W] planes."""
    mu1, mu2 = _filter(x), _filter(y)
    s1 = _filter(x * x) - mu1 * mu1
    s2 = _filter(y * y) - mu2 * mu2
    s12 = _filter(x * y) - mu1 * mu2
    return ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))


def valid_crop(m: torch.Tensor) -> torch.Tensor:
    H, W = m.shape[-2:]
    return m[..., PAD:H - PAD, PAD:W - PAD] if H > 10 and W > 10 else m


def loss_terms(renders: torch.Tensor, target: torch.Tensor, lambda_dssim: float = 0.2, clamp: bool = True):
    """(loss, L1, SSIM) as float64 scalars, differentiable with respect to renders."""
    r = renders_chw(renders).double()
    x = torch.clamp(r, 0.0, 1.0) if clamp else r
    y = target_chw(target, r.shape[1], r.shape[2]).double()
    l1 = (x - y).abs().mean()
    ssim = valid_crop(ssim_map(x, y)).mean()
    return (1.0 - lambda_dssim) * l1 + lambda_dssim * (1.0 - ssim), l1, ssim


def photometric_loss_f64(renders: torch.Tensor, target: torch.Tensor, lambda_dssim: float = 0.2, clamp: bool = True):
    """(loss, L1, SSIM, dLoss/d(renders)): float64 values, the gradient laid out like renders, on renders' device."""
    r = renders.detach().double().requires_grad_(True)
    loss, l1, ssim = loss_terms(r, target.detach(), lambda_dssim, clamp)
    (grad,) = torch.autograd.grad(loss, r)
    return float(loss.detach()), float(l1.detach()), float(ssim.detach()), grad
