"""The bilateral grid of the training iteration (SURVEY.md 8 f5): a per-image affine colour correction that the reference
trains next to the Gaussians when `--bilateral-grid` (use_bilateral_grid) is on.

  BilateralGrid        src/training/components/bilateral_grid.cpp: grids [N, 12, L, H, W] initialised to the identity
                       (:85-91), apply(image, image_idx) (:94-127) and tv_loss() (:131-133), as autograd functions over
                       this library's kernels (csrc/gsb_bilagrid.cu, torch.ops.gsplat_b200.bilagrid_*)
  WarmupExponentialLR  src/training/optimizers/scheduler.cpp:27-63 as the trainer configures it for the grids
                       (trainer.cpp:66-101): linear warm-up from 1 % over 1000 steps, then gamma = 0.01^(1/iterations)

Option naming follows the reference: bilateral_grid_X and _Y are the grid's width and height, bilateral_grid_W its
guidance depth L (BilateralGrid(num_images, grid_W = X, grid_H = Y, grid_L = W))."""
from __future__ import annotations

import torch

from . import _product_ns


def _index(image_idx, device) -> torch.Tensor:
    if isinstance(image_idx, torch.Tensor):
        return image_idx.to(device=device, dtype=torch.int32).reshape(1)
    return torch.tensor([int(image_idx)], dtype=torch.int32, device=device)


class _Slice(torch.autograd.Function):
    """image (unclamped) -> clamp -> slice through grids[image_idx]; gradients for the grids and the unclamped image."""

    @staticmethod
    def forward(ctx, grids, image, image_idx, chw):
        grids_c, image_c = grids.detach().contiguous(), image.detach().contiguous()
        ctx.save_for_backward(grids_c, image_c, image_idx)
        ctx.chw = chw
        return _product_ns().bilagrid_slice(grids_c, image_c, image_idx, chw)

    @staticmethod
    def backward(ctx, v_out):
        grids, image, image_idx = ctx.saved_tensors
        v_grids = torch.zeros_like(grids)
        v_image = _product_ns().bilagrid_slice_backward(grids, image, image_idx, v_out.contiguous(), v_grids, ctx.chw)
        return v_grids, v_image, None, None


class _TVLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids):
        g = grids.detach().contiguous()
        ctx.save_for_backward(g)
        return _product_ns().bilagrid_tv(g, None, False)[0]

    @staticmethod
    def backward(ctx, g_loss):
        (grids,) = ctx.saved_tensors
        w = g_loss.detach().to(torch.float32).reshape(1).contiguous()
        return _product_ns().bilagrid_tv(grids, w, True)[1]


def slice_image(grids, image, image_idx, chw: bool):
    """Differentiable slice of an image laid out [..., 3, H, W] (chw) or [..., H, W, 3] through grids[image_idx]
    (image_idx: int or a one-element device tensor).  The image is clamped to [0, 1] first, as apply() does."""
    return _Slice.apply(grids, image, _index(image_idx, image.device), chw)


def tv_loss(grids):
    """Total-variation loss of grids [N, 12, L, H, W] (a 0-dim tensor)."""
    return _TVLoss.apply(grids)


class BilateralGrid:
    def __init__(self, num_images: int, grid_X: int = 16, grid_Y: int = 16, grid_L: int = 8, device="cuda"):
        self.num_images, self.grid_width, self.grid_height, self.grid_guidance = int(num_images), grid_X, grid_Y, grid_L
        # identity: coefficient 4d+s of every cell is delta(d, s) (bilateral_grid.cpp:85-91)
        eye = torch.eye(4, dtype=torch.float32)[:3]
        grid = eye.repeat(grid_L * grid_Y * grid_X, 1).reshape(1, grid_L, grid_Y, grid_X, 12).permute(0, 4, 1, 2, 3)
        self.grids = grid.repeat(self.num_images, 1, 1, 1, 1).to(device).contiguous().requires_grad_(True)

    def parameters(self) -> torch.Tensor:
        return self.grids

    def apply(self, rgb: torch.Tensor, image_idx: int) -> torch.Tensor:
        """rgb [C,H,W] or [1,C,H,W] -> corrected image of the same shape (bilateral_grid.cpp:94-127)."""
        if not 0 <= int(image_idx) < self.num_images:
            raise ValueError(f"Invalid image index: {image_idx}")
        if rgb.dim() == 4 and rgb.shape[0] == 1:
            img = rgb.squeeze(0)
        elif rgb.dim() == 3:
            img = rgb
        else:
            raise ValueError(f"RGB must be [C, H, W] or [1, C, H, W], got {tuple(rgb.shape)}")
        out = slice_image(self.grids, img, image_idx, chw=True)
        return out.unsqueeze(0) if rgb.dim() == 4 else out

    def tv_loss(self) -> torch.Tensor:
        return tv_loss(self.grids)


class WarmupExponentialLR:
    """The learning rate of the grids' Adam.  As in the reference, step k (1-based) of the optimizer uses the rate set
    after k - 1 scheduler steps: the first step runs at the initial rate, then warm-up from start_factor."""

    def __init__(self, initial_lr: float, iterations: int = 30000, warmup_steps: int = 1000, start_factor: float = 0.01):
        self.initial_lr = float(initial_lr)
        self.gamma = 0.01 ** (1.0 / iterations)
        self.warmup_steps, self.start_factor = int(warmup_steps), float(start_factor)
        self.current_step = 0
        self.lr = self.initial_lr

    def step(self) -> float:
        self.current_step += 1
        if self.current_step <= self.warmup_steps:
            progress = self.current_step / self.warmup_steps
            self.lr = self.initial_lr * (self.start_factor + (1.0 - self.start_factor) * progress)
        else:
            self.lr = self.initial_lr * self.gamma ** (self.current_step - self.warmup_steps)
        return self.lr
