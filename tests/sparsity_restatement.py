"""A torch restatement of the reference's ADMM sparsifier (src/training/components/sparsity_optimizer.cpp and
sparsity_optimizer.hpp) and of the trainer's phase logic around it (trainer.cpp:173-247, 331-361, 707-784), line by
line, on any device.  The tests hold the library's kernels and training steps against it."""
from __future__ import annotations

import numpy as np
import torch

GROUPS = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")


def prune_index(prune_ratio: float, n: int) -> int:
    """static_cast<int>(config_.prune_ratio * z.size(0)): float * int64 is a float32 product."""
    return int(np.float32(np.float32(prune_ratio) * np.float32(n)))


# ---- sparsity_optimizer.hpp: the schedule --------------------------------------------------------------------------
def should_update(it: int, start: int, steps: int, every: int) -> bool:
    r = it - start
    return it >= start and r > 0 and r < steps and r % every == 0


def should_apply_loss(it: int, start: int, steps: int) -> bool:
    return it >= start and it < start + steps


def should_prune(it: int, start: int, steps: int) -> bool:
    return it == start + steps


def post_backward_due(it: int, base: int) -> bool:
    """trainer.cpp:745-754"""
    return it <= base


# ---- sparsity_optimizer.cpp ----------------------------------------------------------------------------------------
def prune_z(z: torch.Tensor, prune_ratio: float) -> torch.Tensor:
    if z.numel() == 0:
        return torch.zeros_like(z)
    index = prune_index(prune_ratio, z.shape[0])
    if index == 0:
        return torch.zeros_like(z)
    z_sorted, _ = torch.sort(z.flatten(), 0)
    z_threshold = z_sorted[index - 1]
    return (z > z_threshold) * z


def initialize(opacities: torch.Tensor, prune_ratio: float):
    """(z, u)"""
    with torch.no_grad():
        opa = torch.sigmoid(opacities).detach().contiguous()
        u = torch.zeros_like(opa)
        z = prune_z(opa + u, prune_ratio)
    return z, u


def update_state(opacities: torch.Tensor, z: torch.Tensor, u: torch.Tensor, prune_ratio: float):
    """(z, u) after update_state; u is updated in place as the reference does."""
    with torch.no_grad():
        opa = torch.sigmoid(opacities).detach().contiguous()
        z_temp = opa + u
        z = prune_z(z_temp, prune_ratio)
        u += opa - z
    return z, u


def loss(opacities: torch.Tensor, z: torch.Tensor, u: torch.Tensor, init_rho: float) -> torch.Tensor:
    """0.5f * init_rho * pow(norm(diff, 2), 2) with diff = sigmoid(o) - z + u; differentiable in opacities."""
    opa = torch.sigmoid(opacities)
    diff = opa - z.detach() + u.detach()
    return float(np.float32(0.5) * np.float32(init_rho)) * torch.pow(torch.norm(diff, 2), 2)


def prune_mask(opacities: torch.Tensor, prune_ratio: float) -> torch.Tensor:
    """get_prune_mask: the n_prune smallest sigmoid(o) (topk, largest=False)."""
    opa = torch.sigmoid(opacities.flatten())
    n_prune = prune_index(prune_ratio, opa.shape[0])
    mask = torch.zeros(opa.shape[0], dtype=torch.bool, device=opa.device)
    if n_prune == 0:
        return mask
    _, idx = torch.topk(opa, n_prune, -1, largest=False)
    mask[idx] = True
    return mask


def remove_gaussians(P: dict, M1: dict, M2: dict, mask: torch.Tensor):
    """default_strategy.cpp:194-227 / mcmc.cpp:404-440: index_select of the six parameters and both moments."""
    keep = (~mask).nonzero().squeeze(-1)
    return ({k: P[k].index_select(0, keep) for k in GROUPS}, {k: M1[k].index_select(0, keep) for k in GROUPS},
            {k: M2[k].index_select(0, keep) for k in GROUPS})


class Sparsifier:
    """ADMMSparsityOptimizer with the trainer's calls: loss_step after the regularisers, after_step after Adam."""

    def __init__(self, start: int, steps: int, init_rho: float = 5e-4, prune_ratio: float = 0.6, every: int = 50):
        self.start, self.steps, self.rho, self.ratio, self.every = start, steps, init_rho, prune_ratio, every
        self.z = self.u = None
        self.done = False

    def loss_step(self, opacity_raw: torch.Tensor, it: int):
        """compute_sparsity_loss (trainer.cpp:173-197): the loss's gradient added into opacity_raw.grad."""
        if self.done or not should_apply_loss(it, self.start, self.steps):
            return None
        if self.z is None:
            self.z, self.u = initialize(opacity_raw.detach(), self.ratio)
        o = opacity_raw.detach().clone().requires_grad_(True)
        value = loss(o, self.z, self.u, self.rho)
        value.backward()
        with torch.no_grad():
            opacity_raw.grad += o.grad
        return value.detach()

    def after_step(self, P: dict, M1: dict, M2: dict, it: int):
        """handle_sparsity_update then apply_sparsity_pruning (trainer.cpp:199-247): the new (P, M1, M2) or None."""
        if self.done:
            return None
        if should_update(it, self.start, self.steps, self.every):
            self.z, self.u = update_state(P["opacity_raw"].detach(), self.z, self.u, self.ratio)
        if should_prune(it, self.start, self.steps):
            self.done = True
            mask = prune_mask(P["opacity_raw"].detach(), self.ratio)
            return remove_gaussians(P, M1, M2, mask)
        return None
