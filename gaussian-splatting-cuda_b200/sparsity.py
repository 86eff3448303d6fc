"""ADMM opacity sparsification, the reference's --enable-sparsity: a mirror of
src/training/components/sparsity_optimizer.cpp on this library's kernels (csrc/gsb_sparsity.cu, gsb_adc.cu).

After `start_iteration` base iterations the trainer runs `sparsify_steps` more.  In that phase every iteration adds
0.5 rho ||sigmoid(o) - z + u||^2 to the loss (its gradient into opacity_raw.grad), every `update_every` iterations the
state is updated (z = prune_z(sigmoid(o) + u), u += sigmoid(o) - z), and the last iteration removes the
(int)(prune_ratio * N) Gaussians of lowest opacity.  The strategy's post_backward runs only up to the base iteration
count.  z and u stay on the device, the prune_z threshold is selected on the device, and the prune compacts into
exact-size rows with N and n_prune known on the host: no iteration of the phase synchronises with the host."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _product_ns, load


@dataclass
class SparsityConfig:
    """ADMMSparsityOptimizer::Config (sparsity_optimizer.hpp); start_iteration is the base iteration count."""
    sparsify_steps: int = 15000
    init_rho: float = 5e-4
    prune_ratio: float = 0.6
    update_every: int = 50
    start_iteration: int = 30000


def prune_count(prune_ratio: float, n: int) -> int:
    """static_cast<int>(prune_ratio * N) with a float ratio and an int64 N: the product is a float32 one."""
    return int(np.float32(np.float32(prune_ratio) * np.float32(n)))


class ADMMSparsity:
    """The sparsifier of one training run.  `done` after the prune (the reference drops it then)."""

    def __init__(self, cfg: SparsityConfig | None = None):
        load()
        self.cfg = cfg or SparsityConfig()
        self.z = self.u = None
        self.rho = None  # [1] device tensor, read by the loss kernel
        self.done = False
        self.last_loss = None
        self.n_pruned = 0

    @property
    def initialized(self) -> bool:
        return self.z is not None

    @property
    def base(self) -> int:
        return self.cfg.start_iteration

    # ---- schedule (sparsity_optimizer.hpp) ------------------------------------------------------------------------
    def should_apply_loss(self, it: int) -> bool:
        c = self.cfg
        return not self.done and c.start_iteration <= it < c.start_iteration + c.sparsify_steps

    def should_update(self, it: int) -> bool:
        c = self.cfg
        r = it - c.start_iteration
        return not self.done and it >= c.start_iteration and 0 < r < c.sparsify_steps and r % c.update_every == 0

    def should_prune(self, it: int) -> bool:
        return not self.done and it == self.cfg.start_iteration + self.cfg.sparsify_steps

    def post_backward_due(self, it: int) -> bool:
        """trainer.cpp:745-754: the strategy's post_backward runs up to the base iteration count, inclusive."""
        return it <= self.cfg.start_iteration

    # ---- state -----------------------------------------------------------------------------------------------------
    def initialize(self, opacity_raw: torch.Tensor) -> None:
        """u = 0, z = prune_z(sigmoid(o) + u) (sparsity_optimizer.cpp:18-43)."""
        o = opacity_raw.detach()
        self.z = torch.empty(o.numel(), dtype=torch.float32, device=o.device)
        self.u = torch.empty_like(self.z)
        self.rho = torch.full((1,), float(self.cfg.init_rho), dtype=torch.float32, device=o.device)
        _product_ns().sparsity_update(o.reshape(-1), self.z, self.u, prune_count(self.cfg.prune_ratio, o.numel()), True)

    def check_rows(self, n: int) -> None:
        if self.initialized and self.z.numel() != n:
            raise ValueError(f"the number of Gaussians changed from {self.z.numel()} to {n} after the sparsity state was "
                             f"initialised: the strategy must not refine at the base iteration {self.base} (the "
                             f"reference fails there with a shape mismatch)")

    def add_loss_gradient(self, opacity_raw: torch.Tensor) -> torch.Tensor:
        """0.5 rho ||sigmoid(o) - z + u||^2 as a [1] device tensor, its gradient added into opacity_raw.grad."""
        self.check_rows(opacity_raw.numel())
        g = opacity_raw.grad
        if g is None:
            g = opacity_raw.grad = torch.zeros_like(opacity_raw)
        o = opacity_raw.detach()
        self.last_loss = _product_ns().sparsity_loss(o.reshape(-1), self.z, self.u, self.rho, g.view(-1))
        return self.last_loss

    def update_state(self, opacity_raw: torch.Tensor) -> None:
        """zt = sigmoid(o) + u; z = prune_z(zt); u += sigmoid(o) - z (sparsity_optimizer.cpp:69-102)."""
        o = opacity_raw.detach()
        self.check_rows(o.numel())
        _product_ns().sparsity_update(o.reshape(-1), self.z, self.u, prune_count(self.cfg.prune_ratio, o.numel()),
                                      False)

    def prune(self, strategy) -> int:
        """get_prune_mask + remove_gaussians (trainer.cpp:216-247): the strategy drops the n_prune rows of lowest
        opacity.  Returns n_prune; the sparsifier is done afterwards."""
        n = strategy.n
        n_prune = prune_count(self.cfg.prune_ratio, n)
        if n_prune > 0:
            strategy.remove_lowest_opacity(n_prune)
        self.n_pruned = n_prune
        self.done = True
        self.z = self.u = None
        return n_prune

    # ---- one iteration's parts, in the trainer's order -------------------------------------------------------------
    def loss_step(self, opacity_raw: torch.Tensor, it: int) -> torch.Tensor | None:
        """After the photometric loss and the regularisers: the lazy initialisation at the first loss iteration, then
        the loss and its gradient.  None when no loss applies."""
        if not self.should_apply_loss(it):
            return None
        if not self.initialized:
            self.initialize(opacity_raw)
        return self.add_loss_gradient(opacity_raw)

    def after_step(self, strategy, it: int) -> bool:
        """After Adam: update_state when due, then the prune when due.  True when the prune replaced the tensors."""
        if self.should_update(it):
            self.update_state(strategy.params["opacity_raw"])
        if self.should_prune(it):
            return self.prune(strategy) > 0
        return False
