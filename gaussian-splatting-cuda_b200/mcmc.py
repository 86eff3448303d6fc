"""The MCMC densification strategy (SURVEY.md 8 f6): a mirror of the reference's src/training/strategies/mcmc.cpp on
this library's kernels (csrc/gsb_mcmc.cu).

  post_backward(iteration)   mcmc.cpp:369-393: SH-degree bump, then -- on a refine iteration -- relocate_gs and
                             add_new_gs, then inject_noise (before_adam) with lr(group 0) * 5e5 (the rate before this
                             iteration's scheduler step)
  regularize(params)         trainer.cpp:132-158: scale_reg * mean(exp(scaling_raw)) + opacity_reg *
                             mean(sigmoid(opacity_raw)), gradients added into the parameters' .grad

Storage is capacity-resident: the six parameters and their Adam moments live in buffers of max(max_cap, N) rows;
params[k] and the optimizer's moments are [:N] views of them.  A growth step writes only the new rows and the sampled
rows and re-creates the views -- params[k] become new leaves without .grad, so FusedAdam skips that iteration's step
and keeps its step counts, as the reference's does after torch::cat (fused_adam.cpp:46-49).  Nothing in a refine reads
a device value on the host: N is known on the host, the dead count and the samples stay on the device.

Reproduced quirks of the reference:
  * relocation zeroes the Adam moments of the SAMPLED rows only; the dead rows it overwrites keep their old moments
    (update_optimizer_for_relocate receives the dead indices and does not use them, mcmc.cpp:84-109);
  * growth leaves the sampled rows' moments alone and appends zero moments;
  * the growth target is (int)(1.05f * N), a float product."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _product_ns, load
from .strategy import PARAM_GROUPS, Strategy


@dataclass
class MCMCConfig:
    """parameter/mcmc_optimization_params.json (the fields the strategy reads)."""
    iterations: int = 30000
    sh_degree: int = 3
    sh_degree_interval: int = 1000
    min_opacity: float = 0.005
    refine_every: int = 100
    start_refine: int = 500
    stop_refine: int = 25000
    opacity_reg: float = 0.01
    scale_reg: float = 0.01
    max_cap: int = 1000000
    noise_lr: float = 5e5  # mcmc.hpp:79


def binomial_table(n_max: int = 51) -> torch.Tensor:
    """C(n, k) for n, k < n_max, computed in float as mcmc.cpp:458-472 does (row n, column k)."""
    b = np.zeros((n_max, n_max), np.float32)
    for n in range(n_max):
        for k in range(n + 1):
            v = np.float32(1.0)
            for i in range(k):
                v = np.float32(v * np.float32(np.float32(n - i) / np.float32(i + 1)))
            b[n, k] = v
    return torch.from_numpy(b)


def growth_count(n: int, max_cap: int) -> int:
    """n_new of add_new_gs (mcmc.cpp:199-201): max(0, min(max_cap, (int)(1.05f * n)) - n)."""
    target = min(max_cap, int(np.float32(np.float32(1.05) * np.float32(n))))
    return max(0, target - n)


class MCMC(Strategy):
    """The strategy over a parameter dict (PARAM_GROUPS -> leaf tensors) and its FusedAdam.  Mutates both in place:
    after a growth step params[k] and optimizer.exp_avg[k] / exp_avg_sq[k] are new [:N] views of the storage."""

    def __init__(self, params: dict, optimizer, cfg: MCMCConfig | None = None, sh_degree: int = 0):
        load()
        self.cfg = cfg or MCMCConfig()
        self.params, self.optimizer = params, optimizer
        self.sh_degree = int(sh_degree)  # the active degree (SplatData::_active_sh_degree)
        self.n = int(params["means"].shape[0])
        dev = params["means"].device
        self.capacity = max(self.cfg.max_cap, self.n)
        self.binoms = binomial_table().to(dev)
        with torch.no_grad():
            self.store = {k: self._resident(params[k]) for k in PARAM_GROUPS}
            self.store_m1 = {k: self._resident(optimizer.exp_avg[k]) for k in PARAM_GROUPS}
            self.store_m2 = {k: self._resident(optimizer.exp_avg_sq[k]) for k in PARAM_GROUPS}
        self._views()
        self.last_samples = None     # the last refine's draws (relocation: the first n_dead are valid)
        self.last_dead = None        # (dead indices, device dead count) of the last relocation
        self.last_grow_samples = None
        self.last_noise = None
        self.refines = 0

    def _resident(self, t: torch.Tensor) -> torch.Tensor:
        buf = torch.zeros((self.capacity,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        buf[:self.n].copy_(t.detach())
        return buf

    def _views(self):
        n = self.n
        for k in PARAM_GROUPS:
            self.params[k] = self.store[k][:n].detach().requires_grad_(True)
            self.optimizer.exp_avg[k] = self.store_m1[k][:n]
            self.optimizer.exp_avg_sq[k] = self.store_m2[k][:n]

    def _lists(self, rows: int | None = None):
        s = slice(0, rows) if rows is not None else slice(None)
        return ([self.store[k][s] for k in PARAM_GROUPS], [self.store_m1[k][s] for k in PARAM_GROUPS],
                [self.store_m2[k][s] for k in PARAM_GROUPS])

    def is_refining(self, iteration: int) -> bool:
        c = self.cfg
        return c.start_refine < iteration < c.stop_refine and iteration % c.refine_every == 0

    def relocate(self) -> None:
        """relocate_gs (mcmc.cpp:112-190): dead rows take relocated copies of opacity-weighted draws from the alive."""
        ns, c, n = _product_ns(), self.cfg, self.n
        p, m1, m2 = self._lists(n)
        dead, n_dead, weights = ns.mcmc_dead(p[5].reshape(-1), p[4], c.min_opacity)
        samples = ns.mcmc_sample(weights, n, n_dead, None, False)
        ns.mcmc_relocate(p, m1, m2, samples, dead, n_dead, self.binoms, c.min_opacity)
        self.last_samples, self.last_dead = samples, (dead, n_dead)

    def grow(self) -> int:
        """add_new_gs (mcmc.cpp:192-347) into the resident storage; returns the number of rows added."""
        ns, c, n = _product_ns(), self.cfg, self.n
        n_new = growth_count(n, self.capacity)
        if n_new == 0:
            return 0
        p, m1, m2 = self._lists()
        samples = ns.mcmc_sample(p[5][:n].reshape(-1), n_new, None, None, True)
        ns.mcmc_grow(p, m1, m2, n, samples, self.binoms, c.min_opacity)
        self.last_grow_samples = samples
        self.n = n + n_new
        self._views()
        return n_new

    def remove_lowest_opacity(self, n_prune: int) -> None:
        """remove_gaussians (mcmc.cpp:404-440) of the n_prune lowest-opacity rows: the kept rows are compacted into
        fresh rows (the compaction must not read and write the same rows), written back to the front of the storage,
        and the views re-created.  Step counts are kept."""
        from .adc import lowest_opacity_removed
        p, m1, m2 = self._lists(self.n)
        out_p, out_m1, out_m2, _ = lowest_opacity_removed(p, m1, m2, n_prune)
        kept = self.n - n_prune
        with torch.no_grad():
            for k, a, b, c in zip(PARAM_GROUPS, out_p, out_m1, out_m2):
                self.store[k][:kept].copy_(a)
                self.store_m1[k][:kept].copy_(b)
                self.store_m2[k][:kept].copy_(c)
        self.n = kept
        self._views()

    def inject_noise(self, lr: float | torch.Tensor) -> None:
        """inject_noise (mcmc.cpp:349-367): lr is group 0's learning rate, a float or a device scalar."""
        P = self.params
        with torch.no_grad():
            noise = torch.randn_like(P["means"])
            args = (P["opacity_raw"].detach().reshape(-1), P["scaling_raw"].detach(), P["rotation_raw"].detach(),
                    noise, P["means"].detach())
            if isinstance(lr, torch.Tensor):
                _product_ns().mcmc_add_noise(*args, lr, self.cfg.noise_lr)
            else:  # (float)lr * _noise_lr, a float product
                _product_ns().add_noise(*args, float(np.float32(lr) * np.float32(self.cfg.noise_lr)))
        self.last_noise = noise

    def regularize(self, params: dict | None = None) -> torch.Tensor:
        """Adds the regularisers' gradients into the parameters' .grad; returns (scale loss, opacity loss) on the
        device.  A group without a gradient is left as it is."""
        P, c = params or self.params, self.cfg
        gs, go = P["scaling_raw"].grad, P["opacity_raw"].grad
        return _product_ns().mcmc_regularize(P["scaling_raw"].detach(), P["opacity_raw"].detach(), c.scale_reg,
                                             c.opacity_reg, gs if c.scale_reg > 0 else None,
                                             go if c.opacity_reg > 0 else None)

    def before_adam(self, lr: float | torch.Tensor) -> None:
        self.inject_noise(lr)

    def refine(self, iteration: int) -> tuple:
        """The SH bump and, on a refine iteration, relocation then growth.  A growth replaces the tensors, so Adam
        skips every group (nothing to step, as after the reference's torch::cat); relocation works in place."""
        if iteration % self.cfg.sh_degree_interval == 0 and self.sh_degree < self.cfg.sh_degree:
            self.sh_degree += 1
        self.replaced = False
        if not self.is_refining(iteration):
            return ()
        self.refines += 1
        self.relocate()
        self.replaced = self.grow() > 0
        return PARAM_GROUPS if self.replaced else ()
