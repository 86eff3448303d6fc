"""Adaptive density control, the reference's default densification strategy: a mirror of
src/training/strategies/default_strategy.cpp on this library's kernels (csrc/gsb_adc.cu).

  post_backward(iteration)   default_strategy.cpp:292-326: SH-degree bump; at stop_refine the statistics become empty
                             (the fastgs backward then stops writing them); before it, on a refine iteration grow_gs
                             (duplicate, split) and prune_gs as ONE compaction into exact-size tensors, then zeroed
                             statistics [2, N]; every reset_every iterations reset_opacity, in place
  regularize(params)         trainer.cpp:132-158, the scale and opacity regularisers (0 by default for this strategy)

A refine reads one small array of device counts back -- the output size and the shape of torch.randn({2, n_split, 3})
depend on it -- and nothing else in an iteration synchronises.  A refine that changed anything replaces all six
tensors and their moments: the new leaves have no .grad, so FusedAdam skips every group that iteration and keeps its
step counts, as the reference's does (fused_adam.cpp:46-66).  A refine that changed nothing keeps the tensors and only
zeroes the statistics.  A reset skips the opacity group only.

On the 3DGUT path the backward writes no statistics: nothing grows, rows are still pruned and opacities reset."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from . import _product_ns, load
from .strategy import PARAM_GROUPS, Strategy


def lowest_opacity_removed(params: list, exp_avg: list, exp_avg_sq: list, n_prune: int):
    """The rows of the six tensors and their moments (PARAM_GROUPS order) without the n_prune rows of lowest
    sigmoid(opacity_raw), in order, in freshly allocated tensors: (params, exp_avg, exp_avg_sq, zeroed statistics
    [2, n_kept]).  The sparsifier's final prune (sparsity_optimizer.cpp:104-143 + remove_gaussians); n_prune and the
    row count are known on the host, so nothing is read back."""
    ns = _product_ns()
    n = int(params[0].shape[0])
    with torch.no_grad():
        counts, ws = ns.sparsity_prune_classify(params[5].reshape(-1), n_prune)
        return ns.adc_apply(params, exp_avg, exp_avg_sq, ws, counts, 0, n - n_prune, None, False)


@dataclass
class DefaultConfig:
    """parameter/default_optimization_params.json (the fields the strategy is given; values already scaled by
    steps_scaler)."""
    iterations: int = 30000
    sh_degree: int = 3
    sh_degree_interval: int = 1000
    refine_every: int = 100
    start_refine: int = 500
    stop_refine: int = 15000
    reset_every: int = 3000
    pause_refine_after_reset: int = 0
    grad_threshold: float = 0.0002
    grow_scale3d: float = 0.01
    prune_opacity: float = 0.005
    prune_scale3d: float = 0.1
    revised_opacity: bool = False
    opacity_reg: float = 0.0
    scale_reg: float = 0.0
    # given to the strategy but not read by it (nor by the reference's): no 2D criteria and no cap on growth
    grow_scale2d: float = 0.05
    prune_scale2d: float = 0.15
    max_cap: int = 1000000


class DefaultStrategy(Strategy):
    """The strategy over a parameter dict (PARAM_GROUPS -> leaf tensors) and its FusedAdam.  Mutates both: after a
    refine that changed the set, params[k] and optimizer.exp_avg[k] / exp_avg_sq[k] are new tensors.  scene_scale is
    the optimizer's (one get_scene_scale() feeds both the means learning rate and the thresholds)."""

    def __init__(self, params: dict, optimizer, cfg: DefaultConfig | None = None, sh_degree: int = 0):
        load()
        self.cfg = cfg or DefaultConfig()
        self.params, self.optimizer = params, optimizer
        self.sh_degree = int(sh_degree)  # the active degree (SplatData::_active_sh_degree)
        self.scene_scale = float(optimizer.cfg.scene_scale)
        dev = params["means"].device
        # strategy_utils.cpp:17 (initialize_gaussians): [2, N] zeros; the fastgs backward accumulates into it
        self.densification_info = torch.zeros((2, self.n), dtype=torch.float32, device=dev)
        self.last_counts = None  # (duplicated, split, pruned, final rows) of the last refine
        self.last_z = None       # the last split's normals [2, n_split, 3]
        self.last_kept_split = 0
        self.refines = 0
        self.resets = 0

    @property
    def n(self) -> int:
        return int(self.params["means"].shape[0])

    def is_refining(self, iteration: int) -> bool:
        """default_strategy.cpp:31-35"""
        c = self.cfg
        return (iteration > c.start_refine and iteration % c.refine_every == 0
                and iteration % c.reset_every >= c.pause_refine_after_reset)

    def regularize(self, params: dict | None = None):
        """The trainer's regularisers added into the parameters' .grad when a weight is > 0; returns (scale loss,
        opacity loss) on the device, or None when both weights are 0."""
        P, c = params or self.params, self.cfg
        if not (c.scale_reg > 0 or c.opacity_reg > 0):
            return None
        gs, go = P["scaling_raw"].grad, P["opacity_raw"].grad
        return _product_ns().mcmc_regularize(P["scaling_raw"].detach(), P["opacity_raw"].detach(), c.scale_reg,
                                             c.opacity_reg, gs if c.scale_reg > 0 else None,
                                             go if c.opacity_reg > 0 else None)

    def grow_and_prune(self, iteration: int) -> bool:
        """grow_gs then prune_gs (default_strategy.cpp:164-249).  True when the set changed (the tensors are new)."""
        ns, c, P = _product_ns(), self.cfg, self.params
        info = self.densification_info
        with torch.no_grad():
            counts, ws = ns.adc_classify(info if info.numel() else None, P["scaling_raw"].detach(),
                                         P["rotation_raw"].detach(), P["opacity_raw"].detach(), c.grad_threshold,
                                         c.grow_scale3d, c.prune_scale3d, self.scene_scale, c.prune_opacity,
                                         iteration > c.reset_every, bool(c.revised_opacity))
            h = counts.tolist()  # the refine's one read-back
            n_dup, n_split, n_prune, n_final = h[:4]
            self.last_counts = (n_dup, n_split, n_prune, n_final)
            self.last_kept_split = h[6]  # the last 2 * last_kept_split rows are split copies
            self.last_z = None
            if n_dup == 0 and n_split == 0 and n_prune == 0:
                if info.numel():
                    info.zero_()
                return False
            z = None
            if n_split > 0:  # default_strategy.cpp:100-104: the same call and shape, drawn only when rows split
                z = torch.randn((2, n_split, 3), device=P["means"].device)
            self.last_z = z
            out_p, out_m1, out_m2, new_info = ns.adc_apply(*self._state(), ws, counts, n_split, n_final, z,
                                                           bool(c.revised_opacity))
        self._install(out_p, out_m1, out_m2)
        self.densification_info = new_info
        return True

    def _state(self):
        """(params, exp_avg, exp_avg_sq) as lists in PARAM_GROUPS order."""
        P, opt = self.params, self.optimizer
        return ([P[k].detach() for k in PARAM_GROUPS], [opt.exp_avg[k] for k in PARAM_GROUPS],
                [opt.exp_avg_sq[k] for k in PARAM_GROUPS])

    def _install(self, params: list, exp_avg: list, exp_avg_sq: list) -> None:
        """New tensors become the leaves and their moments the optimizer's; step counts are kept."""
        for k, p, m1, m2 in zip(PARAM_GROUPS, params, exp_avg, exp_avg_sq):
            self.params[k] = p.requires_grad_(True)
            self.optimizer.exp_avg[k], self.optimizer.exp_avg_sq[k] = m1, m2

    def remove_lowest_opacity(self, n_prune: int) -> None:
        """remove_gaussians (default_strategy.cpp:194-227) of the n_prune lowest-opacity rows: new tensors and
        moments, step counts kept.  Non-empty statistics become zeros [2, n_kept]."""
        out_p, out_m1, out_m2, new_info = lowest_opacity_removed(*self._state(), n_prune)
        self._install(out_p, out_m1, out_m2)
        if self.densification_info.numel():
            self.densification_info = new_info

    def reset_opacity(self) -> None:
        """default_strategy.cpp:251-290 in place."""
        opt = self.optimizer
        with torch.no_grad():
            _product_ns().adc_reset_opacity(self.params["opacity_raw"].detach(), opt.exp_avg["opacity_raw"],
                                            opt.exp_avg_sq["opacity_raw"], self.cfg.prune_opacity)
        self.resets += 1

    def refine(self, iteration: int) -> tuple:
        """post_backward's work without touching gradients; returns the groups whose Adam step this iteration skips
        (all six after a refine that changed the set, the opacity group after a reset).  `replaced` tells whether the
        tensors are new."""
        c = self.cfg
        self.replaced = False
        if iteration % c.sh_degree_interval == 0 and self.sh_degree < c.sh_degree:
            self.sh_degree += 1
        if iteration == c.stop_refine:  # the backward stops accumulating statistics
            self.densification_info = torch.empty(0, dtype=torch.float32, device=self.params["means"].device)
        if iteration >= c.stop_refine:
            return ()
        skip = ()
        if self.is_refining(iteration):
            self.refines += 1
            if self.grow_and_prune(iteration):
                self.replaced = True
                skip = PARAM_GROUPS
        if iteration % c.reset_every == 0 and iteration > 0:
            self.reset_opacity()
            if not skip:
                skip = ("opacity_raw",)
        return skip
