"""Torch restatement of the reference's MCMC strategy (src/training/strategies/mcmc.cpp) and of the trainer's ordering
around it (trainer.cpp:668-756), with the draws INJECTED: relocate_gs / add_new_gs take the sampled indices instead of
calling multinomial_sample, and inject_noise takes the noise.  `relocation(opacities, scales, ratios, binoms, n_max)`
is supplied by the caller (the CPU oracle's, this library's or the reference's kernel).  Works on CPU or CUDA tensors;
parameters and moments are dicts over GROUPS."""
from __future__ import annotations

import numpy as np
import torch

GROUPS = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")


def binoms_exact(n_max: int = 51) -> np.ndarray:
    from math import comb
    return np.array([[comb(n, k) if k <= n else 0 for k in range(n_max)] for n in range(n_max)], np.float64)


def dead_mask(P: dict, min_opacity: float) -> torch.Tensor:
    """mcmc.cpp:119-121"""
    op = torch.sigmoid(P["opacity_raw"].reshape(-1))
    rot = P["rotation_raw"]
    return (op <= min_opacity) | ((rot * rot).sum(-1) < 1e-8)


def _relocate_rows(P: dict, sampled: torch.Tensor, ratios: torch.Tensor, relocation, binoms, min_opacity: float):
    """The sampled rows' new logit opacity and log scale (mcmc.cpp:147-167 / 225-245); written into P."""
    n_max = binoms.shape[0]
    op = torch.sigmoid(P["opacity_raw"].reshape(-1))
    new_op, new_sc = relocation(op[sampled].contiguous(), torch.exp(P["scaling_raw"])[sampled].contiguous(),
                                ratios.to(torch.int32).contiguous(), binoms, n_max)
    new_op = torch.clamp(new_op, min_opacity, 1.0 - 1e-7)
    o = P["opacity_raw"]
    if o.dim() == 2:
        o[sampled] = torch.logit(new_op).unsqueeze(-1)
    else:
        o[sampled] = torch.logit(new_op)
    P["scaling_raw"][sampled] = torch.log(new_sc)


def relocate_gs(P: dict, M1: dict, M2: dict, sampled: torch.Tensor, relocation, binoms, min_opacity: float) -> int:
    """mcmc.cpp:112-190 in place; `sampled` are the n_dead global indices drawn from the alive Gaussians."""
    with torch.no_grad():
        dead = dead_mask(P, min_opacity)
        dead_idx = dead.nonzero().squeeze(-1)
        if dead_idx.numel() == 0 or (~dead).sum() == 0:
            return 0
        sampled = sampled.long()
        assert sampled.numel() == dead_idx.numel()
        n_max = binoms.shape[0]
        ratios = torch.ones_like(P["opacity_raw"].reshape(-1), dtype=torch.int32)
        ratios.index_add_(0, sampled, torch.ones_like(sampled, dtype=torch.int32))
        ratios = ratios[sampled].clamp_max(n_max)
        _relocate_rows(P, sampled, ratios, relocation, binoms, min_opacity)
        for k in GROUPS:
            P[k][dead_idx] = P[k][sampled]
        for k in GROUPS:  # update_optimizer_for_relocate: the SAMPLED rows only (the dead rows keep their moments)
            M1[k][sampled] = 0
            M2[k][sampled] = 0
        return int(dead_idx.numel())


def growth_count(n: int, max_cap: int) -> int:
    """mcmc.cpp:199-201: (int)(1.05f * current_n) is a float product."""
    return max(0, min(max_cap, int(np.float32(np.float32(1.05) * np.float32(n)))) - n)


def add_new_gs(P: dict, M1: dict, M2: dict, sampled: torch.Tensor, relocation, binoms, min_opacity: float):
    """mcmc.cpp:192-347: returns new (P, M1, M2) dicts with the sampled rows appended (torch::cat)."""
    with torch.no_grad():
        sampled = sampled.long()
        n_max = binoms.shape[0]
        counts = torch.zeros_like(P["opacity_raw"].reshape(-1))
        counts.index_add_(0, sampled, torch.ones_like(sampled, dtype=counts.dtype))
        ratios = torch.clamp(counts[sampled] + 1, 1, n_max).to(torch.int32)
        _relocate_rows(P, sampled, ratios, relocation, binoms, min_opacity)
        nP = {k: torch.cat([P[k], P[k][sampled]], 0) for k in GROUPS}
        z = {k: torch.zeros_like(P[k][sampled]) for k in GROUPS}
        return nP, {k: torch.cat([M1[k], z[k]], 0) for k in GROUPS}, {k: torch.cat([M2[k], z[k]], 0) for k in GROUPS}


def regularizer_grads(P: dict, scale_reg: float, opacity_reg: float) -> tuple[dict, torch.Tensor, torch.Tensor]:
    """trainer.cpp:132-158 by autograd: the gradients the two regulariser backward passes add."""
    s = P["scaling_raw"].detach().clone().requires_grad_(True)
    o = P["opacity_raw"].detach().clone().requires_grad_(True)
    ls = scale_reg * torch.exp(s).mean()
    lo = opacity_reg * torch.sigmoid(o).mean()
    ls.backward()
    lo.backward()
    return {"scaling_raw": s.grad, "opacity_raw": o.grad}, ls.detach(), lo.detach()


def adam_step(P: dict, G: dict, M1: dict, M2: dict, lrs: list, steps: dict, iteration: int,
              beta1=0.9, beta2=0.999, eps=1e-15) -> None:
    """FusedAdam (fused_adam.cpp:22-95): groups without a gradient are skipped and keep their step count; shN frozen
    for the first 1000 iterations (its count still advances)."""
    with torch.no_grad():
        for i, k in enumerate(GROUPS):
            if G.get(k) is None or P[k].numel() == 0:
                continue
            steps[k] += 1
            if k == "shN" and iteration <= 1000:
                continue
            t = steps[k]
            g = G[k]
            M1[k].mul_(beta1).add_(g, alpha=1 - beta1)
            M2[k].mul_(beta2).addcmul_(g, g, value=1 - beta2)
            bc1 = 1.0 / (1.0 - beta1 ** t)
            bc2 = 1.0 / np.sqrt(1.0 - beta2 ** t)
            P[k].sub_(lrs[i] * bc1 * M1[k] / (M2[k].sqrt() * bc2 + eps))


class Strategy:
    """post_backward + step of mcmc.cpp with injected draws and noise; keeps P, moments, step counts, the lr schedule
    and the active SH degree like the reference's SplatData / FusedAdam / ExponentialLR."""

    def __init__(self, P, lrs, cfg, relocation, binoms, add_noise, sh_degree=0):
        self.P = {k: v.detach().clone() for k, v in P.items()}
        self.M1 = {k: torch.zeros_like(v) for k, v in self.P.items()}
        self.M2 = {k: torch.zeros_like(v) for k, v in self.P.items()}
        self.steps = {k: 0 for k in GROUPS}
        self.lrs = list(lrs)
        self.gamma = 0.01 ** (1.0 / cfg.iterations)
        self.cfg, self.relocation, self.binoms, self.add_noise = cfg, relocation, binoms, add_noise
        self.sh_degree = sh_degree
        self.ns = []

    def is_refining(self, it):
        c = self.cfg
        return c.start_refine < it < c.stop_refine and it % c.refine_every == 0

    def iteration(self, it, grads: dict, reloc_samples, grow_samples, noise) -> bool:
        """grads: the photometric gradients of this iteration.  Returns True when rows were added (Adam skipped)."""
        c = self.cfg
        G = {k: grads[k].detach().clone() for k in GROUPS}
        rg, _, _ = regularizer_grads(self.P, c.scale_reg, c.opacity_reg)
        G["scaling_raw"] += rg["scaling_raw"]
        G["opacity_raw"] += rg["opacity_raw"]
        if it % c.sh_degree_interval == 0 and self.sh_degree < c.sh_degree:
            self.sh_degree += 1
        grew = False
        if self.is_refining(it):
            relocate_gs(self.P, self.M1, self.M2, reloc_samples, self.relocation, self.binoms, c.min_opacity)
            if growth_count(self.P["means"].shape[0], c.max_cap):
                self.P, self.M1, self.M2 = add_new_gs(self.P, self.M1, self.M2, grow_samples, self.relocation,
                                                      self.binoms, c.min_opacity)
                grew = True
        lr = float(np.float32(self.lrs[0]) * np.float32(c.noise_lr))
        self.add_noise(self.P, noise, lr)
        if not grew:  # the new leaves of add_new_gs have no gradient: FusedAdam steps nothing
            adam_step(self.P, G, self.M1, self.M2, self.lrs, self.steps, it)
        self.lrs[0] *= self.gamma
        self.ns.append(self.P["means"].shape[0])
        return grew
