"""Torch restatement of the reference's default densification strategy (src/training/strategies/default_strategy.cpp:
duplicate, split, remove, grow_gs, prune_gs, reset_opacity, post_backward, is_refining) and of FusedAdam's bookkeeping
around it (a group whose tensor was replaced has no gradient: it is skipped and keeps its step count).
`quats_to_rotmats` is supplied by the caller (this library's or the reference's kernel, or `quats_to_rotmats_torch`),
and the split's normals z are injected or drawn as the reference draws them.  Works on CPU or CUDA tensors;
parameters and moments are dicts over GROUPS."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

GROUPS = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")


def quats_to_rotmats_torch(q: torch.Tensor) -> torch.Tensor:
    """QuatToRotmatCUDA.cu:14-39 in torch (normalising, row-major), for CPU use."""
    q = q * torch.rsqrt((q * q).sum(-1, keepdim=True))
    w, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)
    return R.reshape(-1, 3, 3)


def f32(x: float) -> float:
    return float(np.float32(x))


def is_refining(cfg, it: int) -> bool:
    """default_strategy.cpp:31-35"""
    return it > cfg.start_refine and it % cfg.refine_every == 0 and it % cfg.reset_every >= cfg.pause_refine_after_reset


def _cat_zeros(M: torch.Tensor, n: int) -> torch.Tensor:
    return torch.cat([M, torch.zeros((n,) + tuple(M.shape[1:]), dtype=M.dtype, device=M.device)], 0)


def duplicate(P: dict, M1: dict, M2: dict, is_dup: torch.Tensor):
    """:49-85: the duplicated rows appended, zero moments for them."""
    idx = is_dup.nonzero().squeeze(-1)
    P = {k: torch.cat([P[k], P[k].index_select(0, idx)]) for k in GROUPS}
    return P, {k: _cat_zeros(M1[k], idx.numel()) for k in GROUPS}, {k: _cat_zeros(M2[k], idx.numel()) for k in GROUPS}


def split(P: dict, M1: dict, M2: dict, is_split: torch.Tensor, quats_to_rotmats, revised_opacity: bool, z=None):
    """:87-162: rest rows, then copy 0 of every split row, then copy 1.  Returns (P, M1, M2, z)."""
    idx = is_split.nonzero().squeeze(-1)
    rest = is_split.logical_not().nonzero().squeeze(-1)
    scales = torch.exp(P["scaling_raw"]).index_select(0, idx)
    quats = F.normalize(P["rotation_raw"], dim=-1).index_select(0, idx)
    R = quats_to_rotmats(quats.contiguous())
    n = idx.numel()
    if z is None:
        z = torch.randn((2, n, 3), device=P["means"].device)
    samples = torch.einsum("nij,nj,bnj->bni", R, scales, z)
    out = {}
    for k in GROUPS:
        sampled = P[k].index_select(0, idx)
        repeats = [2] + [1] * (P[k].dim() - 1)
        if k == "means":
            sp = (sampled.unsqueeze(0) + samples).reshape(-1, 3)
        elif k == "scaling_raw":
            sp = torch.log(scales / 1.6).repeat(2, 1)
        elif k == "opacity_raw" and revised_opacity:
            sp = torch.logit(1.0 - torch.sqrt(1.0 - torch.sigmoid(sampled))).repeat(repeats)
        else:
            sp = sampled.repeat(repeats)
        out[k] = torch.cat([P[k].index_select(0, rest), sp], 0)
    return (out, {k: _cat_zeros(M1[k].index_select(0, rest), 2 * n) for k in GROUPS},
            {k: _cat_zeros(M2[k].index_select(0, rest), 2 * n) for k in GROUPS}, z)


def remove(P: dict, M1: dict, M2: dict, is_prune: torch.Tensor):
    """:194-227"""
    keep = is_prune.logical_not().nonzero().squeeze(-1)
    sel = lambda D: {k: D[k].index_select(0, keep) for k in GROUPS}
    return sel(P), sel(M1), sel(M2)


def grow_gs(P, M1, M2, info, cfg, scene_scale, quats_to_rotmats, z=None):
    """:164-192.  Returns (P, M1, M2, n_dup, n_split, z)."""
    grads = info[1] / torch.clamp_min(info[0], 1.0)
    is_grad_high = grads > cfg.grad_threshold
    max_values = torch.exp(P["scaling_raw"]).max(-1).values
    is_small = max_values <= f32(np.float32(cfg.grow_scale3d) * np.float32(scene_scale))
    is_dup = is_grad_high & is_small
    n_dup = int(is_dup.sum())
    is_split = is_grad_high & ~is_small
    n_split = int(is_split.sum())
    if n_dup > 0:
        P, M1, M2 = duplicate(P, M1, M2, is_dup)
    is_split = torch.cat([is_split, torch.zeros(n_dup, dtype=torch.bool, device=is_split.device)])
    if n_split > 0:
        P, M1, M2, z = split(P, M1, M2, is_split, quats_to_rotmats, cfg.revised_opacity, z)
    return P, M1, M2, n_dup, n_split, (z if n_split > 0 else None)


def prune_mask(P: dict, it: int, cfg, scene_scale) -> torch.Tensor:
    """:229-243"""
    is_prune = torch.sigmoid(P["opacity_raw"]).reshape(-1) < cfg.prune_opacity
    rot = P["rotation_raw"]
    is_prune |= (rot * rot).sum(-1) < 1e-8
    if it > cfg.reset_every:
        max_values = torch.exp(P["scaling_raw"]).max(-1).values
        is_prune |= max_values > f32(np.float32(cfg.prune_scale3d) * np.float32(scene_scale))
    return is_prune


def prune_gs(P, M1, M2, it, cfg, scene_scale):
    """:229-249.  Returns (P, M1, M2, n_prune)."""
    is_prune = prune_mask(P, it, cfg, scene_scale)
    n = int(is_prune.sum())
    if n > 0:
        P, M1, M2 = remove(P, M1, M2, is_prune)
    return P, M1, M2, n


def reset_threshold(prune_opacity: float) -> float:
    """:254-260: torch::logit(torch::tensor(2.0f * prune_opacity)).item()"""
    return float(torch.logit(torch.tensor(f32(np.float32(2.0) * np.float32(prune_opacity)))).item())


def reset_opacity(P: dict, M1: dict, M2: dict, cfg) -> None:
    """:251-290, in place on the dicts' entries"""
    P["opacity_raw"] = torch.clamp_max(P["opacity_raw"], reset_threshold(cfg.prune_opacity))
    M1["opacity_raw"] = torch.zeros_like(M1["opacity_raw"])
    M2["opacity_raw"] = torch.zeros_like(M2["opacity_raw"])


def refine(P, M1, M2, info, it, cfg, scene_scale, quats_to_rotmats, z=None):
    """grow_gs then prune_gs.  Returns (P, M1, M2, counts (n_dup, n_split, n_prune, N_final), z)."""
    P, M1, M2, n_dup, n_split, z = grow_gs(P, M1, M2, info, cfg, scene_scale, quats_to_rotmats, z)
    P, M1, M2, n_prune = prune_gs(P, M1, M2, it, cfg, scene_scale)
    return P, M1, M2, (n_dup, n_split, n_prune, int(P["means"].shape[0])), z


class Strategy:
    """post_backward of default_strategy.cpp with FusedAdam's step-count bookkeeping; keeps P, moments, the
    statistics, step counts and the active SH degree like the reference's SplatData / FusedAdam."""

    def __init__(self, P, M1, M2, cfg, scene_scale, quats_to_rotmats, sh_degree=0, steps=None):
        self.P = {k: v.detach().clone() for k, v in P.items()}
        self.M1 = {k: v.detach().clone() for k, v in M1.items()}
        self.M2 = {k: v.detach().clone() for k, v in M2.items()}
        self.cfg, self.scene_scale, self.q2r = cfg, scene_scale, quats_to_rotmats
        self.info = torch.zeros((2, self.P["means"].shape[0]), device=self.P["means"].device)
        self.steps = dict(steps) if steps is not None else {k: 0 for k in GROUPS}
        self.sh_degree = sh_degree
        self.counts = None

    def post_backward(self, it: int, z=None) -> tuple:
        """Returns the groups FusedAdam skips this iteration (their tensors were replaced)."""
        c = self.cfg
        self.counts = None
        if it % c.sh_degree_interval == 0 and self.sh_degree < c.sh_degree:
            self.sh_degree += 1
        if it == c.stop_refine:
            self.info = torch.empty(0, device=self.info.device)
        if it >= c.stop_refine:
            return ()
        skip = ()
        if is_refining(c, it):
            P, M1, M2, counts, _ = refine(self.P, self.M1, self.M2, self.info, it, c, self.scene_scale, self.q2r, z)
            self.counts = counts
            if counts[0] or counts[1] or counts[2]:
                self.P, self.M1, self.M2 = P, M1, M2
                skip = GROUPS
            self.info = torch.zeros((2, self.P["means"].shape[0]), device=self.info.device)
        if it % c.reset_every == 0 and it > 0:
            reset_opacity(self.P, self.M1, self.M2, c)
            skip = skip or ("opacity_raw",)
        return skip

    def adam_bookkeeping(self, skip: tuple) -> None:
        """FusedAdam's step counts: every group with a gradient advances (shN too while frozen)."""
        for k in GROUPS:
            if k not in skip and self.P[k].numel():
                self.steps[k] += 1
