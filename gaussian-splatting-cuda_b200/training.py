"""Host-side mirror of the reference's training iteration around the hot path (SURVEY.md 8 f2 / f3):

  photometric_loss   trainer.cpp:103-126 (L1 + fused SSIM "valid") as one kernel that also returns dLoss/d(render)
  FusedAdam          src/training/optimizers/fused_adam.cpp:22-117 + strategy_utils.cpp:27-55 (per-group learning rates,
                     eps 1e-15, exponential decay of the position learning rate, shN frozen for the first 1000
                     iterations), all groups stepped by ONE kernel launch (gsb_adam_step)
  TrainStep          render (extended operator on the raw tensors) -> loss -> backward -> Adam, with the intersection
                     buffer sized from a capacity so that the iteration has no host read-back
  strategy           optional densification (SURVEY.md 8 f6, strategy.py): MCMC (mcmc.py) or the default strategy
                     (adc.py, whose statistics the fastgs backward accumulates).  After the backward: the regularisers
                     -> post_backward (SH bump, the refine, the pre-Adam hook: MCMC's noise) -> Adam, skipping the
                     groups the refine returns (all six when it replaced the tensors) -> scheduler
  bilateral_grid     optional (SURVEY.md 8 f5, trainer.cpp:662-665,698-705,758-762): render -> slice through the
                     image's grid -> unclamped loss -> + weight * TV of all grids -> backward -> one Adam launch for the
                     Gaussians and the grids (lr from the warm-up/exponential schedule, eps 1e-15)
  sparsity           optional ADMM sparsification with a strategy (sparsity.py, trainer.cpp:173-247,707-784): after
                     the regularisers the sparsity loss's gradient; post_backward only up to the base iteration count;
                     after Adam the state update and, on the last iteration, the prune

Everything that computes lives behind the C ABI; this file only orders the calls, like the reference's trainer does."""
from __future__ import annotations

import dataclasses
import itertools
import math
from dataclasses import dataclass, field

import torch

from . import _product_ns, load, rasterize_fused
from .bilateral import BilateralGrid, WarmupExponentialLR
from .sparsity import ADMMSparsity
from .strategy import PARAM_GROUPS, Strategy


class _PhotometricLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renders, target, lambda_dssim, clamp):
        ns = _product_ns()
        op = ns.photometric_loss_fused if clamp else ns.photometric_loss_fused_unclamped
        stats, v = op(renders.detach().contiguous(), target.contiguous(), float(lambda_dssim), renders.requires_grad)
        ctx.save_for_backward(v)
        ctx.mark_non_differentiable(stats)
        return stats[0], stats

    @staticmethod
    def backward(ctx, g_loss, _g_stats):
        (v,) = ctx.saved_tensors
        return (v * g_loss if v.numel() else None), None, None, None


def photometric_loss_unclamped(renders, target, lambda_dssim: float = 0.2):
    """photometric_loss on an image used as it is (no clamp, no clamp mask): the loss of a bilateral-grid output."""
    load()
    return _PhotometricLoss.apply(renders, target, lambda_dssim, False)


def photometric_loss(renders, target, lambda_dssim: float = 0.2):
    """(loss, stats) with stats = device tensor [loss, l1 mean, ssim mean].  renders [1,H,W,3] unclamped (the blend's
    output); target [3,H,W] (the reference's image layout) or [1,H,W,3]."""
    load()
    return _PhotometricLoss.apply(renders, target, lambda_dssim, True)


@dataclass
class AdamConfig:
    """parameter/*_optimization_params.json defaults (include/core/parameters.hpp)."""
    means_lr: float = 0.00016
    shs_lr: float = 0.0025
    scaling_lr: float = 0.005
    rotation_lr: float = 0.001
    opacity_lr: float = 0.05
    scene_scale: float = 1.0
    iterations: int = 30000
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-15

    def lrs(self):
        return [self.means_lr * self.scene_scale, self.shs_lr, self.shs_lr / 20.0, self.scaling_lr, self.rotation_lr,
                self.opacity_lr]


def _adam_step(groups: list, dyn: torch.Tensor | None = None) -> None:
    """Steps the groups (param, grad, exp_avg, exp_avg_sq, (beta1, beta2, eps), s) in order, one launch per run of
    equal (beta1, beta2, eps).  s is (lr, step count) with the scalars on the host, or the group's row of `dyn`
    (lr, the two bias corrections, enabled) with the scalars on the device."""
    ns = _product_ns()
    with torch.no_grad():
        for (beta1, beta2, eps), run in itertools.groupby(groups, key=lambda g: g[4]):
            p, g, m, v, _, s = (list(x) for x in zip(*run))
            if dyn is None:
                ns.fused_adam_step(p, g, m, v, [lr for lr, _ in s], beta1, beta2, eps, [t for _, t in s])
            else:
                rows = dyn[s[0]:s[-1] + 1]
                ns.fused_adam_step_dynamic(p, g, m, v, rows if len(rows) == len(s) else dyn[s], beta1, beta2, eps)


class FusedAdam:
    """One launch per step for the six SplatData groups.  State tensors are allocated lazily like the reference's."""

    def __init__(self, params: dict, cfg: AdamConfig | None = None):
        self.cfg = cfg or AdamConfig()
        self.params = params
        self.lr = self.cfg.lrs()
        self.gamma = 0.01 ** (1.0 / self.cfg.iterations)  # ExponentialLR on group 0 (strategy_utils.cpp:52-55)
        self.exp_avg = {k: torch.zeros_like(v) for k, v in params.items()}
        self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in params.items()}
        self.steps = {k: 0 for k in params}

    def advance(self, iteration: int, skip=()) -> list:
        """fused_adam.cpp:61-81 for one step: every group not in `skip` advances its step count (a skipped group keeps
        it), and those groups are stepped except shN up to iteration 1000, whose count advances all the same.
        Returns the groups to step."""
        stepped = []
        for k in PARAM_GROUPS:
            if k in skip:
                continue
            self.steps[k] += 1
            if not (k == "shN" and iteration <= 1000):
                stepped.append(k)
        return stepped

    def _group(self, k: str, s):
        p = self.params[k]
        return p, p.grad, self.exp_avg[k], self.exp_avg_sq[k], (self.cfg.beta1, self.cfg.beta2, self.cfg.eps), s

    def step(self, iteration: int, extra=()):
        """Steps the groups that have a gradient, then the `extra` groups (param, grad, exp_avg, exp_avg_sq,
        (beta1, beta2, eps), (lr, step count)): one launch, or one more per change of hyperparameters."""
        absent = [k for k in PARAM_GROUPS if self.params[k].grad is None or self.params[k].numel() == 0]
        groups = [self._group(k, (self.lr[PARAM_GROUPS.index(k)], self.steps[k]))
                  for k in self.advance(iteration, absent)]
        _adam_step(groups + list(extra))
        self.lr[0] *= self.gamma

    def zero_grad(self):
        for p in self.params.values():
            p.grad = None


class _GridState:
    """What the training iteration keeps for the bilateral grids: the device image index, the TV weight as a device
    scalar, the grids' Adam moments and step count, and their learning-rate schedule (trainer.cpp:66-101)."""

    # the grids' own torch::optim::Adam (trainer.cpp:81-83): default betas, eps 1e-15 -- independent of the Gaussians'
    beta1, beta2, eps = 0.9, 0.999, 1e-15

    def __init__(self, grid: BilateralGrid, lr: float, tv_weight: float, iterations: int):
        g = grid.grids
        self.grid = grid
        self.sched = WarmupExponentialLR(lr, iterations)
        self.exp_avg, self.exp_avg_sq = torch.zeros_like(g), torch.zeros_like(g)
        self.steps = 0
        self.idx = torch.zeros(1, dtype=torch.int32, device=g.device)
        self.weight = torch.full((1,), float(tv_weight), dtype=torch.float32, device=g.device)

    def set_image(self, image_idx) -> None:
        if image_idx is None or not 0 <= int(image_idx) < self.grid.num_images:
            raise ValueError(f"a training step with a bilateral grid needs an image index in [0, {self.grid.num_images})")
        self.idx.fill_(int(image_idx))  # a kernel argument: no host buffer to race with

    def tv(self):
        """(TV loss of all grids, weight * its gradient): the buffer the slice backward then adds into."""
        return _product_ns().bilagrid_tv(self.grid.grids.detach(), self.weight, True)

    def advance(self):
        """(lr, step count) of this step; advances the schedule (bilateral_grid_scheduler_->step())."""
        self.steps += 1
        lr = self.sched.lr
        self.sched.step()
        return lr, self.steps

    def adam_group(self, s):
        """The grids' Adam group, with scalars s as _adam_step takes them."""
        g = self.grid.grids
        return g.detach(), g.grad, self.exp_avg, self.exp_avg_sq, (self.beta1, self.beta2, self.eps), s


class _SliceIntoGrad(torch.autograd.Function):
    """Slice for the training step: the backward ADDS the grid gradient into v_grids (the TV gradient of all grids)
    and returns the gradient of the unclamped render only."""

    @staticmethod
    def forward(ctx, image, grids, image_idx, v_grids, chw):
        image = image.detach().contiguous()
        ctx.save_for_backward(image, grids, image_idx, v_grids)
        ctx.chw = chw
        return _product_ns().bilagrid_slice(grids, image, image_idx, chw)

    @staticmethod
    def backward(ctx, v_out):
        image, grids, image_idx, v_grids = ctx.saved_tensors
        return _product_ns().bilagrid_slice_backward(grids, image, image_idx, v_out.contiguous(), v_grids, ctx.chw), \
            None, None, None, None


def _check_sparsity(sparsity, strategy) -> None:
    if sparsity is not None and strategy is None:
        raise ValueError("sparsity needs a strategy: the final prune removes rows from the strategy's tensors, and "
                         "the strategy's post_backward stops after the base iterations")


def _check_step(strategy, sparsity, params, optimizer, sh_degree) -> None:
    """A strategy owns the parameter dict and the optimizer's moments: the step must use the same objects, and the
    degree it renders with is the strategy's active degree (SplatData's, which the strategy raises).  Sparsity needs
    a strategy."""
    _check_sparsity(sparsity, strategy)
    if strategy is None:
        return
    if params is not None and params is not strategy.params:
        raise ValueError("the step's params must be the strategy's params dict (growth replaces its tensors)")
    if optimizer is not None and optimizer is not strategy.optimizer:
        raise ValueError("the step's optimizer must be the strategy's optimizer (growth replaces its moments)")
    if sh_degree is not None and int(sh_degree) != strategy.sh_degree:
        raise ValueError(f"sh_degree {sh_degree} differs from the strategy's active degree {strategy.sh_degree}: "
                         f"pass {type(strategy).__name__}(..., sh_degree=...) or the step the same degree")


class _EagerStep:
    """What TrainStep and FastGsTrainStep share around their render -> loss -> backward (`_forward_backward`)."""

    def __post_init__(self):
        _check_step(self.strategy, self.sparsity, self.params, self.optimizer, self.sh_degree)

    def _grid(self) -> _GridState:
        if self.grid_state is None:
            its = self.optimizer.cfg.iterations if self.optimizer is not None else AdamConfig().iterations
            self.grid_state = _GridState(self.bilateral_grid, self.bilateral_grid_lr, self.tv_loss_weight, its)
        return self.grid_state

    def _begin(self) -> None:
        self.iteration += 1
        if self.strategy is not None:
            self.sh_degree = self.strategy.sh_degree

    def _finish(self, loss, last: dict):
        """After the backward (trainer.cpp:668-762): the regularisers, the sparsity loss's gradient when it applies, the
        strategy's post_backward up to the base iteration count, Adam (the grids' group after the Gaussians'), the
        sparsifier's update and prune."""
        st, sp, it = self.strategy, self.sparsity, self.iteration
        reg = sp_loss = None
        if st is not None:
            with torch.no_grad():
                reg = st.regularize()
                if sp is not None:
                    sp_loss = sp.loss_step(st.params["opacity_raw"], it)
                if sp is None or sp.post_backward_due(it):
                    st.post_backward(it)
        if sp_loss is not None:
            loss = loss.detach() + sp_loss[0]
        if self.optimizer is not None:
            G = self.grid_state
            self.optimizer.step(it, [G.adam_group(G.advance())] if G is not None else ())
            self.optimizer.zero_grad()
            if G is not None:
                G.grid.grids.grad = None
        if sp is not None:
            sp.after_step(st, it)
        self.last = {**last, "reg": reg, "sparsity_loss": sp_loss}
        return loss


@dataclass
class TrainStep(_EagerStep):
    """One training iteration on resident raw parameters: camera + target in, loss (device scalar) out."""
    params: dict
    sh_degree: int
    width: int
    height: int
    lambda_dssim: float = 0.2
    optimizer: FusedAdam | None = None
    capacity: int = 0                    # intersections the buffers are sized for; 0 = size exactly (one read-back)
    iteration: int = 0
    last: dict = field(default_factory=dict)
    bilateral_grid: BilateralGrid | None = None  # use_bilateral_grid: the iteration needs image_idx
    bilateral_grid_lr: float = 2e-3
    tv_loss_weight: float = 10.0                 # mcmc_optimization_params.json (default_optimization_params.json: 5)
    grid_state: _GridState | None = None         # created on first use
    strategy: Strategy | None = None             # densification: owns params and the optimizer's moments
    sparsity: ADMMSparsity | None = None         # ADMM sparsification after the base iterations (needs a strategy)

    def _forward_backward(self, viewmat, K, target, background):
        """render -> loss -> backward, or render -> slice -> unclamped loss -> backward with the grids' gradient (TV
        and slice) left in their .grad: (loss, stats, intersection count)."""
        P = self.params
        out = rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                              self.sh_degree, viewmat, K, self.width, self.height, bg_color=background,
                              isect_capacity=self.capacity)
        if self.bilateral_grid is None:
            loss, stats = photometric_loss(out.render_colors, target, self.lambda_dssim)
            loss.backward()
            return loss, stats, out.n_isects
        G = self._grid()
        tv, v_grids = G.tv()
        sliced = _SliceIntoGrad.apply(out.render_colors, G.grid.grids.detach(), G.idx, v_grids, False)
        loss, stats = photometric_loss_unclamped(sliced, target, self.lambda_dssim)
        loss.backward()
        G.grid.grids.grad = v_grids
        return loss.detach() + G.weight[0] * tv, stats, out.n_isects  # the trainer's loss_value includes the TV term

    def __call__(self, viewmat, K, target, background=None, image_idx=None):
        self._begin()
        if self.bilateral_grid is not None:
            self._grid().set_image(image_idx)
        loss, stats, n = self._forward_backward(viewmat, K, target, background)
        return self._finish(loss, {"n_isects": n, "stats": stats})

    def size_capacity(self, viewmat, K, target, background=None, slack: float = 1.25):
        """An exact (synchronising) render sizes the intersection capacity for the following steps."""
        with torch.no_grad():
            P = self.params
            out = rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                                  self.sh_degree, viewmat, K, self.width, self.height, bg_color=background)
            n = int(out.n_isects.item())
        self.capacity = int(n * slack) + 1024
        return n


@dataclass
class FastGsTrainStep(_EagerStep):
    """One training iteration on the reference's DEFAULT rasterizer path (SURVEY.md 8 f4 + f2 + f3), ordered like
    the reference's trainer (trainer.cpp: fast_rasterize -> photometric loss -> backward -> optimizer step):
    fastgs forward (raw parameters in) -> background composite (fast_rasterizer.cpp:71) -> fused SSIM + L1 loss and
    gradient on the [3,H,W] image -> fastgs backward -> one-launch Adam.  No autograd graph is built: the loss kernel
    returns dLoss/d(image) and the backward takes it directly."""
    params: dict                          # PARAM_GROUPS -> leaf tensors (opacity_raw [N,1] or [N])
    sh_degree: int
    width: int
    height: int
    lambda_dssim: float = 0.2
    optimizer: FusedAdam | None = None
    backend: object = None                # fastgs.FastGsBackend; default: this library
    capacity: int = 0                     # > 0: instance buffer sized from it, no host read-back (rasterization_ext.h)
    iteration: int = 0
    last: dict = field(default_factory=dict)
    bilateral_grid: BilateralGrid | None = None  # use_bilateral_grid: the iteration needs image_idx
    bilateral_grid_lr: float = 2e-3
    tv_loss_weight: float = 10.0
    grid_state: _GridState | None = None         # created on first use
    index_on_device: bool = False                # the caller refreshes grid_state.idx itself (image_idx is not read)
    strategy: Strategy | None = None             # densification: owns params and the optimizer's moments
    sparsity: ADMMSparsity | None = None         # ADMM sparsification after the base iterations (needs a strategy)

    def size_capacity(self, w2c, settings, slack: float = 1.25):
        """One exact (synchronising) forward sizes the instance capacity for the following iterations."""
        from . import fastgs as fg
        be = self.backend or fg.default_backend()
        P = self.params
        with torch.no_grad():
            _, _, ctx = be.forward(P["means"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"].reshape(-1, 1), P["sh0"],
                                   P["shN"], w2c, settings)
        n = int(ctx["ints"][1])
        self.capacity = int(n * slack) + 1024
        return n

    def _forward_backward(self, w2c, settings, target, background, densification_info):
        """forward -> composite -> loss and its gradient [-> slice, unclamped loss, slice backward with the grids'
        gradient left in their .grad] -> backward into the parameters' .grad: (loss, stats, instance count)."""
        from . import fastgs as fg
        be = self.backend or fg.default_backend()
        P = self.params
        G = self._grid() if self.bilateral_grid is not None else None
        with torch.no_grad():
            opac = P["opacity_raw"].reshape(-1, 1)
            image, alpha, ctx = be.forward(P["means"], P["scaling_raw"], P["rotation_raw"], opac, P["sh0"], P["shN"], w2c, settings,
                                           capacity=self.capacity)
            final = image + (1.0 - alpha) * background.reshape(3, 1, 1) if background is not None else image
            if G is None:
                stats, v_final = _product_ns().photometric_loss_fused(final.contiguous(), target.contiguous(),
                                                                      float(self.lambda_dssim), True)
            else:  # slice -> unclamped loss -> slice backward (adds into the TV gradient of all grids)
                ns = _product_ns()
                final = final.contiguous()
                tv, v_grids = G.tv()
                grids = G.grid.grids.detach()
                sliced = ns.bilagrid_slice(grids, final, G.idx, True)
                stats, v_sliced = ns.photometric_loss_fused_unclamped(sliced, target.contiguous(), float(self.lambda_dssim),
                                                                      True)
                v_final = ns.bilagrid_slice_backward(grids, final, G.idx, v_sliced, v_grids, True)
                G.grid.grids.grad = v_grids
            v_alpha = (-(v_final * background.reshape(3, 1, 1)).sum(0, keepdim=True) if background is not None
                       else torch.zeros_like(alpha))
            g = be.backward(ctx, v_final, v_alpha.contiguous(), image, alpha, P["means"], P["scaling_raw"], P["rotation_raw"],
                            P["shN"], w2c, settings, densification_info)
            for k, gk in zip(("means", "scaling_raw", "rotation_raw", "opacity_raw", "sh0", "shN"), g[:6]):
                P[k].grad = gk.reshape(P[k].shape)
        loss = stats[0] if G is None else stats[0] + G.weight[0] * tv
        # capacity mode: the count is a device tensor (compare it with the capacity when convenient)
        return loss, stats, ctx.get("n_instances_dev", int(ctx["ints"][1]))

    def __call__(self, w2c, settings, target, background=None, densification_info=None, image_idx=None):
        self._begin()
        st = self.strategy
        if st is not None:
            settings = dataclasses.replace(settings, active_sh_bases=(self.sh_degree + 1) ** 2)
            if st.densification_info is not None:  # the backward accumulates the strategy's statistics
                if densification_info is not None:
                    raise ValueError("the strategy owns densification_info: do not pass it as well")
                densification_info = st.densification_info
        if self.bilateral_grid is not None and not self.index_on_device:
            self._grid().set_image(image_idx)
        loss, stats, n = self._forward_backward(w2c, settings, target, background, densification_info)
        return self._finish(loss, {"n_instances": n, "stats": stats})


class GraphedTrainStep:
    """The whole iteration -- extended render operator, loss-and-gradient kernel, blend backward, fused back kernel, Adam --
    captured ONCE in a CUDA graph and replayed: one graph launch per iteration instead of ~25 kernel launches and their
    torch bookkeeping.  Possible because nothing inside the iteration needs a host-side value: the intersection buffers
    are sized from a capacity (the count stays on the device, `overflowed()` checks it afterwards) and Adam's
    step-dependent scalars (learning rates, bias corrections, the shN freeze of the first 1000 iterations) are read from a
    small device tensor that is refreshed before every replay.

    Per iteration the host copies the camera (viewmat, K), the background and the target image into static device buffers
    (pinned -> device, on the replay stream) and reads the loss back when it wants to.  The render -> loss -> backward
    part is the eager step's own (`self.step`)."""

    def __init__(self, params: dict, sh_degree: int, width: int, height: int, cfg: AdamConfig | None = None,
                 lambda_dssim: float = 0.2, capacity_slack: float = 1.25, bilateral_grid: BilateralGrid | None = None,
                 bilateral_grid_lr: float = 2e-3, tv_loss_weight: float = 10.0, strategy: Strategy | None = None,
                 sparsity: ADMMSparsity | None = None):
        load()
        _check_step(strategy, sparsity, params, None, sh_degree)
        self.sparsity = sparsity
        self.sparsity_in_graph = False  # the captured part A adds the sparsity loss
        self.hook_in_graph = False      # the captured part B runs the strategy's pre-Adam hook
        self.params, self.sh_degree, self.W, self.H = params, int(sh_degree), int(width), int(height)
        self.lambda_dssim = float(lambda_dssim)
        # with a strategy, its optimizer (whose moments live in the strategy's storage) is the step's
        self.opt = strategy.optimizer if strategy is not None else FusedAdam(params, cfg)
        self.strategy = strategy
        self.graph_b = None
        self.captures = 0
        self.slack = capacity_slack
        dev = params["means"].device
        self.dev = dev
        self.static = {"viewmat": torch.zeros((1, 4, 4), device=dev), "K": torch.zeros((1, 3, 3), device=dev),
                       "background": torch.zeros((1, 3), device=dev),
                       "target": torch.zeros((3, self.H, self.W), device=dev)}
        # with a bilateral grid, its image index is a device input and its Adam scalars are one more row of `dyn`
        self.bilateral_grid = bilateral_grid
        self.grid_state = (_GridState(bilateral_grid, bilateral_grid_lr, tv_loss_weight, self.opt.cfg.iterations)
                           if bilateral_grid is not None else None)
        self.step = TrainStep(params, self.sh_degree, self.W, self.H, self.lambda_dssim, bilateral_grid=bilateral_grid,
                              grid_state=self.grid_state)
        n_rows = len(PARAM_GROUPS) + (1 if bilateral_grid is not None else 0)
        self.dyn = torch.zeros((n_rows, 4), device=dev)
        self.dyn_host = torch.zeros((n_rows, 4)).pin_memory()
        self.graph = None
        self.loss = None
        self.stats = None
        self.n_isects = None
        self.capacity = 0
        self.iteration = 0

    def _forward_backward(self):
        S = self.static
        return self.step._forward_backward(S["viewmat"], S["K"], S["target"], S["background"])

    def _size_capacity(self) -> int:
        S = self.static
        self.step.sh_degree = self.sh_degree
        return self.step.size_capacity(S["viewmat"], S["K"], S["target"], S["background"], self.slack)

    def _set_inputs(self, viewmat, K, target, background):
        S = self.static
        S["viewmat"].copy_(viewmat.reshape(1, 4, 4), non_blocking=True)
        S["K"].copy_(K.reshape(1, 3, 3), non_blocking=True)
        S["target"].copy_(target.reshape(3, self.H, self.W), non_blocking=True)
        if background is not None:
            S["background"].copy_(background.reshape(1, 3), non_blocking=True)

    def _part_a(self):
        """render -> loss -> backward [-> the strategy's regularisers, then in the sparsity phase the sparsity loss
        (rho read on the device: zero on the prune iteration)]: (loss, stats, count)"""
        loss, stats, n = self._forward_backward()
        if self.strategy is not None:
            with torch.no_grad():
                self.strategy.regularize()
                if self.sparsity_in_graph:
                    loss = loss.detach() + self.sparsity.add_loss_gradient(self.params["opacity_raw"])[0]
        return loss, stats, n

    def _part_b(self):
        """[the strategy's pre-Adam hook at group 0's rate, read from `dyn` ->] Adam"""
        if self.strategy is not None and self.hook_in_graph:
            self.strategy.before_adam(self.dyn[0, 0:1])
        self._adam()

    def _adam(self):
        """Adam on the scalars of `dyn`: the non-empty Gaussian groups, then the grids'."""
        groups = [self.opt._group(k, i) for i, k in enumerate(PARAM_GROUPS) if self.params[k].numel() > 0]
        if self.grid_state is not None:
            groups.append(self.grid_state.adam_group(len(PARAM_GROUPS)))
        _adam_step(groups, self.dyn)

    def _body(self):
        loss, stats, n = self._part_a()
        self._part_b()
        return loss, stats, n

    def _warm_up_and_capture(self):
        """Warm-up iterations with every Adam group disabled and a zero hook rate (`dyn` is zero: nothing moves), then
        the capture.  Without a strategy the iteration is one graph.  With one it is two graphs -- (render, loss,
        backward, regularisers) and (pre-Adam hook, Adam) -- so that a refine can run eagerly between them, and the
        warm-up's random draws are undone so that the replays draw what an eager run would.  The strategy's statistics,
        which the warm-up's backward passes accumulate into, are restored too."""
        self.dyn.zero_()
        st, sp = self.strategy, self.sparsity
        self.sparsity_in_graph = sp is not None and sp.initialized and not sp.done
        # post_backward, and with it the hook, must be due on every iteration the graphs serve: without a sparsifier,
        # or before its phase (entering the phase re-captures; the base iteration then runs the hook eagerly)
        self.hook_in_graph = sp is None or not (sp.initialized or sp.done)
        rng = torch.cuda.get_rng_state(self.dev) if st is not None else None
        info = st.densification_info if st is not None else None
        info_before = info.clone() if info is not None and info.numel() else None
        side = torch.cuda.Stream(self.dev)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                for p in self.params.values():
                    p.grad = None
                self._body()
        torch.cuda.current_stream(self.dev).wait_stream(side)
        for p in self.params.values():
            p.grad = None
        if rng is not None:
            torch.cuda.set_rng_state(rng, self.dev)
        if info_before is not None:
            info.copy_(info_before)
        self.graph = torch.cuda.CUDAGraph()
        self.captures += 1
        if st is None:
            with torch.cuda.graph(self.graph):
                self.loss, self.stats, self.n_isects = self._body()
            return
        with torch.cuda.graph(self.graph):
            self.loss, self.stats, self.n_isects = self._part_a()
        self.graph_b = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_b, pool=self.graph.pool()):
            self._part_b()

    def _replay(self):
        """One iteration with a strategy: part A, the refine eagerly when post_backward is due, the Adam scalars with
        the skipped groups disabled (their step counts held), the pre-Adam hook eagerly where part B does not hold it,
        then part B.  A refine that replaced the tensors leaves nothing for part B to step (as FusedAdam after the
        reference's torch::cat): it is not replayed and the next call re-captures.  So does an SH bump, a change of the
        statistics tensor (stop_refine) and the sparsifier's prune.  A refine that works in place keeps the graphs."""
        st, sp, it = self.strategy, self.sparsity, self.iteration
        lr0 = self.opt.lr[0]  # the rate before this iteration's scheduler step
        degree, info = st.sh_degree, st.densification_info
        self.graph.replay()
        post = sp is None or sp.post_backward_due(it)  # no post_backward after the base iterations
        skip = st.refine(it) if post else ()
        replaced = post and st.replaced
        self._set_scalars(skip)
        if post and (replaced or not self.hook_in_graph):
            st.before_adam(lr0)
        if not replaced:
            self.graph_b.replay()
        if sp is not None and sp.after_step(st, it):  # the prune replaced the tensors
            replaced = True
        if replaced or st.sh_degree != degree or st.densification_info is not info:
            self.graph = None

    def _enter_iteration(self) -> None:
        """Before the capture check of iteration self.iteration + 1: the sparsifier's lazy initialisation at its first
        loss iteration, which re-captures part A with the loss in it; rho set to zero where no loss applies."""
        sp = self.sparsity
        if sp is None or sp.done:
            return
        it = self.iteration + 1
        sp.check_rows(self.strategy.n)
        if sp.should_apply_loss(it) and not sp.initialized:
            sp.initialize(self.params["opacity_raw"])
            self.graph = None
        if sp.initialized and not sp.should_apply_loss(it):  # the prune iteration
            sp.rho.zero_()

    def _set_row(self, i: int, lr: float, t: int, beta1: float, beta2: float, enabled: bool) -> None:
        h = self.dyn_host
        h[i, 0] = lr
        h[i, 1] = 1.0 / (1.0 - beta1 ** t)
        h[i, 2] = 1.0 / math.sqrt(1.0 - beta2 ** t)
        h[i, 3] = 1.0 if enabled else 0.0

    def _set_scalars(self, skip: tuple = ()):
        """fused_adam.cpp:61-81 on the host (FusedAdam.advance: step counts, the shN freeze, the skipped groups held and
        disabled), bias corrections, strategy_utils.cpp:52-55 lr; the grids' row from their own Adam and schedule."""
        o = self.opt
        stepped = o.advance(self.iteration, skip)
        for i, k in enumerate(PARAM_GROUPS):
            self._set_row(i, o.lr[i], o.steps[k], o.cfg.beta1, o.cfg.beta2, k in stepped)
        G = self.grid_state
        if G is not None:
            lr, t = G.advance()
            self._set_row(len(PARAM_GROUPS), lr, t, G.beta1, G.beta2, True)
        self.dyn.copy_(self.dyn_host, non_blocking=True)
        o.lr[0] *= o.gamma

    def capture(self, camera, intrinsics, target, background=None, image_idx=None):
        """Sizes the capacity with one exact render, warms up and captures the graph(s).  camera, intrinsics: viewmat
        and K on this path, w2c and the camera position on the fastgs one."""
        self._set_inputs(camera, intrinsics, target, background)
        if self.grid_state is not None:
            self.grid_state.set_image(image_idx)
        if self.strategy is not None:
            self.sh_degree = self.strategy.sh_degree
        n = self._size_capacity()
        self.capacity = self.step.capacity
        self._warm_up_and_capture()
        return n

    def __call__(self, camera, intrinsics, target, background=None, image_idx=None):
        self._enter_iteration()
        if self.graph is None:
            self.capture(camera, intrinsics, target, background, image_idx)
        self.iteration += 1
        self._set_inputs(camera, intrinsics, target, background)
        if self.grid_state is not None:
            self.grid_state.set_image(image_idx)
        if self.strategy is None:
            self._set_scalars()
            self.graph.replay()
        else:
            self._replay()
        return self.loss

    def overflowed(self) -> bool:
        """True when the last iteration had more intersections than the captured buffers hold (re-capture then)."""
        return int(self.n_isects.item()) > self.capacity


class GraphedFastGsTrainStep(GraphedTrainStep):
    """GraphedTrainStep on the fastgs path: fastgs forward (capacity mode) -> background composite -> loss-and-gradient
    kernel -> fastgs backward -> Adam with device-side scalars, captured once and replayed.  The camera pose, camera
    position, background and target are static device buffers refreshed before each replay; the intrinsics and the image
    size are launch arguments and therefore fixed per captured graph (one graph per camera resolution)."""

    def __init__(self, params: dict, sh_degree: int, settings, cfg: AdamConfig | None = None, lambda_dssim: float = 0.2,
                 capacity_slack: float = 1.25, bilateral_grid: BilateralGrid | None = None, bilateral_grid_lr: float = 2e-3,
                 tv_loss_weight: float = 10.0, strategy: Strategy | None = None, sparsity: ADMMSparsity | None = None):
        super().__init__(params, sh_degree, settings.width, settings.height, cfg, lambda_dssim, capacity_slack,
                         bilateral_grid, bilateral_grid_lr, tv_loss_weight, strategy, sparsity)
        from . import fastgs as fg
        dev = self.dev
        self.static = {"w2c": torch.zeros((4, 4), device=dev), "campos": torch.zeros((3,), device=dev),
                       "background": torch.zeros((3,), device=dev), "target": torch.zeros((3, self.H, self.W), device=dev)}
        self.settings = dataclasses.replace(settings, cam_position=self.static["campos"])
        self.be = fg.default_backend()
        self.step = FastGsTrainStep(params, sh_degree, settings.width, settings.height, lambda_dssim, optimizer=None,
                                    backend=self.be, bilateral_grid=bilateral_grid, grid_state=self.grid_state)

    def _forward_backward(self):
        S, st = self.static, self.strategy
        return self.step._forward_backward(S["w2c"], self.settings, S["target"], S["background"],
                                           st.densification_info if st is not None else None)

    def _size_capacity(self) -> int:
        if self.strategy is not None:
            self.settings = dataclasses.replace(self.settings, active_sh_bases=(self.sh_degree + 1) ** 2)
        return self.step.size_capacity(self.static["w2c"], self.settings, self.slack)

    def _set_inputs(self, w2c, cam_position, target, background):
        S = self.static
        S["w2c"].copy_(w2c.reshape(4, 4), non_blocking=True)
        S["campos"].copy_(cam_position.reshape(3), non_blocking=True)
        S["target"].copy_(target.reshape(3, self.H, self.W), non_blocking=True)
        if background is not None:
            S["background"].copy_(background.reshape(3), non_blocking=True)
