"""Host-side mirror of the reference's training iteration around the hot path (SURVEY.md 8 f2 / f3):

  photometric_loss   trainer.cpp:103-126 (L1 + fused SSIM "valid") as one kernel that also returns dLoss/d(render)
  FusedAdam          src/training/optimizers/fused_adam.cpp:22-117 + strategy_utils.cpp:27-55 (per-group learning rates,
                     eps 1e-15, exponential decay of the position learning rate, shN frozen for the first 1000
                     iterations), all groups stepped by ONE kernel launch (gsb_adam_step)
  TrainStep          render (extended operator on the raw tensors) -> loss -> backward -> Adam [-> MCMC noise], with
                     the intersection buffer sized from a capacity so that the iteration has no host read-back
  strategy           optional MCMC densification (SURVEY.md 8 f6, mcmc.py): render -> loss -> backward -> regularisers
                     -> post_backward (SH bump, relocation / growth on refine iterations, noise) -> Adam (nothing to
                     step on a growth iteration) -> scheduler; or the default strategy (adc.py): the fastgs backward
                     accumulates the strategy's statistics -> post_backward (SH bump, duplicate / split / prune on
                     refine iterations, opacity reset) -> Adam (skipping the groups whose tensors were replaced or
                     reset) -> scheduler
  bilateral_grid     optional (SURVEY.md 8 f5, trainer.cpp:662-665,698-705,758-762): render -> slice through the
                     image's grid -> unclamped loss -> + weight * TV of all grids -> backward -> one Adam launch for the
                     Gaussians and the grids (lr from the warm-up/exponential schedule, eps 1e-15)
  sparsity           optional ADMM sparsification with a strategy (sparsity.py, trainer.cpp:173-247,707-784): after
                     the regularisers the sparsity loss's gradient; post_backward only up to the base iteration count;
                     after Adam the state update and, on the last iteration, the prune

Everything that computes lives behind the C ABI; this file only orders the calls, like the reference's trainer does."""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass, field

import torch

from . import _product_ns, load, rasterize_fused
from .adc import DefaultStrategy
from .bilateral import BilateralGrid, WarmupExponentialLR
from .mcmc import MCMC, growth_count
from .sparsity import ADMMSparsity


class _PhotometricLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renders, target, lambda_dssim):
        stats, v = _product_ns().photometric_loss_fused(renders.detach().contiguous(), target.contiguous(),
                                                        float(lambda_dssim), renders.requires_grad)
        ctx.save_for_backward(v)
        ctx.mark_non_differentiable(stats)
        return stats[0], stats

    @staticmethod
    def backward(ctx, g_loss, _g_stats):
        (v,) = ctx.saved_tensors
        return (v * g_loss if v.numel() else None), None, None


class _PhotometricLossUnclamped(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renders, target, lambda_dssim):
        stats, v = _product_ns().photometric_loss_fused_unclamped(renders.detach().contiguous(), target.contiguous(),
                                                                  float(lambda_dssim), renders.requires_grad)
        ctx.save_for_backward(v)
        ctx.mark_non_differentiable(stats)
        return stats[0], stats

    @staticmethod
    def backward(ctx, g_loss, _g_stats):
        (v,) = ctx.saved_tensors
        return (v * g_loss if v.numel() else None), None, None


def photometric_loss_unclamped(renders, target, lambda_dssim: float = 0.2):
    """photometric_loss on an image used as it is (no clamp, no clamp mask): the loss of a bilateral-grid output."""
    load()
    return _PhotometricLossUnclamped.apply(renders, target, lambda_dssim)


def photometric_loss(renders, target, lambda_dssim: float = 0.2):
    """(loss, stats) with stats = device tensor [loss, l1 mean, ssim mean].  renders [1,H,W,3] unclamped (the blend's
    output); target [3,H,W] (the reference's image layout) or [1,H,W,3]."""
    load()
    return _PhotometricLoss.apply(renders, target, lambda_dssim)


PARAM_GROUPS = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")  # order of strategy_utils.cpp:27-55


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

    def step(self, iteration: int, extra: tuple | None = None):
        """extra: one more group (param, grad, exp_avg, exp_avg_sq, lr, step count, (beta1, beta2, eps)), stepped by the
        same launch when its hyperparameters are the Gaussians' and by a second launch otherwise."""
        names, counts = [], []
        for k in PARAM_GROUPS:
            p = self.params[k]
            if p.grad is None or p.numel() == 0:
                continue
            self.steps[k] += 1
            if k == "shN" and iteration <= 1000:  # fused_adam.cpp:68-70: the step count still advances
                continue
            names.append(k)
            counts.append(self.steps[k])
        if names and extra is None:
            with torch.no_grad():
                _product_ns().fused_adam_step([self.params[k] for k in names], [self.params[k].grad for k in names],
                                              [self.exp_avg[k] for k in names], [self.exp_avg_sq[k] for k in names],
                                              [self.lr[PARAM_GROUPS.index(k)] for k in names], self.cfg.beta1,
                                              self.cfg.beta2, self.cfg.eps, counts)
        elif extra is not None:
            p, g, m, v, lr, t, hyper = extra
            c = self.cfg
            ns = _product_ns()
            with torch.no_grad():
                if hyper == (c.beta1, c.beta2, c.eps):
                    ns.fused_adam_step([self.params[k] for k in names] + [p], [self.params[k].grad for k in names] + [g],
                                       [self.exp_avg[k] for k in names] + [m], [self.exp_avg_sq[k] for k in names] + [v],
                                       [self.lr[PARAM_GROUPS.index(k)] for k in names] + [lr], c.beta1, c.beta2, c.eps,
                                       counts + [t])
                else:
                    if names:
                        ns.fused_adam_step([self.params[k] for k in names], [self.params[k].grad for k in names],
                                           [self.exp_avg[k] for k in names], [self.exp_avg_sq[k] for k in names],
                                           [self.lr[PARAM_GROUPS.index(k)] for k in names], c.beta1, c.beta2, c.eps, counts)
                    ns.fused_adam_step([p], [g], [m], [v], [lr], hyper[0], hyper[1], hyper[2], [t])
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

    def adam_group(self):
        """The grids' Adam group for this step; advances the schedule (bilateral_grid_scheduler_->step())."""
        self.steps += 1
        g = self.grid.grids
        group = (g.detach(), g.grad, self.exp_avg, self.exp_avg_sq, self.sched.lr, self.steps,
                 (self.beta1, self.beta2, self.eps))
        self.sched.step()
        return group


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


@dataclass
class TrainStep:
    """One training iteration on resident raw parameters: camera + target in, loss (device scalar) out."""
    params: dict
    sh_degree: int
    width: int
    height: int
    lambda_dssim: float = 0.2
    optimizer: FusedAdam | None = None
    mcmc_noise_lr: float = 0.0          # > 0: gsplat::add_noise every iteration (mcmc.cpp:349-367)
    capacity: int = 0                    # intersections the buffers are sized for; 0 = size exactly (one read-back)
    iteration: int = 0
    last: dict = field(default_factory=dict)
    bilateral_grid: BilateralGrid | None = None  # use_bilateral_grid: the iteration needs image_idx
    bilateral_grid_lr: float = 2e-3
    tv_loss_weight: float = 10.0                 # mcmc_optimization_params.json (default_optimization_params.json: 5)
    grid_state: _GridState | None = None         # created on first use
    strategy: MCMC | DefaultStrategy | None = None  # densification: owns params and the optimizer's moments
    sparsity: ADMMSparsity | None = None            # ADMM sparsification after the base iterations (needs a strategy)

    def __post_init__(self):
        _check_strategy(self.strategy, self.mcmc_noise_lr, self.params, self.optimizer, self.sh_degree)
        _check_sparsity(self.sparsity, self.strategy)

    def _grid(self) -> _GridState:
        if self.grid_state is None:
            its = self.optimizer.cfg.iterations if self.optimizer is not None else AdamConfig().iterations
            self.grid_state = _GridState(self.bilateral_grid, self.bilateral_grid_lr, self.tv_loss_weight, its)
        return self.grid_state

    def __call__(self, viewmat, K, target, background=None, image_idx=None):
        P = self.params
        self.iteration += 1
        if self.strategy is not None:
            self.sh_degree = self.strategy.sh_degree
        out = rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                              self.sh_degree, viewmat, K, self.width, self.height, bg_color=background,
                              isect_capacity=self.capacity)
        extra = None
        if self.bilateral_grid is None:
            loss, stats = photometric_loss(out.render_colors, target, self.lambda_dssim)
            loss.backward()
        else:
            G = self._grid()
            G.set_image(image_idx)
            tv, v_grids = G.tv()
            sliced = _SliceIntoGrad.apply(out.render_colors, G.grid.grids.detach(), G.idx, v_grids, False)
            loss, stats = photometric_loss_unclamped(sliced, target, self.lambda_dssim)
            loss.backward()
            G.grid.grids.grad = v_grids
            loss = loss.detach() + G.weight[0] * tv  # the trainer's loss_value includes the TV term
        reg, sp_loss = _post_backward(self.strategy, self.sparsity, self.iteration)
        if sp_loss is not None:
            loss = loss.detach() + sp_loss[0]
        if self.optimizer is not None:
            if self.bilateral_grid is not None:
                extra = self.grid_state.adam_group()
            self.optimizer.step(self.iteration, extra)
            if self.mcmc_noise_lr > 0.0:
                with torch.no_grad():
                    noise = torch.randn_like(P["means"])
                    _product_ns().add_noise(P["opacity_raw"].detach().reshape(-1), P["scaling_raw"].detach(),
                                            P["rotation_raw"].detach(), noise, P["means"].detach(),
                                            self.mcmc_noise_lr * self.optimizer.lr[0])
            self.optimizer.zero_grad()
        if self.bilateral_grid is not None:
            self.bilateral_grid.grids.grad = None
        if self.sparsity is not None:
            self.sparsity.after_step(self.strategy, self.iteration)
        self.last = {"n_isects": out.n_isects, "stats": stats, "reg": reg, "sparsity_loss": sp_loss}
        return loss

    def size_capacity(self, viewmat, K, target, background=None, slack: float = 1.25):
        """An exact (synchronising) render sizes the intersection capacity for the following steps."""
        with torch.no_grad():
            P = self.params
            out = rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                                  self.sh_degree, viewmat, K, self.width, self.height, bg_color=background)
            n = int(out.n_isects.item())
        self.capacity = int(n * slack) + 1024
        return n


def _check_strategy(strategy, mcmc_noise_lr: float, params=None, optimizer=None, sh_degree=None) -> None:
    """A strategy owns the parameter dict and the optimizer's moments: the step must use the same objects, and the
    degree it renders with is the strategy's active degree (SplatData's, which the strategy raises)."""
    if strategy is None:
        return
    if mcmc_noise_lr > 0.0:
        raise ValueError("mcmc_noise_lr and strategy both add noise: the strategy injects it before Adam, as the "
                         "reference does, so pass one of them")
    if params is not None and params is not strategy.params:
        raise ValueError("the step's params must be the strategy's params dict (growth replaces its tensors)")
    if optimizer is not None and optimizer is not strategy.optimizer:
        raise ValueError("the step's optimizer must be the strategy's optimizer (growth replaces its moments)")
    if sh_degree is not None and int(sh_degree) != strategy.sh_degree:
        raise ValueError(f"sh_degree {sh_degree} differs from the strategy's active degree {strategy.sh_degree}: "
                         f"pass {type(strategy).__name__}(..., sh_degree=...) or the step the same degree")


def _strategy_post_backward(strategy, iteration: int):
    """Regularisers into the gradients, then the strategy's post_backward (trainer.cpp:668-756): on a growth iteration
    the parameters become new leaves without gradients, so the following Adam step skips them (the default strategy
    also drops the opacity gradient after a reset)."""
    if strategy is None:
        return None
    with torch.no_grad():
        reg = strategy.regularize()
        strategy.post_backward(iteration)
    return reg


def _check_sparsity(sparsity, strategy) -> None:
    if sparsity is not None and strategy is None:
        raise ValueError("sparsity needs a strategy: the final prune removes rows from the strategy's tensors, and "
                         "the strategy's post_backward stops after the base iterations")


def _post_backward(strategy, sparsity, iteration: int):
    """(regulariser losses, sparsity loss): the regularisers, the sparsity loss's gradient when it applies
    (trainer.cpp:707-714), then the strategy's post_backward up to the base iteration count (trainer.cpp:745-754)."""
    if sparsity is None:
        return _strategy_post_backward(strategy, iteration), None
    with torch.no_grad():
        reg = strategy.regularize()
        sp = sparsity.loss_step(strategy.params["opacity_raw"], iteration)
        if sparsity.post_backward_due(iteration):
            strategy.post_backward(iteration)
    return reg, sp


def _densification_info(strategy):
    """The default strategy's statistics tensor (empty after stop_refine); None for MCMC or no strategy."""
    return strategy.densification_info if isinstance(strategy, DefaultStrategy) else None


class GraphedTrainStep:
    """The whole iteration -- extended render operator, loss-and-gradient kernel, blend backward, fused back kernel, Adam --
    captured ONCE in a CUDA graph and replayed: one graph launch per iteration instead of ~25 kernel launches and their
    torch bookkeeping.  Possible because nothing inside the iteration needs a host-side value: the intersection buffers
    are sized from a capacity (the count stays on the device, `overflowed()` checks it afterwards) and Adam's
    step-dependent scalars (learning rates, bias corrections, the shN freeze of the first 1000 iterations) are read from a
    small device tensor that is refreshed before every replay.

    Per iteration the host copies the camera (viewmat, K), the background and the target image into static device buffers
    (pinned -> device, on the replay stream) and reads the loss back when it wants to."""

    def __init__(self, params: dict, sh_degree: int, width: int, height: int, cfg: AdamConfig | None = None,
                 lambda_dssim: float = 0.2, capacity_slack: float = 1.25, bilateral_grid: BilateralGrid | None = None,
                 bilateral_grid_lr: float = 2e-3, tv_loss_weight: float = 10.0,
                 strategy: MCMC | DefaultStrategy | None = None, sparsity: ADMMSparsity | None = None):
        load()
        _check_strategy(strategy, 0.0, params, None, sh_degree)
        _check_sparsity(sparsity, strategy)
        self.sparsity = sparsity
        self.sparsity_in_graph = False  # the captured part A adds the sparsity loss (part B then has no MCMC noise)
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
        n_rows = len(PARAM_GROUPS) + (1 if bilateral_grid is not None else 0)
        self.dyn = torch.zeros((n_rows, 4), device=dev)
        self.dyn_host = torch.zeros((n_rows, 4)).pin_memory()
        self.graph = None
        self.loss = None
        self.stats = None
        self.n_isects = None
        self.capacity = 0
        self.iteration = 0

    def _part_a(self):
        """render -> loss -> backward [-> the strategy's regularisers]: (loss, stats, count, grid gradient or None)"""
        P, S = self.params, self.static
        out = rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                              self.sh_degree, S["viewmat"], S["K"], self.W, self.H, bg_color=S["background"],
                              isect_capacity=self.capacity)
        if self.grid_state is None:
            loss, stats = photometric_loss(out.render_colors, S["target"], self.lambda_dssim)
            loss.backward()
            return self._regularize(loss), stats, out.n_isects, None
        G = self.grid_state
        tv, v_grids = G.tv()
        sliced = _SliceIntoGrad.apply(out.render_colors, G.grid.grids.detach(), G.idx, v_grids, False)
        loss, stats = photometric_loss_unclamped(sliced, S["target"], self.lambda_dssim)
        loss.backward()
        return self._regularize(loss.detach() + G.weight[0] * tv), stats, out.n_isects, v_grids

    def _regularize(self, loss):
        """The strategy's regularisers, then, in the sparsity phase, the sparsity loss (rho read on the device: zero
        on the prune iteration).  Returns the iteration's loss."""
        if self.strategy is not None:
            with torch.no_grad():
                self.strategy.regularize()
                if self.sparsity_in_graph:
                    return loss.detach() + self.sparsity.add_loss_gradient(self.params["opacity_raw"])[0]
        return loss

    def _part_b(self, v_grids):
        """[MCMC's noise at the means group's rate, read from `dyn` ->] Adam.  In the sparsity phase the strategy's
        post_backward, and with it the noise, stops: part B is Adam only."""
        if isinstance(self.strategy, MCMC) and not self.sparsity_in_graph:
            self.strategy.inject_noise(self.dyn[0, 0:1])
        self._adam(v_grids)

    def _body(self):
        loss, stats, n, v_grids = self._part_a()
        self._part_b(v_grids)
        return loss, stats, n

    def _warm_up_and_capture(self):
        """Warm-up iterations with every Adam group disabled and a zero noise rate (`dyn` is zero: nothing moves),
        then the capture.  Without a strategy the iteration is one graph.  With one it is two graphs -- (render, loss,
        backward, regularisers) and (noise, Adam) -- so that a refine can run eagerly between them, and the warm-up's
        random draws are undone so that the replays draw what an eager run would.  The default strategy's statistics,
        which the warm-up's backward passes accumulate into, are restored too."""
        self.dyn.zero_()
        sp = self.sparsity
        self.sparsity_in_graph = sp is not None and sp.initialized and not sp.done
        rng = torch.cuda.get_rng_state(self.dev) if self.strategy is not None else None
        info = _densification_info(self.strategy)
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
        if self.strategy is None:
            with torch.cuda.graph(self.graph):
                self.loss, self.stats, self.n_isects = self._body()
            return
        with torch.cuda.graph(self.graph):
            self.loss, self.stats, self.n_isects, v_grids = self._part_a()
        self.graph_b = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_b, pool=self.graph.pool()):
            self._part_b(v_grids)

    def _replay(self):
        """One iteration from the captured graph(s).  With a strategy: part A, then -- on a refine iteration -- the
        refine eagerly, then part B (noise, Adam).  A growth step replaces the parameters, so its noise runs eagerly on
        the new rows, Adam has nothing to step (as FusedAdam after the reference's torch::cat) and the next call
        re-captures; an SH-degree bump re-captures too.  A relocation-only refine works in place: no re-capture."""
        st = self.strategy
        if st is None:
            self.graph.replay()
            return
        sp = self.sparsity
        post = sp is None or sp.post_backward_due(self.iteration)  # no post_backward after the base iterations
        if isinstance(st, DefaultStrategy):
            self._replay_default(st, post)
        else:
            self._replay_mcmc(st, post)
        if sp is not None and sp.after_step(st, self.iteration):  # the prune replaced the tensors
            self.graph = None

    def _replay_mcmc(self, st: MCMC, post: bool):
        lr0 = self.opt.lr[0]  # the rate before this iteration's scheduler step
        grows = post and st.is_refining(self.iteration) and growth_count(st.n, st.capacity) > 0
        self._set_scalars(skip_adam=grows)
        degree = st.sh_degree
        self.graph.replay()
        grew = st.refine(self.iteration) if post else False
        if grew:
            st.inject_noise(lr0)
        else:
            if post and self.sparsity_in_graph:  # the base iteration: its noise is no longer in part B
                st.inject_noise(lr0)
            self.graph_b.replay()
        if grew or st.sh_degree != degree:
            self.graph = None

    def _replay_default(self, st: DefaultStrategy, post: bool = True):
        """Part A, then the eager post_backward, then the Adam scalars with the skipped groups disabled (their step
        counts held), then part B.  A refine that replaced the tensors has nothing left to step: part B is not replayed
        and the next call re-captures.  So does an SH-degree bump, and stop_refine, where the statistics the captured
        backward writes go away.  A reset or a refine that changed nothing works in place and keeps the graphs."""
        degree, info = st.sh_degree, st.densification_info
        self.graph.replay()
        skip = st.refine(self.iteration) if post else ()
        replaced = post and st.replaced
        self._set_scalars(skip_groups=skip)
        if not replaced:
            self.graph_b.replay()
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

    def _adam(self, v_grids=None):
        """One launch for the Gaussians' groups (and the grids' after them), scalars from `dyn`."""
        P = self.params
        names = [k for k in PARAM_GROUPS if P[k].numel() > 0]
        with torch.no_grad():
            if v_grids is None:
                _product_ns().fused_adam_step_dynamic([P[k] for k in names], [P[k].grad for k in names],
                                                      [self.opt.exp_avg[k] for k in names],
                                                      [self.opt.exp_avg_sq[k] for k in names],
                                                      self.dyn[[PARAM_GROUPS.index(k) for k in names]].contiguous()
                                                      if len(names) != len(PARAM_GROUPS) else self.dyn,
                                                      self.opt.cfg.beta1, self.opt.cfg.beta2, self.opt.cfg.eps)
                return
            G, c, ns = self.grid_state, self.opt.cfg, _product_ns()
            rows = [PARAM_GROUPS.index(k) for k in names]
            if (G.beta1, G.beta2, G.eps) == (c.beta1, c.beta2, c.eps):  # one launch for all groups
                rows.append(len(PARAM_GROUPS))
                ns.fused_adam_step_dynamic([P[k] for k in names] + [G.grid.grids.detach()],
                                           [P[k].grad for k in names] + [v_grids],
                                           [self.opt.exp_avg[k] for k in names] + [G.exp_avg],
                                           [self.opt.exp_avg_sq[k] for k in names] + [G.exp_avg_sq],
                                           self.dyn[rows].contiguous() if len(rows) != self.dyn.shape[0] else self.dyn,
                                           c.beta1, c.beta2, c.eps)
                return
            ns.fused_adam_step_dynamic([P[k] for k in names], [P[k].grad for k in names],
                                       [self.opt.exp_avg[k] for k in names], [self.opt.exp_avg_sq[k] for k in names],
                                       self.dyn[rows].contiguous(), c.beta1, c.beta2, c.eps)
            ns.fused_adam_step_dynamic([G.grid.grids.detach()], [v_grids], [G.exp_avg], [G.exp_avg_sq],
                                       self.dyn[len(PARAM_GROUPS):].contiguous(), G.beta1, G.beta2, G.eps)

    def _set_inputs(self, viewmat, K, target, background):
        S = self.static
        S["viewmat"].copy_(viewmat.reshape(1, 4, 4), non_blocking=True)
        S["K"].copy_(K.reshape(1, 3, 3), non_blocking=True)
        S["target"].copy_(target.reshape(3, self.H, self.W), non_blocking=True)
        if background is not None:
            S["background"].copy_(background.reshape(1, 3), non_blocking=True)

    def _set_scalars(self, skip_adam: bool = False, skip_groups: tuple = ()):
        """fused_adam.cpp:61-81 on the host: step counts, bias corrections, the shN freeze; strategy_utils.cpp:52-55 lr.
        skip_adam: an iteration whose Adam step is skipped keeps the step counts (the learning rate still decays).
        skip_groups: those groups are disabled and keep their step counts (a group without a gradient in FusedAdam)."""
        o = self.opt
        for i, k in enumerate(PARAM_GROUPS):
            skipped = skip_adam or k in skip_groups
            o.steps[k] += 0 if skipped else 1
            t = o.steps[k]
            enabled = 0.0 if (k == "shN" and self.iteration <= 1000) or k in skip_groups else 1.0
            self.dyn_host[i, 0] = o.lr[i]
            self.dyn_host[i, 1] = 1.0 / (1.0 - o.cfg.beta1 ** t)
            self.dyn_host[i, 2] = 1.0 / math.sqrt(1.0 - o.cfg.beta2 ** t)
            self.dyn_host[i, 3] = enabled
        if self.grid_state is not None:  # the grids' group: torch.optim.Adam's bias corrections, the scheduled lr
            G, i = self.grid_state, len(PARAM_GROUPS)
            G.steps += 1
            self.dyn_host[i, 0] = G.sched.lr
            self.dyn_host[i, 1] = 1.0 / (1.0 - G.beta1 ** G.steps)
            self.dyn_host[i, 2] = 1.0 / math.sqrt(1.0 - G.beta2 ** G.steps)
            self.dyn_host[i, 3] = 1.0
            G.sched.step()
        self.dyn.copy_(self.dyn_host, non_blocking=True)
        o.lr[0] *= o.gamma

    def capture(self, viewmat, K, target, background=None, image_idx=None):
        """Sizes the intersection capacity with one exact render, warms up and captures the graph."""
        if self.strategy is not None:
            self.sh_degree = self.strategy.sh_degree
        self._set_inputs(viewmat, K, target, background)
        if self.grid_state is not None:
            self.grid_state.set_image(image_idx)
        with torch.no_grad():
            P, S = self.params, self.static
            out = rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                                  self.sh_degree, S["viewmat"], S["K"], self.W, self.H, bg_color=S["background"])
            n = int(out.n_isects.item())
        self.capacity = int(n * self.slack) + 1024
        self._warm_up_and_capture()
        return n

    def __call__(self, viewmat, K, target, background=None, image_idx=None):
        self._enter_iteration()
        if self.graph is None:
            self.capture(viewmat, K, target, background, image_idx)
        self.iteration += 1
        self._set_inputs(viewmat, K, target, background)
        if self.grid_state is not None:
            self.grid_state.set_image(image_idx)
        if self.strategy is None:
            self._set_scalars()
        self._replay()
        return self.loss

    def overflowed(self) -> bool:
        """True when the last iteration had more intersections than the captured buffers hold (re-capture then)."""
        return int(self.n_isects.item()) > self.capacity


@dataclass
class FastGsTrainStep:
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
    index_on_device: bool = False                # the graphed wrapper refreshes grid_state.idx itself before each replay
    strategy: MCMC | DefaultStrategy | None = None  # densification: owns params and the optimizer's moments
    sparsity: ADMMSparsity | None = None            # ADMM sparsification after the base iterations (needs a strategy)

    def __post_init__(self):
        _check_strategy(self.strategy, 0.0, self.params, self.optimizer, self.sh_degree)
        _check_sparsity(self.sparsity, self.strategy)

    def _grid(self) -> _GridState:
        if self.grid_state is None:
            its = self.optimizer.cfg.iterations if self.optimizer is not None else AdamConfig().iterations
            self.grid_state = _GridState(self.bilateral_grid, self.bilateral_grid_lr, self.tv_loss_weight, its)
        return self.grid_state

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

    def __call__(self, w2c, settings, target, background=None, densification_info=None, image_idx=None):
        from . import fastgs as fg
        be = self.backend or fg.default_backend()
        P = self.params
        self.iteration += 1
        if self.strategy is not None:
            self.sh_degree = self.strategy.sh_degree
            settings = dataclasses.replace(settings, active_sh_bases=(self.sh_degree + 1) ** 2)
        if isinstance(self.strategy, DefaultStrategy):  # the backward accumulates the strategy's statistics
            if densification_info is not None:
                raise ValueError("the default strategy owns densification_info: do not pass it as well")
            densification_info = self.strategy.densification_info
        G = None
        if self.bilateral_grid is not None:
            G = self._grid()
            if not self.index_on_device:
                G.set_image(image_idx)
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
        reg, sp_loss = _post_backward(self.strategy, self.sparsity, self.iteration)
        if self.optimizer is not None:
            self.optimizer.step(self.iteration, G.adam_group() if G is not None else None)
            self.optimizer.zero_grad()
            if G is not None:
                G.grid.grids.grad = None
        if self.sparsity is not None:
            self.sparsity.after_step(self.strategy, self.iteration)
        # capacity mode: the count is a device tensor (compare it with the capacity when convenient)
        self.last = {"n_instances": ctx.get("n_instances_dev", int(ctx["ints"][1])), "stats": stats, "reg": reg,
                     "sparsity_loss": sp_loss}
        loss = stats[0] if G is None else stats[0] + G.weight[0] * tv
        return loss if sp_loss is None else loss + sp_loss[0]


class GraphedFastGsTrainStep(GraphedTrainStep):
    """GraphedTrainStep on the fastgs path: fastgs forward (capacity mode) -> background composite -> loss-and-gradient
    kernel -> fastgs backward -> Adam with device-side scalars, captured once and replayed.  The camera pose, camera
    position, background and target are static device buffers refreshed before each replay; the intrinsics and the image
    size are launch arguments and therefore fixed per captured graph (one graph per camera resolution)."""

    def __init__(self, params: dict, sh_degree: int, settings, cfg: AdamConfig | None = None, lambda_dssim: float = 0.2,
                 capacity_slack: float = 1.25, bilateral_grid: BilateralGrid | None = None, bilateral_grid_lr: float = 2e-3,
                 tv_loss_weight: float = 10.0, strategy: MCMC | DefaultStrategy | None = None,
                 sparsity: ADMMSparsity | None = None):
        super().__init__(params, sh_degree, settings.width, settings.height, cfg, lambda_dssim, capacity_slack,
                         bilateral_grid, bilateral_grid_lr, tv_loss_weight, strategy, sparsity)
        from . import fastgs as fg
        dev = self.dev
        self.static = {"w2c": torch.zeros((4, 4), device=dev), "campos": torch.zeros((3,), device=dev),
                       "background": torch.zeros((3,), device=dev), "target": torch.zeros((3, self.H, self.W), device=dev)}
        self.settings = fg.FastGSSettings(cam_position=self.static["campos"], active_sh_bases=settings.active_sh_bases,
                                          width=settings.width, height=settings.height, focal_x=settings.focal_x,
                                          focal_y=settings.focal_y, center_x=settings.center_x, center_y=settings.center_y,
                                          near_plane=settings.near_plane, far_plane=settings.far_plane)
        self.be = fg.default_backend()
        self.step = FastGsTrainStep(params, sh_degree, settings.width, settings.height, lambda_dssim, optimizer=None,
                                    backend=self.be, bilateral_grid=bilateral_grid, grid_state=self.grid_state,
                                    index_on_device=True)

    def _part_a(self):
        S = self.static
        self.step.capacity = self.capacity
        loss = self.step(S["w2c"], self.settings, S["target"], S["background"],
                         densification_info=_densification_info(self.strategy))
        loss = self._regularize(loss)
        return (loss, self.step.last["stats"], self.step.last["n_instances"],
                self.grid_state.grid.grids.grad if self.grid_state is not None else None)

    def _set_inputs(self, w2c, cam_position, target, background):
        S = self.static
        S["w2c"].copy_(w2c.reshape(4, 4), non_blocking=True)
        S["campos"].copy_(cam_position.reshape(3), non_blocking=True)
        S["target"].copy_(target.reshape(3, self.H, self.W), non_blocking=True)
        if background is not None:
            S["background"].copy_(background.reshape(3), non_blocking=True)

    def capture(self, w2c, cam_position, target, background=None, image_idx=None):
        self._set_inputs(w2c, cam_position, target, background)
        if self.grid_state is not None:
            self.grid_state.set_image(image_idx)
        if self.strategy is not None:
            self.sh_degree = self.strategy.sh_degree
            self.settings = dataclasses.replace(self.settings, active_sh_bases=(self.sh_degree + 1) ** 2)
        self.step.capacity = 0
        n = self.step.size_capacity(self.static["w2c"], self.settings, self.slack)
        self.capacity = self.step.capacity
        self._warm_up_and_capture()
        return n

    def __call__(self, w2c, cam_position, target, background=None, image_idx=None):
        self._enter_iteration()
        if self.graph is None:
            self.capture(w2c, cam_position, target, background, image_idx)
        self.iteration += 1
        self._set_inputs(w2c, cam_position, target, background)
        if self.grid_state is not None:
            self.grid_state.set_image(image_idx)
        if self.strategy is None:
            self._set_scalars()
        self._replay()
        return self.loss
