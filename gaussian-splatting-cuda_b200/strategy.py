"""What the training steps ask of a densification strategy (mcmc.MCMC, adc.DefaultStrategy), so that they never ask
which one they hold:

  refine(iteration) -> tuple   the SH-degree bump and the iteration's densification, gradients untouched; returns the
                               Adam groups this iteration's step skips (all six when the tensors were replaced)
  replaced                     the last refine replaced the tensors: params[k] and the moments are new objects
  before_adam(lr)              what runs between the refine and Adam; lr is group 0's rate before this iteration's
                               scheduler step, a float or a device scalar
  post_backward(iteration)     the above in the reference's order; the skipped groups lose their gradient
  regularize()                 the regularisers' gradients into .grad
  sh_degree                    the active degree the step renders with
  densification_info           the statistics the fastgs backward accumulates into, or None"""
from __future__ import annotations

PARAM_GROUPS = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")  # order of strategy_utils.cpp:27-55


class Strategy:
    """The shared part of the protocol: a subclass has `params`, `optimizer`, `sh_degree`, `refine` and `regularize`."""

    replaced = False
    densification_info = None

    def before_adam(self, lr) -> None:
        pass

    def post_backward(self, iteration: int) -> tuple:
        """The refine, the skipped groups' gradients dropped (FusedAdam then leaves them and their step counts alone),
        then the pre-Adam hook at the optimizer's group-0 rate."""
        skip = self.refine(iteration)
        for k in skip:
            self.params[k].grad = None
        self.before_adam(self.optimizer.lr[0])
        return skip
