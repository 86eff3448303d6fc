"""CPU: the sparsifier's torch restatement (tests/sparsity_restatement.py) and the library's host-side schedule and
prune count (sparsity.py) on hand-derived cases: the schedule's edges, prune_z with ties and equal inputs, a zero
index, the float32 index near 2^24, and the loss and its gradient against float64 and finite differences."""
import importlib

import numpy as np
import pytest
import torch

import sparsity_restatement as R


@pytest.fixture(scope="module")
def sp(pkg):
    return importlib.import_module(pkg.__name__ + ".sparsity")


def test_schedule_edges(sp):
    start, steps, every = 30000, 15000, 50
    cfg = sp.SparsityConfig(sparsify_steps=steps, start_iteration=start, update_every=every)
    s = sp.ADMMSparsity.__new__(sp.ADMMSparsity)  # the predicates only: no device state
    s.cfg, s.done = cfg, False
    for it in (start - 1, start, start + 1, start + 50, start + 50 * 7, start + 51, start + steps - 50,
               start + steps - 1, start + steps, start + steps + 1):
        assert s.should_apply_loss(it) == R.should_apply_loss(it, start, steps), it
        assert s.should_update(it) == R.should_update(it, start, steps, every), it
        assert s.should_prune(it) == R.should_prune(it, start, steps), it
        assert s.post_backward_due(it) == R.post_backward_due(it, start), it
    assert not R.should_apply_loss(start - 1, start, steps) and R.should_apply_loss(start, start, steps)
    assert not R.should_update(start, start, steps, every)             # relative 0: no update
    assert R.should_update(start + 50, start, steps, every) and R.should_update(start + 100, start, steps, every)
    assert not R.should_update(start + 51, start, steps, every)
    assert not R.should_update(start + steps, start, steps, every)     # the prune iteration does not update
    assert not R.should_apply_loss(start + steps, start, steps) and R.should_prune(start + steps, start, steps)
    assert R.post_backward_due(start, start) and not R.post_backward_due(start + 1, start)  # base gets both
    s.done = True
    assert not s.should_apply_loss(start) and not s.should_prune(start + steps)


def test_short_schedule():
    start, steps = 20, 120
    upd = [it for it in range(1, 200) if R.should_update(it, start, steps, 50)]
    loss = [it for it in range(1, 200) if R.should_apply_loss(it, start, steps)]
    assert upd == [70, 120] and loss[0] == 20 and loss[-1] == 139
    assert [it for it in range(1, 200) if R.should_prune(it, start, steps)] == [140]


def test_prune_z_ties_and_equal_inputs():
    x = torch.tensor([0.3, 0.1, 0.2, 0.2, 0.2, 0.5, 0.4, 0.2, 0.9, 0.7])  # index (int)(0.6f * 10) = 6
    assert R.prune_index(0.6, 10) == 6
    # sorted: .1 .2 .2 .2 .2 .3 | .4 ...: the threshold is 0.3; every value <= 0.3 becomes 0
    z = R.prune_z(x, 0.6)
    assert torch.equal(z, torch.where(x > 0.3, x, torch.zeros_like(x)))
    # the threshold inside a run of ties: more than `index` zeros
    y = torch.tensor([0.2, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2, 0.9, 0.8, 0.1])
    zy = R.prune_z(y, 0.6)
    assert int((zy == 0).sum()) == 8 > R.prune_index(0.6, 10)
    e = torch.full((7,), 0.25)
    assert not bool(R.prune_z(e, 0.6).any())                         # all equal: everything is zeroed


def test_zero_index_prunes_nothing(sp):
    x = torch.tensor([0.3, 0.1])
    assert R.prune_index(0.4, 2) == 0 and sp.prune_count(0.4, 2) == 0
    assert torch.equal(R.prune_z(x, 0.4), torch.zeros(2))
    assert not bool(R.prune_mask(torch.logit(x), 0.4).any())
    z, u = R.initialize(torch.logit(x), 0.4)
    assert not bool(z.any()) and not bool(u.any())
    assert sp.prune_count(0.6, 1) == 0 and sp.prune_count(0.6, 4) == 2


@pytest.mark.parametrize("n", [2 ** 24 - 3, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 24 + 5, 2 ** 25 + 7, 50_000_011])
def test_float32_index_near_2_24(sp, n):
    want = int(np.float32(np.float32(0.6) * np.float32(n)))
    assert R.prune_index(0.6, n) == want == sp.prune_count(0.6, n)


def test_float32_index_differs_from_exact():
    diffs = [n for n in range(2 ** 24, 2 ** 24 + 64) if R.prune_index(0.6, n) != int(0.6 * n)]
    assert diffs, "the float32 product must differ from the exact one somewhere above 2^24"


def test_loss_and_gradient_against_float64_and_differences():
    g = torch.Generator().manual_seed(3)
    o = torch.randn(257, 1, generator=g)
    z, u = R.initialize(o, 0.6)
    z, u = R.update_state(o + 0.1 * torch.randn(257, 1, generator=g), z, u, 0.6)
    rho = 5e-4
    o32 = o.clone().requires_grad_(True)
    L = R.loss(o32, z, u, rho)
    L.backward()
    o64 = o.double().requires_grad_(True)
    s = torch.sigmoid(o64)
    L64 = 0.5 * rho * ((s - z.double() + u.double()) ** 2).sum()
    L64.backward()
    assert abs(float(L.detach()) - float(L64.detach())) <= 1e-5 * abs(float(L64.detach()))
    # s - z + u cancels where u has absorbed s - z: float32 error relative to the largest gradient
    scale = float(o64.grad.abs().max())
    assert torch.allclose(o32.grad.double(), o64.grad, rtol=1e-5, atol=1e-5 * scale)
    # analytic form of the gradient: rho (s - z + u) s (1 - s)
    sd = torch.sigmoid(o.double())
    assert torch.allclose(o64.grad, rho * (sd - z.double() + u.double()) * sd * (1 - sd), rtol=1e-12, atol=0)
    # central differences in float64
    h = 1e-6
    for i in (0, 17, 256):
        p, m = o.double().clone(), o.double().clone()
        p[i] += h
        m[i] -= h
        f = lambda t: 0.5 * rho * ((torch.sigmoid(t) - z.double() + u.double()) ** 2).sum()
        fd = float((f(p) - f(m)) / (2 * h))
        assert abs(fd - float(o64.grad[i])) <= 1e-5 * scale  # roundoff of the sum over all rows, over 2h


def test_update_and_prune_by_hand():
    o = torch.logit(torch.tensor([[0.9], [0.1], [0.5], [0.3], [0.2]]))
    z, u = R.initialize(o, 0.6)  # index 3: threshold the 3rd smallest (0.3)
    s = torch.sigmoid(o)
    assert torch.equal(z, torch.where(s > s[3], s, torch.zeros_like(s))) and not bool(u.any())
    z2, u2 = R.update_state(o, z, u.clone(), 0.6)
    assert torch.equal(u2, s - z2)
    mask = R.prune_mask(o, 0.6)
    assert mask.tolist() == [False, True, False, True, True]
    P = {k: torch.arange(5.0)[:, None] * (i + 1) for i, k in enumerate(R.GROUPS)}
    P2, _, _ = R.remove_gaussians(P, P, P, mask)
    assert P2["means"].flatten().tolist() == [0.0, 2.0]


def test_sparsity_needs_a_strategy(pkg):
    training = importlib.import_module(pkg.__name__ + ".training")
    with pytest.raises(ValueError, match="needs a strategy"):
        training._check_sparsity(object(), None)
    training._check_sparsity(None, None)
