"""GPU: the MCMC refine of this library against the restatement of mcmc.cpp driven by the REFERENCE's own
gsplat::relocation kernel (oracle/_ref/libgsplat_ref.so, built by oracle/build_ref.py where the reference's sources are
present; skipped otherwise).  Injected draws with duplicates, SH degrees 0 and 3, relocation and growth."""
import importlib

import pytest
import torch

import mcmc_restatement as R
from oracle import ref_ops
from test_gpu_mcmc import _lists, _params

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_ops.available(), reason="oracle/_ref/libgsplat_ref.so not built")]


def _ref_relocation(op, sc, ratios, binoms, n_max):
    return ref_ops._ns().relocation(op, sc, ratios, binoms.to(op.device), n_max)


def _close(got, want):
    # the reference's kernel is built with --use_fast_math and sums the alternating binomial series in another order;
    # at ratios near n_max the float32 series cancels terms up to C(50, 25) ~ 1.3e14, so the two differ in the fourth
    # digit of the scale factor there
    return torch.allclose(got, want, rtol=1e-4, atol=2e-4)


@pytest.mark.parametrize("deg", [0, 3])
def test_relocate_matches_reference_relocation(native, cuda_device, deg):
    mc = importlib.import_module(native.__name__ + ".mcmc")
    N, K = 30_000, (deg + 1) ** 2 - 1
    P, M1, M2 = _params(N, K, cuda_device, seed=30 + deg, dead_frac=0.05)
    dead, n_dead, _ = torch.ops.gsplat_b200.mcmc_dead(P["opacity_raw"], P["rotation_raw"], 0.005)
    n = int(n_dead.item())
    alive = (~R.dead_mask(P, 0.005)).nonzero().squeeze(-1)
    g = torch.Generator(device=cuda_device).manual_seed(deg)
    samples = alive[torch.randint(0, 80, (n,), device=cuda_device, generator=g)]
    samples[:70] = alive[5]  # ratio clamped to 51
    Q = {k: v.clone() for k, v in P.items()}
    Q1, Q2 = {k: v.clone() for k, v in M1.items()}, {k: v.clone() for k, v in M2.items()}
    b = mc.binomial_table().to(cuda_device)
    s32 = torch.zeros(N, dtype=torch.int32, device=cuda_device)
    s32[:n] = samples.int()
    torch.ops.gsplat_b200.mcmc_relocate(*_lists(P, M1, M2), s32, dead, n_dead, b, 0.005)
    R.relocate_gs(Q, Q1, Q2, samples, _ref_relocation, b, 0.005)
    for k in R.GROUPS:
        if k in ("opacity_raw", "scaling_raw"):
            assert _close(P[k], Q[k]), (k, (P[k] - Q[k]).abs().max().item())
        else:
            assert torch.equal(P[k], Q[k]), k
        assert torch.equal(M1[k], Q1[k]) and torch.equal(M2[k], Q2[k]), k


@pytest.mark.parametrize("deg", [0, 3])
def test_grow_matches_reference_relocation(native, cuda_device, deg):
    mc = importlib.import_module(native.__name__ + ".mcmc")
    N, K = 30_000, (deg + 1) ** 2 - 1
    P, M1, M2 = _params(N, K, cuda_device, seed=40 + deg)
    n_new = R.growth_count(N, 10 ** 9)
    g = torch.Generator(device=cuda_device).manual_seed(deg)
    samples = torch.randint(0, 300, (n_new,), device=cuda_device, generator=g)
    cap = N + n_new
    store = {k: torch.zeros((cap,) + tuple(v.shape[1:]), device=cuda_device) for k, v in P.items()}
    s1, s2 = {k: torch.zeros_like(store[k]) for k in P}, {k: torch.zeros_like(store[k]) for k in P}
    for k in P:
        store[k][:N], s1[k][:N], s2[k][:N] = P[k], M1[k], M2[k]
    b = mc.binomial_table().to(cuda_device)
    torch.ops.gsplat_b200.mcmc_grow(*_lists(store, s1, s2), N, samples.int(), b, 0.005)
    Q, Q1, Q2 = R.add_new_gs({k: v.clone() for k, v in P.items()}, M1, M2, samples, _ref_relocation, b, 0.005)
    for k in R.GROUPS:
        if k in ("opacity_raw", "scaling_raw"):
            assert _close(store[k], Q[k]), (k, (store[k] - Q[k]).abs().max().item())
        else:
            assert torch.equal(store[k], Q[k]), k
        assert torch.equal(s1[k], Q1[k]) and torch.equal(s2[k], Q2[k]), k
