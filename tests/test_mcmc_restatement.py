"""CPU: the MCMC restatement (tests/mcmc_restatement.py) against hand-derived cases, the strategy's host-side pieces
(binomial table, growth count), and the C-ABI entry points of the MCMC refine (argument validation, symbols).
No GPU: relocation is the CPU oracle's."""
import ctypes as C
import importlib
import os

import numpy as np
import pytest
import torch

import mcmc_restatement as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def mc(pkg):
    """mcmc.py: its host-side helpers need no native library."""
    return importlib.import_module(pkg.__name__ + ".mcmc")


@pytest.fixture(scope="module")
def relocation(orc):
    def f(op, sc, ratios, binoms, n_max):
        o, s = orc.relocation(op.numpy(), sc.numpy(), ratios.numpy(), binoms.numpy(), n_max)
        return torch.from_numpy(np.asarray(o, np.float32)), torch.from_numpy(np.asarray(s, np.float32))
    return f


def _scene(N, K=3, seed=0, n_dead=0):
    g = torch.Generator().manual_seed(seed)
    P = {"means": torch.randn(N, 3, generator=g), "sh0": torch.randn(N, 1, 3, generator=g),
         "shN": torch.randn(N, K, 3, generator=g), "scaling_raw": torch.randn(N, 3, generator=g) - 3,
         "rotation_raw": torch.randn(N, 4, generator=g), "opacity_raw": torch.randn(N, 1, generator=g)}
    if n_dead:
        P["opacity_raw"][torch.randperm(N, generator=g)[:n_dead]] = -8.0  # sigmoid = 3.4e-4 < 0.005
    M1 = {k: torch.randn(v.shape, generator=g) for k, v in P.items()}
    M2 = {k: torch.rand(v.shape, generator=g) for k, v in P.items()}
    return P, M1, M2


def test_binomial_table_is_exact(mc):
    b = mc.binomial_table().numpy().astype(np.float64)
    ex = R.binoms_exact()
    # the reference multiplies float quotients (n-i)/(i+1), so entries carry the rounding of up to 25 float products
    assert np.array_equal(b == 0, ex == 0) and np.array_equal(b[:, 0], ex[:, 0]) and np.array_equal(b[:, 1], ex[:, 1])
    assert np.all(np.abs(b - ex) <= 1e-5 * ex)


def test_ratio_one_is_the_identity(mc, relocation):
    """One copy: o' = 1 - (1 - o) and the scale factor o / o' -- both the identity up to float rounding."""
    b = mc.binomial_table()
    op = torch.linspace(0.01, 0.99, 97)
    sc = torch.rand(97, 3) + 0.1
    o, s = relocation(op, sc, torch.ones(97, dtype=torch.int32), b, 51)
    assert torch.allclose(o, op, rtol=0, atol=1e-7)
    assert torch.allclose(s, sc, rtol=1e-5, atol=0)  # o / (1 - (1 - o)): one rounding of 1 - o, relative to o >= 0.01


def test_relocate_duplicates_and_moments(mc, relocation):
    """Three dead rows filled from one alive row drawn three times: ratio 4 for it, all copies equal, the sampled row
    carries the same values, its moments are zeroed and the dead rows keep theirs."""
    P, M1, M2 = _scene(12, seed=1)
    P["opacity_raw"][[2, 5, 9]] = -8.0
    b = mc.binomial_table()
    before = {k: v.clone() for k, v in P.items()}
    m1_dead = {k: v[[2, 5, 9]].clone() for k, v in M1.items()}
    n = R.relocate_gs(P, M1, M2, torch.tensor([7, 7, 7]), relocation, b, 0.005)
    assert n == 3
    o, s = relocation(torch.sigmoid(before["opacity_raw"][7]), torch.exp(before["scaling_raw"][7:8]),
                      torch.tensor([4], dtype=torch.int32), b, 51)
    assert torch.equal(P["opacity_raw"][7], torch.logit(torch.clamp(o, 0.005, 1 - 1e-7)))
    assert torch.equal(P["scaling_raw"][7], torch.log(s[0]))
    for k in R.GROUPS:
        for d in (2, 5, 9):
            assert torch.equal(P[k][d], P[k][7]), k
        assert torch.equal(M1[k][7], torch.zeros_like(M1[k][7])) and torch.equal(M2[k][7], torch.zeros_like(M2[k][7]))
        assert torch.equal(M1[k][[2, 5, 9]], m1_dead[k]), k
        untouched = [i for i in range(12) if i not in (2, 5, 7, 9)]
        assert torch.equal(P[k][untouched], before[k][untouched]), k


def test_relocate_nothing_without_dead_or_alive(mc, relocation):
    b = mc.binomial_table()
    P, M1, M2 = _scene(8, seed=2)
    P["opacity_raw"][:] = 3.0
    assert R.relocate_gs(P, M1, M2, torch.tensor([], dtype=torch.long), relocation, b, 0.005) == 0
    P["opacity_raw"][:] = -9.0
    before = {k: v.clone() for k, v in P.items()}
    assert R.relocate_gs(P, M1, M2, torch.zeros(8, dtype=torch.long), relocation, b, 0.005) == 0
    assert all(torch.equal(P[k], before[k]) for k in R.GROUPS)


def test_grow_appends_zero_moments_and_keeps_sampled_moments(mc, relocation):
    b = mc.binomial_table()
    P, M1, M2 = _scene(10, seed=3)
    m1_before = {k: v.clone() for k, v in M1.items()}
    nP, nM1, nM2 = R.add_new_gs(P, M1, M2, torch.tensor([4, 4, 1]), relocation, b, 0.005)
    assert nP["means"].shape[0] == 13
    for k in R.GROUPS:
        assert torch.equal(nP[k][10], nP[k][4]) and torch.equal(nP[k][11], nP[k][4]) and torch.equal(nP[k][12], nP[k][1])
        assert not nM1[k][10:].any() and not nM2[k][10:].any()
        assert torch.equal(nM1[k][:10], m1_before[k]), k


@pytest.mark.parametrize("n,cap,want", [(100, 1000, 4), (1000, 1049, 49), (1000, 1050, 50), (1000, 1000, 0),
                                        (19, 100, 0), (20, 100, 1), (16777216, 10 ** 9, 838860),
                                        (16777217, 10 ** 9, 838859), (6000000, 6000000, 0), (5800000, 6000000, 200000)])
def test_growth_count(mc, n, cap, want):
    """(int)(1.05f * N) - N clamped to the cap: 1.05f * 100 is 104.99999, and above 2^24 N itself rounds."""
    assert R.growth_count(n, cap) == want
    assert mc.growth_count(n, cap) == want


def test_strategy_schedule(mc):
    m = mc
    c = m.MCMCConfig()
    assert (c.refine_every, c.start_refine, c.stop_refine, c.min_opacity, c.max_cap) == (100, 500, 25000, 0.005, 1000000)
    assert (c.scale_reg, c.opacity_reg, c.noise_lr, c.sh_degree_interval) == (0.01, 0.01, 5e5, 1000)
    s = R.Strategy.__new__(R.Strategy)
    s.cfg = c
    ref = [it for it in range(0, 26000) if s.is_refining(it)]
    assert ref[0] == 600 and ref[-1] == 24900 and len(ref) == 244


# ---- C ABI ---------------------------------------------------------------------------------------------------------
OK, E_INVALID, E_WORKSPACE = 0, -1, -3
_buf = np.zeros(1 << 16, np.uint8)
_aligned = (_buf.ctypes.data + 255) // 256 * 256
PTR = C.c_void_p(_aligned)
NULL = C.c_void_p(None)
u32, f32, i32, sz = C.c_uint32, C.c_float, C.c_int32, C.c_size_t


class GsbPhilox(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("offset", C.c_uint64), ("seed_ptr", C.c_void_p), ("offset_ptr", C.c_void_p),
                ("offset_intragraph", C.c_uint64)]


class GsbMcmcRows(C.Structure):
    _fields_ = [("means", C.c_void_p), ("sh0", C.c_void_p), ("shN", C.c_void_p), ("scaling_raw", C.c_void_p),
                ("rotation_raw", C.c_void_p), ("opacity_raw", C.c_void_p), ("shN_rows", C.c_uint32),
                ("exp_avg", C.c_void_p * 6), ("exp_avg_sq", C.c_void_p * 6)]


@pytest.fixture(scope="module")
def lib(pkg):
    path = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsb200.so")
    if not os.path.exists(path):
        pkg.build()
    L = C.CDLL(path)
    L.gsb_mcmc_workspace.restype = C.c_size_t
    return L


def test_mcmc_symbols(lib):
    for n in ("gsb_mcmc_workspace", "gsb_mcmc_dead", "gsb_mcmc_sample", "gsb_mcmc_apply", "gsb_mcmc_add_noise",
              "gsb_mcmc_regularize"):
        assert hasattr(lib, n), n


def test_mcmc_workspace_grows_with_n(lib):
    a, b = lib.gsb_mcmc_workspace(u32(1000)), lib.gsb_mcmc_workspace(u32(2000))
    assert b - a == 8000 and a >= 8000


def test_mcmc_validation(lib):
    ws = lib.gsb_mcmc_workspace(u32(4))
    # N == 0: nothing to do
    assert lib.gsb_mcmc_dead(u32(0), NULL, NULL, f32(0.005), NULL, NULL, NULL, NULL, sz(0), NULL) == OK
    assert lib.gsb_mcmc_sample(u32(0), NULL, 0, u32(4), NULL, NULL, NULL, NULL, NULL, sz(0), NULL) == OK
    assert lib.gsb_mcmc_apply(u32(0), NULL, NULL, u32(4), NULL, NULL, NULL, i32(51), f32(0.005), NULL, sz(0), NULL) == OK
    assert lib.gsb_mcmc_add_noise(u32(0), NULL, NULL, NULL, NULL, NULL, NULL, f32(5e5), NULL) == OK
    assert lib.gsb_mcmc_regularize(u32(0), NULL, NULL, f32(0.01), f32(0.01), NULL, NULL, NULL, NULL, sz(0), NULL) == OK
    # missing pointers
    assert lib.gsb_mcmc_dead(u32(4), PTR, NULL, f32(0.005), PTR, PTR, PTR, PTR, sz(ws), NULL) == E_INVALID
    assert lib.gsb_mcmc_dead(u32(4), PTR, PTR, f32(0.005), PTR, NULL, PTR, PTR, sz(ws), NULL) == E_INVALID
    assert lib.gsb_mcmc_sample(u32(4), PTR, 0, u32(4), NULL, NULL, NULL, PTR, PTR, sz(ws), NULL) == E_INVALID
    assert lib.gsb_mcmc_sample(u32(4), NULL, 0, u32(4), NULL, PTR, NULL, PTR, PTR, sz(ws), NULL) == E_INVALID
    assert lib.gsb_mcmc_apply(u32(4), NULL, PTR, u32(4), NULL, NULL, PTR, i32(51), f32(0.005), PTR, sz(ws), NULL) == E_INVALID
    rows = GsbMcmcRows(means=PTR.value, sh0=PTR.value, shN=None, scaling_raw=PTR.value, rotation_raw=PTR.value,
                       opacity_raw=PTR.value, shN_rows=3)
    assert lib.gsb_mcmc_apply(u32(4), C.byref(rows), PTR, u32(4), NULL, NULL, PTR, i32(51), f32(0.005), PTR, sz(ws),
                              NULL) == E_INVALID  # shN rows without shN
    assert lib.gsb_mcmc_add_noise(u32(4), PTR, PTR, PTR, PTR, PTR, NULL, f32(5e5), NULL) == E_INVALID
    assert lib.gsb_mcmc_regularize(u32(4), PTR, PTR, f32(0.01), f32(0.01), PTR, PTR, NULL, PTR, sz(ws), NULL) == E_INVALID
    # short or misaligned workspace
    assert lib.gsb_mcmc_dead(u32(4), PTR, PTR, f32(0.005), PTR, PTR, PTR, PTR, sz(ws - 1), NULL) == E_WORKSPACE
    assert lib.gsb_mcmc_dead(u32(4), PTR, PTR, f32(0.005), PTR, PTR, PTR, C.c_void_p(_aligned + 8), sz(ws),
                             NULL) == E_WORKSPACE
    ph = GsbPhilox()
    assert lib.gsb_mcmc_sample(u32(4), PTR, 0, u32(4), NULL, NULL, C.byref(ph), PTR, NULL, sz(ws), NULL) == E_WORKSPACE
