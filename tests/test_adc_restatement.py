"""CPU: the default-strategy restatement (tests/adc_restatement.py) against a hand-built 8-row case whose final row
order, moments and counts are written out by hand; is_refining with a pause after reset; the reset threshold; the
statistics at and after stop_refine; and the strategy's configuration."""
import importlib

import numpy as np
import pytest
import torch

import adc_restatement as R


@pytest.fixture(scope="module")
def adc(pkg):
    """adc.py: its configuration and host-side helpers need no native library."""
    return importlib.import_module(pkg.__name__ + ".adc")


SMALL, LARGE, HUGE = float(np.log(0.005)), float(np.log(0.05)), float(np.log(0.2))
ALIVE, DEAD, FAINT = 0.0, -7.0, float(np.log(0.009 / 0.991))  # sigmoid 0.5, 9e-4, 0.009


def _case():
    """Eight rows, thresholds at their defaults (grow 0.01, prune 0.1, opacity 0.005, gradient 2e-4, scene scale 1):
      0  low gradient, small                      kept as it is
      1  high, small                              duplicated
      2  high, large (0.05)                       split; copies at 0.031 kept
      3  high, small, opacity 9e-4                duplicated, and the source and its copy are both pruned
      4  high, huge (0.2)                         split; copies at 0.125 pruned as too big after reset_every
      5  low, huge                                pruned as too big after reset_every
      6  low, small, |q|^2 = 4e-10                pruned
      7  high, large, opacity 0.009               split; revised copies at 0.0045 pruned"""
    high = [0, 1, 1, 1, 1, 0, 0, 1]
    scale = [SMALL, SMALL, LARGE, SMALL, HUGE, HUGE, SMALL, LARGE]
    opac = [ALIVE, ALIVE, ALIVE, DEAD, ALIVE, ALIVE, ALIVE, FAINT]
    N = 8
    P = {"means": torch.arange(N * 3, dtype=torch.float32).reshape(N, 3),
         "sh0": 100 + torch.arange(N * 3, dtype=torch.float32).reshape(N, 1, 3),
         "shN": 200 + torch.arange(N * 3, dtype=torch.float32).reshape(N, 1, 3),
         "scaling_raw": torch.tensor(scale, dtype=torch.float32)[:, None].repeat(1, 3),
         "rotation_raw": torch.tensor([[1.0, 0.0, 0.0, 0.0]] * N),
         "opacity_raw": torch.tensor(opac, dtype=torch.float32)[:, None]}
    P["rotation_raw"][6] = 1e-5
    M1 = {k: 1000 + torch.arange(v.numel(), dtype=torch.float32).reshape(v.shape) for k, v in P.items()}
    M2 = {k: 2000 + torch.arange(v.numel(), dtype=torch.float32).reshape(v.shape) for k, v in P.items()}
    info = torch.stack([torch.ones(N), torch.tensor(high, dtype=torch.float32) * 1e-3])
    z = torch.tensor([[[0.5, -1.0, 2.0], [1.0, 1.0, 1.0], [-2.0, 0.25, 0.0]],
                      [[-0.5, 1.0, -2.0], [0.0, -1.0, 3.0], [1.5, 0.0, -1.0]]])
    return P, M1, M2, info, z


def _check(P0, M10, M20, z, out, want, revised):
    """want: the final rows as (source, kind) with kind 'keep', 'dup' or the split copy 0 / 1 (rank = the source's rank
    among the split rows 2, 4, 7)."""
    P, M1, M2 = out
    assert P["means"].shape[0] == len(want)
    rank = {2: 0, 4: 1, 7: 2}
    for d, (s, kind) in enumerate(want):
        for k in ("sh0", "shN", "rotation_raw"):
            assert torch.equal(P[k][d], P0[k][s]), (d, k)
        if kind in ("keep", "dup"):
            for k in ("means", "scaling_raw", "opacity_raw"):
                assert torch.equal(P[k][d], P0[k][s]), (d, k)
        else:
            sc = torch.exp(P0["scaling_raw"][s])
            # identity rotation: the offset is s * z[b, rank]
            torch.testing.assert_close(P["means"][d], P0["means"][s] + sc * z[kind, rank[s]], rtol=1e-6, atol=1e-6)
            assert torch.equal(P["scaling_raw"][d], torch.log(sc / 1.6))
            o = P0["opacity_raw"][s]
            assert torch.equal(P["opacity_raw"][d],
                               torch.logit(1.0 - torch.sqrt(1.0 - torch.sigmoid(o))) if revised else o)
        for k in R.GROUPS:
            if kind == "keep":
                assert torch.equal(M1[k][d], M10[k][s]) and torch.equal(M2[k][d], M20[k][s]), (d, k)
            else:
                assert not M1[k][d].any() and not M2[k][d].any(), (d, k)


def test_hand_built_refine_before_reset_every(adc):
    """Iteration 20 <= reset_every 30: no too-big pruning.  Grown set: 8 + 2 duplicates + 3 splits = 13 rows; rows 3,
    6 and 3's duplicate are pruned."""
    P0, M10, M20, info, z = _case()
    cfg = adc.DefaultConfig(reset_every=30)
    P, M1, M2, counts, zz = R.refine(P0, M10, M20, info, 20, cfg, 1.0, R.quats_to_rotmats_torch, z)
    assert counts == (2, 3, 3, 10)
    assert zz is z
    want = [(0, "keep"), (1, "keep"), (5, "keep"), (1, "dup"), (2, 0), (4, 0), (7, 0), (2, 1), (4, 1), (7, 1)]
    _check(P0, M10, M20, z, (P, M1, M2), want, revised=False)


def test_hand_built_refine_after_reset_every_revised(adc):
    """Iteration 40 > reset_every 30 with revised_opacity: row 5 and row 4's copies go as too big, row 7's copies as
    too faint; 13 - 8 = 5 rows remain."""
    P0, M10, M20, info, z = _case()
    cfg = adc.DefaultConfig(reset_every=30, revised_opacity=True)
    P, M1, M2, counts, _ = R.refine(P0, M10, M20, info, 40, cfg, 1.0, R.quats_to_rotmats_torch, z)
    assert counts == (2, 3, 8, 5)
    _check(P0, M10, M20, z, (P, M1, M2), [(0, "keep"), (1, "keep"), (1, "dup"), (2, 0), (2, 1)], revised=True)


def test_hand_built_split_copies_kept_without_revised_opacity(adc):
    """Iteration 40 without revised_opacity: row 7's copies keep opacity 0.009 and stay."""
    P0, M10, M20, info, z = _case()
    cfg = adc.DefaultConfig(reset_every=30)
    P, M1, M2, counts, _ = R.refine(P0, M10, M20, info, 40, cfg, 1.0, R.quats_to_rotmats_torch, z)
    assert counts == (2, 3, 6, 7)
    _check(P0, M10, M20, z, (P, M1, M2), [(0, "keep"), (1, "keep"), (1, "dup"), (2, 0), (7, 0), (2, 1), (7, 1)],
           revised=False)


def test_scene_scale_scales_both_thresholds(adc):
    """With scene_scale 10 the grow limit is 0.1: rows 2 and 7 (0.05) duplicate instead of splitting, row 4 (0.2)
    still splits, and nothing is too big for the prune limit 1.0."""
    P0, M10, M20, info, z = _case()
    cfg = adc.DefaultConfig(reset_every=30)
    _, _, _, counts, _ = R.refine(P0, M10, M20, info, 40, cfg, 10.0, R.quats_to_rotmats_torch, z[:, :1])
    # duplicates 1, 2, 3, 7; split 4; pruned 3, its copy and 6
    assert counts == (4, 1, 3, 8 + 4 + 1 - 3)


def test_is_refining_with_pause_after_reset(adc):
    cfg = adc.DefaultConfig(start_refine=500, refine_every=100, reset_every=3000, pause_refine_after_reset=500)
    got = {it: R.is_refining(cfg, it) for it in (500, 600, 650, 2900, 3000, 3100, 3400, 3500, 6000, 6500)}
    assert got == {500: False, 600: True, 650: False, 2900: True, 3000: False, 3100: False, 3400: False, 3500: True,
                   6000: False, 6500: True}
    # the strategy's own predicate is the same function of the configuration
    s = adc.DefaultStrategy.__new__(adc.DefaultStrategy)
    s.cfg = cfg
    assert all(s.is_refining(it) == want for it, want in got.items())


def test_reset_threshold_is_a_float_logit(adc):
    thr = R.reset_threshold(0.005)
    x = np.float32(2.0) * np.float32(0.005)
    assert thr == float(np.float32(np.log(np.float32(x / (np.float32(1) - x)))))
    assert abs(thr - np.log(0.01 / 0.99)) < 1e-6
    P0, M10, M20, _, _ = _case()
    P, M1, M2 = dict(P0), dict(M10), dict(M20)
    R.reset_opacity(P, M1, M2, adc.DefaultConfig())
    o0, o = P0["opacity_raw"].reshape(-1), P["opacity_raw"].reshape(-1)
    assert torch.equal(o, torch.where(o0 > thr, torch.full_like(o0, thr), o0))
    assert o[0] == np.float32(thr) and o[3] == DEAD and o[7] == np.float32(FAINT)
    assert not M1["opacity_raw"].any() and not M2["opacity_raw"].any()
    assert torch.equal(M1["means"], M10["means"])


def test_statistics_at_and_after_stop_refine(adc):
    """At stop_refine the statistics become empty and nothing refines, even on a refine iteration; after it nothing
    happens at all.  Before it, a refine leaves zeroed statistics sized to the new set, and a reset iteration skips
    the opacity group only."""
    P0, M10, M20, info, z = _case()
    cfg = adc.DefaultConfig(start_refine=0, refine_every=10, reset_every=30, stop_refine=50)
    st = R.Strategy(P0, M10, M20, cfg, 1.0, R.quats_to_rotmats_torch)
    st.info = info.clone()
    skip = st.post_backward(20, z)
    assert skip == R.GROUPS and st.counts == (2, 3, 3, 10)
    assert st.info.shape == (2, 10) and not st.info.any()
    st.adam_bookkeeping(skip)
    assert set(st.steps.values()) == {0}
    st2 = R.Strategy(P0, M10, M20, cfg, 1.0, R.quats_to_rotmats_torch)
    st2.info = torch.zeros(2, 8)
    st2.P["opacity_raw"][3] = ALIVE
    st2.P["rotation_raw"][6] = 1.0
    assert st2.post_backward(20) == ()  # a refine that changed nothing: Adam steps every group
    assert st2.counts == (0, 0, 0, 8)
    assert st2.post_backward(30) == ("opacity_raw",) and st2.counts == (0, 0, 0, 8)  # refine, then the reset
    n = st2.P["means"].shape[0]
    st2.info = torch.ones(2, n)
    assert st2.post_backward(50) == () and st2.info.numel() == 0 and st2.counts is None
    assert st2.P["means"].shape[0] == n
    assert st2.post_backward(60) == () and st2.info.numel() == 0


def test_config_fields(adc):
    """The fields default_optimization_params.json gives the strategy, with its values."""
    c = adc.DefaultConfig()
    assert (c.refine_every, c.start_refine, c.stop_refine, c.reset_every, c.pause_refine_after_reset) == \
        (100, 500, 15000, 3000, 0)
    assert (c.grad_threshold, c.grow_scale3d, c.prune_opacity, c.prune_scale3d) == (0.0002, 0.01, 0.005, 0.1)
    assert (c.revised_opacity, c.opacity_reg, c.scale_reg, c.sh_degree_interval) == (False, 0.0, 0.0, 1000)
