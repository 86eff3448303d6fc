"""GPU: the default strategy's refine of this library against the restatement of default_strategy.cpp driven by the
REFERENCE's own gsplat::quats_to_rotmats (oracle/_ref/libgsplat_ref.so, built by oracle/build_ref.py where the
reference's sources are present; skipped otherwise).  SH degrees 0 and 3, with and without revised opacity."""
import importlib

import pytest
import torch

import adc_restatement as R
from oracle import ref_ops
from test_gpu_adc import _assert_rows_equal, _offset_magnitude, _params

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_ops.available(), reason="oracle/_ref/libgsplat_ref.so not built")]


@pytest.mark.parametrize("revised", [False, True])
@pytest.mark.parametrize("K", [0, 15])
def test_refine_matches_reference_composition(native, cuda_device, K, revised):
    adc = importlib.import_module(native.__name__ + ".adc")
    N, it = 200_003, (40 if revised else 20)
    P, M1, M2, info = _params(N, K, cuda_device, "mixed", seed=70 + K)
    cfg = adc.DefaultConfig(reset_every=30, revised_opacity=revised)
    counts, ws = torch.ops.gsplat_b200.adc_classify(info, P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                                                    cfg.grad_threshold, cfg.grow_scale3d, cfg.prune_scale3d, 1.0,
                                                    cfg.prune_opacity, it > cfg.reset_every, revised)
    c = counts.tolist()
    torch.manual_seed(K)
    z = torch.randn((2, c[1], 3), device=cuda_device)
    gp, g1, g2, _ = torch.ops.gsplat_b200.adc_apply([P[k] for k in R.GROUPS], [M1[k] for k in R.GROUPS],
                                                    [M2[k] for k in R.GROUPS], ws, counts, c[1], c[3], z, revised)
    WP, WM1, WM2, wc, _ = R.refine(P, M1, M2, info, it, cfg, 1.0, ref_ops._ns().quats_to_rotmats, z)
    assert tuple(c[:4]) == wc and min(wc[:3]) > 0
    A = _offset_magnitude(native, P, M1, M2, info, it, cfg, z)[c[4] + c[5]:]
    _assert_rows_equal((dict(zip(R.GROUPS, gp)), dict(zip(R.GROUPS, g1)), dict(zip(R.GROUPS, g2)), A),
                       (WP, WM1, WM2), c[4] + c[5], "reference")
