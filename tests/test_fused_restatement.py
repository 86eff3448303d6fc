"""CPU: the float64 restatement of the fused raw-parameter path (fused_restatement.py).  Its hand-written chain rule
against torch autograd through the activations rasterize_from_raw applies, and the clamp rule of the colour at its
boundary."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fused_restatement as fr
import scenes

SH_LAYOUTS = [(0, 1), (0, 16), (1, 16), (2, 16), (3, 16), (4, 25), (2, 25)]


def _random_raw(N, K, seed):
    """Raw parameters in float64: quaternions of norm 0.3 to 3, log-scales about log(0.05), opacities about 0.5."""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((N, 4))
    q *= (rng.random((N, 1)) * 2.7 + 0.3) / np.linalg.norm(q, axis=-1, keepdims=True)
    return dict(means=rng.standard_normal((N, 3)), sh0=rng.standard_normal((N, 1, 3)) * 0.3,
                shN=rng.standard_normal((N, K - 1, 3)) * 0.3, scaling_raw=rng.standard_normal((N, 3)) * 0.5 - 3.0,
                rotation_raw=q, opacity_raw=rng.standard_normal((N, 1)) * 2.0)


@pytest.mark.parametrize("modifier", [1.0, 0.5, 1.7])
@pytest.mark.parametrize("deg,K", SH_LAYOUTS)
def test_chain_matches_autograd(deg, K, modifier):
    N = 257
    raw = _random_raw(N, K, deg * 100 + K + int(modifier * 10))
    norms = np.linalg.norm(raw["rotation_raw"], axis=-1)
    assert norms.min() < 0.5 and norms.max() > 2.5
    rng = np.random.default_rng(K)
    cot = dict(v_means=rng.standard_normal((N, 3)), v_quats=rng.standard_normal((N, 4)),
               v_scales=rng.standard_normal((N, 3)), v_opacities=rng.standard_normal(N),
               v_sh_coeffs=rng.standard_normal((N, K, 3)), v_dirs=rng.standard_normal((N, 3)))
    got = fr.chain_to_raw(raw, cot, deg, modifier)

    # autograd through the torch activations of rasterize_from_raw / rasterize (normalize, exp, * modifier, sigmoid,
    # cat); the colour reads the first (deg + 1)^2 rows of the concatenated coefficients
    P = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in raw.items()}
    T = {k: torch.from_numpy(v) for k, v in cot.items()}
    nb = (deg + 1) ** 2
    campos = torch.tensor([0.3, -0.2, 1.1], dtype=torch.float64)
    quats = F.normalize(P["rotation_raw"], dim=-1)
    scales = torch.exp(P["scaling_raw"]) * modifier
    opac = torch.sigmoid(P["opacity_raw"]).squeeze(-1)
    sh = torch.cat([P["sh0"], P["shN"]], dim=1)[:, :nb]
    dirs = P["means"] - campos
    loss = ((P["means"] * T["v_means"]).sum() + (quats * T["v_quats"]).sum() + (scales * T["v_scales"]).sum() +
            (opac * T["v_opacities"]).sum() + (sh * T["v_sh_coeffs"][:, :nb]).sum() + (dirs * T["v_dirs"]).sum())
    want = dict(zip(fr.RAW, torch.autograd.grad(loss, [P[k] for k in fr.RAW], allow_unused=True)))
    for k in fr.RAW:
        w = np.zeros_like(raw[k]) if want[k] is None else want[k].numpy()
        assert got[k].shape == raw[k].shape, k
        if not np.any(w):  # shN at degree 0
            assert not np.any(got[k]), k
        else:
            e = np.linalg.norm(got[k] - w) / np.linalg.norm(w)
            assert e < 1e-12, (k, e)
    if K > nb:  # the inactive rows of the cotangent are random and must not leak
        assert np.all(got["shN"][:, nb - 1:] == 0.0)


def _exact_minus_half(orc):
    """A float32 sh0 coefficient whose degree-0 colour the float64 oracle evaluates to exactly -0.5."""
    lo = hi = np.float32(-0.5 / 0.2820947917738781)
    cands = [lo]
    for _ in range(16):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        cands += [lo, hi]
    cands = np.array(cands, np.float32)
    dirs = np.tile(np.array([[0.0, 0.0, 1.0]], np.float32), (len(cands), 1))
    col = orc.sh_fwd(0, dirs, np.repeat(cands[:, None, None], 3, -1), precision="f64")[:, 0]
    hit = cands[col == np.float32(-0.5)]
    assert len(hit), "no float32 coefficient gives a colour of exactly -0.5"
    return hit[0]


def test_clamp_passes_the_gradient_at_exactly_minus_half(orc):
    """clamp_min(colour + 0.5, 0) at colour == -0.5: torch passes the gradient (its mask is `>= min`), and so do the
    restatement and the kernel; a colour below -0.5 gets none and one above it all."""
    x = torch.tensor([-0.5, -0.6, -0.4], dtype=torch.float32, requires_grad=True)
    torch.clamp_min(x + 0.5, 0.0).sum().backward()
    assert x.grad.tolist() == [1.0, 0.0, 1.0]

    sc = scenes.scene_small(N=3, width=64, height=48, sh_degree=0)
    sc["means"][:] = [[-0.3, 0.0, 3.0], [0.0, 0.1, 3.2], [0.3, -0.1, 2.8]]
    sc["scales"][:] = 0.1
    c = _exact_minus_half(orc)
    sh0 = np.full((3, 1, 3), 0.2, np.float32)
    sh0[0, 0] = (c, np.float32(-0.6 / 0.2820947917738781), np.float32(0.1))  # exactly -0.5, clamped, passed
    raw = dict(means=sc["means"], sh0=sh0, shN=np.zeros((3, 0, 3), np.float32),
               scaling_raw=np.log(sc["scales"]), rotation_raw=sc["quats"],
               opacity_raw=np.log(sc["opacities"] / (1 - sc["opacities"]))[:, None])
    rng = np.random.default_rng(3)
    vrc = rng.standard_normal((1, 48, 64, 3)).astype(np.float32)
    vra = rng.standard_normal((1, 48, 64, 1)).astype(np.float32)
    out, g = fr.render_raw(orc, raw, 0, sc["viewmats"], sc["Ks"], 64, 48, sc["background"], vrc, vra)
    assert out["masks"][0].all()
    assert out["sh_colors"][0, 0, 0] == np.float32(-0.5) and out["colors"][0, 0, 0] == 0.0
    assert out["sh_colors"][0, 0, 1] < -0.5 < out["sh_colors"][0, 0, 2]
    v_col = out["v_colors"][0, 0]
    assert np.all(v_col != 0.0)
    assert g["sh0"][0, 0, 0] == pytest.approx(0.2820947917738781 * v_col[0], rel=1e-6)
    assert g["sh0"][0, 0, 1] == 0.0
    assert g["sh0"][0, 0, 2] == pytest.approx(0.2820947917738781 * v_col[2], rel=1e-6)

