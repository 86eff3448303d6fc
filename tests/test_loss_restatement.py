"""CPU: the float64 restatement of the training loss (loss_restatement.py) against autograd's finite differences, the
"valid" crop rule, cases whose values follow by hand, and the values of the restatement it replaced."""
import math

import pytest
import torch

import loss_restatement as lr


def _pair(H, W, seed, lo=-0.2, hi=1.2):
    g = torch.Generator().manual_seed(seed)
    renders = torch.rand((1, H, W, 3), generator=g, dtype=torch.float64) * (hi - lo) + lo
    target = torch.rand((3, H, W), generator=g, dtype=torch.float64)
    return renders, target


@pytest.mark.parametrize("clamp", [True, False])
def test_gradcheck(clamp):
    # renders at least 0.1 from the clamp bounds, 15% of them outside [0, 1], and none within 1e-4 of the target: no
    # finite difference crosses a kink of the clamp or of |.|
    r, t = _pair(12, 13, 5, lo=0.1, hi=0.9)
    g = torch.Generator().manual_seed(6)
    outside = torch.rand(r.shape, generator=g, dtype=torch.float64) < 0.15
    u, v = (torch.rand(r.shape, generator=g, dtype=torch.float64) for _ in range(2))
    r = torch.where(outside, torch.where(u < 0.5, -0.15 - 0.3 * v, 1.15 + 0.3 * v), r).requires_grad_(True)
    assert bool(((r < -0.1) | (r > 1.1)).eq(outside).all())
    assert float((r.detach()[0].permute(2, 0, 1) - t).abs().min()) > 1e-4
    assert torch.autograd.gradcheck(lambda x: lr.loss_terms(x, t, 0.2, clamp), (r,), eps=1e-6, atol=1e-9, rtol=1e-6)
    *_, g = lr.photometric_loss_f64(r, t, 0.2, clamp)
    if clamp:  # outside [0, 1] the clamp passes nothing
        assert bool((g[outside] == 0).all()) and bool((g[~outside] != 0).all())
    else:
        assert bool((g != 0).all())


@pytest.mark.parametrize("H,W,cropped", [(10, 11, False), (11, 10, False), (11, 11, True), (12, 21, True)])
def test_valid_crop_rule(H, W, cropped):
    r, t = _pair(H, W, H * 100 + W)
    _, _, ssim, _ = lr.photometric_loss_f64(r, t, 0.2, True)
    m = lr.ssim_map(lr.renders_chw(r).clamp(0, 1), t)
    assert m.shape == (3, H, W)
    want = m[:, 5:H - 5, 5:W - 5].mean() if cropped else m.mean()
    assert ssim == pytest.approx(float(want), abs=1e-15)
    if (H, W) == (11, 11):  # one pixel per channel is left: the centre, whose window touches every pixel
        assert ssim == pytest.approx(float(m[:, 5, 5].mean()), abs=1e-15)
        assert abs(ssim - float(m.mean())) > 1e-3


def test_window_is_sigma_1_5_normalised():
    w = lr.window_1d()
    assert len(w) == 11 and math.fsum(w) == pytest.approx(1.0, abs=1e-15) and w == w[::-1]
    assert w[4] / w[5] == pytest.approx(math.exp(-1.0 / 4.5), rel=1e-15)
    # the taps csrc/gsb_loss.cu keeps in constant memory are these, rounded to float32
    assert w[5] == pytest.approx(0.2660117249, rel=1e-9) and w[0] == pytest.approx(0.001028380084, rel=1e-9)


@pytest.mark.parametrize("clamp", [True, False])
@pytest.mark.parametrize("constant", [True, False])
def test_identical_images_give_ssim_one_and_zero_gradient(clamp, constant):
    """x == y maximises every pixel's luminance and structure factors at 1, so SSIM = 1 and its gradient is 0; the
    L1 term is 0 with subgradient 0."""
    H, W = 23, 31
    t = torch.full((3, H, W), 0.375, dtype=torch.float64) if constant else _pair(H, W, 8, 0.0, 1.0)[1]
    loss, l1, ssim, g = lr.photometric_loss_f64(t.permute(1, 2, 0)[None], t, 0.2, clamp)
    assert l1 == 0.0 and ssim == pytest.approx(1.0, abs=1e-14) and loss == pytest.approx(0.0, abs=1e-14)
    assert float(g.abs().max()) <= 1e-12


@pytest.mark.parametrize("clamp", [True, False])
def test_constant_images_by_hand(clamp):
    """Constant planes a (render) and b (target): every pixel of the cropped map has its window inside the image, so
    sigma^2 = sigma12 = 0 and SSIM = (2ab + C1) / (a^2 + b^2 + C1); a render of 1.3 is clamped to 1."""
    H, W, b = 17, 29, 0.5
    r = torch.full((1, H, W, 3), 1.3, dtype=torch.float64)
    loss, l1, ssim, g = lr.photometric_loss_f64(r, torch.full((3, H, W), b, dtype=torch.float64), 0.2, clamp)
    a = 1.0 if clamp else 1.3
    want = (2 * a * b + lr.C1) / (a * a + b * b + lr.C1)
    # sigma^2 = E[x^2] - mu^2 cancels to ~1e-16, and C2 = 9e-4 alone is left in its denominator
    assert l1 == pytest.approx(a - b, abs=1e-15) and ssim == pytest.approx(want, abs=1e-11)
    assert loss == pytest.approx(0.8 * (a - b) + 0.2 * (1 - want), abs=1e-11)
    if clamp:
        assert bool((g == 0).all())


@pytest.mark.parametrize("clamp", [True, False])
def test_lambda_selects_the_terms(clamp):
    r, t = _pair(19, 27, 9)
    x = r.clone().requires_grad_(True)
    loss, l1, ssim = lr.loss_terms(x, t, 0.0, clamp)
    assert float(loss.detach()) == float(l1.detach())
    (g0,) = torch.autograd.grad(loss, x)
    (gl1,) = torch.autograd.grad(lr.loss_terms(x, t, 0.2, clamp)[1], x)
    assert torch.equal(g0, gl1)
    loss, l1, ssim = lr.loss_terms(x, t, 1.0, clamp)
    assert float(loss.detach()) == 1.0 - float(ssim.detach())
    (g1,) = torch.autograd.grad(loss, x)
    (gs,) = torch.autograd.grad(lr.loss_terms(x, t, 0.2, clamp)[2], x)
    assert torch.allclose(g1, -gs, rtol=1e-13, atol=0)
    # the blend at 0.2 is the weighted sum of the two
    (g2,) = torch.autograd.grad(lr.loss_terms(x, t, 0.2, clamp)[0], x)
    assert torch.allclose(g2, 0.8 * gl1 - 0.2 * gs, rtol=1e-12, atol=1e-18)


def test_layouts_agree():
    r, t = _pair(13, 22, 10)
    loss, l1, ssim, g = lr.photometric_loss_f64(r, t)
    planes = r[0].permute(2, 0, 1).contiguous()
    for rr, gl in ((r, lambda x: x), (planes, lambda x: x.permute(1, 2, 0)[None])):
        for tt in (t, t[None], t.permute(1, 2, 0)[None].contiguous()):
            got = lr.photometric_loss_f64(rr, tt)
            assert got[:3] == (loss, l1, ssim)
            assert torch.equal(gl(got[3]), g)


# The restatement this module replaced (a 2-D grouped conv2d of the same window, [1,H,W,3] renders, clamp always on)
# gave these values, to the last digit printed, on the inputs below: (loss, L1, SSIM, |dLoss/d(render)|_2).
_PREVIOUS = {
    (9, 40, 0.2): (0.43677695988415804, 0.36594226090511167, 0.27988424419965646, 0.029241959287932353),
    (70, 150, 0.2): (0.5018330683494894, 0.37985403329510975, 0.01025079143299243, 0.0057814863504374045),
    (64, 80, 0.5): (0.6891058813230865, 0.38208749310896434, 0.0038757304627912914, 0.012297629425930226),
}


@pytest.mark.parametrize("H,W,lam", list(_PREVIOUS))
def test_agrees_with_the_previous_restatement(H, W, lam):
    g = torch.Generator().manual_seed(H * 1000 + W)
    r = torch.rand((1, H, W, 3), generator=g, dtype=torch.float64) * 1.4 - 0.2
    t = torch.rand((3, H, W), generator=g, dtype=torch.float64)
    loss, l1, ssim, grad = lr.photometric_loss_f64(r, t, lam, True)
    want = _PREVIOUS[(H, W, lam)]
    assert loss == pytest.approx(want[0], abs=1e-14) and l1 == pytest.approx(want[1], abs=1e-14)
    assert ssim == pytest.approx(want[2], abs=1e-14)
    assert float(grad.norm()) == pytest.approx(want[3], rel=1e-12)
