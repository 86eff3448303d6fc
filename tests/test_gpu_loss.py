"""GPU: the training loss kernel (csrc/gsb_loss.cu, through training.photometric_loss and its unclamped variant, the
loss of a bilateral-grid output) against the float64 restatement of loss_restatement.py, at the shapes where its
32x16 tile, 52x36 staged neighbourhood, ragged strips and "valid" crop have edges, in every layout it accepts, at the
clamp's and the L1 subgradient's edges, and on a NaN render."""
import math

import pytest
import torch

import loss_restatement as lr
from parity import rel

pytestmark = pytest.mark.gpu

# An exact zero in the kernel's gradient where the clamp passes it must be a zero of the float64 gradient: no larger
# than this fraction of the largest float64 gradient (float32 rounding of terms that cancel), far below the 1e-4 bound
# on every element's error.
ZERO_TOL = 1e-6


@pytest.fixture(scope="module")
def training(native):
    from gsplat_b200 import training
    return training


def _inputs(H, W, seed, dev):
    """Renders in [-0.2, 1.2) (about 14% clamped) and a target that follows them, so SSIM is mid-range."""
    g = torch.Generator(device=dev).manual_seed(seed)
    renders = torch.rand((1, H, W, 3), device=dev, generator=g) * 1.4 - 0.2
    target = 0.7 * renders[0].permute(2, 0, 1).clamp(0, 1) + 0.3 * torch.rand((3, H, W), device=dev, generator=g)
    return renders, target.contiguous()


def _kernel(training, renders, target, lam, clamp, scale=1.0):
    """([loss, L1, SSIM], d(scale * loss)/d(renders)) from the kernel."""
    r = renders.detach().clone().requires_grad_(True)
    fn = training.photometric_loss if clamp else training.photometric_loss_unclamped
    loss, stats = fn(r, target, lam)
    (loss * scale).backward()
    return [float(v) for v in stats.cpu()], r.grad


def _check(training, tag, renders, target, lam=0.2, clamp=True, zero_tol=ZERO_TOL):
    got, g = _kernel(training, renders, target, lam, clamp)
    *want, g64 = lr.photometric_loss_f64(renders, target, lam, clamp)
    errs = [abs(a - b) for a, b in zip(got, want)]
    gmax = max(float(g64.abs().max()), 1e-30)
    g_rel, g_max = rel(g, g64), float((g.double() - g64).abs().max()) / gmax
    # the clamp mask: no gradient where the clamp was active, and no other zero the float64 gradient does not have
    blocked = ((renders < 0) | (renders > 1)) if clamp else torch.zeros_like(renders, dtype=torch.bool)
    free_zero = (g == 0) & ~blocked
    zero_max = float(g64[free_zero].abs().max()) / gmax if bool(free_zero.any()) else 0.0
    print(f"[{tag}] loss {got[0]:.7f}: err {errs[0]:.1e} (L1 {errs[1]:.1e}, SSIM {errs[2]:.1e}); "
          f"grad rel_l2 {g_rel:.2e}, max|err| / max|g64| {g_max:.1e}; {int(free_zero.sum())} zeros where the clamp "
          f"passes, max|g64| there / max|g64| {zero_max:.1e}")
    for name, e, w in zip(("loss", "L1", "SSIM"), errs, want):
        assert e <= 2e-6 * max(1.0, abs(w)), (name, e, w)
    assert g_rel < 2e-5
    assert g_max <= 1e-4
    assert bool((g[blocked] == 0).all())
    assert zero_max <= zero_tol
    return got, g


SHAPES = [(1, 1), (1, 37), (37, 1), (5, 37), (10, 10), (10, 11), (11, 10), (11, 11), (12, 21),
          (16, 32),  # exactly one tile
          (15, 31), (17, 33),  # a pixel short of it / a pixel past it
          (16, 64), (48, 96),  # tile multiples
          (822, 1237), (1080, 1920)]


@pytest.mark.parametrize("clamp", [True, False], ids=["clamped", "unclamped"])
@pytest.mark.parametrize("H,W", SHAPES)
def test_loss_and_gradient_vs_float64(training, cuda_device, H, W, clamp):
    renders, target = _inputs(H, W, H * 10000 + W, cuda_device)
    _check(training, f"{H}x{W} {'clamped' if clamp else 'unclamped'}", renders, target, 0.2, clamp)


@pytest.mark.parametrize("clamp", [True, False], ids=["clamped", "unclamped"])
def test_every_layout_gives_the_same_loss_and_gradient(training, cuda_device, clamp):
    """Renders [1,H,W,3] or [3,H,W] planes x target [3,H,W], [1,3,H,W] or [1,H,W,3]: the layout only moves the loads and
    stores, so the gradient is bit for bit the same.  So is the loss: each CTA's partial sums are float32 with a fixed
    order, and their double-precision total is exact at this size, whatever order the atomics take."""
    H, W = 70, 150
    renders, target = _inputs(H, W, 70, cuda_device)
    base, g_base = _kernel(training, renders, target, 0.2, clamp)
    planes = renders[0].permute(2, 0, 1).contiguous()
    for r_name, rr, back in (("[1,H,W,3]", renders, lambda x: x), ("[3,H,W]", planes, lambda x: x.permute(1, 2, 0)[None])):
        for t_name, tt in (("[3,H,W]", target), ("[1,3,H,W]", target[None]),
                           ("[1,H,W,3]", target.permute(1, 2, 0)[None].contiguous())):
            got, g = _kernel(training, rr, tt, 0.2, clamp)
            assert got == base, (r_name, t_name, got, base)
            assert g.shape == rr.shape and torch.equal(back(g), g_base), (r_name, t_name)
    _check(training, f"{H}x{W} layouts", renders, target, 0.2, clamp)


def _edge_case(kind, H, W, dev):
    renders, target = _inputs(H, W, 77, dev)
    r, t = renders[0], target  # [H,W,3] view, [3,H,W]
    if kind == "zero_one":  # the clamp's bounds, where torch's inclusive mask passes the gradient
        r[5:30, 10:50] = 0.0
        r[40:66, 90:141] = 1.0
    elif kind == "inf":
        r[5:30, 10:50] = math.inf
        r[40:66, 90:141] = -math.inf
        r[50, 20, 1] = math.inf
    elif kind == "equal":  # render == target bit for bit: L1 subgradient 0
        r[8:40, 30:100] = t.permute(1, 2, 0)[8:40, 30:100]
        r[60, :, 2] = t[2, 60, :]
    elif kind == "constant":
        # sigma^2 = sigma12 = 0 inside the blocks, so C2 alone is left in the denominator.  The values are powers of two:
        # their window sums are exact in float32, so what is checked is the kernel's handling of that denominator, not
        # the cancellation in E[x^2] - mu^2 that float32 shares with the reference's own kernel.
        r[5:30, 10:50] = 0.5
        t[:, 5:30, 10:50] = 0.25
        r[35:66, 80:140] = 0.5
        t[:, 35:66, 80:140] = 0.5
    elif kind == "black":
        renders.zero_()
        target.zero_()
    return renders, target


# an infinite render only has a finite loss through the clamp
EDGES = [(k, c) for k in ("zero_one", "inf", "equal", "constant", "black") for c in (True, False) if c or k != "inf"]


@pytest.mark.parametrize("kind,clamp", EDGES, ids=[f"{k}-{'clamped' if c else 'unclamped'}" for k, c in EDGES])
def test_value_edges(training, cuda_device, kind, clamp):
    H, W = 71, 149
    renders, target = _edge_case(kind, H, W, cuda_device)
    # Next to the block where render == target the true gradient is ~0, the difference of terms of size ~1/C2 that
    # float32 resolves only to a few 1e-5 of the largest gradient: an exact zero there is rounding, held to the 1e-4
    # bound on every element.
    zero_tol = 1e-4 if kind == "constant" else ZERO_TOL
    got, g = _check(training, f"{kind} {'clamped' if clamp else 'unclamped'}", renders, target, 0.2, clamp, zero_tol)
    if kind == "inf":
        assert all(math.isfinite(v) for v in got)
        assert bool((g[renders.isinf()] == 0).all())
    if kind == "black":  # L1 = 0, SSIM = C1 C2 / (C1 C2) = 1, and every term of the gradient has a zero factor
        assert got[1] == 0.0
        assert bool((g == 0).all())


@pytest.mark.parametrize("clamp", [True, False], ids=["clamped", "unclamped"])
@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
def test_lambda_and_upstream_scale(training, cuda_device, lam, clamp):
    renders, target = _inputs(45, 77, 45, cuda_device)
    got, g = _check(training, f"lambda {lam} {'clamped' if clamp else 'unclamped'}", renders, target, lam, clamp)
    if lam == 0.0:
        assert got[0] == got[1]
    _, g17 = _kernel(training, renders, target, lam, clamp, scale=1.7)
    assert torch.equal(g17, g * 1.7)


def _nan_pair(dev):
    """A ragged image with one NaN render value in its interior, and the same image with 0.5 there."""
    H, W = 70, 150
    renders, target = _inputs(H, W, 99, dev)
    bad, fine = renders.clone(), renders.clone()
    bad[0, 33, 77, 1] = math.nan
    fine[0, 33, 77, 1] = 0.5
    return bad, fine, target, (33, 77, 1)


def test_nan_render_clamped(training, cuda_device):
    """torch::clamp keeps NaN, so the reference's loss is NaN; its backward masks the NaN pixel itself to 0.  The loss
    must not hide a diverging model that evaluation would report."""
    bad, fine, target, (y, x, c) = _nan_pair(cuda_device)
    got, g = _kernel(training, bad, target, 0.2, True)
    _, g_fine = _kernel(training, fine, target, 0.2, True)
    print(f"NaN render, clamped: stats {got}; gradient at the pixel {float(g[0, y, x, c])}")
    assert all(math.isnan(v) for v in got)
    assert float(g[0, y, x, c]) == 0.0
    H, W = bad.shape[1:3]
    cheb = torch.maximum((torch.arange(H, device=cuda_device)[:, None] - y).abs(),
                         (torch.arange(W, device=cuda_device)[None, :] - x).abs())
    # farther than the two window radii from the pixel nothing depends on it; the other channels never do
    far = cheb > 10
    assert torch.equal(g[0][far][:, c], g_fine[0][far][:, c])
    others = [k for k in range(3) if k != c]
    assert torch.equal(g[0][..., others], g_fine[0][..., others])
    # within them every SSIM statistic the gradient sums is NaN, and the clamp mask alone gives a 0
    near = (cheb <= 10) & (cheb > 0)
    raw, gc = bad[0, :, :, c], g[0, :, :, c]
    passing = (raw >= 0) & (raw <= 1)
    assert bool(gc[near & passing].isnan().all()) and bool((gc[near & ~passing] == 0).all())


def test_nan_render_unclamped(training, cuda_device):
    bad, _, target, (y, x, c) = _nan_pair(cuda_device)
    got, g = _kernel(training, bad, target, 0.2, False)
    print(f"NaN render, unclamped: stats {got}; gradient at the pixel {float(g[0, y, x, c])}")
    assert all(math.isnan(v) for v in got)
    assert math.isnan(float(g[0, y, x, c]))
