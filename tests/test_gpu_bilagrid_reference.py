"""GPU: the bilateral grid (SURVEY.md 8 f5) against the REFERENCE -- its own kernels (src/training/kernels/
bilateral_grid_{forward,backward,tv}.cu, compiled unmodified into oracle/_ref/libbilagrid_ref.so by
oracle/build_ref_bilagrid.py) live, the same kernels' outputs stored in tests/golden/ref_bilagrid_small.npz (so the
comparison also runs where the reference tree is absent), and its BilateralGrid component (components/bilateral_grid.cpp,
compiled unmodified against include/kernels/bilateral_grid.cuh) run on this library.  Each comparison prints the
reference kernels' own distance from the float64 restatement beside this library's."""
import importlib
import os

import numpy as np
import pytest
import torch

import bilagrid_restatement as R
from parity import rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_bilagrid_small.npz")


@pytest.fixture(scope="module")
def ref_kernels(native):
    so = os.path.join(REF_DIR, "libbilagrid_ref.so")
    if not os.path.exists(so):
        pytest.skip("reference bilateral-grid kernels not built (oracle/build_ref_bilagrid.py)")
    torch.ops.load_library(so)
    return torch.ops.bilagrid_ref


def _grids(n, X, Y, L, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return (R.identity_grids(n, X, Y, L) + 0.2 * torch.randn(n, 12, L, Y, X, generator=g, dtype=torch.float64)).float().to(dev)


def _case(h, w, X, Y, L, dev, seed):
    g = torch.Generator().manual_seed(seed)
    grids = _grids(5, X, Y, L, seed, dev)
    img = (torch.rand(h, w, 3, generator=g) * 1.4 - 0.2).to(dev)
    v_out = torch.randn(h, w, 3, generator=g).to(dev)
    return grids, img, v_out


def _ours(grids, img, v_out, idx, chw=False):
    ns = torch.ops.gsplat_b200
    i = torch.tensor([idx], dtype=torch.int32, device=img.device)
    x = img.permute(2, 0, 1).contiguous() if chw else img
    v = v_out.permute(2, 0, 1).contiguous() if chw else v_out
    out = ns.bilagrid_slice(grids, x, i, chw)
    v_grids = torch.zeros_like(grids)
    v_img = ns.bilagrid_slice_backward(grids, x, i, v, v_grids, chw)
    if chw:
        out, v_img = out.permute(1, 2, 0), v_img.permute(1, 2, 0)
    return out, v_grids, v_img


def _compare_slice(tag, grid, img, v_out, out, v_grid, v_img, ref_out, ref_vg, ref_vi):
    """ours vs the reference kernels' outputs (which take the clamped image and return the gradient with respect to
    it: the clamp mask is applied to them here, as the reference's autograd does through torch::clamp)."""
    mask = ((img >= 0) & (img <= 1)).to(ref_vi.dtype)
    ref_vi = ref_vi * mask
    want = R.slice_fwd(grid.double().cpu(), img.double().cpu())
    want_vg, want_vi = R.slice_bwd(grid.double().cpu(), img.double().cpu(), v_out.double().cpu())
    e_f = float((out.double() - ref_out.double()).abs().max())
    e_vi, e_vg = rel(v_img.cpu(), ref_vi.cpu()), rel(v_grid.cpu(), ref_vg.cpu())
    r_f = float((ref_out.double().cpu() - want).abs().max())
    o_f = float((out.double().cpu() - want).abs().max())
    print(f"[{tag}] vs reference kernels: fwd max|err| {e_f:.2e}, v_input rel_l2 {e_vi:.2e}, v_grid rel_l2 {e_vg:.2e} | "
          f"vs float64: ours fwd {o_f:.2e} v_in {rel(v_img.cpu(), want_vi):.2e} v_grid {rel(v_grid.cpu(), want_vg):.2e}; "
          f"reference fwd {r_f:.2e} v_in {rel(ref_vi.cpu(), want_vi):.2e} v_grid {rel(ref_vg.cpu(), want_vg):.2e}")
    assert e_f <= 1e-5
    assert e_vi <= 1e-5
    assert e_vg <= 1e-4


@pytest.mark.parametrize("h,w,X,Y,L", [(1080, 1920, 16, 16, 8), (97, 173, 16, 16, 8), (23, 40, 16, 16, 8),
                                       (97, 173, 12, 9, 4)])
@pytest.mark.parametrize("chw", [False, True])
def test_slice_vs_reference_kernels(native, ref_kernels, cuda_device, h, w, X, Y, L, chw):
    grids, img, v_out = _case(h, w, X, Y, L, cuda_device, h + w + X)
    out, v_grids, v_img = _ours(grids, img, v_out, 3, chw)
    x = img.clamp(0, 1).contiguous()
    ref_out = ref_kernels.slice_forward(grids[3].contiguous(), x)
    ref_vg, ref_vi = ref_kernels.slice_backward(grids[3].contiguous(), x, v_out)
    torch.cuda.synchronize()
    _compare_slice(f"{h}x{w} grid {X}x{Y}x{L} chw={chw}", grids[3], img, v_out, out, v_grids[3], v_img, ref_out, ref_vg,
                   ref_vi)
    assert int((torch.cat([v_grids[:3].flatten(), v_grids[4:].flatten()]) != 0).sum()) == 0


@pytest.mark.parametrize("N,X,Y,L", [(200, 16, 16, 8), (3, 12, 9, 4)])
def test_tv_vs_reference_kernels(native, ref_kernels, cuda_device, N, X, Y, L):
    grids = _grids(N, X, Y, L, N + X, cuda_device)
    loss, grad = torch.ops.gsplat_b200.bilagrid_tv(grids, torch.tensor([2.5], device=cuda_device), True)
    ref_loss = ref_kernels.tv_forward(grids)
    ref_grad = ref_kernels.tv_backward(grids, torch.tensor(2.5, device=cuda_device))
    want = float(R.tv_loss(grids.double().cpu()))
    e_l = abs(float(loss) - float(ref_loss)) / abs(float(ref_loss))
    e_g = rel(grad.cpu(), ref_grad.cpu())
    print(f"[N={N} {X}x{Y}x{L}] tv vs reference kernels: loss rel {e_l:.2e}, grad rel_l2 {e_g:.2e} | vs float64: ours "
          f"{abs(float(loss) - want) / want:.2e}, reference {abs(float(ref_loss) - want) / want:.2e}")
    assert e_l <= 1e-6 and e_g <= 1e-6


def _golden_case(dev):
    return _case(29, 41, 8, 6, 4, dev, 77)


def test_dump_reference_bilagrid_golden(native, ref_kernels, cuda_device, tmp_path):
    """Writes ref_bilagrid_small.npz (into $GSB_GOLDEN_OUT, else a temporary directory): the reference kernels' outputs
    on a seeded case.  The file is committed as tests/golden/ref_bilagrid_small.npz."""
    grids, img, v_out = _golden_case(cuda_device)
    x = img.clamp(0, 1).contiguous()
    ref_out = ref_kernels.slice_forward(grids[3].contiguous(), x)
    ref_vg, ref_vi = ref_kernels.slice_backward(grids[3].contiguous(), x, v_out)
    tv = ref_kernels.tv_forward(grids)
    tv_g = ref_kernels.tv_backward(grids, torch.tensor(2.5, device=cuda_device))
    out = os.environ.get("GSB_GOLDEN_OUT") or str(tmp_path)
    os.makedirs(out, exist_ok=True)
    c = lambda t: t.detach().cpu().numpy()
    np.savez_compressed(os.path.join(out, "ref_bilagrid_small.npz"), grids=c(grids), image=c(img), v_out=c(v_out),
                        image_idx=np.int32(3), slice_out=c(ref_out), slice_v_grid=c(ref_vg), slice_v_rgb=c(ref_vi),
                        tv=c(tv), tv_weight=np.float32(2.5), tv_grad=c(tv_g))


def test_slice_and_tv_vs_reference_golden(native, cuda_device):
    """The reference kernels' stored outputs (tests/golden/ref_bilagrid_small.npz) against this library."""
    gold = np.load(GOLDEN)
    t = lambda k: torch.from_numpy(gold[k]).to(cuda_device)
    grids, img, v_out, idx = t("grids"), t("image"), t("v_out"), int(gold["image_idx"])
    out, v_grids, v_img = _ours(grids, img, v_out, idx)
    _compare_slice("golden", grids[idx], img, v_out, out, v_grids[idx], v_img, t("slice_out"), t("slice_v_grid"),
                   t("slice_v_rgb"))
    loss, grad = torch.ops.gsplat_b200.bilagrid_tv(grids, torch.tensor([float(gold["tv_weight"])], device=cuda_device), True)
    e_l = abs(float(loss) - float(gold["tv"])) / abs(float(gold["tv"]))
    e_g = rel(grad.cpu(), torch.from_numpy(gold["tv_grad"]))
    print(f"[golden] tv loss rel {e_l:.2e}, grad rel_l2 {e_g:.2e}")
    assert e_l <= 1e-6 and e_g <= 1e-6


def test_reference_component_runs_on_this_library(native, cuda_device):
    """The reference's BilateralGrid (apply, tv_loss, autograd), compiled unmodified against
    include/kernels/bilateral_grid.cuh, gives what the Python mirror gives."""
    so = os.path.join(REF_DIR, "libref_bilagrid_b200.so")
    if not os.path.exists(so):
        pytest.skip("reference component harness not built (oracle/build_ref_bilagrid.py)")
    torch.ops.load_library(so)
    bil = importlib.import_module(native.__name__ + ".bilateral")
    grids = _grids(4, 12, 9, 4, 21, cuda_device)
    g = torch.Generator().manual_seed(22)
    img = (torch.rand(3, 57, 81, generator=g) * 1.4 - 0.2).to(cuda_device)
    v = torch.randn(3, 57, 81, generator=g).to(cuda_device)
    out, tv, g_grids, g_rgb = torch.ops.bilagrid_component.run(grids, img, 2, v, 3.0)
    bg = bil.BilateralGrid(4, grid_X=12, grid_Y=9, grid_L=4, device=cuda_device)
    with torch.no_grad():
        bg.grids.copy_(grids)
    x = img.clone().requires_grad_(True)
    mo = bg.apply(x, 2)
    mt = bg.tv_loss()
    ((mo * v).sum() + 3.0 * mt).backward()
    print(f"component vs mirror: out max|diff| {float((out - mo).abs().max()):.2e}, tv {float(tv):.8e} vs {float(mt):.8e}, "
          f"grad grids rel_l2 {rel(g_grids, bg.grids.grad):.2e}, grad rgb rel_l2 {rel(g_rgb, x.grad):.2e}")
    assert torch.equal(out, mo.detach())
    assert float(tv) == float(mt)
    assert rel(g_grids, bg.grids.grad) <= 1e-6
    assert rel(g_rgb, x.grad) <= 1e-7
