"""GPU: the scalar staging fall-backs of the kernels that load their inputs with TMA bulk copies when the data allows it.

fused_front / fused_back (gsb_fused.cu) and fgs_front / fgs_back (gsb_fastgs.cu) move each 128-Gaussian slab of shN rows
between global and shared memory with one bulk copy when the slab starts 16-byte aligned and holds a whole number of
16-byte words, and with a per-thread copy loop otherwise.  At K = 16 a row is 45 floats, so after a densification or a
prune leaves N % 4 != 0 the last slab takes the copy loop; a contiguous view at a 4-byte offset takes it in every slab.
The SH operator (gsb_sh.cu) and the one-launch Adam step (gsb_optim.cu) have the same kind of dispatch.  Each case below
states the path it selects, proves the selection from the kernel's own rule, and compares the result with the bulk path
(bitwise where only the staging differs) and with an independent computation (the unfused operator sequence, the float64
oracle, or the reference's fastgs kernels)."""
import math

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel, to_dev
from test_gpu_fastgs import PARAMS, _fg, _settings, _weights, grads_close, image_close, reference, run
from test_gpu_fused import RAW, compare, raw_leaves, run_pair

pytestmark = pytest.mark.gpu
SLAB = 128  # kFusedThreads (gsb_fused.cu:28) == kFgsThreads: one CTA stages one slab of rows


# ---------------------------------------------------------------------------------------------------------------------
# the selection rule, stated once
# ---------------------------------------------------------------------------------------------------------------------
def slab_paths(shN):
    """The staging path of every 128-row slab of `shN` [N, R, 3] in fused_front_kernel / fused_back_kernel
    (gsb_fused.cu:105-109, 179-187) and fgs_front_kernel / fgs_back_kernel (gsb_fastgs.cu:179-183, 315-323): a bulk
    (TMA) copy when the slab's first row is 16-byte aligned and cnt * R * 3 is a multiple of 4, the copy loop otherwise."""
    N = shN.shape[0]
    rowf = shN[0].numel() if N else 0
    paths = []
    for g0 in range(0, N, SLAB):
        n_floats = min(SLAB, N - g0) * rowf
        paths.append("bulk" if (shN.data_ptr() + 4 * g0 * rowf) % 16 == 0 and n_floats % 4 == 0 else "scalar")
    return paths


def assert_ragged(shN):
    N, rowf = shN.shape[0], shN[0].numel()
    assert (N % SLAB or SLAB) * rowf % 4 != 0
    assert slab_paths(shN)[-1] == "scalar"


def assert_offset(shN):
    assert shN.data_ptr() % 16 != 0 and shN.is_contiguous()
    assert set(slab_paths(shN)) == {"scalar"}


def assert_bulk(shN):
    assert shN.data_ptr() % 16 == 0 and set(slab_paths(shN)) == {"bulk"}


def describe(tag, shN, N, K, offset=0):
    p = slab_paths(shN)
    print(f"[{tag}] N={N} K={K} offset={offset} floats: {p.count('bulk')} bulk + {p.count('scalar')} scalar slabs, "
          f"last slab {p[-1] if p else '-'}")


def last_slab(N):
    return (N - 1) // SLAB * SLAB


def offset_leaf(values, o):
    """A contiguous view `buf[o : o + n].view(shape)` of a leaf buffer holding `values`, and the buffer."""
    n = values.numel()
    buf = torch.zeros(o + n + 7, device=values.device)
    buf[o:o + n] = values.detach().reshape(-1)
    buf.requires_grad_(True)
    return buf[o:o + n].view(values.shape), buf


def behind_camera(viewmat, r, rng):
    """r world points that sit behind a camera with world-to-camera matrix `viewmat` [4, 4]."""
    R, t = viewmat[:3, :3].astype(np.float64), viewmat[:3, 3].astype(np.float64)
    pc = np.stack([rng.random(r) - 0.5, rng.random(r) - 0.5, -1.0 - rng.random(r)], -1)
    return ((pc - t) @ R).astype(np.float32)  # R^T (p_c - t), row-wise


# ---------------------------------------------------------------------------------------------------------------------
# 1. fused path: ragged last slab
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_scene(N):
    return scenes.scene_small(N=N, width=200, height=120, view=1)  # the scene of test_fused_vs_cpu_oracle at N = 3000


def _append_culled(sc, r, seed=0):
    rng = np.random.default_rng(seed)
    out = dict(sc)
    K = sc["sh_coeffs"].shape[1]
    q = rng.standard_normal((r, 4)).astype(np.float32)
    add = dict(means=behind_camera(sc["viewmats"][0], r, rng), quats=q / np.linalg.norm(q, axis=-1, keepdims=True),
               scales=np.full((r, 3), 0.1, np.float32), opacities=np.full(r, 0.8, np.float32),
               sh_coeffs=((rng.random((r, K, 3)) - 0.5) * 0.3).astype(np.float32))
    for k, v in add.items():
        out[k] = np.concatenate([sc[k], v])
    return out


def _fused(native, sc, deg, dev, shN_offset=None):
    t = to_dev(sc, dev)
    W, H = sc["width"], sc["height"]
    g = torch.Generator(device=dev).manual_seed(3)
    vr = torch.randn((1, H, W, 3), device=dev, generator=g)
    va = torch.randn((1, H, W, 1), device=dev, generator=g)
    P = raw_leaves(native, t, None)
    shN, buf = P["shN"], None
    if shN_offset is not None:
        shN, buf = offset_leaf(P["shN"], shN_offset)
    o = native.rasterize_fused(P["means"], P["sh0"], shN, P["scaling_raw"], P["rotation_raw"], P["opacity_raw"], deg,
                               t["viewmats"], t["Ks"], W, H, bg_color=t["background"])
    ((o.render_colors * vr).sum() + (o.alpha * va).sum()).backward()
    torch.cuda.synchronize()
    grads = {k: (P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])) for k in RAW}
    if buf is not None:
        n = shN.numel()
        grads["shN"] = buf.grad[shN_offset:shN_offset + n].view(shN.shape)
    return dict(o=o, shN=shN, buf=buf, grads=grads)


@pytest.mark.parametrize("r", [1, 2, 3])
def test_fused_appended_culled_rows_scalar_last_slab(native, cuda_device, r):
    base_sc = _oracle_scene(3000)
    sc = _append_culled(base_sc, r, seed=r)
    base = _fused(native, base_sc, 3, cuda_device)
    got = _fused(native, sc, 3, cuda_device)
    N0, N = 3000, 3000 + r
    assert_bulk(base["shN"])  # the last slab of 56 rows is 2520 floats: bulk
    assert_ragged(got["shN"])
    describe("fused appended culled", got["shN"], N, 16)
    vis = (got["o"].radii[0] > 0).all(-1)
    assert not vis[N0:].any()  # the appended rows are culled ...
    assert vis[last_slab(N):].any()  # ... but the scalar-staged slab holds visible Gaussians
    a, b = got["o"], base["o"]
    # staging changes no arithmetic (gsb_fused.cu is built with -fmad=false): the forward is bitwise the same
    assert torch.equal(a.render_colors, b.render_colors) and torch.equal(a.alpha, b.alpha)
    assert torch.equal(a.n_isects, b.n_isects)
    assert torch.equal(a.radii[:, :N0], b.radii) and torch.equal(a.means2d[:, :N0], b.means2d)
    assert torch.equal(a.depths[:, :N0], b.depths)
    for k in RAW:
        # the blend backward sums with float atomics: order-dependent in the last bits only
        e = rel(got["grads"][k][:N0], base["grads"][k])
        print(f"[fused appended culled r={r}] {k}: rel {e:.2e}")
        assert e < 1e-5, (k, e)
        assert not got["grads"][k][N0:].any(), k


def _k_scene(N, K, seed):
    if N <= 3:  # by hand, in view of the identity camera
        sc = scenes.scene_small(N=N, width=160, height=96)
        sc["means"] = np.array([[0.0, 0.0, 3.0], [0.3, 0.1, 2.5], [-0.2, -0.1, 3.5]], np.float32)[:N]
        sc["scales"] = np.array([[0.16, 0.05, 0.1], [0.06, 0.12, 0.08], [0.1, 0.04, 0.14]], np.float32)[:N]
    else:
        sc = scenes.scene_small(N=N, width=160, height=96, view=2)
    rng = np.random.default_rng(seed)
    sc["sh_coeffs"] = ((rng.random((N, K, 3), dtype=np.float32) - 0.5) * 0.6).astype(np.float32)
    return sc


RAGGED = ([(N, 16, 3) for N in (1, 3, 127, 129, 3001, 3003)] +
          [(N, K, deg) for K, deg in ((16, 2), (16, 1), (16, 0), (4, 1), (2, 0)) for N in (129, 3001)])


@pytest.mark.parametrize("N,K,deg", RAGGED)
def test_fused_ragged_counts_vs_unfused(native, cuda_device, N, K, deg):
    """The unfused sequence computes the colour with the SH operator, whose staging is independent of the fused
    kernels'."""
    sc = _k_scene(N, K, seed=N * 31 + K * 7 + deg)
    out = run_pair(native, sc, cuda_device, deg)
    P = raw_leaves(native, to_dev(sc, cuda_device), None, requires_grad=False)
    assert_ragged(P["shN"])
    describe(f"fused ragged deg={deg}", P["shN"], N, K)
    assert bool((out["fused"]["radii"][0, last_slab(N):] > 0).all(-1).any())
    compare(out, N, f"ragged N={N} K={K} deg={deg}")
    # the rows of the scalar-staged slab alone: the whole-tensor bound would let a wrong last slab through
    s = slice(last_slab(N), None)
    assert_grad_close(out["fused"]["grads"]["shN"][s], out["unfused"]["grads"]["shN"][s], "shN (last slab)",
                      N - last_slab(N), rel_tol=2e-4, tag=f"ragged N={N} K={K} deg={deg} fused vs unfused")
    g = out["fused"]["grads"]["shN"]
    if deg < 3 and K > (deg + 1) ** 2:  # inactive degrees get exact zeros (gsb_fused.cu:264-267), copy loop included
        assert not g[:, (deg + 1) ** 2 - 1:].any()
    if deg == 0:  # rows are written but never read
        assert not g.any()


def test_fused_ragged_vs_cpu_oracle(native, orc, cuda_device):
    sc = _oracle_scene(3001)
    W, H = sc["width"], sc["height"]
    rng = np.random.default_rng(4)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    ref = orc.render_pipeline(sc, "f32", True, vrc, vra)
    t = to_dev(sc, cuda_device)
    P = raw_leaves(native, t, None)
    assert_ragged(P["shN"])
    describe("fused ragged vs oracle", P["shN"], 3001, 16)
    o = native.rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"], 3,
                               t["viewmats"], t["Ks"], W, H, bg_color=t["background"])
    assert bool((o.radii[0, last_slab(3001):] > 0).all(-1).any())
    assert abs(int(o.n_isects.item()) - len(ref["flatten_ids"])) <= 8
    ((o.render_colors * torch.from_numpy(vrc).to(cuda_device)).sum() +
     (o.alpha * torch.from_numpy(vra).to(cuda_device)).sum()).backward()
    assert rel(o.render_colors.detach().cpu().numpy(), ref["renders"]) < 1e-4
    op = sc["opacities"].astype(np.float64)
    want = {"means": ref["v_means"] + ref["v_dirs"][0], "sh0": ref["v_sh_coeffs"][:, :1], "shN": ref["v_sh_coeffs"][:, 1:],
            "scaling_raw": ref["v_scales"] * sc["scales"], "rotation_raw": ref["v_quats"],
            "opacity_raw": (ref["v_opacities"][0] * op * (1 - op))[:, None]}
    for k, w in want.items():
        assert_grad_close(P[k].grad, w, k, 3001, tag="fused ragged vs CPU oracle")
    # the rows of the scalar-staged slab alone: the whole-tensor bound would let a wrong last slab through
    s = slice(last_slab(3001), None)
    assert_grad_close(P["shN"].grad[s], want["shN"][s], "shN (last slab)", 3001 - last_slab(3001),
                      tag="fused ragged vs CPU oracle")


# ---------------------------------------------------------------------------------------------------------------------
# 2. fused path: shN as an offset view
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [3000, 3001])
@pytest.mark.parametrize("K,deg", [(16, 3), (9, 2), (25, 4)])
@pytest.mark.parametrize("o", [1, 2, 3, 4])
def test_fused_offset_shN(native, cuda_device, N, K, deg, o):
    sc = _k_scene(N, K, seed=K + deg)
    aligned = _fused(native, sc, deg, cuda_device)
    view = _fused(native, sc, deg, cuda_device, shN_offset=o)
    sv = view["shN"]
    if o == 4:  # control: bulk in every slab but a ragged last one, as for the aligned tensor
        assert sv.data_ptr() % 16 == 0 and set(slab_paths(sv)[:-1]) == {"bulk"}
        assert slab_paths(sv) == slab_paths(aligned["shN"])
    else:  # the copy loop in, the bulk copy out (the shim allocates v_shN aligned)
        assert_offset(sv)
    describe(f"fused offset deg={deg}", sv, N, K, o)
    a, b = view["o"], aligned["o"]
    assert torch.equal(a.render_colors, b.render_colors) and torch.equal(a.alpha, b.alpha)
    assert torch.equal(a.radii, b.radii) and torch.equal(a.n_isects, b.n_isects)
    for k in RAW:
        e = rel(view["grads"][k], aligned["grads"][k])
        assert e < 1e-5, (k, e)  # float atomics in the blend backward
    assert view["grads"]["shN"].any()
    g = view["buf"].grad
    n = sv.numel()
    assert not g[:o].any() and not g[o + n:].any()


# ---------------------------------------------------------------------------------------------------------------------
# 3. fastgs path: the same checks
# ---------------------------------------------------------------------------------------------------------------------
def _prim_rows(buf, N):
    """Per-Gaussian regions of the forward's per-primitive buffer (gsb_fastgs.cu:492-510, 256-byte aligned pieces in a
    256-byte aligned block; the moments are left out: the forward zeroes them) as [N, bytes per row] uint8 views."""
    base = (-buf.data_ptr()) % 256
    out, b = {}, 0
    for name, width in (("recs", 64), ("moments", 64), ("counts", 4), ("boxes", 8), ("masks", 4), ("depths", 4),
                        ("filt0", 16), ("filt1", 8)):
        o = (b + 255) // 256 * 256
        b = o + N * width
        if name != "moments":
            out[name] = buf[base + o:base + b].view(N, width)
    return out


def _fgs(fg, inp, dev, gi, ga, shN_offset=None):
    """fast_rasterize with densification_info, plus the backend's forward buffers on the same inputs."""
    P = {k: torch.from_numpy(np.ascontiguousarray(inp[k])).to(dev).requires_grad_(True) for k in PARAMS}
    shN, buf = P["shN"], None
    if shN_offset is not None:
        shN, buf = offset_leaf(P["shN"], shN_offset)
    w2c = torch.from_numpy(inp["w2c"]).to(dev)
    s = _settings(fg, inp, dev)
    N = P["means"].shape[0]
    dens = torch.zeros((2, N), device=dev)
    image, alpha = fg.fast_rasterize(fg.default_backend(), P["means"], P["scales_raw"], P["rotations_raw"],
                                     P["opacities_raw"], P["sh0"], shN, w2c, s, densification_info=dens)
    ((image * gi).sum() + (alpha * ga).sum()).backward()
    with torch.no_grad():
        _, _, ctx = fg.default_backend().forward(P["means"], P["scales_raw"], P["rotations_raw"], P["opacities_raw"],
                                                 P["sh0"], shN, w2c, s)
    torch.cuda.synchronize()
    grads = {k: P[k].grad for k in PARAMS}
    if buf is not None:
        grads["shN"] = buf.grad[shN_offset:shN_offset + shN.numel()].view(shN.shape)
    return dict(image=image.detach(), alpha=alpha.detach(), grads=grads, dens=dens, shN=shN, buf=buf,
                prim=_prim_rows(ctx["buffers"][0], N), n_inst=int(ctx["ints"][1]))


def _fgs_inputs(N, rest_plus_1=16, active=16, seed=0):
    sc = scenes.scene_small(N=N, width=200, height=120, sh_degree=3, seed=11, view=1)
    if rest_plus_1 != 16:
        rng = np.random.default_rng(seed)
        sc["sh_coeffs"] = ((rng.random((N, rest_plus_1, 3), dtype=np.float32) - 0.5) * 0.6).astype(np.float32)
    inp = scenes.fastgs_inputs(sc)
    inp["active_sh_bases"] = active
    return inp


@pytest.mark.parametrize("r", [1, 2, 3])
def test_fastgs_appended_culled_rows_scalar_last_slab(native, cuda_device, r):
    fg = _fg(native)
    inp0 = _fgs_inputs(3000)
    rng = np.random.default_rng(r)
    inp = dict(inp0)
    add = dict(means=behind_camera(inp0["w2c"], r, rng), scales_raw=np.full((r, 3), np.log(0.1), np.float32),
               rotations_raw=np.tile(np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), (r, 1)),
               opacities_raw=np.full((r, 1), 1.5, np.float32), sh0=rng.standard_normal((r, 1, 3)).astype(np.float32),
               shN=rng.standard_normal((r, 15, 3)).astype(np.float32))
    for k, v in add.items():
        inp[k] = np.concatenate([inp0[k], v])
    gi, ga = _weights(inp0, cuda_device, 11)
    base = _fgs(fg, inp0, cuda_device, gi, ga)
    got = _fgs(fg, inp, cuda_device, gi, ga)
    N0, N = 3000, 3000 + r
    assert_bulk(base["shN"])
    assert_ragged(got["shN"])
    describe("fastgs appended culled", got["shN"], N, 16)
    assert bool((got["dens"][0, last_slab(N):N0] > 0).any())  # the scalar-staged slab holds visible primitives
    assert torch.equal(got["image"], base["image"]) and torch.equal(got["alpha"], base["alpha"])
    assert got["n_inst"] == base["n_inst"]
    for name, rows in got["prim"].items():
        assert torch.equal(rows[:N0], base["prim"][name]), name
    for k in PARAMS:
        e = rel(got["grads"][k][:N0], base["grads"][k])
        print(f"[fastgs appended culled r={r}] {k}: rel {e:.2e}")
        assert e < 1e-5, (k, e)  # float atomics in the blend backward
        assert not got["grads"][k][N0:].any(), k
    assert torch.equal(got["dens"][0, :N0], base["dens"][0]) and rel(got["dens"][1, :N0], base["dens"][1]) < 1e-5
    assert not got["dens"][:, N0:].any()


@pytest.mark.parametrize("N", [129, 3001])
@pytest.mark.parametrize("active", [4, 16])
def test_fastgs_ragged_counts_vs_reference(native, cuda_device, N, active):
    fg = _fg(native)
    inp = _fgs_inputs(N, active=active)
    shN = torch.from_numpy(inp["shN"]).to(cuda_device)
    assert_ragged(shN)
    describe(f"fastgs ragged active={active}", shN, N, 16)
    gi, ga = _weights(inp, cuda_device, 12)
    d1 = torch.zeros((2, N), device=cuda_device)
    d2 = torch.zeros((2, N), device=cuda_device)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga, dens=d1)
    ref = reference(native, inp, cuda_device, gi, ga, dens=d2)
    assert bool((d1[0, last_slab(N):] > 0).any())
    image_close(mine, ref, f"ragged N={N} active {active}, b200 vs reference")
    grads_close(mine, ref, N, f"ragged N={N} active {active}")
    s = slice(last_slab(N), None)
    assert_grad_close(mine["grads"]["shN"][s], ref["grads"]["shN"][s], "shN (last slab)", N - last_slab(N),
                      tag=f"ragged N={N} active {active}")
    assert not mine["grads"]["shN"][:, active - 1:].any()


@pytest.mark.parametrize("N", [3000, 3001])
@pytest.mark.parametrize("bases,active", [(16, 16), (9, 9), (25, 16)])
@pytest.mark.parametrize("o", [1, 2, 3, 4])
def test_fastgs_offset_shN(native, cuda_device, N, bases, active, o):
    fg = _fg(native)
    inp = _fgs_inputs(N, bases, active, seed=bases)
    gi, ga = _weights(inp, cuda_device, 13)
    aligned = _fgs(fg, inp, cuda_device, gi, ga)
    view = _fgs(fg, inp, cuda_device, gi, ga, shN_offset=o)
    sv = view["shN"]
    if o == 4:
        assert sv.data_ptr() % 16 == 0 and set(slab_paths(sv)[:-1]) == {"bulk"}
    else:
        assert_offset(sv)
    describe(f"fastgs offset active={active}", sv, N, bases, o)
    assert torch.equal(view["image"], aligned["image"]) and torch.equal(view["alpha"], aligned["alpha"])
    for name, rows in view["prim"].items():
        assert torch.equal(rows, aligned["prim"][name]), name
    for k in PARAMS:
        e = rel(view["grads"][k], aligned["grads"][k])
        assert e < 1e-5, (k, e)
    assert view["grads"]["shN"].any()
    assert torch.equal(view["dens"][0], aligned["dens"][0]) and rel(view["dens"][1], aligned["dens"][1]) < 1e-5
    g = view["buf"].grad
    assert not g[:o].any() and not g[o + sv.numel():].any()


# ---------------------------------------------------------------------------------------------------------------------
# 4. the SH operator and the one-launch Adam step
# ---------------------------------------------------------------------------------------------------------------------
def max_ulp(a, b):
    """Largest distance in units in the last place between two float32 tensors."""
    def ordered(x):
        i = x.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return int((ordered(a) - ordered(b)).abs().max()) if a.numel() else 0


def sh_k16_path(coeffs, v_coeffs=None, degree=3, fwd=True):
    """gsb_sh_fwd / gsb_sh_bwd / sh_bwd_views_launch (gsb_sh.cu:409, 439, 472): the K = 16 row kernels take degrees
    1-3 forward, 0-3 backward, and need coeffs (and v_coeffs) 16-byte aligned; the generic kernel does the rest."""
    ok = coeffs.shape[-2] == 16 and (1 <= degree <= 3 if fwd else degree <= 3) and coeffs.data_ptr() % 16 == 0
    return ok and (v_coeffs is None or v_coeffs.data_ptr() % 16 == 0)


@pytest.mark.parametrize("K,deg", [(16, 0), (16, 1), (16, 2), (16, 3), (4, 1)])
def test_sh_offset_coeffs_take_the_generic_kernel(native, orc, cuda_device, K, deg):
    """The generic kernel's own 128-bit row loads (K * 3 and the active floats multiples of 4) must not be taken either."""
    rng = np.random.default_rng(50 + deg)
    M = 1501
    dirs = rng.standard_normal((M, 3)).astype(np.float32)
    coeffs = rng.standard_normal((M, K, 3)).astype(np.float32)
    vcol = rng.standard_normal((M, 3)).astype(np.float32)
    masks = rng.random(M) > 0.3
    d, c, v, m = (torch.from_numpy(x).to(cuda_device) for x in (dirs, coeffs, vcol, masks))
    cv, _ = offset_leaf(c, 1)
    cv = cv.detach()
    assert cv.data_ptr() % 16 != 0 and cv.is_contiguous() and not sh_k16_path(cv, degree=deg)
    assert sh_k16_path(c, degree=deg) == (K == 16 and deg >= 1)
    col = native.spherical_harmonics_fwd(deg, d, cv, m)
    col_al = native.spherical_harmonics_fwd(deg, d, c, m)
    np.testing.assert_allclose(col.cpu().numpy()[masks], orc.sh_fwd(deg, dirs, coeffs, masks)[masks], rtol=1e-4, atol=1e-4)
    v_coeffs, v_dirs = native.spherical_harmonics_bwd(K, deg, d, cv, m, v, True)
    assert not sh_k16_path(cv, v_coeffs, deg, fwd=False) and v_coeffs.data_ptr() % 16 == 0
    rc, rd = orc.sh_bwd(deg, dirs, coeffs, masks, vcol)
    np.testing.assert_allclose(v_coeffs.cpu().numpy(), rc, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(v_dirs.cpu().numpy(), rd, rtol=1e-4, atol=2e-4)
    vc_al, vd_al = native.spherical_harmonics_bwd(K, deg, d, c, m, v, True)
    assert sh_k16_path(c, vc_al, deg, fwd=False) == (K == 16)
    print(f"[sh deg={deg} M={M} K={K} offset=1 float: generic kernel; aligned: "
          f"{'K=16 row' if sh_k16_path(c, degree=deg) else 'generic'} fwd, {'K=16 row' if K == 16 else 'generic'} bwd] "
          f"max ULP vs aligned: "
          f"colors {max_ulp(col[m], col_al[m])}, v_coeffs {max_ulp(v_coeffs, vc_al)}, v_dirs {max_ulp(v_dirs, vd_al)}")


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_sh_bwd_views_offset_coeffs(native, orc, cuda_device, deg):
    rng = np.random.default_rng(70 + deg)
    M, V, K = 1501, 3, 16
    means = rng.standard_normal((M, 3)).astype(np.float32) * 3
    campos = rng.standard_normal((V, 3)).astype(np.float32) * 6
    coeffs = rng.standard_normal((M, K, 3)).astype(np.float32)
    vc = rng.standard_normal((V, M, 3)).astype(np.float32)
    vc[rng.random((V, M)) < 0.5] = 0.0
    vm0 = rng.standard_normal((M, 3)).astype(np.float32)
    want_c = np.zeros_like(coeffs, dtype=np.float64)
    want_m = vm0.astype(np.float64)
    for i in range(V):
        a, b = orc.sh_bwd(deg, means - campos[i], coeffs, None, vc[i], True, precision="f64")
        want_c += a
        want_m += b
    d = lambda x: torch.from_numpy(x).to(cuda_device)
    be = native.default_backend()
    cv, _ = offset_leaf(d(coeffs), 3)
    cv = cv.detach()
    assert cv.data_ptr() % 16 != 0 and cv.is_contiguous()
    vm = d(vm0.copy())
    got = be.spherical_harmonics_bwd_views(deg, d(means), d(campos), cv, d(vc), vm)
    assert not sh_k16_path(cv, got, deg, fwd=False)
    assert rel(got.cpu().numpy(), want_c) < 1e-5
    assert rel(vm.cpu().numpy(), want_m) < 1e-5
    vm_al = d(vm0.copy())
    got_al = be.spherical_harmonics_bwd_views(deg, d(means), d(campos), d(coeffs), d(vc), vm_al)
    assert sh_k16_path(d(coeffs), got_al, deg, fwd=False)
    print(f"[sh_bwd_views deg={deg} M={M} V={V} K={K} offset=3 floats: generic kernel] max ULP vs aligned: "
          f"v_coeffs {max_ulp(got, got_al)}, v_means {max_ulp(vm, vm_al)}")


def _adam_groups(dev, sizes, offsets, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for n, o in zip(sizes, offsets):
        four = []
        for j in range(4):
            x = torch.randn(n, device=dev, generator=g)
            if j == 3:
                x = x.abs()  # exp_avg_sq >= 0
            if o:
                buf = torch.zeros(n + o + 3, device=dev)
                buf[o:o + n] = x
                x = buf[o:o + n]
            four.append(x)
        out.append(four)  # param, grad, exp_avg, exp_avg_sq
    return out


def _vector_copies(groups):
    """The same values in 16-byte aligned buffers padded to a multiple of four: every element takes the float4 body."""
    out = []
    for four in groups:
        n = four[0].numel()
        cp = []
        for x in four:
            y = torch.zeros((n + 3) // 4 * 4, device=x.device)
            y[:n] = x
            cp.append(y)
        out.append(cp)
    return out


def adam_group_vec(four):
    """adam_multi_kernel (gsb_optim.cu:52, 101-103): a group takes the float4 body where all four of its pointers are
    16-byte aligned and a whole float4 is left, the scalar loop otherwise."""
    return all(x.data_ptr() % 16 == 0 for x in four)


@pytest.mark.parametrize("dynamic", [False, True])
def test_adam_scalar_and_vector_bodies_agree(native, cuda_device, dynamic):
    dev = cuda_device
    ns = native.ops()
    sizes = [3003, 1001, 4000, 4001, 4002, 4003]  # an offset group, then aligned groups with n % 4 = 0, 1, 2, 3
    offsets = [1, 2, 0, 0, 0, 0]
    if dynamic:  # a zero-size group and a disabled group keep their rows of the scalar table
        sizes += [0, 1003]
        offsets += [0, 0]
    groups = _adam_groups(dev, sizes, offsets, seed=17 + dynamic)
    vec = _vector_copies(groups)
    ref0 = [[x.double().clone() for x in four] for four in groups]
    assert not adam_group_vec(groups[0]) and not adam_group_vec(groups[1])
    assert all(adam_group_vec(f) for f in groups[2:]) and all(adam_group_vec(f) for f in vec)
    for i, (n, o) in enumerate(zip(sizes, offsets)):
        path = "scalar" if not adam_group_vec(groups[i]) else ("float4" if n % 4 == 0 else "float4 + scalar tail")
        print(f"[adam {'dynamic' if dynamic else 'host'} scalars] group {i}: n={n} (n % 4 = {n % 4}) offset={o} floats: {path}")
    b1, b2, eps = 0.9, 0.999, 1e-15
    lrs = [1e-3 * (i + 1) for i in range(len(sizes))]
    steps = [1 + 3 * i for i in range(len(sizes))]
    bc1 = [float(np.float32(1.0 / (1.0 - b1 ** t))) for t in steps]
    bc2 = [float(np.float32(1.0 / math.sqrt(1.0 - b2 ** t))) for t in steps]
    enabled = [1.0] * len(sizes)
    if dynamic:
        enabled[-1] = 0.0
        table = torch.tensor([[lrs[i], bc1[i], bc2[i], enabled[i]] for i in range(len(sizes))], device=dev)
        assert table.data_ptr() % 16 == 0
    for gs in (groups, vec):
        p, gr, m, v = (list(x) for x in zip(*gs))
        if dynamic:
            ns.fused_adam_step_dynamic(p, gr, m, v, table, b1, b2, eps)
        else:
            ns.fused_adam_step(p, gr, m, v, lrs, b1, b2, eps, steps)
    torch.cuda.synchronize()
    for i, n in enumerate(sizes):
        for j in (0, 2, 3):
            assert torch.equal(groups[i][j], vec[i][j][:n]), (i, j)
        p, gr, m, v = ref0[i]
        if not enabled[i]:
            assert torch.equal(groups[i][0].double(), p) and torch.equal(groups[i][2].double(), m), i
            continue
        # the float64 formula of test_fused_adam_matches_reference_formula, with the kernel's float32 coefficients
        fb1, fb2 = float(np.float32(b1)), float(np.float32(b2))
        ob1, ob2 = float(np.float32(1) - np.float32(b1)), float(np.float32(1) - np.float32(b2))
        m1 = fb1 * m + ob1 * gr
        m2 = fb2 * v + ob2 * gr * gr
        want = p - float(np.float32(lrs[i])) * bc1[i] * m1 / (m2.sqrt() * bc2[i] + float(np.float32(eps)))
        if n:
            assert rel(groups[i][0], want) < 1e-6, i
            assert rel(groups[i][2], m1) < 1e-6 and rel(groups[i][3], m2) < 1e-6, i
