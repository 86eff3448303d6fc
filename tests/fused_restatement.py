"""Float64 restatement of the fused raw-parameter render path (rasterize_fused; csrc/gsb_fused.cu), the yardstick of
tests/test_gpu_fused_oracle.py.

Training holds the RAW SplatData tensors; the reference activates them with torch (splat_data.cpp:267-286) before
gs::training::rasterize, which applies the viewer's scaling modifier to the scales:

  scale   = exp(scaling_raw) * scaling_modifier
  opacity = sigmoid(opacity_raw)
  quat    = rotation_raw / |rotation_raw|
  sh      = cat(sh0, shN), of which the colour reads the first (deg + 1)^2 rows
  dirs    = means - campos (the SH view direction)

The forward and the gradients of the activated parameters come from oracle.render_pipeline in float64.  They are
chained to the raw parameters here, in float64, by hand:

  d/d scaling_raw  = v_scale * scale                              (the activated scale, modifier included)
  d/d opacity_raw  = v_opacity * opacity (1 - opacity)
  d/d rotation_raw = (I - q^ q^T) v_quat / |q|,  q^ = q / |q|
  d/d sh0, shN     = the rows of v_sh, zero beyond (deg + 1)^2
  d/d means        = v_means + v_dirs

The clamp of the colour, clamp_min(colour + 0.5, 0) (rasterizer.cpp:266), passes its gradient where colour + 0.5 >= 0:
that is torch's clamp_min backward, which the reference's autograd runs, and the kernel's rule (gsb_fused.cu).
oracle.backward_pipeline applies the same inclusive mask; test_fused_restatement.py pins it at a colour of exactly
-0.5.
"""
from __future__ import annotations

import numpy as np

RAW = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")


def activate(raw: dict, scaling_modifier: float = 1.0) -> dict:
    """The activated parameters of `raw` (numpy; sh0 [N,1,3], shN [N,K-1,3], opacity_raw [N,1]) in float64."""
    q = np.asarray(raw["rotation_raw"], np.float64)
    return dict(means=np.asarray(raw["means"], np.float64),
                quats=q / np.linalg.norm(q, axis=-1, keepdims=True),
                scales=np.exp(np.asarray(raw["scaling_raw"], np.float64)) * scaling_modifier,
                opacities=1.0 / (1.0 + np.exp(-np.asarray(raw["opacity_raw"], np.float64)[:, 0])),
                sh_coeffs=np.concatenate([np.asarray(raw["sh0"], np.float64), np.asarray(raw["shN"], np.float64)], 1))


def chain_to_raw(raw: dict, grads: dict, sh_degree: int, scaling_modifier: float = 1.0) -> dict:
    """Gradients of the raw parameters from those of the activated ones: v_means, v_quats, v_scales [N,3],
    v_opacities [N], v_sh_coeffs [N,K,3] and v_dirs [N,3], all float64."""
    act = activate(raw, scaling_modifier)
    q = np.asarray(raw["rotation_raw"], np.float64)
    qn, inv = act["quats"], 1.0 / np.linalg.norm(q, axis=-1, keepdims=True)
    vq = np.asarray(grads["v_quats"], np.float64)
    o = act["opacities"]
    v_sh = np.array(grads["v_sh_coeffs"], np.float64)
    v_sh[:, (sh_degree + 1) ** 2:] = 0.0  # inactive degrees: the colour does not read them
    return {"means": np.asarray(grads["v_means"], np.float64) + np.asarray(grads["v_dirs"], np.float64),
            "sh0": v_sh[:, :1], "shN": v_sh[:, 1:],
            "scaling_raw": np.asarray(grads["v_scales"], np.float64) * act["scales"],
            "rotation_raw": (vq - (vq * qn).sum(-1, keepdims=True) * qn) * inv,
            "opacity_raw": (np.asarray(grads["v_opacities"], np.float64) * o * (1.0 - o))[:, None]}


def render_raw(orc, raw: dict, sh_degree: int, viewmats, Ks, width: int, height: int, background, v_render_colors,
               v_render_alphas, scaling_modifier: float = 1.0, precision: str = "f64", **camera) -> tuple[dict, dict]:
    """rasterize_fused on the oracle: (render_pipeline's output, the raw-parameter gradients).  `camera`: camera_model,
    radial, tangential, thin_prism as render_pipeline takes them.  The activated parameters reach the oracle rounded
    to float32, as they reach the kernels."""
    act = activate(raw, scaling_modifier)
    scene = {k: v.astype(np.float32) for k, v in act.items()}
    scene.update(sh_degree=sh_degree, viewmats=viewmats, Ks=Ks, width=width, height=height, tile_size=16,
                 background=background)
    out = orc.render_pipeline(scene, precision, True, v_render_colors, v_render_alphas, **camera)
    grads = dict(v_means=out["v_means"], v_quats=out["v_quats"], v_scales=out["v_scales"],
                 v_opacities=out["v_opacities"][0], v_sh_coeffs=out["v_sh_coeffs"], v_dirs=out["v_dirs"][0])
    return out, chain_to_raw(raw, grads, sh_degree, scaling_modifier)
