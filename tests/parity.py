"""Shared comparison helpers of the GPU parity tests.

BASELINE.json's north_star asks for 1e-4 relative on rendered RGB and 1e-3 relative on gradients; "relative"
is the relative L2 error over the whole tensor.  A single whole-tensor number would let a handful of badly
wrong Gaussians pass, so every gradient comparison additionally bounds, PER GAUSSIAN,
  * the fraction of Gaussians whose own relative error exceeds `per_gauss_tol` (a floor of `floor_frac` x the
    RMS row norm keeps Gaussians with a near-zero gradient from counting), and
  * the largest absolute element error relative to the largest reference element.
The blend is only piecewise continuous (alpha >= 1/255 cut, alpha <= 0.999 gate, T <= 1e-4 stop), so a few
Gaussians with a pixel at a decision boundary legitimately differ between any two float implementations;
the bounds are set from the measured float32-vs-float64 noise of the reference formulation itself.
"""
from __future__ import annotations

import numpy as np
import torch


def rel(a, b) -> float:
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        a = torch.as_tensor(a).double()
        b = torch.as_tensor(b).double().to(a.device)
        return float((a - b).norm() / b.norm().clamp_min(1e-30))
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def to_dev(sc, dev):
    return {k: torch.from_numpy(v).to(dev) for k, v in sc.items() if isinstance(v, np.ndarray)}


def grad_metrics(got, want, n_gauss: int, per_gauss_tol: float = 1e-2, floor_frac: float = 1e-2) -> dict:
    """Whole-tensor and per-Gaussian error metrics of a gradient tensor with `n_gauss` rows."""
    g = torch.as_tensor(got).double().reshape(n_gauss, -1)
    w = torch.as_tensor(want).double().to(g.device).reshape(n_gauss, -1)
    if g.numel() == 0:  # e.g. shN of a degree-0 model
        return dict(rel=0.0, frac_bad=0.0, max_abs=0.0, n_bad=0, n_nonzero=0)
    err = (g - w).norm(dim=1)
    ref = w.norm(dim=1)
    nz = ref > 0
    rms = float(ref[nz].pow(2).mean().sqrt()) if bool(nz.any()) else 0.0
    bad = err > per_gauss_tol * (ref + floor_frac * rms)
    wmax = float(w.abs().max())
    return dict(rel=float((g - w).norm() / w.norm().clamp_min(1e-30)),
                frac_bad=float(bad.double().mean()),
                max_abs=float((g - w).abs().max()) / max(wmax, 1e-30),
                n_bad=int(bad.sum()), n_nonzero=int(nz.sum()))


def assert_grad_close(got, want, name: str, n_gauss: int, rel_tol: float = 1e-3, per_gauss_tol: float = 1e-2,
                      frac_tol: float = 2e-3, max_tol: float = 5e-2, tag: str = "") -> dict:
    m = grad_metrics(got, want, n_gauss, per_gauss_tol)
    print(f"[{tag}] {name}: rel_l2 {m['rel']:.2e}; Gaussians off by > {per_gauss_tol:g}: {m['n_bad']} "
          f"({m['frac_bad']:.2e} of {n_gauss}); max |err| / max |ref| {m['max_abs']:.2e}")
    assert m["rel"] < rel_tol, (name, m)
    assert m["frac_bad"] < frac_tol, (name, m)
    assert m["max_abs"] < max_tol, (name, m)
    return m
