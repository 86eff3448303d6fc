"""Python mirror of the reference's evaluation (src/training/metrics/metrics.{hpp,cpp}), on this library's kernels:

  image_metrics      PSNR::compute and SSIM::compute of one view after the clamp (metrics.cpp:40-116, :441) as ONE kernel
                     launch (csrc/gsb_metrics.cu) writing (psnr, ssim) into a device slot: no host read
  EvalMetrics        the result struct and its formats (metrics.hpp:70-104)
  MetricsReporter    metrics.csv (one row per evaluation) and metrics_report.txt (best and final metrics), :187-289
  split_views        the validation split of CameraDataset (dataset.hpp:42-46): views with i % test_every == 0
  MetricsEvaluator   should_evaluate / evaluate / save_report (:291-530): renders every validation view under no_grad,
                     fills one [V,2] device tensor and reads it back once

Deviations from the reference, on purpose:
  * LPIPS needs the reference's TorchScript VGG weights (weights/lpips_vgg.pt), which this repository does not ship.
    Given `lpips_model_path`, the model runs as the reference runs it (inputs 2x - 1, then .mean()).  Without it the
    LPIPS column is nan and the report says "not computed", where the reference refuses to start.
  * gut=True renders through rasterize_fused (the from-world path) instead of the fastgs rasterizer, for models trained
    on that path.  The default renders through fastgs.fast_rasterize with the background composited, as the reference
    does whatever the model was trained with.
  * Evaluation images and depth maps are not written.
As in the reference, no bilateral grid and no pose correction are applied to the evaluated views."""
from __future__ import annotations

import math
import os
import time
from dataclasses import dataclass

import numpy as np
import torch

from . import _product_ns, load, rasterize_fused


def image_metrics(image: torch.Tensor, target: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """(psnr, ssim) of clamp(image, 0, 1) against target as a [2] float32 device tensor (written into `out` when given,
    e.g. one row of a [V,2] tensor).  target: [3,H,W]; image: [3,H,W] (the fastgs layout), or [H,W,3] (the from-world
    blend's, read in place); a leading batch dimension of 1 is dropped from either.  An image whose shape equals the
    target's is read as [3,H,W]."""
    load()
    if image.dim() == 4 and image.shape[0] == 1:
        image = image[0]
    if target.dim() == 4 and target.shape[0] == 1:
        target = target[0]
    hwc = tuple(image.shape) != tuple(target.shape)
    if out is None:
        out = torch.empty(2, dtype=torch.float32, device=target.device)
    _product_ns().image_metrics(image.contiguous(), target.contiguous(), hwc, out)
    return out


def _f32(v) -> float:
    return float(np.float32(v))


def _mean_f32(values) -> float:
    """std::accumulate(begin, end, 0.0f) / size(): float additions in order, then a float division."""
    s = np.float32(0.0)
    for v in values:
        s = np.float32(s + np.float32(v))
    return float(np.float32(s / np.float32(len(values))))


@dataclass
class EvalMetrics:
    """metrics.hpp:70-104.  The values are float32 like the reference's struct."""
    psnr: float = 0.0
    ssim: float = 0.0
    lpips: float = 0.0
    elapsed_time: float = 0.0
    num_gaussians: int = 0
    iteration: int = 0

    def to_string(self) -> str:
        return (f"PSNR: {_f32(self.psnr):.4f}, SSIM: {_f32(self.ssim):.4f}, LPIPS: {_f32(self.lpips):.4f}, "
                f"Time: {_f32(self.elapsed_time):.4f}s/image, #GS: {int(self.num_gaussians)}")

    @staticmethod
    def to_csv_header() -> str:
        return "iteration,psnr,ssim,lpips,time_per_image,num_gaussians"

    def to_csv_row(self) -> str:
        return (f"{int(self.iteration)},{_f32(self.psnr):.6f},{_f32(self.ssim):.6f},{_f32(self.lpips):.6f},"
                f"{_f32(self.elapsed_time):.6f},{int(self.num_gaussians)}")


def _quoted(path: str) -> str:
    """operator<< of std::filesystem::path: std::quoted, escaping '"' and '\\'."""
    return '"' + path.replace("\\", "\\\\").replace('"', '\\"') + '"'


def _best(metrics: list, better) -> EvalMetrics:
    """std::max_element / std::min_element with the reference's comparators: the first element no later one beats."""
    best = metrics[0]
    for m in metrics[1:]:
        if better(m, best):
            best = m
    return best


class MetricsReporter:
    """metrics.cpp:187-289: metrics.csv gets its header when it does not exist yet and one row per add_metrics();
    save_report() writes metrics_report.txt."""

    def __init__(self, output_dir):
        self.output_dir = str(output_dir)
        self.csv_path = os.path.join(self.output_dir, "metrics.csv")
        self.txt_path = os.path.join(self.output_dir, "metrics_report.txt")
        self.all_metrics: list[EvalMetrics] = []
        os.makedirs(self.output_dir, exist_ok=True)
        if not os.path.exists(self.csv_path):
            with open(self.csv_path, "w") as f:
                f.write(EvalMetrics.to_csv_header() + "\n")

    def add_metrics(self, m: EvalMetrics) -> None:
        self.all_metrics.append(m)
        with open(self.csv_path, "a") as f:
            f.write(m.to_csv_row() + "\n")

    def report(self) -> str:
        """The text of metrics_report.txt.  An LPIPS that was not computed (nan) reads "not computed" in the summary."""
        lines = ["==============================================",
                 "3D Gaussian Splatting Evaluation Report",
                 "==============================================",
                 f"Output Directory: {_quoted(self.output_dir)}",
                 f"Generated: {time.strftime('%Y-%m-%d %H:%M:%S', time.localtime())}", ""]
        ms = self.all_metrics
        lp = lambda v: "not computed" if math.isnan(v) else f"{_f32(v):.4f}"
        if ms:
            # metrics.cpp:236-247: the first highest PSNR and SSIM; the LPIPS line uses min_element with a '>' comparator
            bp = _best(ms, lambda a, b: b.psnr < a.psnr)
            bs = _best(ms, lambda a, b: b.ssim < a.ssim)
            bl = _best(ms, lambda a, b: a.lpips > b.lpips)
            fin = ms[-1]
            lines += ["Summary Statistics:", "------------------",
                      f"Best PSNR:  {_f32(bp.psnr):.4f} (at iteration {bp.iteration})",
                      f"Best SSIM:  {_f32(bs.ssim):.4f} (at iteration {bs.iteration})",
                      f"Best LPIPS: {lp(bl.lpips)} (at iteration {bl.iteration})", "",
                      f"Final Metrics (iteration {fin.iteration}):",
                      f"PSNR:  {_f32(fin.psnr):.4f}",
                      f"SSIM:  {_f32(fin.ssim):.4f}",
                      f"LPIPS: {lp(fin.lpips)}",
                      f"Time per image: {_f32(fin.elapsed_time):.4f} seconds",
                      f"Number of Gaussians: {fin.num_gaussians}"]
        lines += ["", "Detailed Results:", "-----------------",
                  f"{'Iteration':>10}{'PSNR':>10}{'SSIM':>10}{'LPIPS':>10}{'Time(s/img)':>15}{'#Gaussians':>15}",
                  "-" * 75]
        for m in ms:
            lines.append(f"{m.iteration:>10}{_f32(m.psnr):>10.4f}{_f32(m.ssim):>10.4f}{_f32(m.lpips):>10.4f}"
                         f"{_f32(m.elapsed_time):>15.4f}{m.num_gaussians:>15}")
        return "\n".join(lines) + "\n"

    def save_report(self) -> None:
        with open(self.txt_path, "w") as f:
            f.write(self.report())


def split_views(n: int, test_every: int = 8) -> tuple[list, list]:
    """(training, validation) view indices of CameraDataset (dataset.hpp:42-46): validation is i % test_every == 0."""
    val = [i for i in range(n) if i % test_every == 0]
    train = [i for i in range(n) if i % test_every != 0]
    return train, val


class MetricsEvaluator:
    """metrics.cpp:291-530.  `views` of evaluate() are (viewmat [4,4] world->camera, K [3,3], width, height, target
    [3,H,W] on the device); `params` is the six raw SplatData tensors a training step holds (for MCMC the [:N] views,
    so that num_gaussians is N)."""

    def __init__(self, enable_eval: bool, eval_steps, output_path, lpips_model_path: str | None = None,
                 gut: bool = False):
        self.enable_eval = bool(enable_eval)
        self.eval_steps = [int(s) for s in eval_steps]
        self.output_path = output_path
        self.gut = bool(gut)
        self.lpips = None
        self.reporter = None
        self.last_views = None  # [V,2] device tensor of the last evaluate(): per-view (psnr, ssim)
        self.last_lpips = None  # [V] device tensor of per-view LPIPS, or None
        if not self.enable_eval:
            return
        if lpips_model_path is not None:
            self.lpips = torch.jit.load(str(lpips_model_path), map_location="cuda")
            self.lpips.eval()
        self.reporter = MetricsReporter(output_path)

    def is_enabled(self) -> bool:
        return self.enable_eval

    def should_evaluate(self, iteration: int) -> bool:
        return self.enable_eval and int(iteration) in self.eval_steps

    def render(self, params: dict, sh_degree: int, view, background) -> torch.Tensor:
        """The evaluated image of one view, unclamped: [3,H,W] from fastgs with the background composited, or
        [1,H,W,3] from the from-world path (gut=True)."""
        viewmat, K, width, height = view[:4]
        P = params
        dev = P["means"].device
        w2c = torch.as_tensor(viewmat, dtype=torch.float32, device=dev).reshape(4, 4)
        with torch.no_grad():
            if self.gut:
                Kd = torch.as_tensor(K, dtype=torch.float32, device=dev).reshape(1, 3, 3)
                bg = background.reshape(1, 3) if background is not None else None
                return rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"],
                                       P["opacity_raw"], int(sh_degree), w2c[None], Kd, int(width), int(height),
                                       bg_color=bg).render_colors
            from . import fastgs as fg
            Kh = torch.as_tensor(K, dtype=torch.float32).detach().cpu().reshape(3, 3)
            st = fg.FastGSSettings(cam_position=torch.linalg.inv_ex(w2c).inverse[:3, 3].contiguous(),
                                   active_sh_bases=(int(sh_degree) + 1) ** 2, width=int(width), height=int(height),
                                   focal_x=float(Kh[0, 0]), focal_y=float(Kh[1, 1]), center_x=float(Kh[0, 2]),
                                   center_y=float(Kh[1, 2]))
            image, _ = fg.fast_rasterize(fg.default_backend(), P["means"], P["scaling_raw"], P["rotation_raw"],
                                         P["opacity_raw"].reshape(-1, 1), P["sh0"], P["shN"], w2c, st,
                                         bg_color=background)
            return image

    def evaluate(self, iteration: int, params: dict, sh_degree: int, views, background) -> EvalMetrics:
        if not self.enable_eval:
            raise RuntimeError("Evaluation is not enabled")
        views = list(views)
        if not views:
            raise ValueError("evaluate() needs at least one validation view")
        dev = params["means"].device
        start = time.perf_counter()
        per_view = torch.empty((len(views), 2), dtype=torch.float32, device=dev)
        lp = torch.empty(len(views), dtype=torch.float32, device=dev) if self.lpips is not None else None
        for v, view in enumerate(views):
            target = view[4]
            image = self.render(params, sh_degree, view, background)
            image_metrics(image, target, per_view[v])
            if lp is not None:
                with torch.no_grad():
                    pred = torch.clamp(image[0].permute(2, 0, 1) if self.gut else image, 0.0, 1.0)
                    lp[v] = self.lpips((2.0 * pred - 1.0)[None].contiguous(),
                                       (2.0 * target - 1.0)[None].contiguous()).mean()
        vals = per_view.cpu().numpy()  # the one read-back of the evaluation
        lps = lp.cpu().numpy() if lp is not None else np.full(len(views), np.nan, np.float32)
        elapsed = time.perf_counter() - start
        self.last_views, self.last_lpips = per_view, lp
        r = EvalMetrics(psnr=_mean_f32(vals[:, 0]), ssim=_mean_f32(vals[:, 1]), lpips=_mean_f32(lps),
                        elapsed_time=float(np.float32(np.float32(elapsed) / np.float32(len(views)))),
                        num_gaussians=int(params["means"].shape[0]), iteration=int(iteration))
        self.reporter.add_metrics(r)
        return r

    def save_report(self) -> None:
        if self.reporter is not None:
            self.reporter.save_report()
