#!/usr/bin/env python
"""bench.py -- Gaussians rasterized/sec (fwd+bwd) on BASELINE.json configs[1] (and configs[4] for N>1).

One "step" = one pass of the hot path over one view of the synthetic scene:
  projection_ut -> SH fwd -> intersect_tile/offset -> blend fwd -> L1 loss grad -> blend bwd -> SH bwd
through the reference-facing API (the gsplat:: shim, driven by the L3 mirror in the package),
exactly the call sequence of gs::training::rasterize + loss.backward() (SURVEY.md section 3.2/3.3).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference] [--config B|D|A]

What the N=1 line carries (BASELINE.md 2.1-2.4):
  value / ms_per_step      EXACTLY K steps, device-resident inputs, CUDA events, barrier + synchronize on both sides
  distribution             20 warm-up + 100 individually timed steps: median / p10 / p90
  ops_ms                   per-operator CUDA-event times of BOTH libraries (this backend and the reference's own
                           gsplat CUDA kernels built unmodified in oracle/_ref) through one harness, same call sites
  e2e / e2e_resident       the same metric with host<->device copies in the timed region, for both libraries
  fused                    the extended operator over the raw SplatData tensors (SURVEY.md 8 f1)
  train                    a training iteration (render + SSIM/L1 loss + backward + Adam), eager and from one CUDA graph
  fastgs, train_fastgs     the reference's DEFAULT rasterizer path (SURVEY.md 8 f4) and a training iteration on it, beside
                           the reference's own fastgs kernels
  configs                  config A (CPU oracle at full size, all cores + 1 thread; GPU beside it) and config D (6 M)
  roofline, cpu_baseline   as the task contract asks

N>1 (launched by torchrun, one rank per GPU): every rank renders its own view of the same 1 M
Gaussians (config E: eight cameras on a ring, taken in the order 0, 180, 90, 270 degrees and then the diagonals, so
that 2 and 4 ranks hold equally expensive views) and the per-Gaussian gradients are exchanged over NCCL; weak scaling,
value = N_gaussians x n_gpus / max-over-ranks time; `exchange.step_without_collectives_ms` is the same step with the
collectives left out.

--impl reference times the reference's CPU path of the same hot path: the oracle port
(oracle/gut_oracle.c, OpenMP over all host cores) on a bounded sample (a sub-frustum crop of the
same scene, same Gaussians-per-pixel density); rank 0 only.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

METRIC = "gaussians_rasterized_per_sec_fwd_bwd"
UNIT = "Gaussians/s"
KERNEL_NAMES = ("projection_ut", "sh_fwd", "isect_count", "isect_depth_sort", "isect_runs", "isect_tile_hist",
                "isect_colscan", "isect_emit", "isect_repair", "isect_keys", "isect_sort", "isect_offsets", "raster_prep", "raster_fwd", "raster_bwd", "raster_finalize", "sh_bwd",
                "sh_bwd_views", "fused_front", "fused_back", "ssim_l1_fwd", "ssim_l1_bwd", "adam_step",
                "fgs_front", "ewa_blend_fwd", "ewa_blend_bwd", "fgs_back")
WORKLOADS = {
    "A": "10k synthetic Gaussians, 256x256, SH deg 0, 1 camera (BASELINE.json configs[0])",
    "B": "1M synthetic Gaussians, 1920x1080, SH deg 3, 16x16 tiles, fwd+bwd on 1xH100 (BASELINE.json configs[1])",
    "D": "6M synthetic Gaussians, 1920x1080, SH deg 3, 16x16 tiles, fwd+bwd on 1xH100 (BASELINE.json configs[3])",
}


# ---------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------
def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            d = json.load(open(p))
            return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3)"


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.index = index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                 "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": float(max(mx)) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def crop_scene(sc, x0, y0, w, h, margin=0.12):
    """Sub-frustum sample of a scene: the Gaussians whose centres project into the window
    (plus a margin) and a camera whose principal point is shifted to the window."""
    V = sc["viewmats"][0].astype(np.float64)
    K = sc["Ks"][0].astype(np.float64)
    pc = sc["means"].astype(np.float64) @ V[:3, :3].T + V[:3, 3]
    u = pc[:, 0] / pc[:, 2] * K[0, 0] + K[0, 2]
    v = pc[:, 1] / pc[:, 2] * K[1, 1] + K[1, 2]
    keep = (pc[:, 2] > 0.01) & (u > x0 - margin * w) & (u < x0 + w * (1 + margin)) & \
           (v > y0 - margin * h) & (v < y0 + h * (1 + margin))
    out = dict(sc)
    for k in ("means", "quats", "scales", "opacities", "sh_coeffs"):
        out[k] = np.ascontiguousarray(sc[k][keep])
    Kc = sc["Ks"].copy()
    Kc[0, 0, 2] -= x0
    Kc[0, 1, 2] -= y0
    out["Ks"] = Kc
    out["width"], out["height"] = w, h
    return out


def oracle_step(orc, sc, target):
    """One fwd+bwd pass of the hot path on the CPU oracle with an L1 loss against `target`."""
    o = orc.render_pipeline(sc, precision="f32")
    diff = o["renders"] - target
    v_rc = (np.sign(diff) / diff.size).astype(np.float32)
    v_ra = np.zeros(o["alphas"].shape, np.float32)
    orc.backward_pipeline(sc, o, v_rc, v_ra, precision="f32")
    return float(np.abs(diff).mean()), o


def make_scene(config, n_gauss=None, view=None):
    import scenes
    if config == "A":
        return scenes.scene_a()
    n = n_gauss or (6_000_000 if config == "D" else 1_000_000)
    return scenes.scene_b(N=n, view=view)


def cpu_sample_scene(n_gauss):
    sc = make_scene("B", n_gauss)
    # central 480x272 window of the 1920x1080 frame: 1/16 of the pixels and ~1/16 of the Gaussians
    w, h = 480, 272
    x0, y0 = (sc["width"] - w) // 2, (sc["height"] - h) // 2
    return crop_scene(sc, x0, y0, w, h), f"central {w}x{h} window of the {sc['width']}x{sc['height']} frame"


def time_oracle_on(sc, steps, warmup, threads=None):
    from oracle import oracle as orc
    orc.build()
    cores = threads or orc.max_threads()
    orc.set_threads(cores)
    target = np.full((1, sc["height"], sc["width"], 3), 0.5, np.float32)
    for _ in range(warmup):
        oracle_step(orc, sc, target)
    t0 = time.perf_counter()
    for _ in range(steps):
        oracle_step(orc, sc, target)
    dt = (time.perf_counter() - t0) / max(steps, 1)
    orc.set_threads(1)
    return dt, cores


def time_oracle(steps, warmup, n_gauss, threads=None):
    sc, what = cpu_sample_scene(n_gauss)
    dt, cores = time_oracle_on(sc, steps, warmup, threads)
    ns = sc["means"].shape[0]
    return {"value": ns / dt, "unit": UNIT, "cores": cores, "kind": "port",
            "sample": f"{what}: {ns} of the {n_gauss} Gaussians (sub-frustum, same per-pixel density), "
                      f"fwd+bwd, {dt * 1e3:.1f} ms/step, oracle/gut_oracle.c with OpenMP"}, dt


def cpu_config_a():
    """BASELINE.md 2.2: the CPU oracle on config A at FULL size, all cores and one thread."""
    sc = make_scene("A")
    n = sc["means"].shape[0]
    dt_all, cores = time_oracle_on(sc, 3, 1)
    dt_one, _ = time_oracle_on(sc, 1, 1, threads=1)
    return {"workload": WORKLOADS["A"], "gaussians": n, "cpu_oracle": {
        "cores": cores, "ms_per_step": dt_all * 1e3, "value": n / dt_all, "unit": UNIT,
        "one_thread": {"ms_per_step": dt_one * 1e3, "value": n / dt_one}}}


# ---------------------------------------------------------------------------------------------
# reference arm
# ---------------------------------------------------------------------------------------------
def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    cb, dt = time_oracle(args.steps, args.warmup, args.gaussians or 1_000_000)
    line = {
        "impl": "reference", "metric": METRIC, "value": cb["value"], "unit": UNIT, "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt * 1e3, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOADS["B"] + "; CPU sample: " + cb["sample"]},
        "cpu_baseline": cb,
        "e2e": {"value": cb["value"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))
    return 0


# ---------------------------------------------------------------------------------------------
# GPU arm
# ---------------------------------------------------------------------------------------------
class TimedBackend:
    """Wraps an OpsBackend: CUDA events on the launching stream around every operator call, so that both libraries are
    timed per operator by the same harness through the same call sites (BASELINE.md 2.1)."""

    OPS = ("projection_ut_3dgs_fused", "spherical_harmonics_fwd", "spherical_harmonics_bwd", "intersect_tile",
           "intersect_offset", "rasterize_to_pixels_from_world_3dgs_fwd", "rasterize_to_pixels_from_world_3dgs_bwd")

    def __init__(self, backend):
        import torch
        self._b, self._torch, self.records = backend, torch, []

    def __getattr__(self, name):
        fn = getattr(self._b, name)
        if name not in self.OPS:
            return fn
        torch = self._torch

        def timed(*a, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **kw)
            e1.record()
            self.records.append((name, e0, e1))
            return r
        return timed

    def summary(self):
        self._torch.cuda.synchronize()
        agg = {}
        for name, e0, e1 in self.records:
            agg.setdefault(name, []).append(e0.elapsed_time(e1))
        self.records = []
        return {k: round(float(np.median(v)), 4) for k, v in agg.items()}


DUMP_GAUSSIAN_SAMPLE = 65536


def dump_outputs(out_dir, wl, names):
    """Writes what the last timed step handed its caller as <out_dir>/<name>.npy (float32; the loss in float64): the
    rendered image and alpha in full, and the parameter gradients on a fixed, seeded sample of Gaussians (all of them
    would be ~240 MB at 1 M), so that two builds can be compared output for output on the same inputs."""
    import torch
    os.makedirs(out_dir, exist_ok=True)
    loss, out = wl.last
    arrays = {"loss": np.asarray(float(loss.detach().item()), np.float64),
              "render_colors": out.render_colors.detach().float().cpu().numpy(),
              "render_alphas": out.alpha.detach().float().cpu().numpy()}
    n = wl.N
    idx = np.arange(n) if n <= DUMP_GAUSSIAN_SAMPLE else \
        np.sort(np.random.default_rng(0).choice(n, DUMP_GAUSSIAN_SAMPLE, replace=False))
    arrays["gaussian_sample_index"] = idx.astype(np.float64)
    sel = torch.from_numpy(idx).to(wl.P["means"].device)
    for k in names:
        arrays[f"grad_{k}"] = wl.P[k].grad.detach().index_select(0, sel).float().cpu().numpy()
    for k, a in arrays.items():
        np.save(os.path.join(out_dir, k + ".npy"), a)


def percentiles(ms):
    a = np.asarray(ms, np.float64)
    return {"n": int(a.size), "median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)),
            "p90_ms": float(np.percentile(a, 90))}


def run_b200(args):
    import torch
    import torch.distributed as dist

    import __graft_entry__ as ge

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise RuntimeError("bench.py needs a CUDA device: the CUDA backend has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    pg2 = None
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        if not args.no_overlap:
            pg2 = dist.new_group()  # second communicator: the geometry all-reduce overlaps the colour all-gather
    pkg = ge.load_package()
    pkg.load()
    from gsplat_b200 import hoststream, multiview
    cabi = ctypes.CDLL(pkg.CABI_PATH)
    cabi.gsb_launch_count.restype = ctypes.c_uint64
    cabi.gsb_profile_read.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_double)]
    names = ("means", "quats", "scales", "opacities", "sh_coeffs")
    raw_names = ("means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw")
    compact = world > 1 and args.exchange in ("compact", "peer")
    peer = {"obj": None, "why": None}   # peer-memory exchange, built with the workload (needs N)

    def sync_all():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        """The contract's timing: `steps` calls bracketed by barrier + synchronize, CUDA events, max over ranks."""
        sync_all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        sync_all()
        return multiview.max_over_ranks(e0.elapsed_time(e1), dev)

    def distribution(fn, warm=20, n=100):
        """BASELINE.md 2.1: 20 warm-up + 100 timed iterations, each between its own pair of events."""
        for _ in range(warm):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
        torch.cuda.synchronize()
        for a, b in ev:
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return percentiles([a.elapsed_time(b) for a, b in ev])

    def read_profile(fn, steps):
        cabi.gsb_profile_enable(1)
        timed(fn, steps)
        prof = {}
        for kname in KERNEL_NAMES:
            tot = ctypes.c_double(0.0)
            n = cabi.gsb_profile_read(kname.encode(), ctypes.byref(tot))
            if n:
                prof[kname] = {"launches": n, "avg_ms": tot.value / n}
        cabi.gsb_profile_enable(0)
        return prof

    class Workload:
        """Device + pinned-host tensors of one config and the step functions over them."""

        def __init__(self, config, n_gauss=None, view=None):
            self.config = config
            sc = make_scene(config, n_gauss, view)
            self.N, self.W, self.H, self.deg = sc["means"].shape[0], sc["width"], sc["height"], sc["sh_degree"]
            self.host = {k: torch.from_numpy(sc[k]).pin_memory() for k in
                         ("means", "quats", "scales", "opacities", "sh_coeffs", "viewmats", "Ks")}
            bg = sc["background"] if sc.get("background") is not None else np.zeros((1, 3), np.float32)
            self.host["background"] = torch.from_numpy(bg).pin_memory()
            rng = np.random.default_rng(123 + rank)
            self.host["target"] = torch.from_numpy(rng.random((1, self.H, self.W, 3), dtype=np.float32)).pin_memory()
            self.P = {k: self.host[k].to(dev).requires_grad_(k in names) for k in self.host}
            self.stats = {}
            self._raw = None
            self.capacity = 0

        # -- operator path: activated parameters in, as gs::training::rasterize hands them to the ops --
        def step(self, Pd=None, backend=None, exchange=True, prof=None):
            Pd = Pd or self.P
            for k in names:
                Pd[k].grad = None
            deferred = pkg.DeferredSHBackward() if compact else None
            out = pkg.rasterize(Pd["means"], Pd["quats"], Pd["scales"], Pd["opacities"], Pd["sh_coeffs"], self.deg,
                                Pd["viewmats"], Pd["Ks"], self.W, self.H, bg_color=Pd["background"], backend=backend,
                                sh_exchange=deferred)
            loss = (out.render_colors - Pd["target"]).abs().mean()
            loss.backward()
            if compact:
                if peer["obj"] is not None:
                    multiview.exchange_gradients_peer(Pd, deferred, peer["obj"], overlap_group=pg2)
                else:
                    multiview.exchange_gradients_compact(Pd, deferred, overlap_group=pg2, local_only=not exchange, prof=prof)
            elif world > 1:
                multiview.allreduce_gradients([Pd[k].grad for k in names])
            self.stats["n_isects"], self.stats["vis"] = out.n_isects, out.visibility
            self.last = (loss, out)
            return loss, out

        # -- raw SplatData: what training holds (log-scales, logits, raw quaternions, sh0 / shN) --
        def raw(self):
            if self._raw is None:
                with torch.no_grad():
                    r = pkg.raw_from_activated(self.P["means"], self.P["quats"], self.P["scales"], self.P["opacities"],
                                               self.P["sh_coeffs"])
                self._raw = {k: v.detach().clone().requires_grad_(True) for k, v in r.items()}
            return self._raw

        def step_raw_unfused(self, backend=None):
            """The reference's own sequence: torch activations (splat_data.cpp:267-286) + the operators + autograd."""
            R = self.raw()
            for k in raw_names:
                R[k].grad = None
            out = pkg.rasterize_from_raw(R, self.deg, self.P["viewmats"], self.P["Ks"], self.W, self.H,
                                         bg_color=self.P["background"], backend=backend)
            loss = (out.render_colors - self.P["target"]).abs().mean()
            loss.backward()
            return loss, out

        def step_fused(self):
            R = self.raw()
            for k in raw_names:
                R[k].grad = None
            out = pkg.rasterize_fused(R["means"], R["sh0"], R["shN"], R["scaling_raw"], R["rotation_raw"],
                                      R["opacity_raw"], self.deg, self.P["viewmats"], self.P["Ks"], self.W, self.H,
                                      bg_color=self.P["background"], isect_capacity=self.capacity)
            loss = (out.render_colors - self.P["target"]).abs().mean()
            loss.backward()
            self.stats["fused_n"] = out.n_isects
            return loss, out

        def size_capacity(self):
            """One exact step sizes flatten_ids for the capacity mode (no host read-back afterwards)."""
            self.raw()
            self.capacity = 0
            _, out = self.step_fused()
            n = int(out.n_isects.item())
            self.capacity = int(n * 1.25) + 1024
            return n

        # -- end-to-end protocols --
        def e2e_staged(self, steps, backend=None):
            """All op inputs from pinned host memory each step, image + all gradients + loss back (hoststream.py)."""
            def staged_step(Pd):
                loss, out = self.step(Pd, backend)
                return loss, out.render_colors
            st = hoststream.HostStagedSteps(dev, self.host, names, staged_step)
            st.run(3)
            losses = []
            ms = timed(lambda: losses.extend(st.run(steps)), 1) / steps
            return ms, st.h2d_bytes, st.d2h_bytes, (losses[-1] if losses else None)

        def e2e_resident(self, steps, fn):
            """Parameters resident (training): camera + target image H2D, loss D2H every step."""
            def one():
                for k in ("viewmats", "Ks", "background", "target"):
                    self.P[k] = self.host[k].to(dev, non_blocking=True)
                loss, _ = fn()
                return float(loss.item())
            one()
            return timed(one, steps) / steps

        def max_tile_list(self):
            """Longest per-tile intersection list of the current view (BASELINE.md 2.1)."""
            with torch.no_grad():
                P = self.P
                radii, m2d, dep, _, _ = pkg.projection_ut_3dgs_fused(P["means"].detach(), P["quats"].detach(),
                                                                     P["scales"].detach(), P["opacities"].detach(),
                                                                     P["viewmats"], P["Ks"], self.W, self.H, 0.3, 0.01,
                                                                     1e4, 0.0)
                tw, th = (self.W + 15) // 16, (self.H + 15) // 16
                _, ids, _ = pkg.intersect_tile(m2d, radii, dep, 1, 16, tw, th, True)
                off = pkg.intersect_offset(ids, 1, tw, th).reshape(-1).long()
                ends = torch.cat([off[1:], torch.tensor([ids.shape[0]], device=dev)])
                return int((ends - off).max().item())

    cfg = args.config if world == 1 else "B"
    # Config E: eight cameras on a ring around the slab, one per rank.  The ring positions are not equally expensive (the
    # four diagonal ones see part of the slab at a third of the distance: 2.45 vs 2.2 ms on one GPU, DESIGN.md 6); ranks
    # take them in the order 0, 180, 90, 270 degrees, then the diagonals, so that 2 and 4 ranks render equally heavy views
    # and the scaling figure measures the exchange, not the scene.  At 8 ranks every position is in use.
    VIEW_ORDER = (0, 4, 2, 6, 1, 5, 3, 7)
    wl = Workload(cfg, args.gaussians, view=(VIEW_ORDER[rank % 8] if world > 1 else None))
    N, W, H = wl.N, wl.W, wl.H
    warm = max(args.warmup, 3)
    if world > 1 and args.exchange == "peer":
        # collective: every rank tries, and every rank falls back if ANY rank failed (the paths must not be mixed)
        try:
            peer["obj"] = multiview.PeerColourExchange(N, dev)
            ok = 1
        except Exception as e:
            peer["why"], ok = repr(e)[:200], 0
        flag = torch.tensor([ok], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            peer["obj"] = None
            peer["why"] = peer["why"] or "another rank could not map symmetric memory"

    # ---- warm-up + device-resident timing (the contract's K steps) -------------------------------------------
    if world > 1:
        # set-up, not warm-up: NCCL builds its rings / channels lazily on the first collectives of each communicator (two
        # here: exchange + overlapped all-reduce).  At 8 ranks the K = 20 loop right after 5 warm-up steps measured 4.05 ms
        # while the e2e_resident loop later in the same run measured 3.44 ms for a superset of the work.
        for _ in range(12):
            wl.step()
        sync_all()
    for _ in range(warm):
        wl.step()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = cabi.gsb_launch_count()
    ms_total = timed(wl.step, args.steps)
    launches = int(cabi.gsb_launch_count() - launches0)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, wl, names)
    ms_step = ms_total / args.steps
    value = N * world / (ms_step * 1e-3)
    prof = read_profile(wl.step, max(args.steps, 10))  # per-kernel events in a SEPARATE pass

    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": warm,
        "ms_per_step": ms_step, "iters_per_sec": 1e3 / ms_step, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "gpu_launches": launches,
        "kernels_ms": {k: round(v["avg_ms"], 4) for k, v in prof.items()},
    }
    cfgd = {"workload": (WORKLOADS[cfg] if world == 1 else
                         f"1M Gaussians x {world} synthetic cameras/step, per-view shard + NCCL gradient exchange "
                         f"({args.exchange}) (BASELINE.json configs[4])"),
            "gaussians": N, "visible": int(wl.stats["vis"].sum().item()), "intersections": wl.stats["n_isects"],
            "image": [W, H], "loss": "L1 vs synthetic target", "parallelism": f"view-dp{world}",
            "l2": "per-step working set (236 B/Gaussian parameters + 64 B records + 12 B/intersection lists + 236 B "
                  "gradients) exceeds the 50 MB L2; no explicit flush"}
    line["config"] = cfgd
    line["intersections_per_sec"] = wl.stats["n_isects"] * world / (ms_step * 1e-3)

    # ---- roofline of the dominant kernel (SURVEY.md 8d algorithmic bytes) ---------------------------------------
    peak, peak_src = load_peaks()
    I, Pn = wl.stats["n_isects"], W * H
    dom = max(prof, key=lambda k: prof[k]["avg_ms"]) if prof else None
    algo = {"raster_bwd": 60 * I + 24 * Pn + 112 * N, "raster_fwd": 48 * I + 20 * Pn}
    if dom in algo:
        achieved = algo[dom] / (prof[dom]["avg_ms"] * 1e-3) / 1e9
        line["roofline"] = {
            "kernel": dom, "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
            "peak_source": peak_src, "algorithmic_bytes_per_launch": algo[dom], "avg_kernel_ms": prof[dom]["avg_ms"],
            "note": "the blend is FP32-issue/LSU/atomic bound by construction (SURVEY.md 8d): the HBM fraction is the "
                    "figure north_star asks for"}

    if args.quick:
        if rank == 0:
            line["clocks"] = sampler.stop()
            print(json.dumps(line))
        if world > 1:
            dist.destroy_process_group()
        return 0

    # ---- distribution + per-op times of this backend -----------------------------------------------------------
    ops_ms = {}
    if world == 1:
        line["distribution"] = distribution(wl.step)
        tb = TimedBackend(pkg.default_backend())
        for _ in range(20):
            wl.step(backend=tb)
        ops_ms["b200"] = tb.summary()
        cfgd["max_tile_list"] = wl.max_tile_list()

    # ---- end-to-end -----------------------------------------------------------------------------------------------
    ms_e2e, h2d, d2h, e2e_loss = wl.e2e_staged(args.steps)
    ms_e2e_res = wl.e2e_resident(args.steps, wl.step)
    clocks = sampler.stop() if rank == 0 else None
    line["e2e"] = {"value": N * world / (ms_e2e * 1e-3), "unit": UNIT, "ms_per_step": ms_e2e,
                   "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h), "loss": e2e_loss,
                   "what": "all op inputs (parameters, camera, target) from pinned host memory each step; image + all "
                           "gradients + loss back to pinned host; copies of neighbouring steps overlap the kernels "
                           "(gsplat_b200.hoststream.HostStagedSteps)"}
    line["e2e_resident"] = {"value": N * world / (ms_e2e_res * 1e-3), "unit": UNIT, "ms_per_step": ms_e2e_res,
                            "what": "parameters resident (as in training); camera + target image H2D, loss D2H per step"}
    line["clocks"] = clocks

    if world > 1:
        # the exchange alone: one coalesced all-reduce of the 236 B/Gaussian gradient set (BASELINE.md config E)
        bufs = [torch.zeros_like(wl.P[k]) for k in names]
        for _ in range(3):
            multiview.allreduce_gradients(bufs)
        ms_ar = timed(lambda: multiview.allreduce_gradients(bufs), 20) / 20
        nbytes = sum(b.numel() * 4 for b in bufs)
        ms_local = None
        if compact and peer["obj"] is None:  # the same step without any collective: what the exchange adds
            for _ in range(3):
                wl.step(exchange=False)
            ms_local = timed(lambda: wl.step(exchange=False), args.steps) / args.steps
            pr = {}
            for _ in range(10):
                wl.step(prof=pr)
            sync_all()
            phases = {k: (round(v, 4) if v is not None else None) for k, v in multiview.phase_times(pr).items()}
        line["exchange"] = {"mode": ("peer" if peer["obj"] is not None else
                                     ("compact" if compact else "allreduce")),
                            "peer_fallback_reason": peer["why"],
                            "overlap": ("geometry all-reduce on a second communicator" if pg2 is not None else "none"),
                            "step_without_collectives_ms": ms_local,
                            "phases_ms": (phases if ms_local is not None else None),
                            "allreduce_236B_ms": ms_ar, "allreduce_bytes": nbytes,
                            "allreduce_bus_GBps": 2.0 * (world - 1) / world * nbytes / (ms_ar * 1e-3) / 1e9,
                            "nvlink4_peak_GBps_per_direction": 450.0,
                            "note": "e2e re-uploads the REPLICATED parameters from every rank through one host: "
                                    "e2e_resident (camera + target in, loss out) is the multi-GPU end-to-end figure"}
    if rank != 0 or world > 1:
        if rank == 0:
            print(json.dumps(line))
        if world > 1:
            dist.destroy_process_group()
        return 0

    # ---- extended operator over the raw SplatData tensors (SURVEY.md 8 f1) -------------------------------------
    try:
        n_f = wl.size_capacity()
        for _ in range(3):
            wl.step_fused()
        ms_f = timed(wl.step_fused, args.steps) / args.steps
        prof_f = read_profile(wl.step_fused, max(args.steps, 10))
        ms_f_res = wl.e2e_resident(args.steps, wl.step_fused)
        assert int(wl.stats["fused_n"].item()) <= wl.capacity
        for _ in range(3):
            wl.step_raw_unfused()
        ms_u = timed(wl.step_raw_unfused, args.steps) / args.steps
        ms_u_res = wl.e2e_resident(args.steps, wl.step_raw_unfused)
        line["fused"] = {
            "what": "rasterize_from_world_fused_fwd/bwd on the raw SplatData tensors (log-scales, logits, raw quaternions, "
                    "sh0/shN), flatten_ids sized from a capacity: no host read-back inside the step",
            "ms_per_step": ms_f, "value": N / (ms_f * 1e-3), "e2e_resident_ms": ms_f_res,
            "distribution": distribution(wl.step_fused), "intersections": n_f,
            "kernels_ms": {k: round(v["avg_ms"], 4) for k, v in prof_f.items()},
            "operator_path_on_raw_tensors": {
                "what": "torch activations (splat_data.cpp:267-286) + the eleven operators + autograd, this backend",
                "ms_per_step": ms_u, "e2e_resident_ms": ms_u_res}}
    except Exception as e:
        line["fused"] = {"unavailable": repr(e)[:300]}

    # ---- same-box GPU baseline: the reference's own gsplat CUDA kernels (oracle/_ref), same call sites ------------
    rb = None
    if not args.no_ref_cuda:
        try:
            from oracle import ref_ops
            if ref_ops.available():
                rb = ref_ops.backend(pkg)
                ref_step = lambda: wl.step(backend=rb)
                for _ in range(3):
                    ref_step()
                ms_ref = timed(ref_step, args.steps) / args.steps
                dist_ref = distribution(ref_step, warm=5, n=50)
                tbr = TimedBackend(rb)
                for _ in range(10):
                    wl.step(backend=tbr)
                ops_ms["reference_cuda"] = tbr.summary()
                ms_ref_e2e, _, _, _ = wl.e2e_staged(args.steps, backend=rb)
                ms_ref_res = wl.e2e_resident(args.steps, ref_step)
                ref_raw = lambda: wl.step_raw_unfused(backend=rb)
                for _ in range(2):
                    ref_raw()
                ms_ref_raw = timed(ref_raw, args.steps) / args.steps
                ms_ref_raw_res = wl.e2e_resident(args.steps, ref_raw)
                fused_res = line["fused"].get("e2e_resident_ms")
                line["reference_cuda"] = {
                    "what": "reference gsplat/*.cu compiled unmodified (-O3 --use_fast_math, sm_90) by oracle/build_ref.py, "
                            "driven through the same L3 call sequence on the same inputs",
                    "ms_per_step": ms_ref, "value": N / (ms_ref * 1e-3), "unit": UNIT, "distribution": dist_ref,
                    "e2e_ms": ms_ref_e2e, "e2e_resident_ms": ms_ref_res,
                    "raw_tensor_sequence": {"ms_per_step": ms_ref_raw, "e2e_resident_ms": ms_ref_raw_res,
                                            "what": "torch activations + the reference's kernels + autograd: what the "
                                                    "reference's trainer runs per step"},
                    "speedup": {"device_resident": ms_ref / ms_step, "e2e": ms_ref_e2e / ms_e2e,
                                "e2e_resident": ms_ref_res / ms_e2e_res,
                                "fused_vs_reference_training_step_e2e_resident":
                                    (ms_ref_raw_res / fused_res) if fused_res else None}}
        except Exception as e:  # the baseline is optional evidence, never a failure of the bench
            line["reference_cuda"] = {"unavailable": repr(e)[:200]}
    line["ops_ms"] = ops_ms

    # ---- training iteration: render -> L1 + SSIM loss -> backward -> Adam (BASELINE.json "iters/sec"; SURVEY.md 8 f2/f3) ----
    def train_block(w, steps):
        from gsplat_b200 import training
        tgt_chw = w.P["target"][0].permute(2, 0, 1).contiguous()
        host_tgt = tgt_chw.cpu().pin_memory()
        out = {}
        P1 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
        ts = training.TrainStep(P1, w.deg, w.W, w.H, optimizer=training.FusedAdam(P1))
        ts.size_capacity(w.P["viewmats"], w.P["Ks"], tgt_chw, w.P["background"])

        def it_b200():
            for k in ("viewmats", "Ks", "background"):
                w.P[k] = w.host[k].to(dev, non_blocking=True)
            tg = host_tgt.to(dev, non_blocking=True)
            return float(ts(w.P["viewmats"], w.P["Ks"], tg, w.P["background"]).item())
        for _ in range(3):
            it_b200()
        ms = timed(it_b200, steps) / steps
        prof_t = read_profile(it_b200, max(steps, 10))
        assert int(ts.last["n_isects"].item()) <= ts.capacity
        out["b200"] = {"ms_per_iter": ms, "iters_per_sec": 1e3 / ms,
                       "kernels_ms": {k: round(v["avg_ms"], 4) for k, v in prof_t.items()},
                       "what": "extended operator on raw tensors + fused SSIM/L1 loss-and-gradient kernel + one-launch Adam; "
                               "camera + target H2D and loss D2H every iteration"}
        try:  # the same iteration captured once in a CUDA graph: one launch per iteration
            P3 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
            gts = training.GraphedTrainStep(P3, w.deg, w.W, w.H)
            gts.capture(w.host["viewmats"].to(dev), w.host["Ks"].to(dev), tgt_chw, w.P["background"])

            def it_graph():
                return float(gts(w.host["viewmats"], w.host["Ks"], host_tgt, w.host["background"]).item())
            for _ in range(3):
                it_graph()
            ms_g = timed(it_graph, steps) / steps
            assert not gts.overflowed()
            out["b200_cuda_graph"] = {"ms_per_iter": ms_g, "iters_per_sec": 1e3 / ms_g,
                                      "what": "the same iteration replayed from one captured CUDA graph (no host "
                                              "read-back inside: capacity-sized intersection buffers, Adam scalars from "
                                              "device memory); camera + target H2D and loss D2H every iteration"}
            del gts, P3
        except Exception as e:
            out["b200_cuda_graph"] = {"unavailable": repr(e)[:300]}
        if rb is not None:
            try:
                from oracle import ref_train
                P2 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
                ropt = ref_train.RefFusedAdam(P2, training.AdamConfig().lrs())
                state = {"it": 0}

                def it_ref():
                    for k in ("viewmats", "Ks", "background"):
                        w.P[k] = w.host[k].to(dev, non_blocking=True)
                    tg = host_tgt.to(dev, non_blocking=True)
                    o = pkg.rasterize_from_raw(P2, w.deg, w.P["viewmats"], w.P["Ks"], w.W, w.H,
                                               bg_color=w.P["background"], backend=rb)
                    loss = ref_train.ref_photometric_loss(o.image, tg, 0.2)
                    loss.backward()
                    state["it"] += 1
                    ropt.step(state["it"], training.PARAM_GROUPS)
                    ropt.zero_grad()
                    return float(loss.item())
                for _ in range(2):
                    it_ref()
                ms_r = timed(it_ref, steps) / steps
                out["reference_cuda"] = {"ms_per_iter": ms_r, "iters_per_sec": 1e3 / ms_r,
                                         "what": "the reference's own kernels for every stage (gsplat operators, ssim.cu, "
                                                 "adam_kernels.cuh) glued by torch exactly as its trainer does"}
                out["speedup"] = ms_r / ms
                if "ms_per_iter" in out.get("b200_cuda_graph", {}):
                    out["speedup_cuda_graph"] = ms_r / out["b200_cuda_graph"]["ms_per_iter"]
            except Exception as e:
                out["reference_cuda"] = {"unavailable": repr(e)[:200]}
        return out

    try:
        line["train"] = train_block(wl, args.steps)
    except Exception as e:
        line["train"] = {"unavailable": repr(e)[:300]}

    # ---- SURVEY.md 8 f4: the reference's default rasterizer (fastgs, EWA) on the same scene: forward + backward -------
    def fastgs_block(w, steps):
        from gsplat_b200 import fastgs as fg
        R = w.raw()
        V = w.P["viewmats"][0].detach()
        K = w.host["Ks"][0]
        campos = (-V[:3, :3].T @ V[:3, 3]).contiguous()
        st = fg.FastGSSettings(cam_position=campos, active_sh_bases=(w.deg + 1) ** 2, width=w.W, height=w.H,
                               focal_x=float(K[0, 0]), focal_y=float(K[1, 1]), center_x=float(K[0, 2]), center_y=float(K[1, 2]))
        names_f = ("means", "scaling_raw", "rotation_raw", "opacity_raw", "sh0", "shN")
        tgt = w.P["target"][0].permute(2, 0, 1).contiguous()
        bgc = w.P["background"][0]
        info = {}

        def make_step(backend):
            def step():
                for k in names_f:
                    R[k].grad = None
                img, alpha = fg.fast_rasterize(backend, R["means"], R["scaling_raw"], R["rotation_raw"],
                                               R["opacity_raw"].reshape(-1, 1), R["sh0"], R["shN"], V, st, bg_color=bgc)
                loss = (img - tgt).abs().mean()
                loss.backward()
                return loss
            return step
        out = {"what": "fast_gs::rasterization forward_wrapper + backward_wrapper through the reference caller's sequence "
                       "(fast_rasterizer.cpp:12-74: raw parameters in, background composite, L1 loss, autograd), "
                       "device-resident"}
        mine = make_step(fg.default_backend())
        for _ in range(3):
            mine()
        ms = timed(mine, steps) / steps
        prof = read_profile(mine, max(steps, 10))
        with torch.no_grad():
            _, _, c = fg.default_backend().forward(R["means"], R["scaling_raw"], R["rotation_raw"], R["opacity_raw"].reshape(-1, 1),
                                                   R["sh0"], R["shN"], V, st)
        out["b200"] = {"ms_per_step": ms, "value": w.N / (ms * 1e-3), "unit": UNIT, "instances": int(c["ints"][1]),
                       "distribution": distribution(mine, warm=5, n=50),
                       "kernels_ms": {k: round(v["avg_ms"], 4) for k, v in prof.items()}}
        del c
        if not args.no_ref_cuda:
            try:
                from oracle import ref_fastgs
                if ref_fastgs.available():
                    rbe = ref_fastgs.backend(fg)
                    ref = make_step(rbe)
                    for _ in range(3):
                        ref()
                    ms_r = timed(ref, steps) / steps
                    with torch.no_grad():
                        _, _, c = rbe.forward(R["means"], R["scaling_raw"], R["rotation_raw"], R["opacity_raw"].reshape(-1, 1),
                                              R["sh0"], R["shN"], V, st)
                    out["reference_cuda"] = {"ms_per_step": ms_r, "value": w.N / (ms_r * 1e-3), "unit": UNIT,
                                             "instances": int(c["ints"][1]), "buckets": int(c["ints"][2]),
                                             "distribution": distribution(ref, warm=3, n=30),
                                             "what": "reference fastgs/rasterization/*.cu compiled unmodified (-O3 "
                                                     "--use_fast_math, sm_90) by oracle/build_ref.py, same call sites"}
                    out["speedup"] = ms_r / ms
                    del c
            except Exception as e:
                out["reference_cuda"] = {"unavailable": repr(e)[:200]}
        return out

    try:
        line["fastgs"] = fastgs_block(wl, args.steps)
    except Exception as e:
        line["fastgs"] = {"unavailable": repr(e)[:300]}

    # ---- a training iteration on the reference's DEFAULT path: fastgs render -> SSIM/L1 loss -> backward -> Adam ---------
    def fastgs_train_block(w, steps):
        from gsplat_b200 import fastgs as fg, training
        V = w.P["viewmats"][0].detach()
        K = w.host["Ks"][0]
        campos = (-V[:3, :3].T @ V[:3, 3]).contiguous()
        st = fg.FastGSSettings(cam_position=campos, active_sh_bases=(w.deg + 1) ** 2, width=w.W, height=w.H,
                               focal_x=float(K[0, 0]), focal_y=float(K[1, 1]), center_x=float(K[0, 2]), center_y=float(K[1, 2]))
        tgt_chw = w.P["target"][0].permute(2, 0, 1).contiguous()
        host_tgt = tgt_chw.cpu().pin_memory()
        host_w2c = V.cpu().pin_memory()
        bgc = w.P["background"][0].detach()
        out = {"what": "fastgs forward -> background composite -> SSIM/L1 loss and gradient -> fastgs backward -> Adam; camera + "
                       "target H2D and loss D2H every iteration"}
        P1 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
        ts = training.FastGsTrainStep(P1, w.deg, w.W, w.H, optimizer=training.FusedAdam(P1))

        def it_b200():
            w2c = host_w2c.to(dev, non_blocking=True)
            tg = host_tgt.to(dev, non_blocking=True)
            return float(ts(w2c, st, tg, bgc).item())
        for _ in range(3):
            it_b200()
        ms = timed(it_b200, steps) / steps
        prof_t = read_profile(it_b200, max(steps, 10))
        out["b200"] = {"ms_per_iter": ms, "iters_per_sec": 1e3 / ms, "kernels_ms": {k: round(v["avg_ms"], 4) for k, v in prof_t.items()},
                       "what": "gsb_fastgs_* + gsb_ssim_l1 on [3,H,W] planes + one-launch Adam; no autograd graph"}
        del ts, P1
        try:  # no read-back (capacity-sized instance buffer), then the same iteration replayed from one CUDA graph
            P3 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
            ts3 = training.FastGsTrainStep(P3, w.deg, w.W, w.H, optimizer=training.FusedAdam(P3))
            ts3.size_capacity(V, st)

            def it_cap():
                w2c = host_w2c.to(dev, non_blocking=True)
                tg = host_tgt.to(dev, non_blocking=True)
                return float(ts3(w2c, st, tg, bgc).item())
            for _ in range(3):
                it_cap()
            ms_c = timed(it_cap, steps) / steps
            assert int(ts3.last["n_instances"].item()) <= ts3.capacity
            out["b200_capacity"] = {"ms_per_iter": ms_c, "iters_per_sec": 1e3 / ms_c,
                                    "what": "forward_capacity (include/fastgs/rasterization_ext.h): no host read-back inside"}
            del ts3, P3
            P4 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
            gts = training.GraphedFastGsTrainStep(P4, w.deg, st)
            host_campos, host_bg = campos.cpu().pin_memory(), bgc.cpu().pin_memory()
            gts.capture(V, campos, tgt_chw, bgc)

            def it_graph():
                return float(gts(host_w2c, host_campos, host_tgt, host_bg).item())
            for _ in range(3):
                it_graph()
            ms_g = timed(it_graph, steps) / steps
            assert not gts.overflowed()
            out["b200_cuda_graph"] = {"ms_per_iter": ms_g, "iters_per_sec": 1e3 / ms_g,
                                      "what": "the same iteration replayed from one captured CUDA graph"}
            del gts, P4
        except Exception as e:
            out["b200_cuda_graph"] = {"unavailable": repr(e)[:300]}
        if not args.no_ref_cuda:
            try:
                from oracle import ref_fastgs, ref_train
                if ref_fastgs.available():
                    rbe = ref_fastgs.backend(fg)
                    P2 = {k: v.detach().clone().requires_grad_(True) for k, v in w.raw().items()}
                    ropt = ref_train.RefFusedAdam(P2, training.AdamConfig().lrs())
                    state = {"it": 0}

                    def it_ref():
                        w2c = host_w2c.to(dev, non_blocking=True)
                        tg = host_tgt.to(dev, non_blocking=True)
                        img, _ = fg.fast_rasterize(rbe, P2["means"], P2["scaling_raw"], P2["rotation_raw"],
                                                   P2["opacity_raw"].reshape(-1, 1), P2["sh0"], P2["shN"], w2c, st, bg_color=bgc)
                        loss = ref_train.ref_photometric_loss(torch.clamp(img, 0.0, 1.0), tg, 0.2)  # trainer.cpp:103-126
                        loss.backward()
                        state["it"] += 1
                        ropt.step(state["it"], training.PARAM_GROUPS)
                        ropt.zero_grad()
                        return float(loss.item())
                    for _ in range(2):
                        it_ref()
                    ms_r = timed(it_ref, steps) / steps
                    out["reference_cuda"] = {"ms_per_iter": ms_r, "iters_per_sec": 1e3 / ms_r,
                                             "what": "the reference's own kernels for every stage (fastgs rasterizer, ssim.cu, "
                                                     "adam_kernels.cuh) glued by torch autograd exactly as its trainer does"}
                    out["speedup"] = ms_r / ms
                    if "ms_per_iter" in out.get("b200_cuda_graph", {}):
                        out["speedup_cuda_graph"] = ms_r / out["b200_cuda_graph"]["ms_per_iter"]
            except Exception as e:
                out["reference_cuda"] = {"unavailable": repr(e)[:200]}
        return out

    try:
        line["train_fastgs"] = fastgs_train_block(wl, args.steps)
    except Exception as e:
        line["train_fastgs"] = {"unavailable": repr(e)[:300]}

    # ---- the other configs of BASELINE.json (N=1 line only) ---------------------------------------------------------
    configs = {}
    if cfg == "B" and not args.no_other_configs:
        try:
            a = cpu_config_a()
            wa = Workload("A")
            for _ in range(5):
                wa.step()
            ms_a = timed(wa.step, 50) / 50
            a["b200"] = {"ms_per_step": ms_a, "value": wa.N / (ms_a * 1e-3), "intersections": wa.stats["n_isects"]}
            if rb is not None:
                for _ in range(3):
                    wa.step(backend=rb)
                ms_ar = timed(lambda: wa.step(backend=rb), 50) / 50
                a["reference_cuda"] = {"ms_per_step": ms_ar, "value": wa.N / (ms_ar * 1e-3)}
            configs["A"] = a
            del wa
        except Exception as e:
            configs["A"] = {"unavailable": repr(e)[:200]}
        try:
            del wl
            torch.cuda.empty_cache()
            wd = Workload("D")
            for _ in range(3):
                wd.step()
            ms_d = timed(wd.step, 20) / 20
            prof_d = read_profile(wd.step, 10)
            d = {"workload": WORKLOADS["D"], "gaussians": wd.N, "intersections": wd.stats["n_isects"],
                 "visible": int(wd.stats["vis"].sum().item()), "ms_per_step": ms_d, "value": wd.N / (ms_d * 1e-3),
                 "distribution": distribution(wd.step, warm=3, n=30),
                 "e2e_resident_ms": wd.e2e_resident(10, wd.step),
                 "kernels_ms": {k: round(v["avg_ms"], 4) for k, v in prof_d.items()}}
            try:
                wd.size_capacity()
                for _ in range(2):
                    wd.step_fused()
                ms_df = timed(wd.step_fused, 20) / 20
                d["fused"] = {"ms_per_step": ms_df, "value": wd.N / (ms_df * 1e-3),
                              "e2e_resident_ms": wd.e2e_resident(10, wd.step_fused)}
            except Exception as e:
                d["fused"] = {"unavailable": repr(e)[:200]}
            if rb is not None:
                for _ in range(2):
                    wd.step(backend=rb)
                ms_dr = timed(lambda: wd.step(backend=rb), 10) / 10
                d["reference_cuda"] = {"ms_per_step": ms_dr, "value": wd.N / (ms_dr * 1e-3),
                                       "speedup_device_resident": ms_dr / ms_d}
            try:
                d["train"] = train_block(wd, 10)
            except Exception as e:
                d["train"] = {"unavailable": repr(e)[:200]}
            try:
                d["fastgs"] = fastgs_block(wd, 10)
            except Exception as e:
                d["fastgs"] = {"unavailable": repr(e)[:200]}
            try:
                d["train_fastgs"] = fastgs_train_block(wd, 10)
            except Exception as e:
                d["train_fastgs"] = {"unavailable": repr(e)[:200]}
            configs["D"] = d
            del wd
        except Exception as e:
            configs["D"] = {"unavailable": repr(e)[:200]}
    if configs:
        line["configs"] = configs

    if not args.no_cpu_baseline:
        cb, _ = time_oracle(1, 1, N if cfg != "A" else 1_000_000)
        line["cpu_baseline"] = cb

    print(json.dumps(line))
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--exchange", choices=("compact", "allreduce", "peer"), default="compact",
                    help="N>1 gradient exchange: compact (all-gather colour gradients + multi-view SH backward) or "
                         "plain all-reduce of the five gradient tensors")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default="B", choices=["A", "B", "D"], help="N=1 workload (BASELINE.json configs)")
    ap.add_argument("--gaussians", type=int, default=None, help="override the config's Gaussian count")
    ap.add_argument("--no-overlap", action="store_true", help="N>1: geometry all-reduce on the compute stream (no second communicator)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-ref-cuda", action="store_true")
    ap.add_argument("--no-other-configs", action="store_true", help="skip the config A / D block of the N=1 line")
    ap.add_argument("--quick", action="store_true", help="device-resident timing only (profiling runs)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the image, alpha, loss and a seeded sample of the parameter "
                         "gradients of the last timed step as DIR/<name>.npy")
    args = ap.parse_args()
    if args.quick:
        args.no_cpu_baseline = args.no_ref_cuda = args.no_other_configs = True
    if args.impl == "reference":
        return run_reference(args)
    return run_b200(args)


if __name__ == "__main__":
    sys.exit(main())
