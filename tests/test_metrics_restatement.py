"""CPU: the restatement of the reference's evaluation metrics (metrics_restatement.py) against a float32 torch conv2d
transcription of metrics.cpp and against the properties of the formula, and the Python mirror's formats and report
(metrics.py) against the reference's (metrics.hpp:78-103, metrics.cpp:212-289) character for character."""
import math
import re

import numpy as np
import pytest
import torch

import metrics_restatement as mr


@pytest.fixture(scope="module")
def M(pkg):
    from gsplat_b200 import metrics
    return metrics


def _pair(H, W, seed):
    rng = np.random.default_rng(seed)
    image = (rng.random((3, H, W)) * 1.4 - 0.2).astype(np.float32)  # exercises the clamp
    target = (0.7 * np.clip(image, 0, 1) + 0.3 * rng.random((3, H, W))).astype(np.float32)  # mid-range SSIM
    return image, target


@pytest.mark.parametrize("H,W", [(540, 960), (37, 53), (4, 9)])
def test_restatement_agrees_with_float32_torch_conv2d(H, W):
    image, target = _pair(H, W, H + W)
    p64, s64 = mr.metrics_f64(image, target)
    p32, s32 = mr.metrics_torch(torch.from_numpy(image), torch.from_numpy(target))
    print(f"[{H}x{W}] psnr {p64:.7f} / {p32:.7f}  ssim {s64:.9f} / {s32:.9f}")
    assert abs(s64 - s32) <= 7e-7
    assert abs(p64 - p32) <= 1e-4


def test_window_is_the_reference_quirk():
    w = mr.window_1d()
    assert w.dtype == np.float32 and w.shape == (11,)
    d2 = (np.arange(11) - 5).astype(np.float32) ** 2
    raw = np.exp(-d2 * np.float32(1.125)).astype(np.float32)  # 1.0f / 2.0f * 1.5f * 1.5f == 1.125f
    np.testing.assert_allclose(w, raw / raw.sum(dtype=np.float32), rtol=2e-7, atol=0)
    assert abs(w[4] / w[5] - np.exp(np.float32(-1.125))) <= 2 * np.spacing(np.float32(0.3247))
    np.testing.assert_allclose(w[:7], [3.65e-13, 9.11e-09, 2.40e-05, 6.65e-03, 1.94e-01, 5.98e-01, 1.94e-01], rtol=3e-3)
    assert np.array_equal(w, w[::-1]) and abs(float(w.sum(dtype=np.float64)) - 1.0) < 1e-6
    # not the training loss's sigma = 1.5 window
    assert w[5] > 0.5


@pytest.mark.parametrize("H,W", [(64, 96), (1, 1), (5, 37)])
def test_identical_images_give_one_and_100_db(H, W):
    rng = np.random.default_rng(3)
    x = rng.random((3, H, W)).astype(np.float32)
    p, s = mr.metrics_f64(x, x)
    assert abs(s - 1.0) <= 1e-6
    assert p == pytest.approx(100.0, abs=1e-9)
    p32, s32 = mr.metrics_torch(torch.from_numpy(x), torch.from_numpy(x))
    assert abs(s32 - 1.0) <= 1e-6 and abs(p32 - 100.0) <= 1e-4


def test_ssim_is_symmetric():
    rng = np.random.default_rng(4)
    a, b = rng.random((3, 41, 29)), rng.random((3, 41, 29))
    assert mr.metrics_f64(a, b)[1] == pytest.approx(mr.metrics_f64(b, a)[1], abs=1e-14)
    assert mr.metrics_f64(a, b)[0] == pytest.approx(mr.metrics_f64(b, a)[0], abs=1e-12)


def test_formats_match_the_reference(M):
    m = M.EvalMetrics(psnr=25.123456789, ssim=0.87654321, lpips=float("nan"), elapsed_time=0.0123,
                      num_gaussians=123456, iteration=7000)
    # the reference's EvalMetrics printed through its own iostream manipulators
    assert M.EvalMetrics.to_csv_header() == "iteration,psnr,ssim,lpips,time_per_image,num_gaussians"
    assert m.to_csv_row() == "7000,25.123457,0.876543,nan,0.012300,123456"
    m.lpips = 0.25
    assert m.to_string() == "PSNR: 25.1235, SSIM: 0.8765, LPIPS: 0.2500, Time: 0.0123s/image, #GS: 123456"


def test_reporter_csv_and_report(M, tmp_path):
    out = tmp_path / "run a"
    rep = M.MetricsReporter(out)
    assert (out / "metrics.csv").read_text() == "iteration,psnr,ssim,lpips,time_per_image,num_gaussians\n"
    E = M.EvalMetrics
    rows = [E(20.0, 0.70, 0.30, 0.01, 1000, 1000), E(25.0, 0.90, 0.35, 0.02, 2000, 2000),
            E(25.0, 0.85, 0.35, 0.03, 3000, 3000), E(24.0, 0.90, 0.20, 0.04, 4000, 4000)]
    for r in rows:
        rep.add_metrics(r)
    csv = (out / "metrics.csv").read_text().splitlines()
    assert len(csv) == 5 and csv[2] == "2000,25.000000,0.900000,0.350000,0.020000,2000"
    M.MetricsReporter(out)  # an existing CSV keeps its rows
    assert len((out / "metrics.csv").read_text().splitlines()) == 5
    rep.save_report()
    text = (out / "metrics_report.txt").read_text()
    assert text.startswith("==============================================\n3D Gaussian Splatting Evaluation Report\n"
                           "==============================================\n" f'Output Directory: "{out}"\n')
    assert re.search(r"\nGenerated: \d{4}-\d\d-\d\d \d\d:\d\d:\d\d\n\n", text)
    # metrics.cpp:236-247: the first of the equal best PSNRs and SSIMs; the LPIPS line takes min_element with a '>'
    # comparator, i.e. the first LARGEST LPIPS
    assert "Best PSNR:  25.0000 (at iteration 2000)\n" in text
    assert "Best SSIM:  0.9000 (at iteration 2000)\n" in text
    assert "Best LPIPS: 0.3500 (at iteration 2000)\n" in text
    assert ("\nFinal Metrics (iteration 4000):\nPSNR:  24.0000\nSSIM:  0.9000\nLPIPS: 0.2000\n"
            "Time per image: 0.0400 seconds\nNumber of Gaussians: 4000\n") in text
    assert text.endswith("\nDetailed Results:\n-----------------\n"
                         " Iteration      PSNR      SSIM     LPIPS    Time(s/img)     #Gaussians\n" + "-" * 75 + "\n"
                         "      1000   20.0000    0.7000    0.3000         0.0100           1000\n"
                         "      2000   25.0000    0.9000    0.3500         0.0200           2000\n"
                         "      3000   25.0000    0.8500    0.3500         0.0300           3000\n"
                         "      4000   24.0000    0.9000    0.2000         0.0400           4000\n")


def test_report_without_lpips_says_not_computed(M, tmp_path):
    rep = M.MetricsReporter(tmp_path)
    rep.add_metrics(M.EvalMetrics(21.5, 0.8, float("nan"), 0.01, 10, 500))
    text = rep.report()
    assert "Best LPIPS: not computed (at iteration 500)\n" in text and "\nLPIPS: not computed\n" in text
    assert (tmp_path / "metrics.csv").read_text().splitlines()[1] == "500,21.500000,0.800000,nan,0.010000,10"


def test_split_views_and_should_evaluate(M, tmp_path):
    train, val = M.split_views(20)
    assert val == [0, 8, 16] and train == [i for i in range(20) if i % 8]
    assert M.split_views(7, test_every=3)[1] == [0, 3, 6]
    ev = M.MetricsEvaluator(True, [7000, 30000], tmp_path)
    assert ev.should_evaluate(7000) and not ev.should_evaluate(7001)
    off = M.MetricsEvaluator(False, [7000], tmp_path / "off")
    assert not off.should_evaluate(7000) and not (tmp_path / "off").exists()
    with pytest.raises(RuntimeError, match="not enabled"):
        off.evaluate(7000, {}, 0, [], None)


def test_float_accumulation_of_the_means(M):
    vals = np.array([30.1, 29.7, 31.3], np.float32)
    s = np.float32(0)
    for v in vals:
        s = np.float32(s + v)
    assert M._mean_f32(vals) == float(np.float32(s / np.float32(3)))
    assert math.isnan(M._mean_f32([float("nan")] * 2))
