"""The float64 restatement of the validation metrics (oracle/metrics_ref.py) checked against itself and known answers:
the torchmetrics SSIM recipe (reflect pad, 2D correlation, crop) and the direct per-window sum agree; identical images,
constant images and uniform offsets give their closed forms; the Gaussian window equals torch's fp32 formula."""
import math

import numpy as np
import pytest
import torch

from oracle import metrics_ref as M

C1, C2 = 0.01 ** 2, 0.03 ** 2


def _pair(H, W, seed, u8_gt):
    rng = np.random.RandomState(seed)
    pred = rng.rand(H, W, 3).astype(np.float32)
    if u8_gt:
        gt = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
    else:  # correlated with pred, so that the covariance term matters
        gt = np.clip(pred + rng.normal(0, 0.1, (H, W, 3)), 0, 1).astype(np.float32)
    return pred, gt


@pytest.mark.parametrize("H,W", [(11, 11), (12, 29), (64, 64), (101, 77)])
@pytest.mark.parametrize("u8_gt", [False, True])
def test_recipe_and_direct_window_sum_agree(H, W, u8_gt):
    pred, gt = _pair(H, W, H * 1000 + W, u8_gt)
    a, b = M.ssim_conv(pred, gt), M.ssim_direct(pred, gt)
    assert abs(a - b) <= 1e-12, (a, b)
    assert -1 <= a <= 1


def test_identical_images():
    pred, _ = _pair(23, 31, 3, False)
    assert M.ssim_conv(pred, pred) == pytest.approx(1.0, abs=1e-12)
    assert M.ssim_direct(pred, pred) == pytest.approx(1.0, abs=1e-12)
    assert M.psnr(pred, pred) == math.inf
    u8 = (pred * 255).astype(np.uint8)
    assert M.psnr(u8, u8) == math.inf and M.ssim_conv(u8, u8) == pytest.approx(1.0, abs=1e-12)


@pytest.mark.parametrize("a,b", [(0.2, 0.7), (0.5, 0.5), (0.0, 1.0), (0.3, 0.35), (0.9, 0.1)])
def test_constant_images_closed_form(a, b):
    """two constant images: (2ab + c1) / (a^2 + b^2 + c1), the variances being zero. The fp32 window sums to S = (sum w)^2
    != 1 by ~1e-7, which leaves (a-b)^2 S(1-S) in the variance terms; the exact value with S is pinned to 1e-12 and the
    closed form to that bound"""
    A, B = np.full((13, 17, 3), a, np.float32), np.full((13, 17, 3), b, np.float32)
    a, b = float(np.float32(a)), float(np.float32(b))
    s1 = float(np.sum(M.gaussian_weights().astype(np.float64)))
    S = s1 * s1
    q, r = a * a + b * b, 2 * a * b
    exact = (r * S * S + C1) * (r * S * (1 - S) + C2) / ((q * S * S + C1) * (q * S * (1 - S) + C2))
    closed = (r + C1) / (q + C1)
    for f in (M.ssim_conv, M.ssim_direct):
        s = f(A, B)
        assert abs(s - exact) <= 1e-12
        assert abs(s - closed) <= (a - b) ** 2 * abs(S * (1 - S)) / C2 + 4 * abs(1 - S) + 1e-12


@pytest.mark.parametrize("delta", [0.5, 0.0390625, 2.0 ** -9, -0.125])
def test_psnr_of_uniform_offset(delta):
    """values on a 2^-10 grid, so that gt + delta is exact in fp32"""
    rng = np.random.RandomState(5)
    gt = (rng.randint(0, 256, (17, 19, 3)) / 1024.0 + 0.25).astype(np.float32)
    pred = (gt + np.float32(delta)).astype(np.float32)
    assert np.array_equal(pred.astype(np.float64) - gt.astype(np.float64), np.full(gt.shape, delta))
    assert M.psnr(pred, gt) == pytest.approx(-20 * math.log10(abs(delta)), abs=1e-12)


def test_gaussian_window_equals_fp32_formula():
    """torchmetrics' 1D window in fp32: exp(-(x / sigma)^2 / 2) over x = -5..5, normalised by its sum"""
    assert M.KSIZE == 11 and M.RADIUS == 5
    dist = torch.arange((1 - M.KSIZE) / 2, (1 + M.KSIZE) / 2, 1, dtype=torch.float32)
    g = torch.exp(-torch.pow(dist / M.SIGMA, 2) / 2)
    g = (g / g.sum()).numpy()
    w = M.gaussian_weights()
    assert w.dtype == np.float32 and np.array_equal(w, g)
    assert np.array_equal(w, w[::-1])


def test_uint8_reads_as_torch_division():
    v = np.arange(256, dtype=np.uint8).reshape(1, -1, 1).repeat(3, 2)
    t = (torch.arange(256, dtype=torch.uint8).float() / 255).numpy()
    assert np.array_equal(M.as_unit(v)[0, :, 0], t.astype(np.float64))


def test_metric_functions_refuse_cpu_tensors():
    from ngp_pl_b200 import metrics
    a, b = torch.rand(12, 12, 3), torch.rand(12, 12, 3)
    for call in (lambda: metrics.psnr(a, b), lambda: metrics.ssim(a, b),
                 lambda: metrics.evaluate(lambda o, d: None, torch.zeros(1, 3, 4), torch.zeros(144, 3), [b], (12, 12))):
        with pytest.raises(RuntimeError):
            call()
