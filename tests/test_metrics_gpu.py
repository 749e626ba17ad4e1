"""ngp_image_metrics (csrc/metrics.cu) and ngp_pl_b200.metrics against the float64 restatement oracle/metrics_ref.py.

The kernel accumulates the windowed moments and every sum in double, so it agrees with the float64 recipe far inside
the 1e-5 (SSIM) and 1e-6 relative (squared error) the reference's fp32 torchmetrics would need; the tests pin 1e-8 and
1e-10 relative."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import metrics_ref as M

pytestmark = pytest.mark.gpu

SIZES = [(11, 11), (13, 37), (200, 150), (800, 800), (45, 70)]  # 45 x 70: no multiple of the 32 x 32 tile either way


def _images(H, W, seed, u8_gt):
    """gt: noise over a smooth ramp, one flat rectangle; pred: gt plus noise, the rectangle flat at another value (flat
    regions whose images differ are where fp32 moments would stray furthest from the float64 recipe)"""
    rng = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    gt = np.clip(0.5 * (yy + xx)[..., None] * np.array([1.0, 0.8, 0.6]) + rng.normal(0, 0.05, (H, W, 3)), 0, 1)
    pred = np.clip(gt + rng.normal(0, 0.08, (H, W, 3)), 0, 1)
    gt[H // 4:H // 2 + 3, W // 5:W // 2 + 4] = 0.2
    pred[H // 4:H // 2 + 3, W // 5:W // 2 + 4] = 0.7
    pred = pred.astype(np.float32)
    gt = np.round(gt * 255).astype(np.uint8) if u8_gt else gt.astype(np.float32)
    return pred, gt


def _run(pred, gt, H, W, data_range=1.0):
    from ngp_pl_b200 import metrics
    out = torch.zeros(2, dtype=torch.float64, device="cuda")
    p = torch.as_tensor(pred).cuda().reshape(H * W, 3)
    g = torch.as_tensor(gt).cuda().reshape(H * W, 3)
    metrics.image_metrics(p, g, H, W, out[0], out[1], metrics.workspace(H, W, "cuda"), data_range)
    return out.cpu().numpy()


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("u8_gt", [False, True])
def test_kernel_matches_float64_recipe(H, W, u8_gt):
    pred, gt = _images(H, W, H * 7 + W, u8_gt)
    sse, ssim = _run(pred, gt, H, W)
    sse_o, ssim_o = M.sse(pred, gt), M.ssim_conv(pred, gt)
    assert abs(ssim - ssim_o) <= 1e-8, (ssim, ssim_o)
    assert abs(sse - sse_o) <= 1e-10 * sse_o, (sse, sse_o)


def test_two_calls_bitwise_equal_and_uint8_is_torch_division():
    H, W = 800, 800
    pred, gt = _images(H, W, 1, True)
    a, b = _run(pred, gt, H, W), _run(pred, gt, H, W)
    assert np.array_equal(a, b)
    gt_f = (torch.as_tensor(gt).float() / 255).numpy()  # what a uint8 image reads as
    assert np.array_equal(_run(pred, gt_f, H, W), a)


def test_data_range_and_identical_images():
    H, W = 37, 29
    pred, gt = _images(H, W, 2, False)
    sse, ssim = _run(pred * 2, gt * 2, H, W, data_range=2.0)
    assert abs(ssim - M.ssim_conv(pred, gt)) <= 1e-8  # c1, c2 scale with data_range^2: SSIM is scale-invariant
    sse, ssim = _run(pred, pred, H, W)
    assert sse == 0.0 and abs(ssim - 1.0) <= 1e-12


def test_bad_arguments_return_einval():
    from ngp_pl_b200 import _lib
    lib = _lib.lib()
    H, W = 16, 16
    p = torch.rand(H * W, 3, device="cuda")
    g = torch.rand(H * W, 3, device="cuda")
    out = torch.zeros(2, dtype=torch.float64, device="cuda")
    ws = torch.zeros(lib.ngp_image_metrics_workspace(4, 64), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    o0, o1 = out[0].data_ptr(), out[1].data_ptr()

    def call(pp, hh, ww, oo0, oo1, wsb):
        return lib.ngp_image_metrics(pp, g.data_ptr(), 0, hh, ww, 1.0, oo0, oo1, ws.data_ptr(), wsb, st)

    n = lib.ngp_image_metrics_workspace(H, W)
    assert 0 < n <= ws.numel()
    assert call(p.data_ptr(), H, W, o0, o1, n) == 0
    for rc in (call(p.data_ptr(), 10, W, o0, o1, n), call(p.data_ptr(), H, 10, o0, o1, n),  # H or W below 11
               call(None, H, W, o0, o1, n), call(p.data_ptr(), H, W, None, o1, n),          # null pointers
               call(p.data_ptr(), H, W, o0, o1, n - 1)):                                     # short workspace
        assert rc == -22
        with pytest.raises(RuntimeError):
            _lib.check(rc, "ngp_image_metrics")
    assert call(p.data_ptr(), 4, 64, o0, None, ws.numel()) == 0  # squared error alone takes any shape
    torch.cuda.synchronize()
    assert out[0].item() == pytest.approx(float(((p[:256].double() - g[:256].double()) ** 2).sum()), rel=1e-12)
    from ngp_pl_b200 import metrics
    with pytest.raises(RuntimeError):
        metrics.ssim(torch.rand(10, 20, 3, device="cuda"), torch.rand(10, 20, 3, device="cuda"))


def test_psnr_and_ssim_functions():
    from ngp_pl_b200 import metrics
    H, W = 120, 90
    pred, gt = _images(H, W, 3, True)
    p = torch.as_tensor(pred).cuda()
    g = torch.as_tensor(gt).cuda()
    s = metrics.ssim(p, g)
    assert s.is_cuda and s.dtype == torch.float32 and s.dim() == 0
    assert abs(float(s) - M.ssim_conv(pred, gt)) <= 1e-6  # fp32 result
    s2 = metrics.ssim(p.permute(2, 0, 1)[None], (g.float() / 255).permute(2, 0, 1)[None])  # the reference's (1, 3, h, w)
    assert float(s2) == float(s)
    # reference metrics.py semantics on a ray batch (8191 rays: no image shape)
    n = 8191
    a = torch.rand(n, 3, device="cuda")
    b = torch.rand(n, 3, device="cuda")
    ps = metrics.psnr(a, b)
    assert ps.is_cuda and ps.dtype == torch.float32
    want = -10 * math.log10(float(((a - b).double() ** 2).mean()))
    assert abs(float(ps) - want) <= 1e-4
    assert float(metrics.psnr(a, a)) == math.inf
    m = torch.rand(n, device="cuda") > 0.5
    assert abs(float(metrics.psnr(a, b, valid_mask=m)) + 10 * math.log10(float(((a - b)[m] ** 2).mean()))) <= 1e-4
    assert metrics.psnr(a, b, reduction='none').shape == (n, 3)


def test_evaluate_equals_host_loop():
    from ngp_pl_b200 import metrics, synth
    from ngp_pl_b200.models.rendering import render
    from test_render_gpu import make_model
    scene = synth.lego_scene(0)
    model = make_model(scene)
    W, H = 64, 48
    K = synth.intrinsics(W=W, H=H, fx=1111.11 * W / 800)
    dirs = synth.ray_directions(K, "cuda")
    poses = torch.as_tensor(synth.camera_poses(3, seed=4321)).cuda()
    images = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8)
                          for i in range(3)])
    outs = []

    def render_fn(o, d):
        outs.append(render(model, o, d, test_time=True))
        return outs[-1]
    res = metrics.evaluate(render_fn, poses, dirs, images, (W, H))
    assert len(outs) == 3
    res_model = metrics.evaluate(model, poses, dirs, images, (W, H))  # the default renderer
    assert res_model["total_samples"] == res["total_samples"]
    assert np.allclose(res_model["ssim_per_view"], res["ssim_per_view"], rtol=0, atol=1e-6)
    total = 0
    for i, out in enumerate(outs):
        total += int(out["total_samples"])
        pred = out["rgb"].float().reshape(H, W, 3).cpu().numpy()
        gt = images[i].reshape(H, W, 3).cpu().numpy()
        assert abs(res["psnr_per_view"][i] - M.psnr(pred, gt)) <= 1e-9
        assert abs(res["ssim_per_view"][i] - M.ssim_conv(pred, gt)) <= 1e-8
        mse = float(((out["rgb"].float() - images[i].float() / 255) ** 2).mean())
        assert abs(res["psnr_per_view"][i] - (-10 * math.log10(mse))) <= 1e-3
    assert res["total_samples"] == total > 0
    assert res["psnr"] == pytest.approx(np.mean(res["psnr_per_view"]), abs=1e-12)
    assert res["ssim"] == pytest.approx(np.mean(res["ssim_per_view"]), abs=1e-12)
