"""Cost of the validation metrics: the ngp_image_metrics kernel on an 800x800 view (CUDA events over many launches), and
metrics.evaluate() against rendering the same views alone, with a model trained for a few hundred steps on the synthetic
Lego scene. Prints one JSON line, with the card's name and power limit.

    python tools/eval_cost.py [--launches 500] [--views 10] [--train-steps 1000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import metrics, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.models.rendering import render  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30)
        return q.stdout.decode().strip()
    except Exception as e:  # the name alone still says what was measured
        return "%s (nvidia-smi: %r)" % (torch.cuda.get_device_name(), e)


def kernel_ms(pred, gt, H, W, launches):
    out = torch.zeros(2, dtype=torch.float64, device="cuda")
    ws = metrics.workspace(H, W, "cuda")
    for _ in range(20):
        metrics.image_metrics(pred, gt, H, W, out[0], out[1], ws)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        metrics.image_metrics(pred, gt, H, W, out[0], out[1], ws)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--views", type=int, default=10)
    ap.add_argument("--train-steps", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    res = {"card": card()}
    scene = synth.lego_scene(0)
    H = W = 800
    K = synth.intrinsics()
    dirs = synth.ray_directions(K, "cuda")
    poses = torch.as_tensor(synth.camera_poses(a.views, seed=4321)).cuda()
    images = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8)
                          for i in range(a.views)])

    # the kernel alone, on a rendered-looking pair (ground truth + noise)
    g = torch.Generator(device="cuda").manual_seed(0)
    pred = (images[0].float() / 255 + 0.05 * torch.randn(H * W, 3, device="cuda", generator=g)).clamp(0, 1)
    res["kernel_ms_800x800_u8_gt"] = kernel_ms(pred, images[0], H, W, a.launches)
    res["kernel_ms_800x800_f32_gt"] = kernel_ms(pred, images[0].float() / 255, H, W, a.launches)
    res["kernel_timing"] = "CUDA events around %d back-to-back launches after 20 warm-ups, one workspace" % a.launches

    # evaluate() vs rendering alone, alternating
    bank = synth.RayBank(scene, n_images=100, device="cuda", seed=0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(a.train_steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr, bank

    def render_only():
        for i in range(a.views):
            o, d = synth.get_rays(dirs, poses[i])
            render(model, o, d, test_time=True)

    def with_metrics():
        return metrics.evaluate(model, poses, dirs, images, (W, H))
    render_only()
    with_metrics()
    t_r, t_e = [], []
    for _ in range(a.repeats):
        for fn, acc in ((render_only, t_r), (with_metrics, t_e)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            acc.append(1e3 * (time.perf_counter() - t0) / a.views)
    res["render_only_ms_per_view"] = t_r
    res["evaluate_ms_per_view"] = t_e
    res["evaluate_over_render"] = min(t_e) / min(t_r)
    res["views"], res["train_steps"] = a.views, a.train_steps
    res["test_psnr"], res["test_ssim"] = out["psnr"], out["ssim"]
    res["view_timing"] = "host clock around %d views ending in a device synchronise, alternating, %d repeats" % (a.views, a.repeats)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
