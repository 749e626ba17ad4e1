"""Cost of writing the validation pass's test-view images at 800x800: ngp_view_images and ngp_png_encode alone (CUDA
events over many launches), metrics.evaluate per view with and without save_dir (alternated, a model trained for a
few hundred steps on the synthetic Lego scene), the PNG sizes against Pillow's compress_level=6 on the same uint8
arrays, and Pillow's host encode time. Prints one JSON line, with the card's name and power limit.

    python tools/image_cost.py [--launches 200] [--views 10] [--train-steps 1000] [--out DIR]
"""
import argparse
import io
import json
import os
import shutil
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import images as I  # noqa: E402
from ngp_pl_b200 import metrics, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.models.rendering import render  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from eval_cost import card  # noqa: E402


def events_ms(fn, launches):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--views", type=int, default=10)
    ap.add_argument("--train-steps", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the saved views (default: a temporary one)")
    a = ap.parse_args()
    res = {"card": card()}
    scene = synth.lego_scene(0)
    H = W = 800
    dirs = synth.ray_directions(synth.intrinsics(), "cuda")
    poses = torch.as_tensor(synth.camera_poses(a.views, seed=4321)).cuda()
    gts = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8)
                       for i in range(a.views)])

    bank = synth.RayBank(scene, n_images=100, device="cuda", seed=0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(a.train_steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr, bank

    # the kernels alone, on the first view's render
    out = render(model, *synth.get_rays(dirs, poses[0]), test_time=True)
    rgb, depth = out["rgb"].float().contiguous(), out["depth"].float().contiguous()
    rgb_img, depth_img = I.view_images(rgb, depth, H, W)
    vws = torch.empty(4096, dtype=torch.uint8, device="cuda")
    res["view_images_ms"] = events_ms(lambda: I.view_images(rgb, depth, H, W, rgb_img, depth_img, vws), a.launches)
    cap, ws = I.png_capacity(H, W), I.png_workspace(H, W, "cuda")
    buf_d = torch.empty(cap, dtype=torch.uint8, device="cuda")
    buf_h = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
    n = torch.zeros(1, dtype=torch.int64, pin_memory=True)
    for name, img in (("rgb", rgb_img), ("depth", depth_img)):
        res["png_encode_ms_%s_device_out" % name] = events_ms(lambda: I.encode_png_into(img, buf_d, n, ws), a.launches)
        res["png_encode_ms_%s_pinned_out" % name] = events_ms(lambda: I.encode_png_into(img, buf_h, n, ws), a.launches)
    res["kernel_timing"] = "CUDA events around %d back-to-back calls after 10 warm-ups" % a.launches

    # evaluate per view with and without save_dir, alternated
    root = a.out or tempfile.mkdtemp(prefix="ngp_images_")
    save = os.path.join(root, "views")

    def plain():
        return metrics.evaluate(model, poses, dirs, gts, (W, H))

    def saving():
        return metrics.evaluate(model, poses, dirs, gts, (W, H), save_dir=save)
    r0, r1 = plain(), saving()
    assert r0 == r1, "evaluate's result changed with save_dir"
    t_p, t_s = [], []
    for _ in range(a.repeats):
        for fn, acc in ((plain, t_p), (saving, t_s)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            acc.append(1e3 * (time.perf_counter() - t0) / a.views)
    res["evaluate_ms_per_view"] = t_p
    res["evaluate_save_dir_ms_per_view"] = t_s
    res["save_dir_extra_ms_per_view"] = min(t_s) - min(t_p)
    res["view_timing"] = "host clock around %d views ending in a device synchronise, alternating, %d repeats" % (
        a.views, a.repeats)

    # sizes against Pillow on the same arrays, and Pillow's host encode time
    from PIL import Image
    ours, pil, pil_ms = {"rgb": 0, "depth": 0}, {"rgb": 0, "depth": 0}, []
    for i in range(a.views):
        for kind, suffix in (("rgb", ".png"), ("depth", "_d.png")):
            data = open(os.path.join(save, "%03d%s" % (i, suffix)), "rb").read()
            ours[kind] += len(data)
            with Image.open(io.BytesIO(data)) as im:
                arr = im.convert("RGB")
            t0 = time.perf_counter()
            b = io.BytesIO()
            arr.save(b, format="PNG", compress_level=6)
            pil_ms.append(1e3 * (time.perf_counter() - t0))
            pil[kind] += len(b.getvalue())
    res["png_bytes_per_view"] = {k: ours[k] / a.views for k in ours}
    res["pillow_level6_bytes_per_view"] = {k: pil[k] / a.views for k in pil}
    res["size_over_pillow"] = {k: ours[k] / pil[k] for k in ours}
    res["pillow_encode_ms_per_image"] = sorted(pil_ms)[len(pil_ms) // 2]
    res["pillow_encode_ms_per_view"] = 2 * res["pillow_encode_ms_per_image"]
    res["views"], res["train_steps"], res["test_psnr"] = a.views, a.train_steps, r0["psnr"]
    if a.out is None:
        shutil.rmtree(root)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
