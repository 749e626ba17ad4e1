"""Cost of the Motion-JPEG videos of the validation pass at 800x800: ngp_jpeg_encode alone into device and into mapped
pinned memory (CUDA events over many launches), metrics.evaluate per view with save_dir alone and with video_fps=30
(alternated windows, a model trained on the synthetic Lego scene), the JPEG bytes per frame at quality 90 against this
project's PNGs and against Pillow's JPEG of the same arrays (libjpeg; the files are expected to be equal), and Pillow's
host encode time. Prints one JSON line, with the card's name and power limit.

    python tools/video_cost.py [--launches 200] [--views 30] [--train-steps 1000] [--out DIR]
"""
import argparse
import io
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import images as I  # noqa: E402
from ngp_pl_b200 import metrics, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.models.rendering import render  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from eval_cost import card  # noqa: E402
from image_cost import events_ms  # noqa: E402

QUALITY = 90


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--views", type=int, default=30, help="per evaluate call; 30 views make a window of over 200 ms")
    ap.add_argument("--train-steps", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the saved views and videos (default: a temporary one)")
    a = ap.parse_args()
    res = {"card": card(), "quality": QUALITY}
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

    # the encoder alone, on the first view's images
    out = render(model, *synth.get_rays(dirs, poses[0]), test_time=True)
    rgb_img, depth_img = I.view_images(out["rgb"].float().contiguous(), out["depth"].float().contiguous(), H, W)
    cap, ws = I.jpeg_capacity(H, W), I.jpeg_workspace(H, W, "cuda")
    buf_d = torch.empty(cap, dtype=torch.uint8, device="cuda")
    buf_h = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
    n = torch.zeros(1, dtype=torch.int64, pin_memory=True)
    for name, img in (("rgb", rgb_img), ("depth", depth_img)):
        res["jpeg_encode_ms_%s_device_out" % name] = events_ms(lambda: I.encode_jpeg_into(img, buf_d, n, ws, QUALITY), a.launches)
        res["jpeg_encode_ms_%s_pinned_out" % name] = events_ms(lambda: I.encode_jpeg_into(img, buf_h, n, ws, QUALITY), a.launches)
    png_ws = I.png_workspace(H, W, "cuda")
    png_d = torch.empty(I.png_capacity(H, W), dtype=torch.uint8, device="cuda")
    res["png_encode_ms_rgb_device_out"] = events_ms(lambda: I.encode_png_into(rgb_img, png_d, n, png_ws), a.launches)
    res["kernel_timing"] = "CUDA events around %d back-to-back calls after 10 warm-ups" % a.launches
    res["jpeg_capacity_bytes"], res["jpeg_workspace_bytes"] = cap, ws.numel()

    # evaluate per view with save_dir alone and with the videos, alternated
    root = a.out or tempfile.mkdtemp(prefix="ngp_video_")
    save, save_v = os.path.join(root, "views"), os.path.join(root, "views_video")

    def saving():
        return metrics.evaluate(model, poses, dirs, gts, (W, H), save_dir=save)

    def video():
        return metrics.evaluate(model, poses, dirs, gts, (W, H), save_dir=save_v, video_fps=30, video_quality=QUALITY)
    r0, r1 = saving(), video()
    assert r0 == r1, "evaluate's result changed with video_fps"
    t_s, t_v = [], []
    for _ in range(a.repeats):
        for fn, acc in ((saving, t_s), (video, t_v)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            acc.append(1e3 * (time.perf_counter() - t0) / a.views)
    res["evaluate_save_dir_ms_per_view"] = t_s
    res["evaluate_video_ms_per_view"] = t_v
    res["video_extra_ms_per_view"] = min(t_v) - min(t_s)
    res["view_timing"] = "host clock around %d views ending in a device synchronise (windows of %.0f ms), alternating, " \
        "%d repeats; the first call of each arm, which allocates the pinned slots for the first time, is not timed" % (
            a.views, min(t_s) * a.views, a.repeats)

    # sizes: the frames of the videos against the PNGs of the same views and against Pillow's JPEG of the same arrays
    from PIL import Image
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from test_jpeg_cpu import parse_avi
    sizes = {}
    pil_ms, equal = [], True
    for kind, suffix in (("rgb", ".png"), ("depth", "_d.png")):
        data = open(os.path.join(save_v, kind + ".avi"), "rb").read()
        frames = [data[p:p + m] for p, m in parse_avi(data)["frames"]]
        assert len(frames) == a.views
        png = pil = 0
        for i, f in enumerate(frames):
            path = os.path.join(save_v, "%03d%s" % (i, suffix))
            png += os.path.getsize(path)
            with Image.open(path) as im:
                arr = im.convert("RGB")
            t0 = time.perf_counter()
            b = io.BytesIO()
            arr.save(b, "JPEG", quality=QUALITY, subsampling=0, optimize=False)
            pil_ms.append(1e3 * (time.perf_counter() - t0))
            pil += len(b.getvalue())
            equal = equal and b.getvalue() == f
        sizes[kind] = {"jpeg_bytes_per_frame": sum(map(len, frames)) / a.views, "png_bytes_per_view": png / a.views,
                       "pillow_jpeg_bytes_per_frame": pil / a.views, "avi_bytes": len(data)}
    res["sizes"] = sizes
    res["frames_equal_pillow_jpeg"] = equal
    res["pillow_jpeg_encode_ms_per_image"] = float(np.median(pil_ms))
    res["views"], res["train_steps"], res["test_psnr"] = a.views, a.train_steps, r0["psnr"]
    if a.out is None:
        shutil.rmtree(root)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
