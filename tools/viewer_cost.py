"""Cost of one interactive-viewer frame at 800x800: show_gui.ViewRenderer.frame (ngp_render_view_frame, one CUDA graph
from the pose to the JPEG) against the same frame composed from the public pieces (synth.get_rays, render(test_time=True,
T_threshold=1e-2, max_samples=100), images.view_images, images.encode_jpeg with its read-back), on a Lego model after
1000 fused-Trainer steps on synth.lego_scene, along an orbit-camera path, in both display modes.

Per arm: the median over alternated windows of at least --window-ms of the wall time per frame (host clock around
whole frames, each ending in a synchronise) and of the device time per frame (CUDA events around each frame). Also the
JPEG bytes per frame of each mode, the card's name, power limit and maximum SM clock, and the SM clock and power draw
after the run. Prints one JSON line.

    python tools/viewer_cost.py [--train-steps 1000] [--poses 24] [--windows 9] [--window-ms 200]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import images as I  # noqa: E402
from ngp_pl_b200 import synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.models.rendering import render  # noqa: E402
from ngp_pl_b200.show_gui import OrbitCamera, ViewRenderer  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from eval_cost import card  # noqa: E402
from png_cost import sm_clock  # noqa: E402

QUALITY = 90
W = H = 800


def composed_frame(model, dirs, pose, mode):
    """the frame from today's public pieces, as a caller without ngp_render_view_frame would build it"""
    c2w = torch.as_tensor(np.asarray(pose, np.float32)[:3, :4]).cuda()
    res = render(model, *synth.get_rays(dirs, c2w), test_time=True, T_threshold=1e-2, max_samples=100)
    rgb_img, depth_img = I.view_images(res["rgb"] if mode == "rgb" else None, res["depth"] if mode == "depth" else None,
                                       H, W)
    return I.encode_jpeg(rgb_img if mode == "rgb" else depth_img, QUALITY)


def window(fn, poses, min_ms):
    """frames along the path, round and round, until min_ms have passed: (wall ms per frame, device ms per frame)"""
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in poses]
    dev_ms, n = [], 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while True:
        for (a, b), pose in zip(ev, poses):
            a.record()
            fn(pose)
            b.record()
        torch.cuda.synchronize()
        dev_ms += [a.elapsed_time(b) for a, b in ev]
        n += len(poses)
        elapsed = 1e3 * (time.perf_counter() - t0)
        if elapsed >= min_ms:
            return elapsed / n, statistics.median(dev_ms), elapsed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train-steps", type=int, default=1000)
    ap.add_argument("--poses", type=int, default=24)
    ap.add_argument("--windows", type=int, default=9)
    ap.add_argument("--window-ms", type=float, default=200.0)
    a = ap.parse_args()
    res = {"card": card(), "size": [W, H], "quality": QUALITY}

    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=100, device="cuda", seed=0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(a.train_steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr, bank

    Kd = synth.intrinsics(W=W, H=H)
    K = np.float32([[Kd["fx"], 0, Kd["cx"]], [0, Kd["fy"], Kd["cy"]], [0, 0, 1]])
    cam = OrbitCamera(K, (W, H), 1.5)
    cam.orbit(0, -700)
    poses = []
    for _ in range(a.poses):
        cam.orbit(360 / 0.05 / a.poses, 0)  # one turn around the model over the path
        poses.append(cam.pose)
    vr = ViewRenderer(model, K, (W, H), 0.0, QUALITY)
    dirs = vr.directions

    arms = {}
    for mode in ("rgb", "depth"):
        arms["view_" + mode] = lambda p, m=mode: vr.frame(p, m)
        arms["composed_" + mode] = lambda p, m=mode: composed_frame(model, dirs, p, m)
    for fn in arms.values():  # warm-up: graphs built, caches allocated
        for p in poses:
            fn(p)
    wall = {k: [] for k in arms}
    dev = {k: [] for k in arms}
    spans = []
    for _ in range(a.windows):
        for k, fn in arms.items():
            w, d, span = window(fn, poses, a.window_ms)
            wall[k].append(w)
            dev[k].append(d)
            spans.append(span)
    for k in arms:
        res["%s_wall_ms_per_frame" % k] = statistics.median(wall[k])
        res["%s_device_ms_per_frame" % k] = statistics.median(dev[k])
    for mode in ("rgb", "depth"):
        res["view_saving_%s_wall_ms" % mode] = res["composed_%s_wall_ms_per_frame" % mode] - res["view_%s_wall_ms_per_frame" % mode]
    res["timing"] = ("medians over %d windows per arm, arms alternated; each window renders the %d-pose path until at "
                     "least %.0f ms have passed (shortest window %.0f ms). wall: host clock per frame, every frame "
                     "ending in a synchronise; device: CUDA events around each frame, median over the window"
                     % (a.windows, a.poses, a.window_ms, min(spans)))

    samples, sizes, same = [], {}, {}
    for mode in ("rgb", "depth"):
        nb, eq = [], 0
        for p in poses:
            jpeg, info = vr.frame(p, mode)
            nb.append(len(jpeg))
            samples.append(info["samples_per_ray"])
            eq += jpeg == composed_frame(model, dirs, p, mode)
        sizes[mode] = float(np.mean(nb))
        same[mode] = eq
    res["jpeg_bytes_per_frame"] = sizes
    res["frames_byte_equal_to_composed"] = {m: "%d/%d" % (same[m], len(poses)) for m in same}
    res["samples_per_ray_mean"] = float(np.mean(samples))
    res["sm_clock_and_power_after"] = sm_clock()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
