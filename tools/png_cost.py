"""Cost and size of the two PNG modes on 800x800 test views of a Lego model trained for --train-steps: the per-image
encode time of ngp_png_encode_mode in each mode (CUDA events over many calls, the modes alternated), metrics.evaluate
per view without save_dir and with it in each mode (alternated), and the files' sizes in each mode against Pillow's
compress_level=6 on the same arrays. Prints one JSON line with the card's name, power limit and maximum SM clock, and
the SM clock read after the timed work.

    python tools/png_cost.py [--launches 200] [--views 10] [--train-steps 1000] [--repeats 5]
"""
import argparse
import io
import json
import os
import shutil
import subprocess
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
from image_cost import events_ms  # noqa: E402

MODES = ("fixed", "dynamic")


def sm_clock():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm,power.draw",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30)
        return q.stdout.decode().strip()
    except Exception as e:
        return "nvidia-smi: %r" % (e,)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--views", type=int, default=10)
    ap.add_argument("--train-steps", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=5)
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

    # the encoder alone on the first view's images, the modes alternated
    out = render(model, *synth.get_rays(dirs, poses[0]), test_time=True)
    rgb_img, depth_img = I.view_images(out["rgb"].float().contiguous(), out["depth"].float().contiguous(), H, W)
    cap = I.png_capacity(H, W)
    ws = {m: I.png_workspace(H, W, "cuda", m) for m in MODES}
    buf_d = torch.empty(cap, dtype=torch.uint8, device="cuda")
    buf_h = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
    n = torch.zeros(1, dtype=torch.int64, pin_memory=True)
    enc = {}
    for _ in range(3):
        for m in MODES:
            for name, img in (("rgb", rgb_img), ("depth", depth_img)):
                for where, buf in (("device", buf_d), ("pinned", buf_h)):
                    t = events_ms(lambda: I.encode_png_into(img, buf, n, ws[m], m), a.launches)
                    enc.setdefault("%s_%s_%s_out" % (m, name, where), []).append(t)
    res["png_encode_ms"] = enc
    res["png_workspace_bytes"] = {m: ws[m].numel() for m in MODES}
    res["kernel_timing"] = "CUDA events around %d back-to-back calls after 10 warm-ups, 3 alternated rounds" % a.launches

    # evaluate per view: no files, and files in each mode, alternated
    root = tempfile.mkdtemp(prefix="ngp_png_cost_")
    dirs_out = {m: os.path.join(root, m) for m in MODES}

    def run(m):
        if m is None:
            return metrics.evaluate(model, poses, dirs, gts, (W, H))
        return metrics.evaluate(model, poses, dirs, gts, (W, H), save_dir=dirs_out[m], png_mode=m)
    r = [run(m) for m in (None,) + MODES]
    assert r[0] == r[1] == r[2], "evaluate's result changed with save_dir or png_mode"
    times = {"none": [], "fixed": [], "dynamic": []}
    for _ in range(a.repeats):
        for m in (None,) + MODES:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(m)
            torch.cuda.synchronize()
            times[m or "none"].append(1e3 * (time.perf_counter() - t0) / a.views)
    res["evaluate_ms_per_view"] = times
    res["dynamic_minus_fixed_ms_per_view"] = min(times["dynamic"]) - min(times["fixed"])
    res["view_timing"] = "host clock around %d views ending in a device synchronise, alternating, %d repeats" % (
        a.views, a.repeats)
    res["sm_clock_and_power_after"] = sm_clock()

    # sizes per view: each mode against Pillow level 6 on the same arrays
    from PIL import Image
    from oracle import png_ref
    size = {m: {"rgb": 0, "depth": 0} for m in MODES + ("pillow6",)}
    for i in range(a.views):
        for kind, suffix in (("rgb", ".png"), ("depth", "_d.png")):
            files = {m: open(os.path.join(dirs_out[m], "%03d%s" % (i, suffix)), "rb").read() for m in MODES}
            arr = png_ref.decode(files["fixed"])
            assert (png_ref.decode(files["dynamic"]) == arr).all()
            b = io.BytesIO()
            Image.fromarray(arr).save(b, format="PNG", compress_level=6)
            for m in MODES:
                size[m][kind] += len(files[m])
            size["pillow6"][kind] += len(b.getvalue())
    res["bytes_per_view"] = {m: {k: v / a.views for k, v in s.items()} for m, s in size.items()}
    res["size_over_pillow6"] = {m: {k: size[m][k] / size["pillow6"][k] for k in ("rgb", "depth")} for m in MODES}
    res["views"], res["train_steps"], res["test_psnr"] = a.views, a.train_steps, r[0]["psnr"]
    shutil.rmtree(root)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
