"""Cost of the scene front end (ngp_pl_b200/datasets.py), one JSON line with the card's name and power limit:

  - load_scene on N RGBA 800x800 NeRF-synthetic views (written from SynthLego into a temporary directory first), split
    into Pillow decode, upload + ngp_stage_image, and the fp32 bank's device memory;
  - the batch assembly kernel (ngp_sample_rays_ex) per 8192-ray batch for uint8 / fp32 banks x all_images / same_image,
    CUDA events over many launches;
  - the captured training step with a uint8 and a fp32 bank of the same 100 views, arms alternated, medians of windows.

    python tools/dataset_cost.py [--views 100] [--launches 2000] [--steps 300] [--windows 5]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from ngp_pl_b200 import _lib, datasets, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from eval_cost import card  # noqa: E402


def write_views(root, scene, n):
    """n RGBA 800x800 views in the NeRF-synthetic layout, traced on the device"""
    import dataset_fixtures as F
    F.write_nerf(root, scene, size=800, splits=(("train", n),), images=False)
    K = synth.intrinsics()
    dirs = synth.ray_directions(K, "cuda")
    for i, c2w in enumerate(synth.camera_poses(n, radius=1.5, seed=0)):
        o, d = synth.get_rays(dirs, torch.as_tensor(c2w, device="cuda"))
        rgb = synth.trace(scene, o, d)
        hit = ~(rgb == scene.bg).all(-1)
        img = torch.cat([(rgb * 255).round().to(torch.uint8), (hit.to(torch.uint8) * 255)[:, None]], -1)
        F.save_png(os.path.join(root, "train", "r_%d.png" % i), img.reshape(800, 800, 4).cpu().numpy())


def load_cost(root):
    m = datasets.scene_meta("nerf", root, "train", 1.0)
    w, h = m.img_wh
    t0 = time.perf_counter()
    imgs = [datasets.decode_image(p) for p in m.image_paths]
    t_decode = time.perf_counter() - t0
    rgb = torch.empty(len(imgs), w * h, 3, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i, im in enumerate(imgs):
        datasets.stage_image(torch.from_numpy(im).to("cuda"), w, h, m.blend_a, rgb[i])
    torch.cuda.synchronize()
    t_stage = time.perf_counter() - t0
    # the kernel alone on one view, device-resident input
    src = torch.from_numpy(imgs[0]).cuda()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        datasets.stage_image(src, w, h, True, rgb[0])
    a.record()
    for _ in range(50):
        datasets.stage_image(src, w, h, True, rgb[0])
    b.record()
    torch.cuda.synchronize()
    t_kernel = a.elapsed_time(b) / 50
    t0 = time.perf_counter()
    datasets.load_scene("nerf", root, "train", 1.0)
    torch.cuda.synchronize()
    t_total = time.perf_counter() - t0
    return dict(views=len(imgs), decode_s=t_decode, upload_stage_s=t_stage, stage_kernel_ms_per_view=t_kernel,
                load_scene_s=t_total, bank_f32_MB=rgb.numel() * 4 / 1e6, bank_u8_MB=rgb.numel() / 1e6)


def sampler_us(bank_u8, bank_f32, launches, n=8192):
    out = {}
    o, d, c = (torch.empty(n, 3, device="cuda") for _ in range(3))
    z = torch.empty(n, device="cuda")
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    for dname, bank, dt in (("u8", bank_u8, 0), ("f32", bank_f32, 1)):
        for sname, s in (("all_images", 0), ("same_image", 1)):
            def go():
                L.ngp_sample_rays_ex(bank.poses.data_ptr(), bank.directions.data_ptr(), bank.rgb.data_ptr(), dt, s,
                                     bank.poses.shape[0], bank.directions.shape[0], n, 7, 0, ctr.data_ptr(), o.data_ptr(),
                                     d.data_ptr(), c.data_ptr(), z.data_ptr(), st)
            for _ in range(50):
                go()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(launches):
                go()
            b.record()
            torch.cuda.synchronize()
            out["%s_%s" % (dname, sname)] = a.elapsed_time(b) * 1e3 / launches
    return out


def step_ms(banks, steps, windows):
    """captured train_step, arms alternated window by window; median ms per step"""
    scene = synth.lego_scene(0)
    trs = {}
    for k, bank in banks.items():
        torch.manual_seed(0)
        tr = Trainer(NGP(scene.scale).cuda(), n_rays=8192)
        tr.attach_bank(bank)
        tr.capture()
        for _ in range(300):
            tr.train_step()
        trs[k] = tr
    res = {k: [] for k in banks}
    for _ in range(windows):
        for k, tr in trs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                tr.train_step()
            torch.cuda.synchronize()
            res[k].append((time.perf_counter() - t0) * 1e3 / steps)
    return {k: statistics.median(v) for k, v in res.items()}, {k: v for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dataset_cost.py measures on a CUDA device; none found")
    scene = synth.lego_scene(0)
    with tempfile.TemporaryDirectory() as root:
        write_views(root, scene, a.views)
        load = load_cost(root)
    bank_u8 = synth.RayBank(scene, n_images=a.views, device="cuda")
    bank_f32 = synth.RayBank(scene, n_images=a.views, device="cuda", store_dtype=torch.float32)
    samp = sampler_us(bank_u8, bank_f32, a.launches)
    med, all_ = step_ms({"u8": bank_u8, "f32": bank_f32}, a.steps, a.windows)
    print(json.dumps(dict(card=card(), load=load, sampler_us_per_8192=samp, step_ms_median=med, step_ms_windows=all_)))


if __name__ == "__main__":
    main()
