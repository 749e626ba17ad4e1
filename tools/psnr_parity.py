"""PSNR parity at matched steps (BASELINE.json: "PSNR parity +-0.1 dB"): train this repo's path and the reference arm
(reference vren kernels + unmodified reference Python + tinycudann stand-in) on the same synthetic Lego scene with the
reference's recipe -- 8192 rays/step, Adam lr 1e-2 eps 1e-15, CosineAnnealingLR(T_max = epochs, eta_min = lr/30) stepped
per 1000-step epoch (train.py:131-137), occupancy refresh every 16 steps with a 256-step warm-up -- for the same number
of steps, and render the same held-out 800x800 views at the same checkpoints. Both arms are scored by
ngp_pl_b200.metrics.evaluate (per-view PSNR and SSIM as the reference's validation pass computes them).

    python tools/psnr_parity.py [steps] [out.json] [--tcnn fast|standin] [--views 8] [--res 800] [--no-cosine]
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import synth  # noqa: E402
from ngp_pl_b200.metrics import evaluate  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.models.rendering import render  # noqa: E402
from ngp_pl_b200.trainer import CosineAnnealingLR, Trainer  # noqa: E402

N_RAYS = 8192


def held_out_views(scene, n_views, res):
    K = synth.intrinsics(W=res, H=res, fx=1111.11 * res / 800)
    dirs = synth.ray_directions(K, "cuda")
    poses = torch.as_tensor(synth.camera_poses(n_views, seed=4321)).cuda()
    images = torch.stack([synth.trace(scene, *synth.get_rays(dirs, poses[i])) for i in range(n_views)])
    return poses, dirs, images


def eval_views(render_fn, views, res):
    poses, dirs, images = views
    return evaluate(render_fn, poses, dirs, images, (res, res))


def checkpoints(steps):
    return sorted({c for c in (1000, 2000, 5000, 10000, 20000, 30000) if c < steps} | {steps})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("steps", nargs="?", type=int, default=10000)
    ap.add_argument("out", nargs="?", default=None)
    ap.add_argument("--tcnn", default="fast", choices=["fast", "standin"])
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--res", type=int, default=800)
    ap.add_argument("--no-cosine", action="store_true")
    ap.add_argument("--skip-reference", action="store_true")
    a = ap.parse_args()
    steps = a.steps
    epochs = max(1, steps // 1000)
    scene = synth.lego_scene(0)
    cps = checkpoints(steps)
    views = held_out_views(scene, a.views, a.res)
    res = {"steps": steps, "rays_per_step": N_RAYS, "views": a.views, "resolution": a.res,
           "lr_schedule": None if a.no_cosine else "CosineAnnealingLR(T_max=%d epochs of 1000 steps, eta_min=lr/30)" % epochs,
           "reference_tcnn": a.tcnn, "checkpoints": cps}

    # ---- this repo -------------------------------------------------------------------------------------------
    bank = synth.RayBank(scene, n_images=100, device="cuda", seed=0)
    model = NGP(scene.scale).cuda()
    sched = None if a.no_cosine else CosineAnnealingLR(1e-2, T_max=epochs, steps_per_epoch=1000)
    tr = Trainer(model, n_rays=N_RAYS, lr=1e-2, lr_schedule=sched)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    curve = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    near = set()
    for c in cps:
        near.update(range(c - 49, c + 1))
    mses = []
    for step in range(1, steps + 1):
        tr.train_step()
        if step in near:  # train PSNR = mean MSE of the 50 batches before a checkpoint (one batch alone is +-0.5 dB noise)
            mses.append(tr.scalars[2].item() / (3 * N_RAYS))
        if step in cps:
            torch.cuda.synchronize()
            ev = eval_views(lambda o, d: render(model, o, d, test_time=True), views, a.res)
            tp = -10 * math.log10(max(float(np.mean(mses[-50:])), 1e-12))
            curve[str(step)] = {"test_psnr": ev["psnr"], "test_ssim": ev["ssim"], "views": ev["psnr_per_view"],
                                "views_ssim": ev["ssim_per_view"], "train_psnr_mean50": tp, "lr": tr.lr,
                                "samples_per_ray": tr.stats()["rm_samples"] / N_RAYS}
            print("b200 step %d: test %.3f dB  test_ssim %.4f  train(mean of 50 batches) %.3f dB  lr %.2e" % (
                step, ev["psnr"], ev["ssim"], tp, tr.lr), flush=True)
    res["b200"] = curve
    res["b200_wall_s"] = time.perf_counter() - t0
    del tr

    # ---- the reference arm -----------------------------------------------------------------------------------
    from oracle import ref_env
    if ref_env.available() and not a.skip_reference:
        ref = ref_env.load_reference(tcnn=a.tcnn)
        bank2 = synth.RayBank(scene, n_images=100, device="cuda", seed=0)
        m2 = ref.NGP(scale=scene.scale).cuda()
        G = m2.grid_size
        m2.register_buffer("density_grid", torch.zeros(m2.cascades, G ** 3, device="cuda"))
        gx = torch.stack(torch.meshgrid(*[torch.arange(G, dtype=torch.int32, device="cuda")] * 3, indexing="ij"), -1).reshape(-1, 3)
        m2.register_buffer("grid_coords", gx)
        opt = torch.optim.Adam(m2.parameters(), lr=1e-2, eps=1e-15, fused=True)
        sch = None if a.no_cosine else torch.optim.lr_scheduler.CosineAnnealingLR(opt, epochs, 1e-2 / 30)
        scaler = torch.amp.GradScaler("cuda")  # PL precision=16 (reference train.py:274)
        loss_fn = ref.losses.NeRFLoss(lambda_distortion=0)

        def ref_render(o, d):
            with torch.autocast("cuda", dtype=torch.float16):
                return ref.render(m2, o, d, test_time=True)
        curve = {}
        mses = []
        t0 = time.perf_counter()
        for step in range(1, steps + 1):
            o, d, rgb = bank2.sample(N_RAYS)
            with torch.autocast("cuda", dtype=torch.float16):
                if (step - 1) % 16 == 0:
                    m2.update_density_grid(0.01 * 1024 / 3 ** 0.5, warmup=(step - 1) < 256)
                r = ref.render(m2, o, d)
                loss = sum(v.mean() for v in loss_fn(r, {"rgb": rgb}).values())
            opt.zero_grad(set_to_none=True)
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()
            if step in near:
                mses.append(((r["rgb"].float() - rgb) ** 2).mean().item())
            if step in cps:
                torch.cuda.synchronize()
                ev = eval_views(ref_render, views, a.res)
                tp = -10 * math.log10(max(float(np.mean(mses[-50:])), 1e-12))
                curve[str(step)] = {"test_psnr": ev["psnr"], "test_ssim": ev["ssim"], "views": ev["psnr_per_view"],
                                    "views_ssim": ev["ssim_per_view"], "train_psnr_mean50": tp, "lr": opt.param_groups[0]["lr"],
                                    "samples_per_ray": float(r["rm_samples"]) / N_RAYS}
                print("reference step %d: test %.3f dB  test_ssim %.4f  train(mean of 50 batches) %.3f dB" % (
                    step, ev["psnr"], ev["ssim"], tp), flush=True)
            if sch is not None and step % 1000 == 0:
                sch.step()  # PL steps the scheduler at the end of every (1000-step) epoch
        res["reference"] = curve
        res["reference_wall_s"] = time.perf_counter() - t0
        res["delta_db"] = {k: res["b200"][k]["test_psnr"] - curve[k]["test_psnr"] for k in curve}
        res["delta_db_final"] = res["delta_db"][str(steps)]
        res["delta_ssim"] = {k: res["b200"][k]["test_ssim"] - curve[k]["test_ssim"] for k in curve}
        res["delta_train_db"] = {k: res["b200"][k]["train_psnr_mean50"] - curve[k]["train_psnr_mean50"] for k in curve}
    print(json.dumps(res))
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
