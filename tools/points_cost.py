"""Cost and quality of the point-cloud export (ngp_pl_b200.points) on the synthetic Lego trained for `--steps` steps,
cameras of 100 views at 800^2:

  stages    for each --num_rays: CUDA-event times of the rays, render and back-projection (summed over the chunks),
            voxel downsampling at --voxel, kNN (k 20), outlier removal and normals, and the end to end time of the
            whole pipeline (extract, outliers, normals; no checkpoint load, no file write), median of --reps
  baseline  the host float64 restatement of stages 5-7 on the same points: scipy cKDTree kNN, outlier rule and
            np.linalg.eigh normals (oracle/points_ref.py)
  quality   distance of the points to the nearest face of the scene's boxes (median and 95th percentile, in units of
            the scene), before and after outlier removal

Prints one JSON line per --num_rays, with the card's name, power limit and clocks read in the same run.

    python tools/points_cost.py [--num_rays 1000000 8000000] [--steps 1000] [--reps 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from mesh_cost import gpu_info  # noqa: E402
from ngp_pl_b200 import points, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from oracle import points_ref as P  # noqa: E402


def trained_lego(steps):
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=100, device="cuda")
    torch.manual_seed(0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr
    return scene, model, bank.poses, bank.directions


def face_distance(scene, p):
    """distance of each point to the nearest face of any of the scene's boxes (float64, numpy)"""
    lo, hi = np.asarray(scene.box_min, np.float64), np.asarray(scene.box_max, np.float64)
    c, h = (lo + hi) / 2, (hi - lo) / 2
    best = np.full(len(p), np.inf)
    for b in range(len(lo)):
        q = np.abs(p - c[b]) - h[b]
        outside = np.sqrt((np.maximum(q, 0) ** 2).sum(1))
        inside = np.minimum(q.max(1), 0)
        best = np.minimum(best, np.abs(outside + inside))
    return best


def event_ms(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_rays", type=int, nargs="+", default=[1000000, 8000000])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--voxel", type=int, default=256)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--baseline_max", type=int, default=2000000, help="skip the host baseline above this many points")
    args = ap.parse_args()
    info = gpu_info()
    t0 = time.perf_counter()
    scene, model, poses, dirs = trained_lego(args.steps)
    train_s = time.perf_counter() - t0
    for R in args.num_rays:
        res = {"num_rays": R, "gpu": info, "train_steps": args.steps, "train_s": round(train_s, 1)}
        points.extract_points(model, poses, dirs, num_rays=R)  # warm-up: module loads and the chunk's graph
        stage = {k: [] for k in ("rays", "render", "backproject", "extract", "voxel", "knn", "outliers", "normals",
                                 "end_to_end")}
        for _ in range(args.reps):
            tm = {}
            ms, pts = event_ms(lambda: points.extract_points(model, poses, dirs, num_rays=R, timings=tm))
            for k in ("rays", "render", "backproject"):
                stage[k].append(tm[k])
            stage["extract"].append(ms)
            stage["voxel"].append(event_ms(lambda: points.voxel_downsample(pts, args.voxel))[0])
            stage["knn"].append(event_ms(lambda: points.knn(pts["points"], args.k))[0])
            ms, kept = event_ms(lambda: points.remove_outliers(pts, args.k, 2.0))
            stage["outliers"].append(ms)
            stage["normals"].append(event_ms(lambda: points.estimate_normals(kept, args.k))[0])
            stage["end_to_end"].append(event_ms(lambda: points.estimate_normals(points.remove_outliers(
                points.extract_points(model, poses, dirs, num_rays=R), args.k, 2.0), args.k))[0])
        res["ms"] = {k: round(sorted(v)[len(v) // 2], 2) for k, v in stage.items()}
        res["points"] = {"extracted": int(pts["points"].shape[0]), "kept": int(kept["points"].shape[0])}
        p = pts["points"].cpu().numpy()
        if len(p) <= args.baseline_max:
            t0 = time.perf_counter()
            ti, td = P.knn_tree(p, args.k)
            keep, *_ = P.outliers(td, 2.0)
            q = p[keep]
            qi, _ = P.knn_tree(q, args.k)
            P.normals(q, pts["view"].cpu().numpy()[keep], qi)
            res["host_baseline_s"] = round(time.perf_counter() - t0, 2)
        else:
            res["host_baseline_s"] = "not measured (more than --baseline_max points)"
        d0 = face_distance(scene, p.astype(np.float64))
        d1 = face_distance(scene, kept["points"].cpu().numpy().astype(np.float64))
        res["face_distance"] = {"before": {"median": float(np.median(d0)), "p95": float(np.percentile(d0, 95))},
                                "after": {"median": float(np.median(d1)), "p95": float(np.percentile(d1, 95))}}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
