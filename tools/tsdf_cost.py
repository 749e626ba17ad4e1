"""Cost and quality of the TSDF mesh (ngp_pl_b200.fusion) on the synthetic Lego trained for `--steps` steps, cameras of
100 views at 800^2 (points_cost.py's scene), at each --resolution:

  ms        CUDA-event times of the render of every training pixel, the integration (state zeroing included), the
            masked marching cubes and the whole extract_mesh_tsdf, median of --reps
  bytes     the integration alone, timed on a fresh state: its state-traffic floor 2 * 24 B * N^3 * ceil(views /
            NGP_TSDF_GROUP) plus one read of the maps (20 B per pixel), and the achieved rate against that floor
  mesh      vertex and triangle counts
  quality   the four numbers of tests/test_mesh_gpu.py::test_extract_mesh_of_a_trained_lego -- vertices within 2
            lattice cells of a box surface overall and of those outside every box, vertices outside every box and
            farther, vertices inside a box and deeper -- for the TSDF mesh and for extract_mesh_sparse at the same
            lattice (threshold 20)

Prints one JSON line per --resolution, with the card's name, power limit and clocks read in the same run.

    python tools/tsdf_cost.py [--resolution 256 512 1024] [--steps 1000] [--reps 3]
"""
import argparse
import json
import math
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from mesh_cost import gpu_info  # noqa: E402
from points_cost import event_ms, trained_lego  # noqa: E402
from ngp_pl_b200 import _lib, fusion, mesh, synth  # noqa: E402


def box_distances(p, scene):
    """whether each vertex lies strictly inside some box, and its distance to the nearest box surface"""
    lo = torch.as_tensor(scene.box_min, device=p.device)[None]
    hi = torch.as_tensor(scene.box_max, device=p.device)[None]
    inb = torch.zeros(p.shape[0], dtype=torch.bool, device=p.device)
    dist = torch.empty(p.shape[0], device=p.device)
    for s in range(0, p.shape[0], 1 << 20):
        q = p[s:s + (1 << 20), None]
        ib = ((q > lo) & (q < hi)).all(-1)
        out = torch.clamp(torch.maximum(lo - q, q - hi), min=0).norm(dim=-1)
        depth = torch.minimum(q - lo, hi - q).min(-1)[0]
        inb[s:s + q.shape[0]] = ib.any(-1)
        dist[s:s + q.shape[0]] = torch.where(ib, depth, out).min(-1)[0]
    return inb, dist


def quality(V, scene, cell):
    inside, dist = box_distances(V, scene)
    near = dist <= 2 * cell
    n = max(V.shape[0], 1)
    return {"within_2_cells": round(float(near.float().sum()) / n, 4),
            "outside_within_2_cells": round(float(near[~inside].float().mean()) if (~inside).any() else 0.0, 4),
            "outside_and_farther": round(float((~inside & ~near).float().sum()) / n, 4),
            "inside_and_deeper": round(float((inside & ~near).float().sum()) / n, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    info = gpu_info()
    t0 = time.perf_counter()
    scene, model, poses, dirs = trained_lego(args.steps)
    train_s = time.perf_counter() - t0
    K = synth.intrinsics()
    Km = [[K["fx"], 0, K["cx"]], [0, K["fy"], K["cy"]], [0, 0, 1]]
    wh = (K["W"], K["H"])
    V, HW = poses.shape[0], K["W"] * K["H"]
    box = (model._xyz_min_host, model._xyz_max_host)
    for res in args.resolution:
        out = {"resolution": res, "gpu": info, "train_steps": args.steps, "train_s": round(train_s, 1), "views": V,
               "image": list(wh)}
        fusion.extract_mesh_tsdf(model, poses, Km, wh, res)  # warm-up: module loads, the render's graph
        stage = {k: [] for k in ("render", "integrate", "mesh", "end_to_end", "integrate_only")}
        for _ in range(args.reps):
            tm = {}
            ms, m = event_ms(lambda: fusion.extract_mesh_tsdf(model, poses, Km, wh, res, timings=tm))
            for k in ("render", "integrate", "mesh"):
                stage[k].append(tm[k])
            stage["end_to_end"].append(ms)
        maps = fusion.render_views(model, poses, dirs)
        for _ in range(args.reps):
            vol = fusion.tsdf_volume(res, box)
            torch.cuda.synchronize()
            stage["integrate_only"].append(event_ms(lambda: fusion.integrate(
                vol, poses, Km, wh, maps["depth"], maps["opacity"], maps["rgb"]))[0])
            del vol
        del maps
        out["ms"] = {k: round(sorted(v)[len(v) // 2], 2) for k, v in stage.items()}
        n = res ** 3
        floor = 2 * fusion.STATE_BYTES * n * math.ceil(V / _lib.NGP_TSDF_GROUP) + fusion.MAP_BYTES * V * HW
        out["integrate_bytes"] = {"floor": floor, "floor_GBps_at_measured": round(floor / out["ms"]["integrate_only"] / 1e6, 1)}
        out["mesh"] = {"vertices": int(m["vertices"].shape[0]), "triangles": int(m["triangles"].shape[0])}
        cell = 1.0 / (res - 1)
        sp = mesh.extract_mesh_sparse(model, res, normals=False)
        out["quality"] = {"tsdf": quality(m["vertices"], scene, cell), "sigma_sparse": quality(sp["vertices"], scene, cell)}
        out["sigma_sparse_vertices"] = int(sp["vertices"].shape[0])
        del m, sp
        torch.cuda.empty_cache()
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
