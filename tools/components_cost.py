"""Cost and effect of the connected components (ngp_pl_b200.components, mesh.remove_small_components):

  occupancy  occupancy_components + remove_floaters(keep_largest=1) on random blobs and floaters at 128^3 with 1 and 6
             cascades, CUDA events, median of --reps (the bitfield restored between repetitions)
  mesh       mesh_components + remove_small_components on the sparse mesh of a trained Lego at each --resolution, and
             extract_mesh_sparse itself for scale; host scipy (oracle/components_ref.py: connected_components and the
             compaction) on the mesh at --baseline_res
  quality    on the trained Lego (cameras over the whole sphere, as tests/test_mesh_gpu.py trains it): the fraction of
             vertices outside every box and farther than 2 lattice cells from any box surface (floaters) and inside a
             box and deeper than 2 cells (cavity shells), before and after each filter; test-view PSNR before and after
             remove_floaters

Prints one JSON line with the card's name, power limit and clocks read in the same run.

    python tools/components_cost.py [--resolution 1024 2048] [--baseline_res 1024] [--steps 2000] [--reps 5]
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
from ngp_pl_b200 import components, mesh, metrics, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from oracle import components_ref as R  # noqa: E402


def event_ms(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def median(v):
    return round(sorted(v)[len(v) // 2], 3)


def trained_lego(steps):
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=100, K=K, device="cuda")
    bank.poses = torch.as_tensor(synth.camera_poses(100, radius=1.5, seed=0, upper_only=False), device="cuda")
    for i in range(100):
        bank.rgb[i] = (synth.trace(scene, *synth.get_rays(bank.directions, bank.poses[i])) * 255).round().to(torch.uint8)
    torch.manual_seed(0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr
    return scene, model


def fractions(scene, v, res):
    """(outside every box and farther than 2 cells, inside a box and deeper than 2 cells) of the vertices v"""
    lo = torch.as_tensor(scene.box_min, device=v.device)[None]
    hi = torch.as_tensor(scene.box_max, device=v.device)[None]
    far_o, deep_i = 0, 0
    for i in range(0, v.shape[0], 1 << 20):
        q = v[i:i + (1 << 20), None]
        inb = ((q > lo) & (q < hi)).all(-1)
        out = torch.clamp(torch.maximum(lo - q, q - hi), min=0).norm(dim=-1)
        depth = torch.minimum(q - lo, hi - q).min(-1)[0]
        dist = torch.where(inb, depth, out).min(-1)[0]
        near = dist <= 2.0 / (res - 1)
        inside = inb.any(-1)
        far_o += int((~inside & ~near).sum())
        deep_i += int((inside & ~near).sum())
    n = max(1, v.shape[0])
    return round(far_o / n, 5), round(deep_i / n, 5)


class Grid(torch.nn.Module):
    def __init__(self, bits, cascades, G, scale):
        super().__init__()
        self.cascades, self.grid_size, self.scale = cascades, G, scale
        self.register_buffer("density_bitfield", bits)


def occupancy_cost(cascades, scale, reps):
    G = 128
    rng = np.random.default_rng(cascades)
    coarse = rng.random((cascades, 16, 16, 16)) < 0.3
    occ = coarse.repeat(8, 1).repeat(8, 2).repeat(8, 3) | (rng.random((cascades, G, G, G)) < 1e-3)
    xyz = R.morton_coords(G)
    bits = torch.as_tensor(np.packbits(occ[:, xyz[:, 0], xyz[:, 1], xyz[:, 2]].reshape(-1), bitorder="little")).cuda()
    g = Grid(bits.clone(), cascades, G, scale)
    comp, clean = [], []
    for _ in range(reps + 1):
        g.density_bitfield.copy_(bits)
        comp.append(event_ms(lambda: components.occupancy_components(g))[0])
        ms, (_, st) = event_ms(lambda: components.remove_floaters(g, keep_largest=1, return_stats=True))
        clean.append(ms)
    return {"cascades": cascades, "G": G, "occupied": int(occ.sum()), "components": st["components"],
            "cleared": st["cleared_cells"] + st["cleared_inner"], "occupancy_components_ms": median(comp[1:]),
            "remove_floaters_ms": median(clean[1:])}


def psnr(model, poses, dirs, images):
    return round(float(metrics.evaluate(model, poses, dirs, images, (800, 800))["psnr"]), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, nargs="+", default=[1024, 2048])
    ap.add_argument("--baseline_res", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--views", type=int, default=10)
    args = ap.parse_args()
    res = {"gpu": gpu_info(), "occupancy": [occupancy_cost(1, 0.5, args.reps), occupancy_cost(6, 16.0, args.reps)]}
    t0 = time.perf_counter()
    scene, model = trained_lego(args.steps)
    res["train"] = {"steps": args.steps, "s": round(time.perf_counter() - t0, 1)}

    dirs = synth.ray_directions(synth.intrinsics(), "cuda")
    poses = torch.as_tensor(synth.camera_poses(args.views, seed=4321, upper_only=False)).cuda()
    images = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8)
                          for i in range(args.views)])
    bits0, dg0 = model.density_bitfield.clone(), model.density_grid.clone()
    q = {"psnr_before": psnr(model, poses, dirs, images)}
    for name, kw in (("keep_largest=1", {"keep_largest": 1}), ("min_cells=64", {"min_cells": 64})):
        _, st = components.remove_floaters(model, return_stats=True, **kw)
        m = mesh.extract_mesh_sparse(model, 512)
        q[name] = {"cleared": st["cleared_cells"] + st["cleared_inner"], "components": st["components"],
                   "psnr": psnr(model, poses, dirs, images),
                   "sparse512_far_deep": fractions(scene, m["vertices"], 512)}
        model.density_bitfield.copy_(bits0)
        model.density_grid.copy_(dg0)
    m = mesh.extract_mesh_sparse(model, 512)
    q["sparse512_far_deep_before"] = fractions(scene, m["vertices"], 512)
    res["occupancy_quality"] = q
    del m

    res["mesh"] = []
    for N in args.resolution:
        torch.cuda.empty_cache()
        ext_ms, m = event_ms(lambda: mesh.extract_mesh_sparse(model, N))
        row = {"resolution": N, "vertices": int(m["vertices"].shape[0]), "triangles": int(m["triangles"].shape[0]),
               "extract_mesh_sparse_ms": round(ext_ms, 1), "far_deep_before": fractions(scene, m["vertices"], N)}
        lab_ms, filt_ms = [], []
        for _ in range(max(2, args.reps // 2) + 1):
            lab_ms.append(event_ms(lambda: mesh.mesh_components(m))[0])
            ms, (o, st) = event_ms(lambda: mesh.remove_small_components(m, keep_largest=1, return_stats=True))
            filt_ms.append(ms)
            del o
        row.update(components=st["components"], mesh_components_ms=median(lab_ms[1:]),
                   remove_small_components_ms=median(filt_ms[1:]))
        lab, siz = mesh.mesh_components(m)
        counts = torch.sort(siz[siz > 0], descending=True)[0].cpu().numpy()
        row["largest_sizes"] = counts[:5].tolist()
        del lab, siz
        for name, kw in (("keep_largest=1", {"keep_largest": 1}), ("min_triangles=1000", {"min_triangles": 1000}),
                         ("min_triangles=10000", {"min_triangles": 10000})):
            o = mesh.remove_small_components(m, **kw)
            row[name] = {"triangles": int(o["triangles"].shape[0]), "far_deep": fractions(scene, o["vertices"], N)}
            del o
        if N == args.baseline_res:
            t = m["triangles"].cpu().numpy()
            v = m["vertices"].cpu().numpy()
            t0 = time.perf_counter()
            lab_o, siz_o = R.mesh_components(t, v.shape[0])
            keep_o, _ = R.select(lab_o, siz_o, keep_largest=1)
            R.mesh_filter(v, t, lab_o, keep_o)
            row["host_scipy_s"] = round(time.perf_counter() - t0, 2)
            del t, v, lab_o, siz_o, keep_o
        res["mesh"].append(row)
        del m
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
