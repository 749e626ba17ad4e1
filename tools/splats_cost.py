"""Cost of the Gaussian-splat export's device stages (ngp_pl_b200.splats) at --points points and --directions
directions, on a model with the reference's grid (L 16, T 2^19) and random weights, points uniform in its box with
random unit normals:

  colors    ngp_splat_colors: density once per point, then the colour MLP at every (point, direction) pair; the colour
            MLP's FLOPs (2 (32 64 + 64 64 + 64 8) per pair: the last layer runs 8 of its 16 outputs) over
            its time
  fit       ngp_splat_fit at SH degree 3 with hemisphere weights
  geometry  ngp_splat_geometry (disc) from the 3 nearest neighbours (the kNN itself is the point export's stage 5, not
            timed here)
  pack      the device-to-host copy of the packed (P, 62) fp32 array that write_splats makes
  render    one 800 x 800 view of all the splats through SplatRenderer's graph, camera at distance 2.5

Each stage is timed with CUDA events: `cold` is its first call in the process (module load, cub's first call, graph
capture for the renderer), `warm` the median of --reps further calls. Prints one JSON line with the card's name, power
limit and clocks read in the same run.

    python tools/splats_cost.py [--points 1000000] [--directions 128] [--reps 5] [--json out.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from mesh_cost import gpu_info  # noqa: E402
from ngp_pl_b200 import points, splats, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--directions", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", type=str, default=None, help="also write the result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "splats_cost measures the GPU; there is no CPU path"
    P, D = args.points, args.directions
    torch.manual_seed(0)
    model = NGP(0.5).cuda()
    with torch.no_grad():
        model.xyz_encoder.params[3072:].uniform_(-1, 1)
    g = torch.Generator().manual_seed(0)
    pts = ((torch.rand(P, 3, generator=g) * 2 - 1) * 0.45).cuda()
    nrm = torch.randn(P, 3, generator=g)
    nrm = (nrm / nrm.norm(dim=1, keepdim=True)).cuda()
    dirs = torch.as_tensor(splats.fibonacci_directions(D)).cuda()
    out = torch.zeros(P, 62, device="cuda")
    _, d2 = points.knn(pts, 3)
    state = {}

    def colors():
        state["sigma"], state["rgb"] = splats.colors_over_directions(model, pts, dirs)

    stages = {
        "colors": colors,
        "fit": lambda: splats.fit_sh(state["rgb"], dirs, nrm, out, 3, 1e-3),
        "geometry": lambda: splats.splat_geometry(pts, nrm, state["sigma"], d2, out, "disc", 0.1),
        "pack": lambda: out.cpu(),
    }
    res = {"points": P, "directions": D}
    for name, fn in stages.items():
        cold = timed(fn)
        warm = sorted(timed(fn) for _ in range(args.reps))[args.reps // 2]
        res[name] = {"cold_ms": round(cold, 3), "warm_ms": round(warm, 3)}
    flops = 2.0 * P * D * (32 * 64 + 64 * 64 + 64 * 8)
    res["colors"]["mlp_tflops"] = round(flops / (res["colors"]["warm_ms"] * 1e-3) / 1e12, 1)
    k = synth.intrinsics(W=800, H=800, fx=1111.11)
    K = np.array([[k["fx"], 0, k["cx"]], [0, k["fy"], k["cy"]], [0, 0, 1]], np.float32)
    pose = torch.as_tensor(synth.camera_poses(1, radius=2.5, seed=0)[0])
    t = {}

    def make():
        t["r"] = splats.SplatRenderer(out, (800, 800))
        t["r"].render(pose, K)

    cold = timed(make)
    r = t["r"]
    warm = sorted(timed(lambda: r.render(pose, K)) for _ in range(args.reps))[args.reps // 2]
    res["render"] = {"cold_ms": round(cold, 3), "warm_ms": round(warm, 3), "keys": int(r.n_keys.item()),
                     "capacity": r.capacity}
    res["gpu"] = gpu_info()
    print(json.dumps(res), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
