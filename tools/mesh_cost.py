"""Cost of mesh extraction on one trained model (synthetic Lego, 1000 training steps) at 256^3, 512^3 and 1024^3:

  density      density_volume (ngp_density_lattice: points generated in the kernel) against the notebook's route,
               model.density on N^3 materialised points (the mesh cell of the reference's test.ipynb), time and peak
               memory of each; and the per-point rate of k_ngp_fwd's density-only path on a 2^22-point batch
  mc           count + emit (marching_cubes at sigma 20, one host read-back of the counts inside)
  extract      the whole extract_mesh(model, N) with normals

CUDA events on the current stream, after one warm-up call of every shape. Arms compared with each other (density_volume
against the materialised route; count + emit with and without normals) are ALTERNATED within every repetition, and
each repetition times a window of back-to-back calls of at least `--window` ms; the per-call time reported is the
median over `--reps` repetitions, with the min and max beside it. Prints one JSON line, with the card's name, power
limit and clocks read in the same run.

    python tools/mesh_cost.py [--res 256 512 1024] [--reps 9] [--window 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import mesh, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE,
                             stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # the numbers are still worth printing; say why the card is not named
        return {"error": repr(e)}


def window_ms(fn, calls):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternated(arms, reps, window):
    """{name: fn} -> {name: {median, min, max} ms per call}: after a warm-up call of each, every repetition times each
    arm in turn over max(1, window / one-call time) back-to-back calls"""
    calls = {}
    for k, fn in arms.items():
        fn()
        torch.cuda.synchronize()
        calls[k] = max(1, int(window / max(window_ms(fn, 1), 1e-3)))
    ts = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            ts[k].append(window_ms(fn, calls[k]) / calls[k])
    return {k: {"median": sorted(v)[len(v) // 2], "min": min(v), "max": max(v), "calls_per_window": calls[k]}
            for k, v in ts.items()}


def peak_mb(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def materialised(model, n):
    lat = mesh.lattice(n, model._xyz_min_host, model._xyz_max_host)
    axes = [torch.tensor(lat.lo[a], device="cuda") + torch.arange(n, device="cuda").float() * torch.tensor(lat.step[a], device="cuda")
            for a in range(3)]
    x = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    return model.density(x).reshape(n, n, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--window", type=float, default=200.0)
    ap.add_argument("--steps", type=int, default=1000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mesh_cost measures the GPU; there is no CPU path"
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=100, K=synth.intrinsics(W=200, H=200, fx=1111.11 / 4), device="cuda")
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(a.steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr, bank
    torch.cuda.empty_cache()

    out = {"gpu": gpu_info(), "model": "NGP(0.5), L=16, T=2^19, Lego after %d steps" % a.steps, "reps": a.reps,
           "window_ms": a.window, "by_res": {}}
    x = torch.rand(1 << 22, 3, device="cuda") - 0.5
    t = alternated({"fwd": lambda: model.density(x)}, a.reps, a.window)["fwd"]
    out["k_ngp_fwd_density_random_points_gpts_per_s"] = (1 << 22) / t["median"] / 1e6
    for n in a.res:
        r = {}
        torch.cuda.empty_cache()
        try:
            t = alternated({"density_volume": lambda: mesh.density_volume(model, n),
                            "materialised": lambda: materialised(model, n)}, a.reps, a.window)
        except torch.OutOfMemoryError:
            t = alternated({"density_volume": lambda: mesh.density_volume(model, n)}, a.reps, a.window)
            t["materialised"] = "out of memory"
        r.update({k + "_ms": v for k, v in t.items()})
        r["density_volume_gpts_per_s"] = n ** 3 / t["density_volume"]["median"] / 1e6
        r["density_volume_peak_mb"] = peak_mb(lambda: mesh.density_volume(model, n))
        if t["materialised"] != "out of memory":
            r["materialised_peak_mb"] = peak_mb(lambda: materialised(model, n))
        torch.cuda.empty_cache()
        sigma = mesh.density_volume(model, n)
        v, tr_ = mesh.marching_cubes(sigma, 20.0)
        r["vertices"], r["triangles"] = v.shape[0], tr_.shape[0]
        del v, tr_
        t = alternated({"count_emit": lambda: mesh.marching_cubes(sigma, 20.0),
                        "count_emit_normals": lambda: mesh.marching_cubes(sigma, 20.0, normals=True)}, a.reps, a.window)
        r.update({k + "_ms": v for k, v in t.items()})
        del sigma
        torch.cuda.empty_cache()
        r["extract_mesh_ms"] = alternated({"x": lambda: mesh.extract_mesh(model, n)}, a.reps, a.window)["x"]
        out["by_res"][str(n)] = r
        print(n, r, file=sys.stderr, flush=True)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
