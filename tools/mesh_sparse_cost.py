"""Cost of sparse mesh extraction (extract_mesh_sparse) against the dense extract_mesh on one trained model (synthetic
Lego, 1000 training steps):

  dense vs sparse   256^3, 512^3, 1024^3 with normals, the two arms ALTERNATED in every repetition, each repetition a
                    window of back-to-back calls of at least `--window` ms; median (min, max) per call over `--reps`
  sparse alone      2048^3 and 4096^3 (no normals at 4096^3), `--reps_large` single calls
  phases            per lattice, CUDA events between the steps of one sparse call: brick mask, pass 1
                    (ngp_mesh_sparse_bricks), pass 2 + count (ngp_mesh_sparse_count), emit; the active / visited /
                    surface brick fractions, the vertex count and the peak memory of the call (max_memory_allocated)
  overlap at 512^3  how many of the dense mesh's vertices (bitwise) the sparse mesh has

Prints one JSON line, with the card's name, power limit and clocks read in the same run.

    python tools/mesh_sparse_cost.py [--reps 7] [--window 300] [--steps 1000]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from mesh_cost import alternated, gpu_info, peak_mb  # noqa: E402
from ngp_pl_b200 import _lib, mesh, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP, _net_struct  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402


def phases(model, n, normals=True):
    """one sparse extraction step by step, with CUDA events between the steps (ms each)"""
    L = _lib.lib()
    lat = mesh.lattice(n, model._xyz_min_host, model._xyz_max_host)
    st = torch.cuda.current_stream().cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    torch.cuda.synchronize()
    ev[0].record()
    mask = mesh._brick_mask(model, lat)
    ev[1].record()
    net, keep = _net_struct(model)
    ws_bytes = L.ngp_mesh_sparse_workspace(C.byref(lat))
    ws = torch.empty(ws_bytes, device="cuda", dtype=torch.uint8)
    bc = (C.c_int64 * 3)()
    _lib.check(L.ngp_mesh_sparse_bricks(C.byref(net), C.byref(lat), 20.0, mask.data_ptr(), bc, ws.data_ptr(), ws_bytes, st), "b")
    ev[2].record()
    sf_bytes = L.ngp_mesh_surface_workspace(C.byref(lat), bc[2])
    sf = torch.empty(sf_bytes, device="cuda", dtype=torch.uint8)
    tot = (C.c_int64 * 2)()
    _lib.check(L.ngp_mesh_sparse_count(C.byref(net), C.byref(lat), 20.0, mask.data_ptr(), bc[2], tot, ws.data_ptr(), ws_bytes,
                                       sf.data_ptr(), sf_bytes, st), "c")
    ev[3].record()
    del ws
    verts = torch.empty(tot[0], 3, device="cuda")
    nrm = torch.empty(tot[0], 3, device="cuda") if normals else None
    tris = torch.empty(tot[1], 3, device="cuda", dtype=torch.int64)
    _lib.check(L.ngp_mesh_sparse_emit(C.byref(lat), 20.0, bc[2], verts.data_ptr(), nrm.data_ptr() if normals else None,
                                      tris.data_ptr(), tot[0], tot[1], sf.data_ptr(), sf_bytes, st), "e")
    ev[4].record()
    torch.cuda.synchronize()
    nb = int(np.prod([(lat.n[a] + 7) // 8 for a in range(3)]))
    return {"mask_ms": ev[0].elapsed_time(ev[1]), "pass1_ms": ev[1].elapsed_time(ev[2]),
            "pass2_count_ms": ev[2].elapsed_time(ev[3]), "emit_ms": ev[3].elapsed_time(ev[4]),
            "bricks": nb, "active_frac": bc[0] / nb, "visited_frac": bc[1] / nb, "surface_frac": bc[2] / nb,
            "surface_ws_mb": sf_bytes / 2 ** 20, "vertices": int(tot[0]), "triangles": int(tot[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--reps_large", type=int, default=3)
    ap.add_argument("--window", type=float, default=300.0)
    ap.add_argument("--steps", type=int, default=1000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mesh_sparse_cost measures the GPU; there is no CPU path"
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
    out = {"gpu": gpu_info(), "model": "NGP(0.5), Lego after %d steps" % a.steps, "reps": a.reps, "res": {}}
    for n in (256, 512, 1024):
        t = alternated({"dense": lambda: mesh.extract_mesh(model, n),
                        "sparse": lambda: mesh.extract_mesh_sparse(model, n)}, a.reps, a.window)
        r = {"dense_ms": t["dense"], "sparse_ms": t["sparse"],
             "dense_peak_mb": peak_mb(lambda: mesh.extract_mesh(model, n)),
             "sparse_peak_mb": peak_mb(lambda: mesh.extract_mesh_sparse(model, n)), "phases": phases(model, n)}
        r["dense_vertices"] = int(mesh.extract_mesh(model, n, normals=False)["vertices"].shape[0])
        out["res"][n] = r
        print(json.dumps({n: r}), flush=True)
    for n in (2048, 4096):
        nrm = n < 4096
        try:
            mesh.extract_mesh_sparse(model, n, normals=nrm)
        except RuntimeError as e:  # the output alone may not fit: report what it needs
            out["res"][n] = {"error": str(e)}
            print(json.dumps({n: out["res"][n]}), flush=True)
            torch.cuda.empty_cache()
            continue
        ts = []
        for _ in range(a.reps_large):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            mesh.extract_mesh_sparse(model, n, normals=nrm)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        r = {"sparse_ms": sorted(ts)[len(ts) // 2], "sparse_ms_all": ts, "normals": nrm,
             "sparse_peak_mb": peak_mb(lambda: mesh.extract_mesh_sparse(model, n, normals=nrm)),
             "phases": phases(model, n, normals=nrm)}
        out["res"][n] = r
        print(json.dumps({n: r}), flush=True)
        torch.cuda.empty_cache()
    d = mesh.extract_mesh(model, 512, normals=False)["vertices"].cpu().numpy().view(np.uint32)
    s = mesh.extract_mesh_sparse(model, 512, normals=False)["vertices"].cpu().numpy().view(np.uint32)
    ds = {tuple(v) for v in d}
    out["overlap_512"] = {"dense_vertices": len(d), "sparse_vertices": len(s),
                          "dense_in_sparse": len(ds & {tuple(v) for v in s})}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
