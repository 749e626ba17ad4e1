"""Cost and quality of mesh simplification (mesh.simplify_mesh) on one trained model (synthetic Lego, 1000 training
steps), next to the extraction it follows:

  cost      512^3 and 1024^3 at grids 128 and 256, 2048^3 at grids 256 and 512 (no normals at 2048^3): simplify time
            (median of `--reps` single calls, CUDA events), its peak memory above the input mesh (max_memory_allocated),
            V' / F', and extract_mesh_sparse's time at that lattice
  quality   the 1024^3 mesh simplified at grid G against extract_mesh_sparse run directly at the lattice whose triangle
            count is within 10 % of the simplified one. Both are compared with the 1024^3 mesh: `--samples` area-uniform
            point samples per surface, nearest neighbours both ways through a uniform grid (torch), and the symmetric mean
            and 95th percentile in 1024^3 lattice steps. The sampling floor is the 1024^3 mesh against itself, sampled
            with a second seed.

Prints one JSON line per part and a final one, with the card's name, power limit and clocks read in the same run.

    python tools/mesh_simplify_cost.py [--reps 5] [--steps 1000] [--samples 16000000]
"""
import argparse
import json
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from mesh_cost import gpu_info  # noqa: E402
from ngp_pl_b200 import mesh, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402


def timed(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        out = None
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2], ts, out


def peak_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20, out


def sample(m, n, seed):
    """n points uniform in area on the mesh's triangles"""
    v, t = m["vertices"], m["triangles"]
    a, b, c = v[t[:, 0]].double(), v[t[:, 1]].double(), v[t[:, 2]].double()
    area = torch.linalg.cross(b - a, c - a).norm(dim=1)
    g = torch.Generator(device=v.device).manual_seed(seed)
    pick = torch.multinomial(area.float(), n, replacement=True, generator=g) if area.numel() < 2 ** 24 else \
        torch.searchsorted(torch.cumsum(area, 0), torch.rand(n, device=v.device, generator=g, dtype=torch.float64) *
                           area.sum()).clamp_(max=area.numel() - 1)
    r1, r2 = torch.rand(n, device=v.device, generator=g, dtype=torch.float64), torch.rand(n, device=v.device, generator=g,
                                                                                        dtype=torch.float64)
    s = r1.sqrt()
    p = (1 - s)[:, None] * a[pick] + (s * (1 - r2))[:, None] * b[pick] + (s * r2)[:, None] * c[pick]
    del a, b, c
    return p.float()


def nearest(q, p, cell, chunk=1 << 18):
    """distance from every q to its nearest p, through a uniform grid of side `cell` over the 27 neighbour cells; inf
    where no p lies in them (the nearest is then farther than `cell`)"""
    lo = torch.minimum(q.min(0).values, p.min(0).values) - cell
    key = lambda x: (((x - lo) / cell).floor().long() * torch.tensor([1 << 42, 1 << 21, 1], device=x.device)).sum(1)  # noqa: E731
    kp = key(p)
    kp, order = torch.sort(kp)
    p = p[order]
    uk, cnt = torch.unique_consecutive(kp, return_counts=True)
    start = torch.cumsum(cnt, 0) - cnt
    M = int(cnt.max())
    slot = torch.arange(M, device=p.device)
    off = torch.stack(torch.meshgrid(*[torch.arange(-1, 2, device=p.device)] * 3, indexing="ij"), -1).reshape(-1, 3)
    koff = (off * torch.tensor([1 << 42, 1 << 21, 1], device=p.device)).sum(1)
    out = torch.empty(q.shape[0], device=q.device)
    for s in range(0, q.shape[0], chunk):
        qq = q[s:s + chunk]
        best = torch.full((qq.shape[0],), float("inf"), device=q.device)
        kq = key(qq)
        for ko in koff:
            nk = kq + ko
            i = torch.searchsorted(uk, nk).clamp_(max=uk.numel() - 1)
            hit = uk[i] == nk
            idx = start[i][:, None] + slot[None, :]
            ok = hit[:, None] & (slot[None, :] < cnt[i][:, None])
            d = (p[idx.clamp_(max=p.shape[0] - 1)] - qq[:, None, :]).norm(dim=2)
            best = torch.minimum(best, torch.where(ok, d, torch.full_like(d, float("inf"))).min(1).values)
        out[s:s + chunk] = best
    return out


def distance(m, ref, n, step, seed=1, seed_ref=2):
    """symmetric mean and 95th percentile of the nearest-sample distance, in lattice steps"""
    a, b = sample(m, n, seed), sample(ref, n, seed_ref)
    cell = 8 * step
    d = torch.cat([nearest(a, b, cell), nearest(b, a, cell)]) / step
    far = float((~torch.isfinite(d)).float().mean())
    d = torch.where(torch.isfinite(d), d, torch.full_like(d, 8.0))  # a lower bound where nothing is within one cell
    return {"mean": float(d.mean()), "p95": float(torch.quantile(d[torch.randperm(d.numel(), device=d.device)[:1 << 24]],
                                                                 0.95)), "beyond_8_steps": far}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=16000000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mesh_simplify_cost measures the GPU; there is no CPU path"
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
    box = (model._xyz_min_host, model._xyz_max_host)
    out = {"gpu": gpu_info(), "model": "NGP(0.5), Lego after %d steps" % a.steps, "reps": a.reps, "cost": {}}
    for n, grids in ((512, (128, 256)), (1024, (128, 256)), (2048, (256, 512))):
        nrm = n < 2048
        ext_ms, ext_all, m = timed(lambda: mesh.extract_mesh_sparse(model, n, normals=nrm), 1 if n == 2048 else a.reps)
        r = {"extract_ms": ext_ms, "extract_ms_all": ext_all, "normals": nrm, "vertices": int(m["vertices"].shape[0]),
             "triangles": int(m["triangles"].shape[0]), "input_mb": sum(t.numel() * t.element_size() for t in m.values()
                                                                        if t is not None) / 2 ** 20, "grid": {}}
        for g in grids:
            ms, all_ms, s = timed(lambda: mesh.simplify_mesh(m, g, box), a.reps)
            del s
            peak, s = peak_above(lambda: mesh.simplify_mesh(m, g, box))
            r["grid"][g] = {"simplify_ms": ms, "simplify_ms_all": all_ms, "peak_mb": peak,
                            "vertices": int(s["vertices"].shape[0]), "triangles": int(s["triangles"].shape[0]),
                            "over_extract": ms / ext_ms}
            del s
        out["cost"][n] = r
        print(json.dumps({n: r}), flush=True)
        del m
        torch.cuda.empty_cache()

    # quality at equal size, against the 1024^3 mesh
    ref = mesh.extract_mesh_sparse(model, 1024, normals=False)
    step = float((model._xyz_max_host[0] - model._xyz_min_host[0]) / 1023)
    q = {"floor": distance(ref, ref, a.samples, step), "grids": {}}
    for g in (128, 256):
        s = mesh.simplify_mesh(ref, g, box)
        target = s["triangles"].shape[0]
        res = int(round(1024 * math.sqrt(target / ref["triangles"].shape[0])))
        for _ in range(6):  # triangle count grows about as res^2
            d = mesh.extract_mesh_sparse(model, res, normals=False)
            f = d["triangles"].shape[0]
            if abs(f - target) <= 0.1 * target:
                break
            res = max(2, int(round(res * math.sqrt(target / max(f, 1)))))
        e = {"simplified": distance(s, ref, a.samples, step), "direct": distance(d, ref, a.samples, step),
             "simplified_triangles": target, "direct_resolution": res, "direct_triangles": f,
             "direct_within_10pct": abs(f - target) <= 0.1 * target}
        e["simplified_lower_error"] = e["simplified"]["mean"] < e["direct"]["mean"]
        q["grids"][g] = e
        print(json.dumps({"quality_grid_%d" % g: e}), flush=True)
        del s, d
    out["quality"] = q
    print(json.dumps(out))


if __name__ == "__main__":
    main()
