"""Cost and colour fidelity of texture baking (mesh.bake_texture, mesh.write_obj) on one trained model (synthetic Lego,
1000 training steps): the 1024^3 sparse mesh simplified at grids 128 and 256, baked at W = 4096 and 8192 with K = 16
samples from offset r = h (the cluster cell side).

  cost      median of `--reps` calls (CUDA events) of each step -- ngp_mesh_texture_atlas, _texels, _bake -- and of the
            PNG encode (images.encode_png, dynamic), the host time of write_obj, the baked texel count and the peak
            memory of bake_texture above its input (max_memory_allocated)
  fidelity  `--points` seeded area-uniform points q of the simplified mesh; the mean absolute 8-bit error against
            render(model, q + 2h n, -n, test_time=True) (n: the interpolated vertex normal) of three colourings: the
            texture with r = h and with r = 0 (bilinear at q's uv), and the simplified mesh's interpolated vertex colours
            (extracted with colors=True)

Prints one JSON line per case and a final one, with the card's name, power limit and clocks read in the same run.

    python tools/mesh_texture_cost.py [--reps 5] [--steps 1000] [--points 1048576] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from mesh_cost import gpu_info  # noqa: E402
from mesh_simplify_cost import peak_above, timed  # noqa: E402
from ngp_pl_b200 import _lib, images, mesh, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP, _net_struct  # noqa: E402
from ngp_pl_b200.models.rendering import render  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402


def steps(model, m, W, r, K, reps):
    """median ms of the three C calls, as bake_texture makes them"""
    L = _lib.lib()
    v, t, nrm = m["vertices"], m["triangles"], m["normals"]
    V, F = v.shape[0], t.shape[0]
    st = torch.cuda.current_stream().cuda_stream
    ws_bytes = L.ngp_mesh_texture_workspace(V, F, W)
    ws = torch.empty(ws_bytes, device="cuda", dtype=torch.uint8)
    uv = torch.empty(F, 3, 2, device="cuda")
    sq = torch.empty(F, 3, device="cuda", dtype=torch.int32)
    cnt = (C.c_int64 * 2)()
    atlas = lambda: _lib.check(L.ngp_mesh_texture_atlas(v.data_ptr(), V, t.data_ptr(), F, W, uv.data_ptr(),  # noqa: E731
                                                         sq.data_ptr(), cnt, ws.data_ptr(), ws_bytes, st), "atlas")
    a_ms, _, _ = timed(atlas, reps)
    n = int(cnt[1])
    tx = torch.empty(n, device="cuda", dtype=torch.int64)
    tri = torch.empty(n, device="cuda", dtype=torch.int32)
    p = torch.empty(n, 3, device="cuda")
    nn = torch.empty(n, 3, device="cuda")
    texels = lambda: _lib.check(L.ngp_mesh_texture_texels(v.data_ptr(), nrm.data_ptr(), V, t.data_ptr(), F, W,  # noqa: E731
                                                          uv.data_ptr(), n, tx.data_ptr(), tri.data_ptr(), p.data_ptr(),
                                                          nn.data_ptr(), ws.data_ptr(), ws_bytes, st), "texels")
    t_ms, _, _ = timed(texels, reps)
    del ws
    tex = torch.empty(W, W, 3, device="cuda", dtype=torch.uint8)
    bb = L.ngp_mesh_texture_bake_workspace(K)
    bws = torch.empty(bb, device="cuda", dtype=torch.uint8)
    net, keep = _net_struct(model)
    bake = lambda: _lib.check(L.ngp_mesh_texture_bake(C.byref(net), W, n, tx.data_ptr(), p.data_ptr(), nn.data_ptr(),  # noqa: E731
                                                      r, K, tex.data_ptr(), bws.data_ptr(), bb, st), "bake")
    b_ms, b_all, _ = timed(bake, reps)
    return {"atlas_ms": a_ms, "texels_ms": t_ms, "bake_ms": b_ms, "bake_ms_all": b_all, "S": int(cnt[0]), "texels": n}


def surface_points(m, n, seed):
    """n seeded area-uniform points: triangle ids and barycentrics"""
    v, t = m["vertices"].double(), m["triangles"]
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    area = torch.linalg.cross(b - a, c - a).norm(dim=1)
    g = torch.Generator(device="cuda").manual_seed(seed)
    pick = torch.searchsorted(torch.cumsum(area, 0), torch.rand(n, device="cuda", generator=g, dtype=torch.float64) *
                              area.sum()).clamp_(max=area.numel() - 1)
    r1, r2 = (torch.rand(n, device="cuda", generator=g, dtype=torch.float64) for _ in range(2))
    s = r1.sqrt()
    bary = torch.stack([1 - s, s * (1 - r2), s * r2], 1)
    return pick, bary


def mix(attr, t, pick, bary):
    return (attr[t[pick]].double() * bary[:, :, None]).sum(1)


def bilinear(tex, uv):
    """texel-centre bilinear lookup of the (W, W, 3) atlas at texel coordinates uv (texel row y is image row W-1-y)"""
    W = tex.shape[0]
    img = tex.flip(0).double()  # row y = texel row y
    x, y = uv[:, 0] - 0.5, uv[:, 1] - 0.5
    x0, y0 = x.floor().long(), y.floor().long()
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    at = lambda i, j: img[j.clamp(0, W - 1), i.clamp(0, W - 1)]  # noqa: E731
    return ((1 - fx) * (1 - fy) * at(x0, y0) + fx * (1 - fy) * at(x0 + 1, y0) + (1 - fx) * fy * at(x0, y0 + 1) +
            fx * fy * at(x0 + 1, y0 + 1))


@torch.no_grad()
def fidelity(model, s, textures, h, n_points):
    t = s["triangles"]
    pick, bary = surface_points(s, n_points, 7)
    q = mix(s["vertices"], t, pick, bary)
    nrm = mix(s["normals"], t, pick, bary)
    nrm = nrm / nrm.norm(dim=1, keepdim=True).clamp_min(1e-30)
    o = (q + 2 * h * nrm).float()
    ref = render(model, o.contiguous(), (-nrm).float().contiguous(), test_time=True)["rgb"].double() * 255
    out = {"vertex_colours": float((mix(s["colors"], t, pick, bary) - ref).abs().mean())}
    for name, tex in textures.items():
        uv = (tex["uv"][pick].double() * bary[:, :, None]).sum(1)
        out[name] = float((bilinear(tex["texture"], uv) - ref).abs().mean())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--points", type=int, default=1 << 20)
    ap.add_argument("--out", type=str, default=None, help="directory for the OBJ files (default: a temporary one)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mesh_texture_cost measures the GPU; there is no CPU path"
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
    out = {"gpu": gpu_info(), "model": "NGP(0.5), Lego after %d steps" % a.steps, "reps": a.reps, "K": 16, "cases": {}}
    raw = mesh.extract_mesh_sparse(model, 1024, normals=True, colors=True)
    out["raw"] = {"vertices": int(raw["vertices"].shape[0]), "triangles": int(raw["triangles"].shape[0])}
    tmpdir = tempfile.TemporaryDirectory()
    tmp = a.out or tmpdir.name
    for g in (128, 256):
        s = mesh.simplify_mesh(raw, g, box)
        h = float(mesh.cluster_grid(box[0], box[1], g).h)
        F = int(s["triangles"].shape[0])
        for W in (4096, 8192):
            key = "grid%d_W%d" % (g, W)
            if F * 16 > W * W:
                out["cases"][key] = {"triangles": F, "refused": "needs W >= %d" % mesh.texture_size_for(F)}
                print(json.dumps({key: out["cases"][key]}), flush=True)
                continue
            r = steps(model, s, W, h, 16, a.reps)
            torch.cuda.empty_cache()
            peak, tex = peak_above(lambda: mesh.bake_texture(model, s, W, h, 16))
            png_ms, _, png = timed(lambda: images.encode_png(tex["texture"], mode="dynamic"), a.reps)
            path = os.path.join(tmp, key + ".obj")
            t0 = time.perf_counter()
            mesh.write_obj(path, s["vertices"], s["triangles"], s["normals"], tex["uv"], tex["texture"])
            obj_s = time.perf_counter() - t0
            tex0 = mesh.bake_texture(model, s, W, 0.0, 16)
            r.update({"triangles": F, "vertices": int(s["vertices"].shape[0]), "h": h, "peak_mb": peak,
                      "png_ms": png_ms, "png_mb": len(png) / 2 ** 20, "write_obj_s": obj_s,
                      "obj_mb": os.path.getsize(path) / 2 ** 20,
                      "bake_plus_png_ms": r["atlas_ms"] + r["texels_ms"] + r["bake_ms"] + png_ms})
            r["mean_abs_error_8bit"] = fidelity(model, s, {"texture_r_h": tex, "texture_r_0": tex0}, h, a.points)
            e = r["mean_abs_error_8bit"]
            r["texture_at_most_half_vertex_error"] = e["texture_r_h"] <= 0.5 * e["vertex_colours"]
            r["r_h_beats_r_0"] = e["texture_r_h"] < e["texture_r_0"]
            out["cases"][key] = r
            print(json.dumps({key: r}), flush=True)
            del tex, tex0
            torch.cuda.empty_cache()
        del s
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    tmpdir.cleanup()


if __name__ == "__main__":
    main()
