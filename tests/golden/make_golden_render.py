"""Render-level golden fixtures: the REAL reference (oracle/_ref: compiled `vren`, unmodified Python) on a GPU, on the
tests' seeded inputs. `python tests/golden/make_golden_render.py OUT_DIR`, then copy OUT_DIR/*.npz into tests/golden/.
Large outputs are stored as a fixed seeded sample (cases.sample_idx) and, where a test checks a whole array bit for bit,
as its SHA-256 (cases.digest)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import ref_env  # noqa: E402

N_GRAD = 4096    # hash-table gradient entries stored: the largest, and a sample of the nonzero ones
N_PIX = 2048     # pixels stored per test-time image
LOSS_RAYS = 32   # rays of the stored render that the loss fixture keeps


def np_(t):
    return t.detach().float().cpu().numpy()


def make_pair(ref, scene):
    from test_render_gpu import make_model
    mine = make_model(scene)
    theirs = ref.NGP(scene.scale).cuda()
    theirs.load_state_dict({k: v.clone() for k, v in mine.state_dict().items()}, strict=True)
    return mine, theirs


def grads_of(model):
    """both MLPs' gradients whole; of the hash table's (sparse, 11.4 M entries) the N_GRAD largest and N_GRAD of the
    nonzero ones (seeded), with their indices; each vector's max |g|"""
    ge = np_(dict(model.named_parameters())["xyz_encoder.params"].grad)
    gr = np_(dict(model.named_parameters())["rgb_net.params"].grad)
    t = ge[3072:]
    nz = np.flatnonzero(t)
    idx = np.union1d(np.argsort(-np.abs(t), kind="stable")[:N_GRAD], nz[cases.sample_idx(nz.size, N_GRAD)]) + 3072
    return dict(g_enc_absmax=np.float32(np.abs(ge).max()), g_rgb_absmax=np.float32(np.abs(gr).max()), g_density_mlp=ge[:3072],
                g_rgb=gr, g_table_idx=idx.astype(np.int32), g_table=ge[idx])


def image(res, prefix=""):
    n = res["rgb"].shape[0]
    idx = cases.sample_idx(n, N_PIX)
    return {prefix + k: np_(res[k])[idx] for k in ("rgb", "opacity", "depth")}


def render_train(ref, out_dir):
    from ngp_pl_b200 import synth
    for which in ("lego", "mip360"):
        scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
        _, theirs = make_pair(ref, scene)
        o, d = cases.rays_from_scene(scene, 2048, 31, extra_edge_cases=False)
        o, d = torch.as_tensor(o).cuda(), torch.as_tensor(d).cuda()
        kw = {} if scene.exp_step_factor == 0 else {"exp_step_factor": scene.exp_step_factor}
        torch.manual_seed(123)
        r = ref.render(theirs, o, d, **kw)
        ra = r["rays_a"][torch.argsort(r["rays_a"][:, 0])]
        tgt = torch.as_tensor(cases.target_rgb(o.shape[0], 31)).cuda()
        theirs.zero_grad()
        l = ref.losses.NeRFLoss(lambda_distortion=0)(r, {"rgb": tgt})
        sum(v.mean() for v in l.values()).backward()
        out = dict(rm_samples=np.int64(int(r["rm_samples"])), counts=ra[:, 2].cpu().numpy().astype(np.int32),
                   rgb=np_(r["rgb"]), opacity=np_(r["opacity"]), depth=np_(r["depth"]), keys=np.array(sorted(r.keys())))
        out.update(grads_of(theirs))
        np.savez_compressed(os.path.join(out_dir, "render_train_%s.npz" % which), **out)


def render_test(ref, out_dir):
    from ngp_pl_b200 import synth
    scene = synth.lego_scene(0)
    _, theirs = make_pair(ref, scene)
    K = synth.intrinsics(W=100, H=100, fx=1111.11 / 8)
    dirs = synth.ray_directions(K, "cuda")
    pose = torch.as_tensor(synth.camera_poses(3)[2]).cuda()
    o, d = synth.get_rays(dirs, pose)
    r = ref.render(theirs, o, d, test_time=True)
    np.savez_compressed(os.path.join(out_dir, "render_test.npz"), total_samples=np.int64(int(r["total_samples"])), **image(r))


def losses(ref, out_dir):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    scene = synth.mip360_scene(0)
    mine, _ = make_pair(ref, scene)
    o, d = cases.rays_from_scene(scene, 1024, 32, extra_edge_cases=False)
    o, d = torch.as_tensor(o).cuda(), torch.as_tensor(d).cuda()
    torch.manual_seed(7)
    r = render(mine, o, d, exp_step_factor=scene.exp_step_factor)
    ra = r["rays_a"][:LOSS_RAYS].clone()
    assert torch.equal(ra[:, 0].cpu(), torch.arange(LOSS_RAYS))
    sel = torch.cat([torch.arange(int(s), int(s) + int(n), device="cuda") for _, s, n in ra.tolist()])
    ra[:, 1] = torch.cumsum(ra[:, 2], 0) - ra[:, 2]
    inp = {"rgb": r["rgb"][:LOSS_RAYS], "opacity": r["opacity"][:LOSS_RAYS], "ws": r["ws"][sel], "deltas": r["deltas"][sel],
           "ts": r["ts"][sel], "rays_a": ra}
    inp = {k: v.detach().clone().contiguous() for k, v in inp.items()}
    for k in ("rgb", "opacity", "ws"):
        inp[k].requires_grad_(True)
    tgt = torch.as_tensor(cases.target_rgb(LOSS_RAYS, 32)).cuda()
    l = ref.losses.NeRFLoss(lambda_distortion=1e-3)(inp, {"rgb": tgt})
    g = torch.autograd.grad(l["distortion"].sum(), inp["ws"])[0]
    out = {"in_" + k: v.detach().cpu().numpy() for k, v in inp.items()}
    out.update(dws=np_(g), **{"loss_" + k: np_(l[k]) for k in ("rgb", "opacity", "distortion")})
    np.savez_compressed(os.path.join(out_dir, "losses.npz"), **out)


def mark_invisible(ref, out_dir):
    from ngp_pl_b200 import synth
    theirs = ref.NGP(2.0).cuda()
    G = 128
    coords = torch.stack(torch.meshgrid(*[torch.arange(G, dtype=torch.int32, device="cuda")] * 3, indexing="ij"), -1).reshape(-1, 3)
    theirs.register_buffer("density_grid", torch.zeros(theirs.cascades, G ** 3, device="cuda"))
    theirs.register_buffer("grid_coords", coords)
    Kd = synth.intrinsics(W=200, H=150, fx=180.0)
    K = torch.tensor([[Kd["fx"], 0, Kd["cx"]], [0, Kd["fy"], Kd["cy"]], [0, 0, 1]], device="cuda")
    poses = torch.as_tensor(synth.camera_poses(6, radius=1.2)).cuda()
    theirs.mark_invisible_cells(K, poses, (200, 150))
    dg = theirs.density_grid.cpu().numpy()
    cg = theirs.count_grid.cpu().numpy()
    assert set(np.unique(dg).tolist()) <= {-1.0, 0.0}
    k = np.round(cg * poses.shape[0])  # count_grid = cameras covering the cell / cameras
    assert np.allclose(cg, k / poses.shape[0]) and k.max() < 256
    np.savez_compressed(os.path.join(out_dir, "mark_invisible.npz"), invisible=np.packbits(dg < 0),
                        cameras_digest=cases.digest(k.astype(np.uint8)), n_cams=np.int64(poses.shape[0]),
                        shape=np.array(dg.shape))


def march_large(ref, out_dir):
    from ngp_pl_b200 import synth
    out = {}
    for tag, scene, esf, n_rays in (("lego", synth.lego_scene(0), 0.0, 1 << 18), ("mip360", synth.mip360_scene(0), 1.0 / 256, 1 << 16)):
        bits = torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda()
        o_np, d_np = cases.rays_from_scene(scene, n_rays, 77)
        o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
        center = torch.zeros(1, 3, device="cuda")
        half = torch.full((1, 3), scene.scale, device="cuda")
        _, hits_r, _ = ref.vren.ray_aabb_intersect(o, d, center, half, 1)
        hits_raw = hits_r.cpu().numpy().copy()
        t0 = hits_r[:, 0, 0]
        hits_r[:, 0, 0] = torch.where((t0 >= 0) & (t0 < 0.01), torch.full_like(t0, 0.01), t0)
        hits = hits_r[:, 0].contiguous()
        noise = torch.rand(n_rays, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
        ra, xyz, _, dl, ts, cnt = ref.vren.raymarching_train(o, d, hits, bits, scene.cascades, scene.scale, esf, noise, 128, 1024)
        tot = int(cnt[0])
        ra = ra[torch.argsort(ra[:, 0])]
        counts = ra[:, 2]
        seg = torch.repeat_interleave(torch.arange(n_rays, device="cuda"), counts)
        starts = torch.cumsum(counts, 0) - counts
        src = ra[:, 1][seg] + (torch.arange(tot, device="cuda") - starts[seg])  # all samples in ray order
        out.update({tag + "_total": np.int64(tot), tag + "_hits_digest": cases.digest(hits_raw),
                    tag + "_counts_digest": cases.digest(counts.cpu().numpy().astype(np.int32)),
                    tag + "_ts_digest": cases.digest(ts[src].cpu().numpy()), tag + "_deltas_digest": cases.digest(dl[src].cpu().numpy()),
                    tag + "_xyzs_digest": cases.digest(xyz[src].cpu().numpy())})
    np.savez_compressed(os.path.join(out_dir, "march_large.npz"), **out)


def composite_test(ref, out_dir):
    c = cases.composite_test_case()
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a)).cuda()  # noqa: E731
    alive, op, dp, rgb = T(c["alive"]), T(c["op0"]), T(c["dp0"]), T(c["rgb0"])
    hits = torch.zeros(c["op0"].shape[0], 2, device="cuda")
    ref.vren.composite_test_fw(T(c["sigmas"]), T(c["rgbs"]), T(c["deltas"]), T(c["ts"]), hits, alive, 1e-2, T(c["neff"]),
                               op, dp, rgb)
    np.savez_compressed(os.path.join(out_dir, "composite_test.npz"), alive=alive.cpu().numpy(), opacity=op.cpu().numpy(),
                        depth=dp.cpu().numpy(), rgb=rgb.cpu().numpy())


def drop_in(out_dir):
    """the reference's Python bound to THIS project's vren / tcnn: a regression snapshot of the drop-in path, not the
    reference's own numbers"""
    from ngp_pl_b200 import synth
    drop = ref_env.load_reference(drop_in=True)
    for which in ("lego", "mip360"):
        scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
        _, theirs = make_pair(drop, scene)
        o, d = cases.rays_from_scene(scene, 2048, 51, extra_edge_cases=False)
        o, d = torch.as_tensor(o).cuda(), torch.as_tensor(d).cuda()
        kw = {} if scene.exp_step_factor == 0 else {"exp_step_factor": scene.exp_step_factor}
        torch.manual_seed(5)
        r = drop.render(theirs, o, d, **kw)
        tgt = torch.as_tensor(cases.target_rgb(o.shape[0], 51)).cuda()
        op = r["opacity"] + 1e-10
        theirs.zero_grad()
        (((r["rgb"] - tgt) ** 2).mean() + (1e-3 * (-op * torch.log(op))).mean()).backward()
        K = synth.intrinsics(W=80, H=60, fx=1111.11 / 10)
        dirs = synth.ray_directions(K, "cuda")
        pose = torch.as_tensor(synth.camera_poses(3, radius=1.5 if which == "lego" else 0.9)[1]).cuda()
        o2, d2 = synth.get_rays(dirs, pose)
        a = drop.render(theirs, o2, d2, test_time=True, **kw)
        out = dict(rm_samples=np.int64(int(r["rm_samples"])), rays_a=r["rays_a"].cpu().numpy().astype(np.int32),
                   ts_digest=cases.digest(r["ts"].detach().cpu().numpy()), rgb=np_(r["rgb"]), opacity=np_(r["opacity"]),
                   depth=np_(r["depth"]), **image(a, "test_"))
        out.update(grads_of(theirs))
        np.savez_compressed(os.path.join(out_dir, "dropin_%s.npz" % which), **out)


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    ref = ref_env.load_reference()
    for f in (render_train, render_test, losses, mark_invisible, march_large, composite_test):
        f(ref, out_dir)
        print(f.__name__, "done", flush=True)
    drop_in(out_dir)
    print("golden written to", out_dir)


if __name__ == "__main__":
    main(sys.argv[1])
