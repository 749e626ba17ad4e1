"""The point-cloud export on an H100 (ngp_pl_b200.points, csrc/points.cu) against its numpy restatement
(oracle/points_ref.py): on a random-weight model and on a synthetic Lego trained as test_mesh_sparse_gpu's, the rays,
the render and the back-projection bitwise, voxel cells exactly, kNN distances, the outlier set and the normals, chunk
independence, determinism, and the CLI's file."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import points_ref as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _random_model():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    scene = synth.lego_scene(0)
    torch.manual_seed(1)
    model = NGP(scene.scale, n_levels=8, log2_hashmap_size=16).cuda()
    with torch.no_grad():
        model.xyz_encoder.params[3072:].uniform_(-1, 1)
        model.density_bitfield.copy_(torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda())
    K = synth.intrinsics(W=96, H=80, fx=120.0)
    return model, torch.as_tensor(synth.camera_poses(12, radius=1.5, seed=3, upper_only=False)), synth.ray_directions(K)


def _lego_cameras():
    from ngp_pl_b200 import synth
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    return torch.as_tensor(synth.camera_poses(60, radius=1.5, seed=0, upper_only=False)), synth.ray_directions(K)


@pytest.fixture(scope="module")
def lego():
    """the synthetic Lego trained for 300 steps, as test_mesh_sparse_gpu's fixture trains it, and its cameras"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=60, K=K, device="cuda")
    bank.poses = torch.as_tensor(synth.camera_poses(60, radius=1.5, seed=0, upper_only=False), device="cuda")
    for i in range(60):
        bank.rgb[i] = (synth.trace(scene, *synth.get_rays(bank.directions, bank.poses[i])) * 255).round().to(torch.uint8)
    torch.manual_seed(0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(300):
        tr.train_step()
    torch.cuda.synchronize()
    del tr
    poses, dirs = _lego_cameras()
    return model, poses, dirs


@pytest.fixture(scope="module", params=["random", "lego"])
def scene(request, lego):
    """(model, poses, directions, min_opacity): the random model is mostly transparent"""
    return _random_model() + (0.02,) if request.param == "random" else lego + (0.5,)


def _render_infer_bg0(model, o, d):
    """ngp_render_infer round by round with render()'s cfg and a black background"""
    from ngp_pl_b200 import _lib
    from ngp_pl_b200.models.networks import _net_struct
    from ngp_pl_b200.models.rendering import MAX_SAMPLES, NEAR_DISTANCE
    N = o.shape[0]
    L = _lib.lib()
    cfg = _lib.NgpInferCfg()
    cfg.n_rays, cfg.cascades, cfg.grid_size, cfg.max_samples = N, model.cascades, model.grid_size, MAX_SAMPLES
    cfg.scale, cfg.exp_step_factor = float(model.scale), 0.0
    cfg.T_threshold, cfg.near_distance = 1e-4, NEAR_DISTANCE
    c, h = model.center.flatten().tolist(), model.half_size.flatten().tolist()
    for k in range(3):
        cfg.center[k], cfg.half_size[k], cfg.bg[k] = c[k], h[k], 0.0
    cfg.sample_budget = MAX_SAMPLES
    cfg.max_round_samples = max(4 * N, 1 << 16)
    ws = torch.empty(L.ngp_render_infer_workspace(N, cfg.max_round_samples), device="cuda", dtype=torch.uint8)
    op, dep, rgb = torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, 3, device="cuda")
    total, alive = torch.zeros(1, device="cuda", dtype=torch.int64), torch.zeros(1, device="cuda", dtype=torch.int32)
    net, keep = _net_struct(model)
    st = torch.cuda.current_stream().cuda_stream
    first = 0
    while True:
        _lib.check(L.ngp_render_infer(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                      op.data_ptr(), dep.data_ptr(), rgb.data_ptr(), total.data_ptr(), first, 8, 0,
                                      alive.data_ptr(), ws.data_ptr(), ws.numel(), st), "render_infer")
        first += 8
        if int(alive.item()) == 0 or first > 2 * MAX_SAMPLES:
            break
    _lib.check(L.ngp_render_infer(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                  op.data_ptr(), dep.data_ptr(), rgb.data_ptr(), total.data_ptr(), first, 0, 1, None,
                                  ws.data_ptr(), ws.numel(), st), "render_infer")
    return op, dep, rgb


def test_rays_render_and_backprojection_bitwise(scene):
    from ngp_pl_b200 import _lib, points
    from ngp_pl_b200.models.rendering import render
    model, poses, dirs, min_op = scene
    R = 40000
    out = points.extract_points(model, poses, dirs, num_rays=R, min_opacity=min_op, return_rays=True)
    n_views, n_pix = poses.shape[0], dirs.shape[0]
    img, pix = P.ray_pixels(n_views, n_pix, R)
    assert np.array_equal(out["img_idx"].cpu().numpy(), img) and np.array_equal(out["pix_idx"].cpu().numpy(), pix)
    o, d = torch.empty(R, 3, device="cuda"), torch.empty(R, 3, device="cuda")
    P_, D_ = poses.cuda().contiguous(), dirs.cuda().contiguous()
    _lib.check(_lib.lib().ngp_gen_rays(out["img_idx"].data_ptr(), out["pix_idx"].data_ptr(), P_.data_ptr(), D_.data_ptr(),
                                       None, n_pix, R, o.data_ptr(), d.data_ptr(), None,
                                       torch.cuda.current_stream().cuda_stream), "gen_rays")
    assert _equal(out["rays_o"], o) and _equal(out["rays_d"], d)
    ref = render(model, o, d, test_time=True, exp_step_factor=0.0)
    assert _equal(out["opacity"], ref["opacity"]) and _equal(out["depth"], ref["depth"])
    op, dep, rgb = _render_infer_bg0(model, o, d)
    assert _equal(out["opacity"], op) and _equal(out["depth"], dep) and _equal(out["rgb"], rgb)
    lo, hi = model._xyz_min_host, model._xyz_max_host
    keep, p, c, v = P.backproject(o.cpu().numpy(), d.cpu().numpy(), op.cpu().numpy(), dep.cpu().numpy(), rgb.cpu().numpy(),
                                  min_op, lo, hi)
    assert keep.sum() > 100
    assert np.array_equal(out["points"].cpu().numpy().view(np.int32), p.view(np.int32))
    assert np.array_equal(out["colors"].cpu().numpy(), c)
    assert np.array_equal(out["view"].cpu().numpy().view(np.int32), v.view(np.int32))


def test_deterministic_and_chunking_changes_only_rounding(scene):
    """two calls are bitwise equal; another chunk size renders the same rays, and changes a ray's opacity and depth
    only by rounding (the wavefront's per-round sample quota, and with it the order of its compositing sums, follows
    the number of rays alive in the batch)"""
    from ngp_pl_b200 import points
    model, poses, dirs, min_op = scene
    kw = dict(num_rays=30000, min_opacity=min_op, bounds=([-0.3] * 3, [0.4] * 3), return_rays=True)
    a = points.extract_points(model, poses, dirs, **kw)
    b = points.extract_points(model, poses, dirs, **kw)
    c = points.extract_points(model, poses, dirs, chunk=4099, **kw)
    for k in a:
        if a[k] is not None:
            assert _equal(a[k], b[k]), k
    for k in ("img_idx", "pix_idx", "rays_o", "rays_d"):
        assert _equal(a[k], c[k]), k
    assert (a["opacity"] - c["opacity"]).abs().max() <= 1e-4
    assert ((a["depth"] - c["depth"]).abs() <= 1e-4 * (1 + a["depth"].abs())).all()
    assert (a["points"] >= -0.3).all() and (a["points"] <= 0.4).all()
    n = min(a["points"].shape[0], c["points"].shape[0])
    assert abs(a["points"].shape[0] - c["points"].shape[0]) <= 0.001 * n + 2
    e = points.estimate_normals(points.remove_outliers(a, 16, 1.5), 16)
    f = points.estimate_normals(points.remove_outliers(b, 16, 1.5), 16)
    for k in ("points", "colors", "view", "normals"):
        assert _equal(e[k], f[k]), k


@pytest.mark.parametrize("grid", [1, 7, 64, 300])
def test_voxel_downsampling(lego, grid):
    from ngp_pl_b200 import mesh, points
    model, poses, dirs = lego
    pts = points.extract_points(model, poses, dirs, num_rays=200000)
    vox = points.voxel_downsample(pts, grid, return_cells=True)
    mn, mx = torch.aminmax(pts["points"], dim=0)
    g = mesh.cluster_grid(mn.cpu().numpy(), mx.cpu().numpy(), grid)
    keys, cnt, pos, col, view = P.voxel(pts["points"].cpu().numpy(), pts["colors"].cpu().numpy(), pts["view"].cpu().numpy(),
                                        list(g.lo), g.h, list(g.n))
    assert np.array_equal(vox["key"].cpu().numpy(), keys) and np.array_equal(vox["count"].cpu().numpy(), cnt)
    got = vox["points"].cpu().numpy()
    ulp = np.spacing(np.abs(pos).astype(np.float32))
    assert (np.abs(got - pos) <= ulp).all()
    assert np.array_equal(vox["colors"].cpu().numpy(), col)
    assert np.abs(vox["view"].cpu().numpy() - view).max() < 1e-6


def _adversarial():
    rng = np.random.RandomState(2)
    base = rng.rand(3000, 3).astype(np.float32)
    t = rng.rand(2000).astype(np.float32)
    return {
        "duplicates": np.concatenate([base, base[:1500], base[:300]]),
        "coplanar": np.concatenate([rng.rand(4000, 2), np.zeros((4000, 1))], 1).astype(np.float32),
        "collinear": np.stack([t, 2 * t, -t], 1).astype(np.float32),
        "cluster_and_far": np.concatenate([rng.rand(3000, 3) * 1e-3, rng.randn(7, 3) * 100]).astype(np.float32),
        "all_equal": np.ones((300, 3), np.float32),
        "n_le_k_plus_1": rng.rand(17, 3).astype(np.float32),
        "two": rng.rand(2, 3).astype(np.float32),
    }


@pytest.mark.parametrize("name", list(_adversarial()))
@pytest.mark.parametrize("k", [1, 16, 64])
def test_knn_exact(name, k):
    from ngp_pl_b200 import points
    p = _adversarial()[name]
    idx, d2 = points.knn(torch.as_tensor(p).cuda(), k)
    ri, rd = P.knn(p, k)
    got = d2.cpu().numpy()
    assert got.shape == rd.shape
    assert (np.abs(got - rd) <= 1e-12 * rd).all()
    assert np.array_equal(idx.cpu().numpy(), ri)


def test_knn_outliers_and_normals_on_lego(lego):
    from ngp_pl_b200 import points
    model, poses, dirs = lego
    pts = points.extract_points(model, poses, dirs, num_rays=60000)
    p = pts["points"].cpu().numpy()
    idx, d2 = points.knn(pts["points"], 20)
    ri, rd = P.knn(p, 20)
    assert (np.abs(d2.cpu().numpy() - rd) <= 1e-12 * rd).all()
    assert np.array_equal(idx.cpu().numpy(), ri)
    kept, stats = points.remove_outliers(pts, 20, 2.0, return_stats=True)
    keep, d, mu, sigma, thr = P.outliers(rd, 2.0)
    assert abs(stats["mean"] - mu) <= 1e-12 * mu and abs(stats["std"] - sigma) <= 1e-10 * sigma
    near = np.abs(d - thr) <= 1e-12 * thr
    got = np.zeros(len(p), bool)
    got[stats["kept"].cpu().numpy()] = True
    assert np.array_equal(got[~near], keep[~near]) and (~keep).sum() > 0
    assert _equal(kept["points"], pts["points"][stats["kept"]])
    nrm = points.estimate_normals(kept, 20)
    q = kept["points"].cpu().numpy()
    ki, _ = P.knn(q, 20)
    rn, gap, zero = P.normals(q, kept["view"].cpu().numpy(), ki)
    gn = nrm["normals"].cpu().numpy().astype(np.float64)
    clear = (gap > 1e-6) & ~zero  # normal error <~ 1e-16 / gap
    assert clear.mean() > 0.5
    # the angle from the cross product: the fp32 normal's length is 1 only to rounding, which arccos of the dot would
    # read as an angle of sqrt(2 eps)
    ang = np.arcsin(np.clip(np.linalg.norm(np.cross(gn, rn), axis=1) / np.linalg.norm(gn, axis=1).clip(1e-30), 0, 1))
    assert ang[clear].max() < 1e-5
    vd = (rn * kept["view"].cpu().numpy()).sum(1)
    sure = clear & (np.abs(vd) > 1e-3)
    assert np.array_equal(np.sign((gn * rn).sum(1))[sure], np.ones(sure.sum()))
    assert ((gn * kept["view"].cpu().numpy()).sum(1) <= 1e-6).all()


def _write_nerf_scene(root, poses, dirs_K):
    """a NeRF-synthetic transforms_train.json whose cameras scene_meta reads back (no images)"""
    os.makedirs(root, exist_ok=True)
    frames = []
    for i, c2w in enumerate(poses):
        m = np.eye(4)
        m[:3] = c2w
        m[:3, 1:3] *= -1
        frames.append({"file_path": "./train/r_%d" % i, "transform_matrix": m.tolist()})
    fx = dirs_K
    json.dump({"camera_angle_x": 2 * math.atan(400 / fx), "frames": frames}, open(os.path.join(root, "transforms_train.json"), "w"))


def test_cli_writes_what_the_api_writes(lego, tmp_path):
    from ngp_pl_b200 import datasets, mesh, points, train
    model, poses, dirs = lego
    root = str(tmp_path / "scene")
    _write_nerf_scene(root, poses.numpy().astype(np.float64), 1111.11)
    meta = datasets.scene_meta("nerf", root, "train", 0.25)
    P_, D_ = torch.as_tensor(meta.poses), torch.as_tensor(meta.directions)
    full = str(tmp_path / "full.ckpt")
    slim = str(tmp_path / "slim.ckpt")
    ck = train.checkpoint(model, D_, P_, 0, 300)
    torch.save(ck, full)
    torch.save(train.slim_state_dict(ck), slim)
    pts = points.extract_points(model, P_, D_, num_rays=50000, min_opacity=0.6)
    pts = points.voxel_downsample(pts, 128)
    pts = points.remove_outliers(pts, 12, 2.5)
    pts = points.estimate_normals(pts, 12)
    api = str(tmp_path / "api.ply")
    mesh.write_ply(api, pts["points"], torch.empty(0, 3, dtype=torch.int64), pts["normals"], pts["colors"])
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    args = ["--num_rays", "50000", "--min_opacity", "0.6", "--voxel", "128", "--nb_neighbors", "12", "--std_ratio", "2.5"]
    outs = []
    for extra in (["--ckpt_path", full], ["--ckpt_path", slim, "--root_dir", root, "--downsample", "0.25"]):
        out = str(tmp_path / ("cli%d.ply" % len(outs)))
        r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.export_points"] + extra + args + ["--out", out], cwd=ROOT,
                           env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        assert "normals" in r.stdout
        outs.append(open(out, "rb").read())
    ref = open(api, "rb").read()
    assert outs[0] == ref and outs[1] == ref
    r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.export_points", "--ckpt_path", slim, "--out",
                        str(tmp_path / "x.ply")], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=600)
    assert r.returncode == 2 and "--root_dir" in r.stderr
