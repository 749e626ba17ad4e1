"""The depth fusion on an H100 (ngp_pl_b200.fusion, csrc/fusion.cu and the TSDF marching cubes of csrc/mesh.cu) against
its numpy restatement (oracle/tsdf_ref.py): the integration bit for bit on random views, grouping and determinism; the
masked marching cubes bit for bit, and as the dense marching cubes where every point is observed; analytic geometry
(a union of boxes, a sphere); a trained Lego; and the CLI's file."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mcubes_ref as R
from oracle import tsdf_ref as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _np_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.int32), np.asarray(b, np.float32).view(np.int32)
    return a.shape == b.shape and np.array_equal(a, b)


def _K(W, H, f):
    return np.float32([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])


def _look_at(pos, target=(0.0, 0.0, 0.0)):
    fwd = np.asarray(target, np.float64) - np.asarray(pos, np.float64)
    fwd /= np.linalg.norm(fwd)
    up = np.array([0, 0, 1.0]) if abs(fwd[2]) < 0.99 else np.array([0, 1.0, 0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    return np.stack([right, down, fwd, np.asarray(pos, np.float64)], 1).astype(np.float32)


def _random_views():
    """12 views of 64x48 around a 48x40x56 lattice: random depth, opacity partly below min_opacity (and some depths
    that overflow t), one camera inside the lattice (points behind it), two grazing views along a lattice plane"""
    from ngp_pl_b200 import synth
    rng = np.random.RandomState(5)
    W, H = 64, 48
    K = _K(W, H, 52.0)
    poses = list(synth.camera_poses(9, radius=1.4, seed=4, upper_only=False))
    poses.append(_look_at([0.05, -0.1, 0.02], [0.6, 0.3, 0.1]))    # inside: half the lattice is behind it
    poses.append(_look_at([1.6, 0.0, 0.0005], [0.0, 0.0, 0.0005]))  # grazing: the optical axis in a lattice plane
    poses.append(_look_at([0.0, -1.5, 0.3], [0.0, 0.0, 0.3]))
    poses = np.stack(poses).astype(np.float32)
    V = len(poses)
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    depth = np.empty((V, H * W), np.float32)
    for v in range(V):
        base = np.linalg.norm(poses[v, :, 3]) if v != 9 else 0.45
        depth[v] = (base + 0.15 * np.sin(xx / 5.0 + v) * np.cos(yy / 7.0 - v) + rng.uniform(-0.02, 0.02, (H, W))).ravel()
    op = rng.uniform(0.2, 1.0, (V, H * W)).astype(np.float32)
    op[rng.rand(V, H * W) < 0.1] = 0.0
    depth *= op
    depth[rng.rand(V, H * W) < 0.01] = 3e38  # t = depth / opacity overflows: not finite, skipped
    rgb = (rng.rand(V, H * W, 3) * op[..., None] * 1.2).astype(np.float32)
    n, lo, hi = (48, 40, 56), np.float32([-0.6, -0.5, -0.7]), np.float32([0.6, 0.5, 0.7])
    return dict(W=W, H=H, K=K, poses=poses, depth=depth, op=op, rgb=rgb, n=n, lo=lo, hi=hi)


def _dev(s):
    return (torch.as_tensor(s["depth"]).cuda(), torch.as_tensor(s["op"]).cuda(), torch.as_tensor(s["rgb"]).cuda())


def _oracle_state(s, vol, views=None):
    from ngp_pl_b200 import datasets
    lat = vol["lattice"]
    x = T.lattice_points(tuple(lat.n), list(lat.lo), list(lat.step))
    st = T.new_state(len(x))
    views = range(len(s["poses"])) if views is None else views
    dirs = datasets.ray_directions(s["W"], s["H"], s["K"]).numpy()
    for v in views:
        T.integrate(st, x, vol["trunc"], s["poses"][v:v + 1], s["K"], s["W"], s["H"], dirs, s["depth"][v:v + 1],
                    s["op"][v:v + 1], s["rgb"][v:v + 1], 0.5)
    return st


@pytest.fixture(scope="module")
def random_volume():
    from ngp_pl_b200 import fusion
    s = _random_views()
    vol = fusion.tsdf_volume(s["n"], (s["lo"], s["hi"]), trunc=0.12)
    d, o, c = _dev(s)
    fusion.integrate(vol, torch.as_tensor(s["poses"]), s["K"], (s["W"], s["H"]), d, o, c, 0.5)
    torch.cuda.synchronize()
    return s, vol


def test_integration_bitwise_grouping_and_determinism(random_volume):
    from ngp_pl_b200 import fusion
    s, vol = random_volume
    st = _oracle_state(s, vol)
    got = {k: vol[k].cpu().numpy().reshape(st[k].shape) for k in ("tsdf", "weight", "color", "color_weight")}
    W = st["weight"]
    assert (W > 0).mean() > 0.2 and (W == 0).mean() > 0.05 and W.max() >= 6
    assert (st["color_weight"] < W).any()
    for k in got:
        assert _np_equal(got[k], st[k]), k
    # one view at a time, and a second call: bitwise the same
    d, o, c = _dev(s)
    one = fusion.tsdf_volume(s["n"], (s["lo"], s["hi"]), trunc=0.12)
    for v in range(len(s["poses"])):
        fusion.integrate(one, torch.as_tensor(s["poses"][v:v + 1]), s["K"], (s["W"], s["H"]), d[v:v + 1], o[v:v + 1],
                         c[v:v + 1], 0.5)
    two = fusion.tsdf_volume(s["n"], (s["lo"], s["hi"]), trunc=0.12)
    fusion.integrate(two, torch.as_tensor(s["poses"]), s["K"], (s["W"], s["H"]), d, o, c, 0.5)
    for k in ("tsdf", "weight", "color", "color_weight"):
        assert _equal(one[k], vol[k]) and _equal(two[k], vol[k]), k


def test_more_views_than_a_group_bitwise():
    """views beyond NGP_TSDF_GROUP go to a second launch; the result is the oracle's all the same"""
    from ngp_pl_b200 import _lib, fusion
    s = _random_views()
    reps = _lib.NGP_TSDF_GROUP // len(s["poses"]) + 2
    for k in ("poses", "depth", "op", "rgb"):
        s[k] = np.concatenate([s[k]] * reps)
    s["n"] = (16, 12, 20)
    vol = fusion.tsdf_volume(s["n"], (s["lo"], s["hi"]), trunc=0.12)
    d, o, c = _dev(s)
    fusion.integrate(vol, torch.as_tensor(s["poses"]), s["K"], (s["W"], s["H"]), d, o, c, 0.5)
    st = _oracle_state(s, vol)
    assert len(s["poses"]) > _lib.NGP_TSDF_GROUP and st["weight"].max() > len(s["poses"]) // reps
    for k in ("tsdf", "weight", "color", "color_weight"):
        assert _np_equal(vol[k].cpu().numpy().reshape(st[k].shape), st[k]), k


def test_masked_marching_cubes_bitwise(random_volume):
    from ngp_pl_b200 import _lib, fusion, mesh
    s, vol = random_volume
    m = fusion.tsdf_mesh(vol, normals=True, colors=True)
    lat = vol["lattice"]
    F, Wt = vol["tsdf"].cpu().numpy(), vol["weight"].cpu().numpy()
    v, t, nr, col = T.masked_marching_cubes(F, Wt, list(lat.lo), list(lat.step), normals=True,
                                           color=vol["color"].cpu().numpy(), color_weight=vol["color_weight"].cpu().numpy())
    assert len(t) > 1000
    assert _np_equal(m["vertices"].cpu().numpy(), v) and np.array_equal(m["triangles"].cpu().numpy(), t)
    assert np.array_equal(m["colors"].cpu().numpy(), col)
    assert np.abs(m["normals"].cpu().numpy().astype(np.float64) - nr).max() < 1e-5
    again = fusion.tsdf_mesh(vol)
    for k in m:
        assert _equal(m[k], again[k]), k
    # observed everywhere: the dense marching cubes of -F at 0
    full = dict(vol, weight=vol["weight"].clamp(min=1))
    fm = fusion.tsdf_mesh(full, normals=True, colors=False)
    dv, dt, dn = mesh.marching_cubes(-vol["tsdf"], 0.0, list(lat.lo), list(lat.step), normals=True)
    assert fm["triangles"].shape[0] > m["triangles"].shape[0]
    assert _equal(fm["vertices"], dv) and _equal(fm["triangles"], dt) and _equal(fm["normals"], dn)
    assert fm["colors"] is None
    # a short capacity is refused as the dense path refuses it, with nothing written
    L = _lib.lib()
    ws_bytes = L.ngp_tsdf_mc_workspace(C.byref(lat))
    ws = torch.empty(ws_bytes, device="cuda", dtype=torch.uint8)
    counts = torch.empty(2, device="cuda", dtype=torch.int64)
    st = torch.cuda.current_stream().cuda_stream
    Fd, Wd = vol["tsdf"], vol["weight"]
    assert L.ngp_tsdf_mc_count(Fd.data_ptr(), Wd.data_ptr(), C.byref(lat), counts.data_ptr(), ws.data_ptr(), ws_bytes, st) == 0
    nv, nt = (int(x) for x in counts.cpu())
    assert (nv, nt) == (len(v), len(t))
    verts = torch.full((nv, 3), 7.0, device="cuda")
    tris = torch.full((nt, 3), -5, device="cuda", dtype=torch.int64)
    for mv, mt in ((nv - 1, nt), (nv, nt - 1)):
        rc = L.ngp_tsdf_mc_emit(Fd.data_ptr(), Wd.data_ptr(), None, None, C.byref(lat), verts.data_ptr(), None, None,
                                tris.data_ptr(), mv, mt, ws.data_ptr(), ws_bytes, st)
        assert rc == -22
    assert (verts == 7.0).all() and (tris == -5).all()


def _trace_depth(scene, o, d):
    """ray parameter of the first box hit along the unnormalised d (inf on a miss), float64"""
    bmin = torch.as_tensor(scene.box_min, device=o.device, dtype=torch.float64)
    bmax = torch.as_tensor(scene.box_max, device=o.device, dtype=torch.float64)
    o, d = o.double()[:, None], d.double()[:, None]
    inv = 1.0 / d
    ta, tb = (bmin - o) * inv, (bmax - o) * inv
    t1 = torch.minimum(ta, tb).max(-1)[0]
    t2 = torch.maximum(ta, tb).min(-1)[0]
    hit = (t1 <= t2) & (t1 > 0)
    return torch.where(hit, t1, torch.full_like(t1, math.inf)).min(-1)[0]


def _exact_maps(hit_t, scene=None, o=None, d=None):
    hit = torch.isfinite(hit_t)
    op = hit.float()
    depth = torch.where(hit, hit_t, torch.zeros_like(hit_t)).float()
    return depth, op


def _segment_distance(p, a, b):
    ab = b - a
    t = ((p - a) @ ab / (ab @ ab)).clamp(0, 1)
    return (p - (a + t[:, None] * ab)).norm(dim=1)


def test_box_union_from_exact_depth():
    """60 views at 200^2 of synth.lego_scene(0), depth traced exactly (opacity 1 on a hit, 0 on a miss), fused on a
    256^3 lattice over [-0.5, 0.5]^3 with tau = 4 steps. Bound on the vertices farther than tau + 2 steps from every
    box edge (so no silhouette or occlusion boundary is within the band around them):
      A point x is projected to the pixel whose centre ray passes nearest; in normalised image coordinates that ray is
      off by at most delta = (sqrt(2) / 2) / f, so at camera depth z it passes at most z delta from x laterally. On a
      face with unit normal n seen at angle theta (cos theta = |n . r| for the unit ray r), the plane's camera depth
      over that offset changes by at most z delta |n_xy| / (cos theta |dir|), and the measured sdf (t - zc) |dir|
      is off by e <= z delta / cos theta from the distance along x's own ray, s / cos theta for x at signed distance
      s from the face. So for s > z_max delta every view's sdf is positive and for s < -z_max delta negative: the
      mean F has the sign of s outside |s| <= B = z_max delta, whatever the views' angles and weights. A crossed
      lattice edge has ends of opposite F, hence ends with s > -B and s < B; s is affine along the edge and changes
      by at most one step over it, so the vertex lies within B + step of the face. z_max = camera radius + the
      largest norm of a box corner. Plus 1e-5 for fp32 rounding."""
    from ngp_pl_b200 import fusion, synth
    scene = synth.lego_scene(0)
    f = 1111.11 / 4
    Kd = synth.intrinsics(W=200, H=200, fx=f)
    K = _K(200, 200, f)
    poses = torch.as_tensor(synth.camera_poses(60, radius=1.5, seed=0, upper_only=False))
    dirs = synth.ray_directions(Kd).cuda()
    ds, os_, cs = [], [], []
    for i in range(60):
        o, d = synth.get_rays(dirs, poses[i].cuda())
        depth, op = _exact_maps(_trace_depth(scene, o, d))
        ds.append(depth)
        os_.append(op)
        cs.append(synth.trace(scene, o, d) * op[:, None])
    res = 256
    vol = fusion.tsdf_volume(res, ([-0.5] * 3, [0.5] * 3))
    fusion.integrate(vol, poses, K, (200, 200), torch.stack(ds), torch.stack(os_), torch.stack(cs), 0.5)
    m = fusion.tsdf_mesh(vol)
    V = m["vertices"].double()
    assert V.shape[0] > 10000
    step = max(vol["lattice"].step)
    tau = vol["trunc"]
    lo, hi = np.asarray(scene.box_min, np.float64), np.asarray(scene.box_max, np.float64)
    z_max = 1.5 + np.linalg.norm(np.maximum(np.abs(lo), np.abs(hi)), axis=1).max()
    bound = z_max * (math.sqrt(2) / 2) / f + step + 1e-5
    edge = torch.full((V.shape[0],), math.inf, device="cuda", dtype=torch.float64)
    for b in range(len(lo)):
        for a in range(3):
            o1, o2 = [x for x in range(3) if x != a]
            for u in (lo[b, o1], hi[b, o1]):
                for w in (lo[b, o2], hi[b, o2]):
                    q0, q1 = np.empty(3), np.empty(3)
                    q0[a], q1[a] = lo[b, a], hi[b, a]
                    q0[o1] = q1[o1] = u
                    q0[o2] = q1[o2] = w
                    edge = torch.minimum(edge, _segment_distance(V, torch.as_tensor(q0, device="cuda"),
                                                                 torch.as_tensor(q1, device="cuda")))
    far = edge > tau + 2 * step
    inb, dist = _box_distances(V, scene)
    assert far.float().mean() > 0.5
    print("box union: %d vertices, %d far from edges; bound %.5f; max distance %.5f, 99.9 %% %.5f"
          % (V.shape[0], int(far.sum()), bound, float(dist[far].max()), float(dist[far].quantile(0.999))))
    assert float(dist[far].max()) <= bound
    assert R.unpaired_edges(m["triangles"].cpu().numpy()).shape[0] < 0.01 * m["triangles"].shape[0]


def _box_distances(p, scene):
    """whether each point lies strictly inside some box, and its distance to the nearest box surface (to a face of a
    box it is in, or to the nearest box from outside) -- the rule of test_mesh_gpu's check"""
    lo = torch.as_tensor(scene.box_min, device=p.device, dtype=p.dtype)[None]
    hi = torch.as_tensor(scene.box_max, device=p.device, dtype=p.dtype)[None]
    q = p[:, None]
    inb = ((q > lo) & (q < hi)).all(-1)
    out = torch.clamp(torch.maximum(lo - q, q - hi), min=0).norm(dim=-1)
    depth = torch.minimum(q - lo, hi - q).min(-1)[0]
    return inb.any(-1), torch.where(inb, depth, out).min(-1)[0]


def test_sphere_is_closed():
    """a sphere of radius 0.3 seen by 100 cameras at distance 1.5 from every side: every surface point is seen by a
    camera within 45 degrees of its normal (checked below), so with tau = 4 steps every lattice point within sqrt(3)
    steps of the surface is observed (sdf >= -sqrt(3) step / cos 45 > -tau), every cell the surface passes through
    emits, and every mesh edge is shared by exactly two triangles"""
    from ngp_pl_b200 import fusion, synth
    r, f, Wp = 0.3, 160.0, 128
    K = _K(Wp, Wp, f)
    Kd = synth.intrinsics(W=Wp, H=Wp, fx=f)
    poses = torch.as_tensor(synth.camera_poses(100, radius=1.5, seed=11, upper_only=False))
    cam = poses[:, :, 3].numpy().astype(np.float64)
    # coverage: every direction on the sphere within 45 degrees of some camera as seen from the surface point
    g = np.random.RandomState(0).normal(size=(20000, 3))
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    to_cam = cam[None] - r * g[:, None]
    cosang = (to_cam * g[:, None]).sum(-1) / np.linalg.norm(to_cam, axis=-1)
    assert cosang.max(1).min() > math.cos(math.radians(45))
    dirs = synth.ray_directions(Kd).cuda()
    ds, os_ = [], []
    for i in range(100):
        o, d = synth.get_rays(dirs, poses[i].cuda())
        o, d = o.double(), d.double()
        b = (o * d).sum(1)
        a = (d * d).sum(1)
        disc = b * b - a * ((o * o).sum(1) - r * r)
        t = (-b - disc.clamp(min=0).sqrt()) / a
        t = torch.where(disc > 0, t, torch.full_like(t, math.inf))
        depth, op = _exact_maps(t)
        ds.append(depth)
        os_.append(op)
    depth, op = torch.stack(ds), torch.stack(os_)
    rgb = op[..., None].expand(-1, -1, 3).contiguous() * 0.5
    vol = fusion.tsdf_volume(128, ([-0.5] * 3, [0.5] * 3))
    fusion.integrate(vol, poses, K, (Wp, Wp), depth, op, rgb, 0.5)
    m = fusion.tsdf_mesh(vol)
    t = m["triangles"].cpu().numpy()
    assert len(t) > 5000
    assert R.unpaired_edges(t).shape[0] == 0
    rad = m["vertices"].double().norm(dim=1)
    assert float((rad - r).abs().max()) < 2 * max(vol["lattice"].step)
    assert (m["colors"].int() - 128).abs().max() <= 1


# ---- trained model -------------------------------------------------------------------------------------------------
def _lego_cameras():
    from ngp_pl_b200 import synth
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    return torch.as_tensor(synth.camera_poses(60, radius=1.5, seed=0, upper_only=False)), synth.ray_directions(K)


@pytest.fixture(scope="module")
def lego():
    """the synthetic Lego trained for 300 steps, as test_points_gpu's fixture trains it, and its cameras"""
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
    return scene, model, poses, dirs


def _render_chunk(model, poses, dirs, k0, B, N):
    """rays k0 .. k0 + B of the view-major pixel list through ngp_gen_rays, spare rays as render_views sets them, and
    one ngp_render_infer_frame of B rays with the export's cfg"""
    from ngp_pl_b200 import _lib, fusion
    from ngp_pl_b200.models.networks import _net_struct
    L = _lib.lib()
    m = min(B, N - k0)
    n_pix = dirs.shape[0]
    k = torch.arange(k0, k0 + m, device="cuda")
    img, pix = k // n_pix, k % n_pix
    o, d = torch.empty(B, 3, device="cuda"), torch.empty(B, 3, device="cuda")
    P_, D_ = poses.cuda().contiguous(), dirs.cuda().contiguous()
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.ngp_gen_rays(img.data_ptr(), pix.data_ptr(), P_.data_ptr(), D_.data_ptr(), None, n_pix, m, o.data_ptr(),
                              d.data_ptr(), None, st), "gen_rays")
    cfg, c, h = fusion._infer_cfg(model, B, 0.0)
    if m < B:
        o[m:] = torch.tensor([c[0], c[1], c[2] + 2 * h[2] + 1.0], device="cuda")
        d[m:] = torch.tensor([0.0, 0.0, 1.0], device="cuda")
    ws = torch.empty(L.ngp_render_infer_workspace(B, cfg.max_round_samples), device="cuda", dtype=torch.uint8)
    op, dep, rgb = torch.empty(B, device="cuda"), torch.empty(B, device="cuda"), torch.empty(B, 3, device="cuda")
    total = torch.zeros(1, device="cuda", dtype=torch.int64)
    net, keep = _net_struct(model)
    _lib.check(L.ngp_render_infer_frame(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                        op.data_ptr(), dep.data_ptr(), rgb.data_ptr(), total.data_ptr(), ws.data_ptr(),
                                        ws.numel(), st), "render_infer_frame")
    return op[:m], dep[:m], rgb[:m]


def test_trained_lego(lego):
    from ngp_pl_b200 import datasets, fusion, mesh
    scene, model, poses, dirs = lego
    assert float(model.scale) <= 0.5  # exp_step_factor 0 by the export's rule, as _render_chunk renders
    B = 1 << 16
    maps = fusion.render_views(model, poses, dirs, chunk=B)
    N = poses.shape[0] * dirs.shape[0]
    flat = {k: maps[k].reshape(N, -1).squeeze(1) for k in maps}
    for k0 in (0, 9 * B, (N - 1) // B * B):
        op, dep, rgb = _render_chunk(model, poses, dirs, k0, B, N)
        m = op.shape[0]
        assert _equal(flat["opacity"][k0:k0 + m], op) and _equal(flat["depth"][k0:k0 + m], dep)
        assert _equal(flat["rgb"][k0:k0 + m], rgb)
    assert (flat["opacity"] > 0.5).float().mean() > 0.05
    res = 128
    K = _K(200, 200, 1111.11 / 4)
    vol = fusion.tsdf_volume(res, (model._xyz_min_host, model._xyz_max_host))
    fusion.integrate(vol, poses, K, (200, 200), maps["depth"], maps["opacity"], maps["rgb"], 0.5)
    # the integration bit for bit on the trained maps
    s = dict(W=200, H=200, K=K, poses=poses.numpy(), depth=maps["depth"].cpu().numpy(), op=maps["opacity"].cpu().numpy(),
             rgb=maps["rgb"].cpu().numpy())
    st = _oracle_state(s, vol)
    for k in ("tsdf", "weight", "color", "color_weight"):
        assert _np_equal(vol[k].cpu().numpy().reshape(st[k].shape), st[k]), k
    m = fusion.tsdf_mesh(vol)
    lat = vol["lattice"]
    v, t, nr, col = T.masked_marching_cubes(st["tsdf"].reshape(lat.n[0], lat.n[1], lat.n[2]),
                                           st["weight"].reshape(lat.n[0], lat.n[1], lat.n[2]), list(lat.lo),
                                           list(lat.step), normals=True, color=st["color"],
                                           color_weight=st["color_weight"].reshape(lat.n[0], lat.n[1], lat.n[2]))
    assert len(t) > 10000
    assert _np_equal(m["vertices"].cpu().numpy(), v) and np.array_equal(m["triangles"].cpu().numpy(), t)
    assert np.array_equal(m["colors"].cpu().numpy(), col)
    assert np.abs(m["normals"].cpu().numpy().astype(np.float64) - nr).max() < 1e-5
    # the whole pipeline gives the same mesh
    e = fusion.extract_mesh_tsdf(model, poses, K, (200, 200), res, chunk=B)
    for k in m:
        assert _equal(m[k], e[k]), k
    # cavities: the fraction of vertices inside the boxes and deeper than 2 cells, against the σ mesh
    sp = mesh.extract_mesh_sparse(model, res, normals=False)
    cell = 1.0 / (res - 1)
    frac = []
    for V in (m["vertices"], sp["vertices"]):
        inb, dist = _box_distances(V, scene)
        frac.append(float((inb & (dist > 2 * cell)).float().mean()))
    print("inside and deeper than 2 cells: TSDF %.4f (%d vertices), sigma %.4f (%d vertices)"
          % (frac[0], m["vertices"].shape[0], frac[1], sp["vertices"].shape[0]))
    assert frac[0] < frac[1]


def test_cpu_tensors_raise(lego, random_volume):
    from ngp_pl_b200 import fusion
    s, vol = random_volume
    d, o, c = _dev(s)
    with pytest.raises(RuntimeError):
        fusion.integrate(vol, s["poses"], s["K"], (s["W"], s["H"]), d.cpu(), o, c, 0.5)
    cpu = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in vol.items()}
    with pytest.raises(RuntimeError):
        fusion.tsdf_mesh(cpu)
    with pytest.raises(RuntimeError):
        fusion.integrate(cpu, s["poses"], s["K"], (s["W"], s["H"]), d, o, c, 0.5)
    with pytest.raises(RuntimeError):
        fusion.tsdf_volume(8, ([0] * 3, [1] * 3), device="cpu")
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(RuntimeError):
            fusion.tsdf_volume(8, ([0] * 3, [1] * 3), trunc=bad)
    for bad in (0.0, 1.5, float("nan")):
        with pytest.raises(RuntimeError):
            fusion.integrate(vol, s["poses"], s["K"], (s["W"], s["H"]), d, o, c, bad)
    with pytest.raises(RuntimeError):
        fusion.integrate(vol, s["poses"], s["K"], (s["W"], s["H"]), d[:, :-1], o, c, 0.5)
    with pytest.raises(RuntimeError):
        fusion.tsdf_volume(4096, ([0] * 3, [1] * 3))  # 1.6 TB of state
    scene, model, poses, dirs = lego
    cpu_model = type(model)(model.scale)
    with pytest.raises(RuntimeError):
        fusion.extract_mesh_tsdf(cpu_model, poses, _K(200, 200, 277.0), (200, 200), 16)


def _write_nerf_scene(root, poses, fx):
    import json
    os.makedirs(root, exist_ok=True)
    frames = []
    for i, c2w in enumerate(poses):
        m = np.eye(4)
        m[:3] = c2w
        m[:3, 1:3] *= -1
        frames.append({"file_path": "./train/r_%d" % i, "transform_matrix": m.tolist()})
    json.dump({"camera_angle_x": 2 * math.atan(400 / fx), "frames": frames},
              open(os.path.join(root, "transforms_train.json"), "w"))


def test_cli_writes_what_the_api_writes(lego, tmp_path):
    from ngp_pl_b200 import datasets, fusion, mesh, train
    scene, model, poses, dirs = lego
    root = str(tmp_path / "scene")
    _write_nerf_scene(root, poses.numpy().astype(np.float64), 1111.11)
    meta = datasets.scene_meta("nerf", root, "train", 0.25)
    P_, D_ = torch.as_tensor(meta.poses), torch.as_tensor(meta.directions)
    ck = str(tmp_path / "full.ckpt")
    torch.save(train.checkpoint(model, D_, P_, 0, 300), ck)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = 96
    m = fusion.extract_mesh_tsdf(model, P_, meta.K, meta.img_wh, res, min_opacity=0.6, trunc=0.05)
    box = (model._xyz_min_host, model._xyz_max_host)
    k = mesh.simplify_mesh(mesh.remove_small_components(m, keep_largest=1), 32, box)
    outs = {}
    for name, ref, extra in (("plain", m, []), ("pieces", k, ["--keep_largest", "1", "--simplify", "32"])):
        api = str(tmp_path / ("api_%s.ply" % name))
        mesh.write_ply(api, **ref)
        out = str(tmp_path / ("cli_%s.ply" % name))
        r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.export_mesh", "--ckpt_path", ck, "--tsdf", "--root_dir", root,
                            "--downsample", "0.25", "--resolution", str(res), "--min_opacity", "0.6", "--tsdf_trunc",
                            "0.05", "--colors", "--out", out] + extra, cwd=ROOT, env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        outs[name] = (open(out, "rb").read(), open(api, "rb").read())
    assert k["triangles"].shape[0] < m["triangles"].shape[0]
    for name, (cli, api) in outs.items():
        assert cli == api, name
