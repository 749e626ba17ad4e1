"""Mesh extraction on the device: ngp_marching_cubes_count / _emit (csrc/mesh.cu) against the numpy restatement
oracle/mcubes_ref.py, ngp_density_lattice (csrc/network.cu) against model.density on materialised points, and
extract_mesh end to end on a trained model."""
import ctypes as C
import math
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import mcubes_ref as R
from test_mesh_cpu import random_field, read_ply, sphere, torus

pytestmark = pytest.mark.gpu


def _iso_field():
    """values on a 1/8 grid (every difference exact in fp32) with a whole plane and isolated points at iso = 0.5"""
    v = (np.random.RandomState(7).randint(0, 9, (17, 19, 23)) / 8).astype(np.float32)
    v[:, 6] = 0.5
    v[3, 4, 5] = v[10, 11, 12] = v[16, 0, 22] = 0.5
    return v, 0.5


def _nan_field():
    v = random_field((21, 18, 25), 3, border=False)
    rng = np.random.RandomState(4)
    v.reshape(-1)[rng.randint(0, v.size, 60)] = np.nan
    return v, 0.5


def _multi_slab():
    from ngp_pl_b200 import _lib
    shape = (4, 800, 700)
    per = max(1, _lib.NGP_MC_SLAB_POINTS // (shape[1] * shape[2]))
    assert math.ceil((shape[0] - 1) / per) >= 3  # cell planes in slabs of `per`: at least three slabs
    return random_field(shape, 5, border=False), 0.5


def _multi_plane_slabs():
    """slabs of several cell planes and a shorter last one: 11 cell planes of 512 x 512 points -> 4 + 4 + 3"""
    from ngp_pl_b200 import _lib
    shape = (12, 512, 512)
    per = max(1, _lib.NGP_MC_SLAB_POINTS // (shape[1] * shape[2]))
    assert per == 4 and [min(per, shape[0] - 1 - i0) for i0 in range(0, shape[0] - 1, per)] == [4, 4, 3]
    v = random_field(shape, 6, border=False)
    v[[4, 8], ::3] = 0.5  # iso values on the planes where two slabs meet
    return v, 0.5


CASES = {
    "rand_2x2x2": lambda: (random_field((2, 2, 2), 0, border=False), 0.5),
    "rand_3x5x7": lambda: (random_field((3, 5, 7), 1, border=False), 0.5),
    "rand_64x48x33": lambda: (random_field((64, 48, 33), 2, border=False), 0.5),
    "rand_200x31x17": lambda: (random_field((200, 31, 17), 3), 0.5),
    "sphere": lambda: (sphere(32, 10.0), 0.0),
    "torus": lambda: (torus(), 0.0),
    "iso_planes_points": _iso_field,
    "nan": _nan_field,
    "multi_slab": _multi_slab,
    "multi_plane_slabs": _multi_plane_slabs,
}


def _same_bits(a, b):
    """bitwise equal, any NaN matching any NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


def _device_mesh(vol, iso, lo=None, step=None):
    from ngp_pl_b200 import mesh
    v, t, n = mesh.marching_cubes(torch.as_tensor(vol).cuda(), iso, lo, step, normals=True)
    return v.cpu().numpy(), t.cpu().numpy(), n.cpu().numpy()


@pytest.mark.parametrize("name", list(CASES))
def test_marching_cubes_matches_oracle(name):
    vol, iso = CASES[name]()
    V, F, N = _device_mesh(vol, iso)
    Vo, Fo, No = R.marching_cubes(vol, iso, normals=True)
    assert V.shape == Vo.shape and F.shape == Fo.shape
    assert _same_bits(V, Vo)
    assert np.array_equal(F, Fo)
    assert np.abs(N - No).max(initial=0.0) <= 1e-5
    assert len(F) > 0


def test_world_space_lattice_matches_oracle():
    vol = random_field((30, 22, 41), 9, border=False)
    lo, step = np.float32([-0.7, 0.25, 3.0]), np.float32([0.013, 0.5, 1.0 / 7])
    V, F, N = _device_mesh(vol, 0.5, lo, step)
    Vo, Fo, No = R.marching_cubes(vol, 0.5, lo, step, normals=True)
    assert _same_bits(V, Vo) and np.array_equal(F, Fo)
    assert np.abs(N - No).max() <= 1e-5


def test_two_calls_bitwise_equal_and_short_capacity_is_refused():
    from ngp_pl_b200 import _lib, mesh
    vol = torch.as_tensor(random_field((64, 48, 33), 11, border=False)).cuda()
    a = mesh.marching_cubes(vol, 0.5, normals=True)
    b = mesh.marching_cubes(vol, 0.5, normals=True)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y)
    L = _lib.lib()
    lat = mesh.lattice(tuple(vol.shape), 0.0, 0.0)
    for k in range(3):
        lat.step[k] = 1.0
    ws_bytes = L.ngp_marching_cubes_workspace(C.byref(lat))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert L.ngp_marching_cubes_count(vol.data_ptr(), C.byref(lat), 0.5, counts.data_ptr(), ws.data_ptr(), ws_bytes, st) == 0
    nv, nt = counts.tolist()
    assert (nv, nt) == (a[0].shape[0], a[1].shape[0])
    sentinel = -12345
    for short_v, short_t in ((1, 0), (0, 1)):
        verts = torch.full((nv + 1, 3), float(sentinel), device="cuda")
        tris = torch.full((nt + 1, 3), sentinel, dtype=torch.int64, device="cuda")
        rc = L.ngp_marching_cubes_emit(vol.data_ptr(), C.byref(lat), 0.5, verts.data_ptr(), None, tris.data_ptr(),
                                       nv - short_v, nt - short_t, ws.data_ptr(), ws_bytes, st)
        assert rc == -22
        torch.cuda.synchronize()
        assert (verts == sentinel).all() and (tris == sentinel).all()  # nothing written, let alone past the capacity
    verts = torch.empty(nv, 3, device="cuda")
    tris = torch.empty(nt, 3, dtype=torch.int64, device="cuda")
    assert L.ngp_marching_cubes_emit(vol.data_ptr(), C.byref(lat), 0.5, verts.data_ptr(), None, tris.data_ptr(), nv, nt,
                                     ws.data_ptr(), ws_bytes, st) == 0
    assert torch.equal(verts.view(torch.int32), a[0].view(torch.int32)) and torch.equal(tris, a[1])
    # bad arguments
    assert L.ngp_marching_cubes_emit(vol.data_ptr(), C.byref(lat), 0.5, verts.data_ptr(), None, tris.data_ptr(), nv, nt,
                                     ws.data_ptr(), ws_bytes - 1, st) == -22
    assert L.ngp_marching_cubes_emit(vol.data_ptr(), C.byref(lat), 0.5, None, None, tris.data_ptr(), nv, nt,
                                     ws.data_ptr(), ws_bytes, st) == -22
    assert L.ngp_marching_cubes_count(None, C.byref(lat), 0.5, counts.data_ptr(), ws.data_ptr(), ws_bytes, st) == -22
    lat.n[1] = 1
    assert L.ngp_marching_cubes_workspace(C.byref(lat)) == 0
    assert L.ngp_marching_cubes_count(vol.data_ptr(), C.byref(lat), 0.5, counts.data_ptr(), ws.data_ptr(), ws_bytes, st) == -22


def test_workspace_grows_with_a_slab_not_the_volume():
    from ngp_pl_b200 import mesh, _lib
    L = _lib.lib()
    ws512 = L.ngp_marching_cubes_workspace(C.byref(mesh.lattice(512, 0.0, 1.0)))
    assert 0 < ws512 < 0.1 * 512 ** 3 * 4
    ws1024 = L.ngp_marching_cubes_workspace(C.byref(mesh.lattice(1024, 0.0, 1.0)))
    assert 0 < ws1024 < 64 << 20


# ---- density on a lattice ----------------------------------------------------------------------------------------------
def _random_model(scale, seed):
    from ngp_pl_b200.models.networks import NGP
    model = NGP(scale).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        p = model.xyz_encoder.params
        p[:3072] = ((torch.rand(3072, generator=g) * 2 - 1) * 0.4).cuda()  # the density MLP
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * 0.5).cuda()
    return model


def _materialised(model, res, lo, hi):
    """model.density on the lattice points built in torch with the documented fp32 formula"""
    from ngp_pl_b200 import mesh
    lat = mesh.lattice(res, lo, hi)
    axes = [torch.tensor(lat.lo[a], dtype=torch.float32, device="cuda") +
            torch.arange(lat.n[a], device="cuda").float() * torch.tensor(lat.step[a], dtype=torch.float32, device="cuda")
            for a in range(3)]
    x = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    return model.density(x).reshape(lat.n[0], lat.n[1], lat.n[2])


@pytest.mark.parametrize("scale,res,bounds", [
    (0.5, 64, None),
    (0.5, (37, 64, 129), None),
    (0.5, (50, 41, 33), ((-0.9, -0.6, -0.5), (0.7, 1.1, 0.5))),  # reaching outside the model's box
    (16.0, 96, None),
    (16.0, (70, 33, 51), ((-20.0, -3.0, -1.0), (2.0, 18.0, 1.0))),
])
def test_density_volume_bitwise_equals_model_density(scale, res, bounds):
    from ngp_pl_b200 import mesh
    model = _random_model(scale, 3)
    sig = mesh.density_volume(model, res, bounds)
    lo, hi = bounds if bounds is not None else (model._xyz_min_host, model._xyz_max_host)
    ref = _materialised(model, res, lo, hi)
    assert sig.shape == ref.shape and sig.is_cuda and sig.dtype == torch.float32
    assert torch.equal(sig.view(torch.int32), ref.view(torch.int32))
    assert sig.std() > 0


# ---- end to end ----------------------------------------------------------------------------------------------------------
def _box_distances(p, scene):
    """for points (V, 3): whether each lies strictly inside some box of the scene, and its distance to the nearest box
    surface (to a face of the box it is in, or to the nearest box from outside)"""
    lo = torch.as_tensor(scene.box_min, device=p.device)[None]
    hi = torch.as_tensor(scene.box_max, device=p.device)[None]
    q = p[:, None]
    inb = ((q > lo) & (q < hi)).all(-1)
    out = torch.clamp(torch.maximum(lo - q, q - hi), min=0).norm(dim=-1)
    depth = torch.minimum(q - lo, hi - q).min(-1)[0]
    return inb.any(-1), torch.where(inb, depth, out).min(-1)[0]


def test_extract_mesh_of_a_trained_lego():
    """Train on the synthetic Lego scene and extract a 128^3 mesh at sigma 20: non-empty, oriented and closed except on
    the lattice boundary, vertices exactly where the lattice puts them in world space, on the scene's box surfaces as
    seen from outside, colours from the fused forward, and a write_ply round trip.

    The cameras cover the whole sphere: with the bank's default upper hemisphere nothing observes the region under the
    base plate, and 21 % of the vertices are floaters there. Where the vertices lie (H100 80GB HBM3, 2000 steps, ~117k
    vertices): 97.7 % of those outside every box are within 2 lattice cells of a box surface, and 0.5 % of all vertices
    are outside every box and farther than 2 cells. Over all vertices the fraction within 2 cells is only 73.7 %, and it
    does not rise from 2000 to 10000 steps: 26 % of the vertices bound cavities deeper than 2 cells inside the solid
    boxes, where no ray reaches and 40 % of the lattice points deeper than 2 cells have sigma <= 20. Marching cubes
    extracts that field faithfully (bitwise against the oracle above); the cavities belong to the trained model. So the
    geometric bounds asserted are on the surface seen from outside: >= 90 % of the vertices outside every box within 2
    cells, and at most 2 % of all vertices outside every box and farther than 2 cells."""
    from ngp_pl_b200 import mesh, synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=100, K=K, device="cuda")
    bank.poses = torch.as_tensor(synth.camera_poses(100, radius=1.5, seed=0, upper_only=False), device="cuda")
    for i in range(100):
        bank.rgb[i] = (synth.trace(scene, *synth.get_rays(bank.directions, bank.poses[i])) * 255).round().to(torch.uint8)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(2000):
        tr.train_step()
    torch.cuda.synchronize()
    assert tr.stats()["psnr"] > 30
    del tr

    res = 128
    m = mesh.extract_mesh(model, res, colors=True)
    V, F = m["vertices"], m["triangles"]
    assert V.shape[0] > 1000 and F.shape[0] > 1000
    # same topology as the index-space mesh of the same volume; open only on the lattice boundary
    Vi, Fi = mesh.marching_cubes(mesh.density_volume(model, res), 20.0)
    assert torch.equal(Fi, F)
    Vi, Fi = Vi.cpu().numpy(), Fi.cpu().numpy()
    bad = R.unpaired_edges(Fi)
    a, b = Vi[bad[:, 0]], Vi[bad[:, 1]]
    assert (((a == 0) & (b == 0)) | ((a == res - 1) & (b == res - 1))).any(1).all()
    # world space: vertex = lo + q * step in fp32 (multiply, then add), q the index-space vertex
    lat = mesh.lattice(res, model._xyz_min_host, model._xyz_max_host)
    lo32, step32 = np.float32(list(lat.lo)), np.float32(list(lat.step))
    assert np.array_equal(V.cpu().numpy().view(np.uint32), (lo32 + Vi * step32).astype(np.float32).view(np.uint32))
    cell = 1.0 / (res - 1)
    inside, dist = _box_distances(V, scene)
    near = dist <= 2 * cell
    frac_outside = float(near[~inside].float().mean())
    floaters = float((~inside & ~near).float().mean())
    print("vertices %d: within 2 cells of a box surface %.4f overall, %.4f of those outside every box; outside and farther "
          "%.4f, inside and deeper %.4f" % (V.shape[0], float(near.float().mean()), frac_outside, floaters,
                                            float((inside & ~near).float().mean())))
    assert frac_outside >= 0.9
    assert floaters <= 0.02
    # colours: the fused forward looking at the surface head-on
    assert m["colors"].dtype == torch.uint8 and m["colors"].shape == V.shape
    d = -m["normals"]
    d[(m["normals"] == 0).all(1)] = torch.tensor([0.0, 0.0, 1.0], device="cuda")  # extract_mesh's view of a flat vertex
    with torch.no_grad():
        _, c = model(V, d)
    assert torch.equal(m["colors"], (c.float() * 255).round().clamp(0, 255).to(torch.uint8))
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "lego.ply")
        mesh.write_ply(p, **m)
        r = read_ply(p)
        v = r["vertex"]
        assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), V.cpu().numpy())
        assert np.array_equal(np.stack([v["nx"], v["ny"], v["nz"]], 1), m["normals"].cpu().numpy())
        assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), m["colors"].cpu().numpy())
        assert np.array_equal(r["face"]["v"], F.cpu().numpy())
