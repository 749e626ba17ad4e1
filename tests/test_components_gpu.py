"""Connected components on the device (csrc/components.cu) against the numpy + scipy restatement
oracle/components_ref.py, bitwise: occupancy labels, sizes, the cleaned bitfield and density_grid; mesh labels and
filtered meshes; and the cleanup end to end on a trained Lego."""
import numpy as np
import pytest
import torch

from oracle import components_ref as R
from test_mesh_cpu import random_field

pytestmark = pytest.mark.gpu

SCALE_FOR = {1: 0.5, 2: 1.0, 3: 2.0, 4: 3.0, 5: 8.0, 6: 16.0}  # scale 3: cascade 3 is 1.5 x cascade 2


class _Grid(torch.nn.Module):
    """the attributes of NGP that the occupancy functions read"""

    def __init__(self, bits, cascades, G, scale, density_grid=None):
        super().__init__()
        self.cascades, self.grid_size, self.scale = cascades, G, scale
        self.register_buffer("density_bitfield", torch.as_tensor(bits).cuda())
        if density_grid is not None:
            self.register_buffer("density_grid", torch.as_tensor(density_grid).cuda())


def _to_morton(occ3d):
    """(C, G, G, G) bool in (x, y, z) order -> (C, G^3) in cell order"""
    G = occ3d.shape[1]
    xyz = R.morton_coords(G)
    return occ3d[:, xyz[:, 0], xyz[:, 1], xyz[:, 2]]


def _blobs(cascades, G, seed, p_float=1e-3):
    """smooth random blobs per cascade (noise at G/8 upsampled, thresholded) plus isolated floaters"""
    rng = np.random.default_rng(seed)
    k = max(1, G // 8)
    coarse = rng.random((cascades, G // k, G // k, G // k)) < 0.3
    occ = coarse.repeat(k, 1).repeat(k, 2).repeat(k, 3)
    occ |= rng.random(occ.shape) < p_float
    return _to_morton(occ)


def _path(G):
    """a serpentine through rows along z at even x and even y (x, y < G / 2), joined at alternating row ends"""
    occ = np.zeros((1, G, G, G), bool)
    h = G // 2
    order = [(x, y) for x in range(0, h, 2) for y in (range(0, h, 2) if (x // 2) % 2 == 0 else range(h - 2, -1, -2))]
    for r, (x, y) in enumerate(order):
        occ[0, x, y, :] = True
        if r + 1 < len(order):
            end = G - 1 if r % 2 == 0 else 0
            nx, ny = order[r + 1]
            occ[0, (x + nx) // 2, (y + ny) // 2, end] = True
    return _to_morton(occ)


def _single_cells(cascades, G):
    occ = np.zeros((cascades, G, G, G), bool)
    for c in range(cascades):
        occ[c, 0, 0, 0] = occ[c, G - 1, G - 1, G - 1] = occ[c, G // 2, 1, G - 3] = True
    return _to_morton(occ)


def _checkerboard(G):
    x, y, z = np.meshgrid(*[np.arange(G)] * 3, indexing="ij")
    return _to_morton(((x + y + z) % 2 == 0)[None]), _to_morton(((x == y) & (y == z))[None] | ((x == G - 1 - y) & (z == 0))[None])


def _joined_by_coarse():
    """two cascade-0 pieces on opposite faces of its box, joined only through a ring of cascade-1 shell cells"""
    G = 16
    occ = np.zeros((2, G, G, G), bool)
    occ[0, 0:2, 6:8, 6:8] = True
    occ[0, G - 2:G, 6:8, 6:8] = True
    occ[1, 3, 7, 7] = True  # cascade 1 (scale 1, 2 x the extent): cells 3 and 12 touch cascade 0's faces
    occ[1, 12, 7, 7] = True
    occ[1, 4:12, 7, 3] = True
    occ[1, 3, 7, 3:8] = True
    occ[1, 12, 7, 3:8] = True
    return _to_morton(occ)


CASES = {
    "empty": lambda: (np.zeros((1, 128 ** 3), bool), 1, 128, 0.5),
    "full": lambda: (np.ones((3, 32 ** 3), bool), 3, 32, 2.0),
    "single_cells": lambda: (_single_cells(3, 16), 3, 16, 2.0),
    "checkerboard": lambda: (_checkerboard(32)[0], 1, 32, 0.5),
    "diagonals": lambda: (_checkerboard(32)[1], 1, 32, 0.5),
    "path": lambda: (_path(256), 1, 256, 0.5),
    "joined_by_coarse": lambda: (_joined_by_coarse(), 2, 16, 1.0),
    "G2": lambda: (np.random.default_rng(5).random((3, 8)) < 0.5, 3, 2, 2.0),
    "G256": lambda: (_blobs(1, 256, 11), 1, 256, 0.5),
    "scale0.7": lambda: (_blobs(2, 64, 12), 2, 64, 0.7),
}
for _c in range(1, 7):
    CASES["G128_c%d" % _c] = (lambda c: lambda: (_blobs(c, 128, c), c, 128, SCALE_FOR[c]))(_c)


def _check_grid(occ, cascades, G, scale, criteria):
    """labels and sizes, then the cleanup under each (keep_largest, min_cells) of criteria, against the oracle"""
    from ngp_pl_b200 import components
    bits = np.packbits(occ.reshape(-1), bitorder="little")
    lab_o, siz_o = R.grid_components(bits, cascades, G, scale)
    g = _Grid(bits, cascades, G, scale)
    lab, siz = components.occupancy_components(g)
    assert np.array_equal(lab.cpu().numpy(), lab_o) and np.array_equal(siz.cpu().numpy(), siz_o)
    lab2, siz2 = components.occupancy_components(g)
    assert torch.equal(lab, lab2) and torch.equal(siz, siz2)
    out = []
    for seed, (keep_largest, min_cells) in enumerate(criteria):
        dg0 = np.random.default_rng(seed).random((cascades, G ** 3)).astype(np.float32)
        keep_o, cnt_o = R.select(lab_o, siz_o, keep_largest, min_cells)
        bits_o, dg_o, n_o = R.grid_clean(bits, dg0, cascades, G, scale, lab_o, keep_o)
        g = _Grid(bits, cascades, G, scale, dg0)
        _, st = components.remove_floaters(g, keep_largest, min_cells, return_stats=True)
        assert np.array_equal(g.density_bitfield.cpu().numpy(), bits_o)
        assert np.array_equal(g.density_grid.cpu().numpy().view(np.uint32), dg_o.view(np.uint32))
        assert (st["components"], st["kept"]) == cnt_o and (st["cleared_cells"], st["cleared_inner"]) == n_o
        out.append((cnt_o, n_o))
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_occupancy_components_and_cleanup_equal_oracle(name):
    occ, cascades, G, scale = CASES[name]()
    (cnt, n), _, _ = _check_grid(occ, cascades, G, scale, [(3, None), (None, 20), (1, 2)])
    print("%s: %d components, cleared %d shell and %d inner cells (keep_largest=3)" % (name, cnt[0], n[0], n[1]))


def test_path_is_one_component():
    from ngp_pl_b200 import components
    occ = _path(256)
    g = _Grid(np.packbits(occ.reshape(-1), bitorder="little"), 1, 256, 0.5)
    lab, siz = components.occupancy_components(g)
    first = int(np.nonzero(occ[0])[0][0])
    assert int(siz[first]) == int(occ.sum()) > 1_000_000 and int((siz > 0).sum()) == 1


def test_occupancy_refusals():
    from ngp_pl_b200 import components
    g = _Grid(np.zeros(128 ** 3 // 8, np.uint8), 1, 128, 0.5)
    for kw in ({}, {"keep_largest": 0}, {"min_cells": -1}, {"keep_largest": 1.5}, {"keep_largest": True}):
        with pytest.raises(RuntimeError):
            components.remove_floaters(g, **kw)
    g.cascades = 2  # bitfield too short for two cascades
    with pytest.raises(RuntimeError):
        components.occupancy_components(g)


# ---- mesh ----------------------------------------------------------------------------------------------------------
def _check_mesh(m, keep_largest=None, min_triangles=None):
    from ngp_pl_b200 import mesh
    V = m["vertices"].shape[0]
    t = m["triangles"].cpu().numpy()
    lab_o, siz_o = R.mesh_components(t, V)
    lab, siz = mesh.mesh_components(m)
    assert np.array_equal(lab.cpu().numpy(), lab_o) and np.array_equal(siz.cpu().numpy(), siz_o)
    lab2, _ = mesh.mesh_components(m)
    assert torch.equal(lab, lab2)
    keep_o, cnt_o = R.select(lab_o, siz_o, keep_largest, min_triangles)
    want = R.mesh_filter(m["vertices"].cpu().numpy(), t, lab_o, keep_o,
                         None if m["normals"] is None else m["normals"].cpu().numpy(),
                         None if m["colors"] is None else m["colors"].cpu().numpy())
    got, st = mesh.remove_small_components(m, keep_largest, min_triangles, return_stats=True)
    assert (st["components"], st["kept"]) == cnt_o
    for k in ("vertices", "triangles", "normals", "colors"):
        if want[k] is None:
            assert got[k] is None
        else:
            assert np.array_equal(got[k].cpu().numpy(), want[k]), k
    return cnt_o


def _soup(V, F, seed, attrs=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = {"vertices": torch.rand(V, 3, generator=g, device="cuda"),
         "triangles": torch.randint(0, V, (F, 3), generator=g, device="cuda", dtype=torch.int64),
         "normals": torch.rand(V, 3, generator=g, device="cuda") if attrs else None,
         "colors": torch.randint(0, 256, (V, 3), generator=g, device="cuda", dtype=torch.uint8) if attrs else None}
    return m


@pytest.mark.parametrize("V,F,seed", [(10, 3, 0), (1000, 400, 1), (100000, 40000, 2), (50000, 200000, 3)])
def test_random_soups_equal_oracle(V, F, seed):
    m = _soup(V, F, seed, attrs=seed % 2 == 0)
    _check_mesh(m, keep_largest=5)
    _check_mesh(m, min_triangles=3)
    _check_mesh(m, keep_largest=2, min_triangles=2)


def _blob_volume(n=96, blobs=60, seed=0):
    rng = np.random.default_rng(seed)
    x = np.arange(n, dtype=np.float32)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    v = np.zeros((n, n, n), np.float32)
    for _ in range(blobs):
        c = rng.uniform(4, n - 4, 3)
        r = rng.uniform(1.0, 6.0)
        v = np.maximum(v, r * r - ((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2))
    return v.astype(np.float32)


def test_marching_cubes_blobs_equal_oracle():
    from ngp_pl_b200 import mesh
    v, t, nrm = mesh.marching_cubes(torch.as_tensor(_blob_volume()).cuda(), 0.0, normals=True)
    m = {"vertices": v, "triangles": t, "normals": nrm, "colors": None}
    cnt = _check_mesh(m, keep_largest=10)
    assert cnt[0] > 20
    _check_mesh(m, min_triangles=200)
    v, t = mesh.marching_cubes(torch.as_tensor(random_field((40, 50, 60), 8)).cuda(), 0.5)
    _check_mesh({"vertices": v, "triangles": t, "normals": None, "colors": None}, min_triangles=10)


def test_twenty_million_triangles_equal_oracle():
    m = _soup(30_000_000, 20_000_000, 4, attrs=False)
    cnt = _check_mesh(m, keep_largest=1000, min_triangles=2)
    print("20 M-triangle soup: %d components, %d kept" % cnt)


def test_nothing_removed_returns_the_input_and_refusals():
    """a mesh whose vertices are all used (marching cubes' are) comes back bitwise when no component is removed"""
    from ngp_pl_b200 import mesh
    v, t, nrm = mesh.marching_cubes(torch.as_tensor(_blob_volume(48, 10, 1)).cuda(), 0.0, normals=True)
    m = {"vertices": v, "triangles": t, "normals": nrm, "colors": None}
    out = mesh.remove_small_components(m, min_triangles=1)
    for k in ("vertices", "triangles", "normals"):
        assert torch.equal(out[k], m[k]), k
    assert out["colors"] is None
    for kw in ({}, {"keep_largest": 0}, {"min_triangles": 0}):
        with pytest.raises(RuntimeError):
            mesh.remove_small_components(m, **kw)
    bad = dict(m, triangles=m["triangles"].clone())
    bad["triangles"][7, 1] = v.shape[0]
    with pytest.raises(RuntimeError, match="outside"):
        mesh.mesh_components(bad)
    empty = {"vertices": torch.zeros(0, 3, device="cuda"), "triangles": torch.zeros(0, 3, device="cuda", dtype=torch.int64),
             "normals": None, "colors": None}
    out = mesh.remove_small_components(empty, keep_largest=1)
    assert out["vertices"].shape == (0, 3) and out["triangles"].shape == (0, 3)


# ---- end to end on the Lego of test_mesh_gpu -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lego():
    """the synthetic Lego of test_mesh_gpu's end-to-end test (cameras over the whole sphere, 2000 steps)"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
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
    for _ in range(2000):
        tr.train_step()
    torch.cuda.synchronize()
    del tr
    return scene, model


def _fractions(m, scene, res):
    from test_mesh_gpu import _box_distances
    inside, dist = _box_distances(m["vertices"], scene)
    near = dist <= 2.0 / (res - 1)
    return float((~inside & ~near).float().mean()), float((inside & ~near).float().mean())


def test_trained_bitfield_equals_oracle(lego):
    _, model = lego
    occ = R.unpack(model.density_bitfield.cpu().numpy(), model.cascades, model.grid_size)
    (cnt, n), _ = _check_grid(occ, model.cascades, model.grid_size, float(model.scale), [(1, None), (None, 50)])
    print("trained Lego bitfield: %d components; keep_largest=1 clears %d cells" % (cnt[0], n[0] + n[1]))


def test_mesh_cleanup_end_to_end(lego):
    from ngp_pl_b200 import components, mesh
    scene, model = lego
    res = 128
    m = mesh.extract_mesh(model, res)
    lab, siz = mesh.mesh_components(m)
    big = int(torch.argmax(siz))
    out = mesh.remove_small_components(m, keep_largest=1)
    assert out["triangles"].shape[0] == int(siz[big])
    # every triangle of the largest component is kept, in order, on the same positions
    tri_big = m["triangles"][lab == big]
    assert torch.equal(m["vertices"][tri_big], out["vertices"][out["triangles"]])
    f0, c0 = _fractions(m, scene, res)
    print("extract_mesh %d^3: %d triangles in %d components; outside-and-far %.4f, inside-and-deep %.4f"
          % (res, m["triangles"].shape[0], int((siz > 0).sum()), f0, c0))
    for k in (1, 2, 5):
        o = mesh.remove_small_components(m, keep_largest=k)
        f, c = _fractions(o, scene, res)
        print("  keep_largest=%d: %d triangles; outside-and-far %.4f, inside-and-deep %.4f" % (k, o["triangles"].shape[0], f, c))
    for n in (100, 1000):
        o = mesh.remove_small_components(m, min_triangles=n)
        f, c = _fractions(o, scene, res)
        print("  min_triangles=%d: %d triangles; outside-and-far %.4f, inside-and-deep %.4f" % (n, o["triangles"].shape[0], f, c))

    # remove_floaters then extract_mesh_sparse == extract_mesh_sparse of a model given the oracle's cleaned bitfield
    bits0 = model.density_bitfield.clone()
    dg0 = model.density_grid.clone()
    lab_o, siz_o = R.grid_components(bits0.cpu().numpy(), model.cascades, model.grid_size, float(model.scale))
    keep_o, _ = R.select(lab_o, siz_o, keep_largest=1)
    bits_o, _, _ = R.grid_clean(bits0.cpu().numpy(), None, model.cascades, model.grid_size, float(model.scale), lab_o, keep_o)
    try:
        model.density_bitfield.copy_(torch.as_tensor(bits_o).cuda())
        want = mesh.extract_mesh_sparse(model, 256)
        model.density_bitfield.copy_(bits0)
        components.remove_floaters(model, keep_largest=1)
        assert torch.equal(model.density_bitfield, torch.as_tensor(bits_o).cuda())
        got = mesh.extract_mesh_sparse(model, 256)
        for k in ("vertices", "triangles", "normals"):
            assert torch.equal(got[k], want[k]), k
        model.density_bitfield.copy_(bits0)
        before = mesh.extract_mesh_sparse(model, 256)
        f0, c0 = _fractions(before, scene, 256)
        f1, c1 = _fractions(got, scene, 256)
        print("extract_mesh_sparse 256^3 before / after remove_floaters(keep_largest=1): %d / %d triangles; "
              "outside-and-far %.4f / %.4f, inside-and-deep %.4f / %.4f"
              % (before["triangles"].shape[0], got["triangles"].shape[0], f0, f1, c0, c1))
    finally:
        model.density_bitfield.copy_(bits0)
        model.density_grid.copy_(dg0)
