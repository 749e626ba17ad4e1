"""CPU tests of mesh simplification: oracle/mesh_simplify.py (the numpy float64 restatement of include/ngp_b200.h's
vertex clustering with quadric-error placement) against hand-checked cases, and `export_mesh --simplify`'s parsing
and refusals (exit status 2, naming the flag, before torch is imported)."""
import os
import subprocess
import sys

import numpy as np

from oracle import mesh_simplify as MS
from oracle.mcubes_ref import marching_cubes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LO4, HI4 = (0, 0, 0), (4, 4, 4)  # grid 4 over these bounds: unit cells, cell (x, y, z) has key (x*4 + y)*4 + z


def cell(x, y, z, d=(0.5, 0.5, 0.5)):
    return [x + d[0], y + d[1], z + d[2]]


def grid_tris(k, a=(1, 0, 0), b=(0, 1, 0), o=(0, 0, 0), flip=False):
    """a (k+1)^2 vertex grid o + i/k a + j/k b, two triangles per quad"""
    i, j = np.meshgrid(np.arange(k + 1), np.arange(k + 1), indexing="ij")
    v = np.asarray(o, np.float64) + (i.reshape(-1, 1) * np.asarray(a) + j.reshape(-1, 1) * np.asarray(b)) / k
    idx = lambda i, j: i * (k + 1) + j  # noqa: E731
    t = []
    for i in range(k):
        for j in range(k):
            q = [idx(i, j), idx(i + 1, j), idx(i + 1, j + 1), idx(i, j + 1)]
            t += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    t = np.array(t, np.int64)
    return v, t[:, ::-1].copy() if flip else t


def box_mesh(k):
    """the six faces of the unit cube, each a k x k grid of its own (outward triangles)"""
    faces = [((0, 1, 0), (0, 0, 1), (0, 0, 0)), ((0, 0, 1), (0, 1, 0), (1, 0, 0)),
             ((0, 0, 1), (1, 0, 0), (0, 0, 0)), ((1, 0, 0), (0, 0, 1), (0, 1, 0)),
             ((1, 0, 0), (0, 1, 0), (0, 0, 0)), ((0, 1, 0), (1, 0, 0), (0, 0, 1))]
    vs, ts, n = [], [], 0
    for a, b, o in faces:
        v, t = grid_tris(k, a, b, o)
        vs.append(v)
        ts.append(t + n)
        n += len(v)
    return np.concatenate(vs).astype(np.float32), np.concatenate(ts)


def test_cluster_grid_rule():
    lo, h, n = MS.cluster_grid((0, 0, 0), (4, 2, 1), 8)
    assert h == np.float32(0.5) and list(n) == [8, 4, 2]
    lo, h, n = MS.cluster_grid((-1, -1, -1), (1, 1, 1), 1)
    assert h == np.float32(2) and list(n) == [1, 1, 1]
    lo, h, n = MS.cluster_grid((0, 0, 0), (3, 1, 0.3), 7)  # ceil rounds the partial cell up, capped at grid
    assert list(n) == [7, 3, 1]
    keys = MS.cluster_keys(np.array([[0.0, 0.0, 0.0], [-9, 0.2, 0.1], [2.99, 0.99, 0.29], [99, 99, 99]], np.float32),
                           lo, h, n)
    assert list(keys) == [0, 0, (6 * 3 + 2) * 1 + 0, (6 * 3 + 2) * 1 + 0]


def test_box_corners_at_grid_2():
    v, t = box_mesh(6)
    r = MS.simplify(v, t, (0, 0, 0), (1, 1, 1), 2)
    assert len(r["vertices"]) == 8
    corners = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float64)  # key order
    assert np.abs(r["positions64"] - corners).max() < 1e-12
    assert np.array_equal(r["vertices"], corners.astype(np.float32))
    assert list(r["key"]) == list(range(8))
    tri = r["triangles"]
    assert len(tri) > 0 and (tri[:, 0] != tri[:, 1]).all() and (tri[:, 1] != tri[:, 2]).all()


def test_tilted_plane_on_plane_and_inside_boxes():
    v, t = grid_tris(16)
    v = np.concatenate([v[:, :2], (0.25 * v[:, 0] + 0.5 * v[:, 1] + 0.125)[:, None]], 1).astype(np.float32)
    lo, hi = (0, 0, 0), (1, 1, 1)
    r = MS.simplify(v, t, lo, hi, 4)
    p = r["positions64"]
    assert len(p) > 4
    assert np.abs(0.25 * p[:, 0] + 0.5 * p[:, 1] + 0.125 - p[:, 2]).max() < 1e-12
    glo, h, n = MS.cluster_grid(lo, hi, 4)
    keys = MS.cluster_keys(v, glo, h, n)
    for q, k in zip(p, r["key"]):
        mine = v[keys == k].astype(np.float64)
        assert (q >= mine.min(0) - 1e-12).all() and (q <= mine.max(0) + 1e-12).all()


def _run(v, t, grid=4, lo=LO4, hi=HI4, **kw):
    return MS.simplify(np.array(v, np.float32), np.array(t, np.int64).reshape(-1, 3), lo, hi, grid, **kw)


def test_degenerate_triangle_removed():
    v = [cell(0, 0, 0), cell(0, 0, 0, (0.6, 0.5, 0.5)), cell(1, 0, 0), cell(0, 1, 0)]
    r = _run(v, [[0, 1, 2], [0, 2, 3]])
    assert r["triangles"].tolist() == [[0, 2, 1]]
    assert r["key"].tolist() == [0, 4, 16]
    # cluster 0 = {v0, v1}: their mean, on the plane z = 0.5 of the one triangle with area
    assert r["vertices"].tolist() == [[np.float32(0.55), 0.5, 0.5], [0.5, 1.5, 0.5], [1.5, 0.5, 0.5]]


def test_duplicates_keep_the_first_and_opposite_pairs_stay():
    A, B, C = cell(0, 0, 0), cell(0, 1, 0), cell(1, 0, 0)
    A2, B2, C2 = cell(0, 0, 0, (0.4, 0.5, 0.5)), cell(0, 1, 0, (0.5, 0.4, 0.5)), cell(1, 0, 0, (0.4, 0.5, 0.5))
    v = [A, B, C, A2, B2, C2]
    tris = [[0, 2, 1],  # (A, C, B)
            [4, 3, 5],  # (B, A, C): a rotation of the first -> dropped
            [3, 4, 5],  # (A, B, C): the opposite orientation -> kept
            [5, 4, 3],  # (C, B, A): a rotation of the first -> dropped
            [1, 0, 5]]  # (B, A, C) again -> dropped
    r = _run(v, tris)
    assert r["key"].tolist() == [0, 4, 16]
    assert r["triangles"].tolist() == [[0, 2, 1], [0, 1, 2]]


def test_vertices_in_ascending_key_order_and_unreferenced_clusters_dropped():
    v = [cell(2, 2, 0), cell(0, 1, 1), cell(1, 1, 0),  # keys 40, 5, 20
         cell(3, 3, 3),  # key 63: only in a collapsed triangle
         cell(3, 0, 0)]  # key 48: in no triangle
    r = _run(v, [[0, 1, 2], [3, 3, 0]])
    assert r["key"].tolist() == [5, 20, 40]
    assert r["triangles"].tolist() == [[2, 0, 1]]
    assert np.array_equal(r["vertices"], np.array([v[1], v[2], v[0]], np.float32))


def test_out_of_bounds_vertices_clamp_to_border_cells():
    v = [[-5.0, 0.5, 9.0], [10.0, 10.0, 10.0], [0.5, 3.5, -1.0]]  # cells (0, 0, 3), (3, 3, 3), (0, 3, 0)
    r = _run(v, [[0, 1, 2]])
    assert r["key"].tolist() == [3, 12, 63]
    assert r["triangles"].tolist() == [[0, 2, 1]]
    assert np.array_equal(r["vertices"], np.array([v[0], v[2], v[1]], np.float32))  # singletons stay where they are


def test_grid_1_and_empty_meshes():
    v, t = box_mesh(3)
    r = MS.simplify(v, t, (0, 0, 0), (1, 1, 1), 1)
    assert r["vertices"].shape == (0, 3) and r["triangles"].shape == (0, 3)
    for v, t in ((np.zeros((0, 3)), np.zeros((0, 3))), (np.ones((4, 3)), np.zeros((0, 3)))):
        r = MS.simplify(v, t, (0, 0, 0), (1, 1, 1), 8, normals=np.zeros((len(v), 3)), colors=np.zeros((len(v), 3)))
        assert r["vertices"].shape == (0, 3) and r["triangles"].shape == (0, 3)
        assert r["normals"].shape == (0, 3) and r["colors"].shape == (0, 3)


def test_normals_and_colours_averaged_exactly():
    v = [cell(0, 0, 0), cell(0, 0, 0, (0.2, 0.3, 0.4)),  # A
         cell(1, 0, 0), cell(1, 0, 0, (0.1, 0.1, 0.1)), cell(1, 0, 0, (0.9, 0.9, 0.9)),  # B
         cell(0, 1, 0)]  # C
    n = [[1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, -1], [0, 0, 0], [0, 3, 4]]
    c = [[10, 20, 30], [11, 20, 255], [0, 0, 0], [1, 1, 1], [1, 1, 1], [7, 8, 9]]
    r = _run(v, [[0, 2, 5], [1, 3, 5]], normals=n, colors=c)
    assert r["triangles"].tolist() == [[0, 2, 1]]
    s = 1 / np.sqrt(2)
    assert np.array_equal(r["normals"], np.array([[s, s, 0], [0, 0.6, 0.8], [0, 0, 0]]))
    assert r["colors"].tolist() == [[11, 20, 143], [7, 8, 9], [1, 1, 1]]


def test_sphere_bounds_and_validity():
    N = 40
    x = np.linspace(-1, 1, N, dtype=np.float32)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    vol = -np.sqrt((X - 0.1) ** 2 + (Y + 0.05) ** 2 + Z ** 2)
    step = np.float32(2 / (N - 1))
    v, t = marching_cubes(vol, -0.7, lo=np.full(3, -1, np.float32), step=np.full(3, step, np.float32))
    for grid in (3, 6, 11):
        r = MS.simplify(v, t, (-1, -1, -1), (1, 1, 1), grid)
        h, tri, out = r["h"], r["triangles"], r["vertices"]
        assert 0 < len(tri) < len(t)
        assert tri.min() >= 0 and tri.max() < len(out) and len(np.unique(tri)) == len(out)
        assert ((tri[:, 0] != tri[:, 1]) & (tri[:, 1] != tri[:, 2]) & (tri[:, 0] != tri[:, 2])).all()
        rot = np.stack([np.roll(tri, -s, 1)[np.arange(len(tri)), :] for s in range(3)])  # (3, F, 3)
        canon = rot[np.argmin(tri, 1), np.arange(len(tri))]
        assert len(np.unique(canon, axis=0)) == len(tri)
        glo, hh, n = MS.cluster_grid((-1, -1, -1), (1, 1, 1), grid)
        keys = MS.cluster_keys(v, glo, hh, n)
        pos = np.searchsorted(r["key"], keys)
        ref = (pos < len(out)) & (r["key"][np.minimum(pos, len(out) - 1)] == keys)
        dist = np.sqrt(((v[ref].astype(np.float64) - out[pos[ref]]) ** 2).sum(1))
        assert ref.mean() > 0.9 and dist.max() <= np.sqrt(3) * h * (1 + 1e-6)


# ---- export_mesh --simplify ------------------------------------------------------------------------------------------
def _cli(argv=None, code=None):
    cmd = [sys.executable, "-c", code] if code is not None else [sys.executable, "-m", "ngp_pl_b200.export_mesh"] + argv
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)


def test_export_mesh_simplify_parses_without_torch():
    code = ("import sys; from ngp_pl_b200 import export_mesh as E\n"
            "print(E.parse_args(['--ckpt_path', %r]).simplify)\n"
            "print(E.parse_args(['--ckpt_path', %r, '--simplify', '256']).simplify)\n"
            "print(E.parse_args(['--ckpt_path', %r, '--simplify', '65536', '--dense']).simplify)\n"
            "print('torch' in sys.modules)\n" % (__file__, __file__, __file__))
    r = _cli(None, code)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines() == ["None", "256", "65536", "False"]


def test_export_mesh_simplify_refusals_exit_2_before_torch(tmp_path):
    ok = os.path.join(str(tmp_path), "m.ckpt")
    open(ok, "wb").close()
    for g in ("0", "65537", "-4", "x"):
        argv = ["--ckpt_path", ok, "--simplify", g]
        r = _cli(argv)
        assert r.returncode == 2 and "--simplify" in r.stderr, (argv, r.returncode, r.stderr)
        code = ("import sys; from ngp_pl_b200 import export_mesh\n"
                "try:\n    export_mesh.main(%r)\n"
                "except SystemExit as e:\n    code = e.code\n"
                "print(code, 'torch' in sys.modules)\n" % (argv,))
        r = _cli(None, code)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)
