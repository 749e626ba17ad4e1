"""Mesh extraction, host side: the generated marching-cubes table (tools/mc_table.py) and its face rule, the numpy
restatement oracle/mcubes_ref.py on analytic and random fields, write_ply, the NgpLattice mirror and the refusal of
CPU tensors. Runs without a GPU."""
import importlib.util
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import mc_table as T
from oracle import mcubes_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gen():
    spec = importlib.util.spec_from_file_location("mc_table_gen", os.path.join(ROOT, "tools", "mc_table.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# ---- the table ---------------------------------------------------------------------------------------------------------
def test_generated_table_is_committed():
    g = _gen()
    tab = g.table()
    assert open(g.HEADER).read() == g.render_header(tab)
    assert open(g.PYMOD).read() == g.render_pymod(tab)
    assert [list(t) for t in T.TRIS] == [[tuple(x) for x in t] for t in tab]


def _crossed(mask):
    return {e for e, (c0, c1, _) in enumerate(T.EDGES) if ((mask >> c0) & 1) != ((mask >> c1) & 1)}


def _undirected_counts(tris):
    cnt = {}
    for t in tris:
        for i in range(3):
            k = frozenset((t[i], t[(i + 1) % 3]))
            cnt[k] = cnt.get(k, 0) + 1
    return cnt


def test_table_uses_exactly_the_crossed_edges_and_at_most_five_triangles():
    assert max(len(t) for t in T.TRIS) == 5
    for m in range(256):
        used = {e for t in T.TRIS[m] for e in t}
        assert used == _crossed(m), m


def test_no_interior_diagonal_joins_two_vertices_of_one_face():
    g = _gen()
    for m in range(256):
        for k, c in _undirected_counts(T.TRIS[m]).items():
            a, b = tuple(k)
            assert c in (1, 2), (m, k)
            if c == 2:  # interior diagonal of a loop's triangulation
                assert not g.same_face(a, b), (m, a, b)
            else:       # a loop segment: drawn on one face
                assert g.same_face(a, b), (m, a, b)


def _face_segments_of_case(g, m, f):
    """directed loop segments of case m lying on face f"""
    fe = g.FACE_EDGES[f]
    cnt = _undirected_counts(T.TRIS[m])
    out = set()
    for t in T.TRIS[m]:
        for i in range(3):
            a, b = t[i], t[(i + 1) % 3]
            if cnt[frozenset((a, b))] == 1 and a in fe and b in fe:
                out.add((a, b))
    return out


def test_face_segments_depend_only_on_the_face_corner_signs():
    g = _gen()
    for f, (ring, _) in enumerate(g.FACES):
        others = [c for c in range(8) if c not in ring]
        for pattern in range(16):
            base = sum(((pattern >> i) & 1) << ring[i] for i in range(4))
            seen = {frozenset(_face_segments_of_case(g, base | sum(((o >> i) & 1) << others[i] for i in range(4)), f))
                    for o in range(16)}
            assert len(seen) == 1, (f, pattern, seen)


# ---- the oracle on analytic and random fields --------------------------------------------------------------------------
def _grid(shape):
    return np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij"), -1)


def sphere(n=32, r=10.0, c=15.5):
    return (r - np.linalg.norm(_grid((n, n, n)) - c, axis=-1)).astype(np.float32)


def torus(n=40, R_=11.0, r=4.0, c=19.5):
    p = _grid((n, n, n)) - c
    q = np.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2) - R_
    return (r - np.sqrt(q ** 2 + p[..., 2] ** 2)).astype(np.float32)


def two_spheres(n=40):
    g = _grid((n, n, n))
    a = 7.0 - np.linalg.norm(g - np.array([11.0, 12.0, 19.5]), axis=-1)
    b = 6.0 - np.linalg.norm(g - np.array([28.0, 26.0, 19.5]), axis=-1)
    return np.maximum(a, b).astype(np.float32)


def random_field(shape, seed, border=True):
    v = np.random.RandomState(seed).rand(*shape).astype(np.float32)
    if border:
        v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = 0, 0, 0, 0, 0, 0
    return v


def test_sphere_closed_oriented_and_normals_radial():
    r = 10.0
    V, F, N = R.marching_cubes(sphere(32, r), 0.0, normals=True)
    assert len(R.unpaired_edges(F)) == 0
    assert R.euler_characteristic(V, F) == 2
    vol = R.signed_volume(V, F)
    exact = 4 / 3 * np.pi * r ** 3
    assert 0 < vol and abs(vol - exact) < 0.01 * exact, (vol, exact)
    rad = (V - 15.5) / np.linalg.norm(V - 15.5, axis=1, keepdims=True)
    assert (np.einsum("ij,ij->i", N, rad) > 0.99).all()


@pytest.mark.parametrize("field,chi", [(torus, 0), (two_spheres, 4)])
def test_topology(field, chi):
    V, F = R.marching_cubes(field(), 0.0)
    assert len(R.unpaired_edges(F)) == 0
    assert R.euler_characteristic(V, F) == chi
    assert R.signed_volume(V, F) > 0


@pytest.mark.parametrize("shape", [(12, 13, 14), (5, 17, 9), (23, 6, 11), (8, 8, 30)])
def test_random_fields_with_outside_border_are_closed(shape):
    for seed in range(10):
        V, F = R.marching_cubes(random_field(shape, seed), 0.5)
        assert len(F) > 0
        assert len(R.unpaired_edges(F)) == 0, (shape, seed)


@pytest.mark.parametrize("shape", [(12, 13, 14), (2, 9, 7), (9, 2, 2), (6, 11, 3)])
def test_random_fields_open_only_on_the_lattice_boundary(shape):
    n = np.array(shape, np.float32) - 1
    for seed in range(5):
        V, F = R.marching_cubes(random_field(shape, 100 + seed, border=False), 0.5)
        bad = R.unpaired_edges(F)
        a, b = V[bad[:, 0]], V[bad[:, 1]]
        on_face = (((a == 0) & (b == 0)) | ((a == n) & (b == n))).any(1)
        assert on_face.all(), (shape, seed)


def test_uniform_volumes_and_two_point_axes():
    for v in (np.ones((5, 6, 7), np.float32), np.zeros((5, 6, 7), np.float32)):
        V, F = R.marching_cubes(v, 0.5)
        assert V.shape == (0, 3) and F.shape == (0, 3)
    v = np.zeros((2, 2, 2), np.float32)
    v[0, 0, 0] = 1
    V, F = R.marching_cubes(v, 0.5)
    assert len(F) == 1
    assert np.allclose(sorted(map(tuple, V)), sorted([(0.5, 0, 0), (0, 0.5, 0), (0, 0, 0.5)]))
    # corner 0 inside: the triangle's normal points away from it
    n = np.cross(V[F[0, 1]] - V[F[0, 0]], V[F[0, 2]] - V[F[0, 0]])
    assert (n > 0).all()


# ---- write_ply ---------------------------------------------------------------------------------------------------------
def read_ply(path):
    """minimal binary little-endian PLY reader for what write_ply writes"""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").split("\n")
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0"
    types = {"float": "<f4", "uchar": "u1"}
    elems, cur = [], None
    for ln in lines[2:]:
        w = ln.split()
        if w[:1] == ["element"]:
            cur = (w[1], int(w[2]), [])
            elems.append(cur)
        elif w[:2] == ["property", "list"]:
            assert w[2:] == ["uchar", "int", "vertex_indices"]
            cur[2].append(("n", "u1"))
            cur[2].append(("v", "<i4", (3,)))
        elif w[:1] == ["property"]:
            cur[2].append((w[2], types[w[1]]))
    out, off = {}, end
    for name, count, fields in elems:
        dt = np.dtype(fields)
        out[name] = np.frombuffer(data, dt, count, off)
        off += dt.itemsize * count
    assert off == len(data)
    return out


def test_write_ply_round_trip():
    from ngp_pl_b200.mesh import write_ply
    V, F, N = R.marching_cubes(sphere(16, 5.0, 7.5), 0.0, normals=True)
    col = np.random.RandomState(0).randint(0, 256, V.shape).astype(np.uint8)
    with tempfile.TemporaryDirectory() as d:
        for kw in ({}, {"normals": N}, {"colors": col}, {"normals": N, "colors": col}):
            p = os.path.join(d, "m.ply")
            write_ply(p, V, F, **kw)
            m = read_ply(p)
            v = m["vertex"]
            assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), V)
            assert (m["face"]["n"] == 3).all() and np.array_equal(m["face"]["v"], F)
            if "normals" in kw:
                assert np.array_equal(np.stack([v["nx"], v["ny"], v["nz"]], 1), N.astype(np.float32))
            if "colors" in kw:
                assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), col)


# ---- ABI mirror and the refusal of CPU tensors ---------------------------------------------------------------------------
def test_lattice_struct_matches_header():
    import ctypes
    from ngp_pl_b200 import _lib
    hdr = os.path.join(ROOT, "include")
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "ngp_b200.h"\nint main(void){printf("%zu %zu %zu %d\\n",'
                           ' sizeof(NgpLattice), offsetof(NgpLattice, lo), offsetof(NgpLattice, step), NGP_MC_SLAB_POINTS);'
                           ' return 0;}\n')
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", hdr, c, "-o", exe])
        size, lo, step, slab = [int(x) for x in subprocess.check_output([exe]).decode().split()]
    assert ctypes.sizeof(_lib.NgpLattice) == size
    assert _lib.NgpLattice.lo.offset == lo and _lib.NgpLattice.step.offset == step
    assert _lib.NGP_MC_SLAB_POINTS == slab


def test_mesh_functions_refuse_cpu_tensors():
    from ngp_pl_b200 import mesh
    from ngp_pl_b200.models.networks import NGP
    model = NGP(0.5, n_levels=4, log2_hashmap_size=14)
    with pytest.raises(RuntimeError):
        mesh.density_volume(model, 8)
    with pytest.raises(RuntimeError):
        mesh.extract_mesh(model, 8)
    with pytest.raises(RuntimeError):
        mesh.marching_cubes(torch.zeros(4, 4, 4), 0.5)


def test_lattice_step_is_fp32():
    from ngp_pl_b200 import mesh
    lat = mesh.lattice((3, 7, 512), (-0.5, -1.0, 0.1), (0.5, 2.0, 0.7))
    for a, (n, lo, hi) in enumerate(zip((3, 7, 512), (-0.5, -1.0, 0.1), (0.5, 2.0, 0.7))):
        assert lat.n[a] == n and lat.lo[a] == np.float32(lo)
        assert lat.step[a] == (np.float32(hi) - np.float32(lo)) / np.float32(n - 1)
    with pytest.raises(RuntimeError):
        mesh.lattice((1, 4, 4), 0.0, 1.0)
