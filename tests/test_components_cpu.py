"""CPU tests of the connected-components restatement (oracle/components_ref.py) against plain breadth-first searches
over brute-force adjacency, of its cross-cascade rule against exact closed-box intersection of every cell pair, and
of the refusals of `python -m ngp_pl_b200.clean_occupancy` and export_mesh's component flags."""
import os
import subprocess
import sys
from collections import deque
from fractions import Fraction

import numpy as np
import pytest

from oracle import components_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bfs_labels(n, is_node, adj):
    """smallest node index of each node's component by BFS from every unvisited node in ascending order"""
    labels = np.full(n, -1, np.int32)
    for s in range(n):
        if not is_node[s] or labels[s] >= 0:
            continue
        labels[s] = s
        q = deque([s])
        while q:
            u = q.popleft()
            for v in adj.get(u, ()):
                if labels[v] < 0:
                    labels[v] = s
                    q.append(v)
    return labels


def _box(c, G, scale, xyz):
    mb = Fraction(R.half_extent(c, scale))
    return [(mb * (Fraction(2 * v, G) - 1), mb * (Fraction(2 * (v + 1), G) - 1)) for v in xyz]


def _meet(b0, b1):
    return all(lo0 <= hi1 and lo1 <= hi0 for (lo0, hi0), (lo1, hi1) in zip(b0, b1))


def _inside(b, mf):
    return all(lo >= -mf and hi <= mf for lo, hi in b)


def _brute_graph(occ, cascades, G, scale):
    """nodes and adjacency from exact rational boxes, every cell pair of a cascade and of consecutive cascades"""
    xyz = R.morton_coords(G)
    G3 = G ** 3
    boxes = [[_box(c, G, scale, xyz[m]) for m in range(G3)] for c in range(cascades)]
    node = np.zeros(cascades * G3, bool)
    for c in range(cascades):
        mf = Fraction(R.half_extent(c - 1, scale)) if c else None
        for m in range(G3):
            node[c * G3 + m] = occ[c, m] and (c == 0 or not _inside(boxes[c][m], mf))
    adj = {}
    for c in range(cascades):
        for a in range(G3):
            if not node[c * G3 + a]:
                continue
            for b in range(G3):
                if b != a and node[c * G3 + b] and np.abs(xyz[a] - xyz[b]).max() == 1:
                    adj.setdefault(c * G3 + a, set()).add(c * G3 + b)
            if c:
                for b in range(G3):
                    if node[(c - 1) * G3 + b] and _meet(boxes[c][a], boxes[c - 1][b]):
                        adj.setdefault(c * G3 + a, set()).add((c - 1) * G3 + b)
                        adj.setdefault((c - 1) * G3 + b, set()).add(c * G3 + a)
    return node, adj


@pytest.mark.parametrize("scale", [0.5, 1.0, 3.0, 16.0, 0.7])
def test_cross_cascade_rule_is_closed_box_intersection(scale):
    G = 4
    cascades = max(1 + int(np.ceil(np.log2(2 * scale))), 2)
    occ = np.ones((cascades, G ** 3), bool)
    node, adj = _brute_graph(occ, cascades, G, scale)
    assert (R.nodes(occ, cascades, G, scale).reshape(-1) == node).all()
    got = set(map(tuple, R.grid_edges(R.nodes(occ, cascades, G, scale), cascades, G, scale).tolist()))
    G3 = G ** 3
    want = {(a, b) for a, bs in adj.items() for b in bs if a // G3 > b // G3}
    got_cross = {e for e in got if e[0] // G3 != e[1] // G3}
    assert got_cross == want


@pytest.mark.parametrize("scale,cascades,G,p", [(0.5, 1, 8, 0.3), (1.0, 2, 4, 0.4), (3.0, 4, 4, 0.25), (0.7, 2, 4, 0.5),
                                                (16.0, 6, 2, 0.5)])
def test_grid_oracle_matches_bfs(scale, cascades, G, p):
    rng = np.random.default_rng(int(scale * 10) + cascades)
    occ = rng.random((cascades, G ** 3)) < p
    bits = np.packbits(occ.reshape(-1), bitorder="little")
    labels, sizes = R.grid_components(bits, cascades, G, scale)
    node, adj = _brute_graph(occ, cascades, G, scale)
    want = _bfs_labels(cascades * G ** 3, node, adj)
    assert (labels == want).all()
    assert (sizes == np.bincount(want[want >= 0], minlength=want.size)).all()


def test_select_ranks_by_size_then_label():
    labels = np.array([0, 0, 2, 2, 4, 4, 4, -1, 8], np.int32)
    sizes = np.zeros(9, np.int32)
    np.add.at(sizes, labels[labels >= 0], 1)
    keep, cnt = R.select(labels, sizes, keep_largest=2)
    assert cnt == (4, 2) and list(np.nonzero(keep)[0]) == [0, 4]
    keep, cnt = R.select(labels, sizes, min_size=2)
    assert cnt == (4, 3) and list(np.nonzero(keep)[0]) == [0, 2, 4]
    keep, cnt = R.select(labels, sizes, keep_largest=1, min_size=4)
    assert cnt == (4, 0) and not keep.any()


def test_inner_cells_follow_the_finer_cascade():
    """scale 1, G 4: cascade 1's cell 1 spans [-0.5, 0] and meets cascade 0's cells 0..2 on an axis, its cell 2 spans
    [0, 0.5] and meets cells 1..3; both are inner"""
    G, cascades, scale = 4, 2, 1.0
    midx = R.morton_index(G)
    occ = np.zeros((cascades, G ** 3), bool)
    occ[0, midx[0, 0, 0]] = True               # a floater of cascade 0 ...
    occ[1, midx[0, 0, 0]] = True               # ... touching a shell cell of cascade 1: a piece of 2
    for z in (1, 2, 3):
        occ[0, midx[3, 3, z]] = True           # the largest piece: 3 cells
    occ[1, midx[1, 1, 1]] = True               # inner, meets the floater only: cleared
    occ[1, midx[2, 2, 2]] = True               # inner, meets the kept piece: stays
    bits = np.packbits(occ.reshape(-1), bitorder="little")
    labels, sizes = R.grid_components(bits, cascades, G, scale)
    assert labels[G ** 3 + midx[1, 1, 1]] == -1 and labels[G ** 3 + midx[0, 0, 0]] == 0
    keep, cnt = R.select(labels, sizes, keep_largest=1)
    assert cnt == (2, 1)
    out, dg, n = R.grid_clean(bits, np.zeros((cascades, G ** 3), np.float32), cascades, G, scale, labels, keep)
    o = R.unpack(out, cascades, G)
    assert all(o[0, midx[3, 3, z]] for z in (1, 2, 3)) and o[1, midx[2, 2, 2]]
    assert not o[0, midx[0, 0, 0]] and not o[1, midx[0, 0, 0]] and not o[1, midx[1, 1, 1]]
    assert n == (2, 1) and o.sum() == 4
    assert (dg == -1).sum() == 3 and dg[1, midx[1, 1, 1]] == -1


def _random_soup(rng, V, F):
    return rng.integers(0, V, size=(F, 3)).astype(np.int64)


@pytest.mark.parametrize("V,F", [(10, 4), (50, 20), (200, 60), (1, 1)])
def test_mesh_oracle_matches_bfs(V, F):
    rng = np.random.default_rng(V + F)
    t = _random_soup(rng, V, F)
    labels, sizes = R.mesh_components(t, V)
    adj = {}
    for a in range(F):
        for b in range(F):
            if a != b and set(t[a]) & set(t[b]):
                adj.setdefault(a, set()).add(b)
    want = _bfs_labels(F, np.ones(F, bool), adj)
    assert (labels == want).all()
    assert (sizes == np.bincount(want, minlength=F)).all()


def test_mesh_filter_keeps_order_and_renumbers():
    v = np.arange(24, dtype=np.float32).reshape(8, 3)
    t = np.array([[5, 6, 7], [0, 1, 2], [2, 3, 1], [4, 4, 4]], np.int64)
    labels, sizes = R.mesh_components(t, 8)
    assert list(labels) == [0, 1, 1, 3] and list(sizes) == [1, 2, 0, 1]
    keep, cnt = R.select(labels, sizes, min_size=2)
    m = R.mesh_filter(v, t, labels, keep, normals=-v)
    assert cnt == (3, 1)
    assert (m["vertices"] == v[:4]).all() and (m["normals"] == -v[:4]).all() and m["colors"] is None
    assert (m["triangles"] == [[0, 1, 2], [2, 3, 1]]).all()


def _run(module, argv):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    code = ("import sys, runpy; sys.argv = [%r] + %r\n"
            "try:\n    runpy.run_module(%r, run_name='__main__')\n"
            "finally:\n    print('torch' in sys.modules, file=sys.stderr)\n" % (module, argv, module))
    return subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True, timeout=300)


def test_clean_occupancy_refusals(tmp_path):
    ok = str(tmp_path / "model.ckpt")
    open(ok, "wb").close()
    out = str(tmp_path / "out.ckpt")
    cases = [
        (["--out", out, "--keep_largest", "1"], "--ckpt_path"),
        (["--ckpt_path", str(tmp_path / "missing.ckpt"), "--out", out, "--keep_largest", "1"], "--ckpt_path"),
        (["--ckpt_path", ok, "--keep_largest", "1"], "--out"),
        (["--ckpt_path", ok, "--out", out], "--keep_largest"),
        (["--ckpt_path", ok, "--out", out, "--keep_largest", "0"], "--keep_largest"),
        (["--ckpt_path", ok, "--out", out, "--min_cells", "-3"], "--min_cells"),
        (["--ckpt_path", ok, "--out", out, "--min_cells", "2.5"], "--min_cells"),
        (["--ckpt_path", ok, "--out", out, "--keep_largest", "1", "--scale", "0"], "--scale"),
        (["--ckpt_path", ok, "--out", ok, "--keep_largest", "1"], "--out"),
        (["--ckpt_path", ok, "--out", str(tmp_path / "no" / "x.ckpt"), "--keep_largest", "1"], "--out"),
    ]
    for argv, flag in cases:
        r = _run("ngp_pl_b200.clean_occupancy", argv)
        assert r.returncode == 2, (argv, r.returncode, r.stderr)
        assert flag in r.stderr, (argv, r.stderr)
        assert r.stderr.strip().splitlines()[-1] == "False", (argv, r.stderr)


def test_export_mesh_component_flag_refusals(tmp_path):
    ok = str(tmp_path / "model.ckpt")
    open(ok, "wb").close()
    for argv, flag in [(["--ckpt_path", ok, "--keep_largest", "0"], "--keep_largest"),
                       (["--ckpt_path", ok, "--min_triangles", "0"], "--min_triangles"),
                       (["--ckpt_path", ok, "--min_triangles", "x"], "--min_triangles")]:
        r = _run("ngp_pl_b200.export_mesh", argv)
        assert r.returncode == 2, (argv, r.returncode, r.stderr)
        assert flag in r.stderr, (argv, r.stderr)
        assert r.stderr.strip().splitlines()[-1] == "False", (argv, r.stderr)
