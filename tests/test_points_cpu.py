"""CPU tests of the point-cloud export's restatement (oracle/points_ref.py) against brute force and analytic cases,
of `python -m ngp_pl_b200.export_points`'s refusals (exit status 2, naming the flag, before torch is imported), and of
a face-less mesh.write_ply round trip."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import points_ref as P
from oracle import mesh_simplify as MS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- stage 1: the ray permutation --------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2, 3, 4, 10, 97, 100, 360, 1000, 2 ** 12, 6 * 7 * 11 * 13, 100 * 640000])
def test_golden_step_is_coprime_and_a_bijection(N):
    g = P.golden_step(N)
    assert math.gcd(g, N) == 1 and (N == 1 or 1 <= g < N)
    assert g >= (P.GOLDEN * N + 5 * 10 ** 9) // 10 ** 10
    for h in range((P.GOLDEN * N + 5 * 10 ** 9) // 10 ** 10, g):
        assert math.gcd(h, N) != 1
    if N <= 10 ** 6:
        img, pix = P.ray_pixels(1, N, N)
        assert sorted(pix.tolist()) == list(range(N))


def test_golden_step_rounds_half_up_exactly():
    # 0.6180339887 N has a fraction of exactly 1/2 at N = 5 10^9 / gcd: compare with exact rationals
    from fractions import Fraction
    for N in (10 ** 10, 2 * 10 ** 10 + 1, 123456789, 2 ** 34 - 3, 2 ** 34 + 17):
        x = Fraction(6180339887, 10 ** 10) * N
        r = math.floor(x + Fraction(1, 2))
        g = P.golden_step(N)
        assert g >= r and all(math.gcd(h, N) != 1 for h in range(r, g))


@pytest.mark.parametrize("n_views,n_pix", [(1, 1), (3, 7), (100, 640000), (2 ** 10, 2 ** 24 + 3)])
def test_ray_pixels_exact_near_2_34(n_views, n_pix):
    N = n_views * n_pix
    R = min(N, 1 << 16)
    img, pix = P.ray_pixels(n_views, n_pix, R)
    g = P.golden_step(N)
    ks = list(range(min(R, 200))) + list(range(max(0, R - 200), R))
    for k in ks:
        q = (k * g) % N
        assert (img[k], pix[k]) == (q // n_pix, q % n_pix)
    q = img * n_pix + pix
    assert len(np.unique(q)) == R and (q >= 0).all() and (q < N).all()
    if n_views > 1 and R >= 4 * n_views:
        counts = np.bincount(img, minlength=n_views)
        assert counts.min() >= 1  # spread over every view


# ---- stage 3: fmaf and back-projection -------------------------------------------------------------------------------
def test_fmaf_rounds_once():
    from fractions import Fraction
    rng = np.random.RandomState(0)
    a = rng.randn(3000).astype(np.float32)
    b = (rng.randn(3000) * 10.0 ** rng.randint(-8, 8, 3000)).astype(np.float32)
    c = (rng.randn(3000) * 10.0 ** rng.randint(-8, 8, 3000)).astype(np.float32)
    # halfway cases of the double sum: c = -a b plus a tiny rest
    a[:20], b[:20] = np.float32(1 + 2 ** -23), np.float32(1 + 2 ** -23)
    c[:20] = np.float32(2 ** -60) * np.arange(1, 21, dtype=np.float32)
    got = P.fmaf(a, b, c)
    for i in range(len(a)):
        x = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(x))
        # the float32 nearest to x (ties to even), from exact rationals
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda f: (abs(Fraction(float(f)) - x), int(np.float32(f).view(np.int32)) & 1))
        assert got[i] == best, (i, a[i], b[i], c[i], got[i], best)


def test_backproject_rules():
    o = np.zeros((6, 3), np.float32)
    d = np.tile(np.float32([0, 0, 2]), (6, 1))
    op = np.float32([1, 0.5, 0.49, 1, 1, 0.5])
    depth = np.float32([0.5, 0.25, 0.2, 3.0, np.inf, 0.5])
    rgb = np.float32([[1, 0.5, 0], [0.5, 0.6, 0.1], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0.25, 0.25, 0.25]])
    keep, p, c, v = P.backproject(o, d, op, depth, rgb, 0.5, [-1, -1, -1], [1, 1, 2])
    assert keep.tolist() == [True, True, False, False, False, True]
    assert np.array_equal(p, np.float32([[0, 0, 1], [0, 0, 1], [0, 0, 2]]))  # the last on the closed box's face
    assert c.tolist() == [[255, 128, 0], [255, 255, 51], [128, 128, 128]]
    assert np.array_equal(v, np.float32([[0, 0, 1]] * 3))


# ---- stage 4: voxel keys ------------------------------------------------------------------------------------------
def test_voxel_keys_are_the_simplification_cells():
    rng = np.random.RandomState(1)
    p = (rng.rand(5000, 3) * [2, 1, 0.5] - [1, 0.5, 0]).astype(np.float32)
    p[:10] = [[5, 5, 5]] * 10  # outside: the border cell
    c = rng.randint(0, 256, (5000, 3)).astype(np.uint8)
    v = rng.randn(5000, 3).astype(np.float32)
    lo, hi = np.float32([-1, -0.5, 0]), np.float32([1, 0.5, 0.5])
    glo, h, n = MS.cluster_grid(lo, hi, 16)
    keys, cnt, pos, col, view = P.voxel(p, c, v, glo, h, n)
    k = MS.cluster_keys(p, glo, h, n)
    assert np.array_equal(keys, np.unique(k)) and cnt.sum() == 5000
    for j in range(0, len(keys), 37):
        m = k == keys[j]
        assert cnt[j] == m.sum()
        assert np.allclose(pos[j], p[m].astype(np.float64).mean(0), rtol=0, atol=1e-12)
        assert (col[j] == np.floor(c[m].astype(np.float64).mean(0) + 0.5)).all()


# ---- stage 5: exact kNN -------------------------------------------------------------------------------------------
def _naive(p, k):
    p = np.asarray(p, np.float32).astype(np.float64)
    out_d = []
    for i in range(len(p)):
        e = [[float(p[j, a]) - float(p[i, a]) for a in range(3)] for j in range(len(p))]
        d = sorted(((e[j][0] * e[j][0] + e[j][1] * e[j][1]) + e[j][2] * e[j][2], j) for j in range(len(p)) if j != i)
        out_d.append([x for x, _ in d[:min(k, len(p) - 1)]])
    return np.array(out_d).reshape(len(p), -1)


def adversarial_sets():
    rng = np.random.RandomState(2)
    sets = {}
    base = rng.rand(60, 3).astype(np.float32)
    sets["duplicates"] = np.concatenate([base, base[:30], base[:10]])
    sets["coplanar"] = np.concatenate([rng.rand(120, 2), np.zeros((120, 1))], 1).astype(np.float32)
    t = rng.rand(100).astype(np.float32)
    sets["collinear"] = np.stack([t, 2 * t, -t], 1).astype(np.float32)
    sets["cluster_and_far"] = np.concatenate([rng.rand(150, 3) * 1e-3, [[100, 0, 0], [0, -100, 0], [0, 0, 100]]]).astype(
        np.float32)
    sets["all_equal"] = np.ones((25, 3), np.float32)
    sets["tiny"] = rng.rand(5, 3).astype(np.float32)
    return sets


@pytest.mark.parametrize("name", list(adversarial_sets()))
@pytest.mark.parametrize("k", [1, 4, 20, 64])
def test_knn_matches_naive(name, k):
    p = adversarial_sets()[name]
    idx, d2 = P.knn(p, k, block=37)
    ref = _naive(p, k)
    assert d2.shape == ref.shape and np.array_equal(d2, ref)
    n = len(p)
    for i in range(n):
        assert i not in idx[i]
        assert len(set(idx[i].tolist())) == idx.shape[1]
        # ties ordered by index
        for a in range(idx.shape[1] - 1):
            assert d2[i, a] < d2[i, a + 1] or idx[i, a] < idx[i, a + 1]


def test_knn_small_n():
    for n in (1, 2, 3):
        p = np.arange(3 * n, dtype=np.float32).reshape(n, 3)
        idx, d2 = P.knn(p, 20)
        assert idx.shape == (n, n - 1)


# ---- stage 6: outliers ---------------------------------------------------------------------------------------------
def test_outliers_remove_isolated_points():
    p = adversarial_sets()["cluster_and_far"]
    idx, d2 = P.knn(p, 8)
    keep, d, mu, sigma, thr = P.outliers(d2, 2.0)
    assert keep[:150].all() and not keep[150:].any()
    assert np.isclose(mu, d.mean()) and np.isclose(sigma, d.std())


# ---- stage 7: normals ------------------------------------------------------------------------------------------------
def test_normals_of_a_plane_face_the_camera():
    rng = np.random.RandomState(3)
    n0 = np.array([1.0, 2.0, 2.0]) / 3
    u = np.cross(n0, [0, 0, 1.0])
    u /= np.linalg.norm(u)
    w = np.cross(n0, u)
    ab = rng.rand(400, 2) * 2 - 1
    p = (ab[:, :1] * u + ab[:, 1:] * w + 0.25 * n0).astype(np.float32)
    views = np.tile(-n0 + [0.1, 0, 0], (400, 1))
    views[::2] = n0  # seen from the other side
    idx, _ = P.knn(p, 12)
    nrm, gap, zero = P.normals(p, views, idx)
    assert not zero.any()
    s = np.where((views @ n0) > 0, -1.0, 1.0)
    assert np.abs(nrm - s[:, None] * n0).max() < 1e-5


def test_normals_of_a_sphere_point_out():
    rng = np.random.RandomState(4)
    x = rng.randn(4000, 3)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    p = (x * 0.5).astype(np.float32)
    idx, _ = P.knn(p, 10)
    nrm, gap, zero = P.normals(p, -x, idx)  # cameras outside look inwards
    cos = (nrm * x).sum(1)
    assert np.median(cos) > 0.999 and cos.min() > 0.98


def test_normals_zero_covariance():
    p = np.ones((5, 3), np.float32)
    idx, _ = P.knn(p, 3)
    nrm, gap, zero = P.normals(p, np.ones((5, 3)), idx)
    assert zero.all() and (nrm == 0).all()


# ---- PLY round trip ------------------------------------------------------------------------------------------------
def _read_ply(path):
    b = open(path, "rb").read()
    end = b.index(b"end_header\n") + len(b"end_header\n")
    head = b[:end].decode().splitlines()
    nv = int([l for l in head if l.startswith("element vertex")][0].split()[-1])
    nf = int([l for l in head if l.startswith("element face")][0].split()[-1])
    props = [l.split() for l in head if l.startswith("property") and "list" not in l]
    dt = [(q[2], "<f4" if q[1] == "float" else "u1") for q in props]
    rec = np.frombuffer(b[end:end + nv * np.dtype(dt).itemsize], dtype=dt)
    assert len(b) == end + nv * np.dtype(dt).itemsize + nf * 13
    return rec, nf


@pytest.mark.parametrize("normals,colors", [(True, True), (False, True), (True, False), (False, False)])
def test_write_ply_point_cloud_round_trip(tmp_path, normals, colors):
    from ngp_pl_b200 import mesh
    rng = np.random.RandomState(5)
    p = rng.randn(100, 3).astype(np.float32)
    n = rng.randn(100, 3).astype(np.float32) if normals else None
    c = rng.randint(0, 256, (100, 3)).astype(np.uint8) if colors else None
    path = str(tmp_path / "p.ply")
    mesh.write_ply(path, p, np.zeros((0, 3), np.int64), n, c)
    rec, nf = _read_ply(path)
    assert nf == 0
    assert np.array_equal(np.stack([rec["x"], rec["y"], rec["z"]], 1), p)
    if normals:
        assert np.array_equal(np.stack([rec["nx"], rec["ny"], rec["nz"]], 1), n)
    if colors:
        assert np.array_equal(np.stack([rec["red"], rec["green"], rec["blue"]], 1), c)


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def _run(argv=None, code=None):
    cmd = [sys.executable, "-c", code] if code is not None else [sys.executable, "-m", "ngp_pl_b200.export_points"] + argv
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)


def test_defaults_parse_without_torch():
    code = ("import sys; from ngp_pl_b200 import export_points as E\n"
            "a = E.parse_args(['--ckpt_path', %r])\n"
            "print(a.scale, a.root_dir, a.dataset_name, a.downsample, a.num_rays, a.min_opacity, a.bounds, a.voxel,"
            " a.nb_neighbors, a.std_ratio, a.keep_outliers, a.no_normals, a.out)\n"
            "print('torch' in sys.modules)\n" % (__file__,))
    r = _run(None, code)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.splitlines()
    assert lines[0] == "0.5 None nerf 1.0 1000000 0.5 None None 20 2.0 False False points.ply"
    assert lines[1] == "False"


def _refused(tmp):
    ok = os.path.join(tmp, "m.ckpt")
    return [
        ([], "--ckpt_path"),
        (["--ckpt_path", os.path.join(tmp, "missing.ckpt")], "--ckpt_path"),
        (["--ckpt_path", ok, "--scale", "0"], "--scale"),
        (["--ckpt_path", ok, "--num_rays", "0"], "--num_rays"),
        (["--ckpt_path", ok, "--num_rays", str(2 ** 28 + 1)], "--num_rays"),
        (["--ckpt_path", ok, "--min_opacity", "0"], "--min_opacity"),
        (["--ckpt_path", ok, "--min_opacity", "1.5"], "--min_opacity"),
        (["--ckpt_path", ok, "--min_opacity", "nan"], "--min_opacity"),
        (["--ckpt_path", ok, "--bounds", "0", "0", "0", "1", "-1", "1"], "--bounds"),
        (["--ckpt_path", ok, "--bounds", "0", "0", "0", "1", "inf", "1"], "--bounds"),
        (["--ckpt_path", ok, "--voxel", "0"], "--voxel"),
        (["--ckpt_path", ok, "--nb_neighbors", "0"], "--nb_neighbors"),
        (["--ckpt_path", ok, "--nb_neighbors", "65"], "--nb_neighbors"),
        (["--ckpt_path", ok, "--std_ratio", "-1"], "--std_ratio"),
        (["--ckpt_path", ok, "--downsample", "0"], "--downsample"),
        (["--ckpt_path", ok, "--dataset_name", "nsvf"], "--dataset_name"),
    ]


def test_refusals_exit_2_before_torch(tmp_path):
    tmp = str(tmp_path)
    open(os.path.join(tmp, "m.ckpt"), "wb").close()
    for argv, flag in _refused(tmp):
        r = _run(argv)
        assert r.returncode == 2, (argv, r.returncode, r.stderr)
        assert flag in r.stderr, (argv, r.stderr)
        code = ("import sys; from ngp_pl_b200 import export_points\n"
                "try:\n    export_points.main(%r)\n"
                "except SystemExit as e:\n    code = e.code\n"
                "print(code, 'torch' in sys.modules)\n" % (argv,))
        r = _run(None, code)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)
