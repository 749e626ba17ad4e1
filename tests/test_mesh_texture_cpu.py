"""CPU tests of the texture atlas rule (oracle/mesh_texture.py, the numpy restatement of include/ngp_b200.h "Texture
baking"): disjoint aligned squares inside the atlas, a maximal S, undistorted counter-clockwise uv with the margin kept,
the band and closest points against brute force, hand cases, the composite's limits, write_obj's files, and the
`export_mesh --texture` flags and refusals."""
import os

import numpy as np
import pytest

from oracle import mesh_texture as MT
from test_export_mesh_cpu import _run


def _random_mesh(seed, F, V=None, scale=1.0):
    rng = np.random.default_rng(seed)
    V = V or max(3, F)
    v = (rng.standard_normal((V, 3)) * scale * np.exp(rng.uniform(-4, 0, (V, 1)))).astype(np.float32)
    t = rng.integers(0, V, (F, 3))
    return v, t


def _squares_ok(at, W):
    sq = at["squares"].astype(np.int64)
    x0, y0, s = sq[:, 0], sq[:, 1], sq[:, 2]
    assert (s >= MT.S_MIN).all() and ((s & (s - 1)) == 0).all()
    assert (x0 % s == 0).all() and (y0 % s == 0).all()
    assert (x0 >= 0).all() and (y0 >= 0).all() and (x0 + s <= W).all() and (y0 + s <= W).all()
    cover = np.zeros((W, W), np.int32)
    for a, b, c in sq:
        cover[b:b + c, a:a + c] += 1
    assert cover.max(initial=0) <= 1
    return sq


def _maximal(at, W):
    S = at["S"]
    assert S == W or (at["hist"] * MT.side(np.arange(64), 2 * S) ** 2).sum() > W * W
    assert (at["hist"] * MT.side(np.arange(64), S) ** 2).sum() <= W * W


@pytest.mark.parametrize("seed,F,W", [(0, 1, 16), (1, 7, 16), (2, 16, 16), (3, 100, 64), (4, 300, 128), (5, 1000, 512)])
def test_squares_disjoint_aligned_and_S_maximal(seed, F, W):
    v, t = _random_mesh(seed, F)
    at = MT.atlas(v, t, W)
    _squares_ok(at, W)
    _maximal(at, W)
    # the packing order: sizes descending, ties by triangle index
    s = at["squares"][at["order"], 2]
    assert (np.diff(s) <= 0).all()
    same = np.diff(s) == 0
    assert (np.diff(at["order"])[same] > 0).all()


def _uv_checks(v, t, at):
    """the double placement is the 3-D triangle scaled by rho (1e-9 relative on every edge), uv is it rounded to fp32
    once, counter-clockwise and at least the margin inside the square"""
    assert np.array_equal(at["uv"], at["uv64"].astype(np.float32))
    u64 = at["uv64"]
    sq = at["squares"].astype(np.int64)
    p = v.astype(np.float64)[t]
    ok = at["k"] < MT.MAX_CLASS
    rho = np.ldexp((sq[:, 2] - 2).astype(np.float64), -at["e"])
    for k in range(3):
        e3 = np.linalg.norm(p[:, (k + 1) % 3] - p[:, k], axis=1) * rho
        e2 = np.linalg.norm(u64[:, (k + 1) % 3] - u64[:, k], axis=1)
        big = ok & (e3 > 1e-6 * (sq[:, 2] - 2))  # shorter edges: relative to the square's inner side
        assert (np.abs(e2 - e3)[big] <= 1e-9 * e3[big]).all(), k
        assert (np.abs(e2 - e3)[ok] <= 1e-9 * (sq[ok, 2] - 2)).all(), k
    uv = at["uv"].astype(np.float64)
    u, w = uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]
    area = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    assert (area >= -1e-9).all()
    lo, hi = sq[:, None, :2] + MT.MARGIN, (sq[:, None, :2] + sq[:, None, 2:] - MT.MARGIN)
    assert (uv >= lo).all() and (uv <= hi).all()


@pytest.mark.parametrize("seed,F,W", [(10, 50, 64), (11, 500, 256), (12, 2000, 256)])
def test_uv_is_the_triangle_scaled_ccw_and_inside_the_margin(seed, F, W):
    v, t = _random_mesh(seed, F)
    at = MT.atlas(v, t, W)
    _uv_checks(v, t, at)


def _brute_band(uv, sq, W):
    """every texel of every square whose open box meets the closed triangle, decided by clipping the triangle to the box"""
    out = set()
    for i in range(uv.shape[0]):
        P = uv[i].astype(np.float64)
        x0, y0, s = sq[i]
        for x in range(x0, x0 + s):
            for y in range(y0, y0 + s):
                if _clip_nonempty(P, x - 0.5, x + 1.5, y - 0.5, y + 1.5):
                    out.add((int(MT.interleave(x, y)), i))
    return out


def _clip_nonempty(P, xl, xh, yl, yh):
    """does the closed triangle P meet the open box? Sutherland-Hodgman clip against the closed box, then: a
    non-degenerate clipped polygon meets the open box, and a degenerate one (a segment or point) must not lie on the
    box's boundary"""
    poly = [tuple(p) for p in P]
    for axis, bound, keep_ge in ((0, xl, True), (0, xh, False), (1, yl, True), (1, yh, False)):
        out = []
        n = len(poly)
        for k in range(n):
            a, b = poly[k], poly[(k + 1) % n]
            ina = a[axis] >= bound if keep_ge else a[axis] <= bound
            inb = b[axis] >= bound if keep_ge else b[axis] <= bound
            if ina:
                out.append(a)
            if ina != inb:
                t = (bound - a[axis]) / (b[axis] - a[axis])
                out.append((a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1])))
        poly = out
        if not poly:
            return False
    q = np.array(poly)
    return bool(((q[:, 0] > xl) & (q[:, 0] < xh) & (q[:, 1] > yl) & (q[:, 1] < yh)).any() or
                ((q[:, 0].max() > xl) and (q[:, 0].min() < xh) and (q[:, 1].max() > yl) and (q[:, 1].min() < yh) and
                 _centroid_inside(q, xl, xh, yl, yh)))


def _centroid_inside(q, xl, xh, yl, yh):
    c = q.mean(0)
    return xl < c[0] < xh and yl < c[1] < yh


@pytest.mark.parametrize("seed,F,W", [(20, 12, 32), (21, 40, 64), (22, 60, 128)])
def test_band_equals_brute_force(seed, F, W):
    v, t = _random_mesh(seed, F)
    at = MT.atlas(v, t, W)
    m, tri = MT.band(at["uv"], at["squares"], W)
    assert (np.diff(m) > 0).all()
    got = set(zip(m.tolist(), tri.tolist()))
    ref = _brute_band(at["uv"], at["squares"].astype(np.int64), W)
    assert got == ref, (len(got ^ ref), sorted(got ^ ref)[:5])


@pytest.mark.parametrize("seed", [30, 31, 32])
def test_closest_points_equal_brute_force(seed):
    v, t = _random_mesh(seed, 30)
    W = 64
    at = MT.atlas(v, t, W)
    m, tri = MT.band(at["uv"], at["squares"], W)
    rot = at["rot"][tri]
    i = np.arange(len(tri))
    uv = at["uv"][tri]
    uvt = np.stack([uv[i, rot % 3], uv[i, (rot + 1) % 3], uv[i, (rot + 2) % 3]], 1).astype(np.float64)
    x, y = MT.deinterleave(m)
    b = MT.closest_bary(uvt, x + 0.5, y + 0.5)
    assert np.allclose(b.sum(1), 1) and (b >= -1e-12).all()
    got = np.einsum("nk,nkd->nd", b, uvt)
    q = np.stack([x + 0.5, y + 0.5], 1)
    # brute force: a fine barycentric grid of each triangle
    g = np.linspace(0, 1, 201)
    bb, cc = np.meshgrid(g, g)
    keep = bb + cc <= 1
    bb, cc = bb[keep], cc[keep]
    pts = uvt[:, None, 0] + bb[None, :, None] * (uvt[:, None, 1] - uvt[:, None, 0]) + \
        cc[None, :, None] * (uvt[:, None, 2] - uvt[:, None, 0])
    dmin = np.sqrt(((pts - q[:, None]) ** 2).sum(-1)).min(1)
    dgot = np.sqrt(((got - q) ** 2).sum(-1))
    span = np.abs(uvt - uvt[:, :1]).max((1, 2))
    assert (dgot <= dmin + 1e-12).all()
    assert (dmin - dgot <= span / 200 + 1e-12).all()


def test_hand_cases():
    W = 16
    # one triangle: S = W, the square is the whole atlas
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    at = MT.atlas(v, [[0, 1, 2]], W)
    assert at["S"] == W and at["squares"].tolist() == [[0, 0, 16]]
    assert at["rot"][0] == 1  # |c - b| = sqrt 2 is the longest: B, C, A
    uv = at["uv"][0].astype(np.float64)
    assert uv[1].tolist() == [1.0, 1.0]  # A' = corner b at the margin
    assert np.isclose(uv[2, 0] - uv[1, 0], 14 * np.sqrt(2) / 2 ** 1) and uv[2, 1] == 1.0
    # an equilateral triangle
    h = np.float32(np.sqrt(3) / 2)
    at = MT.atlas(np.array([[0, 0, 0], [1, 0, 0], [0.5, h, 0]], np.float32), [[0, 1, 2]], W)
    u = at["uv"][0].astype(np.float64)
    e = [np.linalg.norm(u[(k + 1) % 3] - u[k]) for k in range(3)]
    assert np.allclose(e, e[0], rtol=1e-6)
    # a needle, a collinear triangle and three equal corners: all placed, margin kept, band non-empty
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1e-6, 0], [2, 0, 0], [3, 0, 0], [4, 0, 0], [5, 5, 5]], np.float32)
    t = np.array([[0, 1, 2], [3, 4, 5], [6, 6, 6]])
    at = MT.atlas(v, t, W)
    _squares_ok(at, W)
    _uv_checks(v, t, at)
    assert at["k"][2] == MT.MAX_CLASS
    assert np.all(at["uv"][2] == at["uv"][2][0])
    m, tri = MT.band(at["uv"], at["squares"], W)
    assert set(tri.tolist()) == {0, 1, 2}
    assert (tri == 2).sum() == 4  # a point at a texel corner (x0 + 1, y0 + 1): the 2 x 2 texels around it
    p, n, _ = MT.surface(v, t, None, at["rot"], at["uv"], m, tri, W)
    assert np.array_equal(n[tri == 2], np.tile([0, 0, -1], ((tri == 2).sum(), 1)).astype(np.float32))
    assert np.array_equal(p[tri == 2], np.tile(v[6], ((tri == 2).sum(), 1)))
    col = n[tri == 1]  # collinear: no face normal either
    assert np.array_equal(col, np.tile([0, 0, -1], (len(col), 1)).astype(np.float32))


def test_full_atlas_and_one_triangle_more():
    W = 32
    F = W * W // 16
    v, t = _random_mesh(40, F)
    at = MT.atlas(v, t, W)
    assert (at["squares"][:, 2] == 4).all() and at["offset"][-1] == W * W
    _squares_ok(at, W)
    with pytest.raises(ValueError, match="W >= 64"):
        MT.atlas(v, np.concatenate([t, t[:1]]), W)
    assert MT.smallest_size(F + 1) == 64 and MT.smallest_size(F) == 32 and MT.smallest_size(0) == 16


def test_composite_limits():
    rng = np.random.default_rng(0)
    n, K = 50, 16
    c = rng.uniform(0, 1, (n, K + 1, 3))
    sig = rng.uniform(0, 50, (n, K + 1))
    assert np.array_equal(MT.composite(sig, c, 0.0), c[:, K])  # r = 0: delta = 0
    assert np.array_equal(MT.composite(np.zeros((n, K + 1)), c, 0.1), c[:, K])
    assert np.allclose(MT.composite(np.full((n, K + 1), 1e30), c, 0.1), c[:, 0])
    # r = 0: every sample is the surface point
    p = rng.standard_normal((n, 3)).astype(np.float32)
    nr = rng.standard_normal((n, 3)).astype(np.float32)
    o, d, t, delta, x = MT.sample_geometry(p, nr, 0.0, K)
    assert delta == 0 and np.array_equal(o, p) and np.array_equal(x, np.repeat(p[:, None], K + 1, 1))
    o, d, t, delta, x = MT.sample_geometry(p, nr, 0.25, 4)
    assert delta == np.float32(0.125) and t.tolist() == [0.0625, 0.1875, 0.3125, 0.4375, 0.25]
    assert MT.quantise([[0.5 / 255, 1.5 / 255, 2.0]]).tolist() == [[0, 2, 255]]


def _parse_obj(path):
    v, vn, vt, f = [], [], [], []
    for line in open(path):
        w = line.split()
        if not w or w[0].startswith("#"):
            continue
        if w[0] == "v":
            v.append([float(x) for x in w[1:]])
        elif w[0] == "vn":
            vn.append([float(x) for x in w[1:]])
        elif w[0] == "vt":
            vt.append([float(x) for x in w[1:]])
        elif w[0] == "f":
            f.append([[int(y) if y else 0 for y in x.split("/")] for x in w[1:]])
    return np.array(v, np.float32), np.array(vn, np.float32), np.array(vt, np.float32), np.array(f, np.int64)


def test_write_obj_round_trip(tmp_path, monkeypatch):
    import torch
    from ngp_pl_b200 import images, mesh
    v, t = _random_mesh(50, 200, 120)
    nrm = np.random.default_rng(1).standard_normal((120, 3)).astype(np.float32)
    W = 256
    at = MT.atlas(v, t, W)
    monkeypatch.setattr(images, "encode_png", lambda img, mode="fixed": b"\x89PNG-" + mode.encode())
    tex = torch.zeros(W, W, 3, dtype=torch.uint8)
    p = str(tmp_path / "m.obj")
    mesh.write_obj(p, v, t, nrm, at["uv"], tex)
    gv, gn, gt, gf = _parse_obj(p)
    assert np.array_equal(gv, v) and np.array_equal(gn, nrm)
    assert np.array_equal(gt, at["uv"].reshape(-1, 2) / np.float32(W))
    assert np.array_equal(gf[:, :, 0] - 1, t) and np.array_equal(gf[:, :, 2] - 1, t)
    assert np.array_equal(gf[:, :, 1] - 1, np.arange(3 * len(t)).reshape(-1, 3))
    assert "mtllib m.mtl\nusemtl material0\n" in open(p).read()
    assert "map_Kd m.png" in open(str(tmp_path / "m.mtl")).read().splitlines()
    assert open(str(tmp_path / "m.png"), "rb").read() == b"\x89PNG-dynamic"
    # without normals / uv: v//vn, v/vt, v; no MTL
    for kw, width in (({}, 1), ({"normals": nrm}, 3), ({"uv": at["uv"]}, 2)):
        q = str(tmp_path / "n.obj")
        mesh.write_obj(q, v, t, **kw)
        _, _, _, f = _parse_obj(q)
        assert f.shape == (len(t), 3, width) and np.array_equal(f[:, :, 0] - 1, t)
        assert not os.path.exists(str(tmp_path / "n.mtl"))
    with pytest.raises(RuntimeError, match="needs uv"):
        mesh.write_obj(p, v, t, texture=tex)


def test_export_mesh_texture_flags_parse_without_torch():
    code = ("import sys; from ngp_pl_b200 import export_mesh as E\n"
            "a = E.parse_args(['--ckpt_path', %r])\n"
            "print(a.texture, a.texture_offset, a.texture_samples)\n"
            "b = E.parse_args(['--ckpt_path', %r, '--texture', '8192', '--texture_offset', '0', '--texture_samples',"
            " '256', '--out', 'x.OBJ'])\n"
            "print(b.texture, b.texture_offset, b.texture_samples, b.out)\n"
            "print('torch' in sys.modules)\n" % (__file__, __file__))
    r = _run(None, code)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines() == ["None None 16", "8192 0.0 256 x.OBJ", "False"]


def test_export_mesh_texture_refusals(tmp_path):
    ok = str(tmp_path / "m.ckpt")
    open(ok, "wb").close()
    base = ["--ckpt_path", ok, "--out", "m.obj"]
    for argv, flag in ((["--texture", "100"], "--texture"), (["--texture", "8"], "--texture"),
                       (["--texture", "32768"], "--texture"), (["--texture", "64", "--colors"], "--colors"),
                       (["--texture", "64", "--texture_offset", "-1"], "--texture_offset"),
                       (["--texture", "64", "--texture_offset", "nan"], "--texture_offset"),
                       (["--texture", "64", "--texture_samples", "0"], "--texture_samples"),
                       (["--texture", "64", "--texture_samples", "257"], "--texture_samples")):
        r = _run(base + argv)
        assert r.returncode == 2 and flag in r.stderr, (argv, r.stderr)
    r = _run(["--ckpt_path", ok, "--texture", "64", "--out", "m.ply"])
    assert r.returncode == 2 and "--out" in r.stderr, r.stderr
    code = ("import sys; from ngp_pl_b200 import export_mesh\n"
            "try:\n    export_mesh.main(%r)\n"
            "except SystemExit as e:\n    code = e.code\n"
            "print(code, 'torch' in sys.modules)\n" % (base + ["--texture", "100"],))
    r = _run(None, code)
    assert r.stdout.split() == ["2", "False"], (r.stdout, r.stderr)
