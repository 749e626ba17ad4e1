"""CPU tests of the depth fusion's restatement (oracle/tsdf_ref.py) and of `python -m ngp_pl_b200.export_mesh --tsdf`'s
flags: the integration rule against the analytic TSDF of a plane seen head-on, the masked marching cubes against
oracle/mcubes_ref.py where every point is observed and its mask rules where some are not, and the CLI's refusals
(exit status 2, before torch is imported)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mcubes_ref as R
from oracle import tsdf_ref as T
from oracle.mc_table import TRIS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _K(W, H, f):
    return np.float32([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])


def _dirs(W, H, K):
    v, u = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    d = np.stack([(u - K[0, 2] + np.float32(0.5)) / K[0, 0], (v - K[1, 2] + np.float32(0.5)) / K[1, 1], np.ones_like(u)], -1)
    return d.reshape(-1, 3)


def _plane_setup(dtype):
    """one camera at z = -1 looking along +z at the plane z = D - 1 (camera depth D); the right half of the image has
    opacity below min_opacity"""
    W, H, f, D = 32, 24, 30.0, 1.25
    K = _K(W, H, f)
    pose = np.float32([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, -1]])[None]
    dirs = _dirs(W, H, K)
    op = np.ones((1, W * H), np.float32)
    op[0, (np.arange(W * H) % W) >= W // 2 + 4] = 0.3
    depth = (np.float32(D) * op).astype(np.float32)
    rgb = np.tile(np.float32([0.2, 0.4, 0.9]), (1, W * H, 1)) * op[..., None]
    n, lo, hi = (28, 26, 40), np.float32([-0.6, -0.5, -1.2]), np.float32([0.6, 0.5, 0.9])
    step = (hi - lo) / (np.array(n) - 1).astype(np.float32)
    x = T.lattice_points(n, lo, step, dtype)
    return dict(W=W, H=H, K=K, D=D, pose=pose, dirs=dirs, op=op, depth=depth, rgb=rgb, x=x, trunc=0.15)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_plane_seen_head_on(dtype):
    """F = clamp((D - z) |dir| / tau) wherever the point is observed (float64 exactly from the same pixel; float32
    to rounding); points behind the band, behind the camera, outside the image or on a pixel below min_opacity are not
    updated, and W counts the views (integrating the same view twice doubles W and keeps F)"""
    s = _plane_setup(dtype)
    st = T.new_state(len(s["x"]), dtype)
    T.integrate(st, s["x"], s["trunc"], s["pose"], s["K"], s["W"], s["H"], s["dirs"], s["depth"], s["op"], s["rgb"], 0.5,
                dtype)
    x = s["x"].astype(np.float64)
    zc = x[:, 2] + 1.0
    K = s["K"].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        px = K[0, 0] * x[:, 0] / zc + K[0, 2]
        py = K[1, 1] * x[:, 1] / zc + K[1, 2]
    inimg = (zc > 0) & (px >= 0) & (px < s["W"]) & (py >= 0) & (py < s["H"])
    u = np.where(inimg, np.floor(px), 0).astype(np.int64)
    v = np.where(inimg, np.floor(py), 0).astype(np.int64)
    pix = v * s["W"] + u
    dn = np.linalg.norm(s["dirs"].astype(np.float64)[pix], axis=1)
    sdf = (s["D"] - zc) * dn
    tau = s["trunc"]
    lit = inimg & (s["op"][0][pix] >= 0.5)
    obs = lit & (sdf >= -tau)
    # the rule on the boundaries of the band and the image is a comparison of rounded values: keep clear of them
    clear = (np.abs(sdf + tau) > 1e-5) & (np.abs(px - np.round(px)) > 1e-4) & (np.abs(py - np.round(py)) > 1e-4)
    assert obs.sum() > 1000 and (lit & ~obs & clear).sum() > 500 and (~lit & clear).sum() > 1000
    assert np.array_equal((st["weight"] > 0)[clear], obs[clear])
    assert (st["weight"][~obs & clear] == 0).all() and (st["tsdf"][~obs & clear] == 0).all()
    want = np.minimum(1.0, sdf / tau)
    tol = 0 if dtype == np.float64 else 1e-5
    err = np.abs(st["tsdf"][obs & clear].astype(np.float64) - want[obs & clear])
    assert err.max() <= tol + (1e-12 if dtype == np.float64 else 0)
    band = obs & clear & (sdf <= tau)
    assert (st["color_weight"][band] == 1).all() and (st["color_weight"][obs & clear & (sdf > tau + 1e-5)] == 0).all()
    assert np.allclose(st["color"][band], [0.2, 0.4, 0.9], atol=1e-6)
    # a second time: W doubles, F stays (the mean of two equal values)
    F1 = st["tsdf"].copy()
    T.integrate(st, s["x"], s["trunc"], s["pose"], s["K"], s["W"], s["H"], s["dirs"], s["depth"], s["op"], s["rgb"], 0.5,
                dtype)
    assert (st["weight"][obs & clear] == 2).all()
    assert np.array_equal(st["tsdf"][obs & clear], F1[obs & clear])


def test_float32_rule_is_close_to_float64():
    s64, s32 = _plane_setup(np.float64), _plane_setup(np.float32)
    a, b = T.new_state(len(s64["x"]), np.float64), T.new_state(len(s32["x"]), np.float32)
    for s, st, dt in ((s64, a, np.float64), (s32, b, np.float32)):
        T.integrate(st, s["x"], s["trunc"], s["pose"], s["K"], s["W"], s["H"], s["dirs"], s["depth"], s["op"], s["rgb"],
                    0.5, dt)
    both = (a["weight"] > 0) & (b["weight"] > 0)
    assert both.mean() > 0.1 and (a["weight"] != b["weight"]).mean() < 0.01
    assert np.abs(a["tsdf"][both] - b["tsdf"][both]).max() < 1e-5


def test_every_crossed_edge_of_a_case_is_used():
    """the masked rule 'a vertex exists iff a cell around its edge emits' leaves no vertex unreferenced only because
    every crossed edge of a case appears in the case table's triangles"""
    for m, tris in enumerate(TRIS):
        used = {e for t in tris for e in t}
        assert used == T.crossed_edges_of_case(m), m


def _blob(n, seed):
    rng = np.random.RandomState(seed)
    g = np.stack(np.meshgrid(*[np.linspace(-1, 1, k) for k in n], indexing="ij"), -1)
    F = np.ones(n)
    for _ in range(4):
        c, r = rng.uniform(-0.5, 0.5, 3), rng.uniform(0.25, 0.5)
        F = np.minimum(F, (np.linalg.norm(g - c, axis=-1) - r) / 0.3)
    return np.clip(F, -1, 1).astype(np.float32)


def test_masked_marching_cubes_observed_everywhere_is_mcubes_ref():
    n = (19, 23, 17)
    F = _blob(n, 0)
    Wt = np.ones(n, np.int32)
    lo, step = np.float32([-1, -1, -1]), np.float32([0.1, 0.09, 0.12])
    v, t, nr = T.masked_marching_cubes(F, Wt, lo, step, normals=True)
    rv, rt, rn = R.marching_cubes(-F, 0.0, lo, step, normals=True)
    assert len(t) > 200
    assert np.array_equal(v.view(np.int32), rv.view(np.int32)) and np.array_equal(t, rt) and np.array_equal(nr, rn)


def test_masked_marching_cubes_with_holes():
    """no emitted cell has an unobserved corner, every vertex is referenced, every vertex's edge has both ends
    observed and exactly one inside; and colours come from the ends' means"""
    n = (21, 18, 20)
    F = _blob(n, 1)
    rng = np.random.RandomState(3)
    Wt = (rng.rand(*n) > 0.08).astype(np.int32) * rng.randint(1, 5, n).astype(np.int32)
    Wt[5:9, 3:12, :] = 0
    F = np.where(Wt > 0, F, 0).astype(np.float32)
    col = rng.rand(*n, 3).astype(np.float32)
    Wc = np.where((Wt > 0) & (rng.rand(*n) > 0.3) | ((Wt > 0) & (F < 0)), 1, 0).astype(np.int32)
    lo, step = np.float32([0, 0, 0]), np.float32([1, 1, 1])
    v, t, nr, c = T.masked_marching_cubes(F, Wt, lo, step, normals=True, color=col, color_weight=Wc)
    assert len(t) > 100
    assert np.array_equal(np.unique(t), np.arange(len(v)))
    obs = Wt > 0
    # the cell of each triangle: the floor of its centroid in index space lies in the cell (vertices lie on its edges)
    cell = np.floor(v[t].mean(1)).astype(np.int64)
    for c_ in range(8):
        corner = cell + np.array([c_ & 1, (c_ >> 1) & 1, (c_ >> 2) & 1])
        assert obs[tuple(corner.T)].all()
    # fewer triangles than the unmasked mesh of the same values
    _, rt = R.marching_cubes(-F, 0.0, lo, step)
    assert len(t) < len(rt)
    assert c.dtype == np.uint8 and c.shape == v.shape and np.isfinite(nr).all()


def _run(argv=None, code=None):
    cmd = [sys.executable, "-c", code] if code is not None else [sys.executable, "-m", "ngp_pl_b200.export_mesh"] + argv
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)


def test_cli_tsdf_flags_and_defaults_without_torch(tmp_path):
    ck = str(tmp_path / "m.ckpt")
    open(ck, "wb").close()
    code = ("import sys; from ngp_pl_b200 import export_mesh as E\n"
            "a = E.parse_args(['--ckpt_path', %r])\n"
            "print(a.tsdf, a.root_dir, a.dataset_name, a.downsample, a.min_opacity, a.tsdf_trunc)\n"
            "b = E.parse_args(['--ckpt_path', %r, '--tsdf', '--root_dir', %r, '--dataset_name', 'colmap', '--downsample',"
            " '0.25', '--min_opacity', '0.7', '--tsdf_trunc', '0.02', '--resolution', '1024'])\n"
            "print(b.tsdf, b.root_dir == %r, b.dataset_name, b.downsample, b.min_opacity, b.tsdf_trunc, b.resolution)\n"
            "print('torch' in sys.modules)\n" % (ck, ck, str(tmp_path), str(tmp_path)))
    r = _run(None, code)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.splitlines()
    assert lines[0] == "False None nerf 1.0 0.5 None"
    assert lines[1] == "True True colmap 0.25 0.7 0.02 1024"
    assert lines[2] == "False"


def test_cli_tsdf_refusals_exit_2_before_torch(tmp_path):
    ck = str(tmp_path / "m.ckpt")
    open(ck, "wb").close()
    root = str(tmp_path)
    cases = [
        (["--tsdf"], "--root_dir"),
        (["--tsdf", "--root_dir", root, "--dense"], "--dense"),
        (["--tsdf", "--root_dir", root, "--resolution", "1025"], "--resolution"),
        (["--tsdf", "--root_dir", root, "--min_opacity", "0"], "--min_opacity"),
        (["--tsdf", "--root_dir", root, "--min_opacity", "1.5"], "--min_opacity"),
        (["--tsdf", "--root_dir", root, "--min_opacity", "nan"], "--min_opacity"),
        (["--tsdf", "--root_dir", root, "--tsdf_trunc", "0"], "--tsdf_trunc"),
        (["--tsdf", "--root_dir", root, "--tsdf_trunc", "-1"], "--tsdf_trunc"),
        (["--tsdf", "--root_dir", root, "--tsdf_trunc", "inf"], "--tsdf_trunc"),
        (["--tsdf", "--root_dir", root, "--downsample", "0"], "--downsample"),
    ]
    for extra, flag in cases:
        argv = ["--ckpt_path", ck] + extra
        r = _run(argv)
        assert r.returncode == 2 and flag in r.stderr, (argv, r.returncode, r.stderr)
        code = ("import sys; from ngp_pl_b200 import export_mesh\n"
                "try:\n    export_mesh.main(%r)\n"
                "except SystemExit as e:\n    code = e.code\n"
                "print(code, 'torch' in sys.modules)\n" % (argv,))
        r = _run(None, code)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)
