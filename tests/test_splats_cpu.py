"""CPU checks of the Gaussian-splat export's numpy restatement (oracle/splats_ref.py) and host code
(ngp_pl_b200.splats, ngp_pl_b200.export_splats): the SH basis is orthonormal, the fit recovers known coefficients and
ignores back-facing directions, the quaternion takes +z to the normal, the PLY layout is 3DGS's byte for byte, the
brute-force rasteriser reproduces an analytic peak, and the command's refusals (exit status 2, before torch)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import splats_ref as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fib64(n):
    j = np.arange(n, dtype=np.float64)
    z = 1.0 - (2.0 * j + 1.0) / n
    phi = j * (np.pi * (3.0 - np.sqrt(5.0)))
    r = np.sqrt(1.0 - z * z)
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)


def test_sh_basis_is_orthonormal():
    d = _fib64(200000)
    Y = S.sh_basis(d)
    G = Y.T @ Y * (4 * np.pi / d.shape[0])
    assert np.abs(G - np.eye(16)).max() < 1e-4, np.abs(G - np.eye(16)).max()


def test_basis_matches_3dgs_signs():
    # degree 1 is (-C1 y, C1 z, -C1 x), and the host table is the oracle's
    from ngp_pl_b200 import splats
    d = np.array([[0.36, -0.48, 0.8]])
    Y = S.sh_basis(d)[0]
    assert np.allclose(Y[1:4], [-S.C1 * -0.48, S.C1 * 0.8, -S.C1 * 0.36])
    rng = np.random.RandomState(0)
    u = rng.normal(size=(50, 3))
    assert np.array_equal(splats.sh_basis(u), S.sh_basis(u))
    assert np.array_equal(splats.fibonacci_directions(128), S.fibonacci_directions(128))


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_fit_recovers_coefficients(degree):
    rng = np.random.RandomState(degree)
    dirs = S.fibonacci_directions(128)
    nb = (degree + 1) ** 2
    coef = np.zeros((4, 3, 16))
    coef[:, :, :nb] = rng.normal(size=(4, 3, nb)) * 0.3
    colors = np.einsum("pck,dk->pdc", coef, S.sh_basis(dirs)) + 0.5
    got = S.fit(colors, dirs, None, degree, 0.0)
    assert np.abs(got - coef).max() < 1e-9


def test_rank_deficient_fit_is_zero():
    # ridge 0 and 16 directions: about 8 lie in a normal's hemisphere, too few for the 16 degree-3 coefficients
    from ngp_pl_b200 import _lib
    assert S.PIVOT_RTOL == _lib.NGP_SPLAT_PIVOT_RTOL
    rng = np.random.RandomState(5)
    dirs = S.fibonacci_directions(16)
    n = rng.normal(size=(6, 3))
    colors = rng.rand(6, 16, 3)
    assert (S.fit(colors, dirs, n, 3, 0.0) == 0).all()
    assert np.abs(S.fit(colors, dirs, n, 3, 1e-3)).max() > 0  # the ridge makes it solvable
    assert np.abs(S.fit(colors, dirs, n, 1, 0.0)).max() > 0   # and so do fewer coefficients


def test_hemisphere_weights_ignore_back_faces():
    rng = np.random.RandomState(1)
    dirs = S.fibonacci_directions(256)
    n = rng.normal(size=3)
    n /= np.linalg.norm(n)
    w = S.weights(dirs, n)
    dn = dirs.astype(np.float64) @ n
    assert (w[dn >= 0] == 0).all() and (w[dn < 0] > 0).all()
    assert np.array_equal(S.weights(dirs, np.zeros(3)), np.ones(256))
    colors = rng.rand(1, 256, 3)
    spoiled = colors.copy()
    spoiled[0, dn >= 0] = rng.rand(int((dn >= 0).sum()), 3) * 10
    a = S.fit(colors, dirs, n[None], 3, 1e-3)
    b = S.fit(spoiled, dirs, n[None], 3, 1e-3)
    assert np.array_equal(a, b)
    c = S.fit(colors, dirs, None, 3, 1e-3)
    assert not np.allclose(a, c)


def test_quaternion_takes_z_to_the_normal():
    rng = np.random.RandomState(2)
    ns = list(rng.normal(size=(200, 3))) + [np.array([0, 0, 1.0]), np.array([0, 0, -1.0]), np.array([0, 0, 2.5]),
                                            np.array([1e-9, 0, -1.0]), np.array([0, 1.0, 0])]
    for n in ns:
        q = S.quaternion(n)
        assert abs(np.linalg.norm(q) - 1) < 1e-12
        assert np.abs(S.rotation(q) @ [0, 0, 1.0] - n / np.linalg.norm(n)).max() < 1e-7, (n, q)
    assert np.array_equal(S.quaternion([0, 0, 1.0]), [1, 0, 0, 0])
    assert np.array_equal(S.quaternion([0, 0, -1.0]), [0, 1, 0, 0])


def test_geometry_rules():
    pts = np.zeros((3, 3), np.float32)
    nrm = np.array([[0, 0, 1], [0, 0, 0], [1, 0, 0]], np.float32)
    d2 = np.array([[0.01, 0.04, 0.07], [0, 0, 0], [1, 1, 1]])
    out = S.geometry(pts, nrm, np.array([10, 10, 0], np.float32), d2, "disc", 0.1)
    s0 = np.sqrt(0.04)
    assert np.allclose(out[0, S.SCALE:S.SCALE + 3], np.log([s0, s0, 0.1 * s0]))
    assert np.allclose(out[1, S.SCALE:S.SCALE + 3], np.log(np.sqrt(1e-7)))  # floor, and n = 0 falls back to a sphere
    assert np.array_equal(out[1, S.ROT:S.ROT + 4], [1, 0, 0, 0])
    a0 = 1 - np.exp(-10 * 2 * s0)
    assert np.isclose(out[0, S.OPACITY], np.log(a0 / (1 - a0)))
    assert np.isclose(out[2, S.OPACITY], np.log(0.01 / 0.99))  # sigma 0 -> clamped at 0.01
    sph = S.geometry(pts, nrm, np.ones(3, np.float32), d2, "sphere", 0.1)
    assert np.array_equal(sph[:, S.ROT:S.ROT + 4], np.tile([1.0, 0, 0, 0], (3, 1)))


# ---- PLY ---------------------------------------------------------------------------------------------------------------
def _3dgs_attributes():
    # 3DGS's GaussianModel.construct_list_of_attributes with 3 f_dc, 45 f_rest, 3 scales and 4 rotations
    names = ['x', 'y', 'z', 'nx', 'ny', 'nz']
    names += ['f_dc_{}'.format(i) for i in range(3)]
    names += ['f_rest_{}'.format(i) for i in range(45)]
    names.append('opacity')
    names += ['scale_{}'.format(i) for i in range(3)]
    names += ['rot_{}'.format(i) for i in range(4)]
    return names


def test_ply_header_is_3dgs_layout():
    from ngp_pl_b200 import splats
    assert splats.ATTRIBUTES == _3dgs_attributes()
    expect = ("ply\nformat binary_little_endian 1.0\nelement vertex 7\n" +
              "".join("property float %s\n" % a for a in _3dgs_attributes()) + "end_header\n").encode()
    assert splats.ply_header(7) == expect
    assert [S.F_DC, S.F_REST, S.OPACITY, S.SCALE, S.ROT] == [_3dgs_attributes().index(a) for a in
                                                            ("f_dc_0", "f_rest_0", "opacity", "scale_0", "rot_0")]


def test_read_splats_round_trip(tmp_path):
    from ngp_pl_b200 import splats
    rng = np.random.RandomState(3)
    a = rng.normal(size=(11, 62)).astype(np.float32)
    path = str(tmp_path / "s.ply")
    with open(path, "wb") as f:
        f.write(splats.ply_header(11))
        f.write(a.astype("<f4").tobytes())
    b = splats.read_splats(path, device="cpu").numpy()
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    with open(path, "wb") as f:
        f.write(splats.ply_header(11).replace(b"property float rot_3\n", b""))
        f.write(a[:, :61].astype("<f4").tobytes())
    with pytest.raises(ValueError):
        splats.read_splats(path, device="cpu")


# ---- rasteriser oracle ---------------------------------------------------------------------------------------------------
def test_brute_force_rasteriser_peak():
    W, H, f = 32, 24, 30.0
    K = np.array([[f, 0, 16.5], [0, f, 12.5], [0, 0, 1]])  # pixel (16, 12) looks straight down the axis
    pose = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    g = np.zeros(62)
    g[2] = 2.0
    g[S.F_DC:S.F_DC + 3] = [0.5, -0.2, 1.0]
    g[S.SCALE:S.SCALE + 3] = np.log(0.05)
    g[S.ROT] = 1.0
    g[S.OPACITY] = np.log(0.7 / 0.3)
    bg = np.array([0.1, 0.2, 0.3])
    rgb, op = S.rasterize(g[None], pose, K, W, H, bg)
    c = np.maximum(S.C0 * g[S.F_DC:S.F_DC + 3] + 0.5, 0)
    assert np.allclose(rgb[12, 16], 0.7 * c + 0.3 * bg)
    assert np.isclose(op[12, 16], 0.7)
    # one pixel off: the 2D variance is (f s / z)^2 + 0.3
    var = (f * 0.05 / 2.0) ** 2 + 0.3
    assert np.isclose(op[12, 17], 0.7 * np.exp(-0.5 / var))
    assert op.argmax() == 12 * W + 16
    # behind the near plane nothing is drawn
    g2 = g.copy()
    g2[2] = 0.2
    rgb2, op2 = S.rasterize(g2[None], pose, K, W, H, bg)
    assert (op2 == 0).all() and np.allclose(rgb2, bg)


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def _run(argv=None, code=None):
    cmd = [sys.executable, "-c", code] if code is not None else [sys.executable, "-m", "ngp_pl_b200.export_splats"] + argv
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)


def test_defaults_parse_without_torch():
    code = ("import sys; from ngp_pl_b200 import export_splats as E\n"
            "a = E.parse_args(['--ckpt_path', %r])\n"
            "print(a.scale, a.root_dir, a.dataset_name, a.downsample, a.num_rays, a.min_opacity, a.bounds, a.voxel,"
            " a.nb_neighbors, a.std_ratio, a.keep_outliers, a.no_normals, a.out)\n"
            "print(a.sh_degree, a.directions, a.shape, a.flatness, a.ridge, a.preview)\n"
            "print('torch' in sys.modules)\n" % (__file__,))
    r = _run(None, code)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.splitlines()
    assert lines[0] == "0.5 None nerf 1.0 1000000 0.5 None None 20 2.0 False False splats.ply"
    assert lines[1] == "3 128 disc 0.1 0.001 None"
    assert lines[2] == "False"


def _refused(tmp):
    ok = os.path.join(tmp, "m.ckpt")
    return [
        ([], "--ckpt_path"),
        (["--ckpt_path", os.path.join(tmp, "missing.ckpt")], "--ckpt_path"),
        (["--ckpt_path", ok, "--scale", "0"], "--scale"),
        (["--ckpt_path", ok, "--num_rays", "0"], "--num_rays"),
        (["--ckpt_path", ok, "--min_opacity", "1.5"], "--min_opacity"),
        (["--ckpt_path", ok, "--nb_neighbors", "65"], "--nb_neighbors"),
        (["--ckpt_path", ok, "--dataset_name", "nsvf"], "--dataset_name"),
        (["--ckpt_path", ok, "--dataset_name", "rtmv"], "--dataset_name"),
        (["--ckpt_path", ok, "--sh_degree", "4"], "--sh_degree"),
        (["--ckpt_path", ok, "--sh_degree", "-1"], "--sh_degree"),
        (["--ckpt_path", ok, "--directions", "15"], "--directions"),
        (["--ckpt_path", ok, "--directions", "1025"], "--directions"),
        (["--ckpt_path", ok, "--shape", "ellipsoid"], "--shape"),
        (["--ckpt_path", ok, "--flatness", "0"], "--flatness"),
        (["--ckpt_path", ok, "--flatness", "inf"], "--flatness"),
        (["--ckpt_path", ok, "--ridge", "-1e-3"], "--ridge"),
        (["--ckpt_path", ok, "--ridge", "nan"], "--ridge"),
        (["--ckpt_path", ok, "--preview", tmp], "--preview"),
    ]


def test_refusals_exit_2_before_torch(tmp_path):
    tmp = str(tmp_path)
    open(os.path.join(tmp, "m.ckpt"), "wb").close()
    for argv, flag in _refused(tmp):
        r = _run(argv)
        assert r.returncode == 2, (argv, r.returncode, r.stderr)
        assert flag in r.stderr, (argv, r.stderr)
        code = ("import sys; from ngp_pl_b200 import export_splats\n"
                "try:\n    export_splats.main(%r)\n"
                "except SystemExit as e:\n    code = e.code\n"
                "print(code, 'torch' in sys.modules)\n" % (argv,))
        r = _run(None, code)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)
