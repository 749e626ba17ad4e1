"""The Gaussian-splat export on an H100 (ngp_pl_b200.splats, csrc/splats.cu) against NGP.forward and the numpy
restatement (oracle/splats_ref.py): colours over directions bitwise, the SH fit, geometry and opacity, the rasteriser on
small random scenes, determinism, the PLY round trip, and on a synthetic Lego trained for 300 steps the preview PSNR
against the model's own render."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import splats_ref as S

pytestmark = pytest.mark.gpu
# mean preview PSNR of the Lego fixture's export against the model's render over 8 views: 21.25 dB measured on an H100
# 80GB HBM3 (700 W), less 1 dB (a second run gave 21.16: the fixture's training is not bitwise reproducible)
PSNR_FLOOR = 20.25


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _random_model(seed=1, n_levels=8):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    scene = synth.lego_scene(0)
    torch.manual_seed(seed)
    model = NGP(scene.scale, n_levels=n_levels, log2_hashmap_size=16).cuda()
    with torch.no_grad():
        model.xyz_encoder.params[3072:].uniform_(-1, 1)
        model.xyz_encoder.params[:3072].normal_(0, 0.2)
        model.rgb_net.params.normal_(0, 0.2)
    return model


@pytest.mark.parametrize("P,D", [(37, 16), (101, 24), (300, 128)])
def test_colors_over_directions_bitwise(P, D):
    from ngp_pl_b200 import splats
    model = _random_model()
    g = torch.Generator().manual_seed(P)
    pts = ((torch.rand(P, 3, generator=g) * 2 - 1) * model.scale * 0.9).cuda()
    dirs = torch.as_tensor(splats.fibonacci_directions(D)).cuda()
    sigma, rgb = splats.colors_over_directions(model, pts, dirs)
    with torch.no_grad():
        sig_ref, rgb_ref = model(pts.repeat_interleave(D, 0), dirs.repeat(P, 1))
    assert _equal(rgb.float().reshape(-1, 3), rgb_ref)
    assert _equal(sigma, sig_ref.reshape(P, D)[:, 0].contiguous())
    assert (rgb.float() == rgb_ref.reshape(P, D, 3)).all()


def _fit_case(P, D, degree, ridge, with_normals):
    from ngp_pl_b200 import splats
    model = _random_model(2)
    g = torch.Generator().manual_seed(7 + degree)
    pts = ((torch.rand(P, 3, generator=g) * 2 - 1) * model.scale * 0.9).cuda()
    nrm = None
    if with_normals:
        n = torch.randn(P, 3, generator=g)
        n = n / n.norm(dim=1, keepdim=True)
        n[::7] = 0  # n = 0: every direction weighs 1
        nrm = n.float().cuda()
    dirs = torch.as_tensor(splats.fibonacci_directions(D)).cuda()
    _, rgb = splats.colors_over_directions(model, pts, dirs)
    out = torch.full((P, 62), float("nan"), device="cuda")
    splats.fit_sh(rgb, dirs, nrm, out, degree, ridge)
    ref = S.fit(rgb.float().cpu().numpy(), dirs.cpu().numpy(), None if nrm is None else nrm.cpu().numpy(), degree, ridge)
    return out.cpu().numpy(), ref


@pytest.mark.parametrize("degree,ridge,with_normals", [(3, 1e-3, True), (3, 1e-3, False), (2, 1e-2, True),
                                                       (1, 0.0, True), (0, 1e-3, True)])
def test_fit_matches_restatement(degree, ridge, with_normals):
    got, ref = _fit_case(200, 128, degree, ridge, with_normals)
    f_dc, f_rest = S.sh_fields(ref)
    want = np.concatenate([f_dc, f_rest], 1)
    have = got[:, S.F_DC:S.F_REST + 45].astype(np.float64)
    scale = np.abs(want).max(1, keepdims=True)
    assert (np.abs(have - want) <= 1e-6 * scale + 1e-30).all(), np.abs(have - want).max()
    nb = (degree + 1) ** 2
    rest = got[:, S.F_REST:S.F_REST + 45].reshape(-1, 3, 15)
    assert (rest[:, :, nb - 1:] == 0).all()
    assert np.isnan(got[:, :S.F_DC]).all() and np.isnan(got[:, S.OPACITY:]).all()  # nothing else is written


def test_rank_deficient_fit_is_zero():
    # ridge 0 and 16 directions: about 8 lie in each normal's hemisphere, too few for 16 coefficients; rounding leaves
    # tiny positive pivots, which must give the all-zero fallback rather than huge coefficients
    from ngp_pl_b200 import splats
    model = _random_model(3)
    g = torch.Generator().manual_seed(3)
    P = 500
    pts = ((torch.rand(P, 3, generator=g) * 2 - 1) * model.scale * 0.9).cuda()
    n = torch.randn(P, 3, generator=g)
    nrm = (n / n.norm(dim=1, keepdim=True)).float().cuda()
    dirs = torch.as_tensor(splats.fibonacci_directions(16)).cuda()
    _, rgb = splats.colors_over_directions(model, pts, dirs)
    out = torch.full((P, 62), float("nan"), device="cuda")
    splats.fit_sh(rgb, dirs, nrm, out, 3, 0.0)
    assert (out[:, S.F_DC:S.OPACITY] == 0).all()
    assert (S.fit(rgb.float().cpu().numpy(), dirs.cpu().numpy(), nrm.cpu().numpy(), 3, 0.0) == 0).all()
    splats.fit_sh(rgb, dirs, nrm, out, 1, 0.0)  # 4 coefficients: solvable, and the restatement's
    got = out[:, S.F_DC:S.OPACITY].cpu().numpy().astype(np.float64)
    f_dc, f_rest = S.sh_fields(S.fit(rgb.float().cpu().numpy(), dirs.cpu().numpy(), nrm.cpu().numpy(), 1, 0.0))
    want = np.concatenate([f_dc, f_rest], 1)
    assert np.abs(want).max() > 0
    assert (np.abs(got - want) <= 1e-6 * np.abs(want).max(1, keepdims=True)).all()


def _ulps(a, b):
    a = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


@pytest.mark.parametrize("shape", ["disc", "sphere"])
def test_geometry_matches_restatement(shape):
    from ngp_pl_b200 import points, splats
    rng = np.random.RandomState(4)
    P = 3000
    p = torch.as_tensor(rng.rand(P, 3).astype(np.float32)).cuda()
    p[5] = p[4]  # a duplicate: distance 0, the scale floor
    n = rng.normal(size=(P, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    n[::11] = 0
    n[1] = [0, 0, 1]
    n[2] = [0, 0, -1]
    n[3] = [0, 0, -0.99999994]
    nrm = torch.as_tensor(n.astype(np.float32)).cuda()
    sigma = torch.as_tensor((rng.rand(P) * 50).astype(np.float32)).cuda()
    sigma[:3] = torch.tensor([0.0, 1e30, float("inf")])
    _, d2 = points.knn(p, 3)
    out = torch.full((P, 62), float("nan"), device="cuda")
    splats.splat_geometry(p, nrm, sigma, d2, out, shape, 0.1)
    got = out.cpu().numpy()
    ref = S.geometry(p.cpu().numpy(), nrm.cpu().numpy(), sigma.cpu().numpy(), d2.cpu().numpy(), shape, 0.1)
    assert np.array_equal(got[:, :6], ref[:, :6].astype(np.float32))
    assert np.array_equal(got[:, S.ROT:S.ROT + 4], ref[:, S.ROT:S.ROT + 4].astype(np.float32))
    for a, b in ((S.SCALE, S.SCALE + 3), (S.OPACITY, S.OPACITY + 1)):
        assert _ulps(got[:, a:b], ref[:, a:b].astype(np.float32)).max() <= 1
    assert np.isnan(got[:, S.F_DC:S.OPACITY]).all()
    if shape == "disc":
        for i in range(P):
            if n[i].any():
                R = S.rotation(got[i, S.ROT:S.ROT + 4].astype(np.float64))
                assert np.abs(R[:, 2] - n[i] / np.linalg.norm(n[i])).max() < 1e-3


def _random_scene(seed, P, W=32, H=24):
    rng = np.random.RandomState(seed)
    g = np.zeros((P, 62), np.float32)
    g[:, 0:2] = rng.uniform(-1.2, 1.2, (P, 2))
    g[:, 2] = rng.uniform(0.1, 4.0, P)  # some behind the near plane
    g[:, S.F_DC:S.F_DC + 3] = rng.normal(0, 1, (P, 3))
    g[:, S.F_REST:S.F_REST + 45] = rng.normal(0, 0.2, (P, 45))
    g[:, S.OPACITY] = rng.normal(0, 2, P)
    g[:, S.SCALE:S.SCALE + 3] = np.log(rng.uniform(0.01, 0.3, (P, 3)))
    q = rng.normal(size=(P, 4))
    g[:, S.ROT:S.ROT + 4] = q
    f = rng.uniform(20, 40)
    K = np.array([[f, 0, W / 2 + rng.uniform(-3, 3)], [0, f * rng.uniform(0.9, 1.1), H / 2 + rng.uniform(-3, 3)],
                  [0, 0, 1]], np.float32)
    a = rng.normal(size=3) * 0.1
    c, s = np.cos(a), np.sin(a)
    R = (np.array([[1, 0, 0], [0, c[0], -s[0]], [0, s[0], c[0]]]) @ np.array([[c[1], 0, s[1]], [0, 1, 0], [-s[1], 0, c[1]]]) @
         np.array([[c[2], -s[2], 0], [s[2], c[2], 0], [0, 0, 1]]))
    pose = np.concatenate([R, rng.normal(0, 0.1, (3, 1))], 1).astype(np.float32)
    bg = rng.rand(3).astype(np.float32)
    return g, pose, K, bg


@pytest.mark.parametrize("seed", range(6))
def test_rasteriser_matches_restatement(seed):
    from ngp_pl_b200 import splats
    W, H = 32, 24
    g, pose, K, bg = _random_scene(seed, 300, W, H)
    rgb, op = splats.render(torch.as_tensor(g).cuda(), pose, K, (W, H), bg)
    ref_rgb, ref_op = S.rasterize(g, pose, K, W, H, bg)
    err = np.abs(rgb.cpu().numpy().reshape(H, W, 3) - ref_rgb)
    assert err.mean() <= 1e-5, err.mean()
    assert (err.max(2) > 1e-3).mean() <= 1e-3
    err_op = np.abs(op.cpu().numpy().reshape(H, W) - ref_op)
    assert err_op.mean() <= 1e-5 and (err_op > 1e-3).mean() <= 1e-3
    assert ref_op.max() > 0.5  # the scene draws something


def test_renderer_graph_reuse_and_growth():
    from ngp_pl_b200 import splats
    W, H = 64, 48
    g, pose, K, bg = _random_scene(11, 2000, W, H)
    sp = torch.as_tensor(g).cuda()
    _, pose2, _, bg2 = _random_scene(12, 1, W, H)
    r = splats.SplatRenderer(sp, (W, H), capacity=1)  # too small: grows on the first view
    a = r.render(pose, K, bg)
    assert r.capacity >= int(r.n_keys.item()) > 1
    b = r.render(pose2, K, bg2)
    a2 = r.render(pose, K, bg)
    fa, fb = splats.render(sp, pose, K, (W, H), bg), splats.render(sp, pose2, K, (W, H), bg2)
    for x, y in ((a, fa), (b, fb), (a2, fa)):
        assert _equal(x[0], y[0]) and _equal(x[1], y[1])
    empty = splats.render(torch.empty(0, 62, device="cuda"), pose, K, (W, H), bg)
    assert torch.equal(empty[1], torch.zeros(H * W, device="cuda"))
    assert torch.equal(empty[0], torch.as_tensor(bg).cuda().expand(H * W, 3))


def test_renderer_grows_past_one_key_per_thread():
    # more splats than k_splat_keys has threads, and a capacity that overflows at the first key: the count must still
    # reach the host, so the renderer grows and renders what a renderer with ample capacity renders
    from ngp_pl_b200 import splats
    W, H, P = 256, 192, 300000
    rng = np.random.RandomState(21)
    g = np.zeros((P, 62), np.float32)
    g[:, 2] = rng.uniform(1.0, 4.0, P)
    g[:, 0] = rng.uniform(-0.6, 0.6, P) * g[:, 2]
    g[:, 1] = rng.uniform(-0.45, 0.45, P) * g[:, 2]
    g[:, S.F_DC:S.F_DC + 3] = rng.normal(0, 1, (P, 3))
    g[:, S.OPACITY] = rng.normal(-2, 1, P)
    g[:, S.SCALE:S.SCALE + 3] = np.log(rng.uniform(0.002, 0.02, (P, 3)))
    g[:, S.ROT:S.ROT + 4] = rng.normal(size=(P, 4))
    K = np.array([[200.0, 0, W / 2], [0, 200.0, H / 2], [0, 0, 1]], np.float32)
    pose = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    sp = torch.as_tensor(g).cuda()
    small = splats.SplatRenderer(sp, (W, H), capacity=1)
    a = small.render(pose, K, (0.2, 0.3, 0.4))
    need = int(small.n_keys.item())
    assert need > P and small.capacity >= need
    big = splats.SplatRenderer(sp, (W, H), capacity=4 * need)
    b = big.render(pose, K, (0.2, 0.3, 0.4))
    assert int(big.n_keys.item()) == need
    assert _equal(a[0], b[0]) and _equal(a[1], b[1])
    assert b[1].max() > 0.5


# ---- the synthetic Lego ----------------------------------------------------------------------------------------------------
def _lego_intrinsics():
    from ngp_pl_b200 import synth
    k = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    return k, np.array([[k["fx"], 0, k["cx"]], [0, k["fy"], k["cy"]], [0, 0, 1]], np.float32)


@pytest.fixture(scope="module")
def lego():
    """the synthetic Lego trained for 300 steps, as test_points_gpu's fixture trains it, and its cameras"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    k, _ = _lego_intrinsics()
    bank = synth.RayBank(scene, n_images=60, K=k, device="cuda")
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
    poses = torch.as_tensor(synth.camera_poses(60, radius=1.5, seed=0, upper_only=False))
    return model, poses, synth.ray_directions(k)


def test_lego_export_end_to_end(lego, tmp_path):
    from ngp_pl_b200 import splats
    model, poses, dirs = lego
    _, K = _lego_intrinsics()
    kw = dict(num_rays=400000)
    a = splats.extract_splats(model, poses, dirs, **kw)
    b = splats.extract_splats(model, poses, dirs, **kw)
    assert a.shape[0] > 10000 and _equal(a, b)
    assert torch.isfinite(a).all()
    path = str(tmp_path / "lego.ply")
    splats.write_splats(path, a)
    with open(path, "rb") as f:
        assert f.read().startswith(splats.ply_header(a.shape[0]))
    back = splats.read_splats(path)
    assert _equal(back, a)
    views = poses[::8]
    psnr3 = splats.preview(model, back, views, K, (200, 200), dirs, save_dir=str(tmp_path / "preview"))
    assert sorted(os.listdir(tmp_path / "preview"))[:2] == ["000.png", "000_model.png"]
    d0 = splats.extract_splats(model, poses, dirs, sh_degree=0, **kw)
    assert _equal(d0[:, :6], a[:, :6]) and _equal(d0[:, S.OPACITY:], a[:, S.OPACITY:])
    psnr0 = splats.preview(model, d0, views, K, (200, 200), dirs)
    sph = splats.extract_splats(model, poses, dirs, shape="sphere", **kw)
    psnr_s = splats.preview(model, sph, views, K, (200, 200), dirs)
    m3, m0, ms = float(np.mean(psnr3)), float(np.mean(psnr0)), float(np.mean(psnr_s))
    report = {"splats": int(a.shape[0]), "psnr_deg3": psnr3, "mean_deg3": m3, "mean_deg0": m0, "mean_sphere": ms}
    print("splats preview:", json.dumps(report))
    assert m3 >= PSNR_FLOOR, report
    # Against the model's composited render the view-dependent terms buy nothing measurable on this 300-step model
    # (21.25 dB at degree 3 and 21.26 at degree 0 in one run, 21.158 and 21.158 in another): degree 3 may not lose more than 0.1 dB ...
    assert m3 >= m0 - 0.1, report
    # ... and it must reproduce the model's colour over the fitted directions better, in the fit's weighted norm
    sub = a[::97]
    dirs_f = splats.fibonacci_directions(128)
    _, rgb = splats.colors_over_directions(model, sub[:, :3].contiguous(), torch.as_tensor(dirs_f).cuda())
    c = rgb.float().cpu().numpy().astype(np.float64)
    Y = S.sh_basis(dirs_f)
    res = []
    for sp in (sub, d0[::97]):
        h = sp.cpu().numpy().astype(np.float64)
        coef = np.concatenate([h[:, S.F_DC:S.F_DC + 3, None], h[:, S.F_REST:S.F_REST + 45].reshape(-1, 3, 15)], 2)
        w = np.stack([S.weights(dirs_f, n) for n in h[:, 3:6]])
        res.append((w[:, :, None] * (np.einsum("pck,dk->pdc", coef, Y) + 0.5 - c) ** 2).sum())
    assert res[0] < res[1], res
