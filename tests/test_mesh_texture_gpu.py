"""Texture baking on the device (ngp_mesh_texture_atlas / _texels / _bake in csrc/texture.cu, mesh.bake_texture,
mesh.write_obj) against oracle/mesh_texture.py, on meshes of a random-weight model and of a briefly trained Lego (raw,
simplified, and one of more than 4 M triangles at W = 8192): squares bitwise, S, uv within 1 fp32 ulp, the texel map's
(texel, triangle) pairs, points and normals within their rounding, colours against a float64 composite of the model at
the kernel's own sample points, the offset-0 texture bitwise the model's colour, zero texels outside the band,
determinism, the PNG, `export_mesh --texture` and the refusals."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mesh_texture as MT
from test_mesh_sparse_gpu import _level, _random_model, lego  # noqa: F401  (lego: module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ULP = 2.0 ** -23


def _host(m):
    return {k: (None if v is None else v.cpu().numpy()) for k, v in m.items()}


def _sub(m, F):
    return dict(m, triangles=m["triangles"][:F].contiguous())


@torch.no_grad()
def _model_colors(model, x, d, chunk=1 << 22):
    """σ, c of NGP.forward at materialised points x (n, 3) with directions d (n, 3), float32 on the host"""
    sig, rgb = [], []
    for i in range(0, x.shape[0], chunk):
        s, c = model(torch.as_tensor(x[i:i + chunk]).cuda(), torch.as_tensor(d[i:i + chunk]).cuda())
        sig.append(s.float().cpu().numpy())
        rgb.append(c.float().cpu().numpy())
    return np.concatenate(sig), np.concatenate(rgb)


def _check(model, m, W, r, K, sample=None, seed=0):
    """bake_texture against the oracle; returns the bake and the counts that were excluded near a boundary"""
    from ngp_pl_b200 import mesh
    got = mesh.bake_texture(model, m, W, r, K, return_texels=True)
    h = _host(m)
    v, t, nrm = h["vertices"], h["triangles"], h["normals"]
    F = t.shape[0]
    at = MT.atlas(v, t, W)
    g = _host(got)
    assert np.array_equal(g["squares"], at["squares"])
    if F and (at["k"] == 0).any():
        assert g["squares"][:, 2].max() == max(at["S"], MT.S_MIN)
    du = np.abs(g["uv"].astype(np.float64) - at["uv"].astype(np.float64))
    assert (du <= np.spacing(np.abs(at["uv"])).astype(np.float64)).all(), du.max()
    # texel map: (texel, triangle) pairs; a decision within 1e-5 texel of changing may differ
    m_ref, t_ref = MT.band(at["uv"], at["squares"], W)
    pairs = set(zip(g["texel"].tolist(), g["triangle"].tolist())) if F < 2_000_000 else None
    if pairs is not None:
        diff = pairs ^ set(zip(m_ref.tolist(), t_ref.tolist()))
        n_diff = len(diff)
    else:
        same = g["texel"].shape == m_ref.shape and np.array_equal(g["texel"], m_ref) and np.array_equal(g["triangle"], t_ref)
        n_diff = 0 if same else np.setxor1d(g["texel"] * F + g["triangle"], m_ref * F + t_ref).size
    n = g["texel"].shape[0]
    sample = min(sample or n, (1 << 24) // (K + 1))  # host memory of the float64 composite
    print("W %d, F %d: S %d, %d texels, %d pairs differ from the oracle" % (W, F, g["squares"][:, 2].max(initial=0), n,
                                                                           n_diff))
    assert n_diff <= 1e-4 * max(n, 1), n_diff
    assert (np.diff(g["texel"]) > 0).all()
    # points and normals of the device's own map, on a subset for the largest meshes
    idx = np.arange(n) if n <= sample else np.sort(
        np.random.default_rng(seed).choice(n, sample, replace=False))
    p, nn, _ = MT.surface(v, t, nrm, at["rot"], g["uv"], g["texel"][idx], g["triangle"][idx], W)
    gp, gn = g["point"][idx], g["normal"][idx]
    corner = np.abs(v[t[g["triangle"][idx]]]).max(1)  # the point is a convex combination of its corners
    assert (np.abs(gp - p) <= 2 * ULP * corner + 1e-30).all(), np.abs(gp - p).max()
    assert (np.abs(gn - nn) <= 4 * ULP).all(), np.abs(gn - nn).max()
    # colours: a float64 composite of the model at the sample points restated bitwise from the kernel's map
    o, d, tj, delta, x = MT.sample_geometry(gp, gn, r, K)
    dirs = np.repeat(d[:, None], K + 1, 1).reshape(-1, 3)
    sig, rgb = _model_colors(model, x.reshape(-1, 3), dirs)
    C = MT.composite(sig.reshape(-1, K + 1), rgb.reshape(-1, K + 1, 3), delta)
    ref = MT.quantise(C)
    xs, ys = MT.deinterleave(g["texel"][idx])
    tex = g["texture"][W - 1 - ys, xs]
    off = tex != ref
    # the device composites in double with CUDA's exp: within 1e-9 of 255 C64, so only a value that close to a rounding
    # boundary may round the other way
    v255 = 255.0 * C
    near = np.abs(v255 - np.floor(v255) - 0.5) < 1e-9
    assert not (off & ~near).any(), (int((off & ~near).sum()), v255[off & ~near][:5], tex[off & ~near][:5])
    assert off.sum() <= 1e-3 * off.size
    # every texel outside the band is exactly 0
    mask = np.zeros((W, W), bool)
    X, Y = MT.deinterleave(g["texel"])
    mask[W - 1 - Y, X] = True
    assert not g["texture"][~mask].any()
    return got, n_diff, int(off.sum())


@pytest.fixture(scope="module")
def random_mesh():
    from ngp_pl_b200 import mesh
    from test_mesh_sparse_gpu import _lego_bits
    _, bits = _lego_bits()
    model = _random_model(0.5, 4, bits)
    return model, mesh.extract_mesh(model, 128, threshold=_level(model), normals=True)


@pytest.mark.parametrize("F,W,r,K", [(16, 16, 0.01, 16), (256, 64, 0.02, 4), (4000, 256, 0.0, 1), (200000, 2048, 0.008, 16),
                                     (1000000, 4096, 0.03, 33)])
def test_random_weights_dense_mesh(random_mesh, F, W, r, K):
    model, m = random_mesh
    assert m["triangles"].shape[0] >= F
    _check(model, _sub(m, F), W, r, K, sample=1 << 20)


@pytest.fixture(scope="module")
def lego_meshes(lego):  # noqa: F811
    from ngp_pl_b200 import mesh
    raw = mesh.extract_mesh_sparse(lego, 256, normals=True)
    box = (lego._xyz_min_host, lego._xyz_max_host)
    return {"raw": raw, "s64": mesh.simplify_mesh(raw, 64, box), "s128": mesh.simplify_mesh(raw, 128, box)}


@pytest.mark.parametrize("name,W,r,K", [("s64", 1024, 1.0 / 64, 16), ("s64", 8192, 0.0, 16), ("s128", 2048, 1.0 / 128, 16),
                                        ("s128", 4096, 1.0 / 128, 256), ("raw", 4096, 1.0 / 256, 16)])
def test_trained_lego_meshes(lego, lego_meshes, name, W, r, K):  # noqa: F811
    m = lego_meshes[name]
    assert m["triangles"].shape[0] * 16 <= W * W
    _check(lego, m, W, r, K, sample=1 << 20)


def test_trained_lego_above_4M_triangles_at_8192(lego):  # noqa: F811
    from ngp_pl_b200 import mesh
    F = 4_100_000
    m = mesh.extract_mesh_sparse(lego, 640, normals=True)
    assert m["triangles"].shape[0] >= F, m["triangles"].shape[0]
    m = _sub(m, F)
    got, n_diff, n_off = _check(lego, m, 8192, 1.0 / 640, 16, sample=1 << 20)
    assert (got["squares"][:, 2] == 4).float().mean() > 0.9
    torch.cuda.empty_cache()


def test_offset_0_is_the_model_colour_and_two_calls_equal(lego, lego_meshes):  # noqa: F811
    from ngp_pl_b200 import mesh
    m = lego_meshes["s128"]
    a = mesh.bake_texture(lego, m, 4096, 0.0, 8, return_texels=True)
    with torch.no_grad():
        _, c = lego(a["point"], -a["normal"])
    ref = (c.float() * 255).round().clamp(0, 255).to(torch.uint8)
    W = 4096
    xs, ys = (torch.as_tensor(z, device="cuda") for z in MT.deinterleave(a["texel"].cpu().numpy()))
    assert torch.equal(a["texture"][W - 1 - ys, xs], ref)
    b = mesh.bake_texture(lego, m, 4096, 1.0 / 128, 16, return_texels=True)
    b2 = mesh.bake_texture(lego, m, 4096, 1.0 / 128, 16, return_texels=True)
    for k in b:
        x, y = b[k], b2[k]
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y), k


def test_png_of_write_obj_decodes_to_the_texture(lego, lego_meshes, tmp_path):  # noqa: F811
    from PIL import Image
    from ngp_pl_b200 import mesh
    m = lego_meshes["s64"]
    tex = mesh.bake_texture(lego, m, 1024, 1.0 / 64, 16)
    for mode in ("dynamic", "fixed"):
        p = str(tmp_path / ("m_%s.obj" % mode))
        mesh.write_obj(p, m["vertices"], m["triangles"], m["normals"], tex["uv"], tex["texture"], png_mode=mode)
        img = np.asarray(Image.open(io.BytesIO(open(p[:-4] + ".png", "rb").read())).convert("RGB"))
        assert np.array_equal(img, tex["texture"].cpu().numpy())
        assert "map_Kd m_%s.png" % mode in open(p[:-4] + ".mtl").read()


def test_empty_mesh(lego):  # noqa: F811
    from ngp_pl_b200 import mesh
    e = mesh.bake_texture(lego, {"vertices": torch.zeros(0, 3, device="cuda"),
                                 "triangles": torch.zeros(0, 3, dtype=torch.int64, device="cuda"), "normals": None}, 16)
    assert e["uv"].shape == (0, 3, 2) and e["squares"].shape == (0, 3) and not e["texture"].any()


def test_refusals(lego, lego_meshes, monkeypatch):  # noqa: F811
    from ngp_pl_b200 import _lib, mesh
    m = lego_meshes["s64"]
    F = m["triangles"].shape[0]
    cpu = {k: (None if v is None else v.cpu()) for k, v in m.items()}
    with pytest.raises(RuntimeError, match="CUDA"):
        mesh.bake_texture(lego, cpu, 1024)
    for W in (8, 15, 100, 32768, 2.0, True):
        with pytest.raises(RuntimeError, match="power of two"):
            mesh.bake_texture(lego, m, W)
    small = mesh.texture_size_for(F) // 2
    with pytest.raises(RuntimeError, match="size >= %d" % (2 * small)):
        mesh.bake_texture(lego, m, small)
    for r in (-1e-3, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="offset"):
            mesh.bake_texture(lego, m, 1024, r)
    for K in (0, 257, 1.5):
        with pytest.raises(RuntimeError, match="samples"):
            mesh.bake_texture(lego, m, 1024, 0.0, K)
    bad = dict(m, triangles=m["triangles"].clone())
    bad["triangles"][5, 1] = m["vertices"].shape[0]
    with pytest.raises(RuntimeError, match="invalid argument"):
        mesh.bake_texture(lego, bad, 1024)
    L = _lib.lib()
    assert L.ngp_mesh_texture_workspace(3, 1, 24) == 0 and L.ngp_mesh_texture_workspace(3, 17, 16) == 0
    assert L.ngp_mesh_texture_workspace(3, 16, 16) > 0 and L.ngp_mesh_texture_bake_workspace(257) == 0
    monkeypatch.setattr(mesh, "_free_bytes", lambda dev: 1000)
    before = torch.cuda.memory_allocated()
    with pytest.raises(RuntimeError, match="bake_texture: the atlas .* device memory"):
        mesh.bake_texture(lego, m, 1024)
    assert torch.cuda.memory_allocated() == before


def test_export_mesh_texture_equals_write_obj(lego, tmp_path):  # noqa: F811
    from ngp_pl_b200 import mesh, train
    ck = train.checkpoint(lego, torch.zeros(4, 3), torch.zeros(2, 3, 4), 0, 300)
    path = str(tmp_path / "slim.ckpt")
    torch.save(train.slim_state_dict(ck), path)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    out = str(tmp_path / "out" / "t.obj")
    os.makedirs(os.path.dirname(out))
    r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.export_mesh", "--ckpt_path", path, "--resolution", "200",
                        "--simplify", "48", "--texture", "1024", "--out", out], cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "baked a 1024^2 atlas (S = " in r.stdout, r.stdout
    box = (lego._xyz_min_host, lego._xyz_max_host)
    m = mesh.simplify_mesh(mesh.extract_mesh_sparse(lego, 200), 48, box)
    h = float(mesh.cluster_grid(box[0], box[1], 48).h)
    tex = mesh.bake_texture(lego, m, 1024, h, 16)
    ref = str(tmp_path / "ref" / "t.obj")
    os.makedirs(os.path.dirname(ref))
    mesh.write_obj(ref, m["vertices"], m["triangles"], m["normals"], tex["uv"], tex["texture"])
    for ext in (".obj", ".mtl", ".png"):
        assert open(out[:-4] + ext, "rb").read() == open(ref[:-4] + ext, "rb").read(), ext
