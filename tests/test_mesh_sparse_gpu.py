"""Sparse mesh extraction on the device (ngp_mesh_brick_mask, ngp_density_bricks, ngp_mesh_sparse_* in csrc/mesh.cu and
csrc/network.cu): the brick mask bit for bit against oracle/mesh_bricks.py, σ on bricks bitwise against the lattice,
and extract_mesh_sparse bitwise against the dense marching cubes of σ_masked -- built here from density_volume and
occupied_bricks -- on random weights and on a briefly trained Lego, plus the memory bound and the command line."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mesh_bricks as MB
from test_mesh_cpu import read_ply
from test_mesh_sparse_cpu import CASES as MASK_CASES, cascades_of, lattice as np_lattice, random_bitfield

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_model(scale, seed, bitfield=None):
    from ngp_pl_b200.models.networks import NGP
    model = NGP(scale).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        p = model.xyz_encoder.params
        p[:3072] = ((torch.rand(3072, generator=g) * 2 - 1) * 0.4).cuda()
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * 0.5).cuda()
        if bitfield is not None:
            model.density_bitfield.copy_(torch.as_tensor(bitfield))
    return model


def _lego_bits():
    from ngp_pl_b200 import synth
    scene = synth.lego_scene(0)
    return scene, synth.pack_bits(synth.occupancy_grid(scene))


@pytest.fixture(scope="module")
def lego():
    """the synthetic Lego trained for 300 steps"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=60, K=K, device="cuda")
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
    return model


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _oracle_mask(model, res, bounds):
    from ngp_pl_b200 import mesh
    lo, hi = bounds if bounds is not None else (model._xyz_min_host, model._xyz_max_host)
    lat = mesh.lattice(res, lo, hi)
    return MB.brick_mask(model.density_bitfield.cpu().numpy(), model.cascades, model.grid_size, model.scale,
                         list(lat.n), np.float32(list(lat.lo)), np.float32(list(lat.step)))


@pytest.mark.parametrize("case", range(len(MASK_CASES)))
def test_brick_mask_equals_oracle(case):
    from ngp_pl_b200 import mesh
    scale, G, n, bounds, dens = MASK_CASES[case]
    if G != 128:  # the model's grid is 128^3: the mask cases at G = 32 run as 128 with the same density
        G = 128
    model = _random_model(scale, case, random_bitfield(cascades_of(scale), G, dens / 8, case))
    got = mesh.occupied_bricks(model, n, bounds)
    assert got.is_cuda and got.dtype == torch.bool
    assert np.array_equal(got.cpu().numpy(), _oracle_mask(model, n, bounds))


def test_brick_mask_of_a_trained_bitfield(lego):
    from ngp_pl_b200 import mesh
    for res, bounds in ((256, None), ((200, 256, 160), None), (129, ((-0.3, -0.5, -0.2), (0.6, 0.4, 0.45)))):
        got = mesh.occupied_bricks(lego, res, bounds).cpu().numpy()
        ref = _oracle_mask(lego, res, bounds)
        assert np.array_equal(got, ref) and 0 < ref.mean() < 1


def _masked_sigma(model, res, bounds):
    from ngp_pl_b200 import mesh
    sig = mesh.density_volume(model, res, bounds)
    m = mesh.occupied_bricks(model, res, bounds)
    B = 8
    full = m.repeat_interleave(B, 0).repeat_interleave(B, 1).repeat_interleave(B, 2)[:sig.shape[0], :sig.shape[1], :sig.shape[2]]
    return torch.where(full, sig, torch.zeros_like(sig)), sig, m


def test_sigma_on_bricks_equals_density_volume():
    from ngp_pl_b200 import _lib, mesh
    from ngp_pl_b200.models.networks import _net_struct
    scene, bits = _lego_bits()
    model = _random_model(scene.scale, 2, bits)
    res = (70, 45, 61)
    lat = mesh.lattice(res, model._xyz_min_host, model._xyz_max_host)
    sig = mesh.density_volume(model, res)
    nb = [(v + 7) // 8 for v in res]
    bricks = torch.tensor([0, 5, nb[1] * nb[2] + 3, nb[0] * nb[1] * nb[2] - 1, 17], dtype=torch.int32, device="cuda")
    net, keep = _net_struct(model)
    for apron in (0, 1):
        W = 9 + 2 * apron
        out = torch.full((bricks.numel() * W ** 3,), 7.0, device="cuda")
        _lib.check(_lib.lib().ngp_density_bricks(C.byref(net), C.byref(lat), bricks.data_ptr(), bricks.numel(), apron, None,
                                                 out.data_ptr(), torch.cuda.current_stream().cuda_stream), "bricks")
        out = out.view(-1, W, W, W).cpu()
        s = sig.cpu()
        for q, b in enumerate(bricks.tolist()):
            o = [b // (nb[1] * nb[2]) * 8 - apron, (b // nb[2]) % nb[1] * 8 - apron, b % nb[2] * 8 - apron]
            ref = torch.zeros(W, W, W)
            src = [slice(max(o[a], 0), min(o[a] + W, res[a])) for a in range(3)]
            dst = [slice(src[a].start - o[a], src[a].stop - o[a]) for a in range(3)]
            ref[dst[0], dst[1], dst[2]] = s[src[0], src[1], src[2]]
            assert torch.equal(out[q].view(torch.int32), ref.view(torch.int32))


def _level(model):
    """a σ level random weights cross: the 70th percentile of σ on a coarse lattice (σ > 0 everywhere)"""
    from ngp_pl_b200 import mesh
    return float(torch.quantile(mesh.density_volume(model, 48).flatten(), 0.7))


def _check_sparse(model, res, bounds, colors=True, thr=20.0):
    from ngp_pl_b200 import mesh
    sm, _, m = _masked_sigma(model, res, bounds)
    lo, hi = bounds if bounds is not None else (model._xyz_min_host, model._xyz_max_host)
    lat = mesh.lattice(res, lo, hi)
    V, F, N = mesh.marching_cubes(sm, thr, list(lat.lo), list(lat.step), normals=True)
    got, st = mesh.extract_mesh_sparse(model, res, bounds, thr, normals=True, colors=colors, return_stats=True)
    assert _equal(got["vertices"], V) and _equal(got["triangles"], F) and _equal(got["normals"], N)
    if colors:
        ref = mesh._vertex_colors(model, V, N)
        assert _equal(got["colors"], ref)
    assert st["active"] == int(m.sum()) and st["active"] <= st["visited"] and st["surface"] <= st["visited"]
    return got, st


@pytest.mark.parametrize("res,bounds", [
    (64, None), (129, None), (256, None), ((200, 256, 160), None),
    (129, ((-0.45, -0.3, -0.2), (0.3, 0.6, 0.55))),
])
def test_sparse_equals_dense_on_masked_sigma_trained(lego, res, bounds):
    got, st = _check_sparse(lego, res, bounds)
    assert got["vertices"].shape[0] > 0


def test_sparse_equals_dense_at_512(lego):
    got, st = _check_sparse(lego, 512, None, colors=False)
    print("512^3 trained: %d vertices, bricks %s" % (got["vertices"].shape[0], st))


@pytest.mark.parametrize("scale,res,bounds", [
    (0.5, 64, None), (0.5, (200, 256, 160), ((-0.6, -0.5, -0.55), (0.5, 0.7, 0.5))), (16.0, 129, None),
])
def test_sparse_equals_dense_on_masked_sigma_random(scale, res, bounds):
    from ngp_pl_b200 import synth
    if scale == 0.5:
        _, bits = _lego_bits()
    else:
        bits = synth.pack_bits(synth.occupancy_grid(synth.mip360_scene(0)))
    model = _random_model(scale, 4, bits)
    got, st = _check_sparse(model, res, bounds, thr=_level(model))
    assert got["vertices"].shape[0] > 0


def test_all_ones_is_extract_mesh_and_all_zeros_is_empty():
    from ngp_pl_b200 import mesh
    model = _random_model(0.5, 6)
    model.density_bitfield.fill_(255)
    thr = _level(model)
    for res in (64, (40, 33, 71)):
        d = mesh.extract_mesh(model, res, threshold=thr, colors=True)
        s = mesh.extract_mesh_sparse(model, res, threshold=thr, colors=True)
        assert d.keys() == s.keys()
        for k in d:
            assert _equal(d[k], s[k]), k
        assert d["vertices"].shape[0] > 0
    model.density_bitfield.zero_()
    s, st = mesh.extract_mesh_sparse(model, 96, colors=True, return_stats=True)
    assert s["vertices"].shape == (0, 3) and s["triangles"].shape == (0, 3) and s["colors"].shape == (0, 3)
    assert st == {"active": 0, "visited": 0, "surface": 0}


def test_two_calls_bitwise_equal_and_refusals(lego):
    from ngp_pl_b200 import mesh
    a = mesh.extract_mesh_sparse(lego, 200, colors=True)
    b = mesh.extract_mesh_sparse(lego, 200, colors=True)
    for k in a:
        assert _equal(a[k], b[k]), k
    for thr in (0.0, -1.0, float("nan")):
        with pytest.raises(RuntimeError, match="threshold"):
            mesh.extract_mesh_sparse(lego, 64, threshold=thr)
    with pytest.raises(RuntimeError, match="8192"):
        mesh.extract_mesh_sparse(lego, (8193, 8, 8))
    cpu = _random_model(0.5, 1).cpu()
    with pytest.raises(RuntimeError, match="CUDA"):
        mesh.extract_mesh_sparse(cpu, 64)
    with pytest.raises(RuntimeError, match="CUDA"):
        mesh.occupied_bricks(cpu, 64)


def test_memory_at_1024_and_2048(lego):
    from ngp_pl_b200 import mesh
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m, st = mesh.extract_mesh_sparse(lego, 1024, return_stats=True)
    peak = torch.cuda.max_memory_allocated() - base
    print("1024^3: peak %.3f GB, %d vertices, bricks %s" % (peak / 1e9, m["vertices"].shape[0], st))
    assert peak < 1024 ** 3 * 4
    del m
    m, st = mesh.extract_mesh_sparse(lego, 2048, normals=False, return_stats=True)
    print("2048^3: %d vertices, bricks %s" % (m["vertices"].shape[0], st))
    assert m["vertices"].shape[0] > 0


def test_export_mesh_command_equals_write_ply(lego, tmp_path):
    from ngp_pl_b200 import mesh, train
    ck = train.checkpoint(lego, torch.zeros(4, 3), torch.zeros(2, 3, 4), 0, 300)
    for name, obj in (("full.ckpt", ck), ("slim.ckpt", train.slim_state_dict(ck))):
        path = str(tmp_path / name)
        torch.save(obj, path)
        out = str(tmp_path / (name + ".ply"))
        env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.export_mesh", "--ckpt_path", path, "--resolution", "160",
                            "--colors", "--out", out], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        assert "vertices" in r.stdout
        ref = str(tmp_path / (name + ".ref.ply"))
        mesh.write_ply(ref, **mesh.extract_mesh_sparse(lego, 160, colors=True))
        assert open(out, "rb").read() == open(ref, "rb").read()
        assert read_ply(out)["vertex"].shape[0] > 0
    bad = str(tmp_path / "full.ckpt")
    r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.export_mesh", "--ckpt_path", bad, "--scale", "16", "--out",
                        str(tmp_path / "x.ply")], cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT), stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode != 0 and "does not fit NGP(scale=16)" in r.stderr
