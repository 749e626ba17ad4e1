"""End-to-end: ngp_pl_b200's render()/NGP against the UNMODIFIED reference render()/NGP
(oracle/_ref/ngp_pl, driven by the reference's compiled vren + the tinycudann stand-in) on identical
rays, identical weights, identical start jitter (same torch seed -> same torch.rand_like draw).
The reference's results are stored under tests/golden/ (make_golden_render.py).

  marcher        : rm_samples and per-ray sample counts identical
  rgb/depth/opac : the network part is only pinned to fp16 level (tinycudann is absent), so the
                   rendered values agree to ~1e-3 absolute; given IDENTICAL sigmas/rgbs the compositor
                   agrees to 1e-4 relative (tests/test_vren_gpu.py).
"""
import os

import numpy as np
import pytest
import torch

import cases

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def make_model(scene):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    mine = NGP(scene.scale).cuda()
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        p = mine.xyz_encoder.params
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * 0.3).cuda()
        mine.density_bitfield.copy_(torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda())
    return mine


def check_grads(model, g, rel):
    """this build's gradients against the stored ones (make_golden_render.grads_of): both MLPs whole, the hash table at
    its largest and at sampled nonzero entries, each within rel of the stored vector's max |g|, and that max itself"""
    ge = model.xyz_encoder.params.grad.float().cpu().numpy()
    gr = model.rgb_net.params.grad.float().cpu().numpy()
    for what, mine, ref, key in (("density MLP", ge[:3072], g["g_density_mlp"], "g_enc"), ("hash table", ge[g["g_table_idx"]], g["g_table"], "g_enc"),
                                 ("rgb MLP", gr, g["g_rgb"], "g_rgb")):
        s = float(g[key + "_absmax"])
        assert s > 0
        err = np.abs(mine - ref).max()
        assert err < rel * s, "%s grad: %g vs scale %g" % (what, err, s)
    for name, mine in (("g_enc", ge), ("g_rgb", gr)):
        s = float(g[name + "_absmax"])
        assert abs(np.abs(mine).max() - s) < rel * s, "%s: max |g| %g vs the reference's %g" % (name, np.abs(mine).max(), s)


def _rays(scene, n, seed):
    o, d = cases.rays_from_scene(scene, n, seed, extra_edge_cases=False)
    return torch.as_tensor(o).cuda(), torch.as_tensor(d).cuda()


@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_train_render_matches_reference(which):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.losses import NeRFLoss
    from ngp_pl_b200.models.rendering import render
    g = gold("render_train_" + which)
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    mine = make_model(scene)
    o, d = _rays(scene, 2048, 31)
    kw = {} if scene.exp_step_factor == 0 else {"exp_step_factor": scene.exp_step_factor}
    torch.manual_seed(123)
    r_my = render(mine, o, d, **kw)
    assert int(g["rm_samples"]) == int(r_my["rm_samples"]) > 0
    assert (g["counts"] == r_my["rays_a"][:, 2].cpu().numpy()).all()
    for k in ("rgb", "opacity", "depth"):
        err = np.abs(g[k] - r_my[k].detach().float().cpu().numpy()).max()
        assert err < 5e-3 * max(1.0, np.abs(g[k]).max()), "%s differs by %g" % (k, err)
    for k in g["keys"]:
        assert k in r_my, "missing result key " + k

    # gradients of the reference's loss (NeRFLoss, no distortion) through both pipelines
    tgt = torch.as_tensor(cases.target_rgb(o.shape[0], 31)).cuda()
    mine.zero_grad()
    l = NeRFLoss(lambda_distortion=0)(r_my, {"rgb": tgt})
    sum(v.mean() for v in l.values()).backward()
    check_grads(mine, g, 0.06)


def test_test_render_matches_reference():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    g = gold("render_test")
    scene = synth.lego_scene(0)
    mine = make_model(scene)
    K = synth.intrinsics(W=100, H=100, fx=1111.11 / 8)
    dirs = synth.ray_directions(K, "cuda")
    pose = torch.as_tensor(synth.camera_poses(3)[2]).cuda()
    o, d = synth.get_rays(dirs, pose)
    r_my = render(mine, o, d, test_time=True)
    px = cases.sample_idx(o.shape[0], g["rgb"].shape[0])
    for k in ("rgb", "opacity", "depth"):
        err = np.abs(g[k] - r_my[k].detach().float().cpu().numpy()[px])
        assert err.max() < 2e-2 and err.mean() < 1e-3, "%s differs: max %g mean %g" % (k, err.max(), err.mean())
    # a ray's early termination can flip on an fp16-level sigma difference; totals must be close
    a, b = int(g["total_samples"]), int(r_my["total_samples"])
    assert abs(a - b) <= 0.01 * a + 8


def test_losses_match_reference():
    """NeRFLoss incl. the distortion term: this project's module against the reference's losses.py on the stored first 32
    rays of a render"""
    from ngp_pl_b200.losses import NeRFLoss
    g = gold("losses")
    res = {}
    for k in ("rgb", "opacity", "ws", "deltas", "ts", "rays_a"):
        v = torch.as_tensor(g["in_" + k]).cuda()
        res[k] = v.requires_grad_(True) if k in ("rgb", "opacity", "ws") else v
    tgt = torch.as_tensor(cases.target_rgb(res["rgb"].shape[0], 32)).cuda()
    l_my = NeRFLoss(lambda_distortion=1e-3)(res, {"rgb": tgt})
    for k in ("rgb", "opacity", "distortion"):
        assert np.allclose(l_my[k].detach().float().cpu().numpy(), g["loss_" + k], rtol=1e-4, atol=3e-8), k
    # gradient of the distortion term w.r.t. ws
    g_my = torch.autograd.grad(l_my["distortion"].sum(), res["ws"])[0]
    assert np.allclose(g_my.cpu().numpy(), g["dws"], rtol=1e-4, atol=3e-8)


def test_mark_invisible_cells_matches_reference():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    g = gold("mark_invisible")
    mine = NGP(2.0).cuda()
    G = 128
    coords = torch.stack(torch.meshgrid(*[torch.arange(G, dtype=torch.int32, device="cuda")] * 3, indexing="ij"), -1).reshape(-1, 3)
    mine.register_buffer("density_grid", torch.zeros(mine.cascades, G ** 3, device="cuda"))
    mine.register_buffer("grid_coords", coords)
    Kd = synth.intrinsics(W=200, H=150, fx=180.0)
    K = torch.tensor([[Kd["fx"], 0, Kd["cx"]], [0, Kd["fy"], Kd["cy"]], [0, 0, 1]], device="cuda")
    poses = torch.as_tensor(synth.camera_poses(6, radius=1.2)).cuda()
    mine.mark_invisible_cells(K, poses, (200, 150))
    dg = mine.density_grid.cpu().numpy()
    assert tuple(g["shape"]) == dg.shape
    assert set(np.unique(dg).tolist()) <= {-1.0, 0.0}
    assert (np.packbits(dg < 0) == g["invisible"]).all()
    n_cams = int(g["n_cams"])
    cg = mine.count_grid.cpu().numpy()
    k = np.round(cg * n_cams)
    assert np.allclose(cg, k / n_cams)
    assert (cases.digest(k.astype(np.uint8)) == g["cameras_digest"]).all(), "count_grid differs from the reference's"
    assert 0 < (dg < 0).mean() < 1
