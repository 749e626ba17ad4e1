"""GPU tests of the round-2 additions: the reference's learning-rate schedule on the device-resident lr, `erode` on the fused
occupancy refresh, one random background colour per training batch, refreshing the fp16 working copy after outside writes to
the parameters, the whole-frame inference graph, the fwd kernel's unused-slot marker and the launch counter."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import cases
from test_fused_gpu import make_model

pytestmark = pytest.mark.gpu


def test_cosine_schedule_reaches_the_adam_kernel():
    """Trainer(lr_schedule=CosineAnnealingLR) writes lr(epoch) into the device scalar the Adam kernel reads, epoch = step // steps_per_epoch
    (reference train.py:135-137, stepped per epoch by pytorch-lightning)"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import CosineAnnealingLR, Trainer
    scene = synth.lego_scene(0)
    model = make_model(scene)
    sch = CosineAnnealingLR(1e-2, T_max=4, steps_per_epoch=3)
    tr = Trainer(model, n_rays=256, lr=1e-2, lr_schedule=sch)
    o_np, d_np = cases.rays_from_scene(scene, 256, 5, extra_edge_cases=False)
    tr.set_batch(torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda(), torch.rand(256, 3, device="cuda"))
    seen = []
    for step in range(12):
        tr.train_step(sample=False)
        seen.append(float(tr.lr_dev.item()))
    want = [1e-2 / 30 + (1e-2 - 1e-2 / 30) * (1 + math.cos(math.pi * (s // 3) / 4)) / 2 for s in range(12)]
    assert np.allclose(seen, want, rtol=1e-6)
    assert seen[0] == pytest.approx(1e-2) and seen[-1] < seen[0]


def test_fused_refresh_erode_matches_formula():
    """ngp_update_density_grid with count_grid: every cell that is not re-evaluated above its old value decays by
    clamp(decay^(1/count), 0.1, 0.95) (reference networks.py:258-264)"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = make_model(scene, amp=0.0)  # zero table -> h = 0 -> sigma = exp(0) = 1 everywhere
    tr = Trainer(model, n_rays=256, erode=True)
    G3 = model.grid_size ** 3
    with pytest.raises(RuntimeError):
        tr.update_density_grid(warmup=False)  # no count_grid yet
    g = torch.Generator("cuda").manual_seed(3)
    count = torch.rand(model.cascades, G3, device="cuda", generator=g)
    count[:, ::7] = 0.0  # unseen cells: decay^(inf) = 0 -> clamped to 0.1
    model.count_grid = count
    model.density_grid.fill_(100.0)  # old*decay >= 10 > sigma = 1: the maximum keeps the decayed old value in every cell
    tr.update_density_grid(warmup=False, decay=0.95)
    torch.cuda.synchronize()
    d = torch.clamp(0.95 ** (1 / count), 0.1, 0.95)
    assert torch.allclose(model.density_grid, 100.0 * d, rtol=2e-6)
    # and without erode: the plain decay
    tr2 = Trainer(make_model(scene, amp=0.0), n_rays=256)
    tr2.model.density_grid.fill_(100.0)
    tr2.update_density_grid(warmup=False, decay=0.95)
    torch.cuda.synchronize()
    assert torch.allclose(tr2.model.density_grid, torch.full_like(tr2.model.density_grid, 95.0), rtol=2e-6)


def test_random_background_per_batch():
    """Trainer(random_bg=True): one uniform colour per batch composited behind the samples, forward and backward
    (reference rendering.py:153-161); checked against render() + autograd with the same colour"""
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.losses import NeRFLoss
    from ngp_pl_b200.models.custom_functions import RayMarcher
    from ngp_pl_b200.models.rendering import render
    from ngp_pl_b200.trainer import Trainer
    scene = synth.mip360_scene(0)
    n = 1024
    model = make_model(scene)
    o_np, d_np = cases.rays_from_scene(scene, n, 47, extra_edge_cases=False)
    o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
    gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    tr = Trainer(model, n_rays=n, exp_step_factor=scene.exp_step_factor, bg=(0.0,) * 3, random_bg=True)
    tr.set_batch(o, d, gt)
    tr.march()  # draws the jitter and this batch's background
    bg1 = tr.bg.clone()
    noise = tr.noise.clone()
    tr._compute()
    torch.cuda.synchronize()
    assert (bg1 >= 0).all() and (bg1 < 1).all() and bg1.std() > 0
    # reference composition with the same colour: rgb = acc + bg * (1 - opacity)
    RayMarcher.noise_override = noise
    try:
        model.zero_grad()
        res = render(model, o, d, exp_step_factor=scene.exp_step_factor)
    finally:
        RayMarcher.noise_override = None
    rgb = res["rgb"] + bg1 * (1 - res["opacity"])[:, None]  # render() used bg 0 (random_bg not requested)
    assert (tr.rgb - rgb).abs().max().item() < 2e-4
    loss = sum(v.mean() for v in NeRFLoss(lambda_distortion=0)({"rgb": rgb, "opacity": res["opacity"]}, {"rgb": gt}).values())
    loss.backward()
    g_ref = torch.cat([model.xyz_encoder.params.grad, model.rgb_net.params.grad])
    assert (g_ref - tr.G).abs().max().item() < 3e-3 * g_ref.abs().max().item()
    tr.march()
    assert not torch.equal(tr.bg, bg1)  # a new colour for the next batch


def test_outside_parameter_writes_reach_the_kernels():
    """load_state_dict (post hook) and sync_params() refresh the fp16 working copy the kernels read; the stand-alone modules
    re-cast on every training forward (an optimiser writing through p.data does not bump p._version)"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = make_model(scene)
    tr = Trainer(model, n_rays=256)
    other = make_model(scene, seed=5)
    x = (torch.rand(4096, 3, device="cuda") - 0.5)
    want = other.density(x)
    before = model.density(x)
    assert not torch.allclose(before, want)
    model.load_state_dict(other.state_dict(), strict=False)  # (`other` has no density_grid buffer: only a Trainer registers one)
    assert torch.equal(model.density(x), want)
    with torch.no_grad():
        model.xyz_encoder.params.data.mul_(0.5)
    tr.sync_params()
    half = NGP(scene.scale).cuda()
    half.load_state_dict(model.state_dict(), strict=False)
    assert torch.equal(model.density(x), half.density(x))
    # stand-alone module (no Trainer): a write through .data must be seen by the next training forward
    m2 = make_model(scene, seed=7)
    d = torch.randn(4096, 3, device="cuda")
    s0, _ = m2(x, d)
    with torch.no_grad():
        m2.xyz_encoder.params.data.mul_(0.25)  # does not bump _version
    s1, _ = m2(x, d)
    assert not torch.allclose(s0, s1)


def test_position_gradients_fail_loudly():
    from ngp_pl_b200 import synth
    scene = synth.lego_scene(0)
    model = make_model(scene)
    x = (torch.rand(64, 3, device="cuda") - 0.5).requires_grad_(True)
    d = torch.randn(64, 3, device="cuda")
    with pytest.raises(NotImplementedError):
        model(x, d)


@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_frame_graph_inference_equals_round_loop(which):
    """ngp_render_infer_frame (one CUDA graph with a device-side while loop) == ngp_render_infer driven round by round from the
    host: same kernels, same order, so the images are identical. Both are also bitwise the operator loop (fused=False):
    its samples are the wavefront's (both march the reference's test-time sequence), the network evaluates a sample at
    fma(d, t, o) from (ray, t) exactly as the operator loop's marcher rounds xyzs, and both composite with
    composite_ray_serial in the same order -- so total_samples and every image agree exactly."""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    model = make_model(scene)
    K = synth.intrinsics(W=200, H=150, fx=1111.11 / 4)
    dirs = synth.ray_directions(K, "cuda")
    kw = {} if scene.exp_step_factor == 0 else {"exp_step_factor": scene.exp_step_factor}
    for i in range(3):  # the second and third frame replay the cached graph with new rays in the same buffers
        pose = torch.as_tensor(synth.camera_poses(4, radius=synth.camera_radius(scene), upper_only=scene.scale <= 0.5)[i]).cuda()
        o, d = synth.get_rays(dirs, pose)
        a = render(model, o, d, test_time=True, graph=True, **kw)
        assert getattr(model, "_infer_graph_ok", True), "conditional graph nodes should be available on this driver"
        b = render(model, o, d, test_time=True, graph=False, **kw)
        for k in ("rgb", "opacity", "depth"):
            assert torch.equal(a[k], b[k]), k
        assert int(a["total_samples"]) == int(b["total_samples"]) > 0
    c = render(model, o, d, test_time=True, fused=False, **kw)
    assert int(a["total_samples"]) == int(c["total_samples"])
    for k in ("rgb", "opacity", "depth"):
        assert torch.equal(a[k], c[k]), "%s: max |fused - operator loop| = %g" % (k, (a[k] - c[k]).abs().max().item())


def test_forward_skips_unused_slots():
    """ray_idx = -1 marks an unused slot of a rectangular (ray, slot) sample layout: the forward kernel must not touch rays_o /
    rays_d / the table for it, and the other samples' outputs are unchanged"""
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.models.networks import _net_struct
    scene = synth.lego_scene(0)
    model = make_model(scene)
    n_rays, n = 64, 4096
    g = torch.Generator("cuda").manual_seed(0)
    o = (torch.rand(n_rays, 3, device="cuda", generator=g) - 0.5) * 0.2
    d = torch.randn(n_rays, 3, device="cuda", generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    ridx = torch.randint(0, n_rays, (n,), device="cuda", generator=g, dtype=torch.int32)
    ts = torch.rand(n, device="cuda", generator=g) * 0.3
    net, keep = _net_struct(model)
    L = _lib.lib()

    def run(ray_idx):
        smp = _lib.NgpSamples()
        smp.rays_o, smp.rays_d, smp.ray_idx, smp.ts = o.data_ptr(), d.data_ptr(), ray_idx.data_ptr(), ts.data_ptr()
        smp.n = n
        sig = torch.zeros(n, device="cuda")
        rgb = torch.zeros(n, 3, device="cuda")
        _lib.check(L.ngp_net_forward(C.byref(net), C.byref(smp), 1, sig.data_ptr(), rgb.data_ptr(), None, None,
                                     torch.cuda.current_stream().cuda_stream), "fwd")
        torch.cuda.synchronize()
        return sig, rgb
    s0, c0 = run(ridx)
    holes = ridx.clone()
    holes[::3] = -1
    s1, c1 = run(holes)
    keep_mask = holes >= 0
    assert torch.equal(s0[keep_mask], s1[keep_mask]) and torch.equal(c0[keep_mask], c1[keep_mask])
    assert (s1[~keep_mask] == 0).all()  # untouched


def test_launch_counter_counts_graph_replays():
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = make_model(scene)
    bank = synth.RayBank(scene, n_images=4, K=synth.intrinsics(W=64, H=64, fx=100.0), device="cuda")
    tr = Trainer(model, n_rays=512, update_interval=1 << 30)
    tr.attach_bank(bank)
    tr.host_step = 1
    tr.capture(sample=True)
    per_step = tr._graph_nodes[id(tr.g_prepare[0])] + tr._graph_nodes[id(tr.g_compute[0][0])] + tr._graph_nodes[id(tr.g_update[0])]
    assert per_step >= 9  # sample, march, scan, compact | fwd, composite+loss, scale, MLP bwd, scatter | adam, step
    tr.train_step()  # the first step also marches its own batch; from the second on every step replays one graph of each kind
    n0 = tr.launch_count()
    for _ in range(10):
        tr.train_step()
    torch.cuda.synchronize()
    assert tr.launch_count() - n0 == 10 * per_step
    assert int(_lib.lib().ngp_launch_count()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_refresh_picked_ahead_equals_refresh_in_line(which):
    """Trainer(pick_ahead=True) launches the weight-independent half of the NEXT occupancy refresh (cell choice, Morton
    sort, jitter) on its own stream right after a refresh; the grids and bitfields it produces must be bit-identical to
    the single-stream refresh, across the warm-up boundary and for several cascades, and a pick made for other arguments
    (or an older grid) must not be reused."""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    out = []
    for ahead in (True, False):
        model = make_model(scene, amp=0.3)
        tr = Trainer(model, n_rays=256, pick_ahead=ahead, warmup_steps=32)
        grids = []
        for step in (0, 16, 32, 48, 64):  # warm-up, warm-up, then three regular refreshes
            tr.host_step = step
            tr.update_density_grid(warmup=step < tr.warmup_steps)
            assert (tr._picked is not None) == ahead
            grids.append((model.density_grid.clone(), model.density_bitfield.clone()))
        # a refresh the pick was not made for: other step (seed), then a grid written behind the trainer's back
        tr.host_step = 100
        tr.update_density_grid(warmup=False)
        grids.append((model.density_grid.clone(), model.density_bitfield.clone()))
        tr.host_step = 116
        model.density_grid[:, :5000] = -1.0  # bumps the tensor's version counter: the pick made from the old grid is stale
        tr.update_density_grid(warmup=False)
        torch.cuda.synchronize()
        assert (model.density_grid[:, :5000] == -1).all()
        grids.append((model.density_grid.clone(), model.density_bitfield.clone()))
        out.append(grids)
    for (ga, ba), (gb, bb) in zip(*out):
        assert torch.equal(ga, gb)
        # the threshold is min(mean of the positive cells, thr), and that mean is summed in a fixed order (k_grid_merge's
        # per-block partials, added up by k_grid_mean): equal grids give equal bitfields
        assert torch.equal(ba, bb)
