"""GPU tests of the fused, sync-free paths (ngp_render_train_fwd/bwd, ngp_adam_step, ngp_gen_rays,
ngp_update_density_grid, ngp_render_infer) against the operator-by-operator path whose pieces are
pinned to the oracle / reference in test_vren_gpu.py and test_network_gpu.py, and against torch.
"""
import math

import numpy as np
import pytest
import torch

import cases

pytestmark = pytest.mark.gpu


def make_model(scene, amp=0.3, seed=0):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    m = NGP(scene.scale).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        p = m.xyz_encoder.params
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * amp).cuda()
        m.density_bitfield.copy_(torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda())
    return m


@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_fused_train_step_matches_unfused_autograd(which):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    from ngp_pl_b200.models.rendering import render
    from ngp_pl_b200.models.custom_functions import RayMarcher
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    n = 2048
    model = make_model(scene)
    o_np, d_np = cases.rays_from_scene(scene, n, 41, extra_edge_cases=True)
    o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
    gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    bg = (1.0,) * 3 if scene.exp_step_factor == 0 else (0.0,) * 3
    tr = Trainer(model, n_rays=n, exp_step_factor=scene.exp_step_factor, bg=bg, materialize_ws=True)
    tr.set_batch(o, d, gt)
    # fused forward with a known jitter
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    import ctypes as C
    from ngp_pl_b200 import _lib
    tr.noise.copy_(noise)
    _lib.check(_lib.lib().ngp_render_train_fwd(C.byref(tr.net), C.byref(tr.cfg), C.byref(tr.buf), tr._st()), "fwd")
    tr.loss_backward()
    torch.cuda.synchronize()
    st = tr.stats()

    # operator-by-operator path with the same jitter
    RayMarcher.noise_override = noise
    try:
        kw = {} if scene.exp_step_factor == 0 else {"exp_step_factor": scene.exp_step_factor}
        model.zero_grad()
        res = render(model, o, d, **kw)
    finally:
        RayMarcher.noise_override = None
    assert int(res["rm_samples"]) == st["rm_samples"] > 0
    assert int(res["vr_samples"]) == st["vr_samples"]
    assert torch.equal(res["rays_a"][:, 2].int(), tr.n_samples)
    tot = st["rm_samples"]
    # the fused path allocates a ray's segment in arrival order (like the reference's atomic rays_a), the operator path in
    # ray order: sample i of the operator path lives in slot[i] of the fused path's arrays
    ra = res["rays_a"]
    slot = torch.repeat_interleave(tr.offsets.long() - ra[:, 1], ra[:, 2]) + torch.arange(tot, device="cuda")
    assert torch.equal(res["ts"], tr.ts[slot]) and torch.equal(res["deltas"], tr.deltas[slot])
    for k, mine in (("rgb", tr.rgb), ("opacity", tr.opacity), ("depth", tr.depth)):
        assert torch.allclose(res[k].float(), mine, rtol=1e-5, atol=1e-6), k
    assert torch.allclose(res["ws"], tr.ws[slot], rtol=1e-5, atol=1e-7)
    # reference NeRFLoss (losses.py:47-60, no distortion) in torch
    op = res["opacity"] + 1e-10
    loss = ((res["rgb"] - gt) ** 2).mean() + (1e-3 * (-op * torch.log(op))).mean()
    loss.backward()
    assert abs(loss.item() - st["loss"]) < 1e-5 * max(1.0, abs(loss.item()))
    g_ref = torch.cat([model.xyz_encoder.params.grad, model.rgb_net.params.grad])
    g_my = tr.G
    s = g_ref.abs().max().item()
    assert s > 0
    err = (g_ref - g_my).abs().max().item()
    assert err < 2e-3 * s, "fused gradient differs: %g vs scale %g" % (err, s)


def test_adam_matches_torch_adam():
    import ctypes as C
    from ngp_pl_b200 import _lib
    n = 100003  # odd tail exercises the scalar epilogue
    gen = torch.Generator("cuda").manual_seed(0)
    p0 = torch.randn(n + 1, device="cuda", generator=gen)[:n].contiguous()
    p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=1e-2, eps=1e-15)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    ph = torch.zeros(n, device="cuda", dtype=torch.float16)
    lr = torch.full((1,), 1e-2, device="cuda")
    step = torch.zeros(1, device="cuda", dtype=torch.int32)
    st = torch.cuda.current_stream().cuda_stream
    for it in range(5):
        g = torch.randn(n, device="cuda", generator=gen) * (10.0 ** -it)
        g[::7] = 0  # untouched hash entries: zero gradient, parameters still move with the momentum
        p_ref.grad = (g / 2).clone()  # averaged gradient of a 2-rank job
        opt.step()
        gg = g.clone()
        _lib.check(_lib.lib().ngp_adam_step(p.data_ptr(), gg.data_ptr(), m.data_ptr(), v.data_ptr(), ph.data_ptr(), n,
                                            lr.data_ptr(), step.data_ptr(), 0.9, 0.999, 1e-15, 0.5, 1, st), "adam")
        assert gg.abs().max().item() == 0, "gradient buffer must be zeroed for the next step"
        assert torch.allclose(p, p_ref.detach(), rtol=2e-5, atol=2e-6), "step %d" % it
        assert torch.equal(ph, p.half())
    assert int(step) == 5


def test_gen_rays_matches_reference_convention():
    import ctypes as C
    from ngp_pl_b200 import _lib, synth
    K = synth.intrinsics(W=64, H=48, fx=70.0)
    dirs = synth.ray_directions(K, "cuda")
    poses = torch.as_tensor(synth.camera_poses(5)).cuda()
    imgs = torch.randint(0, 256, (5, dirs.shape[0], 3), device="cuda", dtype=torch.uint8)
    n = 1000
    img = torch.randint(0, 5, (n,), device="cuda")
    pix = torch.randint(0, dirs.shape[0], (n,), device="cuda")
    o = torch.empty(n, 3, device="cuda"); d = torch.empty(n, 3, device="cuda"); c = torch.empty(n, 3, device="cuda")
    _lib.check(_lib.lib().ngp_gen_rays(img.data_ptr(), pix.data_ptr(), poses.data_ptr(), dirs.data_ptr(), imgs.data_ptr(),
                                       dirs.shape[0], n, o.data_ptr(), d.data_ptr(), c.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "gen_rays")
    o2, d2 = synth.get_rays(dirs[pix], poses[img])
    assert torch.equal(o, o2)
    assert torch.allclose(d, d2, rtol=1e-6, atol=1e-7)
    assert torch.allclose(c, imgs[img, pix].float() / 255)


def test_sample_rays_draws_uniform_pairs_and_builds_the_same_rays():
    """ngp_sample_rays = device-side draw of (image, pixel) with replacement + ngp_gen_rays + jitter in one kernel."""
    from ngp_pl_b200 import synth, _lib
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=40, H=30, fx=300.0)
    bank = synth.RayBank(scene, n_images=7, K=K, device="cuda")
    n_img, n_pix = bank.poses.shape[0], bank.directions.shape[0]
    n = 20000
    L = _lib.lib()

    def draw(seed, stream, ctr):
        o = torch.empty(n, 3, device="cuda"); d = torch.empty(n, 3, device="cuda"); c = torch.empty(n, 3, device="cuda")
        z = torch.empty(n, device="cuda")
        _lib.check(L.ngp_sample_rays(bank.poses.data_ptr(), bank.directions.data_ptr(), bank.rgb.data_ptr(), n_img, n_pix, n,
                                     seed, stream, ctr.data_ptr(), o.data_ptr(), d.data_ptr(), c.data_ptr(), z.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), "sample_rays")
        return o, d, c, z
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    o, d, c, z = draw(5, 0, ctr)
    assert ctr.tolist() == [1, 0]  # the kernel advanced its own draw counter
    # every ray is exactly what ngp_gen_rays builds for SOME (image, pixel): recover the pair and compare
    origins = bank.poses[:, :, 3]
    im = (o[:, None, :] - origins[None]).abs().sum(-1).argmin(1)
    assert torch.equal(o, origins[im])
    all_d = torch.einsum("pc,ikc->ipk", bank.directions, bank.poses[:, :, :3])  # (n_img, n_pix, 3)
    px = (all_d[im] - d[:, None, :]).abs().sum(-1).argmin(1)
    o2 = torch.empty_like(o); d2 = torch.empty_like(d); c2 = torch.empty_like(c)
    _lib.check(L.ngp_gen_rays(im.data_ptr(), px.data_ptr(), bank.poses.data_ptr(), bank.directions.data_ptr(),
                              bank.rgb.data_ptr(), n_pix, n, o2.data_ptr(), d2.data_ptr(), c2.data_ptr(),
                              torch.cuda.current_stream().cuda_stream), "gen_rays")
    assert torch.equal(d, d2) and torch.equal(c, c2)
    # uniform with replacement over images and pixels, jitter uniform in [0,1)
    cnt = torch.bincount(im, minlength=n_img).float()
    assert (cnt - n / n_img).abs().max() < 6 * (n / n_img) ** 0.5
    assert torch.bincount(px, minlength=n_pix).max() <= 60 and px.unique().numel() > 0.99 * n_pix
    assert 0 <= float(z.min()) and float(z.max()) < 1 and abs(float(z.mean()) - 0.5) < 0.01
    # next draw differs; another stream differs; same (seed, stream, draw) reproduces
    o3, d3, _, z3 = draw(5, 0, ctr)
    assert not torch.equal(d3, d) and not torch.equal(z3, z)
    o4, d4, _, _ = draw(5, 1, torch.zeros(2, dtype=torch.int32, device="cuda"))
    assert not torch.equal(d4, d)
    o5, d5, c5, z5 = draw(5, 0, torch.zeros(2, dtype=torch.int32, device="cuda"))
    assert torch.equal(d5, d) and torch.equal(z5, z) and torch.equal(c5, c)


def test_update_density_grid_semantics():
    from ngp_pl_b200 import synth, vren
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = make_model(scene, amp=0.3)
    with torch.no_grad():
        # keep only the three coarsest levels so that sigma is smooth inside a 1/128 cell
        off3 = int(model.xyz_encoder.meta.offset[3])
        model.xyz_encoder.params[3072 + 2 * off3:] = 0
    tr = Trainer(model, n_rays=256)
    G3 = 128 ** 3
    thr = 0.01 * 1024 / 3 ** 0.5
    # warm-up refresh: every cell evaluated once at a jittered point
    model.density_grid.zero_()
    tr.update_density_grid(thr, warmup=True)
    torch.cuda.synchronize()
    grid = model.density_grid.clone()
    coords = vren.morton3D_invert(torch.arange(G3, device="cuda", dtype=torch.int32)).float()
    centres = (coords / 127 * 2 - 1) * (0.5 - 0.5 / 128)
    sig_c = model.density(centres)
    ratio = (grid[0] / sig_c)
    assert (grid[0] > 0).all()
    assert ratio.median().item() == pytest.approx(1.0, abs=0.05)
    assert ((ratio > 0.5) & (ratio < 2.0)).float().mean().item() > 0.99
    mean = grid[grid > 0].mean().item()
    want = torch.zeros_like(model.density_bitfield)
    vren.packbits(grid, min(mean, thr), want)
    diff = (want ^ model.density_bitfield).to(torch.int32)
    flipped = sum(((diff >> b) & 1).sum().item() for b in range(8))
    assert flipped <= 1e-3 * G3, "bitfield disagrees with packbits(grid, min(mean, thr)) on %d cells" % flipped
    # regular refresh: cells marked -1 stay -1, nothing decays faster than `decay`, sampled cells rise to sigma
    model.density_grid[0, :1000] = -1
    before = model.density_grid.clone()
    tr.host_step = 17
    tr.update_density_grid(thr, warmup=False)
    torch.cuda.synchronize()
    after = model.density_grid
    assert (after[0, :1000] == -1).all()
    rest = before[0, 1000:]
    assert (after[0, 1000:] >= 0.95 * rest - 1e-6).all()
    grown = (after[0, 1000:] > rest * 0.95 + 1e-6).float().mean().item()
    assert 0.2 < grown < 0.55  # ~M uniform + ~M occupied of G^3 cells, with collisions
    # different seeds/steps pick different cells
    tr.host_step = 33
    b2 = model.density_grid.clone()
    tr.update_density_grid(thr, warmup=False)
    assert not torch.equal(b2, model.density_grid)


def frame_rays(which):
    """one 160x120 camera view of the synthetic Lego or mip360 scene"""
    from ngp_pl_b200 import synth
    K = synth.intrinsics(W=160, H=120, fx=1111.11 / 5)
    dirs = synth.ray_directions(K, "cuda")
    pose = torch.as_tensor(synth.camera_poses(3, radius=1.5 if which == "lego" else 0.9)[1]).cuda()
    return synth.get_rays(dirs, pose)


@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_fused_inference_matches_operator_loop(which):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    model = make_model(scene, amp=0.5)
    o, d = frame_rays(which)
    kw = {} if scene.exp_step_factor == 0 else {"exp_step_factor": scene.exp_step_factor}
    a = render(model, o, d, test_time=True, fused=True, **kw)
    b = render(model, o, d, test_time=True, fused=False, **kw)
    for k in ("rgb", "opacity", "depth"):
        err = (a[k] - b[k]).abs()
        assert err.max().item() < 2e-4 * max(1.0, b[k].abs().max().item()), "%s: max err %g" % (k, err.max().item())
    ta, tb = int(a["total_samples"]), int(b["total_samples"])
    # both evaluate the reference's per-round quota max(min(N_rays // N_alive, 64), min_samples) (rendering.py:80) from the same
    # alive counts, so the marched totals agree up to the rays whose termination round moves with the last bits of sigma
    assert ta > 0 and abs(ta - tb) <= 0.01 * tb


@pytest.mark.parametrize("esf", [0.0, 1.0 / 256])
@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_fused_inference_marcher_bitwise_vs_operator_loop(which, esf):
    """The inference wavefront's marcher (k_infer_march: thread per ray with the cached cell visit, warp per ray in the
    late rounds) against raymarching_test, bit for bit. With every MLP weight zero, sigma = exp(0) = 1 and
    rgb = sigmoid(0) = 0.5 exactly in both paths, and both compositing loops do the same serial fp32 operations, so the
    termination rounds, alive counts and quotas agree and any difference comes from the marchers. bg is 0 or 1, so
    bg * (1 - opacity) is exact. (lego, mip360) x (esf 0, 1/256) runs all four step-kind x cascade instances."""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    model = make_model(scene, amp=0.5)
    with torch.no_grad():
        model.xyz_encoder.params[:3072] = 0
        model.rgb_net.params.zero_()
    o, d = frame_rays(which)
    a = render(model, o, d, test_time=True, exp_step_factor=esf)
    b = render(model, o, d, test_time=True, fused=False, exp_step_factor=esf)
    assert int(a["total_samples"]) == int(b["total_samples"]) > 0
    for k in ("opacity", "depth", "rgb"):
        bad = (a[k].view(torch.int32) != b[k].view(torch.int32)).sum().item()
        assert bad == 0, "%s: %d/%d elements differ bitwise" % (k, bad, a[k].numel())


def test_training_converges_and_graph_capture_works():
    """End to end: batch assembly -> fwd -> loss -> bwd -> Adam + occupancy refreshes, CUDA-graph
    captured, on the synthetic Lego scene; PSNR must climb well above the initial ~10 dB."""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=40, K=K, device="cuda")
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=4096, lr=1e-2)
    tr.attach_bank(bank)
    for _ in range(20):  # eager steps first
        tr.train_step()
    tr.capture()
    for _ in range(480):
        tr.train_step()
    torch.cuda.synchronize()
    st = tr.stats()
    assert math.isfinite(st["loss"])
    assert st["psnr"] > 22.0, "training PSNR only %.2f dB after 500 steps" % st["psnr"]
    assert int(tr.step_dev) == 500  # the warm-up run inside capture() is rolled back


@pytest.mark.parametrize("name", cases.MARCH_CASES)
def test_warp_marcher_bit_exact_vs_oracle(name, oracle):
    """the warp-cooperative marcher of the fused path (march_ray_warp) against the serial oracle restatement
    (itself pinned bit-exactly to the reference kernels by tests/golden): counts, ts, deltas"""
    import ctypes as C
    from ngp_pl_b200 import _lib
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    c = cases.march_case(name)
    n = c["o"].shape[0]
    model = NGP(float(c["scale"])).cuda()
    with torch.no_grad():
        model.density_bitfield.copy_(torch.as_tensor(c["bits"]).cuda())
    tr = Trainer(model, n_rays=n, exp_step_factor=float(c["esf"]))
    tr.set_batch(torch.as_tensor(c["o"]).cuda(), torch.as_tensor(c["d"]).cuda(), torch.zeros(n, 3).cuda())
    tr.noise.copy_(torch.as_tensor(c["noise"]).cuda())
    _lib.check(_lib.lib().ngp_render_train_fwd(C.byref(tr.net), C.byref(tr.cfg), C.byref(tr.buf), tr._st()), "fwd")
    torch.cuda.synchronize()
    hits = cases.hits_for(c, oracle)
    ra, xyzs, dirs, deltas, ts = oracle.march_train(c["o"], c["d"], hits, c["bits"], c["cascades"], c["scale"], c["esf"],
                                                    c["noise"], 128, int(tr.cfg.max_samples))
    if name == "full_scale2":
        assert ra[:, 2].max() == 1024
    assert (tr.n_samples.cpu().numpy() == ra[:, 2]).all()
    tot = int(ra[:, 2].sum())
    assert int(tr.counters[0]) == tot
    # the fused path hands every ray a segment of the compact arrays in arrival order (like the reference's atomic rays_a);
    # the segments partition [0, total) and each holds exactly the oracle's samples of its ray, bit for bit
    off = tr.offsets.cpu().numpy().astype(np.int64)
    cnt = ra[:, 2].astype(np.int64)
    order = np.argsort(off, kind="stable")
    nz = order[cnt[order] > 0]
    assert (off[nz] == np.concatenate([[0], np.cumsum(cnt[nz])[:-1]])).all()
    gather = (np.repeat(off - ra[:, 1], cnt) + np.arange(tot)).astype(np.int64)  # oracle sample i (ray order) -> its slot
    assert (tr.ts.cpu().numpy()[gather].view(np.uint32) == ts.view(np.uint32)).all()
    assert (tr.deltas.cpu().numpy()[gather].view(np.uint32) == deltas.view(np.uint32)).all()
    assert (tr.ray_idx.cpu().numpy()[gather] == np.repeat(np.arange(n), cnt)).all()


def test_fused_nvlink_optimizer_step_two_gpus(tmp_path):
    """ngp_adam_step_fused / ngp_adam_step_p2p (reduce-scatter + sharded Adam + all-gather over NVLink peer memory, with
    in-kernel or host barriers, with or without NVLS multicast) == NCCL all-reduce + full Adam, bitwise at N=2
    (tools/check_p2p.py under torchrun). Needs two GPUs; skipped on a 1-GPU box (bench.py's N>1 runs repeat the check on
    their first step and report it in the JSON line as `exchange_check`)."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for k, mode in enumerate(("p2p", "nvls", "p2p_host")):
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", str(29541 + k),
                            os.path.join(root, "tools", "check_p2p.py"), mode],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:]
        assert "MISMATCH" not in r.stdout


def test_fused_trainer_with_distortion_loss_matches_autograd():
    """lambda_distortion > 0 on the fused path (ws materialised, ngp_distortion_loss_fw/bw feeding dL_dws into the
    compositing backward) against render() + NeRFLoss(lambda_distortion) + autograd"""
    import ctypes as C
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.losses import NeRFLoss
    from ngp_pl_b200.trainer import Trainer
    from ngp_pl_b200.models.rendering import render
    from ngp_pl_b200.models.custom_functions import RayMarcher
    scene = synth.mip360_scene(0)
    n, lam = 1024, 1e-2
    model = make_model(scene)
    o_np, d_np = cases.rays_from_scene(scene, n, 43, extra_edge_cases=False)
    o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
    gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    tr = Trainer(model, n_rays=n, exp_step_factor=scene.exp_step_factor, bg=(0.0,) * 3, lambda_distortion=lam)
    tr.set_batch(o, d, gt)
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    tr.noise.copy_(noise)
    _lib.check(_lib.lib().ngp_render_train_fwd(C.byref(tr.net), C.byref(tr.cfg), C.byref(tr.buf), tr._st()), "fwd")
    tr.loss_backward()
    torch.cuda.synchronize()
    st = tr.stats()
    RayMarcher.noise_override = noise
    try:
        model.zero_grad()
        res = render(model, o, d, exp_step_factor=scene.exp_step_factor)
    finally:
        RayMarcher.noise_override = None
    loss = sum(v.mean() for v in NeRFLoss(lambda_distortion=lam)(res, {"rgb": gt}).values())
    loss.backward()
    assert abs(loss.item() - st["loss"]) < 1e-4 * max(1.0, abs(loss.item()))
    g_ref = torch.cat([model.xyz_encoder.params.grad, model.rgb_net.params.grad])
    s = g_ref.abs().max().item()
    assert (g_ref - tr.G).abs().max().item() < 3e-3 * s


def test_backward_visits_only_composited_samples():
    """The samples after a ray's terminating sample get exactly zero gradient (composite_train_bw,
    volumerendering.cu:87-151): the fused backward skips them through the live list. Same gradients as
    the backward over every marched sample."""
    import ctypes as C
    from ngp_pl_b200 import synth, _lib
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    # a briefly trained model: opaque surfaces, so most rays terminate well before their last marched sample
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=40, K=K, device="cuda")
    model = NGP(scene.scale).cuda()
    tr0 = Trainer(model, n_rays=4096, lr=1e-2)
    tr0.attach_bank(bank)
    for _ in range(300):
        tr0.train_step()
    tr0.gather_master_params()
    torch.cuda.synchronize()
    n = 4096
    o, d, gt = bank.sample(n)
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    out = {}
    for skip in (True, False):
        tr = Trainer(model, n_rays=n, skip_dead_samples=skip)
        tr.set_batch(o, d, gt)
        tr.noise.copy_(noise)
        _lib.check(_lib.lib().ngp_render_train_fwd(C.byref(tr.net), C.byref(tr.cfg), C.byref(tr.buf), tr._st()), "fwd")
        tr.loss_backward()
        torch.cuda.synchronize()
        out[skip] = (tr.G.clone(), tr.stats(), tr)
    st = out[True][1]
    assert st["rm_samples"] == out[False][1]["rm_samples"] and st["vr_samples"] == out[False][1]["vr_samples"]
    # live list = composited samples = vr_samples + one terminating sample per terminated ray
    assert st["vr_samples"] <= st["bw_samples"] <= st["vr_samples"] + n
    assert st["bw_samples"] < 0.9 * st["rm_samples"], st
    assert out[False][1]["bw_samples"] == st["rm_samples"]
    tr = out[True][2]
    live = tr.live_idx[:st["bw_samples"]].long()
    assert live.unique().numel() == live.numel()
    dead = torch.ones(st["rm_samples"], dtype=torch.bool, device="cuda")
    dead[live] = False
    assert tr.dsigmas[:st["rm_samples"]][dead].abs().max().item() == 0
    assert tr.drgbs[:st["rm_samples"]][dead].abs().max().item() == 0
    g1, g0 = out[True][0], out[False][0]
    s = g0.abs().max().item()
    assert s > 0
    assert (g1 - g0).abs().max().item() < 2e-4 * s  # fp32 atomics re-associate; fp16 operands are identical


def test_stage_batch_prefetch_matches_set_batch():
    """Host-fed training: stage_batch() (next batch copied + marched on the side stream under the running step) must
    train on exactly the batches / jitter that set_batch() + train_step(sample=False) does."""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=100, H=100, fx=1111.11 / 8)
    bank = synth.RayBank(scene, n_images=10, K=K, device="cuda")
    n = 2048
    host = [tuple(t.cpu().pin_memory() for t in bank.sample(n)) for _ in range(6)]
    logs = []
    for prefetch in (False, True):
        torch.manual_seed(0)
        model = NGP(scene.scale).cuda()
        with torch.no_grad():
            model.density_bitfield.copy_(torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda())
        tr = Trainer(model, n_rays=n, lr=1e-2, seed=3, update_interval=1000)
        tr.set_batch(*host[0])
        tr.capture(sample=False)
        # no occupancy refresh inside the comparison: right after initialisation all cell densities sit on the mean that
        # thresholds them, so the refreshed bitfield would turn on the last bits of the weights, which the two runs'
        # gradient atomics already let drift apart
        tr.host_step = 1
        log = []
        if prefetch:
            tr.stage_batch(*host[0])
        for i in range(6):
            if prefetch:
                tr.train_step(sample=False)
                if i + 1 < 6:
                    tr.stage_batch(*host[i + 1])
            else:
                tr.set_batch(*host[i])
                tr.train_step(sample=False)
            torch.cuda.synchronize()
            st = tr.stats()
            log.append((st["rm_samples"], st["loss"]))
        logs.append(log)
    assert logs[0][0][0] == logs[1][0][0] > 0 and abs(logs[0][0][1] - logs[1][0][1]) < 1e-6  # first step: identical inputs
    for (n0, l0), (n1, l1) in zip(*logs):
        assert abs(n0 - n1) <= 0.02 * n0 and abs(l0 - l1) <= 0.02 * l0  # later: atomics-order noise through Adam only


def test_fused_composite_loss_kernel_matches_separate_kernels():
    """ngp_render_train_step (compositing fw + NeRFLoss + compositing bw in one kernel) against
    ngp_render_train_net + ngp_nerf_loss_grad + ngp_render_train_bwd on the same batch and jitter."""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    n = 4096
    o_np, d_np = cases.rays_from_scene(scene, n, 47, extra_edge_cases=True)
    o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
    gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    out = {}
    for fused in (True, False):
        model = make_model(scene, amp=1.0)
        tr = Trainer(model, n_rays=n, fused_loss=fused)
        assert tr.fused_loss == fused
        tr.set_batch(o, d, gt)
        tr.noise.copy_(noise)
        tr.march(jitter=False)
        tr._compute()
        torch.cuda.synchronize()
        out[fused] = (tr.G.clone(), tr.stats(), tr.rgb.clone(), tr.opacity.clone(), tr.depth.clone(), float(tr.scalars[1]))
    a, b = out[True], out[False]
    for k in ("rm_samples", "vr_samples", "bw_samples"):
        assert a[1][k] == b[1][k] > 0, k
    assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]) and torch.equal(a[4], b[4])  # same forward code
    assert abs(a[1]["loss"] - b[1]["loss"]) < 1e-6 * max(1.0, abs(b[1]["loss"]))
    assert a[5] == b[5]  # same power-of-two loss scale
    s = b[0].abs().max().item()
    assert s > 0 and (a[0] - b[0]).abs().max().item() < 2e-4 * s
