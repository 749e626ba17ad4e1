"""The training step's compositing kernels, sample by sample, against the float64 restatement oracle/composite64.py.

Every per-sample gradient of a training step comes out of k_train_composite_loss (the default, Trainer(fused_loss=True))
or of k_train_composite_fw + k_nerf_loss_grad + k_train_composite_bw (the materialize_ws / distortion-loss path). These
tests read the kernels' own fp32 inputs back (sigmas, rgbs, deltas, ts, offsets, counts), restate compositing, the
background, NeRFLoss and the backward in float64, and hold every output to the derived rounding bound: per ray rgb,
opacity, depth; per sample dL/dsigma and dL/drgb (exactly 0 past the composited samples); the composited counts, the
live list and the sample counters exactly; the loss within gamma_n of the sum; the loss scale exactly. A ray whose
termination the bound cannot decide is reported and left out; at most 1 % of a batch may be.

Batches: random-initialised Lego and mip360 models, a briefly trained Lego, a controlled density (constant sigma, so that
terminations land at chosen lanes of chosen trips) over rays of every length 0..579, a random background, lambda_opacity
1e-3 and 1, and ray counts that leave spare warps in the last block. The separate-kernel path also gets seeded non-zero
dL/ddepth, which the Trainer never passes, and dL/dws, which the Trainer passes only with lambda_distortion > 0 (the
distortion kernel's output; test_distortion_fp64_gpu.py checks that path with the kernel's own dL/dws).
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import cases
from oracle import composite64 as C64
from test_fused_gpu import make_model

pytestmark = pytest.mark.gpu

RATIOS = {}  # quantity -> largest error / (SAFETY bound) over the module's batches


def note(name, r):
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)
    assert r <= 1.0, "%s: error / bound = %.3g" % (name, r)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\ncompositing vs float64, largest error / (%g x bound):" % C64.SAFETY)
    for k in sorted(RATIOS):
        print("  %-28s %.3g" % (k, RATIOS[k]))


def within(name, mine, ref, err, keep):
    note(name, C64.ratio((mine.double() - ref)[keep], err[keep]))


def run_fused(tr, o, d, gt, noise):
    tr.set_batch(o, d, gt)
    tr.noise.copy_(noise)
    tr.march(jitter=False)
    tr._compute()
    torch.cuda.synchronize()


def owner_of_samples(off, cnt, n_tot):
    """ray of every sample slot [0, n_tot)"""
    own = torch.full((n_tot,), -1, dtype=torch.long, device=off.device)
    ray = torch.repeat_interleave(torch.arange(cnt.numel(), device=off.device), cnt.long())
    slot = torch.repeat_interleave(off.long(), cnt.long()) + torch.arange(int(cnt.sum()), device=off.device) - \
        torch.repeat_interleave(torch.cumsum(cnt.long(), 0) - cnt.long(), cnt.long())
    own[slot] = ray
    return own


def check_counts_and_live(tr, f, keep, label):
    """per-ray composited counts (from the live list) equal float64's on decidable rays; the live list is exactly the
    rays' leading composited samples; bw_samples / vr_samples are the sums"""
    st = tr.stats()
    n_tot = st["rm_samples"]
    off, cnt = tr.offsets.long(), tr.n_samples.long()
    assert int(cnt.sum()) == n_tot
    live = tr.live_idx[:st["bw_samples"]].long()
    assert live.unique().numel() == live.numel(), "duplicate live entries"
    own = owner_of_samples(off, cnt, n_tot)
    assert (live >= 0).all() and (live < n_tot).all()
    n_comp_k = torch.bincount(own[live], minlength=cnt.numel())
    # every ray's entries are its leading n_comp_k samples: unique, inside [off, off + n_comp_k)
    assert ((live - off[own[live]]) < n_comp_k[own[live]]).all(), label
    assert torch.equal(n_comp_k[keep], f["n_comp"][keep]), label
    und = ~keep
    total64 = int(f["total"][keep].sum())
    lo = total64 + int((n_comp_k[und] - 1).clamp_min(0).sum())
    hi = total64 + int(n_comp_k[und].sum())
    assert lo <= st["vr_samples"] <= hi, (label, st["vr_samples"], lo, hi)
    if not und.any():
        assert st["vr_samples"] == total64 and st["bw_samples"] == int(f["n_comp"].sum())
    return n_comp_k


def check_backward(tr, f, b, keep, n_tot, label):
    off, cnt = tr.offsets, tr.n_samples
    dsig = C64.pad(tr.dsigmas[:n_tot], off, cnt, f["L"])
    drgb = C64.pad(tr.drgbs[:n_tot], off, cnt, f["L"])
    within("dsigmas", dsig, b["dsig"], b["dsig_err"], keep)
    within("drgbs", drgb, b["drgb"], b["drgb_err"], keep)
    # past each ray's composited samples: exactly zero (decidable rays: float64's count)
    past = (f["valid"] & ~f["comp"])[keep]
    if past.any():
        assert dsig[keep][past].abs().max().item() == 0 and drgb[keep][past].abs().max().item() == 0, label
    return dsig, drgb


def check_loss_scale(tr, n_tot, label):
    want = C64.loss_scale(tr.dsigmas[:n_tot], tr.drgbs[:n_tot], tr.sigmas[:n_tot])
    assert float(tr.scalars[1]) == want, (label, float(tr.scalars[1]), want)


def check_fused_batch(tr, gt, lam, label):
    """everything k_train_composite_loss writes, against float64; returns the forward restatement"""
    n = tr.n_rays
    st = tr.stats()
    n_tot = st["rm_samples"]
    assert n_tot > 0
    bg = tr.bg if tr.random_bg else torch.tensor([tr.cfg.bg[k] for k in range(3)], device="cuda")
    f = C64.forward(tr.sigmas[:n_tot], tr.rgbs[:n_tot], tr.deltas[:n_tot], tr.ts[:n_tot], tr.offsets, tr.n_samples,
                    tr.cfg.T_threshold, "warp")
    keep = ~f["undecidable"]
    n_und = int((~keep).sum())
    print("%s: %d rays, %d samples, %d composited, %d undecidable (%.2f %%)" %
          (label, n, n_tot, int(f["n_comp"].sum()), n_und, 100.0 * n_und / n))
    assert n_und <= 0.01 * n, label
    nl = C64.nerf_loss(f, gt, bg, lam, n)
    within("rgb", tr.rgb, nl["out"], nl["out_err"], keep)
    within("opacity", tr.opacity, f["O"], f["O_err"], keep)
    within("depth", tr.depth, f["D"], f["D_err"], keep)
    b = C64.backward(f, nl["dC"], nl["dO"], dC_err=nl["dC_err"], dO_err=nl["dO_err"])
    check_backward(tr, f, b, keep, n_tot, label)
    check_counts_and_live(tr, f, keep, label)
    check_loss_scale(tr, n_tot, label)
    # the loss: undecidable rays enter with the kernel's own composited output (their float64 twin may hold a sample more)
    loss, err = nl["loss"], nl["loss_err"]
    if n_und:
        und = ~keep
        e_k = tr.rgb[und].double() - gt[und].double()
        op_k = tr.opacity[und].double() + 1e-10
        e_6 = nl["out"][und] - gt[und].double()
        op_6 = f["O"][und] + 1e-10
        loss += float((e_k ** 2).sum() - (e_6 ** 2).sum()) / (3 * n) + \
            lam * float((-op_k * op_k.log()).sum() - (-op_6 * op_6.log()).sum()) / n
    note("loss", abs(st["loss"] - loss) / (C64.SAFETY * err))
    return f


@pytest.mark.parametrize("which,n,lam,random_bg", [
    ("lego", 4101, 1e-3, False),
    ("mip360", 2053, 1e-3, False),
    ("mip360", 1029, 1.0, True),
    ("lego", 3, 1.0, False),
])
def test_fused_step_random_init(which, n, lam, random_bg):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    model = make_model(scene, amp=1.0)
    o_np, d_np = cases.rays_from_scene(scene, max(n, 16), 53, extra_edge_cases=True)
    o, d = torch.as_tensor(o_np[:n]).cuda(), torch.as_tensor(d_np[:n]).cuda()
    gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    bg = (1.0,) * 3 if scene.exp_step_factor == 0 else (0.0,) * 3
    tr = Trainer(model, n_rays=n, exp_step_factor=scene.exp_step_factor, bg=bg, lambda_opacity=lam, random_bg=random_bg)
    assert tr.fused_loss
    run_fused(tr, o, d, gt, noise)
    if random_bg:
        assert tr.bg.std() > 0 and not torch.equal(tr.bg.cpu(), torch.tensor(bg))
    check_fused_batch(tr, gt, lam, "%s n=%d lambda=%g random_bg=%s" % (which, n, lam, random_bg))


def test_fused_step_trained_lego():
    """a briefly trained model: opaque surfaces, rays terminate early, many samples past termination"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=200, H=200, fx=1111.11 / 4)
    bank = synth.RayBank(scene, n_images=40, K=K, device="cuda")
    torch.manual_seed(0)
    model = NGP(scene.scale).cuda()
    tr0 = Trainer(model, n_rays=4096, lr=1e-2)
    tr0.attach_bank(bank)
    for _ in range(300):
        tr0.train_step()
    tr0.gather_master_params()
    torch.cuda.synchronize()
    n = 4101
    o, d, gt = bank.sample(n)
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    for lam in (1e-3, 1.0):
        tr = Trainer(model, n_rays=n, lambda_opacity=lam)
        run_fused(tr, o, d, gt, noise)
        f = check_fused_batch(tr, gt, lam, "trained lego lambda=%g" % lam)
        assert int(f["terminated"].sum()) > 0.2 * n and int(f["n_comp"].sum()) < 0.9 * tr.stats()["rm_samples"]


def controlled_model(scene):
    """hash table = 1 everywhere, W1d = e0 e0^T: every sample's density pre-activation h0 is W2d[0, 0] exactly"""
    from ngp_pl_b200.models.networks import NGP
    torch.manual_seed(0)
    m = NGP(scene.scale).cuda()
    with torch.no_grad():
        p = m.xyz_encoder.params
        p[:3072] = 0
        p[0] = 1.0  # W1d[0, 0]
        p[3072:] = 1.0
        m.density_bitfield.fill_(255)
    return m


def h0_for(k, delta, thr):
    """an fp16 pre-activation h0 whose density exp(h0) makes T_i = exp(-(i + 1) sigma delta) cross T_threshold at
    sample k, as near half a sample from the threshold as fp16 allows"""
    Lth = -math.log(thr)
    want = math.log(Lth / ((k + 0.5) * delta))
    h = torch.tensor([want], dtype=torch.float16)
    assert float(h) > 0
    best = None
    for s in range(-8, 9):
        hv = float((h.view(torch.int16) + s).view(torch.float16))
        x = float(np.float32(math.exp(hv))) * delta
        c = Lth / x
        if math.floor(c) == k and (best is None or abs(c - k - 0.5) < best[0]):
            best = (abs(c - k - 0.5), hv)
    assert best is not None and best[0] < 0.45, (k, best)
    return best[1]


def test_fused_step_controlled_sigma_and_lengths():
    """full occupancy, rays along x from inside the box (every length 0..579 samples), constant density swept so that
    the terminations land on lanes 0 and 31 of trips 0 to 5, at 33, 129, and far beyond the register cache"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = controlled_model(scene)
    n = 8 * 128 + 5
    x0 = torch.linspace(-0.49, 0.56, n)
    o = torch.stack([x0, torch.full((n,), 0.0123), torch.full((n,), -0.0217)], 1).cuda()
    d = torch.tensor([1.0, 0.001, 0.002])
    d = (d / d.norm()).expand(n, 3).contiguous().cuda()
    gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    noise = torch.full((n,), 0.5, device="cuda")
    tr = Trainer(model, n_rays=n, bg=(1.0,) * 3)
    run_fused(tr, o, d, gt, noise)
    n_tot = tr.stats()["rm_samples"]
    deltas = tr.deltas[:n_tot]
    delta = float(deltas[0])
    assert (deltas == delta).all(), "constant step expected with exp_step_factor = 0"
    counts = set(tr.n_samples.tolist())
    assert {0, 1, 31, 32, 33, 127, 128, 129} <= counts, "sample counts must cover the trip edges"
    thr = float(np.float32(tr.cfg.T_threshold))
    targets = [0, 1, 31, 32, 33, 63, 64, 95, 96, 127, 128, 129, 159, 160, 191, 192, 300, 450]
    lanes = set()
    never = 0
    for k in targets:
        h0 = h0_for(k, delta, thr)
        tr.P[2048] = h0  # W2d[0, 0] (the fp16 copy holds it exactly)
        tr.sync_params()
        run_fused(tr, o, d, gt, noise)
        sig = tr.sigmas[:n_tot]
        assert (sig == sig[0]).all(), "density must be constant"
        f = check_fused_batch(tr, gt, 1e-3, "constant sigma %.6g (target k=%d)" % (float(sig[0]), k))
        keep = ~f["undecidable"]
        assert keep.all(), "the controlled terminations are chosen to be decidable"
        term = f["terminated"]
        assert (f["total"][term] == k).all(), "termination must land on sample %d" % k
        if term.any():
            lanes.add(divmod(k, 32))
        never += int((~term & (f["counts"] > 0)).sum())
    for trip in range(5):
        assert (trip, 0) in lanes and (trip, 31) in lanes, trip
    assert any(t >= 5 for t, _ in lanes) and never > 0


def test_separate_kernels_with_depth_and_ws_terms():
    """Trainer(fused_loss=False, materialize_ws=True): k_train_composite_fw's ws / rgb / opacity / depth and
    k_nerf_loss_grad's gradients against float64; then ngp_render_train_bwd with seeded, training-scale dL/drgb,
    dL/dopacity, dL/ddepth and dL/dws into a scratch gradient buffer: dsigmas / drgbs with all four terms"""
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.trainer import Trainer
    L_ = _lib.lib()
    for which, n, random_bg in (("lego", 2053, False), ("mip360", 1029, True)):
        scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
        model = make_model(scene, amp=1.0)
        o_np, d_np = cases.rays_from_scene(scene, n, 59, extra_edge_cases=True)
        o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
        g = torch.Generator("cuda").manual_seed(3)
        gt = torch.rand(n, 3, device="cuda", generator=g)
        noise = torch.rand(n, device="cuda", generator=g)
        bgc = (1.0,) * 3 if scene.exp_step_factor == 0 else (0.0,) * 3
        lam = 1e-3
        tr = Trainer(model, n_rays=n, exp_step_factor=scene.exp_step_factor, bg=bgc, fused_loss=False,
                     materialize_ws=True, random_bg=random_bg)
        assert not tr.fused_loss and tr.ws is not None
        tr.set_batch(o, d, gt)
        tr.noise.copy_(noise)
        tr.march(jitter=False)
        tr.network()
        tr.scalars[2:4].zero_()
        _lib.check(L_.ngp_nerf_loss_grad(C.byref(tr.cfg), C.byref(tr.buf), tr.rgb_gt.data_ptr(), tr.dL_drgb.data_ptr(),
                                         tr.dL_dopacity.data_ptr(), tr._st()), "nerf_loss_grad")
        torch.cuda.synchronize()
        label = "separate %s n=%d random_bg=%s" % (which, n, random_bg)
        n_tot = int(tr.counters[0])
        bg = tr.bg if random_bg else torch.tensor(bgc, device="cuda")
        f = C64.forward(tr.sigmas[:n_tot], tr.rgbs[:n_tot], tr.deltas[:n_tot], tr.ts[:n_tot], tr.offsets, tr.n_samples,
                        tr.cfg.T_threshold, "warp")
        keep = ~f["undecidable"]
        print("%s: %d samples, %d undecidable rays" % (label, n_tot, int((~keep).sum())))
        assert (~keep).sum() <= 0.01 * n
        nl = C64.nerf_loss(f, gt, bg, lam, n)
        within("sep rgb", tr.rgb, nl["out"], nl["out_err"], keep)
        within("sep opacity", tr.opacity, f["O"], f["O_err"], keep)
        within("sep depth", tr.depth, f["D"], f["D_err"], keep)
        within("sep ws", C64.pad(tr.ws[:n_tot], tr.offsets, tr.n_samples, f["L"]), f["w"], f["w_err"], keep)
        within("sep dL_drgb", tr.dL_drgb, nl["dC"], nl["dC_err"], keep)
        within("sep dL_dopacity", tr.dL_dopacity, nl["dL_dopacity"], nl["dL_dopacity_err"], keep)
        assert int(tr.counters[3]) == int(f["total"].sum()) or (~keep).any()

        # seeded upstream gradients at training scale (1 / n_rays), all four terms
        dC = torch.randn(n, 3, device="cuda", generator=g) * (0.5 / n)
        dOp = torch.randn(n, device="cuda", generator=g) * (1e-3 / n)
        dD = torch.randn(n, device="cuda", generator=g) * (0.3 / n)
        dws = torch.randn(tr.capacity, device="cuda", generator=g) * (1e-2 / n)
        ge = torch.zeros(tr.n_enc, device="cuda")
        gr = torch.zeros(tr.n_rgb, device="cuda")
        tr.dsigmas.fill_(float("nan"))
        tr.drgbs.fill_(float("nan"))
        _lib.check(L_.ngp_render_train_bwd(C.byref(tr.net), C.byref(tr.cfg), C.byref(tr.buf), dC.data_ptr(),
                                           dOp.data_ptr(), dD.data_ptr(), dws.data_ptr(), ge.data_ptr(), gr.data_ptr(),
                                           tr._st()), "render_train_bwd")
        torch.cuda.synchronize()
        assert torch.isfinite(tr.dsigmas[:n_tot]).all() and torch.isfinite(tr.drgbs[:n_tot]).all()
        assert ge.abs().max() > 0 and torch.isfinite(ge).all() and torch.isfinite(gr).all()
        b = C64.backward(f, dC, dOp, dD=dD, dws=dws, bg=bg, offsets=tr.offsets)
        b_noD = C64.backward(f, dC, dOp, dws=dws, bg=bg, offsets=tr.offsets)
        dsig, _ = check_backward(tr, f, b, keep, n_tot, label)
        # the depth term is visible: leaving it out of the restatement moves dsig far outside the bound
        assert C64.ratio((dsig - b_noD["dsig"])[keep], b["dsig_err"][keep]) > 10
        check_counts_and_live(tr, f, keep, label)
        check_loss_scale(tr, n_tot, label)
