"""The distortion loss, k_distortion_fw / k_distortion_bw, ray by ray and sample by sample against the float64
restatement oracle/distortion64.py, and the training step at a sample capacity smaller than what its batch marches.

  * The entry points directly (ngp_distortion_loss_fw / _bw, what vren and NeRFLoss call): every ray length from 0 to
    3000, segments in scrambled order with gaps, rows permuted against ray ids, an odd ray count, exact-zero tails, an
    all-zero ray and a weight near 1, on Lego's constant step and a scale-16 scene's exponential step (t to ~50, where
    the formula cancels most). Outputs are NaN-prefilled, so a skipped sample fails; the gaps stay untouched.
  * Segments that cross the arrays' extent n_samples: clipped to it, and the guard region past it is untouched.
  * The Trainer's distortion path (lambda_distortion > 0): per-ray loss and dL/dws against float64, then the compositing
    backward fed the kernel's own dL/dws against composite64, and the loss the step reports.
  * The capacity: max_total_samples below the marched total, first inside larger buffers guarded by a sentinel, then with
    buffers of exactly that size. Every consumer of the sample arrays clips each ray's segment to the capacity.
"""
import pytest
import torch

import cases
from oracle import composite64 as C64
from oracle import distortion64 as D64
from test_fused_gpu import make_model

pytestmark = pytest.mark.gpu

SENT_BITS = 0x7FC0BEEF  # a quiet NaN with a payload no kernel writes: the float buffers' sentinel, compared as bits
SENT_INT = -0x0BADBEE   # the int buffers' sentinel
RATIOS = {}  # quantity -> largest error / (SAFETY bound) over the module's cases
RELERR = {}  # case -> largest |loss error| / |loss| over rays with a loss above 1e-6


def note(name, r):
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)
    assert r <= 1.0, "%s: error / bound = %.3g" % (name, r)


def within(name, mine, ref, err, keep):
    note(name, C64.ratio((mine.double() - ref)[keep], err[keep]))


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nMEASURED distortion loss and capacity vs float64, largest error / (%g x bound):" % C64.SAFETY)
    for k in sorted(RATIOS):
        print("  %-28s %.3g" % (k, RATIOS[k]))
    print("MEASURED distortion loss, largest relative error per case (rays with loss > 1e-6):")
    for k in sorted(RELERR):
        print("  %-28s %.3g" % (k, RELERR[k]))


def sentinel_f32():
    return torch.tensor([SENT_BITS], dtype=torch.int32).view(torch.float32)


def run_fused(tr, o, d, gt, noise):
    """one eager step's march and weight-dependent part (no optimiser)"""
    tr.set_batch(o, d, gt)
    tr.noise.copy_(noise)
    tr.march(jitter=False)
    tr._compute()
    torch.cuda.synchronize()


def call_fw(ws, deltas, ts, rays_a, n_samples, loss, wi, wti):
    from ngp_pl_b200 import _lib
    _lib.check(_lib.lib().ngp_distortion_loss_fw(ws.data_ptr(), deltas.data_ptr(), ts.data_ptr(), rays_a.data_ptr(),
                                                 rays_a.shape[0], n_samples, loss.data_ptr(), wi.data_ptr(), wti.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream), "distortion_fw")


def call_bw(g, wi, wti, ws, deltas, ts, rays_a, n_samples, dws):
    from ngp_pl_b200 import _lib
    _lib.check(_lib.lib().ngp_distortion_loss_bw(g.data_ptr(), wi.data_ptr(), wti.data_ptr(), ws.data_ptr(),
                                                 deltas.data_ptr(), ts.data_ptr(), rays_a.data_ptr(), rays_a.shape[0],
                                                 n_samples, dws.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "distortion_bw")


def nan_like(n):
    return sentinel_f32().cuda().expand(n).contiguous()


def by_ray(rays_a):
    off = torch.zeros(rays_a.shape[0], dtype=torch.long, device=rays_a.device)
    cnt = torch.zeros_like(off)
    off[rays_a[:, 0]] = rays_a[:, 1]
    cnt[rays_a[:, 0]] = rays_a[:, 2]
    return off, cnt


def check_distortion(label, f, b, off, cnt, loss, wi, wti, dws):
    """per-ray loss (by ray) and per-sample scans / dL/dws against the restatement; returns the worst relative loss error"""
    L = f["L"]
    v = f["valid"]
    within("loss", loss, f["loss"], f["loss_err"], torch.ones_like(cnt, dtype=torch.bool))
    within("ws_inc", C64.pad(wi, off, cnt, L)[v], f["W"][v], f["W_err"][v], slice(None))
    within("wts_inc", C64.pad(wti, off, cnt, L)[v], f["WT"][v], f["WT_err"][v], slice(None))
    within("dL_dws", C64.pad(dws, off, cnt, L)[v], b["dws"][v], b["dws_err"][v], slice(None))
    big = f["loss"].abs() > 1e-6
    rel = float(((loss.double() - f["loss"]).abs()[big] / f["loss"][big].abs()).max()) if big.any() else 0.0
    RELERR[label] = max(RELERR.get(label, 0.0), rel)
    return rel


def covered(rays_a, n):
    """mask of the sample slots [0, n) that some ray's segment covers"""
    m = torch.zeros(n + 1, dtype=torch.int32, device=rays_a.device)
    s, c = rays_a[:, 1], rays_a[:, 2]
    m.index_add_(0, s.clamp(max=n), torch.ones_like(s, dtype=torch.int32))
    m.index_add_(0, (s + c).clamp(max=n), -torch.ones_like(s, dtype=torch.int32))
    return torch.cumsum(m, 0)[:n] > 0


def bits(x):
    return x.contiguous().view(torch.int32)


@pytest.mark.parametrize("profile", ["lego", "exp16"])
def test_entry_points_every_length(profile):
    c = cases.distortion_case(11, profile)
    ws, ts, dl = (torch.as_tensor(c[k]).cuda() for k in ("ws", "ts", "deltas"))
    ra = torch.as_tensor(c["rays_a"]).cuda()
    R, n = ra.shape[0], ws.numel()
    g = torch.randn(R, device="cuda", generator=torch.Generator("cuda").manual_seed(7)) * 1e-3
    loss, wi, wti, dws = nan_like(R), nan_like(n), nan_like(n), nan_like(n)
    call_fw(ws, dl, ts, ra, n, loss, wi, wti)
    call_bw(g, wi, wti, ws, dl, ts, ra, n, dws)
    torch.cuda.synchronize()
    off, cnt = by_ray(ra)
    f = D64.forward(ws, dl, ts, off, cnt)
    b = D64.backward(f, g)
    assert torch.isfinite(loss).all()
    rel = check_distortion(profile, f, b, off, cnt, loss, wi, wti, dws)
    # the gaps between segments: untouched
    gap = ~covered(ra, n)
    assert gap.sum() >= R
    for x in (wi, wti, dws):
        assert (bits(x)[gap] == SENT_BITS).all()
    # empty rays: loss exactly 0; the all-zero ray: exactly 0 everywhere
    assert (loss[ra[ra[:, 2] == 0, 0]] == 0).all()
    z = c["special"]["zero"]
    zr, zs = int(ra[z, 0]), int(ra[z, 1])
    assert float(loss[zr]) == 0 and not dws[zs:zs + 64].any() and not wi[zs:zs + 64].any()
    print("%s: %d rays, %d samples, largest relative loss error %.3g" % (profile, R, int(cnt.sum()), rel))


def test_entry_points_clip_to_the_extent():
    """n_samples below the end of some segments: each ray is clipped to it; NaN inputs and sentinel outputs past it"""
    c = cases.distortion_case(12, "exp16")
    ws, ts, dl = (torch.as_tensor(c[k]).cuda() for k in ("ws", "ts", "deltas"))
    ra = torch.as_tensor(c["rays_a"]).cuda()
    R, n = ra.shape[0], ws.numel()
    # the extent: halfway into the long segment that starts nearest the middle of the buffer, so that one ray straddles
    # it and many lie past it
    long_rows = torch.nonzero(ra[:, 2] >= 63)[:, 0]
    row = long_rows[(ra[long_rows, 1] - n // 2).abs().argmin()]
    ext = int(ra[row, 1] + ra[row, 2] // 2)
    for x in (ws, ts, dl):
        x[ext:] = float("nan")
    g = torch.randn(R, device="cuda", generator=torch.Generator("cuda").manual_seed(8)) * 1e-3
    loss, wi, wti, dws = nan_like(R), nan_like(n), nan_like(n), nan_like(n)
    call_fw(ws, dl, ts, ra, ext, loss, wi, wti)
    call_bw(g, wi, wti, ws, dl, ts, ra, ext, dws)
    torch.cuda.synchronize()
    for x in (wi, wti, dws):
        assert (bits(x)[ext:] == SENT_BITS).all(), "a write past the extent"
    off, cnt_full = by_ray(ra)
    cnt = torch.minimum(cnt_full, (ext - off).clamp_min(0))
    past = (cnt == 0) & (cnt_full > 0)
    straddle = (cnt > 0) & (cnt < cnt_full)
    assert past.sum() >= 5 and straddle.any()
    assert (loss[past] == 0).all()
    f = D64.forward(ws[:ext], dl[:ext], ts[:ext], off, cnt)
    b = D64.backward(f, g)
    check_distortion("clipped", f, b, off, cnt, loss, wi, wti, dws)
    # with the full extent the same call writes the whole straddling segment
    call_fw(ws, dl, ts, ra, n, loss, wi, wti)
    torch.cuda.synchronize()
    assert not torch.isfinite(loss[straddle]).all()


# ---- the Trainer --------------------------------------------------------------------------------------------------
def scene_model(which):
    from ngp_pl_b200 import synth
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    return scene, make_model(scene, amp=1.0)


def trained_lego():
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
    torch.cuda.synchronize()
    return scene, model, bank


def batch(scene, n, seed, bank=None):
    if bank is not None:
        o, d, gt = bank.sample(n)
    else:
        o_np, d_np = cases.rays_from_scene(scene, n, seed, extra_edge_cases=True)
        o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
        gt = torch.rand(n, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))
    noise = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(seed + 1))
    return o, d, gt, noise


def background(tr, scene_bg):
    return tr.bg if tr.random_bg else torch.tensor(scene_bg, device="cuda")


def clipped_counts(tr, cap):
    off, cnt = tr.offsets.long(), tr.n_samples.long()
    return off, torch.minimum(cnt, (cap - off).clamp_min(0))


def check_step(tr, gt, bgc, cap, label):
    """everything the step wrote against float64 over each ray's segment clipped to cap (cap = the capacity)"""
    n = tr.n_rays
    off, cnt = clipped_counts(tr, cap)
    lam = tr.cfg.lambda_opacity
    bg = background(tr, bgc)
    f = C64.forward(tr.sigmas[:cap], tr.rgbs[:cap], tr.deltas[:cap], tr.ts[:cap], off, cnt, tr.cfg.T_threshold, "warp")
    keep = ~f["undecidable"]
    n_und = int((~keep).sum())
    assert n_und <= 0.01 * n, label
    nl = C64.nerf_loss(f, gt, bg, lam, n)
    within("rgb", tr.rgb, nl["out"], nl["out_err"], keep)
    within("opacity", tr.opacity, f["O"], f["O_err"], keep)
    within("depth", tr.depth, f["D"], f["D_err"], keep)
    dws = None
    if tr.lambda_distortion > 0:
        fd = D64.forward(tr.ws[:cap], tr.deltas[:cap], tr.ts[:cap], off, cnt)
        bd = D64.backward(fd, tr.dist_dL)
        L = fd["L"]
        v = fd["valid"]
        within("trainer dist_loss", tr.dist_loss, fd["loss"], fd["loss_err"], torch.ones(n, dtype=torch.bool, device="cuda"))
        within("trainer dL_dws", C64.pad(tr.dL_dws[:cap], off, cnt, L)[v], bd["dws"][v], bd["dws_err"][v], slice(None))
        dws = tr.dL_dws
        mean64 = float(fd["loss"].sum()) / n
        err = (float(fd["loss_err"].sum()) + float(C64.gamma(n)) * float(fd["loss"].abs().sum())) / n
        lamd = tr.lambda_distortion
        note("stats distortion", abs(tr.stats()["distortion"] - lamd * mean64) / (C64.SAFETY * lamd * err + 1e-300))
    if tr.fused_loss:
        b = C64.backward(f, nl["dC"], nl["dO"], dC_err=nl["dC_err"], dO_err=nl["dO_err"])
    else:
        within("dL_drgb", tr.dL_drgb, nl["dC"], nl["dC_err"], keep)
        within("dL_dopacity", tr.dL_dopacity, nl["dL_dopacity"], nl["dL_dopacity_err"], keep)
        b = C64.backward(f, tr.dL_drgb, tr.dL_dopacity, dws=dws, bg=bg, offsets=off)
    # check_backward pads with the trainer's own counts: restate with the clipped ones
    dsig = C64.pad(tr.dsigmas[:cap], off, cnt, f["L"])
    drgb = C64.pad(tr.drgbs[:cap], off, cnt, f["L"])
    within("dsigmas", dsig, b["dsig"], b["dsig_err"], keep)
    within("drgbs", drgb, b["drgb"], b["drgb_err"], keep)
    past = (f["valid"] & ~f["comp"])[keep]
    if past.any():
        assert dsig[keep][past].abs().max().item() == 0 and drgb[keep][past].abs().max().item() == 0, label
    # the live list: inside the capacity, exactly the composited samples of the clipped segments
    nb = int(tr.counters[5])
    live = tr.live_idx[:nb].long()
    assert (live >= 0).all() and (live < cap).all(), label
    assert live.unique().numel() == nb
    assert nb == int(f["n_comp"].sum()) or n_und, label
    return f, off, cnt


@pytest.fixture(scope="module")
def trained():
    return trained_lego()


@pytest.mark.parametrize("which,lam", [("lego", 1e-3), ("lego", 1e-2), ("mip360", 1e-3), ("mip360", 1e-2),
                                       ("trained", 1e-3), ("trained", 1e-2)])
def test_trainer_distortion_path(which, lam, request):
    from ngp_pl_b200.trainer import Trainer
    if which == "trained":
        scene, model, bank = request.getfixturevalue("trained")
    else:
        (scene, model), bank = scene_model(which), None
    n = 2053 if which != "mip360" else 1029
    bgc = (1.0,) * 3 if scene.exp_step_factor == 0 else (0.0,) * 3
    tr = Trainer(model, n_rays=n, exp_step_factor=scene.exp_step_factor, bg=bgc, lambda_distortion=lam, log_rows=2)
    assert not tr.fused_loss
    o, d, gt, noise = batch(scene, n, 61, bank)
    run_fused(tr, o, d, gt, noise)
    n_tot = int(tr.counters[0])
    assert n_tot == int(tr.n_samples.sum()) and n_tot > 0
    label = "trainer %s lambda_distortion=%g" % (which, lam)
    check_step(tr, gt, bgc, n_tot, label)
    # the step's log row carries the same distortion (a double sum of the fp32 per-ray losses, then fp32)
    off, cnt = tr.offsets.long(), tr.n_samples.long()
    fd = D64.forward(tr.ws[:n_tot], tr.deltas[:n_tot], tr.ts[:n_tot], off, cnt)
    tr.step_dev.fill_(1)  # as the step's Adam leaves it: the row of step 0
    tr._log_step()
    tr.host_step += 1
    rows = tr.drain_log(wait=True)
    assert len(rows) == 1
    want = lam * float(fd["loss"].sum()) / n
    err = lam * (float(fd["loss_err"].sum()) + float(C64.gamma(n)) * float(fd["loss"].abs().sum())) / n + 2 ** -24 * abs(want)
    note("log row distortion", abs(rows[0]["distortion"] - want) / (C64.SAFETY * err))
    big = fd["loss"].abs() > 1e-6
    if big.any():
        rel = float(((tr.dist_loss.double() - fd["loss"]).abs()[big] / fd["loss"][big].abs()).max())
        RELERR[which] = max(RELERR.get(which, 0.0), rel)
    print("%s: %d rays, %d samples, mean distortion %.4g" % (label, n, n_tot, float(fd["loss"].mean())))


# ---- the capacity -------------------------------------------------------------------------------------------------
PATHS = {"fused": dict(), "separate": dict(fused_loss=False, materialize_ws=True), "distortion": dict(lambda_distortion=1e-2)}
GUARDED = ("ts", "deltas", "ray_idx", "sigmas", "rgbs", "ws", "ws_inc", "wts_inc", "dL_dws", "dsigmas", "drgbs", "live_idx")


def fill_guard(tr, cap):
    guarded = {}
    for name in GUARDED:
        x = getattr(tr, name, None)
        if x is None:
            continue
        x = x.view(x.shape[0], -1)
        if x.dtype == torch.float32:
            x[cap:] = sentinel_f32().cuda()
        else:
            x[cap:] = SENT_INT
        guarded[name] = x
    return guarded


def check_guard(guarded, cap, label):
    for name, x in guarded.items():
        want = SENT_BITS if x.dtype == torch.float32 else SENT_INT
        bad = int((bits(x[cap:]) != want).sum())
        assert bad == 0, "%s: %d entries of %s past the capacity %d changed" % (label, bad, name, cap)


def capacity_step(tr, o, d, gt, noise, cap, marched):
    """one eager step at capacity cap; the marched counts are those of the batch at full capacity"""
    run_fused(tr, o, d, gt, noise)
    assert torch.equal(tr.n_samples.long(), marched), "n_samples keeps the marched counts"
    assert int(tr.counters[0]) == min(int(marched.sum()), cap)
    if tr.fused_loss:
        assert tr.stats()["rm_samples"] == min(int(marched.sum()), cap)


@pytest.mark.parametrize("path", sorted(PATHS))
def test_capacity_below_the_marched_total_guarded(path):
    """the Trainer's buffers at full size, max_total_samples lowered to ~60 % of the marched total, a sentinel from there
    to the end of every per-sample buffer: nothing past the capacity changes and every ray is its clipped segment"""
    from ngp_pl_b200.trainer import Trainer
    scene, model = scene_model("lego")
    n = 2053
    bgc = (1.0,) * 3
    tr = Trainer(model, n_rays=n, bg=bgc, **PATHS[path])
    o, d, gt, noise = batch(scene, n, 67)
    run_fused(tr, o, d, gt, noise)
    marched = tr.n_samples.long().clone()
    total = int(marched.sum())
    # the rays arrive in a different order every run, and a capacity that lands exactly on the end of a ray's segment
    # (about 1 run in 40 here) leaves no ray straddling it: then the step is checked as it is and taken again one sample
    # lower, until some ray straddles the capacity
    for attempt in range(4):
        cap = int(0.6 * total) - attempt
        tr.cfg.max_total_samples = cap
        tr.capacity = cap
        guarded = fill_guard(tr, cap)
        capacity_step(tr, o, d, gt, noise, cap, marched)
        label = "guarded %s cap=%d of %d" % (path, cap, total)
        check_guard(guarded, cap, label)
        _, off, cnt = check_step(tr, gt, bgc, cap, label)
        full = tr.n_samples.long()
        past = (cnt == 0) & (full > 0)
        straddle = (cnt > 0) & (cnt < full)
        if straddle.sum() >= 1:
            break
        # no straddling ray: the capacity is exactly the end of one ray's segment
        assert bool(((off + cnt == cap) & (cnt == full) & (cnt > 0)).any()), label
    assert past.sum() > 10 and straddle.sum() >= 1, label
    # a ray past the capacity renders the background alone
    assert (tr.opacity[past] == 0).all() and (tr.rgb[past] == torch.tensor(bgc, device="cuda")).all()
    if tr.lambda_distortion > 0:
        assert (tr.dist_loss[past] == 0).all()
    print("%s: %d rays past the capacity, %d straddling it" % (label, int(past.sum()), int(straddle.sum())))


@pytest.mark.parametrize("path", sorted(PATHS))
def test_capacity_small_buffers(path):
    """Trainer(max_total_samples=cap): buffers of exactly cap samples, checked against its own offsets (the arrival
    order, and with it which rays are cut, changes from run to run)"""
    from ngp_pl_b200.trainer import Trainer
    scene, model = scene_model("lego")
    n = 2053
    bgc = (1.0,) * 3
    o, d, gt, noise = batch(scene, n, 67)
    probe = Trainer(model, n_rays=n, bg=bgc)
    probe.set_batch(o, d, gt)
    probe.noise.copy_(noise)
    probe.march(jitter=False)
    marched = probe.n_samples.long().clone()
    total = int(marched.sum())
    del probe
    cap = int(0.6 * total)
    tr = Trainer(model, n_rays=n, bg=bgc, max_total_samples=cap, **PATHS[path])
    assert tr.sigmas.shape[0] == cap and tr.ts.shape[0] == cap
    capacity_step(tr, o, d, gt, noise, cap, marched)
    label = "small buffers %s cap=%d of %d" % (path, cap, total)
    _, off, cnt = check_step(tr, gt, bgc, cap, label)
    full = tr.n_samples.long()
    assert ((cnt == 0) & (full > 0)).sum() > 10, label
