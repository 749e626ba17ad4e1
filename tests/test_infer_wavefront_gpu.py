"""The inference wavefront (csrc/infer.cu, behind render(test_time=True)) checked one round at a time against a lockstep
replay of the reference's test-time loop (oracle/infer64.py).

Each round runs alone through ngp_render_infer(first_round=k, n_rounds=1); the workspace is read before and after it
through ngp_render_infer_layout. The replay continues from the device's own alive list every round, and the network's
outputs are taken as given (the network is pinned per sample by test_forward_fp64_gpu.py), so one ray whose termination
falls within rounding distance of T_threshold cannot desynchronise the rest. Per round:
  - the quota, `samples`, the round count and the regime are the reference formula's on the device's alive count;
  - every alive ray's sample count, ts, deltas and ray_idx are bitwise the C oracle's raymarching_test, and a ray that
    used its whole quota resumes bitwise at the reference's hits_t;
  - the slot layout: packed, non-overlapping ranges (thread per ray) or rectangular rows with -1 in the unused slots
    (warp per ray); the network evaluated exactly the used slots, with the outputs of a separate ngp_net_forward;
  - opacity, depth and rgb are the float64 compositing of the device's own network outputs within a derived bound, and
    the next alive list holds exactly the rays that took samples and did not reach T_threshold.
At the end total_samples is the replay's sum of N_eff, the background is rgb + bg * (1 - opacity), and the one-graph
ngp_render_infer_frame gives the same bits."""
import ctypes as C

import numpy as np
import pytest
import torch

import cases
from oracle import infer64
from test_fused_gpu import make_model

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD  # a NaN payload no kernel writes
INFER_STAGE = 8        # warp-per-ray marching from this many samples per ray and round on
DENSE = 8.0


def spec(esf, cascades, grid_size=128, max_samples=1024):
    """(CONST_DT, ONE_CASCADE) of march_dispatch for the test-time marcher (its step bound uses `cascades`)"""
    f = np.float32
    const_dt = esf == 0 and f(1.73205080757) / f(max_samples) <= f(cascades) * f(3.46410161514) / f(grid_size)
    return bool(const_dt), cascades == 1


def view_rays(scene, W, H, pose_i=1):
    from ngp_pl_b200 import synth
    K = synth.intrinsics(W=W, H=H, fx=1111.11 * W / 800)
    dirs = synth.ray_directions(K)
    pose = torch.as_tensor(synth.camera_poses(4, radius=synth.camera_radius(scene), upper_only=scene.scale <= 0.5)[pose_i])
    o, d = synth.get_rays(dirs, pose)
    return o.numpy().astype(np.float32).copy(), d.numpy().astype(np.float32).copy()


def splice_edge_rays(scene, o, d, seed=3):
    """cases.rays_from_scene's edge-case rays (axis-parallel, inside the box before the near plane, pointing away, a miss,
    a grazing ray) written over pixels spread through the view, so they land in different warps"""
    eo, ed = cases.rays_from_scene(scene, 16, seed, extra_edge_cases=True)
    at = np.linspace(0, o.shape[0] - 1, 7).astype(np.int64)
    at[0] = 5
    o[at], d[at] = eo[:7], ed[:7]
    return o, d


# name: scene, exp_step_factor (None: the scene's), rays, T_threshold, sample_budget, max_round_samples (None: the
# render() default), table amplitude (a trailing "d": the density output's weights scaled by DENSE, so that sigma spreads
# over orders of magnitude and rays stop on T_threshold at a spread of samples), expected (CONST_DT, ONE_CASCADE)
CASES = {
    "lego_1ray": ("lego", None, 1, 1e-4, 1024, None, 0.3, (True, True)),
    "lego_31rays": ("lego", None, 31, 1e-4, 1024, None, 0.3, (True, True)),
    "lego_33rays": ("lego", None, 33, 1e-4, 1024, None, "1.0d", (True, True)),
    "lego_view100": ("lego", None, (100, 100), 1e-4, 1024, None, 1.0, (True, True)),
    "mip360_view100": ("mip360", None, (100, 100), 1e-4, 1024, None, 1.0, (False, False)),
    "lego_esf256": ("lego", 1.0 / 256, (100, 100), 1e-4, 1024, None, "1.0d", (False, True)),
    "mip360_esf0": ("mip360", 0.0, (100, 100), 1e-4, 1024, None, "1.0d", (True, False)),
    "lego_T1e-2": ("lego", None, (100, 100), 1e-2, 1024, None, "1.0d", (True, True)),
    "mip360_T1e-2": ("mip360", None, (64, 48), 1e-2, 1024, None, "1.0d", (False, False)),
    "lego_budget3": ("lego", None, (100, 100), 1e-4, 3, None, 1.0, (True, True)),
    "mip360_budget20": ("mip360", None, (100, 100), 1e-4, 20, None, 1.0, (False, False)),
    "mip360_clip": ("mip360", None, (100, 100), 1e-4, 1024, "2n", 1.0, (False, False)),
    "lego_view800": ("lego", None, (800, 800), 1e-4, 1024, None, 1.0, (True, True)),
}


class Wavefront:
    """ngp_render_infer on one set of rays, with its workspace readable field by field"""

    def __init__(self, model, cfg, o, d):
        from ngp_pl_b200 import _lib
        from ngp_pl_b200.models.networks import _net_struct
        self.L = _lib.lib()
        self.model, self.cfg, self.o, self.d = model, cfg, o, d
        self.off, size = _lib.infer_layout(cfg.n_rays, cfg.max_round_samples)
        assert size == self.L.ngp_render_infer_workspace(cfg.n_rays, cfg.max_round_samples)
        self.ws = torch.zeros(size, dtype=torch.uint8, device="cuda")
        n = cfg.n_rays
        self.opacity = torch.zeros(n, device="cuda")
        self.depth = torch.zeros(n, device="cuda")
        self.rgb = torch.zeros(n, 3, device="cuda")
        self.total = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.net, self._keep = _net_struct(model)
        self.st = torch.cuda.current_stream().cuda_stream
        self.cap = int(cfg.max_round_samples)

    def field(self, name, dtype, count):
        a = self.off[name]
        return self.ws[a:a + count * 4].view(dtype)

    def host(self, name, dtype, count):
        return self.field(name, dtype, count).cpu().numpy()

    def counters(self):
        c = self.ws[self.off["counters"]:self.off["counters"] + 72].cpu().numpy()
        counts = c[:8].view(np.int32)
        state = c[32:60].view(np.int32).copy()
        total = int(c[64:72].view(np.int64)[0])
        return counts.copy(), state, total

    def run(self, first_round, n_rounds, finish, total_out=None):
        rc = self.L.ngp_render_infer(C.byref(self.net), C.byref(self.cfg), self.o.data_ptr(), self.d.data_ptr(),
                                     self.model.density_bitfield.data_ptr(), self.opacity.data_ptr(), self.depth.data_ptr(),
                                     self.rgb.data_ptr(), total_out.data_ptr() if total_out is not None else None,
                                     first_round, n_rounds, finish, None, self.ws.data_ptr(), self.ws.numel(), self.st)
        assert rc == 0
        torch.cuda.synchronize()

    def net_forward(self, ray_idx, ts):
        """ngp_net_forward on a compact (ray, t) list"""
        from ngp_pl_b200 import _lib
        n = ray_idx.shape[0]
        ridx = torch.as_tensor(ray_idx, dtype=torch.int32, device="cuda").contiguous()
        tt = torch.as_tensor(ts, dtype=torch.float32, device="cuda").contiguous()
        smp = _lib.NgpSamples()
        smp.rays_o, smp.rays_d, smp.ray_idx, smp.ts, smp.n = self.o.data_ptr(), self.d.data_ptr(), ridx.data_ptr(), tt.data_ptr(), n
        sig = torch.empty(max(n, 1), device="cuda")
        rgb = torch.empty(max(n, 1), 3, device="cuda")
        if n:
            _lib.check(self.L.ngp_net_forward(C.byref(self.net), C.byref(smp), 1, sig.data_ptr(), rgb.data_ptr(), None, None,
                                              self.st), "net_forward")
        torch.cuda.synchronize()
        return sig[:n].cpu().numpy(), rgb[:n].cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def build_case(name):
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.models.rendering import MAX_SAMPLES, NEAR_DISTANCE
    which, esf, rays, T_thr, budget, mrs, amp, want_spec = CASES[name]
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    esf = scene.exp_step_factor if esf is None else esf
    if isinstance(rays, tuple):
        o, d = view_rays(scene, *rays)
        o, d = splice_edge_rays(scene, o, d)
    else:
        o, d = cases.rays_from_scene(scene, rays, 21 + rays, extra_edge_cases=rays >= 16)
    n = o.shape[0]
    model = make_model(scene, amp=float(str(amp).rstrip("d")))
    if str(amp).endswith("d"):
        with torch.no_grad():  # row 0 of the density MLP's output layer (16 x 64 after the 64 x 32 input layer): log sigma
            model.xyz_encoder.params[2048:2112] *= DENSE
    cfg = _lib.NgpInferCfg()
    cfg.n_rays, cfg.cascades, cfg.grid_size, cfg.max_samples = n, model.cascades, model.grid_size, MAX_SAMPLES
    cfg.scale, cfg.exp_step_factor, cfg.T_threshold, cfg.near_distance = float(model.scale), float(esf), T_thr, NEAR_DISTANCE
    c, h = model.center.flatten().tolist(), model.half_size.flatten().tolist()
    bg = 1.0 if esf == 0 else 0.0
    for k in range(3):
        cfg.center[k], cfg.half_size[k], cfg.bg[k] = c[k], h[k], bg
    cfg.sample_budget = budget
    cfg.max_round_samples = 2 * n if mrs == "2n" else max(4 * n, 1 << 16)
    assert spec(esf, model.cascades) == want_spec
    return scene, model, cfg, o, d, esf, want_spec


@pytest.mark.parametrize("name", list(CASES))
def test_wavefront_round_by_round_equals_reference_loop(name):
    scene, model, cfg, o_np, d_np, esf, want_spec = build_case(name)
    n = cfg.n_rays
    o, d = torch.as_tensor(o_np).cuda().contiguous(), torch.as_tensor(d_np).cuda().contiguous()
    wf = Wavefront(model, cfg, o, d)
    rp = infer64.InferReplay(o_np, d_np, model.density_bitfield.cpu().numpy(), model.cascades, model.scale, esf,
                             np.asarray(cfg.center, np.float32), np.asarray(cfg.half_size, np.float32),
                             np.float32(cfg.near_distance), sample_budget=cfg.sample_budget,
                             max_round_samples=cfg.max_round_samples)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = wf.cap

    wf.run(0, 0, 0)  # initialisation only: AABB, near clamp, every ray alive, round 0's bookkeeping
    bits_eq = lambda a, b: np.array_equal(bits(a), bits(b))
    assert bits_eq(wf.host("t_cur", torch.float32, n), rp.hits[:, 0]), "t_cur after init differs from ray_aabb + near clamp"
    assert bits_eq(wf.host("t_end", torch.float32, n), rp.hits[:, 1]), "t_end after init differs from ray_aabb"
    assert (wf.host("alive0", torch.int32, n) == np.arange(n)).all()

    n_eff_sum = 0
    regimes = set()
    max_alive = {0: 0, 1: 0}
    clipped = 0
    borderline = 0
    n_term = 0
    flipped = 0
    worst = 0.0
    k = 0
    while True:
        counts, state, total_before = wf.counters()
        n_alive = int(counts[k & 1])
        S = rp.begin_round(n_alive)
        # ---- quota and stop: the reference's formula on the device's alive count ----
        assert int(state[0]) == S, "round %d: quota %d, the reference's %d (n_alive %d)" % (k, state[0], S, n_alive)
        if S == 0:
            break
        assert int(state[1]) == rp.samples and int(state[3]) == rp.rounds == k + 1
        assert int(state[6]) == 0
        assert int(state[5]) == int(S >= INFER_STAGE)
        warp = S >= INFER_STAGE
        regimes.add(int(warp))
        max_alive[int(warp)] = max(max_alive[int(warp)], n_alive)
        min_samples = 1 if esf == 0 else 4
        if S < max(min(n // n_alive, 64), min_samples):
            clipped += 1
        alive = wf.host("alive%d" % (k & 1), torch.int32, n_alive).astype(np.int64)
        op_b = wf.opacity.cpu().numpy()
        dp_b = wf.depth.cpu().numpy()
        rgb_b = wf.rgb.cpu().numpy()
        wf.field("sigmas", torch.int32, cap).fill_(SENTINEL)
        wf.field("rgbs", torch.int32, 3 * cap).fill_(SENTINEL)

        wf.run(k, 1, 0)

        counts_a, state_a, total_after = wf.counters()
        m = rp.march(alive, S)
        ne = m["n_eff"].astype(np.int64)
        ray_start = wf.host("ray_start", torch.int32, n_alive).astype(np.int64)
        ray_n = wf.host("ray_n", torch.int32, n_alive).astype(np.int64)
        assert (ray_n == ne).all(), "round %d: ray_n differs from raymarching_test's N_eff for rays %s" % (
            k, alive[ray_n != ne][:8])
        marched = int(ne.sum())
        n_eff_sum += marched
        assert total_after - total_before == marched  # state[4] of the round, folded into the total
        used = n_alive * S if warp else marched
        assert used <= cap
        ray_idx = wf.host("ray_idx", torch.int32, max(used, 1))[:used]
        ts = wf.host("ts", torch.float32, max(used, 1))[:used]
        deltas = wf.host("deltas", torch.float32, max(used, 1))[:used]
        # ---- samples: every alive ray's slots hold raymarching_test's row, bit for bit ----
        jj = np.arange(S)[None, :]
        mask = jj < ne[:, None]
        slots = (ray_start[:, None] + jj)[mask]
        assert (ray_idx[slots] == np.broadcast_to(alive[:, None], mask.shape)[mask]).all()
        assert bits_eq(ts[slots], m["ts"][mask]), "round %d: ts differ from raymarching_test's" % k
        assert bits_eq(deltas[slots], m["deltas"][mask]), "round %d: deltas differ from raymarching_test's" % k
        if warp:
            assert (ray_start == np.arange(n_alive) * S).all()
            assert (ray_idx.reshape(n_alive, S)[~mask] == -1).all(), "round %d: unused slots not marked -1" % k
        else:
            nz = ray_n > 0
            order = np.argsort(ray_start[nz], kind="stable")
            st, ln = ray_start[nz][order], ray_n[nz][order]
            assert marched == 0 or (st[0] == 0 and (st[1:] == st[:-1] + ln[:-1]).all() and st[-1] + ln[-1] == marched), \
                "round %d: the claimed sample ranges overlap or leave gaps" % k
        # ---- resume point ----
        t_cur = wf.host("t_cur", torch.float32, n)
        t_end = wf.host("t_end", torch.float32, n)
        full = ne == S
        assert bits_eq(t_cur[alive[full]], rp.hits[alive[full], 0]), "round %d: resume point differs from hits_t" % k
        out = alive[~full]
        assert (t_cur[out] >= t_end[out]).all(), "round %d: a ray that took fewer than S samples is still in the box" % k
        assert not rp.samples_left(out).any(), "round %d: the reference would march more samples for a ray left out" % k
        # ---- network plumbing: the used slots, exactly, with a separate forward's outputs ----
        sig_ws = wf.field("sigmas", torch.float32, cap)
        rgb_ws = wf.field("rgbs", torch.float32, 3 * cap)
        assert (sig_ws.view(torch.int32)[used:] == SENTINEL).all() and (rgb_ws.view(torch.int32)[3 * used:] == SENTINEL).all(), \
            "round %d: the network wrote past the %d slots of the round" % (k, used)
        sig_dev = sig_ws[:used].cpu().numpy()
        rgb_dev = rgb_ws[:3 * used].cpu().numpy().reshape(-1, 3)
        valid = ray_idx >= 0
        s_ref, c_ref = wf.net_forward(ray_idx[valid], ts[valid])
        assert bits_eq(sig_dev[valid], s_ref) and bits_eq(rgb_dev[valid], c_ref), \
            "round %d: the wavefront's network outputs differ from ngp_net_forward on the same (ray, t)" % k
        # ---- compositing and the next alive list ----
        sig_r = np.zeros((n_alive, S), np.float32)
        rgb_r = np.zeros((n_alive, S, 3), np.float32)
        sig_r[mask] = sig_dev[slots]
        rgb_r[mask] = rgb_dev[slots]
        comp = infer64.composite64(sig_r, rgb_r, m["deltas"], m["ts"], ne, op_b[alive], dp_b[alive], rgb_b[alive],
                                   cfg.T_threshold)
        n_next = int(counts_a[(k + 1) & 1])
        op_a = wf.opacity.cpu().numpy()
        got = (op_a[alive], wf.depth.cpu().numpy()[alive], wf.rgb.cpu().numpy()[alive])
        if rp.samples >= cfg.sample_budget:
            # the bookkeeping after this round ends the loop on the budget and clears the next alive count, so the
            # device's termination decisions are not observable: either must match
            assert n_next == 0
            ok_t, jt_t, ratio_t = infer64.composite_match(comp, *got, np.ones(n_alive, bool) & (ne > 0))
            ok_f, jt_f, ratio_f = infer64.composite_match(comp, *got, np.zeros(n_alive, bool))
            ok, jt, ratio = ok_t | ok_f, np.where(ok_t, jt_t, jt_f), np.minimum(ratio_t, ratio_f)
            term = ok_t & (ne > 0)
        else:
            nxt = wf.host("alive%d" % ((k + 1) & 1), torch.int32, n_next).astype(np.int64)
            assert len(np.unique(nxt)) == n_next and np.isin(nxt, alive).all(), "round %d: the next alive list is not a set" % k
            kept = np.isin(alive, nxt)
            assert (ne[kept] > 0).all(), "round %d: a ray without samples stayed alive" % k
            term = ~kept & (ne > 0)
            ok, jt, ratio = infer64.composite_match(comp, *got, term)
        n_term += int(term.sum())
        assert ok.all(), "round %d: %d rays' compositing or termination disagrees with the float64 replay, e.g. ray %d " \
            "(opacity %r vs %r, T_threshold band %s, device stopped: %s)" % (
                k, (~ok).sum(), alive[~ok][0], op_a[alive][~ok][0], comp["O"][~ok][0], (comp["jt_lo"][~ok][0],
                                                                                         comp["jt_hi"][~ok][0]), term[~ok][0])
        band = comp["jt_lo"] < comp["jt_hi"]
        borderline += int(band.sum())
        flipped += int((band & (jt != comp["jt_lo"])).sum())
        worst = max(worst, float(ratio[np.isfinite(ratio)].max(initial=0.0)))
        k += 1
        assert k <= 2 * cfg.sample_budget + 2

    # ---- end of the run ----
    assert rp.samples >= cfg.sample_budget or int(wf.counters()[0][k & 1]) == 0
    op_e, dp_e, rgb_e = wf.opacity.cpu().numpy(), wf.depth.cpu().numpy(), wf.rgb.cpu().numpy()
    total_out = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    wf.run(k, 0, 1, total_out)
    assert int(total_out.item()) == n_eff_sum
    bg = np.asarray(cfg.bg, np.float32)
    want = rgb_e + bg[None, :] * (np.float32(1) - op_e)[:, None]
    assert bits_eq(wf.rgb.cpu().numpy(), want) and bits_eq(wf.opacity.cpu().numpy(), op_e) and bits_eq(wf.depth.cpu().numpy(), dp_e)
    # the one-graph frame on the same inputs
    fr = Wavefront(model, cfg, o, d)
    rc = fr.L.ngp_render_infer_frame(C.byref(fr.net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                     fr.opacity.data_ptr(), fr.depth.data_ptr(), fr.rgb.data_ptr(), fr.total.data_ptr(),
                                     fr.ws.data_ptr(), fr.ws.numel(), fr.st)
    assert rc == 0
    torch.cuda.synchronize()
    assert int(fr.total.item()) == n_eff_sum
    for a, b in ((fr.opacity, wf.opacity), (fr.depth, wf.depth), (fr.rgb, wf.rgb)):
        assert torch.equal(a, b)

    # ---- what the case reached ----
    print("\n%s: spec CONST_DT=%d ONE_CASCADE=%d, %d rounds, total_samples %d, regimes %s, max alive thread/warp %d/%d, "
          "clipped rounds %d, rays stopped by T_threshold %d, in its rounding band %d (device chose the later stop for %d), "
          "worst error/tolerance %.3g" % (name, want_spec[0], want_spec[1], k, n_eff_sum, sorted(regimes), max_alive[0],
                                          max_alive[1], clipped, n_term, borderline, flipped, worst))
    if "T1e-2" in name:
        assert n_term > 0, "rays should stop on T_threshold"
    if cfg.sample_budget >= 1024 and n >= 1000:
        assert regimes == {0, 1}, "both marching regimes should run"
    if name.endswith("clip"):
        assert clipped > 0, "max_round_samples should have clipped the quota"
    if name.endswith("view800"):
        assert max_alive[0] > sms * 16 * 128, "the thread-per-ray and compositing grids should stride"
        assert max_alive[1] > sms * 64, "the warp-per-ray grid should stride"
