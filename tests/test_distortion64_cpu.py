"""oracle/distortion64.py, the float64 distortion-loss restatement the GPU tests hold k_distortion_fw / k_distortion_bw
to, and its rounding bound: the scan identity equals the definition's pair sums, the values agree with the C oracle and
with the reference kernels' own outputs (tests/golden/composite.npz) inside the serial-order bound, and a float32 replay
of the two kernels' exact order -- a 32-lane Hillis-Steele scan with carries, per-lane accumulators and an xor butterfly,
with and without fused multiply-adds -- lies inside the warp-order bound at every ray length the GPU tests use.
A bound that does not cover the reference's own kernels is wrong.
"""
import os

import numpy as np
import pytest
import torch

import cases
from oracle import distortion64 as D64
from test_composite64_cpu import by_ray

F = np.float32
C3, C23 = F(1.0) / F(3.0), F(2.0) / F(3.0)


def T(x):
    return torch.as_tensor(np.ascontiguousarray(x))


def within(name, mine, ref, err, valid=None):
    mine, ref, err = (torch.as_tensor(v).double() for v in (mine, ref, err))
    d = mine - ref
    if valid is not None:
        d, err = d[valid], err[valid]
    assert torch.isfinite(err).all(), name
    r = D64.ratio(d, err)
    assert r <= 1.0, "%s: error / bound = %.3g" % (name, r)
    return r


def oracle64(ws, deltas, ts, rays_a, order, g=None):
    off, cnt = by_ray(rays_a)
    f = D64.forward(T(ws), T(deltas), T(ts), off, cnt, order)
    b = D64.backward(f, T(g)) if g is not None else None
    return f, b, off, cnt


def check_outputs(name, f, b, off, cnt, loss, ws_inc, wts_inc, dws=None):
    """per-ray loss (indexed by ray) and per-sample scans / dL_dws (flat) against the restatement"""
    L = f["L"]
    rs = {"loss": within(name + " loss", loss, f["loss"], f["loss_err"]),
          "ws_inc": within(name + " ws_inc", D64.pad(T(ws_inc), off, cnt, L), f["W"], f["W_err"], f["valid"]),
          "wts_inc": within(name + " wts_inc", D64.pad(T(wts_inc), off, cnt, L), f["WT"], f["WT_err"], f["valid"])}
    if dws is not None:
        rs["dws"] = within(name + " dws", D64.pad(T(dws), off, cnt, L), b["dws"], b["dws_err"], f["valid"])
    return rs


# ---- the two kernels' order, replayed in float32 ------------------------------------------------------------------
def _fma(a, b, c):
    return (a.astype(np.float64) * b + c).astype(F)


def _scan_add(v):
    """inclusive Hillis-Steele scan over the last axis (32 lanes), warp_scan_add's association order"""
    o = 1
    while o < 32:
        v = v + np.concatenate([np.zeros(v.shape[:-1] + (o,), F), v[..., :-o]], -1)
        o <<= 1
    return v


def _butterfly(v):
    """warp_sum: xor butterfly over the last axis, lane 0's value"""
    o = 16
    while o > 0:
        v = v + v[..., np.arange(32) ^ o]
        o >>= 1
    return v[..., 0]


def replay(ws, deltas, ts, rays_a, g, contract):
    """k_distortion_fw then k_distortion_bw, every ray at once -> loss (by ray), ws_inc, wts_inc, dL_dws (flat)"""
    off, cnt = (x.numpy() for x in by_ray(rays_a))
    R = len(cnt)
    trips = max(1, -(-int(cnt.max()) // 32))
    Lp = 32 * trips
    pos = np.arange(Lp)
    valid = pos[None] < cnt[:, None]
    idx = np.where(valid, off[:, None] + pos[None], 0)
    w = np.where(valid, ws[idx], F(0)).astype(F)
    t = np.where(valid, ts[idx], F(0)).astype(F)
    d = np.where(valid, deltas[idx], F(0)).astype(F)
    W, WT = np.zeros((R, Lp), F), np.zeros((R, Lp), F)
    cw, cwt, acc = np.zeros((R, 1), F), np.zeros((R, 1), F), np.zeros((R, 32), F)
    for k in range(trips):
        sl = slice(32 * k, 32 * k + 32)
        wi, v = w[:, sl], valid[:, sl]
        wt = np.where(v, wi * t[:, sl], F(0)).astype(F)
        wi_inc = _scan_add(wi) + cw
        wt_inc = _scan_add(wt) + cwt
        wi_exc, wt_exc = wi_inc - wi, wt_inc - wt
        q = (C3 * wi) * wi
        if contract:
            # what nvcc makes of it: fma(WT, Wx, -fl(W WTx)), then fma(D, 2, fl(q d))
            term = F(2) * _fma(wt_inc, wi_exc, -(wi_inc * wt_exc)) + q * d[:, sl]
        else:
            term = F(2) * (wt_inc * wi_exc - wi_inc * wt_exc) + q * d[:, sl]
        acc = np.where(v, acc + term, acc)
        W[:, sl], WT[:, sl] = wi_inc, wt_inc
        cw, cwt = wi_inc[:, 31:], wt_inc[:, 31:]
    loss = _butterfly(acc)
    # backward: per sample, from the stored scans
    last = np.maximum(cnt - 1, 0)[:, None]
    Wn, WTn = np.take_along_axis(W, last, 1), np.take_along_axis(WT, last, 1)
    Wp = np.concatenate([np.zeros((R, 1), F), W[:, :-1]], 1)
    WTp = np.concatenate([np.zeros((R, 1), F), WT[:, :-1]], 1)
    gg = g[:, None].astype(F)
    if contract:
        head = np.where(pos[None] == 0, F(0), _fma(t, Wp, -WTp))
        tail = _fma(-t, Wn - W, WTn - WT)
        dws = _fma((gg * C23) * w, d, (gg * F(2)) * (head + tail))
    else:
        head = np.where(pos[None] == 0, F(0), t * Wp - WTp)
        tail = (WTn - WT) - t * (Wn - W)
        dws = (gg * F(2)) * (head + tail) + ((gg * C23) * w) * d
    out = [np.full(len(ws), np.nan, F) for _ in range(3)]
    for o, x in zip(out, (W, WT, dws)):
        o[idx[valid]] = x[valid]
    return loss, out[0], out[1], out[2]


# ---- tests --------------------------------------------------------------------------------------------------------
def test_case_layout():
    """the shared GPU case: every length of the list, an odd ray count, gaps, rows permuted against ray ids"""
    c = cases.distortion_case(0, "exp16")
    ra = c["rays_a"]
    assert set(cases.DISTORTION_LENGTHS) <= set(ra[:, 2].tolist()) and len(ra) % 4 != 0
    assert sorted(ra[:, 0].tolist()) == list(range(len(ra))) and (ra[:, 0] != np.arange(len(ra))).any()
    order = np.argsort(ra[:, 1])
    assert (order != np.arange(len(ra))).any()
    ends = ra[order, 1] + ra[order, 2]
    assert (ra[order[1:], 1] > ends[:-1]).all(), "every segment is preceded by a gap"
    off, cnt = by_ray(ra)
    ts = D64.pad(T(c["ts"]), off, cnt)
    assert (ts[:, 1:] >= ts[:, :-1])[D64.pad(T(np.ones_like(c["ts"])), off, cnt)[:, 1:] > 0].all()
    assert 30 < float(ts.max()), "the exponential step reaches the far range"
    w = c["ws"]
    s = c["special"]
    assert not w[ra[s["zero"], 1]:ra[s["zero"], 1] + 64].any() and w.max() == F(1 - 2 ** -20)


@pytest.mark.parametrize("profile", ["lego", "exp16"])
def test_scan_identity_equals_pair_sums(profile):
    """the kernels' formula -- scans, their products and the head / tail brackets -- is the definition: both in float64,
    they agree far inside the fp32 bound (2^-20 of it)"""
    c = cases.distortion_case(1, profile, repeat=1, n_long=1, n_random=9)
    off, cnt = by_ray(c["rays_a"])
    f = D64.forward(T(c["ws"]), T(c["deltas"]), T(c["ts"]), off, cnt)
    g = torch.ones(len(cnt), dtype=torch.float64)
    b = D64.backward(f, g)
    loss, dws = D64.pair_sums(T(c["ws"]), T(c["deltas"]), T(c["ts"]), off, cnt)
    assert D64.ratio(f["loss"] - loss, 2 ** -20 * f["loss_err"]) <= 1
    assert D64.ratio((b["dws"] - dws)[f["valid"]], 2 ** -20 * b["dws_err"][f["valid"]]) <= 1
    assert (loss > 0).sum() > len(cnt) // 2


def test_c_oracle_inside_the_serial_bound(oracle):
    for seed, profile in ((2, "lego"), (3, "exp16")):
        c = cases.distortion_case(seed, profile)
        g = np.random.RandomState(seed).normal(size=len(c["rays_a"])).astype(F)
        f, b, off, cnt = oracle64(c["ws"], c["deltas"], c["ts"], c["rays_a"], "serial", g)
        loss, wi, wti = oracle.distortion_fw(c["ws"], c["deltas"], c["ts"], c["rays_a"])
        dws = oracle.distortion_bw(g, wi, wti, c["ws"], c["deltas"], c["ts"], c["rays_a"])
        rs = check_outputs("C oracle " + profile, f, b, off, cnt, loss, wi, wti, dws)
        print("C oracle, serial bound, %s:" % profile, {k: "%.3g" % v for k, v in rs.items()})


def test_reference_kernels_inside_the_serial_bound():
    """the reference's own distortion kernels on the weights of its compositing forward of composite_case()"""
    gd = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "composite.npz"))
    c = cases.composite_case()
    f, b, off, cnt = oracle64(gd["ws"], c["deltas"], c["ts"], c["rays_a"], "serial", gd["dist_dL"])
    rs = check_outputs("reference", f, b, off, cnt, gd["dist_loss"], gd["ws_inc"], gd["wts_inc"], gd["dist_dws"])
    print("reference kernels, serial bound:", {k: "%.3g" % v for k, v in rs.items()})


@pytest.mark.parametrize("contract", [False, True])
@pytest.mark.parametrize("profile", ["lego", "exp16"])
def test_warp_replay_inside_the_warp_bound(profile, contract):
    c = cases.distortion_case(4, profile)
    g = np.random.RandomState(5).normal(size=len(c["rays_a"])).astype(F)
    f, b, off, cnt = oracle64(c["ws"], c["deltas"], c["ts"], c["rays_a"], "warp", g)
    loss, wi, wti, dws = replay(c["ws"], c["deltas"], c["ts"], c["rays_a"], g, contract)
    rs = check_outputs("replay", f, b, off, cnt, loss, wi, wti, dws)
    print("warp replay (%s, fma=%s), warp bound:" % (profile, contract), {k: "%.3g" % v for k, v in rs.items()})
    # every length of the list is in the case, and the long rays are where the error is largest
    assert set(cases.DISTORTION_LENGTHS) <= set(cnt.tolist())
    assert rs["loss"] > 0 and rs["dws"] > 0


def test_bound_is_not_vacuous():
    """the bound is a few roundings of the cancelling products, not a blanket tolerance: on Lego-like rays it is a
    small fraction of the loss and of dL/dws, and leaving out the 1/3 w^2 d term (under 1 % of a typical loss) falls
    far outside it"""
    c = cases.distortion_case(6, "lego")
    off, cnt = by_ray(c["rays_a"])
    f = D64.forward(T(c["ws"]), T(c["deltas"]), T(c["ts"]), off, cnt)
    b = D64.backward(f, torch.ones(len(cnt), dtype=torch.float64))
    big = f["loss"] > 1e-6
    assert big.sum() > 10
    assert float((f["loss_err"][big] / f["loss"][big]).median()) < 3e-3
    sig = f["valid"] & (b["dws"].abs() > 1e-3)
    assert float((b["dws_err"][sig] / b["dws"][sig].abs()).median()) < 1e-4
    q = (f["w"] ** 2 * f["dl"] / 3).sum(1)
    assert float((q[big] / f["loss"][big]).median()) < 1e-2
    assert D64.ratio(q, f["loss_err"]) > 10
    # an empty ray: loss 0 with bound 0, so anything but an exact 0 fails
    empty = cnt == 0
    assert empty.any() and (f["loss"][empty] == 0).all() and (f["loss_err"][empty] == 0).all()
