"""oracle/composite64.py, the float64 compositing restatement the GPU tests hold the training kernels to, and its
rounding bound: the values agree with the C oracle, and real fp32 implementations lie inside the bound -- the reference's
own CUDA kernels (tests/golden/composite.npz) in the serial order, the numpy float32 replay of the warp algorithm
(test_warp_composite_algorithm_cpu.py) in the warp order. A bound that does not cover the reference's own kernel is wrong.
"""
import os

import numpy as np
import pytest
import torch

import cases
from oracle import composite64 as C64
from test_warp_composite_algorithm_cpu import _warp_composite_loss

F = np.float32


def by_ray(rays_a):
    """rays_a rows (ray, start, count) -> offsets, counts indexed by ray"""
    ra = np.asarray(rays_a)
    off, cnt = np.zeros(len(ra), np.int64), np.zeros(len(ra), np.int64)
    off[ra[:, 0]], cnt[ra[:, 0]] = ra[:, 1], ra[:, 2]
    return torch.as_tensor(off), torch.as_tensor(cnt)


def T(x):
    return torch.as_tensor(np.ascontiguousarray(x))


def fw64(c, sig=None, order="serial"):
    off, cnt = by_ray(c["rays_a"])
    sig = c["sigmas"] if sig is None else sig
    return C64.forward(T(sig), T(c["rgbs"]), T(c["deltas"]), T(c["ts"]), off, cnt, c["T_thr"], order), off, cnt


def within(name, mine, ref, err, keep):
    """|mine - ref| <= SAFETY err on the rays `keep` (per-ray rows of padded / per-ray tensors); returns the ratio"""
    mine, ref, err = (torch.as_tensor(v).double() for v in (mine, ref, err))
    d = (mine - ref)[keep]
    r = C64.ratio(d, err[keep])
    assert r <= 1.0, "%s: error / bound = %.3g" % (name, r)
    assert torch.isfinite(err[keep]).all(), name
    return r


def padded(x, off, cnt, L):
    return C64.pad(T(x), off, cnt, L)


def check_case(c, fw_out, bw_out, sig=None, dO=None, dD=None, dC=None, dws=None):
    """a serial fp32 implementation's forward (total, opacity, depth, rgb, ws by ray) and backward (dsig, drgbs per
    sample) against composite64 with its serial bound"""
    f, off, cnt = fw64(c, sig)
    keep = ~f["undecidable"]
    total, opacity, depth, rgb, ws = fw_out
    assert keep.float().mean() > 0.9, "too many undecidable rays"
    assert torch.equal(T(total)[keep], f["total"][keep])
    rs = [within("opacity", opacity, f["O"], f["O_err"], keep), within("depth", depth, f["D"], f["D_err"], keep),
          within("rgb", rgb, f["C"], f["C_err"], keep),
          within("ws", padded(ws, off, cnt, f["L"]), f["w"], f["w_err"], keep)]
    b = C64.backward(f, T(c["dC"] if dC is None else dC), T(c["dO"] if dO is None else dO),
                     dD=T(c["dD"] if dD is None else dD), dws=T(c["dws"] if dws is None else dws), offsets=off)
    dsig, drgbs = bw_out
    rs.append(within("dsig", padded(dsig, off, cnt, f["L"]), b["dsig"], b["dsig_err"], keep))
    rs.append(within("drgbs", padded(drgbs, off, cnt, f["L"]), b["drgb"], b["drgb_err"], keep))
    return rs, f


def test_reference_kernels_lie_inside_the_serial_bound():
    """the reference's own CUDA compositing forward and backward (with non-zero dD and dws) on cases.composite_case"""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "composite.npz"))
    c = cases.composite_case()
    rs, f = check_case(c, (g["total"], g["opacity"], g["depth"], g["rgb"], g["ws"]), (g["dsig"], g["drgbs"]))
    print("reference kernels, serial bound: error / bound opacity depth rgb ws dsig drgbs =", ["%.3g" % r for r in rs],
          "undecidable rays", int(f["undecidable"].sum()))


@pytest.mark.parametrize("seed,n_rays", [(3, 96), (5, 40)])
def test_c_oracle_agrees_inside_the_serial_bound(seed, n_rays, oracle):
    c = cases.composite_case(seed=seed, n_rays=n_rays)
    fw = oracle.composite_train_fw(c["sigmas"], c["rgbs"], c["deltas"], c["ts"], c["rays_a"], c["T_thr"])
    total, opacity, depth, rgb, ws = fw
    bw = oracle.composite_train_bw(c["dO"], c["dD"], c["dC"], c["dws"], c["sigmas"], c["rgbs"], ws, c["deltas"], c["ts"],
                                   c["rays_a"], opacity, depth, rgb, c["T_thr"])
    check_case(c, fw, bw)


def special_sigmas(c):
    """an opaque first sample, a ray with sigma = 0 everywhere, the 700-sample ray transparent enough never to terminate"""
    ra = c["rays_a"]
    sig = c["sigmas"].copy()
    r_opaque, r_clear, r_long = ra[5], ra[6], ra[4]
    assert r_long[2] == 700
    sig[r_opaque[1]] = 1e9
    sig[r_clear[1]:r_clear[1] + r_clear[2]] = 0
    sig[r_long[1]:r_long[1] + 700] = np.minimum(sig[r_long[1]:r_long[1] + 700], F(0.3))
    return sig, r_opaque, r_clear, r_long


def test_edge_rays_c_oracle(oracle):
    """0, 1, 32, 33 and 700 samples, an opaque first sample (a = 1: T = 0 after it), sigma = 0 everywhere, rays that
    never terminate: values agree with the C oracle and every bound stays finite"""
    c = cases.composite_case(seed=3, n_rays=64, max_n=300)
    sig, r_opaque, r_clear, r_long = special_sigmas(c)
    fw = oracle.composite_train_fw(sig, c["rgbs"], c["deltas"], c["ts"], c["rays_a"], c["T_thr"])
    total, opacity, depth, rgb, ws = fw
    bw = oracle.composite_train_bw(c["dO"], c["dD"], c["dC"], c["dws"], sig, c["rgbs"], ws, c["deltas"], c["ts"],
                                   c["rays_a"], opacity, depth, rgb, c["T_thr"])
    _, f = check_case(c, fw, bw, sig=sig)
    assert set(c["rays_a"][:5, 2].tolist()) == {0, 1, 32, 33, 700}
    ro, rc, rl = int(r_opaque[0]), int(r_clear[0]), int(r_long[0])
    assert f["total"][ro] == 0 and f["n_comp"][ro] == 1 and f["Tinc"][ro, 0] == 0 and f["O"][ro] == 1
    assert f["O"][rc] == 0 and f["total"][rc] == r_clear[2] and not f["terminated"][rc]
    assert not f["terminated"][rl] and f["total"][rl] == 700
    assert not f["undecidable"][[ro, rc, rl]].any()
    b = C64.backward(f, T(c["dC"]), T(c["dO"]), dD=T(c["dD"]), dws=T(c["dws"]), offsets=by_ray(c["rays_a"])[0])
    for k in ("w_err", "dTinc", "C_err", "O_err", "D_err"):
        assert torch.isfinite(f[k]).all(), k
    for k in ("dsig", "dsig_err", "drgb", "drgb_err"):
        assert torch.isfinite(b[k]).all(), k
    # the ray with no samples and the one with sigma = 0 contribute nothing and receive nothing but dO (1 - O) d
    empty = int(np.flatnonzero(c["rays_a"][:, 2] == 0)[0])
    assert f["O"][c["rays_a"][empty, 0]] == 0 and f["n_comp"][c["rays_a"][empty, 0]] == 0
    assert torch.equal(b["drgb"][rc], torch.zeros_like(b["drgb"][rc]))


@pytest.mark.parametrize("seed,bg,lam", [(3, 1.0, 1e-3), (11, 0.0, 1e-3), (7, 0.5, 1.0)])
def test_warp_replay_lies_inside_the_warp_bound(seed, bg, lam):
    """the float32 replay of k_train_composite_loss's warp algorithm -- forward, NeRFLoss and backward -- against
    composite64 + nerf_loss + backward with the warp-order bound, on edge rays and rays beyond the register cache"""
    c = cases.composite_case(seed=seed, n_rays=64, max_n=300)
    sig, r_opaque, r_clear, r_long = special_sigmas(c)
    ra = c["rays_a"]
    n_rays = ra.shape[0]
    gt = np.random.RandomState(seed + 100).rand(n_rays, 3).astype(F)
    bgv = np.full(3, bg, F)
    thr = c["T_thr"]
    f, off, cnt = fw64(c, sig, order="warp")
    L = f["L"]
    nl = C64.nerf_loss(f, T(gt), T(bgv), lam, n_rays)
    b = C64.backward(f, nl["dC"], nl["dO"], dC_err=nl["dC_err"], dO_err=nl["dO_err"])
    out, O, D, tot = (np.zeros((n_rays, 3), F), np.zeros(n_rays, F), np.zeros(n_rays, F), np.zeros(n_rays, np.int64))
    dsig, dcol = np.zeros((n_rays, L), F), np.zeros((n_rays, L, 3), F)
    for ray, s, n in ra:
        sl = slice(s, s + n)
        o_, O_, D_, t_, ds_, dc_, _, _ = _warp_composite_loss(sig[sl], c["deltas"][sl], c["ts"][sl], c["rgbs"][sl], gt[ray],
                                                             bgv, n_rays, lam, thr, cache=4)
        out[ray], O[ray], D[ray], tot[ray] = o_, O_, D_, t_
        dsig[ray, :n], dcol[ray, :n] = ds_, dc_
    keep = ~f["undecidable"]
    assert keep.float().mean() > 0.9
    assert torch.equal(T(tot)[keep], f["total"][keep])
    rs = {"rgb": within("rgb", out, nl["out"], nl["out_err"], keep),
          "opacity": within("opacity", O, f["O"], f["O_err"], keep),
          "depth": within("depth", D, f["D"], f["D_err"], keep),
          "dsig": within("dsig", dsig, b["dsig"], b["dsig_err"], keep),
          "drgbs": within("drgbs", dcol, b["drgb"], b["drgb_err"], keep)}
    print("warp replay, warp bound: error / bound", {k: "%.3g" % v for k, v in rs.items()})


def test_bound_is_not_vacuous():
    """the bound is a few fp32 roundings (and __expf's absolute error per sample) relative to what it bounds, not a
    blanket tolerance: an implementation off by one part in 1e3 falls outside it"""
    c = cases.composite_case()
    f, off, cnt = fw64(c, order="warp")
    keep = ~f["undecidable"] & (f["O"] > 0.1)
    assert float((f["O_err"][keep] / f["O"][keep]).max()) < 1e-4
    assert float((f["C_err"][keep] / f["C"][keep].clamp_min(1e-3)).abs().max()) < 1e-3
    b = C64.backward(f, T(c["dC"]), T(c["dO"]), offsets=off)
    big = b["dsig"].abs() > 1e-3 * b["dsig"].abs().max()
    assert float((b["dsig_err"][big] / b["dsig"][big].abs()).median()) < 1e-3
    assert C64.ratio(1e-3 * f["O"][keep], f["O_err"][keep]) > 1


def test_loss_scale_formula():
    s = torch.tensor([1.0, 2.0, 3.3e7])
    d = torch.tensor([1e-3, -2e-3, 1e-9])
    assert C64.loss_scale(d, torch.zeros(3, 3), s) == 2.0 ** 15  # m = 4e-3: 256 / m = 64000 = 2^15.97
    assert C64.loss_scale(torch.zeros(3), torch.full((3, 3), 0.5), s) == 512.0
    assert C64.loss_scale(torch.zeros(3), torch.zeros(3, 3), s) == 1.0
    assert C64.loss_scale(torch.full((3,), 1e-30), torch.zeros(3, 3), s) == 2.0 ** 60
