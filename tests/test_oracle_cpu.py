"""Pins the CPU oracle (oracle/ngp_oracle.c) to the REAL reference: tests/golden/*.npz were produced by
the reference's own CUDA kernels (oracle/_ref/vren, compiled from the reference's models/csrc) on a
GPU by tests/golden/make_golden.py, on the seeded inputs of tests/cases.py.

  AABB / marcher (train + test)  : BIT-EXACT per ray (counts, t, dt, xyz, mutated hits_t)
  compositing / distortion       : 1e-4 relative (reference uses __expf; sums re-associate)
  packbits / morton              : exact
"""
import os

import numpy as np
import pytest

import cases

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    p = os.path.join(GOLD, name)
    if not os.path.exists(p):
        pytest.fail("golden fixture %s missing (generate with tests/golden/make_golden.py on a GPU box)" % name)
    return np.load(p)


def bits_equal(a, b, what):
    a = np.ascontiguousarray(a, np.float32).view(np.uint32)
    b = np.ascontiguousarray(b, np.float32).view(np.uint32)
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    assert (a == b).all(), "%s: %d/%d elements differ bitwise" % (what, (a != b).sum(), a.size)


def rel_close(a, b, what, rtol=1e-4, atol=1e-6):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    bad = np.abs(a - b) > atol + rtol * np.maximum(np.abs(a), np.abs(b))
    assert not bad.any(), "%s: %d/%d outside tolerance, worst %g" % (what, bad.sum(), bad.size, np.abs(a - b).max())


@pytest.mark.parametrize("name", cases.MARCH_CASES)
def test_aabb_and_train_marcher_bit_exact(name, oracle):
    g = load("march_%s.npz" % name)
    c = cases.march_case(name)
    raw = oracle.ray_aabb(c["o"], c["d"], np.zeros(3, np.float32), np.full(3, c["scale"], np.float32), 0.0)
    bits_equal(raw, g["hits_raw"][:, 0], "ray_aabb_intersect")
    assert ((raw[:, 1] > 0).astype(np.int32) == g["hit_cnt"]).all()
    hits = cases.hits_for(c, oracle)
    bits_equal(hits, g["hits"], "hits_t after the near clamp")
    ra, xyzs, dirs, deltas, ts = oracle.march_train(c["o"], c["d"], hits, c["bits"], c["cascades"], c["scale"], c["esf"],
                                                    c["noise"], 128, 1024)
    assert (ra[:, 2] == g["counts"]).all(), "per-ray sample counts differ from the reference kernel"
    assert ra[:, 2].sum() == int(g["total"])
    bits_equal(ts, g["ts"], "ts")
    bits_equal(deltas, g["deltas"], "deltas")
    bits_equal(xyzs, g["xyzs"], "xyzs")
    bits_equal(dirs, g["dirs"], "dirs")


@pytest.mark.parametrize("name", cases.MARCH_CASES)
def test_test_marcher_bit_exact(name, oracle):
    g = load("march_%s.npz" % name)
    c = cases.march_case(name)
    hits = cases.hits_for(c, oracle).copy()
    n = c["o"].shape[0]
    for rnd, ns in enumerate([1, 2, 4, 64]):
        xyzs, dirs, deltas, ts, neff = oracle.march_test(c["o"], c["d"], hits, np.arange(n), c["bits"], c["cascades"],
                                                         c["scale"], c["esf"], 128, 1024, ns)
        assert (neff == g["test%d_neff" % rnd]).all()
        bits_equal(xyzs, g["test%d_xyzs" % rnd], "round %d xyzs" % rnd)
        bits_equal(deltas, g["test%d_deltas" % rnd], "round %d deltas" % rnd)
        bits_equal(ts, g["test%d_ts" % rnd], "round %d ts" % rnd)
        bits_equal(hits, g["test%d_hits" % rnd], "round %d mutated hits_t" % rnd)


def test_compositing_and_distortion(oracle):
    g = load("composite.npz")
    c = cases.composite_case()
    total, opacity, depth, rgb, ws = oracle.composite_train_fw(c["sigmas"], c["rgbs"], c["deltas"], c["ts"], c["rays_a"], c["T_thr"])
    assert (total == g["total"]).all()
    rel_close(opacity, g["opacity"], "opacity")
    rel_close(depth, g["depth"], "depth")
    rel_close(rgb, g["rgb"], "rgb")
    # per-sample weights a*T with a = 1-exp(-x): __expf's ~1e-7 ABSOLUTE error in exp() is a large RELATIVE
    # error of a small weight, so ws (and dL_drgbs = dC*ws) are pinned absolutely; the 1e-4 relative bar is for the sums
    rel_close(ws, g["ws"], "ws", atol=2e-6)
    dsig, drgbs = oracle.composite_train_bw(c["dO"], c["dD"], c["dC"], c["dws"], c["sigmas"], c["rgbs"], g["ws"], c["deltas"],
                                            c["ts"], c["rays_a"], g["opacity"], g["depth"], g["rgb"], c["T_thr"])
    rel_close(drgbs, g["drgbs"], "dL_drgbs", atol=1e-5)
    rel_close(dsig, g["dsig"], "dL_dsigmas", atol=1e-5)
    loss, wi, wti = oracle.distortion_fw(g["ws"], c["deltas"], c["ts"], c["rays_a"])
    rel_close(loss, g["dist_loss"], "distortion loss", atol=1e-6)
    rel_close(wi, g["ws_inc"], "ws inclusive scan", atol=1e-7)
    dws = oracle.distortion_bw(g["dist_dL"], g["ws_inc"], g["wts_inc"], g["ws"], c["deltas"], c["ts"], c["rays_a"])
    rel_close(dws, g["dist_dws"], "distortion dL_dws", atol=2e-6)


def test_packbits_morton(oracle):
    g = load("bits_morton.npz")
    assert (oracle.packbits(g["grid"], 0.25) == g["bits"]).all()
    assert (oracle.morton3D(g["coords"]) == g["morton"]).all()
    assert (oracle.morton3D_invert(g["morton"]) == g["invert"]).all()
    assert (g["invert"] == g["coords"]).all()


def test_compositing_properties(oracle):
    """size-independent properties: weights sum to opacity <= 1; zero density renders nothing; an opaque
    first sample terminates the ray and total_samples excludes it (volumerendering.cu:28-44)"""
    c = cases.composite_case(seed=5, n_rays=40)
    total, opacity, depth, rgb, ws = oracle.composite_train_fw(c["sigmas"], c["rgbs"], c["deltas"], c["ts"], c["rays_a"], 1e-4)
    for ray, s, n in c["rays_a"]:
        assert abs(ws[s:s + n].sum() - opacity[ray]) < 1e-5 and opacity[ray] <= 1 + 1e-6
    z = np.zeros_like(c["sigmas"])
    total, opacity, depth, rgb, ws = oracle.composite_train_fw(z, c["rgbs"], c["deltas"], c["ts"], c["rays_a"], 1e-4)
    assert opacity.max() == 0 and (total == c["rays_a"][np.argsort(c["rays_a"][:, 0]), 2]).all()
    ra = np.array([[0, 0, 5]], np.int64)
    total, opacity, depth, rgb, ws = oracle.composite_train_fw(np.full(5, 1e9, np.float32), np.ones((5, 3), np.float32),
                                                              np.ones(5, np.float32), np.arange(5, dtype=np.float32), ra, 1e-4)
    assert total[0] == 0 and abs(opacity[0] - 1) < 1e-6 and ws[1:].max() == 0


def test_network_oracles_agree(oracle):
    """the C restatement and the torch restatement of the tinycudann part agree (fp16-ulp level)"""
    import torch
    rng = np.random.RandomState(0)
    L, log2_T = 8, 15
    b = float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / (L - 1))))
    meta, entries = oracle.grid_meta(L, log2_T, 16, b)
    enc = np.concatenate([rng.uniform(-0.25, 0.25, 3072), rng.uniform(-0.5, 0.5, 2 * entries)]).astype(np.float32)
    rgbp = rng.uniform(-0.25, 0.25, 7168).astype(np.float32)
    x = rng.uniform(-0.5, 0.5, (500, 3)).astype(np.float32)
    d = rng.normal(size=(500, 3)).astype(np.float32)
    mn, mx = np.full((1, 3), -0.5, np.float32), np.full((1, 3), 0.5, np.float32)
    sig_c, rgb_c, h_c = oracle.ngp_forward_c(meta, enc, rgbp, mn, mx, x, d)
    sig_t, rgb_t, h_t = oracle.torch_ngp_forward(meta, torch.as_tensor(enc), torch.as_tensor(rgbp), torch.as_tensor(mn),
                                                 torch.as_tensor(mx), torch.as_tensor(x), torch.as_tensor(d))
    assert np.abs(h_c - h_t.numpy()).max() < 0.01 * max(1.0, np.abs(h_c).max())
    assert np.abs(rgb_c - rgb_t.numpy()).max() < 4e-3
