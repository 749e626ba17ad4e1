"""The numpy restatement of the occupancy refresh (oracle/grid_refresh.py) held to independent facts: the C oracle's Morton
order and packbits, exact rational arithmetic for the fma, the textbook rounding bounds for the mean and the erode decay,
and the uniformity of the hashed picks. tests/test_grid_refresh_gpu.py then holds the kernels to the restatement."""
import os
from fractions import Fraction

import numpy as np
import pytest
from scipy import stats

from oracle import grid_refresh as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_morton_matches_the_c_oracle(oracle):
    g = np.load(os.path.join(GOLDEN, "bits_morton.npz"))
    c = g["coords"].astype(np.uint32)
    m = R.morton_encode(c[:, 0], c[:, 1], c[:, 2])
    assert (m.astype(np.int32) == g["morton"]).all()
    assert (R.morton_decode(g["morton"]) == g["invert"]).all()
    rng = np.random.RandomState(4)
    c = rng.randint(0, 1024, (3000, 3)).astype(np.uint32)
    c[:4] = [[0, 0, 0], [1023, 1023, 1023], [1023, 0, 0], [0, 0, 1023]]
    m = R.morton_encode(c[:, 0], c[:, 1], c[:, 2])
    assert (m.astype(np.int32) == oracle.morton3D(c)).all()
    assert (R.morton_decode(m) == c).all()
    # for a power-of-two G the indices of [0, G)^3 are exactly [0, G^3)
    for G in (2, 4, 16, 128):
        ax = np.arange(G, dtype=np.uint32)
        x, y, z = np.meshgrid(ax, ax, ax, indexing="ij")
        assert np.array_equal(np.sort(R.morton_encode(x.ravel(), y.ravel(), z.ravel())), np.arange(G ** 3))


def test_packbits_matches_the_c_oracle(oracle):
    rng = np.random.RandomState(8)
    g = rng.normal(0, 1, 4096 * 8).astype(np.float32)
    g[:64] = np.float32(0.25)  # exactly at the threshold: not above it
    for thr in (0.25, -0.5, 2.0):
        assert np.array_equal(R.packbits(g, thr), oracle.packbits(g, thr))


def _frac(v):
    return Fraction(float(v))


def _round32(q):
    """exact rational -> nearest float32, ties to even"""
    f = np.float32(float(q))  # float(q) is the nearest double; fix a double rounding by hand
    lo, hi = (f, np.nextafter(f, np.float32(np.inf))) if _frac(f) <= q else (np.nextafter(f, np.float32(-np.inf)), f)
    dl, dh = q - _frac(lo), _frac(hi) - q
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (int(lo.view(np.uint32)) & 1) == 0 else hi


def test_fma_restatement_is_exact():
    rng = np.random.RandomState(12)
    a = (rng.uniform(-1, 1, 3000) * 2.0 ** rng.randint(-20, 20, 3000)).astype(np.float32)
    b = (rng.uniform(-1, 1, 3000) * 2.0 ** rng.randint(-20, 20, 3000)).astype(np.float32)
    c = (rng.uniform(-1, 1, 3000) * 2.0 ** rng.randint(-20, 20, 3000)).astype(np.float32)
    # constructed cases: a b + c within 2^-54 of a float32 midpoint, so the float64 sum lands ON the midpoint
    e = 2.0 ** np.arange(-6, 7)
    for sgn in (1.0, -1.0):
        for cc in (1.0, 1.0 + 2.0 ** -23):
            for d in (1.0, -1.0):
                a = np.concatenate([a, np.float32(1 + 2.0 ** -15) * np.ones(e.size, np.float32)])
                b = np.concatenate([b, (sgn * e * 2.0 ** -24 * (1 + d * 2.0 ** -15)).astype(np.float32)])
                c = np.concatenate([c, (sgn * e * cc).astype(np.float32)])
    got = R.fma32(a, b, c)
    want = np.array([_round32(_frac(x) * _frac(y) + _frac(z)) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    assert (naive != want).sum() >= 13, "the constructed halfway cases must defeat a plain double rounding"


@pytest.mark.parametrize("G,scale", [(2, 0.5), (4, 1.0), (16, 3.0), (32, 16.0), (128, 0.5)])
def test_jitter_points_against_the_reference_formula(G, scale):
    """every float32 point lies within 2 ulp(s) of the float64 formula with the same u, inside its cell's box widened by
    one ulp, and the warm-up visits every cell"""
    C = max(1 + int(np.ceil(np.log2(2 * scale))), 1)
    seed = R.refresh_seed(3, 0)
    for c in range(C if G <= 32 else 1):
        cells = np.arange(G ** 3, dtype=np.uint32)
        x = R.jitter(cells, seed, c, G, scale)
        x64, bound = R.jitter_reference(cells, seed, c, G, scale)
        assert np.abs(x.astype(np.float64) - x64).max() <= bound
        lo, hi = R.cell_box(cells, c, G, scale)
        lo32 = np.nextafter(lo.astype(np.float32), np.float32(-np.inf)).astype(np.float64)
        hi32 = np.nextafter(hi.astype(np.float32), np.float32(np.inf)).astype(np.float64)
        assert ((x >= lo32) & (x <= hi32)).all()


def test_mean_bound_covers_fp32_sums():
    """the kernel's fp32 sum chain, emulated in its own order, and other orders each stay within gamma_depth * sum"""
    rng = np.random.RandomState(5)
    for n, blocks in ((8, 1), (4096, 16), (2 ** 21, 1056), (3 * 2 ** 21, 2048)):
        g = np.exp(rng.normal(0, 2, n)).astype(np.float32)
        g[rng.rand(n) < 0.3] = -1.0
        m64, bound = R.mean(g, blocks)
        m32 = _kernel_order_mean(g, blocks)
        assert abs(m32 - m64) <= bound, (n, m32, m64, bound)
        # dropping one block's partial is far outside the bound
        assert abs(_kernel_order_mean(g, blocks, drop_last=True) - m64) > 2 * bound or blocks == 1
        pos = g[g > 0]
        tot = float(pos.astype(np.float64).sum())
        if pos.size <= 4096:
            for order in (pos, pos[::-1]):  # serial, forwards and backwards: depth = number of terms
                s = np.float32(0)
                for v in order:
                    s = np.float32(s + v)
                assert abs(float(s) - tot) <= R.gamma(pos.size) * tot
        pw = pos.copy()
        depth = 0
        while pw.size > 1:  # pairwise: depth = number of levels
            if pw.size % 2:
                pw = np.append(pw, np.float32(0))
            pw = (pw[0::2] + pw[1::2]).astype(np.float32)
            depth += 1
        assert abs(float(pw[0]) - tot) <= R.gamma(depth) * tot


def _kernel_order_mean(g, blocks, drop_last=False):
    """k_grid_merge's per-thread strided sums, warp butterfly, 8 warps, then k_grid_mean, all in float32"""
    T = blocks * 256
    v = np.where(g > 0, g, 0).astype(np.float32)
    k = -(-v.size // T)
    v = np.concatenate([v, np.zeros(k * T - v.size, np.float32)]).reshape(k, T)
    s = np.zeros(T, np.float32)
    for row in v:
        s = (s + row).astype(np.float32)
    w = s.reshape(blocks, 8, 32)
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, :, np.arange(32) ^ o]).astype(np.float32)
    part = np.zeros(blocks, np.float32)
    for j in range(8):
        part = (part + w[:, j, 0]).astype(np.float32)
    if drop_last:
        part = part[:-1]
    t = np.zeros(256, np.float32)
    for b0 in range(0, part.size, 256):
        chunk = part[b0:b0 + 256]
        t[:chunk.size] = (t[:chunk.size] + chunk).astype(np.float32)
    o = 128
    while o:
        t[:o] = (t[:o] + t[o:2 * o]).astype(np.float32)
        o >>= 1
    return float(t[0] / np.float32(int((g > 0).sum())))


def test_erode_bound_covers_float32_power():
    rng = np.random.RandomState(6)
    count = np.concatenate([rng.rand(20000), rng.rand(2000) * 1e-3, [0.0, 1e-30, 1e-45, 1.0, 0.5, 1e-7, 3e-3]]).astype(np.float32)
    for decay in (0.95, 0.5):
        d64, bd = R.erode_decay(count, decay)
        with np.errstate(divide="ignore", over="ignore"):
            y = (np.float32(1) / count).astype(np.float32)
        d32 = np.clip(np.power(np.float32(decay), y), np.float32(0.1), np.float32(0.95)).astype(np.float32)
        assert (np.abs(d32.astype(np.float64) - d64) <= bd).all()
        assert d32[count == 0][0] == np.float32(0.1) and d64[count == 0][0] == np.float32(0.1)
        # the bound is not vacuous: decay^count instead of decay^(1/count) is outside it
        wrong = np.clip(np.power(np.float64(np.float32(decay)), count.astype(np.float64)), 0.1, 0.95)
        assert (np.abs(wrong - d64) > bd).mean() > 0.5


def test_uniform_picks_are_uniform():
    """chi-square of each axis and of the joint cell over fixed seeds: fixed inputs, one fixed answer"""
    G = 16
    for seed, c in ((R.refresh_seed(0, 256), 0), (R.refresh_seed(7, 1024), 3)):
        xyz = R.uniform_coords(seed, c, G, 4 * G ** 3)
        for k in range(3):
            assert stats.chisquare(np.bincount(xyz[:, k], minlength=G)).pvalue > 1e-3
        cells = R.morton_encode(xyz[:, 0], xyz[:, 1], xyz[:, 2])
        assert stats.chisquare(np.bincount(cells, minlength=G ** 3)).pvalue > 1e-3


def test_occupied_picks_follow_the_strict_threshold():
    G, thr = 8, 0.5
    g = np.zeros((1, G ** 3), np.float32)
    g[0, ::5] = 0.75
    g[0, 1::7] = thr  # exactly at thr: not occupied
    keys, occ, draw = R.pick_keys(g[0], thr, 99, 0, G)
    assert np.array_equal(occ, np.flatnonzero(g[0] > thr))
    M = G ** 3 // 4
    assert np.isin(keys[M:], occ).all()
    keys, occ, draw = R.pick_keys(np.zeros(G ** 3, np.float32), thr, 99, 0, G)
    assert occ.size == 0 and (keys[M:] == G ** 3).all()
    cells, tot = R.cascade_cells(np.zeros((2, G ** 3), np.float32), thr, 99, G, False)
    assert tot[0] == 0 and tot[1] == cells[0].size and tot[2] == tot[1] + cells[1].size
    assert cells[0][-1] == G ** 3 and R.cell_index(cells, G)[tot[1] - 1] == -1
    assert (np.diff(cells[0].astype(np.int64)) > 0).all()


def test_threshold_and_nan_mean():
    assert R.threshold(0.5, float("nan")) == np.float32(0.5)
    assert R.threshold(0.5, 0.25) == np.float32(0.25)
    g = np.full(64, -1.0, np.float32)
    m, b = R.mean(g, 1)
    assert np.isnan(m)
    # the reference's min(nan, thr) thresholds at NaN: no bit set, like thr > 0 on a grid with no positive cell
    assert not R.packbits(g, R.threshold(0.5, m)).any() and not (g > np.nan).any()
