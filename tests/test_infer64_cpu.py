"""oracle/infer64.py, the lockstep replay of the reference's test-time loop, checked on the CPU: split into rounds, the
marching walks the same chain of t values as one uninterrupted march, the float64 compositing equals a direct integration
of that sequence, and the quota follows the reference's formula, its budget stop and the per-round capacity clip."""
import numpy as np
import pytest

import cases
from oracle import infer64


def field(xyzs):
    """an analytic density and colour: a few dense blobs over a thin haze, colour varying with position"""
    x = np.asarray(xyzs, np.float64)
    sig = 0.5 + 400.0 * np.exp(-np.sum((x - 0.1) ** 2, -1) / 0.01) + 60.0 * np.exp(-np.sum((x + 0.15) ** 2, -1) / 0.02)
    rgb = 0.5 + 0.5 * np.sin(np.stack([7 * x[..., 0], 5 * x[..., 1] + 1, 3 * x[..., 2] + 2], -1))
    return sig.astype(np.float32), rgb.astype(np.float32)


def run_replay(c, T_threshold=1e-4, sample_budget=1024, max_round_samples=None):
    """the whole loop on the replay alone, float64 accumulators; -> replay, per-ray concatenated ts / deltas, the
    float64 opacity, depth, rgb, the quotas and how each ray left the loop"""
    sc = c["scene"]
    rp = infer64.InferReplay(c["o"], c["d"], c["bits"], c["cascades"], c["scale"], c["esf"], np.zeros(3, np.float32),
                             np.full(3, sc.scale, np.float32), cases.NEAR, sample_budget=sample_budget,
                             max_round_samples=max_round_samples)
    n = rp.n_rays
    hits0 = rp.hits.copy()
    op, dp, rgb = np.zeros(n), np.zeros(n), np.zeros((n, 3))
    ts_all = [[] for _ in range(n)]
    dl_all = [[] for _ in range(n)]
    how = np.full(n, "alive", object)
    n_comp = np.zeros(n, np.int64)  # samples composited: a ray stopped by the threshold marched some it never uses
    alive = np.arange(n)
    quotas = []
    while True:
        S = rp.begin_round(len(alive))
        if S == 0:
            break
        quotas.append((len(alive), S))
        m = rp.march(alive, S)
        sig, col = field(m["xyzs"])
        comp = infer64.composite64(sig, col, m["deltas"], m["ts"], m["n_eff"], op[alive], dp[alive], rgb[alive],
                                   T_threshold)
        jt = comp["jt_lo"]  # float64 accumulators: no fp32 evaluation to match, the float64 decision is the rule
        k = np.minimum(jt + 1, m["n_eff"])
        rows = np.arange(len(alive))
        op[alive], dp[alive], rgb[alive] = comp["O"][rows, k], comp["D"][rows, k], comp["RGB"][rows, k]
        n_comp[alive] += k
        for i, r in enumerate(alive):
            ts_all[r] += list(m["ts"][i, :m["n_eff"][i]])
            dl_all[r] += list(m["deltas"][i, :m["n_eff"][i]])
        term = jt < m["n_eff"]
        how[alive[term]] = "threshold"
        how[alive[m["n_eff"] == 0]] = "left"
        alive = alive[~term & (m["n_eff"] > 0)]
    return rp, hits0, ts_all, dl_all, n_comp, op, dp, rgb, quotas, how


@pytest.mark.parametrize("name,T_threshold,budget", [("lego", 1e-4, 1024), ("lego", 1e-2, 1024), ("mip360", 1e-4, 1024),
                                                     ("lego", 1e-4, 20), ("mip360", 1e-4, 3)])
def test_rounds_are_a_prefix_of_one_march_and_composite_like_one_integration(name, T_threshold, budget, oracle):
    c = cases.march_case(name)
    rp, hits0, ts_all, dl_all, n_comp, op, dp, rgb, quotas, how = run_replay(c, T_threshold, budget)
    n = rp.n_rays
    # (a) every ray's samples, round after round, are bitwise a prefix of one uninterrupted march with a quota of 1024
    h = hits0.copy()
    _, _, dl_full, ts_full, ne_full = oracle.march_test(c["o"], c["d"], h, np.arange(n), c["bits"], c["cascades"],
                                                        c["scale"], c["esf"], 128, 1024, 1024)
    assert ne_full.max() < 1024  # the uninterrupted march is complete: no ray reaches the quota
    for r in range(n):
        k = len(ts_all[r])
        assert k <= ne_full[r]
        np.testing.assert_array_equal(np.array(ts_all[r], np.float32).view(np.uint32), ts_full[r, :k].view(np.uint32))
        np.testing.assert_array_equal(np.array(dl_all[r], np.float32).view(np.uint32), dl_full[r, :k].view(np.uint32))
        if how[r] == "left":  # dropped for an empty round: it had marched its whole sequence
            assert k == ne_full[r]
        elif how[r] == "alive":  # still alive when the budget ran out
            assert rp.samples >= budget
    # (b) the float64 compositing, round by round, equals one integration over that prefix
    assert_integration(c, rp, hits0, n_comp, op, dp, rgb, how, T_threshold, oracle)
    # the run exercised what it is meant to: rays dropped for an empty round, rays stopped by the threshold, and with a
    # small budget rays still alive at the end
    if budget >= 1024:
        assert (how == "left").any() and (how == "threshold").any() and not (how == "alive").any()
    else:
        assert (how == "alive").any(), "the budget should stop the loop with rays still alive"
    print("%s T=%g budget=%d: rounds %d, quotas %s, %s" % (name, T_threshold, budget, rp.rounds, quotas[:12],
                                                          {k: int((how == k).sum()) for k in ("left", "threshold", "alive")}))


def assert_integration(c, rp, hits0, n_comp, op, dp, rgb, how, T_threshold, oracle):
    """direct float64 integration of each ray's concatenated sequence, evaluated at the marcher's own sample points"""
    n = rp.n_rays
    h = hits0.copy()
    xyz_full, _, dl_full, ts_full, ne_full = oracle.march_test(c["o"], c["d"], h, np.arange(n), c["bits"], c["cascades"],
                                                               c["scale"], c["esf"], 128, 1024, 1024)
    for r in range(n):
        k = int(n_comp[r])
        sig, col = field(xyz_full[r, :k])
        x = sig.astype(np.float64) * dl_full[r, :k].astype(np.float64)
        a = -np.expm1(-x)
        T = np.concatenate([[1.0], np.cumprod(np.exp(-x))[:-1]])
        w = a * T
        o_ref = w.sum()
        d_ref = (w * ts_full[r, :k].astype(np.float64)).sum()
        c_ref = (w[:, None] * col.astype(np.float64)).sum(0)
        assert abs(op[r] - o_ref) <= 1e-12 and abs(dp[r] - d_ref) <= 1e-12 * max(1.0, d_ref)
        assert np.abs(rgb[r] - c_ref).max() <= 1e-12
        if how[r] == "threshold":  # stopped at the first sample whose transmittance reached the threshold
            assert 1 - o_ref <= np.float32(T_threshold) * (1 + 1e-9)
            assert k == 1 or 1 - (o_ref - w[-1]) > np.float32(T_threshold) * (1 - 1e-9)
        else:
            assert 1 - o_ref > np.float32(T_threshold) * (1 - 1e-9)


def test_quota_formula_hand_checked():
    q = infer64.quota
    # constant step (min_samples 1): N // n_alive, at most 64
    assert [q(10, a, 0, 1024, 0.0, 1 << 16) for a in (10, 7, 3, 1)] == [1, 1, 3, 10]
    assert q(1000, 1, 0, 1024, 0.0, 1 << 16) == 64
    # exponential step (min_samples 4)
    assert [q(10, a, 0, 1024, 1 / 256, 1 << 16) for a in (10, 7, 3, 2, 1)] == [4, 4, 4, 5, 10]
    # the loop stops once `samples` reached the budget, or when no ray is alive
    assert q(10, 5, 1023, 1024, 0.0, 1 << 16) == 2 and q(10, 5, 1024, 1024, 0.0, 1 << 16) == 0
    assert q(10, 0, 0, 1024, 0.0, 1 << 16) == 0
    # the per-round capacity: max_round_samples // n_alive, at least 1
    assert q(10, 10, 0, 1024, 1 / 256, 12) == 1   # 4 wanted, 12 // 10 = 1 slot each
    assert q(10, 3, 0, 1024, 1 / 256, 12) == 4    # 12 // 3 = 4: fits
    assert q(10, 2, 0, 1024, 1 / 256, 9) == 4     # 9 // 2 = 4 < 5
    assert q(100, 1, 0, 1024, 0.0, 100) == 64


def test_replay_quota_sequence_budget_and_clip():
    """the replay's bookkeeping over a run: `samples` adds up the quotas, a budget stops it, the clip binds"""
    c = cases.march_case("mip360")
    n = c["o"].shape[0]
    rp = infer64.InferReplay(c["o"], c["d"], c["bits"], c["cascades"], c["scale"], c["esf"], np.zeros(3, np.float32),
                             np.full(3, c["scene"].scale, np.float32), cases.NEAR, sample_budget=10,
                             max_round_samples=2 * n)
    got = [rp.begin_round(a) for a in (n, n, 40, 40, 40)]
    # 4 wanted, 2n // n = 2 slots each; then n // 40 = 3 -> min 4, 2n // 40 = 6 fits; budget 10 reached after 2+2+4+4
    assert got == [2, 2, 4, 4, 0]
    assert rp.samples == 12 and rp.rounds == 4
    rp2 = infer64.InferReplay(c["o"], c["d"], c["bits"], c["cascades"], c["scale"], c["esf"], np.zeros(3, np.float32),
                              np.full(3, c["scene"].scale, np.float32), cases.NEAR, sample_budget=3)
    assert [rp2.begin_round(a) for a in (n, n)] == [4, 0]


def test_composite64_termination_band_and_match():
    """a ray whose transmittance lands exactly on the threshold is reported in the band; the fp32 result of either
    decision matches, a result one sample off does not"""
    thr = np.float32(1e-2)
    # one ray, 4 samples; after two samples T = 1e-2 exactly in float64
    a1 = 0.9
    x1 = -np.log1p(-a1)
    x2 = -np.log(0.01 / 0.1)
    sig = np.array([[x1, x2, 1.0, 1.0]], np.float64) / 0.01
    de = np.full((1, 4), 0.01)
    ts = np.array([[0.1, 0.11, 0.12, 0.13]])
    col = np.full((1, 4, 3), 0.5)
    c = infer64.composite64(sig, col, de, ts, np.array([4]), np.zeros(1), np.zeros(1), np.zeros((1, 3)), 1e-2)
    assert abs(c["T"][0, 2] - 0.01) < 1e-8
    assert c["jt_lo"][0] <= 1 < c["jt_hi"][0] or c["jt_lo"][0] < 1 <= c["jt_hi"][0]
    for jt, term in ((1, True), (int(c["jt_hi"][0]), c["jt_hi"][0] < 4)):
        k = min(jt + 1, 4)
        ok, m, _ = infer64.composite_match(c, c["O"][:, k], c["D"][:, k], c["RGB"][:, k], np.array([term]))
        assert ok[0] and m[0] == jt
    ok, _, _ = infer64.composite_match(c, c["O"][:, 4] + 1e-3, c["D"][:, 4], c["RGB"][:, 4], np.array([False]))
    assert not ok[0]
    assert float(thr) == pytest.approx(1e-2)
