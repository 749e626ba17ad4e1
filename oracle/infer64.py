"""The reference's test-time loop (models/rendering.py:46-118) as a lockstep replay -- TEST INFRASTRUCTURE ONLY.

The loop is cut into its three steps so that a caller can drive it from another implementation's state round by round:

    S = replay.begin_round(n_alive)            # the quota, or 0 when `while samples < max_samples and N_alive > 0` ends
    m = replay.march(alive, S)                 # raymarching_test on the C oracle: advances the reference's hits_t
    c = composite64(sigmas, rgbs, deltas, ts, m['n_eff'], opacity, depth, rgb, T_threshold)

The marching keeps the reference's rule that hits_t[r][0] only moves after an occupied sample (the C oracle's
march_test). composite64 restates composite_test_fw_kernel (volumerendering.cu:205-249) in float64: it accumulates onto
the previous opacity, depth and rgb with T = 1 - opacity, and reports, per ray, every accumulated value together with a
first-order bound on what an fp32 evaluation with __expf may differ from it, so that a termination decision that falls
within rounding distance of T_threshold can be told apart from a wrong one.
"""
import numpy as np

from . import oracle

U = 2.0 ** -24  # unit roundoff of fp32


def quota(n_rays, n_alive, samples, sample_budget, exp_step_factor, max_round_samples):
    """N_samples of the coming round (rendering.py:73-81), 0 when the loop is over. max_round_samples (the per-round
    sample capacity) clips the quota to max_round_samples // n_alive, and to at least one sample."""
    if samples >= sample_budget or n_alive <= 0:
        return 0
    min_samples = 1 if exp_step_factor == 0 else 4
    S = max(min(n_rays // n_alive, 64), min_samples)
    share = max_round_samples // n_alive
    if share < S:
        S = max(share, 1)
    return S


class InferReplay:
    """The reference's loop state: hits_t (float32, the marcher's), `samples` requested so far and the rounds run."""

    def __init__(self, rays_o, rays_d, bits, cascades, scale, exp_step_factor, center, half_size, near_distance=0.01,
                 sample_budget=1024, max_round_samples=None, grid_size=128, max_samples=1024):
        self.o = np.ascontiguousarray(rays_o, np.float32)
        self.d = np.ascontiguousarray(rays_d, np.float32)
        self.n_rays = self.o.shape[0]
        self.bits = np.ascontiguousarray(bits, np.uint8)
        self.cascades, self.scale, self.esf = int(cascades), np.float32(scale), np.float32(exp_step_factor)
        self.grid_size, self.max_samples = int(grid_size), int(max_samples)
        self.sample_budget = int(sample_budget)
        self.max_round_samples = int(max_round_samples) if max_round_samples is not None else max(4 * self.n_rays, 1 << 16)
        self.hits = oracle.ray_aabb(self.o, self.d, center, half_size, near_distance)
        self.samples = 0
        self.rounds = 0

    def begin_round(self, n_alive):
        S = quota(self.n_rays, n_alive, self.samples, self.sample_budget, float(self.esf), self.max_round_samples)
        if S:
            self.samples += S
            self.rounds += 1
        return S

    def march(self, alive, S, hits=None):
        """raymarching_test of the rays `alive` (ray ids, in list order) with quota S from `hits` (default: the replay's
        own hits_t, advanced in place) -> dict(xyzs (na,S,3), deltas, ts (na,S), n_eff (na))"""
        h = self.hits if hits is None else hits
        xyzs, _, deltas, ts, n_eff = oracle.march_test(self.o, self.d, h, np.asarray(alive, np.int64), self.bits,
                                                       self.cascades, self.scale, self.esf, self.grid_size,
                                                       self.max_samples, int(S))
        return dict(xyzs=xyzs, deltas=deltas, ts=ts, n_eff=n_eff)

    def samples_left(self, rays):
        """per ray: does the reference's marcher still find a sample from its hits_t (without advancing it)?"""
        if len(rays) == 0:
            return np.zeros(0, bool)
        return self.march(rays, 1, hits=self.hits.copy())["n_eff"] > 0


def composite64(sigmas, rgbs, deltas, ts, n_eff, opacity, depth, rgb, T_threshold):
    """composite_test_fw of one round in float64 for na rays of S slots each (sigmas, deltas, ts (na,S), rgbs (na,S,3),
    n_eff (na)) onto the rays' accumulators before the round (opacity, depth (na), rgb (na,3), any float type).

    Returns a dict of float64 arrays:
      O, D (na,S+1), RGB (na,S+1,3): the accumulators after j = 0..S samples (column 0: before the round);
      bO, bD, bRGB: first-order bounds on |fp32 - float64| of those accumulators, for an fp32 evaluation with
          a = 1 - __expf(-(sigma * delta)) (CUDA's documented error of __expf: 2 + floor(1.173 |x|) ulp), every product,
          sum and fma rounded once (a contracted fma only removes a rounding) and T = 1 - opacity rounded;
      T, bT (na,S+1): the transmittance after j samples and its bound;
    and the fp32 termination index range: jt_lo, jt_hi (na, int). An fp32 evaluation stops after the sample jt
    (transmittance <= T_threshold) with jt_lo <= jt <= jt_hi, jt = n_eff meaning it did not stop; the float64 decision
    is exact for rays with jt_lo == jt_hi. A ray with jt stops compositing after min(jt + 1, n_eff) samples."""
    sg = np.asarray(sigmas, np.float64)
    de = np.asarray(deltas, np.float64)
    tt = np.asarray(ts, np.float64)
    c = np.asarray(rgbs, np.float64)
    ne = np.asarray(n_eff, np.int64)
    na, S = sg.shape
    thr = float(np.float32(T_threshold))
    O = np.zeros((na, S + 1)); D = np.zeros((na, S + 1)); RGB = np.zeros((na, S + 1, 3)); T = np.zeros((na, S + 1))
    bO = np.zeros((na, S + 1)); bD = np.zeros((na, S + 1)); bRGB = np.zeros((na, S + 1, 3)); bT = np.zeros((na, S + 1))
    O[:, 0] = np.asarray(opacity, np.float64)
    D[:, 0] = np.asarray(depth, np.float64)
    RGB[:, 0] = np.asarray(rgb, np.float64)
    T[:, 0] = 1.0 - O[:, 0]
    bT[:, 0] = U * np.abs(T[:, 0])
    x = sg * de
    e = np.exp(-x)
    a = -np.expm1(-x)
    f = e  # 1 - a
    # |fp32 e - e|: the product sigma * delta rounded (relative U, hence |x| U in e) and __expf's error
    be = e * (np.abs(x) * U + (2.0 + np.floor(1.173 * np.abs(x) * (1 + 2 * U))) * 2 * U)
    ba = be + U * np.abs(a)          # a = fl(1 - e)
    bf = ba + U * np.abs(f)          # fl(1 - a)
    for j in range(S):
        live = j < ne
        w = a[:, j] * T[:, j]
        bw = ba[:, j] * T[:, j] + np.abs(a[:, j]) * bT[:, j] + U * np.abs(w)
        w = np.where(live, w, 0.0)
        bw = np.where(live, bw, 0.0)
        O[:, j + 1] = O[:, j] + w
        bO[:, j + 1] = bO[:, j] + bw + np.where(live, U * np.abs(O[:, j + 1]), 0.0)
        D[:, j + 1] = D[:, j] + w * tt[:, j]
        bD[:, j + 1] = bD[:, j] + bw * np.abs(tt[:, j]) + np.where(live, U * np.abs(D[:, j + 1]), 0.0)
        RGB[:, j + 1] = RGB[:, j] + w[:, None] * c[:, j]
        bRGB[:, j + 1] = bRGB[:, j] + bw[:, None] * np.abs(c[:, j]) + np.where(live, U, 0.0)[:, None] * np.abs(RGB[:, j + 1])
        Tn = T[:, j] * f[:, j]
        T[:, j + 1] = np.where(live, Tn, T[:, j])
        bT[:, j + 1] = np.where(live, bT[:, j] * f[:, j] + T[:, j] * bf[:, j] + U * Tn, bT[:, j])
    # fp32 stops after the first sample j with T_fp32[j + 1] <= thr; T_fp32 lies within bT of T
    j = np.arange(S)[None, :]
    in_range = j < ne[:, None]
    maybe = in_range & (T[:, 1:] - bT[:, 1:] <= thr)
    sure = in_range & (T[:, 1:] + bT[:, 1:] <= thr)
    jt_lo = np.where(maybe.any(1), maybe.argmax(1), ne)
    jt_hi = np.where(sure.any(1), sure.argmax(1), ne)
    return dict(O=O, D=D, RGB=RGB, T=T, bO=bO, bD=bD, bRGB=bRGB, bT=bT, jt_lo=jt_lo, jt_hi=jt_hi, n_eff=ne)


def composite_match(c, opacity, depth, rgb, term, slack=2.0, rtol=1e-4, atol=1e-6):
    """Which rays' fp32 results (opacity, depth (na), rgb (na,3), term (na) bool: the ray stopped on T_threshold) agree
    with the float64 composite c of composite64: some termination index jt in [jt_lo, jt_hi] consistent with `term`
    gives values within the tolerance min(slack x the bound, atol + rtol |value|) -- the derived bound, never looser than
    a relative rtol. -> (ok (na) bool, the jt that matched or -1, the smallest error / tolerance over the candidates)"""
    ne = c["n_eff"]
    na = ne.shape[0]
    o = np.asarray(opacity, np.float64)
    dp = np.asarray(depth, np.float64)
    cl = np.asarray(rgb, np.float64)
    term = np.asarray(term, bool)
    ok = np.zeros(na, bool)
    matched = np.full(na, -1, np.int64)
    ratio = np.full(na, np.inf)
    rows = np.arange(na)
    for jt in range(int(c["jt_hi"].max(initial=0)) + 1):
        cand = (jt >= c["jt_lo"]) & (jt <= c["jt_hi"]) & ~ok
        cand &= np.where(term, jt < ne, jt == ne)
        if not cand.any():
            continue
        k = np.minimum(jt + 1, ne)
        def tol(v, b):
            return np.minimum(slack * b, atol + rtol * np.abs(v)) + 1e-30

        r = np.maximum.reduce([np.abs(o - c["O"][rows, k]) / tol(c["O"][rows, k], c["bO"][rows, k]),
                               np.abs(dp - c["D"][rows, k]) / tol(c["D"][rows, k], c["bD"][rows, k]),
                               (np.abs(cl - c["RGB"][rows, k]) / tol(c["RGB"][rows, k], c["bRGB"][rows, k])).max(1)])
        hit = cand & (r <= 1.0)
        ok |= hit
        matched = np.where(hit, jt, matched)
        ratio = np.where(cand, np.minimum(ratio, r), ratio)
    return ok, matched, ratio
