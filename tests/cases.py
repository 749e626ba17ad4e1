"""Deterministic parity cases shared by tests/golden/make_golden.py (runs the REAL reference on a GPU),
the CPU-oracle tests and the GPU parity tests. numpy RandomState only, so every host builds the
same inputs."""
import numpy as np
import torch

from ngp_pl_b200 import synth

NEAR = np.float32(0.01)


def rays_from_scene(scene, n_rays, seed, extra_edge_cases=True):
    rng = np.random.RandomState(seed)
    K = synth.intrinsics()
    dirs = synth.ray_directions(K)
    radius = 1.5 if scene.scale <= 0.5 else 0.9
    poses = torch.as_tensor(synth.camera_poses(8, radius=radius, seed=seed))
    img = rng.randint(0, 8, n_rays)
    pix = rng.randint(0, dirs.shape[0], n_rays)
    o, d = synth.get_rays(dirs[torch.as_tensor(pix)], poses[torch.as_tensor(img)])
    o, d = o.numpy().copy(), d.numpy().copy()
    if extra_edge_cases and n_rays >= 16:
        s = scene.scale
        # axis-parallel rays (1/0 = inf), a ray starting inside the box, a ray pointing away, a grazing ray
        o[0], d[0] = [-2 * s - 1, 0.01, 0.02], [1, 0, 0]
        o[1], d[1] = [0.03, -2 * s - 1, -0.1 * s], [0, 1, 0]
        o[2], d[2] = [0.0, 0.1 * s, 2 * s + 1], [0, 0, -1]
        o[3], d[3] = [0.01, 0.02, 0.03], [0.3, -0.5, 0.8]
        o[4], d[4] = [3 * s, 3 * s, 3 * s], [1, 1, 1]
        o[5], d[5] = [-2 * s, s * 0.999999, 0.0], [1, 0, 1e-4]
        o[6], d[6] = [0.0, 0.0, 0.005], [1, 1, 0]  # starts inside, t0 < NEAR
    return o.astype(np.float32), d.astype(np.float32)


def march_case(name):
    """-> dict(scene, bits, o, d, noise, cascades, scale, esf, grid_size, max_samples)"""
    if name == "lego":
        sc = synth.lego_scene(0)
        bits = synth.pack_bits(synth.occupancy_grid(sc))
        o, d = rays_from_scene(sc, 256, 11)
        esf = 0.0
    elif name == "lego_half_random":
        # what the grid looks like during warm-up: ~half of the cells set, no structure
        sc = synth.lego_scene(0)
        rng = np.random.RandomState(5)
        bits = rng.randint(0, 256, 128 ** 3 // 8).astype(np.uint8)
        o, d = rays_from_scene(sc, 64, 12)
        esf = 0.0
    elif name == "full":
        sc = synth.lego_scene(0)
        bits = np.full(128 ** 3 // 8, 255, np.uint8)  # saturates max_samples on the diagonal
        o, d = rays_from_scene(sc, 32, 13)
        esf = 0.0
    elif name == "full_scale2":
        # scale 2 => 3 cascades, chords several units long at the minimum step: saturates max_samples = 1024
        sc = synth.Scene(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), 2.0, 0.0)
        bits = np.full(sc.cascades * 128 ** 3 // 8, 255, np.uint8)
        o, d = rays_from_scene(sc, 32, 15)
        esf = 0.0
    elif name == "mip360":
        sc = synth.mip360_scene(0)
        bits = synth.pack_bits(synth.occupancy_grid(sc))
        o, d = rays_from_scene(sc, 128, 14)
        esf = 1.0 / 256
    else:
        raise KeyError(name)
    rng = np.random.RandomState(99)
    noise = rng.rand(o.shape[0]).astype(np.float32)
    return dict(scene=sc, bits=bits, o=o, d=d, noise=noise, cascades=sc.cascades, scale=np.float32(sc.scale),
                esf=np.float32(esf), grid_size=128, max_samples=1024)


MARCH_CASES = ["lego", "lego_half_random", "full", "full_scale2", "mip360"]


def composite_case(seed=3, n_rays=96, max_n=300):
    """ragged random samples: sigmas, rgbs, deltas, ts, rays_a (+ upstream gradients)"""
    rng = np.random.RandomState(seed)
    counts = rng.randint(0, max_n, n_rays)
    counts[:4] = [0, 1, 32, 33]
    counts[4] = 700
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    n = int(counts.sum())
    rays_a = np.stack([rng.permutation(n_rays), start, counts], 1).astype(np.int64)
    sig = np.exp(rng.normal(0, 2.5, n)).astype(np.float32)
    sig[rng.rand(n) < 0.3] *= 1e-3
    rgbs = rng.rand(n, 3).astype(np.float32)
    deltas = np.full(n, 1.73205080757 / 1024, np.float32) * rng.uniform(1, 8, n).astype(np.float32)
    ts = np.zeros(n, np.float32)
    for s, c in zip(start, counts):
        ts[s:s + c] = 0.3 + np.cumsum(deltas[s:s + c])
    g = dict(dO=rng.normal(size=n_rays).astype(np.float32), dD=rng.normal(size=n_rays).astype(np.float32),
             dC=rng.normal(size=(n_rays, 3)).astype(np.float32), dws=rng.normal(size=n).astype(np.float32))
    return dict(sigmas=sig, rgbs=rgbs, deltas=deltas, ts=ts, rays_a=rays_a, T_thr=np.float32(1e-4), **g)


DISTORTION_LENGTHS = (0, 1, 2, 31, 32, 33, 63, 64, 65, 1023, 1024, 3000)


def distortion_case(seed=0, profile="lego", lengths=DISTORTION_LENGTHS, repeat=2, n_long=3, n_random=37):
    """ragged weights for the distortion loss: every length `repeat` times (3000: n_long times) plus n_random random
    ones, an odd number of rays in all; the segments lie in scrambled order with gaps between them and rays_a[:, 0] is
    a permutation of the rows. Weights are those of a compositing pass (a_i T_{i-1}, exact zeros once T <= 1e-4), with
    an all-zero ray, a ray cut to zeros at a chosen index and a sample within 2^-20 of 1.
    profile 'lego': t from 0.5 to 1 on, constant step sqrt(3)/1024;
            'exp16': a scale-16 scene's exponential step, dt = clamp(t / 256, sqrt(3)/1024, 16 * 2 sqrt(3)/128)."""
    assert profile in ("lego", "exp16")
    rng = np.random.RandomState(seed)
    counts = [n for n in lengths for _ in range(n_long if n >= 3000 else repeat)]
    counts = np.array(counts + list(rng.randint(0, 200, n_random)), np.int64)
    if len(counts) % 2 == 0:
        counts = np.append(counts, 5)
    R = len(counts)
    gaps = rng.randint(1, 6, R)
    start = np.zeros(R, np.int64)
    at = 0
    for r in rng.permutation(R):  # segments in scrambled order, gaps between them
        at += gaps[r]
        start[r] = at
        at += counts[r]
    n_buf = at + 7
    ws, ts, deltas = np.zeros(n_buf, np.float32), np.zeros(n_buf, np.float32), np.zeros(n_buf, np.float32)
    dmin, dmax = np.float32(1.7320508 / 1024), np.float32(16 * 2 * 1.7320508 / 128)
    for r in range(R):
        n, s = int(counts[r]), int(start[r])
        if profile == "lego":
            dt = np.full(n, dmin, np.float32)
            t = (np.float32(0.5 + 0.5 * rng.rand()) + np.arange(n, dtype=np.float32) * dmin).astype(np.float32)
        else:
            t, dt = np.zeros(n, np.float32), np.zeros(n, np.float32)
            tc = np.float32(rng.uniform(0.05, 1.0))
            for k in range(n):
                dt[k] = np.clip(tc / np.float32(256), dmin, dmax)
                t[k] = tc
                tc = np.float32(tc + dt[k])
        x = np.exp(rng.normal(np.log(10 ** rng.uniform(-3.5, 0)), 1.5, n))
        a = -np.expm1(-x)
        T = np.concatenate([[1.0], np.cumprod(1 - a)[:-1]])
        w = np.where(T > 1e-4, a * T, 0.0).astype(np.float32)
        ws[s:s + n], ts[s:s + n], deltas[s:s + n] = w, t, dt
    by_len = {int(n): r for r, n in enumerate(counts)}
    zero, cut, peak = by_len[64], by_len[1024], by_len[33]
    ws[start[zero]:start[zero] + 64] = 0
    ws[start[cut] + 700:start[cut] + 1024] = 0
    ws[start[peak]:start[peak] + 33] = np.float32(1e-3)
    ws[start[peak] + 5] = np.float32(1 - 2 ** -20)
    ws[start[peak] + 6:start[peak] + 33] = 0
    rays_a = np.stack([rng.permutation(R), start, counts], 1).astype(np.int64)
    return dict(ws=ws, ts=ts, deltas=deltas, rays_a=rays_a, special=dict(zero=zero, cut=cut, peak=peak))


def composite_test_case():
    """one round of the test-time compositor: 150 of 200 rays alive, up to 8 samples each, running ray state"""
    rng = np.random.RandomState(4)
    n_rays, n_alive, ns = 200, 150, 8
    alive = rng.permutation(n_rays)[:n_alive].astype(np.int64)
    sig = np.exp(rng.normal(0, 2.5, (n_alive, ns))).astype(np.float32)
    rgbs = rng.rand(n_alive, ns, 3).astype(np.float32)
    dl = np.full((n_alive, ns), 0.01, np.float32)
    ts = np.cumsum(dl, 1).astype(np.float32)
    neff = rng.randint(0, ns + 1, n_alive).astype(np.int32)
    op0 = (rng.rand(n_rays) * 0.9).astype(np.float32)
    dp0 = rng.rand(n_rays).astype(np.float32)
    rgb0 = rng.rand(n_rays, 3).astype(np.float32)
    return dict(alive=alive, sigmas=sig, rgbs=rgbs, deltas=dl, ts=ts, neff=neff, op0=op0, dp0=dp0, rgb0=rgb0)


def hits_for(case, oracle):
    return oracle.ray_aabb(case["o"], case["d"], np.zeros(3, np.float32), np.full(3, case["scale"], np.float32), NEAR)


# ---- golden fixtures of large outputs (tests/golden/make_golden_render.py and the GPU tests that read them) ----------
SAMPLE_SEED = 1234


def sample_idx(n, k):
    """a fixed, seeded, sorted sample of k of the indices 0..n-1 (all of them when n <= k)"""
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.RandomState(SAMPLE_SEED).choice(n, k, replace=False))


def digest(a):
    """SHA-256 of an array's bytes (C order), as 32 uint8: stands in for a whole array that a test checks bit for bit"""
    import hashlib
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def target_rgb(n, seed):
    """seeded target colours for the loss of a parity render"""
    return np.random.RandomState(seed).rand(n, 3).astype(np.float32)
