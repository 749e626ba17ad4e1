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
