"""The brick mask of sparse mesh extraction, restated in numpy (oracle/mesh_bricks.py): conservative against the
per-point rule it is built to cover, and the mesh of σ_masked closed and oriented where the mask cuts the surface."""
import numpy as np
import pytest

from oracle import mcubes_ref as R
from oracle import mesh_bricks as M
from oracle.grid_refresh import morton_decode
from test_mesh_cpu import random_field


def cascades_of(scale):
    return max(1 + int(np.ceil(np.log2(2 * scale))), 1)


def random_bitfield(cascades, G, density, seed):
    rng = np.random.RandomState(seed)
    bits = rng.rand(cascades * G ** 3) < density
    return np.packbits(bits, bitorder="little")


def blob_bitfield(cascades, G, scale, seed):
    """a few occupied balls of cells in world space, as a trained scene's grid looks"""
    rng = np.random.RandomState(seed)
    centres = rng.uniform(-0.8, 0.8, (3, 3)) * min(scale, 1.0)
    xyz = morton_decode(np.arange(G ** 3, dtype=np.uint32)).astype(np.float64)
    bits = np.zeros((cascades, G ** 3), bool)
    for c in range(cascades):
        mb = min(2.0 ** (c - 1), scale)
        p = (xyz + 0.5) / G * 2 * mb - mb
        for ctr in centres:
            bits[c] |= np.linalg.norm(p - ctr, axis=1) < 0.2 * min(scale, 1.0)
    return np.packbits(bits.reshape(-1), bitorder="little")


def lattice(n, lo, hi):
    n = np.broadcast_to(np.asarray(n, np.int64), (3,))
    lo = np.broadcast_to(np.asarray(lo, np.float32), (3,)).astype(np.float32)
    step = ((np.broadcast_to(np.asarray(hi, np.float32), (3,)) - lo) / (n - 1).astype(np.float32)).astype(np.float32)
    return n, lo, step


# (scale, G, lattice n, bounds or None for the model box, density)
CASES = [
    (0.5, 32, 40, None, 0.002),
    (0.5, 32, (17, 40, 23), None, 0.02),
    (0.5, 128, 65, ((-0.9, -0.6, -0.5), (0.7, 1.1, 0.5)), 0.0005),
    (1.0, 32, 33, None, 0.01),
    (2.0, 32, (31, 26, 45), ((-3.0, -1.0, -0.25), (2.5, 0.75, 3.0)), 0.003),
    (4.0, 32, 57, None, 0.001),
    (8.0, 32, 49, ((-0.3, -0.3, -0.3), (0.3, 0.3, 0.3)), 0.002),
    (16.0, 32, (41, 33, 50), None, 0.0005),
    (16.0, 128, 37, ((-20.0, -3.0, -1.0), (2.0, 18.0, 1.0)), 0.003),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_brick_mask_covers_every_active_point(case):
    scale, G, n, bounds, dens = CASES[case]
    C = cascades_of(scale)
    lo, hi = bounds if bounds is not None else (-scale, scale)
    n, lo, step = lattice(n, lo, hi)
    seen = False
    for bf in (random_bitfield(C, G, dens, case), blob_bitfield(C, G, scale, case)):
        mask = M.brick_mask(bf, C, G, scale, n, lo, step)
        pts = M.point_active(bf, C, G, scale, n, lo, step)
        B = M.B
        assert mask.shape == tuple(-(-int(v) // B) for v in n)
        brick_of = np.repeat(np.repeat(np.repeat(mask, B, 0), B, 1), B, 2)[:n[0], :n[1], :n[2]]
        assert not (pts & ~brick_of).any()
        seen |= bool(pts.any())
    assert seen


def test_empty_and_full_bitfields():
    C, G = cascades_of(2.0), 32
    n, lo, step = lattice(30, -2.0, 2.0)
    assert not M.brick_mask(np.zeros(C * G ** 3 // 8, np.uint8), C, G, 2.0, n, lo, step).any()
    assert M.brick_mask(np.full(C * G ** 3 // 8, 255, np.uint8), C, G, 2.0, n, lo, step).all()
    # a lattice wholly outside the largest cascade's box finds nothing, even with every cell occupied
    n, lo, step = lattice(20, 2.5, 4.0)
    assert not M.brick_mask(np.full(C * G ** 3 // 8, 255, np.uint8), C, G, 2.0, n, lo, step).any()


def test_one_cascade_brick_is_exact():
    """a brick inside one cascade is active iff one of its points is"""
    C, G, scale = 1, 32, 0.5
    n, lo, step = lattice(48, -0.5, 0.5)
    bf = random_bitfield(C, G, 0.001, 3)
    mask = M.brick_mask(bf, C, G, scale, n, lo, step)
    pts = M.point_active(bf, C, G, scale, n, lo, step)
    B = M.B
    per = np.zeros(mask.shape, bool)
    for i, j, k in zip(*np.nonzero(pts)):
        per[i // B, j // B, k // B] = True
    assert np.array_equal(per, mask)


@pytest.mark.parametrize("shape", [(40, 40, 40), (33, 26, 41)])
def test_masked_field_mesh_is_closed_and_oriented(shape):
    sig = random_field(shape, 5) * np.float32(40)  # border 0, iso 20
    nb = tuple(-(-s // M.B) for s in shape)
    mask = np.random.RandomState(1).rand(*nb) < 0.6
    sm = M.masked(sig, mask)
    assert (sm == 0).sum() > (sig == 0).sum()  # the mask cuts the field
    V, F = R.marching_cubes(sm, 20.0)
    assert len(F) > 0 and len(R.unpaired_edges(F)) == 0
    assert R.signed_volume(V, F) > 0
