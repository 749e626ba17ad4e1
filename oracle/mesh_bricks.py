"""numpy restatement of the brick mask of sparse mesh extraction (ngp_mesh_brick_mask, include/ngp_b200.h), and the
per-point occupancy rule it covers.

    occupancy(bitfield, cascades, G)            (cascades, G, G, G) bool, indexed [c, x, y, z]
    brick_mask(bitfield, cascades, G, scale, n, lo, step)   (nb0, nb1, nb2) bool
    point_active(bitfield, cascades, G, scale, n, lo, step) (n0, n1, n2) bool: a cell in the 27-neighbourhood of the
                                                point's cell, in the cascade of its position, is occupied

All arithmetic is the device's fp32: lattice points lo + (float)idx * step, the cascade of a max-norm v from frexpf,
and the cell coordinate (fma(x, 1/mb, 1) * 0.5) * G with fma rounded once (grid_refresh.fma32).
"""
import numpy as np

from .grid_refresh import fma32, morton_decode

B = 8  # NGP_MESH_BRICK

f32 = np.float32


def occupancy(bitfield, cascades, G):
    bits = np.unpackbits(np.asarray(bitfield, np.uint8).reshape(-1), bitorder="little").reshape(cascades, G ** 3)
    xyz = morton_decode(np.arange(G ** 3, dtype=np.uint32)).astype(np.int64)
    occ = np.zeros((cascades, G, G, G), bool)
    occ[:, xyz[:, 0], xyz[:, 1], xyz[:, 2]] = bits.astype(bool)
    return occ


def _box_sums(occ):
    """per cascade the 3-D inclusive prefix sums, padded with a zero plane in front: S[c, x+1, y+1, z+1]"""
    C, G = occ.shape[0], occ.shape[1]
    S = np.zeros((C, G + 1, G + 1, G + 1), np.int64)
    S[:, 1:, 1:, 1:] = occ.astype(np.int64).cumsum(1).cumsum(2).cumsum(3)
    return S


def _box_any(S, c, lo, hi):
    """any occupied cell in cascade c (array) over the inclusive boxes lo..hi (lists of 3 broadcastable arrays)"""
    x0, y0, z0 = lo
    x1, y1, z1 = (h + 1 for h in hi)
    tot = (S[c, x1, y1, z1] - S[c, x0, y1, z1] - S[c, x1, y0, z1] - S[c, x1, y1, z0]
           + S[c, x0, y0, z1] + S[c, x0, y1, z0] + S[c, x1, y0, z0] - S[c, x0, y0, z0])
    return tot > 0


def mip(v, cascades):
    """march.cuh's position rule without the dt term: min(cascades - 1, max(0, e + 1)), frexpf(v, &e)"""
    e = np.frexp(np.asarray(v, f32))[1]
    return np.minimum(cascades - 1, np.maximum(0, e + 1))


def cascade_inv(c, scale):
    mb = np.minimum(f32(2.0 ** (c - 1)), f32(scale))
    return f32(f32(1.0) / mb)


def cell_coord(x, inv, G):
    return (fma32(x, inv, f32(1.0)) * f32(0.5)).astype(f32) * f32(G)


def axis_points(n, lo, step):
    return (f32(lo) + np.arange(n).astype(f32) * f32(step)).astype(f32)


def brick_mask(bitfield, cascades, G, scale, n, lo, step):
    S = _box_sums(occupancy(bitfield, cascades, G))
    n = [int(v) for v in n]
    x0, x1, near, far = [], [], [], []
    for a in range(3):
        nb = -(-n[a] // B)
        pts = axis_points(n[a], lo[a], step[a])
        i0 = np.arange(nb) * B
        p, q = pts[i0], pts[np.minimum(i0 + B - 1, n[a] - 1)]
        a0, a1 = np.minimum(p, q), np.maximum(p, q)
        x0.append(a0)
        x1.append(a1)
        near.append(np.where((a0 <= 0) & (a1 >= 0), f32(0), np.minimum(np.abs(a0), np.abs(a1))))
        far.append(np.maximum(np.abs(a0), np.abs(a1)))
    shape = tuple(len(v) for v in x0)
    grid = np.ix_(*[np.arange(s) for s in shape])
    nearv = np.maximum(np.maximum(near[0][grid[0]], near[1][grid[1]]), near[2][grid[2]])
    farv = np.maximum(np.maximum(far[0][grid[0]], far[1][grid[1]]), far[2][grid[2]])
    c_lo = np.where(nearv > 0, mip(nearv, cascades), 0)
    c_hi = np.where(nearv > 0, mip(farv, cascades), np.maximum(mip(farv, cascades), mip(f32(0), cascades)))
    out = np.zeros(shape, bool)
    for c in range(cascades):
        inv, gs = cascade_inv(c, scale), f32(G)
        inside = np.ones(shape, bool)
        lo3, hi3 = [], []
        for a in range(3):
            v0, v1 = cell_coord(x0[a], inv, G), cell_coord(x1[a], inv, G)
            ins = ~((v1 < 0) | (v0 > gs))
            l = np.maximum(0, np.clip(v0, 0, gs - 1).astype(np.int64) - 1)
            h = np.minimum(G - 1, np.clip(v1, 0, gs - 1).astype(np.int64) + 1)
            inside &= ins[grid[a]]
            lo3.append(l[grid[a]])
            hi3.append(h[grid[a]])
        hit = _box_any(S, np.full(shape, c), lo3, hi3)
        out |= inside & (c_lo <= c) & (c <= c_hi) & hit
    return out


def point_active(bitfield, cascades, G, scale, n, lo, step):
    """the per-point rule the brick mask covers: the point's cascade from its max-norm, its cell (none when it lies
    outside that cascade's box), and any occupied cell among the 27 around it"""
    S = _box_sums(occupancy(bitfield, cascades, G))
    ax = [axis_points(int(n[a]), lo[a], step[a]) for a in range(3)]
    X = np.stack(np.meshgrid(*ax, indexing="ij"), -1)
    c = mip(np.abs(X).max(-1), cascades)
    out = np.zeros(X.shape[:3], bool)
    gs = f32(G)
    for cc in range(cascades):
        sel = c == cc
        if not sel.any():
            continue
        inv = cascade_inv(cc, scale)
        v = cell_coord(X[sel], inv, G)
        inside = ((v >= 0) & (v <= gs)).all(-1)
        cell = np.clip(v, 0, gs - 1).astype(np.int64)
        lo3 = [np.maximum(cell[:, a] - 1, 0) for a in range(3)]
        hi3 = [np.minimum(cell[:, a] + 1, G - 1) for a in range(3)]
        out[sel] = inside & _box_any(S, np.full(cell.shape[0], cc), lo3, hi3)
    return out


def masked(sigma, mask):
    """σ_masked: sigma where the point's brick is active, 0 elsewhere"""
    n = sigma.shape
    m = np.repeat(np.repeat(np.repeat(mask, B, 0), B, 1), B, 2)[:n[0], :n[1], :n[2]]
    return np.where(m, sigma, np.float32(0)).astype(np.float32)
