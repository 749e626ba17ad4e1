"""Plain numpy / scipy float64 restatement of the device point-cloud export (csrc/points.cu), written from the rules of
include/ngp_b200.h ("Point-cloud export"), for the tests and as the host baseline of tools/points_cost.py.

The fp32 stage (back-projection) is restated operation by operation in float32; the neighbour search is a brute-force
O(n^2) scan in float64 (knn) or scipy's cKDTree (knn_tree); normals come from np.linalg.eigh.
"""
import math

import numpy as np

from .mesh_simplify import cluster_keys

GOLDEN = 6180339887


def golden_step(N):
    """the smallest g >= round(0.6180339887 N) (half up, exact integers) with gcd(g, N) = 1"""
    g = max(1, (GOLDEN * int(N) + 5 * 10 ** 9) // 10 ** 10)
    while math.gcd(g, int(N)) != 1:
        g += 1
    return g


def ray_pixels(n_views, n_pix, num_rays):
    """(img_idx, pix_idx) int64 of rays 0 .. R-1, q_k = (k g) mod N in exact integers"""
    N = int(n_views) * int(n_pix)
    R = min(int(num_rays), N)
    g = golden_step(N)
    k = np.arange(R, dtype=np.uint64)
    if (R - 1) * (g if R > 1 else 0) < 2 ** 64:
        q = (k * np.uint64(g)) % np.uint64(N)
    else:
        q = np.array([(int(i) * g) % N for i in range(R)], np.uint64)
    q = q.astype(np.int64)
    return q // n_pix, q % n_pix


def fmaf(a, b, c):
    """a b + c rounded once to float32, for float32 arrays: the fp32 product is exact in double, the sum is rounded to
    odd in double (TwoSum's error decides the last bit), and double -> float32 then rounds as one rounding would"""
    prod = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        s = prod + c
        bb = s - prod
        err = (prod - (s - bb)) + (c - bb)
        adj = (err != 0) & np.isfinite(s) & ((s.view(np.int64) & 1) == 0)
        s = np.where(adj, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def backproject(rays_o, rays_d, opacity, depth, rgb, min_opacity, lo, hi):
    """stage 3 in float32: (keep mask, points, colors, view) for every ray; points etc. of the kept rays only"""
    o = np.asarray(rays_o, np.float32)
    d = np.asarray(rays_d, np.float32)
    a = np.asarray(opacity, np.float32)
    with np.errstate(all="ignore"):
        t = np.asarray(depth, np.float32) / a
        p = fmaf(d, t[:, None], o)
        q = np.minimum(np.asarray(rgb, np.float32) / a[:, None], np.float32(1))
        col = np.rint(np.float32(255) * q)
        ln = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        view = d / ln[:, None]
        keep = (a >= np.float32(min_opacity)) & np.isfinite(p).all(1) & (p >= np.asarray(lo, np.float32)).all(1) & \
               (p <= np.asarray(hi, np.float32)).all(1)
    return keep, p[keep], col[keep].astype(np.uint8), view[keep]


def voxel(points, colors, views, lo, h, n):
    """stage 4: keys (ascending), counts, positions (double means), colours, views (normalised double sums, float64)"""
    p = np.asarray(points, np.float32).reshape(-1, 3)
    key = cluster_keys(p, np.asarray(lo, np.float32), np.float32(h), np.asarray(n, np.int64))
    keys, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    m = len(keys)
    pos = np.zeros((m, 3))
    vs = np.zeros((m, 3))
    cs = np.zeros((m, 3), np.int64)
    np.add.at(pos, inv, p.astype(np.float64))
    np.add.at(vs, inv, np.asarray(views, np.float64))
    np.add.at(cs, inv, np.asarray(colors, np.int64))
    ln = np.sqrt((vs * vs).sum(1))
    view = np.where(ln[:, None] > 0, vs / np.where(ln > 0, ln, 1)[:, None], 0.0)
    col = ((2 * cs + cnt[:, None]) // (2 * cnt[:, None])).astype(np.uint8)
    return keys, cnt, pos / cnt[:, None], col, view


def knn(points, k, block=1024):
    """stage 5 by brute force: idx (n, k') int64 and dist2 (n, k') float64 of the k' = min(k, n - 1) smallest
    (d^2, j), j != i, d^2 = (ex ex + ey ey) + ez ez in float64"""
    p = np.asarray(points, np.float32).reshape(-1, 3).astype(np.float64)
    n = len(p)
    kk = min(k, n - 1)
    idx = np.zeros((n, max(kk, 0)), np.int64)
    d2 = np.zeros((n, max(kk, 0)))
    if kk < 1:
        return idx, d2
    j = np.arange(n)
    for s in range(0, n, block):
        e = p[None, :, :] - p[s:s + block, None, :]
        d = (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]
        for r in range(d.shape[0]):
            i = s + r
            o = np.lexsort((j, d[r]))
            o = o[o != i][:kk]
            idx[i], d2[i] = o, d[r, o]
    return idx, d2


def knn_tree(points, k):
    """stage 5 through scipy's cKDTree (the host baseline; ties in an arbitrary order): idx, dist2"""
    from scipy.spatial import cKDTree
    p = np.asarray(points, np.float32).reshape(-1, 3).astype(np.float64)
    kk = min(k, len(p) - 1)
    d, i = cKDTree(p).query(p, kk + 1)
    d, i = d.reshape(len(p), -1), i.reshape(len(p), -1)
    # drop the point itself (the first of its zero-distance matches may be a duplicate: drop i's own index)
    out_i = np.zeros((len(p), kk), np.int64)
    out_d = np.zeros((len(p), kk))
    for r in range(len(p)):
        m = i[r] != r
        if m.all():
            m[-1] = False
        out_i[r], out_d[r] = i[r][m][:kk], d[r][m][:kk] ** 2
    return out_i, out_d


def outliers(dist2, std_ratio):
    """stage 6: (keep mask, d, mu, sigma, threshold)"""
    d = np.sqrt(np.asarray(dist2, np.float64)).mean(1)
    mu = d.mean()
    sigma = math.sqrt(((d - mu) ** 2).mean())
    thr = mu + std_ratio * sigma
    return d <= thr, d, mu, sigma, thr


def normals(points, views, idx):
    """stage 7 with np.linalg.eigh: (normals (n, 3) float64, relative eigengap (lambda_1 - lambda_0) / lambda_2 (n,),
    zero mask). A normal is only defined to the rounding of the covariance divided by that gap: near-collinear
    neighbourhoods have lambda_0 and lambda_1 both at the rounding level of lambda_2."""
    p = np.asarray(points, np.float32).reshape(-1, 3).astype(np.float64)
    v = np.asarray(views, np.float64).reshape(-1, 3)
    idx = np.asarray(idx, np.int64).reshape(len(p), -1)
    nb = np.concatenate([p[:, None, :], p[idx]], 1)
    e = nb - nb.mean(1, keepdims=True)
    cov = np.einsum("nka,nkb->nab", e, e)
    w, vec = np.linalg.eigh(cov)
    nrm = vec[:, :, 0]
    flip = (nrm * v).sum(1) > 0
    nrm[flip] *= -1
    zero = (cov == 0).all((1, 2))
    nrm[zero] = 0
    with np.errstate(all="ignore"):
        gap = np.where(w[:, 2] > 0, (w[:, 1] - w[:, 0]) / w[:, 2], 0.0)
    return nrm, gap, zero
