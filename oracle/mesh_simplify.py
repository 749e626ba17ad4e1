"""Plain numpy float64 restatement of the device mesh simplification (ngp_mesh_simplify_count / _emit, csrc/mesh.cu),
written from rules 1-6 of include/ngp_b200.h, for the tests: vertex clustering with quadric-error placement.

Clusters, their order and the triangle rules are computed from integer keys (np.unique, stable argsorts), so topology
and vertex order are exact; representatives come from np.linalg.eigh per cluster, in world coordinates.
"""
import numpy as np

CUTOFF = 1e-3


def cluster_grid(lo, hi, grid):
    """(lo fp32[3], h fp32, n int64[3]) of rule 1: h = max(hi - lo) / grid, n = min(grid, max(1, ceil((hi - lo) / h)))"""
    lo = np.asarray(lo, np.float32).reshape(3)
    hi = np.asarray(hi, np.float32).reshape(3)
    ext = hi - lo
    h = np.float32(ext.max() / np.float32(grid))
    n = np.minimum(np.maximum(1, np.ceil(ext / h).astype(np.int64)), int(grid))
    return lo, h, n


def cluster_keys(vertices, lo, h, n):
    """int64 key (c0*n1 + c1)*n2 + c2 of every vertex, c = clamp(floor((v - lo) / h), 0, n - 1) in fp32"""
    v = np.asarray(vertices, np.float32).reshape(-1, 3)
    c = np.floor((v - lo) / h)  # fp32 subtract, fp32 divide
    c = np.clip(c, 0, (n - 1).astype(np.float32)).astype(np.int64)
    return (c[:, 0] * n[1] + c[:, 1]) * n[2] + c[:, 2]


def _segments(cid, C):
    order = np.argsort(cid, kind="stable")
    starts = np.searchsorted(cid[order], np.arange(C))
    return order, starts


def simplify(vertices, triangles, lo, hi, grid, normals=None, colors=None):
    """Returns a dict: 'vertices' (V', 3) float32, 'triangles' (F', 3) int64, 'normals' (V', 3) float64 or None,
    'colors' (V', 3) uint8 or None, and per output vertex 'positions64' (the representative before fp32 rounding),
    'ratio' (its cluster's eigenvalues over the largest, (V', 3)), 'key' (its cluster key) and 'h'."""
    v32 = np.asarray(vertices, np.float32).reshape(-1, 3)
    tris = np.asarray(triangles, np.int64).reshape(-1, 3)
    glo, h, n = cluster_grid(lo, hi, grid)
    V, F = len(v32), len(tris)
    empty = {"vertices": np.zeros((0, 3), np.float32), "triangles": np.zeros((0, 3), np.int64),
             "normals": None if normals is None else np.zeros((0, 3)),
             "colors": None if colors is None else np.zeros((0, 3), np.uint8),
             "positions64": np.zeros((0, 3)), "ratio": np.zeros((0, 3)), "key": np.zeros(0, np.int64), "h": float(h)}
    if V == 0 or F == 0:
        return empty
    assert tris.min() >= 0 and tris.max() < V
    keys, cid = np.unique(cluster_keys(v32, glo, h, n), return_inverse=True)
    cid = cid.reshape(-1)
    C = len(keys)
    v = v32.astype(np.float64)

    # rule 2: quadrics, added to the cluster of every corner
    p0, p1, p2 = v[tris[:, 0]], v[tris[:, 1]], v[tris[:, 2]]
    nt = np.cross(p1 - p0, p2 - p0)
    ln = np.sqrt((nt * nt).sum(1))
    ok = ln > 0
    u = np.zeros_like(nt)
    u[ok] = nt[ok] / ln[ok, None]
    area = np.where(ok, ln / 2, 0.0)
    d = -(u * p0).sum(1)
    A = np.zeros((C, 3, 3))
    b = np.zeros((C, 3))
    for k in range(3):
        ck = cid[tris[:, k]]
        for i in range(3):
            b[:, i] += np.bincount(ck, area * d * u[:, i], minlength=C)
            for j in range(i, 3):
                A[:, i, j] += np.bincount(ck, area * u[:, i] * u[:, j], minlength=C)
    for i in range(3):
        for j in range(i):
            A[:, i, j] = A[:, j, i]

    # rule 3: representatives
    cnt = np.bincount(cid, minlength=C).astype(np.float64)
    xbar = np.stack([np.bincount(cid, v[:, a], minlength=C) for a in range(3)], 1) / cnt[:, None]
    order, starts = _segments(cid, C)
    bmin = np.minimum.reduceat(v[order], starts, axis=0)
    bmax = np.maximum.reduceat(v[order], starts, axis=0)
    lam, E = np.linalg.eigh(A)
    lmax = lam.max(1)
    g = np.einsum("cij,cj->ci", A, xbar) + b
    x = xbar.copy()
    ratio = np.zeros((C, 3))
    pos = lmax > 0
    ratio[pos] = lam[pos] / lmax[pos, None]
    for i in range(3):
        keep = pos & (lam[:, i] > CUTOFF * lmax)
        e = E[:, :, i]
        f = np.where(keep, (e * g).sum(1) / np.where(keep, lam[:, i], 1.0), 0.0)
        x -= e * f[:, None]
    x = np.minimum(np.maximum(x, bmin), bmax)

    # rule 5: triangles
    kc = cid[tris]
    nd = (kc[:, 0] != kc[:, 1]) & (kc[:, 1] != kc[:, 2]) & (kc[:, 0] != kc[:, 2])
    r = np.argmin(kc, 1)
    rot = np.stack([kc[np.arange(F), (r + s) % 3] for s in range(3)], 1)
    idx = np.nonzero(nd)[0]
    if len(idx) == 0:
        return empty
    srt = idx[np.lexsort((idx, rot[idx, 2], rot[idx, 1], rot[idx, 0]))]
    first = np.ones(len(srt), bool)
    first[1:] = (rot[srt[1:]] != rot[srt[:-1]]).any(1)
    kept = np.sort(srt[first])

    # rule 6: referenced clusters in key order
    used = np.unique(kc[kept])
    new = np.full(C, -1, np.int64)
    new[used] = np.arange(len(used))
    out = {"vertices": x[used].astype(np.float32), "triangles": new[kc[kept]], "positions64": x[used],
           "ratio": ratio[used], "key": keys[used], "h": float(h), "normals": None, "colors": None}

    # rule 4: attributes
    if normals is not None:
        nv = np.asarray(normals, np.float32).reshape(-1, 3).astype(np.float64)
        s = np.stack([np.bincount(cid, nv[:, a], minlength=C) for a in range(3)], 1)[used]
        ls = np.sqrt((s * s).sum(1))
        out["normals"] = np.where((ls > 0)[:, None], s / np.where(ls > 0, ls, 1.0)[:, None], 0.0)
    if colors is not None:
        cv = np.asarray(colors, np.uint8).reshape(-1, 3).astype(np.int64)
        s = np.stack([np.bincount(cid, cv[:, a], minlength=C).astype(np.int64) for a in range(3)], 1)[used]
        m = cnt[used].astype(np.int64)[:, None]
        out["colors"] = ((2 * s + m) // (2 * m)).astype(np.uint8)
    return out
