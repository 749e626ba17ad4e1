"""numpy float64 restatement of the texture atlas and bake of include/ngp_b200.h (ngp_mesh_texture_* in
csrc/texture.cu): longest edges and classes, the atlas side S, the Morton packing, the uv placement, the band texels,
their closest points, points and normals, the bake's sample geometry and its composite.

    atlas(vertices, triangles, W)                    -> {'k', 'e', 'rot', 'S', 'order', 'offset', 'squares', 'uv', 'uv64'}
    band(uv, squares, W, tris=None)                  -> texel (Morton, ascending) int64, triangle int32
    box_meets(uv_tri, x, y)                          -> the band test of texel (x, y) against uv triangles (n, 3, 2)
    texels(vertices, triangles, W, normals=None)     -> the whole texel map of atlas + band + surface
    surface(vertices, triangles, normals, rot, uv, texel, tri, W) -> point (n, 3) fp32, normal (n, 3) fp32, bary
    sample_geometry(point, normal, r, K)             -> o (n, 3), d (n, 3), t (K + 1,) fp32 and x (n, K + 1, 3)
    composite(sigma, rgb, delta)                     -> C (n, 3) float64
"""
import numpy as np

from .grid_refresh import fma32

MARGIN = 1
S_MIN = 4
MAX_CLASS = 63


def interleave(x, y):
    """Morton code: x in the even bits, y in the odd bits"""
    x, y = np.asarray(x, np.int64), np.asarray(y, np.int64)
    m = np.zeros(np.broadcast(x, y).shape, np.int64)
    for b in range(16):
        m |= ((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1)
    return m


def deinterleave(m):
    m = np.asarray(m, np.int64)
    x, y = np.zeros_like(m), np.zeros_like(m)
    for b in range(16):
        x |= ((m >> (2 * b)) & 1) << b
        y |= ((m >> (2 * b + 1)) & 1) << b
    return x, y


def smallest_size(F):
    """the smallest power-of-two side >= 16 whose atlas holds F squares of s_min"""
    W = 16
    while F * S_MIN * S_MIN > W * W:
        W *= 2
    return W


def _corners(vertices, triangles, rot):
    """A, B, C (F, 3) float64: the corners rotated by rot"""
    v = np.asarray(vertices, np.float32).astype(np.float64)
    t = np.asarray(triangles, np.int64)
    F = t.shape[0]
    i = np.arange(F)
    return (v[t[i, rot % 3]], v[t[i, (rot + 1) % 3]], v[t[i, (rot + 2) % 3]])


def _norm(d):
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def side(k, S):
    """s = max(s_min, S >> k), 0 for k >= 31"""
    k = np.asarray(k, np.int64)
    return np.maximum(S_MIN, np.where(k < 31, np.int64(S) >> np.minimum(k, 30), 0))


def atlas(vertices, triangles, W):
    v = np.asarray(vertices, np.float32).astype(np.float64)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    F = t.shape[0]
    if F * S_MIN * S_MIN > W * W:
        raise ValueError("an atlas of %d triangles needs W >= %d" % (F, smallest_size(F)))
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    l0, l1, l2 = _norm(b - a), _norm(c - b), _norm(a - c)
    rot = np.where((l0 >= l1) & (l0 >= l2), 0, np.where(l1 >= l2, 1, 2)).astype(np.int64)
    ell = np.choose(rot, [l0, l1, l2])
    _, e = np.frexp(ell)
    e = e.astype(np.int64)
    valid = (ell > 0) & np.isfinite(ell)
    e_top = e[valid].max() if valid.any() else 0
    k = np.where(valid, np.minimum(e_top - e, MAX_CLASS), MAX_CLASS)
    hist = np.bincount(k, minlength=64)
    S = W
    while S > S_MIN and (hist * side(np.arange(64), S) ** 2).sum() > W * W:
        S //= 2
    s = side(k, S)
    order = np.argsort(-s, kind="stable")
    area = s[order] ** 2
    offset = np.zeros(F + 1, np.int64)
    np.cumsum(area, out=offset[1:])
    x0s, y0s = deinterleave(offset[:F])
    x0, y0 = np.empty(F, np.int64), np.empty(F, np.int64)
    x0[order], y0[order] = x0s, y0s
    squares = np.stack([x0, y0, s], 1).astype(np.int32)
    A, B, C = _corners(v, t, rot)
    ok = valid
    ell_ = np.where(ok, ell, 1.0)
    rho = np.ldexp((s - 2 * MARGIN).astype(np.float64), -np.where(ok, e, 0))
    u = (B - A) / ell_[:, None]
    CA = C - A
    w = (CA[:, 0] * u[:, 0] + CA[:, 1] * u[:, 1]) + CA[:, 2] * u[:, 2]
    q = CA - w[:, None] * u
    eta = _norm(q)
    ax, ay = (x0 + MARGIN).astype(np.float64), (y0 + MARGIN).astype(np.float64)
    uvA = np.stack([ax, ay], 1)
    uvB = np.stack([np.where(ok, ax + rho * ell_, ax), ay], 1)
    uvC = np.stack([np.where(ok, ax + rho * w, ax), np.where(ok, ay + rho * eta, ay)], 1)
    uv = np.empty((F, 3, 2), np.float64)
    i = np.arange(F)
    uv[i, rot % 3], uv[i, (rot + 1) % 3], uv[i, (rot + 2) % 3] = uvA, uvB, uvC
    return {"k": k, "e": e, "e_top": e_top, "hist": hist, "rot": rot, "S": S, "order": order, "offset": offset,
            "squares": squares, "uv64": uv, "uv": uv.astype(np.float32)}


def box_meets(uvt, x, y):
    """does the open box (x + 1/2 +- 1, y + 1/2 +- 1) meet the closed triangle uvt (n, 3, 2) fp32? Separating axes in
    double: x, y and the normals of the non-zero edges"""
    p = np.asarray(uvt, np.float32).astype(np.float64)
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    px, py = p[..., 0], p[..., 1]
    meet = (px.max(-1) > x - 0.5) & (px.min(-1) < x + 1.5) & (py.max(-1) > y - 0.5) & (py.min(-1) < y + 1.5)
    cx, cy = x + 0.5, y + 0.5
    for k in range(3):
        nx = -(py[..., (k + 1) % 3] - py[..., k])
        ny = px[..., (k + 1) % 3] - px[..., k]
        d = nx[..., None] * px + ny[..., None] * py
        dc = nx * cx + ny * cy
        rad = np.abs(nx) + np.abs(ny)
        sep = (d.max(-1) <= dc - rad) | (d.min(-1) >= dc + rad)
        meet &= ~(sep & ((nx != 0) | (ny != 0)))
    return meet


def band(uv, squares, W, tris=None, chunk=1 << 22):
    """the baked texels of the triangles `tris` (default all), (texel, triangle) in ascending texel"""
    sq = np.asarray(squares, np.int64)
    tris = np.arange(sq.shape[0]) if tris is None else np.asarray(tris, np.int64)
    out_m, out_t = [], []
    i = 0
    while i < len(tris):
        j, n = i, 0
        while j < len(tris) and (n == 0 or n + sq[tris[j], 2] ** 2 <= chunk):
            n += sq[tris[j], 2] ** 2
            j += 1
        ts = tris[i:j]
        s = sq[ts, 2]
        rep = np.repeat(np.arange(len(ts)), s * s)
        start = np.zeros(len(ts) + 1, np.int64)
        np.cumsum(s * s, out=start[1:])
        loc = np.arange(rep.size) - start[rep]
        lx, ly = deinterleave(loc)
        x, y = sq[ts, 0][rep] + lx, sq[ts, 1][rep] + ly
        keep = box_meets(np.asarray(uv)[ts][rep], x, y)
        out_m.append(interleave(x[keep], y[keep]))
        out_t.append(ts[rep[keep]])
        i = j
    m = np.concatenate(out_m) if out_m else np.zeros(0, np.int64)
    t = np.concatenate(out_t) if out_t else np.zeros(0, np.int64)
    o = np.argsort(m, kind="stable")
    return m[o], t[o].astype(np.int32)


def _cross2(ax, ay, bx, by):
    return ax * by - ay * bx


def closest_bary(uvt, qx, qy):
    """barycentrics (bA, bB, bC) float64 of the closest point of the uv triangles (n, 3, 2) in A, B, C order to (qx, qy):
    the interior when the point is inside a triangle of non-zero area, else the nearest clamped projection onto AB, BC,
    CA, the first on a tie"""
    p = np.asarray(uvt, np.float32).astype(np.float64)
    A, B, C = p[:, 0], p[:, 1], p[:, 2]
    n = p.shape[0]
    area = _cross2(B[:, 0] - A[:, 0], B[:, 1] - A[:, 1], C[:, 0] - A[:, 0], C[:, 1] - A[:, 1])
    dA = _cross2(B[:, 0] - A[:, 0], B[:, 1] - A[:, 1], qx - A[:, 0], qy - A[:, 1])
    dB = _cross2(C[:, 0] - B[:, 0], C[:, 1] - B[:, 1], qx - B[:, 0], qy - B[:, 1])
    dC = _cross2(A[:, 0] - C[:, 0], A[:, 1] - C[:, 1], qx - C[:, 0], qy - C[:, 1])
    inside = (area > 0) & (dA >= 0) & (dB >= 0) & (dC >= 0)
    safe = np.where(area > 0, area, 1.0)
    bary = np.stack([dB / safe, dC / safe, dA / safe], 1)
    best = np.full(n, np.inf)
    bb = np.zeros((n, 3))
    for P, Q, i, j in ((A, B, 0, 1), (B, C, 1, 2), (C, A, 2, 0)):
        ex, ey = Q[:, 0] - P[:, 0], Q[:, 1] - P[:, 1]
        l2 = ex * ex + ey * ey
        t = np.where(l2 > 0, ((qx - P[:, 0]) * ex + (qy - P[:, 1]) * ey) / np.where(l2 > 0, l2, 1.0), 0.0)
        t = np.minimum(np.maximum(t, 0.0), 1.0)
        dx, dy = qx - (P[:, 0] + t * ex), qy - (P[:, 1] + t * ey)
        d2 = dx * dx + dy * dy
        better = d2 < best
        best = np.where(better, d2, best)
        cand = np.zeros((n, 3))
        cand[:, i], cand[:, j] = 1.0 - t, t
        bb = np.where(better[:, None], cand, bb)
    return np.where(inside[:, None], bary, bb)


def surface(vertices, triangles, normals, rot, uv, texel, tri, W):
    """point and normal (n, 3) fp32 of the texels (Morton indices) of triangles `tri`, and their barycentrics"""
    tri = np.asarray(tri, np.int64)
    r = np.asarray(rot, np.int64)[tri]
    t = np.asarray(triangles, np.int64)[tri]
    A, B, C = _corners(vertices, t, r)
    i = np.arange(len(tri))
    u = np.asarray(uv, np.float32)[tri]
    uvt = np.stack([u[i, r % 3], u[i, (r + 1) % 3], u[i, (r + 2) % 3]], 1)
    x, y = deinterleave(texel)
    b = closest_bary(uvt, x + 0.5, y + 0.5)
    eB, eC = B - A, C - A
    p = (A + b[:, 1:2] * eB) + b[:, 2:3] * eC
    fn = np.stack([eB[:, 1] * eC[:, 2] - eB[:, 2] * eC[:, 1], eB[:, 2] * eC[:, 0] - eB[:, 0] * eC[:, 2],
                   eB[:, 0] * eC[:, 1] - eB[:, 1] * eC[:, 0]], 1)
    nrm = fn
    if normals is not None:
        nA, nB, nC = _corners(normals, t, r)
        mix = (b[:, 0:1] * nA + b[:, 1:2] * nB) + b[:, 2:3] * nC
        nrm = np.where((_norm(mix) > 0)[:, None], mix, fn)
    ln = _norm(nrm)
    nrm = np.where((ln > 0)[:, None], nrm / np.where(ln > 0, ln, 1.0)[:, None], np.array([0.0, 0.0, -1.0]))
    return p.astype(np.float32), nrm.astype(np.float32), b


def texels(vertices, triangles, W, normals=None):
    at = atlas(vertices, triangles, W)
    m, t = band(at["uv"], at["squares"], W)
    p, n, _ = surface(vertices, triangles, normals, at["rot"], at["uv"], m, t, W)
    return dict(at, texel=m, triangle=t, point=p, normal=n)


def sample_geometry(point, normal, r, K):
    """o = fmaf(n, r, p), d = -n, delta = (2r)/K, t_j = (j + 1/2) delta (j < K), t_K = r, x_j = fmaf(d, t_j, o): fp32"""
    p, n = np.asarray(point, np.float32), np.asarray(normal, np.float32)
    r = np.float32(r)
    o = fma32(n, r, p)
    d = -n
    delta = np.float32(np.float32(2.0) * r / np.float32(K))
    t = np.empty(K + 1, np.float32)
    t[:K] = (np.arange(K, dtype=np.float32) + np.float32(0.5)) * delta
    t[K] = r
    x = fma32(d[:, None, :], t[None, :, None], o[:, None, :])
    return o, d, t, delta, x


def composite(sigma, rgb, delta):
    """C = sum_{j<K} T_j alpha_j c_j + T_K c_K, alpha_j = 1 - exp(-sigma_j delta), float64; sigma (n, K+1), rgb (n, K+1, 3)"""
    sig = np.asarray(sigma, np.float64)
    c = np.asarray(rgb, np.float64)
    K = sig.shape[1] - 1
    T = np.ones(sig.shape[0])
    C = np.zeros((sig.shape[0], 3))
    for j in range(K):
        a = 1.0 - np.exp(-(sig[:, j] * np.float64(delta)))
        C = C + (T * a)[:, None] * c[:, j]
        T = T * (1.0 - a)
    return C + T[:, None] * c[:, K]


def quantise(C):
    return np.clip(np.rint(255.0 * np.asarray(C, np.float64)), 0, 255).astype(np.uint8)
