"""Plain numpy restatement of the depth fusion (ngp_tsdf_integrate, csrc/fusion.cu) and of the TSDF mesh
(ngp_tsdf_mc_count / _emit, csrc/mesh.cu), written from the rules in include/ngp_b200.h ("Depth fusion (TSDF)"), for
the tests.

integrate() runs the rule in a chosen float type: np.float32 in the kernel's operation order (each numpy operation
rounds once, as the kernel's intrinsics do), so it matches the device bit for bit, or np.float64 for the analytic
geometry tests. masked_marching_cubes() is oracle/mcubes_ref.py's marching cubes with the observed mask: unobserved
points are never inside, cells with an unobserved corner emit nothing, and the vertices are the crossed edges the
emitting cells reference.
"""
import numpy as np

from .mcubes_ref import EDGE_AXIS, EDGE_CORNER, NTRI, TRI_EDGES


def lattice_points(n, lo, step, dtype=np.float32):
    """(n0 n1 n2, 3) points lo + idx * step in linear-index order (fp32 multiply then add for float32)"""
    lo, step = np.asarray(lo, dtype), np.asarray(step, dtype)
    idx = np.stack(np.meshgrid(*[np.arange(k) for k in n], indexing="ij"), -1).reshape(-1, 3)
    return lo + idx.astype(dtype) * step


def new_state(n_points, dtype=np.float32):
    return {"tsdf": np.zeros(n_points, dtype), "weight": np.zeros(n_points, np.int32),
            "color": np.zeros((n_points, 3), dtype), "color_weight": np.zeros(n_points, np.int32)}


def integrate(state, x, trunc, poses, K, W, H, directions, depth, opacity, rgb, min_opacity, dtype=np.float32):
    """apply views (poses (V, 3, 4), depth / opacity (V, H W), rgb (V, H W, 3)) in order to `state` (new_state) at the
    points x (N, 3), in place; returns state"""
    f = dtype
    x = np.asarray(x, f)
    K = np.asarray(K, np.float32).reshape(3, 3)
    fx, fy, cx, cy = f(K[0, 0]), f(K[1, 1]), f(K[0, 2]), f(K[1, 2])
    tau = f(trunc)
    one = f(1)
    dirs = np.asarray(directions, f).reshape(-1, 3)
    dn = np.sqrt((dirs[:, 0] * dirs[:, 0] + dirs[:, 1] * dirs[:, 1]) + dirs[:, 2] * dirs[:, 2])
    poses = np.asarray(poses, f).reshape(-1, 3, 4)
    F, Wt, Col, Wc = state["tsdf"], state["weight"], state["color"], state["color_weight"]
    for v in range(poses.shape[0]):
        R, o = poses[v, :, :3], poses[v, :, 3]
        d = x - o
        cam = [(R[0, c] * d[:, 0] + R[1, c] * d[:, 1]) + R[2, c] * d[:, 2] for c in range(3)]
        xc, yc, zc = cam
        ok = zc > 0
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            px = (fx * xc) / zc + cx
            py = (fy * yc) / zc + cy
        ok &= (px >= 0) & (px < f(W)) & (py >= 0) & (py < f(H))
        sel = np.nonzero(ok)[0]
        pix = np.floor(py[sel]).astype(np.int64) * W + np.floor(px[sel]).astype(np.int64)
        op = np.asarray(opacity[v], f)[pix]
        good = op >= f(min_opacity)
        sel, pix, op = sel[good], pix[good], op[good]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            t = np.asarray(depth[v], f)[pix] / op
        good = np.isfinite(t)
        sel, pix, op, t = sel[good], pix[good], op[good], t[good]
        with np.errstate(over="ignore"):  # t near the fp32 limit: sdf overflows to inf, f = 1, as on the device
            sdf = (t - zc[sel]) * dn[pix]
            good = sdf >= -tau
            sel, pix, op, sdf = sel[good], pix[good], op[good], sdf[good]
            fv = np.minimum(one, sdf / tau)
        w = Wt[sel]
        F[sel] = (F[sel] * w.astype(f) + fv) / (w + 1).astype(f)
        Wt[sel] = w + 1
        band = sdf <= tau
        sc, pc, oc = sel[band], pix[band], op[band]
        c = np.minimum(np.asarray(rgb[v], f).reshape(-1, 3)[pc] / oc[:, None], one)
        wc = Wc[sc]
        Col[sc] = (Col[sc] * wc.astype(f)[:, None] + c) / (wc + 1).astype(f)[:, None]
        Wc[sc] = wc + 1
    return state


def _gradient(vol, obs, pts, step):
    """float64 gradient of vol at lattice points pts (k, 3): central differences, one-sided on the border and next to
    an unobserved neighbour, 0 with neither neighbour observed, divided by step"""
    v = vol.astype(np.float64)
    g = np.zeros(pts.shape, np.float64)
    for a in range(3):
        n = vol.shape[a]
        pl, ph = pts.copy(), pts.copy()
        pl[:, a] = np.maximum(pts[:, a] - 1, 0)
        ph[:, a] = np.minimum(pts[:, a] + 1, n - 1)
        lo = np.where((pts[:, a] > 0) & obs[tuple(pl.T)], pl[:, a], pts[:, a])
        hi = np.where((pts[:, a] + 1 < n) & obs[tuple(ph.T)], ph[:, a], pts[:, a])
        pl[:, a], ph[:, a] = lo, hi
        span = hi - lo
        with np.errstate(divide="ignore", invalid="ignore"):
            ga = (v[tuple(ph.T)] - v[tuple(pl.T)]) / (span * float(step[a]))
        g[:, a] = np.where(span > 0, ga, 0.0)
    return g


def masked_marching_cubes(F, Wt, lo, step, normals=False, color=None, color_weight=None):
    """F (n0, n1, n2) float32, Wt the weights (same shape) -> vertices (V, 3) float32, triangles (F, 3) int64[, normals
    (V, 3) float64][, colors (V, 3) uint8 when color (n0, n1, n2, 3) and color_weight are given]"""
    vol = -np.ascontiguousarray(F, np.float32)
    obs = np.asarray(Wt) > 0
    n0, n1, n2 = vol.shape
    lo, step = np.asarray(lo, np.float32), np.asarray(step, np.float32)
    inside = obs & (vol > 0)
    case = np.zeros((n0 - 1, n1 - 1, n2 - 1), np.int64)
    full = np.ones((n0 - 1, n1 - 1, n2 - 1), bool)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= inside[dx:n0 - 1 + dx, dy:n1 - 1 + dy, dz:n2 - 1 + dz].astype(np.int64) << c
        full &= obs[dx:n0 - 1 + dx, dy:n1 - 1 + dy, dz:n2 - 1 + dz]
    case = np.where(full, case, 0).ravel()  # cell linear index order
    nt = NTRI[case]
    cell = np.repeat(np.arange(case.size), nt)
    k = np.arange(cell.size) - np.repeat(np.cumsum(nt) - nt, nt)
    edges = TRI_EDGES[case[cell], k]
    ci, cj, ck = np.unravel_index(cell, (n0 - 1, n1 - 1, n2 - 1))
    corner = EDGE_CORNER[edges]
    p = np.stack([ci[:, None] + (corner & 1), cj[:, None] + ((corner >> 1) & 1), ck[:, None] + ((corner >> 2) & 1)], -1)
    key = ((p[..., 0] * n1 + p[..., 1]) * n2 + p[..., 2]) * 3 + EDGE_AXIS[edges]
    keys, inv = np.unique(key.ravel(), return_inverse=True)
    tris = inv.reshape(-1, 3).astype(np.int64)
    axis = keys % 3
    p0 = np.stack(np.unravel_index(keys // 3, (n0, n1, n2)), -1)
    p1 = p0.copy()
    p1[np.arange(len(keys)), axis] += 1
    v0, v1 = vol[tuple(p0.T)], vol[tuple(p1.T)]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        t = (np.float32(0) - v0) / (v1 - v0)
        q = p0.astype(np.float32)
        q[np.arange(len(keys)), axis] += t
        verts = lo + q * step
    out = [verts, tris]
    if normals:
        g0, g1 = _gradient(vol, obs, p0, step), _gradient(vol, obs, p1, step)
        nrm = -(g0 + t.astype(np.float64)[:, None] * (g1 - g0))
        ln = np.sqrt((nrm * nrm).sum(1))
        out.append(np.where((ln > 0)[:, None], nrm / np.where(ln > 0, ln, 1)[:, None], 0.0))
    if color is not None:
        col = np.asarray(color, np.float32).reshape(n0, n1, n2, 3)
        wc = np.asarray(color_weight)
        c0, c1 = col[tuple(p0.T)], col[tuple(p1.T)]
        both = (wc[tuple(p0.T)] > 0) & (wc[tuple(p1.T)] > 0)
        in0 = inside[tuple(p0.T)]
        c = np.where(both[:, None], c0 + t[:, None] * (c1 - c0), np.where(in0[:, None], c0, c1))
        out.append(np.clip(np.rint(np.float32(255) * c), 0, 255).astype(np.uint8))
    return tuple(out)


def crossed_edges_of_case(m):
    """the 12-edge indices crossed in case m (corner c inside iff bit c)"""
    from .mc_table import EDGES
    return {e for e, (c0, c1, _a) in enumerate(EDGES) if ((m >> c0) & 1) != ((m >> c1) & 1)}
