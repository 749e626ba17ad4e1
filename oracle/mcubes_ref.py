"""Plain numpy restatement of the device marching cubes (ngp_marching_cubes_count / _emit, csrc/mesh.cu), written from
the rules in include/ngp_b200.h, for the tests. It replaces the mesh cell of the reference's notebook (test.ipynb:
`mcubes.marching_cubes(sigma, 20.)`), whose package is not a dependency here.

Every cell is classified at once; each cell's triangles reference their vertices by the key (lattice point p, axis a)
of the crossed lattice edge, and the distinct keys, sorted, ARE the vertex order (linear index of p, then a). Vertex
positions are computed in np.float32 with the kernel's operation order; normals in float64.
"""
import numpy as np

from .mc_table import EDGES, TRIS

NTRI = np.array([len(t) for t in TRIS], np.int64)
TRI_EDGES = np.full((256, 5, 3), -1, np.int64)
for _m, _tris in enumerate(TRIS):
    for _k, _t in enumerate(_tris):
        TRI_EDGES[_m, _k] = _t
EDGE_CORNER = np.array([e[0] for e in EDGES], np.int64)
EDGE_AXIS = np.array([e[2] for e in EDGES], np.int64)


def _gradient(vol, pts, step):
    """float64 gradient of the volume at lattice points pts (k, 3): central differences, one-sided on the border,
    divided by step"""
    v = vol.astype(np.float64)
    g = np.empty(pts.shape, np.float64)
    for a in range(3):
        n = vol.shape[a]
        lo = np.maximum(pts[:, a] - 1, 0)
        hi = np.minimum(pts[:, a] + 1, n - 1)
        pl, ph = pts.copy(), pts.copy()
        pl[:, a], ph[:, a] = lo, hi
        g[:, a] = (v[tuple(ph.T)] - v[tuple(pl.T)]) / (hi - lo) / float(step[a])
    return g


def marching_cubes(vol, iso, lo=None, step=None, normals=False):
    """vol (n0, n1, n2) float32, inside iff v > iso -> vertices (V, 3) float32, triangles (F, 3) int64[, normals (V, 3)
    float64]. Vertex of lattice edge (p, a): t = (iso - v0) / (v1 - v0), q = p with q_a += t, vertex = lo + q * step."""
    vol = np.ascontiguousarray(vol, np.float32)
    n0, n1, n2 = vol.shape
    assert min(vol.shape) >= 2
    iso = np.float32(iso)
    lo = np.zeros(3, np.float32) if lo is None else np.asarray(lo, np.float32)
    step = np.ones(3, np.float32) if step is None else np.asarray(step, np.float32)
    inside = vol > iso
    case = np.zeros((n0 - 1, n1 - 1, n2 - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= inside[dx:n0 - 1 + dx, dy:n1 - 1 + dy, dz:n2 - 1 + dz].astype(np.int64) << c
    case = case.ravel()  # cell linear index order
    nt = NTRI[case]
    cell = np.repeat(np.arange(case.size), nt)
    k = np.arange(cell.size) - np.repeat(np.cumsum(nt) - nt, nt)  # triangle index within its case
    edges = TRI_EDGES[case[cell], k]  # (F, 3)
    ci, cj, ck = np.unravel_index(cell, (n0 - 1, n1 - 1, n2 - 1))
    corner = EDGE_CORNER[edges]
    p = np.stack([ci[:, None] + (corner & 1), cj[:, None] + ((corner >> 1) & 1), ck[:, None] + ((corner >> 2) & 1)], -1)
    key = ((p[..., 0] * n1 + p[..., 1]) * n2 + p[..., 2]) * 3 + EDGE_AXIS[edges]
    keys, inv = np.unique(key.ravel(), return_inverse=True)
    tris = inv.reshape(-1, 3).astype(np.int64)

    axis = keys % 3
    lin = keys // 3
    p0 = np.stack(np.unravel_index(lin, (n0, n1, n2)), -1)
    p1 = p0.copy()
    p1[np.arange(len(keys)), axis] += 1
    v0 = vol[tuple(p0.T)]
    v1 = vol[tuple(p1.T)]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        t = (iso - v0) / (v1 - v0)  # float32
        q = p0.astype(np.float32)
        q[np.arange(len(keys)), axis] += t
        verts = lo + q * step  # float32, multiply then add
    if not normals:
        return verts, tris
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        g0, g1 = _gradient(vol, p0, step), _gradient(vol, p1, step)
        td = t.astype(np.float64)[:, None]
        nrm = -(g0 + td * (g1 - g0))
        ln = np.sqrt((nrm * nrm).sum(1))
        nrm = np.where((ln > 0)[:, None], nrm / np.where(ln > 0, ln, 1)[:, None], 0.0)
    return verts, tris, nrm


def directed_edges(tris):
    """(3F, 2) directed edges a -> b of the triangles"""
    return np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])


def unpaired_edges(tris):
    """directed edges used more than once, and directed edges whose reverse is not used once: an oriented closed
    surface has none"""
    d = directed_edges(tris)
    if len(d) == 0:
        return d
    m = int(d.max()) + 1
    code = d[:, 0] * m + d[:, 1]
    u, cnt = np.unique(code, return_counts=True)
    rev = d[:, 1] * m + d[:, 0]
    idx = np.searchsorted(u, rev)
    idx = np.minimum(idx, len(u) - 1)
    has_rev = (u[idx] == rev) & (cnt[idx] == 1)
    dup = cnt[np.searchsorted(u, code)] > 1
    return d[dup | ~has_rev]


def euler_characteristic(verts, tris):
    d = np.sort(directed_edges(tris), 1)
    n_edges = len(np.unique(d[:, 0] * (len(verts) + 1) + d[:, 1]))
    return len(verts) - n_edges + len(tris)


def signed_volume(verts, tris):
    v = verts.astype(np.float64)
    a, b, c = v[tris[:, 0]], v[tris[:, 1]], v[tris[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6)
