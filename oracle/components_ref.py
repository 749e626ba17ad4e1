"""numpy + scipy restatement of the connected components of include/ngp_b200.h ("Connected components"): the node and
edge sets built explicitly, scipy.sparse.csgraph.connected_components, each label canonicalised to its component's
smallest node index, and the same selection, inner-cell cleanup and mesh compaction as csrc/components.cu."""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components


def _compact10(v):
    v = v & 0x09249249
    v = (v | (v >> 2)) & 0x030C30C3
    v = (v | (v >> 4)) & 0x0300F00F
    v = (v | (v >> 8)) & 0x030000FF
    v = (v | (v >> 16)) & 0x000003FF
    return v


def morton_coords(G):
    """(G^3, 3) int64: the (x, y, z) of morton code m in row m"""
    m = np.arange(G ** 3, dtype=np.int64)
    return np.stack([_compact10(m), _compact10(m >> 1), _compact10(m >> 2)], 1)


def morton_index(G):
    """(G, G, G) int64: the morton code of (x, y, z)"""
    xyz = morton_coords(G)
    idx = np.empty((G, G, G), np.int64)
    idx[xyz[:, 0], xyz[:, 1], xyz[:, 2]] = np.arange(G ** 3)
    return idx


def half_extent(c, scale):
    """mb_c = fminf(2^(c-1), scale) in fp32, as a Python float"""
    return float(min(np.float32(2.0 ** (c - 1)), np.float32(scale)))


def face(mb, i, G):
    """X_c(i) = mb (2 i / G - 1) in float64 (exact)"""
    return mb * ((2.0 * np.asarray(i, np.float64)) / G - 1.0)


def inner_axis(c, G, scale):
    """(G,) bool: cell x of cascade c >= 1 lies in cascade c - 1's closed box on one axis"""
    mb, mf = half_extent(c, scale), half_extent(c - 1, scale)
    x = np.arange(G)
    return (face(mb, x, G) >= -mf) & (face(mb, x + 1, G) <= mf)


def meet_axis(c, G, scale):
    """(G, G) bool: [s, t] = cell s of cascade c and cell t of cascade c - 1 meet on one axis (closed intervals)"""
    mb, mf = half_extent(c, scale), half_extent(c - 1, scale)
    s = np.arange(G)[:, None]
    t = np.arange(G)[None, :]
    return (face(mf, t, G) <= face(mb, s + 1, G)) & (face(mf, t + 1, G) >= face(mb, s, G))


def unpack(bitfield, cascades, G):
    """(cascades, G^3) bool occupancy in cell order"""
    return np.unpackbits(np.asarray(bitfield, np.uint8), bitorder="little").astype(bool).reshape(cascades, G ** 3)


def nodes(occ, cascades, G, scale):
    """(cascades, G^3) bool: the occupied shell cells"""
    xyz = morton_coords(G)
    node = occ.copy()
    for c in range(1, cascades):
        ia = inner_axis(c, G, scale)
        node[c] &= ~(ia[xyz[:, 0]] & ia[xyz[:, 1]] & ia[xyz[:, 2]])
    return node


def _pairs_meeting(c, G, scale, xyz_s):
    """for cells xyz_s (n, 3) of cascade c: (row into xyz_s, (u, v, w) of cascade c - 1) of every meeting pair"""
    M = meet_axis(c, G, scale)
    lo = np.where(M.any(1), M.argmax(1), 0)
    cnt = M.sum(1)
    W = int(cnt.max()) if cnt.size else 0
    rows, cells = [], []
    for a in range(W):
        for b in range(W):
            for d in range(W):
                off = np.array([a, b, d])
                ok = (off[None, :] < cnt[xyz_s]).all(1)
                r = np.nonzero(ok)[0]
                rows.append(r)
                cells.append(lo[xyz_s[r]] + off[None, :])
    if not rows:
        return np.zeros(0, np.int64), np.zeros((0, 3), np.int64)
    return np.concatenate(rows), np.concatenate(cells)


def grid_edges(node, cascades, G, scale):
    """(E, 2) int64 cell-index pairs: 26-adjacency inside a cascade, closed-box contact with the next finer one"""
    xyz = morton_coords(G)
    midx = morton_index(G)
    G3 = G ** 3
    edges = []
    offs = [(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1) if (dx, dy, dz) > (0, 0, 0)]
    for c in range(cascades):
        m = np.nonzero(node[c])[0]
        p = xyz[m]
        for o in offs:
            q = p + np.array(o)
            ok = ((q >= 0) & (q < G)).all(1)
            j = midx[q[ok, 0], q[ok, 1], q[ok, 2]]
            keep = node[c, j]
            edges.append(np.stack([c * G3 + m[ok][keep], c * G3 + j[keep]], 1))
        if c == 0 or m.size == 0:
            continue
        r, uvw = _pairs_meeting(c, G, scale, p)
        j = midx[uvw[:, 0], uvw[:, 1], uvw[:, 2]]
        keep = node[c - 1, j]
        edges.append(np.stack([c * G3 + m[r[keep]], (c - 1) * G3 + j[keep]], 1))
    return np.concatenate(edges) if edges else np.zeros((0, 2), np.int64)


def components(n, is_node, edges):
    """labels (n,) int32 (smallest node index of the component, -1 off the nodes) and sizes (n,) int32 (at a label)"""
    ids = np.nonzero(is_node)[0]
    pos = np.full(n, -1, np.int64)
    pos[ids] = np.arange(ids.size)
    k = ids.size
    a, b = pos[edges[:, 0]], pos[edges[:, 1]]
    g = sp.coo_matrix((np.ones(a.size, np.int8), (a, b)), shape=(k, k)).tocsr()
    _, comp = connected_components(g, directed=False)
    _, first = np.unique(comp, return_index=True)  # ids ascend, so the first member is the smallest
    lab = ids[first][comp]
    labels = np.full(n, -1, np.int32)
    labels[ids] = lab
    sizes = np.zeros(n, np.int32)
    np.add.at(sizes, lab, 1)
    return labels, sizes


def grid_components(bitfield, cascades, G, scale):
    occ = unpack(bitfield, cascades, G)
    node = nodes(occ, cascades, G, scale)
    return components(cascades * G ** 3, node.reshape(-1), grid_edges(node, cascades, G, scale))


def select(labels, sizes, keep_largest=None, min_size=None):
    """keep (n,) uint8 at the labels and (components, kept): among the keep_largest largest (size descending, ties to the
    smaller label) and at least min_size nodes"""
    n = labels.size
    roots = np.nonzero(labels == np.arange(n))[0]
    order = roots[np.lexsort((roots, -sizes[roots].astype(np.int64)))]
    rank_ok = np.arange(order.size) < (order.size if keep_largest is None else keep_largest)
    size_ok = sizes[order] >= (0 if min_size is None else min_size)
    keep = np.zeros(n, np.uint8)
    keep[order[rank_ok & size_ok]] = 1
    return keep, (int(roots.size), int((rank_ok & size_ok).sum()))


def grid_clean(bitfield, density_grid, cascades, G, scale, labels, keep):
    """(bitfield, density_grid or None, (shell cleared, inner cleared)) after the cleanup, cascade by cascade"""
    occ = unpack(bitfield, cascades, G)
    out = occ.copy()
    removed = np.zeros_like(occ)
    lab = labels.reshape(cascades, G ** 3)
    xyz = morton_coords(G)
    midx = morton_index(G)
    n_shell = n_inner = 0
    for c in range(cascades):
        shell = occ[c] & (lab[c] >= 0)
        drop = np.zeros(G ** 3, bool)
        drop[shell] = keep[lab[c][shell]] == 0
        n_shell += int(drop.sum())
        inner = np.nonzero(occ[c] & (lab[c] < 0))[0]
        if c > 0 and inner.size:
            r, uvw = _pairs_meeting(c, G, scale, xyz[inner])
            j = midx[uvw[:, 0], uvw[:, 1], uvw[:, 2]]
            any_kept = np.zeros(inner.size, bool)
            any_rm = np.zeros(inner.size, bool)
            np.logical_or.at(any_kept, r, out[c - 1, j])
            np.logical_or.at(any_rm, r, removed[c - 1, j])
            d = any_rm & ~any_kept
            drop[inner[d]] = True
            n_inner += int(d.sum())
        out[c] &= ~drop
        removed[c] = drop
    bits = np.packbits(out.reshape(-1), bitorder="little")
    dg = None
    if density_grid is not None:
        dg = np.array(density_grid, np.float32).reshape(cascades, G ** 3).copy()
        dg[removed] = -1.0
    return bits, dg, (n_shell, n_inner)


def mesh_components(triangles, n_vertices):
    """labels (F,) int32 = smallest triangle index of the component (triangles sharing a vertex), sizes (F,) int32"""
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    F = t.shape[0]
    if F == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.int32)
    a = np.concatenate([t[:, 0], t[:, 0]])
    b = np.concatenate([t[:, 1], t[:, 2]])
    g = sp.coo_matrix((np.ones(a.size, np.int8), (a, b)), shape=(n_vertices, n_vertices)).tocsr()
    _, comp = connected_components(g, directed=False)
    tc = comp[t[:, 0]]
    uniq, first = np.unique(tc, return_index=True)
    lut = np.zeros(comp.max() + 1, np.int64)
    lut[uniq] = first
    labels = lut[tc].astype(np.int32)
    sizes = np.bincount(labels, minlength=F).astype(np.int32)
    return labels, sizes


def mesh_filter(vertices, triangles, labels, keep, normals=None, colors=None):
    """the kept triangles in input order and the vertices they use in input order, renumbered"""
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    V = np.asarray(vertices).reshape(-1, 3).shape[0]
    kt = keep[labels].astype(bool) if t.shape[0] else np.zeros(0, bool)
    used = np.zeros(V, bool)
    used[t[kt].reshape(-1)] = True
    newidx = np.cumsum(used) - 1
    pick = lambda a: None if a is None else np.asarray(a).reshape(-1, 3)[used]  # noqa: E731
    return {"vertices": pick(vertices), "triangles": newidx[t[kt]].astype(np.int64), "normals": pick(normals),
            "colors": pick(colors)}
