"""Mesh extraction from a trained model on the device: the mesh cell of the reference's notebook (test.ipynb) without
PyMCubes, trimesh or scikit-image.

    density_volume(model, resolution, bounds=None)                σ on a lattice, (n0, n1, n2) fp32 on the device
    marching_cubes(volume, iso, lo=None, step=None, normals=False) indexed mesh of a σ volume, on the device
    extract_mesh(model, resolution=256, bounds=None, threshold=20.0, normals=True, colors=False)
    occupied_bricks(model, resolution, bounds=None)               brick mask of the occupancy grid, bool on the device
    extract_mesh_sparse(model, resolution=1024, bounds=None, threshold=20.0, normals=True, colors=False,
                        return_stats=False)                       the mesh of σ where the occupancy grid allows a surface
    simplify_mesh(mesh, grid, bounds=None)                        vertex clustering with quadric-error placement
    mesh_components(mesh)                                         component label and size per triangle
    remove_small_components(mesh, keep_largest=None, min_triangles=None, return_stats=False)
                                                                  the mesh without its small pieces
    bake_texture(model, mesh, size=4096, offset=0.0, samples=16, return_texels=False)
                                                                  a per-triangle texture atlas and its colours
    write_ply(path, vertices, triangles, normals=None, colors=None) binary little-endian PLY, numpy only
    write_obj(path, vertices, triangles, normals=None, uv=None, texture=None, png_mode="dynamic")
                                                                  OBJ [+ MTL + PNG encoded on the device]

The σ lattice is evaluated by `ngp_density_lattice` (csrc/network.cu), which generates its points instead of reading
them, and the mesh by `ngp_marching_cubes_count` / `_emit` (csrc/mesh.cu), which work through the volume in slabs;
semantics in include/ngp_b200.h. The only host synchronisations are the read-back of the vertex and triangle counts
and emit's check of the capacities against them. Model and volume must live on a CUDA device, otherwise RuntimeError;
there is no CPU path.

The sparse path (`ngp_mesh_brick_mask`, `ngp_mesh_sparse_*` in csrc/mesh.cu) cuts the lattice into bricks of 8^3
points, evaluates σ only on the bricks near occupied cells of `model.density_bitfield` and keeps σ in memory only for
the bricks a surface passes through; its cost and memory follow the occupied volume and the surface, not N^3.

simplify_mesh (`ngp_mesh_simplify_count` / `_emit`) reduces a mesh to at most one vertex per cell of a grid^3 cluster
grid, placed where the cell's triangle planes meet (quadric error), so thin parts and sharp edges a coarser lattice
would lose keep their place at a fraction of the triangle count.

mesh_components / remove_small_components (`ngp_mesh_components`, `ngp_components_select`, `ngp_mesh_filter_count` /
`_emit` in csrc/components.cu) split a mesh into the pieces that share vertices, on the device, and keep the large ones:
floaters and the closed shells of cavities no ray reaches go, whichever extraction made the mesh.

bake_texture (`ngp_mesh_texture_atlas` / `_texels` / `_bake` in csrc/texture.cu) gives every triangle its own square
of a texture atlas and bakes the model's colours into it through the fused forward, so a simplified mesh keeps the
detail its few vertices cannot hold; write_obj saves mesh, uv and texture for tools that expect a textured OBJ.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .models.networks import _net_struct


def _chk(t, what):
    if not t.is_cuda:
        raise RuntimeError("ngp_pl_b200.mesh.%s needs CUDA tensors (got %s); there is no CPU path" % (what, t.device))


def _st(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _three(v, dtype):
    a = np.asarray(v, dtype).reshape(-1)
    if a.size == 1:
        a = np.repeat(a, 3)
    if a.size != 3:
        raise RuntimeError("ngp_pl_b200.mesh: expected a scalar or 3 values, got %s" % (v,))
    return a


def lattice(resolution, lo, hi):
    """NgpLattice of `resolution` (int or 3 ints, >= 2 each) points from lo to hi (3 values each); step = (hi - lo) /
    (n - 1) in fp32"""
    n = _three(resolution, np.int64)
    if (n < 2).any() or (n >= 2 ** 31).any():
        raise RuntimeError("ngp_pl_b200.mesh: resolution must be at least 2 on every axis, got %s" % (resolution,))
    lo = _three(lo, np.float32)
    step = (_three(hi, np.float32) - lo) / (n - 1).astype(np.float32)  # fp32 throughout
    lat = _lib.NgpLattice()
    for a in range(3):
        lat.n[a], lat.lo[a], lat.step[a] = int(n[a]), float(lo[a]), float(step[a])
    return lat


def _bounds(model, bounds):
    if bounds is None:
        return model._xyz_min_host, model._xyz_max_host
    lo, hi = bounds
    if isinstance(lo, torch.Tensor):
        lo = lo.detach().cpu().numpy()
    if isinstance(hi, torch.Tensor):
        hi = hi.detach().cpu().numpy()
    return lo, hi


def _density(model, lat):
    dev = model.xyz_encoder.params.device
    sigma = torch.empty(lat.n[0], lat.n[1], lat.n[2], device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        net, keep = _net_struct(model)
        _lib.check(_lib.lib().ngp_density_lattice(C.byref(net), C.byref(lat), sigma.data_ptr(), _st(dev)), "ngp_density_lattice")
    return sigma


@torch.no_grad()
def density_volume(model, resolution, bounds=None):
    """σ = model.density at every point of a resolution^3 (or n0 x n1 x n2) lattice spanning `bounds` = (lo, hi)
    (default: the model's box xyz_min .. xyz_max), as a (n0, n1, n2) fp32 tensor on the model's device with axis 0 = x.
    Point (i, j, k) is lo + idx * step with step = (hi - lo) / (n - 1), all in fp32: bitwise what model.density gives
    for the same points materialised as `lo + torch.arange(n).float() * step`. The points themselves are never stored."""
    _chk(model.xyz_encoder.params, "density_volume")
    lo, hi = _bounds(model, bounds)
    return _density(model, lattice(resolution, lo, hi))


def _mc(volume, iso, lat, normals):
    _chk(volume, "marching_cubes")
    if volume.dim() != 3 or volume.dtype != torch.float32:
        raise RuntimeError("ngp_pl_b200.mesh.marching_cubes: expected a 3-D float32 volume, got %s %s"
                           % (tuple(volume.shape), volume.dtype))
    vol = volume.contiguous()
    dev = vol.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_marching_cubes_workspace(C.byref(lat))
        if ws_bytes == 0:
            raise RuntimeError("ngp_pl_b200.mesh.marching_cubes: unsupported volume shape %s" % (tuple(vol.shape),))
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        counts = torch.empty(2, device=dev, dtype=torch.int64)
        st = _st(dev)
        _lib.check(L.ngp_marching_cubes_count(vol.data_ptr(), C.byref(lat), float(iso), counts.data_ptr(), ws.data_ptr(),
                                              ws_bytes, st), "ngp_marching_cubes_count")
        nv, nt = (int(x) for x in counts.cpu())
        verts = torch.empty(nv, 3, device=dev, dtype=torch.float32)
        tris = torch.empty(nt, 3, device=dev, dtype=torch.int64)
        nrm = torch.empty(nv, 3, device=dev, dtype=torch.float32) if normals else None
        if nv > 0:
            _lib.check(L.ngp_marching_cubes_emit(vol.data_ptr(), C.byref(lat), float(iso), verts.data_ptr(),
                                                 nrm.data_ptr() if normals else None, tris.data_ptr(), nv, nt, ws.data_ptr(),
                                                 ws_bytes, st), "ngp_marching_cubes_emit")
    return verts, tris, nrm


@torch.no_grad()
def marching_cubes(volume, iso, lo=None, step=None, normals=False):
    """Indexed triangle mesh of the level set `iso` of a (n0, n1, n2) float32 CUDA volume: vertices (V, 3) float32,
    triangles (F, 3) int64 [, normals (V, 3) float32], all on the volume's device. A value is inside iff v > iso.
    Vertex of lattice edge (p, axis a): lo + q * step, q = p with q_a = p_a + (iso - v0) / (v1 - v0) (fp32). Without
    lo / step the vertices are in index space on the caller's axis order -- the vertex placement of
    mcubes.marching_cubes(volume, iso); only the triangulation of ambiguous faces differs (this one is watertight).
    Triangles are counter-clockwise seen from outside; normals point out of the inside region."""
    _chk(volume, "marching_cubes")
    if volume.dim() != 3:
        raise RuntimeError("ngp_pl_b200.mesh.marching_cubes: expected a 3-D volume, got shape %s" % (tuple(volume.shape),))
    lat = lattice(tuple(volume.shape), 0.0, 0.0)
    lo3, step3 = _three(0.0 if lo is None else lo, np.float32), _three(1.0 if step is None else step, np.float32)
    for a in range(3):
        lat.lo[a], lat.step[a] = float(lo3[a]), float(step3[a])
    verts, tris, nrm = _mc(volume, iso, lat, normals)
    return (verts, tris, nrm) if normals else (verts, tris)


@torch.no_grad()
def extract_mesh(model, resolution=256, bounds=None, threshold=20.0, normals=True, colors=False):
    """density_volume then marching_cubes at `threshold`, with world-space vertices. Returns a dict with 'vertices'
    (V, 3) float32, 'triangles' (F, 3) int64, 'normals' (V, 3) float32 or None, 'colors' (V, 3) uint8 or None, on the
    model's device; `write_ply(path, **mesh)` saves it.

    threshold defaults to the notebook's 20. The notebook's mesh cell has two coordinate quirks that are NOT reproduced:
    its np.meshgrid(x, y, z) uses 'xy' indexing, so x and y come out swapped, and it maps vertices with `vertices / N`,
    which sends lattice index N-1 to (N-1)/N instead of the box edge. Here axis 0 is x and lattice index n-1 lies on hi.

    colors=True evaluates model(vertices, -normals) through the fused forward -- the surface seen head-on -- and returns
    rgb as uint8 (a vertex with a zero normal is seen along -z)."""
    _chk(model.xyz_encoder.params, "extract_mesh")
    lo, hi = _bounds(model, bounds)
    lat = lattice(resolution, lo, hi)
    sigma = _density(model, lat)
    verts, tris, nrm = _mc(sigma, threshold, lat, normals or colors)
    rgb = _vertex_colors(model, verts, nrm) if colors else None
    return {"vertices": verts, "triangles": tris, "normals": nrm if normals else None, "colors": rgb}


def _vertex_colors(model, verts, nrm):
    """rgb of model(verts, -nrm) as uint8; a vertex with a zero normal is seen along -z"""
    d = -nrm
    flat = (nrm == 0).all(1)
    d[flat] = torch.tensor([0.0, 0.0, 1.0], device=d.device)
    rgb = torch.empty(0, 3, device=verts.device, dtype=torch.uint8)
    if verts.shape[0] > 0:
        _, c = model(verts, d)
        rgb = (c.float() * 255).round().clamp(0, 255).to(torch.uint8)
    return rgb


def _brick_mask(model, lat):
    """the brick bitmask (int32 words) of lattice `lat` over the model's occupancy bitfield"""
    dev = model.density_bitfield.device
    _chk(model.density_bitfield, "occupied_bricks")
    G, C_ = int(model.grid_size), int(model.cascades)
    if model.density_bitfield.numel() * 8 != C_ * G ** 3:
        raise RuntimeError("ngp_pl_b200.mesh: density_bitfield has %d bytes, %d cascades of %d^3 cells need %d"
                           % (model.density_bitfield.numel(), C_, G, C_ * G ** 3 // 8))
    L = _lib.lib()
    nbytes = L.ngp_mesh_bricks_bytes(C.byref(lat))
    if nbytes == 0:
        raise RuntimeError("ngp_pl_b200.mesh: the sparse path takes 2..%d points per axis, got %s"
                           % (_lib.NGP_MESH_MAX_N, tuple(lat.n)))
    mask = torch.empty(nbytes // 4, device=dev, dtype=torch.int32)
    with torch.cuda.device(dev):
        _lib.check(L.ngp_mesh_brick_mask(model.density_bitfield.contiguous().data_ptr(), C_, G, float(model.scale),
                                         C.byref(lat), mask.data_ptr(), _st(dev)), "ngp_mesh_brick_mask")
    return mask


@torch.no_grad()
def occupied_bricks(model, resolution, bounds=None):
    """(nb0, nb1, nb2) bool CUDA tensor, nb = ceil(n / 8): the bricks of 8^3 lattice points (lattice as in
    density_volume) near an occupied cell of model.density_bitfield -- the rule of include/ngp_b200.h (brick mask)"""
    _chk(model.xyz_encoder.params, "occupied_bricks")
    lo, hi = _bounds(model, bounds)
    lat = lattice(resolution, lo, hi)
    words = _brick_mask(model, lat)
    B = _lib.NGP_MESH_BRICK
    nb = [(lat.n[a] + B - 1) // B for a in range(3)]
    bits = (words.view(-1, 1) >> torch.arange(32, device=words.device, dtype=torch.int32)) & 1
    return bits.reshape(-1)[:nb[0] * nb[1] * nb[2]].bool().reshape(nb)


def _free_bytes(dev):
    free, _ = torch.cuda.mem_get_info(dev)
    return free + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)


def _need(dev, nbytes, what, fn="extract_mesh_sparse"):
    if nbytes > _free_bytes(dev):
        raise RuntimeError("ngp_pl_b200.mesh.%s: %s need %d bytes of device memory, %d are free"
                           % (fn, what, nbytes, _free_bytes(dev)))


@torch.no_grad()
def extract_mesh_sparse(model, resolution=1024, bounds=None, threshold=20.0, normals=True, colors=False,
                        return_stats=False):
    """The mesh of σ_masked at `threshold`: σ at the points of the bricks occupied_bricks() marks, 0 elsewhere. Returns
    exactly what marching_cubes(σ_masked, threshold) with world-space vertices returns -- the same vertices in the same
    order, triangles and normals, bitwise -- and colours as extract_mesh computes them; the same dict keys as
    extract_mesh. Where the occupancy grid is empty the surface is closed, so the mesh stays watertight. It is not
    extract_mesh's mesh: a surface extract_mesh finds away from occupied cells is not here.

    resolution: 2..8192 points per axis (int or 3 ints); threshold must be > 0. σ is stored only for the bricks a surface
    passes through; RuntimeError, before allocating, when those bricks or the output do not fit in free device memory.
    return_stats=True also returns {'active', 'visited', 'surface'} brick counts."""
    _chk(model.xyz_encoder.params, "extract_mesh_sparse")
    if not threshold > 0:
        raise RuntimeError("ngp_pl_b200.mesh.extract_mesh_sparse: threshold must be > 0, got %r" % (threshold,))
    lo, hi = _bounds(model, bounds)
    lat = lattice(resolution, lo, hi)
    dev = model.xyz_encoder.params.device
    L = _lib.lib()
    iso = float(threshold)
    with torch.cuda.device(dev):
        mask = _brick_mask(model, lat)
        net, keep = _net_struct(model)
        st = _st(dev)
        ws_bytes = L.ngp_mesh_sparse_workspace(C.byref(lat))
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        bc = (C.c_int64 * 3)()
        _lib.check(L.ngp_mesh_sparse_bricks(C.byref(net), C.byref(lat), iso, mask.data_ptr(), bc, ws.data_ptr(), ws_bytes,
                                            st), "ngp_mesh_sparse_bricks")
        n_surf = int(bc[2])
        sf_bytes = L.ngp_mesh_surface_workspace(C.byref(lat), n_surf)
        _need(dev, sf_bytes, "%d surface bricks" % n_surf)
        sf = torch.empty(sf_bytes, device=dev, dtype=torch.uint8)
        tot = (C.c_int64 * 2)()
        _lib.check(L.ngp_mesh_sparse_count(C.byref(net), C.byref(lat), iso, mask.data_ptr(), n_surf, tot, ws.data_ptr(),
                                           ws_bytes, sf.data_ptr(), sf_bytes, st), "ngp_mesh_sparse_count")
        del ws
        nv, nt = int(tot[0]), int(tot[1])
        want_n = normals or colors
        _need(dev, nv * 12 * (2 if want_n else 1) + nt * 24, "%d vertices and %d triangles" % (nv, nt))
        verts = torch.empty(nv, 3, device=dev, dtype=torch.float32)
        tris = torch.empty(nt, 3, device=dev, dtype=torch.int64)
        nrm = torch.empty(nv, 3, device=dev, dtype=torch.float32) if want_n else None
        if nv > 0:
            _lib.check(L.ngp_mesh_sparse_emit(C.byref(lat), iso, n_surf, verts.data_ptr(), nrm.data_ptr() if want_n else None,
                                              tris.data_ptr(), nv, nt, sf.data_ptr(), sf_bytes, st), "ngp_mesh_sparse_emit")
        del sf
    rgb = _vertex_colors(model, verts, nrm) if colors else None
    m = {"vertices": verts, "triangles": tris, "normals": nrm if normals else None, "colors": rgb}
    if return_stats:
        return m, {"active": int(bc[0]), "visited": int(bc[1]), "surface": n_surf}
    return m


def cluster_grid(lo, hi, grid):
    """NgpClusterGrid of rule 1 (include/ngp_b200.h), in fp32: h = max(hi - lo) / grid, n = min(grid, max(1,
    ceil((hi - lo) / h))) cells per axis"""
    lo = _three(lo, np.float32)
    ext = _three(hi, np.float32) - lo
    h = np.float32(ext.max() / np.float32(grid))
    n = np.minimum(np.maximum(1, np.ceil(ext / h).astype(np.int64)), int(grid))
    g = _lib.NgpClusterGrid()
    for a in range(3):
        g.lo[a], g.n[a] = float(lo[a]), int(n[a])
    g.h = float(h)
    return g


@torch.no_grad()
def simplify_mesh(mesh, grid, bounds=None):
    """Vertex clustering with quadric-error placement (Lindstrom 2000; the rule is in include/ngp_b200.h) of a mesh
    dict as extract_mesh / extract_mesh_sparse return it: at most one vertex per cell of a cluster grid of cubes of side
    max(hi - lo) / grid over `bounds` = (lo, hi), placed at the least quadric error of the cell's triangle planes
    within the box of the cell's vertices. Triangles whose corners fall in fewer than three cells are dropped, and so
    is every later triangle with the same cells in the same cyclic order; the mesh need not stay manifold. Returns a
    dict with the same keys: normals are the normalised sums of the cell's normals and colours the rounded means of its
    colours, None where the input's are. Vertices outside the bounds join the border cells.

    grid: 1..65536. bounds=None: the bounding box of the vertices (one device min / max and its read-back). RuntimeError,
    before allocating, for CPU tensors, a grid out of range, lo >= hi on an axis, or a workspace or output that does
    not fit in free device memory. Deterministic: two calls are bitwise equal."""
    verts, tris = mesh["vertices"], mesh["triangles"]
    nrm, col = mesh.get("normals"), mesh.get("colors")
    for t, what in ((verts, "vertices"), (tris, "triangles"), (nrm, "normals"), (col, "colors")):
        if t is not None:
            _chk(t, "simplify_mesh")
    if isinstance(grid, bool) or not isinstance(grid, (int, np.integer)) or not 1 <= grid <= _lib.NGP_SIMPLIFY_MAX_GRID:
        raise RuntimeError("ngp_pl_b200.mesh.simplify_mesh: grid must be an integer in 1..%d, got %r"
                           % (_lib.NGP_SIMPLIFY_MAX_GRID, grid))
    dev = verts.device
    verts = verts.detach().to(torch.float32).reshape(-1, 3).contiguous()
    tris = tris.detach().to(torch.int64).reshape(-1, 3).contiguous()
    V, F = verts.shape[0], tris.shape[0]
    if nrm is not None:
        nrm = nrm.detach().to(torch.float32).reshape(-1, 3).contiguous()
    if col is not None:
        col = col.detach().to(torch.uint8).reshape(-1, 3).contiguous()
    for t, what in ((nrm, "normals"), (col, "colors")):
        if t is not None and t.shape[0] != V:
            raise RuntimeError("ngp_pl_b200.mesh.simplify_mesh: %d %s for %d vertices" % (t.shape[0], what, V))
    if bounds is None:
        if V == 0:
            lo, hi = np.zeros(3, np.float32), np.ones(3, np.float32)
        else:
            mn, mx = torch.aminmax(verts, dim=0)
            lo, hi = mn.cpu().numpy(), mx.cpu().numpy()
            if not (hi - lo).max() > 0:
                raise RuntimeError("ngp_pl_b200.mesh.simplify_mesh: the vertices span no volume (%s .. %s); pass bounds"
                                   % (lo, hi))
    else:
        lo, hi = (_np(b).astype(np.float32).reshape(-1) for b in bounds)
        lo, hi = _three(lo, np.float32), _three(hi, np.float32)
        if not (np.isfinite(lo).all() and np.isfinite(hi).all() and (lo < hi).all()):
            raise RuntimeError("ngp_pl_b200.mesh.simplify_mesh: bounds need lo < hi on every axis, got %s .. %s" % (lo, hi))
    g = cluster_grid(lo, hi, int(grid))
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_mesh_simplify_workspace(V, F)
        if ws_bytes == 0:
            raise RuntimeError("ngp_pl_b200.mesh.simplify_mesh: %d vertices and %d triangles: both must be below 2^31"
                               % (V, F))
        _need(dev, ws_bytes, "the workspace of %d vertices and %d triangles" % (V, F), "simplify_mesh")
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        st = _st(dev)
        tot = (C.c_int64 * 2)()
        _lib.check(L.ngp_mesh_simplify_count(verts.data_ptr(), V, tris.data_ptr(), F, C.byref(g), tot, ws.data_ptr(),
                                             ws_bytes, st), "ngp_mesh_simplify_count")
        nv, nt = int(tot[0]), int(tot[1])
        _need(dev, nv * (12 + (12 if nrm is not None else 0) + (3 if col is not None else 0)) + nt * 24,
              "%d vertices and %d triangles" % (nv, nt), "simplify_mesh")
        out_v = torch.empty(nv, 3, device=dev, dtype=torch.float32)
        out_t = torch.empty(nt, 3, device=dev, dtype=torch.int64)
        out_n = torch.empty(nv, 3, device=dev, dtype=torch.float32) if nrm is not None else None
        out_c = torch.empty(nv, 3, device=dev, dtype=torch.uint8) if col is not None else None
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        if nv > 0:
            _lib.check(L.ngp_mesh_simplify_emit(tris.data_ptr(), V, F, ptr(nrm), ptr(col), out_v.data_ptr(), ptr(out_n),
                                                ptr(out_c), out_t.data_ptr(), nv, nt, ws.data_ptr(), ws_bytes, st),
                       "ngp_mesh_simplify_emit")
        del ws
    return {"vertices": out_v, "triangles": out_t, "normals": out_n, "colors": out_c}


def _mesh_in(mesh, fn):
    verts, tris = mesh["vertices"], mesh["triangles"]
    nrm, col = mesh.get("normals"), mesh.get("colors")
    for t in (verts, tris, nrm, col):
        if t is not None:
            _chk(t, fn)
    verts = verts.detach().to(torch.float32).reshape(-1, 3).contiguous()
    tris = tris.detach().to(torch.int64).reshape(-1, 3).contiguous()
    V = verts.shape[0]
    if nrm is not None:
        nrm = nrm.detach().to(torch.float32).reshape(-1, 3).contiguous()
    if col is not None:
        col = col.detach().to(torch.uint8).reshape(-1, 3).contiguous()
    for t, what in ((nrm, "normals"), (col, "colors")):
        if t is not None and t.shape[0] != V:
            raise RuntimeError("ngp_pl_b200.mesh.%s: %d %s for %d vertices" % (fn, t.shape[0], what, V))
    return verts, tris, nrm, col


def _components(tris, V, fn):
    F = tris.shape[0]
    dev = tris.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_mesh_components_workspace(V, F)
        if ws_bytes == 0:
            raise RuntimeError("ngp_pl_b200.mesh.%s: %d vertices and %d triangles: both must be below 2^31" % (fn, V, F))
        _need(dev, ws_bytes + F * 8, "the components of %d vertices and %d triangles" % (V, F), fn)
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        labels = torch.empty(F, device=dev, dtype=torch.int32)
        sizes = torch.empty(F, device=dev, dtype=torch.int32)
        rc = L.ngp_mesh_components(tris.data_ptr(), V, F, labels.data_ptr(), sizes.data_ptr(), ws.data_ptr(), ws_bytes,
                                   _st(dev))
        if rc == -22 and F > 0:
            raise RuntimeError("ngp_pl_b200.mesh.%s: a triangle index lies outside [0, %d)" % (fn, V))
        _lib.check(rc, "ngp_mesh_components")
    return labels, sizes


@torch.no_grad()
def mesh_components(mesh):
    """Connected components of a mesh dict as extract_mesh / extract_mesh_sparse / simplify_mesh return it: triangles
    that share a vertex index are connected. Returns (labels, sizes), (F,) int32 each on the mesh's device: labels[t] =
    the smallest triangle index of t's component, sizes[l] = the number of triangles of the component labelled l (0 at
    every index that is not a label). RuntimeError for CPU tensors, V or F >= 2^31 or a triangle index outside [0, V).
    Deterministic: two calls are bitwise equal."""
    verts, tris, _, _ = _mesh_in(mesh, "mesh_components")
    return _components(tris, verts.shape[0], "mesh_components")


@torch.no_grad()
def remove_small_components(mesh, keep_largest=None, min_triangles=None, return_stats=False):
    """The mesh without the components that are not among the keep_largest largest (by triangle count, ties to the
    smaller label) or have fewer than min_triangles triangles; at least one criterion is required, and with both a
    component must pass both. Kept triangles stay in input order with their corner order, the vertices they use stay in
    input order and are renumbered; normals and colours go with their vertices. Returns a dict with the same keys as
    the input (a mesh nothing is removed from comes back bitwise); return_stats=True also returns {'components', 'kept'}.
    RuntimeError as mesh_components, and before allocating when the output does not fit in free device memory."""
    from .components import criterion, select_components
    fn = "mesh.remove_small_components"
    keep_largest = criterion(keep_largest, "keep_largest", fn)
    min_triangles = criterion(min_triangles, "min_triangles", fn)
    if keep_largest is None and min_triangles is None:
        raise RuntimeError("ngp_pl_b200.%s: give keep_largest, min_triangles, or both" % fn)
    verts, tris, nrm, col = _mesh_in(mesh, "remove_small_components")
    V, F = verts.shape[0], tris.shape[0]
    dev = verts.device
    labels, sizes = _components(tris, V, "remove_small_components")
    keep, stats = select_components(labels, sizes, keep_largest, min_triangles, fn)
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_mesh_filter_workspace(V, F)
        _need(dev, ws_bytes, "the filter workspace of %d vertices and %d triangles" % (V, F), "remove_small_components")
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        st = _st(dev)
        tot = (C.c_int64 * 2)()
        _lib.check(L.ngp_mesh_filter_count(tris.data_ptr(), V, F, labels.data_ptr(), keep.data_ptr(), tot, ws.data_ptr(),
                                           ws_bytes, st), "ngp_mesh_filter_count")
        del labels, sizes, keep
        nv, nt = int(tot[0]), int(tot[1])
        _need(dev, nv * (12 + (12 if nrm is not None else 0) + (3 if col is not None else 0)) + nt * 24,
              "%d vertices and %d triangles" % (nv, nt), "remove_small_components")
        out_v = torch.empty(nv, 3, device=dev, dtype=torch.float32)
        out_t = torch.empty(nt, 3, device=dev, dtype=torch.int64)
        out_n = torch.empty(nv, 3, device=dev, dtype=torch.float32) if nrm is not None else None
        out_c = torch.empty(nv, 3, device=dev, dtype=torch.uint8) if col is not None else None
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        _lib.check(L.ngp_mesh_filter_emit(verts.data_ptr(), ptr(nrm), ptr(col), tris.data_ptr(), V, F, out_v.data_ptr(),
                                          ptr(out_n), ptr(out_c), out_t.data_ptr(), nv, nt, ws.data_ptr(), ws_bytes, st),
                   "ngp_mesh_filter_emit")
        del ws
    m = {"vertices": out_v, "triangles": out_t, "normals": out_n, "colors": out_c}
    return (m, stats) if return_stats else m


def texture_size_for(n_triangles):
    """the smallest atlas side that holds n_triangles squares of the smallest size"""
    W = _lib.NGP_TEXTURE_MIN_SIZE
    while n_triangles * _lib.NGP_TEXTURE_MIN_SQUARE ** 2 > W * W:
        W *= 2
    return W


@torch.no_grad()
def bake_texture(model, mesh, size=4096, offset=0.0, samples=16, return_texels=False):
    """A texture atlas of side `size` for a mesh dict as extract_mesh / extract_mesh_sparse / simplify_mesh return it,
    and its colours from the model (the rule is in include/ngp_b200.h). Every triangle gets its own power-of-two square,
    packed along the Morton curve, with the triangle placed undistorted one texel inside it. Every texel bilinear
    filtering of a point of a triangle reads is baked: a volume render of `samples` samples along -n from `offset` world
    units outside the surface point the texel maps to, whose own colour is the background (offset 0: the model's colour
    at the point, seen head-on). Other texels are 0.

    Returns {'uv': (F, 3, 2) float32 texel coordinates per corner (divide by size for OBJ's vt), 'squares': (F, 3) int32
    (x0, y0, side), 'texture': (size, size, 3) uint8 (row 0 is the top: texel row y is image row size - 1 - y)} on the
    model's device; return_texels=True adds the texel map: 'texel' (n,) int64 atlas indices (Morton, x in the even bits,
    ascending), 'triangle' (n,) int32, 'point' and 'normal' (n, 3) float32.

    size: a power of two in 16..16384 that holds 16 F texels; offset: >= 0 and finite; samples: 1..256. RuntimeError,
    before allocating, for CPU tensors, a value out of range (a size too small names the one that fits) or memory that
    is not free; also for a triangle index outside [0, V). Deterministic: two calls are bitwise equal."""
    verts, tris, nrm = mesh["vertices"], mesh["triangles"], mesh.get("normals")
    _chk(model.xyz_encoder.params, "bake_texture")
    for t in (verts, tris, nrm):
        if t is not None:
            _chk(t, "bake_texture")
    W = size
    if isinstance(W, bool) or not isinstance(W, (int, np.integer)) or not (
            _lib.NGP_TEXTURE_MIN_SIZE <= W <= _lib.NGP_TEXTURE_MAX_SIZE) or W & (W - 1):
        raise RuntimeError("ngp_pl_b200.mesh.bake_texture: size must be a power of two in %d..%d, got %r"
                           % (_lib.NGP_TEXTURE_MIN_SIZE, _lib.NGP_TEXTURE_MAX_SIZE, size))
    if isinstance(samples, bool) or not isinstance(samples, (int, np.integer)) or not (
            1 <= samples <= _lib.NGP_TEXTURE_MAX_SAMPLES):
        raise RuntimeError("ngp_pl_b200.mesh.bake_texture: samples must be an integer in 1..%d, got %r"
                           % (_lib.NGP_TEXTURE_MAX_SAMPLES, samples))
    r = float(offset)
    if not (r >= 0 and np.isfinite(r)):
        raise RuntimeError("ngp_pl_b200.mesh.bake_texture: offset must be >= 0 and finite, got %r" % (offset,))
    dev = verts.device
    verts = verts.detach().to(torch.float32).reshape(-1, 3).contiguous()
    tris = tris.detach().to(torch.int64).reshape(-1, 3).contiguous()
    V, F = verts.shape[0], tris.shape[0]
    if nrm is not None:
        nrm = nrm.detach().to(torch.float32).reshape(-1, 3).contiguous()
        if nrm.shape[0] != V:
            raise RuntimeError("ngp_pl_b200.mesh.bake_texture: %d normals for %d vertices" % (nrm.shape[0], V))
    W = int(W)
    if F * _lib.NGP_TEXTURE_MIN_SQUARE ** 2 > W * W:
        raise RuntimeError("ngp_pl_b200.mesh.bake_texture: %d triangles need an atlas of size >= %d (%d squares of %d^2 "
                           "texels), got %d" % (F, texture_size_for(F), F, _lib.NGP_TEXTURE_MIN_SQUARE, W))
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_mesh_texture_workspace(V, F, W)
        if ws_bytes == 0:
            raise RuntimeError("ngp_pl_b200.mesh.bake_texture: %d vertices and %d triangles: both must be below 2^31"
                               % (V, F))
        _need(dev, ws_bytes + F * 36 + W * W * 3, "the atlas of %d triangles at size %d" % (F, W), "bake_texture")
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        uv = torch.empty(F, 3, 2, device=dev, dtype=torch.float32)
        squares = torch.empty(F, 3, device=dev, dtype=torch.int32)
        st = _st(dev)
        cnt = (C.c_int64 * 2)()
        _lib.check(L.ngp_mesh_texture_atlas(verts.data_ptr(), V, tris.data_ptr(), F, W, uv.data_ptr(), squares.data_ptr(),
                                            cnt, ws.data_ptr(), ws_bytes, st), "ngp_mesh_texture_atlas")
        n = int(cnt[1])
        bake_bytes = L.ngp_mesh_texture_bake_workspace(int(samples))
        _need(dev, n * 36 + W * W * 3 + bake_bytes, "%d band texels" % n, "bake_texture")
        texel = torch.empty(n, device=dev, dtype=torch.int64)
        tri = torch.empty(n, device=dev, dtype=torch.int32)
        point = torch.empty(n, 3, device=dev, dtype=torch.float32)
        normal = torch.empty(n, 3, device=dev, dtype=torch.float32)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        _lib.check(L.ngp_mesh_texture_texels(verts.data_ptr(), ptr(nrm), V, tris.data_ptr(), F, W, uv.data_ptr(), n,
                                             ptr(texel), ptr(tri), ptr(point), ptr(normal), ws.data_ptr(), ws_bytes, st),
                   "ngp_mesh_texture_texels")
        del ws
        texture = torch.empty(W, W, 3, device=dev, dtype=torch.uint8)
        bws = torch.empty(bake_bytes, device=dev, dtype=torch.uint8)
        net, keep = _net_struct(model)
        _lib.check(L.ngp_mesh_texture_bake(C.byref(net), W, n, ptr(texel), ptr(point), ptr(normal), r, int(samples),
                                           texture.data_ptr(), bws.data_ptr(), bake_bytes, st), "ngp_mesh_texture_bake")
        del bws
    out = {"uv": uv, "squares": squares, "texture": texture}
    if return_texels:
        out.update(texel=texel, triangle=tri, point=point, normal=normal)
    return out


def _np(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _lines(fmt, a, chunk=1 << 18):
    """fmt % row for every row of the 2-D array a, joined: one C-level format per chunk of rows, no per-line loop"""
    parts = []
    for i in range(0, a.shape[0], chunk):
        b = a[i:i + chunk]
        parts.append((fmt * b.shape[0]) % tuple(b.ravel().tolist()))
    return "".join(parts)


def write_obj(path, vertices, triangles, normals=None, uv=None, texture=None, png_mode="dynamic"):
    """Wavefront OBJ: `v` per vertex (%.9g: fp32 round-trips), `vn` per vertex normal, with uv ((F, 3, 2) texel
    coordinates as bake_texture returns them) 3F `vt` lines (uv / size, one per face corner, in face order), and faces
    `f v/vt/vn` (1-based; v//vn, v/vt or v as the attributes present allow). size is texture's side, or the smallest
    power of two >= 16 that holds the uv when no texture is given. With a texture ((W, W, 3) uint8, a device tensor) it
    also writes <stem>.mtl, whose material maps <stem>.png, and that PNG, encoded on the device by images.encode_png
    (png_mode "fixed" or "dynamic")."""
    import os
    v = _np(vertices).astype(np.float32).reshape(-1, 3)
    f = _np(triangles).astype(np.int64).reshape(-1, 3)
    F = f.shape[0]
    stem = os.path.splitext(path)[0]
    base = os.path.basename(stem)
    head = "# ngp_pl_b200 mesh: %d vertices, %d triangles\n" % (v.shape[0], F)
    png = None
    if texture is not None:
        from . import images
        if not (isinstance(texture, torch.Tensor) and texture.dim() == 3 and texture.shape[0] == texture.shape[1]
                and texture.shape[2] == 3 and texture.dtype == torch.uint8):
            raise RuntimeError("ngp_pl_b200.mesh.write_obj: texture must be a (W, W, 3) uint8 tensor")
        if uv is None:
            raise RuntimeError("ngp_pl_b200.mesh.write_obj: a texture needs uv")
        png = images.encode_png(texture.contiguous(), mode=png_mode)
        head += "mtllib %s.mtl\nusemtl material0\n" % base
    text = [head, _lines("v %.9g %.9g %.9g\n", v)]
    if normals is not None:
        text.append(_lines("vn %.9g %.9g %.9g\n", _np(normals).astype(np.float32).reshape(-1, 3)))
    fi = f + 1
    if uv is not None:
        u = _np(uv).astype(np.float32).reshape(F * 3, 2)
        W = texture.shape[0] if texture is not None else 16
        while texture is None and W < u.max(initial=0):
            W *= 2
        text.append(_lines("vt %.9g %.9g\n", u / np.float32(W)))
        vt = np.arange(1, 3 * F + 1, dtype=np.int64).reshape(F, 3)
        if normals is not None:
            text.append(_lines("f %d/%d/%d %d/%d/%d %d/%d/%d\n", np.stack([fi, vt, fi], 2).reshape(F, 9)))
        else:
            text.append(_lines("f %d/%d %d/%d %d/%d\n", np.stack([fi, vt], 2).reshape(F, 6)))
    elif normals is not None:
        text.append(_lines("f %d//%d %d//%d %d//%d\n", np.stack([fi, fi], 2).reshape(F, 6)))
    else:
        text.append(_lines("f %d %d %d\n", fi))
    with open(path, "w", newline="\n") as fh:
        fh.write("".join(text))
    if png is not None:
        with open(stem + ".mtl", "w", newline="\n") as fh:
            fh.write("newmtl material0\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\nmap_Kd %s.png\n" % base)
        with open(stem + ".png", "wb") as fh:
            fh.write(png)


def write_ply(path, vertices, triangles, normals=None, colors=None):
    """Binary little-endian PLY: float x, y, z [, nx, ny, nz] [, uchar red, green, blue] per vertex, and faces as a
    uchar count + int32 indices. Takes tensors (any device) or numpy arrays. Raises if V >= 2^31 (int32 indices)."""
    v = _np(vertices).astype("<f4").reshape(-1, 3)
    f = _np(triangles).reshape(-1, 3)
    if v.shape[0] >= 2 ** 31:
        raise RuntimeError("ngp_pl_b200.mesh.write_ply: %d vertices do not fit PLY's int32 face indices" % v.shape[0])
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    props = ["property float x", "property float y", "property float z"]
    if normals is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        props += ["property float nx", "property float ny", "property float nz"]
    if colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        props += ["property uchar red", "property uchar green", "property uchar blue"]
    rec = np.empty(v.shape[0], dtype=fields)
    rec["x"], rec["y"], rec["z"] = v[:, 0], v[:, 1], v[:, 2]
    if normals is not None:
        n = _np(normals).astype("<f4").reshape(-1, 3)
        rec["nx"], rec["ny"], rec["nz"] = n[:, 0], n[:, 1], n[:, 2]
    if colors is not None:
        c = _np(colors).astype(np.uint8).reshape(-1, 3)
        rec["red"], rec["green"], rec["blue"] = c[:, 0], c[:, 1], c[:, 2]
    face = np.empty(f.shape[0], dtype=[("n", "u1"), ("v", "<i4", (3,))])
    face["n"] = 3
    face["v"] = f.astype("<i4")
    header = "\n".join(["ply", "format binary_little_endian 1.0", "element vertex %d" % v.shape[0]] + props +
                       ["element face %d" % f.shape[0], "property list uchar int vertex_indices", "end_header"]) + "\n"
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(rec.tobytes())
        fh.write(face.tobytes())
