"""Mesh extraction from a trained model on the device: the mesh cell of the reference's notebook (test.ipynb) without
PyMCubes, trimesh or scikit-image.

    density_volume(model, resolution, bounds=None)                σ on a lattice, (n0, n1, n2) fp32 on the device
    marching_cubes(volume, iso, lo=None, step=None, normals=False) indexed mesh of a σ volume, on the device
    extract_mesh(model, resolution=256, bounds=None, threshold=20.0, normals=True, colors=False)
    write_ply(path, vertices, triangles, normals=None, colors=None) binary little-endian PLY, numpy only

The σ lattice is evaluated by `ngp_density_lattice` (csrc/network.cu), which generates its points instead of reading
them, and the mesh by `ngp_marching_cubes_count` / `_emit` (csrc/mesh.cu), which work through the volume in slabs;
semantics in include/ngp_b200.h. The only host synchronisations are the read-back of the vertex and triangle counts
and emit's check of the capacities against them. Model and volume must live on a CUDA device, otherwise RuntimeError;
there is no CPU path.
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
    rgb = None
    if colors:
        d = -nrm
        flat = (nrm == 0).all(1)
        d[flat] = torch.tensor([0.0, 0.0, 1.0], device=d.device)
        rgb = torch.empty(0, 3, device=verts.device, dtype=torch.uint8)
        if verts.shape[0] > 0:
            _, c = model(verts, d)
            rgb = (c.float() * 255).round().clamp(0, 255).to(torch.uint8)
    return {"vertices": verts, "triangles": tris, "normals": nrm if normals else None, "colors": rgb}


def _np(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


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
