"""Gaussian-splat export from a trained model on the device: a 3DGS point_cloud.ply of the point-cloud export's
points, with SH colours fitted to the model's radiance, and a forward splat rasteriser to look at it.

    fibonacci_directions(n)                                 the direction set (n, 3) float32 (host, double, rounded)
    sh_basis(dirs)                                          3DGS's real SH basis (n, 16) float64 at the directions (host)
    colors_over_directions(model, points, dirs)             stage 1: sigma (P,) fp32, rgb (P, D, 3) fp16
    fit_sh(rgb, dirs, normals, splats, degree=3, ridge=1e-3)   stage 2: f_dc / f_rest of splats
    splat_geometry(points, normals, sigma, dist2, splats, shape="disc", flatness=0.1)   stage 3: every other field
    extract_splats(model, poses, directions, ...)           points stages 1-7, then stages 1-3: splats (P, 62) fp32
    write_splats(path, splats) / read_splats(path, device)  the 3DGS binary PLY
    SplatRenderer(splats, img_wh) / render(splats, pose, K, img_wh, bg)   the rasteriser: rgb (H W, 3), opacity (H W)

A splat set is one (P, 62) float32 CUDA tensor whose columns are ATTRIBUTES, the 3DGS file's vertex properties in
order: x y z nx ny nz f_dc_0..2 f_rest_0..44 opacity scale_0..2 rot_0..3. Positions, normals and directions are in the
model's frame, as the mesh and point exports write them; there is no transform back to a COLMAP frame. The rules are in
include/ngp_b200.h ("Gaussian-splat export") and csrc/splats.cu implements them; oracle/splats_ref.py restates them in
numpy. Every stage is deterministic: two calls are bitwise equal. Tensors must live on a CUDA device, otherwise
RuntimeError; there is no CPU path.
"""
import ctypes as C
import gc
import math

import numpy as np
import torch

from . import _lib, points as _points
from .mesh import _chk, _need, _st
from .models.networks import _net_struct

ATTRIBUTES = (["x", "y", "z", "nx", "ny", "nz"] + ["f_dc_%d" % i for i in range(3)] + ["f_rest_%d" % i for i in range(45)] +
              ["opacity"] + ["scale_%d" % i for i in range(3)] + ["rot_%d" % i for i in range(4)])
SHAPES = {"sphere": _lib.NGP_SPLAT_SPHERE, "disc": _lib.NGP_SPLAT_DISC}
CHUNK = 1 << 18          # points per colour evaluation: rgb (CHUNK, D, 3) fp16 is 192 MB at D = 128
C0, C1 = 0.28209479177387814, 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)


def fibonacci_directions(n):
    """(n, 3) float32 unit directions: z_j = 1 - (2j + 1) / n, phi_j = j pi (3 - sqrt 5), computed in double"""
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not (
            _lib.NGP_SPLAT_MIN_DIRS <= n <= _lib.NGP_SPLAT_MAX_DIRS):
        raise RuntimeError("ngp_pl_b200.splats: the number of directions must be an integer in %d..%d, got %r"
                           % (_lib.NGP_SPLAT_MIN_DIRS, _lib.NGP_SPLAT_MAX_DIRS, n))
    j = np.arange(n, dtype=np.float64)
    z = 1.0 - (2.0 * j + 1.0) / n
    phi = j * (math.pi * (3.0 - math.sqrt(5.0)))
    r = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(np.float32)


def sh_basis(dirs):
    """(n, 16) float64: 3DGS's SH basis (sh_utils.py's order and signs) at dirs (n, 3), taken as they are"""
    d = np.asarray(dirs, np.float64).reshape(-1, 3)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    return np.stack([
        np.full_like(x, C0), -C1 * y, C1 * z, -C1 * x,
        C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy),
        C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
        C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy)], 1)


def _dirs_tensor(dirs, dev, fn):
    d = torch.as_tensor(dirs, dtype=torch.float32).to(dev).reshape(-1, 3).contiguous()
    if not _lib.NGP_SPLAT_MIN_DIRS <= d.shape[0] <= _lib.NGP_SPLAT_MAX_DIRS:
        raise RuntimeError("ngp_pl_b200.splats.%s: %d directions: must be %d..%d" % (
            fn, d.shape[0], _lib.NGP_SPLAT_MIN_DIRS, _lib.NGP_SPLAT_MAX_DIRS))
    return d


@torch.no_grad()
def colors_over_directions(model, points, dirs):
    """Stage 1: sigma (P,) float32 and rgb (P, D, 3) float16 of the model at every (point, direction) pair; rgb[i, j] is
    bitwise NGP.forward(points[i], dirs[j])'s colour (its fp16 value) and sigma its density."""
    _chk(points, "colors_over_directions")
    dev = points.device
    p = points.detach().float().reshape(-1, 3).contiguous()
    d = _dirs_tensor(dirs, dev, "colors_over_directions")
    n, D = p.shape[0], d.shape[0]
    with torch.cuda.device(dev):
        _need(dev, n * (4 + 32 + 6 * D), "the colours of %d points over %d directions" % (n, D), "colors_over_directions")
        sigma = torch.empty(n, device=dev, dtype=torch.float32)
        h = torch.empty(n, 16, device=dev, dtype=torch.float16)
        rgb = torch.empty(n, D, 3, device=dev, dtype=torch.float16)
        net, keep = _net_struct(model)
        _lib.check(_lib.lib().ngp_splat_colors(C.byref(net), p.data_ptr(), n, d.data_ptr(), D, sigma.data_ptr(),
                                               h.data_ptr(), rgb.data_ptr(), _st(dev)), "ngp_splat_colors")
        del h
    return sigma, rgb


def _degree(sh_degree):
    if isinstance(sh_degree, bool) or not isinstance(sh_degree, (int, np.integer)) or not 0 <= sh_degree <= 3:
        raise RuntimeError("ngp_pl_b200.splats: sh_degree must be an integer in 0..3, got %r" % (sh_degree,))
    return int(sh_degree)


def _check_splats(splats, fn):
    _chk(splats, fn)
    if splats.dim() != 2 or splats.shape[1] != _lib.NGP_SPLAT_FLOATS or splats.dtype != torch.float32 or \
            not splats.is_contiguous():
        raise RuntimeError("ngp_pl_b200.splats.%s: expected a contiguous (P, %d) float32 splat tensor"
                           % (fn, _lib.NGP_SPLAT_FLOATS))
    return splats.shape[0]


@torch.no_grad()
def fit_sh(rgb, dirs, normals, splats, degree=3, ridge=1e-3):
    """Stage 2 into splats (P, 62): f_dc and f_rest from rgb (P, D, 3) fp16 as colors_over_directions returns it, the
    fit weighted by the hemisphere the normal faces (normals (P, 3) or None: every direction weighs 1)."""
    n = _check_splats(splats, "fit_sh")
    degree = _degree(degree)
    if not (ridge >= 0 and math.isfinite(ridge)):
        raise RuntimeError("ngp_pl_b200.splats.fit_sh: ridge must be >= 0 and finite, got %r" % (ridge,))
    dev = splats.device
    d = _dirs_tensor(dirs, dev, "fit_sh")
    if rgb.shape != (n, d.shape[0], 3) or rgb.dtype != torch.float16 or rgb.device != dev:
        raise RuntimeError("ngp_pl_b200.splats.fit_sh: rgb must be (%d, %d, 3) float16 on %s" % (n, d.shape[0], dev))
    if normals is not None and (normals.shape != (n, 3) or normals.dtype != torch.float32 or normals.device != dev):
        raise RuntimeError("ngp_pl_b200.splats.fit_sh: normals must be (%d, 3) float32 on %s" % (n, dev))
    basis = torch.as_tensor(sh_basis(d.cpu().numpy())).to(dev)
    rgb = rgb.contiguous()
    nrm = None if normals is None else normals.contiguous()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ngp_splat_fit(rgb.data_ptr(), n, d.shape[0], d.data_ptr(), basis.data_ptr(),
                                            None if nrm is None else nrm.data_ptr(), degree, float(ridge),
                                            splats.data_ptr(), _st(dev)), "ngp_splat_fit")
    return splats


@torch.no_grad()
def splat_geometry(points, normals, sigma, dist2, splats, shape="disc", flatness=0.1):
    """Stage 3 into splats: positions, normals, opacity, scales and rotations; dist2 (P, k) float64 from points.knn"""
    n = _check_splats(splats, "splat_geometry")
    if shape not in SHAPES:
        raise RuntimeError("ngp_pl_b200.splats.splat_geometry: shape must be 'disc' or 'sphere', got %r" % (shape,))
    if not (flatness > 0 and math.isfinite(flatness)):
        raise RuntimeError("ngp_pl_b200.splats.splat_geometry: flatness must be positive and finite, got %r" % (flatness,))
    dev = splats.device
    p, s = points.contiguous(), sigma.contiguous()
    d2 = dist2.contiguous()
    if p.shape != (n, 3) or s.shape != (n,) or d2.dim() != 2 or d2.shape[0] != n or d2.dtype != torch.float64:
        raise RuntimeError("ngp_pl_b200.splats.splat_geometry: expected points (%d, 3), sigma (%d,) and dist2 (%d, k) "
                           "float64" % (n, n, n))
    nrm = None if normals is None else normals.contiguous()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ngp_splat_geometry(p.data_ptr(), None if nrm is None else nrm.data_ptr(), s.data_ptr(),
                                                 d2.data_ptr() if d2.numel() else None, d2.shape[1], n, SHAPES[shape],
                                                 float(flatness), splats.data_ptr(), _st(dev)), "ngp_splat_geometry")
    return splats


@torch.no_grad()
def extract_splats(model, poses, directions, num_rays=1000000, min_opacity=0.5, bounds=None, voxel=None, nb_neighbors=20,
                   std_ratio=2.0, keep_outliers=False, normals=True, sh_degree=3, n_directions=128, shape="disc",
                   flatness=0.1, ridge=1e-3, chunk=CHUNK, timings=None):
    """The point-cloud export's stages as export_points runs them (extract_points, voxel_downsample if voxel,
    remove_outliers unless keep_outliers, estimate_normals if normals), then stages 1-3 over n_directions Fibonacci
    directions: a (P, 62) float32 splat tensor in point order. Colours are evaluated `chunk` points at a time. timings
    (a dict) gets the CUDA-event milliseconds of 'points', 'colors', 'fit' and 'geometry'."""
    _degree(sh_degree)
    if isinstance(chunk, bool) or not isinstance(chunk, (int, np.integer)) or chunk < 1:
        raise RuntimeError("ngp_pl_b200.splats.extract_splats: chunk must be a positive integer, got %r" % (chunk,))
    dirs_np = fibonacci_directions(n_directions)
    dev = model.xyz_encoder.params.device
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)] if timings is not None else None
    acc = {"colors": 0.0, "fit": 0.0}
    if ev:
        ev[0].record()
    pts = _points.extract_points(model, poses, directions, num_rays, min_opacity, bounds)
    if voxel is not None:
        pts = _points.voxel_downsample(pts, voxel)
    if not keep_outliers:
        pts = _points.remove_outliers(pts, nb_neighbors, std_ratio)
    if normals:
        pts = _points.estimate_normals(pts, nb_neighbors)
    if ev:
        ev[1].record()
    P = pts["points"].shape[0]
    dirs = torch.as_tensor(dirs_np).to(dev)
    with torch.cuda.device(dev):
        splats = torch.zeros(P, _lib.NGP_SPLAT_FLOATS, device=dev, dtype=torch.float32)
        sigma = torch.empty(P, device=dev, dtype=torch.float32)
        nrm = pts["normals"]
        for k0 in range(0, P, chunk):
            k1 = min(P, k0 + chunk)
            if ev:
                ev[2].record()
            sig, rgb = colors_over_directions(model, pts["points"][k0:k1], dirs)
            sigma[k0:k1] = sig
            if ev:
                ev[3].record()
            fit_sh(rgb, dirs, None if nrm is None else nrm[k0:k1], splats[k0:k1], sh_degree, ridge)
            if ev:
                ev[4].record()
                ev[4].synchronize()
                acc["colors"] += ev[2].elapsed_time(ev[3])
                acc["fit"] += ev[3].elapsed_time(ev[4])
            del rgb
        g0 = torch.cuda.Event(enable_timing=True) if ev else None
        if g0:
            g0.record()
        _, d2 = _points.knn(pts["points"], 3) if P > 1 else (None, torch.empty(P, 0, device=dev, dtype=torch.float64))
        splat_geometry(pts["points"], nrm, sigma, d2, splats, shape, flatness)
        if ev:
            ev[0].synchronize()
            g1 = torch.cuda.Event(enable_timing=True)
            g1.record()
            g1.synchronize()
            timings["points"] = timings.get("points", 0.0) + ev[0].elapsed_time(ev[1])
            timings["colors"] = timings.get("colors", 0.0) + acc["colors"]
            timings["fit"] = timings.get("fit", 0.0) + acc["fit"]
            timings["geometry"] = timings.get("geometry", 0.0) + g0.elapsed_time(g1)
    return splats


def ply_header(n):
    """the 3DGS point_cloud.ply header for n vertices, as bytes"""
    return ("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n +
            "".join("property float %s\n" % a for a in ATTRIBUTES) + "end_header\n").encode("ascii")


def write_splats(path, splats):
    """the 3DGS binary PLY: one device-to-host copy of the packed (P, 62) tensor, then the header and the rows"""
    _check_splats(splats, "write_splats")
    host = splats.detach().cpu().numpy().astype("<f4", copy=False)
    with open(path, "wb") as f:
        f.write(ply_header(host.shape[0]))
        f.write(host.tobytes())


def read_splats(path, device="cuda"):
    """a file with the 3DGS layout (binary little-endian, one vertex element of 62 float properties in ATTRIBUTES
    order, any other elements after it ignored) -> (P, 62) float32 on device. ValueError for any other layout."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.find(b"end_header\n")
    if not data.startswith(b"ply\n") or end < 0:
        raise ValueError("ngp_pl_b200.splats.read_splats: %s is not a PLY file" % path)
    lines = [ln.strip() for ln in data[:end].decode("ascii", "replace").split("\n")[1:] if ln.strip()]
    lines = [ln for ln in lines if not ln.startswith(("comment", "obj_info"))]
    if not lines or lines[0] != "format binary_little_endian 1.0":
        raise ValueError("ngp_pl_b200.splats.read_splats: %s: only binary_little_endian 1.0 is read" % path)
    if len(lines) < 2 or not lines[1].startswith("element vertex "):
        raise ValueError("ngp_pl_b200.splats.read_splats: %s: the first element must be 'vertex'" % path)
    n = int(lines[1].split()[2])
    props = []
    for ln in lines[2:]:
        if ln.startswith("element"):
            break
        props.append(ln)
    if props != ["property float %s" % a for a in ATTRIBUTES]:
        raise ValueError("ngp_pl_b200.splats.read_splats: %s: the vertex properties are not the 3DGS layout (62 floats "
                         "x .. rot_3)" % path)
    body = end + len(b"end_header\n")
    if len(data) < body + 4 * 62 * n:
        raise ValueError("ngp_pl_b200.splats.read_splats: %s is truncated" % path)
    host = np.frombuffer(data, dtype="<f4", count=62 * n, offset=body).reshape(n, 62)
    return torch.from_numpy(host.astype(np.float32)).to(device)


def _view(pose, K, bg):
    pose = np.asarray(torch.as_tensor(pose, dtype=torch.float32).cpu(), np.float32).reshape(12)
    K = np.asarray(torch.as_tensor(K, dtype=torch.float32).cpu(), np.float32).reshape(3, 3)
    bg = np.broadcast_to(np.asarray(bg, np.float32).reshape(-1), (3,))
    v = np.concatenate([pose, [K[0, 0], K[1, 1], K[0, 2], K[1, 2]], bg]).astype(np.float32)
    if not np.isfinite(v).all() or not (v[12] > 0 and v[13] > 0):
        raise RuntimeError("ngp_pl_b200.splats.render: the pose, K and bg must be finite, with fx, fy > 0")
    return torch.from_numpy(v)


class SplatRenderer:
    """The rasteriser for one splat set and one view size: one CUDA graph, replayed for every view (the view goes to a
    device buffer the graph reads). When a view needs more (tile, splat) keys than the graph sorts, the graph is
    captured again with 1.5 times that many and the view rendered again."""

    def __init__(self, splats, img_wh, capacity=None):
        self.n = _check_splats(splats, "SplatRenderer")
        self.splats = splats
        self.W, self.H = int(img_wh[0]), int(img_wh[1])
        if not (1 <= self.W <= _lib.NGP_SPLAT_MAX_SIDE and 1 <= self.H <= _lib.NGP_SPLAT_MAX_SIDE):
            raise RuntimeError("ngp_pl_b200.splats.SplatRenderer: img_wh must be 1..%d per side, got %r"
                               % (_lib.NGP_SPLAT_MAX_SIDE, img_wh))
        self.dev = splats.device
        self.view = torch.zeros(_lib.NGP_SPLAT_VIEW_FLOATS, device=self.dev)
        self.rgb = torch.empty(self.H * self.W, 3, device=self.dev)
        self.opacity = torch.empty(self.H * self.W, device=self.dev)
        self.n_keys = torch.zeros(1, device=self.dev, dtype=torch.int64)
        self.graph = None
        self._setup(capacity if capacity is not None else max(4 * self.n, 1 << 16))

    def _setup(self, capacity):
        capacity = int(min(max(capacity, 1), (1 << 31) - 1))
        self.graph = None
        nbytes = _lib.lib().ngp_splat_render_workspace(self.n, self.W, self.H, capacity)
        if nbytes == 0:
            raise RuntimeError("ngp_pl_b200.splats.SplatRenderer: %d splats at %dx%d with %d keys is out of range"
                               % (self.n, self.W, self.H, capacity))
        self.ws = None
        _need(self.dev, nbytes, "the rasteriser's workspace", "SplatRenderer")
        self.ws = torch.empty(nbytes, device=self.dev, dtype=torch.uint8)
        self.capacity = capacity
        with torch.cuda.device(self.dev):
            self._launch(_st(self.dev))  # eager once: cub's first call and module loading stay out of the capture
            g = torch.cuda.CUDAGraph()
            gc_was_enabled = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.graph(g):
                    self._launch(_st(self.dev))
            finally:
                if gc_was_enabled:
                    gc.enable()
        self.graph = g

    def _launch(self, st):
        _lib.check(_lib.lib().ngp_splat_render(self.splats.data_ptr() if self.n else None, self.n, self.view.data_ptr(),
                                               self.W, self.H, self.capacity, self.rgb.data_ptr(),
                                               self.opacity.data_ptr(), self.n_keys.data_ptr(), self.ws.data_ptr(),
                                               self.ws.numel(), st), "ngp_splat_render")

    @torch.no_grad()
    def render(self, pose, K, bg=(0.0, 0.0, 0.0)):
        """pose (3, 4) c2w (OpenCV axes), K (3, 3) -> rgb (H W, 3), opacity (H W) float32 (copies)"""
        self.view.copy_(_view(pose, K, bg))
        with torch.cuda.device(self.dev):
            self.graph.replay()
            need = int(self.n_keys.item())
            if need > self.capacity:
                self._setup(need + need // 2)
                self.graph.replay()
        return self.rgb.clone(), self.opacity.clone()


def render(splats, pose, K, img_wh, bg=(0.0, 0.0, 0.0)):
    """one view through a fresh SplatRenderer: rgb (H W, 3), opacity (H W). Render many views through one
    SplatRenderer, which keeps its graph."""
    return SplatRenderer(splats, img_wh).render(pose, K, bg)


@torch.no_grad()
def preview(model, splats, poses, K, img_wh, directions, save_dir=None, exp_step_factor=None):
    """Each view of poses through the rasteriser and through the model (render(test_time=True), with the same
    background, which render() picks from exp_step_factor: white when it is 0); per-view PSNR of the splat image against
    the model's, as a list of floats. save_dir: `{i:03d}.png` = the splat image and `{i:03d}_model.png` = the model's,
    (rgb * 255).astype(uint8), PNG-encoded on the device."""
    import os
    from . import images, metrics
    from .models.rendering import default_exp_step_factor, render as render_model
    if exp_step_factor is None:
        exp_step_factor = default_exp_step_factor(model)
    bg = 1.0 if exp_step_factor == 0 else 0.0
    W, H = int(img_wh[0]), int(img_wh[1])
    dev = splats.device
    poses = torch.as_tensor(poses, dtype=torch.float32).to(dev).reshape(-1, 3, 4)
    directions = torch.as_tensor(directions, dtype=torch.float32).to(dev).reshape(-1, 3)
    if directions.shape[0] != W * H:
        raise RuntimeError("ngp_pl_b200.splats.preview: %d directions for a %dx%d view" % (directions.shape[0], W, H))
    if save_dir is not None:
        os.makedirs(save_dir, exist_ok=True)
    rr = SplatRenderer(splats, (W, H))
    out = []
    for i in range(poses.shape[0]):
        rgb, _ = rr.render(poses[i], K, (bg, bg, bg))
        d = directions @ poses[i, :, :3].T
        o = poses[i, :, 3].expand_as(d).contiguous()
        ref = render_model(model, o, d.contiguous(), test_time=True, exp_step_factor=exp_step_factor)["rgb"]
        out.append(float(metrics.psnr(rgb, ref)))
        if save_dir is not None:
            images.write_png(os.path.join(save_dir, "%03d.png" % i), images.rgb_image(rgb, H, W))
            images.write_png(os.path.join(save_dir, "%03d_model.png" % i), images.rgb_image(ref, H, W))
    return out
