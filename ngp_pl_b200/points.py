"""Point-cloud export from a trained model on the device: the training views' rendered depth back-projected to
coloured points, then optional voxel downsampling, statistical outlier removal and normals.

    golden_step(N)                                          the ray-selection step g of N global pixels (host)
    extract_points(model, poses, directions, num_rays=1000000, min_opacity=0.5, bounds=None, exp_step_factor=None,
                   chunk=CHUNK, return_rays=False, timings=None)    stages 1-3: rays, render, back-projection
    voxel_downsample(pts, grid, bounds=None, return_cells=False)   stage 4: one point per occupied cluster-grid cell
    knn(points, k)                                          stage 5: exact k nearest neighbours, (idx, dist2)
    remove_outliers(pts, nb_neighbors=20, std_ratio=2.0, return_stats=False)   stage 6 (Open3D's rule)
    estimate_normals(pts, nb_neighbors=20)                  stage 7: PCA normals facing the cameras

A point dict is {'points' (n, 3) float32, 'colors' (n, 3) uint8, 'view' (n, 3) float32 (the unit direction of the ray
that found the point), 'normals' (n, 3) float32 or None} on the model's device; `mesh.write_ply(path,
pts['points'], empty triangles, pts['normals'], pts['colors'])` saves it. The rules are in include/ngp_b200.h
("Point-cloud export") and csrc/points.cu implements them; oracle/points_ref.py restates them in numpy. Every stage is
deterministic: two calls are bitwise equal. Tensors must live on a CUDA device, otherwise RuntimeError; there is no CPU
path.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .mesh import _chk, _need, _np, _st, _three, cluster_grid
from .models.networks import _net_struct
from .models.rendering import default_exp_step_factor, infer_cfg

CHUNK = 1 << 18          # rays per render: the wavefront's buffers and its cached graph are reused from chunk to chunk
MAX_RAYS = 1 << 28
GOLDEN = 6180339887      # round(0.6180339887 N) = floor((GOLDEN N + 5 10^9) / 10^10)


def golden_step(N):
    """the smallest integer g >= round(0.6180339887 N) (half up, exact integers) with gcd(g, N) = 1: ray k takes the
    global pixel (k g) mod N, a bijection of 0..N-1 that spreads the first rays evenly over views and rows"""
    N = int(N)
    if N < 1:
        raise RuntimeError("ngp_pl_b200.points.golden_step: N must be >= 1, got %d" % N)
    g = max(1, (GOLDEN * N + 5 * 10 ** 9) // 10 ** 10)
    while math.gcd(g, N) != 1:
        g += 1
    return g


def _empty(dev, n=0):
    return {"points": torch.empty(n, 3, device=dev, dtype=torch.float32),
            "colors": torch.empty(n, 3, device=dev, dtype=torch.uint8),
            "view": torch.empty(n, 3, device=dev, dtype=torch.float32), "normals": None}


def _ws(dev, n, what, fn):
    nbytes = _lib.lib().ngp_points_workspace(int(n))
    if nbytes == 0:
        raise RuntimeError("ngp_pl_b200.points.%s: %d %s: must be below 2^31" % (fn, n, what))
    _need(dev, nbytes, "the workspace of %d %s" % (n, what), fn)
    return torch.empty(nbytes, device=dev, dtype=torch.uint8)


def _check_pts(pts, fn):
    p, c, v = pts["points"], pts["colors"], pts["view"]
    for t in (p, c, v):
        _chk(t, fn)
    n = p.shape[0]
    if not (p.shape == (n, 3) and c.shape == (n, 3) and v.shape == (n, 3) and p.dtype == torch.float32 and
            c.dtype == torch.uint8 and v.dtype == torch.float32):
        raise RuntimeError("ngp_pl_b200.points.%s: expected points (n, 3) float32, colors (n, 3) uint8 and view (n, 3) "
                           "float32" % fn)
    return p.contiguous(), c.contiguous(), v.contiguous(), n


def _k(nb_neighbors, fn):
    if isinstance(nb_neighbors, bool) or not isinstance(nb_neighbors, (int, np.integer)) or not (
            1 <= nb_neighbors <= _lib.NGP_POINTS_MAX_K):
        raise RuntimeError("ngp_pl_b200.points.%s: nb_neighbors must be an integer in 1..%d, got %r"
                           % (fn, _lib.NGP_POINTS_MAX_K, nb_neighbors))
    return int(nb_neighbors)


def _render_chunks(model, cfg, poses, directions, step, n, maps, ev=None):
    """Renders rays 0 .. n - 1, cfg.n_rays at a time: ray k through the global pixel (k step) mod (views * pixels) of
    poses x directions (ngp_points_rays), then ngp_render_infer_frame into the (opacity, depth, rgb) tensors that
    maps(k0) returns for the chunk starting at ray k0. Yields (k0, m, idx, o, d) once a chunk's render is enqueued: its
    m rays' (view, pixel) ids, origins and directions, overwritten by the next chunk. ev: CUDA events recorded before
    the rays, before the render and after it."""
    dev, B, L = poses.device, cfg.n_rays, _lib.lib()
    ws = torch.empty(L.ngp_render_infer_workspace(B, cfg.max_round_samples), device=dev, dtype=torch.uint8)
    idx = torch.empty(2, B, device=dev, dtype=torch.int64)
    o, d = torch.empty(B, 3, device=dev), torch.empty(B, 3, device=dev)
    total = torch.zeros(1, device=dev, dtype=torch.int64)
    c, h = model.center.flatten().tolist(), model.half_size.flatten().tolist()
    net, keep = _net_struct(model)
    st = _st(dev)
    for k0 in range(0, n, B):
        m = min(B, n - k0)
        if ev:
            ev[0].record()
        _lib.check(L.ngp_points_rays(poses.shape[0], directions.shape[0], step, k0, m, poses.data_ptr(),
                                     directions.data_ptr(), idx[0].data_ptr(), idx[1].data_ptr(), o.data_ptr(), d.data_ptr(),
                                     st), "ngp_points_rays")
        if m < B:  # the last chunk's spare rays start behind the box and leave it: they never march
            o[m:] = torch.tensor([c[0], c[1], c[2] + 2 * h[2] + 1.0], device=dev)
            d[m:] = torch.tensor([0.0, 0.0, 1.0], device=dev)
        if ev:
            ev[1].record()
        opacity, depth, rgb = maps(k0)
        _lib.check(L.ngp_render_infer_frame(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(),
                                            model.density_bitfield.data_ptr(), opacity.data_ptr(), depth.data_ptr(),
                                            rgb.data_ptr(), total.data_ptr(), ws.data_ptr(), ws.numel(), st),
                   "ngp_render_infer_frame")
        if ev:
            ev[2].record()
        yield k0, m, idx, o, d


@torch.no_grad()
def extract_points(model, poses, directions, num_rays=1000000, min_opacity=0.5, bounds=None, exp_step_factor=None,
                   chunk=CHUNK, return_rays=False, timings=None):
    """Stages 1-3: R = min(num_rays, n_views * n_pix) rays through the pixels golden_step picks, rendered as
    render(model, o, d, test_time=True) renders them (T_threshold 1e-4, 1024 samples) but with a black background,
    and every ray with opacity >= min_opacity whose depth lands in the closed box `bounds` = (lo, hi) (default: the
    model's box [-scale, scale]^3) becomes a point: p = o + d depth / opacity, colour = the rendered colour over
    opacity (the background taken out), view = d / |d|. Points keep the rays' order.

    poses (n_views, 3, 4) and directions (n_pix, 3) as the training set has them (any device); exp_step_factor
    defaults to train.py's rule (1/256 for scale > 0.5, else 0). Rays are rendered `chunk` at a time from the same
    buffers, so the render's cached graph is replayed. The result is a fixed function of the model, the cameras,
    num_rays and chunk: the wavefront's per-round sample quota follows the number of rays alive in the batch, as the
    reference's test-time loop does, and with it the order of the compositing sums and the 1024-sample budget, so
    another chunk changes a ray's opacity and depth by rounding (a ray that hits the budget, by more).

    return_rays=True adds 'img_idx', 'pix_idx' (R,) int64, 'rays_o', 'rays_d' (R, 3), 'opacity', 'depth' (R,) and
    'rgb' (R, 3) of every ray. timings (a dict) gets the CUDA-event milliseconds of 'rays', 'render' and 'backproject'
    summed over the chunks. RuntimeError for CPU tensors, num_rays outside 1..2^28, min_opacity outside (0, 1], a box
    with lo > hi, or outputs that do not fit free device memory."""
    _chk(model.xyz_encoder.params, "extract_points")
    dev = model.xyz_encoder.params.device
    if isinstance(num_rays, bool) or not isinstance(num_rays, (int, np.integer)) or not 1 <= num_rays <= MAX_RAYS:
        raise RuntimeError("ngp_pl_b200.points.extract_points: num_rays must be an integer in 1..2^28, got %r" % (num_rays,))
    if not (0 < min_opacity <= 1):
        raise RuntimeError("ngp_pl_b200.points.extract_points: min_opacity must be in (0, 1], got %r" % (min_opacity,))
    if isinstance(chunk, bool) or not isinstance(chunk, (int, np.integer)) or not 1 <= chunk <= MAX_RAYS:
        raise RuntimeError("ngp_pl_b200.points.extract_points: chunk must be an integer in 1..2^28, got %r" % (chunk,))
    poses = torch.as_tensor(poses, dtype=torch.float32).to(dev).reshape(-1, 3, 4).contiguous()
    directions = torch.as_tensor(directions, dtype=torch.float32).to(dev).reshape(-1, 3).contiguous()
    n_views, n_pix = poses.shape[0], directions.shape[0]
    if n_views < 1 or n_pix < 1:
        raise RuntimeError("ngp_pl_b200.points.extract_points: no cameras (%d poses, %d directions)" % (n_views, n_pix))
    if bounds is None:
        lo, hi = model._xyz_min_host, model._xyz_max_host
    else:
        lo, hi = bounds
    lo, hi = _three(_np(lo), np.float32), _three(_np(hi), np.float32)
    if not (np.isfinite(lo).all() and np.isfinite(hi).all() and (lo <= hi).all()):
        raise RuntimeError("ngp_pl_b200.points.extract_points: bounds need lo <= hi on every axis, got %s .. %s" % (lo, hi))
    box = (C.c_float * 6)(*[float(x) for x in np.concatenate([lo, hi])])
    if exp_step_factor is None:
        exp_step_factor = default_exp_step_factor(model)
    N = n_views * n_pix
    R = min(int(num_rays), N)
    B = min(int(chunk), R)
    L = _lib.lib()
    cfg = infer_cfg(model, B, exp_step_factor, 0.0)
    with torch.cuda.device(dev):
        infer_bytes = L.ngp_render_infer_workspace(B, cfg.max_round_samples)
        pts_bytes = L.ngp_points_workspace(B)
        _need(dev, R * 27 + B * 72 + infer_bytes + pts_bytes + (R * 68 if return_rays else 0),
              "%d rays in chunks of %d" % (R, B), "extract_points")
        pws = _ws(dev, B, "rays", "extract_points")
        opacity, depth, rgb = torch.empty(B, device=dev), torch.empty(B, device=dev), torch.empty(B, 3, device=dev)
        out = _empty(dev, R)
        rays = None
        if return_rays:
            rays = {"img_idx": torch.empty(R, device=dev, dtype=torch.int64), "pix_idx": torch.empty(R, device=dev, dtype=torch.int64),
                    "rays_o": torch.empty(R, 3, device=dev), "rays_d": torch.empty(R, 3, device=dev),
                    "opacity": torch.empty(R, device=dev), "depth": torch.empty(R, device=dev),
                    "rgb": torch.empty(R, 3, device=dev)}
        st = _st(dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timings is not None else None
        acc = [0.0, 0.0, 0.0]
        n_out = 0
        cnt = C.c_int64()
        for k0, m, idx, o, d in _render_chunks(model, cfg, poses, directions, golden_step(N), R,
                                               lambda k0: (opacity, depth, rgb), ev):
            _lib.check(L.ngp_points_backproject(o.data_ptr(), d.data_ptr(), opacity.data_ptr(), depth.data_ptr(),
                                                rgb.data_ptr(), m, float(min_opacity), box,
                                                out["points"][n_out:].data_ptr(), out["colors"][n_out:].data_ptr(),
                                                out["view"][n_out:].data_ptr(), C.byref(cnt), pws.data_ptr(), pws.numel(),
                                                st), "ngp_points_backproject")
            if ev:
                ev[3].record()
                ev[3].synchronize()
                for s in range(3):
                    acc[s] += ev[s].elapsed_time(ev[s + 1])
            if rays is not None:
                rays["img_idx"][k0:k0 + m] = idx[0, :m]
                rays["pix_idx"][k0:k0 + m] = idx[1, :m]
                for key, t in (("rays_o", o), ("rays_d", d), ("opacity", opacity), ("depth", depth), ("rgb", rgb)):
                    rays[key][k0:k0 + m] = t[:m]
            n_out += cnt.value
        del pws
    if timings is not None:
        for s, name in enumerate(("rays", "render", "backproject")):
            timings[name] = timings.get(name, 0.0) + acc[s]
    res = {key: out[key][:n_out].clone() for key in ("points", "colors", "view")}
    res["normals"] = None
    if rays is not None:
        res.update(rays)
    return res


@torch.no_grad()
def voxel_downsample(pts, grid, bounds=None, return_cells=False):
    """Stage 4: one point per occupied cell of mesh.cluster_grid(lo, hi, grid) (cubes of side max(hi - lo) / grid, the
    simplification's cells and keys; points outside the box join the border cells), in ascending cell key: the double
    mean of the members' positions rounded to fp32, the rounded mean colour, the normalised sum of their views.
    bounds=None: the box of the points (one device min / max and its read-back). Normals are dropped (None).
    return_cells=True adds 'key' (m,) int64 cluster keys and 'count' (m,) int32 members."""
    p, c, v, n = _check_pts(pts, "voxel_downsample")
    if isinstance(grid, bool) or not isinstance(grid, (int, np.integer)) or not 1 <= grid <= _lib.NGP_SIMPLIFY_MAX_GRID:
        raise RuntimeError("ngp_pl_b200.points.voxel_downsample: grid must be an integer in 1..%d, got %r"
                           % (_lib.NGP_SIMPLIFY_MAX_GRID, grid))
    dev = p.device
    if bounds is None:
        if n == 0:
            lo, hi = np.zeros(3, np.float32), np.ones(3, np.float32)
        else:
            mn, mx = torch.aminmax(p, dim=0)
            lo, hi = mn.cpu().numpy(), mx.cpu().numpy()
            if not (hi - lo).max() > 0:
                hi = lo + np.float32(1)  # one point, or all alike: a single cell
    else:
        lo, hi = (_three(_np(b), np.float32) for b in bounds)
    if not (np.isfinite(lo).all() and np.isfinite(hi).all() and (lo < hi).all()):
        raise RuntimeError("ngp_pl_b200.points.voxel_downsample: bounds need lo < hi on every axis, got %s .. %s" % (lo, hi))
    g = cluster_grid(lo, hi, int(grid))
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws = _ws(dev, n, "points", "voxel_downsample")
        _need(dev, n * 39, "%d points" % n, "voxel_downsample")
        out = _empty(dev, n)
        key = torch.empty(n, device=dev, dtype=torch.int64)
        cnt = torch.empty(n, device=dev, dtype=torch.int32)
        m = C.c_int64()
        _lib.check(L.ngp_points_voxel(p.data_ptr(), c.data_ptr(), v.data_ptr(), n, C.byref(g), out["points"].data_ptr(),
                                      out["colors"].data_ptr(), out["view"].data_ptr(), key.data_ptr(), cnt.data_ptr(),
                                      C.byref(m), ws.data_ptr(), ws.numel(), _st(dev)), "ngp_points_voxel")
        del ws
    m = m.value
    res = {k: out[k][:m].clone() for k in ("points", "colors", "view")}
    res["normals"] = None
    if return_cells:
        res["key"], res["count"] = key[:m].clone(), cnt[:m].clone()
    return res


@torch.no_grad()
def knn(points, k):
    """Stage 5: for every point the k' = min(k, n - 1) nearest other points, exactly: idx (n, k') int32 and dist2
    (n, k') float64 squared distances (double, from the fp32 coordinates), ordered by distance and then index.
    k: 1..64. RuntimeError for a coordinate that is not finite."""
    _chk(points, "knn")
    k = _k(k, "knn")
    p = points.detach().to(torch.float32).reshape(-1, 3).contiguous()
    n, dev = p.shape[0], p.device
    kk = min(k, n - 1)
    if kk < 1:
        return (torch.empty(n, 0, device=dev, dtype=torch.int32), torch.empty(n, 0, device=dev, dtype=torch.float64))
    with torch.cuda.device(dev):
        ws = _ws(dev, n, "points", "knn")
        _need(dev, n * kk * 12, "the neighbour lists of %d points" % n, "knn")
        idx = torch.empty(n, kk, device=dev, dtype=torch.int32)
        d2 = torch.empty(n, kk, device=dev, dtype=torch.float64)
        _lib.check(_lib.lib().ngp_points_knn(p.data_ptr(), n, kk, idx.data_ptr(), d2.data_ptr(), ws.data_ptr(), ws.numel(),
                                             _st(dev)), "ngp_points_knn")
        del ws
    return idx, d2


@torch.no_grad()
def remove_outliers(pts, nb_neighbors=20, std_ratio=2.0, return_stats=False):
    """Stage 6, Open3D's remove_statistical_outlier: d_i = the mean distance of point i to its k' = min(nb_neighbors,
    n - 1) nearest neighbours; a point is kept iff d_i <= mean + std_ratio * std (population) of the d_i. Order is
    kept; normals are carried along. Fewer than 2 points are all kept. return_stats=True also returns {'mean', 'std',
    'threshold', 'kept' (m,) int64 input indices}."""
    p, c, v, n = _check_pts(pts, "remove_outliers")
    k = _k(nb_neighbors, "remove_outliers")
    if not (std_ratio >= 0 and math.isfinite(std_ratio)):
        raise RuntimeError("ngp_pl_b200.points.remove_outliers: std_ratio must be >= 0 and finite, got %r" % (std_ratio,))
    dev = p.device
    nrm = pts.get("normals")
    if n < 2:
        res = {"points": p.clone(), "colors": c.clone(), "view": v.clone(), "normals": None if nrm is None else nrm.clone()}
        kept = torch.arange(n, device=dev)
        stats = {"mean": 0.0, "std": 0.0, "threshold": 0.0}
    else:
        idx, d2 = knn(p, k)
        del idx
        with torch.cuda.device(dev):
            ws = _ws(dev, n, "points", "remove_outliers")
            _need(dev, n * 31, "%d points" % n, "remove_outliers")
            out = _empty(dev, n)
            kept = torch.empty(n, device=dev, dtype=torch.int32)
            s = (C.c_double * 3)()
            m = C.c_int64()
            _lib.check(_lib.lib().ngp_points_outliers(p.data_ptr(), c.data_ptr(), v.data_ptr(), n, d2.shape[1], d2.data_ptr(),
                                                      float(std_ratio), out["points"].data_ptr(), out["colors"].data_ptr(),
                                                      out["view"].data_ptr(), kept.data_ptr(), s, C.byref(m), ws.data_ptr(),
                                                      ws.numel(), _st(dev)), "ngp_points_outliers")
            del ws, d2
        m = m.value
        kept = kept[:m].long()
        res = {key: out[key][:m].clone() for key in ("points", "colors", "view")}
        res["normals"] = None if nrm is None else nrm[kept]
        stats = {"mean": s[0], "std": s[1], "threshold": s[2]}
    if return_stats:
        stats["kept"] = kept
        return res, stats
    return res


@torch.no_grad()
def estimate_normals(pts, nb_neighbors=20):
    """Stage 7: a copy of the point dict with 'normals': per point, the smallest-eigenvalue eigenvector of the
    covariance of the point and its k' = min(nb_neighbors, n - 1) nearest neighbours (double, cyclic Jacobi), turned to
    face the camera that saw the point (n . view <= 0); (0, 0, 0) where the covariance is 0."""
    p, c, v, n = _check_pts(pts, "estimate_normals")
    k = _k(nb_neighbors, "estimate_normals")
    dev = p.device
    idx, _ = knn(p, k)
    nrm = torch.empty(n, 3, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ngp_points_normals(p.data_ptr(), v.data_ptr(), n, idx.shape[1], idx.data_ptr() if idx.numel() else None,
                                                 nrm.data_ptr(), _st(dev)), "ngp_points_normals")
    return {"points": p, "colors": c, "view": v, "normals": nrm}
