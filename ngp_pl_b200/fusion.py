"""Depth fusion on the device: the training views' rendered depth fused into a truncated signed distance field (TSDF),
and its mesh. A TSDF mesh holds only surfaces the cameras saw -- no cavity inside the solid that no ray reaches, as the
σ level set has -- and needs no σ threshold.

    render_views(model, poses, directions, chunk=points.CHUNK, exp_step_factor=None)
                                                    every pixel of every view: {'opacity', 'depth' (V, HW), 'rgb' (V, HW, 3)}
    tsdf_volume(resolution, bounds, trunc=None, device=None)    an empty TSDF state on a lattice
    integrate(vol, poses, K, img_wh, depth, opacity, rgb, min_opacity=0.5)      fuse depth maps into it, in place
    tsdf_mesh(vol, normals=True, colors=True)       the masked marching cubes of the state: an extract_mesh dict
    extract_mesh_tsdf(model, poses, K, img_wh, resolution=512, bounds=None, trunc=None, min_opacity=0.5, normals=True,
                      colors=True, chunk=points.CHUNK, timings=None)            all of the above

Render: `ngp_points_rays` with step 1 (ray k = view k div HW, pixel k mod HW) and `ngp_render_infer_frame` with the
point-cloud export's configuration (black background, T 1e-4, MAX_SAMPLES), `chunk` rays at a time from the same
buffers; the wavefront's per-round quota follows the batch, so the maps are a fixed function of (model, cameras, chunk).
Integration: `ngp_tsdf_integrate` (csrc/fusion.cu); mesh: `ngp_tsdf_mc_count` / `_emit` (csrc/mesh.cu). The rules are
in include/ngp_b200.h ("Depth fusion (TSDF)") and oracle/tsdf_ref.py restates them in numpy. The mesh dict has
extract_mesh's keys, so remove_small_components, simplify_mesh, bake_texture, write_ply and write_obj take it as it is.
Tensors must live on a CUDA device, otherwise RuntimeError; there is no CPU path. Deterministic: two calls are bitwise
equal.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .mesh import _chk, _need, _np, _st, _three, lattice
from .models.rendering import default_exp_step_factor, infer_cfg
from .points import CHUNK, MAX_RAYS, _render_chunks

STATE_BYTES = 24   # per lattice point: tsdf, weight, colour mean (3), colour weight
MAP_BYTES = 20     # per rendered pixel: opacity, depth, rgb


def _infer_cfg(model, B, exp_step_factor):
    """render_views' configuration for chunks of B rays (the point-cloud export's: black background, T_threshold 1e-4,
    MAX_SAMPLES), with the model's box centre and half size, behind which the spare rays of a short chunk start"""
    return (infer_cfg(model, B, exp_step_factor, 0.0), model.center.flatten().tolist(),
            model.half_size.flatten().tolist())


@torch.no_grad()
def render_views(model, poses, directions, chunk=CHUNK, exp_step_factor=None):
    """opacity, depth (V, HW) and rgb (V, HW, 3) of every pixel of every view, rendered as points.extract_points
    renders its rays (black background; exp_step_factor defaults to train.py's rule), `chunk` rays at a time in view
    then pixel order. RuntimeError for CPU tensors, a bad chunk, or maps that do not fit in free device memory."""
    _chk(model.xyz_encoder.params, "render_views")
    dev = model.xyz_encoder.params.device
    if isinstance(chunk, bool) or not isinstance(chunk, (int, np.integer)) or not 1 <= chunk <= MAX_RAYS:
        raise RuntimeError("ngp_pl_b200.fusion.render_views: chunk must be an integer in 1..2^28, got %r" % (chunk,))
    poses = torch.as_tensor(poses, dtype=torch.float32).to(dev).reshape(-1, 3, 4).contiguous()
    directions = torch.as_tensor(directions, dtype=torch.float32).to(dev).reshape(-1, 3).contiguous()
    V, HW = poses.shape[0], directions.shape[0]
    if V < 1 or HW < 1:
        raise RuntimeError("ngp_pl_b200.fusion.render_views: no cameras (%d poses, %d directions)" % (V, HW))
    if exp_step_factor is None:
        exp_step_factor = default_exp_step_factor(model)
    N = V * HW
    B = min(int(chunk), N)
    n_chunks = (N + B - 1) // B
    cfg = _infer_cfg(model, B, exp_step_factor)[0]
    with torch.cuda.device(dev):
        infer_bytes = _lib.lib().ngp_render_infer_workspace(B, cfg.max_round_samples)
        # the maps are padded to whole chunks, so every chunk renders straight into them
        _need(dev, n_chunks * B * MAP_BYTES + B * 40 + infer_bytes, "the maps of %d views of %d pixels" % (V, HW),
              "render_views")
        opacity = torch.empty(n_chunks * B, device=dev)
        depth = torch.empty(n_chunks * B, device=dev)
        rgb = torch.empty(n_chunks * B, 3, device=dev)
        for _ in _render_chunks(model, cfg, poses, directions, 1, N, lambda k0: (opacity[k0:], depth[k0:], rgb[k0:])):
            pass
    return {"opacity": opacity[:N].view(V, HW), "depth": depth[:N].view(V, HW), "rgb": rgb[:N].view(V, HW, 3)}


def default_trunc(lat):
    """4 times the largest lattice step (fp32)"""
    return float(np.float32(4) * np.float32(max(lat.step)))


def _trunc(trunc, fn):
    t = float(trunc)
    if not (t > 0 and math.isfinite(t) and math.isfinite(float(np.float32(t))) and np.float32(t) > 0):
        raise RuntimeError("ngp_pl_b200.fusion.%s: trunc must be positive and finite, got %r" % (fn, trunc))
    return t


@torch.no_grad()
def tsdf_volume(resolution, bounds, trunc=None, device=None):
    """An empty TSDF state on mesh.lattice(resolution, lo, hi), bounds = (lo, hi): {'tsdf' (n0, n1, n2) float32,
    'weight' int32, 'color' (n0, n1, n2, 3) float32, 'color_weight' int32, all 0, 'lattice' (NgpLattice), 'trunc'}.
    trunc defaults to 4 times the largest lattice step. RuntimeError, before allocating, when the 24 B per point do not
    fit in free device memory."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("ngp_pl_b200.fusion.tsdf_volume needs a CUDA device (got %s); there is no CPU path" % dev)
    lo, hi = bounds
    lo, hi = _three(_np(lo), np.float32), _three(_np(hi), np.float32)
    if not (np.isfinite(lo).all() and np.isfinite(hi).all() and (lo < hi).all()):
        raise RuntimeError("ngp_pl_b200.fusion.tsdf_volume: bounds need lo < hi on every axis, got %s .. %s" % (lo, hi))
    lat = lattice(resolution, lo, hi)
    trunc = default_trunc(lat) if trunc is None else _trunc(trunc, "tsdf_volume")
    n = tuple(int(x) for x in lat.n)
    _need(dev, n[0] * n[1] * n[2] * STATE_BYTES, "the state of a %dx%dx%d lattice" % n, "tsdf_volume")
    return {"tsdf": torch.zeros(n, device=dev, dtype=torch.float32), "weight": torch.zeros(n, device=dev, dtype=torch.int32),
            "color": torch.zeros(n + (3,), device=dev, dtype=torch.float32),
            "color_weight": torch.zeros(n, device=dev, dtype=torch.int32), "lattice": lat, "trunc": trunc}


def _check_vol(vol, fn):
    lat = vol["lattice"]
    n = tuple(int(x) for x in lat.n)
    want = (("tsdf", n, torch.float32), ("weight", n, torch.int32), ("color", n + (3,), torch.float32),
            ("color_weight", n, torch.int32))
    for key, shape, dtype in want:
        t = vol[key]
        _chk(t, fn)
        if tuple(t.shape) != shape or t.dtype != dtype or not t.is_contiguous():
            raise RuntimeError("ngp_pl_b200.fusion.%s: vol['%s'] must be a contiguous %s tensor of shape %s, got %s %s"
                               % (fn, key, dtype, shape, t.dtype, tuple(t.shape)))
    return lat, vol["tsdf"].device


@torch.no_grad()
def integrate(vol, poses, K, img_wh, depth, opacity, rgb, min_opacity=0.5):
    """Fuse depth maps into vol (tsdf_volume) in place, views in pose order, by the rule of include/ngp_b200.h: poses
    (V, 3, 4) [right down front], one pinhole K (3, 3) and img_wh = (W, H); depth, opacity (V, H W) and rgb (V, H W, 3)
    as render_views returns them, or any others (opacity 1 where a depth is known, 0 elsewhere). Returns vol.
    RuntimeError for CPU tensors, bad shapes or min_opacity outside (0, 1]."""
    lat, dev = _check_vol(vol, "integrate")
    trunc = _trunc(vol["trunc"], "integrate")
    if not (0 < min_opacity <= 1):
        raise RuntimeError("ngp_pl_b200.fusion.integrate: min_opacity must be in (0, 1], got %r" % (min_opacity,))
    for t in (depth, opacity, rgb):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError("ngp_pl_b200.fusion.integrate: depth, opacity and rgb must be CUDA tensors")
        _chk(t, "integrate")
    W, H = (int(x) for x in img_wh)
    K = np.asarray(_np(K), np.float32)
    if K.shape != (3, 3) or W < 1 or H < 1:
        raise RuntimeError("ngp_pl_b200.fusion.integrate: expected K (3, 3) and img_wh (W, H) >= 1, got %s and %s"
                           % (K.shape, (W, H)))
    poses = torch.as_tensor(poses, dtype=torch.float32).to(dev)
    if poses.dim() != 3 or tuple(poses.shape[1:]) != (3, 4):
        raise RuntimeError("ngp_pl_b200.fusion.integrate: poses must be (V, 3, 4), got %s" % (tuple(poses.shape),))
    V, HW = poses.shape[0], W * H
    for t, shape, what in ((depth, (V, HW), "depth"), (opacity, (V, HW), "opacity"), (rgb, (V, HW, 3), "rgb")):
        if tuple(t.shape) != shape or t.dtype != torch.float32:
            raise RuntimeError("ngp_pl_b200.fusion.integrate: %s must be float32 %s for %d views of %dx%d, got %s %s"
                               % (what, shape, V, W, H, t.dtype, tuple(t.shape)))
    from .datasets import ray_directions
    dirs = ray_directions(W, H, K).to(dev).contiguous()
    Kc = (C.c_float * 9)(*[float(x) for x in K.reshape(-1)])
    depth, opacity, rgb = depth.contiguous(), opacity.contiguous(), rgb.contiguous()
    poses = poses.contiguous()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ngp_tsdf_integrate(C.byref(lat), float(trunc), V, poses.data_ptr(), Kc, W, H, dirs.data_ptr(),
                                                 depth.data_ptr(), opacity.data_ptr(), rgb.data_ptr(), float(min_opacity),
                                                 vol["tsdf"].data_ptr(), vol["weight"].data_ptr(), vol["color"].data_ptr(),
                                                 vol["color_weight"].data_ptr(), _st(dev)), "ngp_tsdf_integrate")
    return vol


@torch.no_grad()
def tsdf_mesh(vol, normals=True, colors=True):
    """The masked marching cubes of vol (include/ngp_b200.h): the level 0 of F over the observed points, with
    world-space vertices, normals out of the solid and the fused colours (uint8). Returns extract_mesh's dict
    {'vertices', 'triangles', 'normals' or None, 'colors' or None}. Observed everywhere, it is exactly
    mesh.marching_cubes(-F, 0, lo, step, normals=True). RuntimeError, before allocating, when the output does not fit
    in free device memory."""
    lat, dev = _check_vol(vol, "tsdf_mesh")
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_tsdf_mc_workspace(C.byref(lat))
        if ws_bytes == 0:
            raise RuntimeError("ngp_pl_b200.fusion.tsdf_mesh: unsupported lattice %s" % (tuple(lat.n),))
        _need(dev, ws_bytes, "the marching-cubes workspace", "tsdf_mesh")
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        counts = torch.empty(2, device=dev, dtype=torch.int64)
        st = _st(dev)
        F, Wt = vol["tsdf"], vol["weight"]
        _lib.check(L.ngp_tsdf_mc_count(F.data_ptr(), Wt.data_ptr(), C.byref(lat), counts.data_ptr(), ws.data_ptr(), ws_bytes,
                                       st), "ngp_tsdf_mc_count")
        nv, nt = (int(x) for x in counts.cpu())
        _need(dev, nv * (12 + (12 if normals else 0) + (3 if colors else 0)) + nt * 24,
              "%d vertices and %d triangles" % (nv, nt), "tsdf_mesh")
        verts = torch.empty(nv, 3, device=dev, dtype=torch.float32)
        tris = torch.empty(nt, 3, device=dev, dtype=torch.int64)
        nrm = torch.empty(nv, 3, device=dev, dtype=torch.float32) if normals else None
        col = torch.empty(nv, 3, device=dev, dtype=torch.uint8) if colors else None
        if nv > 0:
            _lib.check(L.ngp_tsdf_mc_emit(F.data_ptr(), Wt.data_ptr(), vol["color"].data_ptr(), vol["color_weight"].data_ptr(),
                                          C.byref(lat), verts.data_ptr(), nrm.data_ptr() if normals else None,
                                          col.data_ptr() if colors else None, tris.data_ptr(), nv, nt, ws.data_ptr(),
                                          ws_bytes, st), "ngp_tsdf_mc_emit")
        del ws
    return {"vertices": verts, "triangles": tris, "normals": nrm, "colors": col}


@torch.no_grad()
def extract_mesh_tsdf(model, poses, K, img_wh, resolution=512, bounds=None, trunc=None, min_opacity=0.5, normals=True,
                      colors=True, chunk=CHUNK, timings=None):
    """render_views of every pixel of the views (poses, K, img_wh: the training cameras), integrate into a
    tsdf_volume over `bounds` (default: the model's box) and tsdf_mesh. timings (a dict) gets the CUDA-event
    milliseconds of 'render', 'integrate' and 'mesh'. RuntimeError for CPU tensors, a bad trunc or min_opacity, or a
    state or output that does not fit in free device memory (checked before allocating)."""
    _chk(model.xyz_encoder.params, "extract_mesh_tsdf")
    dev = model.xyz_encoder.params.device
    if not (0 < min_opacity <= 1):
        raise RuntimeError("ngp_pl_b200.fusion.extract_mesh_tsdf: min_opacity must be in (0, 1], got %r" % (min_opacity,))
    if trunc is not None:
        _trunc(trunc, "extract_mesh_tsdf")
    if bounds is None:
        bounds = (model._xyz_min_host, model._xyz_max_host)
    W, H = (int(x) for x in img_wh)
    K = np.asarray(_np(K), np.float32)
    from .datasets import ray_directions
    dirs = ray_directions(W, H, K)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timings is not None else None
    with torch.cuda.device(dev):
        if ev:
            ev[0].record()
        maps = render_views(model, poses, dirs, chunk=chunk)
        if ev:
            ev[1].record()
        vol = tsdf_volume(resolution, bounds, trunc, dev)
        integrate(vol, poses, K, (W, H), maps["depth"], maps["opacity"], maps["rgb"], min_opacity)
        del maps
        if ev:
            ev[2].record()
        m = tsdf_mesh(vol, normals=normals, colors=colors)
        if ev:
            ev[3].record()
            ev[3].synchronize()
            for s, name in enumerate(("render", "integrate", "mesh")):
                timings[name] = timings.get(name, 0.0) + ev[s].elapsed_time(ev[s + 1])
    return m
