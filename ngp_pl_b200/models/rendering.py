"""render(model, rays_o, rays_d, **kwargs) with the reference's signature, kwargs and result keys
(reference models/rendering.py:11-163).

kwargs honoured: test_time, exp_step_factor, T_threshold, max_samples, random_bg, to_cpu, to_numpy,
output_radiance (`exposure` belongs to the HDR tonemapper path, outside the hot path).
Result keys -- train: deltas, ts, rm_samples, vr_samples, opacity, depth, rgb, ws, rays_a;
test: opacity, depth, rgb, total_samples.
"""
import ctypes as C

import torch

from .custom_functions import RayAABBIntersector, RayMarcher, VolumeRenderer
from .. import _lib, vren

MAX_SAMPLES = 1024
NEAR_DISTANCE = 0.01


def default_exp_step_factor(model):
    """train.py's rule, read from the model: 1/256 (exponential steps) for scale > 0.5, else 0 (constant steps)"""
    return 1 / 256 if float(model.scale) > 0.5 else 0.0


def infer_cfg(model, n_rays, exp_step_factor, bg, T_threshold=1e-4, sample_budget=MAX_SAMPLES):
    """NgpInferCfg of the inference wavefront for n_rays rays of model: the marcher's MAX_SAMPLES step bound, the near
    plane NEAR_DISTANCE, background bg in all three channels, the outer loop's sample_budget and per-round sample
    buffers of max(4 n_rays, 2^16), so the per-ray quota is never clipped"""
    cfg = _lib.NgpInferCfg()
    cfg.n_rays, cfg.cascades, cfg.grid_size, cfg.max_samples = n_rays, model.cascades, model.grid_size, MAX_SAMPLES
    cfg.scale, cfg.exp_step_factor = float(model.scale), float(exp_step_factor)
    cfg.T_threshold, cfg.near_distance = float(T_threshold), NEAR_DISTANCE
    c, h = model.center.flatten().tolist(), model.half_size.flatten().tolist()
    for k in range(3):
        cfg.center[k], cfg.half_size[k], cfg.bg[k] = c[k], h[k], bg
    cfg.sample_budget = int(sample_budget)
    cfg.max_round_samples = max(4 * n_rays, 1 << 16)
    return cfg


@torch.amp.autocast('cuda')
def render(model, rays_o, rays_d, **kwargs):
    rays_o = rays_o.contiguous()
    rays_d = rays_d.contiguous()
    _, hits_t, _ = RayAABBIntersector.apply(rays_o, rays_d, model.center, model.half_size, 1)
    # rays starting inside the box begin at the near plane (reference rendering.py:29); branch-free,
    # no boolean-mask index_put (which costs a host sync in the reference)
    t0 = hits_t[:, 0, 0]
    hits_t[:, 0, 0] = torch.where((t0 >= 0) & (t0 < NEAR_DISTANCE), torch.full_like(t0, NEAR_DISTANCE), t0)

    if kwargs.get('test_time', False):
        # default: the sync-free device-side wavefront (ngp_render_infer); fused=False runs the
        # reference-shaped host loop over the unfused operators (kept for operator-level parity)
        fn = _render_rays_test_fused if kwargs.get('fused', True) else _render_rays_test
    else:
        fn = _render_rays_train
    results = fn(model, rays_o, rays_d, hits_t, **kwargs)
    if kwargs.get('to_cpu', False):
        for k, v in results.items():
            if torch.is_tensor(v):
                v = v.cpu()
                if kwargs.get('to_numpy', False):
                    v = v.numpy()
            results[k] = v
    return results


def _background(exp_step_factor, device, random_bg=False):
    if exp_step_factor == 0:  # synthetic scenes: white
        return torch.ones(3, device=device)
    if random_bg:
        return torch.rand(3, device=device)
    return torch.zeros(3, device=device)


@torch.no_grad()
def _render_rays_test_fused(model, rays_o, rays_d, hits_t, **kwargs):
    """Inference as a device-side wavefront. Default: ngp_render_infer_frame -- the whole frame is ONE CUDA graph with a
    device-side while loop, no host read-back (graph=False or a driver without conditional graph nodes: ngp_render_infer,
    `rounds_per_check` rounds per host read of the alive count; the reference synchronises >= 3 times per round)."""
    from .networks import _net_struct
    exp_step_factor = kwargs.get('exp_step_factor', 0.)
    N = rays_o.shape[0]
    dev = rays_o.device
    with torch.cuda.device(dev):
        L = _lib.lib()
        cfg = infer_cfg(model, N, exp_step_factor, 1.0 if exp_step_factor == 0 else 0.0, kwargs.get('T_threshold', 1e-4),
                        kwargs.get('max_samples', MAX_SAMPLES))
        ws_bytes = L.ngp_render_infer_workspace(N, cfg.max_round_samples)
        # persistent per-model buffers: workspace, staged rays and outputs keep their addresses from frame to frame, which
        # is what lets the cached frame graph be replayed
        cache = getattr(model, '_infer_cache', None)
        if cache is None or cache['N'] != N or cache['dev'] != dev or cache['ws'].numel() < ws_bytes:
            cache = dict(N=N, dev=dev, ws=torch.empty(ws_bytes, device=dev, dtype=torch.uint8),
                         o=torch.empty(N, 3, device=dev), d=torch.empty(N, 3, device=dev), opacity=torch.empty(N, device=dev),
                         depth=torch.empty(N, device=dev), rgb=torch.empty(N, 3, device=dev),
                         total=torch.zeros(1, device=dev, dtype=torch.int64), alive=torch.zeros(1, device=dev, dtype=torch.int32),
                         alive_host=torch.zeros(1, dtype=torch.int32).pin_memory())
            model._infer_cache = cache
        ws, o, d = cache['ws'], cache['o'], cache['d']
        opacity, depth, rgb, total = cache['opacity'], cache['depth'], cache['rgb'], cache['total']
        o.copy_(rays_o)
        d.copy_(rays_d)
        net, keep = _net_struct(model)
        st = torch.cuda.current_stream().cuda_stream
        done = False
        if kwargs.get('graph', True) and getattr(model, '_infer_graph_ok', True):
            rc = L.ngp_render_infer_frame(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                          opacity.data_ptr(), depth.data_ptr(), rgb.data_ptr(), total.data_ptr(), ws.data_ptr(),
                                          ws.numel(), st)
            if rc == 0:
                done = True
            elif rc < 0:
                _lib.check(rc, "render_infer_frame")
            else:
                model._infer_graph_ok = False  # conditional graph nodes unavailable: host-chunked rounds from now on
        if not done:
            alive, alive_host = cache['alive'], cache['alive_host']
            chunk = int(kwargs.get('rounds_per_check', 8))
            first = 0
            while True:
                # `chunk` rounds are enqueued back to back; the alive count is read back once per chunk
                rc = L.ngp_render_infer(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                        opacity.data_ptr(), depth.data_ptr(), rgb.data_ptr(), total.data_ptr(), first, chunk, 0,
                                        alive.data_ptr(), ws.data_ptr(), ws.numel(), st)
                _lib.check(rc, "render_infer")
                first += chunk
                alive_host.copy_(alive, non_blocking=True)
                torch.cuda.current_stream().synchronize()
                if int(alive_host[0]) == 0 or first > 2 * cfg.sample_budget:
                    break
            rc = L.ngp_render_infer(C.byref(net), C.byref(cfg), o.data_ptr(), d.data_ptr(), model.density_bitfield.data_ptr(),
                                    opacity.data_ptr(), depth.data_ptr(), rgb.data_ptr(), total.data_ptr(), first, 0, 1, None,
                                    ws.data_ptr(), ws.numel(), st)
            _lib.check(rc, "render_infer(finish)")
        # fresh tensors for the caller (the persistent ones are overwritten by the next frame)
        return {'opacity': opacity.clone(), 'depth': depth.clone(), 'rgb': rgb.clone(), 'total_samples': total[0].clone()}


@torch.no_grad()
def _render_rays_test(model, rays_o, rays_d, hits_t, **kwargs):
    """Inference: alive rays take N more occupied samples per round until their transmittance falls
    below T_threshold or they leave the box (reference rendering.py:46-118)."""
    exp_step_factor = kwargs.get('exp_step_factor', 0.)
    T_threshold = kwargs.get('T_threshold', 1e-4)
    budget = kwargs.get('max_samples', MAX_SAMPLES)
    N_rays = len(rays_o)
    device = rays_o.device
    opacity = torch.zeros(N_rays, device=device)
    depth = torch.zeros(N_rays, device=device)
    rgb = torch.zeros(N_rays, 3, device=device)
    alive = torch.arange(N_rays, device=device)
    min_samples = 1 if exp_step_factor == 0 else 4
    hits = hits_t[:, 0]

    requested = 0
    total_samples = 0
    while requested < budget and len(alive) > 0:
        N_samples = max(min(N_rays // len(alive), 64), min_samples)
        requested += N_samples
        xyzs, dirs, deltas, ts, N_eff = vren.raymarching_test(
            rays_o, rays_d, hits, alive, model.density_bitfield, model.cascades, model.scale, exp_step_factor,
            model.grid_size, MAX_SAMPLES, N_samples)
        total_samples = total_samples + N_eff.sum()
        # padded slots have dirs == 0 (kept for parity with the reference's valid_mask); the network is
        # simply evaluated on every slot: padded slots are never composited (s >= N_eff)
        flat_x = xyzs.reshape(-1, 3)
        flat_d = dirs.reshape(-1, 3)
        valid = ~torch.all(flat_d == 0, dim=1)
        if not bool(valid.any()):
            break
        flat_d = torch.where(valid[:, None], flat_d, torch.tensor([0., 0., 1.], device=device))
        sigmas, rgbs = model(flat_x, flat_d, **kwargs)
        sigmas = torch.where(valid, sigmas.float(), torch.zeros_like(sigmas, dtype=torch.float32))
        rgbs = torch.where(valid[:, None], rgbs.float(), torch.zeros_like(rgbs, dtype=torch.float32))
        vren.composite_test_fw(sigmas.reshape(-1, N_samples).contiguous(), rgbs.reshape(-1, N_samples, 3).contiguous(),
                               deltas, ts, hits, alive, T_threshold, N_eff, opacity, depth, rgb)
        alive = alive[alive >= 0]

    results = {'opacity': opacity, 'depth': depth, 'total_samples': total_samples}
    bg = _background(exp_step_factor, device)
    results['rgb'] = rgb + bg * (1 - opacity)[:, None]
    return results


def _render_rays_train(model, rays_o, rays_d, hits_t, **kwargs):
    """Training: march -> network -> ragged compositing (reference rendering.py:121-163)."""
    exp_step_factor = kwargs.get('exp_step_factor', 0.)
    results = {}
    rays_a, xyzs, dirs, results['deltas'], results['ts'], results['rm_samples'] = RayMarcher.apply(
        rays_o, rays_d, hits_t[:, 0], model.density_bitfield, model.cascades, model.scale, exp_step_factor,
        model.grid_size, MAX_SAMPLES)

    per_sample = {}
    for k, v in kwargs.items():  # per-ray tensor kwargs are expanded to per-sample
        if isinstance(v, torch.Tensor):
            per_sample[k] = torch.repeat_interleave(v[rays_a[:, 0]], rays_a[:, 2], 0)
    kwargs = {**kwargs, **per_sample}
    sigmas, rgbs = model(xyzs, dirs, **kwargs)

    results['vr_samples'], results['opacity'], results['depth'], rgb, results['ws'] = VolumeRenderer.apply(
        sigmas, rgbs.contiguous(), results['deltas'], results['ts'], rays_a, kwargs.get('T_threshold', 1e-4))
    results['rays_a'] = rays_a
    bg = _background(exp_step_factor, rays_o.device, kwargs.get('random_bg', False))
    results['rgb'] = rgb + bg * (1 - results['opacity'])[:, None]
    return results
