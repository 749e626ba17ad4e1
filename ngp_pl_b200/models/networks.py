"""NGP model with the reference's constructor, attributes, buffers and methods
(reference models/networks.py:12-269), evaluated by the fused sm_90a kernels in libngp_b200.so.

State-dict keys match the reference: center, xyz_min, xyz_max, half_size, density_bitfield,
xyz_encoder.params, dir_encoder.params (empty), rgb_net.params (+ density_grid / grid_coords when the
caller registers them, reference train.py:72-76).
"""
import ctypes as C

import numpy as np
import torch
from torch import nn
from torch.amp import custom_bwd, custom_fwd

from .. import _lib, tcnn, vren
from .rendering import NEAR_DISTANCE


def _st():
    return torch.cuda.current_stream().cuda_stream


def _net_struct(model):
    """NgpNet for the C ABI from an NGP module (fp16 working copies are refreshed if params changed)."""
    net = _lib.NgpNet()
    enc_h = model.xyz_encoder.half_params()
    rgb_h = model.rgb_net.half_params()
    net.enc_params_h = enc_h.data_ptr()
    net.rgb_params_h = rgb_h.data_ptr()
    net.meta = model.xyz_encoder.meta
    for k in range(3):
        net.xyz_min[k] = model._xyz_min_host[k]
        net.xyz_max[k] = model._xyz_max_host[k]
    net.rgb_act = model.rgb_net.rgb_act
    return net, (enc_h, rgb_h)


def need_cuda(t, what):
    """there is no CPU path: fail like the reference's TORCH_CHECK(is_cuda) (models/csrc/include/utils.h:4-6)"""
    if not t.is_cuda:
        raise RuntimeError("ngp_pl_b200: %s needs CUDA tensors (got %s); there is no CPU or PyTorch fallback" % (what, t.device))


def _samples_struct(x, d):
    s = _lib.NgpSamples()
    s.xyzs = x.data_ptr()
    s.dirs = d.data_ptr() if d is not None else None
    s.rays_o = None
    s.rays_d = None
    s.ray_idx = None
    s.ts = None
    s.n = x.shape[0]
    return s


def feat_save_bytes(n):
    return ((n + 31) // 32) * 32 * 64


class _NGPForward(torch.autograd.Function):
    """sigmas, rgbs = NGP(x, d): hash grid + density MLP + exp + SH + rgb MLP in one kernel; one kernel back."""

    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x, d, enc_params, rgb_params, model):
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            # tinycudann also returns dL/dx through the hash grid (and dL/dd through SH); the reference needs it only for
            # --optimize_ext (learned pose corrections, train.py:88-91). Not built here: fail loudly instead of silently
            # handing zero gradients to RayMarcher.backward.
            raise NotImplementedError("ngp_pl_b200: gradients w.r.t. sample positions / directions (pose refinement, "
                                      "reference --optimize_ext) are not implemented; detach x and d")
        x = x.contiguous()
        d = d.contiguous()
        n = x.shape[0]
        dev = x.device
        with torch.cuda.device(dev):
            net, keep = _net_struct(model)
            smp = _samples_struct(x, d)
            sig = torch.empty(n, device=dev, dtype=torch.float32)
            rgb = torch.empty(n, 3, device=dev, dtype=torch.float32)
            need_grad = any(ctx.needs_input_grad)
            feat = torch.empty(feat_save_bytes(n), device=dev, dtype=torch.uint8) if need_grad else None
            rc = _lib.lib().ngp_net_forward(C.byref(net), C.byref(smp), 1, sig.data_ptr(), rgb.data_ptr(), None,
                                            feat.data_ptr() if feat is not None else None, _st())
            _lib.check(rc, "net_forward")
        ctx.model = model
        ctx.feat = feat
        ctx.save_for_backward(x, d, sig)
        return sig, rgb

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dL_dsig, dL_drgb):
        x, d, sig = ctx.saved_tensors
        model = ctx.model
        dev = x.device
        n = x.shape[0]
        with torch.cuda.device(dev):
            net, keep = _net_struct(model)
            smp = _samples_struct(x, d)
            g_enc = torch.zeros_like(model.xyz_encoder.params)
            g_rgb = torch.zeros_like(model.rgb_net.params)
            if n > 0:
                dL_dsig = dL_dsig.contiguous().float()
                dL_drgb = dL_drgb.contiguous().float()
                scratch = torch.empty(2, device=dev, dtype=torch.float32)
                L = _lib.lib()
                _lib.check(L.ngp_grad_scale(dL_dsig.data_ptr(), sig.data_ptr(), dL_drgb.data_ptr(), n,
                                            scratch.data_ptr(), scratch[1:].data_ptr(), _st()), "grad_scale")
                ws_bytes = L.ngp_net_backward_workspace(n)
                ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
                rc = L.ngp_net_backward(C.byref(net), C.byref(smp), dL_dsig.data_ptr(), dL_drgb.data_ptr(),
                                        ctx.feat.data_ptr() if ctx.feat is not None else None,
                                        scratch[1:].data_ptr(), g_enc.data_ptr(), g_rgb.data_ptr(), ws.data_ptr(), ws_bytes,
                                        _st())
                _lib.check(rc, "net_backward")
        return None, None, g_enc, g_rgb, None


def _pow2_scale(t):
    """power-of-two loss scale 2^floor(log2(256 / max|t|)) as a device scalar (no host sync); 1 if t == 0"""
    amax = t.detach().abs().max().float()
    s = torch.exp2(torch.floor(torch.log2(256.0 / amax.clamp_min(1e-30)))).clamp(2.0 ** -60, 2.0 ** 60)
    return torch.where(amax > 0, s, torch.ones_like(s)).reshape(1).contiguous()


def _unit_net(module):
    """NgpNet of a stand-alone tcnn.NetworkWithInputEncoding: its input is already in [0,1]^3"""
    net = _lib.NgpNet()
    enc_h = module.half_params()
    net.enc_params_h = enc_h.data_ptr()
    net.rgb_params_h = None
    net.meta = module.meta
    for k in range(3):
        net.xyz_min[k], net.xyz_max[k] = 0.0, 1.0
    net.rgb_act = 1
    return net, enc_h


class _DensityFeatures(torch.autograd.Function):
    """tcnn.NetworkWithInputEncoding.forward stand-alone: x01 (N,3) in [0,1] -> fp16 (N,16)
    (reference call site: networks.py:104  h = self.xyz_encoder(x))."""

    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x01, params, module):
        if ctx.needs_input_grad[0]:
            raise NotImplementedError("ngp_pl_b200: dL/dx through the hash grid (reference --optimize_ext) is not implemented; "
                                      "detach the positions")
        x01 = x01.float().contiguous()  # (cast_inputs only acts under autocast)
        n, dev = x01.shape[0], x01.device
        with torch.cuda.device(dev):
            net, keep = _unit_net(module)
            smp = _samples_struct(x01, None)
            h = torch.empty(n, 16, device=dev, dtype=torch.float16)
            sig = torch.empty(n, device=dev, dtype=torch.float32)
            need = any(ctx.needs_input_grad)
            feat = torch.empty(feat_save_bytes(n), device=dev, dtype=torch.uint8) if need else None
            rc = _lib.lib().ngp_net_forward(C.byref(net), C.byref(smp), 0, sig.data_ptr(), None, h.data_ptr(),
                                            feat.data_ptr() if feat is not None else None, _st())
            _lib.check(rc, "net_forward(features)")
        ctx.module, ctx.feat = module, feat
        ctx.save_for_backward(x01)
        return h

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dL_dh):
        (x01,) = ctx.saved_tensors
        module = ctx.module
        n, dev = x01.shape[0], x01.device
        g = torch.zeros_like(module.params)
        if n > 0:
            with torch.cuda.device(dev):
                net, keep = _unit_net(module)
                smp = _samples_struct(x01, None)
                d = dL_dh.float().contiguous()
                scale = _pow2_scale(d)
                L = _lib.lib()
                ws_bytes = L.ngp_net_backward_workspace(n)
                ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
                rc = L.ngp_enc_backward(C.byref(net), C.byref(smp), d.data_ptr(), ctx.feat.data_ptr(), scale.data_ptr(),
                                        g.data_ptr(), ws.data_ptr(), ws_bytes, _st())
                _lib.check(rc, "enc_backward")
        return None, g, None


class _RgbMlp(torch.autograd.Function):
    """tcnn.Network(32 -> 3).forward stand-alone: x (N,32) -> fp16 (N,3) (reference call site networks.py:145)."""

    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float16)
    def forward(ctx, x, params, module):
        x = x.half().contiguous()  # (cast_inputs only acts under autocast)
        n, dev = x.shape[0], x.device
        with torch.cuda.device(dev):
            wh = module.half_params()
            out = torch.empty(n, 3, device=dev, dtype=torch.float16)
            rc = _lib.lib().ngp_mlp_rgb_forward(wh.data_ptr(), x.data_ptr(), n, module.rgb_act, out.data_ptr(), _st())
            _lib.check(rc, "mlp_rgb_forward")
        ctx.module = module
        ctx.save_for_backward(x)
        return out

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dL_dout):
        (x,) = ctx.saved_tensors
        module = ctx.module
        n, dev = x.shape[0], x.device
        g = torch.zeros_like(module.params)
        dx = torch.zeros(n, 32, device=dev, dtype=torch.float32) if ctx.needs_input_grad[0] else None
        if n > 0:
            with torch.cuda.device(dev):
                wh = module.half_params()
                d = dL_dout.float().contiguous()
                scale = _pow2_scale(d)
                rc = _lib.lib().ngp_mlp_rgb_backward(wh.data_ptr(), x.data_ptr(), d.data_ptr(), n, module.rgb_act,
                                                     scale.data_ptr(), dx.data_ptr() if dx is not None else None,
                                                     g.data_ptr(), _st())
                _lib.check(rc, "mlp_rgb_backward")
        return dx, g, None


def sh_encode(u):
    """tcnn.Encoding(SphericalHarmonics, degree 4): u in [0,1]^3 (N,3) -> fp16 (N,16); no gradient (the
    reference feeds it normalised directions that do not require grad, networks.py:143-144)."""
    u = u.detach().float().contiguous()
    out = torch.empty(u.shape[0], 16, device=u.device, dtype=torch.float16)
    with torch.cuda.device(u.device):
        _lib.check(_lib.lib().ngp_sh_encode(u.data_ptr(), u.shape[0], out.data_ptr(), _st()), "sh_encode")
    return out


class NGP(nn.Module):
    def __init__(self, scale, rgb_act='Sigmoid', n_levels=16, log2_hashmap_size=19, n_features=2, base_resolution=16):
        """`scale`, `rgb_act` as in the reference (networks.py:13). The grid hyper-parameters L / log2_T
        / N_min, hard-coded at networks.py:32, are keyword arguments here so that BASELINE config 1
        (L=4, T=2^14) can be built; the defaults are the reference's."""
        super().__init__()
        self.rgb_act = rgb_act

        # scene bounding box
        self.scale = scale
        self.register_buffer('center', torch.zeros(1, 3))
        self.register_buffer('xyz_min', -torch.ones(1, 3) * scale)
        self.register_buffer('xyz_max', torch.ones(1, 3) * scale)
        self.register_buffer('half_size', (self.xyz_max - self.xyz_min) / 2)
        self._xyz_min_host = [float(np.float32(-scale))] * 3
        self._xyz_max_host = [float(np.float32(scale))] * 3

        # each density grid covers [-2^(k-1), 2^(k-1)]^3 for k in [0, C-1]
        self.cascades = max(1 + int(np.ceil(np.log2(2 * scale))), 1)
        self.grid_size = 128
        self.register_buffer('density_bitfield',
                             torch.zeros(self.cascades * self.grid_size ** 3 // 8, dtype=torch.uint8))

        L, F, log2_T, N_min = n_levels, n_features, log2_hashmap_size, base_resolution
        b = np.exp(np.log(2048 * scale / N_min) / (L - 1))
        self.per_level_scale = float(b)

        self.xyz_encoder = tcnn.NetworkWithInputEncoding(
            n_input_dims=3, n_output_dims=16,
            encoding_config={"otype": "Grid", "type": "Hash", "n_levels": L, "n_features_per_level": F,
                             "log2_hashmap_size": log2_T, "base_resolution": N_min, "per_level_scale": b,
                             "interpolation": "Linear"},
            network_config={"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None",
                            "n_neurons": 64, "n_hidden_layers": 1})
        self.dir_encoder = tcnn.Encoding(n_input_dims=3, encoding_config={"otype": "SphericalHarmonics", "degree": 4})
        self.rgb_net = tcnn.Network(
            n_input_dims=32, n_output_dims=3,
            network_config={"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": self.rgb_act,
                            "n_neurons": 64, "n_hidden_layers": 2})
        if self.rgb_act == 'None':
            # the HDR-NeRF tonemapper MLPs (reference networks.py:79-92) are outside the hot path
            pass

    # ------------------------------------------------------------------ network evaluation
    @torch.no_grad()
    def _density_nograd(self, x):
        need_cuda(x, "NGP.density")
        x = x.contiguous().float()
        n = x.shape[0]
        with torch.cuda.device(x.device):
            net, keep = _net_struct(self)
            smp = _samples_struct(x, None)
            sig = torch.empty(n, device=x.device, dtype=torch.float32)
            rc = _lib.lib().ngp_net_forward(C.byref(net), C.byref(smp), 0, sig.data_ptr(), None, None, None, _st())
            _lib.check(rc, "net_forward(density)")
        return sig

    def density(self, x, return_feat=False):
        """x: (N,3) in [-scale, scale] -> sigmas (N)   (reference networks.py:94-107).
        Differentiable evaluation goes through forward(); density() is what the occupancy-grid update
        calls (under no_grad in the reference as well)."""
        if return_feat:
            raise NotImplementedError("return_feat: use forward(x, d)")
        return self._density_nograd(x)

    def forward(self, x, d, **kwargs):
        """x (N,3) in [-scale,scale], d (N,3) directions -> sigmas (N) fp32, rgbs (N,3)
        (reference networks.py:132-153)."""
        if self.rgb_act == 'None' and not kwargs.get('output_radiance', False):
            raise NotImplementedError("HDR tonemapper path (use_exposure) is outside the hot path")
        need_cuda(x, "NGP.forward")
        self.xyz_encoder._half.training_forward(self.xyz_encoder.params)  # tinycudann re-casts its weights every forward
        self.rgb_net._half.training_forward(self.rgb_net.params)
        sig, rgb = _NGPForward.apply(x, d, self.xyz_encoder.params, self.rgb_net.params, self)
        if self.rgb_act == 'None':
            from .custom_functions import TruncExp
            rgb = TruncExp.apply(rgb)
        return sig, rgb

    # ------------------------------------------------------------------ occupancy grid maintenance
    @torch.no_grad()
    def get_all_cells(self):
        """reference networks.py:155-167"""
        indices = vren.morton3D(self.grid_coords).long()
        return [(indices, self.grid_coords)] * self.cascades

    @torch.no_grad()
    def sample_uniform_and_occupied_cells(self, M, density_threshold):
        """reference networks.py:169-195: M uniform + M occupied cells per cascade."""
        cells = []
        dev = self.density_grid.device
        for c in range(self.cascades):
            coords1 = torch.randint(self.grid_size, (M, 3), dtype=torch.int32, device=dev)
            indices1 = vren.morton3D(coords1).long()
            indices2 = torch.nonzero(self.density_grid[c] > density_threshold)[:, 0]
            if len(indices2) > 0:
                rand_idx = torch.randint(len(indices2), (M,), device=dev)
                indices2 = indices2[rand_idx]
            coords2 = vren.morton3D_invert(indices2.int())
            cells += [(torch.cat([indices1, indices2]), torch.cat([coords1, coords2]))]
        return cells

    @torch.no_grad()
    def mark_invisible_cells(self, K, poses, img_wh, chunk=64 ** 3):
        """Cells that no training camera sees (or that lie closer than NEAR_DISTANCE in front of one) get
        density -1 and are never revived; `count_grid` keeps the fraction of cameras covering each cell (used
        by erode=True). Semantics of reference networks.py:197-238; called once before training (train.py:154-157).
        K (3,3) intrinsics, poses (N,3,4) camera-to-world, img_wh (w, h)."""
        G = self.grid_size
        n_cams = poses.shape[0]
        R_wc = poses[:, :3, :3].transpose(1, 2)            # world -> camera rotations (N,3,3)
        t_wc = -(R_wc @ poses[:, :3, 3:])                   # (N,3,1)
        self.count_grid = torch.zeros_like(self.density_grid)
        w, h = float(img_wh[0]), float(img_wh[1])
        for c, (indices, coords) in enumerate(self.get_all_cells()):
            s, half_cell = self._cascade_extent(c)
            for i in range(0, indices.shape[0], chunk):
                idx = indices[i:i + chunk]
                centres = ((coords[i:i + chunk] / (G - 1) * 2 - 1) * (s - half_cell)).T       # (3,M) world
                uvd = K @ (R_wc @ centres + t_wc)                                               # (N,3,M)
                depth = uvd[:, 2]
                uv = uvd[:, :2] / uvd[:, 2:]
                inside = (depth >= 0) & (uv[:, 0] >= 0) & (uv[:, 0] < w) & (uv[:, 1] >= 0) & (uv[:, 1] < h)
                seen = (inside & (depth >= NEAR_DISTANCE)).sum(0) / n_cams
                too_close = (inside & (depth < NEAR_DISTANCE)).any(0)
                self.count_grid[c, idx] = seen
                self.density_grid[c, idx] = torch.where((seen > 0) & ~too_close, 0.0, -1.0)

    def _cascade_extent(self, c):
        """half extent of cascade c and half a cell of it (reference networks.py:250-251)"""
        s = min(2 ** (c - 1), self.scale)
        return s, s / self.grid_size

    @torch.no_grad()
    def update_density_grid(self, density_threshold, warmup=False, decay=0.95, erode=False):
        """Occupancy refresh, semantics of reference networks.py:240-269: evaluate sigma at one jittered
        point inside every selected cell, grid = max(grid*decay, sigma) except cells marked -1, then
        threshold at min(mean of positive cells, density_threshold) and pack to bits."""
        G = self.grid_size
        fresh = torch.zeros_like(self.density_grid)
        cells = self.get_all_cells() if warmup else self.sample_uniform_and_occupied_cells(G ** 3 // 4, density_threshold)
        for c, (indices, coords) in enumerate(cells):
            s, half_cell = self._cascade_extent(c)
            centers = (coords / (G - 1) * 2 - 1) * (s - half_cell)
            jitter = (torch.rand_like(centers) * 2 - 1) * half_cell
            fresh[c, indices] = self.density(centers + jitter)
        if erode:
            if not hasattr(self, 'count_grid'):
                raise RuntimeError("erode=True needs count_grid (camera coverage); not provided on this path")
            decay = torch.clamp(decay ** (1 / self.count_grid), 0.1, 0.95)
        grid = self.density_grid
        self.density_grid = torch.where(grid < 0, grid, torch.maximum(grid * decay, fresh))
        mean_density = self.density_grid[self.density_grid > 0].mean().item()
        vren.packbits(self.density_grid, min(mean_density, density_threshold), self.density_bitfield)
