"""tinycudann-shaped modules for the three networks reference models/networks.py:36-77 builds.

    import ngp_pl_b200.tcnn as tcnn       # instead of `import tinycudann as tcnn`

Same constructor signatures, one flat fp32 `params` Parameter per module laid out as tinycudann lays
it out (NetworkWithInputEncoding: [network | encoding]; matrices row-major (out, in)), fp16 outputs.
The arithmetic runs in libngp_b200.so; there is no PyTorch fallback. tinycudann itself is absent from
/root/reference, so the semantics follow its published algorithm (SURVEY.md Appendix A; unpinned).

Supported configurations = what the reference's hot path instantiates:
  * NetworkWithInputEncoding(3, 16, HashGrid{L<=16, F=2, T, N_min, b, Linear}, FullyFusedMLP{64, 1 hidden, ReLU, None})
  * Encoding(3, SphericalHarmonics{degree 4})
  * Network(32, 3, FullyFusedMLP{64, 2 hidden, ReLU, Sigmoid|None})
(The HDR tonemapper networks of networks.py:79-92 are outside the hot path.)
"""
import ctypes as C
import math

import torch
from torch import nn
from torch.amp import custom_bwd, custom_fwd

from . import _lib


def _st():
    return torch.cuda.current_stream().cuda_stream


class _HalfCopy:
    """fp16 working copy of an fp32 parameter vector. tinycudann re-casts its parameters on every forward; so does this
    whenever the parameter can have changed behind autograd's back: the modules call `training_forward()` at the top of
    every forward that runs with grad mode on and a parameter that requires grad (an optimiser that writes through `p.data`
    -- apex FusedAdam, the reference's choice at train.py:128-134 -- or an EMA swap does NOT bump `p._version`); otherwise
    (inference) the copy is refreshed only when (pointer, version) changed."""

    def __init__(self):
        self.buf = None
        self.key = None

    def invalidate(self):
        self.key = None

    def training_forward(self, p):
        """called OUTSIDE the autograd.Function (grad mode is off inside Function.forward): re-cast if this is a training forward"""
        if p.requires_grad and torch.is_grad_enabled():
            self.key = None

    def get(self, p):
        key = (p.data_ptr(), p._version, p.device)
        if self.buf is None or self.buf.device != p.device or self.buf.numel() != p.numel():
            self.buf = torch.empty(p.numel(), device=p.device, dtype=torch.float16)
            self.key = None
        if key != self.key:
            with torch.cuda.device(p.device):
                _lib.check(_lib.lib().ngp_cast_params(p.data_ptr(), self.buf.data_ptr(), p.numel(), _st()), "cast_params")
            self.key = key
        return self.buf


class _FixedHalf:
    """fp16 working copy owned by someone else (the Trainer's flat buffer, refreshed by its Adam kernel; after an outside
    write to the fp32 parameters -- load_state_dict, p.data.copy_ -- call Trainer.sync_params())"""

    def __init__(self, buf):
        self.buf = buf

    def invalidate(self):
        pass

    def training_forward(self, p):
        pass

    def get(self, p):
        return self.buf


class Encoding(nn.Module):
    """tcnn.Encoding(n_input_dims=3, {"otype": "SphericalHarmonics", "degree": 4}); reference networks.py:58-65.
    Parameter-free (empty `params`, as in tinycudann)."""

    def __init__(self, n_input_dims, encoding_config, dtype=torch.float16):
        super().__init__()
        if encoding_config.get("otype") != "SphericalHarmonics" or int(encoding_config.get("degree", 4)) != 4 \
                or n_input_dims != 3:
            raise NotImplementedError("only the degree-4 spherical-harmonics encoding of the hot path is provided")
        self.n_input_dims = 3
        self.n_output_dims = 16
        self.params = nn.Parameter(torch.zeros(0, dtype=torch.float32))

    def forward(self, x):
        from .models.networks import need_cuda, sh_encode
        need_cuda(x, "tcnn.Encoding")
        return sh_encode(x)


def _xavier_uniform_(t, fan_out, fan_in):
    bound = math.sqrt(6.0 / (fan_in + fan_out))
    return t.uniform_(-bound, bound)


class NetworkWithInputEncoding(nn.Module):
    """tcnn.NetworkWithInputEncoding(3, 16, grid_config, mlp_config); reference networks.py:36-56."""

    def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, seed=1337):
        super().__init__()
        e, n = encoding_config, network_config
        if n_input_dims != 3 or n_output_dims != 16:
            raise NotImplementedError("hot path uses n_input_dims=3, n_output_dims=16")
        if e.get("otype") not in ("Grid", "HashGrid") or e.get("type", "Hash") != "Hash" or \
                int(e.get("n_features_per_level", 2)) != 2 or e.get("interpolation", "Linear") != "Linear":
            raise NotImplementedError("hash grid with F=2 and linear interpolation only")
        if int(n.get("n_neurons", 64)) != 64 or int(n.get("n_hidden_layers", 1)) != 1 or \
                n.get("activation", "ReLU") != "ReLU" or n.get("output_activation", "None") != "None":
            raise NotImplementedError("density MLP is 32->64(ReLU)->16")
        self.n_levels = int(e["n_levels"])
        self.log2_hashmap_size = int(e["log2_hashmap_size"])
        self.base_resolution = int(e["base_resolution"])
        self.per_level_scale = float(e["per_level_scale"])
        self.n_input_dims, self.n_output_dims = 3, 16
        self.meta, self.n_entries = _lib.grid_meta(self.n_levels, self.log2_hashmap_size, self.base_resolution,
                                                   self.per_level_scale)
        g = torch.Generator().manual_seed(seed)
        p = torch.empty(_lib.NGP_DENSITY_MLP_PARAMS + 2 * self.n_entries, dtype=torch.float32)
        p[:2048].uniform_(-math.sqrt(6.0 / (32 + 64)), math.sqrt(6.0 / (32 + 64)), generator=g)
        p[2048:3072].uniform_(-math.sqrt(6.0 / (64 + 16)), math.sqrt(6.0 / (64 + 16)), generator=g)
        p[3072:].uniform_(-1e-4, 1e-4, generator=g)
        self.params = nn.Parameter(p)
        self._half = _HalfCopy()

    def half_params(self):
        return self._half.get(self.params)

    def forward(self, x):
        """x in [0,1]^3 (N,3) -> fp16 (N,16). Differentiable w.r.t. params."""
        from .models.networks import _DensityFeatures, need_cuda
        need_cuda(x, "tcnn.NetworkWithInputEncoding")
        self._half.training_forward(self.params)
        return _DensityFeatures.apply(x, self.params, self)


class Network(nn.Module):
    """tcnn.Network(32, 3, mlp_config); reference networks.py:67-77."""

    def __init__(self, n_input_dims, n_output_dims, network_config, seed=1338):
        super().__init__()
        n = network_config
        if n_input_dims != 32 or n_output_dims != 3:
            raise NotImplementedError("hot path uses the 32 -> 3 rgb network")
        if int(n.get("n_neurons", 64)) != 64 or int(n.get("n_hidden_layers", 2)) != 2 or n.get("activation", "ReLU") != "ReLU":
            raise NotImplementedError("rgb MLP is 32->64->64->3")
        act = n.get("output_activation", "Sigmoid")
        if act not in ("Sigmoid", "None"):
            raise NotImplementedError("output activation Sigmoid or None")
        self.rgb_act = 1 if act == "Sigmoid" else 0
        self.n_input_dims, self.n_output_dims = 32, 3
        g = torch.Generator().manual_seed(seed)
        p = torch.empty(_lib.NGP_RGB_MLP_PARAMS, dtype=torch.float32)
        p[:2048].uniform_(-math.sqrt(6.0 / (32 + 64)), math.sqrt(6.0 / (32 + 64)), generator=g)
        p[2048:6144].uniform_(-math.sqrt(6.0 / (64 + 64)), math.sqrt(6.0 / (64 + 64)), generator=g)
        p[6144:].uniform_(-math.sqrt(6.0 / (64 + 16)), math.sqrt(6.0 / (64 + 16)), generator=g)
        self.params = nn.Parameter(p)
        self._half = _HalfCopy()

    def half_params(self):
        return self._half.get(self.params)

    def forward(self, x):
        from .models.networks import _RgbMlp, need_cuda
        need_cuda(x, "tcnn.Network")
        self._half.training_forward(self.params)
        return _RgbMlp.apply(x, self.params, self)
