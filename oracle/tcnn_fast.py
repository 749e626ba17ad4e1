"""Performance-grade stand-in for `tinycudann` -- TEST / BASELINE INFRASTRUCTURE ONLY (never imported by ngp_pl_b200/).

`oracle/tcnn_standin.py` is the CHECKER: a per-level / per-corner Python loop with double-precision positions, int64
modulo and fp32 `F.linear`, written to be read against tinycudann's published algorithm, and slow.
Timing the reference arm with it under-states what the reference's csrc + tinycudann path does, so `bench.py --impl
reference` runs THIS module instead: the same three classes, the same parameter layout, seeds and fp16 rounding points,
written the way one writes fast eager PyTorch on a GPU:

  * hash grid: ONE vectorised (n, L, 8) int32 index tensor (hashed levels by `&` with the power-of-two mask, dense levels
    by one conditional subtract; no int64, no `%`, no `.double()`), ONE gather from the fp16 table, ONE weighted sum;
    a `torch.autograd.Function` whose backward is ONE `index_add_` into an fp32 table gradient;
  * SH-4: closed form in fp32, fp16 out;
  * MLPs: fp16 cuBLAS GEMMs (fp32 accumulate) on fp16 activations, as tinycudann's FullyFusedMLP computes.

`tests/test_tcnn_fast_gpu.py` holds it to the checker (outputs to fp16 resolution, parameter gradients to 2 % of max).
It is still a stand-in: tinycudann's fused kernels avoid the (n, L, 8) intermediates this materialises in HBM, so the
real reference is faster than this arm -- the ratio `bench.py` reports against it is an UPPER bound on the true one.
"""
import math

import torch
from torch import nn

from . import oracle as _o

_BUCKET = 32768


def _pad_rows(x):
    """Pad the batch to a multiple of 32768 rows (tinycudann pads to its batch granularity too). The sample count of a
    training step changes every step; without the padding every GEMM sees a new M and cuBLAS(Lt) re-runs its algorithm
    heuristics on the host on every call, which made the arm host-bound."""
    n = x.shape[0]
    nb = (n + _BUCKET - 1) // _BUCKET * _BUCKET
    return x if nb == n else torch.nn.functional.pad(x, (0, 0, 0, nb - n))


_P1 = 2654435761 - (1 << 32)  # the hash primes as int32 bit patterns (two's-complement wraparound = uint32 arithmetic)
_P2 = 805459861


class _GridTables:
    """per-level constants as device tensors, built once per (module, device)"""

    def __init__(self, meta, device):
        L = meta.n_levels
        i32 = dict(dtype=torch.int32, device=device)
        self.L = L
        self.scale = torch.tensor([meta.scale[l] for l in range(L)], dtype=torch.float32, device=device)
        self.res = torch.tensor([meta.res[l] for l in range(L)], **i32)
        self.offset = torch.tensor([meta.offset[l] for l in range(L)], **i32)
        entries = [meta.offset[l + 1] - meta.offset[l] for l in range(L)]
        self.entries = torch.tensor(entries, **i32)
        hashed = [(meta.hashed_mask >> l) & 1 for l in range(L)]
        for l in range(L):
            assert not hashed[l] or entries[l] & (entries[l] - 1) == 0, "hashed levels have power-of-two sizes"
        self.hashed = torch.tensor(hashed, dtype=torch.bool, device=device)
        self.mask = torch.tensor([e - 1 for e in entries], **i32)
        c = torch.arange(8, device=device)
        self.corner = torch.stack([c & 1, (c >> 1) & 1, (c >> 2) & 1], 1).to(torch.int32)  # (8, 3)
        self.cornerb = self.corner.bool()


def _grid_indices_weights(T, x01):
    """x01 (n,3) fp32 -> idx (n,L,8) int32 into the flat table, wts (n,L,8) fp32"""
    pos = torch.addcmul(x01.new_full((1, 1, 1), 0.5), x01[:, None, :], T.scale[None, :, None])  # fma(scale, x, 0.5)
    g = torch.floor(pos)
    w = pos - g                                            # (n, L, 3)
    p = g.to(torch.int32)[:, :, None, :] + T.corner[None, None]   # (n, L, 8, 3)
    px, py, pz = p[..., 0], p[..., 1], p[..., 2]
    res = T.res[None, :, None]
    dense = px + py * res + pz * (res * res)
    dense = torch.where(dense >= T.entries[None, :, None], dense - T.entries[None, :, None], dense)
    hashed = (px ^ (py * _P1) ^ (pz * _P2)) & T.mask[None, :, None]
    idx = torch.where(T.hashed[None, :, None], hashed, dense) + T.offset[None, :, None]
    w1 = w[:, :, None, :]
    wsel = torch.where(T.cornerb[None, None], w1, 1.0 - w1)   # (n, L, 8, 3)
    wts = wsel[..., 0] * wsel[..., 1] * wsel[..., 2]
    return idx, wts


class _GridEncode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x01, table_h, T):
        idx, wts = _grid_indices_weights(T, x01)
        vals = table_h[idx.reshape(-1)].view(idx.shape[0], T.L, 8, 2)       # ONE fp16 gather
        feat = (vals.float() * wts[..., None]).sum(2)                        # fp32 accumulate (n, L, 2)
        ctx.save_for_backward(idx, wts)
        ctx.n_entries = table_h.shape[0]
        return feat.reshape(idx.shape[0], 2 * T.L).half()

    @staticmethod
    def backward(ctx, dfeat):
        idx, wts = ctx.saved_tensors
        n, L = idx.shape[0], idx.shape[1]
        contrib = wts[..., None] * dfeat.float().view(n, L, 1, 2)            # (n, L, 8, 2)
        dtable = torch.zeros(ctx.n_entries, 2, dtype=torch.float32, device=dfeat.device)
        dtable.index_add_(0, idx.reshape(-1), contrib.reshape(-1, 2))        # ONE scatter-add
        return None, dtable, None


class NetworkWithInputEncoding(nn.Module):
    def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, seed=1337):
        super().__init__()
        e = encoding_config
        self.meta, self.n_entries = _o.grid_meta(int(e["n_levels"]), int(e["log2_hashmap_size"]), int(e["base_resolution"]),
                                                 float(torch.tensor(float(e["per_level_scale"]), dtype=torch.float32)))
        self.n_levels = int(e["n_levels"])
        g = torch.Generator().manual_seed(seed)
        p = torch.empty(3072 + 2 * self.n_entries)
        p[:2048].uniform_(-math.sqrt(6 / 96), math.sqrt(6 / 96), generator=g)
        p[2048:3072].uniform_(-math.sqrt(6 / 80), math.sqrt(6 / 80), generator=g)
        p[3072:].uniform_(-1e-4, 1e-4, generator=g)
        self.params = nn.Parameter(p)
        self._tables = None

    def _T(self, device):
        if self._tables is None or self._tables.scale.device != device:
            self._tables = _GridTables(self.meta, device)
        return self._tables

    def forward(self, x01):
        with torch.autocast("cuda", enabled=False):
            ph = self.params.half()                     # tinycudann casts its fp32 master parameters every forward
            feat = _GridEncode.apply(x01.float(), ph[3072:].view(-1, 2), self._T(x01.device))
            if self.n_levels < 16:
                feat = torch.nn.functional.pad(feat, (0, 32 - 2 * self.n_levels))
            n = feat.shape[0]
            hid = torch.relu(_pad_rows(feat) @ ph[:2048].view(64, 32).t())
            return (hid @ ph[2048:3072].view(16, 64).t())[:n]


class Encoding(nn.Module):
    def __init__(self, n_input_dims, encoding_config):
        super().__init__()
        self.params = nn.Parameter(torch.zeros(0))

    def forward(self, u):
        with torch.autocast("cuda", enabled=False):
            return _o.torch_sh4(u.float() * 2 - 1).half()


class Network(nn.Module):
    def __init__(self, n_input_dims, n_output_dims, network_config, seed=1338):
        super().__init__()
        self.n_in, self.n_out = n_input_dims, n_output_dims
        self.sigmoid = network_config.get("output_activation", "None") == "Sigmoid"
        g = torch.Generator().manual_seed(seed)
        p = torch.empty(7168)
        p[:2048].uniform_(-math.sqrt(6 / 96), math.sqrt(6 / 96), generator=g)
        p[2048:6144].uniform_(-math.sqrt(6 / 128), math.sqrt(6 / 128), generator=g)
        p[6144:].uniform_(-math.sqrt(6 / 80), math.sqrt(6 / 80), generator=g)
        self.params = nn.Parameter(p)

    def forward(self, x):
        with torch.autocast("cuda", enabled=False):
            ph = self.params.half()
            n = x.shape[0]
            r1 = torch.relu(_pad_rows(x.half()) @ ph[:2048].view(64, 32).t())
            r2 = torch.relu(r1 @ ph[2048:6144].view(64, 64).t())
            out = (r2 @ ph[6144:].view(16, 64).t())[:n, :self.n_out]
            if self.sigmoid:
                out = torch.sigmoid(out.float()).half()
            return out
