"""The level-major hash-table gradient scatter against the float64 scatter of oracle/grad64.py.

k_grid_scatter_merged takes work items -- a chunk of 256 consecutive samples x a group of levels -- from a device ticket
counter, every chunk of one group before the next group. Only the order of the fp32 reductions may differ from the
float64 sum, so each entry is held to twice the rigorous bound (m_e + 2) 2^-24 sum |contribution_e| of test_backward_fp64
(m_e = the entry's number of contributions), and so are two launches against each other. Entries no sample touches stay
exactly 0. Cases: a Trainer's live batch; counts around a warp and off the chunk; fewer than 16 levels and dense levels
only; the xyzs and the ray layouts, with and without a live list; and a count at which the ticket loop turns several
times for any grid of at most 8 CTAs per SM.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import grad64

pytestmark = pytest.mark.gpu

SCALE = 2.0 ** 5


def _L():
    from ngp_pl_b200 import _lib
    return _lib.lib()


def _chk(rc, what):
    from ngp_pl_b200 import _lib
    _lib.check(rc, what)


def _meta(n_levels, log2_T, base=16, scale_max=2048 * 0.5):
    from ngp_pl_b200 import _lib
    b = float(np.exp(np.log(scale_max / base) / max(n_levels - 1, 1)))
    return _lib.grid_meta(n_levels, log2_T, base, b)


def _net(meta, lo=(0.0, 0.0, 0.0), hi=(1.0, 1.0, 1.0)):
    from ngp_pl_b200 import _lib
    net = _lib.NgpNet()
    net.meta = meta
    for k in range(3):
        net.xyz_min[k], net.xyz_max[k] = lo[k], hi[k]
    net.rgb_act = 1
    return net


def _workspace(cap, seed):
    """feature gradients of every (level, row) slot: random fp16, level-major with stride ceil16(cap)"""
    ws = torch.empty(_L().ngp_net_backward_workspace(cap), device="cuda", dtype=torch.uint8)
    stride = (cap + 15) // 16 * 16
    g = torch.Generator(device="cuda").manual_seed(seed)
    ws[:16 * stride * 4].view(torch.float16).copy_((torch.randn(16 * stride * 2, device="cuda", generator=g) * 30).half())
    return ws


def _dfeat(ws, cap, n):
    """(n, 32) fp16, column 2 level + f: the feature gradients of visit positions 0 .. n"""
    stride = (cap + 15) // 16 * 16
    return ws[:16 * stride * 4].view(torch.float16).view(16, stride, 2)[:, :n].permute(1, 0, 2).reshape(n, 32)


def _scatter(net, smp, ws, total):
    st = torch.tensor([SCALE], device="cuda")
    ge = torch.zeros(3072 + 2 * total, device="cuda")
    _chk(_L().ngp_net_backward_scatter(C.byref(net), C.byref(smp), st.data_ptr(), ge.data_ptr(), ws.data_ptr(), ws.numel(),
                                       torch.cuda.current_stream().cuda_stream), "scatter")
    torch.cuda.synchronize()
    return ge


def _check(net, smp, ws, cap, x01, total):
    """x01: (n, 3) float32, the unit-cube positions of the samples the launch visits, in visit order"""
    n = x01.shape[0]
    ref, Sabs, m = grad64.grid_scatter(net.meta, x01, _dfeat(ws, cap, n), 1.0 / SCALE, total)
    tol = 2 * (m[:, None] + 2) * 2.0 ** -24 * Sabs
    untouched = m == 0
    outs = [_scatter(net, smp, ws, total) for _ in range(2)]
    for ge in outs:
        got = ge[3072:].view(-1, 2).double()
        assert ge[:3072].abs().max() == 0
        assert torch.isfinite(got).all()
        bad = (got - ref).abs() > tol
        assert not bad.any(), "%d table entries off, worst %g" % (int(bad.sum()), float(((got - ref).abs() - tol).max()))
        assert (got[untouched] == 0).all()
    a, b = (ge[3072:].view(-1, 2).double() for ge in outs)
    assert ((a - b).abs() <= tol).all()
    assert (~untouched).any()


def _ray_batch(n_rays, cap, rng):
    """rays through the unit cube sampled at small steps, ray after ray (runs of equal cells at the coarse levels)"""
    o = rng.uniform(0.3, 0.7, (n_rays, 3))
    d = rng.normal(size=(n_rays, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    per = rng.randint(1, 2 * cap // n_rays + 2, n_rays)
    ridx = np.repeat(np.arange(n_rays), per)[:cap]
    ridx = np.concatenate([ridx, rng.randint(0, n_rays, cap - len(ridx))])
    step = 10 ** rng.uniform(-4, -2, n_rays)
    first = np.r_[0, np.flatnonzero(np.diff(ridx)) + 1]
    k = np.arange(cap) - np.repeat(first, np.diff(np.r_[first, cap]))
    ts = np.minimum(k * step[ridx], 0.25).astype(np.float32)
    return o.astype(np.float32), d.astype(np.float32), ridx.astype(np.int32), ts


# (n_levels, log2_T, rows visited, layout, live list); "dense_only" runs its 3 levels at scales 15, 31 and 63
CASES = {
    "n1": (16, 19, 1, "xyzs", False),
    "n31_rays": (16, 19, 31, "rays", False),
    "n33_live": (16, 19, 33, "xyzs", True),
    "off_chunk_rays_live": (16, 19, 256 * 37 + 77, "rays", True),
    "L11": (11, 19, 256 * 20 + 5, "xyzs", False),
    "dense_only": (3, 19, 256 * 9 + 13, "rays", False),
    "loops_xyzs": (16, 19, None, "xyzs", False),
    "loops_rays_live": (16, 19, None, "rays", True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_scatter_vs_float64(case):
    from ngp_pl_b200 import _lib
    n_levels, log2_T, n, layout, live = CASES[case]
    S = torch.cuda.get_device_properties(0).multi_processor_count
    if n is None:
        n = S * 8 * 256 + 4321  # more 256-sample chunks per level than 8 CTAs per SM take in one turn
    meta, total = _meta(n_levels, log2_T, scale_max=64) if case == "dense_only" else _meta(n_levels, log2_T)
    if case == "dense_only":
        assert meta.hashed_mask == 0
    else:
        assert meta.hashed_mask != 0
    net = _net(meta)
    rng = np.random.RandomState(sum(map(ord, case)))
    cap = n + n // 3 + 50 if live else n
    smp = _lib.NgpSamples()
    smp.n = cap
    if layout == "xyzs":
        o, d, ridx, ts = _ray_batch(max(cap // 40, 1), cap, rng)
        x = torch.as_tensor((d[ridx].astype(np.float64) * ts[:, None] + o[ridx]).astype(np.float32)).cuda()
        x[torch.as_tensor(rng.randint(0, cap, cap // 50 + 1)).cuda()] = torch.tensor([1.0, 0.0, 1 - 2 ** -24], device="cuda")
        keep = [x]
        smp.xyzs = x.data_ptr()
        x01 = x
    else:
        o, d, ridx, ts = _ray_batch(max(cap // 40, 1), cap, rng)
        keep = [torch.as_tensor(a).cuda() for a in (o, d, ridx, ts)]
        smp.rays_o, smp.rays_d, smp.ray_idx, smp.ts = (t.data_ptr() for t in keep)
        # the kernel's x = fma(d, t, o): the double product is exact
        x01 = torch.as_tensor((d[ridx].astype(np.float64) * ts[:, None] + o[ridx]).astype(np.float32)).cuda()
    if live:
        g = torch.Generator(device="cuda").manual_seed(5)
        live_full = torch.randperm(cap, device="cuda", generator=g)[:n + 40].to(torch.int32).contiguous()
        n_live = torch.tensor([n], device="cuda", dtype=torch.int32)
        keep += [live_full, n_live]
        smp.live_idx, smp.n_live_dev = live_full.data_ptr(), n_live.data_ptr()
        x01 = x01[live_full[:n].long()]
    ws = _workspace(cap, 11)
    _check(net, smp, ws, cap, x01.contiguous(), total)


def test_trainer_live_batch_vs_float64():
    """the positions and the live list of a Trainer's step: ray-ordered samples of a real march"""
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(0)
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=8, device="cuda", seed=3)
    tr = Trainer(NGP(scene.scale).cuda(), n_rays=8192, update_interval=1 << 30)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(20):
        tr.train_step()
    torch.cuda.synchronize()
    smp = _lib.NgpSamples()
    smp.rays_o, smp.rays_d = tr.rays_o.data_ptr(), tr.rays_d.data_ptr()
    smp.ray_idx, smp.ts = tr.ray_idx.data_ptr(), tr.ts.data_ptr()
    smp.n, smp.n_dev = tr.capacity, tr.counters[2:].data_ptr()
    smp.live_idx, smp.n_live_dev = tr.live_idx.data_ptr(), tr.counters[5:].data_ptr()
    n = int(tr.counters[5])
    assert 1000 < n <= tr.capacity
    rows = tr.live_idx[:n].long()
    r = tr.ray_idx[rows].long()
    x = (tr.rays_d[r].double() * tr.ts[rows].double()[:, None] + tr.rays_o[r].double()).float().cpu()
    lo = torch.tensor(list(tr.net.xyz_min), dtype=torch.float32)
    hi = torch.tensor(list(tr.net.xyz_max), dtype=torch.float32)
    x01 = ((x - lo) / (hi - lo)).cuda()  # to_unit: an fp32 subtract, then a correctly rounded fp32 divide
    net = _lib.NgpNet.from_buffer_copy(tr.net)
    total = int(net.meta.offset[net.meta.n_levels])
    ws = _workspace(tr.capacity, 12)
    _check(net, smp, ws, tr.capacity, x01, total)
