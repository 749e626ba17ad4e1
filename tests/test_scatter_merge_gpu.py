"""The hash-table gradient scatter's corner hand-overs on the device, against the float64 scatter of oracle/grad64.py.

k_grid_scatter_merged sums runs of equal cells into their head and hands the corners a head shares with the next run's
adjacent cell to that run's head (tests/test_scatter_merge_algorithm_cpu.py replays the rule). The samples here are
rays marched along the axes (consecutive cells share a face), along the diagonals of a plane (an edge) and of space (a
vertex), and in random directions, at steps from a fraction of the finest cell to more than the coarsest, so that every
level sees runs, each kind of adjacency and jumps; half the axis-aligned and diagonal rays start with equal coordinates,
so that along (1, 1, 0) and (1, 1, 1) every crossing is exactly an edge or a vertex. Only the order of the fp32 sums may differ from the float64 sum: each entry is held to twice the
bound (m_e + 2) 2^-24 sum |contribution_e| of test_scatter_order_gpu (m_e = the entry's number of contributions), and
entries no sample touches stay exactly 0.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import grad64

pytestmark = pytest.mark.gpu

SCALE = 2.0 ** 5
DIRS = {"face": [(1, 0, 0), (0, -1, 0), (0, 0, 1)], "edge": [(1, 1, 0), (0, -1, 1), (-1, 0, -1)],
        "vertex": [(1, 1, 1), (-1, 1, -1), (1, -1, -1)]}


def _lib():
    from ngp_pl_b200 import _lib as L
    return L


def _meta(n_levels, log2_T, base=16, scale_max=2048 * 0.5):
    b = float(np.exp(np.log(scale_max / base) / max(n_levels - 1, 1)))
    return _lib().grid_meta(n_levels, log2_T, base, b)


def _rays(kinds, n, rng):
    """n positions, ray after ray: each ray takes a direction of one of `kinds` (or a random one), a step between 1e-4 and
    0.06 and 8 to 300 samples, from a point of the 1/1024 lattice near the centre"""
    out = []
    total = 0
    while total < n:
        kind = kinds[rng.randint(len(kinds))]
        d = np.array(DIRS[kind][rng.randint(3)] if kind != "random" else rng.normal(size=3), np.float64)
        d /= np.abs(d).max()  # axis steps equal: the diagonal rays cross every axis's planes together
        step = 10 ** rng.uniform(-4, np.log10(0.06))
        k = rng.randint(8, 301)
        o = np.round(rng.uniform(0.35, 0.65, 3) * 1024) / 1024
        if kind != "random" and rng.rand() < 0.5:
            o[:] = o[0]  # along (1, 1, 0) and (1, 1, 1) the coordinates stay equal: every crossing is an edge / a vertex
        x = o + np.outer(np.arange(k) * step, d)
        x = x[(x >= 0).all(1) & (x < 1).all(1)]
        out.append(x)
        total += len(x)
    return np.concatenate(out)[:n].astype(np.float32)


def _scatter(net, smp, ws, total):
    st = torch.tensor([SCALE], device="cuda")
    ge = torch.zeros(3072 + 2 * total, device="cuda")
    _lib().check(_lib().lib().ngp_net_backward_scatter(C.byref(net), C.byref(smp), st.data_ptr(), ge.data_ptr(),
                                                       ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream),
                 "scatter")
    torch.cuda.synchronize()
    return ge


@pytest.mark.parametrize("kinds,n,live", [
    (("face",), 256 * 40 + 3, False), (("edge",), 256 * 40 + 17, False), (("vertex",), 256 * 40 + 29, False),
    (("face", "edge", "vertex", "random"), 256 * 300 + 77, False), (("face", "edge", "vertex", "random"), 256 * 50 + 5, True)])
def test_adjacent_cells_vs_float64(kinds, n, live):
    L = _lib()
    meta, total = _meta(16, 19)
    net = L.NgpNet()
    net.meta = meta
    for k in range(3):
        net.xyz_min[k], net.xyz_max[k] = 0.0, 1.0
    net.rgb_act = 1
    rng = np.random.RandomState(n)
    x01 = _rays(list(kinds), n, rng)
    cap = n + n // 4 + 40 if live else n
    xs = np.concatenate([x01, rng.uniform(0, 1, (cap - n, 3)).astype(np.float32)])
    if live:  # row s of the visit order is position live[s]: scatter the ray order into a shuffled buffer
        perm = rng.permutation(cap).astype(np.int32)
        buf = np.empty_like(xs)
        buf[perm] = xs
        xs = buf
    x = torch.as_tensor(xs).cuda()
    smp = L.NgpSamples()
    smp.n = cap
    smp.xyzs = x.data_ptr()
    keep = [x]
    if live:
        live_idx = torch.as_tensor(perm).cuda()
        n_live = torch.tensor([n], device="cuda", dtype=torch.int32)
        keep += [live_idx, n_live]
        smp.live_idx, smp.n_live_dev = live_idx.data_ptr(), n_live.data_ptr()
    ws = torch.empty(L.lib().ngp_net_backward_workspace(cap), device="cuda", dtype=torch.uint8)
    stride = (cap + 15) // 16 * 16
    g = torch.Generator(device="cuda").manual_seed(n)
    ws[:16 * stride * 4].view(torch.float16).copy_((torch.randn(16 * stride * 2, device="cuda", generator=g) * 30).half())
    dfeat = ws[:16 * stride * 4].view(torch.float16).view(16, stride, 2)[:, :n].permute(1, 0, 2).reshape(n, 32)
    ref, Sabs, m = grad64.grid_scatter(meta, torch.as_tensor(x01).cuda(), dfeat, 1.0 / SCALE, total)
    tol = 2 * (m[:, None] + 2) * 2.0 ** -24 * Sabs
    untouched = m == 0
    ge = _scatter(net, smp, ws, total)
    got = ge[3072:].view(-1, 2).double()
    assert ge[:3072].abs().max() == 0
    assert torch.isfinite(got).all()
    bad = (got - ref).abs() > tol
    assert not bad.any(), "%d table entries off, worst %g" % (int(bad.sum()), float(((got - ref).abs() - tol).max()))
    assert (got[untouched] == 0).all()
    assert (~untouched).any()
