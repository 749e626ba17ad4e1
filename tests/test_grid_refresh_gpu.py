"""The occupancy-grid refresh (ngp_update_density_grid_pick + _eval, csrc/train.cu) cell by cell against the numpy
restatement in oracle/grid_refresh.py, which tests/test_grid_refresh_cpu.py holds to independent facts.

Each case runs one refresh and reads cell_idx, xyz, tot, tmp and stats back from the workspace (offsets as grid_ws()
lays them out). Bitwise: the distinct cells of every cascade and their slot bases, the jittered points, the scattered
sigma (model.density at the restated points -- test_forward_fp64_gpu.py pins that kernel, and its rows do not depend on
the launch shape), the merged grid without erode and the bitfield at fminf(thr, mean). Bounded: the merged grid with
erode and the mean, each within twice its derived bound; against the float64 threshold only cells within that band may
change sides. Every input is seeded, so each case computes one fixed answer."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import grid_refresh as R
from test_fused_gpu import make_model

pytestmark = pytest.mark.gpu

EINVAL = -22
THR = 0.01 * 1024 / 3 ** 0.5  # the Trainer's default density threshold


def _al256(v):
    return (v + 255) & ~255


class Ws:
    """typed views of the refresh workspace, mirroring grid_ws() in train.cu"""

    def __init__(self, ws, cascades, G):
        g3 = G ** 3
        off = 0

        def take(nbytes):
            nonlocal off
            o = off
            off += _al256(nbytes)
            return o
        o_tmp = take(cascades * g3 * 4)
        take(g3)                 # flags
        take(g3 * 4)             # occ_list
        take(256)                # occ_count
        o_cell = take(cascades * g3 * 4)
        o_xyz = take(cascades * g3 * 12)
        take(cascades * g3 * 4)  # sigma
        o_stats = take(256)
        take(R.MERGE_MAX_BLOCKS * 4)
        take(R.MERGE_MAX_BLOCKS * 4)
        o_tot = take(256)
        take(g3 * 4)             # keys (distinct)
        o_sorted = take(g3 * 4)
        host = ws.cpu()

        def view(o, n, dt):
            return host[o:o + n * 4].view(dt).numpy()
        self.tmp = view(o_tmp, cascades * g3, torch.float32).reshape(cascades, g3)
        self.cell_idx = view(o_cell, cascades * g3, torch.int32)
        self.xyz = view(o_xyz, cascades * g3 * 3, torch.float32).reshape(-1, 3)
        self.stats = view(o_stats, 4, torch.float32)
        self.tot = view(o_tot, 64, torch.int32)
        self.keys_sorted = view(o_sorted, 2 * (g3 // 4), torch.int32).view(np.uint32)


def _lib():
    from ngp_pl_b200 import _lib as L
    return L, L.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _model(scale, seed=0):
    """an NGP of this scale with a random hash table (as make_model draws it)"""
    from ngp_pl_b200.models.networks import NGP
    m = NGP(scale).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        p = m.xyz_encoder.params
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * 0.3).cuda()
    return m


def refresh(model, grid, G, thr, warmup, decay, seed, count=None):
    """one direct-ABI refresh of `grid` (cascades, G^3) in place; returns (bitfield, workspace)"""
    from ngp_pl_b200.models.networks import _net_struct
    _, L = _lib()
    cascades = grid.shape[0]
    nbytes = L.ngp_update_grid_workspace(cascades, G)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    bits = torch.zeros(max(cascades * G ** 3 // 8, 1), dtype=torch.uint8, device="cuda")
    net, keep = _net_struct(model)
    rc = L.ngp_update_density_grid_pick(grid.data_ptr(), cascades, G, float(model.scale), float(thr), int(warmup), seed,
                                        ws.data_ptr(), nbytes, _st())
    assert rc == 0
    rc = L.ngp_update_density_grid_eval(C.byref(net), grid.data_ptr(), bits.data_ptr(),
                                        count.data_ptr() if count is not None else None, cascades, G, float(thr),
                                        int(warmup), float(decay), ws.data_ptr(), nbytes, _st())
    assert rc == 0
    torch.cuda.synchronize()
    return bits, ws


def check(model, old, new, bits, ws, G, thr, warmup, decay, seed, count=None):
    """hold one refresh to the restatement; ws=None checks only what the grid and bitfield show. Returns a summary."""
    cascades = old.shape[0]
    g3 = G ** 3
    old = old.cpu().numpy()
    new = new.cpu().numpy()
    bits = bits.cpu().numpy()
    cells, tot = R.cascade_cells(old, thr, seed, G, warmup)
    n = int(tot[-1])
    cidx = R.cell_index(cells, G)
    xyz = R.refresh_points(cells, seed, G, model.scale)
    sig = model.density(torch.from_numpy(xyz).cuda()).cpu().numpy()
    tmp = R.scatter(cidx, sig, (cascades, g3))
    if ws is not None:
        w = Ws(ws, cascades, G)
        assert np.array_equal(w.tot[:cascades + 1], tot), "slot bases tot[c]"
        for c in range(cascades):
            got = w.cell_idx[tot[c]:tot[c + 1]]
            assert np.array_equal(got, cidx[tot[c]:tot[c + 1]]), "distinct cells of cascade %d" % c
        assert np.array_equal(w.xyz[:n].view(np.uint32), xyz.view(np.uint32)), "jittered points"
        assert np.array_equal(w.tmp.view(np.uint32), tmp.view(np.uint32)), "scattered sigma"
    out = dict(distinct=n - sum(int(k[-1] >= g3) for k in cells) if not warmup else n)
    if count is None:
        want = R.merge(old, tmp, decay)
        assert np.array_equal(new.view(np.uint32), want.view(np.uint32)), "merged grid"
    else:
        val, bound = R.merge_erode(old, tmp, count.cpu().numpy(), decay)
        assert np.array_equal(new[old < 0], old[old < 0]), "cells marked -1 stay -1"
        err = np.abs(new.astype(np.float64) - val)
        assert (err <= 2 * bound).all(), "erode grid outside 2x its bound: %g" % (err / np.maximum(2 * bound, 1e-300)).max()
        out["erode_err"] = float((err / np.where(bound > 0, 2 * bound, np.inf)).max())
    m64, mb = R.mean(new, R.merge_blocks(cascades * g3, _sm_count()))
    if ws is not None:  # without the workspace only the band check below sees the mean
        m32 = float(Ws(ws, cascades, G).stats[2])
        if np.isnan(m64):
            assert np.isnan(m32)
        else:
            assert abs(m32 - m64) <= 2 * mb, "mean %r vs float64 %r, bound %g" % (m32, m64, mb)
            out["mean_err"] = abs(m32 - m64) / (2 * mb)
        t32 = R.threshold(thr, m32)
        assert np.array_equal(bits, R.packbits(new, t32)), "bitfield = packbits(grid, fminf(thr, mean))"
    flat = new.reshape(-1).astype(np.float64)
    t64 = min(float(np.float32(thr)), m64) if not np.isnan(m64) else float("nan")
    above64 = flat > t64
    above = np.unpackbits(bits, bitorder="little")[:flat.size].astype(bool)
    band = np.abs(flat - t64) <= 2 * mb if not np.isnan(m64) else np.zeros(flat.size, bool)
    differ = above != above64
    assert not (differ & ~band).any(), "bits outside the threshold band disagree with the float64 threshold"
    out["band"] = int(band.sum())
    out["band_flipped"] = int(differ.sum())
    assert differ.sum() <= 1e-5 * flat.size
    return out


def _seed_grid(grid, thr, rng):
    """-1 cells, cells exactly at thr (not occupied: the test is strict), cells at 0 and cells at 2 thr (occupied, so
    that the occupied half draws from a real list whatever the network's sigma)"""
    n = grid.numel()
    flat = grid.view(-1)
    k = n // 16
    idx = torch.as_tensor(rng.permutation(n)[:4 * k]).cuda()
    flat[idx[:k]] = -1.0
    flat[idx[k:2 * k]] = float(np.float32(thr))
    flat[idx[2 * k:3 * k]] = 0.0
    flat[idx[3 * k:]] = 2 * float(np.float32(thr))


def _report(tag, out):
    print("%s: %s" % (tag, " ".join("%s=%s" % kv for kv in sorted(out.items()))))


# ---------------------------------------------------------------------------------------------------
# the Trainer's refreshes
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["lego", "mip360"])
def test_trainer_refresh_matches_restatement(which):
    """warm-up from a zero grid, then regular refreshes at steps 256 and 272 with pick_ahead: 272 evaluates the pick the
    side stream made at the end of 256, from the grid 256 left"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0) if which == "lego" else synth.mip360_scene(0)
    model = make_model(scene, amp=0.3)
    tr = Trainer(model, n_rays=256, pick_ahead=False)
    G = model.grid_size
    assert model.cascades == (1 if which == "lego" else 6)
    grid = model.density_grid
    grid.zero_()
    tr.host_step = 0
    old = grid.clone()
    tr.update_density_grid(THR, warmup=True)
    torch.cuda.synchronize()
    _report(which + " warm-up", check(model, old, grid, model.density_bitfield, tr.grid_ws, G, THR, True, 0.95,
                                      tr._refresh_seed(0)))
    _seed_grid(grid, THR, np.random.RandomState(1))
    tr.pick_ahead = True
    tr.host_step = 256
    old = grid.clone()
    tr.update_density_grid(THR, warmup=False)
    torch.cuda.synchronize()
    assert tr._picked is not None
    # the pick for 272 is already running over the workspace: only the grid and the bits are this refresh's
    _report(which + " 256", check(model, old, grid, model.density_bitfield, None, G, THR, False, 0.95,
                                  tr._refresh_seed(256)))
    tr.pick_ahead = False
    tr.host_step = 272
    old = grid.clone()
    tr.update_density_grid(THR, warmup=False)
    torch.cuda.synchronize()
    _report(which + " 272", check(model, old, grid, model.density_bitfield, tr.grid_ws, G, THR, False, 0.95,
                                  tr._refresh_seed(272)))


# ---------------------------------------------------------------------------------------------------
# direct ABI, other grid sizes and scales
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cascades,G,scale,decay", [
    (1, 2, 0.5, 0.95), (1, 2, 0.5, 0.5), (2, 4, 1.0, 0.95), (2, 4, 1.0, 0.5), (4, 16, 3.0, 0.95), (4, 16, 3.0, 0.5),
    (1, 256, 0.5, 0.95)])  # G = 256: 25-bit keys over 2^23 slots; scale 3: s capped at a non-power of two
def test_refresh_other_sizes(cascades, G, scale, decay):
    model = _model(scale)
    assert model.cascades == cascades
    grid = torch.zeros(cascades, G ** 3, device="cuda")
    seed = R.refresh_seed(5, 0)
    old = grid.clone()
    bits, ws = refresh(model, grid, G, THR, True, decay, seed)
    _report("C=%d G=%d warm-up" % (cascades, G), check(model, old, grid, bits, ws, G, THR, True, decay, seed))
    # a threshold inside the warm-up's values, so that the occupied half draws from a real list
    pos = grid[grid > 0]
    thr = float(np.float32(pos.float().quantile(0.6).item())) if pos.numel() else THR
    _seed_grid(grid, thr, np.random.RandomState(2))
    for step in (256, 272):
        seed = R.refresh_seed(5, step)
        old = grid.clone()
        bits, ws = refresh(model, grid, G, thr, False, decay, seed)
        _report("C=%d G=%d step %d" % (cascades, G, step), check(model, old, grid, bits, ws, G, thr, False, decay, seed))


def test_occupancy_edges():
    """cascade 0 with no occupied cell (the "none" key), cascade 1 fully occupied; then an all -1 grid: NaN mean,
    threshold = thr, no bit set"""
    model = _model(1.0)
    G = 16
    grid = torch.zeros(2, G ** 3, device="cuda")
    grid[1] = 2 * THR
    seed = R.refresh_seed(9, 300)
    old = grid.clone()
    bits, ws = refresh(model, grid, G, THR, False, 0.95, seed)
    w = Ws(ws, 2, G)
    assert w.cell_idx[w.tot[1] - 1] == -1 and (w.xyz[w.tot[1] - 1] == 0).all()
    _report("edges", check(model, old, grid, bits, ws, G, THR, False, 0.95, seed))
    grid.fill_(-1.0)
    bits, ws = refresh(model, grid, G, THR, False, 0.95, seed)
    st = Ws(ws, 2, G).stats
    assert np.isnan(st[2]) and st[1] == 0
    assert R.threshold(THR, st[2]) == np.float32(THR)
    assert not bits.any() and (grid == -1).all()
    check(model, torch.full_like(grid, -1.0), grid, bits, ws, G, THR, False, 0.95, seed)


def test_erode_against_camera_coverage():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = make_model(scene, amp=0.3)
    tr = Trainer(model, n_rays=256, pick_ahead=False, erode=True)
    G = model.grid_size
    model.register_buffer("grid_coords", torch.stack(torch.meshgrid(
        *[torch.arange(G, dtype=torch.int32, device="cuda")] * 3, indexing="ij"), -1).reshape(-1, 3))
    K = synth.intrinsics(W=80, H=60, fx=100.0)
    Km = torch.tensor([[K["fx"], 0, K["cx"]], [0, K["fy"], K["cy"]], [0, 0, 1]], dtype=torch.float32, device="cuda")
    poses = torch.as_tensor(synth.camera_poses(12, radius=1.2)).float().cuda()
    model.mark_invisible_cells(Km, poses, (K["W"], K["H"]))
    count = model.count_grid
    rng = np.random.RandomState(3)
    n = count.numel()
    idx = torch.as_tensor(rng.permutation(n)[:3000]).cuda()
    flat = count.view(-1)
    flat[idx[:1000]] = 0.0
    flat[idx[1000:2000]] = 1e-30
    flat[idx[2000:]] = 1.0
    grid = model.density_grid
    assert (grid == -1).any() and (grid == 0).any()
    g = torch.Generator("cuda").manual_seed(4)
    grid.copy_(torch.where(grid < 0, grid, torch.rand(grid.shape, device="cuda", generator=g) * 3 * THR))
    for decay in (0.95, 0.5):
        tr.host_step = 512 if decay == 0.95 else 528
        old = grid.clone()
        tr.update_density_grid(THR, warmup=False, decay=decay)
        torch.cuda.synchronize()
        _report("erode %g" % decay, check(model, old, grid, model.density_bitfield, tr.grid_ws, model.grid_size, THR,
                                          False, decay, tr._refresh_seed(tr.host_step), count=count))


# ---------------------------------------------------------------------------------------------------
# distributions (fixed seeds: deterministic)
# ---------------------------------------------------------------------------------------------------
def test_pick_and_jitter_distributions():
    model = _model(0.5)
    G = 32
    g3 = G ** 3
    M = g3 // 4
    # occupied picks: 128 occupied cells, M = 8192 draws; the sorted picks in the workspace are the restated ones
    grid = torch.zeros(1, g3, device="cuda")
    occ = torch.as_tensor(np.random.RandomState(7).permutation(g3)[:128]).cuda()
    grid[0, occ] = 2 * THR
    seed = R.refresh_seed(11, 256)
    old = grid.clone()
    bits, ws = refresh(model, grid, G, THR, False, 0.95, seed)
    keys, occ_list, draw = R.pick_keys(old.cpu().numpy()[0], THR, seed, 0, G)
    assert np.array_equal(Ws(ws, 1, G).keys_sorted, np.sort(keys)), "sorted picks"
    assert stats.chisquare(np.bincount(draw, minlength=occ_list.size)).pvalue > 1e-3
    # jitter offsets of a warm-up: uniform on [-1, 1) per axis, uncorrelated across axes and with the uniform pick
    # coordinates drawn from the same h
    grid = torch.zeros(1, g3, device="cuda")
    seed = R.refresh_seed(11, 0)
    bits, ws = refresh(model, grid, G, THR, True, 0.95, seed)
    xyz = Ws(ws, 1, G).xyz[:g3].astype(np.float64)
    cc = R.morton_decode(np.arange(g3, dtype=np.uint32)).astype(np.float64)
    s, half = 0.5, 0.5 / G
    off = (xyz - (cc / (G - 1) * 2 - 1) * (s - half)) / half
    assert off.min() >= -1 - 1e-5 and off.max() < 1 + 1e-5
    for k in range(3):
        assert stats.kstest(off[:, k], "uniform", args=(-1, 2)).pvalue > 1e-3
    uni = R.uniform_coords(seed, 0, G, g3).astype(np.float64)
    r = np.corrcoef(np.concatenate([off, uni], 1).T)
    lim = 5 / np.sqrt(g3)
    assert np.abs(r - np.diag(np.diag(r)))[:3].max() < lim
    # distinct count of M uniform picks over an empty grid (the occupied half is the single "none" key)
    for G in (32, 128):
        g3, M = G ** 3, G ** 3 // 4
        grid = torch.zeros(1, g3, device="cuda")
        bits, ws = refresh(model, grid, G, THR, False, 0.95, R.refresh_seed(13, 256))
        d = int(Ws(ws, 1, G).tot[1]) - 1
        n = float(g3)
        mu = n * (1 - (1 - 1 / n) ** M)
        var = n * (n - 1) * (1 - 2 / n) ** M + n * (1 - 1 / n) ** M - n * n * (1 - 1 / n) ** (2 * M)
        assert abs(d - mu) < 5 * np.sqrt(var), (G, d, mu, var)


# ---------------------------------------------------------------------------------------------------
# arguments
# ---------------------------------------------------------------------------------------------------
def test_bad_arguments_are_rejected():
    from ngp_pl_b200.models.networks import _net_struct
    _, L = _lib()
    model = _model(0.5)
    net, keep = _net_struct(model)
    st = _st()

    def pick(grid, cascades, G, ws, nbytes):
        return L.ngp_update_density_grid_pick(grid, cascades, G, 0.5, float(THR), 0, 1, ws, nbytes, st)

    def ev(n, grid, bits, cascades, G, ws, nbytes):
        return L.ngp_update_density_grid_eval(n, grid, bits, None, cascades, G, float(THR), 0, 0.95, ws, nbytes, st)

    def buffers(cascades, G):
        nbytes = L.ngp_update_grid_workspace(cascades, G)
        ws = torch.zeros(max(nbytes, 256), dtype=torch.uint8, device="cuda")
        grid = torch.zeros(max(cascades, 1) * G ** 3 + 8, device="cuda")
        bits = torch.zeros(grid.numel() // 8 + 1, dtype=torch.uint8, device="cuda")
        return ws, nbytes, grid, bits

    # grid sizes that are not powers of two in [2, 1024]: the workspace is real and big enough, so only the size rejects
    for G in (3, 5, 100):
        ws, nbytes, grid, bits = buffers(1, G)
        assert pick(grid.data_ptr(), 1, G, ws.data_ptr(), nbytes) == EINVAL
        assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), 1, G, ws.data_ptr(), nbytes) == EINVAL
    ws, nbytes, grid, bits = buffers(1, 2)
    for G in (1, 1025):
        big = L.ngp_update_grid_workspace(1, G)
        assert pick(grid.data_ptr(), 1, G, ws.data_ptr(), big) == EINVAL
        assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), 1, G, ws.data_ptr(), big) == EINVAL
    # cascades 0 and 63 (tot[63] is the distinct-key counter) on both halves
    for cascades in (0, 63):
        ws, nbytes, grid, bits = buffers(cascades, 2)
        assert pick(grid.data_ptr(), cascades, 2, ws.data_ptr(), nbytes) == EINVAL
        assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), cascades, 2, ws.data_ptr(), nbytes) == EINVAL
    # cascades * G^3 > 2^31 - 1 on _eval
    big = L.ngp_update_grid_workspace(3, 1024)
    assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), 3, 1024, ws.data_ptr(), big) == EINVAL
    assert pick(grid.data_ptr(), 3, 1024, ws.data_ptr(), big) == EINVAL
    # a workspace one byte short, and null pointers
    ws, nbytes, grid, bits = buffers(2, 4)
    assert pick(grid.data_ptr(), 2, 4, ws.data_ptr(), nbytes - 1) == EINVAL
    assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), 2, 4, ws.data_ptr(), nbytes - 1) == EINVAL
    assert pick(None, 2, 4, ws.data_ptr(), nbytes) == EINVAL
    assert pick(grid.data_ptr(), 2, 4, None, nbytes) == EINVAL
    assert ev(None, grid.data_ptr(), bits.data_ptr(), 2, 4, ws.data_ptr(), nbytes) == EINVAL
    assert ev(C.byref(net), None, bits.data_ptr(), 2, 4, ws.data_ptr(), nbytes) == EINVAL
    assert ev(C.byref(net), grid.data_ptr(), None, 2, 4, ws.data_ptr(), nbytes) == EINVAL
    assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), 2, 4, None, nbytes) == EINVAL
    # and the same buffers with valid arguments run
    assert pick(grid.data_ptr(), 2, 4, ws.data_ptr(), nbytes) == 0
    assert ev(C.byref(net), grid.data_ptr(), bits.data_ptr(), 2, 4, ws.data_ptr(), nbytes) == 0
    torch.cuda.synchronize()
