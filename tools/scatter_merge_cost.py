"""Do the hash-table gradient scatter's corner hand-overs pay? Trains BASELINE config 2 and config 5 for 1000 steps as
bench.py does, then takes the live samples of one step and

  * counts, per level, the 8-byte and 16-byte reductions k_grid_scatter_merged issues per live sample, under the rule
    that merges only runs of equal cells ("runs") and under the rule that also hands the corners shared with the next
    run's adjacent cell to that run's head ("runs + hand-over", the kernel's rule). A numpy restatement of the warp, exact
    up to fma rounding of the cell coordinates; no timing;
  * times the scatter as the step launches it, each launch after an Adam step that reads and clears the gradient as in
    the training step (CUDA graphs, CUDA events around the scatter alone, medians). With --compare OTHER.so the same C
    call of another build of the library is timed on the same buffers, alternated launch by launch, and the two builds'
    gradients are compared with the spread between two launches of one build.

    python tools/scatter_merge_cost.py [--iters 60] [--steps 1000] [--workloads c2,c5] [--compare path/to/libngp_b200.so]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P1, P2 = 2654435761, 805459861
M32 = 0xFFFFFFFF
WARP = 32


def _cell_coords(x01, scale):
    """grid_cell's floor(fmaf(scale, x, 0.5)): the float32 product is exact in float64, so one rounding to float32"""
    p = (np.float64(np.float32(scale)) * x01.astype(np.float64) + 0.5).astype(np.float32)
    return np.floor(p).astype(np.int64)


def _corner_entries(g, res, entries, hashed):
    """(..., 3) cells -> (..., 8) entries, k = dx + 2 dy + 4 dz, as grid_corner_indices"""
    gx, gy, gz = (g[..., i].astype(np.uint64) & M32 for i in range(3))
    k = np.arange(8, dtype=np.uint64)
    dx, dy, dz = k & 1, (k >> 1) & 1, k >> 2
    vx, vy, vz = (gx[..., None] + dx) & M32, (gy[..., None] + dy) & M32, (gz[..., None] + dz) & M32
    if hashed:
        return (vx ^ ((vy * P1) & M32) ^ ((vz * P2) & M32)) & np.uint64(entries - 1)
    v = (vx + vy * np.uint64(res) + vz * np.uint64(res * res)) & M32
    v = np.where(v >= entries, v - np.uint64(entries), v)
    return np.minimum(v, np.uint64(entries - 1))


def _shared(o):
    """grid_shared_corners over (..., 3) offsets"""
    m = np.full(o.shape[:-1], 0xFF, np.int64)
    for ax, (lo, hi) in enumerate(((0x55, 0xAA), (0x33, 0xCC), (0x0F, 0xF0))):
        m &= np.where(o[..., ax] > 0, hi, np.where(o[..., ax] < 0, lo, 0xFF))
    return m


def _shift(m, o):
    """m << o for o >= 0, m >> -o otherwise (8-bit masks)"""
    return np.where(o >= 0, m << np.maximum(o, 0), m >> np.maximum(-o, 0)) & 0xFF


def _pairs(own, idx, head):
    """(v2, v4) reductions a head issues for the corner mask `own`"""
    v2 = v4 = 0
    for k in range(0, 8, 2):
        o0, o1 = (own >> k) & 1, (own >> (k + 1)) & 1
        both = (o0 == 1) & (o1 == 1) & ((idx[..., k] ^ idx[..., k + 1]) == 1)
        v4 += int((head & both).sum())
        v2 += int((head & ~both & (o0 == 1)).sum()) + int((head & ~both & (o1 == 1)).sum())
    return v2, v4


def census(x01, meta):
    """x01: (n, 3) float32 unit-cube positions in the scatter's visit order. -> per level (v2, v4) under the two rules"""
    n = x01.shape[0]
    W = (n + WARP - 1) // WARP
    pad = W * WARP - n
    x = np.concatenate([x01, np.zeros((pad, 3), np.float32)]).reshape(W, WARP, 3)
    valid = (np.arange(W * WARP) < n).reshape(W, WARP)
    lane = np.arange(WARP)
    out = []
    for level in range(meta.n_levels):
        res, off = int(meta.res[level]), int(meta.offset[level])
        entries = int(meta.offset[level + 1]) - off
        hashed = bool((meta.hashed_mask >> level) & 1)
        g = _cell_coords(x, meta.scale[level])
        pvalid = np.zeros_like(valid)
        pvalid[:, 1:] = valid[:, :-1]
        same = np.zeros_like(valid)
        same[:, 1:] = (g[:, 1:] == g[:, :-1]).all(-1)
        head = (lane == 0)[None] | ~valid | ~pvalid | ~same
        vh = valid & head
        idx = _corner_entries(g, res, entries, hashed)
        old = _pairs(np.full(valid.shape, 0xFF, np.int64), idx, vh)
        # the link of a head to the previous run's cell (lane - 1 holds it)
        o = np.zeros_like(g)
        o[:, 1:] = g[:, :-1] - g[:, 1:]
        adj = vh & pvalid & (np.abs(o) <= 1).all(-1)
        olin = o[..., 0] + 2 * o[..., 1] + 4 * o[..., 2]
        mine = np.where(adj, _shared(o), 0)
        # the next head of every lane: the first head after it (32: none)
        nxt = np.where(head, lane[None], WARP)
        nh = np.full_like(nxt, WARP)
        nh[:, :-1] = np.minimum.accumulate(nxt[:, ::-1], axis=1)[:, ::-1][:, 1:]
        nhc = np.minimum(nh, WARP - 1)
        n_adj = np.take_along_axis(adj, nhc, 1) & (nh < WARP)
        n_mine = np.take_along_axis(mine, nhc, 1)
        n_o = np.take_along_axis(olin, nhc, 1)  # corner k here is corner k + n_o of the next cell
        send = vh & n_adj
        fwd_out = np.where(send, n_mine & ~_shift(mine, n_o), 0) & 0xFF
        fwd = np.where(send, _shift(fwd_out, -n_o), 0)
        new = _pairs(0xFF & ~fwd, idx, vh)
        out.append((old, new))
    return out


def print_census(cen, n_live, n_levels):
    print("reductions per live sample (8-byte + 16-byte) and their total, per level")
    print("%5s %22s %22s %9s" % ("level", "runs", "runs + hand-over", "saved"))
    tot = [0, 0]
    for level, (old, new) in enumerate(cen):
        a, b = sum(old), sum(new)
        tot[0] += a
        tot[1] += b
        print("%5d %6.3f + %5.3f = %5.3f %6.3f + %5.3f = %5.3f %8.1f%%" % (
            level, old[0] / n_live, old[1] / n_live, a / n_live, new[0] / n_live, new[1] / n_live, b / n_live,
            100.0 * (a - b) / max(a, 1)))
    print("%5s %22.3f %22.3f %8.1f%%" % ("all", tot[0] / n_live, tot[1] / n_live, 100.0 * (tot[0] - tot[1]) / max(tot[0], 1)))


def card(torch):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timings stand without it
        return "nvidia-smi unavailable: %r" % e


def run(workload, steps, iters, compare):
    import torch
    import bench
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(0)
    wl = bench.WORKLOADS[workload]
    scene = bench.make_scene(workload)
    bank = synth.RayBank(scene, n_images=bench.N_TRAIN_IMAGES, device="cuda", seed=0)
    tr = Trainer(NGP(scene.scale).cuda(), n_rays=wl["n_rays"], lr=1e-2, exp_step_factor=scene.exp_step_factor,
                 bg=(scene.bg,) * 3, seed=0)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(steps):
        tr.train_step()
    torch.cuda.synchronize()
    print("== %s, after %d steps" % (wl["name"], steps))
    print("card: %s (name, power limit, SM clock, max SM clock) before timing" % card(torch))
    n = int(tr.counters[5])
    rows = tr.live_idx[:n].long()
    r = tr.ray_idx[rows].long()
    x = (tr.rays_d[r].double() * tr.ts[rows].double()[:, None] + tr.rays_o[r].double()).float().cpu()
    lo = torch.tensor(list(tr.net.xyz_min), dtype=torch.float32)
    hi = torch.tensor(list(tr.net.xyz_max), dtype=torch.float32)
    x01 = ((x - lo) / (hi - lo)).numpy()  # to_unit: an fp32 subtract, then an fp32 divide
    meta = tr.net.meta
    print("live samples %d of %d marched" % (n, int(tr.counters[2])))
    print_census(census(x01, meta), n, meta.n_levels)

    libs = {"this build": _lib.lib()}
    if compare:
        other = C.CDLL(os.path.abspath(compare))
        other.ngp_abi_version.restype = C.c_int
        assert other.ngp_abi_version() == _lib.ABI_VERSION, "the other build has another C ABI"
        for f in ("ngp_net_backward_scatter", "ngp_adam_step"):
            getattr(other, f).argtypes = getattr(libs["this build"], f).argtypes
            getattr(other, f).restype = getattr(libs["this build"], f).restype
        libs["other build"] = other
    smp = _lib.NgpSamples()
    smp.rays_o, smp.rays_d = tr.rays_o.data_ptr(), tr.rays_d.data_ptr()
    smp.ray_idx, smp.ts = tr.ray_idx.data_ptr(), tr.ts.data_ptr()
    smp.n, smp.n_dev = tr.capacity, tr.counters[2:].data_ptr()
    smp.live_idx, smp.n_live_dev = tr.live_idx.data_ptr(), tr.counters[5:].data_ptr()
    net = _lib.NgpNet.from_buffer_copy(tr.net)
    G = tr.G
    P2, M2, V2, Ph2 = tr.P.clone(), tr.M.clone(), tr.V.clone(), tr.Ph.clone()

    def scatter(L, stream):
        _lib.check(L.ngp_net_backward_scatter(C.byref(net), C.byref(smp), tr.scalars[1:].data_ptr(), G.data_ptr(),
                                              tr.bwd_ws.data_ptr(), tr.bwd_ws.numel(), stream.cuda_stream), "scatter")

    def adam(stream):  # reads and clears G, as the step's optimiser does; its own copies of the other state
        _lib.check(libs["this build"].ngp_adam_step(P2.data_ptr(), G.data_ptr(), M2.data_ptr(), V2.data_ptr(), Ph2.data_ptr(),
                                                    tr.n_params, tr.lr_dev.data_ptr(), tr.step_dev.data_ptr(), 0.9, 0.999,
                                                    1e-15, 1.0, 0, stream.cuda_stream), "adam")

    grads = {}
    for k, L in libs.items():
        grads[k] = []
        for _ in range(2):
            G.zero_()
            scatter(L, torch.cuda.current_stream())
            torch.cuda.synchronize()
            grads[k].append(G.clone())
    a0, a1 = grads["this build"]
    spread = (a0 - a1).abs()
    print("gradient: max |G| %.3g; two launches of this build differ by max %.3g" % (a0.abs().max().item(), spread.max().item()))
    if compare:
        b0 = grads["other build"][0]
        d = (a0 - b0).abs()
        nz = (a0 != 0) | (b0 != 0)
        rel = lambda t: (t[nz] / a0.abs()[nz].clamp_min(1e-30)).median().item()
        print("gradient: this build against the other differs by max %.3g, median relative %.3g (two launches of this "
              "build: max %.3g, median relative %.3g); same zero pattern: %s" % (
                  d.max().item(), rel(d), spread.max().item(), rel(spread), bool(((a0 == 0) == (b0 == 0)).all())))

    def graph(fn):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn(s)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn(torch.cuda.current_stream())
        return g

    graphs = {k: graph(lambda s, L=L: scatter(L, s)) for k, L in libs.items()}
    g_adam = graph(adam)
    times = {k: [] for k in graphs}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(iters + 3):
        for k, g in graphs.items():
            g_adam.replay()
            ev[0].record()
            g.replay()
            ev[1].record()
            torch.cuda.synchronize()
            if it >= 3:
                times[k].append(ev[0].elapsed_time(ev[1]) * 1e3)
    print("card: %s after timing" % card(torch))
    print("scatter after an Adam step, %d launches each, alternated: median (min, max) us" % iters)
    for k, v in times.items():
        v = sorted(v)
        print("  %-12s %7.1f (%6.1f, %6.1f)" % (k, v[len(v) // 2], v[0], v[-1]))
    del tr, bank


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--workloads", default="c2,c5")
    ap.add_argument("--compare", default=None, help="another build of libngp_b200.so to time against this one")
    args = ap.parse_args()
    for wl in args.workloads.split(","):
        run(wl, args.steps, args.iters, args.compare)


if __name__ == "__main__":
    main()
