"""Does the order of the hash-table gradient scatter matter? On the buffers of a Trainer after 1000 steps, times the scatter
as the step launches it (all levels in one launch) against the same kernel launched once per level, once per pair of
levels and once per four levels. A launch over a level range is the unchanged C call given a level table shifted to
that range and the workspace shifted to its first level's feature gradients, so each launch reloads the positions.

Each timed launch follows an Adam step that reads and clears the gradient, as in the training step, so the scatter meets
the L2 the optimiser leaves; "warm" repeats the timing back to back and "cold" after a 256 MB flush. CUDA graphs, CUDA
events around the scatter alone, the variants alternated iteration by iteration, medians.

    python tools/scatter_order_cost.py [iterations]
"""
import ctypes as C
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import _lib, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timings stand without it
        return "nvidia-smi unavailable: %r" % e


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 40
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=100, device="cuda")
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(1000):
        tr.train_step()
    torch.cuda.synchronize()
    print("card: %s (name, power limit, SM clock, max SM clock) before timing" % card())
    L = _lib.lib()
    smp = _lib.NgpSamples()
    smp.rays_o, smp.rays_d = tr.rays_o.data_ptr(), tr.rays_d.data_ptr()
    smp.ray_idx, smp.ts = tr.ray_idx.data_ptr(), tr.ts.data_ptr()
    smp.n, smp.n_dev = tr.capacity, tr.counters[2:].data_ptr()
    smp.live_idx, smp.n_live_dev = tr.live_idx.data_ptr(), tr.counters[5:].data_ptr()
    stride = (tr.capacity + 15) // 16 * 16  # feature gradients: one uint32 per (level, sample), level-major
    meta = tr.net.meta
    n_levels = meta.n_levels

    def level_net(l0, n):
        net = _lib.NgpNet.from_buffer_copy(tr.net)
        m = net.meta
        m.n_levels = n
        m.hashed_mask = (meta.hashed_mask >> l0) & ((1 << n) - 1)
        for i in range(_lib.NGP_MAX_LEVELS):
            j = l0 + i if i < n else None
            m.res[i] = meta.res[j] if j is not None else 0
            m.scale[i] = meta.scale[j] if j is not None else 0.0
        for i in range(_lib.NGP_MAX_LEVELS + 1):
            m.offset[i] = meta.offset[l0 + min(i, n)]
        return net

    def launches(group):
        return [(level_net(l0, min(group, n_levels - l0)), l0) for l0 in range(0, n_levels, group)]

    G = tr.G
    P2, M2, V2, Ph2 = tr.P.clone(), tr.M.clone(), tr.V.clone(), tr.Ph.clone()

    def scatter(parts, stream):
        for net, l0 in parts:
            _lib.check(L.ngp_net_backward_scatter(C.byref(net), C.byref(smp), tr.scalars[1:].data_ptr(), G.data_ptr(),
                                                  tr.bwd_ws.data_ptr() + 4 * l0 * stride, tr.bwd_ws.numel(),
                                                  stream.cuda_stream), "scatter")

    def adam(stream):  # reads and clears G, as the step's optimiser does; its own copies of the other state
        _lib.check(L.ngp_adam_step(P2.data_ptr(), G.data_ptr(), M2.data_ptr(), V2.data_ptr(), Ph2.data_ptr(), tr.n_params,
                                   tr.lr_dev.data_ptr(), tr.step_dev.data_ptr(), 0.9, 0.999, 1e-15, 1.0, 0,
                                   stream.cuda_stream), "adam")

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

    variants = {"one launch, 16 levels": launches(n_levels), "per level (16 launches)": launches(1),
                "per pair (8 launches)": launches(2), "per 4 levels (4 launches)": launches(4)}
    # the level ranges add up to the single launch: the same reductions, in another order
    G.zero_()
    scatter(variants["one launch, 16 levels"], torch.cuda.current_stream())
    ref = G.clone()
    for name, parts in variants.items():
        G.zero_()
        scatter(parts, torch.cuda.current_stream())
        d = (G - ref).abs().max().item()
        print("%-28s max |G - G_one_launch| = %.3g (max |G| %.3g)" % (name, d, ref.abs().max().item()))
    graphs = {k: graph(lambda s, p=v: scatter(p, s)) for k, v in variants.items()}
    g_adam = graph(adam)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = {(k, c): [] for k in graphs for c in ("after adam", "warm", "cold")}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(iters + 3):
        for k, g in graphs.items():
            for cond in ("after adam", "warm", "cold"):
                g_adam.replay()
                if cond == "warm":
                    g.replay()
                elif cond == "cold":
                    flush.zero_()
                ev[0].record()
                g.replay()
                ev[1].record()
                torch.cuda.synchronize()
                if it >= 3:
                    times[(k, cond)].append(ev[0].elapsed_time(ev[1]) * 1e3)
    print("card: %s after timing" % card())
    print("live samples %d of %d marched; %d iterations, median (min, max) us" % (int(tr.counters[5]), int(tr.counters[2]), iters))
    print("%-28s %24s %24s %24s" % ("scatter", "after adam (in-step L2)", "warm (back to back)", "cold (256 MB flush)"))
    for k in graphs:
        cells = []
        for cond in ("after adam", "warm", "cold"):
            v = sorted(times[(k, cond)])
            cells.append("%7.1f (%6.1f, %6.1f)" % (v[len(v) // 2], v[0], v[-1]))
        print("%-28s %24s %24s %24s" % (k, *cells))


if __name__ == "__main__":
    main()
