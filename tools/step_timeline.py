"""Timeline of the pipelined training step from in-stream timestamps (there is no nsys in this image).

ngp_trace_set() makes the step's entry points enqueue a one-thread kernel after each of their kernels that appends
{id, %globaltimer}; the stamps are captured into the CUDA graphs, so the timeline is the graph-replayed, two-stream
steady state. Each stamp adds to the launch chain, so the traced step is slower than the untraced one (both are
printed); read it for WHERE time goes, not for absolute numbers.

    python tools/step_timeline.py [steps] [n_steps_to_print] [ddp mode]
    python -m torch.distributed.run --nproc-per-node N ... tools/step_timeline.py 1200 3 nvls     (rank 0 prints)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import _lib, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402

NAMES = {1: "k_sample_rays", 2: "k_train_march", 3: "k_ngp_fwd", 4: "k_train_composite_loss", 5: "k_train_grad_scale",
         6: "k_ngp_bwd3", 7: "k_grid_scatter_merged", 8: "k_adam", 11: "<prepare graph starts>", 13: "<compute graph starts>",
         18: "<update graph starts>", 20: "refresh: memsets", 21: "refresh: k_grid_flags + cub select", 22: "refresh: k_grid_pick",
         30: "  exchange: block 0 enters", 31: "  exchange: start barrier passed (every rank's gradients are complete)",
         32: "  exchange: last block done (reduce-scatter + Adam + all-gather issued)", 33: "  exchange: end barrier passed",
         23: "refresh: k_grid_scatter", 24: "refresh: k_grid_merge + mean", 25: "refresh: packbits"}
SIDE = {1, 2, 11}


WORLD = int(os.environ.get("WORLD_SIZE", "1"))
RANK = int(os.environ.get("RANK", "0"))


def run(steps, trace, mode):
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=100, device="cuda", seed=RANK)
    model = NGP(scene.scale).cuda()
    if WORLD > 1:
        import torch.distributed as dist
        tr = Trainer(model, n_rays=8192, lr=1e-2, process_group=dist.group.WORLD, world_size=WORLD, rank=RANK, seed=RANK, ddp=mode)
    else:
        tr = Trainer(model, n_rays=8192, lr=1e-2)
    tr.attach_bank(bank)
    buf = None
    if trace:
        cap = 32 * (steps + 8)
        buf = torch.zeros(2 + 2 * cap, dtype=torch.int64, device="cuda")
        buf[1] = cap
        _lib.check(_lib.lib().ngp_trace_set(buf.data_ptr()), "trace_set")
    tr.capture(sample=True)
    for _ in range(steps - 100):
        tr.train_step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(100):
        tr.train_step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 100
    if trace:
        _lib.lib().ngp_trace_set(None)
    return ms, buf


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 1200
    n_print = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    mode = sys.argv[3] if len(sys.argv) > 3 else "p2p"
    if WORLD > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    ms_plain, _ = run(steps, False, mode)
    ms_traced, buf = run(steps, True, mode)
    if WORLD > 1:
        torch.distributed.barrier()
        if RANK != 0:
            torch.distributed.destroy_process_group()
            return
    print("world %d mode %s" % (WORLD, mode if WORLD > 1 else "-"))
    print("step: %.4f ms untraced, %.4f ms traced" % (ms_plain, ms_traced))
    b = buf.cpu().tolist()
    n = min(b[0], b[1])
    ev = [(b[3 + 2 * i], b[2 + 2 * i]) for i in range(n)]
    ev.sort()
    # steady state: the last n_print steps, delimited by "<compute graph starts>" stamps, skipping the occupancy refresh
    starts = [i for i, (t, k) in enumerate(ev) if k == 13]
    lo = starts[-(n_print + 3)]
    hi = starts[-3]
    t0 = ev[lo][0]
    last = {"main": t0, "side": None}
    print("%9s %9s  %-6s %s" % ("t (us)", "dur (us)", "stream", "event (dur = since the previous stamp on the same stream)"))
    for t, k in ev[lo:hi + 1]:
        s = "side" if k in SIDE else "main"
        d = (t - last[s]) / 1e3 if last[s] is not None else float("nan")
        last[s] = t
        ind = "        " if s == "side" else ""
        print("%9.1f %9.1f  %-6s %s%s" % ((t - t0) / 1e3, d, s, ind, NAMES.get(k, str(k))))
    # one occupancy-refresh step (every 16th): from the compute-graph start before the last refresh to the one after it
    ref = [i for i, (t, k) in enumerate(ev) if k == 20]
    if ref:
        r = ref[-2] if len(ref) > 1 else ref[-1]
        lo = max(i for i in starts if i < r)
        lo = max(i for i in starts if i < lo)  # one step earlier
        nxt = [i for i in starts if i > r]
        hi = nxt[1] if len(nxt) > 1 else len(ev) - 1
        t0 = ev[lo][0]
        last = {"main": t0, "side": None}
        print("\nacross an occupancy refresh:")
        for t, k in ev[lo:hi + 1]:
            s = "side" if k in SIDE else "main"
            d = (t - last[s]) / 1e3 if last[s] is not None else float("nan")
            last[s] = t
            ind = "        " if s == "side" else ""
            print("%9.1f %9.1f  %-6s %s%s" % ((t - t0) / 1e3, d, s, ind, NAMES.get(k, str(k))))
    # aggregate per kernel over the last 64 steps
    agg = {}
    last = {"main": None, "side": None}
    for t, k in ev[starts[-70]:starts[-3]]:
        s = "side" if k in SIDE else "main"
        if last[s] is not None:
            agg.setdefault(k, []).append((t - last[s]) / 1e3)
        last[s] = t
    print("\nmean interval ending at each stamp, last 67 steps:")
    for k in sorted(agg):
        v = agg[k]
        print("  %-28s %7.1f us  (n=%d, min %.1f, max %.1f)" % (NAMES.get(k, str(k)), sum(v) / len(v), len(v), min(v), max(v)))


if __name__ == "__main__":
    main()
