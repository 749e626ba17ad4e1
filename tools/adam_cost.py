"""How close is the optimiser (k_adam) to what HBM allows, and which bytes does it move that it need not?

Trains a Trainer like bench.py (its scene, seeds, `capture(sample=True)`) for 1000 steps, then takes the state the next
step's optimiser meets (P, M, V and the complete gradient G, via train_step(after_backward=...)) and reports, as one JSON
line:

  census     float4 groups and 32-byte sectors (8 parameters) per table level and for the MLP, groups in the states
               zero    g = m = v = 0            (k_adam stores nothing)
               g       g != 0
               m       g = 0, m != 0
               v       g = 0, m = 0, v != 0     (dormant: the update leaves p and m bitwise as they are)
             sectors as "zero", "g_only" (some g != 0, m = v = 0) and "state" (some m or v != 0); and the HBM bytes
             k_adam moves ("bytes") against those a kernel would move that kept a bitmap of the sectors with m or v != 0,
             loaded only G (and P where g != 0) for the others, and skipped the P and M stores of dormant groups
             ("bytes_bitmap").
  k_adam_us  CUDA events around ngp_adam_step, medians (min, max) in us, each call from the same restored state:
               cold     after a 256 MB flush of L2;
               scatter  right after the hash-table gradient scatter recomputed G (the in-step L2 state);
               march    as "scatter", with the next step's g_prepare graph replayed on a side stream underneath, as the
                        training step runs it.
  ceiling    a plain 128-bit stream kernel with Adam's worst-case read:write mix (reads P, M, V, G; writes P, M, V, the
             fp16 copy and G: 34 B per parameter) over the same buffers, after the same flush, at full occupancy and at
             2 CTAs per SM. It is compiled with nvcc into a temporary directory.

    python tools/adam_cost.py [c2|c5] [iterations]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the workloads, their scenes and image count)
from ngp_pl_b200 import _lib, synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402

STREAM_SRC = r"""
#include <cuda_fp16.h>
#include <cstdint>
// Adam's worst-case traffic without its arithmetic: read p, m, v, g; write p, m, v, the fp16 copy and g = 0
__global__ void k_stream_mix(float4* p, float4* g, float4* m, float4* v, uint2* ph, int64_t n4) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 a = p[i], b = g[i], c = m[i], d = v[i];
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        c.x += b.x; d.x += b.y;
        p[i] = a; m[i] = c; v[i] = d;
        g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w);
        ph[i] = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
    }
}
extern "C" int stream_mix(float* p, float* g, float* m, float* v, void* ph, int64_t n4, int grid, void* st) {
    k_stream_mix<<<grid, 256, 0, (cudaStream_t)st>>>((float4*)p, (float4*)g, (float4*)m, (float4*)v, (uint2*)ph, n4);
    return (int)cudaGetLastError();
}
"""


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timings stand without it
        return "nvidia-smi unavailable: %r" % e


def stream_lib(tmp):
    src, so = os.path.join(tmp, "stream_mix.cu"), os.path.join(tmp, "stream_mix.so")
    open(src, "w").write(STREAM_SRC)
    subprocess.run(["nvcc", "-O3", "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", src, "-o", so],
                   check=True)
    lib = C.CDLL(so)
    lib.stream_mix.restype = C.c_int
    lib.stream_mix.argtypes = [C.c_void_p] * 5 + [C.c_int64, C.c_int, C.c_void_p]
    return lib


def census(tr, P, G, M, V):
    """per part (table level or MLP): counts of groups / sectors per state, the bytes k_adam moves and those a kernel with
    a state bitmap would move"""
    meta = tr.net.meta
    parts = [("L%d" % l, 2 * meta.offset[l], 2 * meta.offset[l + 1]) for l in range(meta.n_levels)]
    parts.append(("mlp", tr.n_enc, tr.n_params))
    out, tot = {}, {}
    for name, lo, hi in parts:
        # whole sectors inside the part only (the few groups of a sector that straddles two parts are left out)
        lo8, hi8 = (lo + 7) // 8 * 8, hi // 8 * 8
        if hi8 <= lo8:
            continue
        g, m, v, p = (t[lo8:hi8].view(-1, 2, 4) for t in (G, M, V, P))
        gz, mz, vz = (g == 0).all(-1), (m == 0).all(-1), (v == 0).all(-1)
        st = {"zero": gz & mz & vz, "g": ~gz, "m": gz & ~mz, "v": gz & mz & ~vz}
        d = {"groups": {k: int(x.sum()) for k, x in st.items()}}
        sec_g = (~gz).any(-1)
        sec_mv = (~mz).any(-1) | (~vz).any(-1)  # the sector's bit in a state bitmap
        d["sectors"] = {"zero": int((~sec_g & ~sec_mv).sum()), "g_only": int((sec_g & ~sec_mv).sum()),
                        "state": int(sec_mv.sum())}
        n_grp = g.shape[0] * 2
        written = n_grp - d["groups"]["zero"]
        old = 64 * n_grp + 56 * written + 16 * d["groups"]["g"]
        # with a bitmap: a clear sector reads G (32 B), and P (32 B) when it has a gradient; a set sector reads all four.
        # Stores per group as k_adam's, but P and M not for a dormant group (v state)
        new = 32 * int((~sec_mv).sum()) + 32 * int((sec_g & ~sec_mv).sum()) + 128 * int(sec_mv.sum()) + \
            56 * written + 16 * d["groups"]["g"] - 32 * d["groups"]["v"]
        d["bytes"], d["bytes_bitmap"] = old, new
        out[name] = d
        for k, x in d["groups"].items():
            tot["groups_" + k] = tot.get("groups_" + k, 0) + x
        for k, x in d["sectors"].items():
            tot["sectors_" + k] = tot.get("sectors_" + k, 0) + x
        tot["bytes"] = tot.get("bytes", 0) + old
        tot["bytes_bitmap"] = tot.get("bytes_bitmap", 0) + new
    return out, tot


def med(v):
    v = sorted(v)
    return {"median": round(v[len(v) // 2], 2), "min": round(v[0], 2), "max": round(v[-1], 2)}


def main():
    wl = sys.argv[1] if len(sys.argv) > 1 else "c2"
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 30
    w = bench.WORKLOADS[wl]
    scene = bench.make_scene(wl)
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    bank = synth.RayBank(scene, n_images=bench.N_TRAIN_IMAGES, device=dev, seed=0)
    tr = Trainer(NGP(scene.scale).to(dev), n_rays=w["n_rays"], lr=1e-2, exp_step_factor=scene.exp_step_factor,
                 bg=(scene.bg,) * 3, seed=0)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(1000):
        tr.train_step()
    snap = {}
    tr.train_step(after_backward=lambda t: snap.update(P=t.P.clone(), G=t.G.clone(), M=t.M.clone(), V=t.V.clone(),
                                                       step=t.step_dev.clone()))
    torch.cuda.synchronize()
    card_before = card()
    L = _lib.lib()
    n = tr.n_params
    parts, tot = census(tr, snap["P"], snap["G"], snap["M"], snap["V"])

    P2, G2, M2, V2, Ph2 = (torch.empty_like(t) for t in (tr.P, tr.G, tr.M, tr.V, tr.Ph))
    step2 = snap["step"].clone()
    smp = _lib.NgpSamples()
    smp.rays_o, smp.rays_d = tr.rays_o.data_ptr(), tr.rays_d.data_ptr()
    smp.ray_idx, smp.ts = tr.ray_idx.data_ptr(), tr.ts.data_ptr()
    smp.n, smp.n_dev = tr.capacity, tr.counters[2:].data_ptr()
    smp.live_idx, smp.n_live_dev = tr.live_idx.data_ptr(), tr.counters[5:].data_ptr()

    def restore(with_g):
        for dst, k in ((P2, "P"), (M2, "M"), (V2, "V")):
            dst.copy_(snap[k])
        if with_g:
            G2.copy_(snap["G"])
        else:
            G2.zero_()

    def scatter(st):
        _lib.check(L.ngp_net_backward_scatter(C.byref(tr.net), C.byref(smp), tr.scalars[1:].data_ptr(), G2.data_ptr(),
                                              tr.bwd_ws.data_ptr(), tr.bwd_ws.numel(), st), "scatter")

    def adam(st):
        _lib.check(L.ngp_adam_step(P2.data_ptr(), G2.data_ptr(), M2.data_ptr(), V2.data_ptr(), Ph2.data_ptr(), n,
                                   tr.lr_dev.data_ptr(), step2.data_ptr(), tr.betas[0], tr.betas[1], tr.eps, 1.0, 0, st), "adam")

    def stream_mix(st):
        rc = sl.stream_mix(P2.data_ptr(), G2.data_ptr(), M2.data_ptr(), V2.data_ptr(), Ph2.data_ptr(), n // 4, grid, st)
        if rc:
            raise RuntimeError("stream_mix launch failed: %d" % rc)

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    main_s, side = torch.cuda.current_stream(), torch.cuda.Stream(dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn, cond):
        v = []
        for it in range(iters + 2):
            restore(with_g=cond == "cold")
            flush.zero_()
            if cond != "cold":
                scatter(main_s.cuda_stream)
            if cond == "march":
                side.wait_stream(main_s)
                with torch.cuda.stream(side):
                    tr.g_prepare[1 - tr._cur].replay()
            ev[0].record()
            fn(main_s.cuda_stream)
            ev[1].record()
            main_s.wait_stream(side)
            torch.cuda.synchronize()
            if it >= 2:
                v.append(ev[0].elapsed_time(ev[1]) * 1e3)
        return med(v)

    res = {"workload": wl, "n_params": n, "card_before": card_before, "census_total": tot, "census_by_part": parts}
    res["k_adam_us"] = {cond: timed(adam, cond) for cond in ("cold", "scatter", "march")}
    # the stream ceiling: the same buffers and bytes, at full occupancy and at k_adam's 2 CTAs per SM
    res["stream_ceiling"] = {}
    with tempfile.TemporaryDirectory() as tmp:
        sl = stream_lib(tmp)
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        for name, grid in (("full occupancy", sms * 8), ("2 CTAs per SM", sms * 2)):
            t = timed(stream_mix, "cold")
            t["TBps"] = round(34 * n / t["median"] / 1e6, 3)
            res["stream_ceiling"][name] = t
    res["card_after"] = card()
    ceil = res["stream_ceiling"]["full occupancy"]["TBps"]
    res["model"] = {"bytes_MB": round(tot["bytes"] / 1e6, 2), "bytes_bitmap_MB": round(tot["bytes_bitmap"] / 1e6, 2),
                    "ceiling_TBps": ceil, "bytes_at_ceiling_us": round(tot["bytes"] / ceil / 1e6, 1),
                    "bytes_bitmap_at_ceiling_us": round(tot["bytes_bitmap"] / ceil / 1e6, 1),
                    "k_adam_cold_TBps": round(tot["bytes"] / res["k_adam_us"]["cold"]["median"] / 1e6, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
