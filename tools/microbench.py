"""Kernel micro-timings on one GPU (CUDA events, warm-up, L2 flush between iterations).
Usage: python tools/microbench.py [out.json]"""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ngp_pl_b200 import _lib, synth, vren  # noqa: E402
from ngp_pl_b200.models import networks as N  # noqa: E402


def timeit(fn, iters=20, warm=5, flush=None):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def main():
    out = {}
    dev = "cuda"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    scene = synth.lego_scene(0)
    model = N.NGP(0.5).cuda()
    with torch.no_grad():
        model.xyz_encoder.params[3072:].uniform_(-0.3, 0.3)
        model.density_bitfield.copy_(torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda())
    K = synth.intrinsics()
    dirs = synth.ray_directions(K, dev)
    poses = torch.as_tensor(synth.camera_poses(100)).cuda()
    g = torch.Generator(dev).manual_seed(0)
    n_rays = 8192
    img = torch.randint(100, (n_rays,), device=dev, generator=g)
    pix = torch.randint(dirs.shape[0], (n_rays,), device=dev, generator=g)
    o, d = synth.get_rays(dirs[pix], poses[img])
    _, hits_t, _ = vren.ray_aabb_intersect(o, d, model.center, model.half_size, 1)
    hits = hits_t[:, 0].contiguous()
    noise = torch.rand(n_rays, device=dev)

    def march():
        return vren.raymarching_train(o, d, hits, model.density_bitfield, 1, 0.5, 0.0, noise, 128, 1024)
    rays_a, xyzs, dd, deltas, ts, counter = march()
    n = int(counter[0])
    out["samples"] = n
    out["march_train_ms"] = timeit(march, flush=flush)
    x, dv = xyzs[:n].contiguous(), dd[:n].contiguous()

    net, keep = N._net_struct(model)
    smp = N._samples_struct(x, dv)
    st = torch.cuda.current_stream().cuda_stream
    sig = torch.empty(n, device=dev); rgb = torch.empty(n, 3, device=dev)
    feat = torch.empty(N.feat_save_bytes(n), device=dev, dtype=torch.uint8)
    L = _lib.lib()
    out["net_fwd_ms"] = timeit(lambda: L.ngp_net_forward(C.byref(net), C.byref(smp), 1, sig.data_ptr(), rgb.data_ptr(), None, feat.data_ptr(), st), flush=flush)
    out["net_fwd_nosave_ms"] = timeit(lambda: L.ngp_net_forward(C.byref(net), C.byref(smp), 1, sig.data_ptr(), rgb.data_ptr(), None, None, st), flush=flush)
    if "--fwd-only" in sys.argv:
        print(json.dumps({"samples": n, "net_fwd_ms": out["net_fwd_ms"], "net_fwd_nosave_ms": out["net_fwd_nosave_ms"]}))
        return
    out["net_density_ms"] = timeit(lambda: L.ngp_net_forward(C.byref(net), C.byref(smp), 0, sig.data_ptr(), None, None, None, st), flush=flush)
    dsig = torch.randn(n, device=dev) * 1e-3; drgb = torch.randn(n, 3, device=dev) * 1e-2
    ge = torch.zeros_like(model.xyz_encoder.params); gr = torch.zeros_like(model.rgb_net.params)
    bws = torch.empty(L.ngp_net_backward_workspace(n), device=dev, dtype=torch.uint8)
    out["net_bwd_ms"] = timeit(lambda: L.ngp_net_backward(C.byref(net), C.byref(smp), dsig.data_ptr(), drgb.data_ptr(), feat.data_ptr(), None, ge.data_ptr(), gr.data_ptr(), bws.data_ptr(), bws.numel(), st), flush=flush)
    out["net_bwd_regather_ms"] = timeit(lambda: L.ngp_net_backward(C.byref(net), C.byref(smp), dsig.data_ptr(), drgb.data_ptr(), None, None, ge.data_ptr(), gr.data_ptr(), bws.data_ptr(), bws.numel(), st), flush=flush)
    out["composite_fw_ms"] = timeit(lambda: vren.composite_train_fw(sig, rgb, deltas[:n], ts[:n], rays_a, 1e-4), flush=flush)
    out["cast_params_ms"] = timeit(lambda: L.ngp_cast_params(model.xyz_encoder.params.data_ptr(), keep[0].data_ptr(), model.xyz_encoder.params.numel(), st), flush=flush)
    out["zero_grad_ms"] = timeit(lambda: ge.zero_(), flush=flush)
    # full-image inference-sized network call
    n_big = 4_000_000
    xb = (torch.rand(n_big, 3, device=dev) - 0.5)
    db = torch.randn(n_big, 3, device=dev)
    smpb = N._samples_struct(xb, db)
    sigb = torch.empty(n_big, device=dev); rgbb = torch.empty(n_big, 3, device=dev)
    out["net_fwd_4M_random_ms"] = timeit(lambda: L.ngp_net_forward(C.byref(net), C.byref(smpb), 1, sigb.data_ptr(), rgbb.data_ptr(), None, None, st), iters=5, warm=2, flush=flush)
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1 and not sys.argv[1].startswith("--"):
        os.makedirs(os.path.dirname(sys.argv[1]) or ".", exist_ok=True)
        json.dump(out, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
