"""Generate tests/golden/*.npz by running the REAL reference kernels (oracle/_ref/vren, compiled from
the reference's models/csrc by oracle/build_ref.py) on a GPU:

    python tests/golden/make_golden.py OUT_DIR

then copy OUT_DIR/*.npz into tests/golden/. Inputs come from tests/cases.py (seeded).
The reference's sample ORDER is nondeterministic (atomics, raymarching.cu:237-241); fixtures are
stored per ray in ray order.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import ref_env  # noqa: E402


def T(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).cuda()
    return t.to(dtype) if dtype is not None else t


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    ref = ref_env.load_reference()
    vren = ref.vren

    # ---- AABB + marcher (train and test) -------------------------------------------------------
    for name in cases.MARCH_CASES:
        c = cases.march_case(name)
        o, d = T(c["o"]), T(c["d"])
        center = torch.zeros(1, 3, device="cuda")
        half = torch.full((1, 3), float(c["scale"]), device="cuda")
        cnt, hits_t, idx = vren.ray_aabb_intersect(o, d, center, half, 1)
        hits_raw = hits_t.clone()
        hits_t[(hits_t[:, 0, 0] >= 0) & (hits_t[:, 0, 0] < 0.01), 0, 0] = 0.01  # rendering.py:29
        hits = hits_t[:, 0].contiguous()
        bits = T(c["bits"])
        rays_a, xyzs, dirs, deltas, ts, counter = vren.raymarching_train(
            o, d, hits, bits, int(c["cascades"]), float(c["scale"]), float(c["esf"]), T(c["noise"]), 128, 1024)
        total = int(counter[0])
        rays_a = rays_a.cpu().numpy()
        order = np.argsort(rays_a[:, 0], kind="stable")
        ra = rays_a[order]
        sel = np.concatenate([np.arange(s, s + n) for _, s, n in ra]) if total > 0 else np.zeros(0, np.int64)
        out = dict(hit_cnt=cnt.cpu().numpy(), hits_raw=hits_raw.cpu().numpy(), hits=hits.cpu().numpy(),
                   counts=ra[:, 2].astype(np.int32), total=np.int64(total),
                   xyzs=xyzs[:total].cpu().numpy()[sel], dirs=dirs[:total].cpu().numpy()[sel],
                   deltas=deltas[:total].cpu().numpy()[sel], ts=ts[:total].cpu().numpy()[sel])
        # test-time marcher: four rounds with N_samples 1, 2, 4, 64 on all rays
        h = hits.clone()
        alive = torch.arange(o.shape[0], device="cuda")
        for rnd, ns in enumerate([1, 2, 4, 64]):
            x2, d2, dl2, t2, neff = vren.raymarching_test(o, d, h, alive, bits, int(c["cascades"]), float(c["scale"]),
                                                          float(c["esf"]), 128, 1024, ns)
            out["test%d_xyzs" % rnd] = x2.cpu().numpy()
            out["test%d_dirs" % rnd] = d2.cpu().numpy()
            out["test%d_deltas" % rnd] = dl2.cpu().numpy()
            out["test%d_ts" % rnd] = t2.cpu().numpy()
            out["test%d_neff" % rnd] = neff.cpu().numpy()
            out["test%d_hits" % rnd] = h.cpu().numpy().copy()
        np.savez_compressed(os.path.join(out_dir, "march_%s.npz" % name), **out)
        print(name, "total", total)

    # ---- compositing -----------------------------------------------------------------------------
    c = cases.composite_case()
    sig, rgbs, dl, ts, ra = T(c["sigmas"]), T(c["rgbs"]), T(c["deltas"]), T(c["ts"]), T(c["rays_a"])
    total, opacity, depth, rgb, ws = vren.composite_train_fw(sig, rgbs, dl, ts, ra, float(c["T_thr"]))
    dsig, drgbs = vren.composite_train_bw(T(c["dO"]), T(c["dD"]), T(c["dC"]), T(c["dws"]), sig, rgbs, ws, dl, ts, ra,
                                          opacity, depth, rgb, float(c["T_thr"]))
    loss, ws_inc, wts_inc = vren.distortion_loss_fw(ws, dl, ts, ra)
    dL = T(np.random.RandomState(8).normal(size=ra.shape[0]).astype(np.float32))
    dws2 = vren.distortion_loss_bw(dL, ws_inc, wts_inc, ws, dl, ts, ra)
    np.savez_compressed(os.path.join(out_dir, "composite.npz"), total=total.cpu().numpy(), opacity=opacity.cpu().numpy(),
                        depth=depth.cpu().numpy(), rgb=rgb.cpu().numpy(), ws=ws.cpu().numpy(), dsig=dsig.cpu().numpy(),
                        drgbs=drgbs.cpu().numpy(), dist_loss=loss.cpu().numpy(), ws_inc=ws_inc.cpu().numpy(),
                        wts_inc=wts_inc.cpu().numpy(), dist_dL=dL.cpu().numpy(), dist_dws=dws2.cpu().numpy())

    # ---- packbits / morton -----------------------------------------------------------------------
    rng = np.random.RandomState(21)
    grid = rng.normal(0, 1, 4096 * 8).astype(np.float32)
    bf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    vren.packbits(T(grid), 0.25, bf)
    coords = rng.randint(0, 128, (4096, 3)).astype(np.int32)
    m = vren.morton3D(T(coords))
    inv = vren.morton3D_invert(m)
    np.savez_compressed(os.path.join(out_dir, "bits_morton.npz"), grid=grid, bits=bf.cpu().numpy(), coords=coords,
                        morton=m.cpu().numpy(), invert=inv.cpu().numpy())
    print("golden written to", out_dir)


if __name__ == "__main__":
    main(sys.argv[1])
