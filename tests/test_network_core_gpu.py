"""The network chains that every network kernel shares (csrc/network.cuh), held bit for bit to
tests/golden/network_core.npz (tests/golden/make_golden_network_core.py), so that a change of one rounding in any of
them -- the density MLP and its fp16 h, the colour MLP and its input, the output activation, sigma = exp(h[0]), the
ray-mode sample position -- is seen in every kernel that runs it:

- ngp_net_forward (k_ngp_fwd): xyzs/dirs and ray layouts (with unused ray_idx = -1 slots and a device count), want_rgb
  1 and 0, rgb_act 1 and 0; sigma, rgb, h_out and the feat_save bytes; one tile and a size at which the ticket loop
  turns several times;
- ngp_density_lattice (the lattice instance of k_ngp_fwd) on two lattices;
- ngp_mlp_rgb_forward (k_mlp_rgb_fwd) with both activations;
- the feature gradients per row at a looping size: dL/dx of ngp_mlp_rgb_backward (k_mlp_rgb_bwd), the workspace of
  ngp_enc_backward (k_enc_bwd) and of ngp_net_backward_mlp (k_ngp_bwd3) with saved features, re-gathered and through
  a live list;
- the weight gradients at sizes where the launch is one CTA, so that each element receives exactly one reduction
  (at looping sizes the fp32 reduction order varies from run to run; test_backward_fp64_gpu.py bounds it there).

Large outputs are pinned by the SHA-256 of their bytes, small ones are stored, so that a failure names the rows.
Regenerate the golden only when what the network computes is meant to change.

With two or more GPUs visible, the kernels that opt in to more than 48 KB of dynamic shared memory also run on device 1
after device 0 in one process: the opt-in is a per-device function attribute.
"""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_core.npz")
SCALE = 2.0 ** 8
N_TILE = 13        # one 16-row tile, its last three rows past the end
N_LOOP = 250_000   # > 4 x (132 SMs x 3 CTAs x 8 warps x 16 rows): every forward warp takes several tiles
N_BWD = 200_000    # > 7 x 132 x 192 rows (k_ngp_bwd3) and > 11 x 132 x 128 rows (module kernels)
N_WG_MOD = 128     # one k_mlp_rgb_bwd / k_enc_bwd block
N_WG_NET = 192     # one k_ngp_bwd3 block


def _L():
    from ngp_pl_b200 import _lib
    return _lib.lib()


def _chk(rc, what):
    from ngp_pl_b200 import _lib
    _lib.check(rc, what)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _np(t):
    return t.detach().contiguous().cpu().numpy()


def _sha(t):
    return np.array(hashlib.sha256(_np(t).tobytes()).hexdigest())


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _model(dev):
    """NGP(0.5) with its seeded initial weights and O(1) features at every hash-grid level"""
    from ngp_pl_b200.models.networks import NGP
    model = NGP(0.5).to(dev)
    with torch.no_grad():
        p = model.xyz_encoder.params
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=_gen(1)) * 2 - 1) * 0.5).to(dev)
    return model


def _points(n, seed, dev):
    g = _gen(seed)
    x = torch.rand(n, 3, generator=g) - 0.5
    d = torch.randn(n, 3, generator=g) * (0.5 + torch.rand(n, 1, generator=g))
    return x.to(dev).contiguous(), d.to(dev).contiguous()


def _xyz_smp(x, d):
    from ngp_pl_b200.models import networks as N
    return N._samples_struct(x, d)


def _rays(n, seed, dev):
    """a rectangular (ray, slot) layout: every 7th slot unused (ray_idx = -1); the device count stops 5 short of n"""
    g = _gen(seed)
    R = 4096
    o = (torch.rand(R, 3, generator=g) - 0.5) * 0.5
    dr = torch.randn(R, 3, generator=g) * 0.2
    ridx = torch.randint(0, R, (n,), generator=g, dtype=torch.int32)
    ridx[::7] = -1
    ts = torch.rand(n, generator=g)
    return [t.to(dev).contiguous() for t in (o, dr, ridx, ts)] + [torch.tensor([max(n - 5, 1)], dtype=torch.int32, device=dev)]


def _ray_smp(o, dr, ridx, ts, n_dev, n, live=None, n_live=None):
    from ngp_pl_b200 import _lib
    s = _lib.NgpSamples()
    s.xyzs = s.dirs = None
    s.rays_o, s.rays_d, s.ray_idx, s.ts = o.data_ptr(), dr.data_ptr(), ridx.data_ptr(), ts.data_ptr()
    s.n = n
    s.n_dev = _ptr(n_dev)
    s.live_idx = _ptr(live)
    s.n_live_dev = _ptr(n_live)
    return s


def _forward(net, smp, n, want_rgb, dev):
    """sigma, rgb, h_out and feat_save of one ngp_net_forward; rows the kernel must not write keep their fill"""
    from ngp_pl_b200.models import networks as N
    sig = torch.full((n,), -7.0, device=dev)
    rgb = torch.full((n, 3), -7.0, device=dev)
    h = torch.zeros(n, 16, dtype=torch.float16, device=dev)
    fs = torch.zeros(N.feat_save_bytes(n), dtype=torch.uint8, device=dev)
    _chk(_L().ngp_net_forward(C.byref(net), C.byref(smp), want_rgb, sig.data_ptr(), rgb.data_ptr() if want_rgb else None,
                              h.data_ptr(), fs.data_ptr(), _st()), "ngp_net_forward")
    return sig, rgb, h, fs


def _workspace(n, dev):
    return torch.zeros(_L().ngp_net_backward_workspace(n), dtype=torch.uint8, device=dev)


def _dfeat(ws, n):
    """the feature-gradient workspace [level][row] (stride ceil16(n)) as (n, 32) fp16, column 2 level + f"""
    stride = (n + 15) // 16 * 16
    return ws[:16 * stride * 4].view(torch.float16).view(16, stride, 2)[:, :n].permute(1, 0, 2).reshape(n, 32)


def _mlp_rgb_backward(rgb_h, xin, dout, act, scale_t, dev):
    n = xin.shape[0]
    dx = torch.zeros(n, 32, device=dev)
    gr = torch.zeros(7168, device=dev)
    _chk(_L().ngp_mlp_rgb_backward(rgb_h.data_ptr(), xin.data_ptr(), dout.data_ptr(), n, act, scale_t.data_ptr(),
                                   dx.data_ptr(), gr.data_ptr(), _st()), "ngp_mlp_rgb_backward")
    return dx, gr


def _enc_backward(model, x01, dh, scale_t, dev):
    """ngp_enc_backward from the features of a want_rgb = 0 forward: its feature-gradient workspace and grad_enc"""
    from ngp_pl_b200.models import networks as N
    n = x01.shape[0]
    unet, keep = N._unit_net(model.xyz_encoder)
    _, _, _, fs = _forward(unet, _xyz_smp(x01, None), n, 0, dev)
    ws = _workspace(n, dev)
    ge = torch.zeros_like(model.xyz_encoder.params)
    _chk(_L().ngp_enc_backward(C.byref(unet), C.byref(_xyz_smp(x01, None)), dh.data_ptr(), fs.data_ptr(), scale_t.data_ptr(),
                               ge.data_ptr(), ws.data_ptr(), ws.numel(), _st()), "ngp_enc_backward")
    return _dfeat(ws, n), ge


def _net_backward_mlp(net, smp, up_sig, up_rgb, fs, n_ws, scale_t, dev):
    ws = _workspace(n_ws, dev)
    ge = torch.zeros(3072, device=dev)
    gr = torch.zeros(7168, device=dev)
    _chk(_L().ngp_net_backward_mlp(C.byref(net), C.byref(smp), up_sig.data_ptr(), up_rgb.data_ptr(), _ptr(fs),
                                   scale_t.data_ptr(), ge.data_ptr(), gr.data_ptr(), ws.data_ptr(), ws.numel(), _st()),
         "ngp_net_backward_mlp")
    return ws, ge, gr


def _upstream(n, seed, dev):
    g = _gen(seed)
    return (torch.randn(n, generator=g) * 1e-2).to(dev), (torch.randn(n, 3, generator=g) * 1e-1).to(dev)


def network_core_outputs():
    """every output the golden pins, as numpy arrays (small runs) or SHA-256 hex digests (large runs)"""
    from ngp_pl_b200 import mesh
    from ngp_pl_b200.models import networks as N
    dev = "cuda"
    out = {}
    model = _model(dev)
    net, keep = N._net_struct(model)
    enc_h, rgb_h = keep
    scale_t = torch.tensor([SCALE], device=dev)

    # ---- ngp_net_forward ----
    for size, n in (("tile", N_TILE), ("loop", N_LOOP)):
        x, d = _points(n, 10 + n, dev)
        o, dr, ridx, ts, n_dev = _rays(n, 20 + n, dev)
        for layout, smp in (("xyz", _xyz_smp(x, d)), ("ray", _ray_smp(o, dr, ridx, ts, n_dev, n))):
            for want_rgb, act in ((1, 1), (1, 0), (0, 1)):
                net.rgb_act = act
                sig, rgb, h, fs = _forward(net, smp, n, want_rgb, dev)
                key = "fwd_%s_%s_rgb%d_act%d_" % (size, layout, want_rgb, act)
                for name, t in (("sigma", sig), ("rgb", rgb), ("h", h.view(torch.int16)), ("feat_save", fs)):
                    if name == "rgb" and not want_rgb:
                        continue
                    out[key + name] = _np(t) if size == "tile" else _sha(t)
    net.rgb_act = 1

    # ---- ngp_density_lattice ----
    for size, res, lo, hi in (("small", (5, 6, 7), -0.5, 0.5), ("large", (64, 65, 67), (-0.45, -0.5, -0.3), (0.5, 0.4, 0.35))):
        lat = mesh.lattice(res, lo, hi)
        sigma = torch.full(res, -7.0, device=dev)
        _chk(_L().ngp_density_lattice(C.byref(net), C.byref(lat), sigma.data_ptr(), _st()), "ngp_density_lattice")
        out["lattice_%s_sigma" % size] = _np(sigma) if size == "small" else _sha(sigma)

    # ---- ngp_mlp_rgb_forward ----
    for size, n in (("tile", N_TILE), ("loop", N_LOOP)):
        xin = ((torch.rand(n, 32, generator=_gen(30 + n)) * 2 - 1) * 2).half().to(dev)
        for act in (1, 0):
            o3 = torch.zeros(n, 3, dtype=torch.float16, device=dev)
            _chk(_L().ngp_mlp_rgb_forward(rgb_h.data_ptr(), xin.data_ptr(), n, act, o3.data_ptr(), _st()), "ngp_mlp_rgb_forward")
            t = o3.view(torch.int16)
            out["mlp_rgb_fwd_%s_act%d" % (size, act)] = _np(t) if size == "tile" else _sha(t)

    # ---- ngp_mlp_rgb_backward: dL/dx per row (looping), dL/dx and grad_rgb in one CTA ----
    for size, n in (("loop", N_BWD), ("cta", N_WG_MOD)):
        g = _gen(40 + n)
        xin = ((torch.rand(n, 32, generator=g) * 2 - 1) * 2).half().to(dev)
        dout = (torch.randn(n, 3, generator=g) * 0.1).to(dev)
        for act in (1, 0):
            dx, gr = _mlp_rgb_backward(rgb_h, xin, dout, act, scale_t, dev)
            if size == "loop":
                out["mlp_rgb_bwd_loop_act%d_dx" % act] = _sha(dx)
            else:
                out["mlp_rgb_bwd_cta_act%d_dx" % act] = _np(dx)
                out["mlp_rgb_bwd_cta_act%d_grad_rgb" % act] = _np(gr)

    # ---- ngp_enc_backward: the feature-gradient workspace per row (looping), grad_enc[:3072] in one CTA ----
    for size, n in (("loop", N_BWD), ("cta", N_WG_MOD)):
        g = _gen(50 + n)
        x01 = torch.rand(n, 3, generator=g).to(dev)
        dh = (torch.randn(n, 16, generator=g) * 0.1).to(dev)
        dfeat, ge = _enc_backward(model, x01, dh, scale_t, dev)
        if size == "loop":
            out["enc_bwd_loop_dfeat"] = _sha(dfeat.view(torch.int16))
        else:
            out["enc_bwd_cta_dfeat"] = _np(dfeat.view(torch.int16))
            out["enc_bwd_cta_grad_enc"] = _np(ge[:3072])

    # ---- ngp_net_backward_mlp: saved features, re-gathered, live list ----
    for size, n in (("loop", N_BWD), ("cta", N_WG_NET)):
        x, d = _points(n, 60 + n, dev)
        up_sig, up_rgb = _upstream(n, 61 + n, dev)
        _, _, _, fs = _forward(net, _xyz_smp(x, d), n, 1, dev)
        for mode, f in (("saved", fs), ("regather", None)):
            ws, ge, gr = _net_backward_mlp(net, _xyz_smp(x, d), up_sig, up_rgb, f, n, scale_t, dev)
            dfeat = _dfeat(ws, n).view(torch.int16)
            key = "net_bwd_%s_%s_" % (size, mode)
            if size == "loop":
                out[key + "dfeat"] = _sha(dfeat)
            else:
                out[key + "dfeat"] = _np(dfeat)
                out[key + "grad_enc"] = _np(ge)
                out[key + "grad_rgb"] = _np(gr)
    # a live list over a ray layout: rows in live-list order, every other slot not visited
    for size, n_live in (("loop", N_BWD), ("cta", N_WG_NET)):
        cap = 2 * n_live + 100
        o, dr, ridx, ts, n_dev = _rays(cap, 70 + n_live, dev)
        smp = _ray_smp(o, dr, ridx, ts, n_dev, cap)
        _, _, _, fs = _forward(net, smp, cap, 1, dev)
        live = torch.randperm(cap - 5, generator=_gen(71 + n_live))[:n_live + 50].to(torch.int32).to(dev)
        n_live_t = torch.tensor([n_live], dtype=torch.int32, device=dev)
        up_sig, up_rgb = _upstream(cap, 72 + n_live, dev)
        ws, ge, gr = _net_backward_mlp(net, _ray_smp(o, dr, ridx, ts, n_dev, cap, live, n_live_t), up_sig, up_rgb, fs,
                                       cap, scale_t, dev)
        dfeat = _dfeat(ws, cap)[:n_live].view(torch.int16)
        key = "net_bwd_%s_live_" % size
        if size == "loop":
            out[key + "dfeat"] = _sha(dfeat)
        else:
            out[key + "dfeat"] = _np(dfeat)
            out[key + "grad_enc"] = _np(ge)
            out[key + "grad_rgb"] = _np(gr)
    torch.cuda.synchronize()
    return out


def _same(key, got, ref):
    if ref.dtype.kind == "U":
        assert str(got) == str(ref), "%s: the SHA-256 of the output bytes changed" % key
        return
    assert got.shape == ref.shape and got.dtype == ref.dtype, "%s: %s %s != %s %s" % (key, got.shape, got.dtype, ref.shape, ref.dtype)
    a = got.view(np.uint8).reshape(got.shape[0], -1) if got.ndim else got.view(np.uint8)
    b = ref.view(np.uint8).reshape(ref.shape[0], -1) if ref.ndim else ref.view(np.uint8)
    rows = np.nonzero((a != b).any(axis=1))[0] if a.ndim == 2 else np.nonzero(a != b)[0]
    assert rows.size == 0, "%s: %d of %d rows differ, first %s" % (key, rows.size, a.shape[0], rows[:10].tolist())


def test_network_chains_bitwise_equal_golden():
    ref = np.load(GOLDEN)
    got = network_core_outputs()
    assert sorted(got) == sorted(ref.files)
    for k in sorted(ref.files):
        _same(k, got[k], ref[k])
    # not vacuous: non-zero sigma, colour and gradients in the stored runs
    assert (ref["fwd_tile_xyz_rgb1_act1_sigma"][:N_TILE] > 0).all()
    assert np.abs(ref["fwd_tile_ray_rgb1_act0_rgb"]).max() > 0
    for k in ("mlp_rgb_bwd_cta_act1_grad_rgb", "enc_bwd_cta_grad_enc", "net_bwd_cta_saved_grad_enc", "net_bwd_cta_live_grad_rgb"):
        assert np.abs(ref[k]).max() > 0, k


def _per_device_run(dev):
    """the module backward kernels, the fused MLP backward (both instances) and the image metrics on one device"""
    from ngp_pl_b200 import metrics
    from ngp_pl_b200.models import networks as N
    from oracle import lpips_ref
    res = {}
    with torch.cuda.device(dev):
        model = _model(dev)
        net, keep = N._net_struct(model)
        enc_h, rgb_h = keep
        scale_t = torch.tensor([SCALE], device=dev)
        n = 3000
        g = _gen(80)
        xin = ((torch.rand(n, 32, generator=g) * 2 - 1) * 2).half().to(dev)
        dout = (torch.randn(n, 3, generator=g) * 0.1).to(dev)
        res["mlp_rgb_bwd_dx"], _ = _mlp_rgb_backward(rgb_h, xin, dout, 1, scale_t, dev)
        x01 = torch.rand(n, 3, generator=g).to(dev)
        dh = (torch.randn(n, 16, generator=g) * 0.1).to(dev)
        res["enc_bwd_dfeat"], _ = _enc_backward(model, x01, dh, scale_t, dev)
        x, d = _points(n, 81, dev)
        up_sig, up_rgb = _upstream(n, 82, dev)
        _, _, _, fs = _forward(net, _xyz_smp(x, d), n, 1, dev)
        for mode, f in (("saved", fs), ("regather", None)):
            ws, _, _ = _net_backward_mlp(net, _xyz_smp(x, d), up_sig, up_rgb, f, n, scale_t, dev)
            res["net_bwd_%s_dfeat" % mode] = _dfeat(ws, n)
        H, W = 40, 30
        pred = torch.rand(H * W, 3, generator=g).to(dev)
        gt = torch.rand(H * W, 3, generator=g).to(dev)
        sse = torch.zeros(1, dtype=torch.float64, device=dev)
        ssim = torch.zeros(1, dtype=torch.float64, device=dev)
        metrics.image_metrics(pred, gt, H, W, sse, ssim, metrics.workspace(H, W, dev))
        res["sse"], res["ssim"] = sse, ssim
        vgg, lin = lpips_ref.random_weights(7)
        lp = torch.zeros(1, dtype=torch.float64, device=dev)
        metrics.lpips_metric(metrics.LpipsNet.from_state_dicts(lpips_ref.fp16_convs(vgg), lin, dev), pred, gt, H, W, lp,
                             metrics.lpips_workspace(H, W, dev))
        res["lpips"] = lp
        torch.cuda.synchronize()
    return {k: v.cpu() for k, v in res.items()}


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_shared_memory_opt_in_per_device():
    """device 1 after device 0 in one process: each kernel that needs more than 48 KB of dynamic shared memory opts in
    on every device it runs on (a failed launch raises in _lib.check), and computes what it computed on device 0"""
    a = _per_device_run("cuda:0")
    b = _per_device_run("cuda:1")
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert a["lpips"].item() > 0 and a["net_bwd_saved_dfeat"].abs().max() > 0
