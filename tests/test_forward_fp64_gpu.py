"""The network forward (k_ngp_fwd: hash gather, trilinear interpolation, density MLP, exp, SH-4, rgb MLP, sigmoid) and the
stand-alone module kernels (k_mlp_rgb_fwd, k_sh_encode) per sample against the float64 reference of oracle/grad64.py, at
sizes where the persistent kernel's ticket loop turns, in every input mode, and with its tile scheduler wrapping.

Sizes derive from the SM count S: k_ngp_fwd runs 3 CTAs of 8 warps per SM, so one wave is W = 24 S warp-tiles of 16
rows; 16 W rows fill it exactly and 8 x 16 W + 7 rows make every warp take eight tiles, the last one partial.

Every bound comes from the arithmetic (grad64): the features within the fp32 fmaf chain's 8 x 2^-24 sum |w t| before
their fp16 rounding; the MLP from the kernel's own fp16 features with every layer's bound carried to the outputs
(mlp_forward(carry=True)), which holds through a ReLU whose mask it leaves open, so no row is excluded; sigma = expf of
the fp16 h0 candidates, widened by expf's 2 ulp. Values are compared with 2 x bound, never with a tolerance relative to a
maximum.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import grad64
from test_backward_fp64_gpu import _L, _chk, _f16, _st, env  # noqa: F401  (env is a fixture)

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _N():
    from ngp_pl_b200.models import networks as N
    return N


def _sizes(S):
    W = 24 * S
    return {"1": 1, "15": 15, "16": 16, "17": 17, "3007": 3007, "16W": 16 * W, "8*16W+7": 8 * 16 * W + 7}


SIZES = ["1", "15", "16", "17", "3007", "16W", "8*16W+7"]


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def _random_table(model, seed, amp=0.5):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        p = model.xyz_encoder.params
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * amp).cuda()
    return model


def _trained_lego():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=40, K=synth.intrinsics(W=200, H=200, fx=1111.11 / 4), device="cuda")
    torch.manual_seed(0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=4096, lr=1e-2)
    tr.attach_bank(bank)
    for _ in range(300):
        tr.train_step()
    tr.gather_master_params()
    torch.cuda.synchronize()
    return model


_MODELS = {}


def _model(name, env):
    """the seeded model of test_backward_fp64_gpu (L = 16, T = 2^19, table amplitude 0.5); L = 4, T = 2^14 (the 32-wide
    first layer is mostly zero padding); scale 16 (six cascades, mostly hashed levels); a model trained 300 steps on the
    synthetic Lego scene (realistic ReLU masks and sigma ranges)"""
    if name not in _MODELS:
        from ngp_pl_b200.models.networks import NGP
        if name == "env":
            m = env["model"]
        elif name == "L4_T14":
            torch.manual_seed(1)
            m = _random_table(NGP(0.5, n_levels=4, log2_hashmap_size=14).cuda(), 2)
        elif name == "scale16":
            torch.manual_seed(3)
            m = _random_table(NGP(16.0).cuda(), 4)
        else:
            m = _trained_lego()
        net, keep = _N()._net_struct(m)
        _MODELS[name] = dict(model=m, net=net, keep=keep, enc_h=_f16(keep[0]), rgb_h=_f16(keep[1]), scale=float(m.scale),
                             meta=m.xyz_encoder.meta, lo=list(m._xyz_min_host), hi=list(m._xyz_max_host))
    return _MODELS[name]


MODELS = ["env", "L4_T14", "scale16", "lego"]


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _points(n, mdl, seed):
    """seeded uniform points and unnormalised directions, with the special points first (as many as fit): the box's
    corners and face centres, points on cell faces of several levels, points one float32 ulp outside the box and well
    outside it (the documented clamp), and very short and very long directions"""
    s = mdl["scale"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.rand(n, 3, device="cuda", generator=g) * 2 - 1) * s
    d = torch.randn(n, 3, device="cuda", generator=g) * (0.5 + 1.5 * torch.rand(n, 1, device="cuda", generator=g))
    sp = []
    c = torch.tensor([[i, j, k] for i in (-1, 1) for j in (-1, 1) for k in (-1, 1)], dtype=torch.float32)
    sp.append(c * s)
    f = torch.zeros(6, 3)
    for a in range(3):
        f[2 * a, a], f[2 * a + 1, a] = -1, 1
    sp.append(f * s)
    meta = mdl["meta"]
    rng = np.random.RandomState(seed)
    for l in range(0, int(meta.n_levels), 3):
        k = rng.randint(0, int(meta.res[l]), (8, 3))
        u = torch.as_tensor(((k - 0.5) / np.float64(meta.scale[l])).clip(0, 1), dtype=torch.float32)
        sp.append(u * 2 * s - s)
    out1 = torch.full((6, 3), 0.0)
    for a in range(3):
        out1[2 * a, a] = float(np.nextafter(np.float32(s), np.float32(np.inf)))
        out1[2 * a + 1, a] = float(np.nextafter(np.float32(-s), np.float32(-np.inf)))
    sp.append(out1)
    sp.append(torch.tensor([[1.5, 0.2, -0.3], [-3.0, 2.5, 0.1], [0.4, -2.0, 3.0], [2.9, 2.9, -2.9]]) * s)
    sp = torch.cat(sp).cuda()
    m = min(n, sp.shape[0])
    x[:m] = sp[:m]
    sc = torch.tensor([1e-6, 1e-3, 1e3, 1e6], device="cuda")
    k = min(n, 4)
    d[n - k:] = d[n - k:] * sc[:k, None]
    return x.contiguous(), d.contiguous()


def _filled(shape, dtype=torch.float32):
    return torch.full(shape, NAN, device="cuda", dtype=dtype)


def _forward(mdl, smp, n, want_rgb=1, net=None, feat_save=True, h_out=True, stream=None):
    """ngp_net_forward with NaN-filled outputs: sigma (n), rgb (n, 3), h (n, 16) fp16, feat_save bytes. With `stream`,
    the outputs are allocated and filled on that stream too, so the fill is ordered before the launch."""
    if stream is not None:
        with torch.cuda.stream(stream):
            return _forward(mdl, smp, n, want_rgb, net, feat_save, h_out)
    N = _N()
    sig, rgb = _filled((n,)), _filled((n, 3)) if want_rgb else None
    h = _filled((n, 16), torch.float16) if h_out else None
    fs = torch.zeros(N.feat_save_bytes(n), device="cuda", dtype=torch.uint8) if feat_save else None
    _chk(_L().ngp_net_forward(C.byref(net if net is not None else mdl["net"]), C.byref(smp), want_rgb, sig.data_ptr(),
                              rgb.data_ptr() if rgb is not None else None, h.data_ptr() if h is not None else None,
                              fs.data_ptr() if fs is not None else None, _st()), "forward")
    return dict(sig=sig, rgb=rgb, h=h, fs=fs)


def _reference(mdl, x01, dirs, fs, n, rgb_act=1):
    """the float64 reference of rows 0..n-1: features from the positions, the MLP from the kernel's own features"""
    feat, d_feat = grad64.grid_encode(mdl["meta"], mdl["enc_h"][3072:].view(-1, 2), x01)
    fk = grad64.decode_feat_save(fs, n)
    f = grad64.mlp_forward(fk, grad64.sh4_64(dirs), mdl["enc_h"][:3072], mdl["rgb_h"], rgb_act, carry=True)
    sig, d_sig = grad64.sigma(f["h"], f["d_h"])
    return dict(feat=feat, d_feat=d_feat, fk=fk, h=f["h"], d_h=f["d_h"], sig=sig, d_sig=d_sig, rgb=f["out"],
                d_rgb=f["d_out"], ambiguous_own=f["ambiguous_own"])


def _ratio(got, want, bound, what):
    """asserts |got - want| <= 2 bound element by element; returns (bitwise fraction, worst |got - want| / (2 bound))"""
    got, want, bound = got.double(), want.double(), bound.double()
    assert torch.isfinite(got).all(), what + ": non-finite values"
    err = (got - want).abs()
    bad = err > 2 * bound
    assert not bad.any(), "%s: %d values outside 2 x bound (worst excess %g)" % (
        what, int(bad.sum()), float((err - 2 * bound).max()))
    r = torch.where(err > 0, err / (2 * bound).clamp_min(1e-300), torch.zeros_like(err))
    # bitwise: against the float64 value rounded to the output's format (fp16 values already are; sigma is fp32)
    return float((got == want.float().double()).double().mean()), float(r.max()) if r.numel() else 0.0


def _check_rows(out, ref, rows, what, rgb=True):
    """the kernel's rows `rows` (bool mask or index) against the reference's rows 0..; returns the measured numbers"""
    m = {}
    m["feat"] = _ratio(ref["fk"], ref["feat"], ref["d_feat"], what + " features")
    m["h"] = _ratio(out["h"][rows].float(), ref["h"], ref["d_h"], what + " h")
    m["sigma"] = _ratio(out["sig"][rows], ref["sig"], ref["d_sig"], what + " sigma")
    if rgb:
        r = out["rgb"][rows]
        assert torch.equal(r, r.half().float()), what + ": rgb not fp16 values"
        m["rgb"] = _ratio(r, ref["rgb"], ref["d_rgb"], what + " rgb")
    amb = ref["ambiguous_own"]
    if amb.numel() >= 10000:
        assert amb.double().mean().item() < 1e-2, "%s: %d rows with open ReLU masks" % (what, int(amb.sum()))
    return m


def _print(what, n, m, ref):
    print("MEASURED %s n=%d: %s; %d / %d rows with a ReLU mask open to the kernel's own accumulation error (checked too)"
          % (what, n, ", ".join("%s %.4f bitwise, worst %.3f of 2x bound" % (k, v[0], v[1]) for k, v in m.items()),
             int(ref["ambiguous_own"].sum()), n))


# ---------------------------------------------------------------------------------------------------------------------
# (a) positions + directions, every model and size
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", MODELS)
def test_forward_rows_vs_float64(env, name, size):
    mdl = _model(name, env)
    n = _sizes(env["S"])[size]
    x, d = _points(n, mdl, 100 + n)
    out = _forward(mdl, _N()._samples_struct(x, d), n)
    # the density-only launch, without feat_save and h_out, gives the same sigma bit for bit
    dens = _forward(mdl, _N()._samples_struct(x, d), n, want_rgb=0, feat_save=False, h_out=False)
    torch.cuda.synchronize()
    assert torch.equal(dens["sig"], out["sig"])
    x01 = grad64.to_unit(x, mdl["lo"], mdl["hi"])
    ref = _reference(mdl, x01, d, out["fs"], n)
    m = _check_rows(out, ref, slice(0, n), "%s n=%d" % (name, n))
    if n >= 3007:
        _print(name, n, m, ref)


# ---------------------------------------------------------------------------------------------------------------------
# (b) ray mode: positions fma(d, t, o), ray_idx = -1 slots left untouched
# ---------------------------------------------------------------------------------------------------------------------
def _ray_smp(o, dr, ridx, ts, n, n_dev=None):
    from ngp_pl_b200 import _lib
    s = _lib.NgpSamples()
    s.xyzs = s.dirs = s.live_idx = s.n_live_dev = None
    s.rays_o, s.rays_d, s.ray_idx, s.ts = o.data_ptr(), dr.data_ptr(), ridx.data_ptr(), ts.data_ptr()
    s.n = n
    s.n_dev = n_dev.data_ptr() if n_dev is not None else None
    return s


@pytest.mark.parametrize("size", ["17", "3007", "8*16W+7"])
@pytest.mark.parametrize("name", ["env", "lego"])
def test_ray_mode_vs_float64(env, name, size):
    mdl = _model(name, env)
    n = _sizes(env["S"])[size]
    s = mdl["scale"]
    g = torch.Generator(device="cuda").manual_seed(7 + n)
    R = 2048
    o = ((torch.rand(R, 3, device="cuda", generator=g) * 2 - 1) * s * 0.8).contiguous()
    dr = torch.randn(R, 3, device="cuda", generator=g) * (0.5 + 1.5 * torch.rand(R, 1, device="cuda", generator=g))
    dr = dr.contiguous()
    ridx = torch.randint(0, R, (n,), device="cuda", generator=g, dtype=torch.int32)
    ridx[2::3] = -1
    ts = (torch.rand(n, device="cuda", generator=g) * s).contiguous()
    out = _forward(mdl, _ray_smp(o, dr, ridx, ts, n), n)
    torch.cuda.synchronize()
    live = ridx >= 0
    for k in ("sig", "rgb", "h"):
        assert torch.isnan(out[k][~live]).all(), "%s written in a ray_idx = -1 slot" % k
    x = grad64.ray_positions(o, dr, ridx, ts)[live]
    li = live.nonzero()[:, 0]
    # the reference runs on the live rows; the kernel's features of them come from its feat_save rows
    fs_live = grad64.encode_feat_save(grad64.decode_feat_save(out["fs"], n)[li])
    ref = _reference(mdl, grad64.to_unit(x, mdl["lo"], mdl["hi"]), dr[ridx[li].long()], fs_live, li.numel())
    m = _check_rows(out, ref, li, "%s ray mode n=%d" % (name, n))
    if n > 3007:
        _print(name + " ray mode", li.numel(), m, ref)


# ---------------------------------------------------------------------------------------------------------------------
# (c) the device-side count n_dev
# ---------------------------------------------------------------------------------------------------------------------
def test_device_count(env):
    mdl = _model("env", env)
    S = env["S"]
    n = 16 * 24 * S + 300
    x, d = _points(n, mdl, 9)
    x01 = grad64.to_unit(x, mdl["lo"], mdl["hi"])
    for v in (n - 4321, 16 * 24 * S + 1, n + 5, 0, -3):
        eff = max(0, min(v, n))
        cnt = torch.tensor([v], device="cuda", dtype=torch.int32)
        smp = _N()._samples_struct(x, d)
        smp.n_dev = cnt.data_ptr()
        out = _forward(mdl, smp, n)
        torch.cuda.synchronize()
        for k in ("sig", "rgb", "h"):
            assert torch.isnan(out[k][eff:]).all(), "n_dev=%d: %s written at or past the count" % (v, k)
        if eff:
            ref = _reference(mdl, x01[:eff], d[:eff], out["fs"], eff)
            _check_rows(out, ref, slice(0, eff), "n_dev=%d" % v)


# ---------------------------------------------------------------------------------------------------------------------
# (d) rgb_act = 0 through the NgpNet field
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", ["17", "8*16W+7"])
def test_rgb_act_none(env, size):
    from ngp_pl_b200 import _lib
    mdl = _model("env", env)
    n = _sizes(env["S"])[size]
    x, d = _points(n, mdl, 11)
    net = _lib.NgpNet.from_buffer_copy(mdl["net"])
    net.rgb_act = 0
    out = _forward(mdl, _N()._samples_struct(x, d), n, net=net)
    torch.cuda.synchronize()
    ref = _reference(mdl, grad64.to_unit(x, mdl["lo"], mdl["hi"]), d, out["fs"], n, rgb_act=0)
    m = _check_rows(out, ref, slice(0, n), "rgb_act=0 n=%d" % n)
    assert (out["rgb"] < 0).any() or (out["rgb"] > 1).any()  # no sigmoid
    if n > 3007:
        _print("rgb_act=0", n, m, ref)


# ---------------------------------------------------------------------------------------------------------------------
# (e) the stand-alone module kernels and the h output of tcnn.NetworkWithInputEncoding
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES)
def test_module_kernels_vs_float64(env, size):
    mdl = _model("env", env)
    n = _sizes(env["S"])[size]
    L = _L()
    g = torch.Generator(device="cuda").manual_seed(13 + n)
    # ngp_mlp_rgb_forward on fp16 inputs, both activations
    xin = (torch.rand(n, 32, device="cuda", generator=g) * 2 - 1).half()
    for act in (1, 0):
        out = _filled((n, 3), torch.float16)
        _chk(L.ngp_mlp_rgb_forward(mdl["rgb_h"].data_ptr(), xin.data_ptr(), n, act, out.data_ptr(), _st()), "mlp_rgb_forward")
        torch.cuda.synchronize()
        f = grad64.rgb_forward(xin, torch.zeros(n, 32, device="cuda"), mdl["rgb_h"], act, carry=True)
        m = _ratio(out, f["out"], f["d_out"], "mlp_rgb_forward act=%d" % act)
        if n > 3007:
            print("MEASURED mlp_rgb_forward act=%d n=%d: %.4f bitwise, worst %.3f of 2x bound" % (act, n, m[0], m[1]))
    # ngp_sh_encode
    u = torch.rand(n, 3, device="cuda", generator=g)
    u[: min(n, 2)] = torch.tensor([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]], device="cuda")[: min(n, 2)]
    sh = _filled((n, 16), torch.float16)
    _chk(L.ngp_sh_encode(u.data_ptr(), n, sh.data_ptr(), _st()), "sh_encode")
    torch.cuda.synchronize()
    v, dv = grad64.sh_encode(u)
    m = _ratio(sh, v, dv, "sh_encode")
    if n > 3007:
        print("MEASURED sh_encode n=%d: %.4f bitwise, worst %.3f of 2x bound" % (n, m[0], m[1]))
    # tcnn.NetworkWithInputEncoding: h from positions in [0, 1]^3, end to end (the features' bounds carried through)
    mod = mdl["model"].xyz_encoder
    x01 = torch.rand(n, 3, device="cuda", generator=g)
    with torch.no_grad():
        h = mod(x01)
    feat, d_feat = grad64.grid_encode(mod.meta, _f16(mod.half_params())[3072:].view(-1, 2), x01)
    f = grad64.mlp_forward(feat, torch.zeros(n, 16, device="cuda", dtype=torch.float64), _f16(mod.half_params())[:3072],
                           mdl["rgb_h"], 1, carry=True, d_feat=d_feat)
    m = _ratio(h, f["h"], f["d_h"], "NetworkWithInputEncoding h")
    if n > 3007:
        print("MEASURED NetworkWithInputEncoding h n=%d: %.4f bitwise, worst %.3f of 2x bound" % (n, m[0], m[1]))


# ---------------------------------------------------------------------------------------------------------------------
# (f) the tile scheduler: slot reuse after the pool wraps, concurrent launches, graph replays
# ---------------------------------------------------------------------------------------------------------------------
def _same(a, b):
    """bitwise equality of two output dicts (NaN-safe)"""
    bits = lambda t: t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)  # noqa: E731
    return all(torch.equal(bits(a[k]), bits(b[k])) for k in ("sig", "rgb", "h") if a[k] is not None)


def test_scheduler_slots_wrap(env):
    """1,100 forward launches interleaved with backward launches (which take slots from the same pool of 1,024): every
    launch equals the first bit for bit, also after every slot has been used and re-armed"""
    mdl = _model("env", env)
    S = env["S"]
    n = 16 * 24 * S + 77
    x, d = _points(n, mdl, 17)
    smp = _N()._samples_struct(x, d)
    first = _forward(mdl, smp, n)
    nb = 3 * 192
    xb, db = x[:nb].contiguous(), d[:nb].contiguous()
    smpb = _N()._samples_struct(xb, db)
    g = torch.Generator(device="cuda").manual_seed(18)
    up_sig = torch.randn(nb, device="cuda", generator=g) * 1e-2
    up_rgb = torch.randn(nb, 3, device="cuda", generator=g) * 1e-1
    ws = torch.empty(_L().ngp_net_backward_workspace(nb), device="cuda", dtype=torch.uint8)
    ge, gr = torch.zeros(mdl["model"].xyz_encoder.params.numel(), device="cuda"), torch.zeros(7168, device="cuda")
    fsb = _forward(mdl, smpb, nb)["fs"]
    bad = []
    out = first
    for i in range(1100):
        out = _forward(mdl, smp, n, h_out=(i % 2 == 0), feat_save=False)
        if not (_same(first, out) if out["h"] is not None else _same(dict(first, h=None), out)):
            bad.append(i)
        if i % 3 == 0:
            _chk(_L().ngp_net_backward(C.byref(mdl["net"]), C.byref(smpb), up_sig.data_ptr(), up_rgb.data_ptr(),
                                       fsb.data_ptr(), env["scale_t"].data_ptr(), ge.data_ptr(), gr.data_ptr(),
                                       ws.data_ptr(), ws.numel(), _st()), "backward")
    torch.cuda.synchronize()
    assert not bad, "launches %s differ from the first" % bad[:10]
    assert torch.isfinite(out["sig"]).all() and torch.isfinite(out["rgb"]).all()


def test_scheduler_concurrent_streams(env):
    """two forwards in flight at once on two streams, with different inputs: each equals its own single-stream run"""
    mdl = _model("env", env)
    S = env["S"]
    n = 4 * 16 * 24 * S + 5
    xa, da = _points(n, mdl, 21)
    xb, db = _points(n, mdl, 22)
    sa, sb = _N()._samples_struct(xa, da), _N()._samples_struct(xb, db)
    ref_a, ref_b = _forward(mdl, sa, n), _forward(mdl, sb, n)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    oks = []
    for _ in range(4):
        a = _forward(mdl, sa, n, stream=s1)
        b = _forward(mdl, sb, n, stream=s2)
        torch.cuda.synchronize()
        oks.append(_same(ref_a, a) and _same(ref_b, b))
    assert all(oks)
    assert not torch.equal(ref_a["sig"], ref_b["sig"])


def test_scheduler_graph_replays(env):
    """a forward captured into a CUDA graph keeps its slot; three replays give the same outputs as an eager launch"""
    mdl = _model("env", env)
    S = env["S"]
    n = 2 * 16 * 24 * S + 9
    x, d = _points(n, mdl, 31)
    smp = _N()._samples_struct(x, d)
    eager = _forward(mdl, smp, n)
    out = dict(sig=_filled((n,)), rgb=_filled((n, 3)), h=_filled((n, 16), torch.float16))
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        _chk(_L().ngp_net_forward(C.byref(mdl["net"]), C.byref(smp), 1, out["sig"].data_ptr(), out["rgb"].data_ptr(),
                                  out["h"].data_ptr(), None, side.cuda_stream), "forward (capture)")
    reps = []
    for _ in range(3):
        for v in out.values():
            v.fill_(NAN)
        graph.replay()
        torch.cuda.synchronize()
        reps.append({k: v.clone() for k, v in out.items()})
    for r in reps:
        assert _same(r, reps[0]) and _same(r, eager)
