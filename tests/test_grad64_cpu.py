"""The float64 backward reference (oracle/grad64.py) against the existing restatements, so that a wrong reference cannot
silently agree with a wrong kernel (tests/test_backward_fp64_gpu.py compares the kernels with it):
  * its network backward against fp32 autograd of oracle.torch_ngp_forward (rgb_act 0 and 1);
  * its table scatter against float64 autograd of oracle.torch_grid_encode (dense, hashed and wrapping corners);
  * its feat_save decoder against a plain encoder of the documented fragment layout;
  * its two halves, rgb_backward and density_backward (the stand-alone module kernels' chains), against float64 autograd
    at the kernels' rounding points, and their bounds around an fp32 restatement of the kernels;
  * mlp_backward(carry=True), whose bounds follow every forward flip to the end: the same values as the one-flip model,
    bounds and undecided rows that contain it, and a fp32 restatement of k_ngp_bwd3 inside its bounds;
  * mlp_backward against its own stored outputs (tests/golden/grad64_mlp_backward.npz), so that a change to the forward
    it shares with mlp_forward shows.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import grad64

GOLDEN_MLP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grad64_mlp_backward.npz")


def _points(n, seed, lo=-0.5, hi=0.5):
    rng = np.random.RandomState(seed)
    x = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    d = (rng.normal(size=(n, 3)) * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    return torch.as_tensor(x), torch.as_tensor(d)


def _params(meta_total, seed, table_amp=0.5):
    """the modules' initialisation (ngp_pl_b200/tcnn.py) with an O(1) table, so every level matters"""
    g = torch.Generator().manual_seed(seed)
    enc = torch.empty(3072 + 2 * meta_total)
    enc[:2048].uniform_(-(6 / 96) ** 0.5, (6 / 96) ** 0.5, generator=g)
    enc[2048:3072].uniform_(-(6 / 80) ** 0.5, (6 / 80) ** 0.5, generator=g)
    enc[3072:].uniform_(-table_amp, table_amp, generator=g)
    rgb = torch.empty(7168)
    rgb[:2048].uniform_(-(6 / 96) ** 0.5, (6 / 96) ** 0.5, generator=g)
    rgb[2048:6144].uniform_(-(6 / 128) ** 0.5, (6 / 128) ** 0.5, generator=g)
    rgb[6144:].uniform_(-(6 / 80) ** 0.5, (6 / 80) ** 0.5, generator=g)
    return enc.half().float(), rgb.half().float()  # fp16-representable masters: the fp16 working copy is exact


@pytest.mark.parametrize("rgb_act", [1, 0])
def test_reference_chain_vs_fp32_autograd(oracle, rgb_act):
    meta, total = oracle.grid_meta(16, 19, 16, float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / 15))))
    enc, rgb = _params(total, 7)
    n = 300
    x, d = _points(n, 3)
    mn, mx = torch.full((1, 3), -0.5), torch.full((1, 3), 0.5)
    x01 = (x - mn) / (mx - mn)
    with torch.no_grad():
        feat = oracle.torch_grid_encode(meta, enc[3072:].view(-1, 2), x01).half()
    rng = np.random.RandomState(4)
    up_sig = torch.as_tensor((rng.normal(size=n) * 1e-2).astype(np.float32))
    up_rgb = torch.as_tensor((rng.normal(size=(n, 3)) * 1e-1).astype(np.float32))
    scale = 2.0 ** 10
    ref = grad64.mlp_backward(feat, grad64.sh4_64(d), enc[:3072], rgb, up_sig, up_rgb, scale, rgb_act)
    # rows whose ReLU masks the reference cannot pin down take no part (their branch may legitimately differ)
    keep = ~ref["ambiguous"]
    assert keep.sum() >= n - 3
    up_sig, up_rgb = up_sig * keep, up_rgb * keep[:, None]
    ref = grad64.mlp_backward(feat, grad64.sh4_64(d), enc[:3072], rgb, up_sig, up_rgb, scale, rgb_act)

    e, r = enc.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    sig, out, _ = oracle.torch_ngp_forward(meta, e, r, mn, mx, x, d, rgb_act=rgb_act)
    ((sig * up_sig).sum() + (out * up_rgb).sum()).backward()
    # autograd differentiates the sigmoid at its unrounded value o' = sigmoid(y), the kernel at o = fp16(o'):
    # |o' (1 - o') - o (1 - o)| <= 2^-11 o, i.e. 2^-11 o / (1 - o) of the out-gradient, carried linearly down the chain
    kappa = 0.0
    if rgb_act == 1:
        o = ref["o"]
        kappa = 2.0 ** -11 * float((o / (1 - o)).max())
    got = grad64.split_dW(e.grad.double(), r.grad.double())
    for k, (v, A, err) in ref["dW"].items():
        # the reference is an fp16-rounded chain, autograd an unrounded fp32 one: they differ by at most the reference's own
        # rounding bound, plus fp32 accumulation (2^-18 A) and the sigmoid term
        tol = err + (2.0 ** -18 + kappa) * A
        assert (got[k] - v).abs().le(tol).all(), "%s: max excess %g" % (k, float(((got[k] - v).abs() - tol).max()))
        assert v.abs().max() > 0
    # the table gradient: the reference's dfeat scattered, against autograd through the fp32 grid encoding
    tg, S, _ = grad64.grid_scatter(meta, x01, ref["dfeat"], 1.0 / scale, total)
    terr, _, _ = grad64.grid_scatter(meta, x01, ref["dfeat_err"] + kappa * ref["dfeat_abs"], 1.0 / scale, total)
    ag = e.grad[3072:].double().view(-1, 2)
    tol = terr + 2.0 ** -18 * grad64.grid_scatter(meta, x01, ref["dfeat_abs"], 1.0 / scale, total)[0] + 1e-30
    assert (ag - tg).abs().le(tol + 2.0 ** -20 * S).all()
    assert tg.abs().max() > 0


@pytest.mark.parametrize("cfg", [(16, 19), (4, 14)])
def test_reference_scatter_vs_float64_autograd(oracle, cfg):
    L, log2_T = cfg
    meta, total = oracle.grid_meta(L, log2_T, 16, float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / 15))))
    assert meta.hashed_mask != 0 and meta.hashed_mask != (1 << L) - 1  # dense and hashed levels both present
    n = 400
    rng = np.random.RandomState(11)
    x01 = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    # upper wrap of the dense levels, the last float below 1, and exact grid vertices of the finest dense level
    x01[:6] = [[1, 1, 1], [0, 0, 0], [1, 0, 1], [1 - 2 ** -24] * 3, [1, 1 - 2 ** -24, 0.5], [0.5, 0.25, 1]]
    l_dense = max(l for l in range(L) if not (meta.hashed_mask >> l) & 1)
    x01[6:20] = (rng.randint(0, int(meta.res[l_dense]), (14, 3)) / np.float32(meta.scale[l_dense])).astype(np.float32)
    x01 = torch.as_tensor(np.clip(x01, 0, 1))
    G = torch.as_tensor(rng.normal(size=(n, 32)).astype(np.float16)).double()
    G[:, 2 * L:] = 0
    table = torch.zeros(total, 2, dtype=torch.float64, requires_grad=True)
    feat = oracle.torch_grid_encode(meta, table, x01)
    (feat * G).sum().backward()
    ref, S, m = grad64.grid_scatter(meta, x01, G.half(), 1.0, total)
    assert (table.grad - ref).abs().le(1e-6 * S).all()
    assert int(m.sum()) == 8 * L * n and (ref != 0).sum() > 0


def _encode_np(feat):
    """feat (n, 32) float16 -> bytes of the fragment layout, written element by element from its description"""
    n = feat.shape[0]
    t = (n + 31) // 32 * 2
    out = np.zeros((t, 2, 32, 4, 2), np.float16)  # tile, kt, lane, word, half
    for row in range(n):
        tile, r = divmod(row, 16)
        g, rh = r % 8, r // 8
        for col in range(32):
            kt, c = divmod(col, 16)
            ch, cc = divmod(c, 8)
            q, half = divmod(cc, 2)
            word = 2 * ch + rh  # x: (g, 2q) y: (g + 8, 2q) z: (g, 2q + 8) w: (g + 8, 2q + 8)
            out[tile, kt, 4 * g + q, word, half] = feat[row, col]
    return out.tobytes()


def test_feat_save_decoder_vs_fragment_layout():
    rng = np.random.RandomState(5)
    for n in (1, 16, 37, 64):
        feat = rng.normal(size=(n, 32)).astype(np.float16)
        raw = torch.frombuffer(bytearray(_encode_np(feat)), dtype=torch.uint8)
        assert torch.equal(grad64.decode_feat_save(raw, n), torch.as_tensor(feat))
        assert torch.equal(grad64.encode_feat_save(torch.as_tensor(feat)), raw)
    # column 2 l (+1) is level l: level q lives in lane q's words x / y of k-tile 0
    raw = np.zeros(2 * 1024, np.uint8).view(np.float16)
    raw.reshape(2, 2, 32, 4, 2)[0, 0, 4 * 3 + 1, 1, 0] = 1.0  # tile 0, kt 0, g = 3, q = 1, word y (row g + 8), low half
    dec = grad64.decode_feat_save(torch.as_tensor(raw.view(np.uint8)), 16)
    assert dec[11, 2].item() == 1.0 and dec.abs().sum().item() == 1.0


def mlp_backward_outputs():
    """mlp_backward on one seeded batch of fp16 features (rgb_act 1 and 0): every output as a named float64 / bool array.
    The weight gradients are kept for rgb_act 1 only (they are most of the bytes)."""
    enc, rgb = _params(0, 13)
    g = torch.Generator().manual_seed(14)
    n = 48
    feat = (torch.rand(n, 32, generator=g) * 2 - 1).half()
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    up_sig = torch.randn(n, generator=g) * 1e-2
    up_rgb = torch.randn(n, 3, generator=g) * 1e-1
    out = {}
    for act in (1, 0):
        ref = grad64.mlp_backward(feat, grad64.sh4_64(d), enc[:3072].half(), rgb.half(), up_sig, up_rgb, 2.0 ** 10, act)
        keys = ["dfeat", "dfeat_err", "dfeat_abs", "ambiguous", "ambiguous_own", "hid", "h", "rin", "r1", "r2", "o"]
        for k in keys:
            out["act%d_%s" % (act, k)] = ref[k].numpy()
        for i, c in enumerate(ref["chain"]):
            out["act%d_chain%d" % (act, i)] = c.numpy()
        if act == 1:
            for k, (v, A, err) in ref["dW"].items():
                out["act1_dW_%s_v" % k], out["act1_dW_%s_A" % k], out["act1_dW_%s_err" % k] = v.numpy(), A.numpy(), err.numpy()
    return out


def test_mlp_backward_unchanged():
    """mlp_backward gives what it gave before its forward recompute became mlp_forward. Bounds and masks must not move;
    2^-40 relative leaves room only for another float64 summation order in the matrix products."""
    want = np.load(GOLDEN_MLP)
    got = mlp_backward_outputs()
    assert sorted(got) == sorted(want.files)
    for k in want.files:
        a, b = got[k], want[k]
        assert a.shape == b.shape and a.dtype == b.dtype, k
        if a.dtype == np.bool_:
            assert (a == b).all(), k
        else:
            assert (np.abs(a - b) <= 2.0 ** -40 * np.abs(b).max()).all(), k


def _within(got, want, bound, keep, what):
    """|got - want| <= 2 bound on the rows in keep; returns the worst ratio |got - want| / (2 bound) there"""
    got, want, bound = got.double(), want.double(), bound.double()
    if got.dim() == 1:
        got, want, bound = got[:, None], want[:, None], bound[:, None]
    err = (got - want).abs()[keep]
    b = 2 * bound[keep]
    bad = err > b
    assert not bad.any(), "%s: %d values outside 2 x bound, worst excess %g" % (what, int(bad.sum()), float((err - b).max()))
    return float((err / b.clamp_min(1e-300)).max())


@pytest.mark.parametrize("cfg", [(16, 19, 1), (4, 14, 1), (16, 19, 0)])
def test_interval_forward_contains_the_fp32_oracles(oracle, cfg):
    """grid_encode, mlp_forward(carry=True) and sigma contain the fp32 outputs of oracle.torch_ngp_forward and of the C
    oracle: both take the kernel's fp16 rounding points, so they differ from the float64 values only by fp32 arithmetic"""
    L, log2_T, act = cfg
    meta, total = oracle.grid_meta(L, log2_T, 16, float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / (L - 1)))))
    enc, rgb = _params(total, 21)
    n = 300
    x, d = _points(n, 22)
    x[:4] = torch.tensor([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5], [0.5, -0.5, 0.0], [0.0, 0.0, 0.0]])
    d[4:8] *= torch.tensor([[1e-6], [1e-3], [1e3], [1e6]])
    mn, mx = torch.full((1, 3), -0.5), torch.full((1, 3), 0.5)
    x01 = grad64.to_unit(x, [-0.5] * 3, [0.5] * 3)
    assert torch.equal(x01, (x - mn) / (mx - mn))
    feat, d_feat = grad64.grid_encode(meta, enc[3072:].half().view(-1, 2), x01)
    f = grad64.mlp_forward(feat, grad64.sh4_64(d), enc[:3072].half(), rgb.half(), act, carry=True, d_feat=d_feat)
    sig, d_sig = grad64.sigma(f["h"], f["d_h"])
    # no row is left out: a carried bound holds through a ReLU whose mask it leaves open (relu and the fp16 rounding are
    # monotone, so the kernel's value lies between the roundings of the interval's ends)
    keep = torch.ones(n, dtype=torch.bool)
    with torch.no_grad():
        ft = oracle.torch_grid_encode(meta, enc[3072:].view(-1, 2), x01)
        sig_t, rgb_t, h_t = oracle.torch_ngp_forward(meta, enc, rgb, mn, mx, x, d, rgb_act=act)
    sig_c, rgb_c, h_c = oracle.ngp_forward_c(meta, enc.numpy(), rgb.numpy(), mn.numpy(), mx.numpy(), x.numpy(), d.numpy(),
                                             rgb_act=act)
    _within(ft, feat, d_feat, keep, "torch features")
    assert (feat[:, 2 * L:] == 0).all() and (d_feat[:, 2 * L:] == 0).all()
    for name, (s_, r_, h_) in {"torch": (sig_t, rgb_t, h_t), "C": tuple(map(torch.as_tensor, (sig_c, rgb_c, h_c)))}.items():
        _within(h_, f["h"], f["d_h"], keep, name + " h")
        _within(s_, sig, d_sig, keep, name + " sigma")
        _within(r_, f["out"], f["d_out"], keep, name + " rgb")
    # the bounds stay tight: most feature bounds are zero (no rounding boundary within reach of the fp32 chain), and the
    # sigmoid's outputs are bounded to a few fp16 ulps even with every feature's possible flip carried through the net
    assert (d_feat == 0).double().mean() > 0.9
    if act == 1:
        assert (f["d_out"] <= 16 * 2.0 ** -11).all()


def test_sh_encode_and_ray_positions_restatements():
    """sh_encode against the fp32 SH of fmaf(u, 2, -1) rounded to fp16; ray_positions bit for bit against float32 fma,
    including sums that the float64 addition rounds onto a float32 halfway point"""
    from oracle.oracle import torch_sh4
    rng = np.random.RandomState(31)
    u = torch.as_tensor(rng.uniform(0, 1, (500, 3)).astype(np.float32))
    u[:3] = torch.tensor([[0, 0, 0], [1, 1, 1], [0.5, 0.25, 0.75]])
    v, dv = grad64.sh_encode(u)
    got = torch_sh4(torch.addcmul(torch.full_like(u, -1.0), u, torch.full_like(u, 2.0))).half().double()
    _within(got, v, dv, torch.ones(500, dtype=torch.bool), "sh")
    # fma(d, t, o) in float32: np.float32 has no fma, so take the correctly rounded exact value from Python fractions
    from fractions import Fraction
    o = rng.uniform(-1, 1, (40, 3)).astype(np.float32)
    dr = rng.normal(size=(40, 3)).astype(np.float32)
    ridx = rng.randint(-1, 40, 300).astype(np.int32)
    ts = rng.uniform(0, 3, 300).astype(np.float32)
    # halfway cases: o = 1, d t = 2^-24 + 2^-60 -> the float64 sum is 1 + 2^-24 exactly (a float32 tie), the fma rounds up
    o[0] = [1.0, 1.0, -1.0]
    dr[0] = [2.0 ** -24 + 2.0 ** -47, -(2.0 ** -24 + 2.0 ** -47), 2.0 ** -25 + 2.0 ** -48]
    ridx[:4] = 0
    ts[:4] = np.float32(1 + 2.0 ** -13)
    x = grad64.ray_positions(torch.as_tensor(o), torch.as_tensor(dr), torch.as_tensor(ridx), torch.as_tensor(ts)).numpy()
    for i in range(300):
        r = ridx[i]
        for k in range(3):
            if r < 0:
                assert x[i, k] == 0
                continue
            exact = Fraction(float(dr[r, k])) * Fraction(float(ts[i])) + Fraction(float(o[r, k]))
            lo = np.float32(float(exact))  # nearest double, then the float32 neighbours around it
            cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
            dist = [abs(Fraction(float(c)) - exact) for c in cands]
            best = min(dist)
            ties = [c for c, e in zip(cands, dist) if e == best]
            want = ties[0] if len(ties) == 1 else [c for c in ties if not (c.view(np.int32) & 1)][0]
            assert x[i, k] == want, (i, k, float(x[i, k]), float(want))


def _ste16(v):
    """fp16 rounding in the forward value, identity in the gradient (autograd then differentiates the unrounded chain at
    the kernel's rounded activations)"""
    return v + (grad64.f16(v.detach()) - v.detach())


@pytest.mark.parametrize("rgb_act", [1, 0])
def test_rgb_backward_vs_float64_autograd_and_fp32(rgb_act):
    """rgb_backward (k_mlp_rgb_bwd's chain from an external fp16 input) against float64 autograd of the rgb net at the
    kernel's rounding points, and its bounds around an fp32 restatement of the kernel"""
    _, rgb = _params(0, 41)
    g = torch.Generator().manual_seed(42)
    n = 300
    rin = (torch.rand(n, 32, generator=g) * 2 - 1).half()
    rin[torch.rand(n, 32, generator=g) < 0.05] = 0  # exact zeros
    up = torch.randn(n, 3, generator=g) * 1e-1
    scale = 2.0 ** 10
    rb = grad64.rgb_backward(rin, torch.zeros(n, 32), rgb.half(), up, scale, rgb_act)
    keep = ~rb["ambiguous"]
    assert keep.sum() >= n - 3
    up = up * keep[:, None]
    rb = grad64.rgb_backward(rin, torch.zeros(n, 32), rgb.half(), up, scale, rgb_act)
    assert (rb["fwd"]["r1"] == 0).any() and (rb["dX"] != 0).all(1).sum() > n // 2

    # float64 autograd; the output derivative is taken at the rounded output o, as the kernel takes it
    W = rgb.double().clone().requires_grad_(True)
    X = rin.double().requires_grad_(True)
    W1, W2, W3 = W[:2048].view(64, 32), W[2048:6144].view(64, 64), W[6144:].view(16, 64)[:3]
    r1 = _ste16(torch.relu(X @ W1.t()))
    r2 = _ste16(torch.relu(r1 @ W2.t()))
    yo = r2 @ W3.t()
    if rgb_act == 1:
        o = grad64.f16(torch.sigmoid(yo.detach()))
        s = o * (1 - o)
    else:
        s = torch.ones_like(yo)
    (yo * s * up.double()).sum().backward()
    got = grad64.split_dW(torch.zeros(3072, dtype=torch.float64), W.grad)
    for k, (v, A, err) in rb["dW"].items():
        assert (got[k] - v).abs().le(err + 1e-12 * A).all(), k
        assert v.abs().max() > 0
    assert (X.grad - rb["dX"]).abs().le(rb["dX_err"]).all()
    assert (got["W3r"][3:] == 0).all() and (rb["dW"]["W3r"][0][3:] == 0).all()

    # fp32 restatement at the kernel's rounding points: fp32 accumulation, fp16 activations and out-gradients
    def r16(v): return v.half().float()
    w = rgb.float()
    w1, w2, w3 = w[:2048].view(64, 32), w[2048:6144].view(64, 64), w[6144:].view(16, 64)
    x = rin.float()
    q1 = r16(torch.relu(x @ w1.t()))
    q2 = r16(torch.relu(q1 @ w2.t()))
    zo = q2 @ w3[:3].t()
    if rgb_act == 1:
        oo = r16(torch.sigmoid(zo))
        so = oo * (1 - oo)
    else:
        so = torch.ones_like(zo)
    dout = torch.zeros(n, 16)
    dout[:, :3] = r16(up * so * scale)
    dr2 = r16((dout @ w3) * (q2 > 0))
    dr1 = r16((dr2 @ w2) * (q1 > 0))
    dX = (dr1 @ w1) * (1 / scale)
    assert (dX.double() - rb["dX"]).abs()[keep].le(rb["dX_err"][keep]).all()
    # the fp32 weight-gradient sums over n rows: at most n roundings of 2^-24 of the running sum
    allow = n * 2.0 ** -24
    fw = {"W3r": dout.t() @ q2, "W2r": dr2.t() @ q1, "W1r": dr1.t() @ x}
    for k, (v, A, err) in rb["dW"].items():
        assert (fw[k].double() / scale - v).abs().le(err + allow * A).all(), k


def test_density_backward_vs_float64_autograd_and_fp32():
    """density_backward (k_enc_bwd's chain from a scaled fp16 dL/dh) against float64 autograd of the density MLP at the
    kernel's rounding points, and its bounds around an fp32 restatement of the kernel"""
    enc, _ = _params(0, 51)
    g = torch.Generator().manual_seed(52)
    n = 300
    feat = (torch.rand(n, 32, generator=g) * 2 - 1).half()
    feat[:, 22:] = 0  # 11 levels: the zero-padded feature columns
    # upstream dL/dh spread over five decades, some exact zeros, scaled as _pow2_scale does
    dL_dh = torch.randn(n, 16, generator=g) * 10 ** (torch.rand(n, 16, generator=g) * 5 - 7)
    dL_dh[torch.rand(n, 16, generator=g) < 0.05] = 0
    scale = 2.0 ** math.floor(math.log2(256 / dL_dh.abs().max().item()))
    dh, dh_err, dh_abs = grad64.scaled_dh(dL_dh, scale)
    assert (dh.abs().max() > 128) and (dh.abs().max() <= 256)
    db = grad64.density_backward(feat, enc[:3072].half(), dh, dh_err, dh_abs, scale)
    keep = ~db["ambiguous"]
    assert keep.sum() >= n - 3
    dh, dh_err, dh_abs = dh * keep[:, None], dh_err * keep[:, None], dh_abs * keep[:, None]
    db = grad64.density_backward(feat, enc[:3072].half(), dh, dh_err, dh_abs, scale)

    W = enc[:3072].double().clone().requires_grad_(True)
    F = feat.double().requires_grad_(True)
    W1, W2 = W[:2048].view(64, 32), W[2048:].view(16, 64)
    hid = _ste16(torch.relu(F @ W1.t()))
    (hid @ W2.t() * dh / scale).sum().backward()
    got = grad64.split_dW(W.grad, torch.zeros(7168, dtype=torch.float64))
    for k, (v, A, err) in db["dW"].items():
        assert (got[k] - v).abs().le(err + 1e-12 * A).all(), k
        assert v.abs().max() > 0
    assert (F.grad * scale - db["dfeat"]).abs().le(db["dfeat_err"]).all()
    assert (got["W1d"][:, 22:] == 0).all() and (db["dW"]["W1d"][0][:, 22:] == 0).all()

    def r16(v): return v.half().float()
    w = enc[:3072].float()
    w1, w2 = w[:2048].view(64, 32), w[2048:].view(16, 64)
    x = feat.float()
    hq = r16(torch.relu(x @ w1.t()))
    d16 = r16(dL_dh * scale) * keep[:, None]
    dhid = r16((d16 @ w2) * (hq > 0))
    dfeat = r16(dhid @ w1)
    assert (dfeat.double() - db["dfeat"]).abs()[keep].le(db["dfeat_err"][keep]).all()
    allow = n * 2.0 ** -24
    fw = {"W2d": d16.t() @ hq, "W1d": dhid.t() @ x}
    for k, (v, A, err) in db["dW"].items():
        assert (fw[k].double() / scale - v).abs().le(err + allow * A).all(), k


@pytest.mark.parametrize("rgb_act", [1, 0])
def test_mlp_backward_carry_contains_one_flip_model_and_fp32(oracle, rgb_act):
    """mlp_backward(carry=True) has mlp_backward's values; its bounds and undecided rows contain the one-flip model's;
    and an fp32 restatement of k_ngp_bwd3's chain (fp32 accumulation, fp16 activations and out-gradients, fp32 SH of the
    normalised direction) lies inside its bounds on every decided row, its weight gradients inside the carried
    weight-gradient bounds; and carry does widen the bounds"""
    from oracle.oracle import torch_sh4
    meta, total = oracle.grid_meta(16, 19, 16, float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / 15))))
    enc, rgb = _params(total, 51)
    n = 3000
    x, d = _points(n, 52)
    x01 = x + 0.5
    with torch.no_grad():
        feat = oracle.torch_grid_encode(meta, enc[3072:].view(-1, 2), x01).half()
    g = torch.Generator().manual_seed(53)
    up_sig = torch.randn(n, generator=g) * 1e-2
    up_rgb = torch.randn(n, 3, generator=g) * 1e-1
    scale = 2.0 ** 8
    args = (feat, grad64.sh4_64(d), enc[:3072].half(), rgb.half(), up_sig, up_rgb, scale, rgb_act)
    one, car = grad64.mlp_backward(*args), grad64.mlp_backward(*args, carry=True)
    for k in ("dfeat", "hid", "h", "rin", "r1", "r2", "o"):
        assert torch.equal(one[k], car[k]), k
    assert (car["dfeat_err"] >= one["dfeat_err"]).all()
    assert (car["ambiguous"] | ~one["ambiguous"]).all() and car["ambiguous"].double().mean() < 0.1
    for k, (v, A, err) in car["dW"].items():
        v1, A1, err1 = one["dW"][k]
        assert torch.equal(v, v1) and torch.equal(A, A1) and (err >= err1).all(), k

    def r16(v): return v.half().float()
    w, wr = enc[:3072].float(), rgb.float()
    w1d, w2d = w[:2048].view(64, 32), w[2048:3072].view(16, 64)
    w1r, w2r, w3r = wr[:2048].view(64, 32), wr[2048:6144].view(64, 64), wr[6144:].view(16, 64)
    hid = r16(torch.relu(feat.float() @ w1d.t()))
    h = r16(hid @ w2d.t())
    dn = d / torch.sqrt((d * d).sum(1, keepdim=True))
    rin = torch.cat([r16(torch_sh4(dn)), h], 1)
    q1 = r16(torch.relu(rin @ w1r.t()))
    q2 = r16(torch.relu(q1 @ w2r.t()))
    zo = q2 @ w3r[:3].t()
    oo = r16(torch.sigmoid(zo)) if rgb_act == 1 else zo
    so = oo * (1 - oo) if rgb_act == 1 else torch.ones_like(zo)
    dout = torch.zeros(n, 16)
    dout[:, :3] = r16(up_rgb * so * scale)
    dr2 = r16((dout @ w3r) * (q2 > 0))
    dr1 = r16((dr2 @ w2r) * (q1 > 0))
    c = dr1 @ w1r[:, 16:]
    c[:, 0] += up_sig * torch.exp(h[:, 0].clamp(-15, 15)) * scale
    dh = r16(c)
    dhid = r16((dh @ w2d) * (hid > 0))
    dfeat = r16(dhid @ w1d)
    keep = ~car["ambiguous"]
    assert ((dfeat.double() - car["dfeat"]).abs() <= car["dfeat_err"])[keep].all()
    # carry widens something: more undecided rows, and wider bounds of the feature and weight gradients
    assert car["ambiguous"].sum() > one["ambiguous"].sum()
    assert (car["dfeat_err"] > one["dfeat_err"]).any()
    assert any((car["dW"][k][2] > one["dW"][k][2]).any() for k in car["dW"])

    # the weight gradients of the fp32 restatement, over the rows the carried model decides (the others get no
    # upstream gradient): within the carried bound plus the fp32 sums' n roundings of 2^-24 of the absolute sum
    up_sig, up_rgb = up_sig * keep, up_rgb * keep[:, None]
    car = grad64.mlp_backward(feat, grad64.sh4_64(d), enc[:3072].half(), rgb.half(), up_sig, up_rgb, scale, rgb_act,
                              carry=True)
    assert not car["ambiguous"][keep].any()
    dout = torch.zeros(n, 16)
    dout[:, :3] = r16(up_rgb * so * scale)
    dr2 = r16((dout @ w3r) * (q2 > 0))
    dr1 = r16((dr2 @ w2r) * (q1 > 0))
    c = dr1 @ w1r[:, 16:]
    c[:, 0] += up_sig * torch.exp(h[:, 0].clamp(-15, 15)) * scale
    dh = r16(c)
    dhid = r16((dh @ w2d) * (hid > 0))
    fw = {"W3r": dout.t() @ q2, "W2r": dr2.t() @ q1, "W1r": dr1.t() @ rin, "W2d": dh.t() @ hid,
          "W1d": dhid.t() @ feat.float()}
    for k, (v, A, err) in car["dW"].items():
        assert (fw[k].double() / scale - v).abs().le(err + n * 2.0 ** -24 * A).all(), k
        assert v.abs().max() > 0, k
