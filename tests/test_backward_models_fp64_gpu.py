"""The MLP backward k_ngp_bwd3 and the hash-table scatter behind it against the float64 reference of oracle/grad64.py on
every model the forward is checked on (test_forward_fp64_gpu: L = 16 / T = 2^19, L = 4 / T = 2^14, scale 16, a trained
Lego), at the forward's special points, with rgb_act = 0, in ray mode with ray_idx = -1 slots and a device-side count,
through a live list, and on the batches of two real Trainer steps.

Sizes derive from the SM count S as in test_backward_fp64_gpu: k_ngp_bwd3 runs min(blocks, S) CTAs over 192-row blocks,
so S * 192 + 1 rows make one CTA take a second block and 8 * S * 192 + 37 rows make every CTA loop.

Every value is compared with 2 x its derived bound, never with a tolerance relative to a maximum:
  * feature gradients: grad64.mlp_backward's per-element bound, on every row whose ReLU masks the bound decides (the rows
    it leaves open are counted and reported, and they are still held to the bitwise saved-vs-re-gathered check);
  * weight gradients: the carried model's operand bound (grad64.mlp_backward(carry=True): every forward flip followed to
    the end, so it holds on every row it decides) plus the fp32 summation allowance of test_backward_fp64_gpu's
    sparse-rows test. The rows the carried model leaves open get zero upstream gradients (which rows are open depends
    on the forward alone), so no allowance is needed. Random-sign upstream gradients cancel in the sums far below that
    bound, so every launch is followed by one with sparse, sign-aligned upstream gradients (_dW_power): one marked row
    per 192-row block, whose contributions add up coherently in some element of every matrix, and the check must have
    the power to see a wrong matrix there (some |dW| > 2 x bound). The Trainer's own step cannot have its upstream
    gradients chosen: its weight gradients are held to the bound with an allowance for the open rows
    (_open_allowance) -- which only catches gross errors -- and the power check runs on its batch with the same
    device inputs;
  * the table gradient: grad64.grid_scatter from the kernel's own feature gradients, with the rigorous per-entry bound of
    test_backward_fp64_gpu's scatter test ((m + 2) 2^-24 sum |contribution|).
"""
import ctypes as C
import math

import pytest
import torch

from oracle import grad64
from test_backward_fp64_gpu import (BLK, SCALE, _L, _bwd_mlp, _check_rows, _chk, _dfeat, _dW, _st, _workspace,  # noqa: F401
                                    env)
from test_forward_fp64_gpu import MODELS, _forward, _model, _points, _ray_smp

pytestmark = pytest.mark.gpu

# a quiet fp16 NaN with a payload no arithmetic produces (the GPU's computed NaN is 0x7FFF): a workspace half holding
# it after a backward was never written
SENTINEL = 0x7E5A


def _sizes(S):
    return {"1": 1, "17": 17, "193": 193, "S*192+1": S * BLK + 1, "8*S*192+37": 8 * S * BLK + 37}


SIZES = ["1", "17", "193", "S*192+1", "8*S*192+37"]


def _net(mdl, rgb_act=None):
    from ngp_pl_b200 import _lib
    net = _lib.NgpNet.from_buffer_copy(mdl["net"])
    if rgb_act is not None:
        net.rgb_act = rgb_act
    return net


def _reference(enc_h, rgb_h, feat, dirs, up_sig, up_rgb, scale=SCALE, rgb_act=1):
    """mlp_backward's one-flip model, and the same with every forward flip carried to the end (carry=True)"""
    a = (feat, grad64.sh4_64(dirs), enc_h[:3072], rgb_h, up_sig, up_rgb, scale, rgb_act)
    return grad64.mlp_backward(*a), grad64.mlp_backward(*a, carry=True)


def _reference_chunked(enc_h, rgb_h, feat, dirs, up_sig, up_rgb, scale, rgb_act, chunk=1 << 17):
    """_reference over row chunks (a Trainer batch is too many rows for the float64 intermediates at once): the per-row
    outputs concatenated, the weight-gradient sums (value, A, err) added"""
    keys = ("dfeat", "dfeat_err", "ambiguous", "ambiguous_own")
    out = [dict(dW={}, **{k: [] for k in keys}), dict(dW={}, **{k: [] for k in keys})]
    for a in range(0, feat.shape[0], chunk):
        sl = slice(a, a + chunk)
        for acc, r in zip(out, _reference(enc_h, rgb_h, feat[sl], dirs[sl], up_sig[sl], up_rgb[sl], scale, rgb_act)):
            for k in keys:
                acc[k].append(r[k])
            for k, v in r["dW"].items():
                acc["dW"][k] = v if k not in acc["dW"] else tuple(x + y for x, y in zip(acc["dW"][k], v))
    for acc in out:
        for k in keys:
            acc[k] = torch.cat(acc[k])
    return out


def _rows(got, ref, refc, n_levels):
    """the feature gradients of the levels < L, row by row. Every row the one-flip model decides lies within its bound,
    except rows where a flip caused by another flip moved the chain: on the trained Lego a flip of hid can move h0 by an
    ulp (0.4 % on exp(h0) at |h0| > 4) or flip a colour-net mask. Those must lie within the carried bound (unless it
    leaves them undecided too) and be rare: at most 0.1 % of the rows. Returns the bitwise fraction (_check_rows), the
    mask of such rows, and the worst |got - reference| / (2 x bound) on the rest"""
    r1, rc = _cols(ref, n_levels), _cols(refc, n_levels)
    diff = (got.double() - r1["dfeat"]).abs()
    two = (diff > r1["dfeat_err"]).any(1) & ~r1["ambiguous"]
    inside = (diff <= rc["dfeat_err"]).all(1) | rc["ambiguous"]
    assert inside[two].all(), "%d rows outside the carried bound" % int((two & ~inside).sum())
    assert int(two.sum()) <= 1e-3 * got.shape[0] + 2, "%d rows outside the one-flip bound" % int(two.sum())
    r1 = dict(r1, ambiguous=r1["ambiguous"] | two)
    return _check_rows(got, r1), two, _dfeat_ratio(got, r1)


def _upstream(sig, seed):
    """upstream gradients shaped like a training step's: dL/drgb ~ 1e-1 and dL/dsigma ~ 1e-2 / max(1, sigma), so the
    density term dL/dsigma exp(h0) stays O(1e-2) and nothing overflows fp16 at the loss scale even where sigma is large"""
    n = sig.shape[0]
    g = torch.Generator(device="cuda").manual_seed(seed)
    up_sig = torch.randn(n, device="cuda", generator=g) * 1e-2 / torch.nan_to_num(sig, nan=1.0).clamp_min(1.0)
    up_rgb = torch.randn(n, 3, device="cuda", generator=g) * 1e-1
    return up_sig.contiguous(), up_rgb.contiguous()


def _backward(net, smp, up_sig, up_rgb, fs, n_ws, n_params, scale_t, full=True):
    """ngp_net_backward (or only its MLP half) into zeroed gradients and a workspace filled with SENTINEL"""
    ws = _workspace(n_ws)
    ws.view(torch.int16).fill_(SENTINEL)
    ge = torch.zeros(n_params if full else 3072, device="cuda")
    gr = torch.zeros(7168, device="cuda")
    fn = _L().ngp_net_backward if full else _L().ngp_net_backward_mlp
    _chk(fn(C.byref(net), C.byref(smp), up_sig.data_ptr(), up_rgb.data_ptr(), fs.data_ptr() if fs is not None else None,
            scale_t.data_ptr(), ge.data_ptr(), gr.data_ptr(), ws.data_ptr(), ws.numel(), _st()), "backward")
    return ge, gr, ws


def _untouched(ws, n_ws, rows, n_levels=16):
    """workspace halves of rows `rows` (all levels < n_levels) still hold SENTINEL"""
    d = _dfeat(ws, n_ws).view(torch.int16)[rows, :2 * n_levels]
    return bool((d == SENTINEL).all())


def _dfeat_ratio(got, ref):
    """worst |got - reference| / (2 x bound) over the rows the bound decides"""
    amb = ref["ambiguous"]
    err = (got.double() - ref["dfeat"]).abs()[~amb]
    b = ref["dfeat_err"][~amb]
    r = torch.where(err > 0, err / (2 * b).clamp_min(1e-300), torch.zeros_like(err))
    return float(r.max()) if r.numel() else 0.0


def _open_allowance(enc_h, rgb_h, feat, dirs, up_sig, up_rgb, scale, rgb_act):
    """for rows whose ReLU masks the reference leaves open (the kernel may take either branch): a bound of what those rows
    contribute to each weight gradient in any branch -- the absolute-value out-gradient chain with every mask open
    (|o (1 - o)| <= 1/4; exp(h0) widened by h0's fp16 ulp) times the layer inputs widened by their carried forward bounds,
    with 2^-7 for the chain's fp16 roundings and accumulations. -> {name: (out, in) float64}, unscaled"""
    d = torch.float64
    if feat.shape[0] == 0:
        return {}
    f = grad64.mlp_forward(feat, grad64.sh4_64(dirs), enc_h[:3072], rgb_h, rgb_act, carry=True)
    Wr, Wd = rgb_h.to(d), enc_h[:3072].to(d)
    W1r, W2r, W3r = Wr[:2048].view(64, 32).abs(), Wr[2048:6144].view(64, 64).abs(), Wr[6144:7168].view(16, 64).abs()
    W2d = Wd[2048:3072].view(16, 64).abs()
    dout = torch.zeros(feat.shape[0], 16, dtype=d, device=feat.device)
    dout[:, :3] = up_rgb.to(d).abs() * (0.25 if rgb_act == 1 else 1.0) * scale
    dr2 = dout @ W3r
    dr1 = dr2 @ W2r
    dh = dr1 @ W1r[:, 16:]
    h0 = f["h"][:, 0]
    dh[:, 0] += up_sig.to(d).abs() * torch.exp((h0 + 2.0 ** -9 * h0.abs() + f["d_h"][:, 0]).clamp(max=15)) * scale
    dhid = dh @ W2d
    wid = lambda k: f[k].abs() + f["d_" + k]  # noqa: E731
    c = (1 + 2.0 ** -7) / scale
    return {"W3r": c * dout.t() @ wid("r2"), "W2r": c * dr2.t() @ wid("r1"), "W1r": c * dr1.t() @ wid("rin"),
            "W2d": c * dh.t() @ wid("hid"), "W1d": c * dhid.t() @ feat.to(d).abs()}


def _sum_allowance(n, S):
    """fp32 summation of the weight gradients: 12 k-steps per 192-row block, ceil(blocks / S) blocks per CTA, then S CTA
    reductions, each rounding by <= 2^-24 of the absolute sum (2^-22 a step leaves room for the tensor core's own
    accumulation); never below test_backward_fp64_gpu's 2^-14"""
    n_add = 12 * math.ceil(math.ceil(n / BLK) / S) + S
    return max(2.0 ** -14, n_add * 2.0 ** -22)


def _check_dW(ge, gr, ref, allow_open, sum_allow, what):
    """every weight-gradient element within 2 x its bound; returns the worst |got - reference| / (2 x bound)"""
    got = _dW(ge, gr)
    worst = 0.0
    for k, (v, A, err) in ref["dW"].items():
        bound = err + sum_allow * A + 2 * allow_open.get(k, 0.0)
        e = (got[k] - v).abs()
        assert torch.isfinite(got[k]).all(), "%s %s: non-finite" % (what, k)
        bad = e > 2 * bound
        assert not bad.any(), "%s %s: %d elements outside 2 x bound, worst excess %g" % (
            what, k, int(bad.sum()), float((e - 2 * bound).max()))
        r = torch.where(e > 0, e / (2 * bound).clamp_min(1e-300), torch.zeros_like(e))
        worst = max(worst, float(r.max()))
    return worst


def _open_rows(enc_h, rgb_h, feat, dirs, rgb_act=1):
    """the rows whose ReLU masks the carried model leaves open: a property of the forward alone"""
    return grad64.mlp_forward(feat, grad64.sh4_64(dirs), enc_h[:3072], rgb_h, rgb_act, carry=True)["ambiguous"]


def _dW_power(net, smp, fs, n_ws, sample, feat, dirs, sig, ok, enc_h, rgb_h, scale, scale_t, S, what, rgb_act=1):
    """the weight gradients of a launch with sparse upstream gradients, against float64 with the carried bound, and with
    the power to fail. Launch row r stands for sample sample[r] (its upstream slot); feat / dirs / sig are per row; ok
    marks the rows that may carry a gradient (valid, and decided by the carried model). Marked rows: every row below
    2 x 192, else one random row per 192-row block. They take turns in three groups:
      A  dL/dsigma > 0, no colour gradient: dh = (dh0 > 0, 0, ...), so dW2d[0, :] = sum dh0 hid (hid >= 0) adds up;
      B  dL/dsigma with the sign of the row's first feature, no colour gradient: dW1d[i, 0] = sum [hid_i > 0] dh0 W2d[0, i]
         feat_0 has one sign for each i and adds up;
      C  dL/dred > 0 only: dout >= 0 in one column, so dW3r[0, :] = sum dout r2 and dW2r[j, :] = sum [r2_j > 0] dout
         W3r[0, j] r1 (r1, r2 >= 0) add up; dW1r's inputs (SH) change sign, so it has only its sum over fewer rows.
    Returns (worst |got - reference| / (2 x bound), the smallest over the matrices of max |reference| / (2 x bound))."""
    n = ok.shape[0]
    g = torch.Generator(device="cuda").manual_seed(n)
    if n < 2 * BLK:
        rows = torch.arange(n, device="cuda")
    else:
        nb = (n + BLK - 1) // BLK
        size = torch.clamp(n - torch.arange(nb, device="cuda") * BLK, max=BLK)
        rows = torch.arange(nb, device="cuda") * BLK + (torch.rand(nb, device="cuda", generator=g) * size).long()
    rows = rows[ok[rows]]
    k = rows.numel()
    grp = torch.arange(k, device="cuda") % 3
    amp = SCALE / scale  # the out-gradients' size at 2^8 whatever the launch's loss scale: a Trainer's is far larger
    m = 1e-2 * amp / torch.nan_to_num(sig[rows], nan=1.0).clamp_min(1.0)
    sgn = torch.where(feat[rows, 0] >= 0, 1.0, -1.0).to(m.dtype)
    ups = torch.where(grp == 0, m, torch.where(grp == 1, sgn * m, torch.zeros_like(m)))
    upr = torch.zeros(k, 3, device="cuda")
    upr[:, 0] = torch.randn(k, device="cuda", generator=g).abs() * 1e-1 * amp * (grp == 2)
    up_sig = torch.zeros(n_ws, device="cuda")
    up_rgb = torch.zeros(n_ws, 3, device="cuda")
    up_sig[sample[rows]] = ups
    up_rgb[sample[rows]] = upr
    ge, gr, _ = _backward(net, smp, up_sig, up_rgb, fs, n_ws, 3072, scale_t, full=False)
    torch.cuda.synchronize()
    ref = grad64.mlp_backward(feat[rows], grad64.sh4_64(dirs[rows]), enc_h[:3072], rgb_h, ups, upr, scale, rgb_act,
                              carry=True)
    assert not ref["ambiguous"].any()
    got = _dW(ge, gr)
    worst, power = 0.0, float("inf")
    for key, (v, A, err) in ref["dW"].items():
        bound = err + _sum_allowance(n, S) * A
        e = (got[key] - v).abs()
        assert torch.isfinite(got[key]).all(), "%s sparse %s: non-finite" % (what, key)
        bad = e > 2 * bound
        assert not bad.any(), "%s sparse %s: %d elements outside 2 x bound, worst excess %g" % (
            what, key, int(bad.sum()), float((e - 2 * bound).max()))
        worst = max(worst, float(torch.where(e > 0, e / (2 * bound).clamp_min(1e-300), torch.zeros_like(e)).max()))
        p = float(torch.where(v != 0, v.abs() / (2 * bound).clamp_min(1e-300), torch.zeros_like(v)).max())
        if k >= 64:
            # a matrix written as zero (a dropped flush, a skipped layer) falls outside the bound somewhere. (With a
            # handful of marked rows a group may have no gradient at all: a saturated sigmoid gives o (1 - o) = 0.)
            assert p > 1, "%s sparse %s: no element the check could find wrong (power %.3g)" % (what, key, p)
        power = min(power, p)
    return worst, power


def _check_table(ge, meta, x01, dfeat, scale, total, what):
    """the table gradient against grad64.grid_scatter of the kernel's own feature gradients; returns the worst ratio"""
    ref, Sabs, m = grad64.grid_scatter(meta, x01, dfeat, 1.0 / scale, total)
    got = ge[3072:3072 + 2 * total].view(-1, 2).double()
    assert torch.isfinite(got).all(), what + ": non-finite table gradient"
    tol = (m[:, None] + 2) * 2.0 ** -24 * Sabs
    e = (got - ref).abs()
    bad = e > 2 * tol
    assert not bad.any(), "%s: %d table entries outside 2 x bound, worst excess %g" % (
        what, int(bad.sum()), float((e - 2 * tol).max()))
    assert ((got != 0) == (ref != 0)).double().mean() > 0.999
    r = torch.where(e > 0, e / (2 * tol).clamp_min(1e-300), torch.zeros_like(e))
    return float(r.max())


def _cols(ref, n_levels):
    """the reference's feature gradients of the levels < L (the only workspace halves the kernel writes)"""
    return dict(ref, dfeat=ref["dfeat"][:, :2 * n_levels], dfeat_err=ref["dfeat_err"][:, :2 * n_levels])


def _pad32(dfeat):
    """(n, 2 L) feature gradients -> (n, 32), zero for the levels >= L (which grid_scatter does not read)"""
    out = torch.zeros(dfeat.shape[0], 32, dtype=torch.float32, device=dfeat.device)
    out[:, :dfeat.shape[1]] = dfeat.float()
    return out


def _padding_zero(ge, n_levels):
    """dW1d's columns of the levels >= L (first-layer input padding) are exactly zero"""
    W1d = _dW(ge, torch.zeros(7168, device=ge.device))["W1d"]
    return bool((W1d[:, 2 * n_levels:] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# (a) positions + directions with the special points: feature, weight and table gradients, every model and size
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", MODELS)
def test_rows_vs_float64(env, name, size):
    from ngp_pl_b200.models import networks as N
    mdl = _model(name, env)
    S = env["S"]
    n = _sizes(S)[size]
    L_ = int(mdl["meta"].n_levels)
    total = int(mdl["meta"].offset[L_])
    x, d = _points(n, mdl, 200 + n)
    smp = N._samples_struct(x, d)
    out = _forward(mdl, smp, n)
    up_sig, up_rgb = _upstream(out["sig"], 300 + n)
    feat = grad64.decode_feat_save(out["fs"], n)
    opn = _open_rows(mdl["enc_h"], mdl["rgb_h"], feat, d)
    up_sig, up_rgb = up_sig * ~opn, up_rgb * ~opn[:, None]
    ref, refc = _reference(mdl["enc_h"], mdl["rgb_h"], feat, d, up_sig, up_rgb)
    net = _net(mdl)
    # the whole backward from the saved features, into a workspace whose every half starts as SENTINEL: the levels >= L
    # are never written by the MLP backward and never read by the scatter
    ge, gr, ws = _backward(net, smp, up_sig, up_rgb, out["fs"], n, 3072 + 2 * total, env["scale_t"])
    # the MLP half from re-gathered features: the same fp16 features enter the same chain, bit for bit
    _, _, ws0 = _bwd_mlp(dict(net=net, scale_t=env["scale_t"]), smp, up_sig, up_rgb, None)
    torch.cuda.synchronize()
    got = _dfeat(ws, n)
    bits = got.view(torch.int16)
    assert (bits[:, 2 * L_:] == SENTINEL).all(), "workspace rows of levels >= L written"
    got = got[:, :2 * L_]
    eq, two, rf = _rows(got, ref, refc, L_)
    assert torch.equal(_dfeat(ws0, n)[:, :2 * L_].view(torch.int16), got.view(torch.int16)), "re-gathered != saved"
    rw = _check_dW(ge, gr, refc, {}, _sum_allowance(n, S), "%s n=%d" % (name, n))
    pw = _dW_power(net, smp, out["fs"], n, torch.arange(n, device="cuda"), feat, d, out["sig"], ~opn, mdl["enc_h"],
                   mdl["rgb_h"], SCALE, env["scale_t"], S, "%s n=%d" % (name, n))
    assert _padding_zero(ge, L_), "dW1d padding columns not zero"
    x01 = grad64.to_unit(x, mdl["lo"], mdl["hi"])
    rt = _check_table(ge, mdl["meta"], x01, _pad32(got), SCALE, total, "%s n=%d" % (name, n))
    if n > 10000:
        _print(name, n, eq, rf, rw, rt, ref, refc, two, pw)


def _print(what, n, eq, rf, rw, rt, ref, refc, two, pw):
    print("MEASURED %s n=%d: dfeat %.4f bitwise, worst %.3f of 2x bound; dW worst %.3f; table worst %.3f; sparse dW "
          "worst %.3f, power %.1f; rows undecided: %d own, %d one-flip, %d carried; %d held to the carried bound"
          % (what, n, eq, rf, rw, rt, pw[0], pw[1], int(ref["ambiguous_own"].sum()), int(ref["ambiguous"].sum()),
             int(refc["ambiguous"].sum()), int(two.sum())))


# ---------------------------------------------------------------------------------------------------------------------
# (b) rgb_act = 0 through the NgpNet field: the out-gradient is up x scale, without the sigmoid derivative
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["env", "lego"])
def test_rgb_act_none(env, name):
    from ngp_pl_b200.models import networks as N
    mdl = _model(name, env)
    S = env["S"]
    n = 8 * S * BLK + 37
    L_ = int(mdl["meta"].n_levels)
    x, d = _points(n, mdl, 17)
    smp = N._samples_struct(x, d)
    net = _net(mdl, rgb_act=0)
    out = _forward(mdl, smp, n, net=net)
    up_sig, up_rgb = _upstream(out["sig"], 18)
    feat = grad64.decode_feat_save(out["fs"], n)
    opn = _open_rows(mdl["enc_h"], mdl["rgb_h"], feat, d, 0)
    up_sig, up_rgb = up_sig * ~opn, up_rgb * ~opn[:, None]
    ref, refc = _reference(mdl["enc_h"], mdl["rgb_h"], feat, d, up_sig, up_rgb, rgb_act=0)
    ge, gr, ws = _backward(net, smp, up_sig, up_rgb, out["fs"], n, 3072, env["scale_t"], full=False)
    _, _, ws0 = _bwd_mlp(dict(net=net, scale_t=env["scale_t"]), smp, up_sig, up_rgb, None)
    torch.cuda.synchronize()
    got = _dfeat(ws, n)[:, :2 * L_]
    eq, two, rf = _rows(got, ref, refc, L_)
    assert torch.equal(_dfeat(ws0, n)[:, :2 * L_].view(torch.int16), got.view(torch.int16)), "re-gathered != saved"
    rw = _check_dW(ge, gr, refc, {}, _sum_allowance(n, S), "rgb_act=0 %s" % name)
    pw = _dW_power(net, smp, out["fs"], n, torch.arange(n, device="cuda"), feat, d, out["sig"], ~opn, mdl["enc_h"],
                   mdl["rgb_h"], SCALE, env["scale_t"], S, "rgb_act=0 %s" % name, rgb_act=0)
    # the sigmoid's derivative (<= 1/4) would move the rgb out-gradient far outside the bound
    assert (out["rgb"] < 0).any() or (out["rgb"] > 1).any()
    _print("rgb_act=0 " + name, n, eq, rf, rw, 0.0, ref, refc, two, pw)


# ---------------------------------------------------------------------------------------------------------------------
# (c) ray mode: positions fma(d, t, o), directions from rays_d through ray_idx, -1 slots, the count on the device; then
#     the same batch through a live list
# ---------------------------------------------------------------------------------------------------------------------
def _ray_batch(mdl, n, seed):
    """rays with unnormalised directions (four of them scaled by 1e-6 ... 1e6, their samples' t scaled back), every
    third slot -1, samples inside and outside the box"""
    s = mdl["scale"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    R = 2048
    o = ((torch.rand(R, 3, device="cuda", generator=g) * 2 - 1) * s * 0.8).contiguous()
    dr = torch.randn(R, 3, device="cuda", generator=g) * (0.5 + 1.5 * torch.rand(R, 1, device="cuda", generator=g))
    rs = torch.ones(R, device="cuda")
    rs[:4] = torch.tensor([1e-6, 1e-3, 1e3, 1e6], device="cuda")
    dr = (dr * rs[:, None]).contiguous()
    ridx = torch.randint(0, R, (n,), device="cuda", generator=g, dtype=torch.int32)
    ridx[:8] = torch.arange(8, device="cuda", dtype=torch.int32) % 4
    ridx[2::3] = -1
    ts = (torch.rand(n, device="cuda", generator=g) * 1.2 * s / rs[ridx.long().clamp_min(0)]).contiguous()
    return o, dr, ridx, ts


@pytest.mark.parametrize("name", ["env", "scale16", "lego"])
def test_ray_mode_vs_float64(env, name):
    mdl = _model(name, env)
    S = env["S"]
    n = 8 * S * BLK + 37
    n_dev_v = n - 1234  # rows at and past the device count are not samples
    L_ = int(mdl["meta"].n_levels)
    total = int(mdl["meta"].offset[L_])
    o, dr, ridx, ts = _ray_batch(mdl, n, 40)
    n_dev = torch.tensor([n_dev_v], device="cuda", dtype=torch.int32)
    out = _forward(mdl, _ray_smp(o, dr, ridx, ts, n, n_dev), n)
    slot = torch.arange(n, device="cuda")
    live = (ridx >= 0) & (slot < n_dev_v)
    li = live.nonzero()[:, 0]
    up_sig, up_rgb = _upstream(out["sig"], 41)
    # a slot that is not a sample carries NaN upstream gradients: reading them would poison the weight gradients
    up_sig[~live] = float("nan")
    up_rgb[~live] = float("nan")
    feat_all = grad64.decode_feat_save(out["fs"], n)
    dirs_all = dr[ridx.long().clamp_min(0)]
    feat, dirs = feat_all[li], dirs_all[li]
    opn = torch.zeros(n, dtype=torch.bool, device="cuda")
    opn[li] = _open_rows(mdl["enc_h"], mdl["rgb_h"], feat, dirs)
    up_sig[opn] = 0.0
    up_rgb[opn] = 0.0
    ref, refc = _reference(mdl["enc_h"], mdl["rgb_h"], feat, dirs, up_sig[li], up_rgb[li])
    x01 = grad64.to_unit(grad64.ray_positions(o, dr, ridx, ts)[li], mdl["lo"], mdl["hi"])
    n_params = 3072 + 2 * total
    dense = {}
    for mode, fs in (("saved", out["fs"]), ("re-gathered", None)):
        if fs is None:  # the re-gathered path has no live list and no scatter of its own: the MLP half
            ge, gr, ws = _backward(_net(mdl), _ray_smp(o, dr, ridx, ts, n, n_dev), up_sig, up_rgb, None, n, 3072,
                                   env["scale_t"], full=False)
        else:
            ge, gr, ws = _backward(_net(mdl), _ray_smp(o, dr, ridx, ts, n, n_dev), up_sig, up_rgb, fs, n, n_params,
                                   env["scale_t"])
        torch.cuda.synchronize()
        what = "%s ray mode %s" % (name, mode)
        assert _untouched(ws, n, ~live, L_), what + ": a -1 slot's or a row past the count's workspace written"
        got = _dfeat(ws, n)[li][:, :2 * L_]
        eq, two, rf = _rows(got, ref, refc, L_)
        rw = _check_dW(ge, gr, refc, {}, _sum_allowance(n, S), what)
        pw = _dW_power(_net(mdl), _ray_smp(o, dr, ridx, ts, n, n_dev), fs, n, slot, feat_all, dirs_all, out["sig"],
                       live & ~opn, mdl["enc_h"], mdl["rgb_h"], SCALE, env["scale_t"], S, what)
        rt = _check_table(ge, mdl["meta"], x01, _pad32(got), SCALE, total, what) if fs is not None else 0.0
        dense[mode] = (got, ge, gr)
        _print(what, li.numel(), eq, rf, rw, rt, ref, refc, two, pw)
    assert torch.equal(dense["saved"][0].view(torch.int16), dense["re-gathered"][0].view(torch.int16)), \
        "re-gathered != saved"

    # the live list: a permutation of the live slots plus some -1 slots (which the kernel must skip), past its count
    # more entries that must not be visited
    g = torch.Generator(device="cuda").manual_seed(42)
    neg = (ridx < 0).nonzero()[:, 0]
    pick = torch.cat([li, neg[torch.randperm(neg.numel(), device="cuda", generator=g)[:500]]])
    pick = pick[torch.randperm(pick.numel(), device="cuda", generator=g)]
    n_live = pick.numel()
    live_full = torch.cat([pick, slot[:777]]).to(torch.int32).contiguous()
    n_live_t = torch.tensor([n_live], device="cuda", dtype=torch.int32)
    smp = _ray_smp(o, dr, ridx, ts, n, n_dev)
    smp.live_idx, smp.n_live_dev = live_full.data_ptr(), n_live_t.data_ptr()
    ge, gr, ws = _backward(_net(mdl), smp, up_sig, up_rgb, out["fs"], n, n_params, env["scale_t"])
    torch.cuda.synchronize()
    what = "%s live list" % name
    is_live = live[pick.long()]
    rows = torch.arange(n, device="cuda")
    assert _untouched(ws, n, rows[n_live:], L_), what + ": a row past the live count written"
    assert _untouched(ws, n, rows[:n_live][~is_live], L_), what + ": the row of a -1 slot written"
    # each live row is the dense launch's row of its sample, bit for bit
    pos = torch.full((n,), -1, dtype=torch.long, device="cuda")
    pos[li] = torch.arange(li.numel(), device="cuda")
    got = _dfeat(ws, n)[:n_live][is_live][:, :2 * L_]
    assert torch.equal(got.view(torch.int16), dense["saved"][0][pos[pick[is_live].long()]].view(torch.int16))
    rw = _check_dW(ge, gr, refc, {}, _sum_allowance(n_live, S), what)
    x01l = grad64.to_unit(grad64.ray_positions(o, dr, ridx, ts)[pick], mdl["lo"], mdl["hi"])
    rt = _check_table(ge, mdl["meta"], x01l[is_live], _pad32(got), SCALE, total, what)
    pk = pick.long()
    pw = _dW_power(_net(mdl), smp, out["fs"], n, pk, feat_all[pk], dirs_all[pk], out["sig"][pk], live[pk] & ~opn[pk],
                   mdl["enc_h"], mdl["rgb_h"], SCALE, env["scale_t"], S, what)
    print("MEASURED %s n_live=%d: dW worst %.3f of 2x bound; table worst %.3f; sparse dW worst %.3f, power %.1f"
          % (what, n_live, rw, rt, pw[0], pw[1]))


# ---------------------------------------------------------------------------------------------------------------------
# (d) the Trainer's own batches: one step each of a config 5 shaped and a config 1 shaped Trainer; the backward's device
#     inputs are read back after it ran and its three outputs held to float64
# ---------------------------------------------------------------------------------------------------------------------
def _trainer_step(cfg):
    from ngp_pl_b200 import _lib, synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(0)
    if cfg == "c5":  # unbounded mip360-shaped scene, scale 16 (6 cascades), exp_step_factor 1/256, black background
        scene = synth.mip360_scene(0)
        model = NGP(scene.scale).cuda()
    else:            # the Lego-shaped scene on the L = 4, T = 2^14 model
        scene = synth.lego_scene(0)
        model = NGP(scene.scale, n_levels=4, log2_hashmap_size=14).cuda()
    bank = synth.RayBank(scene, n_images=8, device="cuda", seed=3)
    tr = Trainer(model, n_rays=4096, lr=1e-2, exp_step_factor=scene.exp_step_factor, bg=(scene.bg,) * 3)
    tr.attach_bank(bank)
    snap = {}

    def hook(t):  # after the backward, before the optimiser consumes the gradient and the weights change
        snap.update(G=t.G.clone(), Ph=t.Ph.clone(), ws=t.bwd_ws.clone(), dsig=t.dsigmas.clone(), drgb=t.drgbs.clone(),
                    scale=float(t.scalars[1]), live=t.live_idx.clone(), counters=t.counters.clone(),
                    fs=t.feat_save.clone(), rays_o=t.rays_o.clone(), rays_d=t.rays_d.clone(), ray_idx=t.ray_idx.clone(),
                    ts=t.ts.clone(), sig=t.sigmas.clone())

    tr.train_step(after_backward=hook)
    torch.cuda.synchronize()
    # the network as the backward saw it: the step's fp16 weights, before the optimiser changed them
    net = _lib.NgpNet.from_buffer_copy(tr.net)
    net.enc_params_h = snap["Ph"].data_ptr()
    net.rgb_params_h = snap["Ph"][tr.n_enc:].data_ptr()
    snap["net"] = net
    snap.update(cap=tr.capacity, n_enc=tr.n_enc, rgb_act=int(tr.net.rgb_act), meta=model.xyz_encoder.meta,
                lo=list(model._xyz_min_host), hi=list(model._xyz_max_host), cascades=model.cascades)
    return snap


@pytest.mark.parametrize("cfg", ["c5", "c1"])
def test_trainer_step_vs_float64(env, cfg):
    t = _trainer_step(cfg)
    S = env["S"]
    L_ = int(t["meta"].n_levels)
    total = int(t["meta"].offset[L_])
    assert (t["cascades"], L_) == ((6, 16) if cfg == "c5" else (1, 4))
    cap, n_enc = t["cap"], t["n_enc"]
    n = int(t["counters"][5])
    assert 1000 < n <= int(t["counters"][2]) <= cap
    scale = t["scale"]
    assert scale > 0 and math.frexp(scale)[0] == 0.5, "loss scale %r is not a power of two" % scale
    rows = t["live"][:n].long()
    r = t["ray_idx"][rows].long()
    assert (r >= 0).all()
    enc_h, rgb_h = t["Ph"][:3072], t["Ph"][n_enc:n_enc + 7168]
    feat = grad64.decode_feat_save(t["fs"], cap)[rows]
    dirs = t["rays_d"][r]
    up_sig, up_rgb = t["dsig"][rows], t["drgb"][rows]
    assert up_rgb.abs().max() > 0 and up_sig.abs().max() > 0
    ref, refc = _reference_chunked(enc_h, rgb_h, feat, dirs, up_sig, up_rgb, scale, t["rgb_act"])
    got = _dfeat(t["ws"], cap)[:n][:, :2 * L_]
    eq, two, rf = _rows(got, ref, refc, L_)
    op = refc["ambiguous"] | two
    allow = _open_allowance(enc_h, rgb_h, feat[op], dirs[op], up_sig[op], up_rgb[op], scale, t["rgb_act"])
    G = t["G"]
    rw = _check_dW(G[:n_enc], G[n_enc:n_enc + 7168], refc, allow, _sum_allowance(n, S), "trainer " + cfg)
    assert _padding_zero(G[:n_enc], L_)
    x01 = grad64.to_unit(grad64.ray_positions(t["rays_o"], t["rays_d"], t["ray_idx"][rows], t["ts"][rows]),
                         t["lo"], t["hi"])
    rt = _check_table(G[:n_enc], t["meta"], x01, _pad32(got), scale, total, "trainer " + cfg)
    # the step's own weight gradients are held only to the bound with the open rows' allowance (their upstream gradients
    # are the loss's); the power check reruns the MLP backward on the step's batch -- its rays, live list, saved
    # features, weights and loss scale -- with sparse sign-aligned upstream gradients
    from ngp_pl_b200 import _lib
    smp = _lib.NgpSamples()
    smp.xyzs = smp.dirs = None
    smp.rays_o, smp.rays_d = t["rays_o"].data_ptr(), t["rays_d"].data_ptr()
    smp.ray_idx, smp.ts = t["ray_idx"].data_ptr(), t["ts"].data_ptr()
    smp.n, smp.n_dev = cap, t["counters"][2:].data_ptr()
    smp.live_idx, smp.n_live_dev = t["live"].data_ptr(), t["counters"][5:].data_ptr()
    pw = _dW_power(t["net"], smp, t["fs"], cap, rows, feat, dirs, t["sig"][rows], ~refc["ambiguous"], enc_h, rgb_h,
                   scale, torch.tensor([scale], device="cuda"), S, "trainer " + cfg, rgb_act=t["rgb_act"])
    _print("trainer " + cfg, n, eq, rf, rw, rt, ref, refc, two, pw)
