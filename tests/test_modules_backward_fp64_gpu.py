"""The stand-alone module backward kernels (k_mlp_rgb_bwd behind ngp_mlp_rgb_backward, k_enc_bwd behind ngp_enc_backward)
and the drop-in chain that feeds them, against the float64 reference of oracle/grad64.py (rgb_backward, density_backward,
grid_scatter).

These kernels serve every caller that runs the reference's NGP one module at a time (xyz_encoder, SH, rgb_net). They
have their own out-gradient construction, tail handling, weight-gradient tile maps and persistent 128-row block loop,
none of it shared with k_ngp_bwd3. Each runs min(blocks, S) CTAs over 128-row blocks (S = SM count), so the sizes
straddle one tile, one block and one wave.

Every comparison is within 2 x the derived bound. Weight gradients add the fp32 summation allowance of _allow(). Rows
whose ReLU masks the reference cannot decide get a zero upstream gradient, so they contribute an exact zero on both
sides.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import grad64
from test_backward_fp64_gpu import MOD_BLK, SCALE, _chk, _dfeat, _f16, _L, _smp, _st, _workspace, env  # noqa: F401
from test_forward_fp64_gpu import _ratio

pytestmark = pytest.mark.gpu

SIZES = ["1", "15", "16", "17", "127", "128", "129", "S*128-1", "S*128+1", "8*S*128+37"]
SENTINEL = -12345.0


def _sizes(S):
    return {"1": 1, "15": 15, "16": 16, "17": 17, "127": 127, "128": 128, "129": 129, "S*128-1": S * MOD_BLK - 1,
            "S*128+1": S * MOD_BLK + 1, "8*S*128+37": 8 * S * MOD_BLK + 37}


def _allow(n, S):
    """fp32 summation allowance of a module kernel's weight gradient, relative to A = sum |products|. A CTA adds 8
    k-steps (16-row mma) per block into its accumulators for ceil(blocks / S) blocks; each mma may round by 4 x 2^-24 of
    the running sum (ACC32 = 2^-20 for 4 k-steps). Then up to S CTA partials meet in global memory, one rounding each."""
    blocks = (n + MOD_BLK - 1) // MOD_BLK
    return (4 * 8 * math.ceil(blocks / S) + S + 1) * 2.0 ** -24


def _check_dW(got, ref_dW, allow, what):
    """every weight-gradient element within 2 x (operand bound + allow A); returns {name: (bitwise, worst ratio)}"""
    out = {}
    for k, (v, A, err) in ref_dW.items():
        out[k] = _ratio(got[k], v, err + allow * A, "%s %s" % (what, k))
        assert v.abs().max() > 0 or A.max() == 0, k
    return out


def _amb_rows(amb_own, amb):
    if amb.numel() >= 10000:
        # as in test_backward_fp64_gpu._check_rows: masks left open by a pre-activation's own accumulation error stay
        # under 0.1 % of the rows; counting one-ulp flips of the layer before, under 1 %
        assert amb_own.double().mean().item() < 1e-3, "%d ambiguous rows (own)" % int(amb_own.sum())
        assert amb.double().mean().item() < 1e-2, "%d ambiguous rows" % int(amb.sum())


# ---------------------------------------------------------------------------------------------------------------------
# ngp_mlp_rgb_backward
# ---------------------------------------------------------------------------------------------------------------------
def _rgb_inputs(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(n, 32, device="cuda", generator=g) * 2 - 1
    x[torch.rand(n, 32, device="cuda", generator=g) < 0.05] = 0  # exact zeros
    up = torch.randn(n, 3, device="cuda", generator=g) * 1e-1
    return x.half().contiguous(), up.contiguous()


def _rgb_ref(env, x, up, act, scale=SCALE):
    """rgb_backward with the ambiguous rows' upstream gradients zeroed: (reference, masked upstream)"""
    n = x.shape[0]
    zero = torch.zeros(n, 32, device="cuda")
    f = grad64.rgb_forward(x, zero, env["rgb_h"], act)
    _amb_rows(f["ambiguous_own"], f["ambiguous"])
    up = (up * ~f["ambiguous"][:, None]).contiguous()
    return grad64.rgb_backward(x, zero, env["rgb_h"], up, scale, act), up


def _rgb_bwd(env, x, up, act, n=None, dx=True, gr=None, scale_t=None):
    n = x.shape[0] if n is None else n
    gr = torch.zeros(7168, device="cuda") if gr is None else gr
    dX = torch.full((n + 40, 32), SENTINEL, device="cuda") if dx else None  # 40 rows past n must stay untouched
    st = env["scale_t"] if scale_t is None else scale_t
    _chk(_L().ngp_mlp_rgb_backward(env["rgb_h"].data_ptr(), x.data_ptr(), up.data_ptr(), n, act, st.data_ptr(),
                                   dX.data_ptr() if dx else None, gr.data_ptr(), _st()), "mlp_rgb_backward")
    return dX, gr


def _rgb_dW(gr):
    return {k: v.double() for k, v in grad64.split_dW(torch.zeros(3072, device="cuda"), gr).items() if k[-1] == "r"}


@pytest.mark.parametrize("act", [1, 0])
@pytest.mark.parametrize("size", SIZES)
def test_mlp_rgb_backward_vs_float64(env, size, act):
    S = env["S"]
    n = _sizes(S)[size]
    x, up = _rgb_inputs(n, 100 + 2 * n + act)
    ref, up = _rgb_ref(env, x, up, act)
    assert (ref["fwd"]["r1"] == 0).any() and (ref["fwd"]["r2"] == 0).any()  # negative pre-activations occur
    dX, gr = _rgb_bwd(env, x, up, act)
    _, gr0 = _rgb_bwd(env, x, up, act, dx=False)  # dL_dx = NULL: the weight gradients alone
    torch.cuda.synchronize()
    assert (dX[n:] == SENTINEL).all(), "rows past n written"
    mx = _ratio(dX[:n], ref["dX"], ref["dX_err"], "dL/dx")
    allow = _allow(n, S)
    got = _rgb_dW(gr)
    mw = _check_dW(got, ref["dW"], allow, "grad_rgb")
    _check_dW(_rgb_dW(gr0), ref["dW"], allow, "grad_rgb (dL_dx = NULL)")
    # W3r is 16 x 64 with rows 3..15 zero-padded: no gradient may reach them
    assert (got["W3r"][3:] == 0).all() and (_rgb_dW(gr0)["W3r"][3:] == 0).all()
    assert (ref["dX"] != 0).any()
    if n > 10000:
        print("MEASURED mlp_rgb_backward act=%d n=%d: dL/dx %.4f bitwise, worst %.3f of 2x bound; " % (act, n, *mx)
              + ", ".join("%s %.4f / %.3g" % (k, *v) for k, v in mw.items()) + " (bitwise / worst of 2x bound)")


# ---------------------------------------------------------------------------------------------------------------------
# ngp_enc_backward
# ---------------------------------------------------------------------------------------------------------------------
_ENC = {}


def _enc_module(env, L_, log2_T):
    """a tcnn.NetworkWithInputEncoding with a random O(1) table, so every level matters"""
    key = (L_, log2_T)
    if key not in _ENC:
        from ngp_pl_b200 import tcnn
        if key == (16, 19):
            m = env["model"].xyz_encoder
        else:
            b = float(np.exp(np.log(2048 * 0.5 / 16) / (L_ - 1)))
            m = tcnn.NetworkWithInputEncoding(
                3, 16, {"otype": "Grid", "type": "Hash", "n_levels": L_, "n_features_per_level": 2,
                        "log2_hashmap_size": log2_T, "base_resolution": 16, "per_level_scale": b, "interpolation": "Linear"},
                {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64,
                 "n_hidden_layers": 1}).cuda()
            g = torch.Generator().manual_seed(L_ * 100 + log2_T)
            with torch.no_grad():
                m.params[3072:] = ((torch.rand(m.params.numel() - 3072, generator=g) * 2 - 1) * 0.5).cuda()
        _ENC[key] = m
    return _ENC[key]


def _enc_forward(mod, x01):
    """the module's forward through ngp_net_forward (unit box, no rgb): h and the saved features"""
    from ngp_pl_b200.models import networks as N
    n = x01.shape[0]
    unet, keep = N._unit_net(mod)
    fs = torch.zeros(N.feat_save_bytes(n), device="cuda", dtype=torch.uint8)
    h = torch.empty(n, 16, device="cuda", dtype=torch.float16)
    sig = torch.empty(n, device="cuda")
    _chk(_L().ngp_net_forward(C.byref(unet), C.byref(_smp(x01, None)), 0, sig.data_ptr(), None, h.data_ptr(), fs.data_ptr(),
                              _st()), "forward")
    return h, fs


def _enc_bwd(mod, x01, dL_dh, fs, st, n=None):
    from ngp_pl_b200.models import networks as N
    n = x01.shape[0] if n is None else n
    unet, keep = N._unit_net(mod)
    ws = _workspace(n)
    ge = torch.zeros_like(mod.params)
    _chk(_L().ngp_enc_backward(C.byref(unet), C.byref(_smp(x01, None, n)), dL_dh.data_ptr(), fs.data_ptr(), st.data_ptr(),
                               ge.data_ptr(), ws.data_ptr(), ws.numel(), _st()), "enc_backward")
    return ge, ws


def _enc_inputs(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x01 = torch.rand(n, 3, device="cuda", generator=g)
    dL_dh = torch.randn(n, 16, device="cuda", generator=g) * 1e-1
    dL_dh[torch.rand(n, 16, device="cuda", generator=g) < 0.05] = 0
    return x01.contiguous(), dL_dh


def _enc_ref(mod, feat, dL_dh, scale=SCALE):
    """density_backward from the kernel's own features, the ambiguous rows' upstream gradients zeroed"""
    enc_h = _f16(mod.half_params())[:3072]
    dh = grad64.scaled_dh(dL_dh, scale)
    db = grad64.density_backward(feat, enc_h, *dh, scale)
    _amb_rows(db["ambiguous_own"], db["ambiguous"])
    dL_dh = (dL_dh * ~db["ambiguous"][:, None]).contiguous()
    return grad64.density_backward(feat, enc_h, *grad64.scaled_dh(dL_dh, scale), scale), dL_dh


def _enc_dW(ge):
    return {k: v.double() for k, v in grad64.split_dW(ge, torch.zeros(7168, device="cuda")).items() if k[-1] == "d"}


def _table_check(mod, x01, dfeat, got, inv_scale, what):
    """the table gradient against grid_scatter of the kernel's own feature gradients: each of the m_e products rounds
    once, each of the <= m_e + 1 fp32 additions once; entries no sample touches stay exactly 0"""
    ref, Sabs, m = grad64.grid_scatter(mod.meta, x01, dfeat, inv_scale, mod.n_entries)
    got = got[3072:].view(-1, 2).double()
    r = _ratio(got, ref, (m[:, None] + 2) * 2.0 ** -24 * Sabs, what)
    assert (got[m == 0] == 0).all(), what + ": untouched entries written"
    assert (ref != 0).any()
    return r


@pytest.mark.parametrize("cfg", ["L16_T19", "L11_T19", "L4_T14"])
@pytest.mark.parametrize("size", SIZES)
def test_enc_backward_vs_float64(env, size, cfg):
    L_, log2_T = {"L16_T19": (16, 19), "L11_T19": (11, 19), "L4_T14": (4, 14)}[cfg]
    S = env["S"]
    n = _sizes(S)[size]
    mod = _enc_module(env, L_, log2_T)
    x01, dL_dh = _enc_inputs(n, 200 + 3 * n + L_)
    _, fs = _enc_forward(mod, x01)
    feat = grad64.decode_feat_save(fs, n)
    assert (feat[:, 2 * L_:] == 0).all()
    ref, dL_dh = _enc_ref(mod, feat, dL_dh)
    ge, ws = _enc_bwd(mod, x01, dL_dh, fs, env["scale_t"])
    torch.cuda.synchronize()
    dfeat = _dfeat(ws, n)
    mf = _ratio(dfeat[:, :2 * L_], ref["dfeat"][:, :2 * L_], ref["dfeat_err"][:, :2 * L_], "dfeat")
    got = _enc_dW(ge)
    mw = _check_dW(got, ref["dW"], _allow(n, S), "grad_enc")
    # the first layer is zero-padded to 32 inputs: no gradient may reach the columns of absent levels
    assert (got["W1d"][:, 2 * L_:] == 0).all()
    # (grid_scatter reads the present levels' columns only: the workspace rows of absent levels are never written)
    mt = _table_check(mod, x01, dfeat, ge, 1.0 / SCALE, "table")
    if n > 10000:
        print("MEASURED enc_backward %s n=%d: dfeat %.4f bitwise, worst %.3f; " % (cfg, n, *mf)
              + ", ".join("%s %.4f / %.3g" % (k, *v) for k, v in mw.items())
              + "; table worst %.3g (bitwise / worst of 2x bound)" % mt[1])


# ---------------------------------------------------------------------------------------------------------------------
# every 128-row block counts: sparse upstream gradients, full launch vs compact launch vs float64
# ---------------------------------------------------------------------------------------------------------------------
def _sparse_rows(n, seed, ok):
    """marked rows, all of them where ok (the reference pins their masks down): 0, 15, 16, 127, one random row in every
    7th 128-row block and every row of the last, partial block. -> (the rows of the marked blocks, the mark, the blocks)"""
    n_blk = (n + MOD_BLK - 1) // MOD_BLK
    rng = np.random.RandomState(seed)
    okc = ok.cpu().numpy()
    marked = {r for r in (0, 15, 16, 127) if okc[r]}
    for b in range(0, n_blk - 1, 7):
        cand = np.nonzero(okc[b * MOD_BLK:(b + 1) * MOD_BLK])[0]
        marked.add(b * MOD_BLK + int(cand[rng.randint(len(cand))]))
    marked |= {r for r in range((n_blk - 1) * MOD_BLK, n) if okc[r]}
    blocks = sorted({r // MOD_BLK for r in marked})
    assert 0 in blocks and n_blk - 1 in blocks
    rows = torch.cat([torch.arange(b * MOD_BLK, min((b + 1) * MOD_BLK, n)) for b in blocks]).cuda()
    mark = torch.zeros(n, dtype=torch.bool, device="cuda")
    mark[torch.tensor(sorted(marked), device="cuda")] = True
    return rows, mark, blocks


def _block_effect(dO, In, rows, blocks, A, tol, scale):
    """smallest, over the marked blocks, of the largest |one block's contribution| / tol: > 1 means dropping or doubling
    any one block moves some element of the weight gradient past the tolerance. dO, In: compact rows."""
    starts = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(torch.tensor(
        [min((b + 1) * MOD_BLK, int(rows.max()) + 1) - b * MOD_BLK for b in blocks]), 0)])
    worst = float("inf")
    for i in range(len(blocks)):
        a, b = int(starts[i]), int(starts[i + 1])
        c = dO[a:b].t() @ In[a:b] / scale
        worst = min(worst, float((c.abs() / tol.clamp_min(1e-300)).max()))
    return worst


def test_module_weight_gradients_every_block_counts(env):
    S = env["S"]
    n = 8 * S * MOD_BLK + 37
    allow = _allow(n, S) + _allow(n, S)  # the full and the compact launch each round by up to their allowance
    # ---- ngp_mlp_rgb_backward ----
    x, up = _rgb_inputs(n, 301)
    ok = ~grad64.rgb_forward(x, torch.zeros(n, 32, device="cuda"), env["rgb_h"], 1)["ambiguous"]
    rows, mark, blocks = _sparse_rows(n, 302, ok)
    up = (up * mark[:, None]).contiguous()
    xc, upc = x[rows].contiguous(), up[rows].contiguous()
    ref = grad64.rgb_backward(xc, torch.zeros(rows.numel(), 32, device="cuda"), env["rgb_h"], upc, SCALE, 1)
    assert not ref["ambiguous"][mark[rows]].any()
    dX_f, gr_f = _rgb_bwd(env, x, up, 1)
    dX_c, gr_c = _rgb_bwd(env, xc, upc, 1)
    torch.cuda.synchronize()
    assert torch.equal(dX_f[:n][rows], dX_c[:rows.numel()])
    full, comp = _rgb_dW(gr_f), _rgb_dW(gr_c)
    for k, (v, A, err) in ref["dW"].items():
        _ratio(full[k], comp[k], allow * A, "rgb full vs compact " + k)
    _check_dW(comp, ref["dW"], _allow(rows.numel(), S), "rgb compact")
    eff = _block_effect(ref["dout"], ref["fwd"]["r2"], rows, blocks, ref["dW"]["W3r"][1], 2 * allow * ref["dW"]["W3r"][1],
                        SCALE)
    assert eff > 1, "a dropped block could hide under the allowance: %g" % eff

    # ---- ngp_enc_backward ----
    mod = _enc_module(env, 16, 19)
    x01, dL_dh = _enc_inputs(n, 303)
    _, fs = _enc_forward(mod, x01)
    feat = grad64.decode_feat_save(fs, n)
    z16 = torch.zeros(n, 16, device="cuda", dtype=torch.float64)
    ok = ~grad64.density_backward(feat, _f16(mod.half_params())[:3072], z16, z16, z16, SCALE)["ambiguous"]
    rows, mark, blocks = _sparse_rows(n, 304, ok)
    dL_dh = (dL_dh * mark[:, None]).contiguous()
    x01c, dhc = x01[rows].contiguous(), dL_dh[rows].contiguous()
    _, fsc = _enc_forward(mod, x01c)
    featc = grad64.decode_feat_save(fsc, rows.numel())
    assert torch.equal(featc, feat[rows])
    ref, dhc2 = _enc_ref(mod, featc, dhc)
    assert torch.equal(dhc2, dhc)
    ge_f, ws_f = _enc_bwd(mod, x01, dL_dh, fs, env["scale_t"])
    ge_c, ws_c = _enc_bwd(mod, x01c, dhc, fsc, env["scale_t"])
    torch.cuda.synchronize()
    assert torch.equal(_dfeat(ws_f, n)[rows], _dfeat(ws_c, rows.numel()))
    full, comp = _enc_dW(ge_f), _enc_dW(ge_c)
    for k, (v, A, err) in ref["dW"].items():
        _ratio(full[k], comp[k], allow * A, "enc full vs compact " + k)
    _check_dW(comp, ref["dW"], _allow(rows.numel(), S), "enc compact")
    dh = grad64.scaled_dh(dhc, SCALE)[0]
    eff_e = _block_effect(dh, ref["hid"], rows, blocks, ref["dW"]["W2d"][1], 2 * allow * ref["dW"]["W2d"][1], SCALE)
    assert eff_e > 1, "a dropped block could hide under the allowance: %g" % eff_e
    print("MEASURED every block counts: smallest one-block effect / tolerance: rgb %.3g, enc %.3g (allowance %.3g A)"
          % (eff, eff_e, allow))


# ---------------------------------------------------------------------------------------------------------------------
# loss scale
# ---------------------------------------------------------------------------------------------------------------------
def _centre(chain, amp_target=16.0):
    mid = torch.cat([v[v != 0].abs() for v in chain]).median().item()
    return 2.0 ** round(math.log2(amp_target / mid))


def _fits(chain, n):
    """rows whose every out-gradient value stays a normal fp16 number at 2^-6 and finite at 2^6 (factor 2 of room)"""
    ok = torch.ones(n, dtype=torch.bool, device="cuda")
    for v in chain:
        ok &= ((v == 0) | (v.abs() >= 2.0 ** -14 * 2 ** 6 * 2)).all(1) & (v.abs() <= 65504.0 / 2 ** 6 / 2).all(1)
    return ok


def test_module_loss_scale_is_exact(env):
    """scales 2^-6 and 2^6 against 1: dL/dx, the feature gradients / scale and (one block: one CTA adds in a fixed order)
    the weight gradients bit for bit, wherever nothing under- or overflows"""
    S = env["S"]
    mod = _enc_module(env, 16, 19)
    for n in (MOD_BLK, 2 * S * MOD_BLK + 5):
        x, up = _rgb_inputs(n, 400 + n)
        ref, up = _rgb_ref(env, x, up, 1, scale=1.0)
        up = up * _centre([ref["dout"], ref["dr2"], ref["dr1"]])
        ref = grad64.rgb_backward(x, torch.zeros(n, 32, device="cuda"), env["rgb_h"], up, 1.0, 1)
        ok = _fits([ref["dout"], ref["dr2"], ref["dr1"]], n)
        assert ok.double().mean() > 0.2
        up = (up * ok[:, None]).contiguous()
        x01, dL_dh = _enc_inputs(n, 500 + n)
        _, fs = _enc_forward(mod, x01)
        feat = grad64.decode_feat_save(fs, n)
        db, dL_dh = _enc_ref(mod, feat, dL_dh, scale=1.0)
        dL_dh = dL_dh * _centre([grad64.scaled_dh(dL_dh, 1.0)[0], db["dhid"], db["dfeat"]])
        db, _ = _enc_ref(mod, feat, dL_dh, scale=1.0)
        ok = _fits([grad64.scaled_dh(dL_dh, 1.0)[0], db["dhid"], db["dfeat"]], n)
        assert ok.double().mean() > 0.2
        dL_dh = (dL_dh * ok[:, None]).contiguous()
        outs = []
        for e in (0, -6, 6):
            st = torch.tensor([2.0 ** e], device="cuda")
            dX, gr = _rgb_bwd(env, x, up, 1, scale_t=st)
            ge, ws = _enc_bwd(mod, x01, dL_dh, fs, st)
            torch.cuda.synchronize()
            outs.append((dX, gr, _dfeat(ws, n).float() * 2.0 ** -e, ge[:3072]))
        for o in outs[1:]:
            assert torch.equal(o[0], outs[0][0]) and torch.equal(o[2], outs[0][2])
            if n == MOD_BLK:
                assert torch.equal(o[1], outs[0][1]) and torch.equal(o[3], outs[0][3])
        assert outs[0][0][:n].abs().max() > 0 and outs[0][2].abs().max() > 0


def test_pow2_scale_range_and_zero_upstream(env):
    from ngp_pl_b200 import tcnn
    from ngp_pl_b200.models import networks as N
    g = torch.Generator(device="cuda").manual_seed(61)
    for amax in (1e-8, 1e-3, 1e4):
        t = torch.randn(3000, 3, device="cuda", generator=g)
        t = t / t.abs().max() * amax
        s = float(N._pow2_scale(t))
        assert s == 2.0 ** round(math.log2(s)), s
        m = float(t.abs().max()) * s
        assert 128 < m <= 256, (amax, s, m)
    assert float(N._pow2_scale(torch.zeros(5, 16, device="cuda"))) == 1.0
    # an all-zero upstream gradient: scale 1 and exactly zero gradients through both modules
    net = tcnn.Network(32, 3, {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "Sigmoid",
                               "n_neurons": 64, "n_hidden_layers": 2}).cuda()
    mod = _enc_module(env, 4, 14)
    x01 = torch.rand(1000, 3, device="cuda", generator=g)
    h = mod(x01)
    rin = torch.cat([torch.rand(1000, 16, device="cuda", generator=g).half(), h], 1)
    out = net(rin)
    mod.params.grad = None
    out.backward(torch.zeros_like(out))
    assert torch.equal(net.params.grad, torch.zeros_like(net.params))
    assert torch.equal(mod.params.grad, torch.zeros_like(mod.params))
    mod.params.grad = None


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in chain: the reference's unmodified NGP on ngp_pl_b200.tcnn, end to end
# ---------------------------------------------------------------------------------------------------------------------
TEXP_ERR = 2.0 ** -21  # fp32 expf (2 ulp) and the fp32 product dL/dsigma exp(h0) (half an ulp), relative


def test_dropin_module_chain_vs_float64(env, monkeypatch):
    """reference NGP.forward under autocast (as its precision-16 training runs), then backward from upstream gradients
    spread over 1e-7 ... 1e-2, against the float64 composition rgb_backward -> autograd's fp16 roundings ->
    density_backward -> grid_scatter, with the loss scale each module's _pow2_scale computes"""
    from oracle import ref_env
    from ngp_pl_b200.models import networks as N
    if not ref_env.python_available():
        pytest.skip("the reference's Python is not staged under oracle/_ref")
    ref_mod = ref_env.load_reference(drop_in=True)
    S = env["S"]
    n = 2 * S * MOD_BLK + 77
    torch.manual_seed(0)
    model = ref_mod.NGP(0.5).cuda()
    g = torch.Generator().manual_seed(71)
    with torch.no_grad():
        p = model.xyz_encoder.params
        p[3072:] = ((torch.rand(p.numel() - 3072, generator=g) * 2 - 1) * 0.5).cuda()
    gc = torch.Generator(device="cuda").manual_seed(72)
    x = (torch.rand(n, 3, device="cuda", generator=gc) - 0.5).contiguous()
    d = torch.randn(n, 3, device="cuda", generator=gc)

    rec = {}
    hooks = [model.xyz_encoder.register_forward_hook(lambda m, i, o: rec.update(x01=i[0].detach(), h=o.detach())),
             model.rgb_net.register_forward_hook(lambda m, i, o: rec.update(rin=i[0].detach()))]
    with torch.autocast("cuda", torch.float16):
        sig, rgb = model(x, d)
    for hk in hooks:
        hk.remove()
    assert rgb.dtype == torch.float16 and sig.dtype == torch.float32 and rec["rin"].dtype == torch.float16
    x01, h, rin = rec["x01"].float().contiguous(), rec["h"], rec["rin"]
    assert torch.equal(rin[:, 16:], h)
    enc_h, rgb_h = _f16(model.xyz_encoder.half_params()), _f16(model.rgb_net.half_params())
    # the features, bit for bit: the forward kernel is deterministic
    h2, fs = _enc_forward(model.xyz_encoder, x01)
    assert torch.equal(h2, h)
    feat = grad64.decode_feat_save(fs, n)

    # rows whose ReLU masks the reference cannot decide get no upstream gradient
    zero = torch.zeros(n, 32, device="cuda")
    fr = grad64.rgb_forward(rin, zero, rgb_h, 1)
    fd = grad64.density_backward(feat, enc_h[:3072], torch.zeros(n, 16, device="cuda", dtype=torch.float64),
                                 torch.zeros(n, 16, device="cuda", dtype=torch.float64),
                                 torch.zeros(n, 16, device="cuda", dtype=torch.float64), 1.0)
    _amb_rows(fr["ambiguous_own"] | fd["ambiguous_own"], fr["ambiguous"] | fd["ambiguous"])
    live = ~(fr["ambiguous"] | fd["ambiguous"])

    def spread(*shape):
        mag = 10 ** (torch.rand(*shape, device="cuda", generator=gc) * 5 - 7)
        return torch.where(torch.rand(*shape, device="cuda", generator=gc) < 0.5, -mag, mag)
    up_sig = spread(n) * live
    up_rgb = spread(n, 3) * live[:, None]

    calls = []
    orig = N._pow2_scale

    def spy(t):
        s = orig(t)
        calls.append((t.detach().clone(), s.clone()))
        return s
    monkeypatch.setattr(N, "_pow2_scale", spy)
    torch.autograd.backward([sig, rgb], [up_sig, up_rgb])
    monkeypatch.setattr(N, "_pow2_scale", orig)
    torch.cuda.synchronize()
    assert [c[0].shape for c in calls] == [(n, 3), (n, 16)]
    (d_rgb, s_r), (d_h, s_e) = calls

    def check_scale(t, s):
        m = t.abs().max().double()
        s = float(s)
        assert s == 2.0 ** math.floor(math.log2(256.0 / float(m))) and 128 < float(m) * s <= 256
        return s
    # rgb_net's upstream gradient is rgb's: fp16, so autograd casts dL/drgb to fp16
    up16 = grad64.f16(up_rgb.double())
    assert torch.equal(d_rgb.double(), up16)
    s_r = check_scale(d_rgb, s_r)
    rb = grad64.rgb_backward(rin, zero, rgb_h, up16, s_r, 1)
    # dL/dh: _RgbMlp returns dL/dx in fp32 for an fp16 input, autograd casts it to fp16 (unscaled); TruncExp returns
    # dL/dsigma exp(clamp(h0, +-15)) in fp32, cast to fp16; the two meet in column 0 as an fp16 sum
    dxh, d_dxh, _ = grad64._rounded(rb["dX"][:, 16:], rb["dX_err"][:, 16:], False)
    t = up_sig.double() * torch.exp(h[:, 0].double().clamp(-15, 15))
    tv, d_t, _ = grad64._rounded(t, TEXP_ERR * t.abs(), False)
    y, e = dxh.clone(), d_dxh.clone()
    y[:, 0] += tv
    e[:, 0] += d_t
    dLdh, d_dLdh, _ = grad64._rounded(y, e, False)
    m_dh = _ratio(d_h, dLdh, d_dLdh, "dL/dh")
    s_e = check_scale(d_h, s_e)
    # k_enc_bwd scales the fp16 dL/dh and rounds it to fp16 once
    dh, dh_err, _ = grad64._rounded(dLdh * s_e, d_dLdh * s_e, False)
    db = grad64.density_backward(feat, enc_h[:3072], dh, dh_err, dLdh.abs() * s_e + d_dLdh * s_e, s_e)

    ge, gr = model.xyz_encoder.params.grad, model.rgb_net.params.grad
    allow = _allow(n, S)
    mw = _check_dW({k: v.double() for k, v in grad64.split_dW(ge, gr).items()}, dict(rb["dW"], **db["dW"]), allow,
                   "drop-in")
    tg, Sabs, m = grad64.grid_scatter(model.xyz_encoder.meta, x01, db["dfeat"], 1.0 / s_e, model.xyz_encoder.n_entries)
    terr, _, _ = grad64.grid_scatter(model.xyz_encoder.meta, x01, db["dfeat_err"], 1.0 / s_e, model.xyz_encoder.n_entries)
    Sall, _, _ = grad64.grid_scatter(model.xyz_encoder.meta, x01, db["dfeat"].abs() + db["dfeat_err"], 1.0 / s_e,
                                     model.xyz_encoder.n_entries)
    got_t = ge[3072:].view(-1, 2).double()
    mt = _ratio(got_t, tg, terr.abs() + (m[:, None] + 2) * 2.0 ** -24 * Sall, "drop-in table")
    assert (got_t[m == 0] == 0).all() and (tg != 0).any()
    nz = d_h[live] != 0
    sub = (d_h[live].abs() < 2.0 ** -14) & nz
    print("MEASURED drop-in chain n=%d: dL/dh %.4f bitwise, worst %.3f of 2x bound; %.4f of dL/dh in fp16's subnormal "
          "range, %.4f exactly zero; " % (n, *m_dh, sub.double().mean(), (~nz).double().mean())
          + ", ".join("%s %.4f / %.3g" % (k, *v) for k, v in mw.items())
          + "; table %.4f / %.3g (bitwise / worst of 2x bound)" % mt)
