"""float64 restatement of the network forward, the network backward and the hash-table scatter -- TEST INFRASTRUCTURE ONLY.

Nothing under ngp_pl_b200/ imports this. It is plain torch (any device), so the GPU tests run it on CUDA at training
sizes and the CPU suite checks it against oracle.torch_ngp_forward / torch_grid_encode on small inputs.

mlp_backward() restates k_ngp_bwd3 at the kernel's own fp16 rounding points:
  forward, from the fp16 features:  hid = fp16(relu(feat W1d^T)),  h = fp16(hid W2d^T),  rin = [fp16(SH(d)) | h],
                                    r1 = fp16(relu(rin W1r^T)),  r2 = fp16(relu(r1 W2r^T)),  o = fp16(sigmoid(r2 W3r^T))
  out-gradient chain (scaled by the power-of-two loss scale, each step rounded to fp16):
      dout = up o (1 - o) scale      dr2 = [r2 > 0] dout W3r      dr1 = [r1 > 0] dr2 W2r
      dh   = dr1 W1r[:, 16:]  (+ up_sig exp(clamp(h0, +-15)) scale in column 0)
      dhid = [hid > 0] dh W2d        dfeat = dhid W1d
  weight gradients: dW = sum_rows dOut^T In / scale, in float64.
Every value comes with a rigorous bound of how far the kernel's may lie from it (`err`), built from
  * one fp16 ulp (2^-10 relative: the rounding plus a flip of the last bit by a different fp32 accumulation order) and
    one smallest subnormal (2^-24) per rounding, applied to the absolute-value chain |dout| |W3r| ... |W1d| (`abs`);
  * 2^-20 of sum|terms| for the kernel's fp32 tensor-core accumulation (K <= 64 exact products, <= 4 fp32 additions);
  * the forward values the kernel may round the other way: where an activation's fp32 accumulation error straddles an
    fp16 rounding boundary, the kernel's value may be one ulp off; that difference is carried one layer on, into the next
    layer's ReLU masks, the sigmoid derivative, exp(h0) and the weight gradients' inputs. (A flip caused by another
    flip is modelled only with carry=True, which follows every flip to the forward's outputs.)
A row whose ReLU masks are not determined by those intervals is flagged in `ambiguous`: there the kernel and the
reference may take different branches and no rounding bound applies. `ambiguous_own` flags the subset where the
pre-activation's own accumulation error alone (|z| <= 2^-20 sum|terms|) leaves the mask open.

rgb_backward() and density_backward() are the two halves of that chain on their own, as the stand-alone module kernels
run them: k_mlp_rgb_bwd from an fp16 input matrix to dL/dx in fp32 (no fp16 rounding), k_enc_bwd from a scaled fp16
dL/dh to the feature gradients. mlp_backward() composes them with the one rounding k_ngp_bwd3 adds in between.

mlp_forward() is that forward on its own, as intervals (with carry=True every bound is followed to the outputs);
grid_encode(), sigma(), sh_encode(), ray_positions() and to_unit() restate the rest of k_ngp_fwd / k_sh_encode: the
hash-grid features, sigma = expf(h0), the stand-alone SH encoding and the sample positions, each with its derived bound
(or bit for bit where the arithmetic allows).

grid_scatter() restates k_grid_scatter_merged: corner weights in float32 exactly as grid_cell / grid_corner_weights
compute them (bit for bit), indices as grid_corner_indices (dense wrap included), contributions w g / scale summed in
float64, with the per-entry sum of |contribution| and the number of contributions.
"""
import torch

ULP16 = 2.0 ** -10   # one fp16 ulp, relative (normal range): a rounding (2^-11) plus a flipped last bit
SUB16 = 2.0 ** -24   # smallest fp16 subnormal: absolute floor of a rounding
ACC32 = 2.0 ** -20   # fp32 tensor-core accumulation of <= 64 fp16 products, relative to sum |terms|
ACC32_OUT = 2.0 ** -24  # one fp32 rounding of a stored result, relative
SH_ERR = 2.0 ** -19  # absolute error of the kernel's fp32 SH-4 of a normalised direction (|SH| <= 3, degree <= 3)
SIG_ERR = 2.0 ** -19  # absolute error of the kernel's fp32 sigmoid 1 / (1 + __expf(-x))
M32 = 0xFFFFFFFF


def f16(x):
    """round to fp16 (nearest even), back in x's dtype"""
    return x.to(torch.float16).to(x.dtype)


# ---------------------------------------------------------------------------------------------------
# feat_save: the forward's saved features, in mma A-fragment order
# [16-row tile][kt][lane = 4g + q][word x, y, z, w] of half2: x / y = rows g / g + 8 at columns 16 kt + 2q (+1),
# z / w = rows g / g + 8 at columns 16 kt + 8 + 2q (+1); column 2 l (+1) holds level l's features.
# ---------------------------------------------------------------------------------------------------
def decode_feat_save(fs, n):
    """fs: uint8 tensor (>= ceil(n/16) * 1024 bytes) -> (n, 32) float16 features"""
    t = (n + 15) // 16
    h = fs[:t * 1024].contiguous().view(torch.float16).view(t, 2, 8, 4, 2, 2, 2)  # tile kt g q col-half row-half f
    return h.permute(0, 5, 2, 1, 4, 3, 6).reshape(t * 16, 32)[:n]


def encode_feat_save(feat):
    """inverse of decode_feat_save: (n, 32) float16 -> uint8 tensor of ceil(n/32) * 32 * 64 bytes (zero rows padded)"""
    n = feat.shape[0]
    t = (n + 31) // 32 * 2
    pad = torch.zeros(t * 16, 32, dtype=torch.float16, device=feat.device)
    pad[:n] = feat
    h = pad.view(t, 2, 8, 2, 2, 4, 2)  # tile row-half g kt col-half q f
    return h.permute(0, 3, 2, 5, 4, 1, 6).contiguous().view(torch.uint8).reshape(-1)


def sh4_64(dirs):
    """SH-4 of the normalised directions, in float64 (rounded to fp16 by mlp_backward)"""
    from .oracle import torch_sh4
    d = dirs.double()
    return torch_sh4(d / d.norm(dim=1, keepdim=True))


# ---------------------------------------------------------------------------------------------------
# network backward
# ---------------------------------------------------------------------------------------------------
def _rounded(y, e, relu):
    """fp16 value of y and how far the kernel's may be from it when its pre-rounding value is only known to +- e;
    for a ReLU, also whether the mask is undetermined"""
    r = (lambda v: f16(v.clamp_min(0))) if relu else f16
    a, lo, hi = r(y), r(y - e), r(y + e)
    amb = ((lo > 0) != (hi > 0)).any(1) if relu else None
    return a, torch.maximum(hi - a, a - lo), amb


def _fwd(x, dx, W, relu, carry=False):
    """one forward layer from inputs the kernel may have rounded differently by up to dx: the fp16 output, by how much the
    kernel's may differ (one ulp where its own fp32 accumulation error straddles a rounding boundary; with `carry`, also
    what dx moves the pre-activation by) and, for a ReLU, the rows whose mask the accumulation error together with dx
    leaves undetermined"""
    Wa = W.abs()
    y = x @ W.t()
    e_own = ACC32 * (x.abs() @ Wa.t())
    a, d, amb_own = _rounded(y, e_own, relu)
    if relu or carry:
        _, d_all, amb = _rounded(y, e_own + dx @ Wa.t(), relu)
        if carry:
            d = d_all
    return a, d, (amb, amb_own) if relu else None


def _chain(g, err, ab, W, mask):
    """one dgrad step g W (masked), rounded to fp16: value, error bound, absolute-value chain"""
    Wa = W.abs()
    y, a, e = g @ W, ab @ Wa, err @ Wa
    if mask is not None:
        y, a, e = y * mask, a * mask, e * mask
    return f16(y), _round_err(e + ACC32 * a, a), a


def _round_err(e, a):
    """error after rounding a value whose pre-rounding error is e and whose absolute-value chain is a"""
    return (1 + ULP16) * e + ULP16 * a + SUB16 * (a > 0)


def _wgrad(dO, dO_err, dO_abs, In, In_err, scale):
    """dW = dO^T In / scale, its absolute-value sum A and the bound of the kernel's deviation (operand errors only)"""
    v = dO.t() @ In / scale
    A = dO_abs.t() @ In.abs() / scale
    err = (dO_err.t() @ In.abs() + (dO.abs() + dO_err).t() @ In_err) / scale
    return v, A, err


def rgb_forward(rin, d_rin, rgb_params, rgb_act=1, carry=False):
    """the rgb net 32 -> 64 -> 64 -> 3 from fp16 inputs rin (n, 32) the kernel may hold differently by up to d_rin, at the
    kernel's rounding points (see mlp_forward for the dict it returns; k_mlp_rgb_fwd runs this alone)"""
    dt = torch.float64
    Wr = rgb_params.to(dt)
    W1r, W2r, W3r = Wr[:2048].view(64, 32), Wr[2048:6144].view(64, 64), Wr[6144:7168].view(16, 64)
    rin, d_rin = rin.to(dt), d_rin.to(dt)
    r1, d_r1, amb_r1 = _fwd(rin, d_rin, W1r, True, carry)
    r2, d_r2, amb_r2 = _fwd(r1, d_r1, W2r, True, carry)
    W3 = W3r[:3]
    yo = r2 @ W3.t()
    eo = ACC32 * (r2.abs() @ W3.abs().t()) + d_r2 @ W3.abs().t()
    f = dict(rin=rin, d_rin=d_rin, r1=r1, d_r1=d_r1, r2=r2, d_r2=d_r2, yo=yo, d_yo=eo,
             ambiguous=amb_r1[0] | amb_r2[0], ambiguous_own=amb_r1[1] | amb_r2[1])
    if rgb_act == 1:
        # the kernel's fp32 sigmoid of its accumulator, within SIG_ERR of the sigmoid of a value in yo +- eo, then rounded
        # to fp16: both steps are monotone, so its output lies between the roundings of the two ends
        def sgm(v): return torch.sigmoid(v)
        o = f16(sgm(yo))
        s = o * (1 - o)
        o_lo, o_hi = f16(sgm(yo - eo) - SIG_ERR), f16(sgm(yo + eo) + SIG_ERR)
        ds = torch.maximum((o_lo * (1 - o_lo) - s).abs(), (o_hi * (1 - o_hi) - s).abs())
        f.update(out=o, d_out=torch.maximum(o_hi - o, o - o_lo), s=s, d_s=ds)
    else:
        o, d_o, _ = _rounded(yo, eo, False)
        f.update(out=o, d_out=d_o)
    return f


def mlp_forward(feat, sh, enc_mlp, rgb_params, rgb_act=1, carry=False, d_feat=None):
    """the network forward from fp16 features at the kernel's rounding points, as intervals (k_ngp_fwd's MLP part, and
    what k_ngp_bwd3 recomputes). feat (n, 32) fp16 features, sh (n, 16) float64 SH-4 (unrounded), enc_mlp (>= 3072) /
    rgb_params (7168) fp16 weights. Returns a dict of float64 tensors:
      hid, h, rin = [fp16(sh) | h], r1, r2: fp16 values, each with d_<name>, how far the kernel's value may be from it;
      yo (n, 3): the rgb net's pre-activation, d_yo its bound (fp32 accumulation plus what d_r2 moves);
      out (n, 3): the rgb output, an fp16 value (half_round), d_out its bound; for rgb_act 1 also s = out (1 - out)
      and d_s, what the sigmoid derivative of the kernel's output may differ by;
      ambiguous / ambiguous_own (n) bool: rows whose ReLU masks are undetermined (module docstring).
    carry=False is the backward's model: d_<name> is one flip of the value's own rounding, and a flip reaches only the
    next layer's masks. carry=True bounds the forward's outputs: every layer's bound also carries what its inputs'
    bounds move it by, so a value rounded the other way is followed to the outputs. d_feat: how far the kernel's
    features may lie from feat (grid_encode's bound); None when feat are the kernel's own (feat_save)."""
    dt = torch.float64
    feat = feat.to(dt)
    d_feat = torch.zeros_like(feat) if d_feat is None else d_feat.to(dt)
    Wd = enc_mlp.to(dt)
    W1d, W2d = Wd[:2048].view(64, 32), Wd[2048:3072].view(16, 64)
    hid, d_hid, amb_hid = _fwd(feat, d_feat, W1d, True, carry)
    h, d_h, _ = _fwd(hid, d_hid, W2d, False, carry)
    shr, d_sh, _ = _rounded(sh.to(dt), SH_ERR, False)
    f = rgb_forward(torch.cat([shr, h], 1), torch.cat([d_sh, d_h], 1), rgb_params, rgb_act, carry)
    f.update(hid=hid, d_hid=d_hid, h=h, d_h=d_h, ambiguous=amb_hid[0] | f["ambiguous"],
             ambiguous_own=amb_hid[1] | f["ambiguous_own"])
    return f


def rgb_backward(rin, d_rin, rgb_params, up_rgb, scale, rgb_act=1, carry=False):
    """k_mlp_rgb_bwd's chain from fp16 inputs rin (n, 32) the kernel may hold differently by up to d_rin (0 when they are
    the kernel's own input), fp32 upstream gradients up_rgb (n, 3) and the power-of-two loss scale:
      dout = fp16(up o (1 - o) scale),  dr2 = fp16([r2 > 0] dout W3r),  dr1 = fp16([r1 > 0] dr2 W2r)
      dX   = (dr1 W1r) / scale in fp32: all 32 columns, no fp16 rounding
    Returns a dict: dX (n, 32, unscaled), dX_err (its bound: the operand errors and the fp32 accumulation of dr1 W1r,
    plus one fp32 rounding), dX_abs; dout / dr2 / dr1 with _err / _abs (scaled); dW {W3r, W2r, W1r: (value, A, err)}
    (unscaled); ambiguous / ambiguous_own (n) bool; the forward dict `fwd` (rgb_forward's). carry: the forward's bounds
    carry what d_rin and every earlier flip move each layer by (rgb_forward(carry=True)), and so do the masks, the sigmoid
    derivative and the weight gradients' inputs that depend on them."""
    dt = torch.float64
    Wr = rgb_params.to(dt)
    W1r, W2r, W3r = Wr[:2048].view(64, 32), Wr[2048:6144].view(64, 64), Wr[6144:7168].view(16, 64)
    up_rgb = up_rgb.to(dt)
    f = rgb_forward(rin, d_rin, rgb_params, rgb_act, carry)
    rin, d_rin, r1, d_r1, r2, d_r2, yo = f["rin"], f["d_rin"], f["r1"], f["d_r1"], f["r2"], f["d_r2"], f["yo"]
    n = rin.shape[0]
    if rgb_act == 1:
        s, ds = f["s"], f["d_s"]
    else:
        s, ds = torch.ones_like(yo), torch.zeros_like(yo)

    dout = torch.zeros(n, 16, dtype=dt, device=rin.device)
    dout_abs, dout_err = torch.zeros_like(dout), torch.zeros_like(dout)
    v = up_rgb * s * scale
    dout[:, :3] = f16(v)
    dout_abs[:, :3] = v.abs()
    dout_err[:, :3] = _round_err(ACC32 * v.abs() + up_rgb.abs() * ds * scale, v.abs())
    dr2, dr2_err, dr2_abs = _chain(dout, dout_err, dout_abs, W3r, (r2 > 0).to(dt))
    dr1, dr1_err, dr1_abs = _chain(dr2, dr2_err, dr2_abs, W2r, (r1 > 0).to(dt))
    W1a = W1r.abs()
    y, a = dr1 @ W1r, dr1_abs @ W1a
    e = dr1_err @ W1a + ACC32 * a
    # the fp32 accumulator times 1 / scale (a power of two: exact) is stored once, rounded to fp32; 2^-149 is its
    # subnormal floor
    dX_err = (e + ACC32_OUT * (y.abs() + e)) / scale + 2.0 ** -149
    dW = {
        "W3r": _wgrad(dout, dout_err, dout_abs, r2, d_r2, scale),
        "W2r": _wgrad(dr2, dr2_err, dr2_abs, r1, d_r1, scale),
        "W1r": _wgrad(dr1, dr1_err, dr1_abs, rin, d_rin, scale),
    }
    return dict(dX=y / scale, dX_err=dX_err, dX_abs=a / scale, dout=dout, dout_err=dout_err, dout_abs=dout_abs,
                dr2=dr2, dr2_err=dr2_err, dr2_abs=dr2_abs, dr1=dr1, dr1_err=dr1_err, dr1_abs=dr1_abs, dW=dW,
                ambiguous=f["ambiguous"], ambiguous_own=f["ambiguous_own"], fwd=f)


def scaled_dh(dL_dh, scale):
    """k_enc_bwd's out-gradient: dh = fp16(dL_dh scale), a single rounding of an fp32 product (no accumulation).
    -> (value, bound, absolute value), float64 (n, 16), scaled"""
    v = dL_dh.double() * scale
    return f16(v), _round_err(torch.zeros_like(v), v.abs()), v.abs()


def density_backward(feat, enc_mlp, dh, dh_err, dh_abs, scale):
    """k_enc_bwd's chain (and the density half of k_ngp_bwd3's) from the fp16 features feat (n, 32) and the scaled fp16
    out-gradient dh (n, 16), which the kernel may hold differently by up to dh_err (dh_abs: its absolute-value chain):
      dhid = fp16([hid > 0] dh W2d),  dfeat = fp16(dhid W1d)
    Returns a dict: dhid / dfeat (scaled, like the kernel's workspace) with _err / _abs; dW {W2d, W1d: (value, A, err)}
    (unscaled); hid, d_hid; ambiguous / ambiguous_own (n) bool: rows whose hidden-layer ReLU mask is open."""
    dt = torch.float64
    feat = feat.to(dt)
    Wd = enc_mlp.to(dt)
    W1d, W2d = Wd[:2048].view(64, 32), Wd[2048:3072].view(16, 64)
    hid, d_hid, amb = _fwd(feat, torch.zeros_like(feat), W1d, True)
    dhid, dhid_err, dhid_abs = _chain(dh, dh_err, dh_abs, W2d, (hid > 0).to(dt))
    dfeat, dfeat_err, dfeat_abs = _chain(dhid, dhid_err, dhid_abs, W1d, None)
    dW = {
        "W2d": _wgrad(dh, dh_err, dh_abs, hid, d_hid, scale),
        "W1d": _wgrad(dhid, dhid_err, dhid_abs, feat, torch.zeros_like(feat), scale),
    }
    return dict(dhid=dhid, dhid_err=dhid_err, dhid_abs=dhid_abs, dfeat=dfeat, dfeat_err=dfeat_err, dfeat_abs=dfeat_abs,
                dW=dW, hid=hid, d_hid=d_hid, ambiguous=amb[0], ambiguous_own=amb[1])


def mlp_backward(feat, sh, enc_mlp, rgb_params, up_sig, up_rgb, scale, rgb_act=1, carry=False):
    """feat (n, 32) fp16 features, sh (n, 16) float64 SH-4 (unrounded), enc_mlp (>= 3072) / rgb_params (7168) fp16 weights,
    up_sig (n), up_rgb (n, 3) fp32 upstream gradients, scale the power-of-two loss scale (a number).
    Returns a dict: dfeat (n, 32, scaled by `scale`, like the kernel's workspace), dfeat_err, dfeat_abs, ambiguous (n) bool,
    dW {name: (value, A, err)} for W3r, W2r, W1r, W2d, W1d (unscaled), and the forward activations.
    It is rgb_backward, then the sum k_ngp_bwd3 rounds once: dh = fp16(dr1 W1r[:, 16:] + up_sig exp(h0) scale in
    column 0), then density_backward.
    carry=False models one flip per row: an activation may round the other way where its own accumulation error
    straddles a boundary, and that flip reaches the next layer only. carry=True follows every flip to the end of the
    forward (mlp_forward(carry=True)): a flip of hid moves h, which may move h0 by an ulp (and exp(h0) with it) or flip a
    ReLU mask of the colour net. The values are the same; the bounds and the undecided rows can only grow. Trained
    weights, whose out-gradients cancel heavily, need it."""
    dt = torch.float64
    feat = feat.to(dt)
    Wr = rgb_params.to(dt)
    W1r = Wr[:2048].view(64, 32)
    up_sig = up_sig.to(dt)

    # ---- forward recompute with the kernel's rounding points, as intervals ----
    f = mlp_forward(feat, sh, enc_mlp, rgb_params, rgb_act, carry)
    hid, h, d_h, rin, r1, r2, yo = f["hid"], f["h"], f["d_h"], f["rin"], f["r1"], f["r2"], f["yo"]
    if rgb_act == 1:
        o = f["out"]

    # ---- out-gradient chain ----
    rb = rgb_backward(rin, f["d_rin"], rgb_params, up_rgb, scale, rgb_act, carry)
    dout, dr2, dr1, dr1_err, dr1_abs = rb["dout"], rb["dr2"], rb["dr1"], rb["dr1_err"], rb["dr1_abs"]
    Wh = W1r[:, 16:]
    y, a, e = dr1 @ Wh, dr1_abs @ Wh.abs(), dr1_err @ Wh.abs()
    # density branch d sigma / d h0 = exp(clamp(h0, -15, 15)), h0 possibly off by d_h[:, 0]
    def texp(x): return torch.exp(x.clamp(-15, 15))
    h0, dh0 = h[:, 0], d_h[:, 0]
    t = up_sig * texp(h0) * scale
    dt0 = up_sig.abs() * scale * torch.maximum((texp(h0 + dh0) - texp(h0)).abs(), (texp(h0 - dh0) - texp(h0)).abs())
    y[:, 0] += t
    a[:, 0] += t.abs()
    e[:, 0] += dt0
    dh, dh_err, dh_abs = f16(y), _round_err(e + ACC32 * a, a), a
    db = density_backward(feat, enc_mlp, dh, dh_err, dh_abs, scale)

    dW = dict(rb["dW"])
    dW.update(db["dW"])
    return dict(dfeat=db["dfeat"], dfeat_err=db["dfeat_err"], dfeat_abs=db["dfeat_abs"], dW=dW,
                ambiguous=f["ambiguous"], ambiguous_own=f["ambiguous_own"],
                hid=hid, h=h, rin=rin, r1=r1, r2=r2, o=o if rgb_act == 1 else yo,
                chain=[dout, dr2, dr1, dh, db["dhid"], db["dfeat"]])


# layout of the five weight gradients in the flat parameter-gradient vectors: (vector, offset, shape)
DW_LAYOUT = {"W1d": ("enc", 0, (64, 32)), "W2d": ("enc", 2048, (16, 64)),
             "W1r": ("rgb", 0, (64, 32)), "W2r": ("rgb", 2048, (64, 64)), "W3r": ("rgb", 6144, (16, 64))}


def split_dW(grad_enc, grad_rgb):
    """the five weight gradients of flat gradient vectors, as (out, in) matrices"""
    src = {"enc": grad_enc, "rgb": grad_rgb}
    return {k: src[v][o:o + s[0] * s[1]].view(*s) for k, (v, o, s) in DW_LAYOUT.items()}


# ---------------------------------------------------------------------------------------------------
# network forward: the features, sigma, the stand-alone SH encoding and the ray-mode positions
# ---------------------------------------------------------------------------------------------------
EXP_ERR = 2.0 ** -22   # relative error of expf (2 ulp: CUDA C++ Programming Guide; the build does not use fast-math)
FMA_CHAIN = 8 * 2.0 ** -24  # grid_lookup's 8-step fmaf chain: one fp32 rounding a step, each <= 2^-24 sum |w_k t_k|


def grid_encode(meta, table_h, x01):
    """encode_rows (grid_lookup, then pack_half2) as intervals. table_h (entries, 2) fp16 table, x01 (n, 3) float32.
    Returns float64 (n, 32) tensors: feat = fp16 of the float64 sum_k w_k t_k (column 2 l + f; levels >= n_levels are
    exactly 0) and d_feat, how far the kernel's fp16 value may lie from it. The weights and indices are the kernel's bit
    for bit (corner_weights, corner_indices: the dense wrap and the clamp outside the box included), so the products
    w_k t_k (24 x 11 bits) are exact and only the fp32 chain and the fp16 rounding are left."""
    n = x01.shape[0]
    feat = torch.zeros(n, 32, dtype=torch.float64, device=x01.device)
    d_feat = torch.zeros_like(feat)
    t = table_h.double()
    for l in range(int(meta.n_levels)):
        off = int(meta.offset[l])
        entries = int(meta.offset[l + 1]) - off
        w, gi = corner_weights(x01, meta.scale[l])
        idx = corner_indices(gi, int(meta.res[l]), entries, bool((int(meta.hashed_mask) >> l) & 1)) + off
        c = w.double()[:, :, None] * t[idx]
        a, d, _ = _rounded(c.sum(1), FMA_CHAIN * c.abs().sum(1), False)
        feat[:, 2 * l:2 * l + 2], d_feat[:, 2 * l:2 * l + 2] = a, d
    return feat, d_feat


def sigma(h, d_h):
    """sigma = expf(h0) of the kernel's fp16 h0, which lies in h[:, 0] +- d_h[:, 0]: (float64 exp(h0), bound)"""
    h0, d0 = h[:, 0], d_h[:, 0]
    s = torch.exp(h0)
    lo, hi = torch.exp(h0 - d0), torch.exp(h0 + d0)
    return s, torch.maximum(hi - s, s - lo) + EXP_ERR * hi + 2.0 ** -148  # + two fp32 subnormal steps


def sh_encode(u):
    """k_sh_encode: SH-4 of fmaf(u, 2, -1) (one float32 rounding of the exact 2u - 1), in float64, then rounded to fp16
    as intervals: (value, bound). For u in [0, 1]^3 the kernel's fp32 SH is within SH_ERR of the float64 one."""
    from .oracle import torch_sh4
    x = (u.double() * 2 - 1).float().double()
    a, d, _ = _rounded(torch_sh4(x), SH_ERR, False)
    return a, d


def ray_positions(rays_o, rays_d, ray_idx, ts):
    """load_sample's ray-mode position x = fma(d, t, o) in float32, bit for bit; (n, 3), 0 where ray_idx < 0.
    The float64 product d t is exact; the float64 sum s = d t + o is rounded at most once and TwoSum gives its exact
    residual r. Rounding s to float32 gives the fma's result unless s is exactly halfway between two floats while
    r != 0 -- then the fma rounds towards r."""
    live = ray_idx >= 0
    r = ray_idx.long().clamp_min(0)
    p = rays_d[r].double() * ts.double()[:, None]
    o = rays_o[r].double()
    s = p + o
    bp = s - o
    res = (p - bp) + (o - (s - bp))
    x = s.float()
    xd = x.double()
    nb = torch.where(s > xd, torch.nextafter(x, torch.full_like(x, float("inf"))),
                     torch.nextafter(x, torch.full_like(x, -float("inf"))))
    tie = (s != xd) & ((s - xd) == (nb.double() - s)) & (res != 0)
    x = torch.where(tie & (res > 0), torch.maximum(x, nb), torch.where(tie & (res < 0), torch.minimum(x, nb), x))
    return torch.where(live[:, None], x, torch.zeros_like(x))


def to_unit(x, xyz_min, xyz_max):
    """to_unit: __fdiv_rn(x - xyz_min, xyz_max - xyz_min) in float32, bit for bit (a float32 difference and quotient are
    exact in float64 -- 53 >= 2 x 24 + 2 -- so one rounding to float32 each is the kernel's)"""
    mn = torch.tensor(xyz_min, dtype=torch.float64, device=x.device)
    mx = torch.tensor(xyz_max, dtype=torch.float64, device=x.device)
    num = (x.double() - mn).float().double()
    den = (mx - mn).float().double()
    return (num / den).float()


# ---------------------------------------------------------------------------------------------------
# hash-table scatter
# ---------------------------------------------------------------------------------------------------
def corner_weights(x01, scale_l):
    """the 8 trilinear weights (n, 8) in float32, k = dx + 2 dy + 4 dz, bit-identical to grid_cell + grid_corner_weights,
    and the cell's integer corner (n, 3) int64"""
    pos = (x01.double() * float(scale_l) + 0.5).float()  # fmaf: the double product of two floats is exact
    g = torch.floor(pos)
    w = pos - g
    u = 1.0 - w
    a00, a10, a01, a11 = u[:, 0] * u[:, 1], w[:, 0] * u[:, 1], u[:, 0] * w[:, 1], w[:, 0] * w[:, 1]
    uz, wz = u[:, 2], w[:, 2]
    return torch.stack([a00 * uz, a10 * uz, a01 * uz, a11 * uz, a00 * wz, a10 * wz, a01 * wz, a11 * wz], 1), g.long()


def corner_indices(gi, res, entries, hashed):
    """grid_corner_indices: (n, 8) int64 entry indices inside the level"""
    gx, gy, gz = gi[:, 0] & M32, gi[:, 1] & M32, gi[:, 2] & M32
    if hashed:
        mask = entries - 1
        x0, x1 = gx, (gx + 1) & M32
        y0 = (gy * 2654435761) & M32
        y1 = (y0 + 2654435761) & M32
        z0 = (gz * 805459861) & M32
        z1 = (z0 + 805459861) & M32
        t00, t10, t01, t11 = y0 ^ z0, y1 ^ z0, y0 ^ z1, y1 ^ z1
        idx = [x0 ^ t00, x1 ^ t00, x0 ^ t10, x1 ^ t10, x0 ^ t01, x1 ^ t01, x0 ^ t11, x1 ^ t11]
        return torch.stack([i & mask for i in idx], 1)
    r2 = (res * res) & M32
    b00 = (gx + gy * res + gz * r2) & M32
    b10, b01 = (b00 + res) & M32, (b00 + r2) & M32
    b11 = (b10 + r2) & M32
    raw = torch.stack([b00, b00 + 1, b10, b10 + 1, b01, b01 + 1, b11, b11 + 1], 1) & M32
    raw = torch.where(raw >= entries, raw - entries, raw)
    return raw.clamp_max(entries - 1)


def grid_scatter(meta, x01, dfeat, inv_scale, n_entries):
    """meta: NgpGridMeta-like; x01 (n, 3) float32 in the unit cube; dfeat (n, 32) fp16 feature gradients (column 2 l + f,
    scaled); inv_scale a power of two. -> (grad (n_entries, 2), sum |contribution| (n_entries, 2), count (n_entries)),
    float64 / int64, on x01's device"""
    dev = x01.device
    grad = torch.zeros(n_entries, 2, dtype=torch.float64, device=dev)
    S = torch.zeros_like(grad)
    m = torch.zeros(n_entries, dtype=torch.int64, device=dev)
    dfeat = dfeat.double()
    for l in range(int(meta.n_levels)):
        off = int(meta.offset[l])
        entries = int(meta.offset[l + 1]) - off
        hashed = bool((int(meta.hashed_mask) >> l) & 1)
        w, gi = corner_weights(x01, meta.scale[l])
        idx = corner_indices(gi, int(meta.res[l]), entries, hashed) + off
        c = w.double()[:, :, None] * dfeat[:, None, 2 * l:2 * l + 2] * inv_scale  # exact: 24 x 11 bits
        grad.index_add_(0, idx.reshape(-1), c.reshape(-1, 2))
        S.index_add_(0, idx.reshape(-1), c.abs().reshape(-1, 2))
        m.index_add_(0, idx.reshape(-1), torch.ones(idx.numel(), dtype=torch.int64, device=dev))
    return grad, S, m
