"""float64 restatement of the training compositor, its backward and NeRFLoss, with a bound on how far an fp32
implementation may lie from every value -- TEST INFRASTRUCTURE ONLY.

Nothing under ngp_pl_b200/ imports this. It is plain torch on any device, vectorised over rays in a padded (ray, sample)
layout with a loop over the sample position, so the GPU tests run it on CUDA at training sizes and the CPU suite holds it
to the C oracle, to the reference kernels' own outputs (tests/golden/composite.npz) and to a float32 replay of the warp
algorithm.

Semantics (the reference's serial loops, computed in float64 from the kernel's own fp32 inputs):
  forward   volumerendering.cu:6-45   a_i = 1 - exp(-s_i d_i),  w_i = a_i T_{i-1},  T_i = T_{i-1} (1 - a_i),  T_{-1} = 1;
            sample i is composited iff i = 0 or T_{i-1} > T_threshold (the sample on which T drops to <= T_threshold is
            the last one), total_samples excludes that terminating sample;
            C = sum w c,  O = sum w,  D = sum w t
  background rendering.py:160-161     out = C + bg (1 - O)
  NeRFLoss  losses.py:47-60           mean over 3 n of (out - gt)^2 + lambda mean(-o log o), o = O + 1e-10:
            dL/dout = 2 (out - gt) / (3 n),  dL/dO = lambda (-log o - 1) / n - dL/dout . bg (the background's share)
  backward  volumerendering.cu:87-151 dL/drgb_i = dC w_i,
            dL/dsigma_i = d_i [ dC.(c_i T_i - (C - r_i)) + dO (1 - O) + dD (t_i T_i - (D - d_i)) + T_i dws_i - (S - s_i) ]
            with r_i, d_i, s_i the inclusive prefixes of w c, w t, dws w and S the last of the latter.

The bound (`*_err`) is first order in the fp32 unit roundoff u = 2^-24: every product or quotient adds u times its
magnitude, errors of operands propagate through |partial derivatives|, and each rounding has an absolute floor of 2^-126
(flush to zero). Tests compare with SAFETY (= 2) times the bound, which covers the second-order terms. Step by step:
  * x = fl(s d): u x.  e = __expf(-x): CUDA documents at most 2 + floor(1.173 |x|) ulp, one ulp <= 2^-23 e, plus e u x
    from the rounded argument.  a = fl(1 - e): de + u a.  om = fl(1 - a) (the factor of the product scan): da + u om.
  * Transmittance. Lane l of trip k computes T_i (i = 32 k + l) as a Hillis-Steele product scan of the trip's 32 factors
    times the carry of the previous trip. A product of m factors has m - 1 roundings whatever its tree, so the scan's
    depth of 5 does not help: T_i carries l in-trip roundings, one carry multiply and the carry's own 32 k - 1, i.e. i in
    all, exactly as the serial loop T *= 1 - a. In both orders
        dT_i = om_i dT_{i-1} + T_{i-1} dom_i + u T_i,
    which is the first-order expansion of sum_j (dom_j / om_j + u) times T_i written without dividing by om_j (om_j = 0
    for an opaque sample).
  * w_i = fl(a_i T_{i-1}): da_i T_{i-1} + a_i dT_{i-1} + u w_i.
  * Sums of products, bounded by gamma_k sum |terms| (gamma_k = k u / (1 - k u)) plus the operands' errors. The number
    of roundings k depends on the evaluation order (`order`):
      warp    per-lane fma accumulators over ceil(n_comp / 32) trips, then a 5-level butterfly: k = ceil(n_comp / 32) + 6;
              inclusive prefixes in trip k: the product, a 5-level add scan and one carry add per earlier trip: k = 6 + trip;
              S = sum dws ws over all n samples by lane then butterfly: k = ceil(n / 32) + 6;
      serial  the reference's running sums: k = n_comp + 1 (forward), i + 2 (prefix at sample i), n + 1 (S; any order of
              n terms, which also covers thrust's scan).
    One more rounding than a fused multiply-add needs is counted everywhere, so an implementation that rounds the
    product separately (the numpy replay) is covered too.
  * The backward's brackets c T - (C - r): |c| dT + u |c T| + (dC_sum + dr + u |C - r|) + u |bracket|. The cancellation
    C - r near the end of a ray is the reference's too: its bound is absolute in dC_sum + dr, not relative to C - r.
  * g = sum of the terms: sum of their bounds + (terms) u sum |terms|;  dsig = fl(d g): d dg + u |dsig|.
  * The loss gradients from the kernel's own out and O: dL/dout through e = fl(out - gt), 2 e, * fl(1/n), * fl(1/3)
    (4 roundings); log through logf (1 ulp) and the quotient d(op) / op.
Termination: the kernel's T_i and float64's are only known to lie within SAFETY dT_i of each other. A ray on which some
|T_i - T_threshold| <= SAFETY dT_i, for i up to the float64 termination index + 1, is `undecidable`: there the kernel may
composite one sample more or less, and no rounding bound applies. Such rays are reported, not hidden in the tolerance.
"""
import math

import torch

U = 2.0 ** -24       # fp32 unit roundoff (round to nearest)
ULP = 2.0 ** -23     # one fp32 ulp relative to the value it is measured at (upper bound over a binade)
TINY = 2.0 ** -126   # absolute floor of one fp32 rounding when subnormals flush to zero
SAFETY = 2.0         # the tests compare with SAFETY * bound: second-order terms of the first-order bound
SIGMA_CLAMP = 3.2690173e6  # exp(15): the largest density the network emits (the loss-scale maximum clamps with it)


def gamma(k):
    k = k.double() if torch.is_tensor(k) else torch.tensor(float(k), dtype=torch.float64)
    return k * U / (1 - k * U)


def pad(x, offsets, counts, L=None):
    """ragged per-sample values (N,) or (N, 3) at offsets / counts -> (R, L) or (R, L, 3) float64, 0 past each ray"""
    offsets, counts = offsets.long(), counts.long()
    if L is None:
        L = max(int(counts.max()) if counts.numel() else 0, 1)
    pos = torch.arange(L, device=offsets.device)
    valid = pos[None] < counts[:, None]
    xf = torch.cat([x.double(), torch.zeros((1,) + tuple(x.shape[1:]), dtype=torch.float64, device=x.device)])
    idx = torch.where(valid, offsets[:, None] + pos[None], xf.shape[0] - 1)
    return xf[idx]


def forward(sigmas, rgbs, deltas, ts, offsets, counts, T_thr, order="warp"):
    """compositing forward of every ray. sigmas, deltas, ts (N,), rgbs (N, 3) fp32 as the kernel read them; offsets,
    counts (R,) int. Returns a dict of padded per-sample tensors and per-ray results, each value with its bound `*_err`."""
    assert order in ("warp", "serial")
    counts = counts.long()
    dev = counts.device
    R = counts.numel()
    L = max(int(counts.max()) if R else 0, 1)
    pos = torch.arange(L, device=dev)
    valid = pos[None] < counts[:, None]
    sg, dl, t = (pad(v, offsets, counts, L) for v in (sigmas, deltas, ts))
    c = pad(rgbs, offsets, counts, L)
    thr = float(torch.tensor(float(T_thr), dtype=torch.float32))  # the kernel compares with the fp32 threshold

    x = sg * dl  # exact: the product of two floats fits a double
    e = torch.exp(-x)
    a = -torch.expm1(-x)
    de = (2 + torch.floor(1.173 * x)) * ULP * e + e * U * x + TINY
    da = torch.where(valid, de + U * a + TINY, 0)
    dom = torch.where(valid, da + U * e + TINY, 0)
    om = torch.where(valid, e, 1)

    Tinc, dTinc = torch.empty_like(x), torch.empty_like(x)
    T = torch.ones(R, dtype=torch.float64, device=dev)
    dT = torch.zeros_like(T)
    for j in range(L):
        Tn = T * om[:, j]
        dT = om[:, j] * dT + T * dom[:, j] + (U * Tn + TINY) * valid[:, j]
        T = Tn
        Tinc[:, j], dTinc[:, j] = T, dT
    one = torch.ones(R, 1, dtype=torch.float64, device=dev)
    Texc = torch.cat([one, Tinc[:, :-1]], 1)
    dTexc = torch.cat([one * 0, dTinc[:, :-1]], 1)

    comp = valid & ((pos[None] == 0) | (Texc > thr))
    a = torch.where(valid, a, 0)
    w = torch.where(comp, a * Texc, 0)
    dw = torch.where(comp, da * Texc + a * dTexc + U * w + TINY, 0)
    n_comp = comp.sum(1)
    terminated = (valid & (Tinc <= thr)).any(1)
    total = n_comp - terminated.long()

    if order == "warp":
        k_fw = (n_comp + 31) // 32 + 6
    else:
        k_fw = n_comp + 1
    gf = gamma(k_fw)
    ca, ta = c.abs(), t.abs()
    C = (w[..., None] * c).sum(1)
    C_err = (dw[..., None] * ca).sum(1) + gf[:, None] * (w[..., None] * ca).sum(1)
    O = w.sum(1)
    O_err = dw.sum(1) + gf * O
    D = (w * t).sum(1)
    D_err = (dw * ta).sum(1) + gf * (w * ta).sum(1)

    # termination decided by the same comparisons in both: undecidable where one of them is within the bound
    first = torch.where((valid & (Tinc <= thr)).any(1), (valid & (Tinc <= thr)).float().argmax(1), counts - 1)
    near = valid & ((Tinc - thr).abs() <= SAFETY * dTinc) & (pos[None] <= first[:, None] + 1)
    undecidable = near.any(1)
    return dict(order=order, thr=thr, L=L, counts=counts, valid=valid, comp=comp, sg=sg, dl=dl, t=t, c=c, a=a, da=da,
                Tinc=Tinc, dTinc=dTinc, Texc=Texc, dTexc=dTexc, w=w, w_err=dw, n_comp=n_comp, total=total,
                terminated=terminated, undecidable=undecidable, C=C, C_err=C_err, O=O, O_err=O_err, D=D, D_err=D_err)


def with_background(fw, bg):
    """out = C + bg (1 - O) as the kernels form it (rest = fl(1 - O), fl(bg rest), fl(C + .)); bg (3,) or (R, 3)"""
    bg = torch.as_tensor(bg, dtype=torch.float64, device=fw["C"].device).expand_as(fw["C"])
    rest = 1 - fw["O"]
    out = fw["C"] + bg * rest[:, None]
    out_err = fw["C_err"] + bg.abs() * (fw["O_err"] + U * rest.abs())[:, None] + U * (bg * rest[:, None]).abs() + \
        U * out.abs()
    return out, out_err


def nerf_loss(fw, gt, bg, lam, n_rays):
    """NeRFLoss on the composited output and its per-ray gradients, as the kernels form them from their own out and O.
    dL_dopacity is what ngp_nerf_loss_grad writes, dO the opacity gradient with the background's share that the fused
    kernel uses. loss / loss_err: the batch loss (stats()["loss"]), its fp32 sums in any order."""
    out, out_err = with_background(fw, bg)
    bg = torch.as_tensor(bg, dtype=torch.float64, device=out.device).expand_as(out)
    gt = gt.double()
    e = out - gt
    e_err = out_err + U * e.abs()
    k = 2.0 / (3 * n_rays)
    dC = k * e
    dC_err = k * e_err + 4 * U * dC.abs()
    op = fw["O"] + 1e-10
    op_err = fw["O_err"] + U * op
    lg = torch.log(op)
    lg_err = op_err / op + ULP * lg.abs() + TINY
    A = -lg - 1
    dLdO = lam * A / n_rays
    dLdO_err = lam / n_rays * (lg_err + U * A.abs() + 4 * U * A.abs())  # fl(-lg - 1), fp32 lambda, * , fl(1/n), *
    cb = (dC * bg).sum(1)
    dO = dLdO - cb
    dO_err = dLdO_err + (dC_err * bg.abs()).sum(1) + 3 * U * (dC * bg).abs().sum(1) + U * dO.abs()
    se = (e * e).sum(1)
    se_err = (2 * e.abs() * e_err).sum(1) + 3 * U * se
    ent = -op * lg
    ent_err = lg.abs() * op_err + op * lg_err + U * ent.abs()
    gR = gamma(fw["counts"].numel())
    loss = float(se.sum()) / (3 * n_rays) + lam * float(ent.sum()) / n_rays
    loss_err = float(se_err.sum() + gR * se.sum()) / (3 * n_rays) + lam * float(ent_err.sum() + gR * ent.abs().sum()) / n_rays
    return dict(out=out, out_err=out_err, dC=dC, dC_err=dC_err, dL_dopacity=dLdO, dL_dopacity_err=dLdO_err, dO=dO,
                dO_err=dO_err, loss=loss, loss_err=loss_err)


def _bracket(v, Tinc, dTinc, tot, tot_err, pre, pre_err):
    """v T - (tot - pre) as the kernels form it, and its bound"""
    behind = tot[:, None] - pre
    X = v * Tinc - behind
    X_err = v.abs() * dTinc + U * (v * Tinc).abs() + tot_err[:, None] + pre_err + U * behind.abs() + U * X.abs()
    return X, X_err


def backward(fw, dC, dO, dD=None, dws=None, dC_err=None, dO_err=None, bg=None, offsets=None):
    """compositing backward: (dsig, dsig_err) (R, L) and (drgb, drgb_err) (R, L, 3), exactly 0 past n_comp.
    dC (R, 3), dO (R,), dD (R,) are the upstream gradients the kernel uses (with bounds dC_err / dO_err when the kernel
    computed them itself); dws (N,) per-sample dL/dws at `offsets` (read against the forward's ws).
    bg: the separate backward kernel's convention -- it recovers C = out - bg (1 - O) from the stored output and routes
    the background's share into dO itself; None: C and dO are the fused kernel's own."""
    order, valid, comp, w, dw = fw["order"], fw["valid"], fw["comp"], fw["w"], fw["w_err"]
    Tinc, dTinc, c, t = fw["Tinc"], fw["dTinc"], fw["c"], fw["t"]
    dev = w.device
    R, L = w.shape
    z = torch.zeros(R, dtype=torch.float64, device=dev)
    dC = dC.double()
    dO = dO.double()
    dC_err = z[:, None].expand_as(dC) if dC_err is None else dC_err
    dO_err = z if dO_err is None else dO_err
    C, C_err = fw["C"], fw["C_err"]
    if bg is not None:
        out, _ = with_background(fw, bg)
        C_err = C_err + U * (out.abs() + C.abs())  # fl(fl(C + b) - b)
        bgt = torch.as_tensor(bg, dtype=torch.float64, device=dev).expand_as(dC)
        cb = (dC * bgt).sum(1)
        dO = dO - cb
        dO_err = dO_err + (dC_err * bgt.abs()).sum(1) + 3 * U * (dC * bgt).abs().sum(1) + U * dO.abs()
    pos = torch.arange(L, device=dev)
    if order == "warp":
        k_pre = 6 + pos // 32
    else:
        k_pre = pos + 2
    gp = gamma(k_pre)[None]

    terms, errs = [], []
    wc = w[..., None] * c
    r = torch.cumsum(wc, 1)
    r_err = torch.cumsum(dw[..., None] * c.abs(), 1) + gp[..., None] * torch.cumsum(wc.abs(), 1)
    for ch in range(3):
        X, X_err = _bracket(c[..., ch], Tinc, dTinc, C[:, ch], C_err[:, ch], r[..., ch], r_err[..., ch])
        terms.append(dC[:, ch, None] * X)
        errs.append(dC_err[:, ch, None] * X.abs() + dC[:, ch, None].abs() * X_err + U * terms[-1].abs())
    rest = 1 - fw["O"]
    terms.append((dO * rest)[:, None].expand(R, L))
    errs.append((dO_err * rest.abs() + dO.abs() * (fw["O_err"] + U * rest.abs()) + U * (dO * rest).abs())[:, None].expand(R, L))
    if dD is not None:
        dD = dD.double()
        wt = w * t
        d_pre = torch.cumsum(wt, 1)
        d_err = torch.cumsum(dw * t.abs(), 1) + gp * torch.cumsum(wt.abs(), 1)
        X, X_err = _bracket(t, Tinc, dTinc, fw["D"], fw["D_err"], d_pre, d_err)
        terms.append(dD[:, None] * X)
        errs.append(dD[:, None].abs() * X_err + U * terms[-1].abs())
    if dws is not None:
        dv = pad(dws, offsets, fw["counts"], L)
        dvw = dv * w
        s_pre = torch.cumsum(dvw, 1)
        s_err = torch.cumsum(dv.abs() * dw, 1) + gp * torch.cumsum(dvw.abs(), 1)
        k_S = (fw["counts"] + 31) // 32 + 6 if order == "warp" else fw["counts"] + 1
        S = dvw.sum(1)
        S_err = (dv.abs() * dw).sum(1) + gamma(k_S) * dvw.abs().sum(1)
        X, X_err = _bracket(dv, Tinc, dTinc, S, S_err, s_pre, s_err)
        terms.append(X)
        errs.append(X_err)
    g = sum(terms)
    g_err = sum(errs) + len(terms) * U * sum(v.abs() for v in terms)
    dsig = torch.where(comp, fw["dl"] * g, 0)
    dsig_err = torch.where(comp, fw["dl"] * g_err + U * dsig.abs() + TINY, 0)
    drgb = torch.where(comp[..., None], dC[:, None, :] * w[..., None], 0)
    drgb_err = torch.where(comp[..., None], dC_err[:, None, :] * w[..., None] + dC[:, None, :].abs() * dw[..., None] +
                           U * drgb.abs() + TINY, 0)
    return dict(dsig=dsig, dsig_err=dsig_err, drgb=drgb, drgb_err=drgb_err)


def loss_scale(dsig, drgb, sig):
    """the power-of-two loss scale k_train_grad_scale derives from the compositing backward's outputs, recomputed in fp32
    as the kernels do: m = max(|dsig min(sigma, exp(15))|, |drgb|), scale = 2^clamp(floor(log2(256 / m)), -60, 60)"""
    f = torch.float32
    m = torch.maximum((dsig.to(f) * sig.to(f).clamp_max(SIGMA_CLAMP)).abs().max(), drgb.to(f).abs().max())
    if not (0 < float(m) < math.inf):
        return 1.0
    _, e = torch.frexp(torch.tensor(256.0, dtype=f, device=m.device) / m)
    return math.ldexp(1.0, max(-60, min(60, int(e) - 1)))


def ratio(err, bound):
    """largest |err| / (SAFETY bound) (0 where both are 0; inf where the bound is 0 and err is not)"""
    err, bound = err.double().abs(), SAFETY * bound.double()
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0
