"""float64 restatement of the distortion loss and its gradient, with a bound on how far an fp32 implementation may lie
from every value -- TEST INFRASTRUCTURE ONLY.

Nothing under ngp_pl_b200/ imports this. Plain torch on any device, in composite64's padded (ray, sample) layout, so the
GPU tests run it on CUDA at training sizes and the CPU suite holds it to the C oracle, to the reference kernels' own
outputs (tests/golden/composite.npz) and to a float32 replay of k_distortion_fw / k_distortion_bw.

Semantics (reference losses.cu:10-174, Mip-NeRF 360's distortion loss), from the kernel's own fp32 ws, ts, deltas:
  W_i, WT_i   inclusive scans of w and w t over the ray
  loss        sum_i 2 (WT_i W_{i-1} - W_i WT_{i-1}) + 1/3 w_i^2 d_i
              = sum_i sum_j w_i w_j |t_i - t_j| + 1/3 sum_i w_i^2 d_i     (t non-decreasing along the ray)
  dL/dw_i     g [2 (head_i + tail_i) + 2/3 w_i d_i],  head_i = t_i W_{i-1} - WT_{i-1},  tail_i = (WT_n - WT_i) - t_i (W_n - W_i)
              = g [2 sum_j w_j |t_i - t_j| + 2/3 w_i d_i]
The products in the loss and in the brackets are each about t W^2 while their difference is about w W dt: the formula
cancels, most on long rays at large t. The bound therefore is absolute in the magnitudes of the cancelling products,
never relative to the result.

The bound (`*_err`) is first order in u = 2^-24, composite64's method and constants (U, TINY, SAFETY, gamma):
  * wt = fl(w t): u |w t|.
  * Scans of non-negative terms: gamma_k sum |terms| plus the terms' own errors. warp: a 5-level Hillis-Steele add scan
    per 32-sample trip, the add of the previous trip's carry and one carry add per earlier trip, k = 6 + trip;
    serial: k = i + 1 at sample i, which covers any order of the i + 1 terms (the C oracle's loop, thrust's scan).
  * The loss terms 2 (WT_i Wx_i - W_i WTx_i), with the exclusive values the kernel forms as Wx = fl(W - w),
    WTx = fl(WT - wt): to first order the scan errors dW, dWT and the rounding dwt of wt enter as
    |wt| dW + |w| dWT + |W| dwt (the products' shares of them cancel), the roundings of Wx, WTx and of the two products
    as 2 u (|WT Wx| + |W WTx|), and the difference adds u |D|.
  * The backward brackets: |a| db + |b| da + u |ab| for each product, u |a - b| for each difference; their operands are
    the stored scans, whose errors do not cancel there.
  * 1/3 w w d and g 2/3 w d: four roundings (the constant and three products).
  * The loss: the terms' errors plus gamma_k sum |terms|; warp: per-lane accumulators over ceil(n / 32) trips and a
    5-level butterfly, k = ceil(n / 32) + 6; serial (any order of n terms): k = n + 1.
  * Every rounding also has an absolute floor TINY (flush to zero).
One rounding more than a fused multiply-add needs is counted everywhere, so contracted and uncontracted code are both
covered. There is no data-dependent branch in these kernels: every ray is decidable.
"""
import torch

from oracle.composite64 import SAFETY, TINY, U, gamma, pad, ratio  # noqa: F401  (SAFETY, ratio: for the tests)


def _at_last(x, counts):
    """x[r, counts[r] - 1] (0 for an empty ray)"""
    idx = (counts - 1).clamp_min(0)[:, None]
    return torch.where(counts > 0, x.gather(1, idx)[:, 0], torch.zeros_like(x[:, 0]))


def forward(ws, deltas, ts, offsets, counts, order="warp"):
    """distortion loss of every ray. ws, deltas, ts (N,) fp32 as the kernel read them; offsets, counts (R,) int, indexed
    by ray. Returns the padded per-sample scans W, WT and the per-ray loss, each with its bound `*_err`, and what
    backward() needs."""
    assert order in ("warp", "serial")
    counts = counts.long()
    dev = counts.device
    R = counts.numel()
    L = max(int(counts.max()) if R else 0, 1)
    pos = torch.arange(L, device=dev)
    valid = pos[None] < counts[:, None]
    w, t, dl = (pad(v, offsets, counts, L) for v in (ws, ts, deltas))
    wt = w * t  # exact: the product of two floats fits a double
    wt_err = torch.where(valid, U * wt.abs() + TINY, 0)

    k_scan = (6 + pos // 32) if order == "warp" else (pos + 1)
    gs = gamma(k_scan)[None]
    kt = k_scan[None].double() * TINY
    W = torch.cumsum(w, 1)
    WT = torch.cumsum(wt, 1)
    W_err = torch.where(valid, gs * torch.cumsum(w.abs(), 1) + kt, 0)
    WT_err = torch.where(valid, torch.cumsum(wt_err, 1) + gs * torch.cumsum(wt.abs(), 1) + kt, 0)

    # D = WT Wx - W WTx with the kernel's exclusive values Wx = fl(W - w), WTx = fl(WT - wt). To first order the scans'
    # errors enter only through WT - WTx = wt and W - Wx = w (and the rounding of wt through W): the scans' share does
    # not cancel, the four roundings of the two exclusive values and the two products, each about |P1| or |P2|, do.
    Wx, WTx = W - w, WT - wt
    P1, P2 = WT * Wx, W * WTx
    D = w * (t * Wx - WTx)  # = P1 - P2, without float64's own cancellation
    D_err = wt.abs() * W_err + w.abs() * WT_err + W.abs() * wt_err + 2 * U * (P1.abs() + P2.abs()) + U * D.abs() + \
        5 * TINY
    q = w * w * dl / 3
    q_err = 4 * U * q.abs() + TINY
    s = torch.where(valid, 2 * D + q, 0)
    s_err = torch.where(valid, 2 * D_err + q_err + U * s.abs() + TINY, 0)
    k_acc = (counts + 31) // 32 + 6 if order == "warp" else counts + 1
    loss = s.sum(1)
    loss_err = s_err.sum(1) + gamma(k_acc) * s.abs().sum(1) + k_acc.double() * TINY
    loss_err = torch.where(counts > 0, loss_err, 0)
    return dict(order=order, L=L, counts=counts, valid=valid, w=w, t=t, dl=dl, W=W, W_err=W_err, WT=WT, WT_err=WT_err,
                terms=s, terms_err=s_err, loss=loss, loss_err=loss_err)


def backward(fw, g):
    """dL/dws of every sample, padded (R, L), exactly 0 past each ray, for the per-ray upstream gradient g (R,) (fp32
    as the kernel read it). Reads the forward's scans as the kernel reads ws_inc / wts_inc."""
    valid, w, t, dl, counts = fw["valid"], fw["w"], fw["t"], fw["dl"], fw["counts"]
    W, W_err, WT, WT_err = fw["W"], fw["W_err"], fw["WT"], fw["WT_err"]
    g = g.double()[:, None]
    R, L = w.shape
    z = torch.zeros(R, 1, dtype=torch.float64, device=w.device)
    Wp, Wp_err = torch.cat([z, W[:, :-1]], 1), torch.cat([z, W_err[:, :-1]], 1)
    WTp, WTp_err = torch.cat([z, WT[:, :-1]], 1), torch.cat([z, WT_err[:, :-1]], 1)
    first = torch.arange(L, device=w.device)[None] == 0
    tWp = t * Wp
    head = torch.where(first, 0, tWp - WTp)
    head_err = torch.where(first, 0, t.abs() * Wp_err + U * tWp.abs() + WTp_err + U * head.abs() + 2 * TINY)
    Wn, Wn_err = _at_last(W, counts)[:, None], _at_last(W_err, counts)[:, None]
    WTn, WTn_err = _at_last(WT, counts)[:, None], _at_last(WT_err, counts)[:, None]
    a = WTn - WT
    a_err = WTn_err + WT_err + U * a.abs() + TINY
    b = Wn - W
    b_err = Wn_err + W_err + U * b.abs() + TINY
    tb = t * b
    tb_err = t.abs() * b_err + U * tb.abs() + TINY
    tail = a - tb
    tail_err = a_err + tb_err + U * tail.abs() + TINY
    hs = head + tail
    hs_err = head_err + tail_err + U * hs.abs() + TINY
    p = 2 * g * hs
    p_err = 2 * g.abs() * hs_err + U * p.abs() + TINY
    r = g * (2.0 / 3.0) * w * dl
    r_err = 4 * U * r.abs() + TINY
    dws = torch.where(valid, p + r, 0)
    dws_err = torch.where(valid, p_err + r_err + U * dws.abs() + TINY, 0)
    return dict(dws=dws, dws_err=dws_err)


def pair_sums(ws, deltas, ts, offsets, counts):
    """the definition, O(n^2) per ray: loss = sum_ij w_i w_j |t_i - t_j| + 1/3 sum_i w_i^2 d_i and
    dL/dw_i / g = 2 sum_j w_j |t_i - t_j| + 2/3 w_i d_i, in float64 (padded (R,) and (R, L)); rays one at a time"""
    counts = counts.long()
    R = counts.numel()
    L = max(int(counts.max()) if R else 0, 1)
    w, t, dl = (pad(v, offsets, counts, L) for v in (ws, ts, deltas))
    loss = torch.zeros(R, dtype=torch.float64, device=w.device)
    dws = torch.zeros(R, L, dtype=torch.float64, device=w.device)
    for r in range(R):
        n = int(counts[r])
        wr, tr, dr = w[r, :n], t[r, :n], dl[r, :n]
        Aw = (tr[:, None] - tr[None]).abs() @ wr
        loss[r] = (wr * Aw).sum() + (wr * wr * dr).sum() / 3
        dws[r, :n] = 2 * Aw + (2.0 / 3.0) * wr * dr
    return loss, dws
