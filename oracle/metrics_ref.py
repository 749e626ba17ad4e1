"""Float64 restatement of the validation metrics of the reference's train.py:193-237, written from the formulas:

    PSNR (metrics.py:14-15, torchmetrics PeakSignalNoiseRatio(data_range=1)):  -10 * log10(sse / (3 * H * W))
    SSIM (torchmetrics StructuralSimilarityIndexMeasure(data_range=1), defaults):
        Gaussian window, sigma = 1.5, int(3.5 * sigma + 0.5) * 2 + 1 = 11 taps; fp32 1D weights exp(-(x / sigma)^2 / 2)
        normalised to sum 1; the 2D window is the outer product of the 1D one.
        c1 = (0.01 * data_range)^2, c2 = (0.03 * data_range)^2
        per channel the five windowed moments mu_p, mu_t, E[p^2], E[t^2], E[pt];
        s = (2 mu_p mu_t + c1)(2 (E[pt] - mu_p mu_t) + c2) / ((mu_p^2 + mu_t^2 + c1)(E[p^2] - mu_p^2 + E[t^2] - mu_t^2 + c2))
        torchmetrics reflect-pads by 5, correlates, and crops 5 off every side again: only windows lying wholly inside the
        image count (centres [5, H-5) x [5, W-5)); the result is the mean over those centres and the three channels.
    The variances are NOT clamped at zero: the torchmetrics releases of the reference's pytorch-lightning 1.7.7 era do not
    clamp them (later releases clamp E[p^2] - mu_p^2 and E[t^2] - mu_t^2 at 0; the two differ only where a variance rounds
    below zero, which float64 over [0, 1] images does not reach beyond ~1e-17).

Two independent computations of the SSIM: `ssim_conv` (the torchmetrics recipe as written: reflect pad, full 2D correlation
with the 11 x 11 window, crop) and `ssim_direct` (a sum over each fully-inside 11 x 11 window, one centre at a time).
Images are (H, W, 3) arrays: float32 in [0, 1], or uint8 read as value / 255 in fp32 (how the training images are
stored and how torch's `.float() / 255` reads them).
"""
import numpy as np

SIGMA = 1.5
KSIZE = int(3.5 * SIGMA + 0.5) * 2 + 1  # 11
RADIUS = (KSIZE - 1) // 2                # 5


def gaussian_weights(sigma=SIGMA, ksize=KSIZE):
    """fp32 1D window: e_i = fp32(exp(-(x_i / sigma)^2 / 2)) with x_i / sigma, its square and the halving in fp32;
    S = fp32(sum of the e_i) rounded once (the float64 sum of 11 fp32 values spanning 17 binades is exact);
    w_i = e_i / S in fp32. libngp_b200 builds its window with the same operations."""
    x = np.arange((1 - ksize) / 2, (1 + ksize) / 2, 1, dtype=np.float32)
    a = x / np.float32(sigma)
    arg = -(a * a) / np.float32(2)
    e = np.exp(arg.astype(np.float64)).astype(np.float32)
    s = np.float32(np.sum(e.astype(np.float64)))
    return e / s


def as_unit(img):
    """(H, W, 3) image as float64 values in [0, 1]: uint8 -> fp32(v / 255), fp32 as is"""
    img = np.asarray(img)
    if img.dtype == np.uint8:
        return (img.astype(np.float32) / np.float32(255)).astype(np.float64)
    return img.astype(np.float32).astype(np.float64)


def sse(pred, gt):
    d = as_unit(pred) - as_unit(gt)
    return float(np.sum(d * d))


def psnr(pred, gt):
    """-10 log10(mse); +inf for identical images, as torch's log10(0) = -inf gives the reference"""
    p = as_unit(pred)
    with np.errstate(divide="ignore"):
        return float(-10 * np.log10(sse(pred, gt) / p.size))


def _constants(data_range):
    return (0.01 * data_range) ** 2, (0.03 * data_range) ** 2


def _ssim_map(mu_p, mu_t, e_pp, e_tt, e_pt, c1, c2):
    mpp, mtt, mpt = mu_p * mu_p, mu_t * mu_t, mu_p * mu_t
    upper = 2 * (e_pt - mpt) + c2
    lower = (e_pp - mpp) + (e_tt - mtt) + c2
    return ((2 * mpt + c1) * upper) / ((mpp + mtt + c1) * lower)


def ssim_conv(pred, gt, data_range=1.0):
    """(a) the torchmetrics recipe: reflect pad by RADIUS, 2D correlation with the outer-product window (the output of
    torch's conv2d at every position of the padded image), crop RADIUS off every side, mean over centres and channels"""
    p, t = as_unit(pred), as_unit(gt)
    H, W, C = p.shape
    if H < KSIZE or W < KSIZE:
        raise ValueError("SSIM needs an image of at least %d x %d" % (KSIZE, KSIZE))
    w1 = gaussian_weights().astype(np.float64)
    w2 = np.outer(w1, w1)
    c1, c2 = _constants(data_range)
    r = RADIUS
    total = 0.0
    for c in range(C):
        planes = [p[..., c], t[..., c], p[..., c] * p[..., c], t[..., c] * t[..., c], p[..., c] * t[..., c]]
        moments = []
        for x in planes:
            xp = np.pad(x, r, mode="reflect")
            acc = np.zeros((H, W))
            for i in range(KSIZE):
                for j in range(KSIZE):
                    acc += w2[i, j] * xp[i:i + H, j:j + W]
            moments.append(acc)
        s = _ssim_map(*moments, c1, c2)
        total += float(np.sum(s[r:H - r, r:W - r]))
    return total / (C * (H - 2 * r) * (W - 2 * r))


def ssim_direct(pred, gt, data_range=1.0):
    """(b) one fully-inside window at a time: the five weighted moments of the 11 x 11 patch around each centre"""
    p, t = as_unit(pred), as_unit(gt)
    H, W, C = p.shape
    if H < KSIZE or W < KSIZE:
        raise ValueError("SSIM needs an image of at least %d x %d" % (KSIZE, KSIZE))
    w1 = gaussian_weights().astype(np.float64)
    w2 = np.outer(w1, w1)[:, :, None]
    c1, c2 = _constants(data_range)
    r = RADIUS
    total = 0.0
    for y in range(r, H - r):
        for x in range(r, W - r):
            pp, tt = p[y - r:y + r + 1, x - r:x + r + 1], t[y - r:y + r + 1, x - r:x + r + 1]
            mu_p, mu_t = (w2 * pp).sum((0, 1)), (w2 * tt).sum((0, 1))
            e_pp, e_tt, e_pt = (w2 * pp * pp).sum((0, 1)), (w2 * tt * tt).sum((0, 1)), (w2 * pp * tt).sum((0, 1))
            total += float(np.sum(_ssim_map(mu_p, mu_t, e_pp, e_tt, e_pt, c1, c2)))
    return total / (C * (H - 2 * r) * (W - 2 * r))
