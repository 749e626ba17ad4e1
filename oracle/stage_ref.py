"""numpy float32 restatement of the image staging kernel (ngp_pl_b200/csrc/stage.cu, ngp_stage_image), i.e. of the
reference's `read_image` (datasets/color_utils.py:19-31): uint8 -> /255 -> alpha blend -> cv2.resize(INTER_LINEAR).

cv2 does not document the evaluation order of its fp32 bilinear path. Measured against cv2.resize (opencv 4.13) over
random sizes from 2 to 300 per axis, down- and up-scaling, exact halving included (no INTER_AREA shortcut on fp32):
the result is bitwise
    f = (d + 0.5) * (S / D) - 0.5   (float64),   s = floor(f),   a = float32(f - s)
    clamp: s < 0 -> (0, a = 0);  s >= S - 1 -> (S - 1, a = 0)
    t = fma(a, p[s + 1] - p[s], p[s])   (float32, one rounding)
along x on the two source rows, then along y. tests/test_datasets_cpu.py holds this module to cv2 and the kernel is held
to the golden files it produces (tests/golden/datasets_*.npz), never to cv2 on the GPU machine.
"""
import numpy as np

f32, f64 = np.float32, np.float64


def fma32(a, b, c):
    """float32 fma(a, b, c) with a single rounding. a*b is exact in float64; the float64 sum is rounded to odd (TwoSum
    error term) so that the final cast to float32 rounds correctly, with no double-rounding case left."""
    a, b, c = (np.asarray(v, f32).astype(f64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    bits = s.view(np.int64)
    inexact_even = (err != 0) & ((bits & 1) == 0)
    s = np.where(inexact_even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def to_unit(img_u8, blend_a=True):
    """uint8 (H, W, C in {3, 4}) -> float32 (H, W, 3), reference color_utils.py:20-26"""
    img = img_u8.astype(f32) / f32(255.0)
    if img.shape[2] == 4:
        c, a = img[..., :3], img[..., -1:]
        img = c * a + (f32(1) - a) if blend_a else c * a
    return img.astype(f32)


def _coeffs(S, D):
    f = (np.arange(D, dtype=f64) + 0.5) * (S / D) - 0.5
    s = np.floor(f).astype(np.int64)
    a = (f - s).astype(f32)
    lo = s < 0
    s, a = np.where(lo, 0, s), np.where(lo, f32(0), a)
    hi = s >= S - 1
    s, a = np.where(hi, S - 1, s), np.where(hi, f32(0), a)
    return s, np.minimum(s + 1, S - 1), a


def resize_linear(img, w, h):
    """cv2.resize(img, (w, h)) for a float32 (H0, W0, C) image, C > 0, H0, W0 >= 2 (or no size change)"""
    img = np.asarray(img, f32)
    H0, W0 = img.shape[:2]
    if (w, h) == (W0, H0):
        return img.copy()
    x0, x1, ax = _coeffs(W0, w)
    y0, y1, ay = _coeffs(H0, h)
    p0, p1 = img[:, x0], img[:, x1]
    t = fma32(ax[None, :, None], p1 - p0, p0)
    t0, t1 = t[y0], t[y1]
    return fma32(ay[:, None, None], t1 - t0, t0)


def stage_image(img_u8, w, h, blend_a=True):
    """what ngp_stage_image writes: float32 (h*w, 3)"""
    return resize_linear(to_unit(img_u8, blend_a), w, h).reshape(-1, 3)
