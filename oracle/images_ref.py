"""numpy restatement of the validation pass's test-view images (reference train.py:215-221) -- TEST INFRASTRUCTURE ONLY.

rgb_image(rgb, H, W)      (rgb_pred * 255).astype(np.uint8) on an (H*W, 3) float32 render
depth_image(depth, H, W)  depth2img (train.py:45-50): per-view min/max normalisation in float32, * 255, uint8, then
                          cv2.applyColorMap(COLORMAP_TURBO) -- here from oracle/turbo_table.py, the table the kernel
                          uses, so no OpenCV is needed; cv2's B, G, R order is kept, as the reference's _d.png files hold it

The casts follow numpy on x86: NaN -> 0. Kept in float32 throughout, as numpy >= 1 computes depth2img on a float32 map.
"""
import numpy as np

from .turbo_table import TURBO_BGR

_TURBO = np.array(TURBO_BGR, dtype=np.uint8)


def _to_u8(x):
    """float32 -> uint8 by truncation, NaN -> 0 (for x in [0, 256) or NaN, where numpy's cast is defined)"""
    x = np.asarray(x, np.float32)
    out = np.zeros(x.shape, np.uint8)
    ok = ~np.isnan(x)
    out[ok] = x[ok].astype(np.uint8)
    return out


def rgb_image(rgb, H, W):
    rgb = np.asarray(rgb, np.float32).reshape(H, W, 3)
    return _to_u8(rgb * np.float32(255))


def depth_index(depth):
    d = np.asarray(depth, np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        n = (d - d.min()) / (d.max() - d.min())
        return _to_u8(n * np.float32(255))


def depth_image(depth, H, W):
    return _TURBO[depth_index(np.asarray(depth, np.float32).reshape(H, W))]
