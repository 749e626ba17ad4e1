"""Test-view images on the host: the generated turbo table, oracle/images_ref.py against the reference's own depth2img
(tests/golden/images.npz, tests/golden/make_golden_images.py), the PNG restatement oracle/png_ref.py against its
decoder and Pillow, the capacity formula, the filter tie rule, and the refusal of CPU tensors."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import images_ref as R
from oracle import png_ref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "images.npz")
SIZES = [(1, 1), (1, 23), (19, 1), (17, 13), (64, 48)]
KINDS = ["noise", "flat", "gradient"]


def make_image(H, W, kind, seed=0):
    if kind == "noise":
        return np.random.RandomState(seed + H * 131 + W).randint(0, 256, (H, W, 3)).astype(np.uint8)
    if kind == "flat":
        return np.full((H, W, 3), 255, np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    return np.stack([xx * 255 // max(W - 1, 1), yy * 255 // max(H - 1, 1), (xx + 2 * yy) % 256], -1).astype(np.uint8)


def test_turbo_table_regenerates_identically():
    pytest.importorskip("cv2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "turbo_table.py"), "--check"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert r.returncode == 0, r.stdout.decode()


def test_images_ref_equals_reference_depth2img():
    z = np.load(GOLDEN)
    names = sorted(k[6:] for k in z.files if k.startswith("depth_"))
    assert names == ["constant", "lego", "nan", "ramp", "smooth", "zero_bg"]
    for n in names:
        d, want = z["depth_" + n], z["img_" + n]
        got = R.depth_image(d, *d.shape)
        assert got.dtype == np.uint8 and got.shape == want.shape
        assert np.array_equal(got, want), n
    # the constant and NaN maps are index 0 everywhere
    for n in ("constant", "nan"):
        assert (z["img_" + n] == R.depth_image(np.zeros((1, 1), np.float32), 1, 1)[0, 0]).all()


def test_rgb_ref_is_numpy_cast():
    v = np.array([0, 1 / 255, 0.5, 254.9999 / 255, 1.0, np.nextafter(np.float32(256 / 255), np.float32(0)), np.nan],
                 np.float32)
    rgb = np.repeat(v[:, None], 3, 1)
    got = R.rgb_image(rgb, 1, len(v))
    want = np.where(np.isnan(rgb), 0, np.nan_to_num(rgb) * np.float32(255)).astype(np.uint8).reshape(1, len(v), 3)
    assert np.array_equal(got, want)
    assert got[0, :, 0].tolist() == [0, 1, 127, 254, 255, 255, 0]


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("kind", KINDS)
def test_png_restatement_round_trips(H, W, kind):
    img = make_image(H, W, kind)
    data = P.encode(img)
    assert len(data) <= P.capacity(H, W)
    assert np.array_equal(P.decode(data), img)  # every chunk CRC and the Adler-32 checked
    Image = pytest.importorskip("PIL.Image")
    with Image.open(io.BytesIO(data)) as im:
        assert im.mode == "RGB" and im.size == (W, H)
        assert np.array_equal(np.array(im), img)


def test_noise_takes_the_stored_fallback_and_flat_compresses():
    H, W = 64, 48
    assert len(P.encode(make_image(H, W, "noise"))) == P.capacity(H, W)  # every segment stored
    assert len(P.encode(make_image(H, W, "flat"))) < P.capacity(H, W) // 10


def test_capacity_formula_matches_library():
    from ngp_pl_b200 import _lib
    lib = _lib.lib()
    for H, W in SIZES + [(800, 800), (3, 21845), (2, 40000)]:
        assert lib.ngp_png_capacity(H, W) == P.capacity(H, W)
        assert lib.ngp_png_workspace(H, W) > 0
    for H, W in [(0, 5), (5, 0), (-1, 3), (1 << 20, 1 << 12)]:  # empty, or an IDAT over 2^31 - 1 bytes
        assert lib.ngp_png_capacity(H, W) == 0 and lib.ngp_png_workspace(H, W) == 0


def test_filter_tie_goes_to_lowest_type():
    # Up and Paeth both filter this row to zeros; None, Sub and Average do not
    x, up = [10] * 6, [10] * 6
    f, out = P.filter_row(x, up)
    assert f == 2 and out == [0] * 6
    # a repeated pixel on the first row: Sub alone is the smallest
    f, out = P.filter_row([1, 200, 3, 1, 200, 3], [0] * 6)
    assert f == 1 and out == [1, 200, 3, 0, 0, 0]
    # one pixel on the first row: all five filters give the same bytes, None wins
    f, out = P.filter_row([1, 2, 3], [0, 0, 0])
    assert f == 0 and out == [1, 2, 3]


def test_cpu_tensors_are_refused(tmp_path):
    from ngp_pl_b200 import images
    with pytest.raises(RuntimeError):
        images.rgb_image(torch.zeros(4, 3), 2, 2)
    with pytest.raises(RuntimeError):
        images.depth_image(torch.zeros(4), 2, 2)
    with pytest.raises(RuntimeError):
        images.encode_png(torch.zeros(2, 2, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        images.write_png(str(tmp_path / "a.png"), torch.zeros(2, 2, 3, dtype=torch.uint8))
    assert not os.path.exists(tmp_path / "a.png")
