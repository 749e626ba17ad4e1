"""The JPEG restatement oracle/jpeg_ref.py against libjpeg (through Pillow: quality=q, subsampling=0, optimize=False), and
images.AviWriter against a RIFF walker written here and, where it is installed, OpenCV. No GPU."""
import io
import struct

import numpy as np
import pytest

from oracle import jpeg_ref as J

SIZES = [(1, 1), (7, 9), (8, 8), (17, 33), (100, 100)]
KINDS = ["noise", "ramp", "flat", "checker", "view"]
QUALITIES = [1, 50, 75, 90, 100]


def make_image(H, W, kind, seed=0):
    yy, xx = np.mgrid[0:H, 0:W]
    if kind == "noise":
        return np.random.RandomState(seed + H * 131 + W).randint(0, 256, (H, W, 3)).astype(np.uint8)
    if kind == "ramp":
        return np.stack([xx * 255 // max(W - 1, 1), yy * 255 // max(H - 1, 1), (xx + yy) * 255 // max(H + W - 2, 1)],
                        -1).astype(np.uint8)
    if kind == "flat":
        return np.full((H, W, 3), (200, 30, 255), np.uint8)
    if kind == "checker":  # saturated, per pixel: the largest coefficient categories, and 0xFF bytes to stuff
        c = (((yy + xx) & 1) * 255).astype(np.uint8)
        return np.stack([c, 255 - c, c], -1)
    # like a rendered view: a shaded, textured disc on a white background, with a little sensor-like noise
    r = np.hypot(yy - H / 2, xx - W / 2) / (0.4 * max(H, W))
    shade = np.clip(1 - r * r, 0, 1) ** 0.5
    tex = 0.5 + 0.5 * np.sin(xx / 3.0) * np.cos(yy / 5.0)
    rgb = np.stack([shade * (0.3 + 0.7 * tex), shade * 0.6, shade * (1 - 0.5 * tex)], -1)
    rgb = np.where((r < 1)[..., None], rgb, 1.0) + np.random.RandomState(seed).randn(H, W, 3) * 0.004
    return (np.clip(rgb, 0, 1) * 255).astype(np.uint8)


def pillow_encode(img, quality):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "JPEG", quality=quality, subsampling=0, optimize=False)
    return buf.getvalue()


def pillow_decode(data, H, W):
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        assert im.mode == "RGB" and im.size == (W, H) and im.format == "JPEG"
        return np.array(im)


def segments(data):
    """{marker: [payloads]} of the segments before the entropy-coded data, and the data itself (between SOS and EOI)"""
    assert data[:2] == b"\xff\xd8" and data[-2:] == b"\xff\xd9"
    p, segs = 2, {}
    while True:
        assert data[p] == 0xFF
        marker, n = data[p + 1], int.from_bytes(data[p + 2:p + 4], "big")
        segs.setdefault(marker, []).append(data[p + 4:p + 2 + n])
        p += 2 + n
        if marker == 0xDA:
            return segs, data[p:-2]


def assert_equals_libjpeg(img, quality):
    ours, theirs = J.encode(img, quality), pillow_encode(img, quality)
    (a, scan_a), (b, scan_b) = segments(ours), segments(theirs)
    for marker in (0xDB, 0xC0, 0xC4, 0xDA):  # DQT, SOF0, DHT, SOS
        assert a[marker] == b[marker], hex(marker)
    assert scan_a == scan_b
    assert len(ours) == 623 + len(scan_a) + 2
    return ours, theirs


@pytest.mark.parametrize("quality", QUALITIES)
@pytest.mark.parametrize("kind", KINDS)
def test_restatement_equals_libjpeg(kind, quality):
    for H, W in SIZES:
        img = make_image(H, W, kind)
        ours, _ = assert_equals_libjpeg(img, quality)
        pillow_decode(ours, H, W)


@pytest.mark.parametrize("kind,quality", [("view", 90), ("noise", 100), ("checker", 1)])
def test_restatement_equals_libjpeg_800(kind, quality):
    img = make_image(800, 800, kind)
    ours, _ = assert_equals_libjpeg(img, quality)
    pillow_decode(ours, 800, 800)


def test_stuffing_and_large_categories_are_exercised():
    zz = J.coefficients(make_image(100, 100, "checker"), 100)
    assert np.abs(zz[:, :, 1:]).max() >= 512  # AC category 10
    assert np.abs(np.diff(zz[:, 0, 0])).max() >= 1  # DC differences present
    _, scan = segments(J.encode(make_image(100, 100, "noise"), 100))
    assert b"\xff\x00" in scan and scan.count(b"\xff") == scan.count(b"\xff\x00")


@pytest.mark.parametrize("kind", ["ramp", "view"])
def test_quality_90_psnr(kind):
    H, W = 100, 100
    img = make_image(H, W, kind)
    dec = pillow_decode(J.encode(img, 90), H, W)
    mse = np.mean((dec.astype(np.float64) - img) ** 2)
    assert 10 * np.log10(255 ** 2 / mse) >= 35


def test_stages():
    assert np.array_equal(J.ycc(np.array([[[255, 255, 255], [0, 0, 0], [255, 0, 0]]], np.uint8)),
                          [[[255, 128, 128], [0, 128, 128], [76, 85, 255]]])
    flat = J.fdct(np.full((8, 8), 100))
    assert flat[0, 0] == 100 * 64 and not flat.reshape(-1)[1:].any()  # scaled by 8: DC = 8 * mean * 8
    assert np.array_equal(J.quant_tables(50)[0], J.Q_LUMA) and (J.quant_tables(100) == 1).all()
    assert J.quant_tables(1).max() == 255
    assert np.array_equal(J.quantise(np.array([[12, -12, 11, -11]] * 16).reshape(8, 8), np.full(64, 3))[0, :4], [1, -1, 0, 0])
    with pytest.raises(ValueError):
        J.quant_tables(0)


# ---------------------------------------------------------------------------------------------------------------------
# AviWriter
# ---------------------------------------------------------------------------------------------------------------------
def riff_chunks(data, lo, hi):
    """[(tag, list type or None, payload offset, payload length)] of the chunks in data[lo:hi]"""
    out = []
    while lo < hi:
        tag, n = data[lo:lo + 4], struct.unpack_from("<I", data, lo + 4)[0]
        out.append((tag, data[lo + 8:lo + 12] if tag in (b"RIFF", b"LIST") else None, lo + 8, n))
        lo += 8 + n + (n & 1)
    assert lo == hi
    return out


def parse_avi(data):
    (tag, kind, p, n), = riff_chunks(data, 0, len(data))
    assert (tag, kind) == (b"RIFF", b"AVI ") and n == len(data) - 8
    top = riff_chunks(data, p + 4, p + n)
    assert [(t, k) for t, k, _, _ in top] == [(b"LIST", b"hdrl"), (b"LIST", b"movi"), (b"idx1", None)]
    hdrl = riff_chunks(data, top[0][2] + 4, top[0][2] + top[0][3])
    assert [(t, k) for t, k, _, _ in hdrl] == [(b"avih", None), (b"LIST", b"strl")]
    avih = struct.unpack_from("<14I", data, hdrl[0][2])
    strl = riff_chunks(data, hdrl[1][2] + 4, hdrl[1][2] + hdrl[1][3])
    assert [t for t, _, _, _ in strl] == [b"strh", b"strf"] and hdrl[0][3] == 56 and strl[0][3] == 56 and strl[1][3] == 40
    strh = struct.unpack_from("<4s4sIHHIIIIIIIIhhhh", data, strl[0][2])
    strf = struct.unpack_from("<IiiHH4sIiiII", data, strl[1][2])
    movi_tag = top[1][2]  # offset of 'movi'
    frames = riff_chunks(data, movi_tag + 4, movi_tag + top[1][3])
    assert all(t == b"00dc" for t, _, _, _ in frames)
    index = [struct.unpack_from("<4sIII", data, top[2][2] + 16 * i) for i in range(top[2][3] // 16)]
    return {"avih": avih, "strh": strh, "strf": strf, "movi_tag": movi_tag,
            "frames": [(p, n) for _, _, p, n in frames], "index": index}


def test_avi_writer(tmp_path):
    from ngp_pl_b200 import images
    H, W = 17, 33
    frames = []
    for q in range(60, 100):  # until both parities of length are present
        frames.append(J.encode(make_image(H, W, "view", seed=q), q))
        if len(frames) >= 4 and len({len(f) & 1 for f in frames}) == 2:
            break
    assert len({len(f) & 1 for f in frames}) == 2
    path = str(tmp_path / "v.avi")
    w = images.AviWriter(path, W, H, 30)
    for f in frames:
        w.add(f)
    w.close()
    w.close()  # idempotent
    data = open(path, "rb").read()
    a = parse_avi(data)
    largest = max(len(f) for f in frames)
    assert a["avih"][0] == 33333 and a["avih"][3] & 0x10 and a["avih"][4] == len(frames) and a["avih"][6] == 1
    assert a["avih"][7] == largest and a["avih"][8:10] == (W, H)
    assert a["strh"][:2] == (b"vids", b"MJPG") and a["strh"][6:8] == (1, 30) and a["strh"][9] == len(frames)
    assert a["strh"][10] == largest and a["strh"][-2:] == (W, H)
    assert a["strf"][:6] == (40, W, H, 1, 24, b"MJPG")
    assert len(a["frames"]) == len(a["index"]) == len(frames)
    for f, (p, n), (tag, flags, off, size) in zip(frames, a["frames"], a["index"]):
        assert data[p:p + n] == f and p % 2 == 0
        assert (tag, flags, size) == (b"00dc", 0x10, len(f)) and a["movi_tag"] + off + 8 == p
        if n & 1:
            assert data[p + n] == 0

    w = images.AviWriter(str(tmp_path / "ntsc.avi"), W, H, 30000 / 1001)
    w.close()
    a = parse_avi(open(str(tmp_path / "ntsc.avi"), "rb").read())
    assert a["strh"][6:8] == (1001, 30000) and a["frames"] == [] and a["avih"][4] == 0

    try:
        import cv2
    except ImportError:
        return
    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        return
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == len(frames) and cap.get(cv2.CAP_PROP_FPS) == 30
    assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (W, H)
    for f in frames:
        ok, bgr = cap.read()
        assert ok
        assert np.abs(bgr[..., ::-1].astype(np.int32) - pillow_decode(f, H, W)).mean() <= 2
    assert not cap.read()[0]


def test_avi_writer_refuses_to_pass_2_31(tmp_path):
    from ngp_pl_b200 import images

    class Huge:  # stands for a frame of n bytes without holding them
        def __init__(self, n):
            self.n = n

        def __len__(self):
            return self.n

    w = images.AviWriter(str(tmp_path / "big.avi"), 8, 8, 30)
    w.add(J.encode(make_image(8, 8, "ramp"), 90))
    with pytest.raises(RuntimeError, match="2\\^31"):
        w.add(Huge((1 << 31) - 300))
    w.close()
    assert len(parse_avi(open(str(tmp_path / "big.avi"), "rb").read())["frames"]) == 1
    with pytest.raises(RuntimeError):
        images.AviWriter(str(tmp_path / "x.avi"), 8, 8, 0)


def test_cpu_tensors_are_refused():
    import torch
    from ngp_pl_b200 import images
    img = torch.zeros(8, 8, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        images.encode_jpeg(img)
    with pytest.raises(RuntimeError, match="CUDA"):
        images.write_jpeg("unused.jpg", img)
    with pytest.raises(RuntimeError, match="CUDA"):
        images.render_video(lambda o, d: {}, torch.zeros(1, 3, 4), torch.zeros(64, 3), (8, 8), "unused")
