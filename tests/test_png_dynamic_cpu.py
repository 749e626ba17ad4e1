"""The dynamic PNG mode's host restatement, oracle/png_dynamic_ref.py: files that zlib, png_ref.decode and Pillow
read back to the image, package-merge code lengths against unrestricted Huffman and brute force, the block-header edge
cases, the capacity bound on noise, and the size on two 800x800 proxies of rendered views."""
import glob
import heapq
import io
import itertools
import os
import zlib

import numpy as np
import pytest

from oracle import images_ref as R
from oracle import png_dynamic_ref as D
from oracle import png_ref as P
from test_images_cpu import GOLDEN, ROOT, make_image

G = D.G
WIDE = 10922  # L = 32767: 2L and L + 3 exceed 32768, L - 3 and L do not
SIZES = [(1, 1), (1, 23), (19, 1), (G - 1, 7), (G, 7), (G + 1, 7), (2 * G + 5, 11), (64, 48), (3, WIDE)]


def _smooth(H, W):
    yy, xx = np.mgrid[0:H, 0:W]
    v = 127.5 + 60 * np.sin(xx / 7.0) * np.cos(yy / 11.0) + 40 * np.sin((xx + yy) / 23.0)
    return np.stack([v, v * 0.8, 255 - v], -1).astype(np.uint8)


def make(H, W, kind):
    return _smooth(H, W) if kind == "smooth" else make_image(H, W, kind)


def _pillow(data):
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        assert im.mode == "RGB"
        return np.array(im)


def _check(img):
    data, modes = D.encode(img, return_modes=True)
    H, W = img.shape[:2]
    assert len(data) <= P.capacity(H, W)
    assert np.array_equal(P.decode(data), img)  # chunk CRCs and the Adler-32 checked
    assert np.array_equal(_pillow(data), img)
    assert len(modes) == -(-H // G)
    return data, modes


def test_filtered_stream_equals_png_ref():
    for H, W in SIZES[:-1] + [(5, 300)]:
        for kind in ("noise", "flat", "gradient", "smooth"):
            img = make(H, W, kind)
            assert D.filtered_stream(img) == P.filtered_stream(img), (H, W, kind)


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("kind", ["noise", "flat", "gradient", "smooth"])
def test_round_trips(H, W, kind):
    _check(make(H, W, kind))


def test_round_trips_goldens_and_fixture_pngs():
    z = np.load(GOLDEN)
    imgs = [z[k] for k in z.files if k.startswith("img_")]
    from PIL import Image
    pngs = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "datasets", "lego", "*", "*.png")))[:3]
    pngs += sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "datasets", "*", "images*", "*.png")))[:3]
    assert len(pngs) == 6
    for p in pngs:
        with Image.open(p) as im:
            imgs.append(np.ascontiguousarray(np.array(im.convert("RGB"))))
    for img in imgs:
        _check(img)


def test_wide_rows_drop_far_candidates():
    L = 3 * WIDE + 1
    assert D.distances(L) == [1, 2, 3, 4, 6, 9, 12, L - 3, L]
    assert D.distances(4) == [1, 2, 3, 4, 6, 7, 8, 9, 12]  # L - 3 = 1 and L = 4 coincide with small candidates
    # rows 1 and 2 repeat row 0: matches at distance L cover them
    row = make_image(1, WIDE, "noise")
    data, modes = _check(np.concatenate([row] * 3))
    assert modes == [D.DYNAMIC] and len(data) < 3 * WIDE * 3 // 2


def _huffman_cost(counts):
    h = [c for c in counts if c]
    if len(h) < 2:
        return sum(h)
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        cost += a + b
        heapq.heappush(h, a + b)
    return cost


def _kraft(lens):
    return sum(2.0 ** -n for n in lens if n)


def _histograms():
    rng = np.random.RandomState(5)
    out = [[1, 1], [5, 0, 0, 7], [1] * 286, [2 ** 20] + [1] * 285, [0] * 200 + [3, 9]]
    out.append([int(x) for x in (2.0 ** np.arange(30)).astype(np.int64)])  # Fibonacci-like skew: needs the limit
    out.append([int(x) for x in np.round(1.618 ** np.arange(40)).astype(np.int64)])
    for n in (2, 3, 19, 30, 286):
        for scale in (3, 1000, 10 ** 7):
            c = rng.randint(0, scale, n).tolist()
            c[rng.randint(n)] += 1
            out.append(c)
        out.append(rng.geometric(0.2, n).tolist())
    return out


@pytest.mark.parametrize("limit", [7, 15])
def test_code_lengths_limit_kraft_and_optimality(limit):
    for c in _histograms():
        used = sum(1 for x in c if x)
        if used > 2 ** limit:
            continue
        lens = D.code_lengths(c, limit)
        assert max(lens) <= limit
        assert all((n > 0) == (x > 0) for n, x in zip(lens, c))
        if used >= 2:
            assert _kraft(lens) == 1.0
        cost = sum(n * x for n, x in zip(lens, c))
        free = D.code_lengths(c, 64)  # no limit in effect: package-merge is then plain Huffman
        assert sum(n * x for n, x in zip(free, c)) == _huffman_cost(c)
        if max(free) <= limit:
            assert cost == _huffman_cost(c)


def test_code_lengths_beat_brute_force_on_small_alphabets():
    rng = np.random.RandomState(9)
    for _ in range(60):
        n = rng.randint(2, 6)
        c = (rng.geometric(0.3, n) ** 3).tolist()
        limit = rng.randint(int(np.ceil(np.log2(n))), 5)
        lens = D.code_lengths(c, limit)
        best = min(sum(a * b for a, b in zip(ls, c)) for ls in itertools.product(range(1, limit + 1), repeat=n)
                   if _kraft(ls) <= 1)
        assert sum(a * b for a, b in zip(lens, c)) <= best
        assert max(lens) <= limit


def test_single_symbol_and_empty_alphabets():
    assert D.code_lengths([0, 0, 4, 0], 15) == [0, 0, 1, 0]
    assert D.code_lengths([0] * 30, 15) == [0] * 30


def _inflate(block):
    d = zlib.decompressobj(-15)
    return d.decompress(block) + d.flush()


def test_header_without_matches():
    """a group of literals only: no distance code used, distance code 0 gets length 1"""
    rng = np.random.RandomState(2)
    H, L = 4, 301
    s = bytes(rng.choice([0, 1, 2, 255], H * L, p=[0.7, 0.1, 0.1, 0.1]).astype(np.uint8))
    zeros = [0] * (H * L)
    block, mode = D.group_block(s, zeros, zeros, list(range(H)), L, True)
    assert mode == D.DYNAMIC
    assert _inflate(block) == s
    _, dd_len, _, _ = D.dynamic_header(np.bincount(np.frombuffer(s, np.uint8), minlength=286) + np.eye(286, dtype=int)[256],
                                       np.zeros(30, int))
    assert dd_len == [1] + [0] * 29


def test_header_with_one_distance_code():
    """runs of random bytes: every match is at distance 1, the one distance code gets length 1"""
    rng = np.random.RandomState(3)
    s = bytes(np.repeat(rng.randint(0, 256, 300), rng.randint(4, 20, 300)).astype(np.uint8))
    L = len(s)
    best, dist = D.match_table(s, 1, L)
    sym, _, _, dc, _, _ = D.group_tokens(s, best.tolist(), dist.tolist(), [0], L)
    assert set(dc[dc >= 0].tolist()) == {0}
    ll = np.bincount(sym, minlength=286)
    ll[256] += 1
    _, dd_len, _, _ = D.dynamic_header(ll, np.bincount(dc[dc >= 0], minlength=30))
    assert dd_len == [1] + [0] * 29
    block, mode = D.group_block(s, best.tolist(), dist.tolist(), [0], L, True)
    assert mode == D.DYNAMIC
    assert _inflate(block) == s


def test_fixed_wins_on_a_tiny_group_and_noise_is_stored():
    _, modes = _check(make_image(1, 1, "gradient"))
    assert modes == [D.FIXED]
    H, W = 2 * G + 5, 48
    data, modes = _check(make_image(H, W, "noise"))
    assert modes == [D.STORED] * 3
    assert len(data) <= P.capacity(H, W)
    assert len(data) < len(P.encode(make_image(H, W, "noise")))  # a group stored whole: fewer block headers


@pytest.fixture(scope="module")
def proxies():
    """the 80x80 Lego golden view and its depth image, upscaled to 800x800 (not trained renders)"""
    from PIL import Image
    z = np.load(GOLDEN)
    rgb = np.asarray(Image.fromarray(z["img_lego"]).resize((800, 800), Image.BILINEAR))
    d = np.asarray(Image.fromarray(z["depth_lego"]).resize((800, 800), Image.BILINEAR))
    return {"rgb": np.ascontiguousarray(rgb), "depth": np.ascontiguousarray(R.depth_image(d.ravel(), 800, 800))}


@pytest.mark.parametrize("name", ["rgb", "depth"])
def test_proxy_sizes(proxies, name):
    img = proxies[name]
    data, modes = _check(img)
    fixed = len(P.encode(img))
    assert len(data) <= 0.6 * fixed, (len(data), fixed)
    assert set(modes) == {D.DYNAMIC}
