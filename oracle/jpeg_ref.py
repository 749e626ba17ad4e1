"""Host restatement of ngp_jpeg_encode (csrc/jpeg.cu), byte for byte, in integer numpy: the stream include/ngp_b200.h
specifies, one function per stage. tests/test_jpeg_cpu.py pins it to libjpeg (through Pillow, quality=q, subsampling=0,
optimize=False): DQT, SOF0 and the entropy-coded bytes are equal; tests/test_jpeg_gpu.py holds the device encoder to it.

    ycc(img)                (H, W, 3) uint8 RGB -> (H, W, 3) int32 Y, Cb, Cr (16-bit fixed point, libjpeg's rounding)
    blocks(ycc)             edge-replicated to multiples of 8, level-shifted: (n_mcu, 3, 8, 8) int32, MCU raster order
    fdct(b)                 the accurate integer forward DCT ("islow"): (..., 8, 8) -> (..., 8, 8), scaled by 8
    quant_tables(quality)   the two Annex K tables scaled by libjpeg's rule: (2, 64) int32, natural order
    quantise(c, q)          round-half-away division by 8 q
    scan_bits(zz)           (n_mcu, 3, 64) zig-zagged coefficients -> per slot (value, length) of its codes
    encode(img, quality)    the whole file
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                   14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39,
                   46, 53, 60, 61, 54, 47, 55, 62, 63])

Q_LUMA = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51,
          87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101,
          72, 92, 95, 98, 112, 100, 103, 99]
Q_CHROMA = [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
            99, 99, 99, 99] + [99] * 32

# Annex K.3: (number of codes of each length 1..16, the symbols in code order)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
    0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
    0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
    0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
    0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
    0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
    0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])


def huffman_codes(bits, vals):
    """canonical codes of a (bits, vals) table (Annex C): code[symbol], length[symbol] as (256,) int64, length 0 = absent"""
    code = np.zeros(256, np.int64)
    length = np.zeros(256, np.int64)
    c, k = 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            code[vals[k]], length[vals[k]] = c, n
            c, k = c + 1, k + 1
        c <<= 1
    return code, length


def ycc(img):
    r, g, b = (img[..., i].astype(np.int64) for i in range(3))
    half = 1 << 15
    off = (128 << 16) + half - 1
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + off) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + off) >> 16
    return np.stack([y, cb, cr], -1).astype(np.int32)


def blocks(c):
    H, W = c.shape[:2]
    c = np.pad(c, ((0, -H % 8), (0, -W % 8), (0, 0)), mode="edge") - 128
    h, w = c.shape[0] // 8, c.shape[1] // 8
    return c.reshape(h, 8, w, 8, 3).transpose(0, 2, 4, 1, 3).reshape(h * w, 3, 8, 8)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _pass(d, first):
    """one 1-D pass of the Loeffler-Ligtenberg-Moschytz DCT along the last axis; 13-bit constants, 2-bit pass-1 scale"""
    d = [d[..., i] for i in range(8)]
    t0, t7, t1, t6 = d[0] + d[7], d[0] - d[7], d[1] + d[6], d[1] - d[6]
    t2, t5, t3, t4 = d[2] + d[5], d[2] - d[5], d[3] + d[4], d[3] - d[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    n = 13 - 2 if first else 13 + 2
    o = [None] * 8
    o[0] = (t10 + t11) << 2 if first else _descale(t10 + t11, 2)
    o[4] = (t10 - t11) << 2 if first else _descale(t10 - t11, 2)
    z1 = (t12 + t13) * 4433
    o[2] = _descale(z1 + t13 * 6270, n)
    o[6] = _descale(z1 - t12 * 15137, n)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * 9633
    t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
    z1, z2 = z1 * -7373, z2 * -20995
    z3, z4 = z3 * -16069 + z5, z4 * -3196 + z5
    o[7] = _descale(t4 + z1 + z3, n)
    o[5] = _descale(t5 + z2 + z4, n)
    o[3] = _descale(t6 + z2 + z3, n)
    o[1] = _descale(t7 + z1 + z4, n)
    return np.stack(o, -1)


def fdct(b):
    rows = _pass(b.astype(np.int64), True)
    return np.swapaxes(_pass(np.swapaxes(rows, -1, -2), False), -1, -2)


def quant_tables(quality):
    if not 1 <= quality <= 100:
        raise ValueError("quality must be 1..100")
    s = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((np.array([Q_LUMA, Q_CHROMA], np.int64) * s + 50) // 100, 1, 255).astype(np.int32)


def quantise(c, q):
    q8 = q.astype(np.int64).reshape(8, 8) * 8
    return (np.sign(c) * ((np.abs(c) + (q8 >> 1)) // q8)).astype(np.int32)


def coefficients(img, quality):
    """(n_mcu, 3, 64) int32: the quantised coefficients of every block, zig-zagged"""
    q = quant_tables(quality)
    c = fdct(blocks(ycc(img)))
    out = np.stack([quantise(c[:, k], q[min(k, 1)]) for k in range(3)], 1)
    return out.reshape(len(out), 3, 64)[:, :, ZIGZAG]


def _category(v):
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    for k in range(12):
        n += a >> k > 0
    return n


def scan_bits(zz):
    """Per coefficient slot of the interleaved scan, its codes as one (value, length <= 60) pair, both (n_mcu, 3, 64)
    int64: slot 0 the DC difference (to the same component of the previous MCU), a non-zero AC slot its ZRLs, run/size
    code and magnitude bits, slot 63 the EOB when the last coefficient is zero; every other slot is empty."""
    zz = zz.astype(np.int64)
    n = len(zz)
    val = np.zeros(zz.shape, np.int64)
    length = np.zeros(zz.shape, np.int64)
    diff = zz[:, :, 0] - np.concatenate([np.zeros((1, 3), np.int64), zz[:-1, :, 0]])
    k = np.arange(64)
    # index of the previous non-zero coefficient (0 = the DC slot) for every AC slot
    nz = np.where(zz != 0, k, 0)
    nz[:, :, 0] = 0
    prev = np.maximum.accumulate(nz, axis=2)
    prev = np.concatenate([np.zeros((n, 3, 1), np.int64), prev[:, :, :-1]], 2)
    run = k - prev - 1
    for comp in range(3):
        dc_code, dc_len = huffman_codes(*(DC_LUMA if comp == 0 else DC_CHROMA))
        ac_code, ac_len = huffman_codes(*(AC_LUMA if comp == 0 else AC_CHROMA))
        d = diff[:, comp]
        cat = _category(d)
        extra = np.where(d < 0, d - 1, d) & ((1 << cat) - 1)
        val[:, comp, 0] = (dc_code[cat] << cat) | extra
        length[:, comp, 0] = dc_len[cat] + cat
        v = zz[:, comp, 1:]
        r = run[:, comp, 1:]
        cat = _category(v)
        assert cat.max(initial=0) <= 10 and _category(d).max(initial=0) <= 11
        extra = np.where(v < 0, v - 1, v) & ((1 << cat) - 1)
        sym = ((r & 15) << 4) | cat
        a_val = (ac_code[sym] << cat) | extra
        a_len = ac_len[sym] + cat
        zrl = r >> 4
        for j in (1, 2, 3):  # ZRLs in front
            m = zrl >= j
            a_val = np.where(m, a_val | (ac_code[0xF0] << a_len), a_val)
            a_len = np.where(m, a_len + ac_len[0xF0], a_len)
        live = v != 0
        val[:, comp, 1:] = np.where(live, a_val, 0)
        length[:, comp, 1:] = np.where(live, a_len, 0)
        eob = zz[:, comp, 63] == 0
        val[:, comp, 63] = np.where(eob, ac_code[0], val[:, comp, 63])
        length[:, comp, 63] = np.where(eob, ac_len[0], length[:, comp, 63])
    return val, length


def pack(val, length):
    """the slots' codes MSB first, the last byte padded with 1-bits, 0xFF followed by 0x00"""
    val, length = val.reshape(-1), length.reshape(-1)
    keep = length > 0
    val, length = val[keep], length[keep]
    total = int(length.sum())
    start = np.cumsum(length) - length
    owner = np.repeat(np.arange(len(val)), length)
    j = np.arange(total) - start[owner]
    bits = ((val[owner] >> (length[owner] - 1 - j)) & 1).astype(np.uint8)
    bits = np.concatenate([bits, np.ones(-total % 8, np.uint8)])
    data = np.packbits(bits)
    ff = np.flatnonzero(data == 0xFF)
    return np.insert(data, ff + 1, 0).tobytes()


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def headers(H, W, quality):
    """SOI, JFIF APP0 (1.01, no density unit, 1 x 1), DQT 0, DQT 1, SOF0, DHT DC0, AC0, DC1, AC1, SOS: 623 bytes"""
    q = quant_tables(quality)
    out = b"\xff\xd8" + _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in range(2):
        out += _segment(0xDB, bytes([t]) + bytes(q[t][ZIGZAG].astype(np.uint8)))
    out += _segment(0xC0, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") +
                    bytes([3, 1, 0x11, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for tc_th, (bits, vals) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        out += _segment(0xC4, bytes([tc_th]) + bytes(bits) + bytes(vals))
    return out + _segment(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


def encode(img, quality=90):
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
    H, W = int(img.shape[0]), int(img.shape[1])
    return headers(H, W, quality) + pack(*scan_bits(coefficients(img, quality))) + b"\xff\xd9"
