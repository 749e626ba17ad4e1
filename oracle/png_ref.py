"""Host restatement of the device PNG encoder (ngp_png_encode, include/ngp_b200.h) and an independent decoder -- TEST
INFRASTRUCTURE ONLY.

encode(img)       the encoder's byte stream, byte for byte, for an (H, W, 3) uint8 image: libpng's filter heuristic per
                  row, one deflate segment per filtered row (greedy parse over distances 1, 3, L, 2L, one fixed-Huffman
                  block or stored blocks, then an empty stored block), zlib header 78 01 and Adler-32, CRC-32 per chunk.
                  Plain Python loops: meant for small images.
capacity(H, W)    ngp_png_capacity's formula
filter_row(...)   the filter choice of one row (type, filtered bytes)
decode(data)      chunk parse with zlib.crc32 per chunk, zlib.decompress (which checks the Adler-32) and the five
                  unfilters -> (H, W, 3) uint8; written from the PNG specification, sharing no code with encode
"""
import struct
import zlib

import numpy as np

STORED_MAX = 65535
MAX_DIST = 32768


def stored_len(L):
    return L + 5 * (-(-L // STORED_MAX)) + 5


def capacity(H, W):
    return 63 + H * stored_len(3 * W + 1)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)


def filter_row(x, up):
    """x, up: the row and the row above (zeros for row 0), sequences of 3W ints -> (type, filtered bytes)"""
    n = len(x)
    cands = []
    for f in range(5):
        out = []
        for j in range(n):
            a = x[j - 3] if j >= 3 else 0
            b = up[j]
            c = up[j - 3] if j >= 3 else 0
            pred = (0, a, b, (a + b) >> 1, _paeth(a, b, c))[f]
            out.append((x[j] - pred) & 0xff)
        cands.append((sum(v if v < 128 else 256 - v for v in out), f, out))
    s, f, out = min(cands, key=lambda c: (c[0], c[1]))  # ties: the lowest type
    return f, out


class _Bits:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def put(self, v, nb):  # LSB first
        self.acc |= v << self.n
        self.n += nb
        while self.n >= 8:
            self.out.append(self.acc & 0xff)
            self.acc >>= 8
            self.n -= 8

    def huff(self, code, nb):  # Huffman codes go MSB first
        self.put(int(format(code, "0%db" % nb)[::-1], 2), nb)

    def flush(self):
        if self.n:
            self.out.append(self.acc & 0xff)
        self.acc, self.n = 0, 0


def _length_code(n):
    if n == 258:
        return 285, 0, 0
    v = n - 3
    if v < 8:
        return 257 + v, 0, 0
    e = v.bit_length() - 1 - 2
    return 261 + 4 * e + ((v >> e) & 3), e, v & ((1 << e) - 1)


def _dist_code(d):
    v = d - 1
    if v < 4:
        return v, 0, 0
    e = v.bit_length() - 1 - 1
    return 2 * e + 2 + ((v >> e) & 1), e, v & ((1 << e) - 1)


def parse(s, p0, L):
    """greedy tokens of the segment s[p0:p0+L]: ('lit', byte) or ('match', length, distance)"""
    toks, j = [], 0
    while j < L:
        p = p0 + j
        best, best_d = 0, 0
        for d in (1, 3, L, 2 * L):
            if d > MAX_DIST or p < d:
                continue
            m = 0
            while m < 258 and j + m < L and s[p + m] == s[p - d + m]:
                m += 1
            if m > best:
                best, best_d = m, d
        if best >= 3:
            toks.append(("match", best, best_d))
            j += best
        else:
            toks.append(("lit", s[p]))
            j += 1
    return toks


def segment(s, p0, L, last):
    """the deflate bytes of one segment"""
    b = _Bits()
    b.put(0, 1)
    b.put(1, 2)  # BTYPE 01
    for t in parse(s, p0, L):
        if t[0] == "lit":
            v = t[1]
            if v < 144:
                b.huff(0x30 + v, 8)
            else:
                b.huff(0x190 + v - 144, 9)
        else:
            sym, e, x = _length_code(t[1])
            if sym < 280:
                b.huff(sym - 256, 7)
            else:
                b.huff(0xC0 + sym - 280, 8)
            b.put(x, e)
            dc, de, dx = _dist_code(t[2])
            b.huff(dc, 5)
            b.put(dx, de)
    b.huff(0, 7)  # end of block
    b.put(int(last), 1)
    b.put(0, 2)  # empty stored block
    b.flush()
    fixed = bytes(b.out) + b"\x00\x00\xff\xff"
    if stored_len(L) <= len(fixed):
        out = bytearray()
        data = bytes(s[p0:p0 + L])
        for i in range(0, L, STORED_MAX):
            chunk = data[i:i + STORED_MAX]
            out += bytes([0]) + struct.pack("<HH", len(chunk), 0xffff ^ len(chunk)) + chunk
        out += bytes([int(last), 0, 0, 0xff, 0xff])
        return bytes(out)
    return fixed


def _chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data))


def filtered_stream(img):
    img = np.asarray(img, np.uint8)
    H, W, _ = img.shape
    s, prev = bytearray(), [0] * (3 * W)
    for r in range(H):
        x = img[r].reshape(-1).tolist()
        f, out = filter_row(x, prev)
        s.append(f)
        s += bytes(out)
        prev = x
    return bytes(s)


def encode(img):
    img = np.asarray(img, np.uint8)
    H, W, C = img.shape
    assert C == 3
    L = 3 * W + 1
    s = filtered_stream(img)
    z = b"\x78\x01" + b"".join(segment(s, r * L, L, r == H - 1) for r in range(H)) + struct.pack(">I", zlib.adler32(s))
    ihdr = struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)
    return b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", z) + _chunk(b"IEND", b"")


def decode(data, check_crc=True):
    """-> (H, W, 3) uint8; raises ValueError on a bad signature, chunk CRC or layout"""
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("not a PNG signature")
    pos, idat, hdr, end = 8, bytearray(), None, False
    while pos < len(data):
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        (crc,) = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        if check_crc and crc != zlib.crc32(kind + body):
            raise ValueError("bad CRC in chunk %r" % kind)
        if kind == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"IDAT":
            idat += body
        elif kind == b"IEND":
            end = True
            pos += 12 + n
            break
        pos += 12 + n
    if hdr is None or not end or pos != len(data):
        raise ValueError("missing IHDR / IEND or trailing bytes")
    W, H, depth, ctype, comp, filt, interlace = hdr
    if (depth, ctype, comp, filt, interlace) != (8, 2, 0, 0, 0):
        raise ValueError("not an 8-bit RGB non-interlaced PNG: %s" % (hdr,))
    raw = zlib.decompress(bytes(idat))  # checks the Adler-32
    L = 3 * W + 1
    if len(raw) != H * L:
        raise ValueError("decompressed %d bytes, expected %d" % (len(raw), H * L))
    out = np.zeros((H, 3 * W), np.uint8)
    prev = [0] * (3 * W)
    for r in range(H):
        f = raw[r * L]
        row = np.frombuffer(raw, np.uint8, 3 * W, r * L + 1)
        if f == 0:
            cur = row.tolist()
        elif f == 1:  # Sub: a running sum per channel
            cur = (np.cumsum(row.reshape(W, 3).astype(np.int64), 0) & 0xff).reshape(-1).tolist()
        elif f == 2:
            cur = ((row.astype(np.int64) + np.array(prev)) & 0xff).tolist()
        elif f in (3, 4):
            x, cur = row.tolist(), [0] * (3 * W)
            for j in range(3 * W):
                a = cur[j - 3] if j >= 3 else 0
                b = prev[j]
                if f == 3:
                    pred = (a + b) >> 1
                else:
                    c = prev[j - 3] if j >= 3 else 0
                    pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                    pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
                cur[j] = (x[j] + pred) & 0xff
        else:
            raise ValueError("filter type %d" % f)
        out[r] = cur
        prev = cur
    return out.reshape(H, W, 3)
