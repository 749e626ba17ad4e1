"""Host restatement of the device PNG encoder's dynamic mode (ngp_png_encode_mode(..., NGP_PNG_DYNAMIC),
include/ngp_b200.h) -- TEST INFRASTRUCTURE ONLY.

encode(img)            the mode's byte stream, byte for byte, for an (H, W, 3) uint8 image: png_ref's filters, a lazy
                       parse per row over eleven candidate distances, one block per group of G rows coded with dynamic
                       Huffman, fixed Huffman or stored blocks (the shortest), then an empty stored block per group
filtered_stream(img)   png_ref.filtered_stream, vectorised (the same bytes; tests hold the two equal)
distances(L)           the candidate distances of a row of L bytes, ascending and distinct
code_lengths(c, limit) length-limited Huffman code lengths by package-merge
group_block(...)       the bytes of one group and the coding chosen for it
Matching and bit packing are numpy; the parse walk is a plain loop over each row's tokens.
"""
import struct
import zlib

import numpy as np

from oracle import png_ref

G = 32
MAX_DIST = 32768
MAX_MATCH = 258
STORED_MAX = 65535
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
DYNAMIC, FIXED, STORED = 0, 1, 2


def distances(L):
    return sorted({d for d in (1, 2, 3, 4, 6, 9, 12, L - 3, L, L + 3, 2 * L) if 1 <= d <= MAX_DIST})


def filtered_stream(img):
    """(H, W, 3) uint8 -> the filtered stream, H segments of [type, 3W filtered bytes], as png_ref.filter_row picks"""
    img = np.asarray(img, np.uint8)
    H, W, _ = img.shape
    x = img.reshape(H, 3 * W).astype(np.int32)
    up = np.vstack([np.zeros((1, 3 * W), np.int32), x[:-1]])
    a = np.hstack([np.zeros((H, 3), np.int32), x[:, :-3]])[:, :3 * W]
    c = np.hstack([np.zeros((H, 3), np.int32), up[:, :-3]])[:, :3 * W]
    p = a + up - c
    pa, pb, pc = np.abs(p - a), np.abs(p - up), np.abs(p - c)
    paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, up, c))
    cand = np.stack([x, x - a, x - up, x - ((a + up) >> 1), x - paeth]) & 0xff  # (5, H, 3W)
    cost = np.where(cand < 128, cand, 256 - cand).sum(-1)  # (5, H)
    f = np.argmin(cost, 0)  # ties: the lowest type
    rows = cand[f, np.arange(H)]
    return np.hstack([f[:, None], rows]).astype(np.uint8).reshape(-1).tobytes()


def match_table(s, H, L):
    """(best length, best distance) per stream position: lengths < 3 are 0"""
    s = np.frombuffer(s, np.uint8)
    N = H * L
    ds = distances(L)
    col = np.arange(L)
    runs = np.zeros((len(ds), N), np.int32)
    for k, d in enumerate(ds):
        eq = np.zeros(N, bool)
        if d < N:
            eq[d:] = s[d:] == s[:-d]
        nxt = np.where(eq.reshape(H, L), L, col[None, :])
        nxt = np.minimum.accumulate(nxt[:, ::-1], 1)[:, ::-1]  # the first mismatch at or after j, or the row's end
        runs[k] = np.minimum(nxt - col[None, :], MAX_MATCH).reshape(-1)
    k = np.argmax(runs, 0)  # a tie goes to the smaller distance
    best = runs[k, np.arange(N)]
    dist = np.asarray(ds)[k]
    keep = best >= 3
    return np.where(keep, best, 0), np.where(keep, dist, 0)


def parse_row(best, j0, L):
    """token start positions and lengths (1 = a literal) of the row at j0: lazy matching by one step"""
    b = best[j0:j0 + L]
    b1 = b[1:] + [0]
    starts, j = [], 0
    while j < L:
        m = b[j]
        starts.append(j)
        j += m if (m and not b1[j] > m) else 1
    return starts


def _length_codes():
    sym, ext, val = np.zeros(259, np.int64), np.zeros(259, np.int64), np.zeros(259, np.int64)
    for n in range(3, 259):
        sym[n], ext[n], val[n] = png_ref._length_code(n)
    return sym, ext, val


LEN_SYM, LEN_EXT, LEN_VAL = _length_codes()
LL_EXTRA = np.zeros(286, np.int64)
LL_EXTRA[257:285] = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4
DIST_EXTRA = np.array([0, 0, 0, 0] + [e for e in range(1, 14) for _ in (0, 1)], np.int64)


def _dist_codes(d):
    v = np.asarray(d, np.int64) - 1
    e = np.maximum(np.frexp(np.maximum(v, 1))[1].astype(np.int64) - 2, 0)  # bit_length(v) - 2
    code = np.where(v < 4, v, 2 * e + 2 + ((v >> e) & 1))
    ext = np.where(v < 4, 0, e)
    return code, ext, v & ((1 << ext) - 1)


def code_lengths(counts, limit):
    """package-merge: optimal code lengths <= limit for the symbols with a non-zero count; items sorted by (count,
    symbol), an item before a package of equal weight; one used symbol gets length 1"""
    counts = [int(c) for c in counts]
    lens = [0] * len(counts)
    items = sorted((c, i) for i, c in enumerate(counts) if c)
    n = len(items)
    if n == 0:
        return lens
    if n == 1:
        lens[items[0][1]] = 1
        return lens
    w = [c for c, _ in items]
    cur, flags = list(w), [[True] * n]
    for _ in range(limit - 1):
        pk = [cur[2 * k] + cur[2 * k + 1] for k in range(len(cur) // 2)]
        merged, f, i, j = [], [], 0, 0
        while i < n or j < len(pk):
            if j == len(pk) or (i < n and w[i] <= pk[j]):
                merged.append(w[i])
                f.append(True)
                i += 1
            else:
                merged.append(pk[j])
                f.append(False)
                j += 1
        cur = merged
        flags.append(f)
    k = 2 * n - 2
    for f in reversed(flags):
        ni = sum(f[:k])
        for r in range(ni):
            lens[items[r][1]] += 1
        k = 2 * (k - ni)
    return lens


def canonical(lens):
    """RFC 1951 3.2.2 codes, bit-reversed for LSB-first output"""
    mx = max(lens) if lens else 0
    bl = [0] * (mx + 2)
    for n in lens:
        if n:
            bl[n] += 1
    nxt, code = [0] * (mx + 2), 0
    for b in range(1, mx + 1):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = [0] * len(lens)
    for i, n in enumerate(lens):
        if n:
            out[i] = int(format(nxt[n], "0%db" % n)[::-1], 2)
            nxt[n] += 1
    return out


def rle(lens):
    """zlib's send_tree over one alphabet's lengths: (code-length symbol, extra value, extra bits)"""
    out = []
    n_max = len(lens)
    prev, nextlen, count = -1, lens[0], 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(n_max):
        cur = nextlen
        nextlen = lens[n + 1] if n + 1 < n_max else 0xffff
        count += 1
        if count < max_count and cur == nextlen:
            continue
        if count < min_count:
            out += [(cur, 0, 0)] * count
        elif cur != 0:
            if cur != prev:
                out.append((cur, 0, 0))
                count -= 1
            out.append((16, count - 3, 2))
        elif count <= 10:
            out.append((17, count - 3, 3))
        else:
            out.append((18, count - 11, 7))
        count, prev = 0, cur
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif cur == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


FIXED_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8  # RFC 1951 3.2.6: 288 symbols, 286 and 287 unused
FIXED_DD = [5] * 30


def _pack(vals, nbits):
    """LSB-first bit string of the fields (value, nbits) in order -> (bytes, total bits)"""
    vals, nbits = np.asarray(vals, np.int64), np.asarray(nbits, np.int64)
    keep = nbits > 0
    vals, nbits = vals[keep], nbits[keep]
    total = int(nbits.sum())
    start = np.cumsum(nbits) - nbits
    idx = np.repeat(np.arange(len(nbits)), nbits)
    pos = np.arange(total) - start[idx]
    bits = ((vals[idx] >> pos) & 1).astype(np.uint8)
    return np.packbits(bits, bitorder="little").tobytes(), total


def dynamic_header(ll, dd):
    """the code of one group's histograms: (ll lengths, dd lengths, header fields [(value, nbits)], header bits)"""
    ll_len = code_lengths(ll, 15)
    dd_len = code_lengths(dd, 15)
    if not any(dd_len):
        dd_len[0] = 1
    nlit = max(257, 1 + max(i for i, n in enumerate(ll_len) if n))
    ndist = max(1, 1 + max(i for i, n in enumerate(dd_len) if n))
    seq = rle(ll_len[:nlit]) + rle(dd_len[:ndist])
    cl = [0] * 19
    for sym, _, _ in seq:
        cl[sym] += 1
    cl_len = code_lengths(cl, 7)
    cl_code = canonical(cl_len)
    ncl = 19
    while ncl > 4 and cl_len[CL_ORDER[ncl - 1]] == 0:
        ncl -= 1
    fields = [(0, 1), (2, 2), (nlit - 257, 5), (ndist - 1, 5), (ncl - 4, 4)]
    fields += [(cl_len[CL_ORDER[i]], 3) for i in range(ncl)]
    for sym, v, e in seq:
        fields += [(cl_code[sym], cl_len[sym]), (v, e)]
    return ll_len, dd_len, fields, sum(nb for _, nb in fields)


def group_tokens(s, best, dist, rows, L):
    """the tokens of rows as arrays: ll symbol, length extra (value, bits), distance code, distance extra"""
    sym, lv, lb, dc, dv, db = [], [], [], [], [], []
    for r in rows:
        j0 = r * L
        st = np.asarray(parse_row(best, j0, L), np.int64)
        m = np.asarray([best[j0 + j] for j in st.tolist()], np.int64)
        nxt = np.append(st[1:], L)
        is_m = (nxt - st) > 1
        p = j0 + st
        lit = np.frombuffer(s, np.uint8)[p].astype(np.int64)
        mm = np.where(is_m, m, 3)
        sym.append(np.where(is_m, LEN_SYM[mm], lit))
        lv.append(np.where(is_m, LEN_VAL[mm], 0))
        lb.append(np.where(is_m, LEN_EXT[mm], 0))
        dcode, dext, dval = _dist_codes(np.where(is_m, np.asarray([dist[q] for q in p.tolist()], np.int64), 1))
        dc.append(np.where(is_m, dcode, -1))
        dv.append(np.where(is_m, dval, 0))
        db.append(np.where(is_m, dext, 0))
    return [np.concatenate(a) for a in (sym, lv, lb, dc, dv, db)]


def group_block(s, best, dist, rows, L, last):
    """the bytes of one group (its block and the empty stored block after it) and the coding chosen"""
    sym, lv, lb, dc, dv, db = group_tokens(s, best, dist, rows, L)
    ll = np.bincount(sym, minlength=286)
    ll[256] += 1
    dd = np.bincount(dc[dc >= 0], minlength=30)
    extra = int(lb.sum() + db.sum())
    ll_len, dd_len, head, head_bits = dynamic_header(ll, dd)
    dyn_bits = head_bits + int(np.dot(ll, ll_len) + np.dot(dd, dd_len)) + extra
    fix_bits = 3 + int(np.dot(ll, FIXED_LL[:286]) + np.dot(dd, FIXED_DD)) + extra
    n = len(rows) * L
    sizes = [(dyn_bits + 3 + 7) // 8 + 4, (fix_bits + 3 + 7) // 8 + 4, n + 5 * (-(-n // STORED_MAX)) + 5]
    mode = min(range(3), key=lambda k: (sizes[k], k))
    if mode == STORED:
        data = s[rows[0] * L:rows[0] * L + n]
        out = bytearray()
        for i in range(0, n, STORED_MAX):
            chunk = data[i:i + STORED_MAX]
            out += bytes([0]) + struct.pack("<HH", len(chunk), 0xffff ^ len(chunk)) + chunk
        out += bytes([int(last), 0, 0, 0xff, 0xff])
        return bytes(out), mode
    if mode == FIXED:
        ll_len, dd_len, head = FIXED_LL, FIXED_DD, [(0, 1), (1, 2)]
    ll_code, dd_code = np.asarray(canonical(ll_len), np.int64), np.asarray(canonical(dd_len), np.int64)
    ll_len, dd_len = np.asarray(ll_len, np.int64), np.asarray(dd_len, np.int64)
    is_m = dc >= 0
    dci = np.where(is_m, dc, 0)
    tv = np.stack([ll_code[sym], lv, np.where(is_m, dd_code[dci], 0), dv], 1).reshape(-1)
    tb = np.stack([ll_len[sym], lb, np.where(is_m, dd_len[dci], 0), db], 1).reshape(-1)
    hv, hb = zip(*head)
    vals = np.concatenate([hv, tv, [ll_code[256], int(last), 0]])
    nbits = np.concatenate([hb, tb, [ll_len[256], 1, 2]])
    data, total = _pack(vals, nbits)
    assert total == (dyn_bits if mode == DYNAMIC else fix_bits) + 3
    out = data + b"\x00\x00\xff\xff"
    assert len(out) == sizes[mode]
    return out, mode


def deflate(s, H, L):
    """the deflate stream of the filtered stream s and each group's coding"""
    best, dist = match_table(s, H, L)
    best, dist = best.tolist(), dist.tolist()
    parts, modes = [], []
    for g0 in range(0, H, G):
        rows = list(range(g0, min(g0 + G, H)))
        data, mode = group_block(s, best, dist, rows, L, rows[-1] == H - 1)
        parts.append(data)
        modes.append(mode)
    return b"".join(parts), modes


def encode(img, return_modes=False):
    img = np.asarray(img, np.uint8)
    H, W, C = img.shape
    assert C == 3
    L = 3 * W + 1
    s = filtered_stream(img)
    body, modes = deflate(s, H, L)
    z = b"\x78\x01" + body + struct.pack(">I", zlib.adler32(s))
    ihdr = struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)
    png = b"\x89PNG\r\n\x1a\n" + png_ref._chunk(b"IHDR", ihdr) + png_ref._chunk(b"IDAT", z) + png_ref._chunk(b"IEND", b"")
    return (png, modes) if return_modes else png
