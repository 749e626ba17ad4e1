// Test-view images of the validation pass (reference train.py:215-221, depth2img at train.py:45-50): the quantised RGB
// and turbo depth images, and a PNG encoder, on the device. The layouts, the exact arithmetic and the byte stream are
// specified in include/ngp_b200.h; oracle/images_ref.py and oracle/png_ref.py restate them on the host.
//
// PNG: the filtered image is one byte stream of H segments of L = 3W + 1 bytes (filter type + filtered row). Each
// segment is deflated on its own by one warp -- a greedy parse over four candidate distances, coded as one fixed-Huffman
// block or stored -- and ends with an empty stored block, so every segment starts on a byte boundary and the segments
// concatenate into one deflate stream. The Adler-32 and the IDAT CRC-32 are combined from per-segment values.
// The opt-in dynamic mode (ngp_png_encode_mode) keeps the filters and the assembly but deflates one block per group of
// 32 rows, with Huffman tables built on the device from the group's histograms (oracle/png_dynamic_ref.py restates it).
#include "common.cuh"
#include "ngp_b200.h"
#include "turbo_table.cuh"

#include <algorithm>

namespace {

constexpr int VI_THREADS = 256;
constexpr int VI_PARTIALS = 256;  // min/max blocks; NGP_VIEW_IMAGES_WORKSPACE = 16 bytes each
constexpr uint32_t ADLER_MOD = 65521u;
constexpr uint32_t CRC_POLY = 0xedb88320u;
constexpr int PNG_WARPS = 4;            // rows per block of the filter and deflate kernels
constexpr int PNG_HEAD = 8 + 25 + 8;    // signature, IHDR chunk, IDAT length + type
constexpr int PNG_TAIL = 4 + 4 + 12;    // Adler-32, IDAT CRC, IEND chunk
constexpr int64_t STORED_MAX = 65535;   // bytes of one stored block
constexpr int64_t MAX_DIST = 32768;
constexpr int MAX_MATCH = 258;

// x^(2^k) mod P for the CRC-32 polynomial P, reflected (bit 31 = x^0); period 32 in k (zlib's x2n_table)
__constant__ uint32_t X2N[32] = {
    0x40000000, 0x20000000, 0x08000000, 0x00800000, 0x00008000, 0xedb88320, 0xb1e6b092, 0xa06a2517,
    0xed627dae, 0x88d14467, 0xd7bbfe6a, 0xec447f11, 0x8e7ea170, 0x6427800e, 0x4d47bae0, 0x09fe548f,
    0x83852d0f, 0x30362f1a, 0x7b5a9cc3, 0x31fec169, 0x9fec022a, 0x6c8dedc4, 0x15d6874d, 0x5fde7a4e,
    0xbad90e37, 0x2e4e5eef, 0x4eaba214, 0xa8a472c0, 0x429a969e, 0x148d302a, 0xc40ba6d0, 0xc4e22c3c};

struct PngRow {
    uint32_t len;   // segment bytes
    uint32_t crc;   // CRC-32 of the segment
    uint32_t a, b;  // sum d_i, sum (L - i) d_i over the segment's uncompressed bytes, mod 65521
};

// ---------------------------------------------------------------------------------------------------------------------
// View images
// ---------------------------------------------------------------------------------------------------------------------
struct MinMax {
    float mn, mx;
    int nan, pad;
};

__device__ __forceinline__ uint8_t quantise(float v) {  // trunc(v) for v in [0, 256); NaN -> 0 (cvt.rzi.sat)
    return (uint8_t)min(__float2uint_rz(v), 255u);
}

__device__ void block_minmax(float& mn, float& mx, int& nan) {
    __shared__ float s_mn[VI_THREADS / 32], s_mx[VI_THREADS / 32];
    __shared__ int s_nan[VI_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        nan |= __shfl_xor_sync(0xffffffffu, nan, o);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        s_mn[w] = mn;
        s_mx[w] = mx;
        s_nan[w] = nan;
    }
    __syncthreads();
    mn = s_mn[0];
    mx = s_mx[0];
    nan = s_nan[0];
    for (int i = 1; i < VI_THREADS / 32; ++i) {
        mn = fminf(mn, s_mn[i]);
        mx = fmaxf(mx, s_mx[i]);
        nan |= s_nan[i];
    }
}

__global__ void __launch_bounds__(VI_THREADS) k_depth_minmax(const float* __restrict__ depth, int64_t n, MinMax* part) {
    float mn = __int_as_float(0x7f800000), mx = -__int_as_float(0x7f800000);
    int nan = 0;
    for (int64_t i = blockIdx.x * (int64_t)VI_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * VI_THREADS) {
        const float d = depth[i];
        if (d != d) nan = 1;
        else {
            mn = fminf(mn, d);
            mx = fmaxf(mx, d);
        }
    }
    block_minmax(mn, mx, nan);
    if (threadIdx.x == 0) part[blockIdx.x] = MinMax{mn, mx, nan, 0};
}

__global__ void __launch_bounds__(VI_THREADS) k_view_images(const float* __restrict__ rgb, const float* __restrict__ depth,
                                                            int64_t n, const MinMax* __restrict__ part, int n_part,
                                                            uint8_t* __restrict__ rgb_img, uint8_t* __restrict__ depth_img) {
    float mn = __int_as_float(0x7f800000), mx = -__int_as_float(0x7f800000);
    int nan = 0;
    if (depth_img) {
        // every block reduces the partials in the same order: one min/max for the whole view
        for (int i = threadIdx.x; i < n_part; i += VI_THREADS) {
            mn = fminf(mn, part[i].mn);
            mx = fmaxf(mx, part[i].mx);
            nan |= part[i].nan;
        }
        block_minmax(mn, mx, nan);
    }
    const float range = __fsub_rn(mx, mn);
    for (int64_t i = blockIdx.x * (int64_t)VI_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * VI_THREADS) {
        if (rgb_img) {
#pragma unroll
            for (int k = 0; k < 3; ++k) rgb_img[3 * i + k] = quantise(__fmul_rn(rgb[3 * i + k], 255.0f));
        }
        if (depth_img) {
            // numpy: NaN anywhere makes min and max NaN, and every pixel NaN; a constant map is 0/0 = NaN; NaN -> 0
            const int idx = nan ? 0 : quantise(__fmul_rn(__fdiv_rn(__fsub_rn(depth[i], mn), range), 255.0f));
#pragma unroll
            for (int k = 0; k < 3; ++k) depth_img[3 * i + k] = TURBO_BGR[3 * idx + k];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// CRC-32 and Adler-32 helpers
// ---------------------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {  // a * b mod P, reflected
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}

__device__ __forceinline__ uint32_t x8nmodp(uint64_t n) {  // x^(8 n) mod P
    uint32_t p = 1u << 31;  // x^0
    int k = 3;
    while (n) {
        if (n & 1) p = multmodp(X2N[k & 31], p);
        n >>= 1;
        ++k;
    }
    return p;
}

// CRC of A || B from crc(A), crc(B) and len(B) (zlib's crc32_combine)
__device__ __forceinline__ uint32_t crc_combine(uint32_t c1, uint32_t c2, uint64_t len2) {
    return multmodp(x8nmodp(len2), c1) ^ c2;
}

__device__ void crc_table(uint32_t* tab) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = (uint32_t)i;
        for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
        tab[i] = c;
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------------------
// PNG: filters (one warp per row)
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (uint8_t)((pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c));
}

__device__ __forceinline__ uint8_t filt_byte(int f, int x, int a, int b, int c) {
    switch (f) {
        case 0: return (uint8_t)x;
        case 1: return (uint8_t)(x - a);
        case 2: return (uint8_t)(x - b);
        case 3: return (uint8_t)(x - ((a + b) >> 1));
        default: return (uint8_t)(x - paeth(a, b, c));
    }
}

__global__ void __launch_bounds__(PNG_WARPS * 32) k_png_filter(const uint8_t* __restrict__ img, int H, int W,
                                                               uint8_t* __restrict__ filt, PngRow* __restrict__ rows) {
    const int lane = threadIdx.x & 31;
    const int64_t RB = 3 * (int64_t)W, L = RB + 1;
    for (int64_t r = blockIdx.x * (int64_t)PNG_WARPS + (threadIdx.x >> 5); r < H; r += (int64_t)gridDim.x * PNG_WARPS) {
        const uint8_t* x = img + r * RB;
        const uint8_t* up = r > 0 ? x - RB : nullptr;
        unsigned long long s[5] = {0, 0, 0, 0, 0};
        for (int64_t j = lane; j < RB; j += 32) {
            const int xv = x[j], a = j >= 3 ? x[j - 3] : 0, b = up ? up[j] : 0, c = (up && j >= 3) ? up[j - 3] : 0;
#pragma unroll
            for (int f = 0; f < 5; ++f) {
                const int v = filt_byte(f, xv, a, b, c);
                s[f] += v < 128 ? v : 256 - v;  // |filtered byte read as int8|
            }
        }
        int best = 0;
        unsigned long long best_s = 0;
#pragma unroll
        for (int f = 0; f < 5; ++f) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s[f] += __shfl_xor_sync(0xffffffffu, s[f], o);
            if (f == 0 || s[f] < best_s) {  // ties: the lowest filter type
                best = f;
                best_s = s[f];
            }
        }
        uint8_t* out = filt + r * L;
        // Adler-32 parts over the segment's bytes d_i, i = 0..L-1 (d_0 = the filter type)
        unsigned long long sa = 0, sb = 0;
        if (lane == 0) {
            out[0] = (uint8_t)best;
            sa = (unsigned)best;
            sb = (unsigned long long)(L % ADLER_MOD) * (unsigned)best;
        }
        for (int64_t j = lane; j < RB; j += 32) {
            const int xv = x[j], a = j >= 3 ? x[j - 3] : 0, b = up ? up[j] : 0, c = (up && j >= 3) ? up[j - 3] : 0;
            const uint8_t v = filt_byte(best, xv, a, b, c);
            out[1 + j] = v;
            sa += v;
            sb += (unsigned long long)((L - 1 - j) % ADLER_MOD) * v;
            if ((j >> 5) % 4096 == 4095) {  // keep the sums far from overflow on very wide rows
                sa %= ADLER_MOD;
                sb %= ADLER_MOD;
            }
        }
        sa %= ADLER_MOD;
        sb %= ADLER_MOD;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if (lane == 0) {
            rows[r].a = (uint32_t)(sa % ADLER_MOD);
            rows[r].b = (uint32_t)(sb % ADLER_MOD);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// PNG: deflate of one segment per warp
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rev_bits(uint32_t code, int n) { return __brev(code) >> (32 - n); }

// the token at a parse position as LSB-first bits: a literal, or length + distance codes with their extra bits
__device__ __forceinline__ void token_bits(uint32_t t, uint32_t lit, int64_t L, uint32_t& code, int& nb) {
    if (t == 0) {
        if (lit < 144) {
            code = rev_bits(0x30 + lit, 8);
            nb = 8;
        } else {
            code = rev_bits(0x190 + lit - 144, 9);
            nb = 9;
        }
        return;
    }
    const uint32_t len = t & 511, k = t >> 9;
    const uint32_t d = k == 0 ? 1u : k == 1 ? 3u : (uint32_t)(k == 2 ? L : 2 * L);
    uint32_t sym, le = 0, lx = 0;
    if (len == 258) sym = 285;
    else {
        const uint32_t v = len - 3;
        if (v < 8) sym = 257 + v;
        else {
            le = 31 - __clz(v) - 2;
            sym = 261 + 4 * le + ((v >> le) & 3);
            lx = v & ((1u << le) - 1);
        }
    }
    if (sym < 280) {
        code = rev_bits(sym - 256, 7);
        nb = 7;
    } else {
        code = rev_bits(0xC0 + sym - 280, 8);
        nb = 8;
    }
    code |= lx << nb;
    nb += le;
    const uint32_t v = d - 1;
    uint32_t dc = v, de = 0, dx = 0;
    if (v >= 4) {
        de = 31 - __clz(v) - 1;
        dc = 2 * de + 2 + ((v >> de) & 1);
        dx = v & ((1u << de) - 1);
    }
    code |= rev_bits(dc, 5) << nb;
    nb += 5;
    code |= dx << nb;
    nb += de;
}

__device__ __forceinline__ void put_bits(uint32_t* buf, int64_t n_words, int64_t off, uint32_t code, int nb) {
    const int64_t w = off >> 5;
    const int sh = (int)(off & 31);
    if (w < n_words) atomicOr(buf + w, code << sh);
    if (sh + nb > 32 && w + 1 < n_words) atomicOr(buf + w + 1, code >> (32 - sh));
}

__host__ __device__ __forceinline__ int64_t stored_len(int64_t L) {  // the stored segment, its sync block included
    return L + 5 * ((L + STORED_MAX - 1) / STORED_MAX) + 5;
}

__global__ void __launch_bounds__(PNG_WARPS * 32) k_png_deflate(const uint8_t* __restrict__ filt, int H, int W,
                                                                uint16_t* __restrict__ tok_ws, uint8_t* __restrict__ seg,
                                                                int64_t seg_stride, PngRow* __restrict__ rows) {
    __shared__ uint32_t s_crc[256];
    crc_table(s_crc);
    const int lane = threadIdx.x & 31;
    const int64_t L = 3 * (int64_t)W + 1;
    const int64_t n_chunks = (L + 31) / 32;
    const int64_t dist[4] = {1, 3, L, 2 * L};  // ascending: a tie in length goes to the smaller distance
    for (int64_t r = blockIdx.x * (int64_t)PNG_WARPS + (threadIdx.x >> 5); r < H; r += (int64_t)gridDim.x * PNG_WARPS) {
        const int64_t p0 = r * L;
        uint16_t* tok = tok_ws + p0;
        // 1. longest match per position, back to front: run_d(j) = (s[p] == s[p-d]) ? 1 + run_d(j+1) : 0, stopping at the
        //    segment's end; tok = length | distance index << 9, or 0 for a literal (no match of 3 or more)
        uint32_t carry[4] = {0, 0, 0, 0};
        for (int64_t c = n_chunks - 1; c >= 0; --c) {
            const int64_t j = c * 32 + lane, p = p0 + j;
            const bool in = j < L;
            const uint8_t v = in ? filt[p] : 0;
            uint32_t best_len = 0, best_k = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int64_t d = dist[k];
                const bool eq = in && d <= MAX_DIST && p >= d && filt[p - d] == v;
                const uint32_t above = __ballot_sync(0xffffffffu, !eq) >> lane;
                uint32_t run = above ? (uint32_t)(__ffs(above) - 1) : 32 - lane + carry[k];
                run = min(run, (uint32_t)MAX_MATCH);
                carry[k] = __shfl_sync(0xffffffffu, run, 0);
                if (run > best_len) {
                    best_len = run;
                    best_k = k;
                }
            }
            if (in) tok[j] = best_len >= 3 ? (uint16_t)(best_len | (best_k << 9)) : 0;
        }
        // 2. clear the segment buffer, then the greedy parse front to back, one 32-position chunk at a time: the walk
        //    hops through the chunk by shuffles, and the tokens it lands on are coded in parallel at offsets from a scan.
        //    Bits past the buffer are dropped: they belong to a fixed block longer than the stored one, which is not used.
        uint8_t* out = seg + r * seg_stride;
        uint32_t* ow = reinterpret_cast<uint32_t*>(out);
        const int64_t n_words = seg_stride / 4;
        for (int64_t w = lane; w < n_words; w += 32) ow[w] = 0;
        __syncwarp();
        if (lane == 0) atomicOr(ow, 2u);  // BFINAL 0, BTYPE 01 (fixed Huffman)
        int64_t bit = 3, next = 0;
        for (int64_t c = 0; c < n_chunks; ++c) {
            const int64_t base = c * 32, j = base + lane;
            const uint32_t t = j < L ? tok[j] : 0;
            const uint32_t lit = j < L ? filt[p0 + j] : 0;
            uint32_t starts = 0;
            while (next < base + 32 && next < L) {
                const int i = (int)(next - base);
                const uint32_t ti = __shfl_sync(0xffffffffu, t, i);
                starts |= 1u << i;
                next += ti ? (ti & 511) : 1;
            }
            uint32_t code = 0;
            int nb = 0;
            if ((starts >> lane) & 1) token_bits(t, lit, L, code, nb);
            int inc = nb;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += u;
            }
            if (nb) put_bits(ow, n_words, bit + inc - nb, code, nb);
            bit += __shfl_sync(0xffffffffu, inc, 31);
        }
        bit += 7;  // end of block, code 0000000
        const bool last = r == H - 1;
        const int64_t fixed_len = (bit + 3 + 7) / 8 + 4;  // + the sync block's 3 header bits, padding, LEN, NLEN
        const int64_t st_len = stored_len(L);
        __syncwarp();
        int64_t len;
        if (st_len <= fixed_len) {
            // stored blocks of at most 65535 bytes (header byte 0: BFINAL 0, BTYPE 00, padding), then the sync block
            len = st_len;
            for (int64_t b0 = 0, q = 0; b0 < L; b0 += STORED_MAX, q += STORED_MAX + 5) {
                const int64_t n = min(STORED_MAX, L - b0);
                if (lane < 5) {  // 00, LEN, NLEN (little-endian)
                    const uint32_t len_nlen = (uint32_t)n | ((uint32_t)~n << 16);
                    out[q + lane] = lane == 0 ? 0 : (uint8_t)(len_nlen >> (8 * (lane - 1)));
                }
                for (int64_t i = lane; i < n; i += 32) out[q + 5 + i] = filt[p0 + b0 + i];
            }
            if (lane < 5) out[st_len - 5 + lane] = lane == 0 ? (uint8_t)last : lane < 3 ? 0 : 0xff;  // BFINAL, 0000, ffff
        } else {
            len = fixed_len;
            if (lane == 0) {
                if (last) put_bits(ow, n_words, bit, 1u, 1);  // the sync block's BFINAL
                put_bits(ow, n_words, (fixed_len - 2) * 8, 0xffffu, 16);  // LEN = 0000, NLEN = ffff
            }
        }
        __syncwarp();
        // 3. CRC-32 of the segment: per-lane slices combined in lane order
        const int64_t slice = (len + 31) / 32, lo = min(len, lane * slice), hi = min(len, lo + slice);
        uint32_t crc = ~0u;
        for (int64_t i = lo; i < hi; ++i) crc = s_crc[(crc ^ __ldcg(out + i)) & 0xff] ^ (crc >> 8);
        crc = ~crc;
        uint64_t n = (uint64_t)(hi - lo);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t c2 = __shfl_down_sync(0xffffffffu, crc, o);
            const uint64_t n2 = __shfl_down_sync(0xffffffffu, n, o);
            if ((lane & (2 * o - 1)) == 0) {
                crc = crc_combine(crc, c2, n2);
                n += n2;
            }
        }
        if (lane == 0) {
            rows[r].len = (uint32_t)len;
            rows[r].crc = crc;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// PNG: assembly -- offsets, checksums, headers (one block), then the compaction of the segments
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FIN_THREADS = 512;

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24);
    p[1] = (uint8_t)(v >> 16);
    p[2] = (uint8_t)(v >> 8);
    p[3] = (uint8_t)v;
}

// writes the n low bytes of v big-endian at out[i], updating the running (pre-inverted) CRC c
__device__ __forceinline__ void put_crc(uint8_t* out, int64_t i, uint32_t v, int n, const uint32_t* tab, uint32_t& c) {
    for (int k = n - 1; k >= 0; --k, ++i) {
        const uint8_t b = (uint8_t)(v >> (8 * k));
        out[i] = b;
        c = tab[(c ^ b) & 0xff] ^ (c >> 8);
    }
}

struct Adler {
    uint32_t a, b;
    uint64_t n;
};

__device__ __forceinline__ Adler adler_combine(Adler x, Adler y) {  // x's bytes, then y's
    return Adler{(x.a + y.a) % ADLER_MOD,
                 (uint32_t)((x.b + (uint64_t)(y.n % ADLER_MOD) * x.a + y.b) % ADLER_MOD), x.n + y.n};
}

// rows: the Adler-32 parts of the H filtered rows; segs: the byte length and CRC of the n_seg deflate segments, in
// stream order (the rows themselves in the fixed mode, the row groups in the dynamic mode)
__global__ void __launch_bounds__(FIN_THREADS) k_png_finish(const PngRow* __restrict__ rows, int H,
                                                            const PngRow* __restrict__ segs, int n_seg, int W, int64_t L,
                                                            int64_t* __restrict__ offs, uint8_t* __restrict__ out,
                                                            int64_t* __restrict__ out_len) {
    __shared__ uint32_t s_tab[256];
    __shared__ int64_t s_sum[FIN_THREADS];
    __shared__ uint32_t s_crc[FIN_THREADS];
    __shared__ uint64_t s_clen[FIN_THREADS];
    __shared__ Adler s_ad[FIN_THREADS];
    crc_table(s_tab);
    const int t = threadIdx.x;
    const int64_t q = (n_seg + FIN_THREADS - 1) / FIN_THREADS, r0 = min((int64_t)n_seg, t * q),
                  r1 = min((int64_t)n_seg, r0 + q);
    const int64_t qa = (H + FIN_THREADS - 1) / FIN_THREADS, a0 = min((int64_t)H, t * qa), a1 = min((int64_t)H, a0 + qa);
    int64_t sum = 0;
    uint32_t crc = 0;
    uint64_t clen = 0;
    Adler ad{0, 0, 0};
    for (int64_t r = r0; r < r1; ++r) {
        const PngRow seg = segs[r];
        sum += seg.len;
        crc = crc_combine(crc, seg.crc, seg.len);
        clen += seg.len;
    }
    for (int64_t r = a0; r < a1; ++r) ad = adler_combine(ad, Adler{rows[r].a, rows[r].b, (uint64_t)L});
    s_sum[t] = sum;
    s_crc[t] = crc;
    s_clen[t] = clen;
    s_ad[t] = ad;
    __syncthreads();
    for (int o = 1; o < FIN_THREADS; o <<= 1) {  // inclusive scan of the byte counts
        const int64_t u = t >= o ? s_sum[t - o] : 0;
        __syncthreads();
        s_sum[t] += u;
        __syncthreads();
    }
    int64_t off = s_sum[t] - sum;
    for (int64_t r = r0; r < r1; ++r) {
        offs[r] = off;
        off += segs[r].len;
    }
    for (int o = 1; o < FIN_THREADS; o <<= 1) {  // checksums: a fixed-order tree over the threads' row ranges
        if ((t & (2 * o - 1)) == 0 && t + o < FIN_THREADS) {
            s_crc[t] = crc_combine(s_crc[t], s_crc[t + o], s_clen[t + o]);
            s_clen[t] += s_clen[t + o];
            s_ad[t] = adler_combine(s_ad[t], s_ad[t + o]);
        }
        __syncthreads();
    }
    if (t != 0) return;
    const int64_t z = 2 + s_sum[FIN_THREADS - 1] + 4;  // IDAT data: zlib header, segments, Adler-32
    const uint64_t sig = 0x0a1a0a0d474e5089ull;        // 89 'P' 'N' 'G' 0d 0a 1a 0a
    for (int i = 0; i < 8; ++i) out[i] = (uint8_t)(sig >> (8 * i));
    put_be32(out + 8, 13);
    uint32_t c = ~0u;  // running CRC (pre-inverted) of the bytes put_crc writes
    put_crc(out, 12, 0x49484452u, 4, s_tab, c);  // "IHDR"
    put_crc(out, 16, (uint32_t)W, 4, s_tab, c);
    put_crc(out, 20, (uint32_t)H, 4, s_tab, c);
    put_crc(out, 24, 0x08020000u, 4, s_tab, c);  // 8-bit, colour type 2 (RGB), compression 0, filter 0
    put_crc(out, 28, 0u, 1, s_tab, c);           // no interlace
    put_be32(out + 29, ~c);
    put_be32(out + 33, (uint32_t)z);
    c = ~0u;
    put_crc(out, 37, 0x49444154u, 4, s_tab, c);  // "IDAT"
    put_crc(out, 41, 0x7801u, 2, s_tab, c);      // zlib: deflate, 32 KiB window, FCHECK
    uint32_t crc_idat = crc_combine(~c, s_crc[0], s_clen[0]);
    const Adler a = s_ad[0];
    const uint32_t adler = ((uint32_t)((a.b + a.n % ADLER_MOD) % ADLER_MOD) << 16) | ((a.a + 1) % ADLER_MOD);
    const int64_t e = PNG_HEAD + z - 4;
    c = ~0u;
    put_crc(out, e, adler, 4, s_tab, c);
    crc_idat = crc_combine(crc_idat, ~c, 4);
    put_be32(out + e + 4, crc_idat);
    put_be32(out + e + 8, 0);
    put_be32(out + e + 12, 0x49454e44u);  // "IEND"
    put_be32(out + e + 16, 0xae426082u);  // its CRC
    *out_len = PNG_HEAD + z + PNG_TAIL - 4;
}

__global__ void __launch_bounds__(PNG_WARPS * 32) k_png_copy(const uint8_t* __restrict__ seg, int64_t seg_stride, int H,
                                                             const PngRow* __restrict__ rows, const int64_t* __restrict__ offs,
                                                             uint8_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = blockIdx.x * (int64_t)PNG_WARPS + (threadIdx.x >> 5); r < H; r += (int64_t)gridDim.x * PNG_WARPS) {
        const uint8_t* src = seg + r * seg_stride;
        uint8_t* dst = out + PNG_HEAD + 2 + offs[r];
        const int64_t n = rows[r].len;
        for (int64_t i = lane; i < n; i += 32) dst[i] = src[i];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// PNG, dynamic mode: a lazy parse over eleven distances per row (warp), one block per group of PNG_GROUP rows coded
// with package-merge Huffman tables, fixed Huffman or stored (one CTA per group), the rows' tokens OR-ed into the
// group's buffer at offsets from the tables kernel (warp per row), and a CRC per group
// ---------------------------------------------------------------------------------------------------------------------
constexpr int PNG_GROUP = 32;         // rows per block; also the warps of k_png_tables, one per row
constexpr int N_LL = 286, N_DD = 30;  // literal/length and distance alphabets
constexpr int N_SYM = N_LL + N_DD;    // one row's histogram: N_LL literal/length counts, then N_DD distance counts
constexpr int MAX_CANDS = 11;
constexpr int PM_MAX = N_LL;
enum { MODE_DYNAMIC = 0, MODE_FIXED = 1, MODE_STORED = 2 };

struct PngDists {  // the candidate distances of the row length, ascending and distinct
    int64_t d[MAX_CANDS];
    int n;
};

struct GroupCode {
    int mode;
    uint32_t code[N_SYM];  // bit-reversed code | length << 16, literal/length then distance
};

__host__ __forceinline__ PngDists png_dists(int64_t L) {
    const int64_t c[MAX_CANDS] = {1, 2, 3, 4, 6, 9, 12, L - 3, L, L + 3, 2 * L};
    int64_t s[MAX_CANDS];
    std::copy(c, c + MAX_CANDS, s);
    std::sort(s, s + MAX_CANDS);
    PngDists y{};
    for (int i = 0; i < MAX_CANDS; ++i)
        if (s[i] >= 1 && s[i] <= MAX_DIST && (y.n == 0 || s[i] != y.d[y.n - 1])) y.d[y.n++] = s[i];
    return y;
}

__device__ __forceinline__ uint32_t len_sym(uint32_t len, uint32_t& ext, uint32_t& val) {  // RFC 1951 3.2.5
    ext = 0;
    val = 0;
    if (len == 258) return 285;
    const uint32_t v = len - 3;
    if (v < 8) return 257 + v;
    ext = 31 - __clz(v) - 2;
    val = v & ((1u << ext) - 1);
    return 261 + 4 * ext + ((v >> ext) & 3);
}

__device__ __forceinline__ uint32_t dist_sym(uint32_t d, uint32_t& ext, uint32_t& val) {
    const uint32_t v = d - 1;
    ext = 0;
    val = 0;
    if (v < 4) return v;
    ext = 31 - __clz(v) - 1;
    val = v & ((1u << ext) - 1);
    return 2 * ext + 2 + ((v >> ext) & 1);
}

__host__ __device__ __forceinline__ int sym_extra(int s) {  // extra bits of a histogram slot
    if (s < N_LL) return (s >= 265 && s < 285) ? (s - 261) / 4 : 0;
    const int c = s - N_LL;
    return c < 4 ? 0 : c / 2 - 1;
}

// the parse at a position whose best match is t and whose successor's is tn: the token's length, 1 for a literal
__device__ __forceinline__ uint32_t lazy_adv(uint32_t t, uint32_t tn) {
    const uint32_t m = t & 511;
    return (m && (tn & 511) <= m) ? m : 1;
}

__global__ void __launch_bounds__(PNG_WARPS * 32) k_png_parse(const uint8_t* __restrict__ filt, int H, int W,
                                                              PngDists dists, uint16_t* __restrict__ tok_ws,
                                                              uint32_t* __restrict__ starts, uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_hist[PNG_WARPS][N_SYM];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t L = 3 * (int64_t)W + 1;
    const int64_t n_chunks = (L + 31) / 32;
    uint32_t* sh = s_hist[wib];
    for (int64_t r = blockIdx.x * (int64_t)PNG_WARPS + wib; r < H; r += (int64_t)gridDim.x * PNG_WARPS) {
        const int64_t p0 = r * L;
        uint16_t* tok = tok_ws + p0;
        for (int i = lane; i < N_SYM; i += 32) sh[i] = 0;
        // 1. longest match per position, as k_png_deflate's step 1 over the candidate list
        uint32_t carry[MAX_CANDS];
#pragma unroll
        for (int k = 0; k < MAX_CANDS; ++k) carry[k] = 0;
        for (int64_t c = n_chunks - 1; c >= 0; --c) {
            const int64_t j = c * 32 + lane, p = p0 + j;
            const bool in = j < L;
            const uint8_t v = in ? filt[p] : 0;
            uint32_t best_len = 0, best_k = 0;
#pragma unroll
            for (int k = 0; k < MAX_CANDS; ++k) {
                if (k < dists.n) {
                    const int64_t d = dists.d[k];
                    const bool eq = in && p >= d && filt[p - d] == v;
                    const uint32_t above = __ballot_sync(0xffffffffu, !eq) >> lane;
                    uint32_t run = above ? (uint32_t)(__ffs(above) - 1) : 32 - lane + carry[k];
                    run = min(run, (uint32_t)MAX_MATCH);
                    carry[k] = __shfl_sync(0xffffffffu, run, 0);
                    if (run > best_len) {
                        best_len = run;
                        best_k = k;
                    }
                }
            }
            if (in) tok[j] = best_len >= 3 ? (uint16_t)(best_len | (best_k << 9)) : 0;
        }
        __syncwarp();
        // 2. the lazy parse front to back, walked by shuffles as in k_png_deflate; the tokens' symbols are counted
        int64_t next = 0;
        for (int64_t c = 0; c < n_chunks; ++c) {
            const int64_t base = c * 32, j = base + lane;
            const uint32_t t = j < L ? tok[j] : 0;
            const uint32_t adv = lazy_adv(t, j + 1 < L ? tok[j + 1] : 0);
            uint32_t st = 0;
            while (next < base + 32 && next < L) {
                const int i = (int)(next - base);
                st |= 1u << i;
                next += __shfl_sync(0xffffffffu, adv, i);
            }
            if ((st >> lane) & 1) {
                uint32_t e, x;
                if (adv == 1) atomicAdd(sh + filt[p0 + j], 1u);
                else {
                    atomicAdd(sh + len_sym(adv, e, x), 1u);
                    atomicAdd(sh + N_LL + dist_sym((uint32_t)dists.d[t >> 9], e, x), 1u);
                }
            }
            if (lane == 0) starts[r * n_chunks + c] = st;
        }
        __syncwarp();
        for (int i = lane; i < N_SYM; i += 32) hist[r * N_SYM + i] = sh[i];
        __syncwarp();
    }
}

struct PmScratch {
    unsigned long long w[PM_MAX], cur[2 * PM_MAX], pk[PM_MAX];
    uint16_t sym[PM_MAX];
    uint8_t flag[15][2 * PM_MAX];
};

// Code lengths <= limit for the symbols of cnt[0..n_alpha) with a non-zero count, by package-merge: items sorted by
// (count, symbol), an item before a package of equal weight; one used symbol gets length 1. Called by every thread of a
// block of at least 2 * PM_MAX threads.
__device__ void package_merge(const uint32_t* cnt, int n_alpha, int limit, uint8_t* len, PmScratch& s) {
    const int t = threadIdx.x;
    if (t < n_alpha) {
        len[t] = 0;
        if (cnt[t]) {
            int rank = 0;
            for (int j = 0; j < n_alpha; ++j) rank += cnt[j] && (cnt[j] < cnt[t] || (cnt[j] == cnt[t] && j < t));
            s.w[rank] = cnt[t];
            s.sym[rank] = (uint16_t)t;
        }
    }
    const int n = __syncthreads_count(t < n_alpha && cnt[t]);
    if (n <= 1) {
        if (n == 1 && t == 0) len[s.sym[0]] = 1;
        __syncthreads();
        return;
    }
    if (t < n) {
        s.cur[t] = s.w[t];
        s.flag[0][t] = 1;
    }
    int size = n;
    __syncthreads();
    for (int lv = 1; lv < limit; ++lv) {
        const int np = size / 2;
        if (t < np) s.pk[t] = s.cur[2 * t] + s.cur[2 * t + 1];
        __syncthreads();
        if (t < n) {  // an item goes after the packages lighter than it
            const unsigned long long x = s.w[t];
            int lo = 0, hi = np;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (s.pk[mid] < x) lo = mid + 1;
                else hi = mid;
            }
            s.cur[t + lo] = x;
            s.flag[lv][t + lo] = 1;
        }
        if (t < np) {  // a package goes after the items no heavier than it
            const unsigned long long x = s.pk[t];
            int lo = 0, hi = n;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (s.w[mid] <= x) lo = mid + 1;
                else hi = mid;
            }
            s.cur[t + lo] = x;
            s.flag[lv][t + lo] = 0;
        }
        size = n + np;
        __syncthreads();
    }
    // the first 2n - 2 entries of the last list; a package among the first k entries of a list stands for the first 2
    // entries of the list below it, an item for one more bit of its symbol
    int k = 2 * n - 2;
    for (int lv = limit - 1; lv >= 0; --lv) {
        const int ni = __syncthreads_count(t < k && s.flag[lv][t]);
        if (t < ni) len[s.sym[t]] += 1;
        k = 2 * (k - ni);
    }
    __syncthreads();
}

// RFC 1951 3.2.2 canonical codes of len[0..n), bit-reversed, as code | length << 16; all threads of the block
__device__ void canonical_codes(const uint8_t* len, int n, uint32_t* code, uint32_t* next) {
    const int t = threadIdx.x;
    __syncthreads();
    if (t == 0) {
        uint32_t bl[16] = {0};
        for (int i = 0; i < n; ++i) bl[len[i]]++;
        uint32_t c = 0;
        bl[0] = 0;
        for (int b = 1; b < 16; ++b) {
            c = (c + bl[b - 1]) << 1;
            next[b] = c;
        }
    }
    __syncthreads();
    if (t < n) {
        const int l = len[t];
        uint32_t c = 0;
        if (l) {
            c = next[l];
            for (int j = 0; j < t; ++j) c += len[j] == l;
            c = rev_bits(c, l) | ((uint32_t)l << 16);
        }
        code[t] = c;
    }
    __syncthreads();
}

// zlib's send_tree over len[0..n): code-length symbols and their extra values appended to sym / val at *m
__device__ void rle_lengths(const uint8_t* len, int n, uint8_t* sym, uint8_t* val, int& m) {
    int prev = -1, nextlen = len[0], count = 0;
    int max_count = nextlen == 0 ? 138 : 7, min_count = nextlen == 0 ? 3 : 4;
    for (int i = 0; i < n; ++i) {
        const int cur = nextlen;
        nextlen = i + 1 < n ? len[i + 1] : 0xffff;
        if (++count < max_count && cur == nextlen) continue;
        if (count < min_count) {
            for (; count > 0; --count) {
                sym[m] = (uint8_t)cur;
                val[m++] = 0;
            }
        } else if (cur != 0) {
            if (cur != prev) {
                sym[m] = (uint8_t)cur;
                val[m++] = 0;
                --count;
            }
            sym[m] = 16;
            val[m++] = (uint8_t)(count - 3);
        } else if (count <= 10) {
            sym[m] = 17;
            val[m++] = (uint8_t)(count - 3);
        } else {
            sym[m] = 18;
            val[m++] = (uint8_t)(count - 11);
        }
        count = 0;
        prev = cur;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (cur == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}

__device__ __forceinline__ int fixed_len(int s) {
    if (s >= N_LL) return 5;
    return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
}

__device__ __forceinline__ uint32_t fixed_code(int s) {
    if (s >= N_LL) return rev_bits(s - N_LL, 5) | (5u << 16);
    if (s < 144) return rev_bits(0x30 + s, 8) | (8u << 16);
    if (s < 256) return rev_bits(0x190 + s - 144, 9) | (9u << 16);
    if (s < 280) return rev_bits(s - 256, 7) | (7u << 16);
    return rev_bits(0xC0 + s - 280, 8) | (8u << 16);
}

__device__ __forceinline__ void block_add(unsigned long long* acc, unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(acc, v);
}

constexpr int TAB_THREADS = PNG_GROUP * 32;
__constant__ uint8_t CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// One CTA per group: the group's histogram (a fixed-order sum of its rows'), the three codings' exact sizes, the choice,
// then the whole block but the rows' tokens: the zeroed buffer, the header, end-of-block and the empty stored block, or
// the stored blocks; the code table and each row's bit offset for k_png_emit.
__global__ void __launch_bounds__(TAB_THREADS) k_png_tables(const uint8_t* __restrict__ filt, int H, int W,
                                                            const uint32_t* __restrict__ hist, uint8_t* __restrict__ seg,
                                                            int64_t seg_stride, GroupCode* __restrict__ codes,
                                                            int64_t* __restrict__ row_off, PngRow* __restrict__ grp) {
    __shared__ PmScratch s_pm;
    __shared__ uint32_t s_cnt[N_SYM];
    __shared__ uint8_t s_len[N_SYM];
    __shared__ uint32_t s_code[N_SYM];
    __shared__ uint32_t s_cl_cnt[19], s_cl_code[19], s_next[16];
    __shared__ uint8_t s_cl_len[19];
    __shared__ uint8_t s_seq_sym[N_SYM], s_seq_val[N_SYM];
    __shared__ int s_nseq, s_nlit, s_ndist, s_ncl, s_mode;
    __shared__ int64_t s_glen;  // the group's bytes: shared, never read back from grp (written by thread 0 only)
    __shared__ unsigned long long s_bits[3];  // dynamic data bits, fixed data bits, extra bits
    __shared__ unsigned long long s_row_bits[PNG_GROUP];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int g = blockIdx.x;
    const int64_t L = 3 * (int64_t)W + 1;
    const int r0 = g * PNG_GROUP, nr = min(PNG_GROUP, H - r0);
    if (t < N_SYM) {
        uint32_t c = t == 256;  // end of block
        for (int r = r0; r < r0 + nr; ++r) c += hist[(int64_t)r * N_SYM + t];
        s_cnt[t] = c;
    }
    if (t < 3) s_bits[t] = 0;
    if (t < 19) s_cl_cnt[t] = 0;
    __syncthreads();
    package_merge(s_cnt, N_LL, 15, s_len, s_pm);
    package_merge(s_cnt + N_LL, N_DD, 15, s_len + N_LL, s_pm);
    if (t == 0) {
        int nd = 0;
        for (int i = 0; i < N_DD; ++i) nd += s_len[N_LL + i] != 0;
        if (nd == 0) s_len[N_LL] = 1;  // no distance code used: code 0 of length 1
        int nlit = 257, ndist = 1;
        for (int i = 257; i < N_LL; ++i)
            if (s_len[i]) nlit = i + 1;
        for (int i = 1; i < N_DD; ++i)
            if (s_len[N_LL + i]) ndist = i + 1;
        int m = 0;
        rle_lengths(s_len, nlit, s_seq_sym, s_seq_val, m);
        rle_lengths(s_len + N_LL, ndist, s_seq_sym, s_seq_val, m);
        for (int i = 0; i < m; ++i) s_cl_cnt[s_seq_sym[i]]++;
        s_nseq = m;
        s_nlit = nlit;
        s_ndist = ndist;
    }
    __syncthreads();
    package_merge(s_cl_cnt, 19, 7, s_cl_len, s_pm);
    canonical_codes(s_cl_len, 19, s_cl_code, s_next);
    canonical_codes(s_len, N_LL, s_code, s_next);
    canonical_codes(s_len + N_LL, N_DD, s_code + N_LL, s_next);
    // exact sizes: the token bits under each code, the dynamic header
    {
        const unsigned long long c = t < N_SYM ? s_cnt[t] : 0;
        block_add(&s_bits[0], t < N_SYM ? c * s_len[t] : 0);
        block_add(&s_bits[1], t < N_SYM ? c * fixed_len(t) : 0);
        block_add(&s_bits[2], t < N_SYM ? c * sym_extra(t) : 0);
    }
    __syncthreads();
    if (t == 0) {
        int ncl = 19;
        while (ncl > 4 && s_cl_len[CL_ORDER[ncl - 1]] == 0) --ncl;
        int64_t head = 3 + 14 + 3 * ncl;
        for (int i = 0; i < s_nseq; ++i) {
            const int sy = s_seq_sym[i];
            head += s_cl_len[sy] + (sy == 16 ? 2 : sy == 17 ? 3 : sy == 18 ? 7 : 0);
        }
        const int64_t dyn = head + (int64_t)(s_bits[0] + s_bits[2]), fix = 3 + (int64_t)(s_bits[1] + s_bits[2]);
        const int64_t n = nr * L;
        const int64_t sz[3] = {(dyn + 3 + 7) / 8 + 4, (fix + 3 + 7) / 8 + 4, n + 5 * ((n + STORED_MAX - 1) / STORED_MAX) + 5};
        int mode = 0;
        for (int k = 1; k < 3; ++k)
            if (sz[k] < sz[mode]) mode = k;  // a tie: dynamic, then fixed, then stored
        s_ncl = ncl;
        s_mode = mode;
        s_bits[0] = mode == MODE_DYNAMIC ? head : 3;  // the first token's bit
        s_glen = sz[mode];
        grp[g].len = (uint32_t)sz[mode];
    }
    __syncthreads();
    const int mode = s_mode;
    const bool last = g == (H - 1) / PNG_GROUP;
    uint8_t* out = seg + g * seg_stride;
    const int64_t len = s_glen;
    if (mode == MODE_STORED) {
        const uint8_t* src = filt + r0 * L;
        const int64_t n = nr * L;
        for (int64_t b0 = 0, q = 0; b0 < n; b0 += STORED_MAX, q += STORED_MAX + 5) {
            const int64_t m = min(STORED_MAX, n - b0);
            if (t < 5) {
                const uint32_t len_nlen = (uint32_t)m | ((uint32_t)~m << 16);
                out[q + t] = t == 0 ? 0 : (uint8_t)(len_nlen >> (8 * (t - 1)));
            }
            for (int64_t i = t; i < m; i += TAB_THREADS) out[q + 5 + i] = src[b0 + i];
        }
        if (t < 5) out[len - 5 + t] = t == 0 ? (uint8_t)last : t < 3 ? 0 : 0xff;
        if (t == 0) codes[g].mode = mode;
        return;
    }
    // the rows' bit counts under the chosen code (warp w: row r0 + w), their scan, the code table
    if (t < N_SYM) {
        const uint32_t c = mode == MODE_DYNAMIC ? s_code[t] : fixed_code(t);
        s_code[t] = c;
        codes[g].code[t] = c;
    }
    if (t == 0) codes[g].mode = mode;
    __syncthreads();
    if (w < nr) {
        const uint32_t* h = hist + (int64_t)(r0 + w) * N_SYM;
        unsigned long long b = 0;
        for (int i = lane; i < N_SYM; i += 32) b += (unsigned long long)h[i] * ((s_code[i] >> 16) + sym_extra(i));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
        if (lane == 0) s_row_bits[w] = b;
    }
    uint32_t* ow = reinterpret_cast<uint32_t*>(out);
    const int64_t n_words = seg_stride / 4;
    for (int64_t i = t; i < (len + 3) / 4; i += TAB_THREADS) ow[i] = 0;
    __syncthreads();
    if (t == 0) {
        int64_t bit = (int64_t)s_bits[0];
        for (int r = 0; r < nr; ++r) {
            row_off[r0 + r] = bit;
            bit += (int64_t)s_row_bits[r];
        }
        // end of block, the empty stored block's BFINAL, its LEN 0000 and NLEN ffff
        put_bits(ow, n_words, bit, s_code[256] & 0xffff, s_code[256] >> 16);
        bit += s_code[256] >> 16;
        if (last) put_bits(ow, n_words, bit, 1u, 1);
        put_bits(ow, n_words, (len - 2) * 8, 0xffffu, 16);
        if (mode == MODE_FIXED) put_bits(ow, n_words, 0, 2u, 3);
        else {  // BFINAL 0, BTYPE 10, HLIT, HDIST, HCLEN, the code-length code, the run-length coded lengths
            put_bits(ow, n_words, 0, 4u | (uint32_t)(s_nlit - 257) << 3 | (uint32_t)(s_ndist - 1) << 8 |
                                         (uint32_t)(s_ncl - 4) << 13, 17);
            int64_t b = 17;
            for (int i = 0; i < s_ncl; ++i, b += 3) put_bits(ow, n_words, b, s_cl_len[CL_ORDER[i]], 3);
            for (int i = 0; i < s_nseq; ++i) {
                const int sy = s_seq_sym[i];
                const int nb = s_cl_code[sy] >> 16, ne = sy == 16 ? 2 : sy == 17 ? 3 : sy == 18 ? 7 : 0;
                put_bits(ow, n_words, b, (s_cl_code[sy] & 0xffff) | (uint32_t)s_seq_val[i] << nb, nb + ne);
                b += nb + ne;
            }
        }
    }
}

__device__ __forceinline__ void put_bits64(uint32_t* buf, int64_t n_words, int64_t off, unsigned long long code, int nb) {
    const int64_t w = off >> 5;
    const int sh = (int)(off & 31);
    if (w < n_words) atomicOr(buf + w, (uint32_t)(code << sh));
    if (sh + nb > 32 && w + 1 < n_words) atomicOr(buf + w + 1, (uint32_t)(code >> (32 - sh)));
    if (sh + nb > 64 && w + 2 < n_words) atomicOr(buf + w + 2, (uint32_t)(code >> (64 - sh)));
}

// one warp per row: the row's tokens, coded with its group's table, OR-ed in at the row's bit offset
__global__ void __launch_bounds__(PNG_WARPS * 32) k_png_emit(const uint8_t* __restrict__ filt, int H, int W,
                                                             PngDists dists, const uint16_t* __restrict__ tok_ws,
                                                             const uint32_t* __restrict__ starts,
                                                             const GroupCode* __restrict__ codes,
                                                             const int64_t* __restrict__ row_off, uint8_t* __restrict__ seg,
                                                             int64_t seg_stride) {
    const int lane = threadIdx.x & 31;
    const int64_t L = 3 * (int64_t)W + 1;
    const int64_t n_chunks = (L + 31) / 32;
    for (int64_t r = blockIdx.x * (int64_t)PNG_WARPS + (threadIdx.x >> 5); r < H; r += (int64_t)gridDim.x * PNG_WARPS) {
        const int64_t g = r / PNG_GROUP;
        const GroupCode* gc = codes + g;
        if (gc->mode == MODE_STORED) continue;
        const int64_t p0 = r * L;
        const uint16_t* tok = tok_ws + p0;
        uint32_t* ow = reinterpret_cast<uint32_t*>(seg + g * seg_stride);
        const int64_t n_words = seg_stride / 4;
        int64_t bit = row_off[r];
        for (int64_t c = 0; c < n_chunks; ++c) {
            const int64_t j = c * 32 + lane;
            unsigned long long code = 0;
            int nb = 0;
            if ((starts[r * n_chunks + c] >> lane) & 1) {
                const uint32_t t = tok[j];
                const uint32_t adv = lazy_adv(t, j + 1 < L ? tok[j + 1] : 0);
                if (adv == 1) {
                    const uint32_t e = gc->code[filt[p0 + j]];
                    code = e & 0xffff;
                    nb = e >> 16;
                } else {
                    uint32_t ext, val;
                    uint32_t e = gc->code[len_sym(adv, ext, val)];
                    code = (e & 0xffff) | (unsigned long long)val << (e >> 16);
                    nb = (e >> 16) + ext;
                    const uint32_t ds = dist_sym((uint32_t)dists.d[t >> 9], ext, val);
                    e = gc->code[N_LL + ds];
                    code |= (unsigned long long)((e & 0xffff) | val << (e >> 16)) << nb;
                    nb += (e >> 16) + ext;
                }
            }
            int inc = nb;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += u;
            }
            if (nb) put_bits64(ow, n_words, bit + inc - nb, code, nb);
            bit += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
}

constexpr int GCRC_THREADS = 256;

// the CRC-32 of each group's bytes: per-thread slices combined in a fixed-order tree
__global__ void __launch_bounds__(GCRC_THREADS) k_png_group_crc(const uint8_t* __restrict__ seg, int64_t seg_stride,
                                                                PngRow* __restrict__ grp) {
    __shared__ uint32_t s_tab[256];
    __shared__ uint32_t s_crc[GCRC_THREADS];
    __shared__ uint64_t s_n[GCRC_THREADS];
    crc_table(s_tab);
    const int t = threadIdx.x;
    const uint8_t* src = seg + blockIdx.x * seg_stride;
    const int64_t len = grp[blockIdx.x].len;
    const int64_t slice = (len + GCRC_THREADS - 1) / GCRC_THREADS, lo = min(len, t * slice), hi = min(len, lo + slice);
    uint32_t crc = ~0u;
    for (int64_t i = lo; i < hi; ++i) crc = s_tab[(crc ^ src[i]) & 0xff] ^ (crc >> 8);
    s_crc[t] = ~crc;
    s_n[t] = (uint64_t)(hi - lo);
    __syncthreads();
    for (int o = 1; o < GCRC_THREADS; o <<= 1) {
        if ((t & (2 * o - 1)) == 0) {
            s_crc[t] = crc_combine(s_crc[t], s_crc[t + o], s_n[t + o]);
            s_n[t] += s_n[t + o];
        }
        __syncthreads();
    }
    if (t == 0) grp[blockIdx.x].crc = s_crc[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// workspace layout
// ---------------------------------------------------------------------------------------------------------------------
struct PngLayout {
    int64_t L, seg_stride, filt, tok, seg, rows, offs, total;
};

__host__ __forceinline__ int64_t align256(int64_t x) { return (x + 255) & ~(int64_t)255; }

bool png_layout(int H, int W, PngLayout& y) {
    if (H < 1 || W < 1) return false;
    y.L = 3 * (int64_t)W + 1;
    if (2 + 4 + (int64_t)H * stored_len(y.L) > INT32_MAX) return false;  // the IDAT length field
    y.seg_stride = (stored_len(y.L) + 15) & ~(int64_t)15;
    y.filt = 0;
    y.tok = align256((int64_t)H * y.L);
    y.seg = y.tok + align256((int64_t)H * y.L * 2);
    y.rows = y.seg + align256((int64_t)H * y.seg_stride);
    y.offs = y.rows + align256((int64_t)H * sizeof(PngRow));
    y.total = y.offs + align256((int64_t)H * 8);
    return true;
}

struct PngDynLayout {
    int64_t L, n_groups, n_chunks, seg_stride, filt, tok, starts, hist, row_off, rows, codes, grp, offs, seg, total;
};

bool png_dyn_layout(int H, int W, PngDynLayout& y) {
    PngLayout f;
    if (!png_layout(H, W, f)) return false;
    y.L = f.L;
    y.n_groups = (H + PNG_GROUP - 1) / PNG_GROUP;
    y.n_chunks = (y.L + 31) / 32;
    const int64_t n = std::min(H, PNG_GROUP) * y.L;  // a whole group stored: never longer than its rows stored one by one
    y.seg_stride = (n + 5 * ((n + STORED_MAX - 1) / STORED_MAX) + 5 + 15) & ~(int64_t)15;
    y.filt = 0;
    y.tok = align256((int64_t)H * y.L);
    y.starts = y.tok + align256((int64_t)H * y.L * 2);
    y.hist = y.starts + align256((int64_t)H * y.n_chunks * 4);
    y.row_off = y.hist + align256((int64_t)H * N_SYM * 4);
    y.rows = y.row_off + align256((int64_t)H * 8);
    y.codes = y.rows + align256((int64_t)H * sizeof(PngRow));
    y.grp = y.codes + align256(y.n_groups * (int64_t)sizeof(GroupCode));
    y.offs = y.grp + align256(y.n_groups * (int64_t)sizeof(PngRow));
    y.seg = y.offs + align256(y.n_groups * 8);
    y.total = y.seg + align256(y.n_groups * y.seg_stride);
    return true;
}

int grid_for(int64_t n_rows) { return (int)std::min<int64_t>((n_rows + PNG_WARPS - 1) / PNG_WARPS, 32LL * ngp_sm_count()); }

}  // namespace

extern "C" int ngp_view_images(const float* rgb, const float* depth, int H, int W, uint8_t* rgb_img, uint8_t* depth_img,
                               void* workspace, size_t workspace_bytes, void* stream) {
    if (H < 1 || W < 1 || (!rgb_img && !depth_img)) return NGP_EINVAL;
    if (rgb_img && (!ngp_dev_ptr(rgb, false) || !ngp_dev_ptr(rgb_img, false))) return NGP_EINVAL;
    if (depth_img && (!ngp_dev_ptr(depth, false) || !ngp_dev_ptr(depth_img, false) || !ngp_dev_ptr(workspace, false) ||
                      workspace_bytes < NGP_VIEW_IMAGES_WORKSPACE || ((uintptr_t)workspace & 15)))
        return NGP_EINVAL;
    const cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = (int64_t)H * W;
    const int grid = (int)std::min<int64_t>(ngp_div_up(n, VI_THREADS), 8LL * ngp_sm_count());
    MinMax* part = reinterpret_cast<MinMax*>(workspace);
    int n_part = 0;
    if (depth_img) {
        n_part = (int)std::min<int64_t>(VI_PARTIALS, ngp_div_up(n, 4 * VI_THREADS));
        k_depth_minmax<<<n_part, VI_THREADS, 0, st>>>(depth, n, part);
        NGP_CHECK_LAUNCH();
    }
    k_view_images<<<grid, VI_THREADS, 0, st>>>(rgb, depth, n, part, n_part, rgb_img, depth_img);
    NGP_CHECK_LAUNCH();
    return 0;
}

extern "C" size_t ngp_png_workspace(int H, int W) {
    PngLayout y;
    return png_layout(H, W, y) ? (size_t)y.total : 0;
}

extern "C" size_t ngp_png_capacity(int H, int W) {
    PngLayout y;
    return png_layout(H, W, y) ? (size_t)(PNG_HEAD + PNG_TAIL + 2 + (int64_t)H * stored_len(y.L)) : 0;
}

extern "C" int ngp_png_encode(const uint8_t* img, int H, int W, uint8_t* out, size_t out_capacity, int64_t* out_len,
                              void* workspace, size_t workspace_bytes, void* stream) {
    PngLayout y;
    if (!png_layout(H, W, y)) return NGP_EINVAL;
    if (!ngp_dev_ptr(img, false) || !ngp_dev_ptr(workspace, false) || !ngp_dev_ptr(out, true) || !ngp_dev_ptr(out_len, true))
        return NGP_EINVAL;
    if (workspace_bytes < (size_t)y.total || out_capacity < ngp_png_capacity(H, W) || ((uintptr_t)workspace & 255) ||
        ((uintptr_t)out_len & 7))
        return NGP_EINVAL;
    const cudaStream_t st = (cudaStream_t)stream;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    uint8_t* filt = ws + y.filt;
    uint16_t* tok = reinterpret_cast<uint16_t*>(ws + y.tok);
    uint8_t* seg = ws + y.seg;
    PngRow* rows = reinterpret_cast<PngRow*>(ws + y.rows);
    int64_t* offs = reinterpret_cast<int64_t*>(ws + y.offs);
    const int grid = grid_for(H);
    k_png_filter<<<grid, PNG_WARPS * 32, 0, st>>>(img, H, W, filt, rows);
    NGP_CHECK_LAUNCH();
    k_png_deflate<<<grid, PNG_WARPS * 32, 0, st>>>(filt, H, W, tok, seg, y.seg_stride, rows);
    NGP_CHECK_LAUNCH();
    k_png_finish<<<1, FIN_THREADS, 0, st>>>(rows, H, rows, H, W, y.L, offs, out, out_len);
    NGP_CHECK_LAUNCH();
    k_png_copy<<<grid, PNG_WARPS * 32, 0, st>>>(seg, y.seg_stride, H, rows, offs, out);
    NGP_CHECK_LAUNCH();
    return 0;
}

extern "C" size_t ngp_png_workspace_mode(int H, int W, int mode) {
    if (mode == NGP_PNG_FIXED) return ngp_png_workspace(H, W);
    PngDynLayout y;
    return mode == NGP_PNG_DYNAMIC && png_dyn_layout(H, W, y) ? (size_t)y.total : 0;
}

extern "C" int ngp_png_encode_mode(const uint8_t* img, int H, int W, int mode, uint8_t* out, size_t out_capacity,
                                   int64_t* out_len, void* workspace, size_t workspace_bytes, void* stream) {
    if (mode == NGP_PNG_FIXED) return ngp_png_encode(img, H, W, out, out_capacity, out_len, workspace, workspace_bytes, stream);
    PngDynLayout y;
    if (mode != NGP_PNG_DYNAMIC || !png_dyn_layout(H, W, y)) return NGP_EINVAL;
    if (!ngp_dev_ptr(img, false) || !ngp_dev_ptr(workspace, false) || !ngp_dev_ptr(out, true) || !ngp_dev_ptr(out_len, true))
        return NGP_EINVAL;
    if (workspace_bytes < (size_t)y.total || out_capacity < ngp_png_capacity(H, W) || ((uintptr_t)workspace & 255) ||
        ((uintptr_t)out_len & 7))
        return NGP_EINVAL;
    const cudaStream_t st = (cudaStream_t)stream;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    uint8_t* filt = ws + y.filt;
    uint16_t* tok = reinterpret_cast<uint16_t*>(ws + y.tok);
    uint32_t* starts = reinterpret_cast<uint32_t*>(ws + y.starts);
    uint32_t* hist = reinterpret_cast<uint32_t*>(ws + y.hist);
    int64_t* row_off = reinterpret_cast<int64_t*>(ws + y.row_off);
    PngRow* rows = reinterpret_cast<PngRow*>(ws + y.rows);
    GroupCode* codes = reinterpret_cast<GroupCode*>(ws + y.codes);
    PngRow* grp = reinterpret_cast<PngRow*>(ws + y.grp);
    int64_t* offs = reinterpret_cast<int64_t*>(ws + y.offs);
    uint8_t* seg = ws + y.seg;
    const PngDists dists = png_dists(y.L);
    const int grid = grid_for(H), n_groups = (int)y.n_groups;
    k_png_filter<<<grid, PNG_WARPS * 32, 0, st>>>(img, H, W, filt, rows);
    NGP_CHECK_LAUNCH();
    k_png_parse<<<grid, PNG_WARPS * 32, 0, st>>>(filt, H, W, dists, tok, starts, hist);
    NGP_CHECK_LAUNCH();
    k_png_tables<<<n_groups, TAB_THREADS, 0, st>>>(filt, H, W, hist, seg, y.seg_stride, codes, row_off, grp);
    NGP_CHECK_LAUNCH();
    k_png_emit<<<grid, PNG_WARPS * 32, 0, st>>>(filt, H, W, dists, tok, starts, codes, row_off, seg, y.seg_stride);
    NGP_CHECK_LAUNCH();
    k_png_group_crc<<<n_groups, GCRC_THREADS, 0, st>>>(seg, y.seg_stride, grp);
    NGP_CHECK_LAUNCH();
    k_png_finish<<<1, FIN_THREADS, 0, st>>>(rows, H, grp, n_groups, W, y.L, offs, out, out_len);
    NGP_CHECK_LAUNCH();
    k_png_copy<<<grid_for(n_groups), PNG_WARPS * 32, 0, st>>>(seg, y.seg_stride, n_groups, grp, offs, out);
    NGP_CHECK_LAUNCH();
    return 0;
}
