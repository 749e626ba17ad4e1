// Baseline JPEG of an (H, W, 3) uint8 device image, written by the device: ngp_jpeg_encode. The byte stream is specified
// in include/ngp_b200.h and restated in oracle/jpeg_ref.py; all arithmetic is integer and in libjpeg's order, so the
// files equal libjpeg's for the same settings (quality q, 4:4:4, the Annex K tables, the accurate integer DCT).
//
// Seven kernels: k_jpeg_dct (8 threads per MCU: colour conversion, row pass, column pass, quantisation, zig-zag),
// k_jpeg_count (a warp per MCU: the coded bits of its three blocks), k_jpeg_scan (one block: bit offsets),
// k_jpeg_emit (a warp per MCU: its codes OR-ed into the zeroed bit stream at its offset; OR is order-free),
// k_jpeg_ff (a warp per 512 stream bytes: how many are 0xFF), k_jpeg_scan again, k_jpeg_expand (a warp per 512 bytes:
// the stuffed bytes into out; block 0 also writes the headers, EOI and *out_len).
#include "common.cuh"
#include "ngp_b200.h"

#include <algorithm>

namespace {

constexpr int JPEG_HEAD = 623;          // SOI .. SOS
constexpr int JPEG_BLOCK_BYTES = 208;   // a block codes to at most 20 (DC) + 63 * 26 (AC) = 1658 bits
constexpr int JPEG_CHUNK = 512;         // stream bytes per warp in the stuffing kernels
constexpr int JPEG_THREADS = 256;
constexpr int JPEG_WARPS = JPEG_THREADS / 32;
constexpr int SCAN_THREADS = 1024;

// ---------------------------------------------------------------------------------------------------------------------
// tables (ITU-T T.81 Annex K), the derived Huffman codes and the header template, all made at compile time
// ---------------------------------------------------------------------------------------------------------------------
constexpr uint8_t ZIGZAG[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
constexpr uint8_t Q_BASE[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
     103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

struct HuffSpec {
    uint8_t bits[16];   // codes of each length 1..16
    uint8_t vals[162];  // symbols in code order
    int n;
};
// in DHT order: DC luminance, AC luminance, DC chrominance, AC chrominance
constexpr HuffSpec HUFF[4] = {
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12},
    {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
     {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
      0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
      0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
      0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
      0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
      0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
      0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
      0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
     162},
    {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12},
    {{0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
     {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
      0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
      0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
      0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
      0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
      0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
      0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
      0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
     162}};

// JFIF 1.01, no density unit, 1 x 1, no thumbnail; Y, Cb, Cr sampled 1 x 1 with quantisation tables 0, 1, 1; one scan of
// the three with Huffman tables 0, 1, 1 over coefficients 0..63
constexpr uint8_t JFIF[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
constexpr uint8_t SOF_COMPONENTS[10] = {3, 1, 0x11, 0, 2, 0x11, 1, 3, 0x11, 1};
constexpr uint8_t SOS[10] = {3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};

struct Tables {
    uint32_t code[4][256];  // canonical Huffman codes (Annex C), (code << 8) | length per symbol, tables in HUFF's order
    uint8_t zigzag[64], zz_pos[64];  // zig-zag position -> natural index, and back
    uint8_t q_base[128];             // Q_BASE
    uint8_t head[JPEG_HEAD];
    int dqt[2], sof_size;   // offsets in head of the two tables' 64 entries and of the height / width fields
};

constexpr Tables make_tables() {
    Tables t{};
    for (int k = 0; k < 4; ++k) {
        uint32_t c = 0;
        int v = 0;
        for (int n = 1; n <= 16; ++n) {
            for (int i = 0; i < HUFF[k].bits[n - 1]; ++i) t.code[k][HUFF[k].vals[v++]] = (c++ << 8) | (uint32_t)n;
            c <<= 1;
        }
    }
    for (int i = 0; i < 64; ++i) t.zigzag[i] = ZIGZAG[i], t.zz_pos[ZIGZAG[i]] = (uint8_t)i;
    for (int i = 0; i < 128; ++i) t.q_base[i] = Q_BASE[i >> 6][i & 63];
    int p = 0;
    auto put = [&](int b) { t.head[p++] = (uint8_t)b; };
    auto seg = [&](int marker, int payload) { put(0xFF), put(marker), put((payload + 2) >> 8), put((payload + 2) & 255); };
    put(0xFF), put(0xD8);
    seg(0xE0, 14);
    for (int b : JFIF) put(b);
    for (int k = 0; k < 2; ++k) {
        seg(0xDB, 65), put(k);
        t.dqt[k] = p;
        p += 64;
    }
    seg(0xC0, 15), put(8);
    t.sof_size = p;
    p += 4;
    for (int b : SOF_COMPONENTS) put(b);
    for (int k = 0; k < 4; ++k) {
        seg(0xC4, 17 + HUFF[k].n), put(((k & 1) << 4) | (k >> 1));
        for (int i = 0; i < 16; ++i) put(HUFF[k].bits[i]);
        for (int i = 0; i < HUFF[k].n; ++i) put(HUFF[k].vals[i]);
    }
    seg(0xDA, 10);
    for (int b : SOS) put(b);
    if (p != JPEG_HEAD) t.sof_size = -1;  // caught by the static_assert below
    return t;
}
constexpr Tables TABLES_HOST = make_tables();
static_assert(TABLES_HOST.sof_size > 0, "the header template is not JPEG_HEAD bytes");
__device__ const Tables TABLES = make_tables();

// libjpeg's quality scaling of a base table entry
__device__ __forceinline__ int quant_entry(int base, int quality) {
    const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    return min(max((base * s + 50) / 100, 1), 255);
}

// ---------------------------------------------------------------------------------------------------------------------
// colour conversion, forward DCT, quantisation
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// One 1-D pass of the Loeffler-Ligtenberg-Moschytz DCT with 13-bit constants. The first (row) pass leaves its results
// scaled up by 4; the second (column) pass removes that, and both leave the factor sqrt(8) per pass of the unnormalised
// transform: the block comes out scaled by 8, which the quantiser divides away.
template <bool FIRST>
__device__ __forceinline__ void dct_pass(int (&d)[8]) {
    constexpr int N = FIRST ? 13 - 2 : 13 + 2;
    const int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    const int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    d[0] = FIRST ? (t10 + t11) * 4 : descale(t10 + t11, 2);
    d[4] = FIRST ? (t10 - t11) * 4 : descale(t10 - t11, 2);
    int z1 = (t12 + t13) * 4433;
    d[2] = descale(z1 + t13 * 6270, N);
    d[6] = descale(z1 - t12 * 15137, N);
    z1 = t4 + t7;
    int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
    const int z5 = (z3 + z4) * 9633;
    z1 *= -7373, z2 *= -20995;
    z3 = z3 * -16069 + z5, z4 = z4 * -3196 + z5;
    d[7] = descale(t4 * 2446 + z1 + z3, N);
    d[5] = descale(t5 * 16819 + z2 + z4, N);
    d[3] = descale(t6 * 25172 + z2 + z3, N);
    d[1] = descale(t7 * 12299 + z1 + z4, N);
}

// 8 threads per MCU: thread t converts row t of the 8 x 8 pixels (the last column / row replicated past the edge) and,
// per component, runs the row pass on it, the column pass on column t after a transpose through shared memory, divides
// by 8 q rounding half away from zero and stores the block zig-zagged, 64 int16 at coef[(mcu * 3 + component) * 64].
__global__ void __launch_bounds__(JPEG_THREADS) k_jpeg_dct(const uint8_t* __restrict__ img, int H, int W, int quality,
                                                           int mcus_x, int n_mcu, int16_t* __restrict__ coef) {
    __shared__ int q8[2][64];
    __shared__ int tile[JPEG_THREADS / 8][8][9];
    __shared__ __align__(16) int16_t zz[JPEG_THREADS / 8][64];
    if (threadIdx.x < 128) q8[threadIdx.x >> 6][threadIdx.x & 63] = 8 * quant_entry(TABLES.q_base[threadIdx.x], quality);
    __syncthreads();
    const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
    const int mcu = blockIdx.x * (JPEG_THREADS / 8) + g;
    const bool live = mcu < n_mcu;
    const int m = live ? mcu : n_mcu - 1;
    const int y = min((m / mcus_x) * 8 + t, H - 1), x0 = (m % mcus_x) * 8;
    const uint8_t* row = img + (int64_t)y * W * 3;
    int r[8], gr[8], b[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint8_t* p = row + 3 * min(x0 + i, W - 1);
        r[i] = p[0], gr[i] = p[1], b[i] = p[2];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        int d[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {  // 16-bit fixed point, then the level shift
            if (c == 0) d[i] = ((19595 * r[i] + 38470 * gr[i] + 7471 * b[i] + 32768) >> 16) - 128;
            if (c == 1) d[i] = ((-11059 * r[i] - 21709 * gr[i] + 32768 * b[i] + (128 << 16) + 32767) >> 16) - 128;
            if (c == 2) d[i] = ((32768 * r[i] - 27439 * gr[i] - 5329 * b[i] + (128 << 16) + 32767) >> 16) - 128;
        }
        dct_pass<true>(d);
#pragma unroll
        for (int i = 0; i < 8; ++i) tile[g][t][i] = d[i];
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = tile[g][i][t];
        dct_pass<false>(d);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int q = q8[c > 0][i * 8 + t];
            const int a = (abs(d[i]) + (q >> 1)) / q;
            zz[g][TABLES.zz_pos[i * 8 + t]] = (int16_t)(d[i] < 0 ? -a : a);
        }
        __syncwarp();
        if (live) reinterpret_cast<uint4*>(coef + ((int64_t)mcu * 3 + c) * 64)[t] = reinterpret_cast<const uint4*>(zz[g])[t];
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// entropy coding
// ---------------------------------------------------------------------------------------------------------------------
// The codes of one block, as 64 independent slots: lane l of the warp holds slots l and l + 32 of the zig-zag sequence.
// Slot 0 is the DC difference, a non-zero AC slot is its ZRLs (one per 16 zeros of its run), run/size code and magnitude
// bits, slot 63 is the EOB when the last coefficient is zero, every other slot is empty. At most 3 * 11 + 16 + 10 = 59
// bits per slot, right-aligned in val.
struct Slots {
    uint64_t val[2];
    int len[2];
};

__device__ __forceinline__ void magnitude(int v, int& cat, uint32_t& extra) {
    cat = 32 - __clz(abs(v));
    extra = (uint32_t)(v < 0 ? v - 1 : v) & ((1u << cat) - 1);
}

__device__ __forceinline__ Slots block_slots(const int16_t* __restrict__ blk, int prev_dc, int comp, int lane) {
    const uint32_t* dc = TABLES.code[comp ? 2 : 0];
    const uint32_t* ac = TABLES.code[comp ? 3 : 1];
    const int v[2] = {blk[lane], blk[lane + 32]};
    // coefficients present, the DC slot counted as one so that a run starts after it
    const uint64_t present = __ballot_sync(0xffffffffu, v[0] != 0) | 1u | ((uint64_t)__ballot_sync(0xffffffffu, v[1] != 0) << 32);
    Slots s;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int k = lane + 32 * h;
        s.val[h] = 0, s.len[h] = 0;
        int cat;
        uint32_t extra;
        if (k == 0) {
            magnitude(v[0] - prev_dc, cat, extra);
            const uint32_t e = __ldg(dc + cat);
            s.val[h] = ((uint64_t)(e >> 8) << cat) | extra, s.len[h] = (int)(e & 255) + cat;
        } else if (v[h] != 0) {
            const int run = k - 1 - (63 - __clzll((long long)(present & ((1ull << k) - 1))));
            magnitude(v[h], cat, extra);
            const uint32_t e = __ldg(ac + (((run & 15) << 4) | cat)), zrl = __ldg(ac + 0xF0);
            s.val[h] = ((uint64_t)(e >> 8) << cat) | extra, s.len[h] = (int)(e & 255) + cat;
            for (int j = 0; j < (run >> 4); ++j) s.val[h] |= (uint64_t)(zrl >> 8) << s.len[h], s.len[h] += (int)(zrl & 255);
        } else if (k == 63) {
            const uint32_t e = __ldg(ac);
            s.val[h] = e >> 8, s.len[h] = (int)(e & 255);
        }
    }
    return s;
}

__device__ __forceinline__ int prev_dc_of(const int16_t* __restrict__ coef, int64_t mcu, int comp) {
    return mcu > 0 ? coef[((mcu - 1) * 3 + comp) * 64] : 0;
}

__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_scan_int(int v, int lane) {  // inclusive
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    return v;
}

__global__ void __launch_bounds__(JPEG_THREADS) k_jpeg_count(const int16_t* __restrict__ coef, int n_mcu,
                                                             uint32_t* __restrict__ bits) {
    const int lane = threadIdx.x & 31;
    const int mcu = blockIdx.x * JPEG_WARPS + (threadIdx.x >> 5);
    if (mcu >= n_mcu) return;
    int n = 0;
    for (int c = 0; c < 3; ++c) {
        const Slots s = block_slots(coef + ((int64_t)mcu * 3 + c) * 64, prev_dc_of(coef, mcu, c), c, lane);
        n += s.len[0] + s.len[1];
    }
    n = warp_sum_int(n);
    if (lane == 0) bits[mcu] = (uint32_t)n;
}

// out[i] = in[0] + .. + in[i - 1], *total = the sum of all n; one block, in and out may be the same array
__global__ void __launch_bounds__(SCAN_THREADS) k_jpeg_scan(const uint32_t* in, uint32_t* out, int n, uint32_t* total) {
    __shared__ uint32_t warp_tot[SCAN_THREADS / 32];
    const int per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
    const int lo = min(threadIdx.x * per, n), hi = min(lo + per, n);
    uint32_t mine = 0;
    for (int i = lo; i < hi; ++i) mine += in[i];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t incl = (uint32_t)warp_scan_int((int)mine, lane);
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    if (w == 0) {
        const uint32_t t = warp_tot[lane];
        warp_tot[lane] = (uint32_t)warp_scan_int((int)t, lane) - t;
    }
    __syncthreads();
    uint32_t run = warp_tot[w] + incl - mine;
    for (int i = lo; i < hi; ++i) {
        const uint32_t v = in[i];
        out[i] = run;
        run += v;
    }
    if (threadIdx.x == SCAN_THREADS - 1) *total = run;
}

// ORs the low `len` (< 64) bits of val into the stream at bit position pos, most significant bit first. The stream is
// addressed as 32-bit words holding their four bytes in stream order, hence the byte swap.
__device__ __forceinline__ void put_bits(uint32_t* __restrict__ stream, uint32_t pos, uint64_t val, int len) {
    if (len == 0) return;
    const uint64_t left = val << (64 - len);
    const int s = pos & 31;
    const uint64_t hi = left >> s;
    const uint32_t w[3] = {(uint32_t)(hi >> 32), (uint32_t)hi, s ? (uint32_t)((left << (64 - s)) >> 32) : 0u};
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (w[i]) atomicOr(stream + (pos >> 5) + i, __byte_perm(w[i], 0, 0x0123));
}

__global__ void __launch_bounds__(JPEG_THREADS) k_jpeg_emit(const int16_t* __restrict__ coef, int n_mcu,
                                                            const uint32_t* __restrict__ offs, const uint32_t* __restrict__ total,
                                                            uint32_t* __restrict__ stream) {
    const int lane = threadIdx.x & 31;
    const int mcu = blockIdx.x * JPEG_WARPS + (threadIdx.x >> 5);
    if (mcu >= n_mcu) return;
    uint32_t pos = offs[mcu];
    for (int c = 0; c < 3; ++c) {
        const Slots s = block_slots(coef + ((int64_t)mcu * 3 + c) * 64, prev_dc_of(coef, mcu, c), c, lane);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int incl = warp_scan_int(s.len[h], lane);
            put_bits(stream, pos + (uint32_t)(incl - s.len[h]), s.val[h], s.len[h]);
            pos += (uint32_t)__shfl_sync(0xffffffffu, incl, 31);
        }
    }
    const int pad = (int)(-*total & 7u);  // the last byte is filled with 1-bits
    if (mcu == n_mcu - 1 && lane == 0) put_bits(stream, pos, (1u << pad) - 1, pad);
}

// ---------------------------------------------------------------------------------------------------------------------
// byte stuffing and assembly
// ---------------------------------------------------------------------------------------------------------------------
// the number of 0xFF among the bytes [first, first + 16) of the stream that lie before n_bytes
__device__ __forceinline__ int count_ff(uint4 v, int64_t first, int64_t n_bytes) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int n = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) n += (first + i < n_bytes) && ((w[i >> 2] >> (8 * (i & 3))) & 255u) == 255u;
    return n;
}

__global__ void __launch_bounds__(JPEG_THREADS) k_jpeg_ff(const uint4* __restrict__ stream, const uint32_t* __restrict__ total,
                                                          int n_chunks, uint32_t* __restrict__ ff) {
    const int lane = threadIdx.x & 31;
    const int64_t n_bytes = ((int64_t)*total + 7) >> 3;
    for (int ch = blockIdx.x * JPEG_WARPS + (threadIdx.x >> 5); ch < n_chunks; ch += gridDim.x * JPEG_WARPS) {
        const int64_t first = (int64_t)ch * JPEG_CHUNK + lane * 16;
        int n = 0;
        if ((int64_t)ch * JPEG_CHUNK < n_bytes) n = warp_sum_int(count_ff(stream[first >> 4], first, n_bytes));
        if (lane == 0) ff[ch] = (uint32_t)n;
    }
}

__global__ void __launch_bounds__(JPEG_THREADS) k_jpeg_expand(const uint4* __restrict__ stream, const uint32_t* __restrict__ total,
                                                              int n_chunks, const uint32_t* __restrict__ ff_before,
                                                              const uint32_t* __restrict__ ff_total, int H, int W, int quality,
                                                              uint8_t* __restrict__ out, int64_t* __restrict__ out_len) {
    __shared__ uint8_t stage[JPEG_WARPS][2 * JPEG_CHUNK];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t n_bytes = ((int64_t)*total + 7) >> 3;
    if (blockIdx.x == 0) {
        for (int i = threadIdx.x; i < JPEG_HEAD; i += JPEG_THREADS) {
            int b = TABLES.head[i];
            for (int k = 0; k < 2; ++k)
                if (i >= TABLES.dqt[k] && i < TABLES.dqt[k] + 64) b = quant_entry(TABLES.q_base[k * 64 + TABLES.zigzag[i - TABLES.dqt[k]]], quality);
            const int s = i - TABLES.sof_size;
            if (s >= 0 && s < 4) b = ((s < 2 ? H : W) >> (s & 1 ? 0 : 8)) & 255;
            out[i] = (uint8_t)b;
        }
        if (threadIdx.x == 0) {
            const int64_t end = JPEG_HEAD + n_bytes + *ff_total;
            out[end] = 0xFF, out[end + 1] = 0xD9;
            *out_len = end + 2;
        }
    }
    for (int ch = blockIdx.x * JPEG_WARPS + w; ch < n_chunks; ch += gridDim.x * JPEG_WARPS) {
        const int64_t base = (int64_t)ch * JPEG_CHUNK;
        if (base >= n_bytes) break;
        const int64_t first = base + lane * 16;
        const uint4 v = stream[first >> 4];
        const int mine = count_ff(v, first, n_bytes);
        const int incl = warp_scan_int(mine, lane);
        int p = lane * 16 + incl - mine;
        const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const uint8_t b = (uint8_t)(wd[i >> 2] >> (8 * (i & 3)));
            if (first + i < n_bytes) {
                stage[w][p++] = b;
                if (b == 0xFF) stage[w][p++] = 0;
            }
        }
        const int n_out = (int)min((int64_t)JPEG_CHUNK, n_bytes - base) + __shfl_sync(0xffffffffu, incl, 31);
        __syncwarp();
        uint8_t* dst = out + JPEG_HEAD + base + ff_before[ch];
        for (int i = lane; i < n_out; i += 32) dst[i] = stage[w][i];
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// workspace layout
// ---------------------------------------------------------------------------------------------------------------------
struct JpegLayout {
    int mcus_x, n_mcu, n_chunks;
    int64_t stream_bytes;  // the largest unstuffed scan, a multiple of JPEG_CHUNK
    int64_t coef, bits, totals, stream, ff, total;
};

int64_t align256(int64_t x) { return (x + 255) & ~(int64_t)255; }

bool jpeg_layout(int H, int W, JpegLayout& y) {
    if (H < 1 || W < 1 || H > 65535 || W > 65535) return false;  // SOF0 holds the size in 16 bits
    const int64_t n_mcu = (int64_t)((H + 7) / 8) * ((W + 7) / 8);
    if (n_mcu * 3 * JPEG_BLOCK_BYTES * 8 > INT32_MAX) return false;  // bit offsets are 32-bit
    y.mcus_x = (W + 7) / 8, y.n_mcu = (int)n_mcu;
    // + 8: put_bits may touch (with zeros only) two words past the last code
    y.stream_bytes = (n_mcu * 3 * JPEG_BLOCK_BYTES + 8 + JPEG_CHUNK - 1) / JPEG_CHUNK * JPEG_CHUNK;
    y.n_chunks = (int)(y.stream_bytes / JPEG_CHUNK);
    y.coef = 0;
    y.bits = align256(n_mcu * 3 * 64 * 2);
    y.totals = y.bits + align256(n_mcu * 4);
    y.stream = y.totals + 256;
    y.ff = y.stream + align256(y.stream_bytes);
    y.total = y.ff + align256((int64_t)y.n_chunks * 4);
    return true;
}

}  // namespace

extern "C" size_t ngp_jpeg_workspace(int H, int W) {
    JpegLayout y;
    return jpeg_layout(H, W, y) ? (size_t)y.total : 0;
}

extern "C" size_t ngp_jpeg_capacity(int H, int W) {
    JpegLayout y;
    return jpeg_layout(H, W, y) ? (size_t)(JPEG_HEAD + 2 * (int64_t)y.n_mcu * 3 * JPEG_BLOCK_BYTES + 2) : 0;
}

extern "C" int ngp_jpeg_encode(const uint8_t* img, int H, int W, int quality, uint8_t* out, size_t out_capacity,
                               int64_t* out_len, void* workspace, size_t workspace_bytes, void* stream) {
    JpegLayout y;
    if (!jpeg_layout(H, W, y) || quality < 1 || quality > 100) return NGP_EINVAL;
    if (!ngp_dev_ptr(img, false) || !ngp_dev_ptr(workspace, false) || !ngp_dev_ptr(out, true) || !ngp_dev_ptr(out_len, true))
        return NGP_EINVAL;
    if (workspace_bytes < (size_t)y.total || out_capacity < ngp_jpeg_capacity(H, W) || ((uintptr_t)workspace & 255) ||
        ((uintptr_t)out_len & 7))
        return NGP_EINVAL;
    const cudaStream_t st = (cudaStream_t)stream;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    int16_t* coef = reinterpret_cast<int16_t*>(ws + y.coef);
    uint32_t* bits = reinterpret_cast<uint32_t*>(ws + y.bits);      // per MCU: coded bits, then bit offset
    uint32_t* totals = reinterpret_cast<uint32_t*>(ws + y.totals);  // [0] bits of the scan, [1] its 0xFF bytes
    uint32_t* bitstream = reinterpret_cast<uint32_t*>(ws + y.stream);
    uint32_t* ff = reinterpret_cast<uint32_t*>(ws + y.ff);          // per chunk: 0xFF bytes, then 0xFF bytes before it
    const int mcu_grid = ngp_div_up(y.n_mcu, JPEG_WARPS);
    const int chunk_grid = std::min(ngp_div_up(y.n_chunks, JPEG_WARPS), 8 * ngp_sm_count());
    NGP_CUDA(cudaMemsetAsync(bitstream, 0, (size_t)y.stream_bytes, st));
    k_jpeg_dct<<<ngp_div_up(y.n_mcu, JPEG_THREADS / 8), JPEG_THREADS, 0, st>>>(img, H, W, quality, y.mcus_x, y.n_mcu, coef);
    NGP_CHECK_LAUNCH();
    k_jpeg_count<<<mcu_grid, JPEG_THREADS, 0, st>>>(coef, y.n_mcu, bits);
    NGP_CHECK_LAUNCH();
    k_jpeg_scan<<<1, SCAN_THREADS, 0, st>>>(bits, bits, y.n_mcu, totals);
    NGP_CHECK_LAUNCH();
    k_jpeg_emit<<<mcu_grid, JPEG_THREADS, 0, st>>>(coef, y.n_mcu, bits, totals, bitstream);
    NGP_CHECK_LAUNCH();
    k_jpeg_ff<<<chunk_grid, JPEG_THREADS, 0, st>>>(reinterpret_cast<const uint4*>(bitstream), totals, y.n_chunks, ff);
    NGP_CHECK_LAUNCH();
    k_jpeg_scan<<<1, SCAN_THREADS, 0, st>>>(ff, ff, y.n_chunks, totals + 1);
    NGP_CHECK_LAUNCH();
    k_jpeg_expand<<<chunk_grid, JPEG_THREADS, 0, st>>>(reinterpret_cast<const uint4*>(bitstream), totals, y.n_chunks, ff,
                                                      totals + 1, H, W, quality, out, out_len);
    NGP_CHECK_LAUNCH();
    return 0;
}
