// Multiresolution hash-grid encoding (Instant-NGP), F = 2 features per level, fp16 table.
//
// The reference delegates this to tinycudann (reference models/networks.py:36-56), which is NOT in
// /root/reference. The arithmetic restated here is tiny-cuda-nn's published GridEncoding
// (SURVEY.md Appendix A, "[tcnn-memory]"; parity unpinned, see DESIGN.md):
//   scale_l = exp2f(l*log2f(b))*N_min - 1 ; res_l = ceil(scale_l)+1 ; entries_l = min(align8(res^3), T)
//   pos = fmaf(scale_l, x, 0.5) ; g = floor(pos) ; w = pos - g
//   index(p) = dense ? p.x + p.y*res + p.z*res^2 : p.x ^ p.y*2654435761 ^ p.z*805459861 ;  index %= entries_l
//   value = sum over the 8 corners of prod(w or 1-w) * table[offset_l + index]   (fp32 accumulate)
#pragma once
#include "common.cuh"
#include "../../include/ngp_b200.h"

__device__ __forceinline__ uint32_t grid_corner_index(uint32_t px, uint32_t py, uint32_t pz, uint32_t res,
                                                      uint32_t entries, bool hashed) {
    uint32_t idx;
    if (hashed) {
        idx = px ^ (py * 2654435761u) ^ (pz * 805459861u);
        // hashed levels always have 2^log2_T entries
        idx &= (entries - 1u);
    } else {
        idx = px + py * res + pz * res * res;
        // For inputs in [0,1]^3 only the +1 corner on the upper boundary can run past the level and
        // then idx < 2*entries, so one conditional subtract IS the modulo. The clamp keeps inputs from
        // outside the unit cube memory-safe (tiny-cuda-nn would wrap them with a true %).
        idx = idx >= entries ? idx - entries : idx;
        idx = min(idx, entries - 1u);
    }
    return idx;
}

struct GridCell {
    uint32_t gx, gy, gz;
    float wx, wy, wz;
};

__device__ __forceinline__ GridCell grid_cell(float x01, float y01, float z01, float scale) {
    GridCell c;
    float p, f;
    p = fmaf(scale, x01, 0.5f); f = floorf(p); c.gx = (uint32_t)(int)f; c.wx = p - f;
    p = fmaf(scale, y01, 0.5f); f = floorf(p); c.gy = (uint32_t)(int)f; c.wy = p - f;
    p = fmaf(scale, z01, 0.5f); f = floorf(p); c.gz = (uint32_t)(int)f; c.wz = p - f;
    return c;
}

// The 8 corner indices of a cell, k = dx + 2*dy + 4*dz. Same values as grid_corner_index() corner by corner, with the
// per-axis terms shared: hashed = two xors per corner (LOP3), dense = one 3-input add + the boundary wrap.
__device__ __forceinline__ void grid_corner_indices(const GridCell& c, uint32_t res, uint32_t entries, bool hashed,
                                                    uint32_t (&idx)[8]) {
    if (hashed) {
        const uint32_t mask = entries - 1u;  // hashed levels always have 2^log2_T entries
        const uint32_t x0 = c.gx, x1 = c.gx + 1u;
        const uint32_t y0 = c.gy * 2654435761u, y1 = y0 + 2654435761u;
        const uint32_t z0 = c.gz * 805459861u, z1 = z0 + 805459861u;
        const uint32_t t00 = y0 ^ z0, t10 = y1 ^ z0, t01 = y0 ^ z1, t11 = y1 ^ z1;
        idx[0] = (x0 ^ t00) & mask; idx[1] = (x1 ^ t00) & mask;
        idx[2] = (x0 ^ t10) & mask; idx[3] = (x1 ^ t10) & mask;
        idx[4] = (x0 ^ t01) & mask; idx[5] = (x1 ^ t01) & mask;
        idx[6] = (x0 ^ t11) & mask; idx[7] = (x1 ^ t11) & mask;
    } else {
        const uint32_t r2 = res * res;
        const uint32_t b00 = c.gx + c.gy * res + c.gz * r2;
        const uint32_t b10 = b00 + res, b01 = b00 + r2, b11 = b10 + r2;
        const uint32_t last = entries - 1u;
        uint32_t v;
        // one conditional subtract IS the modulo for inputs in the unit cube; the clamp keeps outside inputs memory-safe
#define NGP_WRAP(dst, val) v = (val); v = v >= entries ? v - entries : v; dst = min(v, last)
        NGP_WRAP(idx[0], b00); NGP_WRAP(idx[1], b00 + 1u);
        NGP_WRAP(idx[2], b10); NGP_WRAP(idx[3], b10 + 1u);
        NGP_WRAP(idx[4], b01); NGP_WRAP(idx[5], b01 + 1u);
        NGP_WRAP(idx[6], b11); NGP_WRAP(idx[7], b11 + 1u);
#undef NGP_WRAP
    }
}

// the 8 trilinear weights, k = dx + 2*dy + 4*dz (same products as ((k&1)?wx:1-wx) * ((k&2)?wy:1-wy) * ((k&4)?wz:1-wz))
__device__ __forceinline__ void grid_corner_weights(const GridCell& c, float (&w)[8]) {
    const float ux = 1.0f - c.wx, uy = 1.0f - c.wy, uz = 1.0f - c.wz;
    const float a00 = ux * uy, a10 = c.wx * uy, a01 = ux * c.wy, a11 = c.wx * c.wy;
    w[0] = a00 * uz; w[1] = a10 * uz; w[2] = a01 * uz; w[3] = a11 * uz;
    w[4] = a00 * c.wz; w[5] = a10 * c.wz; w[6] = a01 * c.wz; w[7] = a11 * c.wz;
}

// base + idx * BYTES as ONE IMAD.WIDE.U32 (the compiler otherwise folds the level offset back into a 64-bit add chain:
// four instructions per corner)
template <int BYTES>
__device__ __forceinline__ const void* entry_ptr(const void* base, uint32_t idx) {
    uint64_t a;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(a) : "r"(idx), "n"(BYTES), "l"((uint64_t)base));
    return (const void*)a;
}

// Trilinear lookup of one (sample, level): 8 independent 4-byte gathers, then 8 FMAs per feature.
__device__ __forceinline__ float2 grid_lookup(const uint32_t* __restrict__ table /* half2 per entry */,
                                              const NgpGridMeta& m, int level, float x01, float y01, float z01) {
    const uint32_t res = m.res[level];
    const uint32_t off = m.offset[level];
    const uint32_t entries = m.offset[level + 1] - off;
    const bool hashed = (m.hashed_mask >> level) & 1u;
    const GridCell c = grid_cell(x01, y01, z01, m.scale[level]);
    uint32_t idx[8], v[8];
    grid_corner_indices(c, res, entries, hashed, idx);
    const uint32_t* lvl = table + off;
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __ldg(reinterpret_cast<const uint32_t*>(entry_ptr<4>(lvl, idx[k])));
    float w[8];
    grid_corner_weights(c, w);
    float f0 = 0.f, f1 = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float2 t = unpack_half2(v[k]);
        f0 = fmaf(w[k], t.x, f0);
        f1 = fmaf(w[k], t.y, f1);
    }
    return make_float2(f0, f1);
}

// The two x-corners of a cell (k, k+1) sit in ONE aligned entry pair whenever their indices differ only in bit 0: for a
// hashed level whenever gx is even ((x ^ t) and ((x+1) ^ t)), for a dense level whenever the first index is even (and the
// pair does not straddle the wrap). The scatter uses that: one 16-byte red.global.add.v4.f32 instead of two 8-byte ones
// (one L2 atomic transaction). The same trick in the GATHER (aligned 8-byte pair load + predicated load of the unpaired
// corner) and a software-pipelined gather were slower than the plain eight 4-byte loads and are not kept.
// the corner contributions acc[2k], acc[2k+1] of one cell that the bit mask `own` selects into the gradient table of a
// level, x-pairs merged when both are owned and aligned
__device__ __forceinline__ void grid_scatter_cell_owned(const float* lvl /* level base, float2 per entry */, const uint32_t (&idx)[8],
                                                        const float (&acc)[16], uint32_t own) {
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
        const bool o0 = (own >> k) & 1u, o1 = (own >> (k + 1)) & 1u;
        if (o0 && o1 && (idx[k] ^ idx[k + 1]) == 1u) {
            float* p = const_cast<float*>(reinterpret_cast<const float*>(entry_ptr<8>(lvl, idx[k] & ~1u)));
            if (idx[k] & 1u) red_add_f32x4(p, acc[2 * k + 2], acc[2 * k + 3], acc[2 * k], acc[2 * k + 1]);
            else red_add_f32x4(p, acc[2 * k], acc[2 * k + 1], acc[2 * k + 2], acc[2 * k + 3]);
        } else {
            if (o0)
                red_add_f32x2(const_cast<float*>(reinterpret_cast<const float*>(entry_ptr<8>(lvl, idx[k]))), acc[2 * k], acc[2 * k + 1]);
            if (o1)
                red_add_f32x2(const_cast<float*>(reinterpret_cast<const float*>(entry_ptr<8>(lvl, idx[k + 1]))), acc[2 * k + 2],
                              acc[2 * k + 3]);
        }
    }
}

// Corners two cells share. Corner k = dx + 2*dy + 4*dz of cell c is the grid vertex c + (dx, dy, dz); if the cell
// c + d is adjacent (every |d_i| <= 1), that vertex is its corner k - (d.x + 2*d.y + 4*d.z) whenever every component of
// k - d stays in {0, 1}. The bit mask of those k (in c's numbering): along an axis with d_i = +1 only the upper corners are
// shared, with d_i = -1 only the lower ones, with d_i = 0 both. A shared vertex has one table entry on every level:
// the hash and the dense wrap and clamp are functions of the vertex alone (grid_corner_indices).
__device__ __forceinline__ uint32_t grid_shared_corners(int dx, int dy, int dz) {
    const uint32_t mx = dx > 0 ? 0xAAu : dx < 0 ? 0x55u : 0xFFu;
    const uint32_t my = dy > 0 ? 0xCCu : dy < 0 ? 0x33u : 0xFFu;
    const uint32_t mz = dz > 0 ? 0xF0u : dz < 0 ? 0x0Fu : 0xFFu;
    return mx & my & mz;
}

__device__ __forceinline__ bool grid_cells_adjacent(int dx, int dy, int dz) {
    return (unsigned)(dx + 1) <= 2u && (unsigned)(dy + 1) <= 2u && (unsigned)(dz + 1) <= 2u;
}

// Scatter of one (sample, level) gradient into the fp32 gradient table: 8 vector reductions of 8 B.
__device__ __forceinline__ void grid_scatter(float* __restrict__ grad /* float2 per entry */, const NgpGridMeta& m, int level,
                                             float x01, float y01, float z01, float g0, float g1) {
    const uint32_t res = m.res[level];
    const uint32_t off = m.offset[level];
    const uint32_t entries = m.offset[level + 1] - off;
    const bool hashed = (m.hashed_mask >> level) & 1u;
    const GridCell c = grid_cell(x01, y01, z01, m.scale[level]);
    uint32_t idx[8];
    grid_corner_indices(c, res, entries, hashed, idx);
    float w[8];
    grid_corner_weights(c, w);
    const float* lvl = grad + 2 * (size_t)off;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        red_add_f32x2(const_cast<float*>(reinterpret_cast<const float*>(entry_ptr<8>(lvl, idx[k]))), w[k] * g0, w[k] * g1);
}

// Degree-4 real spherical harmonics of a unit vector (16 coefficients), tiny-cuda-nn's ordering and
// constants (SURVEY.md Appendix A).
__device__ __forceinline__ void sh4(float x, float y, float z, float* __restrict__ o) {
    const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}
