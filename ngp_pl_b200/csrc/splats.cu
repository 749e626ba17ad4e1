// Gaussian-splat export (include/ngp_b200.h, "Gaussian-splat export"; numpy restatement: oracle/splats_ref.py).
//
// colours : the hash grid and density MLP run once per point (ngp_net_forward, want_rgb 0, h kept), then one warp per
//           16 (point, direction) rows runs the network core's colour chain (network.cuh: color_input, color_mlp,
//           rgb_out) on mma.sync with the point's h fragment read back from global memory: the colour of a row is the
//           one ngp_net_forward computes for the same (p, d), bit for bit.
// fit     : one warp per point. Lane l owns row l / 2 of the 16 x 16 Gram matrix (eight columns) and that row of the
//           three right-hand sides; the directions are visited in order (fixed-order double sums), then a right-looking
//           Cholesky over the warp in shared memory and one lane per channel substitutes.
// geometry: one thread per point; the scale, the shortest-arc quaternion and the opacity, in double.
// render  : 3DGS's forward rasteriser: project + cull + EWA covariance per splat, a scan of the tiles each touches,
//           (tile, depth) keys radix-sorted, per-tile ranges, and one 16 x 16 block per tile blending front to back. The
//           key capacity is fixed per call (no read-back), so the whole chain can be captured in a CUDA graph.
// No float atomics anywhere: two calls are bitwise equal.
#include "network.cuh"
#include "../../include/ngp_b200.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define SPL_THREADS 256
#define SPL_MIN_BLOCKS 3
#define FIT_WARPS 8
#define SPL_TILE 16
#define SPL_MAX_ITEMS ((int64_t)1 << 31)

static size_t spl_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int spl_grid(int64_t items, int threads, int per_sm) {
    const int64_t want = (items + threads - 1) / threads, cap = (int64_t)ngp_sm_count() * per_sm;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

// ---- 1. colours over directions ---------------------------------------------------------------------------------------
struct SplDir {
    float dx, dy, dz;
};

__global__ void __launch_bounds__(SPL_THREADS, SPL_MIN_BLOCKS)
k_splat_colors(const NgpNet net, const uint32_t* __restrict__ h, int64_t n_points, const float* __restrict__ dirs,
               int n_dirs, __half* __restrict__ rgb) {
    __shared__ __align__(16) MlpWeightsFwd sw;
    load_weights_fwd(sw, reinterpret_cast<const __half*>(net.enc_params_h), reinterpret_cast<const __half*>(net.rgb_params_h),
                     threadIdx.x, SPL_THREADS);
    __syncthreads();
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int64_t n = n_points * n_dirs, n_tiles = (n + 15) / 16;
    const int64_t n_warps = (int64_t)gridDim.x * (SPL_THREADS / 32);
    for (int64_t tile = (int64_t)blockIdx.x * (SPL_THREADS / 32) + (threadIdx.x >> 5); tile < n_tiles; tile += n_warps) {
        SplDir s[1][2];
        uint32_t hA[1][1][4];
        bool valid[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int64_t row = tile * 16 + g + 8 * hh;
            valid[hh] = row < n;
            const int64_t p = valid[hh] ? row / n_dirs : 0;
            const int j = valid[hh] ? (int)(row - p * n_dirs) : 0;
            s[0][hh].dx = __ldg(dirs + 3 * j);
            s[0][hh].dy = __ldg(dirs + 3 * j + 1);
            s[0][hh].dz = __ldg(dirs + 3 * j + 2);
            // the h fragment words k_ngp_fwd holds for this row: columns 2q..2q+1 and 2q+8..2q+9
            hA[0][0][hh] = __ldg(h + 8 * p + q);
            hA[0][0][2 + hh] = __ldg(h + 8 * p + 4 + q);
        }
        uint32_t inA[1][2][4];
        color_input<1>(s, hA, q, inA);
        float oC[1][1][4];
        color_mlp<1>(inA, sw.w1r, sw.w2r, sw.w3r, oC, g, q, [](int, const auto&) {});
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int64_t row = tile * 16 + g + 8 * hh;
            if (!valid[hh] || q > 1) continue;
            const __half2 o = rgb_out(oC[0][0][2 * hh], oC[0][0][2 * hh + 1], net.rgb_act);
            if (q == 0) {
                rgb[3 * row] = __low2half(o);
                rgb[3 * row + 1] = __high2half(o);
            } else {
                rgb[3 * row + 2] = __low2half(o);
            }
        }
    }
}

extern "C" int ngp_splat_colors(const NgpNet* net, const float* points, int64_t n_points, const float* dirs, int n_dirs,
                                float* sigma, uint16_t* h, uint16_t* rgb, void* stream) {
    if (!net || !net->enc_params_h || !net->rgb_params_h || !points || !dirs || !sigma || !h || !rgb) return NGP_EINVAL;
    if (n_points < 0 || n_points >= SPL_MAX_ITEMS || n_dirs < NGP_SPLAT_MIN_DIRS || n_dirs > NGP_SPLAT_MAX_DIRS)
        return NGP_EINVAL;
    if (n_points == 0) return 0;
    NgpSamples smp = {};
    smp.xyzs = points;
    smp.n = n_points;
    const int rc = ngp_net_forward(net, &smp, 0, sigma, nullptr, h, nullptr, stream);
    if (rc) return rc;
    const int64_t n_tiles = (n_points * n_dirs + 15) / 16;
    k_splat_colors<<<spl_grid(n_tiles, SPL_THREADS / 32, SPL_MIN_BLOCKS), SPL_THREADS, 0, (cudaStream_t)stream>>>(
        *net, reinterpret_cast<const uint32_t*>(h), n_points, dirs, n_dirs, reinterpret_cast<__half*>(rgb));
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---- 2. SH fit ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FIT_WARPS * 32)
k_splat_fit(const __half* __restrict__ rgb, int64_t n_points, int n_dirs, const float* __restrict__ dirs,
            const double* __restrict__ basis, const float* __restrict__ normals, int nb, double ridge, float* __restrict__ out) {
    __shared__ double sA[FIT_WARPS][16][17];
    __shared__ double sB[FIT_WARPS][3][16];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int r = lane >> 1, c0 = 8 * (lane & 1);
    double(&A)[16][17] = sA[w];
    double(&B)[3][16] = sB[w];
    for (int64_t p = (int64_t)blockIdx.x * FIT_WARPS + w; p < n_points; p += (int64_t)gridDim.x * FIT_WARPS) {
        double nx = 0.0, ny = 0.0, nz = 0.0;
        if (normals) {
            nx = normals[3 * p];
            ny = normals[3 * p + 1];
            nz = normals[3 * p + 2];
        }
        const bool hemi = nx != 0.0 || ny != 0.0 || nz != 0.0;
        double G[8], b[3], wsum = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) G[k] = 0.0;
        b[0] = b[1] = b[2] = 0.0;
        const __half* cp = rgb + p * n_dirs * 3;
        for (int j0 = 0; j0 < n_dirs; j0 += 32) {
            const int j = j0 + lane;
            double wj = 0.0, cj[3] = {0.0, 0.0, 0.0};
            if (j < n_dirs) {
                wj = 1.0;
                if (hemi) {
                    const double dn = __dadd_rn(__dadd_rn(__dmul_rn((double)dirs[3 * j], nx), __dmul_rn((double)dirs[3 * j + 1], ny)),
                                                __dmul_rn((double)dirs[3 * j + 2], nz));
                    wj = dn < 0.0 ? -dn : 0.0;
                }
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) cj[ch] = (double)__half2float(cp[3 * j + ch]) - 0.5;
            }
            const int m = n_dirs - j0 < 32 ? n_dirs - j0 : 32;
            for (int t = 0; t < m; ++t) {
                const double wt = __shfl_sync(0xffffffffu, wj, t);
                const double e0 = __shfl_sync(0xffffffffu, cj[0], t), e1 = __shfl_sync(0xffffffffu, cj[1], t),
                             e2 = __shfl_sync(0xffffffffu, cj[2], t);
                if (wt == 0.0) continue;  // warp-uniform
                const double* y = basis + (int64_t)(j0 + t) * 16;
                const double yr = __ldg(y + r) * wt;
#pragma unroll
                for (int k = 0; k < 8; ++k) G[k] += yr * __ldg(y + c0 + k);
                b[0] += yr * e0;
                b[1] += yr * e1;
                b[2] += yr * e2;
                wsum += wt;
            }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) A[r][c0 + k] = G[k] + (r == c0 + k ? ridge * wsum : 0.0);
        if (c0 == 0)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) B[ch][r] = b[ch];
        __syncwarp();
        // right-looking Cholesky of the leading nb x nb block, lower triangle in place; a pivot at most
        // NGP_SPLAT_PIVOT_RTOL times the largest diagonal entry marks it singular (rounding leaves a rank-deficient
        // block tiny positive pivots, whose solve would be huge)
        double dmax = lane < nb ? A[lane][lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
        const double tiny = NGP_SPLAT_PIVOT_RTOL * dmax;
        bool ok = dmax > 0.0;
        for (int k = 0; k < nb; ++k) {
            const double piv = A[k][k];
            ok = ok && piv > tiny;
            const double d = ok ? sqrt(piv) : 1.0;
            __syncwarp();
            if (lane > k && lane < nb) A[lane][k] /= d;
            if (lane == k) A[k][k] = d;
            __syncwarp();
            for (int e = lane; e < 256; e += 32) {
                const int i = e >> 4, jj = e & 15;
                if (i > k && jj > k && jj <= i && i < nb) A[i][jj] -= A[i][k] * A[jj][k];
            }
            __syncwarp();
        }
        if (lane < 3) {
            double* x = B[lane];
            for (int i = 0; i < nb; ++i) {
                double v = x[i];
                for (int k = 0; k < i; ++k) v -= A[i][k] * x[k];
                x[i] = v / A[i][i];
            }
            for (int i = nb - 1; i >= 0; --i) {
                double v = x[i];
                for (int k = i + 1; k < nb; ++k) v -= A[k][i] * x[k];
                x[i] = v / A[i][i];
            }
        }
        __syncwarp();
        for (int e = lane; e < 48; e += 32) {
            const int ch = e >> 4, k = e & 15;
            const float v = (ok && k < nb) ? (float)B[ch][k] : 0.f;
            out[p * NGP_SPLAT_FLOATS + (k == 0 ? NGP_SPLAT_F_DC + ch : NGP_SPLAT_F_REST + 15 * ch + k - 1)] = v;
        }
        __syncwarp();
    }
}

extern "C" int ngp_splat_fit(const uint16_t* rgb, int64_t n_points, int n_dirs, const float* dirs, const double* basis,
                             const float* normals, int degree, double ridge, float* splats, void* stream) {
    if (!rgb || !dirs || !basis || !splats || n_points < 0 || n_points >= SPL_MAX_ITEMS || n_dirs < NGP_SPLAT_MIN_DIRS ||
        n_dirs > NGP_SPLAT_MAX_DIRS || degree < 0 || degree > 3 || !(ridge >= 0.0) || !isfinite(ridge))
        return NGP_EINVAL;
    if (n_points == 0) return 0;
    k_splat_fit<<<spl_grid(n_points, FIT_WARPS, 16), FIT_WARPS * 32, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __half*>(rgb), n_points, n_dirs, dirs, basis, normals, (degree + 1) * (degree + 1), ridge,
        splats);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---- 3. geometry and opacity ------------------------------------------------------------------------------------------------
__global__ void k_splat_geometry(const float* __restrict__ points, const float* __restrict__ normals,
                                 const float* __restrict__ sigma, const double* __restrict__ dist2, int k, int64_t n,
                                 int disc, float flatness, float* __restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float* o = out + i * NGP_SPLAT_FLOATS;
        double nv[3] = {0.0, 0.0, 0.0};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            o[a] = points[3 * i + a];
            const float f = normals ? normals[3 * i + a] : 0.f;
            o[3 + a] = f;
            nv[a] = f;
        }
        // s = sqrt(max(mean of the first min(k, 3) squared distances, 1e-7)), summed left to right
        const int kk = k < 3 ? k : 3;
        double m = 0.0;
        for (int a = 0; a < kk; ++a) m = __dadd_rn(m, dist2[i * k + a]);
        if (kk > 0) m = __ddiv_rn(m, (double)kk);
        const double s = __dsqrt_rn(m > 1e-7 ? m : 1e-7);
        double qw = 1.0, qx = 0.0, qy = 0.0, qz = 0.0, s_n = s;
        const bool has_n = nv[0] != 0.0 || nv[1] != 0.0 || nv[2] != 0.0;
        if (disc && has_n) {
            const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nv[0], nv[0]), __dmul_rn(nv[1], nv[1])),
                                                    __dmul_rn(nv[2], nv[2])));
            const double ux = __ddiv_rn(nv[0], len), uy = __ddiv_rn(nv[1], len), uz = __ddiv_rn(nv[2], len);
            // shortest arc z -> u: (1 + u.z, z x u) normalised; u = -z exactly: a half turn about x
            const double w = __dadd_rn(1.0, uz), x = -uy, y = ux;
            const double nq = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(w, w), __dmul_rn(x, x)), __dmul_rn(y, y)));
            if (nq > 0.0) {
                qw = __ddiv_rn(w, nq);
                qx = __ddiv_rn(x, nq);
                qy = __ddiv_rn(y, nq);
            } else {
                qw = 0.0;
                qx = 1.0;
                qy = 0.0;
            }
            s_n = __dmul_rn((double)flatness, s);
        }
        double alpha = 1.0 - exp(-(double)sigma[i] * 2.0 * s);
        alpha = alpha < 0.01 ? 0.01 : (alpha > 0.99 ? 0.99 : alpha);  // NaN (sigma inf * 0) cannot occur: s > 0
        o[NGP_SPLAT_OPACITY] = (float)log(alpha / (1.0 - alpha));
        const double ls = log(s);
        o[NGP_SPLAT_SCALE] = (float)ls;
        o[NGP_SPLAT_SCALE + 1] = (float)ls;
        o[NGP_SPLAT_SCALE + 2] = (float)log(s_n);
        o[NGP_SPLAT_ROT] = (float)qw;
        o[NGP_SPLAT_ROT + 1] = (float)qx;
        o[NGP_SPLAT_ROT + 2] = (float)qy;
        o[NGP_SPLAT_ROT + 3] = (float)qz;
    }
}

extern "C" int ngp_splat_geometry(const float* points, const float* normals, const float* sigma, const double* dist2, int k,
                                  int64_t n_points, int shape, float flatness, float* splats, void* stream) {
    if (!points || !sigma || !splats || n_points < 0 || n_points >= SPL_MAX_ITEMS || k < 0 || k > NGP_POINTS_MAX_K ||
        (k > 0 && !dist2) || (shape != NGP_SPLAT_SPHERE && shape != NGP_SPLAT_DISC) || !(flatness > 0.f) ||
        !isfinite(flatness))
        return NGP_EINVAL;
    if (n_points == 0) return 0;
    k_splat_geometry<<<spl_grid(n_points, 256, 16), 256, 0, (cudaStream_t)stream>>>(points, normals, sigma, dist2, k, n_points,
                                                                                   shape == NGP_SPLAT_DISC, flatness, splats);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---- 4. rasteriser ------------------------------------------------------------------------------------------------------------
#define SH_C0 0.28209479177387814f
#define SH_C1 0.4886025119029199f
__constant__ float c_sh_c2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                                 0.5462742152960396f};
__constant__ float c_sh_c3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                                 -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

// coefficient k of channel ch of splat g
__device__ __forceinline__ float sh_coef(const float* __restrict__ g, int ch, int k) {
    return k == 0 ? g[NGP_SPLAT_F_DC + ch] : g[NGP_SPLAT_F_REST + 15 * ch + k - 1];
}

// 3DGS's computeColorFromSH at degree 3 (coefficients above the file's degree are 0), + 0.5, clamped at 0
__device__ float sh_color(const float* __restrict__ g, int ch, float x, float y, float z) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    float r = SH_C0 * sh_coef(g, ch, 0);
    r = r - SH_C1 * y * sh_coef(g, ch, 1) + SH_C1 * z * sh_coef(g, ch, 2) - SH_C1 * x * sh_coef(g, ch, 3);
    r = r + c_sh_c2[0] * xy * sh_coef(g, ch, 4) + c_sh_c2[1] * yz * sh_coef(g, ch, 5) +
        c_sh_c2[2] * (2.0f * zz - xx - yy) * sh_coef(g, ch, 6) + c_sh_c2[3] * xz * sh_coef(g, ch, 7) +
        c_sh_c2[4] * (xx - yy) * sh_coef(g, ch, 8);
    r = r + c_sh_c3[0] * y * (3.0f * xx - yy) * sh_coef(g, ch, 9) + c_sh_c3[1] * xy * z * sh_coef(g, ch, 10) +
        c_sh_c3[2] * y * (4.0f * zz - xx - yy) * sh_coef(g, ch, 11) +
        c_sh_c3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh_coef(g, ch, 12) +
        c_sh_c3[4] * x * (4.0f * zz - xx - yy) * sh_coef(g, ch, 13) + c_sh_c3[5] * z * (xx - yy) * sh_coef(g, ch, 14) +
        c_sh_c3[6] * x * (xx - 3.0f * yy) * sh_coef(g, ch, 15);
    return fmaxf(r + 0.5f, 0.f);
}

struct SplWs {
    float2* xy;
    float4* conic;  // conic a, b, c and opacity
    float* rgb;     // 3 per splat
    float* depth;
    int4* rect;
    int64_t* touched;  // inclusive scan in place
    uint64_t* key[2];
    int32_t* val[2];
    int2* ranges;
    void* temp;
    size_t temp_bytes, total;
};

static size_t spl_temp_bytes(int64_t n, int64_t cap, int end_bit) {
    size_t t = 0, tb = 0;
    cub::DeviceScan::InclusiveSum(nullptr, t, (int64_t*)nullptr, (int64_t*)nullptr, (int)(n > 0 ? n : 1));
    tb = t;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v(nullptr, nullptr);
    t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, k, v, (int)(cap > 0 ? cap : 1), 0, end_bit);
    return t > tb ? t : tb;
}

static int spl_bits(uint64_t x) {  // bits that hold 0..x, at least 1
    int b = 1;
    while (b < 64 && (x >> b)) ++b;
    return b;
}

static SplWs spl_layout(char* base, int64_t n, int W, int H, int64_t cap) {
    SplWs w = {};
    const int64_t n_tiles = (int64_t)((W + SPL_TILE - 1) / SPL_TILE) * ((H + SPL_TILE - 1) / SPL_TILE);
    const int end_bit = 32 + spl_bits((uint64_t)n_tiles);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* p = base ? base + off : nullptr;
        off += spl_align(bytes);
        return p;
    };
    w.xy = (float2*)take(8 * (size_t)n);
    w.conic = (float4*)take(16 * (size_t)n);
    w.rgb = (float*)take(12 * (size_t)n);
    w.depth = (float*)take(4 * (size_t)n);
    w.rect = (int4*)take(16 * (size_t)n);
    w.touched = (int64_t*)take(8 * (size_t)n);
    for (int b = 0; b < 2; ++b) {
        w.key[b] = (uint64_t*)take(8 * (size_t)cap);
        w.val[b] = (int32_t*)take(4 * (size_t)cap);
    }
    w.ranges = (int2*)take(8 * (size_t)n_tiles);
    w.temp_bytes = spl_temp_bytes(n, cap, end_bit);
    w.temp = take(w.temp_bytes);
    w.total = off;
    return w;
}

static bool spl_sizes_ok(int64_t n, int W, int H, int64_t cap) {
    return n >= 0 && n < SPL_MAX_ITEMS && W >= 1 && H >= 1 && W <= NGP_SPLAT_MAX_SIDE && H <= NGP_SPLAT_MAX_SIDE &&
           cap >= 1 && cap < SPL_MAX_ITEMS;
}

extern "C" size_t ngp_splat_render_workspace(int64_t n_splats, int W, int H, int64_t capacity) {
    if (!spl_sizes_ok(n_splats, W, H, capacity)) return 0;
    return spl_layout(nullptr, n_splats, W, H, capacity).total;
}

// view: pose (3 x 4, row-major R | o), fx, fy, cx, cy, bg (3)
__global__ void k_splat_project(const float* __restrict__ splats, int64_t n, const float* __restrict__ view, int W, int H,
                                int gx, int gy, SplWs w) {
    __shared__ float v[NGP_SPLAT_VIEW_FLOATS];
    if (threadIdx.x < NGP_SPLAT_VIEW_FLOATS) v[threadIdx.x] = view[threadIdx.x];
    __syncthreads();
    const float fx = v[12], fy = v[13], cx = v[14], cy = v[15];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float* g = splats + i * NGP_SPLAT_FLOATS;
        w.touched[i] = 0;
        const float d0 = g[0] - v[3], d1 = g[1] - v[7], d2 = g[2] - v[11];
        // camera frame: R^T (p - o)
        const float xc = v[0] * d0 + v[4] * d1 + v[8] * d2;
        const float yc = v[1] * d0 + v[5] * d1 + v[9] * d2;
        const float zc = v[2] * d0 + v[6] * d1 + v[10] * d2;
        if (!(zc > 0.2f)) continue;
        // world covariance R_q diag(s^2) R_q^T
        float qw = g[NGP_SPLAT_ROT], qx = g[NGP_SPLAT_ROT + 1], qy = g[NGP_SPLAT_ROT + 2], qz = g[NGP_SPLAT_ROT + 3];
        const float qn = sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
        if (!(qn > 0.f)) continue;
        qw /= qn; qx /= qn; qy /= qn; qz /= qn;
        const float Rq[3][3] = {{1.f - 2.f * (qy * qy + qz * qz), 2.f * (qx * qy - qw * qz), 2.f * (qx * qz + qw * qy)},
                                {2.f * (qx * qy + qw * qz), 1.f - 2.f * (qx * qx + qz * qz), 2.f * (qy * qz - qw * qx)},
                                {2.f * (qx * qz - qw * qy), 2.f * (qy * qz + qw * qx), 1.f - 2.f * (qx * qx + qy * qy)}};
        float s2[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float s = expf(g[NGP_SPLAT_SCALE + a]);
            s2[a] = s * s;
        }
        float S[3][3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) S[a][b] = Rq[a][0] * s2[0] * Rq[b][0] + Rq[a][1] * s2[1] * Rq[b][1] + Rq[a][2] * s2[2] * Rq[b][2];
        // EWA: J at the point with x/z, y/z clamped to 1.3 x the half field of view; T = J W with W = R^T
        const float limx = 1.3f * (0.5f * W / fx), limy = 1.3f * (0.5f * H / fy);
        const float tx = fminf(limx, fmaxf(-limx, xc / zc)) * zc, ty = fminf(limy, fmaxf(-limy, yc / zc)) * zc;
        const float j00 = fx / zc, j02 = -(fx * tx) / (zc * zc), j11 = fy / zc, j12 = -(fy * ty) / (zc * zc);
        float T[2][3];
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            T[0][b] = j00 * v[4 * b] + j02 * v[4 * b + 2];
            T[1][b] = j11 * v[4 * b + 1] + j12 * v[4 * b + 2];
        }
        float TS[2][3];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) TS[a][b] = T[a][0] * S[0][b] + T[a][1] * S[1][b] + T[a][2] * S[2][b];
        const float ca = TS[0][0] * T[0][0] + TS[0][1] * T[0][1] + TS[0][2] * T[0][2] + 0.3f;
        const float cb = TS[0][0] * T[1][0] + TS[0][1] * T[1][1] + TS[0][2] * T[1][2];
        const float cc = TS[1][0] * T[1][0] + TS[1][1] * T[1][1] + TS[1][2] * T[1][2] + 0.3f;
        const float det = ca * cc - cb * cb;
        if (!(det > 0.f)) continue;
        const float det_inv = 1.f / det;
        const float mid = 0.5f * (ca + cc);
        const float l1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det)), l2 = mid - sqrtf(fmaxf(0.1f, mid * mid - det));
        const float radius = ceilf(3.f * sqrtf(fmaxf(l1, l2)));
        const float px = fx * xc / zc + cx - 0.5f, py = fy * yc / zc + cy - 0.5f;
        int4 rc;
        rc.x = min(gx, max(0, (int)((px - radius) / SPL_TILE)));
        rc.y = min(gy, max(0, (int)((py - radius) / SPL_TILE)));
        rc.z = min(gx, max(0, (int)((px + radius + SPL_TILE - 1) / SPL_TILE)));
        rc.w = min(gy, max(0, (int)((py + radius + SPL_TILE - 1) / SPL_TILE)));
        const int64_t tiles = (int64_t)(rc.z - rc.x) * (rc.w - rc.y);
        if (tiles == 0) continue;
        const float inv = 1.f / sqrtf(d0 * d0 + d1 * d1 + d2 * d2);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) w.rgb[3 * i + ch] = sh_color(g, ch, d0 * inv, d1 * inv, d2 * inv);
        w.xy[i] = make_float2(px, py);
        w.conic[i] = make_float4(cc * det_inv, -cb * det_inv, ca * det_inv, 1.f / (1.f + expf(-g[NGP_SPLAT_OPACITY])));
        w.depth[i] = zc;
        w.rect[i] = rc;
        w.touched[i] = tiles;
    }
}

// after the inclusive scan of touched: splat i's keys go to slots [touched[i] - tiles, touched[i]), those below cap
// (the count is written by one thread on its own: a thread whose splat runs past cap still takes its later splats)
__global__ void k_splat_keys(int64_t n, int64_t cap, int gx, SplWs w, int64_t* __restrict__ n_keys) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_keys = w.touched[n - 1];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t end = w.touched[i], start = i ? w.touched[i - 1] : 0;
        if (end == start || start >= cap) continue;
        const int4 rc = w.rect[i];
        const uint64_t dk = __float_as_uint(w.depth[i]);
        int64_t s = start;
        for (int y = rc.y; y < rc.w && s < cap; ++y)
            for (int x = rc.x; x < rc.z && s < cap; ++x, ++s) {
                w.key[0][s] = ((uint64_t)(y * gx + x) << 32) | dk;
                w.val[0][s] = (int32_t)i;
            }
    }
}

__global__ void k_splat_ranges(const uint64_t* __restrict__ keys, int64_t cap, const int64_t* __restrict__ n_keys,
                               int64_t n_tiles, int2* __restrict__ ranges) {
    const int64_t m = *n_keys < cap ? *n_keys : cap;
    for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < m; s += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = (int64_t)(keys[s] >> 32);
        if (t >= n_tiles) continue;
        if (s == 0 || (int64_t)(keys[s - 1] >> 32) != t) ranges[t].x = (int)s;
        if (s == m - 1 || (int64_t)(keys[s + 1] >> 32) != t) ranges[t].y = (int)s + 1;
    }
}

#define BLEND_THREADS (SPL_TILE * SPL_TILE)
__global__ void __launch_bounds__(BLEND_THREADS)
k_splat_blend(const int2* __restrict__ ranges, const int32_t* __restrict__ vals, SplWs w, int W, int H, int gx,
              const float* __restrict__ view, float* __restrict__ out_rgb, float* __restrict__ out_op) {
    __shared__ int32_t s_id[BLEND_THREADS];
    __shared__ float2 s_xy[BLEND_THREADS];
    __shared__ float4 s_co[BLEND_THREADS];
    const int tile = blockIdx.x, tx = tile % gx, ty = tile / gx;
    const int x = tx * SPL_TILE + (threadIdx.x % SPL_TILE), y = ty * SPL_TILE + (threadIdx.x / SPL_TILE);
    const bool inside = x < W && y < H;
    bool done = !inside;
    const int2 rg = ranges[tile];
    const int rounds = (rg.y - rg.x + BLEND_THREADS - 1) / BLEND_THREADS;
    int todo = rg.y - rg.x;
    float T = 1.f, C[3] = {0.f, 0.f, 0.f};
    const float pxf = (float)x, pyf = (float)y;
    for (int r = 0; r < rounds; ++r, todo -= BLEND_THREADS) {
        if (__syncthreads_count(done) == BLEND_THREADS) break;
        const int k = rg.x + r * BLEND_THREADS + threadIdx.x;
        if (k < rg.y) {
            const int id = vals[k];
            s_id[threadIdx.x] = id;
            s_xy[threadIdx.x] = w.xy[id];
            s_co[threadIdx.x] = w.conic[id];
        }
        __syncthreads();
        const int m = todo < BLEND_THREADS ? todo : BLEND_THREADS;
        for (int j = 0; !done && j < m; ++j) {
            const float2 xy = s_xy[j];
            const float4 co = s_co[j];
            const float dx = xy.x - pxf, dy = xy.y - pyf;
            const float power = -0.5f * (co.x * dx * dx + co.z * dy * dy) - co.y * dx * dy;
            if (power > 0.f) continue;
            const float alpha = fminf(0.99f, co.w * expf(power));
            if (alpha < 1.f / 255.f) continue;
            const float test_T = T * (1.f - alpha);
            if (test_T < 0.0001f) {
                done = true;
                continue;
            }
            const float* c = w.rgb + 3 * (int64_t)s_id[j];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) C[ch] += c[ch] * alpha * T;
            T = test_T;
        }
    }
    if (inside) {
        const int64_t p = (int64_t)y * W + x;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) out_rgb[3 * p + ch] = C[ch] + T * view[16 + ch];
        out_op[p] = 1.f - T;
    }
}

extern "C" int ngp_splat_render(const float* splats, int64_t n_splats, const float* view, int W, int H, int64_t capacity,
                                float* rgb, float* opacity, int64_t* n_keys, void* workspace, size_t workspace_bytes,
                                void* stream) {
    if (!spl_sizes_ok(n_splats, W, H, capacity) || (n_splats > 0 && !splats) || !view || !rgb || !opacity || !n_keys ||
        !workspace)
        return NGP_EINVAL;
    SplWs w = spl_layout((char*)workspace, n_splats, W, H, capacity);
    if (workspace_bytes < w.total || ((uintptr_t)workspace & 255)) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int gx = (W + SPL_TILE - 1) / SPL_TILE, gy = (H + SPL_TILE - 1) / SPL_TILE;
    const int64_t n_tiles = (int64_t)gx * gy;
    const int end_bit = 32 + spl_bits((uint64_t)n_tiles);
    NGP_CUDA(cudaMemsetAsync(w.ranges, 0, 8 * (size_t)n_tiles, st));
    if (n_splats == 0) {
        NGP_CUDA(cudaMemsetAsync(n_keys, 0, sizeof(int64_t), st));
    } else {
        k_splat_project<<<spl_grid(n_splats, 256, 8), 256, 0, st>>>(splats, n_splats, view, W, H, gx, gy, w);
        NGP_CHECK_LAUNCH();
        size_t tb = w.temp_bytes;
        NGP_CUDA(cub::DeviceScan::InclusiveSum(w.temp, tb, w.touched, w.touched, (int)n_splats, st));
        NGP_CUDA(cudaMemsetAsync(w.key[0], 0xff, 8 * (size_t)capacity, st));
        k_splat_keys<<<spl_grid(n_splats, 256, 8), 256, 0, st>>>(n_splats, capacity, gx, w, n_keys);
        NGP_CHECK_LAUNCH();
        cub::DoubleBuffer<uint64_t> k(w.key[0], w.key[1]);
        cub::DoubleBuffer<int32_t> v(w.val[0], w.val[1]);
        tb = w.temp_bytes;
        NGP_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, k, v, (int)capacity, 0, end_bit, st));
        k_splat_ranges<<<spl_grid(capacity, 256, 8), 256, 0, st>>>(k.Current(), capacity, n_keys, n_tiles, w.ranges);
        NGP_CHECK_LAUNCH();
        w.key[0] = k.Current();
        w.val[0] = v.Current();
    }
    k_splat_blend<<<(unsigned)n_tiles, BLEND_THREADS, 0, st>>>(w.ranges, w.val[0], w, W, H, gx, view, rgb, opacity);
    NGP_CHECK_LAUNCH();
    return 0;
}
