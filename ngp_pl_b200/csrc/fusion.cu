// Depth fusion (include/ngp_b200.h, "Depth fusion (TSDF)"; numpy restatement: oracle/tsdf_ref.py).
//
// integrate: one thread per lattice point, consecutive threads along k, grid-stride over the lattice. A launch takes up
//            to NGP_TSDF_GROUP views: each block copies their poses to shared memory once, and each thread reads its
//            point's state, applies the views in pose order in registers and writes the state back only when a view
//            observed the point. So a launch moves at most one read and one write of the state per point, and the
//            result does not depend on how the views are grouped into launches.
// The marching cubes of a TSDF volume are mesh.cu's dense kernels on a masked value accessor (McTsdf there).
// This file is compiled with -fmad=false, and every fp32 operation of the rule is written as a rounded intrinsic: the
// restatement in np.float32 matches it bit for bit. No atomics: two calls are bitwise equal.
#include "common.cuh"
#include "../../include/ngp_b200.h"

#define TSDF_THREADS 256

static int tsdf_grid(int64_t items) {
    const int64_t want = (items + TSDF_THREADS - 1) / TSDF_THREADS, cap = (int64_t)ngp_sm_count() * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

__global__ void __launch_bounds__(TSDF_THREADS) k_tsdf_integrate(
    const NgpLattice lat, float tau, int n_views, const float* __restrict__ poses, float fx, float fy, float cx, float cy,
    int W, int H, const float* __restrict__ dirs, const float* __restrict__ depth, const float* __restrict__ opacity,
    const float* __restrict__ rgb, float min_opacity, float* __restrict__ tsdf, int32_t* __restrict__ weight,
    float* __restrict__ color, int32_t* __restrict__ color_weight) {
    __shared__ float sp[NGP_TSDF_GROUP * 12];
    for (int x = threadIdx.x; x < n_views * 12; x += blockDim.x) sp[x] = poses[x];
    __syncthreads();
    const int64_t n1 = lat.n[1], n2 = lat.n[2], n = (int64_t)lat.n[0] * n1 * n2, hw = (int64_t)W * H;
    const float fW = (float)W, fH = (float)H;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = p % n2, ij = p / n2, j = ij % n1, i = ij / n1;
        const float x[3] = {__fadd_rn(lat.lo[0], __fmul_rn((float)i, lat.step[0])),
                            __fadd_rn(lat.lo[1], __fmul_rn((float)j, lat.step[1])),
                            __fadd_rn(lat.lo[2], __fmul_rn((float)k, lat.step[2]))};
        float F = tsdf[p];
        int32_t w = weight[p];
        const int32_t w_in = w;
        float c[3] = {0.f, 0.f, 0.f};
        int32_t wc = color_weight[p];
        const int32_t wc_in = wc;
        bool c_loaded = false;
        for (int v = 0; v < n_views; ++v) {
            const float* P = sp + 12 * v;  // row r: R[r][0..2], o[r]
            const float d0 = __fsub_rn(x[0], P[3]), d1 = __fsub_rn(x[1], P[7]), d2 = __fsub_rn(x[2], P[11]);
            // 1. camera coordinates R^T (x - o)
            const float zc = __fadd_rn(__fadd_rn(__fmul_rn(P[2], d0), __fmul_rn(P[6], d1)), __fmul_rn(P[10], d2));
            if (!(zc > 0.f)) continue;
            const float xc = __fadd_rn(__fadd_rn(__fmul_rn(P[0], d0), __fmul_rn(P[4], d1)), __fmul_rn(P[8], d2));
            const float yc = __fadd_rn(__fadd_rn(__fmul_rn(P[1], d0), __fmul_rn(P[5], d1)), __fmul_rn(P[9], d2));
            // 2. pixel
            const float px = __fadd_rn(__fdiv_rn(__fmul_rn(fx, xc), zc), cx);
            const float py = __fadd_rn(__fdiv_rn(__fmul_rn(fy, yc), zc), cy);
            if (!(px >= 0.f && px < fW && py >= 0.f && py < fH)) continue;
            const int64_t pix = (int64_t)floorf(py) * W + (int64_t)floorf(px);
            const int64_t q = v * hw + pix;
            // 3. depth along the pixel's ray
            const float op = __ldg(opacity + q);
            if (!(op >= min_opacity)) continue;
            const float t = __fdiv_rn(__ldg(depth + q), op);
            if (!isfinite(t)) continue;
            // 4. signed distance along the ray, Open3D's depth-to-distance multiplier |dir_p|
            const float dx = __ldg(dirs + 3 * pix), dy = __ldg(dirs + 3 * pix + 1), dz = __ldg(dirs + 3 * pix + 2);
            const float dn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            const float sdf = __fmul_rn(__fsub_rn(t, zc), dn);
            if (!(sdf >= -tau)) continue;
            // 5. distance mean
            const float f = fminf(1.f, __fdiv_rn(sdf, tau));
            F = __fdiv_rn(__fadd_rn(__fmul_rn(F, (float)w), f), (float)(w + 1));
            ++w;
            // 6. colour mean inside the band
            if (sdf <= tau) {
                if (!c_loaded) {
                    c[0] = color[3 * p], c[1] = color[3 * p + 1], c[2] = color[3 * p + 2];
                    c_loaded = true;
                }
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const float cv = fminf(__fdiv_rn(__ldg(rgb + 3 * q + ch), op), 1.f);
                    c[ch] = __fdiv_rn(__fadd_rn(__fmul_rn(c[ch], (float)wc), cv), (float)(wc + 1));
                }
                ++wc;
            }
        }
        if (w != w_in) {
            tsdf[p] = F;
            weight[p] = w;
        }
        if (wc != wc_in) {
            color[3 * p] = c[0], color[3 * p + 1] = c[1], color[3 * p + 2] = c[2];
            color_weight[p] = wc;
        }
    }
}

extern "C" int ngp_tsdf_integrate(const NgpLattice* lat, float trunc, int n_views, const float* poses, const float* K, int W,
                                  int H, const float* directions, const float* depth, const float* opacity, const float* rgb,
                                  float min_opacity, float* tsdf, int32_t* weight, float* color, int32_t* color_weight,
                                  void* stream) {
    if (!lat || !K || !tsdf || !weight || !color || !color_weight) return NGP_EINVAL;
    for (int a = 0; a < 3; ++a)
        if (lat->n[a] < 1) return NGP_EINVAL;
    if (!(trunc > 0.f) || !isfinite(trunc) || !(min_opacity > 0.f && min_opacity <= 1.f)) return NGP_EINVAL;
    if (n_views < 0 || W < 1 || H < 1 || (int64_t)W * H >= ((int64_t)1 << 31)) return NGP_EINVAL;
    if (n_views == 0) return 0;
    if (!poses || !directions || !depth || !opacity || !rgb) return NGP_EINVAL;
    const float fx = K[0], fy = K[4], cx = K[2], cy = K[5];
    const int64_t n = (int64_t)lat->n[0] * lat->n[1] * lat->n[2], hw = (int64_t)W * H;
    cudaStream_t st = (cudaStream_t)stream;
    for (int v0 = 0; v0 < n_views; v0 += NGP_TSDF_GROUP) {
        const int nv = n_views - v0 < NGP_TSDF_GROUP ? n_views - v0 : NGP_TSDF_GROUP;
        k_tsdf_integrate<<<tsdf_grid(n), TSDF_THREADS, 0, st>>>(
            *lat, trunc, nv, poses + 12 * (int64_t)v0, fx, fy, cx, cy, W, H, directions, depth + v0 * hw,
            opacity + v0 * hw, rgb + 3 * v0 * hw, min_opacity, tsdf, weight, color, color_weight);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}
