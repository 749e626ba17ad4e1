// Per-view image metrics of the reference's validation pass (train.py:193-237): the sum of squared errors behind
// PSNR (metrics.py:14-15, torchmetrics PeakSignalNoiseRatio(data_range=1)) and the mean SSIM of torchmetrics'
// StructuralSimilarityIndexMeasure(data_range=1) with its defaults: 11-tap Gaussian window, sigma 1.5, only windows
// lying wholly inside the image (torchmetrics reflect-pads and crops the padding off again), no clamping of the
// variances. The restatement the tests compare against is oracle/metrics_ref.py.
//
// One launch per view. A block owns a 32 x 32 tile of window centres: it stages the tile plus its 5-pixel halo of one
// channel in shared memory, runs the horizontal 11-tap pass for the five moments (p, t, p^2, t^2, pt) over the 42 staged
// rows, then the vertical pass, each thread walking 4 consecutive centres of one column. The moments are accumulated in
// double: SSIM divides variance differences by c2 = 9e-4, so fp32 rounding of the 121-tap sums (~1e-7) would show as
// ~1e-4 in the SSIM of flat regions whose two images differ. The squared error of the block's 1024 pixels (a linear
// range, so the loads are coalesced) rides along. Per-block partials are summed by the last block to arrive, in block
// order, in double: two calls give bitwise equal results.
#include <math.h>

#include "common.cuh"
#include "../../include/ngp_b200.h"

#define MET_R 5                         // window radius: int(3.5 * 1.5 + 0.5) = 5, 11 taps
#define MET_K (2 * MET_R + 1)
#define MET_TX 32                       // tile width = threads per row
#define MET_TY 32                       // tile height
#define MET_THREADS 256                 // 32 x 8 threads, 4 centre rows each
#define MET_ROWS (MET_TY / (MET_THREADS / MET_TX))
#define MET_SW (MET_TX + 2 * MET_R)     // staged width
#define MET_SH (MET_TY + 2 * MET_R)     // staged height
#define MET_PIX (MET_TX * MET_TY)       // pixels of the squared error per block
#define MET_HEADER 16                   // arrival counter, padded so the partials are 16-B aligned

struct MetWindow {
    float w[MET_K];
};

struct MetSmem {
    float p[MET_SH][MET_SW];
    float t[MET_SH][MET_SW];
    double h[5][MET_SH][MET_TX];        // horizontal pass: the five moments of each staged row
    double red[2][MET_THREADS / 32];
    int last;
};

// fp32(v / 255) for every uint8 v, i.e. torch's `.float() / 255`, folded by the compiler: v * fp32(1/255) differs in 126
// of the 256 values, and an IEEE division in the loops would be a called slow path that spills
#define MET_U8_1(i) ((float)(i) / 255.0f)
#define MET_U8_4(i) MET_U8_1(i), MET_U8_1((i) + 1), MET_U8_1((i) + 2), MET_U8_1((i) + 3)
#define MET_U8_16(i) MET_U8_4(i), MET_U8_4((i) + 4), MET_U8_4((i) + 8), MET_U8_4((i) + 12)
#define MET_U8_64(i) MET_U8_16(i), MET_U8_16((i) + 16), MET_U8_16((i) + 32), MET_U8_16((i) + 48)
__device__ const float g_met_u8_unit[256] = {MET_U8_64(0), MET_U8_64(64), MET_U8_64(128), MET_U8_64(192)};

template <bool GT_U8>
__device__ __forceinline__ float gt_at(const void* __restrict__ gt, int64_t i) {
    if (GT_U8) return __ldg(g_met_u8_unit + __ldg(reinterpret_cast<const uint8_t*>(gt) + i));
    return __ldg(reinterpret_cast<const float*>(gt) + i);
}

// the 11-tap window of the oracle (oracle/metrics_ref.py gaussian_weights), built on the host with the same operations
static MetWindow met_window() {
    MetWindow m;
    float e[MET_K];
    double s = 0.0;  // exact: 11 fp32 values spanning 17 binades
    for (int i = 0; i < MET_K; ++i) {
        const float a = (float)(i - MET_R) / 1.5f;
        const float arg = -(a * a) / 2.0f;
        e[i] = (float)exp((double)arg);
        s += (double)e[i];
    }
    const float sf = (float)s;
    for (int i = 0; i < MET_K; ++i) m.w[i] = e[i] / sf;
    return m;
}

static inline int64_t met_tiles(int H, int W) { return (int64_t)ngp_div_up(W, MET_TX) * ngp_div_up(H, MET_TY); }

template <bool GT_U8, bool SSIM>
__global__ void __launch_bounds__(MET_THREADS)
k_image_metrics(const float* __restrict__ pred, const void* __restrict__ gt, int H, int W, MetWindow win, double c1, double c2,
                double* __restrict__ out_sse, double* __restrict__ out_ssim, unsigned int* __restrict__ counter,
                double2* __restrict__ partials) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MetSmem& S = *reinterpret_cast<MetSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int blk = blockIdx.y * gridDim.x + blockIdx.x;
    const int64_t n_val = 3 * (int64_t)H * W;

    // squared error of the pixels [blk * 1024, blk * 1024 + 1024)
    double sse = 0.0;
    {
        const int64_t base = (int64_t)blk * (3 * MET_PIX);
        for (int i = tid; i < 3 * MET_PIX; i += MET_THREADS) {
            const int64_t j = base + i;
            if (j < n_val) {
                const double d = (double)__ldg(pred + j) - (double)gt_at<GT_U8>(gt, j);
                sse = fma(d, d, sse);
            }
        }
    }

    double ssim = 0.0;
    if (SSIM) {
        const int x0 = blockIdx.x * MET_TX, y0 = blockIdx.y * MET_TY;
        // block-uniform: does the tile hold any window centre of [R, H-R) x [R, W-R)?
        if (x0 < W - MET_R && x0 + MET_TX > MET_R && y0 < H - MET_R && y0 + MET_TY > MET_R) {
            const int tx = lane, ty0 = warp * MET_ROWS;
            for (int ch = 0; ch < 3; ++ch) {
                for (int i = tid; i < MET_SH * MET_SW; i += MET_THREADS) {
                    const int r = i / MET_SW, c = i - r * MET_SW;
                    const int gy = y0 - MET_R + r, gx = x0 - MET_R + c;
                    float pv = 0.f, tv = 0.f;
                    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
                        const int64_t j = 3 * ((int64_t)gy * W + gx) + ch;
                        pv = __ldg(pred + j);
                        tv = gt_at<GT_U8>(gt, j);
                    }
                    S.p[r][c] = pv;
                    S.t[r][c] = tv;
                }
                __syncthreads();
                for (int i = tid; i < MET_SH * MET_TX; i += MET_THREADS) {
                    const int r = i / MET_TX, c = i - r * MET_TX;
                    double mp = 0.0, mt = 0.0, mpp = 0.0, mtt = 0.0, mpt = 0.0;
#pragma unroll
                    for (int k = 0; k < MET_K; ++k) {
                        const double pv = S.p[r][c + k], tv = S.t[r][c + k];
                        const double wp = (double)win.w[k] * pv, wt = (double)win.w[k] * tv;  // exact products
                        mp += wp;
                        mt += wt;
                        mpp = fma(wp, pv, mpp);
                        mtt = fma(wt, tv, mtt);
                        mpt = fma(wp, tv, mpt);
                    }
                    S.h[0][r][c] = mp;
                    S.h[1][r][c] = mt;
                    S.h[2][r][c] = mpp;
                    S.h[3][r][c] = mtt;
                    S.h[4][r][c] = mpt;
                }
                __syncthreads();
                double acc[MET_ROWS][5];
#pragma unroll
                for (int o = 0; o < MET_ROWS; ++o)
#pragma unroll
                    for (int m = 0; m < 5; ++m) acc[o][m] = 0.0;
#pragma unroll
                for (int r = 0; r < MET_ROWS + MET_K - 1; ++r) {
                    double hv[5];
#pragma unroll
                    for (int m = 0; m < 5; ++m) hv[m] = S.h[m][ty0 + r][tx];
#pragma unroll
                    for (int o = 0; o < MET_ROWS; ++o) {
                        const int k = r - o;
                        if (k >= 0 && k < MET_K) {
#pragma unroll
                            for (int m = 0; m < 5; ++m) acc[o][m] = fma((double)win.w[k], hv[m], acc[o][m]);
                        }
                    }
                }
                const int cx = x0 + tx;
#pragma unroll
                for (int o = 0; o < MET_ROWS; ++o) {
                    const int cy = y0 + ty0 + o;
                    if (cx >= MET_R && cx < W - MET_R && cy >= MET_R && cy < H - MET_R) {
                        const double mpp = acc[o][0] * acc[o][0], mtt = acc[o][1] * acc[o][1], mpt = acc[o][0] * acc[o][1];
                        const double upper = 2.0 * (acc[o][4] - mpt) + c2;
                        const double lower = (acc[o][2] - mpp) + (acc[o][3] - mtt) + c2;
                        ssim += ((2.0 * mpt + c1) * upper) / ((mpp + mtt + c1) * lower);
                    }
                }
                __syncthreads();  // S.p / S.t are restaged for the next channel
            }
        }
    }

    // block partial in a fixed order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sse += __shfl_xor_sync(0xffffffffu, sse, o);
        ssim += __shfl_xor_sync(0xffffffffu, ssim, o);
    }
    if (lane == 0) {
        S.red[0][warp] = sse;
        S.red[1][warp] = ssim;
    }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b = 0.0;
        for (int w = 0; w < MET_THREADS / 32; ++w) {
            a += S.red[0][w];
            b += S.red[1][w];
        }
        partials[blk] = make_double2(a, b);
        __threadfence();
        S.last = atomicAdd(counter, 1u) == gridDim.x * gridDim.y - 1;
    }
    __syncthreads();
    if (!S.last) return;

    // the last block: partials in block order, each thread a fixed strided subset, then the same fixed tree
    __threadfence();
    const int n_blk = gridDim.x * gridDim.y;
    double a = 0.0, b = 0.0;
    for (int i = tid; i < n_blk; i += MET_THREADS) {
        const double2 v = __ldcg(partials + i);
        a += v.x;
        b += v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    __syncthreads();
    if (lane == 0) {
        S.red[0][warp] = a;
        S.red[1][warp] = b;
    }
    __syncthreads();
    if (tid == 0) {
        a = 0.0;
        b = 0.0;
        for (int w = 0; w < MET_THREADS / 32; ++w) {
            a += S.red[0][w];
            b += S.red[1][w];
        }
        *out_sse = a;
        if (SSIM) *out_ssim = b / (3.0 * (double)(H - 2 * MET_R) * (double)(W - 2 * MET_R));
        *counter = 0u;  // re-armed for the next launch on this workspace
    }
}

extern "C" size_t ngp_image_metrics_workspace(int H, int W) {
    if (H < 1 || W < 1) return 0;
    return MET_HEADER + sizeof(double2) * (size_t)met_tiles(H, W);
}

template <bool GT_U8, bool SSIM>
static int met_launch(dim3 grid, cudaStream_t st, const float* pred, const void* gt, int H, int W, const MetWindow& win,
                      double c1, double c2, double* out_sse, double* out_ssim, void* workspace) {
    static bool attr = false;
    if (!attr) {
        NGP_CUDA(cudaFuncSetAttribute(k_image_metrics<GT_U8, SSIM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(MetSmem)));
        attr = true;
    }
    k_image_metrics<GT_U8, SSIM><<<grid, MET_THREADS, sizeof(MetSmem), st>>>(
        pred, gt, H, W, win, c1, c2, out_sse, out_ssim, reinterpret_cast<unsigned int*>(workspace),
        reinterpret_cast<double2*>(reinterpret_cast<unsigned char*>(workspace) + MET_HEADER));
    NGP_CHECK_LAUNCH();
    return 0;
}

extern "C" int ngp_image_metrics(const float* pred, const void* gt, int gt_is_u8, int H, int W, float data_range,
                                 double* out_sse, double* out_ssim, void* workspace, size_t workspace_bytes, void* stream) {
    if (!pred || !gt || !out_sse || !workspace || H < 1 || W < 1) return NGP_EINVAL;
    if (out_ssim && (H < MET_K || W < MET_K || !(data_range > 0.f))) return NGP_EINVAL;
    if ((((uintptr_t)out_sse) & 7) || (((uintptr_t)out_ssim) & 7) || (((uintptr_t)workspace) & 15)) return NGP_EINVAL;
    // grid limits: 65535 tile rows; fewer than 2^31 blocks
    if (ngp_div_up(H, MET_TY) > 65535 || met_tiles(H, W) >= ((int64_t)1 << 31)) return NGP_EINVAL;
    if (workspace_bytes < ngp_image_metrics_workspace(H, W)) return NGP_EINVAL;
    const MetWindow win = met_window();
    const double dr = (double)data_range, c1 = (0.01 * dr) * (0.01 * dr), c2 = (0.03 * dr) * (0.03 * dr);
    const cudaStream_t st = (cudaStream_t)stream;
    if (out_ssim) {
        const dim3 grid(ngp_div_up(W, MET_TX), ngp_div_up(H, MET_TY));
        return gt_is_u8 ? met_launch<true, true>(grid, st, pred, gt, H, W, win, c1, c2, out_sse, out_ssim, workspace)
                        : met_launch<false, true>(grid, st, pred, gt, H, W, win, c1, c2, out_sse, out_ssim, workspace);
    }
    const dim3 grid(ngp_div_up((int64_t)H * W, MET_PIX));
    return gt_is_u8 ? met_launch<true, false>(grid, st, pred, gt, H, W, win, c1, c2, out_sse, nullptr, workspace)
                    : met_launch<false, false>(grid, st, pred, gt, H, W, win, c1, c2, out_sse, nullptr, workspace);
}
