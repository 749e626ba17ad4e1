// LPIPS v0.1 with the VGG-16 backbone, the perceptual distance of the reference's validation pass (opt.py:55-56,
// train.py:65-68, 209-213: torchmetrics LearnedPerceptualImagePatchSimilarity('vgg')). The restatement the tests compare
// against is oracle/lpips_ref.py. The two images of a view run as one batch of two, so every weight tile a block loads
// serves both:
//
//   k_lpips_input    pred fp32 / gt fp32-or-uint8 (H*W, 3) -> x = clamp(2v - 1, -1, 1), (x - shift) / scale -> NHWC fp16,
//                    channels zero-padded to 16 (image 0 = pred, image 1 = gt)
//   k_lpips_conv     3x3 conv (padding 1) + bias + ReLU as an implicit GEMM: M = 2*h*w pixels, N = C_out, K = 9*C_in, fp16
//                    operands from a 4-stage cp.async pipeline, mma.sync.m16n8k16 with ldmatrix (mlp.cuh), fp32
//                    accumulation, fp16 NHWC out. conv1_1 is the same kernel with C_in = 16 (3 channels + zeros).
//   k_lpips_pool     2x2 max-pool, stride 2, rounding down
//   k_lpips_head     at a tap: per pixel, unit-normalise both feature vectors (f / (|f| + 1e-10)), the lin-weighted
//                    squared difference; a warp per pixel, fixed-order per-block partial sums in double
//   k_lpips_final    partials of each tap in block order -> tap mean; the five means added in tap order -> *out
//
// No atomics anywhere: two calls are bitwise equal, and swapping the images gives the bitwise same value (both images
// run through identical code; the head's difference is formed without contraction, so it only changes sign).
#include <math.h>

#include "common.cuh"
#include "mlp.cuh"
#include "../../include/ngp_b200.h"

#define LP_LAYERS 13
#define LP_TAPS 5
#define LP_C0 16                 // conv1_1 input channels after zero padding
#define LP_THREADS 256
#define LP_STAGES 4
#define LP_HEAD_PIX 64           // pixels per head block: 8 warps x 8 pixels
#define LP_MIN 16                // below 16 pixels on a side relu5_3 is empty

// VGG-16 features[0:30]: output channels of the 13 convolutions; a pool (features 4, 9, 16, 23) precedes layers 2, 4, 7, 10,
// and the taps relu1_2 .. relu5_3 follow layers 1, 3, 6, 9, 12
static const int kCout[LP_LAYERS] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
static const int kTapC[LP_TAPS] = {64, 128, 256, 512, 512};
static inline int lp_cin(int l) { return l == 0 ? LP_C0 : kCout[l - 1]; }
static inline bool lp_pool_before(int l) { return l == 2 || l == 4 || l == 7 || l == 10; }
static inline int lp_tap_after(int l) { return l == 1 ? 0 : l == 3 ? 1 : l == 6 ? 2 : l == 9 ? 3 : l == 12 ? 4 : -1; }

// byte offsets of the packed weights (include/ngp_b200.h): fp16 conv weights of every layer, then fp32 biases, then fp32
// lin weights
struct LpLayout {
    size_t w[LP_LAYERS], b[LP_LAYERS], lin[LP_TAPS], total;
};
static LpLayout lp_layout() {
    LpLayout L;
    size_t o = 0;
    for (int l = 0; l < LP_LAYERS; ++l) {
        L.w[l] = o;
        o += sizeof(__half) * 9 * (size_t)lp_cin(l) * kCout[l];
    }
    for (int l = 0; l < LP_LAYERS; ++l) {
        L.b[l] = o;
        o += sizeof(float) * kCout[l];
    }
    for (int t = 0; t < LP_TAPS; ++t) {
        L.lin[t] = o;
        o += sizeof(float) * kTapC[t];
    }
    L.total = o;
    return L;
}

// spatial size at each tap: halved (rounding down) by each pool
static inline void lp_tap_hw(int H, int W, int t, int& h, int& w) {
    h = H >> t;
    w = W >> t;
}
static inline int64_t lp_head_blocks(int64_t hw) { return (hw + LP_HEAD_PIX - 1) / LP_HEAD_PIX; }

// ---- input ----------------------------------------------------------------------------------------------------------

// fp32(v / 255) for every uint8 v, i.e. torch's `.float() / 255` (as metrics.cu reads a uint8 ground truth)
#define LP_U8_1(i) ((float)(i) / 255.0f)
#define LP_U8_4(i) LP_U8_1(i), LP_U8_1((i) + 1), LP_U8_1((i) + 2), LP_U8_1((i) + 3)
#define LP_U8_16(i) LP_U8_4(i), LP_U8_4((i) + 4), LP_U8_4((i) + 8), LP_U8_4((i) + 12)
#define LP_U8_64(i) LP_U8_16(i), LP_U8_16((i) + 16), LP_U8_16((i) + 32), LP_U8_16((i) + 48)
__device__ const float g_lp_u8_unit[256] = {LP_U8_64(0), LP_U8_64(64), LP_U8_64(128), LP_U8_64(192)};

// LPIPS ScalingLayer constants (shift, scale per RGB channel)
__constant__ float c_lp_shift[3] = {-0.030f, -0.088f, -0.188f};
__constant__ float c_lp_scale[3] = {0.458f, 0.448f, 0.450f};

template <bool GT_U8>
__global__ void __launch_bounds__(LP_THREADS) k_lpips_input(const float* __restrict__ pred, const void* __restrict__ gt,
                                                            int64_t hw, __half* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * LP_THREADS + threadIdx.x;  // pixel of the batch of two
    if (i >= 2 * hw) return;
    const bool is_gt = i >= hw;
    const int64_t p = is_gt ? i - hw : i;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (!is_gt) v[c] = __ldg(pred + 3 * p + c);
        else if (GT_U8) v[c] = __ldg(g_lp_u8_unit + __ldg(reinterpret_cast<const uint8_t*>(gt) + 3 * p + c));
        else v[c] = __ldg(reinterpret_cast<const float*>(gt) + 3 * p + c);
    }
    uint32_t h[8];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float x = fminf(fmaxf(__fsub_rn(__fmul_rn(2.f, v[c]), 1.f), -1.f), 1.f);
        v[c] = __fdiv_rn(__fsub_rn(x, c_lp_shift[c]), c_lp_scale[c]);
    }
    h[0] = pack_half2(v[0], v[1]);
    h[1] = pack_half2(v[2], 0.f);
#pragma unroll
    for (int k = 2; k < 8; ++k) h[k] = 0u;
    uint4* o = reinterpret_cast<uint4*>(out + LP_C0 * i);
    o[0] = make_uint4(h[0], h[1], h[2], h[3]);
    o[1] = make_uint4(h[4], h[5], h[6], h[7]);
}

// ---- convolution ----------------------------------------------------------------------------------------------------

// 16-byte cp.async that writes zeros when `valid` is false (src-size 0 reads nothing)
__device__ __forceinline__ void cp_async_16_zfill(void* smem_dst, const void* gmem_src, bool valid) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gmem_src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// Block tile BM pixels x BN output channels, K in chunks of BK channels of one tap (C_in % BK == 0, C_out % BN == 0);
// WM x WN warps, each owning a (BM/WM) x (BN/WN) tile. Shared rows are padded by 8 halfs so that the eight rows one
// ldmatrix reads fall into disjoint banks.
template <int BM, int BN, int BK, int WM, int WN>
struct LpConv {
    static constexpr int LD = BK + 8;
    static constexpr int WTM = BM / WM, WTN = BN / WN, MT = WTM / 16, NT = WTN / 8;
    static constexpr int CPR = BK / 8;                                  // 16-byte chunks per row
    static constexpr int A_CHUNKS = BM * CPR, B_CHUNKS = BN * CPR;
    static constexpr int A_PER = (A_CHUNKS + LP_THREADS - 1) / LP_THREADS, B_PER = (B_CHUNKS + LP_THREADS - 1) / LP_THREADS;
    static constexpr int STAGE = (BM + BN) * LD;                        // halfs per stage
    static constexpr size_t SMEM = sizeof(__half) * LP_STAGES * STAGE;
    static_assert(WM * WN * 32 == LP_THREADS, "8 warps");
    static_assert(MT >= 1 && NT % 2 == 0, "tile shape");
};

template <int BM, int BN, int BK, int WM, int WN>
__global__ void __launch_bounds__(LP_THREADS, 2)
k_lpips_conv(const __half* __restrict__ in, const __half* __restrict__ wt, const float* __restrict__ bias,
             __half* __restrict__ out, int H, int W, int Cin, int Cout) {
    using T = LpConv<BM, BN, BK, WM, WN>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __half* smem = reinterpret_cast<__half*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t hw = (int64_t)H * W, M = 2 * hw;
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int cblk = Cin / BK, n_k = 9 * cblk;

    // the A rows this thread stages: fixed over the K loop, so their pixel coordinates are decoded once
    int ay[T::A_PER], ax[T::A_PER];
    int64_t abase[T::A_PER];  // element offset of (image, 0, 0, 0)
    const int acol = 8 * (tid % T::CPR);
#pragma unroll
    for (int j = 0; j < T::A_PER; ++j) {
        const int64_t m = m0 + (tid + j * LP_THREADS) / T::CPR;
        if (m < M && tid + j * LP_THREADS < T::A_CHUNKS) {
            const int64_t b = m / hw, r = m - b * hw;
            ay[j] = (int)(r / W);
            ax[j] = (int)(r - (int64_t)ay[j] * W);
            abase[j] = b * hw * Cin;
        } else {
            ay[j] = -4;  // every tap reads out of bounds: zero rows
            ax[j] = 0;
            abase[j] = 0;
        }
    }

    auto load_stage = [&](int kc, int s) {
        const int tap = kc / cblk, c0 = (kc - tap * cblk) * BK;
        const int dy = tap / 3 - 1, dx = tap % 3 - 1;
        __half* sA = smem + s * T::STAGE;
        __half* sB = sA + BM * T::LD;
#pragma unroll
        for (int j = 0; j < T::A_PER; ++j) {
            const int id = tid + j * LP_THREADS;
            if (T::A_CHUNKS % LP_THREADS == 0 || id < T::A_CHUNKS) {
                const int row = id / T::CPR;
                const int yy = ay[j] + dy, xx = ax[j] + dx;
                const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
                const __half* src = ok ? in + abase[j] + ((int64_t)yy * W + xx) * Cin + c0 + acol : in;
                cp_async_16_zfill(sA + row * T::LD + acol, src, ok);
            }
        }
#pragma unroll
        for (int j = 0; j < T::B_PER; ++j) {
            const int id = tid + j * LP_THREADS;
            if (T::B_CHUNKS % LP_THREADS == 0 || id < T::B_CHUNKS) {
                const int row = id / T::CPR, col = 8 * (id % T::CPR);
                cp_async_16(sB + row * T::LD + col, wt + (int64_t)(n0 + row) * 9 * Cin + tap * Cin + c0 + col);
            }
        }
    };

    float acc[T::MT][T::NT][4];
#pragma unroll
    for (int i = 0; i < T::MT; ++i)
#pragma unroll
        for (int j = 0; j < T::NT; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < LP_STAGES - 1; ++s) {
        if (s < n_k) load_stage(s, s);
        cp_async_commit();
    }

    const int wm = warp / WN, wn = warp % WN;
    const int lrow = lane & 7, lt = lane >> 3;
    for (int kc = 0; kc < n_k; ++kc) {
        cp_async_wait<LP_STAGES - 2>();
        __syncthreads();  // stage kc has landed for every thread; stage kc - 1 is no longer read
        if (kc + LP_STAGES - 1 < n_k) load_stage(kc + LP_STAGES - 1, (kc + LP_STAGES - 1) % LP_STAGES);
        cp_async_commit();
        const __half* sA = smem + (kc % LP_STAGES) * T::STAGE;
        const __half* sB = sA + BM * T::LD;
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
            uint32_t a[T::MT][4];
#pragma unroll
            for (int i = 0; i < T::MT; ++i)
                ldmatrix_x4(a[i], sA + (wm * T::WTM + 16 * i + (lane & 15)) * T::LD + 16 * kk + 8 * (lane >> 4));
#pragma unroll
            for (int j = 0; j < T::NT; j += 2) {
                uint32_t b[4];
                ldmatrix_x4(b, sB + (wn * T::WTN + 8 * (j + (lt >> 1)) + lrow) * T::LD + 16 * kk + 8 * (lt & 1));
#pragma unroll
                for (int i = 0; i < T::MT; ++i) {
                    mma_16816(acc[i][j], a[i], b[0], b[1]);
                    mma_16816(acc[i][j + 1], a[i], b[2], b[3]);
                }
            }
        }
    }
    cp_async_wait<0>();

    // bias + ReLU, fp16 NHWC: pixel m's channels are row m of the output
    const int g = lane >> 2, q = lane & 3;
#pragma unroll
    for (int j = 0; j < T::NT; ++j) {
        const int col = n0 + wn * T::WTN + 8 * j + 2 * q;
        const float b0 = __ldg(bias + col), b1 = __ldg(bias + col + 1);
#pragma unroll
        for (int i = 0; i < T::MT; ++i) {
#pragma unroll
            for (int hlf = 0; hlf < 2; ++hlf) {
                const int64_t m = m0 + wm * T::WTM + 16 * i + g + 8 * hlf;
                if (m < M)
                    *reinterpret_cast<uint32_t*>(out + m * Cout + col) =
                        pack_half2(fmaxf(acc[i][j][2 * hlf] + b0, 0.f), fmaxf(acc[i][j][2 * hlf + 1] + b1, 0.f));
            }
        }
    }
}

template <int BM, int BN, int BK, int WM, int WN>
static int lp_conv_launch(const __half* in, const __half* wt, const float* bias, __half* out, int H, int W, int Cin,
                          int Cout, cudaStream_t st) {
    using T = LpConv<BM, BN, BK, WM, WN>;
    NGP_CUDA((ngp_smem_opt_in<k_lpips_conv<BM, BN, BK, WM, WN>>((int)T::SMEM)));
    const dim3 grid(ngp_div_up(2 * (int64_t)H * W, BM), Cout / BN);
    k_lpips_conv<BM, BN, BK, WM, WN><<<grid, LP_THREADS, T::SMEM, st>>>(in, wt, bias, out, H, W, Cin, Cout);
    NGP_CHECK_LAUNCH();
    return 0;
}

// conv1_1 (C_in 16); conv1_2 (C_out 64); every wider layer
static int lp_conv(const __half* in, const __half* wt, const float* bias, __half* out, int H, int W, int Cin, int Cout,
                   cudaStream_t st) {
    if (Cin == LP_C0) return lp_conv_launch<128, 64, 16, 4, 2>(in, wt, bias, out, H, W, Cin, Cout, st);
    if (Cout == 64) return lp_conv_launch<128, 64, 32, 4, 2>(in, wt, bias, out, H, W, Cin, Cout, st);
    return lp_conv_launch<128, 128, 32, 2, 4>(in, wt, bias, out, H, W, Cin, Cout, st);
}

// ---- pool -----------------------------------------------------------------------------------------------------------

// in (2, H, W, C) -> out (2, H/2, W/2, C); a thread owns 8 channels of one output pixel
__global__ void __launch_bounds__(LP_THREADS) k_lpips_pool(const __half* __restrict__ in, __half* __restrict__ out, int H,
                                                           int W, int C) {
    const int Ho = H >> 1, Wo = W >> 1, c8 = C >> 3;
    const int64_t i = (int64_t)blockIdx.x * LP_THREADS + threadIdx.x;
    if (i >= 2 * (int64_t)Ho * Wo * c8) return;
    const int c = (int)(i % c8);
    const int64_t p = i / c8;
    const int x = (int)(p % Wo);
    const int64_t by = p / Wo;
    const int y = (int)(by % Ho), b = (int)(by / Ho);
    const uint4* r0 = reinterpret_cast<const uint4*>(in + (((int64_t)b * H + 2 * y) * W + 2 * x) * C) + c;
    const uint4* r1 = r0 + (int64_t)W * c8;
    const uint4 v[4] = {__ldg(r0), __ldg(r0 + c8), __ldg(r1), __ldg(r1 + c8)};
    uint4 o;
    uint32_t* po = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        __half2 m = reinterpret_cast<const __half2*>(&v[0])[k];
#pragma unroll
        for (int e = 1; e < 4; ++e) m = __hmax2(m, reinterpret_cast<const __half2*>(&v[e])[k]);
        po[k] = *reinterpret_cast<uint32_t*>(&m);
    }
    reinterpret_cast<uint4*>(out)[i] = o;
}

// ---- head -----------------------------------------------------------------------------------------------------------

// f (2, hw, C) at one tap; partials[block] = sum over the block's LP_HEAD_PIX pixels of sum_c lin_c (f0^ - f1^)^2 in
// double. Lane l holds channels 2l, 2l + 1 of every 64-channel group.
template <int C>
__global__ void __launch_bounds__(LP_THREADS) k_lpips_head(const __half* __restrict__ f, const float* __restrict__ lin,
                                                           int64_t hw, double* __restrict__ partials) {
    constexpr int G = C / 64;
    __shared__ double red[LP_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[2 * G];
#pragma unroll
    for (int j = 0; j < G; ++j) {
        w[2 * j] = __ldg(lin + 64 * j + 2 * lane);
        w[2 * j + 1] = __ldg(lin + 64 * j + 2 * lane + 1);
    }
    double acc = 0.0;
    for (int k = 0; k < LP_HEAD_PIX / (LP_THREADS / 32); ++k) {
        const int64_t p = (int64_t)blockIdx.x * LP_HEAD_PIX + k * (LP_THREADS / 32) + warp;
        if (p >= hw) break;  // warp-uniform
        float a[2 * G], b[2 * G];
        const uint32_t* pa = reinterpret_cast<const uint32_t*>(f + p * C) + lane;
        const uint32_t* pb = reinterpret_cast<const uint32_t*>(f + (hw + p) * C) + lane;
#pragma unroll
        for (int j = 0; j < G; ++j) {
            const float2 u = unpack_half2(__ldg(pa + 32 * j)), v = unpack_half2(__ldg(pb + 32 * j));
            a[2 * j] = u.x;
            a[2 * j + 1] = u.y;
            b[2 * j] = v.x;
            b[2 * j + 1] = v.y;
        }
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int j = 0; j < 2 * G; ++j) {
            sa = fmaf(a[j], a[j], sa);
            sb = fmaf(b[j], b[j], sb);
        }
        // xor butterflies: every lane ends with the bitwise same sums
        sa = warp_sum(sa);
        sb = warp_sum(sb);
        const float ia = 1.f / (sqrtf(sa) + 1e-10f), ib = 1.f / (sqrtf(sb) + 1e-10f);
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < 2 * G; ++j) {
            const float e = __fsub_rn(__fmul_rn(a[j], ia), __fmul_rn(b[j], ib));  // no contraction: swapping negates e
            d = fmaf(w[j], __fmul_rn(e, e), d);
        }
        d = warp_sum(d);
        acc += (double)d;
    }
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < LP_THREADS / 32; ++i) s += red[i];
        partials[blockIdx.x] = s;
    }
}

struct LpTaps {
    int64_t n_blk[LP_TAPS], off[LP_TAPS];
    double hw[LP_TAPS];
};

// out = sum over taps (in order) of (sum of the tap's partials in block order, per-thread strided then a fixed tree) / hw
__global__ void __launch_bounds__(LP_THREADS) k_lpips_final(const double* __restrict__ partials, LpTaps taps,
                                                            double* __restrict__ out) {
    __shared__ double red[LP_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double total = 0.0;
    for (int t = 0; t < LP_TAPS; ++t) {
        double s = 0.0;
        for (int64_t i = tid; i < taps.n_blk[t]; i += LP_THREADS) s += partials[taps.off[t] + i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[warp] = s;
        __syncthreads();
        if (tid == 0) {
            double b = 0.0;
            for (int i = 0; i < LP_THREADS / 32; ++i) b += red[i];
            total += b / taps.hw[t];
        }
        __syncthreads();
    }
    if (tid == 0) *out = total;
}

template <int C>
static int lp_head_launch(const __half* f, const float* lin, int64_t hw, double* partials, cudaStream_t st) {
    k_lpips_head<C><<<(unsigned)lp_head_blocks(hw), LP_THREADS, 0, st>>>(f, lin, hw, partials);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---- entry points ---------------------------------------------------------------------------------------------------

static inline size_t lp_act_bytes(int H, int W) { return (size_t)2 * H * W * 64 * sizeof(__half); }

static LpTaps lp_taps(int H, int W) {
    LpTaps T;
    int64_t off = 0;
    for (int t = 0; t < LP_TAPS; ++t) {
        int h, w;
        lp_tap_hw(H, W, t, h, w);
        T.hw[t] = (double)h * w;
        T.n_blk[t] = lp_head_blocks((int64_t)h * w);
        T.off[t] = off;
        off += T.n_blk[t];
    }
    return T;
}

extern "C" size_t ngp_lpips_weights_bytes(void) { return lp_layout().total; }

extern "C" size_t ngp_lpips_workspace(int H, int W) {
    if (H < LP_MIN || W < LP_MIN || (int64_t)H * W > NGP_LPIPS_MAX_PIXELS) return 0;
    const LpTaps T = lp_taps(H, W);
    return 2 * lp_act_bytes(H, W) + sizeof(double) * (size_t)(T.off[LP_TAPS - 1] + T.n_blk[LP_TAPS - 1]);
}

static bool lp_on_device(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();  // a failed query is not an error of the next launch
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

extern "C" int ngp_lpips(const void* weights, const float* pred, const void* gt, int gt_is_u8, int H, int W, double* out,
                         void* workspace, size_t workspace_bytes, void* stream) {
    if (!weights || !pred || !gt || !out || !workspace) return NGP_EINVAL;
    const size_t need = ngp_lpips_workspace(H, W);
    if (need == 0 || workspace_bytes < need) return NGP_EINVAL;
    if ((((uintptr_t)weights) & 15) || (((uintptr_t)workspace) & 15) || (((uintptr_t)out) & 7) ||
        (((uintptr_t)pred) & 3) || (!gt_is_u8 && (((uintptr_t)gt) & 3)))
        return NGP_EINVAL;
    if (!lp_on_device(weights) || !lp_on_device(pred) || !lp_on_device(gt) || !lp_on_device(out) ||
        !lp_on_device(workspace))
        return NGP_EINVAL;
    const cudaStream_t st = (cudaStream_t)stream;
    const LpLayout L = lp_layout();
    const unsigned char* wb = reinterpret_cast<const unsigned char*>(weights);
    __half* buf[2] = {reinterpret_cast<__half*>(workspace),
                      reinterpret_cast<__half*>(reinterpret_cast<unsigned char*>(workspace) + lp_act_bytes(H, W))};
    double* partials = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(workspace) + 2 * lp_act_bytes(H, W));
    const LpTaps T = lp_taps(H, W);

    const int64_t hw = (int64_t)H * W;
    if (gt_is_u8) k_lpips_input<true><<<ngp_div_up(2 * hw, LP_THREADS), LP_THREADS, 0, st>>>(pred, gt, hw, buf[0]);
    else k_lpips_input<false><<<ngp_div_up(2 * hw, LP_THREADS), LP_THREADS, 0, st>>>(pred, gt, hw, buf[0]);
    NGP_CHECK_LAUNCH();
    int cur = 0, h = H, w = W;
    for (int l = 0; l < LP_LAYERS; ++l) {
        if (lp_pool_before(l)) {
            const int C = kCout[l - 1];
            k_lpips_pool<<<ngp_div_up(2 * (int64_t)(h >> 1) * (w >> 1) * (C / 8), LP_THREADS), LP_THREADS, 0, st>>>(
                buf[cur], buf[cur ^ 1], h, w, C);
            NGP_CHECK_LAUNCH();
            cur ^= 1;
            h >>= 1;
            w >>= 1;
        }
        const int rc = lp_conv(buf[cur], reinterpret_cast<const __half*>(wb + L.w[l]),
                               reinterpret_cast<const float*>(wb + L.b[l]), buf[cur ^ 1], h, w, lp_cin(l), kCout[l], st);
        if (rc) return rc;
        cur ^= 1;
        const int t = lp_tap_after(l);
        if (t >= 0) {
            const float* lin = reinterpret_cast<const float*>(wb + L.lin[t]);
            const int64_t thw = (int64_t)h * w;
            int r;
            switch (kTapC[t]) {
                case 64: r = lp_head_launch<64>(buf[cur], lin, thw, partials + T.off[t], st); break;
                case 128: r = lp_head_launch<128>(buf[cur], lin, thw, partials + T.off[t], st); break;
                case 256: r = lp_head_launch<256>(buf[cur], lin, thw, partials + T.off[t], st); break;
                default: r = lp_head_launch<512>(buf[cur], lin, thw, partials + T.off[t], st); break;
            }
            if (r) return r;
        }
    }
    k_lpips_final<<<1, LP_THREADS, 0, st>>>(partials, T, out);
    NGP_CHECK_LAUNCH();
    return 0;
}
