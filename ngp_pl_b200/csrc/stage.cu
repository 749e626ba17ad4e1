// Image staging for the training bank (reference datasets/color_utils.py:19-31, `read_image`): a decoded uint8 image on
// the device -> one fp32 (h*w, 3) row of the bank, bitwise what
//     img = imread(path).astype(np.float32) / 255.0
//     img = img[..., :3] * img[..., -1:] + (1 - img[..., -1:])      (4 channels, blend_a)   or   img[..., :3] * img[..., -1:]
//     img = cv2.resize(img, (w, h))                                    (INTER_LINEAR on fp32)
// computes. Every operation is written with an explicitly rounded intrinsic so that no FMA contraction changes a bit.
//
// cv2's fp32 bilinear path (measured against cv2.resize 4.13 on the host, oracle/stage_ref.py) evaluates, per axis,
//     f  = (d + 0.5) * (S / D) - 0.5          in double
//     s  = floor(f),  a = (float)(f - s)       clamped to (0, 0) below the first and to (S-1, 0) past the last sample
//     t  = fma(a, p[s+1] - p[s], p[s])         in fp32 (a single rounding)
// first along x on the two source rows, then along y on the two results. With (w, h) == (W0, H0) cv2 copies.
#include "common.cuh"

namespace {

__device__ __forceinline__ float stage_px(const uint8_t* __restrict__ src, int64_t p, int C, int blend_a, int k) {
    const uint8_t* q = src + p * C;
    float c = __fdiv_rn((float)q[k], 255.0f);
    if (C == 4) {
        const float a = __fdiv_rn((float)q[3], 255.0f);
        c = __fmul_rn(c, a);
        if (blend_a) c = __fadd_rn(c, __fsub_rn(1.0f, a));
    }
    return c;
}

__device__ __forceinline__ void lin_coeff(int d, int S, int D, int& s0, int& s1, float& a) {
    const double f = __dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), __ddiv_rn((double)S, (double)D)), 0.5);
    int s = (int)floor(f);
    a = __double2float_rn(__dsub_rn(f, (double)s));
    if (s < 0) {
        s = 0;
        a = 0.0f;
    }
    if (s >= S - 1) {
        s = S - 1;
        a = 0.0f;
    }
    s0 = s;
    s1 = min(s + 1, S - 1);
}

__global__ void k_stage_image(const uint8_t* __restrict__ src, int H0, int W0, int C, int blend_a, int h, int w,
                              float* __restrict__ dst) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)h * w) return;
    if (h == H0 && w == W0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) dst[3 * i + k] = stage_px(src, i, C, blend_a, k);
        return;
    }
    const int y = (int)(i / w), x = (int)(i % w);
    int x0, x1, y0, y1;
    float ax, ay;
    lin_coeff(x, W0, w, x0, x1, ax);
    lin_coeff(y, H0, h, y0, y1, ay);
    const int64_t r0 = (int64_t)y0 * W0, r1 = (int64_t)y1 * W0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float p00 = stage_px(src, r0 + x0, C, blend_a, k), p01 = stage_px(src, r0 + x1, C, blend_a, k);
        const float p10 = stage_px(src, r1 + x0, C, blend_a, k), p11 = stage_px(src, r1 + x1, C, blend_a, k);
        const float t0 = __fmaf_rn(ax, __fsub_rn(p01, p00), p00);
        const float t1 = __fmaf_rn(ax, __fsub_rn(p11, p10), p10);
        dst[3 * i + k] = __fmaf_rn(ay, __fsub_rn(t1, t0), t0);
    }
}

}  // namespace

extern "C" int ngp_stage_image(const uint8_t* src, int src_h, int src_w, int channels, int blend_a, int dst_h, int dst_w,
                               float* dst, void* stream) {
    if (!src || !dst || src_h < 1 || src_w < 1 || dst_h < 1 || dst_w < 1 || (channels != 3 && channels != 4)) return NGP_EINVAL;
    // cv2 treats a single source row or column differently; the loaders never resize one
    if ((src_h != dst_h || src_w != dst_w) && (src_h < 2 || src_w < 2)) return NGP_EINVAL;
    const int64_t n = (int64_t)dst_h * dst_w;
    k_stage_image<<<ngp_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(src, src_h, src_w, channels, blend_a, dst_h, dst_w,
                                                                         dst);
    NGP_CHECK_LAUNCH();
    return 0;
}
