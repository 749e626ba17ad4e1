// Stand-alone kernels behind the tinycudann-shaped modules (ngp_pl_b200/tcnn.py) for callers that use the
// three modules of reference models/networks.py:36-77 one by one, exactly as the reference's own
// NGP.forward does (xyz_encoder(x) -> h ; dir_encoder((d+1)/2) ; rgb_net(cat[d, h])):
//   ngp_sh_encode        tcnn.Encoding(SphericalHarmonics, degree 4)
//   ngp_mlp_rgb_forward  tcnn.Network(32 -> 64 -> 64 -> 3)              forward on an (N,32) fp16 matrix
//   ngp_mlp_rgb_backward                                               dL/dx (N,32) + weight gradients
//   ngp_enc_backward     tcnn.NetworkWithInputEncoding backward from dL/dh (N,16): weight gradients +
//                        feature gradients for ngp_net_backward_scatter (its forward is ngp_net_forward
//                        with want_rgb = 0 and h_out)
// The fused NGP kernels (network.cu) are the hot path; these run the same network chains (network.cuh) in the simple
// 8-warp / stage-everything form, with their own mma.sync weight-gradient loops.
#include "common.cuh"
#include "network.cuh"
#include "../../include/ngp_b200.h"

// ---------------------------------------------------------------------------------------------------
// SH-4 of u in [0,1]^3 (tinycudann maps its input to 2u-1)
// ---------------------------------------------------------------------------------------------------
__global__ void k_sh_encode(const float* __restrict__ u, int64_t n, __half* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float sh[16];
    sh4(fmaf(u[3 * i], 2.0f, -1.0f), fmaf(u[3 * i + 1], 2.0f, -1.0f), fmaf(u[3 * i + 2], 2.0f, -1.0f), sh);
    uint4* o = reinterpret_cast<uint4*>(out + 16 * i);
    o[0] = make_uint4(pack_half2(sh[0], sh[1]), pack_half2(sh[2], sh[3]), pack_half2(sh[4], sh[5]), pack_half2(sh[6], sh[7]));
    o[1] = make_uint4(pack_half2(sh[8], sh[9]), pack_half2(sh[10], sh[11]), pack_half2(sh[12], sh[13]), pack_half2(sh[14], sh[15]));
}
extern "C" int ngp_sh_encode(const float* u01, int64_t n, uint16_t* out_half, void* stream) {
    if (n < 0 || (n > 0 && (!u01 || !out_half)) || (((uintptr_t)out_half) & 15)) return NGP_EINVAL;
    if (n == 0) return 0;
    k_sh_encode<<<ngp_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(u01, n, (__half*)out_half);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------------
#define MOD_WARPS 8
#define MOD_THREADS (MOD_WARPS * 32)
#define MOD_ROWS (MOD_WARPS * 16)

// A fragments (K = 32) of 16 rows of a row-major fp16 matrix X (n, 32) in global memory
__device__ __forceinline__ void load_rows32(const __half* __restrict__ X, int64_t base, int64_t n, uint32_t (&A)[1][2][4], int g, int q) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t row = base + g + 8 * h;
        const bool ok = row < n;
        const uint32_t* r = reinterpret_cast<const uint32_t*>(X + row * 32);
#pragma unroll
        for (int kt = 0; kt < 2; ++kt) {
            A[0][kt][h] = ok ? __ldg(r + 8 * kt + q) : 0u;
            A[0][kt][2 + h] = ok ? __ldg(r + 8 * kt + 4 + q) : 0u;
        }
    }
}

template <int KT>
__device__ __forceinline__ void stage_rows(__half* __restrict__ dst, int ld, int row0, const uint32_t (&A)[KT][4], int g, int q) {
#pragma unroll
    for (int kt = 0; kt < KT; ++kt) {
        uint32_t* r0 = reinterpret_cast<uint32_t*>(dst + (row0 + g) * ld + 16 * kt + 2 * q);
        uint32_t* r1 = reinterpret_cast<uint32_t*>(dst + (row0 + g + 8) * ld + 16 * kt + 2 * q);
        r0[0] = A[kt][0]; r1[0] = A[kt][1]; r0[4] = A[kt][2]; r1[4] = A[kt][3];
    }
}

__device__ __forceinline__ void wgrad_acc(float (&acc)[4], const __half* __restrict__ dOut, int ld_o, int mt,
                                          const __half* __restrict__ In, int ld_i, int nt, int lane) {
    const int ra = (lane & 7) + 8 * ((lane >> 4) & 1), ca = 16 * mt + 8 * ((lane >> 3) & 1);
    const int rb = (lane & 7) + 8 * ((lane >> 3) & 1), cb = 8 * nt;
#pragma unroll
    for (int ks = 0; ks < MOD_ROWS / 16; ++ks) {
        uint32_t a[4], b0, b1;
        ldmatrix_x4_trans(a, dOut + (16 * ks + ra) * ld_o + ca);
        ldmatrix_x2_trans(b0, b1, In + (16 * ks + rb) * ld_i + cb);
        mma_16816(acc, a, b0, b1);
    }
}
__device__ __forceinline__ void wgrad_out(const float (&acc)[4], float* __restrict__ dW, int in_dim, int mt, int nt, float inv_scale,
                                          int g, int q) {
    red_add_f32x2(dW + (16 * mt + g) * in_dim + 8 * nt + 2 * q, acc[0] * inv_scale, acc[1] * inv_scale);
    red_add_f32x2(dW + (16 * mt + g + 8) * in_dim + 8 * nt + 2 * q, acc[2] * inv_scale, acc[3] * inv_scale);
}

// ---------------------------------------------------------------------------------------------------
// rgb MLP 32 -> 64 -> 64 -> 3 on an external input matrix
// ---------------------------------------------------------------------------------------------------
struct RgbW {
    __half w1r[64 * LD32];
    __half w2r[64 * LD64];
    __half w3r[16 * LD64];
};
__device__ __forceinline__ void load_rgb_weights(RgbW& s, const __half* __restrict__ wr, int tid, int nthreads) {
    load_matrix(s.w1r, LD32, wr, 64, 32, tid, nthreads);
    load_matrix(s.w2r, LD64, wr + 2048, 64, 64, tid, nthreads);
    load_matrix(s.w3r, LD64, wr + 2048 + 4096, 16, 64, tid, nthreads);
    cp_async_wait_all();
}

__global__ void __launch_bounds__(MOD_THREADS)
k_mlp_rgb_fwd(const __half* __restrict__ wr, const __half* __restrict__ X, int64_t n, int act, __half* __restrict__ out3) {
    __shared__ __align__(16) RgbW sw;
    load_rgb_weights(sw, wr, threadIdx.x, MOD_THREADS);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int64_t n_tiles = (n + 15) / 16;
    for (int64_t tile = (int64_t)blockIdx.x * MOD_WARPS + warp; tile < n_tiles; tile += (int64_t)gridDim.x * MOD_WARPS) {
        const int64_t base = tile * 16;
        uint32_t inA[1][2][4];
        load_rows32(X, base, n, inA, g, q);
        float oC[1][1][4];
        color_mlp<1>(inA, sw.w1r, sw.w2r, sw.w3r, oC, g, q, [](int, const auto&) {});
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = base + g + 8 * h;
            if (row >= n || q > 1) continue;
            const __half2 o = rgb_out(oC[0][0][2 * h], oC[0][0][2 * h + 1], act);
            if (q == 0) {
                out3[3 * row] = __low2half(o);
                out3[3 * row + 1] = __high2half(o);
            } else {
                out3[3 * row + 2] = __low2half(o);
            }
        }
    }
}

extern "C" int ngp_mlp_rgb_forward(const uint16_t* rgb_params_h, const uint16_t* x_half, int64_t n, int rgb_act,
                                   uint16_t* out_half3, void* stream) {
    if (n < 0 || !rgb_params_h || (n > 0 && (!x_half || !out_half3)) || (((uintptr_t)x_half) & 3)) return NGP_EINVAL;
    if (n == 0) return 0;
    const int64_t want = ((n + 15) / 16 + MOD_WARPS - 1) / MOD_WARPS;
    const int grid = (int)(want < (int64_t)ngp_sm_count() * 4 ? want : ngp_sm_count() * 4);
    k_mlp_rgb_fwd<<<grid, MOD_THREADS, 0, (cudaStream_t)stream>>>((const __half*)rgb_params_h, (const __half*)x_half, n, rgb_act,
                                                                 (__half*)out_half3);
    NGP_CHECK_LAUNCH();
    return 0;
}

struct RgbBwdSmem {
    RgbW w;
    __half rin[MOD_ROWS * LD32];
    __half r1[MOD_ROWS * LD64];
    __half r2[MOD_ROWS * LD64];
    __half dr1[MOD_ROWS * LD64];
    __half dr2[MOD_ROWS * LD64];
    __half dout[MOD_ROWS * LD16];
};

// 56 wgrad tiles (W1r 16, W2r 32, W3r 8), 7 per warp
struct ModTile { int mat, mt, nt; };
__device__ __forceinline__ ModTile rgb_tile_of(int t) {
    ModTile w;
    if (t < 16) { w.mat = 0; w.mt = t >> 2; w.nt = t & 3; }
    else if (t < 48) { w.mat = 1; w.mt = (t - 16) >> 3; w.nt = (t - 16) & 7; }
    else { w.mat = 2; w.mt = 0; w.nt = t - 48; }
    return w;
}

__global__ void __launch_bounds__(MOD_THREADS, 1)
k_mlp_rgb_bwd(const __half* __restrict__ wr, const __half* __restrict__ X, const float* __restrict__ dL_dout3, int64_t n, int act,
              const float* __restrict__ loss_scale, float* __restrict__ dL_dX, float* __restrict__ grad_rgb) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    RgbBwdSmem& S = *reinterpret_cast<RgbBwdSmem*>(smem_raw);
    load_rgb_weights(S.w, wr, threadIdx.x, MOD_THREADS);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int64_t n_blks = ((n + 15) / 16 + MOD_WARPS - 1) / MOD_WARPS;
    const float scale = loss_scale ? *loss_scale : 1.0f;
    const float inv_scale = 1.0f / scale;
    float acc[7][4];
#pragma unroll
    for (int j = 0; j < 7; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;

    for (int64_t blk = blockIdx.x; blk < n_blks; blk += gridDim.x) {
        const int64_t base = (blk * MOD_WARPS + warp) * 16;
        uint32_t inA[1][2][4];
        load_rows32(X, base, n, inA, g, q);
        uint32_t r1A[1][4][4], r2A[1][4][4];
        float oC[1][1][4];
        color_mlp<1>(inA, S.w.w1r, S.w.w2r, S.w.w3r, oC, g, q, [&](int l, const uint32_t (&r)[1][4][4]) {
#pragma unroll
            for (int kt = 0; kt < 4; ++kt)
#pragma unroll
                for (int e = 0; e < 4; ++e) (l == 1 ? r1A : r2A)[0][kt][e] = r[0][kt][e];
        });
        uint32_t doutA[1][1][4];
        doutA[0][0][2] = 0u; doutA[0][0][3] = 0u;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = base + g + 8 * h;
            float d0 = 0.f, d1 = 0.f;
            if (row < n && q < 2) {
                float s0 = oC[0][0][2 * h], s1 = oC[0][0][2 * h + 1];
                rgb_out_grad(s0, s1, act);
                if (q == 0) {
                    d0 = __ldg(dL_dout3 + 3 * row) * s0 * scale;
                    d1 = __ldg(dL_dout3 + 3 * row + 1) * s1 * scale;
                } else {
                    d0 = __ldg(dL_dout3 + 3 * row + 2) * s0 * scale;
                }
            }
            doutA[0][0][h] = pack_half2(d0, d1);
        }
        uint32_t dr2A[1][4][4], dr1A[1][4][4];
        {
            float c[1][8][4];
            mlp_layer_dgrad<16, 64, LD64>(doutA, S.w.w3r, c, lane);
            relu_bwd_to_frag<1, 64>(c, r2A, dr2A);
        }
        {
            float c[1][8][4];
            mlp_layer_dgrad<64, 64, LD64>(dr2A, S.w.w2r, c, lane);
            relu_bwd_to_frag<1, 64>(c, r1A, dr1A);
        }
        {
            float c[1][4][4];
            mlp_layer_dgrad<64, 32, LD32>(dr1A, S.w.w1r, c, lane);
            if (dL_dX) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t row = base + g + 8 * h;
                    if (row >= n) continue;
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        *reinterpret_cast<float2*>(dL_dX + row * 32 + 8 * j + 2 * q) =
                            make_float2(c[0][j][2 * h] * inv_scale, c[0][j][2 * h + 1] * inv_scale);
                }
            }
        }
        const int row0 = 16 * warp;
        stage_rows<2>(S.rin, LD32, row0, inA[0], g, q);
        stage_rows<4>(S.r1, LD64, row0, r1A[0], g, q);
        stage_rows<4>(S.r2, LD64, row0, r2A[0], g, q);
        stage_rows<4>(S.dr1, LD64, row0, dr1A[0], g, q);
        stage_rows<4>(S.dr2, LD64, row0, dr2A[0], g, q);
        stage_rows<1>(S.dout, LD16, row0, doutA[0], g, q);
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const ModTile w = rgb_tile_of(warp * 7 + j);
            if (w.mat == 0) wgrad_acc(acc[j], S.dr1, LD64, w.mt, S.rin, LD32, w.nt, lane);
            else if (w.mat == 1) wgrad_acc(acc[j], S.dr2, LD64, w.mt, S.r1, LD64, w.nt, lane);
            else wgrad_acc(acc[j], S.dout, LD16, w.mt, S.r2, LD64, w.nt, lane);
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 7; ++j) {
        const ModTile w = rgb_tile_of(warp * 7 + j);
        if (w.mat == 0) wgrad_out(acc[j], grad_rgb, 32, w.mt, w.nt, inv_scale, g, q);
        else if (w.mat == 1) wgrad_out(acc[j], grad_rgb + 2048, 64, w.mt, w.nt, inv_scale, g, q);
        else wgrad_out(acc[j], grad_rgb + 2048 + 4096, 64, w.mt, w.nt, inv_scale, g, q);
    }
}

extern "C" int ngp_mlp_rgb_backward(const uint16_t* rgb_params_h, const uint16_t* x_half, const float* dL_dout3, int64_t n,
                                    int rgb_act, const float* loss_scale, float* dL_dx, float* grad_rgb, void* stream) {
    // x_half is read as uint32 (load_rows32), dL_dx written as float2
    if (n < 0 || !rgb_params_h || !grad_rgb || (n > 0 && (!x_half || !dL_dout3)) || (((uintptr_t)x_half) & 3) ||
        (((uintptr_t)dL_dx) & 7))
        return NGP_EINVAL;
    if (n == 0) return 0;
    NGP_CUDA(ngp_smem_opt_in<k_mlp_rgb_bwd>((int)sizeof(RgbBwdSmem)));
    const int64_t n_blks = ((n + 15) / 16 + MOD_WARPS - 1) / MOD_WARPS;
    const int grid = (int)(n_blks < (int64_t)ngp_sm_count() ? n_blks : ngp_sm_count());
    k_mlp_rgb_bwd<<<grid, MOD_THREADS, sizeof(RgbBwdSmem), (cudaStream_t)stream>>>(
        (const __half*)rgb_params_h, (const __half*)x_half, dL_dout3, n, rgb_act, loss_scale, dL_dx, grad_rgb);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// backward of tcnn.NetworkWithInputEncoding from dL/dh (N,16)
// ---------------------------------------------------------------------------------------------------
struct EncBwdSmem {
    __half w1d[64 * LD32];
    __half w2d[16 * LD64];
    __half feat[MOD_ROWS * LD32];
    __half hid[MOD_ROWS * LD64];
    __half dhid[MOD_ROWS * LD64];
    __half dh[MOD_ROWS * LD16];
};

__global__ void __launch_bounds__(MOD_THREADS, 1)
k_enc_bwd(const __half* __restrict__ wd, const uint4* __restrict__ feat_save, const float* __restrict__ dL_dh, int64_t n,
          int n_levels, const float* __restrict__ loss_scale, float* __restrict__ grad_enc, uint32_t* __restrict__ dfeat,
          int64_t dfeat_stride) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    EncBwdSmem& S = *reinterpret_cast<EncBwdSmem*>(smem_raw);
    load_matrix(S.w1d, LD32, wd, 64, 32, threadIdx.x, MOD_THREADS);
    load_matrix(S.w2d, LD64, wd + 2048, 16, 64, threadIdx.x, MOD_THREADS);
    cp_async_wait_all();
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int64_t n_mtiles = (n + 15) / 16;
    const int64_t n_blks = (n_mtiles + MOD_WARPS - 1) / MOD_WARPS;
    const float scale = loss_scale ? *loss_scale : 1.0f;
    const float inv_scale = 1.0f / scale;
    float acc[3][4];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
    for (int64_t blk = blockIdx.x; blk < n_blks; blk += gridDim.x) {
        const int64_t mtile = blk * MOD_WARPS + warp;
        const int64_t base = mtile * 16;
        uint32_t featA[1][2][4];
#pragma unroll
        for (int kt = 0; kt < 2; ++kt) {
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (base < n) v = __ldg(feat_save + (mtile * 2 + kt) * 32 + lane);
            featA[0][kt][0] = v.x; featA[0][kt][1] = v.y; featA[0][kt][2] = v.z; featA[0][kt][3] = v.w;
        }
        uint32_t hidA[1][4][4];
        density_hidden<1>(featA, S.w1d, hidA, g, q);
        uint32_t dhA[1][1][4];
        {
            float c[1][2][4];
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t row = base + g + 8 * h;
                    float2 v = make_float2(0.f, 0.f);
                    if (row < n) v = __ldg(reinterpret_cast<const float2*>(dL_dh + row * 16 + 8 * j + 2 * q));
                    c[0][j][2 * h] = v.x * scale;
                    c[0][j][2 * h + 1] = v.y * scale;
                }
            to_frag<1, 16>(c, dhA);
        }
        uint32_t dhidA[1][4][4];
        {
            float c[1][8][4];
            mlp_layer_dgrad<16, 64, LD64>(dhA, S.w2d, c, lane);
            relu_bwd_to_frag<1, 64>(c, hidA, dhidA);
        }
        {
            float c[1][4][4];
            mlp_layer_dgrad<64, 32, LD32>(dhidA, S.w1d, c, lane);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = base + g + 8 * h;
                if (row >= n) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int level = 4 * j + q;
                    if (level < n_levels) dfeat[(int64_t)level * dfeat_stride + row] = pack_half2(c[0][j][2 * h], c[0][j][2 * h + 1]);
                }
            }
        }
        const int row0 = 16 * warp;
        stage_rows<2>(S.feat, LD32, row0, featA[0], g, q);
        stage_rows<4>(S.hid, LD64, row0, hidA[0], g, q);
        stage_rows<4>(S.dhid, LD64, row0, dhidA[0], g, q);
        stage_rows<1>(S.dh, LD16, row0, dhA[0], g, q);
        __syncthreads();
        // 24 tiles: W1d (4 x 4) -> warps take tiles 3w, 3w+1, 3w+2 of the list [W1d 0..15 | W2d 16..23]
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int t = warp * 3 + j;
            if (t < 16) wgrad_acc(acc[j], S.dhid, LD64, t >> 2, S.feat, LD32, t & 3, lane);
            else wgrad_acc(acc[j], S.dh, LD16, 0, S.hid, LD64, t - 16, lane);
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const int t = warp * 3 + j;
        if (t < 16) wgrad_out(acc[j], grad_enc, 32, t >> 2, t & 3, inv_scale, g, q);
        else wgrad_out(acc[j], grad_enc + 2048, 64, 0, t - 16, inv_scale, g, q);
    }
}

extern "C" int ngp_enc_backward(const NgpNet* net, const NgpSamples* smp, const float* dL_dh, const void* feat_save,
                                const float* loss_scale, float* grad_enc, void* workspace, size_t workspace_bytes, void* stream) {
    if (!net || !smp || smp->n < 0 || !grad_enc) return NGP_EINVAL;
    if (net->meta.n_levels < 1 || net->meta.n_levels > NGP_MAX_LEVELS) return NGP_EINVAL;
    if (smp->n == 0) return 0;
    if (!dL_dh || !feat_save || !workspace || workspace_bytes < ngp_net_backward_workspace(smp->n)) return NGP_EINVAL;
    // dL_dh is read as float2, feat_save as uint4
    if ((((uintptr_t)dL_dh) & 7) || (((uintptr_t)feat_save) & 15)) return NGP_EINVAL;
    NGP_CUDA(ngp_smem_opt_in<k_enc_bwd>((int)sizeof(EncBwdSmem)));
    const int64_t n_mtiles = (smp->n + 15) / 16;
    const int64_t n_blks = (n_mtiles + MOD_WARPS - 1) / MOD_WARPS;
    const int grid = (int)(n_blks < (int64_t)ngp_sm_count() ? n_blks : ngp_sm_count());
    k_enc_bwd<<<grid, MOD_THREADS, sizeof(EncBwdSmem), (cudaStream_t)stream>>>(
        (const __half*)net->enc_params_h, (const uint4*)feat_save, dL_dh, smp->n, net->meta.n_levels, loss_scale, grad_enc,
        (uint32_t*)workspace, n_mtiles * 16);
    NGP_CHECK_LAUNCH();
    return ngp_net_backward_scatter(net, smp, loss_scale, grad_enc, workspace, workspace_bytes, stream);
}
