// Warp-level tensor-core building blocks for the two 64-wide MLPs of NGP (the only dense contraction
// on the path). One warp owns MT row tiles of 16 samples; activations stay in mma fragments in
// registers from the hash gather to the output (the C fragment of layer i IS the A fragment of layer
// i+1 after ReLU + fp16 packing), weights live in shared memory, accumulation is fp32.
//
// mma.sync.m16n8k16 fragment layout (g = lane>>2, q = lane&3):
//   A (16x16 row-major): a0=(g, 2q..2q+1) a1=(g+8, 2q..) a2=(g, 2q+8..) a3=(g+8, 2q+8..)
//   B (16x8  col-major): b0=(k=2q..2q+1, n=g)   b1=(k=2q+8.., n=g)
//   C (16x8)           : c0,c1=(g, 2q..2q+1)    c2,c3=(g+8, 2q..2q+1)
// A weight matrix W[out][in] stored row-major is exactly the col-major B operand of Y = X * W^T.
#pragma once
#include "common.cuh"

__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ldmatrix (no transpose): four / two 8x8 b16 tiles; lane l supplies the address of row (l&7) of tile (l>>3).
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t& r0, uint32_t& r1, const void* smem_row) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(a));
}

// C[mt][N/8][4] = A[mt][K/16][4] x W^T, W = [N][LD] halfs in shared memory (LD = K + 8: rows are 16-byte aligned and
// eight consecutive rows fall into disjoint banks). The B fragments of TWO n-tiles (b0,b1 of tile j and of tile j+1) come
// from one ldmatrix.x4 -- row n of W, k = 0..7 / 8..15 of the k-step is exactly the (k = 2q.., n = g) fragment layout --
// instead of four 32-bit shared loads.
template <int MT, int K, int N, int LD>
__device__ __forceinline__ void mlp_layer(const uint32_t (&A)[MT][K / 16][4], const __half* __restrict__ W,
                                          float (&C)[MT][N / 8][4], int g, int q) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) C[mt][j][e] = 0.f;
    const int lane = 4 * g + q;
    const int lrow = lane & 7, lt = lane >> 3;  // ldmatrix: this lane addresses row lrow of tile lt
#pragma unroll
    for (int kt = 0; kt < K / 16; ++kt) {
        if (N / 8 >= 2) {
#pragma unroll
            for (int j = 0; j + 1 < N / 8; j += 2) {
                uint32_t b[4];
                ldmatrix_x4(b, W + (8 * (j + (lt >> 1)) + lrow) * LD + 16 * kt + 8 * (lt & 1));
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    mma_16816(C[mt][j], A[mt][kt], b[0], b[1]);
                    mma_16816(C[mt][j + 1], A[mt][kt], b[2], b[3]);
                }
            }
        } else {
            uint32_t b0, b1;
            ldmatrix_x2(b0, b1, W + lrow * LD + 16 * kt + 8 * (lt & 1));
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) mma_16816(C[mt][0], A[mt][kt], b0, b1);
        }
    }
}

// ReLU + fp16 pack: C fragments of a layer with N outputs -> A fragments (N/16 k-tiles) of the next.
template <int MT, int N>
__device__ __forceinline__ void relu_to_frag(const float (&C)[MT][N / 8][4], uint32_t (&A)[MT][N / 16][4]) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int kt = 0; kt < N / 16; ++kt) {
            A[mt][kt][0] = pack_half2(fmaxf(C[mt][2 * kt][0], 0.f), fmaxf(C[mt][2 * kt][1], 0.f));
            A[mt][kt][1] = pack_half2(fmaxf(C[mt][2 * kt][2], 0.f), fmaxf(C[mt][2 * kt][3], 0.f));
            A[mt][kt][2] = pack_half2(fmaxf(C[mt][2 * kt + 1][0], 0.f), fmaxf(C[mt][2 * kt + 1][1], 0.f));
            A[mt][kt][3] = pack_half2(fmaxf(C[mt][2 * kt + 1][2], 0.f), fmaxf(C[mt][2 * kt + 1][3], 0.f));
        }
}

// plain fp16 pack (no activation)
template <int MT, int N>
__device__ __forceinline__ void to_frag(const float (&C)[MT][N / 8][4], uint32_t (&A)[MT][N / 16][4]) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int kt = 0; kt < N / 16; ++kt) {
            A[mt][kt][0] = pack_half2(C[mt][2 * kt][0], C[mt][2 * kt][1]);
            A[mt][kt][1] = pack_half2(C[mt][2 * kt][2], C[mt][2 * kt][3]);
            A[mt][kt][2] = pack_half2(C[mt][2 * kt + 1][0], C[mt][2 * kt + 1][1]);
            A[mt][kt][3] = pack_half2(C[mt][2 * kt + 1][2], C[mt][2 * kt + 1][3]);
        }
}

// Backward through ReLU: gradient C fragments masked by the sign of the saved (post-ReLU, fp16)
// activation fragments, then packed to fp16 A fragments for the next dgrad.
__device__ __forceinline__ uint32_t mask_pack(float lo, float hi, uint32_t act) {
    const float2 a = unpack_half2(act);
    return pack_half2(a.x > 0.f ? lo : 0.f, a.y > 0.f ? hi : 0.f);
}
template <int MT, int N>
__device__ __forceinline__ void relu_bwd_to_frag(const float (&dC)[MT][N / 8][4], const uint32_t (&act)[MT][N / 16][4],
                                                 uint32_t (&dA)[MT][N / 16][4]) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int kt = 0; kt < N / 16; ++kt) {
            dA[mt][kt][0] = mask_pack(dC[mt][2 * kt][0], dC[mt][2 * kt][1], act[mt][kt][0]);
            dA[mt][kt][1] = mask_pack(dC[mt][2 * kt][2], dC[mt][2 * kt][3], act[mt][kt][1]);
            dA[mt][kt][2] = mask_pack(dC[mt][2 * kt + 1][0], dC[mt][2 * kt + 1][1], act[mt][kt][2]);
            dA[mt][kt][3] = mask_pack(dC[mt][2 * kt + 1][2], dC[mt][2 * kt + 1][3], act[mt][kt][3]);
        }
}

// ---- shared-memory weight block -----------------------------------------------------------------
// operands W[out][in] (+8 halfs of row padding); the backward reads the same block (mlp_layer_dgrad).
#define LD32 40
#define LD64 72
#define LD16 24
struct MlpWeightsFwd {
    __half w1d[64 * LD32];  // density 32 -> 64
    __half w2d[16 * LD64];  // density 64 -> 16
    __half w1r[64 * LD32];  // rgb 32 -> 64
    __half w2r[64 * LD64];  // rgb 64 -> 64
    __half w3r[16 * LD64];  // rgb 64 -> 16 (3 used)
};

// Row-major [rows][cols] global matrix -> padded shared rows, 16 bytes per cp.async (cols % 8 == 0, ld % 8 == 0, both
// bases 16-B aligned). The copies are asynchronous: call cp_async_wait_all() (+ __syncthreads()) before reading.
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

__device__ __forceinline__ void load_matrix(__half* dst, int ld, const __half* __restrict__ src, int rows, int cols,
                                            int tid, int nthreads) {
    const int cpr = cols >> 3;  // 16-byte chunks per row
    for (int i = tid; i < rows * cpr; i += nthreads) {
        const int r = i / cpr, c = i - r * cpr;
        cp_async_16(dst + r * ld + 8 * c, src + r * cols + 8 * c);
    }
}
__device__ __forceinline__ void load_weights_fwd(MlpWeightsFwd& s, const __half* __restrict__ wd, const __half* __restrict__ wr,
                                                 int tid, int nthreads) {
    load_matrix(s.w1d, LD32, wd, 64, 32, tid, nthreads);
    load_matrix(s.w2d, LD64, wd + 2048, 16, 64, tid, nthreads);
    if (wr) {
        load_matrix(s.w1r, LD32, wr, 64, 32, tid, nthreads);
        load_matrix(s.w2r, LD64, wr + 2048, 64, 64, tid, nthreads);
        load_matrix(s.w3r, LD64, wr + 2048 + 4096, 16, 64, tid, nthreads);
    }
    cp_async_wait_all();
}

// ldmatrix with transpose: four 8x8 b16 tiles; lane l supplies the address of row (l&7) of tile (l>>3).
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* smem_row) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(a));
}

// ---- backward (network.cu: k_ngp_bwd3, modules.cu) ------------------------------------------------

// dX[16 x N] = dY[16 x K] * W[K rows (out)][N cols (in)]  with W row-major (LD halfs per row) in shared
// memory: the B fragments (k = out row, n = in column) are the TRANSPOSE of what a plain 32-bit load of
// W gives, so they are fetched with ldmatrix.trans (two n-tiles per x4), no transposed weight copy needed.
template <int K, int N, int LD>
__device__ __forceinline__ void mlp_layer_dgrad(const uint32_t (&A)[1][K / 16][4], const __half* __restrict__ W,
                                                float (&C)[1][N / 8][4], int lane) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) C[0][j][e] = 0.f;
    const int row = (lane & 7) + 8 * ((lane >> 3) & 1);
    const int col = 8 * (lane >> 4);
#pragma unroll
    for (int kt = 0; kt < K / 16; ++kt) {
#pragma unroll
        for (int j = 0; j < N / 8; j += 2) {
            uint32_t b[4];
            ldmatrix_x4_trans(b, W + (16 * kt + row) * LD + 8 * j + col);
            mma_16816(C[0][j], A[0][kt], b[0], b[1]);
            mma_16816(C[0][j + 1], A[0][kt], b[2], b[3]);
        }
    }
}
