// The network's forward chains, written once for every kernel that runs them: k_ngp_fwd (network.cu), the
// forward recompute of k_ngp_bwd3 (network.cu) and the module kernels (modules.cu). Their fp16 rounding points, the
// form of the sigmoid and the order in which h feeds the colour net are what the float64 tests and the goldens pin.
// A kernel that keeps or stages a hidden activation gets it through a callback, called where the activation is
// produced, so that the kernel's instruction order is that of the chain written out in place.
#pragma once
#include "hashgrid.cuh"
#include "mlp.cuh"

__device__ __forceinline__ float half_round(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float lo_half(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu))); }

__device__ __forceinline__ float sel4(int q, float a, float b, float c, float d) {
    return q == 0 ? a : (q == 1 ? b : (q == 2 ? c : d));
}

// density MLP, first layer: 32 -> 64 (ReLU)
template <int MT>
__device__ __forceinline__ void density_hidden(const uint32_t (&featA)[MT][2][4], const __half* __restrict__ w1d,
                                               uint32_t (&hidA)[MT][4][4], int g, int q) {
    float c[MT][8][4];
    mlp_layer<MT, 32, 64, LD32>(featA, w1d, c, g, q);
    relu_to_frag<MT, 64>(c, hidA);
}

// density MLP 32 -> 64 (ReLU) -> 16 -> the fp16 h fragments (tinycudann returns fp16); on_hidden(hidA) sees the hidden
// activations
template <int MT, typename OnHidden>
__device__ __forceinline__ void density_mlp(const uint32_t (&featA)[MT][2][4], const __half* __restrict__ w1d,
                                            const __half* __restrict__ w2d, uint32_t (&hA)[MT][1][4], int g, int q,
                                            OnHidden&& on_hidden) {
    uint32_t hidA[MT][4][4];
    density_hidden<MT>(featA, w1d, hidA, g, q);
    on_hidden(hidA);
    float c[MT][2][4];
    mlp_layer<MT, 64, 16, LD64>(hidA, w2d, c, g, q);
    to_frag<MT, 16>(c, hA);
}

// sigma = exp(h[:,0]) in fp32 (reference networks.py:105, custom_functions.py:162-167), from a word of the h fragment
__device__ __forceinline__ float sigma_of_h(uint32_t h01) { return expf(lo_half(h01)); }

// SH-4 of the normalised direction, this lane's words of the colour input's k-tile 0
__device__ __forceinline__ void sh_rows(float dx, float dy, float dz, int q, uint32_t& lo, uint32_t& hi) {
    const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
    float sh[16];
    sh4(dx * inv, dy * inv, dz * inv, sh);
    lo = pack_half2(sel4(q, sh[0], sh[2], sh[4], sh[6]), sel4(q, sh[1], sh[3], sh[5], sh[7]));
    hi = pack_half2(sel4(q, sh[8], sh[10], sh[12], sh[14]), sel4(q, sh[9], sh[11], sh[13], sh[15]));
}

// the colour net's input [SH16(dir) | h16]: rows g and g + 8 of tile mt have the view directions s[mt][0], s[mt][1]
// (anything with members dx, dy, dz)
template <int MT, typename Dir>
__device__ __forceinline__ void color_input(const Dir (&s)[MT][2], const uint32_t (&hA)[MT][1][4], int q,
                                            uint32_t (&inA)[MT][2][4]) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int h = 0; h < 2; ++h) sh_rows(s[mt][h].dx, s[mt][h].dy, s[mt][h].dz, q, inA[mt][0][h], inA[mt][0][2 + h]);
#pragma unroll
        for (int e = 0; e < 4; ++e) inA[mt][1][e] = hA[mt][0][e];
    }
}

// colour MLP 32 -> 64 (ReLU) -> 64 (ReLU) -> 16 from its input fragments to the output accumulators; only output columns
// 0..7 are computed (rgb = 0..2). on_hidden(1, r1A) and on_hidden(2, r2A) see the two hidden activations.
template <int MT, typename OnHidden>
__device__ __forceinline__ void color_mlp(const uint32_t (&inA)[MT][2][4], const __half* __restrict__ w1r,
                                          const __half* __restrict__ w2r, const __half* __restrict__ w3r,
                                          float (&oC)[MT][1][4], int g, int q, OnHidden&& on_hidden) {
    uint32_t r1A[MT][4][4];
    {
        float c[MT][8][4];
        mlp_layer<MT, 32, 64, LD32>(inA, w1r, c, g, q);
        relu_to_frag<MT, 64>(c, r1A);
    }
    on_hidden(1, r1A);
    uint32_t r2A[MT][4][4];
    {
        float c[MT][8][4];
        mlp_layer<MT, 64, 64, LD64>(r1A, w2r, c, g, q);
        relu_to_frag<MT, 64>(c, r2A);
    }
    on_hidden(2, r2A);
    mlp_layer<MT, 64, 8, LD64>(r2A, w3r, oC, g, q);
}

__device__ __forceinline__ float sigmoid(float v) { return 1.0f / (1.0f + __expf(-v)); }
// the output activation of a lane's two output columns, rounded to fp16 as tinycudann returns it: sigmoid (rgb_act 1)
// or none
__device__ __forceinline__ __half2 rgb_out(float a, float b, int act) {
    if (act == 1) {
        a = sigmoid(a);
        b = sigmoid(b);
    }
    return __floats2half2_rn(a, b);
}
// its derivative at the same two pre-activations, taken at the rounded outputs o: o (1 - o) for the sigmoid, 1 for none
__device__ __forceinline__ void rgb_out_grad(float& a, float& b, int act) {
    float s0 = 1.0f, s1 = 1.0f;
    if (act == 1) {
        const float o0 = half_round(sigmoid(a));
        const float o1 = half_round(sigmoid(b));
        s0 = o0 * (1.0f - o0);
        s1 = o1 * (1.0f - o1);
    }
    a = s0;
    b = s1;
}
