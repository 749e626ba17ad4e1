// Front-to-back alpha compositing along one ray: the warp sweeps (32 samples per trip, transmittance as a warp-wide
// inclusive product scan with a carry between trips) and the serial loop of the test-time path. Every compositing
// kernel goes through this file, so the arithmetic and its order exist once.
//
// Semantics follow reference models/csrc/volumerendering.cu:6-45 (forward) and :87-151 (backward):
//   a_i = 1 - __expf(-sigma_i*delta_i);  w_i = a_i * T_{i-1};  T_i = T_{i-1}*(1-a_i)
//   the sample on which T first drops to <= T_threshold IS accumulated, later ones are not,
//   total_samples excludes that terminating sample, ws stays 0 past it.
// The reference accumulates serially per ray; a warp scan re-associates the fp32 sums/products
// (~1e-7 relative), which is inside the 1e-4 relative budget of the parity tests but not bit-exact.
#pragma once
#include "common.cuh"

// One ray's samples: pointers at its first sample (rgb holds three floats per sample).
struct RaySamples {
    const float *sg, *de, *t, *rgb;
};

struct CLSample {
    float sg, de, ti;
    float3 c;
};

// Sample i of the ray; zeros past its n samples.
__device__ __forceinline__ void cl_load(CLSample& x, const RaySamples& s, int i, int n) {
    x.sg = 0.f; x.de = 0.f; x.ti = 0.f; x.c = make_float3(0.f, 0.f, 0.f);
    if (i < n) {
        x.sg = __ldg(s.sg + i);
        x.de = __ldg(s.de + i);
        x.ti = __ldg(s.t + i);
        x.c = make_float3(__ldg(s.rgb + 3 * i), __ldg(s.rgb + 3 * i + 1), __ldg(s.rgb + 3 * i + 2));
    }
}

// What one trip hands to the next.
struct TripCarry {
    float T = 1.0f;    // transmittance after the trip's last sample
    int n_comp = 0;    // samples composited so far
    bool done = false; // the ray terminated inside the trip
};

struct TripHead {
    bool valid, comp;  // comp: the transmittance BEFORE the sample is still above the threshold (the first always is)
    float T_inc, w;    // transmittance after the sample, its weight (0 unless comp)
};

// Sample i = base + lane of one trip: its weight from the warp-wide transmittance scan, and the carry to the next trip.
__device__ __forceinline__ TripHead trip_head(TripCarry& c, const CLSample& x, int i, int n, float T_threshold, int lane) {
    TripHead h;
    h.valid = i < n;
    const float a = h.valid ? 1.0f - __expf(-(x.sg * x.de)) : 0.f;
    h.T_inc = warp_scan_mul(1.0f - a, lane) * c.T;
    float T_exc = __shfl_up_sync(0xffffffffu, h.T_inc, 1);
    if (lane == 0) T_exc = c.T;
    h.comp = h.valid && (i == 0 || T_exc > T_threshold);
    h.w = h.comp ? a * T_exc : 0.f;
    c.n_comp += __popc(__ballot_sync(0xffffffffu, h.comp));
    c.done = __ballot_sync(0xffffffffu, h.valid && !(h.T_inc > T_threshold)) != 0u;
    c.T = __shfl_sync(0xffffffffu, h.T_inc, 31);
    return h;
}

struct CompositeOut {
    float r, g, b, depth, opacity;
    int n_composited;   // samples that received a non-zero weight slot (includes the terminating one)
    int total_samples;  // reference `total_samples[ray]`
};

// The sweeps below walk a ray trip by trip until it terminates. The first CACHE trips come from `cache` (samples the
// caller holds in registers, loaded with cl_load); later trips load their samples from `s`.

// Forward of one ray by one warp. ws (may be null) receives every sample's weight, 0 past termination.
template <int CACHE>
__device__ __forceinline__ CompositeOut composite_ray_warp(const RaySamples& s, int n, float T_threshold, int lane,
                                                           const CLSample* cache, float* ws) {
    float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_d = 0.f, acc_o = 0.f;
    TripCarry c;
    auto trip = [&](int base, const CLSample& x) {
        const int i = base + lane;
        const TripHead h = trip_head(c, x, i, n, T_threshold, lane);
        if (h.comp) {
            acc_r = fmaf(h.w, x.c.x, acc_r);
            acc_g = fmaf(h.w, x.c.y, acc_g);
            acc_b = fmaf(h.w, x.c.z, acc_b);
            acc_d = fmaf(h.w, x.ti, acc_d);
            acc_o += h.w;
        }
        if (ws && h.valid) ws[i] = h.w;
    };
    int base = 0;
#pragma unroll
    for (int k = 0; k < CACHE; ++k)
        if (k * 32 < n && !c.done) { trip(k * 32, cache[k]); base = k * 32 + 32; }
    for (; base >= CACHE * 32 && base < n && !c.done; base += 32) {
        CLSample x;
        cl_load(x, s, base + lane, n);
        trip(base, x);
    }
    if (ws)
        for (int i = base + lane; i < n; i += 32) ws[i] = 0.f;  // past the terminating trip

    CompositeOut o;
    o.r = warp_sum(acc_r);
    o.g = warp_sum(acc_g);
    o.b = warp_sum(acc_b);
    o.depth = warp_sum(acc_d);
    o.opacity = warp_sum(acc_o);
    o.n_composited = c.n_comp;
    o.total_samples = c.done ? c.n_comp - 1 : c.n_comp;
    return o;
}

struct CompositeBwdOut {
    int n_composited;  // the ray's leading samples, terminating one included: only those get a non-zero gradient
    float m;           // this lane's max of |dL/drgb| and |dL/dsigma * min(sigma, 3.2690173e6)| (fp16 loss scale)
};

// Backward of the above for one ray by one warp, from the upstream gradients dC, dO, dD of the composited colour,
// opacity and depth (C, O, D). dsig / drgb receive every sample's gradient, 0 past termination.
// DEPTH_WS adds the depth term and the ws term (dws = dL/dws, null for none; ws = the forward's weights, read whenever
// dws is not null, so it must not be null then); without it dD and the ws gradient are taken to be zero and their scans
// are skipped.
template <int CACHE, bool DEPTH_WS>
__device__ __forceinline__ CompositeBwdOut composite_ray_warp_bwd(const RaySamples& s, int n, float T_threshold, int lane,
                                                                  const CLSample* cache, float3 dC, float dO, float dD,
                                                                  float3 C, float O, float D, const float* dws,
                                                                  const float* ws, float* dsig, float* drgb) {
    // total of dL/dws * ws over the ray (ws is 0 past termination)
    float s_tot = 0.f;
    if (DEPTH_WS && dws) {
        for (int i = lane; i < n; i += 32) s_tot = fmaf(__ldg(dws + i), __ldg(ws + i), s_tot);
        s_tot = warp_sum(s_tot);
    }
    const float dO_term = dO * (1.0f - O);
    float m = 0.f;
    TripCarry c;
    float pr = 0.f, pg = 0.f, pb = 0.f, pd = 0.f, ps = 0.f;  // inclusive prefixes carried between trips
    auto trip = [&](int base, const CLSample& x) {
        const int i = base + lane;
        const TripHead h = trip_head(c, x, i, n, T_threshold, lane);
        const float r_inc = warp_scan_add(h.w * x.c.x, lane) + pr;
        const float g_inc = warp_scan_add(h.w * x.c.y, lane) + pg;
        const float b_inc = warp_scan_add(h.w * x.c.z, lane) + pb;
        float d_inc = 0.f, s_inc = 0.f, dw = 0.f;
        if (DEPTH_WS) {
            float wv = 0.f;
            if (h.valid && dws) {
                dw = __ldg(dws + i);
                wv = __ldg(ws + i);
            }
            d_inc = warp_scan_add(h.w * x.ti, lane) + pd;
            s_inc = warp_scan_add(dw * wv, lane) + ps;
        }
        if (h.valid) {
            float3 dcv = make_float3(0.f, 0.f, 0.f);
            float dsv = 0.f;
            if (h.comp) {
                dcv = make_float3(dC.x * h.w, dC.y * h.w, dC.z * h.w);
                float g = dC.x * (x.c.x * h.T_inc - (C.x - r_inc)) + dC.y * (x.c.y * h.T_inc - (C.y - g_inc)) +
                          dC.z * (x.c.z * h.T_inc - (C.z - b_inc)) + dO_term;
                if (DEPTH_WS) g = g + dD * (x.ti * h.T_inc - (D - d_inc)) + (h.T_inc * dw - (s_tot - s_inc));
                dsv = x.de * g;
            }
            drgb[3 * i] = dcv.x; drgb[3 * i + 1] = dcv.y; drgb[3 * i + 2] = dcv.z;
            dsig[i] = dsv;
            m = fmaxf(m, fmaxf(fabsf(dcv.x), fmaxf(fabsf(dcv.y), fabsf(dcv.z))));
            m = fmaxf(m, fabsf(dsv * fminf(x.sg, 3.2690173e6f)));
        }
        pr = __shfl_sync(0xffffffffu, r_inc, 31);
        pg = __shfl_sync(0xffffffffu, g_inc, 31);
        pb = __shfl_sync(0xffffffffu, b_inc, 31);
        if (DEPTH_WS) {
            pd = __shfl_sync(0xffffffffu, d_inc, 31);
            ps = __shfl_sync(0xffffffffu, s_inc, 31);
        }
    };
    int base = 0;
#pragma unroll
    for (int k = 0; k < CACHE; ++k)
        if (k * 32 < n && !c.done) { trip(k * 32, cache[k]); base = k * 32 + 32; }
    for (; base >= CACHE * 32 && base < n && !c.done; base += 32) {
        CLSample x;
        cl_load(x, s, base + lane, n);
        trip(base, x);
    }
    for (int i = base + lane; i < n; i += 32) {  // past the terminating trip
        drgb[3 * i] = 0.f; drgb[3 * i + 1] = 0.f; drgb[3 * i + 2] = 0.f;
        dsig[i] = 0.f;
    }
    return {c.n_comp, m};
}

// Test-time compositing of one ray by one thread, serially: its n samples start at index `first` of the sample arrays
// `s` and are composited onto what earlier rounds accumulated in r, g, b, depth, opacity. Returns true when the ray
// terminated: its transmittance fell to T_threshold. (The index type is the caller's: the arrays are kernel arguments,
// and adding `first` to them once per ray would hold four 64-bit pointers per thread.)
template <class I>
__device__ __forceinline__ bool composite_ray_serial(const RaySamples& s, I first, int n, float T_threshold, float& r,
                                                     float& g, float& b, float& depth, float& opacity) {
    float T = 1.0f - opacity;
    for (int j = 0; j < n; ++j) {
        const I k = first + j;
        const float a = 1.0f - __expf(-(__ldg(s.sg + k) * __ldg(s.de + k)));
        const float w = a * T;
        r = fmaf(w, __ldg(s.rgb + 3 * k), r);
        g = fmaf(w, __ldg(s.rgb + 3 * k + 1), g);
        b = fmaf(w, __ldg(s.rgb + 3 * k + 2), b);
        depth = fmaf(w, __ldg(s.t + k), depth);
        opacity += w;
        T *= 1.0f - a;
        if (T <= T_threshold) return true;
    }
    return false;
}

// NeRFLoss of one ray (reference losses.py:47-60, lambda_distortion = 0) over a batch of n rays (inv_n = 1/n): its
// squared colour error and opacity entropy, and its gradients with respect to the ray's colour and opacity.
struct NerfLossRay {
    float3 dC;
    // n * dL/dopacity, before any background routing. The caller scales it by inv_n; the fused kernel folds the
    // background routing into that multiply (one rounding), the separate path rounds dL/dopacity first.
    float dO_n;
    float se, ent;
};
__device__ __forceinline__ NerfLossRay nerf_loss_ray(float3 rgb, float3 rgb_gt, float opacity, float lambda_opacity,
                                                     float inv_n) {
    NerfLossRay l;
    const float ex = rgb.x - rgb_gt.x, ey = rgb.y - rgb_gt.y, ez = rgb.z - rgb_gt.z;
    l.dC = make_float3(2.0f * ex * inv_n * (1.0f / 3.0f), 2.0f * ey * inv_n * (1.0f / 3.0f), 2.0f * ez * inv_n * (1.0f / 3.0f));
    l.se = ex * ex + ey * ey + ez * ez;
    const float op = opacity + 1e-10f;
    const float lg = logf(op);
    l.ent = -op * lg;
    l.dO_n = lambda_opacity * (-lg - 1.0f);
    return l;
}
