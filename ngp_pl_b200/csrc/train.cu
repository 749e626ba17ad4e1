// Fused training path for sm_90a: everything render(test_time=False) does (reference
// models/rendering.py:11-43,:121-163) plus loss, optimiser, batch assembly and the occupancy-grid
// refresh, as a handful of stream-ordered launches with NO host synchronisation (sample counts never
// leave the device), so a whole optimiser step can be captured in one CUDA graph.
#include "common.cuh"
#include "march.cuh"
#include "composite.cuh"
#include "../../include/ngp_b200.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

// -------------------------------------------------------------------------------------------------
// 1. AABB + near clamp + jittered march, ONE pass: samples go to a per-ray staging row
//    (reference intersection.cu:25-56, rendering.py:29, raymarching.cu:166-235)
// -------------------------------------------------------------------------------------------------
template <bool CONST_DT, bool ONE_CASCADE>
__global__ void k_train_march(const NgpTrainCfg cfg, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                              const float* __restrict__ noise, const uint8_t* __restrict__ bitfield,
                              float* __restrict__ stage_t, float* __restrict__ stage_dt, int* __restrict__ n_samples,
                              int* __restrict__ offsets, int* __restrict__ ray_idx, float* __restrict__ ts,
                              float* __restrict__ deltas, int* __restrict__ counters, int* __restrict__ acc) {
    // one WARP per ray (march_ray_warp): 32 chain points probed side by side, same t sequence as the serial loop
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r < cfg.n_rays) {
        const MarchConst c = make_march_const(bitfield, cfg.cascades, cfg.grid_size, cfg.max_samples, cfg.scale,
                                              cfg.exp_step_factor, cfg.scale);
        const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                            rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
        const float2 tt = ray_aabb(ray, cfg.center[0], cfg.center[1], cfg.center[2], cfg.half_size[0], cfg.half_size[1],
                                   cfg.half_size[2]);
        float t1 = -1.0f, t2 = -1.0f;
        if (tt.y > 0.0f) {
            t1 = fmaxf(tt.x, 0.0f);
            t2 = tt.y;
        }
        if (t1 >= 0.0f && t1 < cfg.near_distance) t1 = cfg.near_distance;
        const float t = march_jitter(t1, noise[r], c);
        float* st = stage_t + (size_t)r * cfg.max_samples;
        float* sd = stage_dt + (size_t)r * cfg.max_samples;
        const int n = march_ray_warp<CONST_DT, ONE_CASCADE>(ray, c, t, t2, cfg.max_samples, lane, [&](int k, float ts_, float dts) {
            st[k] = ts_;
            sd[k] = dts;
        });
        // The ray's segment of the compact per-sample arrays: claimed with one atomic, in arrival order like the reference's
        // rays_a (raymarching.cu:237-241) -- every consumer goes through offsets[ray] / n_samples[ray], none needs the
        // segments sorted by ray. Replaces a prefix-sum kernel and a compaction kernel; the staging row just written by this
        // warp is still in L1/L2 when it is copied out.
        int start = 0;
        if (lane == 0) {
            start = atomicAdd(&acc[0], n);
            n_samples[r] = n;
            offsets[r] = start;
        }
        start = __shfl_sync(0xffffffffu, start, 0);
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            const int64_t s = (int64_t)start + i;
            if (s < cfg.max_total_samples) {
                ray_idx[s] = r;
                ts[s] = st[i];
                deltas[s] = sd[i];
            }
        }
    }
    // the last block to finish publishes the total and re-arms the accumulators (the network kernels read counters[0];
    // a trainer may already be marching the NEXT batch into another buffer set, with its own counters and accumulators)
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&acc[1], 1) == (int)gridDim.x - 1) {
            const int tot = atomicAdd(&acc[0], 0);
            counters[0] = (int)((int64_t)tot < cfg.max_total_samples ? tot : cfg.max_total_samples);
            counters[1] = 0;
            counters[4] = 0;
            acc[0] = 0;
            acc[1] = 0;
        }
    }
}

// 5. ragged compositing of the network outputs, one warp per ray, + background
__global__ void k_train_composite_fw(const NgpTrainCfg cfg, const int* __restrict__ n_samples, const int* __restrict__ offsets,
                                     const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                     const float* __restrict__ deltas, const float* __restrict__ ts,
                                     float* __restrict__ rgb, float* __restrict__ opacity, float* __restrict__ depth,
                                     float* __restrict__ ws, int* __restrict__ counters, const float* __restrict__ bg_dev) {
    const float bg[3] = {bg_dev ? bg_dev[0] : cfg.bg[0], bg_dev ? bg_dev[1] : cfg.bg[1], bg_dev ? bg_dev[2] : cfg.bg[2]};
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= cfg.n_rays) return;
    const int64_t start = offsets[w];
    int n = n_samples[w];
    if (start + n > cfg.max_total_samples) n = (int)max((int64_t)0, cfg.max_total_samples - start);
    const float* sg = sigmas + start;
    const float* dl = deltas + start;
    const float* tt = ts + start;
    const float* cl = rgbs + 3 * start;
    float* wo = ws ? ws + start : nullptr;
    const CompositeOut o = composite_ray_warp(
        n, cfg.T_threshold, lane,
        [&](int i) { return __ldg(sg + i); }, [&](int i) { return __ldg(dl + i); }, [&](int i) { return __ldg(tt + i); },
        [&](int i) { return make_float3(__ldg(cl + 3 * i), __ldg(cl + 3 * i + 1), __ldg(cl + 3 * i + 2)); },
        [&](int i, float v) { if (wo) wo[i] = v; });
    if (lane == 0) {
        const float rest = 1.0f - o.opacity;  // rgb += bg * (1 - opacity), reference rendering.py:160-161
        opacity[w] = o.opacity;
        depth[w] = o.depth;
        rgb[3 * w] = o.r + bg[0] * rest;
        rgb[3 * w + 1] = o.g + bg[1] * rest;
        rgb[3 * w + 2] = o.b + bg[2] * rest;
        if (o.total_samples) atomicAdd(&counters[1], o.total_samples);
    }
}

extern "C" size_t ngp_train_scan_temp_bytes(int n_rays) {
    (void)n_rays;
    return 256;  // two int32 accumulators of the march kernel's segment allocation (zero-initialised ONCE by the caller)
}

static NgpSamples train_samples(const NgpTrainCfg* cfg, const NgpTrainBuffers* b) {
    NgpSamples s;
    s.xyzs = nullptr; s.dirs = nullptr;
    s.rays_o = b->rays_o; s.rays_d = b->rays_d;
    s.ray_idx = b->ray_idx; s.ts = b->ts;
    s.n = cfg->max_total_samples;
    s.n_dev = b->counters;
    s.live_idx = nullptr;
    s.n_live_dev = nullptr;
    return s;
}

static int check_train_args(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* b) {
    if (!net || !cfg || !b) return NGP_EINVAL;
    if (cfg->n_rays < 1 || cfg->cascades < 1 || cfg->grid_size < 1 || cfg->grid_size > 1024 || cfg->max_samples < 1 ||
        cfg->max_total_samples < 1 || cfg->max_total_samples > 0x7fffffffll)
        return NGP_EINVAL;
    if (!b->rays_o || !b->rays_d || !b->noise || !b->density_bitfield || !b->stage_t || !b->stage_dt || !b->n_samples ||
        !b->offsets || !b->counters || !b->rgb || !b->opacity || !b->depth || !b->ray_idx || !b->ts || !b->deltas ||
        !b->sigmas || !b->rgbs || !b->scalars || !b->scan_temp)
        return NGP_EINVAL;
    return 0;
}

// first half of the forward: AABB + march + segment allocation + compaction in ONE kernel. Depends only on the rays, the jitter
// and the occupancy bitfield (NOT on the network weights), so a trainer may run it for step i+1 while the
// optimiser of step i is still updating the weights.
extern "C" int ngp_render_train_march(const NgpTrainCfg* cfg, const NgpTrainBuffers* b, void* stream) {
    NgpNet dummy;
    int rc = check_train_args(&dummy, cfg, b);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int n = cfg->n_rays;
    const bool const_dt = march_const_dt(cfg->exp_step_factor, cfg->max_samples, cfg->scale, cfg->grid_size);
    const dim3 mg(ngp_div_up((int64_t)n * 32, 128));
    // accumulators of the march kernel's segment allocation: two ints at the head of scan_temp, zero between launches
    // (zeroed once by the caller -- torch allocates scan_temp zero-filled in the Trainer -- and re-armed by the kernel)
    int* acc = (int*)b->scan_temp;
    march_dispatch(const_dt, cfg->cascades, [&](auto cd, auto oc) {
        k_train_march<decltype(cd)::value, decltype(oc)::value><<<mg, 128, 0, st>>>(
            *cfg, b->rays_o, b->rays_d, b->noise, b->density_bitfield, b->stage_t, b->stage_dt, b->n_samples, b->offsets,
            b->ray_idx, b->ts, b->deltas, b->counters, acc);
    });
    NGP_CHECK_LAUNCH();
    NGP_TRACE(2, st);
    return 0;
}

// second half of the forward: network on the marched samples + ragged compositing
extern "C" int ngp_render_train_net(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* b, void* stream) {
    int rc = check_train_args(net, cfg, b);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int n = cfg->n_rays;
    const NgpSamples smp = train_samples(cfg, b);
    rc = ngp_net_forward(net, &smp, 1, b->sigmas, b->rgbs, nullptr, b->feat_save, stream);
    if (rc) return rc;
    k_train_composite_fw<<<ngp_div_up((int64_t)n * 32, 128), 128, 0, st>>>(*cfg, b->n_samples, b->offsets, b->sigmas, b->rgbs,
                                                                            b->deltas, b->ts, b->rgb, b->opacity, b->depth,
                                                                            b->ws, b->counters, b->bg_dev);
    NGP_CHECK_LAUNCH();
    return 0;
}

extern "C" int ngp_render_train_fwd(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* b, void* stream) {
    int rc = ngp_render_train_march(cfg, b, stream);
    if (rc) return rc;
    return ngp_render_train_net(net, cfg, b, stream);
}

// -------------------------------------------------------------------------------------------------
// backward: compositing backward per ray (+ running max for the fp16 loss scale), then the network
// -------------------------------------------------------------------------------------------------
__global__ void k_train_composite_bw(const NgpTrainCfg cfg, const int* __restrict__ n_samples, const int* __restrict__ offsets,
                                     const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                     const float* __restrict__ deltas, const float* __restrict__ ts,
                                     const float* __restrict__ ws, const float* __restrict__ rgb,
                                     const float* __restrict__ opacity, const float* __restrict__ depth,
                                     const float* __restrict__ dL_drgb, const float* __restrict__ dL_dopacity,
                                     const float* __restrict__ dL_ddepth, const float* __restrict__ dL_dws,
                                     float* __restrict__ dsigmas, float* __restrict__ drgbs, float* __restrict__ amax,
                                     int* __restrict__ live_idx, int* __restrict__ counters, const float* __restrict__ bg_dev) {
    const float bg[3] = {bg_dev ? bg_dev[0] : cfg.bg[0], bg_dev ? bg_dev[1] : cfg.bg[1], bg_dev ? bg_dev[2] : cfg.bg[2]};
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= cfg.n_rays) return;
    const int64_t start = offsets[w];
    int n = n_samples[w];
    if (start + n > cfg.max_total_samples) n = (int)max((int64_t)0, cfg.max_total_samples - start);
    if (n == 0) return;
    const float* sg = sigmas + start;
    const float* dl = deltas + start;
    const float* tt = ts + start;
    const float* cl = rgbs + 3 * start;
    const float* wv = ws ? ws + start : nullptr;
    const float* dw = dL_dws ? dL_dws + start : nullptr;
    float* ds = dsigmas + start;
    float* dc = drgbs + 3 * start;
    const float3 dC = make_float3(dL_drgb[3 * w], dL_drgb[3 * w + 1], dL_drgb[3 * w + 2]);
    // the forward output is acc + bg*(1-O): undo the background to get the accumulated colour, and
    // route its gradient into the opacity gradient
    const float O = opacity[w];
    const float rest = 1.0f - O;
    const float3 C = make_float3(rgb[3 * w] - bg[0] * rest, rgb[3 * w + 1] - bg[1] * rest, rgb[3 * w + 2] - bg[2] * rest);
    const float dO = dL_dopacity[w] - (dC.x * bg[0] + dC.y * bg[1] + dC.z * bg[2]);
    const float dD = dL_ddepth ? dL_ddepth[w] : 0.f;
    float m = 0.f;
    const int n_comp = composite_ray_warp_bwd(
        n, cfg.T_threshold, lane, dO, dD, dC, O, depth[w], C,
        [&](int i) { return __ldg(sg + i); }, [&](int i) { return __ldg(dl + i); }, [&](int i) { return __ldg(tt + i); },
        [&](int i) { return make_float3(__ldg(cl + 3 * i), __ldg(cl + 3 * i + 1), __ldg(cl + 3 * i + 2)); },
        [&](int i) { return dw ? __ldg(dw + i) : 0.f; }, [&](int i) { return (dw && wv) ? __ldg(wv + i) : 0.f; },
        [&](int i, float v) {
            ds[i] = v;
            m = fmaxf(m, fabsf(v * fminf(__ldg(sg + i), 3.2690173e6f)));
        },
        [&](int i, float3 v) {
            dc[3 * i] = v.x; dc[3 * i + 1] = v.y; dc[3 * i + 2] = v.z;
            m = fmaxf(m, fmaxf(fabsf(v.x), fmaxf(fabsf(v.y), fabsf(v.z))));
        });
    m = warp_max(m);
    if (lane == 0 && m > 0.f && m < INFINITY) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));
    // the composited samples are the ray's leading n_comp: append them to the list the network backward visits
    // (every other sample has dsigmas = drgbs = 0 exactly and would only add zeros)
    if (live_idx) {
        int at = 0;
        if (lane == 0) at = atomicAdd(&counters[4], n_comp);
        at = __shfl_sync(0xffffffffu, at, 0);
        for (int i = lane; i < n_comp; i += 32) live_idx[at + i] = (int)(start + i);
    }
}

__global__ void k_train_grad_scale(float* __restrict__ scalars, int* __restrict__ counters, const int fused_loss) {
    // the live list is complete: publish its length and re-arm the append counter, so that counters[4] is zero
    // whenever a compositing backward starts, whatever the caller's order of calls
    counters[5] = counters[4];
    counters[4] = 0;
    // fused compositing + loss kernel: publish its sums ([4],[5] -> [2],[3]) and this step's sample counts, re-arm
    // (unconditionally: a step whose sums are exactly zero must not leave the previous step's numbers behind)
    if (fused_loss) {
        scalars[2] = scalars[4];
        scalars[3] = scalars[5];
        scalars[4] = 0.f;
        scalars[5] = 0.f;
        counters[2] = counters[0];
        counters[3] = counters[1];
    }
    const float m = scalars[0];
    float s = 1.0f;
    if (m > 0.f && m < INFINITY) {
        int e;
        frexpf(256.0f / m, &e);
        e = max(-60, min(60, e - 1));
        s = scalbnf(1.0f, e);
    }
    scalars[1] = s;
    scalars[0] = 0.f;
}

// compositing forward + NeRFLoss + compositing backward of one ray in ONE pass by one warp (the loss gradient of a ray
// depends on that ray's composited colour / opacity only): k_train_composite_fw + k_nerf_loss_grad + k_train_composite_bw
// without the two extra launches and with the second sweep over the ray's samples hitting L1/L2.
#define CL_WARPS 8  // rays per block of k_train_composite_loss
#define CL_CACHE 4  // trips (of 32 samples) of a ray held in registers between the forward and the backward sweep (64 regs)
struct CLSample {
    float sg, de, ti;
    float3 c;
};
__device__ __forceinline__ CLSample cl_load(const float* __restrict__ sg, const float* __restrict__ dl,
                                            const float* __restrict__ tt, const float* __restrict__ cl, int i) {
    CLSample x;
    x.sg = __ldg(sg + i);
    x.de = __ldg(dl + i);
    x.ti = __ldg(tt + i);
    x.c = make_float3(__ldg(cl + 3 * i), __ldg(cl + 3 * i + 1), __ldg(cl + 3 * i + 2));
    return x;
}
__global__ void __launch_bounds__(CL_WARPS * 32) k_train_composite_loss(const NgpTrainCfg cfg, const int* __restrict__ n_samples, const int* __restrict__ offsets,
                                       const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                       const float* __restrict__ deltas, const float* __restrict__ ts,
                                       const float* __restrict__ rgb_gt, float* __restrict__ rgb, float* __restrict__ opacity,
                                       float* __restrict__ depth, float* __restrict__ dsigmas, float* __restrict__ drgbs,
                                       float* __restrict__ scalars, int* __restrict__ live_idx, int* __restrict__ counters,
                                       const float* __restrict__ bg_dev) {
    const float bg[3] = {bg_dev ? bg_dev[0] : cfg.bg[0], bg_dev ? bg_dev[1] : cfg.bg[1], bg_dev ? bg_dev[2] : cfg.bg[2]};
    const int lane = threadIdx.x & 31;
    // (n_rays is a multiple of the rays per block or the last block's spare warps idle on ray n_rays - 1 with n = 0 and
    // contribute nothing: every warp must reach the block barriers below)
    const int w_raw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const bool real = w_raw < cfg.n_rays;
    const int w = real ? w_raw : cfg.n_rays - 1;
    const int64_t start = offsets[w];
    int n = real ? n_samples[w] : 0;
    if (start + n > cfg.max_total_samples) n = (int)max((int64_t)0, cfg.max_total_samples - start);
    const float* sg = sigmas + start;
    const float* dl = deltas + start;
    const float* tt = ts + start;
    const float* cl = rgbs + 3 * start;
    // The ray's first CL_CACHE trips of 32 samples are loaded up front (independent loads, one exposed latency instead of
    // one per trip) and kept in registers for the backward sweep; longer rays continue trip by trip from memory. The
    // kernel is two waves of warps and lasts as long as its longest rays: with the generic helpers (a dependent load ->
    // scan chain per trip, twice) those chains were what it waited on. Arithmetic and its order are those of
    // composite_ray_warp / composite_ray_warp_bwd (composite.cuh), minus the depth and ws scans whose gradients are zero.
    CLSample sm[CL_CACHE];
#pragma unroll
    for (int k = 0; k < CL_CACHE; ++k) {
        const int i = k * 32 + lane;
        sm[k].sg = 0.f; sm[k].de = 0.f; sm[k].ti = 0.f; sm[k].c = make_float3(0.f, 0.f, 0.f);
        if (i < n) sm[k] = cl_load(sg, dl, tt, cl, i);
    }
    CompositeOut o;
    {
        float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_d = 0.f, acc_o = 0.f, T_carry = 1.0f;
        int n_comp = 0;
        bool done = false;
        auto trip = [&](int base, const CLSample& x) {
            const int i = base + lane;
            const bool valid = i < n;
            const float a = valid ? 1.0f - __expf(-(x.sg * x.de)) : 0.f;
            const float T_inc = warp_scan_mul(1.0f - a, lane) * T_carry;
            float T_exc = __shfl_up_sync(0xffffffffu, T_inc, 1);
            if (lane == 0) T_exc = T_carry;
            const bool comp = valid && (i == 0 || T_exc > cfg.T_threshold);
            const float w = comp ? a * T_exc : 0.f;
            if (comp) {
                acc_r = fmaf(w, x.c.x, acc_r);
                acc_g = fmaf(w, x.c.y, acc_g);
                acc_b = fmaf(w, x.c.z, acc_b);
                acc_d = fmaf(w, x.ti, acc_d);
                acc_o += w;
            }
            n_comp += __popc(__ballot_sync(0xffffffffu, comp));
            done = __ballot_sync(0xffffffffu, valid && !(T_inc > cfg.T_threshold)) != 0u;
            T_carry = __shfl_sync(0xffffffffu, T_inc, 31);
        };
#pragma unroll
        for (int k = 0; k < CL_CACHE; ++k)
            if (k * 32 < n && !done) trip(k * 32, sm[k]);
        for (int base = CL_CACHE * 32; base < n && !done; base += 32) {
            CLSample x;
            x.sg = 0.f; x.de = 0.f; x.ti = 0.f; x.c = make_float3(0.f, 0.f, 0.f);
            if (base + lane < n) x = cl_load(sg, dl, tt, cl, base + lane);
            trip(base, x);
        }
        o.r = warp_sum(acc_r);
        o.g = warp_sum(acc_g);
        o.b = warp_sum(acc_b);
        o.depth = warp_sum(acc_d);
        o.opacity = warp_sum(acc_o);
        o.n_composited = n_comp;
        o.total_samples = done ? n_comp - 1 : n_comp;
    }
    const float rest = 1.0f - o.opacity;  // rgb += bg * (1 - opacity), reference rendering.py:160-161
    const float3 out = make_float3(o.r + bg[0] * rest, o.g + bg[1] * rest, o.b + bg[2] * rest);
    // NeRFLoss (reference losses.py:47-60, lambda_distortion = 0) and its per-ray gradients
    const float inv_n = 1.0f / (float)cfg.n_rays;
    const float ex = out.x - rgb_gt[3 * w], ey = out.y - rgb_gt[3 * w + 1], ez = out.z - rgb_gt[3 * w + 2];
    const float3 dC = make_float3(2.0f * ex * inv_n * (1.0f / 3.0f), 2.0f * ey * inv_n * (1.0f / 3.0f), 2.0f * ez * inv_n * (1.0f / 3.0f));
    const float op = o.opacity + 1e-10f;
    const float lg = logf(op);
    if (lane == 0 && real) {
        opacity[w] = o.opacity;
        depth[w] = o.depth;
        rgb[3 * w] = out.x; rgb[3 * w + 1] = out.y; rgb[3 * w + 2] = out.z;
    }
    // backward: the background term routes the colour gradient into the opacity gradient
    float m = 0.f;
    int n_comp = 0;
    if (n > 0) {
        const float dO = cfg.lambda_opacity * (-lg - 1.0f) * inv_n - (dC.x * bg[0] + dC.y * bg[1] + dC.z * bg[2]);
        float* ds = dsigmas + start;
        float* dc = drgbs + 3 * start;
        const float3 C = make_float3(o.r, o.g, o.b);
        const float dO_term = dO * (1.0f - o.opacity);
        float T_carry = 1.0f, pr = 0.f, pg = 0.f, pb = 0.f;
        bool done = false;
        auto trip = [&](int base, const CLSample& x) {
            const int i = base + lane;
            const bool valid = i < n;
            const float a = valid ? 1.0f - __expf(-(x.sg * x.de)) : 0.f;
            const float T_inc = warp_scan_mul(1.0f - a, lane) * T_carry;
            float T_exc = __shfl_up_sync(0xffffffffu, T_inc, 1);
            if (lane == 0) T_exc = T_carry;
            const bool comp = valid && (i == 0 || T_exc > cfg.T_threshold);
            const float w = comp ? a * T_exc : 0.f;
            const float r_inc = warp_scan_add(w * x.c.x, lane) + pr;
            const float g_inc = warp_scan_add(w * x.c.y, lane) + pg;
            const float b_inc = warp_scan_add(w * x.c.z, lane) + pb;
            if (valid) {
                float3 dcv = make_float3(0.f, 0.f, 0.f);
                float dsv = 0.f;
                if (comp) {
                    dcv = make_float3(dC.x * w, dC.y * w, dC.z * w);
                    const float g = dC.x * (x.c.x * T_inc - (C.x - r_inc)) + dC.y * (x.c.y * T_inc - (C.y - g_inc)) +
                                    dC.z * (x.c.z * T_inc - (C.z - b_inc)) + dO_term;
                    dsv = x.de * g;
                }
                dc[3 * i] = dcv.x; dc[3 * i + 1] = dcv.y; dc[3 * i + 2] = dcv.z;
                ds[i] = dsv;
                m = fmaxf(m, fmaxf(fabsf(dcv.x), fmaxf(fabsf(dcv.y), fabsf(dcv.z))));
                m = fmaxf(m, fabsf(dsv * fminf(x.sg, 3.2690173e6f)));
            }
            n_comp += __popc(__ballot_sync(0xffffffffu, comp));
            done = __ballot_sync(0xffffffffu, valid && !(T_inc > cfg.T_threshold)) != 0u;
            T_carry = __shfl_sync(0xffffffffu, T_inc, 31);
            pr = __shfl_sync(0xffffffffu, r_inc, 31);
            pg = __shfl_sync(0xffffffffu, g_inc, 31);
            pb = __shfl_sync(0xffffffffu, b_inc, 31);
        };
        int base = 0;
#pragma unroll
        for (int k = 0; k < CL_CACHE; ++k)
            if (k * 32 < n && !done) { trip(k * 32, sm[k]); base = k * 32 + 32; }
        for (; base >= CL_CACHE * 32 && base < n && !done; base += 32) {
            CLSample x;
            x.sg = 0.f; x.de = 0.f; x.ti = 0.f; x.c = make_float3(0.f, 0.f, 0.f);
            if (base + lane < n) x = cl_load(sg, dl, tt, cl, base + lane);
            trip(base, x);
        }
        for (int i = base + lane; i < n; i += 32) {  // past the terminating trip: zero gradients
            dc[3 * i] = 0.f; dc[3 * i + 1] = 0.f; dc[3 * i + 2] = 0.f;
            ds[i] = 0.f;
        }
        m = warp_max(m);
    }
    // Per-ray sums, the loss-scale maximum and the live-list allocation go through ONE set of atomics per BLOCK (8 rays):
    // five same-address atomics per ray serialise in the L2 atomic unit.
    __shared__ float s_se[CL_WARPS], s_ent[CL_WARPS], s_m[CL_WARPS];
    __shared__ int s_tot[CL_WARPS], s_comp[CL_WARPS], s_base;
    const int wib = threadIdx.x >> 5;
    if (lane == 0) {
        s_se[wib] = ex * ex + ey * ey + ez * ez;
        s_ent[wib] = -op * lg;
        s_m[wib] = (m > 0.f && m < INFINITY) ? m : 0.f;
        s_tot[wib] = o.total_samples;
        s_comp[wib] = n_comp;
    }
    __syncthreads();
    if (wib == 0) {
        const bool has = lane < CL_WARPS && (blockIdx.x * CL_WARPS + lane) < cfg.n_rays;
        float se = has ? s_se[lane] : 0.f, ent = has ? s_ent[lane] : 0.f, mm = has ? s_m[lane] : 0.f;
        int tot = has ? s_tot[lane] : 0, comp = has ? s_comp[lane] : 0;
        int pre = comp;  // inclusive prefix of the rays' composited counts
#pragma unroll
        for (int o2 = 1; o2 < CL_WARPS; o2 <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, pre, o2);
            if (lane >= o2) pre += u;
        }
        if (has) s_comp[lane] = pre - comp;  // exclusive offset of ray `lane` inside the block's range
        se = warp_sum(se);
        ent = warp_sum(ent);
        mm = warp_max(mm);
#pragma unroll
        for (int o2 = 16; o2 > 0; o2 >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o2);
        const int block_comp = __shfl_sync(0xffffffffu, pre, CL_WARPS - 1);
        if (lane == 0) {
            if (tot) atomicAdd(&counters[1], tot);
            atomicAdd(&scalars[4], se);
            atomicAdd(&scalars[5], ent);
            if (mm > 0.f) atomicMax(reinterpret_cast<int*>(scalars), __float_as_int(mm));
            s_base = (live_idx && block_comp) ? atomicAdd(&counters[4], block_comp) : 0;
        }
    }
    __syncthreads();
    if (live_idx && n_comp > 0) {
        const int at = s_base + s_comp[wib];
        for (int i = lane; i < n_comp; i += 32) live_idx[at + i] = (int)(start + i);
    }
}

// One call for the weight-dependent part of a training step with the plain NeRFLoss (no distortion term):
// network forward -> {compositing, loss, compositing backward} -> loss scale -> MLP backward -> table scatter.
extern "C" int ngp_render_train_step(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* b, const float* rgb_gt,
                                     float* grad_enc, float* grad_rgb, void* stream) {
    int rc = check_train_args(net, cfg, b);
    if (rc) return rc;
    if (!rgb_gt || !b->dsigmas || !b->drgbs || !b->feat_save || !grad_enc || !grad_rgb) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int n = cfg->n_rays;
    NgpSamples smp = train_samples(cfg, b);
    NGP_TRACE(13, st);
    rc = ngp_net_forward(net, &smp, 1, b->sigmas, b->rgbs, nullptr, b->feat_save, stream);
    if (rc) return rc;
    k_train_composite_loss<<<ngp_div_up(n, CL_WARPS), CL_WARPS * 32, 0, st>>>(
        *cfg, b->n_samples, b->offsets, b->sigmas, b->rgbs, b->deltas, b->ts, rgb_gt, b->rgb, b->opacity, b->depth, b->dsigmas,
        b->drgbs, b->scalars, b->live_idx, b->counters, b->bg_dev);
    NGP_CHECK_LAUNCH();
    NGP_TRACE(4, st);
    k_train_grad_scale<<<1, 1, 0, st>>>(b->scalars, b->counters, 1);
    NGP_CHECK_LAUNCH();
    NGP_TRACE(5, st);
    if (b->live_idx) {
        smp.live_idx = b->live_idx;
        smp.n_live_dev = b->counters + 5;
    }
    return ngp_net_backward(net, &smp, b->dsigmas, b->drgbs, b->feat_save, b->scalars + 1, grad_enc, grad_rgb,
                            b->bwd_workspace, b->bwd_workspace_bytes, stream);
}

extern "C" int ngp_render_train_bwd(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* b,
                                    const float* dL_drgb, const float* dL_dopacity, const float* dL_ddepth,
                                    const float* dL_dws, float* grad_enc, float* grad_rgb, void* stream) {
    int rc = check_train_args(net, cfg, b);
    if (rc) return rc;
    if (!dL_drgb || !dL_dopacity || !b->dsigmas || !b->drgbs || !grad_enc || !grad_rgb) return NGP_EINVAL;
    if (dL_dws && !b->ws) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int n = cfg->n_rays;
    k_train_composite_bw<<<ngp_div_up((int64_t)n * 32, 128), 128, 0, st>>>(
        *cfg, b->n_samples, b->offsets, b->sigmas, b->rgbs, b->deltas, b->ts, b->ws, b->rgb, b->opacity, b->depth, dL_drgb,
        dL_dopacity, dL_ddepth, dL_dws, b->dsigmas, b->drgbs, b->scalars, b->live_idx, b->counters, b->bg_dev);
    NGP_CHECK_LAUNCH();
    k_train_grad_scale<<<1, 1, 0, st>>>(b->scalars, b->counters, 0);
    NGP_CHECK_LAUNCH();
    NgpSamples smp = train_samples(cfg, b);
    if (b->live_idx && b->feat_save) {
        smp.live_idx = b->live_idx;
        smp.n_live_dev = b->counters + 5;
    }
    return ngp_net_backward(net, &smp, b->dsigmas, b->drgbs, b->feat_save, b->scalars + 1, grad_enc, grad_rgb,
                            b->bwd_workspace, b->bwd_workspace_bytes, stream);
}

// -------------------------------------------------------------------------------------------------
// NeRFLoss and its per-ray gradients (reference losses.py:47-60 with lambda_distortion = 0)
// -------------------------------------------------------------------------------------------------
__global__ void k_nerf_loss_grad(const NgpTrainCfg cfg, const float* __restrict__ rgb, const float* __restrict__ opacity,
                                 const float* __restrict__ rgb_gt, float* __restrict__ dL_drgb, float* __restrict__ dL_dopacity,
                                 float* __restrict__ scalars, int* __restrict__ counters) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    float se = 0.f, ent = 0.f;
    if (r < cfg.n_rays) {
        const float inv_n = 1.0f / (float)cfg.n_rays;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float e = rgb[3 * r + c] - rgb_gt[3 * r + c];
            se += e * e;
            dL_drgb[3 * r + c] = 2.0f * e * inv_n * (1.0f / 3.0f);
        }
        const float o = opacity[r] + 1e-10f;
        const float lg = logf(o);
        ent = -o * lg;
        dL_dopacity[r] = cfg.lambda_opacity * (-lg - 1.0f) * inv_n;
    }
    se = warp_sum(se);
    ent = warp_sum(ent);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&scalars[2], se);
        atomicAdd(&scalars[3], ent);
    }
    // snapshot of this step's sample counts (counters[0..1] are reused by the next step's march, which a
    // trainer may run ahead of time)
    if (r == 0) {
        counters[2] = counters[0];
        counters[3] = counters[1];
    }
}

extern "C" int ngp_nerf_loss_grad(const NgpTrainCfg* cfg, const NgpTrainBuffers* b, const float* rgb_gt, float* dL_drgb,
                                  float* dL_dopacity, void* stream) {
    if (!cfg || !b || !rgb_gt || !dL_drgb || !dL_dopacity || cfg->n_rays < 1) return NGP_EINVAL;
    k_nerf_loss_grad<<<ngp_div_up(cfg->n_rays, 256), 256, 0, (cudaStream_t)stream>>>(*cfg, b->rgb, b->opacity, rgb_gt, dL_drgb,
                                                                                      dL_dopacity, b->scalars, b->counters);
    NGP_CHECK_LAUNCH();
    return 0;
}

// -------------------------------------------------------------------------------------------------
// fused Adam (+ fp16 re-cast + gradient zeroing), 128-bit accesses
// -------------------------------------------------------------------------------------------------
__global__ void k_adam(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                       __half* __restrict__ ph, int64_t n, const float* __restrict__ lr_dev, const int* __restrict__ step_dev,
                       float beta1, float beta2, float eps, float grad_mul) {
    const int t = *step_dev + 1;
    const float lr = *lr_dev;
    const float bc1 = 1.0f - powf(beta1, (float)t);
    const float bc2 = 1.0f - powf(beta2, (float)t);
    const float step_size = lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    const int64_t n4 = n >> 2;
    // fp32 params, moments and the consumed gradients stream through L2 (evict first); the fp16 working copy the
    // forward gathers from is kept (evict last); the zeroed gradients (next step's reduction target) stay normal
    const uint64_t stream_pol = l2_policy_evict_first(), keep_pol = l2_policy_evict_last();
    // two 64-byte groups per thread and trip: all eight 128-bit loads are issued before the first use, so the stream keeps
    // ~15 MB in flight even when the next step's march shares the SMs' issue slots
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < n4; i0 += 2 * stride) {
        const int64_t i1 = i0 + stride;
        const bool two = i1 < n4;
        float4 pv[2], gv[2], mv[2], vv[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int64_t i = u ? i1 : i0;
            if (u == 0 || two) {
                pv[u] = ld_f4_hint(reinterpret_cast<const float4*>(p) + i, stream_pol);
                gv[u] = ld_f4_hint(reinterpret_cast<const float4*>(g) + i, stream_pol);
                mv[u] = ld_f4_hint(reinterpret_cast<const float4*>(m) + i, stream_pol);
                vv[u] = ld_f4_hint(reinterpret_cast<const float4*>(v) + i, stream_pol);
            }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            if (u == 1 && !two) break;
            const int64_t i = u ? i1 : i0;
            float* pp = &pv[u].x; float* gp = &gv[u].x; float* mp = &mv[u].x; float* vp = &vv[u].x;
            // Stores that cannot change memory are skipped (bitwise the same result, 18 of the 34 bytes per parameter):
            // a hash-table entry no ray has touched yet has g = m = v = 0, its update is p -= lr * 0 / (0 + eps);
            // and a gradient that already is zero needs no clearing. Most of the fine levels' entries are in one of the
            // two states at any step.
            const bool g_zero = gp[0] == 0.f && gp[1] == 0.f && gp[2] == 0.f && gp[3] == 0.f;
            if (g_zero && mp[0] == 0.f && mp[1] == 0.f && mp[2] == 0.f && mp[3] == 0.f && vp[0] == 0.f && vp[1] == 0.f &&
                vp[2] == 0.f && vp[3] == 0.f)
                continue;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float gr = gp[k] * grad_mul;
                mp[k] = beta1 * mp[k] + (1.0f - beta1) * gr;
                vp[k] = beta2 * vp[k] + (1.0f - beta2) * gr * gr;
                const float denom = sqrtf(vp[k]) * inv_sqrt_bc2 + eps;
                pp[k] -= step_size * (mp[k] / denom);
            }
            st_f4_hint(reinterpret_cast<float4*>(p) + i, pv[u], stream_pol);
            st_f4_hint(reinterpret_cast<float4*>(m) + i, mv[u], stream_pol);
            st_f4_hint(reinterpret_cast<float4*>(v) + i, vv[u], stream_pol);
            if (!g_zero) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ph) {
                uint2 h;
                h.x = pack_half2(pv[u].x, pv[u].y);
                h.y = pack_half2(pv[u].z, pv[u].w);
                st_u2_hint(reinterpret_cast<uint2*>(ph) + i, h, keep_pol);
            }
        }
    }
    // tail
    for (int64_t i = (n4 << 2) + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gr = g[i] * grad_mul;
        m[i] = beta1 * m[i] + (1.0f - beta1) * gr;
        v[i] = beta2 * v[i] + (1.0f - beta2) * gr * gr;
        p[i] -= step_size * (m[i] / (sqrtf(v[i]) * inv_sqrt_bc2 + eps));
        g[i] = 0.f;
        if (ph) ph[i] = __float2half_rn(p[i]);
    }
}
__global__ void k_step_inc(int* step) { *step += 1; }

extern "C" int ngp_adam_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, uint16_t* params_half, int64_t n,
                             const float* lr_dev, int32_t* step_dev, float beta1, float beta2, float eps, float grad_mul,
                             int increment_step, void* stream) {
    if (!params || !grads || !exp_avg || !exp_avg_sq || !lr_dev || !step_dev || n < 0) return NGP_EINVAL;
    if ((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) || (((uintptr_t)params_half) & 7))
        return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (n > 0) {
        // 2 resident blocks per SM (two 64-byte groups per thread in flight) saturate HBM and leave registers for the
        // next step's march, which a trainer overlaps with this kernel on another stream
        int grid = ngp_div_up((n >> 2) + 1, 256);
        const int cap = ngp_sm_count() * 2;
        if (grid > cap) grid = cap;
        NGP_TRACE(18, st);
        k_adam<<<grid, 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, (__half*)params_half, n, lr_dev, step_dev, beta1,
                                      beta2, eps, grad_mul);
        NGP_CHECK_LAUNCH();
        NGP_TRACE(8, st);
    }
    if (increment_step) {
        k_step_inc<<<1, 1, 0, st>>>(step_dev);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

// -------------------------------------------------------------------------------------------------
// Data-parallel optimiser step fused with its collective over NVLink peer memory (one kernel):
//   reduce-scatter : rank r sums ITS 1/N shard of the gradient straight out of every peer's gradient
//                    buffer (128-bit P2P loads over NVLink / NVSwitch; no staging copy, no NCCL),
//   Adam           : on that shard only (optimiser state and its HBM traffic are sharded N ways),
//   all-gather     : the updated fp16 parameters of the shard are stored into EVERY peer's working copy.
// Replaces all_reduce(45.8 MB) + a full-size Adam pass. The caller brackets it with two cross-GPU
// barriers (all gradients complete before; all parameter stores landed after) and clears its own
// gradient buffer afterwards. The fp32 master copy of a shard lives on its owner only.
// -------------------------------------------------------------------------------------------------
#define NGP_MAX_PEERS 16
struct PeerPtrs {
    const float* grads[NGP_MAX_PEERS];
    __half* params_half[NGP_MAX_PEERS];
};

__global__ void k_adam_p2p(const PeerPtrs peers, const int world, float* __restrict__ p, float* __restrict__ m,
                           float* __restrict__ v, const int64_t lo4, const int64_t hi4, const float* __restrict__ lr_dev,
                           const int* __restrict__ step_dev, float beta1, float beta2, float eps, float grad_mul) {
    const int t = *step_dev + 1;
    const float lr = *lr_dev;
    const float bc1 = 1.0f - powf(beta1, (float)t);
    const float bc2 = 1.0f - powf(beta2, (float)t);
    const float step_size = lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    const uint64_t stream_pol = l2_policy_evict_first();
    for (int64_t i = lo4 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < hi4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 part[NGP_MAX_PEERS];
#pragma unroll
        for (int r = 0; r < NGP_MAX_PEERS; ++r)
            if (r < world) part[r] = __ldcg(reinterpret_cast<const float4*>(peers.grads[r]) + i);  // all loads in flight
#pragma unroll
        for (int r = 0; r < NGP_MAX_PEERS; ++r)
            if (r < world) { g.x += part[r].x; g.y += part[r].y; g.z += part[r].z; g.w += part[r].w; }
        float4 pv = ld_f4_hint(reinterpret_cast<const float4*>(p) + i, stream_pol);
        float4 mv = ld_f4_hint(reinterpret_cast<const float4*>(m) + i, stream_pol);
        float4 vv = ld_f4_hint(reinterpret_cast<const float4*>(v) + i, stream_pol);
        float* pp = &pv.x; float* gp = &g.x; float* mp = &mv.x; float* vp = &vv.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float gr = gp[k] * grad_mul;
            mp[k] = beta1 * mp[k] + (1.0f - beta1) * gr;
            vp[k] = beta2 * vp[k] + (1.0f - beta2) * gr * gr;
            pp[k] -= step_size * (mp[k] / (sqrtf(vp[k]) * inv_sqrt_bc2 + eps));
        }
        st_f4_hint(reinterpret_cast<float4*>(p) + i, pv, stream_pol);
        st_f4_hint(reinterpret_cast<float4*>(m) + i, mv, stream_pol);
        st_f4_hint(reinterpret_cast<float4*>(v) + i, vv, stream_pol);
        uint2 h;
        h.x = pack_half2(pv.x, pv.y);
        h.y = pack_half2(pv.z, pv.w);
#pragma unroll
        for (int r = 0; r < NGP_MAX_PEERS; ++r)
            if (r < world) reinterpret_cast<uint2*>(peers.params_half[r])[i] = h;
    }
}

extern "C" int ngp_adam_step_p2p(int world, int rank, const uint64_t* peer_grads, float* params, float* exp_avg,
                                 float* exp_avg_sq, const uint64_t* peer_params_half, int64_t n, const float* lr_dev,
                                 int32_t* step_dev, float beta1, float beta2, float eps, int increment_step, void* stream) {
    if (world < 1 || world > NGP_MAX_PEERS || rank < 0 || rank >= world || !peer_grads || !peer_params_half || !params ||
        !exp_avg || !exp_avg_sq || !lr_dev || !step_dev || n < 0 || (n & 3))
        return NGP_EINVAL;
    PeerPtrs pp;
    for (int r = 0; r < NGP_MAX_PEERS; ++r) {
        pp.grads[r] = r < world ? (const float*)(uintptr_t)peer_grads[r] : nullptr;
        pp.params_half[r] = r < world ? (__half*)(uintptr_t)peer_params_half[r] : nullptr;
        if (r < world && (((uintptr_t)pp.grads[r] & 15) || ((uintptr_t)pp.params_half[r] & 7))) return NGP_EINVAL;
    }
    if (((uintptr_t)params | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    // contiguous shard of float4 elements owned by this rank
    const int64_t n4 = n >> 2;
    const int64_t base = n4 / world, extra = n4 % world;
    const int64_t lo4 = rank * base + (rank < extra ? rank : extra);
    const int64_t hi4 = lo4 + base + (rank < extra ? 1 : 0);
    if (hi4 > lo4) {
        int grid = ngp_div_up(hi4 - lo4, 256);
        const int cap = ngp_sm_count() * 4;
        if (grid > cap) grid = cap;
        k_adam_p2p<<<grid, 256, 0, st>>>(pp, world, params, exp_avg, exp_avg_sq, lo4, hi4, lr_dev, step_dev, beta1, beta2,
                                          eps, 1.0f / (float)world);
        NGP_CHECK_LAUNCH();
    }
    if (increment_step) {
        k_step_inc<<<1, 1, 0, st>>>(step_dev);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

// -------------------------------------------------------------------------------------------------
// The same exchange as ONE self-synchronising kernel (no host-side barriers, CUDA-graph capturable):
//   start barrier : block 0 tells every peer "my gradients are complete" (flag store, release.sys) and waits for
//                   the same word from every peer, then releases the other blocks through a local flag;
//   body          : reduce-scatter (peer loads, or ONE multimem.ld_reduce per 16 bytes when the buffers have an
//                   NVLS multicast mapping: the switch sums the N copies, 1/N of the inbound NVLink bytes)
//                   -> Adam on the owned shard -> all-gather of the new fp16 parameters (peer stores, or ONE
//                   multimem.st); every block also clears its slice of `zero_buf`, the gradient buffer the NEXT
//                   step accumulates into (gradient buffers alternate, so nobody clears a buffer a peer may still read);
//   end barrier   : the last block to finish fences, tells every peer "my parameter stores are done", waits for the
//                   same from every peer and bumps the epoch. The kernel therefore ends only when this rank's fp16
//                   working copy is complete and every peer is done reading this rank's gradients.
// Flags are monotonically increasing epochs (never reset), so replays need no re-arming. A rank that waits more
// than ~4 s (a peer died) sets sync[2] = 1 and carries on; the host checks it (ngp_fused_sync_error).
// -------------------------------------------------------------------------------------------------
struct FusedPeers {
    const float* grads[NGP_MAX_PEERS];
    __half* params_half[NGP_MAX_PEERS];
    uint32_t* flags[NGP_MAX_PEERS];  // per rank: [0,world) arrive slots, [NGP_MAX_PEERS, NGP_MAX_PEERS+world) done slots
    const float* mc_grads;           // multicast (NVLS) alias of the gradient buffer, or nullptr
    __half* mc_params_half;          // multicast alias of the fp16 working copy, or nullptr
};
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// spin until *p has reached epoch e (wrap-safe); false on timeout
template <bool SYS>
__device__ __forceinline__ bool wait_epoch(const uint32_t* p, uint32_t e) {
    const long long t0 = clock64();
    for (;;) {
        const uint32_t v = SYS ? ld_acquire_sys(p) : ld_acquire_gpu(p);
        if ((int32_t)(v - e) >= 0) return true;
        if (clock64() - t0 > 8000000000ll) return false;
        __nanosleep(64);
    }
}
__device__ __forceinline__ float4 multimem_ld_reduce_f4(const float* mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st_u2(void* mc, uint2 v) {
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(mc), "f"(__uint_as_float(v.x)),
                 "f"(__uint_as_float(v.y))
                 : "memory");
}

// sync (local device memory, uint32): [0] epoch of the last completed call, [1] finished-block counter, [2] error flag,
// [3] go flag (start barrier passed, written by block 0)
template <int W>  // W >= world: bounds the peer-load registers (16 float4 in flight per thread would halve the occupancy)
__global__ void __launch_bounds__(256, 3)
k_adam_fused(const FusedPeers peers, const int world, const int rank, float* __restrict__ p, float* __restrict__ m,
             float* __restrict__ v, const int64_t lo4, const int64_t hi4, float4* __restrict__ zero_buf, const int64_t zero_n4,
             uint32_t* __restrict__ sync, const float* __restrict__ lr_dev, const int* __restrict__ step_dev, float beta1,
             float beta2, float eps, float grad_mul, unsigned long long* __restrict__ trace) {
    __shared__ uint32_t s_e;
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) trace_mark(trace, 30);  // (debugging aid, see common.cuh)
    // ---- start barrier ----
    if (threadIdx.x == 0) s_e = sync[0] + 1u;  // sync[0] is only written by the last block of the previous call
    __syncthreads();
    const uint32_t e = s_e;
    // The clear of the next step's gradient buffer is local and needs nobody's permission (its last readers were the peers
    // of the PREVIOUS exchange, which ended with a barrier): every block but the one that runs the start barrier does its
    // share first, i.e. while this rank waits for the slowest rank's gradients; block 0 does its share after the barrier.
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (blockIdx.x != 0)
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < zero_n4; i += (int64_t)gridDim.x * blockDim.x)
            zero_buf[i] = z4;
    if (blockIdx.x == 0) {
        if ((int)threadIdx.x < world) {
            st_release_sys(peers.flags[threadIdx.x] + rank, e);
            if (!wait_epoch<true>(peers.flags[rank] + threadIdx.x, e)) sync[2] = 1u;
        }
        __syncthreads();
        if (threadIdx.x == 0) st_release_gpu(&sync[3], e);
        if (trace && threadIdx.x == 0) trace_mark(trace, 31);
        for (int64_t i = threadIdx.x; i < zero_n4; i += (int64_t)gridDim.x * blockDim.x) zero_buf[i] = z4;
    } else {
        if (threadIdx.x == 0 && !wait_epoch<false>(&sync[3], e)) sync[2] = 1u;
        __syncthreads();
    }
    const int t = *step_dev + 1;
    const float lr = *lr_dev;
    const float bc1 = 1.0f - powf(beta1, (float)t);
    const float bc2 = 1.0f - powf(beta2, (float)t);
    const float step_size = lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    const uint64_t stream_pol = l2_policy_evict_first();
    const bool mc_in = peers.mc_grads != nullptr, mc_out = peers.mc_params_half != nullptr;
    // U float4 groups per thread per trip, their remote loads issued back to back before anything waits on them: one
    // multimem.ld_reduce (or one round of peer loads) per trip would make the loop a chain of ~30 NVLink round trips per
    // thread
    constexpr int U = W <= 2 ? 4 : (W <= 4 ? 2 : 1);  // peer-load path: U * W float4 in flight per thread
    constexpr int UM = 4;                             // multimem path: the switch reduces, one float4 per group
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nthr = (int64_t)gridDim.x * blockDim.x;
    auto update = [&](const int64_t i, float4 g) {
        float4 pv = ld_f4_hint(reinterpret_cast<const float4*>(p) + i, stream_pol);
        float4 mv = ld_f4_hint(reinterpret_cast<const float4*>(m) + i, stream_pol);
        float4 vv = ld_f4_hint(reinterpret_cast<const float4*>(v) + i, stream_pol);
        float* pp = &pv.x; float* gp = &g.x; float* mp = &mv.x; float* vp = &vv.x;
        // untouched entries (g = m = v = 0 on every rank): nothing changes, nothing to store or to send (see k_adam)
        if (gp[0] == 0.f && gp[1] == 0.f && gp[2] == 0.f && gp[3] == 0.f && mp[0] == 0.f && mp[1] == 0.f && mp[2] == 0.f &&
            mp[3] == 0.f && vp[0] == 0.f && vp[1] == 0.f && vp[2] == 0.f && vp[3] == 0.f)
            return;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float gr = gp[k] * grad_mul;
            mp[k] = beta1 * mp[k] + (1.0f - beta1) * gr;
            vp[k] = beta2 * vp[k] + (1.0f - beta2) * gr * gr;
            pp[k] -= step_size * (mp[k] / (sqrtf(vp[k]) * inv_sqrt_bc2 + eps));
        }
        st_f4_hint(reinterpret_cast<float4*>(p) + i, pv, stream_pol);
        st_f4_hint(reinterpret_cast<float4*>(m) + i, mv, stream_pol);
        st_f4_hint(reinterpret_cast<float4*>(v) + i, vv, stream_pol);
        uint2 h;
        h.x = pack_half2(pv.x, pv.y);
        h.y = pack_half2(pv.z, pv.w);
        if (mc_out) {
            multimem_st_u2(reinterpret_cast<uint2*>(peers.mc_params_half) + i, h);
        } else {
#pragma unroll
            for (int r = 0; r < W; ++r)
                if (r < world) reinterpret_cast<uint2*>(peers.params_half[r])[i] = h;
        }
    };
    if (mc_in) {
        for (int64_t i0 = lo4 + tid; i0 < hi4; i0 += nthr * UM) {
            float4 g[UM];
#pragma unroll
            for (int u = 0; u < UM; ++u)
                if (i0 + u * nthr < hi4) g[u] = multimem_ld_reduce_f4(peers.mc_grads + 4 * (i0 + u * nthr));
#pragma unroll
            for (int u = 0; u < UM; ++u)
                if (i0 + u * nthr < hi4) update(i0 + u * nthr, g[u]);
        }
    } else {
        for (int64_t i0 = lo4 + tid; i0 < hi4; i0 += nthr * U) {
            float4 part[U][W];
#pragma unroll
            for (int u = 0; u < U; ++u)
#pragma unroll
                for (int r = 0; r < W; ++r)
                    if (r < world && i0 + u * nthr < hi4)
                        part[u][r] = __ldcg(reinterpret_cast<const float4*>(peers.grads[r]) + i0 + u * nthr);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (i0 + u * nthr >= hi4) break;
                float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int r = 0; r < W; ++r)
                    if (r < world) { g.x += part[u][r].x; g.y += part[u][r].y; g.z += part[u][r].z; g.w += part[u][r].w; }
                update(i0 + u * nthr, g);
            }
        }
    }
    // ---- end barrier: last block to finish ----
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        if (atomicAdd(&sync[1], 1u) == gridDim.x - 1u) {
            __threadfence_system();
            sync[1] = 0u;
            if (trace) trace_mark(trace, 32);
            for (int r = 0; r < world; ++r) st_release_sys(peers.flags[r] + NGP_MAX_PEERS + rank, e);
            for (int r = 0; r < world; ++r)
                if (!wait_epoch<true>(peers.flags[rank] + NGP_MAX_PEERS + r, e)) sync[2] = 1u;
            sync[0] = e;
            __threadfence();
            if (trace) trace_mark(trace, 33);
        }
    }
}

extern "C" int ngp_adam_step_fused(int world, int rank, const uint64_t* peer_grads, const uint64_t* peer_params_half,
                                   const uint64_t* peer_flags, uint64_t mc_grads, uint64_t mc_params_half, float* params,
                                   float* exp_avg, float* exp_avg_sq, int64_t n, float* zero_buf, uint32_t* sync,
                                   const float* lr_dev, int32_t* step_dev, float beta1, float beta2, float eps,
                                   int increment_step, void* stream) {
    if (world < 1 || world > NGP_MAX_PEERS || rank < 0 || rank >= world || !peer_grads || !peer_params_half || !peer_flags ||
        !params || !exp_avg || !exp_avg_sq || !sync || !lr_dev || !step_dev || n < 0 || (n & 3))
        return NGP_EINVAL;
    FusedPeers pp;
    for (int r = 0; r < NGP_MAX_PEERS; ++r) {
        pp.grads[r] = r < world ? (const float*)(uintptr_t)peer_grads[r] : nullptr;
        pp.params_half[r] = r < world ? (__half*)(uintptr_t)peer_params_half[r] : nullptr;
        pp.flags[r] = r < world ? (uint32_t*)(uintptr_t)peer_flags[r] : nullptr;
        if (r < world && (((uintptr_t)pp.grads[r] & 15) || ((uintptr_t)pp.params_half[r] & 7) || ((uintptr_t)pp.flags[r] & 3) ||
                          !pp.flags[r]))
            return NGP_EINVAL;
    }
    pp.mc_grads = (const float*)(uintptr_t)mc_grads;
    pp.mc_params_half = (__half*)(uintptr_t)mc_params_half;
    if ((mc_grads & 15) || (mc_params_half & 7)) return NGP_EINVAL;
    if (((uintptr_t)params | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq | (uintptr_t)zero_buf) & 15) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n4 = n >> 2;
    const int64_t base = n4 / world, extra = n4 % world;
    const int64_t lo4 = rank * base + (rank < extra ? rank : extra);
    const int64_t hi4 = lo4 + base + (rank < extra ? 1 : 0);
    // every block passes both barriers, so the grid must not exceed what is guaranteed to become resident while others
    // spin: blocks only wait on block 0 (the first one dispatched) and on peers, never on later blocks of this grid
    int64_t work = hi4 - lo4;
    if (zero_buf && n4 > work) work = n4;
    int grid = ngp_div_up(work > 0 ? work : 1, 256 * 4);
    // Resident blocks per SM. The kernel is NVLink-bound and spends part of its life waiting at its barriers, and while 3
    // blocks per SM are resident (80 registers x 768 threads) no block of the next step's run-ahead march fits beside
    // them: with two ranks half the table per rank makes the kernel's own speed win (3), beyond that the march's share of
    // the SMs (2). NGP_FUSED_BLOCKS_PER_SM (env, read once) overrides.
    static int per_sm_env = -1;
    if (per_sm_env < 0) {
        const char* e = getenv("NGP_FUSED_BLOCKS_PER_SM");
        per_sm_env = e ? atoi(e) : 0;
        if (per_sm_env < 0 || per_sm_env > 3) per_sm_env = 0;
    }
    const int per_sm = per_sm_env ? per_sm_env : (world <= 2 ? 3 : 2);
    const int cap = ngp_sm_count() * per_sm;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
#define NGP_LAUNCH_FUSED(W)                                                                                                \
    k_adam_fused<W><<<grid, 256, 0, st>>>(pp, world, rank, params, exp_avg, exp_avg_sq, lo4, hi4, (float4*)zero_buf,       \
                                          zero_buf ? n4 : 0, sync, lr_dev, step_dev, beta1, beta2, eps, 1.0f / (float)world, \
                                          g_ngp_trace)
    NGP_TRACE(18, st);
    if (world <= 2) NGP_LAUNCH_FUSED(2);
    else if (world <= 4) NGP_LAUNCH_FUSED(4);
    else if (world <= 8) NGP_LAUNCH_FUSED(8);
    else NGP_LAUNCH_FUSED(16);
#undef NGP_LAUNCH_FUSED
    NGP_CHECK_LAUNCH();
    NGP_TRACE(8, st);
    if (increment_step) {
        k_step_inc<<<1, 1, 0, st>>>(step_dev);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

// -------------------------------------------------------------------------------------------------
// batch assembly (reference train.py:78-91, datasets/ray_utils.py:46-70)
// -------------------------------------------------------------------------------------------------
__global__ void k_gen_rays(const int64_t* __restrict__ img_idx, const int64_t* __restrict__ pix_idx,
                           const float* __restrict__ poses, const float* __restrict__ directions,
                           const uint8_t* __restrict__ images, int64_t n_pix, int n, float* __restrict__ rays_o,
                           float* __restrict__ rays_d, float* __restrict__ rgb_gt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t im = img_idx[i], px = pix_idx[i];
    const float* P = poses + 12 * im;
    const float dx = directions[3 * px], dy = directions[3 * px + 1], dz = directions[3 * px + 2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        // rays_d = directions @ R^T  ->  d_k = sum_c dir_c * R[k][c]
        rays_d[3 * i + k] = fmaf(dz, P[4 * k + 2], fmaf(dy, P[4 * k + 1], dx * P[4 * k]));
        rays_o[3 * i + k] = P[4 * k + 3];
    }
    if (images && rgb_gt) {
        const uint8_t* c = images + 3 * (im * n_pix + px);
        rgb_gt[3 * i] = c[0] * (1.0f / 255.0f);
        rgb_gt[3 * i + 1] = c[1] * (1.0f / 255.0f);
        rgb_gt[3 * i + 2] = c[2] * (1.0f / 255.0f);
    }
}

extern "C" int ngp_gen_rays(const int64_t* img_idx, const int64_t* pix_idx, const float* poses, const float* directions,
                            const uint8_t* images, int64_t n_pix, int n, float* rays_o, float* rays_d, float* rgb_gt,
                            void* stream) {
    if (n < 0 || !img_idx || !pix_idx || !poses || !directions || !rays_o || !rays_d) return NGP_EINVAL;
    if (n == 0) return 0;
    k_gen_rays<<<ngp_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(img_idx, pix_idx, poses, directions, images, n_pix, n,
                                                                      rays_o, rays_d, rgb_gt);
    NGP_CHECK_LAUNCH();
    return 0;
}

// Batch assembly in ONE kernel: draws the (image, pixel) pair of every ray and its start jitter from a counter-based
// generator (Philox-4x32-10 keyed by (seed, stream), counter = (draw, ray)) and builds the ray as k_gen_rays does.
// `draw` lives on the device (rng_draw[0], advanced by the kernel's last block), so a CUDA-graph replay draws a new batch.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += 0x9E3779B9u;
        key.y += 0xBB67AE85u;
    }
    return ctr;
}

__global__ void k_sample_rays(const float* __restrict__ poses, const float* __restrict__ directions,
                              const uint8_t* __restrict__ images, uint32_t n_img, uint32_t n_pix, int n, uint32_t seed,
                              uint32_t stream_id, int* __restrict__ rng_draw, float* __restrict__ rays_o,
                              float* __restrict__ rays_d, float* __restrict__ rgb_gt, float* __restrict__ noise) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t draw = (uint32_t)rng_draw[0];
    if (i < n) {
        const uint4 r = philox4x32_10(make_uint4((uint32_t)i, draw, 0u, 0u), make_uint2(seed, stream_id));
        // uniform integers by multiply-high (bias < n/2^32), like torch's random_(0, n) up to the generator
        const uint32_t im = __umulhi(r.x, n_img), px = __umulhi(r.y, n_pix);
        noise[i] = (float)(r.z >> 8) * (1.0f / 16777216.0f);
        const float* P = poses + 12 * (size_t)im;
        const float dx = directions[3 * (size_t)px], dy = directions[3 * (size_t)px + 1], dz = directions[3 * (size_t)px + 2];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            rays_d[3 * i + k] = fmaf(dz, P[4 * k + 2], fmaf(dy, P[4 * k + 1], dx * P[4 * k]));
            rays_o[3 * i + k] = P[4 * k + 3];
        }
        const uint8_t* c = images + 3 * ((size_t)im * n_pix + px);
        rgb_gt[3 * i] = c[0] * (1.0f / 255.0f);
        rgb_gt[3 * i + 1] = c[1] * (1.0f / 255.0f);
        rgb_gt[3 * i + 2] = c[2] * (1.0f / 255.0f);
    }
    // the last block to finish advances the draw counter (every block has read it by then)
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&rng_draw[1], 1) == (int)gridDim.x - 1) {
            rng_draw[1] = 0;
            rng_draw[0] = (int)(draw + 1u);
        }
    }
}

extern "C" int ngp_sample_rays(const float* poses, const float* directions, const uint8_t* images, int n_img, int64_t n_pix,
                               int n, uint32_t seed, uint32_t stream_id, int32_t* rng_draw, float* rays_o, float* rays_d,
                               float* rgb_gt, float* noise, void* stream) {
    if (n < 0 || n_img < 1 || n_pix < 1 || n_pix > 0xffffffffll || !poses || !directions || !images || !rng_draw || !rays_o ||
        !rays_d || !rgb_gt || !noise)
        return NGP_EINVAL;
    if (n == 0) return 0;
    NGP_TRACE(11, (cudaStream_t)stream);
    k_sample_rays<<<ngp_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(poses, directions, images, (uint32_t)n_img,
                                                                         (uint32_t)n_pix, n, seed, stream_id, rng_draw, rays_o,
                                                                         rays_d, rgb_gt, noise);
    NGP_CHECK_LAUNCH();
    NGP_TRACE(1, (cudaStream_t)stream);
    return 0;
}

// -------------------------------------------------------------------------------------------------
// occupancy-grid refresh on the device (reference networks.py:169-195, :240-269)
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pcg_hash(uint32_t v) {
    uint32_t s = v * 747796405u + 2891336453u;
    uint32_t w = ((s >> ((s >> 28u) + 4u)) ^ s) * 277803737u;
    return (w >> 22u) ^ w;
}
__device__ __forceinline__ float u01(uint32_t h) { return (float)(h >> 8) * (1.0f / 16777216.0f); }

struct GridUpd {
    int cascades, grid_size, warmup;
    uint32_t g3, M;
    float scale;
    uint32_t seed;
};

// flag[c*g3 + i] = density_grid > thr  (input of the stream compaction that lists occupied cells)
__global__ void k_grid_flags(const float* __restrict__ grid, int64_t n, float thr, uint8_t* __restrict__ flags) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) flags[i] = grid[i] > thr ? 1 : 0;
}

// Pick the cells to refresh. Slot layout per cascade:
//   warmup : g3 slots, slot i = Morton index i (no pick, no sort)
//   else   : 2*M slots, [0,M) uniform random cells, [M,2M) random occupied cells (key = g3, "none", if there are none)
// The picked Morton indices are then SORTED (cub radix sort) before the density is evaluated: the result of the refresh does
// not depend on the order the cells are evaluated in (it is scattered back per cell), but the evaluation does -- 1M cells in
// random order make every hash-grid gather of a warp hit 32 different sectors; in Morton order neighbouring threads share
// cells on the coarse levels, like consecutive samples of a ray do.
__global__ void k_grid_pick_cells(const GridUpd u, int c, const int* __restrict__ occ_list, const int* __restrict__ occ_count,
                                  uint32_t* __restrict__ keys) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2u * u.M) return;
    const uint32_t h = pcg_hash(u.seed ^ pcg_hash(i + 0x9e3779b9u * (uint32_t)(c + 1)));
    uint32_t idx;
    if (i < u.M) {
        // uniform cell: three independent coordinates, then Morton order (reference networks.py:182-184)
        const uint32_t G = (uint32_t)u.grid_size;
        const uint32_t cx = pcg_hash(h) % G, cy = pcg_hash(h ^ 0x68bc21ebu) % G, cz = pcg_hash(h ^ 0x02e5be93u) % G;
        idx = morton_encode3(cx, cy, cz);
    } else {
        const int cnt = *occ_count;
        idx = cnt <= 0 ? u.g3 : (uint32_t)occ_list[pcg_hash(h ^ 0x7feb352du) % (uint32_t)cnt];
    }
    keys[i] = idx;
}

// One jittered point inside each picked cell. Warm-up (keys == nullptr): slot i of cascade c is cell i. Otherwise `keys`
// are this cascade's picked cells sorted AND de-duplicated (*n_keys of them): a cell picked more than once is evaluated once
// -- the reference's index_put keeps an arbitrary one of the duplicates' values, and with ~150 k occupied cells drawn
// 524 k times most picks ARE duplicates -- so the density pass runs over the distinct cells only. Slots of successive
// cascades are appended: tot[c] = first slot of cascade c, tot[cascades] = number of slots of this refresh.
// cell_idx = c * g3 + cell (-1: nothing to evaluate).
__global__ void k_grid_jitter(const GridUpd u, int c, const uint32_t* __restrict__ keys, const int* __restrict__ n_keys,
                              int* __restrict__ tot, int* __restrict__ cell_idx, float* __restrict__ xyz) {
    const uint32_t n = keys ? (uint32_t)*n_keys : u.g3;
    const uint32_t base = keys ? (uint32_t)tot[c] : (uint32_t)c * u.g3;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) tot[c + 1] = (int)(base + n);  // read by the next cascade's launch / the second half only
    if (i >= n) return;
    const uint32_t m = keys ? keys[i] : i;
    const size_t at = (size_t)base + i;
    if (m >= u.g3) {  // the "no occupied cell" key
        cell_idx[at] = -1;
        xyz[3 * at] = 0.f; xyz[3 * at + 1] = 0.f; xyz[3 * at + 2] = 0.f;
        return;
    }
    cell_idx[at] = (int)((uint32_t)c * u.g3 + m);
    uint32_t h = pcg_hash(u.seed ^ pcg_hash(i + 0x9e3779b9u * (uint32_t)(c + 1)));
    const float G1 = (float)(u.grid_size - 1);
    const float s = fminf(scalbnf(1.0f, c - 1), u.scale);
    const float half_cell = s / (float)u.grid_size;
    const uint32_t cc[3] = {morton_compact10(m), morton_compact10(m >> 1), morton_compact10(m >> 2)};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        h = pcg_hash(h + 0x85ebca6bu);
        const float centre = ((float)cc[k] / G1 * 2.0f - 1.0f) * (s - half_cell);
        xyz[3 * at + k] = centre + (u01(h) * 2.0f - 1.0f) * half_cell;
    }
}

// tmp[cell] = sigma over the first *n_dev slots (n_dev == nullptr: all n_cap); cell_idx = cascade * g3 + cell
__global__ void k_grid_scatter(const int* __restrict__ cell_idx, const float* __restrict__ sigma, const int* __restrict__ n_dev,
                               uint32_t n_cap, float* __restrict__ tmp) {
    const uint32_t n = n_dev ? min((uint32_t)max(*n_dev, 0), n_cap) : n_cap;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = cell_idx[i];
        if (c >= 0) tmp[c] = sigma[i];
    }
}

// grid = grid < 0 ? grid : max(grid*decay, tmp); sum / count of the positive cells per block, into part / part_n[block]
// erode (count_grid != NULL, reference networks.py:258-260): cells seen by few cameras decay faster,
// decay_i = clamp(decay^(1/count_i), 0.1, 0.95)
__global__ void k_grid_merge(float* __restrict__ grid, const float* __restrict__ tmp, int64_t n, float decay,
                             const float* __restrict__ count_grid, float* __restrict__ part, unsigned* __restrict__ part_n) {
    float s = 0.f;
    unsigned cnt = 0u;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float g = grid[i];
        float d = decay;
        if (count_grid) d = fminf(fmaxf(powf(decay, 1.0f / count_grid[i]), 0.1f), 0.95f);
        if (!(g < 0.f)) g = fmaxf(g * d, tmp[i]);
        grid[i] = g;
        if (g > 0.f) { s += g; cnt += 1u; }
    }
    // per-block partials, summed in a fixed order by k_grid_mean: float atomics would make the mean -- the occupancy
    // threshold, near which most cells sit right after initialisation -- depend on the order blocks finish in
    __shared__ float sh_s[8];
    __shared__ unsigned sh_c[8];
    s = warp_sum(s);
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0) {
        sh_s[threadIdx.x >> 5] = s;
        sh_c[threadIdx.x >> 5] = cnt;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float bs = 0.f;
        unsigned bc = 0u;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { bs += sh_s[w]; bc += sh_c[w]; }
        part[blockIdx.x] = bs;
        part_n[blockIdx.x] = bc;
    }
}
#define MERGE_MAX_BLOCKS 2048
// one block of 256 threads: stats[0] = sum, [1] = count, [2] = mean of the positive cells (NaN when there is none, like the
// reference's empty .mean()), every partial added in the same order every time
__global__ void k_grid_mean(const float* __restrict__ part, const unsigned* __restrict__ part_n, int n_blocks,
                            float* __restrict__ stats) {
    __shared__ float sh_s[256];
    __shared__ unsigned long long sh_c[256];
    float s = 0.f;
    unsigned long long c = 0ull;
    for (int b = threadIdx.x; b < n_blocks; b += 256) { s += part[b]; c += part_n[b]; }
    sh_s[threadIdx.x] = s;
    sh_c[threadIdx.x] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) { sh_s[threadIdx.x] += sh_s[threadIdx.x + o]; sh_c[threadIdx.x] += sh_c[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        stats[0] = sh_s[0];
        stats[1] = (float)sh_c[0];
        stats[2] = sh_s[0] / (float)sh_c[0];
    }
}

// workspace layout (all 256-byte aligned), C = cascades:
//   tmp (C*g3 f32) | flags (g3 u8) | occ_list (g3 i32) | occ_count (i32) | cell_idx (C*g3 i32, cascade offset included)
//   | xyz (C*g3*3 f32) | sigma (C*g3 f32) | stats (4 f32) | tot (C+1 i32) + n_unique (i32 at [63]) | keys (g3 u32)
//   | keys_sorted (g3 u32) | cub temp
static size_t al256(size_t v) { return (v + 255) & ~(size_t)255; }
static int key_bits(size_t g3) {  // bits of the largest key, g3 ("none")
    int b = 1;
    while (((size_t)1 << b) <= g3) ++b;
    return b;
}
static size_t cub_temp_bytes(size_t g3) {
    size_t sel = 0, srt = 0;
    cub::DeviceSelect::Flagged(nullptr, sel, cub::CountingInputIterator<int>(0), (const uint8_t*)nullptr, (int*)nullptr,
                               (int*)nullptr, (int)g3);
    cub::DeviceRadixSort::SortKeys(nullptr, srt, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)g3, 0, key_bits(g3));
    size_t unq = 0;
    cub::DeviceSelect::Unique(nullptr, unq, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int*)nullptr, (int)g3);
    if (unq > sel) sel = unq;
    return al256(sel > srt ? sel : srt);
}
struct GridWs {
    float* tmp; uint8_t* flags; int* occ_list; int* occ_count; int* cell_idx; float* xyz; float* sigma; float* stats;
    float* part; unsigned* part_n;  // k_grid_merge's per-block partials
    int* tot;  // [0..C]: first slot of each cascade / total; [63]: number of distinct keys of the cascade being picked
    uint32_t* keys; uint32_t* keys_sorted; void* cub_temp; size_t cub_bytes; size_t total;
};
static GridWs grid_ws(void* workspace, int cascades, size_t g3) {
    GridWs g;
    char* w = (char*)workspace;
    const size_t C = (size_t)cascades;
    g.tmp = (float*)w; w += al256(C * g3 * 4);
    g.flags = (uint8_t*)w; w += al256(g3);
    g.occ_list = (int*)w; w += al256(g3 * 4);
    g.occ_count = (int*)w; w += 256;
    g.cell_idx = (int*)w; w += al256(C * g3 * 4);
    g.xyz = (float*)w; w += al256(C * g3 * 12);
    g.sigma = (float*)w; w += al256(C * g3 * 4);
    g.stats = (float*)w; w += 256;
    g.part = (float*)w; w += al256(MERGE_MAX_BLOCKS * 4);
    g.part_n = (unsigned*)w; w += al256(MERGE_MAX_BLOCKS * 4);
    g.tot = (int*)w; w += 256;
    g.keys = (uint32_t*)w; w += al256(g3 * 4);
    g.keys_sorted = (uint32_t*)w; w += al256(g3 * 4);
    g.cub_temp = w;
    g.cub_bytes = cub_temp_bytes(g3);
    g.total = (size_t)(w - (char*)workspace) + g.cub_bytes;
    return g;
}
extern "C" size_t ngp_update_grid_workspace(int cascades, int grid_size) {
    if (cascades < 1 || grid_size < 1) return 0;
    return grid_ws(nullptr, cascades, (size_t)grid_size * grid_size * grid_size).total;
}

// First half of the refresh: everything that depends on the OLD density grid and the seed but not on the weights -- which
// cells to re-evaluate (sorted) and a jittered point in each, plus clearing the scratch grid. A trainer runs it on a side
// stream any time after the previous refresh, so that only the second half sits between two training steps.
extern "C" int ngp_update_density_grid_pick(const float* density_grid, int cascades, int grid_size, float scale,
                                            float density_threshold, int warmup, uint32_t seed, void* workspace,
                                            size_t workspace_bytes, void* stream) {
    if (!density_grid || !workspace || cascades < 1 || cascades > 62 || grid_size < 2 || grid_size > 1024) return NGP_EINVAL;
    if ((int64_t)cascades * grid_size * grid_size * grid_size > 0x7fffffffll) return NGP_EINVAL;  // cell_idx = c * g3 + cell
    if (workspace_bytes < ngp_update_grid_workspace(cascades, grid_size)) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t g3 = (size_t)grid_size * grid_size * grid_size;
    const GridWs g = grid_ws(workspace, cascades, g3);
    size_t cub_bytes = g.cub_bytes;
    GridUpd u;
    u.cascades = cascades; u.grid_size = grid_size; u.warmup = warmup ? 1 : 0;
    u.g3 = (uint32_t)g3; u.M = (uint32_t)(g3 / 4); u.scale = scale; u.seed = seed;
    NGP_CUDA(cudaMemsetAsync(g.tmp, 0, cascades * g3 * 4, st));
    NGP_CUDA(cudaMemsetAsync(g.stats, 0, 16, st));
    NGP_COUNT_LAUNCHES(2);
    NGP_TRACE(20, st);
    const uint32_t n_slots = warmup ? (uint32_t)g3 : 2u * u.M;
    NGP_CUDA(cudaMemsetAsync(g.tot, 0, 256, st));
    NGP_COUNT_LAUNCHES(1);
    for (int c = 0; c < cascades; ++c) {
        if (!warmup) {
            k_grid_flags<<<ngp_div_up(g3, 256), 256, 0, st>>>(density_grid + c * g3, (int64_t)g3, density_threshold, g.flags);
            NGP_CHECK_LAUNCH();
            NGP_CUDA(cub::DeviceSelect::Flagged(g.cub_temp, cub_bytes, cub::CountingInputIterator<int>(0), g.flags, g.occ_list,
                                                g.occ_count, (int)g3, st));
            NGP_COUNT_LAUNCHES(2);  // cub: init + sweep kernels
            NGP_TRACE(21, st);
            k_grid_pick_cells<<<ngp_div_up(n_slots, 256), 256, 0, st>>>(u, c, g.occ_list, g.occ_count, g.keys);
            NGP_CHECK_LAUNCH();
            NGP_CUDA(cub::DeviceRadixSort::SortKeys(g.cub_temp, cub_bytes, (const uint32_t*)g.keys, g.keys_sorted, (int)n_slots,
                                                    0, key_bits(g3), st));
            NGP_COUNT_LAUNCHES(2 + (key_bits(g3) + 7) / 8);  // cub onesweep: histogram + scan + one kernel per 8-bit digit
            NGP_CUDA(cub::DeviceSelect::Unique(g.cub_temp, cub_bytes, (const uint32_t*)g.keys_sorted, g.keys, g.tot + 63,
                                               (int)n_slots, st));
            NGP_COUNT_LAUNCHES(2);
        }
        k_grid_jitter<<<ngp_div_up(n_slots, 256), 256, 0, st>>>(u, c, warmup ? nullptr : g.keys, g.tot + 63, g.tot, g.cell_idx,
                                                                g.xyz);
        NGP_CHECK_LAUNCH();
        NGP_TRACE(22, st);
    }
    return 0;
}

// Second half: the density at the picked points (ONE pass over the slots of all cascades), the merge and the bitfield.
extern "C" int ngp_update_density_grid_eval(const NgpNet* net, float* density_grid, uint8_t* density_bitfield,
                                            const float* count_grid, int cascades, int grid_size, float density_threshold,
                                            int warmup, float decay, void* workspace, size_t workspace_bytes, void* stream) {
    if (!net || !density_grid || !density_bitfield || !workspace || cascades < 1 || grid_size < 2 || grid_size > 1024)
        return NGP_EINVAL;
    if (workspace_bytes < ngp_update_grid_workspace(cascades, grid_size)) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t g3 = (size_t)grid_size * grid_size * grid_size;
    const GridWs g = grid_ws(workspace, cascades, g3);
    const size_t n_slots = warmup ? g3 : 2 * (g3 / 4);
    const size_t n_all = n_slots * (size_t)cascades;  // capacity; the regular refresh evaluates tot[cascades] distinct cells
    NgpSamples smp;
    smp.xyzs = g.xyz; smp.dirs = nullptr; smp.rays_o = nullptr; smp.rays_d = nullptr; smp.ray_idx = nullptr; smp.ts = nullptr;
    smp.n = (int64_t)n_all; smp.n_dev = warmup ? nullptr : g.tot + cascades; smp.live_idx = nullptr; smp.n_live_dev = nullptr;
    int rc = ngp_net_forward(net, &smp, 0, g.sigma, nullptr, nullptr, nullptr, stream);
    if (rc) return rc;
    int sgrid = ngp_div_up(n_all, 256);
    if (sgrid > ngp_sm_count() * 16) sgrid = ngp_sm_count() * 16;
    k_grid_scatter<<<sgrid, 256, 0, st>>>(g.cell_idx, g.sigma, smp.n_dev, (uint32_t)n_all, g.tmp);
    NGP_CHECK_LAUNCH();
    NGP_TRACE(23, st);
    int grid = ngp_div_up((int64_t)cascades * g3, 256);
    if (grid > ngp_sm_count() * 8) grid = ngp_sm_count() * 8;
    if (grid > MERGE_MAX_BLOCKS) grid = MERGE_MAX_BLOCKS;
    k_grid_merge<<<grid, 256, 0, st>>>(density_grid, g.tmp, (int64_t)cascades * g3, decay, count_grid, g.part, g.part_n);
    NGP_CHECK_LAUNCH();
    k_grid_mean<<<1, 256, 0, st>>>(g.part, g.part_n, grid, g.stats);
    NGP_CHECK_LAUNCH();
    NGP_TRACE(24, st);
    // threshold = min(mean, density_threshold) evaluated on the device (fminf ignores a NaN mean)
    rc = ngp_packbits(density_grid, 0, (int64_t)cascades * g3 / 8, density_threshold, g.stats + 2, density_bitfield, stream);
    NGP_TRACE(25, st);
    return rc;
}

extern "C" int ngp_update_density_grid(const NgpNet* net, float* density_grid, uint8_t* density_bitfield,
                                       const float* count_grid, int cascades, int grid_size, float scale,
                                       float density_threshold, int warmup, float decay, uint32_t seed, void* workspace,
                                       size_t workspace_bytes, void* stream) {
    if (!net || !density_bitfield) return NGP_EINVAL;
    int rc = ngp_update_density_grid_pick(density_grid, cascades, grid_size, scale, density_threshold, warmup, seed, workspace,
                                          workspace_bytes, stream);
    if (rc) return rc;
    return ngp_update_density_grid_eval(net, density_grid, density_bitfield, count_grid, cascades, grid_size, density_threshold,
                                        warmup, decay, workspace, workspace_bytes, stream);
}
