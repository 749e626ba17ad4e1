// Sync-free inference render for sm_90a: what render(test_time=True) does (reference
// models/rendering.py:46-118) as a device-side wavefront.
//
// The reference loops on the host: march N more samples for every alive ray, evaluate the network,
// composite, drop converged rays (boolean-mask compaction => >= 3 host syncs per round, tens of rounds
// per image). Here the alive list (ping-pong), the per-round sample quota and the convergence test all
// stay on the device. Per round every alive ray receives the reference's sample quota
// max(min(N_rays // N_alive, 64), min_samples) (rendering.py:73,80), computed ON the device from the alive
// counter, and a ray leaves the alive list exactly when the reference's composite_test_fw drops it
// (volumerendering.cu:221-248) -- so the rounds, the per-round quotas and total_samples are the reference's.
// Each ray sees exactly the reference's sample sequence (raymarching_test_kernel semantics, incl. its
// `cascades`-as-scale quirk) and the same front-to-back accumulation order, so results differ from the
// reference only by the fp16-level network difference (T is resumed as 1 - opacity, volumerendering.cu:230).
// One round = THREE launches: march, network, compositing (whose last block does the next round's bookkeeping).
#include "common.cuh"
#include "march.cuh"
#include "../../include/ngp_b200.h"
#include <string.h>

// per-round bookkeeping (1 thread), the head of the reference's loop (rendering.py:75-81):
//   while samples < max_samples:  N_alive = len(alive); if N_alive == 0: break
//       N_samples = max(min(N_rays // N_alive, 64), min_samples);  samples += N_samples
// computed from the device-side alive count. N_alive * N_samples <= max(N_rays, min_samples * N_alive) <= 4 * N_rays, the
// capacity of the per-round sample buffers (max_round_samples), so the quota never has to be clipped.
// Two marching regimes (one kernel, chosen per round on the device):
//   N_samples <  INFER_STAGE (at least N_rays/8 rays alive, few samples each) -> one THREAD per ray: one visit per empty
//       CELL is ~5x less work than probing every chain point, and there are enough rays to fill the GPU; samples staged in
//       shared memory and appended compactly (one atomic per warp);
//   N_samples >= INFER_STAGE (few rays, many samples each) -> one WARP per ray (march_ray_warp: 32 chain points probed side
//       by side), samples written straight to the ray's own N_samples slots, unused slots marked ray_idx = -1 (the network
//       kernel skips their gathers).
//   On rounds of 2-7 samples per ray the warp regime is slower than thread-per-ray, so it is kept for the late rounds
//   only, and the thread-per-ray visit is specialised (no frexp/scalbn/division with one cascade, constant step).
// state: [0] N_samples of this round (0 = loop over)  [1] `samples` so far  [2] slots the network evaluates this round
//        [3] rounds run  [4] samples marched this round  [5] 1 = warp-per-ray regime  [6] finished-block ticket
#define INFER_STAGE 8  // thread-per-ray regime below this many samples per ray and round (= its staging slots per thread)
__device__ __forceinline__ void infer_begin_round(const NgpInferCfg& cfg, int* __restrict__ alive_count,
                                                  int* __restrict__ next_count, int* __restrict__ state,
                                                  int64_t* __restrict__ total) {
    *total += state[4];
    state[4] = 0;
    state[2] = 0;
    *next_count = 0;
    int n_alive = *alive_count;
    if (state[1] >= cfg.sample_budget) {
        n_alive = 0;
        *alive_count = 0;
    }
    int S = 0;
    if (n_alive > 0) {
        const int min_samples = cfg.exp_step_factor == 0.0f ? 1 : 4;
        S = max(min(cfg.n_rays / n_alive, 64), min_samples);
        const int64_t share = cfg.max_round_samples / n_alive;  // (never binds for max_round_samples >= 4 * n_rays)
        if (share < S) S = (int)(share < 1 ? 1 : share);
        state[1] += S;
        state[3] += 1;
        const bool warp_regime = S >= INFER_STAGE;
        state[5] = warp_regime ? 1 : 0;
        if (warp_regime) state[2] = n_alive * S;  // rectangular slots; the thread-per-ray regime counts as it appends
    }
    state[0] = S;
}

// init: AABB (+ near clamp), zero the accumulators. EVERY ray enters the first alive list, in order, like the reference's
// alive_indices = arange(N_rays) (rendering.py:71): rays that miss the box take no sample in round 0 and are dropped by
// its compositing (composite_test_fw: N_eff == 0 -> not alive), so the per-round quota N_rays // N_alive of the following
// rounds sees the same alive counts as the reference's loop. Thread 0 also does the bookkeeping of round 0 (the counters
// were cleared by the memset before this kernel).
__global__ void k_infer_init(const NgpInferCfg cfg, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                             float* __restrict__ t_cur, float* __restrict__ t_end, float* __restrict__ opacity,
                             float* __restrict__ depth, float* __restrict__ rgb, int* __restrict__ alive,
                             int* __restrict__ alive_count, int* __restrict__ next_count, int* __restrict__ state,
                             int64_t* __restrict__ total) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) {
        *alive_count = cfg.n_rays;
        infer_begin_round(cfg, alive_count, next_count, state, total);
    }
    if (r >= cfg.n_rays) return;
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
    t_cur[r] = t1;
    t_end[r] = t2;
    opacity[r] = 0.f;
    depth[r] = 0.f;
    rgb[3 * r] = 0.f; rgb[3 * r + 1] = 0.f; rgb[3 * r + 2] = 0.f;
    alive[r] = r;
}

// one round of marching; the regime (state[5]) is uniform over the grid
#define INFER_THREADS 128
template <bool CONST_DT, bool ONE_CASCADE>
__global__ void __launch_bounds__(INFER_THREADS)
k_infer_march(const NgpInferCfg cfg, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
              const uint8_t* __restrict__ bitfield, float* __restrict__ t_cur, const float* __restrict__ t_end,
              const int* __restrict__ alive, const int* __restrict__ alive_count, int* __restrict__ ray_start,
              int* __restrict__ ray_n, int* __restrict__ ray_idx, float* __restrict__ ts, float* __restrict__ deltas,
              int* __restrict__ state) {
    __shared__ float2 stage[INFER_THREADS][INFER_STAGE - 1];
    const int S = state[0];
    if (S <= 0) return;
    const int lane = threadIdx.x & 31;
    const int n_alive = *alive_count;
    const MarchConst c = make_march_const(bitfield, cfg.cascades, cfg.grid_size, cfg.max_samples, cfg.scale, cfg.exp_step_factor,
                                          (float)cfg.cascades);
    if (!state[5]) {
        // ---- thread per ray: up to S < INFER_STAGE occupied samples per ray, staged, then one atomic per warp claims a
        //      contiguous range of the compact sample arrays; whole warps stride over the alive list ----
        const int n_pad = (n_alive + 31) & ~31;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pad; i += gridDim.x * blockDim.x) {
            float2* my = stage[threadIdx.x];
            int n = 0, r = -1;
            float t = 0.f;
            if (i < n_alive) {
                r = alive[i];
                const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                                    rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
                t = t_cur[r];
                const float t2 = t_end[r];
                float dt;
                MarchCache cache;
                while (t < t2 && n < S) {
                    if (march_visit_t<CONST_DT, ONE_CASCADE>(ray, c, t, dt, &cache)) {
                        my[n] = make_float2(t, dt);
                        t = __fadd_rn(t, dt);
                        ++n;
                    }
                }
            }
            int pre = n;  // inclusive prefix of the counts across the warp
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, pre, o);
                if (lane >= o) pre += u;
            }
            const int warp_total = __shfl_sync(0xffffffffu, pre, 31);
            int base = 0;
            if (lane == 31 && warp_total > 0) {
                base = atomicAdd(&state[2], warp_total);
                atomicAdd(&state[4], warp_total);
            }
            base = __shfl_sync(0xffffffffu, base, 31);
            if (r < 0) continue;
            const int start = base + pre - n;  // n_alive * S <= capacity, so this always fits
            ray_start[i] = start;
            ray_n[i] = n;
            t_cur[r] = t;
            for (int k = 0; k < n; ++k) {
                ray_idx[start + k] = r;
                ts[start + k] = my[k].x;
                deltas[start + k] = my[k].y;
            }
        }
        return;
    }
    // ---- warp per ray: same sample sequence, 32 chain points probed at a time (march_ray_warp); ray i owns slots
    //      [i*S, (i+1)*S). Lanes 0..7 hold {ox,oy,oz,dx,dy,dz,t,t2} of the NEXT ray (one load each) while this one is marched ----
    const int n_warps = (gridDim.x * blockDim.x) >> 5;
    int marched = 0;
    int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int r_next = i < n_alive ? alive[i] : -1;
    auto fetch = [&](int r) -> float {
        if (r < 0 || lane > 7) return 0.f;
        if (lane < 3) return rays_o[3 * r + lane];
        if (lane < 6) return rays_d[3 * r + lane - 3];
        return lane == 6 ? t_cur[r] : t_end[r];
    };
    float v_next = fetch(r_next);
    for (; i < n_alive; i += n_warps) {
        const int r = r_next;
        const float v = v_next;
        const int i2 = i + n_warps;
        r_next = i2 < n_alive ? alive[i2] : -1;
        v_next = fetch(r_next);
        const MarchRay ray = make_march_ray(__shfl_sync(0xffffffffu, v, 0), __shfl_sync(0xffffffffu, v, 1), __shfl_sync(0xffffffffu, v, 2),
                                            __shfl_sync(0xffffffffu, v, 3), __shfl_sync(0xffffffffu, v, 4), __shfl_sync(0xffffffffu, v, 5));
        const float t = __shfl_sync(0xffffffffu, v, 6);
        const float t2 = __shfl_sync(0xffffffffu, v, 7);
        const int64_t base = (int64_t)i * S;
        float resume = t;
        const int n = march_ray_warp<CONST_DT, ONE_CASCADE>(ray, c, t, t2, S, lane, [&](int k, float tk, float dk) {
            ray_idx[base + k] = r;
            ts[base + k] = tk;
            deltas[base + k] = dk;
        }, &resume);
        for (int k = n + lane; k < S; k += 32) ray_idx[base + k] = -1;  // unused slots
        if (lane == 0) {
            ray_start[i] = (int)base;
            ray_n[i] = n;
            // a ray that took fewer than S samples has left the box: nothing more to march (the reference keeps its t there too)
            t_cur[r] = n < S ? fmaxf(resume, t2) : resume;
            marched += n;
        }
    }
    if (lane == 0 && marched) atomicAdd(&state[4], marched);
}

// composite this round's samples of every alive ray (one thread per ray, <= 64 samples, same serial order as the
// reference's composite_test_fw_kernel) and append the survivors to the next alive list. The LAST block to finish does the
// next round's bookkeeping (infer_begin_round on the swapped lists) and, inside the frame graph, sets the WHILE node's
// condition (`handle` != 0 on the second round of the loop body).
__global__ void k_infer_composite(const NgpInferCfg cfg, const float* __restrict__ sigmas,
                                  const float* __restrict__ rgbs, const float* __restrict__ deltas,
                                  const float* __restrict__ ts, const int* __restrict__ ray_start,
                                  const int* __restrict__ ray_n, const int* __restrict__ alive,
                                  int* __restrict__ alive_count, float* __restrict__ opacity,
                                  float* __restrict__ depth, float* __restrict__ rgb, int* __restrict__ next_alive,
                                  int* __restrict__ next_count, int* __restrict__ state, int64_t* __restrict__ total,
                                  const cudaGraphConditionalHandle handle, const int set_cond) {
    const int lane = threadIdx.x & 31;
    const int n_alive = *alive_count;
    const int n_pad = (n_alive + 31) & ~31;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pad; i += gridDim.x * blockDim.x) {
        bool keep = false;
        int r = -1;
        if (i < n_alive) {
            r = alive[i];
            const int n = ray_n[i];
            const int start = ray_start[i];
            float o = opacity[r], d = depth[r];
            float cr = rgb[3 * r], cg = rgb[3 * r + 1], cb = rgb[3 * r + 2];
            float T = 1.0f - o;
            bool term = false;
            for (int s = 0; s < n; ++s) {
                const int k = start + s;
                const float a = 1.0f - __expf(-(__ldg(sigmas + k) * __ldg(deltas + k)));
                const float w = a * T;
                cr = fmaf(w, __ldg(rgbs + 3 * k), cr);
                cg = fmaf(w, __ldg(rgbs + 3 * k + 1), cg);
                cb = fmaf(w, __ldg(rgbs + 3 * k + 2), cb);
                d = fmaf(w, __ldg(ts + k), d);
                o += w;
                T *= 1.0f - a;
                if (T <= cfg.T_threshold) {
                    term = true;
                    break;
                }
            }
            opacity[r] = o;
            depth[r] = d;
            rgb[3 * r] = cr; rgb[3 * r + 1] = cg; rgb[3 * r + 2] = cb;
            // the reference's rule (composite_test_fw, volumerendering.cu:221-224,:245-248): a ray leaves the alive list when it
            // got no sample this round or its transmittance fell to the threshold -- a ray that ran out of box with SOME samples
            // stays for one more (empty) round, and counts in that round's N_alive
            keep = !term && n > 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (m) {
            int base = 0;
            const int leader = __ffs(m) - 1;
            if (lane == leader) base = atomicAdd(next_count, __popc(m));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (keep) next_alive[base + __popc(m & ((1u << lane) - 1u))] = r;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&state[6], 1) == (int)gridDim.x - 1) {  // every block's appends are visible
            state[6] = 0;
            infer_begin_round(cfg, next_count, alive_count, state, total);  // the lists swap roles
            if (set_cond) cudaGraphSetConditional(handle, state[0] > 0 ? 1u : 0u);
        }
    }
}

__global__ void k_infer_finish(const NgpInferCfg cfg, const float* __restrict__ opacity, float* __restrict__ rgb,
                               const int* __restrict__ state, int64_t* __restrict__ total, int64_t* __restrict__ total_out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0 && total_out) *total_out = *total + state[4];
    if (r >= cfg.n_rays) return;
    const float rest = 1.0f - opacity[r];  // reference rendering.py:112-116
    rgb[3 * r] += cfg.bg[0] * rest;
    rgb[3 * r + 1] += cfg.bg[1] * rest;
    rgb[3 * r + 2] += cfg.bg[2] * rest;
}

struct InferWs {
    float *t_cur, *t_end;
    int* alive[2];
    int *ray_start, *ray_n, *ray_idx;
    float *ts, *deltas, *sigmas, *rgbs;
    int *counters, *alive_cnt, *state;
    int64_t* total;
};
static InferWs infer_ws(const NgpInferCfg* cfg, void* workspace) {
    const size_t nr = ((size_t)cfg->n_rays * 4 + 255) & ~(size_t)255;
    const size_t ns = ((size_t)cfg->max_round_samples * 4 + 255) & ~(size_t)255;
    char* w = (char*)workspace;
    InferWs W;
    W.t_cur = (float*)w; w += nr;
    W.t_end = (float*)w; w += nr;
    W.alive[0] = (int*)w; w += nr;
    W.alive[1] = (int*)w; w += nr;
    W.ray_start = (int*)w; w += nr;
    W.ray_n = (int*)w; w += nr;
    W.ray_idx = (int*)w; w += ns;
    W.ts = (float*)w; w += ns;
    W.deltas = (float*)w; w += ns;
    W.sigmas = (float*)w; w += ns;
    W.rgbs = (float*)w; w += 3 * ns;
    W.counters = (int*)w;  // [0],[1] alive counts (ping-pong)  [8..11] state  [16..17] int64 total
    W.alive_cnt = W.counters;
    W.state = W.counters + 8;
    W.total = (int64_t*)(W.counters + 16);
    return W;
}

// one round of the wavefront on stream st; the ping-pong role of the two alive lists is given by `cur`
static int infer_round(const NgpNet* net, const NgpInferCfg* cfg, const InferWs& W, const float* rays_o, const float* rays_d,
                       const uint8_t* density_bitfield, float* opacity, float* depth, float* rgb, int cur, cudaStream_t st,
                       cudaGraphConditionalHandle handle = 0, int set_cond = 0);

extern "C" size_t ngp_render_infer_workspace(int n_rays, int64_t max_round_samples) {
    if (n_rays < 1 || max_round_samples < 1) return 0;
    const size_t nr = ((size_t)n_rays * 4 + 255) & ~(size_t)255;
    const size_t ns = ((size_t)max_round_samples * 4 + 255) & ~(size_t)255;
    // t_cur, t_end, alive[2], ray_start, ray_n  |  ray_idx, ts, deltas, sigmas, rgbs(3)  |  counters
    return 6 * nr + 7 * ns + 4096;
}

// Runs rounds [first_round, first_round + n_rounds) of the wavefront. first_round == 0 also initialises
// (AABB, accumulators, first alive list); finish != 0 adds the background and writes total_samples.
// alive_count_out (device int32*, optional) receives the number of rays still alive after the last round
// of this call: the caller may read it back every few rounds to stop early (the ONLY host sync of the
// path, amortised over n_rounds), or never read it and simply run enough rounds.
extern "C" int ngp_render_infer(const NgpNet* net, const NgpInferCfg* cfg, const float* rays_o, const float* rays_d,
                                const uint8_t* density_bitfield, float* opacity, float* depth, float* rgb,
                                int64_t* total_samples, int first_round, int n_rounds, int finish, int* alive_count_out,
                                void* workspace, size_t workspace_bytes, void* stream) {
    if (!net || !cfg || !rays_o || !rays_d || !density_bitfield || !opacity || !depth || !rgb || !workspace) return NGP_EINVAL;
    if (cfg->n_rays < 1 || cfg->cascades < 1 || cfg->grid_size < 1 || cfg->grid_size > 1024 || cfg->max_samples < 1 ||
        cfg->max_round_samples < cfg->n_rays || cfg->max_round_samples > 0x7fffffffll || cfg->sample_budget < 1 ||
        first_round < 0 || n_rounds < 0)
        return NGP_EINVAL;
    if (workspace_bytes < ngp_render_infer_workspace(cfg->n_rays, cfg->max_round_samples)) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int n = cfg->n_rays;
    const InferWs W = infer_ws(cfg, workspace);
    int* alive_cnt = W.alive_cnt;
    int* state = W.state;
    int64_t* total = W.total;

    if (first_round == 0) {
        NGP_CUDA(cudaMemsetAsync(W.counters, 0, 4096, st));
        NGP_COUNT_LAUNCHES(1);
        k_infer_init<<<ngp_div_up(n, 256), 256, 0, st>>>(*cfg, rays_o, rays_d, W.t_cur, W.t_end, opacity, depth, rgb, W.alive[0],
                                                          alive_cnt, alive_cnt + 1, W.state, W.total);
        NGP_CHECK_LAUNCH();
    }
    for (int round = first_round; round < first_round + n_rounds; ++round) {
        int rc = infer_round(net, cfg, W, rays_o, rays_d, density_bitfield, opacity, depth, rgb, round & 1, st);
        if (rc) return rc;
    }
    if (alive_count_out)
        NGP_CUDA(cudaMemcpyAsync(alive_count_out, alive_cnt + ((first_round + n_rounds) & 1), sizeof(int),
                                 cudaMemcpyDeviceToDevice, st));
    if (finish) {
        k_infer_finish<<<ngp_div_up(n, 256), 256, 0, st>>>(*cfg, opacity, rgb, state, total, total_samples);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

static int infer_round(const NgpNet* net, const NgpInferCfg* cfg, const InferWs& W, const float* rays_o, const float* rays_d,
                       const uint8_t* density_bitfield, float* opacity, float* depth, float* rgb, int cur, cudaStream_t st,
                       cudaGraphConditionalHandle handle, int set_cond) {
    const int n = cfg->n_rays;
    const int nxt = cur ^ 1;
    // persistent-style grids (the kernels stride over the device-side alive count): enough blocks to fill the GPU, never
    // tens of thousands of blocks that find nothing to do in the late rounds
    const int sms = ngp_sm_count();
    const int grid_m = (int)min((int64_t)ngp_div_up(n, INFER_THREADS), (int64_t)sms * 16);
    const int grid_c = (int)min((int64_t)ngp_div_up(n, 128), (int64_t)sms * 16);
    // the test-time step bounds use `cascades` where the train kernel uses `scale` (reference raymarching.cu:370,399)
    const bool const_dt = march_const_dt(cfg->exp_step_factor, cfg->max_samples, (float)cfg->cascades, cfg->grid_size);
    march_dispatch(const_dt, cfg->cascades, [&](auto cd, auto oc) {
        k_infer_march<decltype(cd)::value, decltype(oc)::value><<<grid_m, INFER_THREADS, 0, st>>>(
            *cfg, rays_o, rays_d, density_bitfield, W.t_cur, W.t_end, W.alive[cur], W.alive_cnt + cur, W.ray_start, W.ray_n,
            W.ray_idx, W.ts, W.deltas, W.state);
    });
    NGP_CHECK_LAUNCH();
    NgpSamples smp;
    smp.xyzs = nullptr; smp.dirs = nullptr; smp.rays_o = rays_o; smp.rays_d = rays_d; smp.ray_idx = W.ray_idx; smp.ts = W.ts;
    smp.n = cfg->max_round_samples; smp.n_dev = W.state + 2; smp.live_idx = nullptr; smp.n_live_dev = nullptr;
    int rc = ngp_net_forward(net, &smp, 1, W.sigmas, W.rgbs, nullptr, nullptr, (void*)st);
    if (rc) return rc;
    k_infer_composite<<<grid_c, 128, 0, st>>>(*cfg, W.sigmas, W.rgbs, W.deltas, W.ts, W.ray_start, W.ray_n, W.alive[cur],
                                               W.alive_cnt + cur, opacity, depth, rgb, W.alive[nxt], W.alive_cnt + nxt, W.state,
                                               W.total, handle, set_cond);
    NGP_CHECK_LAUNCH();
    return 0;
}

// -------------------------------------------------------------------------------------------------
// The whole frame as ONE CUDA graph with a device-side loop: init -> WHILE(alive rays left and sample budget not used up)
// { two rounds (the alive lists ping-pong) } -> finish. The loop is a conditional WHILE node whose condition the last block
// of the second round's compositing kernel sets (cudaGraphSetConditional: another round is due), so the host enqueues one
// graph launch per frame and never reads anything back. The instantiated graph is cached per (device, arguments): a
// caller that renders frame after frame from the same buffers pays the build once.
// -------------------------------------------------------------------------------------------------
struct InferGraphKey {
    NgpNet net;
    NgpInferCfg cfg;
    const void *rays_o, *rays_d, *bitfield, *opacity, *depth, *rgb, *total, *workspace;
    int device;
};
struct InferGraphEntry {
    InferGraphKey key;
    cudaGraphExec_t exec;
    cudaGraph_t graph;
    bool used;
};
#define INFER_GRAPH_CACHE 8
static InferGraphEntry g_infer_graphs[INFER_GRAPH_CACHE];
static unsigned g_infer_graph_clock = 0;

static int build_infer_graph(const InferGraphKey& k, InferGraphEntry* e) {
    const NgpNet* net = &k.net;
    const NgpInferCfg* cfg = &k.cfg;
    const float* rays_o = (const float*)k.rays_o;
    const float* rays_d = (const float*)k.rays_d;
    const uint8_t* bitfield = (const uint8_t*)k.bitfield;
    float* opacity = (float*)k.opacity;
    float* depth = (float*)k.depth;
    float* rgb = (float*)k.rgb;
    const InferWs W = infer_ws(cfg, (void*)k.workspace);
    const int n = cfg->n_rays;
    cudaStream_t cs;
    NGP_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    cudaGraph_t g = nullptr;
    int rc = 0;
    do {
        if ((rc = (int)cudaGraphCreate(&g, 0))) break;
        // ---- head: clear the counters, AABB + first alive list ----
        if ((rc = (int)cudaStreamBeginCaptureToGraph(cs, g, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal))) break;
        cudaMemsetAsync(W.counters, 0, 4096, cs);
        k_infer_init<<<ngp_div_up(n, 256), 256, 0, cs>>>(*cfg, rays_o, rays_d, W.t_cur, W.t_end, opacity, depth, rgb, W.alive[0],
                                                          W.alive_cnt, W.alive_cnt + 1, W.state, W.total);
        cudaStreamCaptureStatus status;
        const cudaGraphNode_t* deps = nullptr;
        size_t n_deps = 0;
        if ((rc = (int)cudaStreamGetCaptureInfo(cs, &status, nullptr, nullptr, &deps, &n_deps))) break;
        cudaGraphNode_t head_tail[8];
        if (n_deps > 8) { rc = NGP_EINVAL; break; }
        for (size_t i = 0; i < n_deps; ++i) head_tail[i] = deps[i];
        cudaGraph_t tmp = nullptr;
        if ((rc = (int)cudaStreamEndCapture(cs, &tmp))) break;
        // ---- the WHILE node ----
        cudaGraphConditionalHandle handle;
        if ((rc = (int)cudaGraphConditionalHandleCreate(&handle, g, 1, cudaGraphCondAssignDefault))) break;
        cudaGraphNodeParams cp = {};
        cp.type = cudaGraphNodeTypeConditional;
        cp.conditional.handle = handle;
        cp.conditional.type = cudaGraphCondTypeWhile;
        cp.conditional.size = 1;
        cudaGraphNode_t loop;
        if ((rc = (int)cudaGraphAddNode(&loop, g, head_tail, n_deps, &cp))) break;
        cudaGraph_t body = cp.conditional.phGraph_out[0];
        if ((rc = (int)cudaStreamBeginCaptureToGraph(cs, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal))) break;
        for (int half = 0; half < 2 && !rc; ++half)  // the second round's compositing sets the loop condition
            rc = infer_round(net, cfg, W, rays_o, rays_d, bitfield, opacity, depth, rgb, half, cs, handle, half);
        int rc2 = (int)cudaStreamEndCapture(cs, &tmp);
        if (rc) break;
        if ((rc = rc2)) break;
        // ---- tail: background + total ----
        if ((rc = (int)cudaStreamBeginCaptureToGraph(cs, g, &loop, nullptr, 1, cudaStreamCaptureModeThreadLocal))) break;
        k_infer_finish<<<ngp_div_up(n, 256), 256, 0, cs>>>(*cfg, opacity, rgb, W.state, W.total, (int64_t*)k.total);
        if ((rc = (int)cudaStreamEndCapture(cs, &tmp))) break;
        cudaGraphExec_t exec = nullptr;
        if ((rc = (int)cudaGraphInstantiate(&exec, g, 0))) break;
        e->exec = exec;
        e->graph = g;
        e->key = k;
        e->used = true;
        g = nullptr;
    } while (0);
    if (rc) {
        // leave no capture open on the private stream
        cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(cs, &status) == cudaSuccess && status != cudaStreamCaptureStatusNone) {
            cudaGraph_t junk = nullptr;
            cudaStreamEndCapture(cs, &junk);
        }
        cudaGetLastError();
    }
    if (g) cudaGraphDestroy(g);
    cudaStreamDestroy(cs);
    return rc;
}

extern "C" int ngp_render_infer_frame(const NgpNet* net, const NgpInferCfg* cfg, const float* rays_o, const float* rays_d,
                                      const uint8_t* density_bitfield, float* opacity, float* depth, float* rgb,
                                      int64_t* total_samples, void* workspace, size_t workspace_bytes, void* stream) {
    if (!net || !cfg || !rays_o || !rays_d || !density_bitfield || !opacity || !depth || !rgb || !workspace) return NGP_EINVAL;
    if (cfg->n_rays < 1 || cfg->cascades < 1 || cfg->grid_size < 1 || cfg->grid_size > 1024 || cfg->max_samples < 1 ||
        cfg->max_round_samples < cfg->n_rays || cfg->max_round_samples > 0x7fffffffll || cfg->sample_budget < 1)
        return NGP_EINVAL;
    if (workspace_bytes < ngp_render_infer_workspace(cfg->n_rays, cfg->max_round_samples)) return NGP_EINVAL;
    InferGraphKey k;
    memset(&k, 0, sizeof(k));
    k.net = *net;
    k.cfg = *cfg;
    k.rays_o = rays_o; k.rays_d = rays_d; k.bitfield = density_bitfield; k.opacity = opacity; k.depth = depth; k.rgb = rgb;
    k.total = total_samples; k.workspace = workspace;
    NGP_CUDA(cudaGetDevice(&k.device));
    InferGraphEntry* hit = nullptr;
    InferGraphEntry* victim = &g_infer_graphs[g_infer_graph_clock % INFER_GRAPH_CACHE];
    for (int i = 0; i < INFER_GRAPH_CACHE; ++i) {
        InferGraphEntry* e = &g_infer_graphs[i];
        if (e->used && memcmp(&e->key, &k, sizeof(k)) == 0) { hit = e; break; }
        if (!e->used) victim = e;
    }
    if (!hit) {
        if (victim->used) {
            cudaGraphExecDestroy(victim->exec);
            cudaGraphDestroy(victim->graph);
            victim->used = false;
        }
        int rc = build_infer_graph(k, victim);
        if (rc) return rc;
        ++g_infer_graph_clock;
        hit = victim;
    }
    NGP_CUDA(cudaGraphLaunch(hit->exec, (cudaStream_t)stream));
    return 0;
}
