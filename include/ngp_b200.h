/* ngp_b200.h -- C ABI of the H100-native (sm_90a) hot path of kwea123/ngp_pl.
 *
 * This is the drop-in boundary. The reference's native surface for this path is the pybind11 module
 * `vren` (reference models/csrc/binding.cpp:234-250, prototypes in models/csrc/include/utils.h:9-126)
 * plus the tinycudann modules its models/networks.py:36-77 instantiates. Each entry point below names
 * the reference interface it replaces. Conventions:
 *   - plain device pointers + sizes; no torch types; the CALLER owns and allocates every buffer
 *     (workspace sizes are queried with the *_workspace functions);
 *   - `stream` is a cudaStream_t passed as void*; every launch is asynchronous on that stream;
 *   - return 0 on success, a cudaError_t (>0) on a CUDA failure, NGP_EINVAL (-22) on a bad argument;
 *   - all tensors are dense row-major ("contiguous" in the reference's CHECK_INPUT sense).
 */
#ifndef NGP_B200_H
#define NGP_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NGP_MAX_LEVELS 16
#define NGP_ABI_VERSION 15

int ngp_abi_version(void); /* == NGP_ABI_VERSION of the header the caller was built against */

/* Number of kernel launches this library has issued in this process so far -- eager launches and launches recorded
 * into a CUDA graph under stream capture alike (cub's kernels launched on its behalf included; a graph REPLAY does not
 * pass through the library, so a caller multiplies a graph's recorded count by its replays). Evidence for bench.py's
 * `gpu_launches`; no reference counterpart. */
unsigned long long ngp_launch_count(void);

/* Debugging aid (tools/step_timeline.py; no reference counterpart): install a device buffer of 2 + 2*capacity uint64
 * (buf[0] = 0, buf[1] = capacity, written by the caller) and the training-step entry points enqueue a one-thread kernel
 * after each of their kernels that appends {id, %globaltimer ns}. Recorded into CUDA graphs like any other launch, so
 * install it before capturing; NULL turns it off (the default). */
int ngp_trace_set(void* buf);

/* ----------------------------------------------------------------------------------------------
 * The twelve vren operators
 * -------------------------------------------------------------------------------------------- */

/* vren.ray_aabb_intersect (binding.cpp:4-16, intersection.cu:25-100). hits_t (n_rays,max_hits,2) and
 * hits_voxel_idx (n_rays,max_hits) are filled with -1 then written in hit order; hit_cnt (n_rays).
 * The reference sorts hits by t1 afterwards with torch ops; the Python shim does the same when
 * max_hits > 1 (the hot path uses n_voxels = max_hits = 1, where the sort is the identity). */
int ngp_ray_aabb_intersect(const float* rays_o, const float* rays_d, const float* centers, const float* half_sizes,
                           int n_rays, int n_voxels, int max_hits, int* hit_cnt, float* hits_t,
                           int64_t* hits_voxel_idx, void* stream);

/* vren.ray_sphere_intersect (binding.cpp:19-31, intersection.cu:103-197). */
int ngp_ray_sphere_intersect(const float* rays_o, const float* rays_d, const float* centers, const float* radii,
                             int n_rays, int n_spheres, int max_hits, int* hit_cnt, float* hits_t,
                             int64_t* hits_sphere_idx, void* stream);

/* vren.packbits (binding.cpp:34-43, raymarching.cu:122-161). dtype 0=f32 1=f16 2=f64; n_bytes = size of
 * density_bitfield; optional thr_dev (device float*): effective threshold = min(thr, *thr_dev), which
 * keeps `min(mean_density, thr)` of networks.py:266-269 on the device. */
int ngp_packbits(const void* density_grid, int dtype, int64_t n_bytes, float thr, const float* thr_dev,
                 uint8_t* density_bitfield, void* stream);

/* vren.morton3D / vren.morton3D_invert (binding.cpp:46-57, raymarching.cu:62-119); coords int32 (n,3). */
int ngp_morton3D(const int* coords, int n, int* indices, void* stream);
int ngp_morton3D_invert(const int* indices, int n, int* coords, void* stream);

/* vren.raymarching_train (binding.cpp:60-81, raymarching.cu:166-332). hits_t is (n_rays,2). Outputs:
 * rays_a int64 (n_rays,3) = [ray_idx,start_idx,N_samples] ordered by ray index; xyzs,dirs (>=total,3);
 * deltas,ts (>=total); counter int32[2] = [total_samples, n_rays]. Rows past `total` are not written. */
size_t ngp_raymarching_train_workspace(int n_rays);                     /* minimum (serial two-pass kernels) */
size_t ngp_raymarching_train_workspace2(int n_rays, int max_samples);   /* + staging rows: enables the warp-per-ray marcher */
int ngp_raymarching_train(const float* rays_o, const float* rays_d, const float* hits_t,
                          const uint8_t* density_bitfield, int cascades, float scale, float exp_step_factor,
                          const float* noise, int grid_size, int max_samples, int n_rays,
                          int64_t* rays_a, float* xyzs, float* dirs, float* deltas, float* ts, int* counter,
                          void* workspace, size_t workspace_bytes, void* stream);

/* vren.raymarching_test (binding.cpp:84-106, raymarching.cu:335-454). hits_t (n_rays_total,2) is
 * MUTATED ([r][0] advanced); outputs are (n_alive,N_samples[,3]) with zero padding. */
int ngp_raymarching_test(const float* rays_o, const float* rays_d, float* hits_t, const int64_t* alive_indices,
                         const uint8_t* density_bitfield, int cascades, float scale, float exp_step_factor,
                         int grid_size, int max_samples, int N_samples, int n_alive,
                         float* xyzs, float* dirs, float* deltas, float* ts, int* N_eff_samples, void* stream);

/* vren.composite_train_fw (binding.cpp:109-126, volumerendering.cu:6-84). */
int ngp_composite_train_fw(const float* sigmas, const float* rgbs, const float* deltas, const float* ts,
                           const int64_t* rays_a, float T_threshold, int n_rays, int64_t n_samples,
                           int64_t* total_samples, float* opacity, float* depth, float* rgb, float* ws, void* stream);

/* vren.composite_train_bw (binding.cpp:129-163, volumerendering.cu:87-202). */
int ngp_composite_train_bw(const float* dL_dopacity, const float* dL_ddepth, const float* dL_drgb, const float* dL_dws,
                           const float* sigmas, const float* rgbs, const float* ws, const float* deltas, const float* ts,
                           const int64_t* rays_a, const float* opacity, const float* depth, const float* rgb,
                           float T_threshold, int n_rays, int64_t n_samples, float* dL_dsigmas, float* dL_drgbs,
                           void* stream);

/* vren.composite_test_fw (binding.cpp:166-194, volumerendering.cu:205-285); alive_indices, opacity,
 * depth, rgb are updated in place. */
int ngp_composite_test_fw(const float* sigmas, const float* rgbs, const float* deltas, const float* ts,
                          const float* hits_t, int64_t* alive_indices, float T_threshold, const int* N_eff_samples,
                          int n_alive, int N_samples, float* opacity, float* depth, float* rgb, void* stream);

/* vren.distortion_loss_fw / _bw (binding.cpp:197-231, losses.cu:10-174). n_samples is the extent of the per-sample
 * arrays (ws, deltas, ts, the scans, dL_dws): each ray's segment [start, start + count) is clipped to it, and a ray
 * clipped to nothing gets loss 0 and no per-sample writes. */
int ngp_distortion_loss_fw(const float* ws, const float* deltas, const float* ts, const int64_t* rays_a, int n_rays,
                           int64_t n_samples, float* loss, float* ws_inclusive_scan, float* wts_inclusive_scan,
                           void* stream);
int ngp_distortion_loss_bw(const float* dL_dloss, const float* ws_inclusive_scan, const float* wts_inclusive_scan,
                           const float* ws, const float* deltas, const float* ts, const int64_t* rays_a, int n_rays,
                           int64_t n_samples, float* dL_dws, void* stream);

/* ----------------------------------------------------------------------------------------------
 * The network the reference builds from tinycudann modules (models/networks.py:36-77):
 *   xyz_encoder = HashGrid(L levels, F=2, T=2^log2_T, N_min, b) -> MLP 32->64(ReLU)->16
 *   dir_encoder = SH degree 4 ;  rgb_net = MLP 32->64->64->3(pad 16), Sigmoid
 * Parameter layout (tinycudann's): xyz_encoder.params = [W1 64x32 | W2 16x64 | table entries*2],
 * rgb_net.params = [W1 64x32 | W2 64x64 | W3 16x64], every matrix row-major (out,in).
 * -------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n_levels;
    uint32_t hashed_mask;                 /* bit l set: level l is hashed (res^3 > entries) */
    uint32_t offset[NGP_MAX_LEVELS + 1];  /* in entries (one entry = F=2 features) */
    uint32_t res[NGP_MAX_LEVELS];
    float scale[NGP_MAX_LEVELS];
} NgpGridMeta;

/* Host-side: level table of the hash grid (no GPU needed) for the encoding config the reference builds at
 * models/networks.py:32-33,39-49 (L, F=2, log2_T, N_min, b = exp(log(2048*scale/N_min)/(L-1))). Returns total entries,
 * 0 on bad input. */
uint32_t ngp_grid_meta(int n_levels, int log2_hashmap_size, int base_resolution, float per_level_scale,
                       NgpGridMeta* out);

#define NGP_DENSITY_MLP_PARAMS 3072 /* 64*32 + 16*64 */
#define NGP_RGB_MLP_PARAMS 7168     /* 64*32 + 64*64 + 16*64 */

/* fp32 -> fp16 working copy of a parameter vector (the tinycudann modules of models/networks.py:36-77 keep one flat fp32
 * `params` and cast it to fp16 on every forward). */
int ngp_cast_params(const float* src, uint16_t* dst_half, int64_t n, void* stream);

typedef struct {
    const uint16_t* enc_params_h; /* fp16 xyz_encoder params: [3072 MLP | table] */
    const uint16_t* rgb_params_h; /* fp16 rgb_net params (7168) */
    NgpGridMeta meta;
    float xyz_min[3];
    float xyz_max[3];
    int32_t rgb_act; /* 1 = Sigmoid (reference default), 0 = None */
} NgpNet;

/* Sample positions are given EITHER as xyzs+dirs (n,3) arrays (ray_idx == NULL) -- the signature of
 * NGP.forward(x, d), networks.py:132 -- OR as (rays_o, rays_d, ray_idx, ts): x = fma(d, t, o). */
typedef struct {
    const float* xyzs;
    const float* dirs;
    const float* rays_o;
    const float* rays_d;
    const int32_t* ray_idx;
    const float* ts;
    int64_t n;            /* number of samples, or the CAPACITY when n_dev is set */
    const int32_t* n_dev; /* optional device int32: the kernels read the sample count from here (no host sync) */
    /* backward only (ngp_net_backward*; a live list needs feat_save): visit just the samples live_idx[0 .. *n_live_dev),
     * i.e. those whose upstream gradient can be non-zero -- the samples past a ray's termination receive exactly
     * zero gradient from composite_train_bw (volumerendering.cu:87-151) and contribute +0 to every sum. NULL = all. */
    const int32_t* live_idx;
    const int32_t* n_live_dev;
} NgpSamples;

/* Fused forward of NGP.forward (networks.py:132-153): hash gather + trilinear + density MLP +
 * exp + SH + rgb MLP + sigmoid, one kernel. sigmas fp32 (n), rgbs fp32 (n,3) (values are
 * fp16-representable, as tinycudann returns fp16). feat_save (optional, 64 B/sample, opaque fragment
 * order) keeps the encoded features for ngp_net_backward. want_rgb = 0 evaluates NGP.density only. */
int ngp_net_forward(const NgpNet* net, const NgpSamples* smp, int want_rgb, float* sigmas, float* rgbs,
                    uint16_t* h_out /* optional fp16 (n,16) */, void* feat_save /* 16-B aligned */, void* stream);

size_t ngp_net_backward_workspace(int64_t n); /* 64 B per sample: feature gradients [level][sample] */
/* Fused backward of NGP.forward (what autograd runs through models/networks.py:132-153 and TruncExp.backward,
 * models/custom_functions.py:168-173): recomputes the MLP activations from feat_save (or by re-gathering when NULL),
 * back-propagates dL/dsigmas (n) and dL/drgbs (n,3), accumulates
 *   grad_enc (fp32, same layout as xyz_encoder.params) and grad_rgb (fp32, 7168)   with atomics (+=).
 * loss_scale (device float*, optional) is the power-of-two the fp16 gradient operands are scaled by
 * internally (results are un-scaled); NULL = 1. Two kernels: the MLP backward (dgrad + wgrad on tensor
 * cores) writes the feature gradients to `workspace`; the scatter kernel (one thread per sample and level,
 * duplicate cells merged inside the warp) turns them into vector reductions on the table gradient.
 * With smp->n_dev the workspace must cover the capacity smp->n. */
int ngp_net_backward(const NgpNet* net, const NgpSamples* smp, const float* dL_dsigmas, const float* dL_drgbs,
                     const void* feat_save, const float* loss_scale, float* grad_enc, float* grad_rgb,
                     void* workspace, size_t workspace_bytes, void* stream);

/* The two halves of ngp_net_backward, individually callable (profiling; overlapping them with other work).
 * Both launch as programmatic dependents of the kernel before them on the stream (they may start under its tail):
 * the MLP half reads the fp16 weights, and the scatter half the sample count, live list and sample positions, before
 * waiting for that kernel, so these must not be written by the kernel issued immediately before the call. */
int ngp_net_backward_mlp(const NgpNet* net, const NgpSamples* smp, const float* dL_dsigmas, const float* dL_drgbs,
                         const void* feat_save, const float* loss_scale, float* grad_enc, float* grad_rgb,
                         void* workspace, size_t workspace_bytes, void* stream);
int ngp_net_backward_scatter(const NgpNet* net, const NgpSamples* smp, const float* loss_scale, float* grad_enc,
                             void* workspace, size_t workspace_bytes, void* stream);

/* Stand-alone module kernels for callers that use the three tinycudann modules one by one, as the
 * reference's NGP.forward does (models/networks.py:104,144-145); see ngp_pl_b200/tcnn.py.
 *   ngp_sh_encode        : tcnn.Encoding(SphericalHarmonics deg 4): u in [0,1]^3 (n,3) fp32 -> fp16 (n,16)
 *   ngp_mlp_rgb_forward  : tcnn.Network 32->64->64->3 on x fp16 (n,32) -> fp16 (n,3)
 *   ngp_mlp_rgb_backward : dL/dout fp32 (n,3) -> dL/dx fp32 (n,32) (optional) and grad_rgb (+=, fp32 7168)
 *   ngp_enc_backward     : tcnn.NetworkWithInputEncoding backward from dL/dh fp32 (n,16); forward is
 *                          ngp_net_forward(want_rgb=0, h_out, feat_save); workspace as ngp_net_backward
 * Alignment (NGP_EINVAL otherwise, before any device work): x_half 4 B, dL_dx and dL_dh 8 B, out_half and
 * feat_save 16 B. */
int ngp_sh_encode(const float* u01, int64_t n, uint16_t* out_half, void* stream);
int ngp_mlp_rgb_forward(const uint16_t* rgb_params_h, const uint16_t* x_half, int64_t n, int rgb_act, uint16_t* out_half3,
                        void* stream);
int ngp_mlp_rgb_backward(const uint16_t* rgb_params_h, const uint16_t* x_half, const float* dL_dout3, int64_t n, int rgb_act,
                         const float* loss_scale, float* dL_dx, float* grad_rgb, void* stream);
int ngp_enc_backward(const NgpNet* net, const NgpSamples* smp, const float* dL_dh, const void* feat_save,
                     const float* loss_scale, float* grad_enc, void* workspace, size_t workspace_bytes, void* stream);

/* loss_scale helper (the role PL's GradScaler plays for Trainer(precision=16), train.py:274, and tinycudann's fixed
 * loss_scale = 128): *scale_out = 2^floor(log2(256 / max(|dL_dsigmas*sigma'|, |dL_drgbs|))) (1 if all zero). */
int ngp_grad_scale(const float* dL_dsigmas, const float* sigmas, const float* dL_drgbs, int64_t n,
                   float* scratch /* 1 float */, float* scale_out, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Fused training path: the body of render(..., test_time=False) (reference models/rendering.py:11-43,
 * :121-163) without a single host synchronisation -- AABB + near clamp + march + segment allocation (one
 * kernel: per-ray staging, one atomicAdd per ray hands out its segment, coalesced copy-out) -> ngp_net_forward ->
 * ragged compositing, and its backward.
 * All sample counts stay on the device; every per-sample buffer is sized for `max_total_samples`
 * (n_rays * max_samples can never overflow).
 * -------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n_rays, cascades, grid_size, max_samples;
    float scale, exp_step_factor, T_threshold, near_distance;
    float center[3], half_size[3], bg[3];
    float lambda_opacity;      /* NeRFLoss lambda_opacity (reference losses.py:41) */
    int64_t max_total_samples; /* capacity of the per-sample buffers */
} NgpTrainCfg;

typedef struct {
    /* inputs */
    const float* rays_o;          /* (n_rays,3) */
    const float* rays_d;          /* (n_rays,3) unnormalised */
    const float* noise;           /* (n_rays) start jitter in [0,1) */
    const uint8_t* density_bitfield;
    /* per-ray */
    float* stage_t;               /* (n_rays*max_samples) marcher staging */
    float* stage_dt;              /* (n_rays*max_samples) */
    int32_t* n_samples;           /* (n_rays) marched samples per ray == rays_a[:,2] */
    int32_t* offsets;             /* (n_rays) first sample of the ray == rays_a[:,1]; segments are handed out in arrival order
                                     (like the reference's atomic rays_a, raymarching.cu:237-241) and partition [0, total) */
    int32_t* counters;            /* int32[8]: [0] marched samples (rm_samples), [1] composited (vr_samples) of the step in flight;
                                     [2],[3] the same, snapshotted by ngp_nerf_loss_grad for the last completed step;
                                     [4] append cursor of live_idx while the compositing backward runs (0 otherwise), [5] length of live_idx,
                                     [6..7] free for the caller (the Trainer keeps its ngp_sample_rays draw counter there) */
    float* rgb;                   /* (n_rays,3) composited colour incl. background */
    float* opacity;               /* (n_rays) */
    float* depth;                 /* (n_rays) */
    /* per-sample (capacity max_total_samples) */
    int32_t* ray_idx;
    float* ts;
    float* deltas;
    float* sigmas;
    float* rgbs;                  /* (S,3) */
    float* ws;                    /* (S) optional (NULL: not materialised) */
    float* dsigmas;               /* (S)   backward scratch */
    float* drgbs;                 /* (S,3) backward scratch */
    int32_t* live_idx;            /* (S) optional: samples with a non-zero upstream gradient, built by the compositing
                                     backward; the network backward then visits only those */
    void* feat_save;              /* ceil32(S)*64 bytes */
    float* scalars;               /* float[8]: [0] amax scratch, [1] loss scale, [2] sum sq err, [3] sum opacity entropy of the last
                                     step, [4],[5] their accumulators inside ngp_render_train_step (zero otherwise) */
    void* scan_temp;
    size_t scan_temp_bytes;
    void* bwd_workspace;          /* ngp_net_backward_workspace(max_total_samples) bytes */
    size_t bwd_workspace_bytes;
    const float* bg_dev;          /* optional device float[3]: background colour of THIS batch, overrides cfg.bg (the
                                     reference's random_bg draws one colour per training batch, rendering.py:153-161) */
} NgpTrainBuffers;

size_t ngp_train_scan_temp_bytes(int n_rays); /* NgpTrainBuffers.scan_temp size; the buffer must be ZERO-INITIALISED once by the caller
                                                 (accumulators of the march kernel's segment allocation, re-armed by the kernel) */

/* forward = __render_rays_train (models/rendering.py:121-163) incl. the AABB test and near clamp of render() (:25-29):
 * fills per-ray rgb/opacity/depth (+ws) and everything the backward needs */
int ngp_render_train_fwd(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* buf, void* stream);
/* its two halves: _march (AABB + march + segment allocation + copy-out; independent of the weights, so it may overlap the
 * optimiser of the previous step) and _net (network + compositing). _fwd == _march then _net. */
int ngp_render_train_march(const NgpTrainCfg* cfg, const NgpTrainBuffers* buf, void* stream);
int ngp_render_train_net(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* buf, void* stream);

/* Weight-dependent part of one training step with the plain NeRFLoss (losses.py:47-60, no distortion term) in one call:
 * network forward -> ONE kernel for {compositing forward, loss + its per-ray gradients, compositing backward} -> loss
 * scale -> MLP backward -> table scatter. Equivalent to ngp_render_train_net + ngp_nerf_loss_grad + ngp_render_train_bwd
 * (needs dsigmas, drgbs, feat_save; fills rgb/opacity/depth, scalars[2..3], counters[2..3]). */
int ngp_render_train_step(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* b, const float* rgb_gt,
                          float* grad_enc, float* grad_rgb, void* stream);

/* backward of the above from per-ray gradients = VolumeRenderer.backward (models/custom_functions.py:148-159) followed by
 * the network backward (dL_ddepth / dL_dws may be NULL = 0); accumulates (+=) into the fp32 gradient vectors laid out like
 * the parameter vectors. */
int ngp_render_train_bwd(const NgpNet* net, const NgpTrainCfg* cfg, const NgpTrainBuffers* buf,
                         const float* dL_drgb, const float* dL_dopacity, const float* dL_ddepth, const float* dL_dws,
                         float* grad_enc, float* grad_rgb, void* stream);

/* NeRFLoss (reference losses.py:47-60, distortion off) and its per-ray gradients, on the device:
 * loss = mean((rgb-gt)^2) + lambda_opacity*mean(-o*log(o)), o = opacity+1e-10.
 * Adds the two sums into buf->scalars[2], [3] (caller zeroes them) and writes dL_drgb (n,3), dL_dopacity (n). */
int ngp_nerf_loss_grad(const NgpTrainCfg* cfg, const NgpTrainBuffers* buf, const float* rgb_gt,
                       float* dL_drgb, float* dL_dopacity, void* stream);

/* Fused Adam over a flat fp32 vector (apex FusedAdam semantics as the reference uses it, train.py:131:
 * adam_w_mode, weight_decay 0, bias correction, eps): p -= lr * m_hat / (sqrt(v_hat) + eps), with
 * g = grads * grad_mul (1/world_size after a sum all-reduce). The bias corrections are apex's: 1 - beta^t computed in
 * double and rounded to float once (in float, 1 - powf(0.999, t) loses ~100 roundings to cancellation at small t).
 * ngp_adam_step_p2p / _fused share this update: on the same inputs they agree with it bit for bit. Also refreshes
 * the fp16 working copy and
 * zeroes the gradient for the next step in the same pass. lr and step live on the device
 * (lr_dev[0], step_dev[0] = number of completed steps; the kernel uses t = step+1 and a follow-up
 * single-thread kernel increments it) so a captured CUDA graph never needs re-capturing. Launched as a programmatic
 * dependent of the kernel before it on the stream: params, exp_avg, exp_avg_sq, lr and step are read before waiting
 * for that kernel, so they must not be written by the kernel issued immediately before the call. */
int ngp_adam_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, uint16_t* params_half, int64_t n,
                  const float* lr_dev, int32_t* step_dev, float beta1, float beta2, float eps, float grad_mul,
                  int increment_step, void* stream);

/* Data-parallel optimiser step FUSED with its collective over NVLink peer memory (N ranks of one node); replaces the DDP
 * gradient all-reduce (train.py:269-272, DDPPlugin) + FusedAdam.step (train.py:131-137) of the reference:
 * rank `rank` reduces its 1/N shard of the gradient directly from every rank's gradient buffer (P2P loads),
 * applies Adam (mean gradient, same semantics as ngp_adam_step) to that shard of params / exp_avg /
 * exp_avg_sq, and stores the shard's new fp16 parameters into every rank's working copy (P2P stores).
 * peer_grads / peer_params_half: HOST arrays of `world` device addresses valid on this rank (symmetric
 * memory; index = rank). The caller must barrier across ranks before (all gradients written) and after
 * (all parameter stores visible), then clear its own gradient buffer. n must be a multiple of 4. */
int ngp_adam_step_p2p(int world, int rank, const uint64_t* peer_grads, float* params, float* exp_avg, float* exp_avg_sq,
                      const uint64_t* peer_params_half, int64_t n, const float* lr_dev, int32_t* step_dev, float beta1,
                      float beta2, float eps, int increment_step, void* stream);

/* The same exchange as ONE self-synchronising, CUDA-graph-capturable kernel (no host-side barriers):
 *   start barrier (flag words in symmetric memory) -> reduce-scatter + Adam on the owned shard + all-gather of the
 *   new fp16 parameters -> end barrier; the kernel ends only when this rank's working copy is complete and every
 *   peer is done reading this rank's gradients.
 * peer_flags: HOST array of `world` device addresses of each rank's flag block (>= 32 uint32, symmetric memory,
 * zero-initialised once, never reset). mc_grads / mc_params_half: NVLS multicast aliases of the gradient buffer /
 * the fp16 working copy (0 = none): with them the reduction is one multimem.ld_reduce and the all-gather one
 * multimem.st per 16 bytes (the switch sums / replicates; summation order then differs from NCCL's).
 * zero_buf (may be NULL): a LOCAL fp32 buffer of n elements cleared inside the kernel -- the gradient buffer the
 * NEXT step accumulates into; gradient buffers must alternate between steps, the buffer being reduced is left
 * untouched. sync: >= 4 uint32 of local device memory, zero-initialised once ([2] != 0 afterwards = a peer never
 * arrived: timeout). n must be a multiple of 4. */
int ngp_adam_step_fused(int world, int rank, const uint64_t* peer_grads, const uint64_t* peer_params_half,
                        const uint64_t* peer_flags, uint64_t mc_grads, uint64_t mc_params_half, float* params,
                        float* exp_avg, float* exp_avg_sq, int64_t n, float* zero_buf, uint32_t* sync,
                        const float* lr_dev, int32_t* step_dev, float beta1, float beta2, float eps,
                        int increment_step, void* stream);

/* Per-step training log (Trainer(log_rows=R); the reference logs train/loss, train/psnr, train/rm_s, train/vr_s and lr
 * every step, train.py:175-183): one single-block kernel that writes one row of a caller-owned device ring
 * log[rows][8] (int32 words) without any host counter, so that one captured CUDA graph writes the right row on every
 * replay. Launch it after the step's optimiser, which has advanced *step_dev: the row is (*step_dev - 1) mod rows and
 * holds
 *   [0] scalars[2] (sum of squared errors, fp32 bits)   [1] scalars[3] (sum of opacity entropy, fp32 bits)
 *   [2] counters[2] (ray-marched samples)                [3] counters[3] (volume-rendered samples)
 *   [4] counters[5] (samples the backward visited)       [5] *lr_dev (fp32 bits)
 *   [6] sum of dist_loss[0 .. n_dist) (fp32 bits; 0 when n_dist == 0, fixed-order double reduction)
 *   [7] *step_dev - 1 (the step's index)
 * scalars / counters: the step's NgpTrainBuffers fields. dist_loss may be NULL when n_dist == 0. Launched as a
 * programmatic dependent of the kernel before it; it reads nothing before that kernel has completed, and the kernel
 * after it starts once it has completed. */
int ngp_train_log_step(const float* scalars, const int32_t* counters, const float* lr_dev, const int32_t* step_dev,
                       const float* dist_loss, int64_t n_dist, int32_t* log, int rows, void* stream);

/* Batch assembly on the device (reference train.py:78-91 + datasets/ray_utils.py:46-70 + base.py:22-30):
 * rays_d = directions[pix] @ R^T, rays_o = c2w[:,3], rgb_gt = images[img, pix] / 255. */
int ngp_gen_rays(const int64_t* img_idx, const int64_t* pix_idx, const float* poses /* (n_img,3,4) */,
                 const float* directions /* (n_pix,3) */, const uint8_t* images /* (n_img,n_pix,3) or NULL */,
                 int64_t n_pix, int n, float* rays_o, float* rays_d, float* rgb_gt, void* stream);

/* The same with the random draw on the device, in one kernel: every ray gets a uniform (image, pixel) pair with
 * replacement (reference datasets/base.py:22-30, ray sampling strategy 'all_images') and its start jitter noise[i] in [0,1)
 * (reference custom_functions.py:84) from Philox-4x32-10 keyed by (seed, stream_id) with counter (ray, draw); rng_draw is a
 * device int32[2] {draw counter, scratch 0}, advanced by the kernel, so CUDA-graph replays draw fresh batches. */
int ngp_sample_rays(const float* poses, const float* directions, const uint8_t* images, int n_img, int64_t n_pix, int n,
                    uint32_t seed, uint32_t stream_id, int32_t* rng_draw, float* rays_o, float* rays_d, float* rgb_gt,
                    float* noise, void* stream);

/* ngp_sample_rays for any bank: image_dtype 0 = uint8 (rgb_gt = v/255, bitwise ngp_sample_rays) or 1 = float32 (rgb_gt = the
 * stored value); strategy 0 = 'all_images' (bitwise ngp_sample_rays) or 1 = 'same_image' (reference datasets/base.py:27-28:
 * ONE image per batch, drawn as umulhi(Philox(counter (0, draw, 1, 0)).x, n_img) -- a counter no per-ray draw uses -- while
 * pixels and jitter are those 'all_images' draws). Other values return NGP_EINVAL. */
int ngp_sample_rays_ex(const float* poses, const float* directions, const void* images /* (n_img,n_pix,3) */, int image_dtype,
                       int strategy, int n_img, int64_t n_pix, int n, uint32_t seed, uint32_t stream_id, int32_t* rng_draw,
                       float* rays_o, float* rays_d, float* rgb_gt, float* noise, void* stream);

/* Image staging (reference datasets/color_utils.py:19-31, read_image(path, (dst_w, dst_h), blend_a)): a decoded uint8
 * (src_h, src_w, channels) image, channels 3 or 4, becomes fp32 (dst_h*dst_w, 3): v/255 correctly rounded; with 4 channels
 * c*a + (1-a) (blend_a != 0) or c*a; then cv2.resize's INTER_LINEAR on fp32 when the size changes (a copy otherwise).
 * Bitwise equal to the reference's arithmetic (oracle/stage_ref.py states the evaluation order). A resize needs
 * src_h, src_w >= 2. */
int ngp_stage_image(const uint8_t* src, int src_h, int src_w, int channels, int blend_a, int dst_h, int dst_w, float* dst,
                    void* stream);

/* Occupancy-grid refresh on the device (reference networks.py:240-269 + :169-195), no host sync:
 * picks cells (all cells when warmup, else M uniform + M occupied per cascade), evaluates sigma at a
 * jittered point of each, grid = grid<0 ? grid : max(grid*decay, sigma), threshold = min(mean of
 * positive cells, density_threshold), packs the bitfield. With count_grid (networks.py:258-260, `erode`): per-cell
 * decay = clamp(decay^(1/count), 0.1, 0.95). workspace: see ngp_update_grid_workspace. */
size_t ngp_update_grid_workspace(int cascades, int grid_size);
int ngp_update_density_grid(const NgpNet* net, float* density_grid /* (cascades, G^3) */, uint8_t* density_bitfield,
                            const float* count_grid /* (cascades, G^3) camera coverage for `erode`, or NULL */,
                            int cascades, int grid_size, float scale, float density_threshold, int warmup, float decay,
                            uint32_t seed, void* workspace, size_t workspace_bytes, void* stream);
/* The same refresh in two halves, ngp_update_density_grid == pick then eval on one stream. `pick` needs only the OLD grid
 * and the seed (which cells, sorted in Morton order, and the jittered point in each; clears the scratch grid), so a trainer
 * runs it on a side stream any time after the previous refresh and only `eval` (density at the points, merge, threshold,
 * bitfield) sits between two training steps. A cell picked more than once is evaluated once (the reference's index_put
 * keeps an arbitrary one of the duplicates), at a point hashed from the cell's rank among the cascade's distinct picks in
 * Morton order -- not from any of its pick slots. grid_size must be a power of two in [2, 1024], cascades in [1, 62] and
 * cascades * grid_size^3 < 2^31; both halves return NGP_EINVAL otherwise. Both halves must see the same workspace,
 * cascades, grid_size, threshold and warmup, and nothing else may touch the workspace in between. */
int ngp_update_density_grid_pick(const float* density_grid, int cascades, int grid_size, float scale, float density_threshold,
                                 int warmup, uint32_t seed, void* workspace, size_t workspace_bytes, void* stream);
int ngp_update_density_grid_eval(const NgpNet* net, float* density_grid, uint8_t* density_bitfield, const float* count_grid,
                                 int cascades, int grid_size, float density_threshold, int warmup, float decay, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Fused inference path: render(..., test_time=True) (reference models/rendering.py:46-118) as a
 * device-side wavefront without host synchronisation. rays are (n_rays,3); outputs opacity, depth
 * (n_rays), rgb (n_rays,3, background included); total_samples (device int64, optional) = the
 * reference's result['total_samples'].
 * -------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n_rays, cascades, grid_size, max_samples; /* max_samples: the marcher's MAX_SAMPLES (step lower bound) */
    float scale, exp_step_factor, T_threshold, near_distance;
    float center[3], half_size[3], bg[3];
    int32_t sample_budget;      /* reference kwarg `max_samples` of the outer loop (default 1024) */
    int64_t max_round_samples;  /* capacity of the per-round sample buffers, shared fairly by the alive rays */
} NgpInferCfg;

size_t ngp_render_infer_workspace(int n_rays, int64_t max_round_samples); /* workspace of ngp_render_infer */

/* Where the wavefront keeps its per-round state inside that workspace, for callers that inspect it between rounds of
 * ngp_render_infer. Fills offsets[NGP_INFER_LAYOUT_FIELDS] with the byte offset of each array below (offsets may be
 * NULL) and returns the workspace size, ngp_render_infer_workspace's value; 0 when n_rays or max_round_samples < 1.
 *   per ray r (n_rays entries):        T_CUR (float) next parameter to march from; T_END (float) the box exit
 *                                      (-1 for a miss)
 *   per alive-list position i:         ALIVE0 / ALIVE1 (int32) the two alive lists, ray ids; round k reads list k & 1
 *                                      and appends the survivors to the other, in no particular order;
 *                                      RAY_START / RAY_N (int32) first slot and sample count of alive[i] this round
 *   per slot (max_round_samples):      RAY_IDX (int32, -1 = unused slot), TS, DELTAS, SIGMAS (float), RGBS (float x 3)
 *   COUNTERS: int32 alive counts of list 0 and 1 at bytes 0 and 4; int32 state[7] at NGP_INFER_STATE_OFFSET:
 *     state[0] N_samples of the coming round (0 = loop over)  [1] samples requested so far (the reference's `samples`)
 *     [2] slots the network evaluates this round  [3] rounds run  [4] samples marched this round
 *     [5] 1 = warp-per-ray marching (N_samples >= 8), 0 = thread-per-ray  [6] finished-block ticket (0 between rounds);
 *   and the int64 running total of marched samples at NGP_INFER_TOTAL_OFFSET (total_samples = it + state[4]).
 * In the thread-per-ray regime the rays' slot ranges are packed into [0, state[2]); in the warp-per-ray regime ray i
 * owns slots [i * N_samples, (i + 1) * N_samples) and state[2] = N_alive * N_samples. */
#define NGP_INFER_T_CUR 0
#define NGP_INFER_T_END 1
#define NGP_INFER_ALIVE0 2
#define NGP_INFER_ALIVE1 3
#define NGP_INFER_RAY_START 4
#define NGP_INFER_RAY_N 5
#define NGP_INFER_RAY_IDX 6
#define NGP_INFER_TS 7
#define NGP_INFER_DELTAS 8
#define NGP_INFER_SIGMAS 9
#define NGP_INFER_RGBS 10
#define NGP_INFER_COUNTERS 11
#define NGP_INFER_LAYOUT_FIELDS 12
#define NGP_INFER_STATE_OFFSET 32 /* bytes into COUNTERS */
#define NGP_INFER_TOTAL_OFFSET 64 /* bytes into COUNTERS */
size_t ngp_render_infer_layout(int n_rays, int64_t max_round_samples, int64_t* offsets);
/* Runs rounds [first_round, first_round+n_rounds) of the wavefront (first_round == 0 initialises; finish != 0
 * adds the background and writes total_samples). Per round every alive ray takes up to the reference's quota
 * N_samples = max(min(n_rays / n_alive, 64), min_samples) (rendering.py:73,80; min_samples = 1 if exp_step_factor == 0
 * else 4), evaluated on the device from the alive count; the alive-list rules are composite_test_fw's
 * (volumerendering.cu:221-248), so total_samples reproduces the operator loop's. alive_count_out (device int32*,
 * optional) gets the number of rays still alive afterwards -- reading it back every few rounds is the only host
 * synchronisation of the path. Requires max_round_samples >= 4 * n_rays for the quota never to be clipped
 * (>= n_rays to run at all). */
int ngp_render_infer(const NgpNet* net, const NgpInferCfg* cfg, const float* rays_o, const float* rays_d,
                     const uint8_t* density_bitfield, float* opacity, float* depth, float* rgb, int64_t* total_samples,
                     int first_round, int n_rounds, int finish, int* alive_count_out,
                     void* workspace, size_t workspace_bytes, void* stream);

/* The same wavefront for a WHOLE frame as one CUDA graph with a device-side loop (a conditional WHILE node whose
 * condition a kernel sets from the alive count): init -> while (rays alive and samples < sample_budget) { round } ->
 * finish. One graph launch per call, no host read-back at all (the reference's loop synchronises >= 3 times per round,
 * rendering.py:75-105). The instantiated graph is cached per (device, every pointer argument, *net, *cfg) -- up to 8
 * entries, rebuilt on a miss -- so callers should render from the same buffers frame after frame. Not thread-safe.
 * Returns a cudaError_t if the driver cannot build conditional graph nodes (callers may then fall back to
 * ngp_render_infer). */
int ngp_render_infer_frame(const NgpNet* net, const NgpInferCfg* cfg, const float* rays_o, const float* rays_d,
                           const uint8_t* density_bitfield, float* opacity, float* depth, float* rgb, int64_t* total_samples,
                           void* workspace, size_t workspace_bytes, void* stream);

/* One frame of the interactive viewer (the reference's show_gui.py render_cam: get_rays, render(test_time=True),
 * depth2img) as ONE cached CUDA graph, from camera pose to JPEG file:
 *   1. a memcpy node copies the 3x4 camera-to-world pose (12 floats, row-major [R | t]) from `pose`, which must be
 *      pinned host memory, into the workspace -- every launch reads the buffer's contents at that moment, so moving the
 *      camera never rebuilds the graph;
 *   2. rays_d = directions @ R^T, rays_o = t for every pixel (directions (H*W, 3) device), with ngp_gen_rays' arithmetic:
 *      rays_o / rays_d (H*W, 3) are bitwise ngp_gen_rays with img_idx = 0, pix_idx = 0 .. H*W-1 on that pose;
 *   3. the wavefront of ngp_render_infer_frame on those rays (opacity, depth, rgb as it writes them);
 *   4. ngp_view_images of the chosen output only (mode 0: rgb_img of rgb, 1: depth_img of depth), then ngp_jpeg_encode
 *      of that image at view->quality into jpeg.
 * stats (int64[2]): [0] the JPEG's length, [1] total_samples. jpeg and stats may be device memory or mapped pinned host
 * memory (as for ngp_jpeg_encode), so only the file's bytes cross PCIe; nothing in the call synchronises the stream.
 * Graphs are cached as ngp_render_infer_frame's are (up to 8, per device, every pointer argument, *net, *cfg and *view):
 * the two modes are two entries, and toggling between them rebuilds nothing once both exist. Not thread-safe.
 * workspace: ngp_render_view_workspace(cfg, view) bytes, 256-B aligned -- ngp_render_infer_workspace's, then the pose,
 * the ngp_view_images workspace, the (H, W, 3) display image and the ngp_jpeg_workspace(H, W) -- or 0 when
 * H * W != cfg->n_rays or ngp_jpeg_workspace(H, W) is 0. NGP_EINVAL for H * W != n_rays, an unknown mode, a quality
 * outside 1..100, jpeg_capacity < ngp_jpeg_capacity(H, W), a NULL pointer, a pose that is not pinned host memory, another
 * pointer the device cannot reach, stats not 8-B aligned, a short or misaligned workspace, and everything
 * ngp_render_infer_frame refuses. A cudaError_t if the driver cannot build conditional graph nodes; there is no other
 * path. */
typedef struct {
    int32_t mode;    /* 0 = rgb_img, 1 = depth_img (ngp_view_images' two outputs) */
    int32_t quality; /* JPEG quality 1..100 */
    int32_t H, W;    /* H * W == cfg->n_rays */
} NgpViewCfg;
size_t ngp_render_view_workspace(const NgpInferCfg* cfg, const NgpViewCfg* view);
int ngp_render_view_frame(const NgpNet* net, const NgpInferCfg* cfg, const NgpViewCfg* view, const float* directions,
                          const float* pose, const uint8_t* density_bitfield, float* rays_o, float* rays_d, float* opacity,
                          float* depth, float* rgb, uint8_t* jpeg, size_t jpeg_capacity, int64_t* stats,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Validation metrics of one rendered view (reference train.py:193-237): the per-image PSNR of torchmetrics'
 * PeakSignalNoiseRatio(data_range=1) / metrics.py:14-15 and SSIM of StructuralSimilarityIndexMeasure(data_range=1)
 * (11-tap Gaussian window, sigma 1.5, only windows wholly inside the image, variances not clamped).
 * -------------------------------------------------------------------------------------------- */
size_t ngp_image_metrics_workspace(int H, int W); /* bytes; the buffer must be ZERO-INITIALISED once by the caller (an
                                                     arrival counter the kernel re-arms); one launch at a time uses it */
/* pred: fp32 (H*W,3) in the reference's '(h w) c' pixel order; gt: the same layout, uint8 read as v/255 in fp32
 * (gt_is_u8 != 0) or fp32. Writes, on the device, *out_sse = sum of squared errors over all 3*H*W values (double; PSNR =
 * -10 log10(sse / (3*H*W)) for data_range 1) and *out_ssim = the mean SSIM over the window centres [5,H-5) x [5,W-5) and
 * the three channels (double; c1 = (0.01 data_range)^2, c2 = (0.03 data_range)^2). out_ssim may be NULL: then only the
 * squared error is computed and any H, W >= 1 will do (a flat list of n pixels is H = 1, W = n). NGP_EINVAL for a NULL
 * pred, gt, out_sse or workspace, H or W < 11 with out_ssim, data_range <= 0, or a short workspace. One kernel; the
 * result does not depend on scheduling (per-block partials summed in block order), so two calls are bitwise equal. */
int ngp_image_metrics(const float* pred, const void* gt, int gt_is_u8, int H, int W, float data_range, double* out_sse,
                      double* out_ssim, void* workspace, size_t workspace_bytes, void* stream);

/* LPIPS v0.1, VGG-16 backbone, of one view: the reference's --eval_lpips (train.py:65-68, 209-213), torchmetrics
 * LearnedPerceptualImagePatchSimilarity('vgg') of clip(2 pred - 1, -1, 1) and clip(2 gt - 1, -1, 1). The inputs are in
 * [0, 1]; the kernel applies the clip, the LPIPS scaling layer, VGG-16 features[0:30] (3x3 convs with padding 1 + ReLU,
 * 2x2 max-pools rounding down) and, at relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3, the spatial mean of
 * sum_c lin_c (f_pred / (|f_pred| + 1e-10) - f_gt / (|f_gt| + 1e-10))_c^2; *out (double, on the device) = the sum of the
 * five means. Convolutions in fp16 on tensor cores with fp32 accumulation and fp16 activations; the head in fp32 per pixel
 * and double over pixels, in a fixed order: two calls are bitwise equal, and so are LPIPS(a, b) and LPIPS(b, a).
 *
 * weights: ngp_lpips_weights_bytes() bytes, 16-B aligned, packed as
 *   for each conv l = 0..12 (features 0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28; C_out = 64 64 128 128 256 256 256
 *   512 512 512 512 512 512, C_in the previous C_out, 16 for l = 0):
 *       fp16 w_l[C_out][3][3][C_in]  (K-major: row n holds k = (ky*3 + kx)*C_in + c; torchvision's weight[n][c][ky][kx];
 *                                     l = 0 has channels 3..15 zero)
 *   for each conv l = 0..12: fp32 bias_l[C_out]
 *   for each tap t = 0..4 (C = 64 128 256 512 512): fp32 lin_t[C]  (LPIPS lin{t}.model.1.weight, non-negative)
 * pred: fp32 (H*W, 3); gt: the same layout, uint8 read as v/255 in fp32 (gt_is_u8 != 0) or fp32. All device pointers.
 * workspace (uninitialised is fine): ngp_lpips_workspace(H, W) =
 *   2 * (2*H*W*64*2)                       two ping-pong fp16 NHWC activation buffers, sized for the 64-channel
 *                                          full-resolution layers (every later layer is smaller)
 *   + 8 * sum_{t=0..4} ceil((H>>t)*(W>>t) / 64)   per-block double partials of the five heads
 * (~330 MB at 800x800), or 0 when H or W < 16 (relu5_3 would be empty) or H*W > NGP_LPIPS_MAX_PIXELS. NGP_EINVAL for
 * such a size, a NULL or non-device pointer, a misaligned weights / workspace (16 B) or out (8 B), or a short workspace.
 * 24 kernels on `stream`, no synchronisation, no allocation. */
#define NGP_LPIPS_MAX_PIXELS (1 << 26)
size_t ngp_lpips_weights_bytes(void);
size_t ngp_lpips_workspace(int H, int W);
int ngp_lpips(const void* weights, const float* pred, const void* gt, int gt_is_u8, int H, int W, double* out,
              void* workspace, size_t workspace_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Mesh extraction of a trained model. Replaces the mesh cell of the reference's test.ipynb, which evaluates
 * model.density on an N^3 np.meshgrid materialised on the host and runs mcubes.marching_cubes(sigma, 20.) on the CPU.
 * A lattice has n[a] >= 2 points on axis a; point (i, j, k) lies at x_a = lo[a] + (float)idx_a * step[a] (an fp32
 * multiply, then an fp32 add; axis 0 is x) and has linear index (i*n1 + j)*n2 + k.
 * -------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n[3];
    float lo[3];
    float step[3]; /* (hi - lo) / (n - 1) in fp32 */
} NgpLattice;

/* sigma (n0*n1*n2 fp32, linear-index order) = NGP.density at every lattice point: bitwise what ngp_net_forward(want_rgb
 * = 0) gives for the same points materialised as xyzs. The points are computed in the kernel, never stored. Points
 * outside the model's box are allowed (the encoding treats them as ngp_net_forward does). */
int ngp_density_lattice(const NgpNet* net, const NgpLattice* lat, float* sigma, void* stream);

/* Marching cubes on a volume (n0*n1*n2 fp32 in linear-index order) at level `iso`:
 *   - a lattice value is inside iff v > iso (NaN is outside); a lattice edge is crossed iff exactly one end is inside;
 *   - one vertex per crossed edge, shared by every cell using it, owned by the edge's lower end p and its axis a and
 *     ordered by (linear index of p, a); t = (iso - v0) / (v1 - v0), q = p with q_a = (float)p_a + t, vertex =
 *     lo + q * step per axis (fp32, multiply then add, no contraction);
 *   - triangles ordered by cell linear index (i*(n1-1) + j)*(n2-1) + k, then by the case table's order (tools/mc_table.py:
 *     generated from a face rule that makes the mesh watertight, at most 5 triangles a cell), counter-clockwise seen from
 *     outside: the triangle normals point out of the inside region;
 *   - normals (optional): the volume gradient (central differences, one-sided on the lattice border, divided by step)
 *     interpolated with t between the edge's ends, negated and normalised; a zero gradient gives (0, 0, 0);
 *   - no float atomics: two calls are bitwise equal.
 * The volume is processed in slabs of max(1, NGP_MC_SLAB_POINTS / (n1*n2)) cell planes, so the workspace grows with one
 * slab, not with the volume. `count` writes {n_vertices, n_triangles} to the device int64[2] `counts`; the caller reads
 * them back, allocates, and calls `emit` with the same volume, lattice, iso and workspace, nothing else touching the
 * workspace in between. `emit` checks the capacities against the totals `count` left in the workspace and returns
 * NGP_EINVAL when they are short, having written nothing: that check is a 16-byte read-back and stream synchronisation,
 * a second host synchronisation besides the caller's read-back of `counts` (cheap: that one has already drained the
 * stream), and it makes `emit` unusable under stream capture. Both return NGP_EINVAL for a NULL
 * pointer (other than normals), an n[a] < 2, n1*n2 > 2^26 or a short workspace. vertices, normals: (V, 3) fp32;
 * triangles: (F, 3) int64. */
#define NGP_MC_SLAB_POINTS (1 << 20)
size_t ngp_marching_cubes_workspace(const NgpLattice* lat); /* bytes; 0 for a lattice the functions reject */
int ngp_marching_cubes_count(const float* volume, const NgpLattice* lat, float iso, int64_t* counts, void* workspace,
                             size_t workspace_bytes, void* stream);
int ngp_marching_cubes_emit(const float* volume, const NgpLattice* lat, float iso, float* vertices, float* normals,
                            int64_t* triangles, int64_t max_vertices, int64_t max_triangles, void* workspace,
                            size_t workspace_bytes, void* stream);

/* Sparse mesh extraction: sigma and marching cubes only where the occupancy grid says the field can have a surface.
 * The lattice (n[a] in [2, NGP_MESH_MAX_N]) is cut into bricks of NGP_MESH_BRICK (B) points per axis: point (i, j, k)
 * belongs to brick (i/B, j/B, k/B), bricks on the upper border may be partial, there are nb[a] = ceil(n[a]/B) per axis
 * and brick (bi, bj, bk) has linear index (bi*nb1 + bj)*nb2 + bk. A brick mask holds bit (b & 31) of word b >> 5 for
 * brick b, ngp_mesh_bricks_bytes(lat) bytes.
 *
 * Brick mask (ngp_mesh_brick_mask; numpy restatement: oracle/mesh_bricks.py). From the brick's lower and upper corner
 * points x0, x1 (per axis: the lattice formula at b*B and at min(b*B + B - 1, n - 1)):
 *   - near = max_a (0 if the axis interval [x0, x1] holds 0, else min(|x0|, |x1|)), far = max_a max(|x0|, |x1|);
 *   - mip(v) = min(cascades - 1, max(0, e + 1)) with frexpf(v, &e): the marcher's position rule (march.cuh march_probe)
 *     without its dt term, i.e. the finest cascade whose box holds a point of max-norm v; mip(0) = min(cascades - 1, 1);
 *   - the cascades taken are c_lo = (near > 0 ? mip(near) : 0) .. c_hi = max(mip(far), near > 0 ? 0 : mip(0));
 *   - in cascade c, mb = fminf(scalbnf(1, c - 1), scale), inv = 1/mb (fp32 division), and a coordinate x has cell
 *     coordinate v = (fma(x, inv, 1) * 0.5) * G (fp32, the marcher's cell formula, monotone in x). A point with v < 0 or
 *     v > G on some axis lies outside cascade c's box: if the brick's [v(x0), v(x1)] lies wholly outside [0, G] on an
 *     axis, cascade c contributes nothing (points outside the largest cascade's box find no occupancy: no clamping to
 *     its border cells). Otherwise the cell range is [(int)clamp(v(x0), 0, G-1) - 1, (int)clamp(v(x1), 0, G-1) + 1]
 *     clipped to [0, G) -- the brick's cells widened by one on every side;
 *   - the brick is active iff a bit of density_bitfield (cell c*G^3 + morton(x, y, z)) is set in one of those ranges.
 * This is a superset of the per-point rule "a cell in the 27-neighbourhood of the point's cell, in the cascade of its
 * position, is occupied", and exact for a brick that lies in one cascade.
 *
 * sigma_masked is sigma (bitwise ngp_density_lattice) at the points of active bricks and 0 at every other point. The
 * sparse extraction returns exactly ngp_marching_cubes_count / _emit of sigma_masked at `iso`: the same vertices in the
 * same order, the same triangles and the same normals, bitwise. iso must be > 0 (the 0 fill would count as inside
 * otherwise); a surface that runs into an inactive brick is closed there. No float atomics: two calls are bitwise equal.
 *
 * Three steps, each a host call:
 *   1. ngp_mesh_sparse_bricks: a brick is *visited* when its (B+1)^3 block (the brick plus a one-point apron on the
 *      upper side, clipped to the lattice) holds a point of an active brick. Pass 1 walks the visited bricks in linear
 *      order, NGP_MESH_CHUNK_BRICKS at a time, evaluates sigma_masked on their blocks and keeps the *surface* bricks:
 *      those with a crossed cell (lower corner in the brick) or a crossed edge (lower end in the brick). Every crossed
 *      cell and edge lies in a visited brick, since an unvisited block is all 0. Writes {active, visited, surface}
 *      brick counts to the host int64[3] `counts` (two read-backs, so the call synchronises the stream).
 *   2. ngp_mesh_sparse_count: evaluates sigma_masked again on the surface bricks' (B+3)^3 blocks (one point of apron
 *      below, two above: what the normals' central differences reach) and stores them in `surface_ws`, counts the
 *      vertices and triangles of each row of each brick and scans them in the lattice's linear order (rows of B points
 *      ordered by (i, j, brick column), which is point order and cell order). Writes {n_vertices, n_triangles} to the
 *      host int64[2] `counts` (a read-back).
 *   3. ngp_mesh_sparse_emit: writes the mesh as ngp_marching_cubes_emit does, including its capacity check (a
 *      read-back; NGP_EINVAL with nothing written when max_vertices or max_triangles is short).
 * The same lattice, iso, mask, net and workspaces go to every step, nothing else touching the workspaces in between.
 * Device memory: the mask, `workspace` (fixed: two more brick bitmasks, a word prefix and one chunk of sigma blocks)
 * and `surface_ws` (grows with the surface bricks, 4 (B+3)^3 + 16 B^2 + 28 bytes each), never with the active bricks.
 * All return NGP_EINVAL for a NULL pointer (other than normals), a lattice outside the limits, iso <= 0 (or NaN) or a
 * short workspace; the workspace queries return 0 for a lattice outside the limits. */
#define NGP_MESH_BRICK 8
#define NGP_MESH_MAX_N 8192
#define NGP_MESH_CHUNK_BRICKS (1 << 16)
size_t ngp_mesh_bricks_bytes(const NgpLattice* lat);
/* The brick mask of `lat` over an occupancy bitfield (cascades * G^3 bits, G a power of two in [2, 1024], cascades in
 * [1, 62], scale > 0), one thread per brick, no atomics. */
int ngp_mesh_brick_mask(const uint8_t* density_bitfield, int cascades, int grid_size, float scale, const NgpLattice* lat,
                        uint32_t* mask, void* stream);
/* sigma_masked on the blocks of a list of bricks (linear indices, any order): brick s's block is the (W)^3 points from
 * b*B - apron on each axis, W = B + 1 + 2 * apron (apron 0 or 1), written to sigma[s*W^3 + (li*W + lj)*W + lk]; 0 at
 * points outside the lattice and at points of bricks whose bit in `mask` is clear (mask NULL: every brick active). The
 * points are those of ngp_density_lattice, through the same network kernel, so sigma is bitwise its value there. */
int ngp_density_bricks(const NgpNet* net, const NgpLattice* lat, const int32_t* bricks, int64_t n_bricks, int apron,
                       const uint32_t* mask, float* sigma, void* stream);
size_t ngp_mesh_sparse_workspace(const NgpLattice* lat);
int ngp_mesh_sparse_bricks(const NgpNet* net, const NgpLattice* lat, float iso, const uint32_t* mask, int64_t* counts,
                           void* workspace, size_t workspace_bytes, void* stream);
size_t ngp_mesh_surface_workspace(const NgpLattice* lat, int64_t n_surface);
int ngp_mesh_sparse_count(const NgpNet* net, const NgpLattice* lat, float iso, const uint32_t* mask, int64_t n_surface,
                          int64_t* counts, void* workspace, size_t workspace_bytes, void* surface_ws, size_t surface_bytes,
                          void* stream);
int ngp_mesh_sparse_emit(const NgpLattice* lat, float iso, int64_t n_surface, float* vertices, float* normals,
                         int64_t* triangles, int64_t max_vertices, int64_t max_triangles, void* surface_ws,
                         size_t surface_bytes, void* stream);

/* Mesh simplification: vertex clustering with quadric-error placement (Lindstrom, "Out-of-core simplification of large
 * polygonal models", SIGGRAPH 2000). Input: V vertices (V, 3) fp32, F triangles (F, 3) int64, optional normals (V, 3)
 * fp32 and colours (V, 3) uint8. numpy float64 restatement: oracle/mesh_simplify.py.
 *   1. Cluster grid (computed on the host in fp32 from bounds lo < hi and grid g in 1..65536): cubes of side
 *      h = max_a(hi_a - lo_a) / g, n_a = min(g, max(1, ceil((hi_a - lo_a) / h))) cells on axis a. Vertex cell
 *      c_a = clamp(floor(__fdiv_rn(__fsub_rn(v_a, lo_a), h)), 0, n_a - 1) -- vertices outside the bounds clamp to the
 *      border cells -- and cluster key (c0*n1 + c1)*n2 + c2 (int64). A cluster is the set of vertices of one key.
 *   2. Quadrics: per triangle, in double, n_t = (v1 - v0) x (v2 - v0) of the fp32 positions, area = |n_t| / 2,
 *      u = n_t / |n_t|, d = -u.v0; area * [u; d][u; d]^T is added to the cluster of each of its three corners (a cluster
 *      holding two corners gets it twice), collapsing triangles included; |n_t| = 0 contributes nothing. Evaluated in
 *      the cell-local coordinates of the receiving cluster (origin lo + c * h), which leaves A unchanged.
 *   3. Representative: x_bar = mean of the cluster's vertices, A and b of its summed quadric (error x^T A x + 2 b^T x +
 *      c); with A's eigenpairs (lambda_i, e_i), x = x_bar - sum over lambda_i > 1e-3 * lambda_max of
 *      e_i (e_i^T (A x_bar + b)) / lambda_i (x = x_bar when lambda_max = 0); clamped to the axis-aligned box of the
 *      cluster's vertices and rounded to fp32. Every vertex therefore lies within sqrt(3) * h of its representative.
 *      The eigensolve is NGP_SIMPLIFY_JACOBI_SWEEPS cyclic Jacobi sweeps in double.
 *   4. Normals: the normalised double sum of the cluster's input normals, exactly 0 when that sum is 0. Colours:
 *      floor(mean + 1/2) per channel, from exact integer sums.
 *   5. Triangles: each maps to its three cluster keys; one with two equal keys is dropped; of triangles whose key
 *      triples are the same cyclic rotation, only the first in input order is kept (opposite orientations are both
 *      kept: the result need not be manifold). Kept triangles stay in input order, with their corner order.
 *   6. Vertices: one per cluster referenced by a kept triangle, in ascending key order, numbered 0..V'-1.
 *   7. Determinism: sorted segment reductions in a fixed order (radix sorts, then lane-strided sums and a fixed shuffle
 *      tree per segment), no float atomics: two calls are bitwise equal.
 * ngp_mesh_simplify_count computes clusters, quadrics, representatives and kept triangles into the workspace and writes
 * {V', F'} to the host int64[2] `counts` (one read-back: the call synchronises the stream). Triangle indices are
 * checked on the device: an index outside [0, V) makes count return NGP_EINVAL (the kernels never read through it).
 * ngp_mesh_simplify_emit, with the same triangles, V, F and workspace and nothing else touching the workspace in
 * between, checks max_vertices / max_triangles against {V', F'} (a read-back; NGP_EINVAL with nothing written when
 * short) and writes out_vertices (V', 3) fp32, out_triangles (F', 3) int64, and out_normals (V', 3) fp32 / out_colors
 * (V', 3) uint8 where both that input and that output pointer are non-NULL.
 * ngp_mesh_simplify_workspace(V, F) is about 52 V + 52 F bytes plus cub's temporary storage (sort keys and ids of the
 * vertices and of the 3F corners), or 0 for V or F outside [0, 2^31). Both calls return NGP_EINVAL for V or F outside
 * [0, 2^31), a NULL pointer that is needed or a short workspace, and count also for a grid with n_a outside
 * 1..NGP_SIMPLIFY_MAX_GRID or h not positive and finite. V = 0 or F = 0 gives an empty mesh. */
#define NGP_SIMPLIFY_MAX_GRID 65536
#define NGP_SIMPLIFY_JACOBI_SWEEPS 8
typedef struct {
    float lo[3];
    float h;
    int32_t n[3];
} NgpClusterGrid;
size_t ngp_mesh_simplify_workspace(int64_t n_vertices, int64_t n_triangles);
int ngp_mesh_simplify_count(const float* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            const NgpClusterGrid* grid, int64_t* counts, void* workspace, size_t workspace_bytes,
                            void* stream);
int ngp_mesh_simplify_emit(const int64_t* triangles, int64_t n_vertices, int64_t n_triangles, const float* normals,
                           const uint8_t* colors, float* out_vertices, float* out_normals, uint8_t* out_colors,
                           int64_t* out_triangles, int64_t max_vertices, int64_t max_triangles, void* workspace,
                           size_t workspace_bytes, void* stream);

/* Texture baking: a per-triangle texture atlas of side W (a power of two in [16, 16384]) and its colours from the model.
 * Input: V vertices (V, 3) fp32, F triangles (F, 3) int64 (counter-clockwise seen from outside), optional normals
 * (V, 3) fp32. Margin m = 1 texel, smallest square s_min = 4. numpy float64 restatement: oracle/mesh_texture.py.
 *   1. Longest edge, in double on the fp32 positions: the edge lengths |b-a|, |c-b|, |a-c| of corners (a, b, c); the
 *      first maximum is the longest. The corners rotated so that it runs from the first to the second are A, B, C (the
 *      same cyclic order). l = |B - A|, frexp(l) = f * 2^e with f in [1/2, 1); e_top = max e over the triangles with
 *      l > 0 and finite; class k = min(e_top - e, 63), and k = 63 for l = 0 or not finite.
 *   2. Square side s = max(s_min, S >> k) (0 for k >= 31, so s_min), S the largest power of two in [s_min, W] with
 *      sum s^2 <= W^2, found on the host from a device histogram of the classes (64 bins, one read-back). F s_min^2 > W^2
 *      is refused.
 *   3. Packing: the squares ordered by s descending, ties by triangle index. Square i's Morton offset is the exclusive
 *      sum of s^2 before it; its lower-left texel (x0, y0) is that offset with x in the even bits and y in the odd bits
 *      (y from the bottom). Every earlier square is at least as large and every area a power of 4 times s^2, so each
 *      square is an aligned s x s block and no two overlap. Texel (x, y) has atlas index m = interleave(x, y), the same
 *      Morton code, so square i holds the atlas indices [offset_i, offset_i + s_i^2).
 *   4. Placement, a similarity transform, in double and rounded to fp32 once: rho = (s - 2m) / 2^e texels per world
 *      unit, u = (B - A) / l, w = (C - A).u, eta = |(C - A) - w u|; A' = (x0 + m, y0 + m), B' = A' + (rho l, 0),
 *      C' = A' + rho (w, eta) (A' = B' = C' for l = 0 or not finite). uv (F, 3, 2) lists the corners in the triangle's
 *      own order. AB is the longest edge, so 0 <= w <= l, eta < l: the triangle keeps m texels from the square's sides
 *      and stays counter-clockwise.
 *   5. Band: texel (x, y) of triangle i's square is baked when the open box (x + 1/2 +- 1, y + 1/2 +- 1) meets the
 *      closed uv triangle (every texel bilinear filtering of a point of the triangle reads): separating-axis tests in
 *      double on the fp32 uv along x, y and the normals of the triangle's non-zero edges, an axis separating when the
 *      triangle's interval [lo, hi] has hi <= box_lo or lo >= box_hi. Every other texel of the atlas is (0, 0, 0).
 *      A baked texel maps to the closest point of the uv triangle to its centre (the interior when the centre is inside
 *      a triangle of non-zero area, else the nearest of the clamped projections onto AB, BC, CA, the first on a tie), in
 *      double; its barycentrics give p = A + bB (B - A) + bC (C - A) and n = the normalised bA nA + bB nB + bC nC when
 *      the mesh has normals and that mix is non-zero, else the normalised (B - A) x (C - A), else (0, 0, -1); both are
 *      rounded to fp32. The texel map lists the baked texels in ascending atlas index.
 *   6. Bake, K samples (1..256) from offset r >= 0, all fp32: o = fmaf(n, r, p), d = -n, delta = (2r) / K,
 *      t_j = (j + 1/2) delta for j < K, t_K = r, x_j = fmaf(d, t_j, o) -- ngp_net_forward's ray mode, which evaluates
 *      (sigma_j, c_j) = NGP.forward(x_j, d). Composite in double: T_0 = 1, alpha_j = 1 - exp(-sigma_j delta),
 *      T_{j+1} = T_j (1 - alpha_j), C = sum_{j<K} T_j alpha_j c_j + T_K c_K (the surface's own colour is the background);
 *      texel = rint(255 C) clamped to [0, 255]. r = 0 gives rint(255 NGP.forward(p, d)). Image row W - 1 - y holds
 *      texel row y.
 * No float atomics: two calls are bitwise equal.
 *
 * ngp_mesh_texture_atlas: steps 1-5 up to the band count. Writes uv, squares (F, 3) int32 (x0, y0, s), and {S, number
 * of band texels} to the host int64[2] `counts` (two read-backs: the call synchronises the stream). Triangle indices are
 * checked on the device: an index outside [0, V) returns NGP_EINVAL.
 * ngp_mesh_texture_texels, with the same vertices, triangles, W and workspace and nothing else touching the workspace in
 * between: the texel map, texel (n) int64 atlas indices, triangle (n) int32, point (n, 3) and normal (n, 3) fp32, with
 * n = counts[1]; NGP_EINVAL when max_texels < n (a read-back, nothing written).
 * ngp_mesh_texture_workspace(V, F, W) is about 32 F + 4 W^2 bytes plus cub's temporary storage, or 0 for V or F outside
 * [0, 2^31) or W not a power of two in [16, 16384]. Both calls return NGP_EINVAL for those sizes, F s_min^2 > W^2, a
 * NULL pointer that is needed or a short workspace.
 * ngp_mesh_texture_bake: texture (W, W, 3) uint8 from the texel map (texel, point, normal of n texels), in chunks of
 * max(1, NGP_TEXTURE_CHUNK_SAMPLES / (K + 1)) texels, so the workspace, ngp_mesh_texture_bake_workspace(K) bytes (0 for
 * K outside 1..256), grows with one chunk. NGP_EINVAL for a bad size, r negative or not finite, a NULL pointer that is
 * needed, a short workspace, or a texel index outside [0, W^2) (checked on the device, such a texel is not written; a
 * read-back at the end, so the call synchronises the stream). */
#define NGP_TEXTURE_MIN_SIZE 16
#define NGP_TEXTURE_MAX_SIZE 16384
#define NGP_TEXTURE_MIN_SQUARE 4
#define NGP_TEXTURE_MARGIN 1
#define NGP_TEXTURE_MAX_SAMPLES 256
#define NGP_TEXTURE_CHUNK_SAMPLES (1 << 22)
size_t ngp_mesh_texture_workspace(int64_t n_vertices, int64_t n_triangles, int size);
int ngp_mesh_texture_atlas(const float* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                           int size, float* uv, int32_t* squares, int64_t* counts, void* workspace, size_t workspace_bytes,
                           void* stream);
int ngp_mesh_texture_texels(const float* vertices, const float* normals, int64_t n_vertices, const int64_t* triangles,
                            int64_t n_triangles, int size, const float* uv, int64_t max_texels, int64_t* texel,
                            int32_t* triangle, float* point, float* normal, void* workspace, size_t workspace_bytes,
                            void* stream);
size_t ngp_mesh_texture_bake_workspace(int samples);
int ngp_mesh_texture_bake(const NgpNet* net, int size, int64_t n_texels, const int64_t* texel, const float* point,
                          const float* normal, float offset, int samples, uint8_t* texture, void* workspace,
                          size_t workspace_bytes, void* stream);

/* Point-cloud export: a coloured point cloud with normals from the training views' rendered depth. numpy float64
 * restatement: oracle/points_ref.py. Stages (ngp_pl_b200/points.py runs them in this order):
 *   1. Rays, no RNG: N = n_views * n_pix global pixels, R = min(num_rays, N). Ray k takes q_k = (k g) mod N, the
 *      product exact (128-bit), with g the smallest integer >= round(0.6180339887 N) (half up, exact integers) coprime
 *      to N, found on the host; k -> q_k is then a bijection of 0..N-1, so the first R rays have no duplicate. View
 *      q div n_pix, pixel q mod n_pix; the rays are ngp_gen_rays' on that (img_idx, pix_idx) list.
 *   2. Render: ngp_render_infer_frame with bg = 0 (opacity, depth and rgb as it writes them), in batches of a fixed
 *      ray count: its per-round quota follows the batch's alive count, so the batch size is part of the result.
 *   3. Back-projection, fp32: t = __fdiv_rn(depth, opacity), p = fmaf(d, t, o) per axis, colour = rint(255 min(
 *      __fdiv_rn(rgb, opacity), 1)), view = d / sqrt((dx dx + dy dy) + dz dz) (each operation rounded). A ray is kept
 *      iff opacity >= min_opacity (in (0, 1]), p is finite and p lies in the closed box bounds[0..2] .. bounds[3..5].
 *      Kept points stay in ray order.
 *   4. Voxel downsampling on a cluster grid (rule 1 of the mesh simplification: the same cell and key): one point per
 *      occupied cell, in ascending key. Position = the double mean of the members rounded to fp32, colour =
 *      floor(mean + 1/2) from integer sums, view = the normalised double sum of the members' views (0 when it is 0).
 *   5. k nearest neighbours, k in 1..min(NGP_POINTS_MAX_K, n - 1): for every point the k smallest pairs (d^2, j) over
 *      the other points j (duplicates included), d^2 = (ex ex + ey ey) + ez ez in double of e = p_j - p_i from the fp32
 *      coordinates, ordered by d^2 and then j. Exact: a uniform grid (at most NGP_POINTS_KNN_MAX_CELLS cells) searched
 *      ring by ring until no unvisited cell can hold a closer point.
 *   6. Statistical outlier removal: d_i = the mean of sqrt(d^2) over the k neighbours; mu and sigma (population) of the
 *      d_i in double, fixed-order reductions; a point is kept iff d_i <= mu + std_ratio sigma, in order.
 *   7. Normals: the covariance sum (x - m)(x - m)^T over the point and its k neighbours about their mean m, in double;
 *      the eigenvector of the smallest eigenvalue (the first on a tie) from NGP_SIMPLIFY_JACOBI_SWEEPS cyclic Jacobi
 *      sweeps, negated when n . view > 0, rounded to fp32; (0, 0, 0) when the covariance is 0.
 * No float atomics: two calls are bitwise equal.
 *
 * ngp_points_rays: rays k0 .. k0 + n - 1 (k0 + n <= N, 1 <= g < N or g = 1 for N = 1): img_idx, pix_idx (n) int64 and
 * rays_o, rays_d (n, 3) fp32 from poses (n_views, 3, 4) and directions (n_pix, 3).
 * ngp_points_backproject: stage 3 over n rays; the kept points go to points (3 fp32), colors (3 uint8) and views
 * (3 fp32) from their first row, and their number to the host int64 *count (one read-back: the call synchronises the
 * stream). bounds is host memory.
 * ngp_points_voxel: stage 4 into outputs of capacity n; out_keys (int64 cluster keys) and out_counts (int32 members) may
 * be NULL; the number of cells to *count (a read-back).
 * ngp_points_knn: stage 5; idx (n, k) int32 and dist2 (n, k) double. One read-back (the box). NGP_EINVAL also for a
 * coordinate that is not finite.
 * ngp_points_outliers: stage 6 over dist2 (n, k) as ngp_points_knn writes it (n >= 2); the kept points to the out arrays
 * (capacity n), their input indices to kept (may be NULL), {mu, sigma, threshold} to the host double stats[3] (may be
 * NULL) and their number to *count (a read-back).
 * ngp_points_normals: stage 7 with idx (n, k) from ngp_points_knn (k may be 0: every normal is then 0); no read-back.
 * ngp_points_workspace(n) covers every call above for up to n points or rays (0 for n outside [0, 2^31)). All calls
 * return NGP_EINVAL for sizes out of range, a NULL pointer that is needed or a short workspace. */
#define NGP_POINTS_MAX_K 64
#define NGP_POINTS_KNN_MAX_CELLS (1 << 22)
size_t ngp_points_workspace(int64_t n);
int ngp_points_rays(int64_t n_views, int64_t n_pix, int64_t g, int64_t k0, int n, const float* poses,
                    const float* directions, int64_t* img_idx, int64_t* pix_idx, float* rays_o, float* rays_d, void* stream);
int ngp_points_backproject(const float* rays_o, const float* rays_d, const float* opacity, const float* depth,
                           const float* rgb, int64_t n, float min_opacity, const float* bounds, float* points,
                           uint8_t* colors, float* views, int64_t* count, void* workspace, size_t workspace_bytes,
                           void* stream);
int ngp_points_voxel(const float* points, const uint8_t* colors, const float* views, int64_t n, const NgpClusterGrid* grid,
                     float* out_points, uint8_t* out_colors, float* out_views, int64_t* out_keys, int32_t* out_counts,
                     int64_t* count, void* workspace, size_t workspace_bytes, void* stream);
int ngp_points_knn(const float* points, int64_t n, int k, int32_t* idx, double* dist2, void* workspace,
                   size_t workspace_bytes, void* stream);
int ngp_points_outliers(const float* points, const uint8_t* colors, const float* views, int64_t n, int k,
                        const double* dist2, double std_ratio, float* out_points, uint8_t* out_colors, float* out_views,
                        int32_t* kept, double* stats, int64_t* count, void* workspace, size_t workspace_bytes,
                        void* stream);
int ngp_points_normals(const float* points, const float* views, int64_t n, int k, const int32_t* idx, float* normals,
                       void* stream);

/* ----------------------------------------------------------------------------------------------
 * Depth fusion (TSDF): depth maps rendered from the training views (or any others) fused into a truncated signed
 * distance field on a lattice, and its mesh. A TSDF mesh holds only surfaces the cameras saw: no cavity no ray reaches,
 * and no sigma threshold. numpy restatement: oracle/tsdf_ref.py (np.float32, bit for bit).
 *
 * Lattice: an NgpLattice as mesh.lattice(resolution, lo, hi) builds it (the points of ngp_density_lattice). State per
 * point p (linear index): tsdf F (fp32), weight W (int32, the number of observations), color (3 fp32, a mean) and
 * color_weight Wc (int32) -- 24 B. Initial state: all 0.
 * Views: poses (n_views, 3, 4) fp32, R | o with the loaders' [right down front] axes; one pinhole K (3x3 fp32, host,
 * row-major: fx = K[0], cx = K[2], fy = K[4], cy = K[5]) and W x H pixels; directions (H W, 3) fp32, the table
 * datasets.ray_directions builds from that K (camera-frame z = 1); per view and pixel depth, opacity (fp32) and rgb
 * (3 fp32) as ngp_render_infer_frame writes them. t = depth / opacity is the ray parameter along the unnormalised
 * direction, i.e. the camera-frame z of the surface.
 *
 * One observation of point x (x_a = lo[a] + (float)idx_a step[a], multiply then add) by view v, views in pose order;
 * the view is skipped as soon as a condition fails. Every fp32 operation is rounded on its own (no contraction), sums
 * left to right:
 *   1. d = x - o; (xc, yc, zc) = R^T d, component c = (R[0][c] d0 + R[1][c] d1) + R[2][c] d2. Require zc > 0.
 *   2. px = (fx xc) / zc + cx, py = (fy yc) / zc + cy. Require 0 <= px < W and 0 <= py < H (NaN fails); pixel
 *      u = floor(px), v = floor(py): the pixel whose direction passes nearest.
 *   3. op = opacity of the pixel; require op >= min_opacity (NaN fails); t = depth / op, required finite.
 *   4. |dir| = sqrt((dx dx + dy dy) + dz dz) of the pixel's direction; sdf = (t - zc) |dir|. Require sdf >= -trunc.
 *   5. f = fminf(1, sdf / trunc); F <- (F (float)W + f) / (float)(W + 1); W <- W + 1.
 *   6. Only if sdf <= trunc: per channel c = fminf(rgb / op, 1) (the colour rule of the point-cloud export);
 *      color <- (color (float)Wc + c) / (float)(Wc + 1); Wc <- Wc + 1.
 * There are no float atomics, and the result does not depend on how the views are split into calls: two calls are
 * bitwise equal, and views integrated one call at a time give the result of one call with all of them.
 *
 * ngp_tsdf_integrate applies n_views views to the state in place, NGP_TSDF_GROUP views per launch (each launch reads
 * and writes a point's 24 B at most once: the state traffic is at most 2 * 24 * N * ceil(n_views / NGP_TSDF_GROUP)
 * bytes for N points). depth / opacity (n_views, H W), rgb (n_views, H W, 3). NGP_EINVAL for a NULL pointer that is
 * needed, n[a] < 1, trunc not positive and finite, min_opacity outside (0, 1], n_views < 0, W or H < 1 or W H >= 2^31.
 * No read-back.
 *
 * Masked marching cubes (the TSDF mesh): the rules of ngp_marching_cubes_* on v = -F at iso 0, except at unobserved
 * points (W = 0):
 *   - a point is inside iff it is observed and F < 0; an edge is crossed iff both ends are observed and exactly one
 *     is inside;
 *   - a cell emits triangles iff its 8 corners are observed;
 *   - a vertex exists iff its edge is crossed and one of the cells around the edge emits (every crossed edge of a cell
 *     is used by the case table, so no vertex is left unreferenced); vertex order is still (linear index of p, a);
 *   - normals: the dense gradient rule, a neighbour with W = 0 treated like one past the lattice border (one-sided
 *     difference, 0 when neither neighbour along the axis is observed);
 *   - colours (optional, (V, 3) uint8): the colour means of the edge's ends interpolated with the vertex's t, c0 + t
 *     (c1 - c0), when both have Wc > 0, else the inside end's mean (it has Wc >= 1); rint(255 c) clamped to 0..255.
 * So a volume observed everywhere gives exactly ngp_marching_cubes_* of -F at iso 0. The protocol, workspace and
 * refusals are those of ngp_marching_cubes_count / _emit (ngp_tsdf_mc_workspace is ngp_marching_cubes_workspace);
 * emit also refuses colors without color / color_weight. */
#define NGP_TSDF_GROUP 64
int ngp_tsdf_integrate(const NgpLattice* lat, float trunc, int n_views, const float* poses, const float* K, int W, int H,
                       const float* directions, const float* depth, const float* opacity, const float* rgb,
                       float min_opacity, float* tsdf, int32_t* weight, float* color, int32_t* color_weight, void* stream);
size_t ngp_tsdf_mc_workspace(const NgpLattice* lat);
int ngp_tsdf_mc_count(const float* tsdf, const int32_t* weight, const NgpLattice* lat, int64_t* counts, void* workspace,
                      size_t workspace_bytes, void* stream);
int ngp_tsdf_mc_emit(const float* tsdf, const int32_t* weight, const float* color, const int32_t* color_weight,
                     const NgpLattice* lat, float* vertices, float* normals, uint8_t* colors, int64_t* triangles,
                     int64_t max_vertices, int64_t max_triangles, void* workspace, size_t workspace_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Gaussian-splat export: 3D Gaussians in the layout of 3DGS's point_cloud.ply (Kerbl et al. 2023), one per point of the
 * point-cloud export (stages 1-7 above), with SH colours fitted to the model's radiance, and a forward splat rasteriser
 * with the 3DGS reference rasteriser's rules. numpy restatement: oracle/splats_ref.py (float64). Positions, normals and
 * directions are in the model's frame, as the mesh and point exports write them.
 *
 * A splat is NGP_SPLAT_FLOATS fp32, in 3DGS's construct_list_of_attributes order: x y z, nx ny nz (the point's normal;
 * 3DGS writes zeros), f_dc_0..2, f_rest_0..44, opacity, scale_0..2, rot_0..3 (w x y z). f_rest is channel-major:
 * f_rest[15 c + k - 1] is coefficient k = 1..15 of channel c. Opacity is stored as logit(alpha), scales as log(s).
 * SH basis (3DGS's sh_utils.py): C0 = 0.28209479177387814; degree 1: -C1 y, C1 z, -C1 x with C1 = 0.4886025119029199;
 * degree 2: C2_0 xy, C2_1 yz, C2_2 (2zz - xx - yy), C2_3 xz, C2_4 (xx - yy) with C2 = {1.0925484305920792,
 * -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396}; degree 3: C3_0 y (3xx - yy),
 * C3_1 xyz, C3_2 y (4zz - xx - yy), C3_3 z (2zz - 3xx - 3yy), C3_4 x (4zz - xx - yy), C3_5 z (xx - yy),
 * C3_6 x (xx - 3yy) with C3 = {-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
 * -0.4570457994644658, 1.445305721320277, -0.5900435899266435}. A splat's colour seen along the unit direction u is
 * max(0, sum_k a_k Y_k(u) + 0.5) per channel.
 *
 * Stages, per point p with normal n (0 when normals are left out):
 *   1. Colours over directions: D directions d_j (NGP_SPLAT_MIN_DIRS..NGP_SPLAT_MAX_DIRS; the host computes a Fibonacci
 *      sphere z_j = 1 - (2j + 1) / D, phi_j = j pi (3 - sqrt 5) in double and rounds it to fp32). sigma(p) and the fp16
 *      geometric feature h(p) come from ngp_net_forward (density only); then the colour MLP runs on [SH16(d_j) | h(p)]
 *      through the network core's colour chain. c(p, d_j) is bitwise the rgb ngp_net_forward returns for (p, d_j), and
 *      is stored as that fp16 value (exact).
 *   2. SH fit of degree L in 0..3, n_b = (L + 1)^2 basis functions, basis table Y (D, 16) double evaluated at the fp32
 *      d_j: w_j = max(0, -((d_jx n_x + d_jy n_y) + d_jz n_z)) in double when n != 0, else 1. In double:
 *      (sum_j w_j y_j y_j^T + ridge (sum_j w_j) I) a_c = sum_j w_j y_j (c_c(p, d_j) - 0.5) over the leading n_b x n_b
 *      block, by Cholesky, one matrix for the three channels; the sums run over j in order. Coefficients above degree L
 *      are 0, and all of them are 0 when a pivot of the (right-looking) factorisation is at most NGP_SPLAT_PIVOT_RTOL times
 *      the largest diagonal entry of the block: a rank-deficient system, e.g. ridge 0 with fewer than n_b directions in
 *      the hemisphere. Equal to the restatement within 1e-6 relative (the
 *      sums' order and the solver's differ; the ridge keeps the system conditioned).
 *   3. Geometry (no contraction, each double operation rounded as numpy's): m = the left-to-right double sum of the
 *      first min(k, 3) squared neighbour distances of ngp_points_knn over min(k, 3) (0 for k = 0), s = sqrt(max(m,
 *      1e-7)). NGP_SPLAT_SPHERE, or n = 0: scales (s, s, s), rotation (1, 0, 0, 0). NGP_SPLAT_DISC: u = n / |n|,
 *      scales (s, s, flatness s) and rotation (1 + u_z, -u_y, u_x, 0) / its norm, the shortest arc taking +z to u, or
 *      (0, 1, 0, 0) when that norm is 0 (u = -z). alpha = clamp(1 - exp(-sigma 2 s), 0.01, 0.99). The rotation is the
 *      restatement's bit for bit; log(s), log(flatness s) and logit(alpha) come from the device's double log / exp and
 *      are within one fp32 ulp of it.
 * No float atomics: two calls are bitwise equal.
 *
 * ngp_splat_colors: sigma (n) fp32, h (n, 16) fp16 scratch, rgb (n, D, 3) fp16 for points (n, 3) and dirs (D, 3) fp32.
 * ngp_splat_fit: stage 2 from rgb as ngp_splat_colors writes it and basis (D, 16) double; normals may be NULL; writes
 * f_dc and f_rest of splats (n, NGP_SPLAT_FLOATS) and nothing else. ngp_splat_geometry: stage 3 from dist2 (n, k) of
 * ngp_points_knn (k in 0..NGP_POINTS_MAX_K) and sigma; normals may be NULL; writes every other field of splats.
 * No read-back in either. NGP_EINVAL for n outside [0, 2^31), D or L out of range, a negative or non-finite ridge, a
 * flatness not positive and finite, an unknown shape or a NULL pointer that is needed.
 *
 * Rasteriser (ngp_splat_render), forward only, after the 3DGS reference rasteriser:
 *   - view (device, NGP_SPLAT_VIEW_FLOATS fp32): the c2w pose (3 x 4, R | o, OpenCV axes: x right, y down, z forward),
 *     fx, fy, cx, cy (pixel centres at i + 0.5, as the loaders' ray directions have them), bg (3).
 *   - Per splat, fp32: camera point c = R^T (p - o), culled unless c_z > 0.2. Sigma = R_q diag(s^2) R_q^T with R_q from
 *     the normalised quaternion and s = exp(scale). EWA: t_x = clamp(c_x / c_z, +-1.3 W / (2 fx)) c_z (y likewise with
 *     H, fy), J = [[fx / c_z, 0, -fx t_x / c_z^2], [0, fy / c_z, -fy t_y / c_z^2]], Sigma2D = J R^T Sigma R J^T + 0.3 I;
 *     culled unless det > 0. Radius ceil(3 sqrt(lambda_max)) with lambda = mid +- sqrt(max(0.1, mid^2 - det)). Centre
 *     (fx c_x / c_z + cx - 0.5, fy c_y / c_z + cy - 0.5) in pixel-centre coordinates. Tiles of NGP_SPLAT_TILE^2 pixels:
 *     the rectangle [(int)((x - r) / 16), (int)((x + r + 15) / 16)) per axis clamped to the grid; culled when empty.
 *     Colour at u = normalise(p - o) as above; opacity sigmoid(logit).
 *   - Keys (tile << 32 | depth bits), one per touched tile, radix-sorted (stable: ties keep splat order), then per-tile
 *     ranges. Per pixel, front to back: power = -(a dx^2 + c dy^2) / 2 - b dx dy with d = centre - pixel; skipped when
 *     power > 0; alpha = min(0.99, o exp(power)), skipped below 1/255; stop when T (1 - alpha) < 1e-4; C += c alpha T.
 *     rgb = C + T bg (H W, 3) and opacity = 1 - T (H W), fp32.
 *   - At most `capacity` keys are sorted: the call reads nothing back. The number of keys the view needs goes to the
 *     device int64 *n_keys; when it exceeds capacity the image is incomplete and the caller renders again with a
 *     larger one. So one call with fixed sizes can be captured in a CUDA graph and replayed for any view.
 * ngp_splat_render_workspace(n, W, H, capacity) is about 64 n + 24 capacity bytes plus cub's temporary storage; 0 (and
 * NGP_EINVAL from the render) for n outside [0, 2^31), W or H outside 1..NGP_SPLAT_MAX_SIDE or capacity outside
 * [1, 2^31); the workspace must be 256-B aligned. */
#define NGP_SPLAT_FLOATS 62
#define NGP_SPLAT_F_DC 6
#define NGP_SPLAT_F_REST 9
#define NGP_SPLAT_OPACITY 54
#define NGP_SPLAT_SCALE 55
#define NGP_SPLAT_ROT 58
#define NGP_SPLAT_MIN_DIRS 16
#define NGP_SPLAT_MAX_DIRS 1024
#define NGP_SPLAT_SPHERE 0
#define NGP_SPLAT_DISC 1
#define NGP_SPLAT_VIEW_FLOATS 19
#define NGP_SPLAT_TILE 16
#define NGP_SPLAT_MAX_SIDE 16384
#define NGP_SPLAT_PIVOT_RTOL 1e-10
int ngp_splat_colors(const NgpNet* net, const float* points, int64_t n_points, const float* dirs, int n_dirs, float* sigma,
                     uint16_t* h, uint16_t* rgb, void* stream);
int ngp_splat_fit(const uint16_t* rgb, int64_t n_points, int n_dirs, const float* dirs, const double* basis,
                  const float* normals, int degree, double ridge, float* splats, void* stream);
int ngp_splat_geometry(const float* points, const float* normals, const float* sigma, const double* dist2, int k,
                       int64_t n_points, int shape, float flatness, float* splats, void* stream);
size_t ngp_splat_render_workspace(int64_t n_splats, int W, int H, int64_t capacity);
int ngp_splat_render(const float* splats, int64_t n_splats, const float* view, int W, int H, int64_t capacity, float* rgb,
                     float* opacity, int64_t* n_keys, void* workspace, size_t workspace_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Connected components (numpy + scipy restatement: oracle/components_ref.py), to remove floaters from the occupancy
 * grid and small pieces from extracted meshes. One union-find core: parent is int32, one entry per node, the edges are
 * generated by kernels and never stored; a link always hooks the larger root under the smaller, so a node's label is
 * the smallest node index of its component, whatever the schedule. Sizes are exact integer counts. No float atomics:
 * two calls are bitwise equal.
 *
 * Occupancy graph (ngp_grid_components): cell i = c G^3 + morton(x, y, z) of density_bitfield; cascade c has half
 * extent mb_c = fminf(2^(c-1), scale) (fp32, the marcher's) and cell x of it spans [X_c(x), X_c(x + 1)] on an axis,
 * X_c(x) = mb_c (2x / G - 1) in double -- exact, so every comparison below is exact.
 *   - Shell and inner cells: a cell of cascade c >= 1 is *inner* when its closed box lies in cascade c - 1's closed box
 *     (X_c(x) >= -mb_{c-1} and X_c(x + 1) <= mb_{c-1} on every axis); every other cell, and every cell of cascade 0, is
 *     a *shell* cell.
 *   - Nodes: the occupied shell cells. Edges: 26-adjacency between nodes of one cascade; and a node (x, y, z) of cascade
 *     c >= 1 with a node (u, v, w) of cascade c - 1 when their closed boxes meet, i.e. per axis
 *     X_{c-1}(u) <= X_c(x + 1) and X_{c-1}(u + 1) >= X_c(x). No edges between cascades further apart.
 *   - labels (C G^3 int32): the component label of a node, -1 for every other cell (it also serves as the parent
 *     array); sizes (C G^3 int32): at a label, the number of nodes of that component, 0 elsewhere.
 * ngp_grid_components_clean, after ngp_components_select on those labels and sizes (n = C G^3), cascade by cascade
 * from c = 0: an occupied shell cell is cleared iff keep[label] is 0; an occupied inner cell of cascade c is cleared
 * iff the occupied cells of cascade c - 1 its closed box meets (by the rule of the edges) include a cleared cell and
 * no cell left occupied. A cleared cell's bit is cleared in density_bitfield (in place) and, when density_grid (C G^3
 * fp32) is not NULL, its value set to -1, the marker update_density_grid never revives. removed: C G^3 / 8 bytes of
 * scratch (no initialisation). cleared (device int64[2], may be NULL): {shell cells cleared, inner cells cleared}.
 * Both return NGP_EINVAL for a NULL pointer that is needed, G not a power of two in [2, 1024], cascades outside
 * [1, 62], cascades G^3 >= 2^31 or scale not positive and finite. Three kernels, and one per cascade; no read-back.
 *
 * Selection (ngp_components_select, any graph): a component is kept iff it is among the keep_largest largest -- ranked
 * by size descending, ties to the smaller label -- and has at least min_size nodes (keep_largest = INT64_MAX and
 * min_size = 0 leave a criterion out). keep (n bytes): 1 at a kept label, 0 everywhere else. counts (host int64[2]):
 * {components, kept components}. Roots compacted with a scan, sizes radix-sorted descending with the labels as values;
 * two read-backs, so the call synchronises the stream. NGP_EINVAL for n outside [0, 2^31), a negative criterion, a
 * NULL pointer that is needed or a short workspace; ngp_components_select_workspace(n) is about 20 n bytes plus cub's
 * temporary storage (0 for n outside the range).
 *
 * Mesh graph (ngp_mesh_components): F triangles (F, 3) int64 over V vertices are connected when they share a vertex
 * index (the marching cubes, sparse and simplified meshes share their vertices, so this is their connectivity). The
 * nodes of the union-find are the vertices, each triangle hooking its corners; labels (F int32) = the smallest triangle
 * index of the triangle's component and sizes (F int32) = at a label, the component's number of triangles, 0 elsewhere.
 * Triangle indices are checked on the device (one read-back: the call synchronises the stream); an index outside
 * [0, V) returns NGP_EINVAL. ngp_mesh_components_workspace(V, F) is about 8 V bytes.
 * Filtering, with keep from ngp_components_select on those labels and sizes (n = F): the triangles whose label is
 * kept, in input order, and the vertices they use, in input order, the indices renumbered. ngp_mesh_filter_count
 * writes {V', F'} to the host int64[2] counts (one read-back); ngp_mesh_filter_emit, with the same triangles, V, F and
 * workspace and nothing else touching the workspace in between, checks max_vertices / max_triangles against them (a
 * read-back; NGP_EINVAL with nothing written when short) and writes out_vertices (V', 3) fp32, out_triangles (F', 3)
 * int64, and out_normals (V', 3) fp32 / out_colors (V', 3) uint8 where both that input and that output are not NULL.
 * ngp_mesh_filter_workspace(V, F) is about 4 (V + F) bytes plus cub's temporary storage. All mesh calls return
 * NGP_EINVAL for V or F outside [0, 2^31), a NULL pointer that is needed or a short workspace; the workspace queries
 * return 0 there. */
int ngp_grid_components(const uint8_t* density_bitfield, int cascades, int grid_size, float scale, int32_t* labels,
                        int32_t* sizes, void* stream);
int ngp_grid_components_clean(uint8_t* density_bitfield, float* density_grid, int cascades, int grid_size, float scale,
                              const int32_t* labels, const uint8_t* keep, uint8_t* removed, int64_t* cleared,
                              void* stream);
size_t ngp_components_select_workspace(int64_t n);
int ngp_components_select(const int32_t* labels, const int32_t* sizes, int64_t n, int64_t keep_largest, int64_t min_size,
                          uint8_t* keep, int64_t* counts, void* workspace, size_t workspace_bytes, void* stream);
size_t ngp_mesh_components_workspace(int64_t n_vertices, int64_t n_triangles);
int ngp_mesh_components(const int64_t* triangles, int64_t n_vertices, int64_t n_triangles, int32_t* labels,
                        int32_t* sizes, void* workspace, size_t workspace_bytes, void* stream);
size_t ngp_mesh_filter_workspace(int64_t n_vertices, int64_t n_triangles);
int ngp_mesh_filter_count(const int64_t* triangles, int64_t n_vertices, int64_t n_triangles, const int32_t* labels,
                          const uint8_t* keep, int64_t* counts, void* workspace, size_t workspace_bytes, void* stream);
int ngp_mesh_filter_emit(const float* vertices, const float* normals, const uint8_t* colors, const int64_t* triangles,
                         int64_t n_vertices, int64_t n_triangles, float* out_vertices, float* out_normals,
                         uint8_t* out_colors, int64_t* out_triangles, int64_t max_vertices, int64_t max_triangles,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------
 * Test-view images of the validation pass (reference train.py:215-221): `{idx:03d}.png` holds (rgb_pred*255).astype(np.uint8)
 * and `{idx:03d}_d.png` depth2img(depth) (train.py:45-50; show_gui.py uses it for its depth view), and an 8-bit RGB PNG
 * encoder for both, so that only the compressed file crosses to the host.
 * -------------------------------------------------------------------------------------------- */
#define NGP_VIEW_IMAGES_WORKSPACE 4096 /* bytes, 16-B aligned; no initialisation needed */
/* rgb (H*W, 3) fp32 and depth (H*W) fp32, as render(test_time=True) returns them -> rgb_img and depth_img, uint8
 * (H, W, 3), bitwise the reference's arrays:
 *   rgb_img   = (uint8) trunc(__fmul_rn(v, 255.f)): numpy's cast for every v in [0, 256/255), the range the renderer
 *               produces; NaN -> 0 as x86 numpy gives. Other values (negative, >= 256/255, inf) are outside the contract:
 *               they saturate to 0 / 255, which numpy does not promise;
 *   depth_img = depth2img(depth): mn, mx = the exact min and max over the view (order-free: block partials), NaN
 *               propagating as numpy's min / max do; idx = trunc(__fmul_rn(__fdiv_rn(__fsub_rn(d, mn), __fsub_rn(mx, mn)),
 *               255.f)), all float32 as numpy >= 1 computes it; a NaN idx (a constant map's 0/0, or NaN anywhere in the
 *               view) is 0, as numpy on x86 gives; then the 256-entry table of cv2.applyColorMap(COLORMAP_TURBO)
 *               (csrc/turbo_table.cuh, generated by tools/turbo_table.py). The channels are cv2's B, G, R in that order:
 *               the reference hands cv2's BGR array to imageio.imsave as RGB, so its _d.png files hold blue in the red
 *               position, and so does depth_img. Depths with an infinity are outside the contract.
 * Either output may be NULL (its input is then not read), not both; workspace is needed with depth_img only.
 * NGP_EINVAL for H or W < 1, a NULL or non-device pointer that is used, or a short / misaligned workspace.
 * Two kernels with depth_img (min/max partials, then the images), one without; no synchronisation. */
int ngp_view_images(const float* rgb, const float* depth, int H, int W, uint8_t* rgb_img, uint8_t* depth_img,
                    void* workspace, size_t workspace_bytes, void* stream);

/* One complete 8-bit RGB PNG of img (H, W, 3) uint8 (device): signature, IHDR (8-bit, colour type 2, no interlace), one
 * IDAT, IEND. The file goes to out and its length, an int64, to *out_len -- both written by the device; out and out_len
 * may be device memory or mapped pinned host memory (cudaHostAlloc; with unified addressing its host pointer is its
 * device pointer), so only the file's bytes cross PCIe. Nothing in the call synchronises the stream.
 *
 * The byte stream is fixed by this algorithm (oracle/png_ref.py restates it byte for byte):
 *   - Filters, one per row, libpng's heuristic: the type f in None, Sub, Up, Average, Paeth (0..4; bpp 3, the row above
 *     row 0 is zeros) minimising sum |filtered byte read as int8| over the row's 3W bytes; a tie goes to the lowest f.
 *     Row r of the filtered stream is the segment [f, filtered bytes], L = 3W + 1 bytes, at stream position r*L.
 *   - Deflate, one segment per row. A greedy LZ77 parse from the segment's first byte over the candidate distances
 *     1, 3, L and 2L, a candidate dropped when it exceeds 32768 or reaches before the stream start. At position p the
 *     match length for d is the number of bytes s[p+i] == s[p-d+i], at most 258 and never past the segment's end; the
 *     longest wins, a tie to the smaller distance; a length >= 3 is emitted as (length, distance) and the parse skips
 *     it, otherwise the byte is a literal. The segment is coded as one fixed-Huffman block (BFINAL 0, BTYPE 01, then the
 *     tokens and end-of-block), or as stored blocks of at most 65535 bytes each (BFINAL 0, BTYPE 00) when those are no
 *     longer. Either way an empty stored block follows (3 header bits, padding to the byte, LEN 0000, NLEN ffff), so the
 *     next segment starts on a byte boundary; the last segment's empty block carries BFINAL = 1.
 *   - Assembly: zlib header 78 01, the segments in row order (offsets from a scan of their byte lengths), the Adler-32
 *     combined from per-segment (sum d_i, sum (L - i) d_i) pairs in row order. The IDAT CRC-32 is combined from
 *     per-segment CRCs with crc32_combine (a multiplication by x^(8 len) mod P from a table of x^(2^k)).
 *   - All arithmetic is integer and fixed-order: two calls give the same bytes.
 * Sizes: ngp_png_capacity(H, W) = 63 + H * S with S = L + 5 * ceil(L / 65535) + 5 (every segment stored: the largest
 * file the encoder can write); ngp_png_workspace(H, W) = 256-B-aligned regions for the filtered stream (H*L), the match
 * table (2 H L), the segments (H * round_up(S, 16)), per-row records (16 H) and offsets (8 H); both are 0 for H or W < 1
 * or an IDAT that could exceed 2^31 - 1 bytes (6 + H * S). NGP_EINVAL for such a size, a NULL or non-device pointer, a
 * workspace short or not 256-B aligned, out_len not 8-B aligned, or out_capacity < ngp_png_capacity(H, W).
 * Four kernels (filter, deflate, assembly, compaction). */
size_t ngp_png_workspace(int H, int W);
size_t ngp_png_capacity(int H, int W);
int ngp_png_encode(const uint8_t* img, int H, int W, uint8_t* out, size_t out_capacity, int64_t* out_len,
                   void* workspace, size_t workspace_bytes, void* stream);

/* The same file in a chosen deflate mode: NGP_PNG_FIXED is ngp_png_encode's stream byte for byte (and its workspace);
 * NGP_PNG_DYNAMIC is a smaller stream of the same image, fixed by this algorithm (oracle/png_dynamic_ref.py restates it
 * byte for byte):
 *   - Filters and their Adler-32 parts: as ngp_png_encode. L = 3W + 1.
 *   - Match search, each row on its own: the candidate distances are the distinct values of 1, 2, 3, 4, 6, 9, 12, L-3,
 *     L, L+3 and 2L that lie in 1..32768, a candidate dropped at a position p < d. The match length for d at p is the
 *     number of bytes s[p+i] == s[p-d+i], at most 258 and never past the row's end; the longest wins, a tie to the
 *     smaller distance; best(p) is that length when it is >= 3, else 0 (best = 0 past the row's end).
 *   - Lazy parse by one step from the row's first byte: at p, when best(p) >= 3 and best(p+1) <= best(p), the match
 *     (best(p), its distance) is emitted and the parse skips it; otherwise the byte is a literal and the parse moves on
 *     by one. Tokens are coded with RFC 1951's length and distance codes and extra bits.
 *   - Groups: rows 32g .. 32g + 31 (the last group shorter) form one block, their tokens concatenated bit by bit, then
 *     end-of-block. Histograms: the group's literal/length symbols plus one end-of-block, and its distance codes.
 *   - Dynamic code: lengths by package-merge, limit 15 for both alphabets; items sorted by (count, symbol) ascending,
 *     an item before a package of equal weight; the first 2n - 2 entries of the last list give the lengths. A single
 *     used symbol gets length 1; with no distance code used, distance code 0 gets length 1. Canonical codes (RFC 1951
 *     3.2.2). HLIT = max(257, last used literal/length + 1), HDIST = max(1, last nonzero distance length + 1). The two
 *     length lists are run-length coded separately by zlib's send_tree rules (16: 3-6 repeats of the previous length,
 *     17: 3-10 zeros, 18: 11-138 zeros); the code-length code by package-merge with limit 7 over those symbols,
 *     HCLEN = the RFC's permutation order trimmed of trailing zero lengths, at least 4.
 *   - Each group is coded as one dynamic block (BTYPE 10), one fixed block (BTYPE 01) or stored blocks of at most 65535
 *     bytes of the group's filtered bytes (BTYPE 00), whichever is shortest in bytes with the empty stored block that
 *     follows it (3 header bits, padding, LEN 0000, NLEN ffff), a tie in that order; BFINAL is 0 on each, and 1 on the
 *     last group's empty block. Every group therefore starts on a byte boundary.
 *   - Assembly as ngp_png_encode with the groups in place of the rows: offsets from a scan of the groups' lengths, the
 *     IDAT CRC-32 combined from per-group CRCs; the Adler-32 still from per-row parts.
 *   - All arithmetic is integer and fixed-order: two calls give the same bytes.
 * ngp_png_capacity bounds both modes (a group stored whole is never longer than its rows stored one by one).
 * ngp_png_workspace_mode(H, W, NGP_PNG_DYNAMIC) covers the filtered stream, the match table (2 H L), token-start masks,
 * per-row histograms (1264 H), row offsets, the group tables and buffers; it is 0 where ngp_png_workspace is, and for
 * an unknown mode. ngp_png_encode_mode returns NGP_EINVAL for an unknown mode and for everything ngp_png_encode
 * refuses. Dynamic mode: seven kernels (filter, match and parse, tables, emission, group CRCs, assembly, compaction);
 * no synchronisation. */
#define NGP_PNG_FIXED 0
#define NGP_PNG_DYNAMIC 1
size_t ngp_png_workspace_mode(int H, int W, int mode);
int ngp_png_encode_mode(const uint8_t* img, int H, int W, int mode, uint8_t* out, size_t out_capacity, int64_t* out_len,
                        void* workspace, size_t workspace_bytes, void* stream);

/* One complete baseline JPEG of img (H, W, 3) uint8 RGB (device), for the Motion-JPEG videos of the test views. As with
 * ngp_png_encode the file goes to out and its length, an int64, to *out_len, both written by the device; out and out_len
 * may be device memory or mapped pinned host memory; nothing in the call synchronises the stream.
 *
 * One fixed format; quality (1..100) is the only choice. The byte stream (oracle/jpeg_ref.py restates it byte for byte,
 * and it is the file libjpeg writes for the same quality with 4:4:4 sampling, its default tables and its accurate
 * integer DCT, e.g. Pillow's save(quality=q, subsampling=0, optimize=False)):
 *   - Segments: SOI; APP0 JFIF 1.01, density unit 0, 1 x 1, no thumbnail; DQT table 0; DQT table 1 (8-bit entries in
 *     zig-zag order); SOF0 (baseline sequential DCT, 8-bit, H, W, components 1, 2, 3 = Y, Cb, Cr, each sampled 1 x 1,
 *     quantisation tables 0, 1, 1); DHT DC 0, AC 0, DC 1, AC 1: the "typical" tables of ITU-T T.81 Annex K.3; SOS (one
 *     interleaved scan, Huffman tables 0, 1, 1, coefficients 0..63); the entropy-coded data; EOI. No restart intervals.
 *     The segments before the data are 623 bytes.
 *   - Quantisation tables: the Annex K.1 luminance and chrominance tables scaled as libjpeg does, s = 5000 / quality
 *     below 50 and 200 - 2 quality from 50, entry = (base * s + 50) / 100 in integers, clamped to 1..255.
 *   - Colour: Y = (19595 R + 38470 G + 7471 B + 32768) >> 16, Cb = (-11059 R - 21709 G + 32768 B + 8421375) >> 16,
 *     Cr = (32768 R - 27439 G - 5329 B + 8421375) >> 16 (8421375 = (128 << 16) + 32767). The image is cut into 8 x 8
 *     blocks, the last column and row repeated up to a multiple of 8; 128 is subtracted from every sample.
 *   - Forward DCT: the Loeffler-Ligtenberg-Moschytz factorisation in 32-bit integers with 13-bit constants, rows then
 *     columns, the row pass scaled up by 4 and every product sum rounded by adding half before the arithmetic shift;
 *     the block comes out scaled by 8. Quantisation: sign(c) * ((|c| + 4 q) / (8 q)), i.e. rounding half away from zero.
 *   - Entropy coding: an MCU is the Y, Cb, Cr blocks of one 8 x 8 area, MCUs in raster order. Per block: the difference
 *     of the DC coefficient to the same component's DC of the previous MCU (0 before the first) as its size category's
 *     code and that many magnitude bits (a negative value v as the low bits of v - 1); the AC coefficients in zig-zag
 *     order as run/size codes with magnitude bits, a run over 15 as ZRL codes, and EOB unless coefficient 63 is not
 *     zero. Bits are packed most significant first, the last byte is filled with 1-bits, and every 0xFF byte of the
 *     data is followed by a 0x00.
 *   - All arithmetic is integer and order-free (codes are OR-ed into a zeroed stream): two calls give the same bytes.
 * Sizes, with B = 3 * ceil(H / 8) * ceil(W / 8) blocks: a block codes to at most 20 + 63 * 26 = 1658 bits, taken as 208
 * bytes, and stuffing at most doubles them, so ngp_jpeg_capacity(H, W) = 623 + 416 B + 2. ngp_jpeg_workspace(H, W) =
 * 256-B-aligned regions for the coefficients (128 B), per-MCU bit counts (4 B / 3), the unstuffed stream (208 B + 8
 * rounded up to 512) and per-512-byte 0xFF counts, plus 256 bytes. Both are 0 for H or W outside 1..65535 (the SOF0
 * fields) or 1664 B > 2^31 - 1 (bit offsets are 32-bit: about 27 million pixels). NGP_EINVAL for such a size, a quality
 * outside 1..100, a NULL or non-device pointer, a workspace short or not 256-B aligned, out_len not 8-B aligned, or
 * out_capacity < ngp_jpeg_capacity(H, W). One memset of the stream and seven kernels (DCT, bit counts, scan, code
 * emission, 0xFF counts, scan, stuffing and assembly). */
size_t ngp_jpeg_workspace(int H, int W);
size_t ngp_jpeg_capacity(int H, int W);
int ngp_jpeg_encode(const uint8_t* img, int H, int W, int quality, uint8_t* out, size_t out_capacity, int64_t* out_len,
                    void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NGP_B200_H */
