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
#define NGP_ABI_VERSION 3

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

/* vren.distortion_loss_fw / _bw (binding.cpp:197-231, losses.cu:10-174). */
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

/* The two halves of ngp_net_backward, individually callable (profiling; overlapping them with other work). */
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
 *                          ngp_net_forward(want_rgb=0, h_out, feat_save); workspace as ngp_net_backward */
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
 * g = grads * grad_mul (1/world_size after a sum all-reduce). Also refreshes the fp16 working copy and
 * zeroes the gradient for the next step in the same pass. lr and step live on the device
 * (lr_dev[0], step_dev[0] = number of completed steps; the kernel uses t = step+1 and a follow-up
 * single-thread kernel increments it) so a captured CUDA graph never needs re-capturing. */
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
 * bitfield) sits between two training steps. A cell picked more than once is evaluated once, at its first pick's point
 * (the reference's index_put keeps an arbitrary one of the duplicates). Both halves must see the same workspace, cascades, grid_size, threshold and
 * warmup, and nothing else may touch the workspace in between. */
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

#ifdef __cplusplus
}
#endif
#endif /* NGP_B200_H */
