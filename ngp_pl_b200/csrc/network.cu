// Fused NGP network kernels for sm_90a: hash-grid gather + trilinear interpolation + density MLP +
// exp + SH-4 + rgb MLP + sigmoid in ONE forward kernel, and ONE backward kernel that recomputes the
// activations, runs dgrad/wgrad on the tensor cores and scatters hash-table gradients with 8-byte
// vector reductions. Replaces the three tinycudann modules of reference models/networks.py:36-77 and
// the glue of NGP.density / NGP.forward (networks.py:94-107, :132-153).
#include "common.cuh"
#include "network.cuh"
#include "wgmma.cuh"
#include "../../include/ngp_b200.h"
#include <math.h>

extern "C" int ngp_abi_version(void) { return NGP_ABI_VERSION; }

unsigned long long g_ngp_launch_count = 0;
extern "C" unsigned long long ngp_launch_count(void) { return __atomic_load_n(&g_ngp_launch_count, __ATOMIC_RELAXED); }

// ---- step timeline (debugging aid, see common.cuh) -------------------------------------------------------------------
unsigned long long* g_ngp_trace = nullptr;
__global__ void k_trace_stamp(unsigned long long* buf, int id) { trace_mark(buf, id); }
void ngp_trace_stamp(int id, cudaStream_t st) { k_trace_stamp<<<1, 1, 0, st>>>(g_ngp_trace, id); }
// buf: device array of 2 + 2 * capacity u64, buf[0] = 0 (cursor) and buf[1] = capacity set by the caller; nullptr = off
extern "C" int ngp_trace_set(void* buf) {
    g_ngp_trace = (unsigned long long*)buf;
    return 0;
}

// -------------------------------------------------------------------------------------------------
// host: level table (tiny-cuda-nn GridEncoding constructor semantics, SURVEY.md Appendix A)
// -------------------------------------------------------------------------------------------------
extern "C" uint32_t ngp_grid_meta(int n_levels, int log2_hashmap_size, int base_resolution, float per_level_scale,
                                  NgpGridMeta* out) {
    if (!out || n_levels < 1 || n_levels > NGP_MAX_LEVELS || log2_hashmap_size < 3 || log2_hashmap_size > 28 ||
        base_resolution < 1 || !(per_level_scale >= 1.0f))
        return 0;
    const float log2_b = log2f(per_level_scale);
    uint64_t offset = 0;
    out->n_levels = n_levels;
    out->hashed_mask = 0;
    for (int l = 0; l < NGP_MAX_LEVELS; ++l) {
        out->offset[l] = 0; out->res[l] = 0; out->scale[l] = 0.f;
    }
    for (int l = 0; l < n_levels; ++l) {
        const float scale = exp2f((float)l * log2_b) * (float)base_resolution - 1.0f;
        const uint32_t res = (uint32_t)ceilf(scale) + 1u;
        const uint64_t dense = (uint64_t)res * res * res;
        uint64_t entries = (dense + 7u) / 8u * 8u;
        const uint64_t cap = 1ull << log2_hashmap_size;
        if (entries > cap) entries = cap;
        if (dense > entries) out->hashed_mask |= (1u << l);
        out->offset[l] = (uint32_t)offset;
        out->res[l] = res;
        out->scale[l] = scale;
        offset += entries;
        if (offset > 0xffffffffull) return 0;
    }
    for (int l = n_levels; l <= NGP_MAX_LEVELS; ++l) out->offset[l] = (uint32_t)offset;
    return (uint32_t)offset;
}

// -------------------------------------------------------------------------------------------------
// fp32 master params -> fp16 working copy
// -------------------------------------------------------------------------------------------------
__global__ void k_cast_params(const float* __restrict__ src, __half* __restrict__ dst, int64_t n) {
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n && ((((uintptr_t)src) & 15) == 0) && ((((uintptr_t)dst) & 7) == 0)) {
        const float4 v = *reinterpret_cast<const float4*>(src + i);
        uint2 o;
        o.x = pack_half2(v.x, v.y);
        o.y = pack_half2(v.z, v.w);
        *reinterpret_cast<uint2*>(dst + i) = o;
    } else {
        for (int64_t k = i; k < n && k < i + 4; ++k) dst[k] = __float2half_rn(src[k]);
    }
}
extern "C" int ngp_cast_params(const float* src, uint16_t* dst_half, int64_t n, void* stream) {
    if (n < 0) return NGP_EINVAL;
    if (n == 0) return 0;
    k_cast_params<<<ngp_div_up((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(src, (__half*)dst_half, n);
    NGP_CHECK_LAUNCH();
    return 0;
}

// -------------------------------------------------------------------------------------------------
// Dynamic tile scheduling for the persistent kernels: warps (forward) / CTAs (backward) take the next tile from a
// device counter instead of striding, so a CTA that becomes resident late -- the trainer runs the next step's
// march on a second stream under these kernels -- simply takes fewer tiles instead of stretching the kernel by a
// whole extra wave. A slot is {next tile, finished CTAs}; the last CTA to finish re-arms it. Slots rotate per
// launch, so launches that may overlap on different streams never share one.
// -------------------------------------------------------------------------------------------------
#define NGP_SCHED_EAGER 1024  // rotated by eager launches (a collision needs two launches 1024 apart to overlap in time)
#define NGP_SCHED_GRAPH 1024  // handed out once each to launches recorded into CUDA graphs (their slot is baked in)
__device__ int g_sched[NGP_SCHED_EAGER + NGP_SCHED_GRAPH][2];
// nullptr => the kernel falls back to static striding (no current device / not queryable)
static int* sched_slot(cudaStream_t st) {
    static int* bases[64] = {nullptr};  // per device: a __device__ symbol has one address per device
    static unsigned eager_seq[64] = {0}, graph_seq[64] = {0};  // per device too (slots live in per-device memory)
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    int* base = __atomic_load_n(&bases[dev], __ATOMIC_ACQUIRE);
    if (!base) {
        void* p = nullptr;
        if (cudaGetSymbolAddress(&p, g_sched) != cudaSuccess) return nullptr;
        base = (int*)p;
        __atomic_store_n(&bases[dev], base, __ATOMIC_RELEASE);  // every thread computes the same address
    }
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) return nullptr;
    if (cs != cudaStreamCaptureStatusNone) {
        // a captured launch keeps its slot for the life of the graph; when the pool is used up the slots are handed out
        // again round-robin (two graphs then share one only if 1,024 captures lie between them AND they overlap in time)
        const unsigned k = __atomic_fetch_add(&graph_seq[dev], 1u, __ATOMIC_RELAXED);
        return base + 2 * (size_t)(NGP_SCHED_EAGER + k % NGP_SCHED_GRAPH);
    }
    return base + 2 * (size_t)(__atomic_fetch_add(&eager_seq[dev], 1u, __ATOMIC_RELAXED) % NGP_SCHED_EAGER);
}
__device__ __forceinline__ void sched_finish(int* sched) {
    if (!sched) return;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&sched[1], 1) == (int)gridDim.x - 1) {  // every CTA is past its last grab
            sched[0] = 0;
            sched[1] = 0;
            __threadfence();
        }
    }
}

// -------------------------------------------------------------------------------------------------
// sample access
// -------------------------------------------------------------------------------------------------
struct SampleIn {
    float x, y, z;     // world position
    float dx, dy, dz;  // (unnormalised) view direction
};
// number of live samples: from the device counter when one is given (clamped to the capacity)
__device__ __forceinline__ int64_t sample_count(const NgpSamples& s) {
    if (s.n_dev) {
        const int64_t v = (int64_t)__ldg(s.n_dev);
        return v < s.n ? (v < 0 ? 0 : v) : s.n;
    }
    return s.n;
}

// Backward-only compaction: when live_idx is given, the backward kernels visit samples live_idx[0 .. *n_live_dev)
// only (the ones whose upstream gradient can be non-zero) and index their per-sample outputs by that position.
__device__ __forceinline__ int64_t bwd_count(const NgpSamples& s) {
    if (s.live_idx) {
        const int64_t v = (int64_t)__ldg(s.n_live_dev);
        return v < s.n ? (v < 0 ? 0 : v) : s.n;
    }
    return sample_count(s);
}

// the sample at t on ray r, with the rounding of the marcher's sample position (march.cuh: x = fma(d, t, o))
__device__ __forceinline__ SampleIn ray_sample(const NgpSamples& s, int r, float t) {
    SampleIn o;
    o.dx = __ldg(s.rays_d + 3 * r); o.dy = __ldg(s.rays_d + 3 * r + 1); o.dz = __ldg(s.rays_d + 3 * r + 2);
    o.x = __fmaf_rn(o.dx, t, __ldg(s.rays_o + 3 * r));
    o.y = __fmaf_rn(o.dy, t, __ldg(s.rays_o + 3 * r + 1));
    o.z = __fmaf_rn(o.dz, t, __ldg(s.rays_o + 3 * r + 2));
    return o;
}

__device__ __forceinline__ SampleIn load_sample(const NgpSamples& s, int64_t i, bool& valid) {
    SampleIn o;
    if (!valid) {
        o.x = o.y = o.z = 0.f;
        o.dx = 0.f; o.dy = 0.f; o.dz = 1.f;
        return o;
    }
    if (s.ray_idx) {
        const int r = __ldg(s.ray_idx + i);
        if (r < 0) {  // an unused slot of a rectangular (ray, slot) layout (ngp_render_infer's warp-per-ray rounds)
            valid = false;
            o.x = o.y = o.z = 0.f;
            o.dx = 0.f; o.dy = 0.f; o.dz = 1.f;
            return o;
        }
        o = ray_sample(s, r, __ldg(s.ts + i));
    } else {
        o.x = __ldg(s.xyzs + 3 * i); o.y = __ldg(s.xyzs + 3 * i + 1); o.z = __ldg(s.xyzs + 3 * i + 2);
        if (s.dirs) {
            o.dx = __ldg(s.dirs + 3 * i); o.dy = __ldg(s.dirs + 3 * i + 1); o.dz = __ldg(s.dirs + 3 * i + 2);
        } else {
            o.dx = 0.f; o.dy = 0.f; o.dz = 1.f;
        }
    }
    return o;
}

// a point of a lattice, generated from its row-major index: x = lo + (float)i * step, an fp32 multiply then an fp32 add,
// so the points are bitwise those a caller materialises with the same formula
__device__ __forceinline__ int64_t sample_count(const NgpLattice& lat) { return (int64_t)lat.n[0] * lat.n[1] * lat.n[2]; }
__device__ __forceinline__ void lattice_point(const NgpLattice& lat, int64_t i, int64_t j, int64_t k, SampleIn& s) {
    s.x = __fadd_rn(lat.lo[0], __fmul_rn((float)i, lat.step[0]));
    s.y = __fadd_rn(lat.lo[1], __fmul_rn((float)j, lat.step[1]));
    s.z = __fadd_rn(lat.lo[2], __fmul_rn((float)k, lat.step[2]));
}
__device__ __forceinline__ SampleIn load_sample(const NgpLattice& lat, int64_t row, bool& valid) {
    SampleIn s;
    s.x = s.y = s.z = 0.f;
    s.dx = 0.f; s.dy = 0.f; s.dz = 1.f;
    if (valid) {
        const int64_t n1 = lat.n[1], n2 = lat.n[2];
        const int64_t k = row % n2, ij = row / n2;
        const int64_t j = ij % n1, i = ij / n1;
        lattice_point(lat, i, j, k, s);
    }
    return s;
}

// the points of a list of lattice bricks (sparse mesh extraction, csrc/mesh.cu): brick s's block is W^3 points from
// b*B - apron per axis, row s*W^3 + (li*W + lj)*W + lk. Points outside the lattice or in a brick whose mask bit is clear
// are not evaluated (the caller has zeroed sigma); the others are lattice points, bitwise.
struct BrickRows {
    NgpLattice lat;
    const int32_t* bricks;
    const uint32_t* mask;  // NULL: every brick active
    int64_t n_bricks;
    int32_t nb1, nb2, apron, width;
};
__device__ __forceinline__ int64_t sample_count(const BrickRows& b) {
    return b.n_bricks * (int64_t)(b.width * b.width * b.width);
}
__device__ __forceinline__ SampleIn load_sample(const BrickRows& b, int64_t row, bool& valid) {
    SampleIn s;
    s.x = s.y = s.z = 0.f;
    s.dx = 0.f; s.dy = 0.f; s.dz = 1.f;
    if (!valid) return s;
    const int w = b.width, w3 = w * w * w;
    const int brick = __ldg(b.bricks + row / w3), l = (int)(row % w3);
    const int bk = brick % b.nb2, bij = brick / b.nb2, bj = bij % b.nb1, bi = bij / b.nb1;
    const int64_t i = (int64_t)bi * NGP_MESH_BRICK - b.apron + l / (w * w);
    const int64_t j = (int64_t)bj * NGP_MESH_BRICK - b.apron + (l / w) % w;
    const int64_t k = (int64_t)bk * NGP_MESH_BRICK - b.apron + l % w;
    if (i < 0 || j < 0 || k < 0 || i >= b.lat.n[0] || j >= b.lat.n[1] || k >= b.lat.n[2]) {
        valid = false;
        return s;
    }
    if (b.mask) {
        const int64_t pb = ((i / NGP_MESH_BRICK) * b.nb1 + j / NGP_MESH_BRICK) * b.nb2 + k / NGP_MESH_BRICK;
        if (!((__ldg(b.mask + (pb >> 5)) >> (pb & 31)) & 1u)) {
            valid = false;
            return s;
        }
    }
    lattice_point(b.lat, i, j, k, s);
    return s;
}

// x01 = (x - xyz_min) / (xyz_max - xyz_min)   (reference networks.py:103)
__device__ __forceinline__ void to_unit(const NgpNet& net, const SampleIn& s, float& u, float& v, float& w) {
    u = __fdiv_rn(s.x - net.xyz_min[0], net.xyz_max[0] - net.xyz_min[0]);
    v = __fdiv_rn(s.y - net.xyz_min[1], net.xyz_max[1] - net.xyz_min[1]);
    w = __fdiv_rn(s.z - net.xyz_min[2], net.xyz_max[2] - net.xyz_min[2]);
}

// Encode the rows this lane owns into the A fragments of the first density layer.
// Lane (g,q) owns rows {g, g+8} of each 16-row tile and levels {q, q+4, q+8, q+12}.
template <int MT>
__device__ __forceinline__ void encode_rows(const NgpNet& net, const uint32_t* __restrict__ table,
                                            const float (&u)[MT][2][3], const bool (&valid)[MT][2],
                                            uint32_t (&featA)[MT][2][4], int q) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int level = 4 * j + q;
                float2 f = make_float2(0.f, 0.f);
                if (valid[mt][h] && level < net.meta.n_levels)
                    f = grid_lookup(table, net.meta, level, u[mt][h][0], u[mt][h][1], u[mt][h][2]);
                featA[mt][j >> 1][2 * (j & 1) + h] = pack_half2(f.x, f.y);
            }
}

// -------------------------------------------------------------------------------------------------
// forward. Rows: the samples of an NgpSamples, or the points of an NgpLattice generated from the row index (mesh
// extraction, ngp_pl_b200/mesh.py: density only, 4 B a point written).
// -------------------------------------------------------------------------------------------------
#define FWD_MT 1            // 16-row tiles a warp takes at a time
#define FWD_THREADS 256
#define FWD_MIN_BLOCKS 3    // CTAs per SM: 24 warps
template <typename Rows>
__global__ void __launch_bounds__(FWD_THREADS, FWD_MIN_BLOCKS)
k_ngp_fwd(const NgpNet net, const Rows smp, const int want_rgb, float* __restrict__ sigmas, float* __restrict__ rgbs,
          __half* __restrict__ h_out, uint4* __restrict__ feat_save, int* __restrict__ sched) {
    __shared__ __align__(16) MlpWeightsFwd sw;
    // (eager callers may write the weights or the samples with the kernel right before this one: wait first)
    pdl_wait();
    pdl_trigger();
    const __half* wd = reinterpret_cast<const __half*>(net.enc_params_h);
    const __half* wr = want_rgb ? reinterpret_cast<const __half*>(net.rgb_params_h) : nullptr;
    load_weights_fwd(sw, wd, wr, threadIdx.x, FWD_THREADS);
    __syncthreads();
    const uint32_t* table = reinterpret_cast<const uint32_t*>(wd + NGP_DENSITY_MLP_PARAMS);

    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int64_t n = sample_count(smp);
    const int64_t n_tiles = (n + 16 * FWD_MT - 1) / (16 * FWD_MT);
    const int n_warps = (int)gridDim.x * (FWD_THREADS / 32);
    int grabbed = (int)blockIdx.x * (FWD_THREADS / 32) + (threadIdx.x >> 5);  // static striding when there is no slot
    if (sched && lane == 0) grabbed = atomicAdd(&sched[0], 1);
    for (;;) {
        const int64_t tile = __shfl_sync(0xffffffffu, grabbed, 0);
        if (tile >= n_tiles) break;
        if (!sched) grabbed += n_warps;
        else if (lane == 0) grabbed = atomicAdd(&sched[0], 1);  // the next ticket travels while this tile is computed
        const int64_t base = tile * 16 * FWD_MT;
        SampleIn sm[FWD_MT][2];
        bool valid[FWD_MT][2];
        float u[FWD_MT][2][3];
#pragma unroll
        for (int mt = 0; mt < FWD_MT; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = base + 16 * mt + g + 8 * h;
                valid[mt][h] = row < n;
                sm[mt][h] = load_sample(smp, row, valid[mt][h]);
                to_unit(net, sm[mt][h], u[mt][h][0], u[mt][h][1], u[mt][h][2]);
            }

        uint32_t featA[FWD_MT][2][4];
        encode_rows<FWD_MT>(net, table, u, valid, featA, q);

        if (feat_save) {
#pragma unroll
            for (int mt = 0; mt < FWD_MT; ++mt)
#pragma unroll
                for (int kt = 0; kt < 2; ++kt)
                    feat_save[((tile * FWD_MT + mt) * 2 + kt) * 32 + lane] =
                        make_uint4(featA[mt][kt][0], featA[mt][kt][1], featA[mt][kt][2], featA[mt][kt][3]);
        }

        uint32_t hA[FWD_MT][1][4];
        density_mlp<FWD_MT>(featA, sw.w1d, sw.w2d, hA, g, q, [](const auto&) {});
#pragma unroll
        for (int mt = 0; mt < FWD_MT; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = base + 16 * mt + g + 8 * h;
                if (valid[mt][h]) {
                    if (q == 0) sigmas[row] = sigma_of_h(hA[mt][0][h]);
                    if (h_out) {
                        uint32_t* ho = reinterpret_cast<uint32_t*>(h_out + row * 16);
                        ho[q] = hA[mt][0][h];
                        ho[4 + q] = hA[mt][0][2 + h];
                    }
                }
            }
        if (!want_rgb) continue;

        uint32_t inA[FWD_MT][2][4];
        color_input<FWD_MT>(sm, hA, q, inA);
        float oC[FWD_MT][1][4];
        color_mlp<FWD_MT>(inA, sw.w1r, sw.w2r, sw.w3r, oC, g, q, [](int, const auto&) {});
#pragma unroll
        for (int mt = 0; mt < FWD_MT; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = base + 16 * mt + g + 8 * h;
                if (!valid[mt][h] || q > 1) continue;
                const float2 o = __half22float2(rgb_out(oC[mt][0][2 * h], oC[mt][0][2 * h + 1], net.rgb_act));
                if (q == 0) {
                    rgbs[3 * row] = o.x;
                    rgbs[3 * row + 1] = o.y;
                } else {
                    rgbs[3 * row + 2] = o.x;
                }
            }
    }
    sched_finish(sched);
}

static int fwd_grid(int64_t n) {
    const int64_t n_tiles = (n + 16 * FWD_MT - 1) / (16 * FWD_MT);
    const int64_t want = (n_tiles + FWD_THREADS / 32 - 1) / (FWD_THREADS / 32);
    const int64_t cap = (int64_t)ngp_sm_count() * FWD_MIN_BLOCKS;
    return (int)(want < cap ? want : cap);
}

extern "C" int ngp_net_forward(const NgpNet* net, const NgpSamples* smp, int want_rgb, float* sigmas, float* rgbs,
                               uint16_t* h_out, void* feat_save, void* stream) {
    if (!net || !smp || smp->n < 0 || !sigmas || (want_rgb && !rgbs)) return NGP_EINVAL;
    if (net->meta.n_levels < 1 || net->meta.n_levels > NGP_MAX_LEVELS) return NGP_EINVAL;
    if (smp->n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(ngp_launch_pdl(k_ngp_fwd<NgpSamples>, fwd_grid(smp->n), FWD_THREADS, 0, st, *net, *smp, want_rgb, sigmas, rgbs,
                            (__half*)h_out, (uint4*)feat_save, sched_slot(st)));
    NGP_CHECK_LAUNCH();
    NGP_TRACE(3, st);
    return 0;
}

// density on a lattice: static striding (no scheduler slot), sigma only
extern "C" int ngp_density_lattice(const NgpNet* net, const NgpLattice* lat, float* sigma, void* stream) {
    if (!net || !lat || !sigma || !net->enc_params_h) return NGP_EINVAL;
    if (net->meta.n_levels < 1 || net->meta.n_levels > NGP_MAX_LEVELS) return NGP_EINVAL;
    for (int a = 0; a < 3; ++a)
        if (lat->n[a] < 2) return NGP_EINVAL;
    const int64_t n = (int64_t)lat->n[0] * lat->n[1] * lat->n[2];
    k_ngp_fwd<NgpLattice><<<fwd_grid(n), FWD_THREADS, 0, (cudaStream_t)stream>>>(*net, *lat, 0, sigma, nullptr, nullptr, nullptr,
                                                                                  nullptr);
    NGP_CHECK_LAUNCH();
    return 0;
}

// sigma_masked on the blocks of a brick list (include/ngp_b200.h): zero the blocks, then evaluate the points that count
extern "C" int ngp_density_bricks(const NgpNet* net, const NgpLattice* lat, const int32_t* bricks, int64_t n_bricks, int apron,
                                  const uint32_t* mask, float* sigma, void* stream) {
    if (!net || !lat || !bricks || !sigma || !net->enc_params_h || n_bricks < 0 || (apron != 0 && apron != 1)) return NGP_EINVAL;
    if (net->meta.n_levels < 1 || net->meta.n_levels > NGP_MAX_LEVELS) return NGP_EINVAL;
    for (int a = 0; a < 3; ++a)
        if (lat->n[a] < 2 || lat->n[a] > NGP_MESH_MAX_N) return NGP_EINVAL;
    if (n_bricks == 0) return 0;
    BrickRows b;
    b.lat = *lat;
    b.bricks = bricks;
    b.mask = mask;
    b.n_bricks = n_bricks;
    b.nb1 = (lat->n[1] + NGP_MESH_BRICK - 1) / NGP_MESH_BRICK;
    b.nb2 = (lat->n[2] + NGP_MESH_BRICK - 1) / NGP_MESH_BRICK;
    b.apron = apron;
    b.width = NGP_MESH_BRICK + 1 + 2 * apron;
    const int64_t n = n_bricks * (int64_t)(b.width * b.width * b.width);
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(cudaMemsetAsync(sigma, 0, n * sizeof(float), st));
    k_ngp_fwd<BrickRows><<<fwd_grid(n), FWD_THREADS, 0, st>>>(*net, b, 0, sigma, nullptr, nullptr, nullptr, nullptr);
    NGP_CHECK_LAUNCH();
    return 0;
}

// -------------------------------------------------------------------------------------------------
// backward: the dgrad chain stays on mma.sync fragments in twelve ROW warps, but the five WEIGHT-GRADIENT GEMMs
// (dW = dOut^T * In over the 192 staged rows of a block: K = 192, M = 64, N <= 64) are issued by a dedicated MMA WARPGROUP
// (warps 12-15) as wgmma.mma_async with both operands read from shared memory through matrix descriptors and the fp32
// accumulators in that warpgroup's registers (64 x 160, 80 a thread, alive for the CTA's whole lifetime). The activations
// are staged in the canonical MN-major no-swizzle layout (wgmma.cuh); the out-gradient of a layer goes to one of two
// buffers, so the tensor core can still be reading layer L's while the warps stage layer L+1's.
// Synchronisation is by mbarriers, not CTA barriers: a row thread that has staged its rows of a layer ARRIVES on that
// layer's `staged` barrier and carries on with its dgrad; the MMA warpgroup WAITS on it, issues the 12 wgmma of the layer's
// GEMM, waits for them and arrives on the `done` barrier of the buffer they read, which row threads wait on only before they
// overwrite that buffer two layers later. One CTA barrier per 192-row block is left (ticket broadcast + reuse of the
// activation tiles). Twelve row warps: a 512-thread block keeps the 128 registers a thread the row path needs without
// spilling (sixteen would leave 96).
// The encoded features come from the forward's feat_save or, with REGATHER (no feat_save), from the hash table again
// through the forward's own encode_rows, so both give the same fp16 values.
// -------------------------------------------------------------------------------------------------
#define B3_WARPS 12
#define B3_ROW_THREADS (B3_WARPS * 32)
#define B3_THREADS (B3_ROW_THREADS + 128)
#define B3_ROWS (B3_WARPS * 16)
struct Bwd3Smem {
    MlpWeightsFwd wf;
    __align__(128) __half feat[B3_ROWS * 32];
    __align__(128) __half hid[B3_ROWS * 64];
    __align__(128) __half rin[B3_ROWS * 32];
    __align__(128) __half r1[B3_ROWS * 64];
    __align__(128) __half r2[B3_ROWS * 64];
    __align__(128) __half dbuf[2][B3_ROWS * 64];  // out-gradient of the layer being processed, alternating
    __align__(8) uint64_t done[2];                // completion of the MMAs that read dbuf[b] (one arrival per MMA warp)
    uint64_t staged[5];                           // all rows of layer L are staged (one arrival per row warp and block)
    int blk[2];
};

// A fragments of this warp's 16 rows <-> canonical tile of C channels (32-bit accesses; a warp touches 128 contiguous bytes)
template <int KT>
__device__ __forceinline__ void stage_canon(__half* __restrict__ dst, int C, int row0, const uint32_t (&A)[KT][4], int g, int q) {
    __half* b0 = dst + (row0 >> 3) * (C * 8) + g * 8 + 2 * q;
    __half* b1 = b0 + C * 8;
#pragma unroll
    for (int kt = 0; kt < KT; ++kt) {
        *reinterpret_cast<uint32_t*>(b0 + (2 * kt) * 64) = A[kt][0];
        *reinterpret_cast<uint32_t*>(b1 + (2 * kt) * 64) = A[kt][1];
        *reinterpret_cast<uint32_t*>(b0 + (2 * kt + 1) * 64) = A[kt][2];
        *reinterpret_cast<uint32_t*>(b1 + (2 * kt + 1) * 64) = A[kt][3];
    }
}
template <int KT>
__device__ __forceinline__ void load_canon(const __half* __restrict__ src, int C, int row0, uint32_t (&A)[1][KT][4], int g, int q) {
    const __half* b0 = src + (row0 >> 3) * (C * 8) + g * 8 + 2 * q;
    const __half* b1 = b0 + C * 8;
#pragma unroll
    for (int kt = 0; kt < KT; ++kt) {
        A[0][kt][0] = *reinterpret_cast<const uint32_t*>(b0 + (2 * kt) * 64);
        A[0][kt][1] = *reinterpret_cast<const uint32_t*>(b1 + (2 * kt) * 64);
        A[0][kt][2] = *reinterpret_cast<const uint32_t*>(b0 + (2 * kt + 1) * 64);
        A[0][kt][3] = *reinterpret_cast<const uint32_t*>(b1 + (2 * kt + 1) * 64);
    }
}
// D[64][N] += A^T B over the B3_ROWS staged rows: A = tile of 64 channels (M), B = tile of N channels; the whole MMA
// warpgroup executes it and returns when the MMAs have completed (their operands may then be overwritten)
template <int N>
__device__ __forceinline__ void wgmma_wgrad(float (&d)[N / 2], const __half* A, const __half* B) {
    const uint32_t lbo_a = 64u * 16u, lbo_b = (uint32_t)N * 16u;  // bytes between 8-row blocks: C/8 * 128
    uint64_t ad = wgmma_smem_desc(A, lbo_a, 128), bd = wgmma_smem_desc(B, lbo_b, 128);
    const uint64_t a_step = (uint64_t)((2u * lbo_a) >> 4), b_step = (uint64_t)((2u * lbo_b) >> 4);  // 16 rows, in 16-byte units
    wgmma_fence_operand(d);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < B3_ROWS / 16; ++ks) {
        wgmma_f16<N>(d, ad, bd);
        ad += a_step;  // the start-address field is the low 14 bits; the tiles end below 256 KB, so no carry leaves it
        bd += b_step;
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(d);
}
// this thread's fragment of a D[64][N] accumulator (rows m0, m0 + 8; columns 8 j + 2 q, + 1) * inv_scale -> dW by fp32
// reductions: dW[m][n] (row-major, ld) or, TRANSPOSED, dW[n][m]
template <int N, bool TRANSPOSED>
__device__ __forceinline__ void wgmma_acc_flush(const float (&d)[N / 2], float* dW, int ld, int m0, int q, float inv_scale) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + 8 * h, c = 8 * j + 2 * q;
            const float v0 = d[4 * j + 2 * h] * inv_scale, v1 = d[4 * j + 2 * h + 1] * inv_scale;
            if (TRANSPOSED) {
                asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dW + c * ld + m), "f"(v0) : "memory");
                asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dW + (c + 1) * ld + m), "f"(v1) : "memory");
            } else {
                red_add_f32x2(dW + m * ld + c, v0, v1);
            }
        }
}

template <bool REGATHER>
__global__ void __launch_bounds__(B3_THREADS, 1)
k_ngp_bwd3(const NgpNet net, const NgpSamples smp, const float* __restrict__ dL_dsigmas, const float* __restrict__ dL_drgbs,
           const uint4* __restrict__ feat_save, const float* __restrict__ loss_scale, float* __restrict__ grad_enc,
           float* __restrict__ grad_rgb, uint32_t* __restrict__ dfeat, const int64_t dfeat_stride, int* __restrict__ sched) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Bwd3Smem& S = *reinterpret_cast<Bwd3Smem*>(smem_raw);
    const __half* wd = reinterpret_cast<const __half*>(net.enc_params_h);
    const __half* wr = reinterpret_cast<const __half*>(net.rgb_params_h);
    // Before waiting on the kernel that publishes the live count and the loss scale: stage the weights (the fp16 working
    // copy, written by the previous step's optimiser), initialise the barriers and take the first ticket (the scheduler
    // slot is this launch's own).
    load_weights_fwd(S.wf, wd, wr, threadIdx.x, B3_THREADS);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const bool mma_wg = warp >= B3_WARPS;
    const int32_t* __restrict__ live = smp.live_idx;
    const int row0 = 16 * warp;

    if (threadIdx.x == 0) {
        mbar_init(&S.done[0], 4);
        mbar_init(&S.done[1], 4);
#pragma unroll
        for (int l = 0; l < 5; ++l) mbar_init(&S.staged[l], B3_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        S.blk[0] = sched ? atomicAdd(&sched[0], 1) : (int)blockIdx.x;
    }
    pdl_wait();
    pdl_trigger();
    const int64_t n = bwd_count(smp);
    const int64_t n_mtiles = (n + 15) / 16;
    const int64_t n_blks = (n_mtiles + B3_WARPS - 1) / B3_WARPS;
    const float scale = loss_scale ? *loss_scale : 1.0f;
    const float inv_scale = 1.0f / scale;
    __syncthreads();
    uint32_t commits[2] = {0u, 0u};  // MMA batches signalled on done[b] so far (every thread counts the same)

    if (mma_wg) {
        // ================= MMA warpgroup: one GEMM per layer, as soon as the layer's rows are staged =================
        // accumulators: W3r^T [in 64][out 16], W2r [64][64], W1r [64][32], W2d^T [in 64][out 16], W1d [64][32]
        float a3r[8], a2r[32], a1r[16], a2d[8], a1d[16];
#pragma unroll
        for (int i = 0; i < 8; ++i) a3r[i] = a2d[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) a1r[i] = a1d[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) a2r[i] = 0.f;
        auto signal = [&](int b) {  // the GEMM that read dbuf[b] has completed
            __syncwarp();
            if (lane == 0) mbar_arrive(&S.done[b]);
        };
        int n_done = 0;  // blocks processed by this CTA
        for (int it = 0;; ++it) {
            const int64_t blk = S.blk[it & 1];
            if (blk >= n_blks) break;
            ++n_done;
            __syncthreads();  // (the block's CTA barrier: see the row warps)
            const uint32_t par = (uint32_t)it & 1u;
            mbar_wait(&S.staged[0], par);
            wgmma_wgrad<16>(a3r, S.r2, S.dbuf[0]);   signal(0);
            mbar_wait(&S.staged[1], par);
            wgmma_wgrad<64>(a2r, S.dbuf[1], S.r1);   signal(1);
            mbar_wait(&S.staged[2], par);
            wgmma_wgrad<32>(a1r, S.dbuf[0], S.rin);  signal(0);
            mbar_wait(&S.staged[3], par);
            wgmma_wgrad<16>(a2d, S.hid, S.dbuf[1]);  signal(1);
            mbar_wait(&S.staged[4], par);
            wgmma_wgrad<32>(a1d, S.dbuf[0], S.feat); signal(0);
        }
        sched_finish(sched);
        // ---- flush the weight gradients: registers -> fp32 reductions ----
        if (n_done > 0) {
            const int m0 = 16 * (warp - B3_WARPS) + g;
            wgmma_acc_flush<16, true>(a3r, grad_rgb + 2048 + 4096, 64, m0, q, inv_scale);  // W3r (16 x 64), accumulated transposed
            wgmma_acc_flush<64, false>(a2r, grad_rgb + 2048, 64, m0, q, inv_scale);        // W2r (64 x 64)
            wgmma_acc_flush<32, false>(a1r, grad_rgb, 32, m0, q, inv_scale);               // W1r (64 x 32)
            wgmma_acc_flush<16, true>(a2d, grad_enc + 2048, 64, m0, q, inv_scale);         // W2d (16 x 64), transposed
            wgmma_acc_flush<32, false>(a1d, grad_enc, 32, m0, q, inv_scale);               // W1d (64 x 32)
        }
        return;
    }

    // ---- software-pipelined row fetch (row warps): state of the NEXT block's two rows of this lane ----
    bool pre_valid[2] = {false, false};
    int64_t pre_src[2] = {0, 0};
    int pre_ridx[2] = {-1, -1};
    float pre_t[2] = {0.f, 0.f};
    float pre_up[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    uint32_t pre_feat[2][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
    auto fetch_hop1 = [&](int64_t nblk) {  // which sample does each of my rows stand for
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = (nblk * B3_WARPS + warp) * 16 + g + 8 * h;
            pre_valid[h] = nblk < n_blks && row < n;
            pre_src[h] = pre_valid[h] ? (live ? (int64_t)__ldg(live + row) : row) : 0;
        }
    };
    auto fetch_hop2 = [&](int64_t nblk) {  // everything that is indexed by the sample
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t sidx = pre_src[h];
            pre_ridx[h] = -1;
            pre_up[h][0] = pre_up[h][1] = pre_up[h][2] = 0.f;
            if (pre_valid[h]) {
                if (smp.ray_idx) {
                    pre_ridx[h] = __ldg(smp.ray_idx + sidx);
                    pre_t[h] = __ldg(smp.ts + sidx);
                }
                if (q == 0) {
                    pre_up[h][0] = __ldg(dL_dsigmas + sidx);
                    pre_up[h][1] = __ldg(dL_drgbs + 3 * sidx);
                    pre_up[h][2] = __ldg(dL_drgbs + 3 * sidx + 1);
                } else if (q == 1) {
                    pre_up[h][1] = __ldg(dL_drgbs + 3 * sidx + 2);
                }
            }
            if constexpr (!REGATHER) {
                // this lane's four words of the row out of the forward's fragment-order save (word x/z = row g, y/w = row
                // g+8 of the 16-row tile that holds the sample)
                const uint32_t* fs = reinterpret_cast<const uint32_t*>(feat_save);
                const int64_t t2 = (sidx >> 4) * 2;
                const int r = (int)(sidx & 15);
                const int64_t w0 = (r & 7) * 4 + q;
                const int sub = r >> 3;
#pragma unroll
                for (int kt = 0; kt < 2; ++kt) {
                    const uint32_t* p = fs + ((t2 + kt) * 32 + w0) * 4 + sub;
                    pre_feat[kt][h] = pre_valid[h] ? __ldg(p) : 0u;
                    pre_feat[kt][2 + h] = pre_valid[h] ? __ldg(p + 2) : 0u;
                }
            }
        }
        (void)nblk;
    };
    fetch_hop1(S.blk[0]);
    fetch_hop2(S.blk[0]);

    // wait until the most recent MMA batch that read dbuf[b] (and everything issued before it) has completed
    auto wait_buf = [&](int b) {
        if (commits[b]) mbar_wait(&S.done[b], (commits[b] - 1u) & 1u);
    };

    for (int it = 0;; ++it) {
        const int64_t blk = S.blk[it & 1];
        if (blk >= n_blks) break;
        if (threadIdx.x == 0) S.blk[(it + 1) & 1] = sched ? atomicAdd(&sched[0], 1) : (int)(blk + gridDim.x);

        // ================= row warps =================
        // The rows of THIS block were fetched while the previous block was processed (hop 1: live index, right after that
        // block's barrier; hop 2: ray index, t, upstream gradients, saved features, half-way through it), so only the last
        // hop -- the ray's origin and direction, L1/L2 hits shared by the rays' consecutive samples -- is on the critical
        // path here. (Three dependent global loads at the top of every block were 15 % of the stall samples.)
        const int64_t mtile = blk * B3_WARPS + warp;
        const int64_t base = mtile * 16;
        bool valid[2];
        float up_sig[2], up_c0[2], up_c1[2];
        SampleIn sm[1][2];
        uint32_t featA[1][2][4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            valid[h] = pre_valid[h];
            up_sig[h] = pre_up[h][0]; up_c0[h] = pre_up[h][1]; up_c1[h] = pre_up[h][2];
#pragma unroll
            for (int kt = 0; kt < 2; ++kt) {
                featA[0][kt][h] = pre_feat[kt][h];
                featA[0][kt][2 + h] = pre_feat[kt][2 + h];
            }
            if (valid[h] && pre_ridx[h] >= 0) {
                sm[0][h] = ray_sample(smp, pre_ridx[h], pre_t[h]);
            } else {
                bool v = valid[h];
                sm[0][h] = load_sample(smp, pre_src[h], v);  // (xyzs / dirs layout, or an invalid row)
                valid[h] = v;
            }
        }
        if constexpr (REGATHER) {
            const uint32_t* table = reinterpret_cast<const uint32_t*>(wd + NGP_DENSITY_MLP_PARAMS);
            const bool v[1][2] = {{valid[0], valid[1]}};
            float u[1][2][3];
#pragma unroll
            for (int h = 0; h < 2; ++h) to_unit(net, sm[0][h], u[0][h][0], u[0][h][1], u[0][h][2]);
            encode_rows<1>(net, table, u, v, featA, q);
        }
        // the previous block's GEMMs still read feat / hid / rin / r1 / r2: its last batch (W1d, buffer 0) completes after
        // every earlier one (the MMAs of one thread complete in order). The CTA barrier also publishes the next ticket and
        // keeps a fast thread from arriving on a `staged` barrier whose previous phase is still open.
        wait_buf(0);
        __syncthreads();
        const int64_t nblk = S.blk[(it + 1) & 1];  // published by the barrier
        fetch_hop1(nblk);

        // ---- forward recompute, staging each activation as soon as it exists ----
        stage_canon<2>(S.feat, 32, row0, featA[0], g, q);
        float h0[2];
        uint32_t hA[1][1][4];
        density_mlp<1>(featA, S.wf.w1d, S.wf.w2d, hA, g, q,
                       [&](const auto& hid) { stage_canon<4>(S.hid, 64, row0, hid[0], g, q); });
        h0[0] = lo_half(hA[0][0][0]);
        h0[1] = lo_half(hA[0][0][1]);
        uint32_t doutA[1][1][4];
        {
            uint32_t inA[1][2][4];
            color_input<1>(sm, hA, q, inA);
            stage_canon<2>(S.rin, 32, row0, inA[0], g, q);
            float oC[1][1][4];
            color_mlp<1>(inA, S.wf.w1r, S.wf.w2r, S.wf.w3r, oC, g, q,
                         [&](int l, const auto& r) { stage_canon<4>(l == 1 ? S.r1 : S.r2, 64, row0, r[0], g, q); });
            doutA[0][0][2] = 0u;
            doutA[0][0][3] = 0u;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float d0 = 0.f, d1 = 0.f;
                if (valid[h] && q < 2) {
                    float s0 = oC[0][0][2 * h], s1 = oC[0][0][2 * h + 1];
                    rgb_out_grad(s0, s1, net.rgb_act);
                    d0 = up_c0[h] * s0 * scale;
                    d1 = (q == 0) ? up_c1[h] * s1 * scale : 0.f;
                }
                doutA[0][0][h] = pack_half2(d0, d1);
            }
        }

        // ---- layer rgb-3 : dW3r^T[in 64][out 16] = r2^T dout ; buffer 0 (free: waited above) ----
        stage_canon<1>(S.dbuf[0], 16, row0, doutA[0], g, q);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.staged[0]);
        commits[0] += 1u;
        uint32_t dA[1][4][4];  // out-gradient fragments of the 64-wide layers, reused
        {
            float c[1][8][4];
            mlp_layer_dgrad<16, 64, LD64>(doutA, S.wf.w3r, c, lane);
            uint32_t act[1][4][4];
            load_canon<4>(S.r2, 64, row0, act, g, q);
            relu_bwd_to_frag<1, 64>(c, act, dA);
        }
        // ---- layer rgb-2 : dW2r[out 64][in 64] = dr2^T r1 ; buffer 1 ----
        wait_buf(1);
        stage_canon<4>(S.dbuf[1], 64, row0, dA[0], g, q);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.staged[1]);
        commits[1] += 1u;
        {
            float c[1][8][4];
            mlp_layer_dgrad<64, 64, LD64>(dA, S.wf.w2r, c, lane);
            uint32_t act[1][4][4];
            load_canon<4>(S.r1, 64, row0, act, g, q);
            relu_bwd_to_frag<1, 64>(c, act, dA);
        }
        fetch_hop2(nblk);  // the next block's live indices have long arrived
        // ---- layer rgb-1 : dW1r[out 64][in 32] = dr1^T rin ; buffer 0 ; only the h half of its input needs a gradient ----
        wait_buf(0);
        stage_canon<4>(S.dbuf[0], 64, row0, dA[0], g, q);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.staged[2]);
        commits[0] += 1u;
        uint32_t dhA[1][1][4];
        {
            float c[1][2][4];
            mlp_layer_dgrad<64, 16, LD32>(dA, S.wf.w1r + 16, c, lane);
            if (q == 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (valid[h]) c[0][0][2 * h] += up_sig[h] * expf(fminf(fmaxf(h0[h], -15.f), 15.f)) * scale;
            }
            to_frag<1, 16>(c, dhA);
        }
        // ---- layer density-2 : dW2d^T[in 64][out 16] = hid^T dh ; buffer 1 ----
        wait_buf(1);
        stage_canon<1>(S.dbuf[1], 16, row0, dhA[0], g, q);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.staged[3]);
        commits[1] += 1u;
        {
            float c[1][8][4];
            mlp_layer_dgrad<16, 64, LD64>(dhA, S.wf.w2d, c, lane);
            uint32_t act[1][4][4];
            load_canon<4>(S.hid, 64, row0, act, g, q);
            relu_bwd_to_frag<1, 64>(c, act, dA);
        }
        // ---- layer density-1 : dW1d[out 64][in 32] = dhid^T feat ; buffer 0 -> feature gradients ----
        wait_buf(0);
        stage_canon<4>(S.dbuf[0], 64, row0, dA[0], g, q);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.staged[4]);
        commits[0] += 1u;
        {
            float c[1][4][4];
            mlp_layer_dgrad<64, 32, LD32>(dA, S.wf.w1d, c, lane);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = base + g + 8 * h;
                if (!valid[h]) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int level = 4 * j + q;
                    if (level < net.meta.n_levels)
                        dfeat[(int64_t)level * dfeat_stride + row] = pack_half2(c[0][j][2 * h], c[0][j][2 * h + 1]);
                }
            }
        }
    }

    sched_finish(sched);  // (the MMA warpgroup flushes the weight gradients)
}

// -------------------------------------------------------------------------------------------------
// hash-table gradient scatter: one thread per (sample, level), a warp = 32 CONSECUTIVE samples of one
// level. Consecutive samples of a ray fall into the same cell at the coarse levels, so equal cells are
// contiguous lane runs: their 16 corner contributions are summed with a segmented shuffle reduction and
// only the head of each run issues the 8 vector reductions (fewer, and far less contended, L2 atomics).
// At the finer levels a run's next cell is mostly the neighbour across a face, an edge or a vertex, whose shared corners
// are the same grid vertices and so the same table entries: a head hands those sums to the next head through shared
// memory instead of issuing them (tests/test_scatter_merge_algorithm_cpu.py replays the rule lane by lane).
//
// Level-major order: a work item is a chunk of SCATTER_THREADS consecutive samples x a group of SCATTER_GROUP
// levels, and the tickets of the device counter hand out every chunk of one group before the next group. So
// the reductions in flight hit one group's slice of the fp32 gradient (4 MB per hashed level at T = 2^19)
// instead of the whole table (45.8 MB, about the size of the L2): a line stays in L2 across its reductions
// instead of making a round trip to HBM for each. Group g holds levels g, g + G, g + 2G, ... (G groups), so
// the small dense levels share their group with hashed ones rather than taking every SM's reductions alone.
// An item reloads its chunk's positions; a larger group spends fewer reloads on a larger working set.
// -------------------------------------------------------------------------------------------------
#define SCATTER_THREADS 256
#define SCATTER_MIN_BLOCKS 5  // CTAs per SM: 40 warps (48 registers)
#define SCATTER_GROUP 2       // levels per work item: 1 and 4 were slower (DESIGN.md section 9)
__global__ void __launch_bounds__(SCATTER_THREADS, SCATTER_MIN_BLOCKS)
k_grid_scatter_merged(const NgpNet net, const NgpSamples smp, const uint32_t* __restrict__ dfeat, const int64_t dfeat_stride,
                      const float* __restrict__ loss_scale, float* __restrict__ grad_table, int* __restrict__ sched) {
    __shared__ int s_item[2];
    // corners handed from a run head to the next (float2 per corner, indexed by the receiving lane; 9 slots per lane
    // spread the lanes over the banks)
    __shared__ float2 s_hand[SCATTER_THREADS / 32][32][9];
    const int lane = threadIdx.x & 31;
    const int64_t n = bwd_count(smp);
    const int n_levels = net.meta.n_levels;
    const int n_groups = (n_levels + SCATTER_GROUP - 1) / SCATTER_GROUP;
    const int64_t n_chunks = (n + SCATTER_THREADS - 1) / SCATTER_THREADS;
    const int64_t n_items = n_chunks * n_groups;

    // an item's positions are computed once and reused for the levels of its group (dfeat is indexed by s, the position
    // by the sample it stands for)
    bool valid;
    float u, v, w;
    int64_t s;
    int group;
    auto take = [&](int64_t item) {
        group = (int)(item / n_chunks);
        s = (item - group * n_chunks) * SCATTER_THREADS + threadIdx.x;
        valid = s < n;
        const SampleIn sm = load_sample(smp, (valid && smp.live_idx) ? (int64_t)__ldg(smp.live_idx + s) : s, valid);
        to_unit(net, sm, u, v, w);
    };
    // the first item's positions (the count, the live list and the positions were written two or more kernels earlier)
    // are loaded before waiting on the MLP backward, whose feature gradients are the first thing read after it
    if (threadIdx.x == 0) s_item[0] = sched ? atomicAdd(&sched[0], 1) : (int)blockIdx.x;
    __syncthreads();
    int64_t item = s_item[0];
    if (item < n_items) take(item);
    pdl_wait();
    pdl_trigger();
    const float inv_scale = loss_scale ? 1.0f / *loss_scale : 1.0f;
    for (int it = 0; item < n_items; ++it) {
        // the next ticket travels while this item is scattered
        if (threadIdx.x == 0) s_item[(it + 1) & 1] = sched ? atomicAdd(&sched[0], 1) : (int)(item + gridDim.x);
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        // the per-level feature gradient is the one load on the critical path of a level: fetch the NEXT level's while
        // this level's shuffles and reductions run
        uint32_t d_next = valid ? __ldg(dfeat + (int64_t)group * dfeat_stride + s) : 0u;
        for (int level = group; level < n_levels; level += n_groups) {
            const uint32_t d_cur = d_next;
            if (valid && level + n_groups < n_levels) d_next = __ldg(dfeat + (int64_t)(level + n_groups) * dfeat_stride + s);
            const uint32_t res = net.meta.res[level];
            const uint32_t off = net.meta.offset[level];
            const uint32_t entries = net.meta.offset[level + 1] - off;
            const bool hashed = (net.meta.hashed_mask >> level) & 1u;
            const GridCell c = grid_cell(u, v, w, net.meta.scale[level]);
            float2 gr = make_float2(0.f, 0.f);
            if (valid) {
                gr = unpack_half2(d_cur);
                gr.x *= inv_scale;
                gr.y *= inv_scale;
            }
            float acc[16];
            {
                float wk[8];
                grid_corner_weights(c, wk);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    acc[2 * k] = wk[k] * gr.x;
                    acc[2 * k + 1] = wk[k] * gr.y;
                }
            }
            // runs of equal cells (an invalid lane never joins a run)
            const uint32_t px = __shfl_up_sync(0xffffffffu, c.gx, 1), py = __shfl_up_sync(0xffffffffu, c.gy, 1),
                           pz = __shfl_up_sync(0xffffffffu, c.gz, 1);
            const bool pvalid = lane > 0 && ((vmask >> (lane - 1)) & 1u);
            const bool head = lane == 0 || !valid || !pvalid || px != c.gx || py != c.gy || pz != c.gz;
            const unsigned heads = __ballot_sync(0xffffffffu, head);
            const unsigned later = lane == 31 ? 0u : (heads >> (lane + 1));
            const int run_end = later ? lane + __ffs(later) - 1 : 31;
            // A valid head whose previous lane is valid starts a run right after another run, whose cell is px, py, pz.
            // If the two cells are adjacent, its link holds the corners they share (bits 0-7, in this cell's numbering)
            // and 8 + o, where corner k of the previous cell is corner k + o here (bits 8-11). 0: no link.
            uint32_t link = 0u;
            if (valid && pvalid && head) {
                const int ox = (int)(px - c.gx), oy = (int)(py - c.gy), oz = (int)(pz - c.gz);
                if (grid_cells_adjacent(ox, oy, oz))
                    link = grid_shared_corners(ox, oy, oz) | (uint32_t)(ox + 2 * oy + 4 * oz + 8) << 8;
            }
            if (heads != 0xffffffffu) {
                // longest run in the warp bounds the depth of the segmented reduction (warp-uniform)
                unsigned cont = ~heads;  // bit i set: lane i continues the run of lane i-1
                int max_run = 1;
                while (cont) {
                    cont &= cont >> 1;
                    ++max_run;
                }
                for (int d = 1; d < max_run; d <<= 1) {
                    const bool take = lane + d <= run_end;
#pragma unroll
                    for (int k = 0; k < 16; ++k) {
                        const float o = __shfl_down_sync(0xffffffffu, acc[k], d);
                        if (take) acc[k] += o;
                    }
                }
            }
            // Corners shared with the next run's cell, in one pass. A head hands the corners it shares with the next head's
            // cell to that head, except those it shares with the previous head's cell too: it may receive those, so it
            // issues them itself. A corner handed over is one the receiver issues (never one it hands on), so every
            // contribution reaches memory once, after at most one hop.
            const uint32_t nlink = __shfl_sync(0xffffffffu, link, (run_end + 1) & 31);  // lane 0 has no link
            uint32_t fwd = 0u, fwd_out = 0u;  // corners handed over, in this cell's and in the next cell's numbering
            if (valid && head && nlink) {
                const int o = (int)(nlink >> 8) - 8;  // corner k here is corner k + o of the next cell
                const uint32_t mine = link & 0xFFu;
                fwd_out = nlink & 0xFFu & ~(o >= 0 ? mine << o : mine >> -o);
                fwd = o >= 0 ? fwd_out >> o : fwd_out << -o;
                float2* dst = s_hand[threadIdx.x >> 5][run_end + 1];
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if ((fwd >> k) & 1u) dst[k + o] = make_float2(acc[2 * k], acc[2 * k + 1]);
            }
            const int phead = lane == 0 ? 0 : 31 - __clz(heads & ((1u << lane) - 1u));
            const uint32_t recv = __shfl_sync(0xffffffffu, fwd_out, phead);  // what the previous head handed over
            __syncwarp();
            if (valid && head) {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (link && ((recv >> k) & 1u)) {
                        const float2 t = s_hand[threadIdx.x >> 5][lane][k];
                        acc[2 * k] += t.x;
                        acc[2 * k + 1] += t.y;
                    }
                uint32_t idx[8];
                grid_corner_indices(c, res, entries, hashed, idx);
                const float* lvl = grad_table + 2 * (size_t)off;
                // 16-byte reductions for aligned x-corner pairs this head issues both of, 8-byte otherwise
                grid_scatter_cell_owned(lvl, idx, acc, 0xFFu & ~fwd);
            }
            __syncwarp();  // read before the next level's hand-over writes
        }
        __syncthreads();
        item = s_item[(it + 1) & 1];
        if (item < n_items) take(item);
    }
    sched_finish(sched);
}

// workspace of ngp_net_backward: the feature gradients, one half2 per (level, sample): 64 B per sample
extern "C" size_t ngp_net_backward_workspace(int64_t n) {
    if (n < 0) return 0;
    const int64_t n16 = (n + 15) / 16 * 16;
    return (size_t)n16 * NGP_MAX_LEVELS * sizeof(uint32_t);
}

static int check_bwd_args(const NgpNet* net, const NgpSamples* smp, void* workspace, size_t workspace_bytes) {
    if (!net || !smp || smp->n < 0) return NGP_EINVAL;
    if (net->meta.n_levels < 1 || net->meta.n_levels > NGP_MAX_LEVELS) return NGP_EINVAL;
    if (smp->n > 0 && (!workspace || workspace_bytes < ngp_net_backward_workspace(smp->n))) return NGP_EINVAL;
    return 0;
}

// first half: MLP backward (dgrad + wgrad), feature gradients -> workspace
extern "C" int ngp_net_backward_mlp(const NgpNet* net, const NgpSamples* smp, const float* dL_dsigmas, const float* dL_drgbs,
                                    const void* feat_save, const float* loss_scale, float* grad_enc, float* grad_rgb,
                                    void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_bwd_args(net, smp, workspace, workspace_bytes);
    if (rc) return rc;
    if (!dL_dsigmas || !dL_drgbs || !grad_enc || !grad_rgb) return NGP_EINVAL;
    if (smp->live_idx && (!smp->n_live_dev || !feat_save)) return NGP_EINVAL;  // a live list needs the saved features
    if (smp->n == 0) return 0;
    const int smem = (int)sizeof(Bwd3Smem) + 128;
    NGP_CUDA(feat_save ? ngp_smem_opt_in<k_ngp_bwd3<false>>(smem) : ngp_smem_opt_in<k_ngp_bwd3<true>>(smem));
    const int64_t n_mtiles = (smp->n + 15) / 16;
    const int64_t n_blks = (n_mtiles + B3_WARPS - 1) / B3_WARPS;
    const int grid = (int)(n_blks < (int64_t)ngp_sm_count() ? n_blks : ngp_sm_count());
    auto* kernel = feat_save ? k_ngp_bwd3<false> : k_ngp_bwd3<true>;
    NGP_CUDA(ngp_launch_pdl(kernel, grid, B3_THREADS, sizeof(Bwd3Smem) + 128, (cudaStream_t)stream, *net, *smp, dL_dsigmas,
                            dL_drgbs, (const uint4*)feat_save, loss_scale, grad_enc, grad_rgb, (uint32_t*)workspace,
                            n_mtiles * 16, sched_slot((cudaStream_t)stream)));
    NGP_CHECK_LAUNCH();
    NGP_TRACE(6, (cudaStream_t)stream);
    return 0;
}

// second half: feature gradients in workspace -> hash-table gradient
extern "C" int ngp_net_backward_scatter(const NgpNet* net, const NgpSamples* smp, const float* loss_scale, float* grad_enc,
                                        void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_bwd_args(net, smp, workspace, workspace_bytes);
    if (rc) return rc;
    if (!grad_enc || (smp->live_idx && !smp->n_live_dev)) return NGP_EINVAL;
    if (smp->n == 0) return 0;
    const int64_t n_mtiles = (smp->n + 15) / 16;
    // persistent: as many CTAs as are resident at once, at most one per item of the capacity
    const int n_groups = (net->meta.n_levels + SCATTER_GROUP - 1) / SCATTER_GROUP;
    int64_t gx = (smp->n + SCATTER_THREADS - 1) / SCATTER_THREADS * n_groups;
    const int64_t cap = (int64_t)ngp_sm_count() * SCATTER_MIN_BLOCKS;
    if (gx > cap) gx = cap;
    NGP_CUDA(ngp_launch_pdl(k_grid_scatter_merged, (unsigned)gx, SCATTER_THREADS, 0, (cudaStream_t)stream, *net, *smp,
                            (const uint32_t*)workspace, n_mtiles * 16, loss_scale, grad_enc + NGP_DENSITY_MLP_PARAMS,
                            sched_slot((cudaStream_t)stream)));
    NGP_CHECK_LAUNCH();
    NGP_TRACE(7, (cudaStream_t)stream);
    return 0;
}

extern "C" int ngp_net_backward(const NgpNet* net, const NgpSamples* smp, const float* dL_dsigmas, const float* dL_drgbs,
                                const void* feat_save, const float* loss_scale, float* grad_enc, float* grad_rgb,
                                void* workspace, size_t workspace_bytes, void* stream) {
    int rc = ngp_net_backward_mlp(net, smp, dL_dsigmas, dL_drgbs, feat_save, loss_scale, grad_enc, grad_rgb, workspace,
                                  workspace_bytes, stream);
    if (rc) return rc;
    return ngp_net_backward_scatter(net, smp, loss_scale, grad_enc, workspace, workspace_bytes, stream);
}

// -------------------------------------------------------------------------------------------------
// loss-scale helper
// -------------------------------------------------------------------------------------------------
__global__ void k_grad_amax(const float* __restrict__ dsig, const float* __restrict__ sig, const float* __restrict__ drgb,
                            int64_t n, float* __restrict__ amax) {
    float m = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float s = fminf(sig[i], 3.2690173e6f);  // exp(15): the TruncExp backward clamp
        m = fmaxf(m, fabsf(dsig[i] * s));
        m = fmaxf(m, fmaxf(fabsf(drgb[3 * i]), fmaxf(fabsf(drgb[3 * i + 1]), fabsf(drgb[3 * i + 2]))));
    }
    m = warp_max(m);
    // non-negative floats order like their bit patterns
    if ((threadIdx.x & 31) == 0 && m > 0.f && m < INFINITY) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));
}
__global__ void k_grad_scale(float* __restrict__ amax, float* __restrict__ scale_out) {
    const float m = *amax;
    float s = 1.0f;
    if (m > 0.f && m < INFINITY) {
        int e;
        frexpf(256.0f / m, &e);  // 256/m = f * 2^e, f in [0.5,1)  ->  2^(e-1) <= 256/m
        e = max(-60, min(60, e - 1));
        s = scalbnf(1.0f, e);
    }
    *scale_out = s;
    *amax = 0.f;
}
extern "C" int ngp_grad_scale(const float* dL_dsigmas, const float* sigmas, const float* dL_drgbs, int64_t n,
                              float* scratch, float* scale_out, void* stream) {
    if (n < 0 || !scratch || !scale_out) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(cudaMemsetAsync(scratch, 0, sizeof(float), st));
    if (n > 0) {
        int grid = ngp_div_up(n, 256);
        if (grid > 4 * ngp_sm_count()) grid = 4 * ngp_sm_count();
        k_grad_amax<<<grid, 256, 0, st>>>(dL_dsigmas, sigmas, dL_drgbs, n, scratch);
        NGP_CHECK_LAUNCH();
    }
    k_grad_scale<<<1, 1, 0, st>>>(scratch, scale_out);
    NGP_CHECK_LAUNCH();
    return 0;
}
