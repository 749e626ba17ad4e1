// The twelve `vren` operators of kwea123/ngp_pl re-implemented for sm_90a behind a C ABI.
// Each entry point cites the reference operator it replaces (reference models/csrc/binding.cpp and
// the kernel behind it). Plain device pointers and sizes only; the caller owns every buffer.
#include "common.cuh"
#include "march.cuh"
#include "composite.cuh"
#include "../../include/ngp_b200.h"
#include <cub/device/device_scan.cuh>

// ---------------------------------------------------------------------------------------------
// ray_aabb_intersect  (reference binding.cpp:4-16 -> intersection.cu:25-100)
// ---------------------------------------------------------------------------------------------
__global__ void k_fill_hits(int64_t n, float* __restrict__ hits_t, int64_t* __restrict__ hits_idx, int* __restrict__ hit_cnt,
                            int64_t n_rays) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) {
        hits_t[2 * i] = -1.0f;
        hits_t[2 * i + 1] = -1.0f;
        hits_idx[i] = -1;
    }
    if (i < n_rays) hit_cnt[i] = 0;
}

__global__ void k_ray_aabb(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                           const float* __restrict__ centers, const float* __restrict__ half_sizes,
                           int n_rays, int n_voxels, int max_hits,
                           int* __restrict__ hit_cnt, float* __restrict__ hits_t, int64_t* __restrict__ hits_idx) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = blockIdx.y;
    if (r >= n_rays || v >= n_voxels) return;
    const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                        rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
    const float2 tt = ray_aabb(ray, centers[3 * v], centers[3 * v + 1], centers[3 * v + 2],
                               half_sizes[3 * v], half_sizes[3 * v + 1], half_sizes[3 * v + 2]);
    if (tt.y > 0.0f) {
        const int cnt = atomicAdd(&hit_cnt[r], 1);
        if (cnt < max_hits) {
            const int64_t k = (int64_t)r * max_hits + cnt;
            hits_t[2 * k] = fmaxf(tt.x, 0.0f);
            hits_t[2 * k + 1] = tt.y;
            hits_idx[k] = v;
        }
    }
}

extern "C" int ngp_ray_aabb_intersect(const float* rays_o, const float* rays_d, const float* centers,
                                      const float* half_sizes, int n_rays, int n_voxels, int max_hits,
                                      int* hit_cnt, float* hits_t, int64_t* hits_voxel_idx, void* stream) {
    if (n_rays < 0 || n_voxels < 0 || max_hits < 1) return NGP_EINVAL;
    if (n_rays == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = (int64_t)n_rays * max_hits;
    k_fill_hits<<<ngp_div_up(n, 256), 256, 0, st>>>(n, hits_t, hits_voxel_idx, hit_cnt, n_rays);
    NGP_CHECK_LAUNCH();
    if (n_voxels > 0) {
        dim3 grid(ngp_div_up(n_rays, 128), n_voxels);
        k_ray_aabb<<<grid, 128, 0, st>>>(rays_o, rays_d, centers, half_sizes, n_rays, n_voxels, max_hits,
                                          hit_cnt, hits_t, hits_voxel_idx);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------
// ray_sphere_intersect  (reference binding.cpp:19-31 -> intersection.cu:103-197). Exported by the
// reference but never called from its Python; kept so the operator table is complete.
// ---------------------------------------------------------------------------------------------
__global__ void k_ray_sphere(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                             const float* __restrict__ centers, const float* __restrict__ radii,
                             int n_rays, int n_spheres, int max_hits,
                             int* __restrict__ hit_cnt, float* __restrict__ hits_t, int64_t* __restrict__ hits_idx) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = blockIdx.y;
    if (r >= n_rays || s >= n_spheres) return;
    const float ox = rays_o[3 * r], oy = rays_o[3 * r + 1], oz = rays_o[3 * r + 2];
    const float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
    const float cx = ox - centers[3 * s], cy = oy - centers[3 * s + 1], cz = oz - centers[3 * s + 2];
    const float rad = radii[s];
    const float a = dx * dx + dy * dy + dz * dz;
    const float half_b = dx * cx + dy * cy + dz * cz;
    const float c = cx * cx + cy * cy + cz * cz - rad * rad;
    const float disc = half_b * half_b - a * c;
    if (disc < 0.0f) return;
    const float sq = sqrtf(disc);
    const float t1 = (-half_b - sq) / a, t2 = (-half_b + sq) / a;
    if (t2 > 0.0f) {
        const int cnt = atomicAdd(&hit_cnt[r], 1);
        if (cnt < max_hits) {
            const int64_t k = (int64_t)r * max_hits + cnt;
            hits_t[2 * k] = fmaxf(t1, 0.0f);
            hits_t[2 * k + 1] = t2;
            hits_idx[k] = s;
        }
    }
}

extern "C" int ngp_ray_sphere_intersect(const float* rays_o, const float* rays_d, const float* centers,
                                        const float* radii, int n_rays, int n_spheres, int max_hits,
                                        int* hit_cnt, float* hits_t, int64_t* hits_sphere_idx, void* stream) {
    if (n_rays < 0 || n_spheres < 0 || max_hits < 1) return NGP_EINVAL;
    if (n_rays == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = (int64_t)n_rays * max_hits;
    k_fill_hits<<<ngp_div_up(n, 256), 256, 0, st>>>(n, hits_t, hits_sphere_idx, hit_cnt, n_rays);
    NGP_CHECK_LAUNCH();
    if (n_spheres > 0) {
        dim3 grid(ngp_div_up(n_rays, 128), n_spheres);
        k_ray_sphere<<<grid, 128, 0, st>>>(rays_o, rays_d, centers, radii, n_rays, n_spheres, max_hits,
                                            hit_cnt, hits_t, hits_sphere_idx);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------
// packbits  (reference binding.cpp:34-43 -> raymarching.cu:122-161): bit i of byte n = grid[8n+i] > thr
// A thread packs 4 output bytes from 32 consecutive densities (128-bit loads), so a warp reads 4 KB
// contiguous and writes 128 B contiguous.
// ---------------------------------------------------------------------------------------------
// density > threshold evaluated in the wider of the two types, as C++ promotion does in the reference
template <typename T> __device__ __forceinline__ bool above(T v, float thr);
template <> __device__ __forceinline__ bool above<float>(float v, float thr) { return v > thr; }
template <> __device__ __forceinline__ bool above<double>(double v, float thr) { return v > (double)thr; }
template <> __device__ __forceinline__ bool above<__half>(__half v, float thr) { return __half2float(v) > thr; }

template <typename T>
__global__ void k_packbits(const T* __restrict__ grid, int64_t n_bytes, float thr, const float* __restrict__ thr_dev,
                           uint8_t* __restrict__ bits) {
    const int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (n >= n_bytes) return;
    if (thr_dev) thr = fminf(thr, *thr_dev);
    const T* g = grid + 8 * n;
    uint32_t b = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) b |= above<T>(g[i], thr) ? (1u << i) : 0u;
    bits[n] = (uint8_t)b;
}

__global__ void k_packbits_f32x4(const float4* __restrict__ grid, int64_t n_words, float thr,
                                 const float* __restrict__ thr_dev, uint32_t* __restrict__ bits) {
    const int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (n >= n_words) return;
    if (thr_dev) thr = fminf(thr, *thr_dev);
    const float4* g = grid + 8 * n;
    uint32_t b = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float4 v = __ldg(g + i);
        b |= (v.x > thr ? 1u : 0u) << (4 * i);
        b |= (v.y > thr ? 1u : 0u) << (4 * i + 1);
        b |= (v.z > thr ? 1u : 0u) << (4 * i + 2);
        b |= (v.w > thr ? 1u : 0u) << (4 * i + 3);
    }
    bits[n] = b;
}

// dtype: 0 = float32, 1 = float16, 2 = float64. thr_dev (optional, device float*) lets the caller keep
// min(mean_density, thr) on the device: effective threshold = min(thr, *thr_dev).
extern "C" int ngp_packbits(const void* density_grid, int dtype, int64_t n_bytes, float thr, const float* thr_dev,
                            uint8_t* bitfield, void* stream) {
    if (n_bytes < 0 || dtype < 0 || dtype > 2) return NGP_EINVAL;
    if (n_bytes == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0 && (n_bytes % 4) == 0 && (((uintptr_t)density_grid) % 16) == 0 && (((uintptr_t)bitfield) % 4) == 0) {
        const int64_t nw = n_bytes / 4;
        k_packbits_f32x4<<<ngp_div_up(nw, 256), 256, 0, st>>>((const float4*)density_grid, nw, thr, thr_dev,
                                                               (uint32_t*)bitfield);
    } else if (dtype == 0) {
        k_packbits<float><<<ngp_div_up(n_bytes, 256), 256, 0, st>>>((const float*)density_grid, n_bytes, thr, thr_dev, bitfield);
    } else if (dtype == 1) {
        k_packbits<__half><<<ngp_div_up(n_bytes, 256), 256, 0, st>>>((const __half*)density_grid, n_bytes, thr, thr_dev, bitfield);
    } else {
        k_packbits<double><<<ngp_div_up(n_bytes, 256), 256, 0, st>>>((const double*)density_grid, n_bytes, thr, thr_dev, bitfield);
    }
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// morton3D / morton3D_invert  (reference binding.cpp:46-57 -> raymarching.cu:62-119)
// Valid domain: 0 <= coord < 1024 (the occupancy grid uses < 128).
// ---------------------------------------------------------------------------------------------
__global__ void k_morton3d(const int* __restrict__ coords, int n, int* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = (int)morton_encode3((uint32_t)coords[3 * i], (uint32_t)coords[3 * i + 1], (uint32_t)coords[3 * i + 2]);
}
__global__ void k_morton3d_invert(const int* __restrict__ idx, int n, int* __restrict__ coords) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t v = (uint32_t)idx[i];
    coords[3 * i] = (int)morton_compact10(v);
    coords[3 * i + 1] = (int)morton_compact10(v >> 1);
    coords[3 * i + 2] = (int)morton_compact10(v >> 2);
}
extern "C" int ngp_morton3D(const int* coords, int n, int* indices, void* stream) {
    if (n < 0) return NGP_EINVAL;
    if (n == 0) return 0;
    k_morton3d<<<ngp_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(coords, n, indices);
    NGP_CHECK_LAUNCH();
    return 0;
}
extern "C" int ngp_morton3D_invert(const int* indices, int n, int* coords, void* stream) {
    if (n < 0) return NGP_EINVAL;
    if (n == 0) return 0;
    k_morton3d_invert<<<ngp_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(indices, n, coords);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// raymarching_train  (reference binding.cpp:60-81 -> raymarching.cu:166-332)
// Three launches instead of one kernel with two global atomics: count -> exclusive scan -> write.
// Sample ranges are therefore ordered by ray index and the whole op is deterministic (the
// reference's start_idx / rays_a row order depend on atomic arrival order); per-ray contents are
// bit-identical. Outputs beyond counter[0] rows are never written (the reference zero-fills 268 MB).
// ---------------------------------------------------------------------------------------------
__global__ void k_march_train_count(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                    const float* __restrict__ hits_t, const float* __restrict__ noise,
                                    const uint8_t* __restrict__ bitfield, int cascades, int grid_size, float scale,
                                    float esf, int max_samples, int n_rays, int* __restrict__ n_samples) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const MarchConst c = make_march_const(bitfield, cascades, grid_size, max_samples, scale, esf, scale);
    const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                        rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
    const float t2 = hits_t[2 * r + 1];
    float t = march_jitter(hits_t[2 * r], noise[r], c);
    int n = 0;
    float dt;
    while (0.0f <= t && t < t2 && n < max_samples) {
        if (march_visit_t<false, false>(ray, c, t, dt)) {
            t = __fadd_rn(t, dt);
            ++n;
        }
    }
    n_samples[r] = n;
}

__global__ void k_march_train_write(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                    const float* __restrict__ hits_t, const float* __restrict__ noise,
                                    const uint8_t* __restrict__ bitfield, int cascades, int grid_size, float scale,
                                    float esf, int max_samples, int n_rays,
                                    const int* __restrict__ n_samples, const int* __restrict__ offsets,
                                    int64_t* __restrict__ rays_a, float* __restrict__ xyzs, float* __restrict__ dirs,
                                    float* __restrict__ deltas, float* __restrict__ ts, int* __restrict__ counter) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const int n_tot = n_samples[r];
    const int start = offsets[r];
    rays_a[3 * r] = r;
    rays_a[3 * r + 1] = start;
    rays_a[3 * r + 2] = n_tot;
    if (r == n_rays - 1) {
        counter[0] = start + n_tot;
        counter[1] = n_rays;
    }
    if (n_tot == 0) return;
    const MarchConst c = make_march_const(bitfield, cascades, grid_size, max_samples, scale, esf, scale);
    const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                        rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
    const float t2 = hits_t[2 * r + 1];
    float t = march_jitter(hits_t[2 * r], noise[r], c);
    int n = 0;
    float dt;
    while (t < t2 && n < n_tot) {
        if (march_visit_t<false, false>(ray, c, t, dt)) {
            const int64_t s = (int64_t)start + n;
            xyzs[3 * s] = __fmaf_rn(ray.dx, t, ray.ox);
            xyzs[3 * s + 1] = __fmaf_rn(ray.dy, t, ray.oy);
            xyzs[3 * s + 2] = __fmaf_rn(ray.dz, t, ray.oz);
            dirs[3 * s] = ray.dx; dirs[3 * s + 1] = ray.dy; dirs[3 * s + 2] = ray.dz;
            ts[s] = t;
            deltas[s] = dt;
            t = __fadd_rn(t, dt);
            ++n;
        }
    }
}

static size_t scan_temp_bytes(int n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const int*)nullptr, (int*)nullptr, n);
    return (bytes + 255) & ~(size_t)255;
}

// Warp-per-ray variant (march.cuh: march_ray_warp, bit-exact with the serial loop): ONE march into a per-ray
// staging row of (t, dt), prefix sum, then a coalesced expansion to xyzs/dirs/deltas/ts. Used whenever the
// staging rows fit the workspace budget; the serial two-pass kernels above remain for very large ray counts. They
// are not only a memory fallback: at 2^18 rays and max_samples 1024 on the mip360-shaped scene (6 cascades,
// exp_step_factor 1/256) they take 5.4 ms against 7.1 ms for the warp-per-ray path (Lego: 2.5 ms against 1.9 ms),
// measured on an H100 80GB HBM3 at a 400 W power limit.
#define NGP_MARCH_STAGE_BUDGET (512ull << 20)

template <bool CONST_DT, bool ONE_CASCADE>
__global__ void k_march_train_stage(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                    const float* __restrict__ hits_t, const float* __restrict__ noise,
                                    const uint8_t* __restrict__ bitfield, int cascades, int grid_size, float scale, float esf,
                                    int max_samples, int n_rays, float2* __restrict__ stage, int* __restrict__ n_samples) {
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rays) return;
    const MarchConst c = make_march_const(bitfield, cascades, grid_size, max_samples, scale, esf, scale);
    const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                        rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
    const float t2 = hits_t[2 * r + 1];
    const float t = march_jitter(hits_t[2 * r], noise[r], c);
    float2* st = stage + (size_t)r * max_samples;
    const int n = march_ray_warp<CONST_DT, ONE_CASCADE>(ray, c, t, t2, max_samples, lane,
                                                        [&](int k, float ts, float dts) { st[k] = make_float2(ts, dts); });
    if (lane == 0) n_samples[r] = n;
}

__global__ void k_march_train_expand(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                     const float2* __restrict__ stage, int max_samples, int n_rays,
                                     const int* __restrict__ n_samples, const int* __restrict__ offsets,
                                     int64_t* __restrict__ rays_a, float* __restrict__ xyzs, float* __restrict__ dirs,
                                     float* __restrict__ deltas, float* __restrict__ ts, int* __restrict__ counter) {
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rays) return;
    const int n = n_samples[r];
    const int64_t start = offsets[r];
    if (lane == 0) {
        rays_a[3 * r] = r;
        rays_a[3 * r + 1] = start;
        rays_a[3 * r + 2] = n;
        if (r == n_rays - 1) {
            counter[0] = (int)(start + n);
            counter[1] = n_rays;
        }
    }
    const float ox = rays_o[3 * r], oy = rays_o[3 * r + 1], oz = rays_o[3 * r + 2];
    const float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
    const float2* st = stage + (size_t)r * max_samples;
    for (int k = lane; k < n; k += 32) {
        const float2 v = st[k];
        const int64_t s = start + k;
        xyzs[3 * s] = __fmaf_rn(dx, v.x, ox);
        xyzs[3 * s + 1] = __fmaf_rn(dy, v.x, oy);
        xyzs[3 * s + 2] = __fmaf_rn(dz, v.x, oz);
        dirs[3 * s] = dx; dirs[3 * s + 1] = dy; dirs[3 * s + 2] = dz;
        ts[s] = v.x;
        deltas[s] = v.y;
    }
}

static bool march_use_stage(int n_rays, int max_samples) {
    return (unsigned long long)n_rays * (unsigned long long)max_samples * sizeof(float2) <= NGP_MARCH_STAGE_BUDGET;
}

extern "C" size_t ngp_raymarching_train_workspace2(int n_rays, int max_samples) {
    if (n_rays <= 0) return 256;
    const size_t ints = (((size_t)n_rays * sizeof(int)) + 255) & ~(size_t)255;
    size_t bytes = 2 * ints + scan_temp_bytes(n_rays);
    if (max_samples > 0 && march_use_stage(n_rays, max_samples)) bytes += (size_t)n_rays * max_samples * sizeof(float2) + 256;
    return bytes;
}
extern "C" size_t ngp_raymarching_train_workspace(int n_rays) { return ngp_raymarching_train_workspace2(n_rays, 0); }

static inline int march_block(int n_rays) { return n_rays >= ngp_sm_count() * 128 * 4 ? 128 : 32; }

extern "C" int ngp_raymarching_train(const float* rays_o, const float* rays_d, const float* hits_t,
                                     const uint8_t* density_bitfield, int cascades, float scale, float exp_step_factor,
                                     const float* noise, int grid_size, int max_samples, int n_rays,
                                     int64_t* rays_a, float* xyzs, float* dirs, float* deltas, float* ts, int* counter,
                                     void* workspace, size_t workspace_bytes, void* stream) {
    if (n_rays < 0 || cascades < 1 || grid_size < 1 || grid_size > 1024 || max_samples < 1) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_rays == 0) {
        NGP_CUDA(cudaMemsetAsync(counter, 0, 2 * sizeof(int), st));
        return 0;
    }
    if (workspace_bytes < ngp_raymarching_train_workspace(n_rays)) return NGP_EINVAL;
    const size_t ints = (((size_t)n_rays * sizeof(int)) + 255) & ~(size_t)255;
    int* n_samples = (int*)workspace;
    int* offsets = (int*)((char*)workspace + ints);
    void* temp = (char*)workspace + 2 * ints;
    size_t temp_bytes = scan_temp_bytes(n_rays);
    // the caller sized the workspace with ngp_raymarching_train_workspace2: warp-per-ray path with staging rows
    if (march_use_stage(n_rays, max_samples) && workspace_bytes >= ngp_raymarching_train_workspace2(n_rays, max_samples)) {
        float2* stage = (float2*)((((uintptr_t)temp + temp_bytes) + 255) & ~(uintptr_t)255);
        const bool const_dt = march_const_dt(exp_step_factor, max_samples, scale, grid_size);
        const dim3 mg(ngp_div_up((int64_t)n_rays * 32, 128));
        march_dispatch(const_dt, cascades, [&](auto cd, auto oc) {
            k_march_train_stage<decltype(cd)::value, decltype(oc)::value><<<mg, 128, 0, st>>>(
                rays_o, rays_d, hits_t, noise, density_bitfield, cascades, grid_size, scale, exp_step_factor, max_samples,
                n_rays, stage, n_samples);
        });
        NGP_CHECK_LAUNCH();
        NGP_CUDA(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, n_samples, offsets, n_rays, st));
        NGP_COUNT_LAUNCHES(2);  // cub: init + sweep kernels
        k_march_train_expand<<<mg, 128, 0, st>>>(rays_o, rays_d, stage, max_samples, n_rays, n_samples, offsets, rays_a, xyzs,
                                                 dirs, deltas, ts, counter);
        NGP_CHECK_LAUNCH();
        return 0;
    }
    const int bs = march_block(n_rays);
    k_march_train_count<<<ngp_div_up(n_rays, bs), bs, 0, st>>>(rays_o, rays_d, hits_t, noise, density_bitfield, cascades,
                                                                grid_size, scale, exp_step_factor, max_samples, n_rays,
                                                                n_samples);
    NGP_CHECK_LAUNCH();
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, n_samples, offsets, n_rays, st));
    NGP_COUNT_LAUNCHES(2);  // cub: init + sweep kernels
    k_march_train_write<<<ngp_div_up(n_rays, bs), bs, 0, st>>>(rays_o, rays_d, hits_t, noise, density_bitfield, cascades,
                                                                grid_size, scale, exp_step_factor, max_samples, n_rays,
                                                                n_samples, offsets, rays_a, xyzs, dirs, deltas, ts, counter);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// raymarching_test  (reference binding.cpp:84-106 -> raymarching.cu:335-454)
// Rectangular (n_alive, N_samples) outputs, zero-filled where no sample was produced (the reference
// relies on dirs==0 to detect padding, rendering.py:91); hits_t[r][0] is advanced in place.
// ---------------------------------------------------------------------------------------------
__global__ void k_march_test(const float* __restrict__ rays_o, const float* __restrict__ rays_d, float* __restrict__ hits_t,
                             const int64_t* __restrict__ alive, const uint8_t* __restrict__ bitfield, int cascades,
                             int grid_size, float scale, float esf, int n_samples_max, int max_samples, int n_alive,
                             float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas,
                             float* __restrict__ ts, int* __restrict__ n_eff) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int64_t r = alive[n];
    // the reference passes `cascades` where calc_dt expects `scale` (raymarching.cu:370,399)
    const MarchConst c = make_march_const(bitfield, cascades, grid_size, max_samples, scale, esf, (float)cascades);
    const MarchRay ray = make_march_ray(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2],
                                        rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]);
    float t = hits_t[2 * r];
    const float t2 = hits_t[2 * r + 1];
    int s = 0;
    float dt;
    const int64_t row = (int64_t)n * n_samples_max;
    while (t < t2 && s < n_samples_max) {
        if (march_visit_t<false, false>(ray, c, t, dt)) {
            const int64_t k = row + s;
            xyzs[3 * k] = __fmaf_rn(ray.dx, t, ray.ox);
            xyzs[3 * k + 1] = __fmaf_rn(ray.dy, t, ray.oy);
            xyzs[3 * k + 2] = __fmaf_rn(ray.dz, t, ray.oz);
            dirs[3 * k] = ray.dx; dirs[3 * k + 1] = ray.dy; dirs[3 * k + 2] = ray.dz;
            ts[k] = t;
            deltas[k] = dt;
            t = __fadd_rn(t, dt);
            hits_t[2 * r] = t;
            ++s;
        }
    }
    n_eff[n] = s;  // slots s.. keep the zeros of the memsets below
}

extern "C" int ngp_raymarching_test(const float* rays_o, const float* rays_d, float* hits_t, const int64_t* alive_indices,
                                    const uint8_t* density_bitfield, int cascades, float scale, float exp_step_factor,
                                    int grid_size, int max_samples, int N_samples, int n_alive,
                                    float* xyzs, float* dirs, float* deltas, float* ts, int* N_eff_samples, void* stream) {
    if (n_alive < 0 || cascades < 1 || grid_size < 1 || grid_size > 1024 || max_samples < 1 || N_samples < 1) return NGP_EINVAL;
    if (n_alive == 0) return 0;
    // zero padding of the rectangular outputs (the reference allocates them with torch::zeros, raymarching.cu:423-426):
    // four streaming memsets instead of strided stores from the marching threads
    const size_t slots = (size_t)n_alive * N_samples;
    NGP_CUDA(cudaMemsetAsync(xyzs, 0, slots * 3 * sizeof(float), (cudaStream_t)stream));
    NGP_CUDA(cudaMemsetAsync(dirs, 0, slots * 3 * sizeof(float), (cudaStream_t)stream));
    NGP_CUDA(cudaMemsetAsync(deltas, 0, slots * sizeof(float), (cudaStream_t)stream));
    NGP_CUDA(cudaMemsetAsync(ts, 0, slots * sizeof(float), (cudaStream_t)stream));
    NGP_COUNT_LAUNCHES(4);
    const int bs = n_alive >= ngp_sm_count() * 128 * 4 ? 128 : 64;
    k_march_test<<<ngp_div_up(n_alive, bs), bs, 0, (cudaStream_t)stream>>>(
        rays_o, rays_d, hits_t, alive_indices, density_bitfield, cascades, grid_size, scale, exp_step_factor, N_samples,
        max_samples, n_alive, xyzs, dirs, deltas, ts, N_eff_samples);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// composite_train_fw / composite_train_bw  (reference binding.cpp:109-163 -> volumerendering.cu:6-202)
// One warp per ray (the reference uses one thread per ray).
// ---------------------------------------------------------------------------------------------
__global__ void k_composite_train_fw(const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                     const float* __restrict__ deltas, const float* __restrict__ ts,
                                     const int64_t* __restrict__ rays_a, float T_threshold, int n_rays,
                                     int64_t* __restrict__ total_samples, float* __restrict__ opacity,
                                     float* __restrict__ depth, float* __restrict__ rgb, float* __restrict__ ws) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n_rays) return;
    const int64_t ray = rays_a[3 * w];
    const int64_t start = rays_a[3 * w + 1];
    const int n = (int)rays_a[3 * w + 2];
    const RaySamples smp{sigmas + start, deltas + start, ts + start, rgbs + 3 * start};
    const CompositeOut o = composite_ray_warp<0>(smp, n, T_threshold, lane, nullptr, ws + start);
    if (lane == 0) {
        opacity[ray] = o.opacity;
        depth[ray] = o.depth;
        rgb[3 * ray] = o.r;
        rgb[3 * ray + 1] = o.g;
        rgb[3 * ray + 2] = o.b;
        total_samples[ray] = o.total_samples;
    }
}

extern "C" int ngp_composite_train_fw(const float* sigmas, const float* rgbs, const float* deltas, const float* ts,
                                      const int64_t* rays_a, float T_threshold, int n_rays, int64_t n_samples,
                                      int64_t* total_samples, float* opacity, float* depth, float* rgb, float* ws,
                                      void* stream) {
    (void)n_samples;
    if (n_rays < 0) return NGP_EINVAL;
    if (n_rays == 0) return 0;
    k_composite_train_fw<<<ngp_div_up((int64_t)n_rays * 32, 128), 128, 0, (cudaStream_t)stream>>>(
        sigmas, rgbs, deltas, ts, rays_a, T_threshold, n_rays, total_samples, opacity, depth, rgb, ws);
    NGP_CHECK_LAUNCH();
    return 0;
}

__global__ void k_composite_train_bw(const float* __restrict__ dL_dopacity, const float* __restrict__ dL_ddepth,
                                     const float* __restrict__ dL_drgb, const float* __restrict__ dL_dws,
                                     const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                     const float* __restrict__ ws, const float* __restrict__ deltas,
                                     const float* __restrict__ ts, const int64_t* __restrict__ rays_a,
                                     const float* __restrict__ opacity, const float* __restrict__ depth,
                                     const float* __restrict__ rgb, float T_threshold, int n_rays,
                                     float* __restrict__ dL_dsigmas, float* __restrict__ dL_drgbs) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n_rays) return;
    const int64_t ray = rays_a[3 * w];
    const int64_t start = rays_a[3 * w + 1];
    const int n = (int)rays_a[3 * w + 2];
    const RaySamples smp{sigmas + start, deltas + start, ts + start, rgbs + 3 * start};
    composite_ray_warp_bwd<0, true>(smp, n, T_threshold, lane, nullptr,
                                    make_float3(dL_drgb[3 * ray], dL_drgb[3 * ray + 1], dL_drgb[3 * ray + 2]),
                                    dL_dopacity[ray], dL_ddepth[ray],
                                    make_float3(rgb[3 * ray], rgb[3 * ray + 1], rgb[3 * ray + 2]), opacity[ray],
                                    depth[ray], dL_dws + start, ws + start, dL_dsigmas + start, dL_drgbs + 3 * start);
}

extern "C" int ngp_composite_train_bw(const float* dL_dopacity, const float* dL_ddepth, const float* dL_drgb,
                                      const float* dL_dws, const float* sigmas, const float* rgbs, const float* ws,
                                      const float* deltas, const float* ts, const int64_t* rays_a, const float* opacity,
                                      const float* depth, const float* rgb, float T_threshold, int n_rays,
                                      int64_t n_samples, float* dL_dsigmas, float* dL_drgbs, void* stream) {
    (void)n_samples;
    if (n_rays < 0) return NGP_EINVAL;
    if (n_rays == 0) return 0;
    k_composite_train_bw<<<ngp_div_up((int64_t)n_rays * 32, 128), 128, 0, (cudaStream_t)stream>>>(
        dL_dopacity, dL_ddepth, dL_drgb, dL_dws, sigmas, rgbs, ws, deltas, ts, rays_a, opacity, depth, rgb, T_threshold,
        n_rays, dL_dsigmas, dL_drgbs);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// composite_test_fw  (reference binding.cpp:166-194 -> volumerendering.cu:205-285)
// Rows are short (N_samples <= 64) and rectangular: one thread per alive ray, like the reference,
// accumulating in registers and writing the per-ray accumulators once.
// ---------------------------------------------------------------------------------------------
__global__ void k_composite_test_fw(const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                    const float* __restrict__ deltas, const float* __restrict__ ts,
                                    int64_t* __restrict__ alive, float T_threshold, const int* __restrict__ n_eff,
                                    int n_alive, int n_samples_max, float* __restrict__ opacity,
                                    float* __restrict__ depth, float* __restrict__ rgb) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int ne = n_eff[n];
    if (ne == 0) {
        alive[n] = -1;
        return;
    }
    const int64_t r = alive[n];
    float o = opacity[r], d = depth[r];
    float cr = rgb[3 * r], cg = rgb[3 * r + 1], cb = rgb[3 * r + 2];
    const int64_t row = (int64_t)n * n_samples_max;
    if (composite_ray_serial(RaySamples{sigmas, deltas, ts, rgbs}, row, ne, T_threshold, cr, cg, cb, d, o)) alive[n] = -1;
    opacity[r] = o;
    depth[r] = d;
    rgb[3 * r] = cr; rgb[3 * r + 1] = cg; rgb[3 * r + 2] = cb;
}

extern "C" int ngp_composite_test_fw(const float* sigmas, const float* rgbs, const float* deltas, const float* ts,
                                     const float* hits_t, int64_t* alive_indices, float T_threshold,
                                     const int* N_eff_samples, int n_alive, int N_samples,
                                     float* opacity, float* depth, float* rgb, void* stream) {
    (void)hits_t;  // unused by the reference kernel as well (volumerendering.cu:205-249)
    if (n_alive < 0 || N_samples < 1) return NGP_EINVAL;
    if (n_alive == 0) return 0;
    k_composite_test_fw<<<ngp_div_up(n_alive, 128), 128, 0, (cudaStream_t)stream>>>(
        sigmas, rgbs, deltas, ts, alive_indices, T_threshold, N_eff_samples, n_alive, N_samples, opacity, depth, rgb);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// distortion_loss_fw / distortion_loss_bw  (reference binding.cpp:197-231 -> losses.cu:10-174)
// One warp per ray; the four thrust scans + elementwise torch ops + reduce of the reference become
// one pass.
// Every ray's segment is clipped to the n_samples entries the per-sample arrays hold (the Trainer's capacity may be smaller
// than what its batch marched, as in train.cu): a ray clipped to nothing gets loss 0 and no per-sample writes.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int distortion_extent(int64_t start, int64_t n, int64_t n_samples) {
    return (int)max((int64_t)0, min(n, n_samples - start));
}

__global__ void k_distortion_fw(const float* __restrict__ ws, const float* __restrict__ deltas, const float* __restrict__ ts,
                                const int64_t* __restrict__ rays_a, int n_rays, int64_t n_samples,
                                float* __restrict__ loss, float* __restrict__ ws_inc, float* __restrict__ wts_inc) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n_rays) return;
    const int64_t ray = rays_a[3 * w];
    const int64_t start = rays_a[3 * w + 1];
    const int n = distortion_extent(start, rays_a[3 * w + 2], n_samples);
    float cw = 0.f, cwt = 0.f, acc = 0.f;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool valid = i < n;
        const float wi = valid ? ws[start + i] : 0.f;
        const float wt = valid ? wi * ts[start + i] : 0.f;
        const float wi_inc = warp_scan_add(wi, lane) + cw;
        const float wt_inc = warp_scan_add(wt, lane) + cwt;
        if (valid) {
            const float wi_exc = wi_inc - wi, wt_exc = wt_inc - wt;
            ws_inc[start + i] = wi_inc;
            wts_inc[start + i] = wt_inc;
            acc += 2.0f * (wt_inc * wi_exc - wi_inc * wt_exc) + (1.0f / 3.0f) * wi * wi * deltas[start + i];
        }
        cw = __shfl_sync(0xffffffffu, wi_inc, 31);
        cwt = __shfl_sync(0xffffffffu, wt_inc, 31);
    }
    acc = warp_sum(acc);
    if (lane == 0) loss[ray] = acc;
}

extern "C" int ngp_distortion_loss_fw(const float* ws, const float* deltas, const float* ts, const int64_t* rays_a,
                                      int n_rays, int64_t n_samples, float* loss, float* ws_inclusive_scan,
                                      float* wts_inclusive_scan, void* stream) {
    if (n_rays < 0 || n_samples < 0) return NGP_EINVAL;
    if (n_rays == 0) return 0;
    k_distortion_fw<<<ngp_div_up((int64_t)n_rays * 32, 128), 128, 0, (cudaStream_t)stream>>>(
        ws, deltas, ts, rays_a, n_rays, n_samples, loss, ws_inclusive_scan, wts_inclusive_scan);
    NGP_CHECK_LAUNCH();
    return 0;
}

__global__ void k_distortion_bw(const float* __restrict__ dL_dloss, const float* __restrict__ ws_inc,
                                const float* __restrict__ wts_inc, const float* __restrict__ ws,
                                const float* __restrict__ deltas, const float* __restrict__ ts,
                                const int64_t* __restrict__ rays_a, int n_rays, int64_t n_samples,
                                float* __restrict__ dL_dws) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n_rays) return;
    const int64_t ray = rays_a[3 * w];
    const int64_t start = rays_a[3 * w + 1];
    const int n = distortion_extent(start, rays_a[3 * w + 2], n_samples);
    if (n <= 0) return;
    const float g = dL_dloss[ray];
    const float ws_sum = ws_inc[start + n - 1];
    const float wts_sum = wts_inc[start + n - 1];
    for (int i = lane; i < n; i += 32) {
        const int64_t s = start + i;
        const float t = ts[s];
        const float head = (i == 0) ? 0.f : (t * ws_inc[s - 1] - wts_inc[s - 1]);
        const float tail = wts_sum - wts_inc[s] - t * (ws_sum - ws_inc[s]);
        dL_dws[s] = g * 2.0f * (head + tail) + g * (2.0f / 3.0f) * ws[s] * deltas[s];
    }
}

extern "C" int ngp_distortion_loss_bw(const float* dL_dloss, const float* ws_inclusive_scan, const float* wts_inclusive_scan,
                                      const float* ws, const float* deltas, const float* ts, const int64_t* rays_a,
                                      int n_rays, int64_t n_samples, float* dL_dws, void* stream) {
    if (n_rays < 0 || n_samples < 0) return NGP_EINVAL;
    if (n_rays == 0) return 0;
    k_distortion_bw<<<ngp_div_up((int64_t)n_rays * 32, 128), 128, 0, (cudaStream_t)stream>>>(
        dL_dloss, ws_inclusive_scan, wts_inclusive_scan, ws, deltas, ts, rays_a, n_rays, n_samples, dL_dws);
    NGP_CHECK_LAUNCH();
    return 0;
}
