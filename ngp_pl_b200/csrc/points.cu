// Point-cloud export (include/ngp_b200.h, "Point-cloud export"; numpy restatement: oracle/points_ref.py).
//
// rays       : one thread per ray computes its global pixel q = (k g) mod N in 128-bit integers and splits it into view
//              and pixel; ngp_gen_rays then builds the rays with the training batch's arithmetic.
// backproject: one thread per ray decides whether it is kept, a scan of the flags numbers the kept rays in ascending
//              order, one thread per ray writes its point, colour and view at its number; one count read-back.
// voxel      : cell key per point (the simplification's rule 1, csrc/cluster.cuh) -> radix sort (key, point) -> cells
//              = runs of equal keys in key order -> one warp per cell sums its members in a fixed order.
// knn        : the points' bounding box (one read-back) sets a uniform grid; keys radix-sorted, cell starts by binary
//              search; one thread per point, in cell order, visits the cells ring by ring (Chebyshev distance r around
//              its own) and keeps the k smallest (d^2, j) pairs until no unvisited cell can hold a closer point.
// outliers   : one thread per point takes its mean neighbour distance, one block reduces mean and deviation in a fixed
//              order, a scan of the keep flags compacts the points.
// normals    : one thread per point, covariance in double and the simplification's Jacobi eigensolve.
// This file is compiled with -fmad=false: its double arithmetic rounds operation by operation as numpy's does, so the
// squared distances and with them the neighbour lists and their order are those of the restatement. No float atomics:
// two calls are bitwise equal.
#include "common.cuh"
#include "../../include/ngp_b200.h"
#include "cluster.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define PT_THREADS 256
#define PT_MAX_ITEMS ((int64_t)1 << 31)
#define PT_STATS_THREADS 1024

static size_t pt_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int pt_grid(int64_t items) {
    const int64_t want = (items + PT_THREADS - 1) / PT_THREADS, cap = (int64_t)ngp_sm_count() * 16;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

static int pt_bits(uint64_t x) {  // bits that hold 0..x, at least 1
    int b = 1;
    while (b < 64 && (x >> b)) ++b;
    return b;
}

// ---- 1. ray selection ---------------------------------------------------------------------------------------------
__global__ void k_pt_index(int64_t N, int64_t n_pix, uint64_t g, int64_t k0, int n, int64_t* __restrict__ img,
                           int64_t* __restrict__ pix) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned __int128 prod = (unsigned __int128)(uint64_t)(k0 + i) * g;
        const int64_t q = (int64_t)(prod % (unsigned __int128)(uint64_t)N);
        img[i] = q / n_pix;
        pix[i] = q % n_pix;
    }
}

extern "C" int ngp_points_rays(int64_t n_views, int64_t n_pix, int64_t g, int64_t k0, int n, const float* poses,
                               const float* directions, int64_t* img_idx, int64_t* pix_idx, float* rays_o, float* rays_d,
                               void* stream) {
    if (n_views < 1 || n_pix < 1 || n_views > INT64_MAX / n_pix || n < 0 || k0 < 0 || !img_idx || !pix_idx || !poses ||
        !directions || !rays_o || !rays_d)
        return NGP_EINVAL;
    const int64_t N = n_views * n_pix;
    if (g < 1 || (N > 1 && g >= N) || k0 + n > N) return NGP_EINVAL;
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    k_pt_index<<<pt_grid(n), PT_THREADS, 0, st>>>(N, n_pix, (uint64_t)g, k0, n, img_idx, pix_idx);
    NGP_CHECK_LAUNCH();
    return ngp_gen_rays(img_idx, pix_idx, poses, directions, nullptr, n_pix, n, rays_o, rays_d, nullptr, stream);
}

// ---- 3. back-projection ---------------------------------------------------------------------------------------------
struct PtRay {
    float p[3], v[3];
    uint8_t c[3];
    bool keep;
};

__device__ __forceinline__ PtRay pt_ray(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ op,
                                        const float* __restrict__ depth, const float* __restrict__ rgb, int64_t i,
                                        float min_opacity, const float (&lo)[3], const float (&hi)[3]) {
    PtRay r;
    const float a = op[i], t = __fdiv_rn(depth[i], a);
    r.keep = a >= min_opacity;
    float dd[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        dd[k] = d[3 * i + k];
        r.p[k] = fmaf(dd[k], t, o[3 * i + k]);
        r.keep = r.keep && isfinite(r.p[k]) && r.p[k] >= lo[k] && r.p[k] <= hi[k];
        r.c[k] = (uint8_t)rintf(__fmul_rn(255.f, fminf(__fdiv_rn(rgb[3 * i + k], a), 1.f)));
    }
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dd[0], dd[0]), __fmul_rn(dd[1], dd[1])), __fmul_rn(dd[2], dd[2])));
#pragma unroll
    for (int k = 0; k < 3; ++k) r.v[k] = __fdiv_rn(dd[k], len);
    return r;
}

struct PtBox {
    float lo[3], hi[3];
};

__global__ void k_pt_flags(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ op,
                           const float* __restrict__ depth, const float* __restrict__ rgb, int64_t n, float min_opacity,
                           const PtBox box, int32_t* __restrict__ flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = i < n && pt_ray(o, d, op, depth, rgb, i, min_opacity, box.lo, box.hi).keep;
}

__global__ void k_pt_emit(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ op,
                          const float* __restrict__ depth, const float* __restrict__ rgb, int64_t n, float min_opacity,
                          const PtBox box, const int32_t* __restrict__ pos, float* __restrict__ points,
                          uint8_t* __restrict__ colors, float* __restrict__ views) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t at = pos[i];
        if (pos[i + 1] == at) continue;
        const PtRay r = pt_ray(o, d, op, depth, rgb, i, min_opacity, box.lo, box.hi);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            points[3 * at + k] = r.p[k];
            colors[3 * at + k] = r.c[k];
            views[3 * at + k] = r.v[k];
        }
    }
}

// workspace of the scans (backproject, outliers): flags / positions (n + 1 int32) | per-point double (n) | stats
// (4 double) | cub temp
struct PtScanWs {
    int32_t* pos;
    double* val;
    double* stats;
    void* temp;
    size_t temp_bytes, total;
};

static PtScanWs pt_scan_ws(int64_t n, void* base) {
    PtScanWs w;
    size_t t = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, n + 1);
    w.temp_bytes = pt_align(t);
    char* p = (char*)base;
    size_t off = 0;
    w.pos = (int32_t*)(p + off); off += pt_align((n + 1) * 4);
    w.val = (double*)(p + off); off += pt_align(n * 8);
    w.stats = (double*)(p + off); off += 256;
    w.temp = p + off; off += w.temp_bytes;
    w.total = off;
    return w;
}

// ---- 4. voxel downsampling ----------------------------------------------------------------------------------------
// workspace: header (int64 cells) | keys x2 (n uint64) | ids x2 (n int32) | heads / scan (n int32) | cell starts (n + 1
// int32) | cub temp
struct PtVoxWs {
    int64_t* hdr;
    uint64_t* key[2];
    int32_t* val[2];
    int32_t* scan;
    int32_t* cseg;
    void* temp;
    size_t temp_bytes, total;
};

static PtVoxWs pt_vox_ws(int64_t n, void* base) {
    PtVoxWs w;
    size_t tb = 0, t;
    cub::DoubleBuffer<uint64_t> k64(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v32(nullptr, nullptr);
    t = 0; cub::DeviceRadixSort::SortPairs(nullptr, t, k64, v32, n, 0, 64); tb = t > tb ? t : tb;
    t = 0; cub::DeviceScan::InclusiveSum(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, n); tb = t > tb ? t : tb;
    w.temp_bytes = pt_align(tb);
    char* p = (char*)base;
    size_t off = 0;
    w.hdr = (int64_t*)(p + off); off += 256;
    for (int i = 0; i < 2; ++i) { w.key[i] = (uint64_t*)(p + off); off += pt_align(n * 8); }
    for (int i = 0; i < 2; ++i) { w.val[i] = (int32_t*)(p + off); off += pt_align(n * 4); }
    w.scan = (int32_t*)(p + off); off += pt_align(n * 4);
    w.cseg = (int32_t*)(p + off); off += pt_align((n + 1) * 4);
    w.temp = p + off; off += w.temp_bytes;
    w.total = off;
    return w;
}

__global__ void k_pt_vkey(const float* __restrict__ pts, int64_t n, const NgpClusterGrid g, uint64_t* __restrict__ key,
                          int32_t* __restrict__ val) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        key[i] = ms_key(pts + 3 * i, g);
        val[i] = (int32_t)i;
    }
}

__global__ void k_pt_heads(const uint64_t* __restrict__ key, int64_t n, int32_t* __restrict__ head) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        head[i] = i == 0 || key[i] != key[i - 1];
}

// scan: inclusive scan of the heads (cell number + 1 at each sorted position)
__global__ void k_pt_cells(const uint64_t* __restrict__ key, const int32_t* __restrict__ scan, int64_t n,
                           int32_t* __restrict__ cseg, int64_t* __restrict__ hdr) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t c = scan[i] - 1;
        if (i == 0 || key[i] != key[i - 1]) cseg[c] = (int32_t)i;
        if (i == n - 1) {
            cseg[c + 1] = (int32_t)n;
            hdr[0] = c + 1;
        }
    }
}

// one warp per cell: the double mean of its positions, the normalised double sum of its views, floor(mean + 1/2) of
// its colours from integer sums
__global__ void k_pt_vemit(const float* __restrict__ pts, const uint8_t* __restrict__ col, const float* __restrict__ view,
                           const uint64_t* __restrict__ key, const int32_t* __restrict__ perm, const int32_t* __restrict__ cseg,
                           const int64_t* __restrict__ hdr, float* __restrict__ out_p, uint8_t* __restrict__ out_c,
                           float* __restrict__ out_v, int64_t* __restrict__ out_key, int32_t* __restrict__ out_n) {
    const int lane = threadIdx.x & 31;
    const int64_t C = hdr[0], warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; c < C; c += warps) {
        const int64_t s0 = cseg[c], s1 = cseg[c + 1];
        double sp[3] = {0.0, 0.0, 0.0}, sv[3] = {0.0, 0.0, 0.0};
        unsigned long long sc[3] = {0, 0, 0};
        for (int64_t i = s0 + lane; i < s1; i += 32) {
            const int64_t j = perm[i];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                sp[a] += (double)__ldg(pts + 3 * j + a);
                sv[a] += (double)__ldg(view + 3 * j + a);
                sc[a] += __ldg(col + 3 * j + a);
            }
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            sp[a] = ms_wsum(sp[a]);
            sv[a] = ms_wsum(sv[a]);
            for (int o = 16; o > 0; o >>= 1) sc[a] += __shfl_down_sync(0xffffffffu, sc[a], o);
        }
        if (lane != 0) continue;
        const int64_t m = s1 - s0;
        const double len = sqrt(sv[0] * sv[0] + sv[1] * sv[1] + sv[2] * sv[2]);
        for (int a = 0; a < 3; ++a) {
            out_p[3 * c + a] = (float)(sp[a] / (double)m);
            out_v[3 * c + a] = len > 0.0 ? (float)(sv[a] / len) : 0.f;
            out_c[3 * c + a] = (uint8_t)((2 * sc[a] + (unsigned long long)m) / (2 * (unsigned long long)m));
        }
        if (out_key) out_key[c] = (int64_t)key[s0];
        if (out_n) out_n[c] = (int32_t)m;
    }
}

static bool pt_n_ok(int64_t n) { return n >= 0 && n < PT_MAX_ITEMS; }

// ---- 5. k nearest neighbours ----------------------------------------------------------------------------------------
struct PtKnnGrid {
    double lo[3], h;
    int32_t n[3];
};

// cells of the search grid: at most about 2 per point, and never more than NGP_POINTS_KNN_MAX_CELLS
static int64_t pt_knn_cells(int64_t n) {
    const int64_t c = 2 * n;
    return c < 1 ? 1 : (c > NGP_POINTS_KNN_MAX_CELLS ? NGP_POINTS_KNN_MAX_CELLS : c);
}

// workspace: header (6 float box + bad flag) | block partials | keys x2 (n uint32) | ids x2 (n int32) | cell starts
// (cells + 1 int32) | cub temp
#define PT_BOX_BLOCKS 256
struct PtKnnWs {
    float* box;
    float* part;
    uint32_t* key[2];
    int32_t* val[2];
    int32_t* start;
    void* temp;
    size_t temp_bytes, total;
};

static PtKnnWs pt_knn_ws(int64_t n, void* base) {
    PtKnnWs w;
    size_t t = 0;
    cub::DoubleBuffer<uint32_t> k32(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v32(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, t, k32, v32, n, 0, 32);
    w.temp_bytes = pt_align(t);
    const int64_t cells = pt_knn_cells(n);
    char* p = (char*)base;
    size_t off = 0;
    w.box = (float*)(p + off); off += 256;
    w.part = (float*)(p + off); off += pt_align(PT_BOX_BLOCKS * 7 * 4);
    for (int i = 0; i < 2; ++i) { w.key[i] = (uint32_t*)(p + off); off += pt_align(n * 4); }
    for (int i = 0; i < 2; ++i) { w.val[i] = (int32_t*)(p + off); off += pt_align(n * 4); }
    w.start = (int32_t*)(p + off); off += pt_align((cells + 1) * 4);
    w.temp = p + off; off += w.temp_bytes;
    w.total = off;
    return w;
}

// the box of the points: block partials (min x y z, max x y z, non-finite count) in a fixed order, then one block
__global__ void k_pt_box_part(const float* __restrict__ pts, int64_t n, float* __restrict__ part) {
    __shared__ float s[7][PT_THREADS];
    float v[7] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY, 0.f};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        for (int a = 0; a < 3; ++a) {
            const float x = pts[3 * i + a];
            if (!isfinite(x)) v[6] = 1.f;
            v[a] = fminf(v[a], x);
            v[3 + a] = fmaxf(v[3 + a], x);
        }
    for (int k = 0; k < 7; ++k) s[k][threadIdx.x] = v[k];
    __syncthreads();
    for (int o = PT_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o)
            for (int k = 0; k < 7; ++k) {
                const float a = s[k][threadIdx.x], b = s[k][threadIdx.x + o];
                s[k][threadIdx.x] = k < 3 ? fminf(a, b) : fmaxf(a, b);
            }
        __syncthreads();
    }
    if (threadIdx.x < 7) part[blockIdx.x * 7 + threadIdx.x] = s[threadIdx.x][0];
}

__global__ void k_pt_box(const float* __restrict__ part, int blocks, float* __restrict__ box) {
    const int k = threadIdx.x;
    if (k >= 7) return;
    float v = part[k];
    for (int b = 1; b < blocks; ++b) v = k < 3 ? fminf(v, part[7 * b + k]) : fmaxf(v, part[7 * b + k]);
    box[k] = v;
}

__device__ __forceinline__ int pt_kcell(float x, double lo, double h, int n) {
    const double q = floor(((double)x - lo) / h);
    return q < 0.0 ? 0 : (q > (double)(n - 1) ? n - 1 : (int)q);
}

__global__ void k_pt_kkey(const float* __restrict__ pts, int64_t n, const PtKnnGrid g, uint32_t* __restrict__ key,
                          int32_t* __restrict__ val) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = pt_kcell(pts[3 * i], g.lo[0], g.h, g.n[0]);
        const int c1 = pt_kcell(pts[3 * i + 1], g.lo[1], g.h, g.n[1]);
        const int c2 = pt_kcell(pts[3 * i + 2], g.lo[2], g.h, g.n[2]);
        key[i] = ((uint32_t)c0 * g.n[1] + c1) * g.n[2] + c2;
        val[i] = (int32_t)i;
    }
}

// start[c] = the first sorted position with a key >= c, c = 0 .. cells
__global__ void k_pt_starts(const uint32_t* __restrict__ key, int64_t n, int64_t cells, int32_t* __restrict__ start) {
    for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c <= cells; c += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = n;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (key[mid] < (uint32_t)c) lo = mid + 1;
            else hi = mid;
        }
        start[c] = (int32_t)lo;
    }
}

// (d, j) < (d', j'): distance first, then index
__device__ __forceinline__ bool pt_less(double d, int32_t j, double d2, int32_t j2) { return d < d2 || (d == d2 && j < j2); }

// offer the points of one cell to the sorted list (bd, bj) of the k smallest (d^2, j) pairs of point i so far
__device__ __forceinline__ void pt_visit(const float* __restrict__ pts, const int32_t* __restrict__ order,
                                         const int32_t* __restrict__ start, uint32_t cell, int32_t i, double x, double y,
                                         double z, int k, int& cnt, double* bd, int32_t* bj) {
    const int32_t s0 = start[cell], s1 = start[cell + 1];
    for (int32_t s = s0; s < s1; ++s) {
        const int32_t j = order[s];
        if (j == i) continue;
        const double ex = (double)pts[3 * j] - x, ey = (double)pts[3 * j + 1] - y, ez = (double)pts[3 * j + 2] - z;
        const double d = ex * ex + ey * ey + ez * ez;
        if (cnt == k && !pt_less(d, j, bd[k - 1], bj[k - 1])) continue;
        int p = cnt < k ? cnt++ : k - 1;
        while (p > 0 && pt_less(d, j, bd[p - 1], bj[p - 1])) {
            bd[p] = bd[p - 1];
            bj[p] = bj[p - 1];
            --p;
        }
        bd[p] = d;
        bj[p] = j;
    }
}

// one thread per point, the points taken in cell order so that a warp's points share their cells
__global__ void __launch_bounds__(PT_THREADS) k_pt_knn(const float* __restrict__ pts, int64_t n, int k, const PtKnnGrid g,
                                                       const int32_t* __restrict__ order, const int32_t* __restrict__ start,
                                                       int32_t* __restrict__ out_idx, double* __restrict__ out_d2) {
    double bd[NGP_POINTS_MAX_K];
    int32_t bj[NGP_POINTS_MAX_K];
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int32_t i = order[t];
        const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
        const int c[3] = {pt_kcell(pts[3 * i], g.lo[0], g.h, g.n[0]), pt_kcell(pts[3 * i + 1], g.lo[1], g.h, g.n[1]),
                          pt_kcell(pts[3 * i + 2], g.lo[2], g.h, g.n[2])};
        int rmax = 0;
        for (int a = 0; a < 3; ++a) rmax = max(rmax, max(c[a], g.n[a] - 1 - c[a]));
        int cnt = 0;
        for (int r = 0; r <= rmax; ++r) {
            // the cells at Chebyshev distance r inside the grid: whole z columns where |dx| or |dy| is r, else dz = +-r
            const int x0 = max(-r, -c[0]), x1 = min(r, g.n[0] - 1 - c[0]);
            const int y0 = max(-r, -c[1]), y1 = min(r, g.n[1] - 1 - c[1]);
            const int z0 = max(-r, -c[2]), z1 = min(r, g.n[2] - 1 - c[2]);
            for (int dx = x0; dx <= x1; ++dx)
                for (int dy = y0; dy <= y1; ++dy) {
                    const uint32_t col = ((uint32_t)(c[0] + dx) * g.n[1] + (c[1] + dy)) * g.n[2] + c[2];
                    if (dx == -r || dx == r || dy == -r || dy == r) {
                        for (int dz = z0; dz <= z1; ++dz) pt_visit(pts, order, start, col + dz, i, x, y, z, k, cnt, bd, bj);
                    } else {
                        if (z0 == -r) pt_visit(pts, order, start, col - r, i, x, y, z, k, cnt, bd, bj);
                        if (z1 == r) pt_visit(pts, order, start, col + r, i, x, y, z, k, cnt, bd, bj);
                    }
                }
            // every unvisited point lies in a cell at Chebyshev distance > r: at least r h away on some axis (less a
            // margin for the rounding of the cell coordinates)
            const double lb = (double)r * g.h * (1.0 - 1.0 / (1 << 20));
            if (cnt == k && bd[k - 1] < lb * lb) break;
        }
        for (int q = 0; q < k; ++q) {
            out_idx[(int64_t)i * k + q] = bj[q];
            out_d2[(int64_t)i * k + q] = bd[q];
        }
    }
}

// ---- 6. statistical outlier removal ----------------------------------------------------------------------------------
__global__ void k_pt_meand(const double* __restrict__ d2, int64_t n, int k, double* __restrict__ md) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int q = 0; q < k; ++q) s += sqrt(d2[i * k + q]);
        md[i] = s / (double)k;
    }
}

__device__ double pt_block_sum(double v, double* sh) {  // fixed tree over PT_STATS_THREADS threads; every thread gets it
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = PT_STATS_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    const double s = sh[0];
    __syncthreads();
    return s;
}

// one block: stats = {mean, population standard deviation, threshold}
__global__ void __launch_bounds__(PT_STATS_THREADS) k_pt_stats(const double* __restrict__ md, int64_t n, double std_ratio,
                                                                 double* __restrict__ stats) {
    __shared__ double sh[PT_STATS_THREADS];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += PT_STATS_THREADS) s += md[i];
    const double mu = pt_block_sum(s, sh) / (double)n;
    s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += PT_STATS_THREADS) s += (md[i] - mu) * (md[i] - mu);
    const double sigma = sqrt(pt_block_sum(s, sh) / (double)n);
    if (threadIdx.x == 0) {
        stats[0] = mu;
        stats[1] = sigma;
        stats[2] = mu + std_ratio * sigma;
    }
}

__global__ void k_pt_keep(const double* __restrict__ md, int64_t n, const double* __restrict__ stats, int32_t* __restrict__ flag) {
    const double thr = stats[2];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = i < n && md[i] <= thr;
}

__global__ void k_pt_compact(const float* __restrict__ pts, const uint8_t* __restrict__ col, const float* __restrict__ view,
                             int64_t n, const int32_t* __restrict__ pos, float* __restrict__ out_p, uint8_t* __restrict__ out_c,
                             float* __restrict__ out_v, int32_t* __restrict__ kept) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t at = pos[i];
        if (pos[i + 1] == at) continue;
        for (int a = 0; a < 3; ++a) {
            out_p[3 * at + a] = pts[3 * i + a];
            out_c[3 * at + a] = col[3 * i + a];
            out_v[3 * at + a] = view[3 * i + a];
        }
        if (kept) kept[at] = (int32_t)i;
    }
}

// ---- 7. normals -----------------------------------------------------------------------------------------------------
__global__ void k_pt_normals(const float* __restrict__ pts, const float* __restrict__ view, int64_t n, int k,
                             const int32_t* __restrict__ idx, float* __restrict__ nrm) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double m[3];
        for (int a = 0; a < 3; ++a) m[a] = (double)pts[3 * i + a];
        for (int q = 0; q < k; ++q) {
            const int64_t j = idx[i * k + q];
            for (int a = 0; a < 3; ++a) m[a] += (double)pts[3 * j + a];
        }
        for (int a = 0; a < 3; ++a) m[a] /= (double)(k + 1);
        double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, E[3][3];
        for (int q = -1; q < k; ++q) {
            const int64_t j = q < 0 ? i : idx[i * k + q];
            const double e[3] = {(double)pts[3 * j] - m[0], (double)pts[3 * j + 1] - m[1], (double)pts[3 * j + 2] - m[2]};
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) A[a][b] += e[a] * e[b];
        }
        bool zero = true;
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) zero = zero && A[a][b] == 0.0;
        if (zero) {
            for (int a = 0; a < 3; ++a) nrm[3 * i + a] = 0.f;
            continue;
        }
        ms_jacobi(A, E);
        int s = 0;
        for (int a = 1; a < 3; ++a)
            if (A[a][a] < A[s][s]) s = a;
        const double dot = E[0][s] * (double)view[3 * i] + E[1][s] * (double)view[3 * i + 1] + E[2][s] * (double)view[3 * i + 2];
        const double sg = dot > 0.0 ? -1.0 : 1.0;
        for (int a = 0; a < 3; ++a) nrm[3 * i + a] = (float)(sg * E[a][s]);
    }
}

// ---- entry points ---------------------------------------------------------------------------------------------------
extern "C" size_t ngp_points_workspace(int64_t n) {
    if (!pt_n_ok(n)) return 0;
    size_t a = pt_scan_ws(n, nullptr).total, b = pt_vox_ws(n, nullptr).total, c = pt_knn_ws(n, nullptr).total;
    a = a > b ? a : b;
    return a > c ? a : c;
}

#define PT_WS_CHECK(w)                                                \
    do {                                                              \
        if (!workspace || workspace_bytes < (w).total) return NGP_EINVAL; \
    } while (0)

extern "C" int ngp_points_backproject(const float* rays_o, const float* rays_d, const float* opacity, const float* depth,
                                      const float* rgb, int64_t n, float min_opacity, const float* bounds, float* points,
                                      uint8_t* colors, float* views, int64_t* count, void* workspace, size_t workspace_bytes,
                                      void* stream) {
    if (!pt_n_ok(n) || !count || !bounds || !(min_opacity > 0.f && min_opacity <= 1.f)) return NGP_EINVAL;
    if (n > 0 && (!rays_o || !rays_d || !opacity || !depth || !rgb || !points || !colors || !views)) return NGP_EINVAL;
    const PtScanWs w = pt_scan_ws(n, workspace);
    PT_WS_CHECK(w);
    PtBox box;
    for (int a = 0; a < 3; ++a) {
        box.lo[a] = bounds[a];
        box.hi[a] = bounds[3 + a];
        if (!(box.lo[a] <= box.hi[a])) return NGP_EINVAL;
    }
    *count = 0;
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    k_pt_flags<<<pt_grid(n + 1), PT_THREADS, 0, st>>>(rays_o, rays_d, opacity, depth, rgb, n, min_opacity, box, w.pos);
    NGP_CHECK_LAUNCH();
    size_t tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.pos, w.pos, n + 1, st));
    NGP_COUNT_LAUNCHES(2);
    k_pt_emit<<<pt_grid(n), PT_THREADS, 0, st>>>(rays_o, rays_d, opacity, depth, rgb, n, min_opacity, box, w.pos, points,
                                                 colors, views);
    NGP_CHECK_LAUNCH();
    int32_t m;
    NGP_CUDA(cudaMemcpyAsync(&m, w.pos + n, sizeof(m), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    *count = m;
    return 0;
}

extern "C" int ngp_points_voxel(const float* points, const uint8_t* colors, const float* views, int64_t n,
                                const NgpClusterGrid* grid, float* out_points, uint8_t* out_colors, float* out_views,
                                int64_t* out_keys, int32_t* out_counts, int64_t* count, void* workspace,
                                size_t workspace_bytes, void* stream) {
    if (!pt_n_ok(n) || !count || !grid || !(grid->h > 0.f) || !isfinite(grid->h)) return NGP_EINVAL;
    for (int a = 0; a < 3; ++a)
        if (grid->n[a] < 1 || grid->n[a] > NGP_SIMPLIFY_MAX_GRID || !isfinite(grid->lo[a])) return NGP_EINVAL;
    if (n > 0 && (!points || !colors || !views || !out_points || !out_colors || !out_views)) return NGP_EINVAL;
    const PtVoxWs w = pt_vox_ws(n, workspace);
    PT_WS_CHECK(w);
    *count = 0;
    if (n == 0) return 0;
    const NgpClusterGrid g = *grid;
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(cudaMemsetAsync(w.hdr, 0, 256, st));
    k_pt_vkey<<<pt_grid(n), PT_THREADS, 0, st>>>(points, n, g, w.key[0], w.val[0]);
    NGP_CHECK_LAUNCH();
    cub::DoubleBuffer<uint64_t> vk(w.key[0], w.key[1]);
    cub::DoubleBuffer<int32_t> vv(w.val[0], w.val[1]);
    size_t tb = w.temp_bytes;
    const int kbits = pt_bits((uint64_t)g.n[0] * g.n[1] * g.n[2] - 1);
    NGP_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, vk, vv, n, 0, kbits, st));
    k_pt_heads<<<pt_grid(n), PT_THREADS, 0, st>>>(vk.Current(), n, w.scan);
    NGP_CHECK_LAUNCH();
    tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::InclusiveSum(w.temp, tb, w.scan, w.scan, n, st));
    NGP_COUNT_LAUNCHES(2);
    k_pt_cells<<<pt_grid(n), PT_THREADS, 0, st>>>(vk.Current(), w.scan, n, w.cseg, w.hdr);
    NGP_CHECK_LAUNCH();
    k_pt_vemit<<<pt_grid(32 * n), PT_THREADS, 0, st>>>(points, colors, views, vk.Current(), vv.Current(), w.cseg, w.hdr,
                                                       out_points, out_colors, out_views, out_keys, out_counts);
    NGP_CHECK_LAUNCH();
    int64_t h;
    NGP_CUDA(cudaMemcpyAsync(&h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    *count = h;
    return 0;
}

extern "C" int ngp_points_knn(const float* points, int64_t n, int k, int32_t* idx, double* dist2, void* workspace,
                              size_t workspace_bytes, void* stream) {
    if (!pt_n_ok(n) || k < 1 || k > NGP_POINTS_MAX_K || k > n - 1 || !points || !idx || !dist2) return NGP_EINVAL;
    const PtKnnWs w = pt_knn_ws(n, workspace);
    PT_WS_CHECK(w);
    cudaStream_t st = (cudaStream_t)stream;
    const int blocks = (int)(n < (int64_t)PT_BOX_BLOCKS * PT_THREADS ? (n + PT_THREADS - 1) / PT_THREADS : PT_BOX_BLOCKS);
    k_pt_box_part<<<blocks, PT_THREADS, 0, st>>>(points, n, w.part);
    NGP_CHECK_LAUNCH();
    k_pt_box<<<1, 32, 0, st>>>(w.part, blocks, w.box);
    NGP_CHECK_LAUNCH();
    float box[7];
    NGP_CUDA(cudaMemcpyAsync(box, w.box, sizeof(box), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    if (box[6] != 0.f) return NGP_EINVAL;  // a coordinate that is not finite
    // cubes of side h = (largest extent) / G, G = floor(cbrt(cells)); an axis without extent has one cell
    const int64_t cells_max = pt_knn_cells(n);
    int64_t G = 1;
    while ((G + 1) * (G + 1) * (G + 1) <= cells_max) ++G;
    PtKnnGrid g;
    double ext = 0.0;
    for (int a = 0; a < 3; ++a) ext = fmax(ext, (double)box[3 + a] - (double)box[a]);
    g.h = ext > 0.0 ? ext / (double)G : 1.0;
    for (int a = 0; a < 3; ++a) {
        g.lo[a] = box[a];
        const double c = ceil(((double)box[3 + a] - (double)box[a]) / g.h);
        g.n[a] = (int32_t)(c < 1.0 ? 1.0 : (c > (double)G ? (double)G : c));
    }
    const int64_t cells = (int64_t)g.n[0] * g.n[1] * g.n[2];
    k_pt_kkey<<<pt_grid(n), PT_THREADS, 0, st>>>(points, n, g, w.key[0], w.val[0]);
    NGP_CHECK_LAUNCH();
    cub::DoubleBuffer<uint32_t> kk(w.key[0], w.key[1]);
    cub::DoubleBuffer<int32_t> kv(w.val[0], w.val[1]);
    size_t tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, kk, kv, n, 0, pt_bits((uint64_t)cells - 1), st));
    k_pt_starts<<<pt_grid(cells + 1), PT_THREADS, 0, st>>>(kk.Current(), n, cells, w.start);
    NGP_CHECK_LAUNCH();
    k_pt_knn<<<pt_grid(n), PT_THREADS, 0, st>>>(points, n, k, g, kv.Current(), w.start, idx, dist2);
    NGP_CHECK_LAUNCH();
    return 0;
}

extern "C" int ngp_points_outliers(const float* points, const uint8_t* colors, const float* views, int64_t n, int k,
                                   const double* dist2, double std_ratio, float* out_points, uint8_t* out_colors,
                                   float* out_views, int32_t* kept, double* stats, int64_t* count, void* workspace,
                                   size_t workspace_bytes, void* stream) {
    if (!pt_n_ok(n) || n < 2 || k < 1 || k > NGP_POINTS_MAX_K || k > n - 1 || !(std_ratio >= 0.0) || !isfinite(std_ratio) ||
        !points || !colors || !views || !dist2 || !out_points || !out_colors || !out_views || !count)
        return NGP_EINVAL;
    const PtScanWs w = pt_scan_ws(n, workspace);
    PT_WS_CHECK(w);
    cudaStream_t st = (cudaStream_t)stream;
    k_pt_meand<<<pt_grid(n), PT_THREADS, 0, st>>>(dist2, n, k, w.val);
    NGP_CHECK_LAUNCH();
    k_pt_stats<<<1, PT_STATS_THREADS, 0, st>>>(w.val, n, std_ratio, w.stats);
    NGP_CHECK_LAUNCH();
    k_pt_keep<<<pt_grid(n + 1), PT_THREADS, 0, st>>>(w.val, n, w.stats, w.pos);
    NGP_CHECK_LAUNCH();
    size_t tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.pos, w.pos, n + 1, st));
    NGP_COUNT_LAUNCHES(2);
    k_pt_compact<<<pt_grid(n), PT_THREADS, 0, st>>>(points, colors, views, n, w.pos, out_points, out_colors, out_views, kept);
    NGP_CHECK_LAUNCH();
    int32_t m;
    double s[3];
    NGP_CUDA(cudaMemcpyAsync(&m, w.pos + n, sizeof(m), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaMemcpyAsync(s, w.stats, sizeof(s), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    *count = m;
    if (stats)
        for (int q = 0; q < 3; ++q) stats[q] = s[q];
    return 0;
}

extern "C" int ngp_points_normals(const float* points, const float* views, int64_t n, int k, const int32_t* idx,
                                  float* normals, void* stream) {
    if (!pt_n_ok(n) || k < 0 || k > NGP_POINTS_MAX_K || (n > 0 && k > n - 1) || (n > 0 && (!points || !views || !normals)) ||
        (n > 0 && k > 0 && !idx))
        return NGP_EINVAL;
    if (n == 0) return 0;
    k_pt_normals<<<pt_grid(n), PT_THREADS, 0, (cudaStream_t)stream>>>(points, views, n, k, idx, normals);
    NGP_CHECK_LAUNCH();
    return 0;
}
