// Texture baking of a mesh (include/ngp_b200.h, "Texture baking"; numpy restatement: oracle/mesh_texture.py).
//
// atlas : one thread per triangle finds its longest edge and class (a device max of the exponents, a 64-bin integer
//         histogram), the host picks S from the histogram, a stable radix sort orders the squares by size, a scan of
//         their areas gives the Morton offsets, and one thread per triangle places its uv. Then one thread per atlas
//         texel (Morton index m) finds its square by binary search over the offsets and runs the band test; a scan of
//         the flags numbers the band texels in ascending m.
// texels: one thread per atlas texel writes the band texel's entry of the texel map: closest point, point, normal.
// bake  : per chunk of texels, one thread per sample writes the rays and sample distances, ngp_net_forward evaluates
//         the samples in ray mode, one thread per texel composites in double and writes the texel.
// This file is compiled with -fmad=false: its double arithmetic rounds operation by operation as numpy's does, so
// classes, squares, uv and the band decisions are those of the restatement. fmaf is written out where the rule has it.
// No float atomics: two calls are bitwise equal.
#include "common.cuh"
#include "../../include/ngp_b200.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define TX_THREADS 256
#define TX_MAX_ITEMS ((int64_t)1 << 31)
#define TX_EBIAS 2048  // exponents are stored biased, so that 0 means "no triangle with a length"

static size_t tx_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int tx_grid(int64_t items) {
    const int64_t want = (items + TX_THREADS - 1) / TX_THREADS, cap = (int64_t)ngp_sm_count() * 16;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

static bool tx_size_ok(int W) {
    return W >= NGP_TEXTURE_MIN_SIZE && W <= NGP_TEXTURE_MAX_SIZE && (W & (W - 1)) == 0;
}

static bool tx_sizes_ok(int64_t V, int64_t F, int W) {
    return V >= 0 && F >= 0 && V < TX_MAX_ITEMS && F < TX_MAX_ITEMS && tx_size_ok(W) &&
           F * NGP_TEXTURE_MIN_SQUARE * NGP_TEXTURE_MIN_SQUARE <= (int64_t)W * W;
}

// workspace: header (int64 bad flag, int32 biased top exponent, 64-bin histogram) | e (F int32) | rot (F int32) |
// sort keys x2 (F uint32) | ids x2 (F int32) | offsets (F + 1 int64) | band flags / scan (W^2 + 1 int32) | cub temp
struct TxWs {
    int64_t* hdr;
    int* etop;
    unsigned long long* hist;
    int32_t* e;
    int32_t* rot;
    uint32_t* key[2];
    int32_t* val[2];
    int64_t* off;
    int32_t* scan;
    void* temp;
    size_t temp_bytes;
    size_t total;
};

static TxWs tx_ws(int64_t F, int W, void* base) {
    TxWs w;
    const int64_t A = (int64_t)W * W;
    size_t tb = 0, t;
    t = 0; cub::DeviceRadixSort::SortPairs(nullptr, t, (uint32_t*)nullptr, (uint32_t*)nullptr, (int32_t*)nullptr,
                                           (int32_t*)nullptr, F, 0, 4); tb = t > tb ? t : tb;
    t = 0; cub::DeviceScan::ExclusiveSum(nullptr, t, (int64_t*)nullptr, (int64_t*)nullptr, F + 1); tb = t > tb ? t : tb;
    t = 0; cub::DeviceScan::ExclusiveSum(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, A + 1); tb = t > tb ? t : tb;
    w.temp_bytes = tx_align(tb);
    char* p = (char*)base;
    size_t off = 0;
    w.hdr = (int64_t*)p; off += 1024;
    w.etop = (int*)(p + 8);
    w.hist = (unsigned long long*)(p + 16);
    w.e = (int32_t*)(p + off); off += tx_align(F * 4);
    w.rot = (int32_t*)(p + off); off += tx_align(F * 4);
    for (int i = 0; i < 2; ++i) { w.key[i] = (uint32_t*)(p + off); off += tx_align(F * 4); }
    for (int i = 0; i < 2; ++i) { w.val[i] = (int32_t*)(p + off); off += tx_align(F * 4); }
    w.off = (int64_t*)(p + off); off += tx_align((F + 1) * 8);
    w.scan = (int32_t*)(p + off); off += tx_align((A + 1) * 4);
    w.temp = p + off; off += w.temp_bytes;
    w.total = off;
    return w;
}

extern "C" size_t ngp_mesh_texture_workspace(int64_t n_vertices, int64_t n_triangles, int size) {
    if (!tx_sizes_ok(n_vertices, n_triangles, size)) return 0;
    return tx_ws(n_triangles, size, nullptr).total;
}

__device__ __forceinline__ uint32_t tx_compact(uint64_t m) {  // the even bits of m
    m &= 0x5555555555555555ull;
    m = (m | (m >> 1)) & 0x3333333333333333ull;
    m = (m | (m >> 2)) & 0x0f0f0f0f0f0f0f0full;
    m = (m | (m >> 4)) & 0x00ff00ff00ff00ffull;
    m = (m | (m >> 8)) & 0x0000ffff0000ffffull;
    m = (m | (m >> 16)) & 0x00000000ffffffffull;
    return (uint32_t)m;
}

__device__ __forceinline__ double tx_len(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

__device__ __forceinline__ void tx_load(const float* __restrict__ v, int64_t i, double (&p)[3]) {
    for (int a = 0; a < 3; ++a) p[a] = (double)__ldg(v + 3 * i + a);
}

// the triangle's vertex indices rotated by rot; false for an index outside [0, V)
__device__ __forceinline__ bool tx_tri(const int64_t* __restrict__ tris, int64_t t, int64_t V, int rot, int64_t (&idx)[3]) {
    bool ok = true;
    for (int k = 0; k < 3; ++k) {
        idx[k] = __ldg(tris + 3 * t + (rot + k) % 3);
        ok = ok && idx[k] >= 0 && idx[k] < V;
    }
    return ok;
}

__device__ __forceinline__ bool tx_valid(double l) { return l > 0.0 && isfinite(l); }

__global__ void k_tx_class(const float* __restrict__ verts, int64_t V, const int64_t* __restrict__ tris, int64_t F,
                           int32_t* __restrict__ e, int32_t* __restrict__ rot, int64_t* __restrict__ hdr, int* __restrict__ etop) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < F; t += (int64_t)gridDim.x * blockDim.x) {
        int64_t idx[3];
        if (!tx_tri(tris, t, V, 0, idx)) {
            hdr[0] = 1;  // every writer stores the same value
            e[t] = 0;
            rot[t] = 0;
            continue;
        }
        double a[3], b[3], c[3];
        tx_load(verts, idx[0], a);
        tx_load(verts, idx[1], b);
        tx_load(verts, idx[2], c);
        const double l0 = tx_len(b[0] - a[0], b[1] - a[1], b[2] - a[2]);
        const double l1 = tx_len(c[0] - b[0], c[1] - b[1], c[2] - b[2]);
        const double l2 = tx_len(a[0] - c[0], a[1] - c[1], a[2] - c[2]);
        const int r = (l0 >= l1 && l0 >= l2) ? 0 : (l1 >= l2 ? 1 : 2);
        const double l = r == 0 ? l0 : (r == 1 ? l1 : l2);
        int ex = 0;
        frexp(l, &ex);
        rot[t] = r;
        e[t] = tx_valid(l) ? ex + TX_EBIAS : 0;
        if (tx_valid(l)) atomicMax(etop, ex + TX_EBIAS);  // integer max: order-free
    }
}

__device__ __forceinline__ int tx_class(int32_t eb, int etop) {
    if (eb == 0) return 63;
    const int k = etop - eb;
    return k < 63 ? k : 63;
}

__host__ __device__ __forceinline__ int64_t tx_side(int k, int64_t S) {
    const int64_t s = k < 31 ? (S >> k) : 0;
    return s > NGP_TEXTURE_MIN_SQUARE ? s : NGP_TEXTURE_MIN_SQUARE;
}

__global__ void k_tx_hist(const int32_t* __restrict__ e, int64_t F, const int* __restrict__ etop,
                          unsigned long long* __restrict__ hist) {
    __shared__ unsigned long long h[64];
    for (int i = threadIdx.x; i < 64; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const int top = *etop;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < F; t += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(h + tx_class(e[t], top), 1ull);
    __syncthreads();
    for (int i = threadIdx.x; i < 64; i += blockDim.x)
        if (h[i]) atomicAdd(hist + i, h[i]);  // integer sums: order-free
}

// sort key: log2(max size) - log2(s), so ascending keys are descending sizes; the ids start as the triangle index
__global__ void k_tx_key(const int32_t* __restrict__ e, int64_t F, const int* __restrict__ etop, int64_t S,
                         uint32_t* __restrict__ key, int32_t* __restrict__ val) {
    const int top = *etop;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < F; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = tx_side(tx_class(e[t], top), S);
        key[t] = (uint32_t)(__clzll(s) - __clzll((int64_t)NGP_TEXTURE_MAX_SIZE));
        val[t] = (int32_t)t;
    }
}

__global__ void k_tx_area(const int32_t* __restrict__ e, const int32_t* __restrict__ order, int64_t F,
                          const int* __restrict__ etop, int64_t S, int64_t* __restrict__ area) {
    const int top = *etop;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= F; i += (int64_t)gridDim.x * blockDim.x) {
        if (i == F) {
            area[F] = 0;
            continue;
        }
        const int64_t s = tx_side(tx_class(e[order[i]], top), S);
        area[i] = s * s;
    }
}

// square and uv of the triangle at sorted position i (step 4 of the rule)
__global__ void k_tx_place(const float* __restrict__ verts, const int64_t* __restrict__ tris, int64_t F,
                           const int32_t* __restrict__ e, const int32_t* __restrict__ rot, const int32_t* __restrict__ order,
                           const int64_t* __restrict__ off, const int* __restrict__ etop, int64_t S, float* __restrict__ uv,
                           int32_t* __restrict__ squares) {
    const int top = *etop;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < F; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = order[i];
        const int32_t eb = e[t];
        const int64_t s = tx_side(tx_class(eb, top), S);
        const uint64_t o = (uint64_t)off[i];
        const int64_t x0 = tx_compact(o), y0 = tx_compact(o >> 1);
        squares[3 * t] = (int32_t)x0;
        squares[3 * t + 1] = (int32_t)y0;
        squares[3 * t + 2] = (int32_t)s;
        const int r = rot[t];
        const double ax = (double)(x0 + NGP_TEXTURE_MARGIN), ay = (double)(y0 + NGP_TEXTURE_MARGIN);
        double bx = ax, cx = ax, cy = ay;
        if (eb != 0) {
            int64_t idx[3];
            for (int k = 0; k < 3; ++k) idx[k] = __ldg(tris + 3 * t + (r + k) % 3);
            double A[3], B[3], C[3];
            tx_load(verts, idx[0], A);
            tx_load(verts, idx[1], B);
            tx_load(verts, idx[2], C);
            const double l = tx_len(B[0] - A[0], B[1] - A[1], B[2] - A[2]);
            const double rho = ldexp((double)(s - 2 * NGP_TEXTURE_MARGIN), -(eb - TX_EBIAS));
            double u[3], ca[3], q[3];
            for (int a = 0; a < 3; ++a) {
                u[a] = (B[a] - A[a]) / l;
                ca[a] = C[a] - A[a];
            }
            const double w = (ca[0] * u[0] + ca[1] * u[1]) + ca[2] * u[2];
            for (int a = 0; a < 3; ++a) q[a] = ca[a] - w * u[a];
            const double eta = tx_len(q[0], q[1], q[2]);
            bx = ax + rho * l;
            cx = ax + rho * w;
            cy = ay + rho * eta;
        }
        float* p = uv + 6 * t;
        p[2 * r] = (float)ax;
        p[2 * r + 1] = (float)ay;
        p[2 * ((r + 1) % 3)] = (float)bx;
        p[2 * ((r + 1) % 3) + 1] = (float)ay;
        p[2 * ((r + 2) % 3)] = (float)cx;
        p[2 * ((r + 2) % 3) + 1] = (float)cy;
    }
}

__device__ __forceinline__ int64_t tx_rank(const int64_t* __restrict__ off, int64_t F, int64_t m) {  // off[i] <= m < off[i+1]
    int64_t lo = 0, hi = F;  // off[0] = 0 <= m
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(off + mid) <= m) lo = mid;
        else hi = mid;
    }
    return lo;
}

// step 5's band test of texel (x, y) against the uv triangle p
__device__ bool tx_meets(const double (&px)[3], const double (&py)[3], double x, double y) {
    if (!(fmax(px[0], fmax(px[1], px[2])) > x - 0.5) || !(fmin(px[0], fmin(px[1], px[2])) < x + 1.5) ||
        !(fmax(py[0], fmax(py[1], py[2])) > y - 0.5) || !(fmin(py[0], fmin(py[1], py[2])) < y + 1.5))
        return false;
    const double cx = x + 0.5, cy = y + 0.5;
    for (int k = 0; k < 3; ++k) {
        const int k1 = k == 2 ? 0 : k + 1;
        const double nx = -(py[k1] - py[k]), ny = px[k1] - px[k];
        if (nx == 0.0 && ny == 0.0) continue;
        double lo = INFINITY, hi = -INFINITY;
        for (int j = 0; j < 3; ++j) {
            const double d = nx * px[j] + ny * py[j];
            lo = fmin(lo, d);
            hi = fmax(hi, d);
        }
        const double dc = nx * cx + ny * cy, rad = fabs(nx) + fabs(ny);
        if (hi <= dc - rad || lo >= dc + rad) return false;
    }
    return true;
}

__device__ __forceinline__ void tx_uv(const float* __restrict__ uv, int64_t t, double (&px)[3], double (&py)[3]) {
    for (int k = 0; k < 3; ++k) {
        px[k] = (double)__ldg(uv + 6 * t + 2 * k);
        py[k] = (double)__ldg(uv + 6 * t + 2 * k + 1);
    }
}

// flag[m] for every atlas texel m < W^2: 1 when m lies in a square and passes its triangle's band test
__global__ void k_tx_band(const float* __restrict__ uv, const int32_t* __restrict__ order, const int64_t* __restrict__ off,
                          int64_t F, int64_t A, int32_t* __restrict__ flag) {
    const int64_t used = off[F];
    for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m <= A; m += (int64_t)gridDim.x * blockDim.x) {
        int32_t f = 0;
        if (m < used) {
            const int64_t t = order[tx_rank(off, F, m)];
            double px[3], py[3];
            tx_uv(uv, t, px, py);
            f = tx_meets(px, py, (double)tx_compact((uint64_t)m), (double)tx_compact((uint64_t)m >> 1));
        }
        flag[m] = f;
    }
}

extern "C" int ngp_mesh_texture_atlas(const float* vertices, int64_t n_vertices, const int64_t* triangles,
                                      int64_t n_triangles, int size, float* uv, int32_t* squares, int64_t* counts,
                                      void* workspace, size_t workspace_bytes, void* stream) {
    const int64_t V = n_vertices, F = n_triangles, A = (int64_t)size * size;
    if (!counts || !workspace || !tx_sizes_ok(V, F, size) || (F > 0 && (!vertices || !triangles || !uv || !squares)))
        return NGP_EINVAL;
    const TxWs w = tx_ws(F, size, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(cudaMemsetAsync(w.hdr, 0, 1024, st));
    if (F == 0) {
        NGP_CUDA(cudaMemsetAsync(w.scan, 0, (A + 1) * sizeof(int32_t), st));
        NGP_CUDA(cudaMemsetAsync(w.off, 0, 8, st));
        NGP_CUDA(cudaStreamSynchronize(st));
        counts[0] = size;
        counts[1] = 0;
        return 0;
    }
    k_tx_class<<<tx_grid(F), TX_THREADS, 0, st>>>(vertices, V, triangles, F, w.e, w.rot, w.hdr, w.etop);
    NGP_CHECK_LAUNCH();
    k_tx_hist<<<tx_grid(F), TX_THREADS, 0, st>>>(w.e, F, w.etop, w.hist);
    NGP_CHECK_LAUNCH();
    int64_t bad = 0;
    unsigned long long hist[64];
    NGP_CUDA(cudaMemcpyAsync(&bad, w.hdr, sizeof(bad), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaMemcpyAsync(hist, w.hist, sizeof(hist), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    if (bad) return NGP_EINVAL;
    int64_t S = size;
    for (; S > NGP_TEXTURE_MIN_SQUARE; S >>= 1) {
        unsigned long long sum = 0;
        for (int k = 0; k < 64; ++k) sum += hist[k] * (unsigned long long)(tx_side(k, S) * tx_side(k, S));
        if (sum <= (unsigned long long)A) break;
    }
    k_tx_key<<<tx_grid(F), TX_THREADS, 0, st>>>(w.e, F, w.etop, S, w.key[0], w.val[0]);
    NGP_CHECK_LAUNCH();
    size_t tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, w.key[0], w.key[1], w.val[0], w.val[1], F, 0, 4, st));
    NGP_COUNT_LAUNCHES(4);
    const int32_t* order = w.val[1];
    k_tx_area<<<tx_grid(F + 1), TX_THREADS, 0, st>>>(w.e, order, F, w.etop, S, w.off);
    NGP_CHECK_LAUNCH();
    tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.off, w.off, F + 1, st));
    NGP_COUNT_LAUNCHES(2);
    k_tx_place<<<tx_grid(F), TX_THREADS, 0, st>>>(vertices, triangles, F, w.e, w.rot, order, w.off, w.etop, S, uv, squares);
    NGP_CHECK_LAUNCH();
    k_tx_band<<<tx_grid(A + 1), TX_THREADS, 0, st>>>(uv, order, w.off, F, A, w.scan);
    NGP_CHECK_LAUNCH();
    tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.scan, w.scan, A + 1, st));
    NGP_COUNT_LAUNCHES(2);
    int32_t n = 0;
    NGP_CUDA(cudaMemcpyAsync(&n, w.scan + A, sizeof(n), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    counts[0] = S;
    counts[1] = n;
    return 0;
}

// the closest point of the uv triangle (A, B, C) to q as barycentrics (step 5)
__device__ void tx_closest(const double (&px)[3], const double (&py)[3], double qx, double qy, double (&b)[3]) {
    const double area = (px[1] - px[0]) * (py[2] - py[0]) - (py[1] - py[0]) * (px[2] - px[0]);
    const double dA = (px[1] - px[0]) * (qy - py[0]) - (py[1] - py[0]) * (qx - px[0]);
    const double dB = (px[2] - px[1]) * (qy - py[1]) - (py[2] - py[1]) * (qx - px[1]);
    const double dC = (px[0] - px[2]) * (qy - py[2]) - (py[0] - py[2]) * (qx - px[2]);
    if (area > 0.0 && dA >= 0.0 && dB >= 0.0 && dC >= 0.0) {
        b[0] = dB / area;
        b[1] = dC / area;
        b[2] = dA / area;
        return;
    }
    double best = INFINITY;
    for (int k = 0; k < 3; ++k) {
        const int k1 = k == 2 ? 0 : k + 1;
        const double ex = px[k1] - px[k], ey = py[k1] - py[k];
        const double l2 = ex * ex + ey * ey;
        double t = l2 > 0.0 ? ((qx - px[k]) * ex + (qy - py[k]) * ey) / l2 : 0.0;
        t = fmin(fmax(t, 0.0), 1.0);
        const double dx = qx - (px[k] + t * ex), dy = qy - (py[k] + t * ey);
        const double d2 = dx * dx + dy * dy;
        if (d2 < best) {
            best = d2;
            b[0] = b[1] = b[2] = 0.0;
            b[k] = 1.0 - t;
            b[k1] = t;
        }
    }
}

__global__ void k_tx_texels(const float* __restrict__ verts, const float* __restrict__ nrm_in, const int64_t* __restrict__ tris,
                            const float* __restrict__ uv, const int32_t* __restrict__ order, const int32_t* __restrict__ rot,
                            const int64_t* __restrict__ off, int64_t F, int64_t A, const int32_t* __restrict__ scan,
                            int64_t* __restrict__ texel, int32_t* __restrict__ tri, float* __restrict__ point,
                            float* __restrict__ normal) {
    for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < A; m += (int64_t)gridDim.x * blockDim.x) {
        const int32_t pos = scan[m];
        if (scan[m + 1] == pos) continue;
        const int64_t t = order[tx_rank(off, F, m)];
        const int r = rot[t];
        double ux[3], uy[3], px[3], py[3];
        tx_uv(uv, t, ux, uy);
        for (int k = 0; k < 3; ++k) {
            px[k] = ux[(r + k) % 3];
            py[k] = uy[(r + k) % 3];
        }
        double b[3];
        tx_closest(px, py, (double)tx_compact((uint64_t)m) + 0.5, (double)tx_compact((uint64_t)m >> 1) + 0.5, b);
        int64_t idx[3];
        for (int k = 0; k < 3; ++k) idx[k] = __ldg(tris + 3 * t + (r + k) % 3);
        double P[3][3];
        for (int k = 0; k < 3; ++k) tx_load(verts, idx[k], P[k]);
        double eB[3], eC[3], n[3];
        for (int a = 0; a < 3; ++a) {
            eB[a] = P[1][a] - P[0][a];
            eC[a] = P[2][a] - P[0][a];
            point[3 * (int64_t)pos + a] = (float)((P[0][a] + b[1] * eB[a]) + b[2] * eC[a]);
        }
        double len = 0.0;
        if (nrm_in) {
            double N[3][3];
            for (int k = 0; k < 3; ++k) tx_load(nrm_in, idx[k], N[k]);
            for (int a = 0; a < 3; ++a) n[a] = (b[0] * N[0][a] + b[1] * N[1][a]) + b[2] * N[2][a];
            len = tx_len(n[0], n[1], n[2]);
        }
        if (!(len > 0.0)) {
            n[0] = eB[1] * eC[2] - eB[2] * eC[1];
            n[1] = eB[2] * eC[0] - eB[0] * eC[2];
            n[2] = eB[0] * eC[1] - eB[1] * eC[0];
            len = tx_len(n[0], n[1], n[2]);
        }
        for (int a = 0; a < 3; ++a)
            normal[3 * (int64_t)pos + a] = len > 0.0 ? (float)(n[a] / len) : (a == 2 ? -1.f : 0.f);
        texel[pos] = m;
        tri[pos] = (int32_t)t;
    }
}

extern "C" int ngp_mesh_texture_texels(const float* vertices, const float* normals, int64_t n_vertices,
                                       const int64_t* triangles, int64_t n_triangles, int size, const float* uv,
                                       int64_t max_texels, int64_t* texel, int32_t* triangle, float* point, float* normal,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    const int64_t V = n_vertices, F = n_triangles, A = (int64_t)size * size;
    if (!workspace || !tx_sizes_ok(V, F, size) || max_texels < 0 || (F > 0 && (!vertices || !triangles || !uv)))
        return NGP_EINVAL;
    const TxWs w = tx_ws(F, size, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    int32_t n = 0;
    NGP_CUDA(cudaMemcpyAsync(&n, w.scan + A, sizeof(n), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    if (n > max_texels) return NGP_EINVAL;
    if (n == 0) return 0;
    if (!texel || !triangle || !point || !normal) return NGP_EINVAL;
    k_tx_texels<<<tx_grid(A), TX_THREADS, 0, st>>>(vertices, normals, triangles, uv, w.val[1], w.rot, w.off, F, A, w.scan,
                                                    texel, triangle, point, normal);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// bake
// ---------------------------------------------------------------------------------------------------------------------
struct TbWs {
    int* bad;
    float* o;
    float* d;
    int32_t* ridx;
    float* ts;
    float* sig;
    float* rgb;
    int64_t chunk;  // texels per chunk
    size_t total;
};

static TbWs tb_ws(int K, void* base) {
    TbWs w;
    const int64_t R = K + 1, c = NGP_TEXTURE_CHUNK_SAMPLES / R > 1 ? NGP_TEXTURE_CHUNK_SAMPLES / R : 1, n = c * R;
    char* p = (char*)base;
    size_t off = 0;
    w.bad = (int*)p; off += 256;
    w.o = (float*)(p + off); off += tx_align(c * 12);
    w.d = (float*)(p + off); off += tx_align(c * 12);
    w.ridx = (int32_t*)(p + off); off += tx_align(n * 4);
    w.ts = (float*)(p + off); off += tx_align(n * 4);
    w.sig = (float*)(p + off); off += tx_align(n * 4);
    w.rgb = (float*)(p + off); off += tx_align(n * 12);
    w.chunk = c;
    w.total = off;
    return w;
}

extern "C" size_t ngp_mesh_texture_bake_workspace(int samples) {
    if (samples < 1 || samples > NGP_TEXTURE_MAX_SAMPLES) return 0;
    return tb_ws(samples, nullptr).total;
}

// one thread per sample of texels [c0, c0 + nc): its ray and t (step 6); the sample's first thread writes the ray
__global__ void k_tx_rays(const float* __restrict__ point, const float* __restrict__ normal, int64_t c0, int64_t nc, int K,
                          float r, float delta, float* __restrict__ o, float* __restrict__ d, int32_t* __restrict__ ridx,
                          float* __restrict__ ts) {
    const int64_t n = nc * (K + 1);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t x = i / (K + 1);
        const int j = (int)(i - x * (K + 1));
        ridx[i] = (int32_t)x;
        ts[i] = j < K ? __fmul_rn((float)j + 0.5f, delta) : r;
        if (j == 0)
            for (int a = 0; a < 3; ++a) {
                const float nv = __ldg(normal + 3 * (c0 + x) + a);
                o[3 * x + a] = __fmaf_rn(nv, r, __ldg(point + 3 * (c0 + x) + a));
                d[3 * x + a] = -nv;
            }
    }
}

__global__ void k_tx_composite(const float* __restrict__ sig, const float* __restrict__ rgb, const int64_t* __restrict__ texel,
                               int64_t c0, int64_t nc, int K, float delta, int64_t W, uint8_t* __restrict__ tex,
                               int* __restrict__ bad) {
    for (int64_t x = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; x < nc; x += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = __ldg(texel + c0 + x);
        if (m < 0 || m >= W * W) {
            *bad = 1;  // every writer stores the same value
            continue;
        }
        const float* s = sig + x * (K + 1);
        const float* c = rgb + 3 * x * (K + 1);
        double T = 1.0, C[3] = {0.0, 0.0, 0.0};
        for (int j = 0; j < K; ++j) {
            const double a = 1.0 - exp(-((double)s[j] * (double)delta));
            const double wt = T * a;
            for (int k = 0; k < 3; ++k) C[k] = C[k] + wt * (double)c[3 * j + k];
            T = T * (1.0 - a);
        }
        const int64_t px = tx_compact((uint64_t)m), py = tx_compact((uint64_t)m >> 1);
        uint8_t* out = tex + 3 * ((W - 1 - py) * W + px);
        for (int k = 0; k < 3; ++k) {
            const double v = rint(255.0 * (C[k] + T * (double)c[3 * K + k]));
            out[k] = (uint8_t)fmin(fmax(v, 0.0), 255.0);
        }
    }
}

extern "C" int ngp_mesh_texture_bake(const NgpNet* net, int size, int64_t n_texels, const int64_t* texel, const float* point,
                                     const float* normal, float offset, int samples, uint8_t* texture, void* workspace,
                                     size_t workspace_bytes, void* stream) {
    const int K = samples;
    if (!net || !texture || !workspace || !tx_size_ok(size) || K < 1 || K > NGP_TEXTURE_MAX_SAMPLES || n_texels < 0 ||
        n_texels > (int64_t)size * size || !(offset >= 0.f) || !isfinite(offset) ||
        (n_texels > 0 && (!texel || !point || !normal)))
        return NGP_EINVAL;
    const TbWs w = tb_ws(K, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t W = size;
    NGP_CUDA(cudaMemsetAsync(texture, 0, W * W * 3, st));
    NGP_CUDA(cudaMemsetAsync(w.bad, 0, sizeof(int), st));
    const float delta = (2.f * offset) / (float)K;  // host fp32: one rounding each
    for (int64_t c0 = 0; c0 < n_texels; c0 += w.chunk) {
        const int64_t nc = n_texels - c0 < w.chunk ? n_texels - c0 : w.chunk;
        k_tx_rays<<<tx_grid(nc * (K + 1)), TX_THREADS, 0, st>>>(point, normal, c0, nc, K, offset, delta, w.o, w.d, w.ridx,
                                                                 w.ts);
        NGP_CHECK_LAUNCH();
        NgpSamples smp = {};
        smp.rays_o = w.o;
        smp.rays_d = w.d;
        smp.ray_idx = w.ridx;
        smp.ts = w.ts;
        smp.n = nc * (K + 1);
        const int rc = ngp_net_forward(net, &smp, 1, w.sig, w.rgb, nullptr, nullptr, stream);
        if (rc) return rc;
        k_tx_composite<<<tx_grid(nc), TX_THREADS, 0, st>>>(w.sig, w.rgb, texel, c0, nc, K, delta, W, texture, w.bad);
        NGP_CHECK_LAUNCH();
    }
    int bad = 0;
    NGP_CUDA(cudaMemcpyAsync(&bad, w.bad, sizeof(bad), cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    return bad ? NGP_EINVAL : 0;
}
