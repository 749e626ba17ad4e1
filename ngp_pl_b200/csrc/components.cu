// Connected components on the device (include/ngp_b200.h, "Connected components"; numpy + scipy restatement:
// oracle/components_ref.py). One union-find core serves two implicit graphs:
//
// core      : parent is int32, one entry per node; a kernel generates the edges and hooks their endpoints' roots,
//             the larger root under the smaller, with atomicCAS (retried from the new root on failure). find() splits
//             paths as it walks them: a plain store of a grandparent into a non-root, which no CAS ever targets.
//             Links always point to a smaller index, so once every edge is hooked each tree's root is the smallest
//             node of its component and a compression pass (label = find) gives labels that do not depend on the
//             schedule. Component sizes are integer atomics on the root.
// select    : roots (label == index) compacted in ascending order with a cub scan, sizes radix-sorted descending with
//             the root as value (the sort is stable, so equal sizes keep the smaller label first), a keep byte per root.
// occupancy : nodes are the occupied shell cells of density_bitfield, edges their 26-neighbours in the cascade and the
//             cells of the next finer cascade whose closed boxes meet theirs. Cell box coordinates mb (2 i / G - 1)
//             are exact in double (mb is an fp32 value, 2 i / G a dyadic rational of at most 11 bits), so every box
//             test is an exact comparison. Cleanup runs cascade by cascade, fine to coarse, one thread per bitfield
//             byte: a shell cell follows its component, an inner cell the finer cells its box meets.
// mesh      : nodes are vertices and each triangle hooks its corners; a triangle's label is the smallest triangle
//             index of its component (atomicMin per root). Filtering flags triangles and the vertices they use, two
//             cub scans number them in input order, one read-back of the counts.
// No float atomics: two calls are bitwise equal.
#include "common.cuh"
#include "march.cuh"
#include "../../include/ngp_b200.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define CC_THREADS 256

static size_t cc_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int cc_grid(int64_t items) {
    const int64_t want = (items + CC_THREADS - 1) / CC_THREADS, cap = (int64_t)ngp_sm_count() * 32;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

#define CC_LOOP(i, n) for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// ---- union-find core ------------------------------------------------------------------------------------------------
// SPLIT: path splitting while linking. The compression pass walks without it: a split there could store an
// intermediate ancestor over a label another thread has just finalised.
template <bool SPLIT = true>
__device__ __forceinline__ int32_t uf_find(int32_t* p, int32_t x) {
    volatile int32_t* vp = p;
    int32_t cur = vp[x];
    if (cur != x) {
        int32_t prev = x, next;
        while (cur > (next = vp[cur])) {
            if (SPLIT) vp[prev] = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

__device__ __forceinline__ void uf_union(int32_t* p, int32_t a, int32_t b) {
    a = uf_find(p, a);
    b = uf_find(p, b);
    while (a != b) {
        if (a < b) {
            const int32_t t = a;
            a = b;
            b = t;
        }
        const int32_t old = atomicCAS(&p[a], a, b);
        if (old == a) return;
        a = uf_find(p, old);
        b = uf_find(p, b);
    }
}

// label = root for every node (parent >= 0), size of the root's component += 1
__global__ void k_cc_compress(int32_t* __restrict__ p, int64_t n, int32_t* __restrict__ sizes) {
    CC_LOOP(i, n) {
        if (p[i] < 0) continue;
        const int32_t r = uf_find<false>(p, (int32_t)i);
        p[i] = r;
        if (sizes) atomicAdd(&sizes[r], 1);
    }
}

// ---- occupancy-grid geometry ----------------------------------------------------------------------------------------
struct CcGrid {
    int cascades, G;
    uint32_t G3;
    float scale;
};

__device__ __forceinline__ double cc_mb(int c, float scale) { return (double)fminf(scalbnf(1.0f, c - 1), scale); }
// lower face of cell i of a cascade of half extent mb (i = G: the upper face of cell G - 1); exact in double
__device__ __forceinline__ double cc_x(double mb, int i, int G) { return mb * ((2.0 * i) / G - 1.0); }

// whether cell (x, y, z) of cascade c >= 1 lies wholly inside cascade c - 1's closed box
__device__ __forceinline__ bool cc_inner(const CcGrid& g, int c, int x, int y, int z) {
    if (c == 0) return false;
    const double mb = cc_mb(c, g.scale), mf = cc_mb(c - 1, g.scale);
    const int v[3] = {x, y, z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (!(cc_x(mb, v[a], g.G) >= -mf && cc_x(mb, v[a] + 1, g.G) <= mf)) return false;
    return true;
}

// the cells t of cascade c - 1 on one axis whose closed interval meets that of cell s of cascade c:
// x_{c-1}(t) <= x_c(s + 1) and x_{c-1}(t + 1) >= x_c(s); an estimate widened by one, then narrowed exactly
__device__ __forceinline__ int2 cc_range(double mb, double mf, int s, int G) {
    const double lo = cc_x(mb, s, G), hi = cc_x(mb, s + 1, G);
    int a = (int)floor((lo / mf + 1.0) * 0.5 * G) - 1, b = (int)floor((hi / mf + 1.0) * 0.5 * G) + 1;
    a = max(a, 0);
    b = min(b, G - 1);
    while (a <= b && !(cc_x(mf, a + 1, G) >= lo)) ++a;
    while (b >= a && !(cc_x(mf, b, G) <= hi)) --b;
    return make_int2(a, b);
}

__device__ __forceinline__ void cc_decode(uint32_t m, int& x, int& y, int& z) {
    x = (int)morton_compact10(m);
    y = (int)morton_compact10(m >> 1);
    z = (int)morton_compact10(m >> 2);
}

__device__ __forceinline__ bool cc_bit(const uint8_t* bits, int64_t i) { return (bits[i >> 3] >> (i & 7)) & 1; }

// labels[i] = i for an occupied shell cell (a node), -1 otherwise
__global__ void k_cc_grid_init(const uint8_t* __restrict__ bits, const CcGrid g, int32_t* __restrict__ labels,
                               int32_t* __restrict__ sizes) {
    const int64_t n = (int64_t)g.cascades * g.G3;
    CC_LOOP(i, n) {
        const int c = (int)(i / g.G3);
        int x, y, z;
        cc_decode((uint32_t)(i - (int64_t)c * g.G3), x, y, z);
        labels[i] = cc_bit(bits, i) && !cc_inner(g, c, x, y, z) ? (int32_t)i : -1;
        sizes[i] = 0;
    }
}

__global__ void k_cc_grid_link(const CcGrid g, int32_t* __restrict__ p) {
    const int64_t n = (int64_t)g.cascades * g.G3;
    CC_LOOP(i, n) {
        if (p[i] < 0) continue;
        const int c = (int)(i / g.G3);
        const int64_t base = (int64_t)c * g.G3;
        int x, y, z;
        cc_decode((uint32_t)(i - base), x, y, z);
        // the 13 neighbours after (x, y, z) in lexicographic offset order: every 26-edge once
        for (int d = 14; d < 27; ++d) {
            const int X = x + d / 9 - 1, Y = y + (d / 3) % 3 - 1, Z = z + d % 3 - 1;
            if (X < 0 || Y < 0 || Z < 0 || X >= g.G || Y >= g.G || Z >= g.G) continue;
            const int64_t j = base + morton_encode3((uint32_t)X, (uint32_t)Y, (uint32_t)Z);
            if (p[j] >= 0) uf_union(p, (int32_t)i, (int32_t)j);
        }
        if (c == 0) continue;
        const double mb = cc_mb(c, g.scale), mf = cc_mb(c - 1, g.scale);
        const int2 rx = cc_range(mb, mf, x, g.G), ry = cc_range(mb, mf, y, g.G), rz = cc_range(mb, mf, z, g.G);
        const int64_t fine = base - g.G3;
        for (int X = rx.x; X <= rx.y; ++X)
            for (int Y = ry.x; Y <= ry.y; ++Y)
                for (int Z = rz.x; Z <= rz.y; ++Z) {
                    const int64_t j = fine + morton_encode3((uint32_t)X, (uint32_t)Y, (uint32_t)Z);
                    if (p[j] >= 0) uf_union(p, (int32_t)i, (int32_t)j);
                }
    }
}

static bool cc_grid_ok(int cascades, int G) {
    return G >= 2 && G <= 1024 && (G & (G - 1)) == 0 && cascades >= 1 && cascades <= 62 &&
           (int64_t)cascades * G * G * G < ((int64_t)1 << 31);
}

extern "C" int ngp_grid_components(const uint8_t* density_bitfield, int cascades, int grid_size, float scale,
                                   int32_t* labels, int32_t* sizes, void* stream) {
    if (!density_bitfield || !labels || !sizes || !cc_grid_ok(cascades, grid_size) || !(scale > 0) || !isfinite(scale))
        return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const CcGrid g{cascades, grid_size, (uint32_t)grid_size * grid_size * grid_size, scale};
    const int64_t n = (int64_t)cascades * g.G3;
    k_cc_grid_init<<<cc_grid(n), CC_THREADS, 0, st>>>(density_bitfield, g, labels, sizes);
    NGP_CHECK_LAUNCH();
    k_cc_grid_link<<<cc_grid(n), CC_THREADS, 0, st>>>(g, labels);
    NGP_CHECK_LAUNCH();
    k_cc_compress<<<cc_grid(n), CC_THREADS, 0, st>>>(labels, n, sizes);
    NGP_CHECK_LAUNCH();
    return 0;
}

// ---- selection ------------------------------------------------------------------------------------------------------
// workspace: header (int64[4]) | positions (n + 1 int32) | sizes x2 (n uint32) | labels x2 (n int32) | cub temp
struct CcSelWs {
    int64_t* hdr;
    int32_t* pos;
    uint32_t* key[2];
    int32_t* val[2];
    void* temp;
    size_t temp_bytes, total;
};

static CcSelWs cc_sel_ws(int64_t n, void* base) {
    CcSelWs w;
    size_t tb = 0, t = 0;
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairsDescending(nullptr, t, k, v, (int)n, 0, 32);
    tb = t;
    t = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1));
    tb = t > tb ? t : tb;
    w.temp_bytes = cc_align(tb);
    char* p = (char*)base;
    size_t off = 0;
    w.hdr = (int64_t*)(p + off); off += 256;
    w.pos = (int32_t*)(p + off); off += cc_align((n + 1) * 4);
    for (int i = 0; i < 2; ++i) { w.key[i] = (uint32_t*)(p + off); off += cc_align(n * 4); }
    for (int i = 0; i < 2; ++i) { w.val[i] = (int32_t*)(p + off); off += cc_align(n * 4); }
    w.temp = p + off; off += w.temp_bytes;
    w.total = off;
    return w;
}

__global__ void k_cc_root_flags(const int32_t* __restrict__ labels, int64_t n, int32_t* __restrict__ flag) {
    CC_LOOP(i, n + 1) flag[i] = i < n && labels[i] == (int32_t)i;
}

__global__ void k_cc_root_scatter(const int32_t* __restrict__ labels, const int32_t* __restrict__ sizes, int64_t n,
                                  const int32_t* __restrict__ pos, uint32_t* __restrict__ key, int32_t* __restrict__ val,
                                  int64_t* __restrict__ hdr) {
    CC_LOOP(i, n) {
        if (labels[i] != (int32_t)i) continue;
        key[pos[i]] = (uint32_t)sizes[i];
        val[pos[i]] = (int32_t)i;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        hdr[0] = pos[n];
        hdr[1] = 0;
    }
}

// rank r of the sorted roots is kept iff r < keep_largest and its size >= min_size
__global__ void k_cc_keep(const uint32_t* __restrict__ key, const int32_t* __restrict__ val, int64_t R,
                          int64_t keep_largest, int64_t min_size, uint8_t* __restrict__ keep,
                          unsigned long long* __restrict__ kept) {
    CC_LOOP(r, R) {
        if (r < keep_largest && (int64_t)key[r] >= min_size) {
            keep[val[r]] = 1;
            atomicAdd(kept, 1ull);
        }
    }
}

extern "C" size_t ngp_components_select_workspace(int64_t n) {
    if (n < 0 || n >= ((int64_t)1 << 31)) return 0;
    return cc_sel_ws(n, nullptr).total;
}

extern "C" int ngp_components_select(const int32_t* labels, const int32_t* sizes, int64_t n, int64_t keep_largest,
                                     int64_t min_size, uint8_t* keep, int64_t* counts, void* workspace,
                                     size_t workspace_bytes, void* stream) {
    if (n < 0 || n >= ((int64_t)1 << 31) || !counts || (n > 0 && (!labels || !sizes || !keep || !workspace)))
        return NGP_EINVAL;
    if (keep_largest < 0 || min_size < 0) return NGP_EINVAL;
    counts[0] = counts[1] = 0;
    if (n == 0) return 0;
    const CcSelWs w = cc_sel_ws(n, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    k_cc_root_flags<<<cc_grid(n + 1), CC_THREADS, 0, st>>>(labels, n, w.pos);
    NGP_CHECK_LAUNCH();
    size_t tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.pos, w.pos, (int)(n + 1), st));
    NGP_COUNT_LAUNCHES(1);
    k_cc_root_scatter<<<cc_grid(n), CC_THREADS, 0, st>>>(labels, sizes, n, w.pos, w.key[0], w.val[0], w.hdr);
    NGP_CHECK_LAUNCH();
    int64_t R = 0;
    NGP_CUDA(cudaMemcpyAsync(&R, w.hdr, 8, cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    NGP_CUDA(cudaMemsetAsync(keep, 0, (size_t)n, st));
    if (R == 0) return 0;
    cub::DoubleBuffer<uint32_t> k(w.key[0], w.key[1]);
    cub::DoubleBuffer<int32_t> v(w.val[0], w.val[1]);
    tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceRadixSort::SortPairsDescending(w.temp, tb, k, v, (int)R, 0, 32, st));
    NGP_COUNT_LAUNCHES(1);
    k_cc_keep<<<cc_grid(R), CC_THREADS, 0, st>>>(k.Current(), v.Current(), R, keep_largest, min_size, keep,
                                                  (unsigned long long*)(w.hdr + 1));
    NGP_CHECK_LAUNCH();
    int64_t h[2];
    NGP_CUDA(cudaMemcpyAsync(h, w.hdr, 16, cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    counts[0] = h[0];
    counts[1] = h[1];
    return 0;
}

// ---- occupancy cleanup ----------------------------------------------------------------------------------------------
// one thread per bitfield byte of cascade c: bits holds the cleaned cascades < c and the input from c on; removed gets
// the cells of c that are cleared. A shell node is cleared iff its component is not kept; an occupied inner cell iff
// the cells of cascade c - 1 its closed box meets include a cleared one and no occupied one left standing.
__global__ void k_cc_grid_clean(uint8_t* __restrict__ bits, float* __restrict__ density_grid, const CcGrid g, int c,
                                const int32_t* __restrict__ labels, const uint8_t* __restrict__ keep,
                                uint8_t* __restrict__ removed, unsigned long long* __restrict__ cleared) {
    const int64_t nb = g.G3 >> 3, base = (int64_t)c * g.G3;
    const double mb = cc_mb(c, g.scale), mf = c > 0 ? cc_mb(c - 1, g.scale) : 0.0;
    CC_LOOP(b, nb) {
        const int64_t byte = (base >> 3) + b;
        const uint8_t in = bits[byte];
        uint8_t out = in, rm = 0;
        unsigned long long n_shell = 0, n_inner = 0;
        for (int k = 0; k < 8; ++k) {
            if (!((in >> k) & 1)) continue;
            const int64_t i = byte * 8 + k;
            bool drop;
            if (labels[i] >= 0) {
                drop = !keep[labels[i]];
                n_shell += drop;
            } else {
                int x, y, z;
                cc_decode((uint32_t)(i - base), x, y, z);
                const int2 rx = cc_range(mb, mf, x, g.G), ry = cc_range(mb, mf, y, g.G), rz = cc_range(mb, mf, z, g.G);
                bool any_rm = false, any_kept = false;
                const int64_t fine = base - g.G3;
                for (int X = rx.x; X <= rx.y && !any_kept; ++X)
                    for (int Y = ry.x; Y <= ry.y && !any_kept; ++Y)
                        for (int Z = rz.x; Z <= rz.y; ++Z) {
                            const int64_t j = fine + morton_encode3((uint32_t)X, (uint32_t)Y, (uint32_t)Z);
                            any_kept = any_kept || cc_bit(bits, j);
                            any_rm = any_rm || cc_bit(removed, j);
                        }
                drop = any_rm && !any_kept;
                n_inner += drop;
            }
            if (drop) {
                out &= (uint8_t)~(1u << k);
                rm |= (uint8_t)(1u << k);
                if (density_grid) density_grid[i] = -1.0f;
            }
        }
        bits[byte] = out;
        removed[byte] = rm;
        if (cleared && n_shell) atomicAdd(&cleared[0], n_shell);
        if (cleared && n_inner) atomicAdd(&cleared[1], n_inner);
    }
}

extern "C" int ngp_grid_components_clean(uint8_t* density_bitfield, float* density_grid, int cascades, int grid_size,
                                         float scale, const int32_t* labels, const uint8_t* keep, uint8_t* removed,
                                         int64_t* cleared, void* stream) {
    if (!density_bitfield || !labels || !keep || !removed || !cc_grid_ok(cascades, grid_size) || !(scale > 0) ||
        !isfinite(scale))
        return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const CcGrid g{cascades, grid_size, (uint32_t)grid_size * grid_size * grid_size, scale};
    if (cleared) NGP_CUDA(cudaMemsetAsync(cleared, 0, 16, st));
    for (int c = 0; c < cascades; ++c) {
        k_cc_grid_clean<<<cc_grid(g.G3 >> 3), CC_THREADS, 0, st>>>(density_bitfield, density_grid, g, c, labels, keep,
                                                                   removed, (unsigned long long*)cleared);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}

// ---- mesh -----------------------------------------------------------------------------------------------------------
// components workspace: header (int32 flag) | parent (V int32) | smallest triangle per root (V int32)
struct CcMeshWs {
    int32_t* flag;
    int32_t* parent;
    int32_t* first;
    size_t total;
};

static CcMeshWs cc_mesh_ws(int64_t V, void* base) {
    CcMeshWs w;
    char* p = (char*)base;
    size_t off = 0;
    w.flag = (int32_t*)(p + off); off += 256;
    w.parent = (int32_t*)(p + off); off += cc_align(V * 4);
    w.first = (int32_t*)(p + off); off += cc_align(V * 4);
    w.total = off;
    return w;
}

__global__ void k_cc_mesh_init(int32_t* __restrict__ parent, int32_t* __restrict__ first, int64_t V) {
    CC_LOOP(i, V) {
        parent[i] = (int32_t)i;
        first[i] = INT32_MAX;
    }
}

__device__ __forceinline__ bool cc_tri(const int64_t* __restrict__ tris, int64_t t, int64_t V, int32_t (&v)[3]) {
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int64_t x = tris[3 * t + k];
        ok = ok && x >= 0 && x < V;
        v[k] = (int32_t)x;
    }
    return ok;
}

__global__ void k_cc_mesh_link(const int64_t* __restrict__ tris, int64_t F, int64_t V, int32_t* __restrict__ parent,
                               int32_t* __restrict__ flag) {
    CC_LOOP(t, F) {
        int32_t v[3];
        if (!cc_tri(tris, t, V, v)) {
            *flag = 1;
            continue;
        }
        uf_union(parent, v[0], v[1]);
        uf_union(parent, v[0], v[2]);
    }
}

__global__ void k_cc_mesh_first(const int64_t* __restrict__ tris, int64_t F, int64_t V, const int32_t* __restrict__ parent,
                                int32_t* __restrict__ first) {
    CC_LOOP(t, F) {
        int32_t v[3];
        if (cc_tri(tris, t, V, v)) atomicMin(&first[parent[v[0]]], (int32_t)t);
    }
}

__global__ void k_cc_mesh_label(const int64_t* __restrict__ tris, int64_t F, int64_t V, const int32_t* __restrict__ parent,
                                const int32_t* __restrict__ first, int32_t* __restrict__ labels,
                                int32_t* __restrict__ sizes) {
    CC_LOOP(t, F) {
        int32_t v[3];
        if (!cc_tri(tris, t, V, v)) continue;
        const int32_t l = first[parent[v[0]]];
        labels[t] = l;
        atomicAdd(&sizes[l], 1);
    }
}

static bool cc_mesh_ok(int64_t V, int64_t F) { return V >= 0 && F >= 0 && V < ((int64_t)1 << 31) && F < ((int64_t)1 << 31); }

extern "C" size_t ngp_mesh_components_workspace(int64_t n_vertices, int64_t n_triangles) {
    if (!cc_mesh_ok(n_vertices, n_triangles)) return 0;
    return cc_mesh_ws(n_vertices, nullptr).total;
}

extern "C" int ngp_mesh_components(const int64_t* triangles, int64_t n_vertices, int64_t n_triangles, int32_t* labels,
                                   int32_t* sizes, void* workspace, size_t workspace_bytes, void* stream) {
    const int64_t V = n_vertices, F = n_triangles;
    if (!cc_mesh_ok(V, F) || !workspace || (F > 0 && (!triangles || !labels || !sizes))) return NGP_EINVAL;
    const CcMeshWs w = cc_mesh_ws(V, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    if (F == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(cudaMemsetAsync(w.flag, 0, 4, st));
    NGP_CUDA(cudaMemsetAsync(sizes, 0, (size_t)F * 4, st));
    k_cc_mesh_init<<<cc_grid(V), CC_THREADS, 0, st>>>(w.parent, w.first, V);
    NGP_CHECK_LAUNCH();
    k_cc_mesh_link<<<cc_grid(F), CC_THREADS, 0, st>>>(triangles, F, V, w.parent, w.flag);
    NGP_CHECK_LAUNCH();
    k_cc_compress<<<cc_grid(V), CC_THREADS, 0, st>>>(w.parent, V, nullptr);
    NGP_CHECK_LAUNCH();
    k_cc_mesh_first<<<cc_grid(F), CC_THREADS, 0, st>>>(triangles, F, V, w.parent, w.first);
    NGP_CHECK_LAUNCH();
    k_cc_mesh_label<<<cc_grid(F), CC_THREADS, 0, st>>>(triangles, F, V, w.parent, w.first, labels, sizes);
    NGP_CHECK_LAUNCH();
    int32_t bad = 0;
    NGP_CUDA(cudaMemcpyAsync(&bad, w.flag, 4, cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    return bad ? NGP_EINVAL : 0;
}

// filter workspace: header (int64[4]: V', F', bad) | triangle positions (F + 1 int32) | vertex positions (V + 1 int32) |
// cub temp
struct CcFilterWs {
    int64_t* hdr;
    int32_t* tpos;
    int32_t* vpos;
    void* temp;
    size_t temp_bytes, total;
};

static CcFilterWs cc_filter_ws(int64_t V, int64_t F, void* base) {
    CcFilterWs w;
    size_t tb = 0, t = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, (int)(F + 1));
    tb = t;
    t = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, (int)(V + 1));
    tb = t > tb ? t : tb;
    w.temp_bytes = cc_align(tb);
    char* p = (char*)base;
    size_t off = 0;
    w.hdr = (int64_t*)(p + off); off += 256;
    w.tpos = (int32_t*)(p + off); off += cc_align((F + 1) * 4);
    w.vpos = (int32_t*)(p + off); off += cc_align((V + 1) * 4);
    w.temp = p + off; off += w.temp_bytes;
    w.total = off;
    return w;
}

__global__ void k_cc_filter_flags(const int64_t* __restrict__ tris, int64_t F, int64_t V, const int32_t* __restrict__ labels,
                                  const uint8_t* __restrict__ keep, int32_t* __restrict__ tflag, int32_t* __restrict__ vflag,
                                  int64_t* __restrict__ hdr) {
    CC_LOOP(t, F + 1) {
        if (t == F) {
            tflag[F] = 0;
            continue;
        }
        int32_t v[3];
        const int32_t l = labels[t];
        const bool ok = cc_tri(tris, t, V, v) && l >= 0 && l < F;
        if (!ok) hdr[2] = 1;
        const bool k = ok && keep[l];
        tflag[t] = k;
        if (k) {
            vflag[v[0]] = 1;
            vflag[v[1]] = 1;
            vflag[v[2]] = 1;
        }
    }
}

__global__ void k_cc_filter_totals(const int32_t* __restrict__ tpos, int64_t F, const int32_t* __restrict__ vpos, int64_t V,
                                   int64_t* __restrict__ hdr) {
    hdr[0] = vpos[V];
    hdr[1] = tpos[F];
}

extern "C" size_t ngp_mesh_filter_workspace(int64_t n_vertices, int64_t n_triangles) {
    if (!cc_mesh_ok(n_vertices, n_triangles)) return 0;
    return cc_filter_ws(n_vertices, n_triangles, nullptr).total;
}

extern "C" int ngp_mesh_filter_count(const int64_t* triangles, int64_t n_vertices, int64_t n_triangles,
                                     const int32_t* labels, const uint8_t* keep, int64_t* counts, void* workspace,
                                     size_t workspace_bytes, void* stream) {
    const int64_t V = n_vertices, F = n_triangles;
    if (!cc_mesh_ok(V, F) || !workspace || !counts || (F > 0 && (!triangles || !labels || !keep))) return NGP_EINVAL;
    const CcFilterWs w = cc_filter_ws(V, F, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    NGP_CUDA(cudaMemsetAsync(w.hdr, 0, 32, st));
    NGP_CUDA(cudaMemsetAsync(w.vpos, 0, (size_t)(V + 1) * 4, st));
    if (F > 0) {
        k_cc_filter_flags<<<cc_grid(F + 1), CC_THREADS, 0, st>>>(triangles, F, V, labels, keep, w.tpos, w.vpos, w.hdr);
        NGP_CHECK_LAUNCH();
    } else {
        NGP_CUDA(cudaMemsetAsync(w.tpos, 0, 4, st));
    }
    size_t tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.tpos, w.tpos, (int)(F + 1), st));
    NGP_COUNT_LAUNCHES(1);
    tb = w.temp_bytes;
    NGP_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.vpos, w.vpos, (int)(V + 1), st));
    NGP_COUNT_LAUNCHES(1);
    k_cc_filter_totals<<<1, 1, 0, st>>>(w.tpos, F, w.vpos, V, w.hdr);
    NGP_CHECK_LAUNCH();
    int64_t h[3];
    NGP_CUDA(cudaMemcpyAsync(h, w.hdr, 24, cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    if (h[2]) return NGP_EINVAL;
    counts[0] = h[0];
    counts[1] = h[1];
    return 0;
}

__global__ void k_cc_filter_vertices(const float* __restrict__ verts, const float* __restrict__ nrm,
                                     const uint8_t* __restrict__ col, int64_t V, const int32_t* __restrict__ vpos,
                                     float* __restrict__ ov, float* __restrict__ on, uint8_t* __restrict__ oc) {
    CC_LOOP(i, V) {
        const int64_t at = vpos[i];
        if (vpos[i + 1] == at) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            ov[3 * at + k] = verts[3 * i + k];
            if (on) on[3 * at + k] = nrm[3 * i + k];
            if (oc) oc[3 * at + k] = col[3 * i + k];
        }
    }
}

__global__ void k_cc_filter_triangles(const int64_t* __restrict__ tris, int64_t F, const int32_t* __restrict__ tpos,
                                      const int32_t* __restrict__ vpos, int64_t* __restrict__ ot) {
    CC_LOOP(t, F) {
        const int64_t at = tpos[t];
        if (tpos[t + 1] == at) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) ot[3 * at + k] = vpos[tris[3 * t + k]];
    }
}

extern "C" int ngp_mesh_filter_emit(const float* vertices, const float* normals, const uint8_t* colors,
                                    const int64_t* triangles, int64_t n_vertices, int64_t n_triangles, float* out_vertices,
                                    float* out_normals, uint8_t* out_colors, int64_t* out_triangles, int64_t max_vertices,
                                    int64_t max_triangles, void* workspace, size_t workspace_bytes, void* stream) {
    const int64_t V = n_vertices, F = n_triangles;
    if (!cc_mesh_ok(V, F) || !workspace || (F > 0 && !triangles) || (V > 0 && !vertices)) return NGP_EINVAL;
    const CcFilterWs w = cc_filter_ws(V, F, workspace);
    if (workspace_bytes < w.total) return NGP_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    int64_t h[2];
    NGP_CUDA(cudaMemcpyAsync(h, w.hdr, 16, cudaMemcpyDeviceToHost, st));
    NGP_CUDA(cudaStreamSynchronize(st));
    if (h[0] > max_vertices || h[1] > max_triangles || (h[0] > 0 && !out_vertices) || (h[1] > 0 && !out_triangles))
        return NGP_EINVAL;
    float* on = normals ? out_normals : nullptr;
    uint8_t* oc = colors ? out_colors : nullptr;
    if (h[0] > 0) {
        k_cc_filter_vertices<<<cc_grid(V), CC_THREADS, 0, st>>>(vertices, normals, colors, V, w.vpos, out_vertices, on, oc);
        NGP_CHECK_LAUNCH();
    }
    if (h[1] > 0) {
        k_cc_filter_triangles<<<cc_grid(F), CC_THREADS, 0, st>>>(triangles, F, w.tpos, w.vpos, out_triangles);
        NGP_CHECK_LAUNCH();
    }
    return 0;
}
