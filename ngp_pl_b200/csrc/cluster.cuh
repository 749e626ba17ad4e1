// Device arithmetic shared by the mesh simplification (csrc/mesh.cu) and the point-cloud export (csrc/points.cu): the
// cluster-grid cell of rule 1 of the simplification (include/ngp_b200.h), the fixed-order warp sum of its reductions
// and its cyclic Jacobi eigensolve.
#pragma once
#include "../../include/ngp_b200.h"

__device__ __forceinline__ int ms_cell(float v, float lo, float h, int n) {
    const float q = floorf(__fdiv_rn(__fsub_rn(v, lo), h));
    return (int)fminf(fmaxf(q, 0.f), (float)(n - 1));  // NaN -> 0
}

// cluster key (c0*n1 + c1)*n2 + c2 of the point p[0..2]
__device__ __forceinline__ uint64_t ms_key(const float* __restrict__ p, const NgpClusterGrid& g) {
    const int c0 = ms_cell(__ldg(p), g.lo[0], g.h, g.n[0]);
    const int c1 = ms_cell(__ldg(p + 1), g.lo[1], g.h, g.n[1]);
    const int c2 = ms_cell(__ldg(p + 2), g.lo[2], g.h, g.n[2]);
    return ((uint64_t)c0 * g.n[1] + c1) * g.n[2] + c2;
}

__device__ __forceinline__ double ms_wsum(double v) {  // fixed shuffle tree: lane 0 holds the sum
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// eigen-decomposition of the symmetric 3x3 a (cyclic Jacobi, NGP_SIMPLIFY_JACOBI_SWEEPS sweeps): eigenvalues on a's diagonal,
// eigenvectors in e's columns
static __device__ void ms_jacobi(double (&a)[3][3], double (&e)[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) e[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < NGP_SIMPLIFY_JACOBI_SWEEPS; ++sweep)
        for (int r = 0; r < 3; ++r) {
            const int p = r == 2 ? 1 : 0, q = r == 0 ? 1 : 2;
            const double apq = a[p][q];
            if (apq == 0.0) continue;
            const double th = (a[q][q] - a[p][p]) / (2.0 * apq);
            const double t = fabs(th) > 1e150 ? 0.5 / th : (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
            const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
            for (int k = 0; k < 3; ++k) {
                const double kp = a[k][p], kq = a[k][q];
                a[k][p] = c * kp - s * kq;
                a[k][q] = s * kp + c * kq;
            }
            for (int k = 0; k < 3; ++k) {
                const double pk = a[p][k], qk = a[q][k];
                a[p][k] = c * pk - s * qk;
                a[q][k] = s * pk + c * qk;
            }
            a[p][q] = a[q][p] = 0.0;
            for (int k = 0; k < 3; ++k) {
                const double kp = e[k][p], kq = e[k][q];
                e[k][p] = c * kp - s * kq;
                e[k][q] = s * kp + c * kq;
            }
        }
}
