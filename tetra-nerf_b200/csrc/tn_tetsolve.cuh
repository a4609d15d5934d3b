// tn_tetsolve.cuh -- the spatial gradient of a function that is affine inside one tetrahedron, shared by the normal map (tn_normals.cu)
// and the ray gradients of the training step (tn_ray_grads.cu).
//
// With b(x) = E^-1 (x - x_v0), E = [x_v1 - x_v0 | x_v2 - x_v0 | x_v3 - x_v0], a function of the weights has the spatial gradient
// E^-T q, q = its gradient in b; E^-T = cof(E) / det(E).  E is formed from the fp32 positions, the cofactors and the determinant in
// float64: the differences are exact, so slivers lose no bits to cancellation.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tn {

// cf[k] = column k of cof(E): e2 x e3, e3 x e1, e1 x e2; det = e1 . (e2 x e3).  grad = sum_k q_k cf[k] / det (no solve when det == 0).
__device__ __forceinline__ void tet_cofactors(const float *__restrict__ xyz, const uint32_t (&vs)[4], double (&cf)[3][3], double &det) {
    double x[4][3];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) x[k][c] = (double)__ldg(xyz + 3 * (size_t)vs[k] + c);
    double e[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) e[k][c] = x[k + 1][c] - x[0][c];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double *a = e[(k + 1) % 3], *b = e[(k + 2) % 3];
        cf[k][0] = a[1] * b[2] - a[2] * b[1];
        cf[k][1] = a[2] * b[0] - a[0] * b[2];
        cf[k][2] = a[0] * b[1] - a[1] * b[0];
    }
    det = e[0][0] * cf[0][0] + e[0][1] * cf[0][1] + e[0][2] * cf[0][2];
}

}  // namespace tn
