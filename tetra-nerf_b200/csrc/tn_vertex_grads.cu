// tn_vertex_grads.cu -- gradient of the fused training step at the mesh vertex positions (DESIGN.md §4.9), for refining the point cloud.
//
// With the sample distances and the matched tetrahedra held fixed, a fine sample's weights b = E^-1 (x_i - x_v0) (b_0 = 1 - sum b_k) move
// with the vertices; the vertex half of the reference's add_barycentrics_grad is
//   dL/dx_vj += -b_j m_i,   m_i = dL/dx_i = E_i^-T q_i   (the per-sample vector k_ray_grads writes),   j = 0..3.
// Unmatched samples, flat tetrahedra and empty rays carry m_i = 0 and contribute nothing.
//
// k_vertex_grads (default mode): one thread per sample row, float reductions into [V,3], like the field gradient of k_mlp_bwd.
// k_det_vertex_grads (deterministic mode): one warp per vertex over the (vertex, row * 4 + k) pairs that the field gradient already sorted
// stably by vertex; lane l sums entries l, l + 32, ... in float64, a fixed butterfly combines the lanes: the result is bitwise reproducible.
#include "tn_common.cuh"
#include "tn_sort.cuh"

namespace tn {

__device__ __forceinline__ float slot_weight(const float *__restrict__ bary, uint64_t row, uint32_t k) {  // as k_det_field_grad
    const float *c = bary + 3 * (size_t)row;
    const float b0 = __ldg(c), b1 = __ldg(c + 1), b2 = __ldg(c + 2);
    return k == 0 ? 1.0f - ((b0 + b1) + b2) : (k == 1 ? b0 : (k == 2 ? b1 : b2));
}

__global__ void __launch_bounds__(256) k_vertex_grads(const VertexGradsLaunch p) {
    const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= (uint64_t)*p.n_active * p.S) return;
    const uint4 v = __ldg(p.vi + row);
    if (v.x == TN_EMPTY) return;
    const float4 m = __ldg(p.gx + row);
    if (m.x == 0.f && m.y == 0.f && m.z == 0.f) return;  // flat tetrahedron (or a zero gradient): nothing to add
    const uint32_t vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {
        const float w = slot_weight(p.bary, row, k);
        float *g = p.grad_xyz + 3 * (size_t)vs[k];
        atomicAdd(g, -(w * m.x));
        atomicAdd(g + 1, -(w * m.y));
        atomicAdd(g + 2, -(w * m.z));
    }
}

__global__ void __launch_bounds__(256) k_det_vertex_grads(const VertexGradsLaunch p) {
    const uint32_t v = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31u;
    if (v >= p.V) return;
    const uint32_t lo = lower_bound_u32(p.keys, p.n, v), hi = lower_bound_u32(p.keys, p.n, v + 1);
    double a[3] = {0.0, 0.0, 0.0};
    for (uint32_t i = lo + lane; i < hi; i += 32) {
        const uint32_t e = __ldg(p.vals + i);
        const uint64_t row = e >> 2;
        const double w = (double)slot_weight(p.bary, row, e & 3u);
        const float4 m = __ldg(p.gx + row);
        a[0] -= w * (double)m.x;
        a[1] -= w * (double)m.y;
        a[2] -= w * (double)m.z;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[c] += __shfl_xor_sync(0xffffffffu, a[c], o);
    if (lane == 0)
        for (int c = 0; c < 3; ++c) p.grad_xyz[3 * (size_t)v + c] = (float)a[c];
}

int launch_vertex_grads(const VertexGradsLaunch &a, cudaStream_t s) {
    if (a.keys == nullptr) {
        TN_CUDA(cudaMemsetAsync(a.grad_xyz, 0, sizeof(float) * 3 * (size_t)a.V, s));
        const uint64_t rows = (uint64_t)a.R * a.S;
        k_vertex_grads<<<(uint32_t)((rows + 255) / 256), 256, 0, s>>>(a);
    } else {
        k_det_vertex_grads<<<(uint32_t)(((uint64_t)a.V * 32 + 255) / 256), 256, 0, s>>>(a);
    }
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

}  // namespace tn
