// tn_ray_grads.cu -- gradients of the fused training step at the ray origins and directions (DESIGN.md §4.8), for a camera optimizer.
//
// The sample distances t_i (midpoints of the fine bins, what the matcher used) are constants, so a sample sits at x_i = o + t_i d.  The
// feature there is the tetrahedron's affine interpolant f(x) = F_v0 + sum_k b_k(x) (F_vk - F_v0), b(x) = E^-1 (x - x_v0), so with
// g_i = dL/df_i (the dX row of k_mlp_bwd) and q_ik = g_i . (F_vk - F_v0):
//   dL/dx_i = E_i^-T q_i,   dL/do = sum_i dL/dx_i,   dL/dd = sum_i t_i dL/dx_i + J_enc(d)^T W4[:, :27]^T g_dirbias.
// Unmatched samples and flat tetrahedra (det E = 0) contribute 0; empty rays get 0.
//
// k_ray_grads: one warp per active ray.  Per group of 32 samples, the warp forms each sample's q with coalesced float2 loads of its dX
// row and four field rows and a butterfly sum; the sample's lane keeps q and solves E^-T q in float64 (tn_tetsolve.cuh).  Every lane
// sums its samples in sample order, the lanes are combined by a fixed butterfly: the result does not depend on scheduling.
#include "tn_common.cuh"
#include "tn_direnc.cuh"
#include "tn_tetsolve.cuh"

namespace tn {

constexpr int RG_WARPS = 4;

__device__ __forceinline__ float warp_sum_fixed(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_fixed(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(RG_WARPS * 32) k_ray_grads(const RayGradsLaunch p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * RG_WARPS + warp;
    if (slot >= *p.n_active) return;
    const uint32_t S = p.S, ray = p.ray_list[slot];
    const float *eb = p.ebins + (size_t)slot * (S + 1);
    double go[3] = {0.0, 0.0, 0.0}, gd[3] = {0.0, 0.0, 0.0};  // this lane's samples: sum dL/dx, sum t dL/dx
    const uint32_t fp = field_pos(2u * (uint32_t)lane);  // where the lane's feature pair (2 lane, +1) sits in a field-shadow row
    for (uint32_t base = 0; base < S; base += 32) {
        const uint32_t j = base + (uint32_t)lane;
        const size_t row = (size_t)slot * S + j;
        const uint4 v = j < S ? __ldg(p.vi + row) : make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
        float q[3] = {0.f, 0.f, 0.f};  // q of sample `base + lane`
        const uint32_t m = min(32u, S - base);
        for (uint32_t k = 0; k < m; ++k) {
            const uint32_t v0 = __shfl_sync(0xffffffffu, v.x, k);
            if (v0 == TN_EMPTY) continue;  // (warp-uniform)
            const uint32_t v1 = __shfl_sync(0xffffffffu, v.y, k), v2 = __shfl_sync(0xffffffffu, v.z, k), v3 = __shfl_sync(0xffffffffu, v.w, k);
            const float2 g = __ldg(reinterpret_cast<const float2 *>(p.dx + ((size_t)slot * S + base + k) * 64) + lane);
            const float2 f0 = __ldg(reinterpret_cast<const float2 *>(p.fshadow + (size_t)v0 * 64 + fp));
            const float2 f1 = __ldg(reinterpret_cast<const float2 *>(p.fshadow + (size_t)v1 * 64 + fp));
            const float2 f2 = __ldg(reinterpret_cast<const float2 *>(p.fshadow + (size_t)v2 * 64 + fp));
            const float2 f3 = __ldg(reinterpret_cast<const float2 *>(p.fshadow + (size_t)v3 * 64 + fp));
            float a = fmaf(g.y, f1.y - f0.y, g.x * (f1.x - f0.x));
            float b = fmaf(g.y, f2.y - f0.y, g.x * (f2.x - f0.x));
            float c = fmaf(g.y, f3.y - f0.y, g.x * (f3.x - f0.x));
            a = warp_sum_fixed(a); b = warp_sum_fixed(b); c = warp_sum_fixed(c);
            if ((uint32_t)lane == k) { q[0] = a; q[1] = b; q[2] = c; }
        }
        if (j < S) {
            float4 gx = make_float4(0.f, 0.f, 0.f, 0.f);
            if (v.x != TN_EMPTY) {
                const uint32_t vs[4] = {v.x, v.y, v.z, v.w};
                double cf[3][3], det;
                tet_cofactors(p.xyz, vs, cf, det);
                if (det != 0.0) {
                    const double inv = 1.0 / det;
                    double x[3];
#pragma unroll
                    for (int c = 0; c < 3; ++c) x[c] = ((double)q[0] * cf[0][c] + (double)q[1] * cf[1][c] + (double)q[2] * cf[2][c]) * inv;
                    const double t = (double)((eb[j + 1] + eb[j]) / 2.f);  // the distance the sample was matched at (k_sample_fine)
#pragma unroll
                    for (int c = 0; c < 3; ++c) { go[c] += x[c]; gd[c] = fma(t, x[c], gd[c]); }
                    gx = make_float4((float)x[0], (float)x[1], (float)x[2], 0.f);
                }
            }
            p.gx[row] = gx;
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { go[c] = warp_sum_fixed(go[c]); gd[c] = warp_sum_fixed(gd[c]); }
    // direction encoding: lane k < 27 forms h_k = (W4[:, :27]^T g_dirbias)_k and its term h_k d enc_k / d d_axis
    const float *enc = p.enc + (size_t)slot * 27;
    const float dx = enc[24], dy = enc[25], dz = enc[26];
    float e[3] = {0.f, 0.f, 0.f};
    if (lane < 27) {
        const float *gdb = p.g_dirbias + (size_t)slot * 128;
        float h = 0.f;
        for (int o = 0; o < 128; ++o) h = fmaf(__ldg(p.w4dir + o * 27 + lane), __ldg(gdb + o), h);
        int axis = 0;
        const float jac = encode_direction_deriv(lane, dx, dy, dz, axis);
        e[axis] = h * jac;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) e[c] = warp_sum_fixed(e[c]);
    if (lane == 0) {
        if (p.grad_o != nullptr)
            for (int c = 0; c < 3; ++c) p.grad_o[3 * (size_t)ray + c] = (float)go[c];
        if (p.grad_d != nullptr)
            for (int c = 0; c < 3; ++c) p.grad_d[3 * (size_t)ray + c] = (float)(gd[c] + (double)e[c]);
    }
}

int launch_ray_grads(const RayGradsLaunch &a, cudaStream_t s) {
    // every ray's gradients: 0 for the empty ones, written by k_ray_grads for the others
    if (a.grad_o != nullptr) TN_CUDA(cudaMemsetAsync(a.grad_o, 0, sizeof(float) * 3 * (size_t)a.R, s));
    if (a.grad_d != nullptr) TN_CUDA(cudaMemsetAsync(a.grad_d, 0, sizeof(float) * 3 * (size_t)a.R, s));
    k_ray_grads<<<(a.R + RG_WARPS - 1) / RG_WARPS, RG_WARPS * 32, 0, s>>>(a);
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

}  // namespace tn
