// tn_composite.cuh -- warp-level scans and RaySamples.get_weights, shared by the compositing kernels of the fused render
// (tn_render.cu) and the normal-map compositing (tn_normals.cu), so that both derive their weights from the same code (static: each
// translation unit keeps its own copy).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tn {

__device__ __forceinline__ float warp_incl_scan_f(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// in-place inclusive scan of a[0..n) in shared memory by one warp; returns the total
static __device__ float smem_scan_add(float *a, uint32_t n, int lane) {
    float carry = 0.f;
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t i = base + lane;
        float v = i < n ? a[i] : 0.f;
        v = warp_incl_scan_f(v, lane) + carry;
        if (i < n) a[i] = v;
        carry = __shfl_sync(0xffffffffu, v, 31);
    }
    __syncwarp();
    return carry;
}
__device__ __forceinline__ float nan_to_num_f(float x) {  // torch.nan_to_num defaults
    if (isnan(x)) return 0.f;
    if (isinf(x)) return x > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
    return x;
}

// RaySamples.get_weights on staged deltas/densities: w[j] (in place over `dd`), using `tr` as scratch
static __device__ void weights_from_density(float *dd, float *tr, uint32_t S, int lane) {
    for (uint32_t j = lane; j < S; j += 32) tr[j] = dd[j];
    __syncwarp();
    smem_scan_add(tr, S, lane);  // inclusive cumsum of delta*density
    for (uint32_t j = lane; j < S; j += 32) {
        const float excl = j == 0 ? 0.f : tr[j - 1];
        const float alpha = 1.f - expf(-dd[j]);
        const float T = expf(-excl);
        dd[j] = nan_to_num_f(alpha * T);
    }
    __syncwarp();
}

}  // namespace tn
