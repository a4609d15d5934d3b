// tn_background.cu -- the training backward of the learned background (DESIGN.md §4.16): with s = grad_rgb (1 - accumulation) per ray
// (grad_rgb on empty rays), the map gradient is s scattered to each ray's four texels with their bilinear weights, and the direction
// gradient gains (d bg / d d)^T s on every ray.
//   default mode:       one thread per ray, float atomics into the map gradient;
//   deterministic mode: one thread per ray writes its four (texel, 4 ray + corner) pairs, a stable radix sort orders them by texel, and
//                       one thread per texel sums its entries in sorted (= ray, corner) order -- the same shape as the field gradient's
//                       k_det_field_keys / k_det_field_grad, so the map gradient is bitwise reproducible.
// The direction term is per ray, without reductions, in both modes.
#include <cub/cub.cuh>

#include "tn_background.cuh"
#include "tn_common.cuh"
#include "tn_sort.cuh"

namespace tn {

__device__ __forceinline__ float bg_corner_weight(const BgTaps &t, uint32_t k) {  // bilinear weight of corner k (00, 01, 10, 11)
    const float wu = (k & 1u) ? t.fu : 1.f - t.fu, wv = (k & 2u) ? t.fv : 1.f - t.fv;
    return wu * wv;
}

template <bool DET>
__global__ void __launch_bounds__(256) k_bg_rays(const BackgroundGradsLaunch p) {
    const uint32_t ray = blockIdx.x * blockDim.x + threadIdx.x;
    if (ray >= p.R) return;
    const float *d = p.dirs + 3 * (size_t)ray;
    const BgTaps t = bg_taps(p.H, p.W, d[0], d[1], d[2]);
    const float s[3] = {p.s[3 * (size_t)ray], p.s[3 * (size_t)ray + 1], p.s[3 * (size_t)ray + 2]};
    const uint32_t tex[4] = {t.t00, t.t01, t.t10, t.t11};
    if constexpr (DET) {
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) { p.keys[4 * (size_t)ray + k] = tex[k]; p.vals[4 * (size_t)ray + k] = 4u * ray + k; }
    } else if (p.grad_map != nullptr) {
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
            const float w = bg_corner_weight(t, k);
#pragma unroll
            for (int c = 0; c < 3; ++c) atomicAdd(p.grad_map + 3 * (size_t)tex[k] + c, w * s[c]);
        }
    }
    if (p.grad_d != nullptr) {
        float g[3];
        bg_grad_direction(p.map, p.H, p.W, t, s, g);
#pragma unroll
        for (int c = 0; c < 3; ++c) p.grad_d[3 * (size_t)ray + c] += g[c];
    }
}

// deterministic mode, after the sort: texel x sums w_k s over its entries in sorted order
__global__ void __launch_bounds__(256) k_bg_texels(const BackgroundGradsLaunch p, const uint32_t *__restrict__ keys,
                                                   const uint32_t *__restrict__ vals) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= p.H * p.W) return;
    const uint32_t n = 4 * p.R, lo = lower_bound_u32(keys, n, x), hi = lower_bound_u32(keys, n, x + 1);
    float acc[3] = {0.f, 0.f, 0.f};
    for (uint32_t e = lo; e < hi; ++e) {
        const uint32_t v = __ldg(vals + e), ray = v >> 2;
        const float *d = p.dirs + 3 * (size_t)ray;
        const float w = bg_corner_weight(bg_taps(p.H, p.W, d[0], d[1], d[2]), v & 3u);
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = fmaf(w, p.s[3 * (size_t)ray + c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) p.grad_map[3 * (size_t)x + c] = acc[c];
}

int launch_background_grads(const BackgroundGradsLaunch &a, DevArray<uint8_t> &tmp, cudaStream_t s) {
    const uint32_t blocks = (a.R + 255) / 256;
    if (!a.det || a.grad_map == nullptr) {  // (without a map gradient only the per-ray direction term is left)
        if (a.grad_map != nullptr) TN_CUDA(cudaMemsetAsync(a.grad_map, 0, sizeof(float) * 3 * (size_t)a.H * a.W, s));
        k_bg_rays<false><<<blocks, 256, 0, s>>>(a);
    } else {
        k_bg_rays<true><<<blocks, 256, 0, s>>>(a);
        const uint32_t n = 4 * a.R;
        const int end_bit = radix_end_bit(a.H * a.W);
        TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
            return cub::DeviceRadixSort::SortPairs(t, bytes, a.keys, a.keys + n, a.vals, a.vals + n, (int)n, 0, end_bit, s);
        }));
        k_bg_texels<<<(a.H * a.W + 255) / 256, 256, 0, s>>>(a, a.keys + n, a.vals + n);
    }
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

}  // namespace tn
