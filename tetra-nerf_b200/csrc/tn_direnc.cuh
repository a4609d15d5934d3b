// tn_direnc.cuh -- the direction encoding of the colour head, shared by the render (k_sample_fine / k_dirbias_only) and the surface
// extraction (tn_surface.cu).
#pragma once
#include <cuda_runtime.h>

namespace tn {

// NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0, max_freq_exp=4, include_input=True), model.py:426-432:
// enc = [sin(2 pi d_a f) for a, f] ++ [sin(2 pi d_a f + pi/2) for a, f] ++ d
__device__ __forceinline__ void encode_direction(float dx, float dy, float dz, float (&enc)[27]) {
    const float dd[3] = {dx, dy, dz};
    const float two_pi = 6.283185307179586f, half_pi = 1.5707963267948966f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float sc = two_pi * dd[a];
#pragma unroll
        for (int f = 0; f < 4; ++f) {
            const float freq = f == 0 ? 1.0f : (f == 1 ? 2.5198421f : (f == 2 ? 6.3496042f : 16.0f));  // 2**linspace(0,4,4)
            const float si = sc * freq;
            enc[a * 4 + f] = sinf(si);
            enc[12 + a * 4 + f] = sinf(si + half_pi);
        }
        enc[24 + a] = dd[a];
    }
}

// the Jacobian of encode_direction: entry k depends on the direction's component `axis` only; returns d enc[k] / d d_axis
// (sin(s f d_a) -> s f cos(s f d_a), sin(s f d_a + pi/2) -> s f cos(s f d_a + pi/2), d_a -> 1; s = 2 pi)
__device__ __forceinline__ float encode_direction_deriv(int k, float dx, float dy, float dz, int &axis) {
    const float two_pi = 6.283185307179586f, half_pi = 1.5707963267948966f;
    if (k >= 24) { axis = k - 24; return 1.0f; }
    const int a = (k % 12) / 4, f = k % 4;
    axis = a;
    const float da = a == 0 ? dx : (a == 1 ? dy : dz);
    const float freq = f == 0 ? 1.0f : (f == 1 ? 2.5198421f : (f == 2 ? 6.3496042f : 16.0f));
    const float si = two_pi * da * freq;
    return two_pi * freq * cosf(k < 12 ? si : si + half_pi);
}

}  // namespace tn
