// tn_background.cuh -- the learned direction-dependent background (DESIGN.md §4.16): the lookup the pixel-writing kernels of the fused
// render composite with, and its derivatives for the training backward (tn_background.cu).
//
// B f32[H,W,3], W = 2H, row-major, in the model's world frame (z up).  For a ray direction d, n = d / |d|:
//   u = W (atan2(n_y, n_x) / 2 pi + 1/2) - 1/2   (columns taken modulo W: the map wraps in u)
//   v = H (1 - n_z) / 2 - 1/2, clamped to [0, H - 1]   (equal-area in v)
//   i0 = floor(u), fu = u - i0;  j0 = floor(v), j1 = min(j0 + 1, H - 1), fv = v - j0
//   bg(d) = lerp(lerp(B[j0,i0], B[j0,i0+1], fu), lerp(B[j1,i0], B[j1,i0+1], fu), fv),  lerp(a, b, t) = a + t (b - a)
// In that form a constant map returns its constant exactly, so an all-c map gives the bits of the constant background c.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tn {

// below this n_x^2 + n_y^2 (|n_z| > 1 - 5e-9) the u-derivative is taken as 0: at the poles u is undefined and its derivative
// ~ W / (2 pi rho) unbounded, while bg itself stays continuous there (every column of the clamped row meets at the pole)
constexpr float BG_POLE_EPS = 1e-8f;

struct BgTaps {
    uint32_t t00, t01, t10, t11;  // texel indices j * W + i of B[j0,i0], B[j0,i1], B[j1,i0], B[j1,i1]
    float fu, fv;
    bool v_in;                    // v was not clamped (its derivative counts)
    float nx, ny, nz, inv_len;    // the unit direction and 1 / |d|
};

__device__ __forceinline__ BgTaps bg_taps(uint32_t H, uint32_t W, float dx, float dy, float dz) {
    BgTaps t;
    t.inv_len = 1.f / sqrtf(dx * dx + dy * dy + dz * dz);
    t.nx = dx * t.inv_len; t.ny = dy * t.inv_len; t.nz = dz * t.inv_len;
    const float u = (float)W * (atan2f(t.ny, t.nx) * 0.15915494309189535f + 0.5f) - 0.5f;
    const float v_raw = (float)H * (1.f - t.nz) * 0.5f - 0.5f;
    const float v = fminf(fmaxf(v_raw, 0.f), (float)(H - 1));  // (a NaN direction clamps to row 0: no index leaves the map)
    t.v_in = v_raw >= 0.f && v_raw <= (float)(H - 1);
    const float fi = floorf(u), fj = floorf(v);
    t.fu = u - fi; t.fv = v - fj;
    int i0 = (int)fi % (int)W;
    if (i0 < 0) i0 += (int)W;
    const uint32_t i1 = (uint32_t)i0 + 1u == W ? 0u : (uint32_t)i0 + 1u;
    const uint32_t j0 = min((uint32_t)fj, H - 1), j1 = min(j0 + 1u, H - 1);
    t.t00 = j0 * W + (uint32_t)i0; t.t01 = j0 * W + i1; t.t10 = j1 * W + (uint32_t)i0; t.t11 = j1 * W + i1;
    return t;
}

__device__ __forceinline__ float bg_lerp(float a, float b, float t) { return a + t * (b - a); }

// bg(d), channel c, of the taps
__device__ __forceinline__ float bg_channel(const float *__restrict__ B, const BgTaps &t, int c) {
    const float top = bg_lerp(__ldg(B + 3 * (size_t)t.t00 + c), __ldg(B + 3 * (size_t)t.t01 + c), t.fu);
    const float bot = bg_lerp(__ldg(B + 3 * (size_t)t.t10 + c), __ldg(B + 3 * (size_t)t.t11 + c), t.fu);
    return bg_lerp(top, bot, t.fv);
}

__device__ __forceinline__ void bg_lookup(const float *__restrict__ B, uint32_t H, uint32_t W, float dx, float dy, float dz, float &r,
                                          float &g, float &b) {
    const BgTaps t = bg_taps(H, W, dx, dy, dz);
    r = bg_channel(B, t, 0); g = bg_channel(B, t, 1); b = bg_channel(B, t, 2);
}

// (d bg / d d)^T s for the per-channel weights s: through dbg/du, dbg/dv, then u(n), v(n) and n = d / |d|
__device__ __forceinline__ void bg_grad_direction(const float *__restrict__ B, uint32_t H, uint32_t W, const BgTaps &t, const float s[3],
                                                  float out[3]) {
    float gu = 0.f, gv = 0.f;  // s . dbg/du, s . dbg/dv
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float b00 = __ldg(B + 3 * (size_t)t.t00 + c), b01 = __ldg(B + 3 * (size_t)t.t01 + c);
        const float b10 = __ldg(B + 3 * (size_t)t.t10 + c), b11 = __ldg(B + 3 * (size_t)t.t11 + c);
        gu += s[c] * ((1.f - t.fv) * (b01 - b00) + t.fv * (b11 - b10));
        gv += s[c] * (bg_lerp(b10, b11, t.fu) - bg_lerp(b00, b01, t.fu));
    }
    const float rho2 = t.nx * t.nx + t.ny * t.ny;
    float gn[3] = {0.f, 0.f, 0.f};  // dL/dn
    if (rho2 >= BG_POLE_EPS) {      // du/dn = W / (2 pi rho^2) (-n_y, n_x, 0)
        const float k = gu * (float)W * 0.15915494309189535f / rho2;
        gn[0] = -k * t.ny; gn[1] = k * t.nx;
    }
    if (t.v_in) gn[2] = gv * (-0.5f * (float)H);  // dv/dn_z = -H / 2
    const float dot = gn[0] * t.nx + gn[1] * t.ny + gn[2] * t.nz;  // dn/dd = (I - n n^T) / |d|
    out[0] = (gn[0] - dot * t.nx) * t.inv_len;
    out[1] = (gn[1] - dot * t.ny) * t.inv_len;
    out[2] = (gn[2] - dot * t.nz) * t.inv_len;
}

}  // namespace tn
