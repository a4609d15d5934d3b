// tn_ops.cu -- find_visited_cells, interpolate_values, interpolate_values_backward (stand-alone ops
// of the pybind surface; the fused render path in tn_render.cu does the same arithmetic in-kernel).
//
// Replaces src/tetrahedra_tracer.cu:115-290.  Arithmetic contract with oracle/tetra_oracle.cpp:
//   matcher : mult = (d - t_in) / (t_out - t_in)  [IEEE div],  b = (1-mult)*c1 + mult*c2 with every
//             op individually rounded (the reference is built --use_fast_math, cmake/FindTorch.cmake:33;
//             its result differs by a few ulp and is checked against oracle/_ref on the GPU box);
//   interp  : out = fma(w_k, F[v_{k+1}], out) for k = 0..D-2, then fma(1 - sum(w), F[v_0], out)
//             -- the FFMA chain nvcc emits for tetrahedra_tracer.cu:211-219.
#include <cub/cub.cuh>

#include "tn_common.cuh"

namespace tn {

// ---- find_matched_cells (tetrahedra_tracer.cu:115-161) : literal, one thread per ray ----------
__global__ void k_match(uint32_t R, uint32_t S, uint32_t M, const uint32_t *__restrict__ num, const uint32_t *__restrict__ cells,
                        const float2 *__restrict__ hd, const float *__restrict__ bary, const float *__restrict__ sd,
                        const uint4 *__restrict__ verts, uint32_t *__restrict__ cell_out, uint4 *__restrict__ verts_out,
                        uint8_t *__restrict__ mask_out, float *__restrict__ bary_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    const uint32_t n = num[i];
    const size_t row = (size_t)i * M;
    uint32_t p = 0;
    bool done = false;
    for (uint32_t j = 0; j < S; ++j) {
        const size_t g = (size_t)i * S + j;
        uint32_t oc = TN_EMPTY;
        uint4 ov = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
        uint8_t om = 0;
        float b0 = 0.f, b1 = 0.f, b2 = 0.f;
        if (!done) {
            const float cd = sd[g];
            while (p < n && hd[row + p].y < cd) p++;
            if (p >= n) done = true;  // "there will be no more matches on this ray" (:137-140)
            else {
                const float2 h = hd[row + p];
                if (h.x <= cd) {
                    om = 1;
                    oc = cells[row + p];
                    ov = verts[row + p];
                    const float mult = __fdiv_rn(__fsub_rn(cd, h.x), __fsub_rn(h.y, h.x));
                    const float omm = __fsub_rn(1.0f, mult);
                    const float *c = bary + 6 * (row + p);
                    b0 = __fadd_rn(__fmul_rn(omm, c[0]), __fmul_rn(mult, c[3]));
                    b1 = __fadd_rn(__fmul_rn(omm, c[1]), __fmul_rn(mult, c[4]));
                    b2 = __fadd_rn(__fmul_rn(omm, c[2]), __fmul_rn(mult, c[5]));
                }
            }
        }
        cell_out[g] = oc; verts_out[g] = ov; mask_out[g] = om;
        bary_out[3 * g] = b0; bary_out[3 * g + 1] = b1; bary_out[3 * g + 2] = b2;
    }
}

// ---- find_matched_cells, one warp per ray ---------------------------------------------------------
// The reference's loop (tetrahedra_tracer.cu:129-160) is serial in the samples only through its pointer p, which never moves
// back: p_j = first p >= p_{j-1} with t_out[p] >= d_j.  When t_out is non-decreasing along the ray (checked per ray; true
// unless sub-eps slivers were swapped by the pairing) this is a running maximum of independent lower bounds,
// p_j = max_{i<=j} lower_bound(t_out, d_i) -- for sorted AND for unsorted samples -- so the warp takes 32 samples at a time:
// binary search in shared memory, warp max-scan, carry.  Rays that fail the check run the literal loop on one lane.
constexpr int MATCH_WARPS = 4;
__global__ void __launch_bounds__(MATCH_WARPS * 32) k_match_warp(uint32_t R, uint32_t S, uint32_t M, const uint32_t *__restrict__ num,
                                                                 const uint32_t *__restrict__ cells, const float2 *__restrict__ hd,
                                                                 const float *__restrict__ bary, const float *__restrict__ sd,
                                                                 const uint4 *__restrict__ verts, uint32_t *__restrict__ cell_out,
                                                                 uint4 *__restrict__ verts_out, uint8_t *__restrict__ mask_out,
                                                                 float *__restrict__ bary_out) {
    extern __shared__ float s_tout[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * MATCH_WARPS + warp;
    if (i >= R) return;
    float *t_out = s_tout + (size_t)warp * M;
    const uint32_t n = min(num[i], M);
    const size_t row = (size_t)i * M;
    for (uint32_t k = lane; k < n; k += 32) t_out[k] = hd[row + k].y;
    __syncwarp();
    bool mono = true;
    for (uint32_t k = lane + 1; k < n; k += 32) mono = mono && !(t_out[k] < t_out[k - 1]);
    mono = __all_sync(0xffffffffu, mono);
    uint32_t carry = 0;     // the reference's pointer p after the previous sample
    bool done = false;      // (only used by the literal fallback)
    for (uint32_t base = 0; base < S; base += 32) {
        const uint32_t j = base + (uint32_t)lane;
        const bool valid = j < S;
        const size_t g = (size_t)i * S + j;
        const float cd = valid ? sd[g] : 0.f;
        uint32_t p;
        if (mono) {
            uint32_t lo = 0, hi = valid ? n : 0u;  // first p with t_out[p] >= cd  (a NaN sample compares false: lo stays 0, as the loop)
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (t_out[mid] < cd) lo = mid + 1; else hi = mid; }
            p = lo;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t q = __shfl_up_sync(0xffffffffu, p, o); if (lane >= o) p = max(p, q); }
            p = max(p, carry);
            carry = __shfl_sync(0xffffffffu, p, 31);
        } else {
            // literal pointer walk for this group of 32 samples, one lane, results broadcast
            uint32_t mine = n;
            if (lane == 0) {
                for (uint32_t q = 0; q < 32 && base + q < S; ++q) {
                    uint32_t pq = n;
                    if (!done) {
                        const float c = sd[(size_t)i * S + base + q];
                        while (carry < n && t_out[carry] < c) carry++;
                        if (carry >= n) done = true;
                        pq = carry;
                    }
                    s_tout[MATCH_WARPS * (size_t)M + warp * 32 + q] = __uint_as_float(pq);
                }
            }
            __syncwarp();
            mine = __float_as_uint(s_tout[MATCH_WARPS * (size_t)M + warp * 32 + lane]);
            __syncwarp();
            p = mine;
        }
        if (!valid) continue;
        uint32_t oc = TN_EMPTY;
        uint4 ov = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
        uint8_t om = 0;
        float b0 = 0.f, b1 = 0.f, b2 = 0.f;
        if (p < n) {  // p >= n: "there will be no more matches on this ray" (:137-140)
            const float2 h = hd[row + p];
            if (h.x <= cd) {
                om = 1;
                oc = cells[row + p];
                ov = verts[row + p];
                const float mult = __fdiv_rn(__fsub_rn(cd, h.x), __fsub_rn(h.y, h.x));
                const float omm = __fsub_rn(1.0f, mult);
                const float *c = bary + 6 * (row + p);
                b0 = __fadd_rn(__fmul_rn(omm, c[0]), __fmul_rn(mult, c[3]));
                b1 = __fadd_rn(__fmul_rn(omm, c[1]), __fmul_rn(mult, c[4]));
                b2 = __fadd_rn(__fmul_rn(omm, c[2]), __fmul_rn(mult, c[5]));
            }
        }
        cell_out[g] = oc; verts_out[g] = ov; mask_out[g] = om;
        bary_out[3 * g] = b0; bary_out[3 * g + 1] = b1; bary_out[3 * g + 2] = b2;
    }
}

// ---- [C,V] -> [V,C] ---------------------------------------------------------------------------
// rows_on_x: the row tiles are indexed by blockIdx.x (the grid's y extent is limited to 65535 blocks: the LONG dimension,
// the vertex count, must always travel on x)
__global__ void k_transpose(const float *__restrict__ in, float *__restrict__ out, uint32_t rows, uint32_t cols, bool rows_on_x) {
    __shared__ float tile[32][33];
    const uint32_t bx = (rows_on_x ? blockIdx.y : blockIdx.x) * 32, by = (rows_on_x ? blockIdx.x : blockIdx.y) * 32;
    for (uint32_t r = threadIdx.y; r < 32; r += blockDim.y) {
        const uint32_t y = by + r, x = bx + threadIdx.x;
        if (y < rows && x < cols) tile[r][threadIdx.x] = in[(size_t)y * cols + x];
    }
    __syncthreads();
    for (uint32_t r = threadIdx.y; r < 32; r += blockDim.y) {
        const uint32_t x = bx + r, y = by + threadIdx.x;
        if (y < rows && x < cols) out[(size_t)x * rows + y] = tile[threadIdx.x][r];
    }
}

// ---- interpolate_values (tetrahedra_tracer.cu:195-221) ----------------------------------------
// row-major field [V,C]: one warp per sample, lanes over features (coalesced 4C-byte vertex rows)
template <int D>
__global__ void k_interp_rows(uint32_t N, uint32_t C, const uint32_t *__restrict__ vi, const float *__restrict__ w,
                              const float *__restrict__ frow, float *__restrict__ out) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= N) return;
    uint32_t v[D];
    float wk[D];
    float weight = 0.f;
#pragma unroll
    for (int k = 0; k < D; ++k) v[k] = vi[(size_t)i * D + k];
#pragma unroll
    for (int k = 0; k < D - 1; ++k) { wk[k] = w[(size_t)i * (D - 1) + k]; weight = __fadd_rn(weight, wk[k]); }
    const float w0 = __fsub_rn(1.0f, weight);
    for (uint32_t j = lane; j < C; j += 32) {
        float o = 0.f;
#pragma unroll
        for (int k = 0; k < D - 1; ++k)
            if (v[k + 1] != TN_EMPTY) o = __fmaf_rn(wk[k], frow[(size_t)v[k + 1] * C + j], o);
        if (v[0] != TN_EMPTY) o = __fmaf_rn(w0, frow[(size_t)v[0] * C + j], o);
        out[(size_t)i * C + j] = o;
    }
}
// C == 64 (the model's field_dim): half a warp per sample, 4 features per lane -> every vertex row is one 256-byte burst of
// 16-byte loads and two samples share each instruction; same FMA chain per element as k_interp_rows
template <int D>
__global__ void k_interp_rows64(uint32_t N, const uint32_t *__restrict__ vi, const float *__restrict__ w, const float4 *__restrict__ frow,
                                float4 *__restrict__ out) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const uint32_t l16 = threadIdx.x & 15u;
    if (i >= N) return;
    uint32_t v[D];
    float wk[D];
    float weight = 0.f;
#pragma unroll
    for (int k = 0; k < D; ++k) v[k] = vi[(size_t)i * D + k];
#pragma unroll
    for (int k = 0; k < D - 1; ++k) { wk[k] = w[(size_t)i * (D - 1) + k]; weight = __fadd_rn(weight, wk[k]); }
    const float w0 = __fsub_rn(1.0f, weight);
    float4 f[D];
#pragma unroll
    for (int k = 0; k < D; ++k) f[k] = v[k] != TN_EMPTY ? __ldg(frow + (size_t)v[k] * 16 + l16) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < D - 1; ++k)
        if (v[k + 1] != TN_EMPTY) {
            o.x = __fmaf_rn(wk[k], f[k + 1].x, o.x); o.y = __fmaf_rn(wk[k], f[k + 1].y, o.y);
            o.z = __fmaf_rn(wk[k], f[k + 1].z, o.z); o.w = __fmaf_rn(wk[k], f[k + 1].w, o.w);
        }
    if (v[0] != TN_EMPTY) {
        o.x = __fmaf_rn(w0, f[0].x, o.x); o.y = __fmaf_rn(w0, f[0].y, o.y);
        o.z = __fmaf_rn(w0, f[0].z, o.z); o.w = __fmaf_rn(w0, f[0].w, o.w);
    }
    out[(size_t)i * 16 + l16] = o;
}

// ---- interpolate_values_backward (tetrahedra_tracer.cu:223-248) -------------------------------
template <int D>
__global__ void k_interp_bwd(uint32_t N, uint32_t C, uint32_t V, const uint32_t *__restrict__ vi, const float *__restrict__ w,
                             const float *__restrict__ gin, float *__restrict__ gfield) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)N * C) return;
    const uint32_t i = (uint32_t)(idx / C), j = (uint32_t)(idx % C);
    const float g = gin[idx];
    float weight = 0.f;
#pragma unroll
    for (int k = 0; k < D - 1; ++k) {
        const float wk = w[(size_t)i * (D - 1) + k];
        const uint32_t v = vi[(size_t)i * D + k + 1];
        if (v != TN_EMPTY) atomicAdd(&gfield[(size_t)j * V + v], __fmul_rn(wk, g));
        weight = __fadd_rn(weight, wk);
    }
    const uint32_t v0 = vi[(size_t)i * D];
    if (v0 != TN_EMPTY) atomicAdd(&gfield[(size_t)j * V + v0], __fmul_rn(__fsub_rn(1.0f, weight), g));
}

// `shadow`: the [V,C] row-major shadow of the field (tn_make_field_shadow)
template <int D>
static void interp_fwd(uint32_t N, uint32_t C, const uint32_t *vi, const float *w, const float *shadow, float *out, cudaStream_t s) {
    const uint32_t threads = 256;
    if (C == 64 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)shadow & 15) == 0)
        k_interp_rows64<D><<<(uint32_t)(((size_t)N * 16 + threads - 1) / threads), threads, 0, s>>>(N, vi, w, (const float4 *)shadow, (float4 *)out);
    else
        k_interp_rows<D><<<(uint32_t)(((size_t)N * 32 + threads - 1) / threads), threads, 0, s>>>(N, C, vi, w, shadow, out);
}
// The same sums accumulated into a row-major [V,C] shadow: lane l of a (sample, vertex) pair adds 4 consecutive features
// with ONE 16-byte vector reduction (red.global.add.v4.f32, sm_90+), so a vertex row takes C/4 coalesced atomics instead of
// C scalar ones spread over C different cache lines of the feature-major gradient.  The caller transposes the shadow.
template <int D>
__global__ void k_interp_bwd_rows(uint32_t N, uint32_t C4, const uint32_t *__restrict__ vi, const float *__restrict__ w,
                                  const float4 *__restrict__ gin, float4 *__restrict__ grow) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // (sample, 4-feature group)
    if (idx >= (size_t)N * C4) return;
    const uint32_t i = (uint32_t)(idx / C4), j = (uint32_t)(idx % C4);
    const float4 g = __ldg(gin + idx);
    float weight = 0.f;
#pragma unroll
    for (int k = 0; k < D; ++k) {
        // k < D-1: vertex k+1 with weight w[k]; k == D-1: vertex 0 with the remaining weight (tetrahedra_tracer.cu:231-247)
        float wk;
        uint32_t v;
        if (k < D - 1) { wk = w[(size_t)i * (D - 1) + k]; v = vi[(size_t)i * D + k + 1]; weight = __fadd_rn(weight, wk); }
        else { wk = __fsub_rn(1.0f, weight); v = vi[(size_t)i * D]; }
        if (v == TN_EMPTY) continue;
        float4 *dst = grow + (size_t)v * C4 + j;
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(__fmul_rn(wk, g.x)), "f"(__fmul_rn(wk, g.y)),
                     "f"(__fmul_rn(wk, g.z)), "f"(__fmul_rn(wk, g.w))
                     : "memory");
    }
}

template <int D>
static int interp_bwd(uint32_t N, uint32_t C, uint32_t V, const uint32_t *vi, const float *w, const float *gin, float *gfield,
                      float *scratch, cudaStream_t s) {
    if (scratch && (C & 3u) == 0 && ((uintptr_t)gin & 15) == 0 && ((uintptr_t)scratch & 15) == 0) {
        TN_CUDA(cudaMemsetAsync(scratch, 0, sizeof(float) * (size_t)C * V, s));
        const size_t total = (size_t)N * (C / 4);
        k_interp_bwd_rows<D><<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(N, C / 4, vi, w, (const float4 *)gin, (float4 *)scratch);
        dim3 tb(32, 8), tg((V + 31) / 32, (C + 31) / 32);
        k_transpose<<<tg, tb, 0, s>>>(scratch, gfield, V, C, true);  // [V,C] -> [C,V]
        return TN_OK;
    }
    TN_CUDA(cudaMemsetAsync(gfield, 0, sizeof(float) * (size_t)C * V, s));  // py_binding.cpp:360
    const size_t total = (size_t)N * C;
    k_interp_bwd<D><<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(N, C, V, vi, w, gin, gfield);
    return TN_OK;
}

// ---- deterministic interpolate_values_backward --------------------------------------------------------------------------------
// The (vertex, entry) pairs of the N x D vertex slots (entry = i * D + k) are sorted by vertex with a stable radix sort (the input is
// in entry order, so equal vertices keep it); then one warp per vertex sums w_k g[i] over its entries in that order into a row-major
// [V,C] accumulator, which is transposed to [C,V].  The products are the reference's (__fmul_rn(w_k, g)); only the order of the sum
// is fixed, so the result does not depend on scheduling.
__global__ void k_ivb_keys(uint32_t n, uint32_t V, const uint32_t *__restrict__ vi, uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const uint32_t v = vi[e];
    keys[e] = v < V ? v : V;  // empty slots (E) sort behind every vertex
    vals[e] = e;
}
__device__ __forceinline__ uint32_t lower_bound_keys(const uint32_t *__restrict__ a, uint32_t n, uint32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(a + mid) < x) lo = mid + 1; else hi = mid; }
    return lo;
}
template <int D>
__global__ void __launch_bounds__(256) k_ivb_det(uint32_t V, uint32_t C, uint32_t n, const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                 const float *__restrict__ w, const float *__restrict__ gin, float *__restrict__ grow) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (v >= V) return;
    const uint32_t lo = lower_bound_keys(keys, n, v), hi = lower_bound_keys(keys, n, v + 1);
    for (uint32_t c0 = 0; c0 < C; c0 += 32) {
        const uint32_t c = c0 + lane;
        float acc = 0.f;
        for (uint32_t b = lo; b < hi; b += 32) {
            uint32_t i = 0;
            float wk = 0.f;
            if (b + lane < hi) {  // this lane's entry: sample i, vertex slot k (k_interp_bwd: slot k >= 1 has w[k-1], slot 0 the rest)
                const uint32_t e = __ldg(vals + b + lane), k = e % D;
                i = e / D;
                if (k > 0) wk = __ldg(w + (size_t)i * (D - 1) + k - 1);
                else {
                    float weight = 0.f;
#pragma unroll
                    for (int q = 0; q < D - 1; ++q) weight = __fadd_rn(weight, __ldg(w + (size_t)i * (D - 1) + q));
                    wk = __fsub_rn(1.0f, weight);
                }
            }
            const uint32_t m = min(32u, hi - b);
            for (uint32_t j = 0; j < m; ++j) {
                const uint32_t ij = __shfl_sync(0xffffffffu, i, j);
                const float wj = __shfl_sync(0xffffffffu, wk, j);
                if (c < C) acc = __fadd_rn(acc, __fmul_rn(wj, __ldg(gin + (size_t)ij * C + c)));
            }
        }
        if (c < C) grow[(size_t)v * C + c] = acc;
    }
}

}  // namespace tn

extern "C" int tn_find_visited_cells(tn_tracer *h, uint32_t R, uint32_t S, uint32_t M, const uint32_t *d_num, const uint32_t *d_cells,
                                     const float *d_bary, const float *d_dist, const uint32_t *d_verts, const float *d_sample_dist,
                                     uint32_t *d_cell_out, uint32_t *d_verts_out, uint8_t *d_mask_out, float *d_bary_out, void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (R == 0 || S == 0) return TN_OK;
    tn::DeviceGuard g(h->device);
    const size_t smem = sizeof(float) * ((size_t)tn::MATCH_WARPS * M + tn::MATCH_WARPS * 32);
    if (smem <= 200 * 1024) {
        TN_CUDA(cudaFuncSetAttribute(tn::k_match_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        tn::k_match_warp<<<(R + tn::MATCH_WARPS - 1) / tn::MATCH_WARPS, tn::MATCH_WARPS * 32, smem, (cudaStream_t)stream>>>(
            R, S, M, d_num, d_cells, (const float2 *)d_dist, d_bary, d_sample_dist, (const uint4 *)d_verts, d_cell_out, (uint4 *)d_verts_out,
            d_mask_out, d_bary_out);
    } else {  // absurdly large M: the literal one-thread-per-ray form
        tn::k_match<<<(R + 63) / 64, 64, 0, (cudaStream_t)stream>>>(R, S, M, d_num, d_cells, (const float2 *)d_dist, d_bary, d_sample_dist,
                                                                   (const uint4 *)d_verts, d_cell_out, (uint4 *)d_verts_out, d_mask_out,
                                                                   d_bary_out);
    }
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

// [C,V] feature-major field -> [V,C] row-major shadow (one vertex = one contiguous row); callers that interpolate the same
// field more than once (coarse + fine pass of a training step) build it once and use tn_interpolate_values_shadow
extern "C" int tn_make_field_shadow(int device, uint32_t C, uint32_t V, const float *d_field, float *d_shadow, void *stream) {
    if (C == 0 || V == 0) return TN_OK;
    tn::DeviceGuard g(device);
    dim3 tb(32, 8), tg((V + 31) / 32, (C + 31) / 32);
    tn::k_transpose<<<tg, tb, 0, (cudaStream_t)stream>>>(d_field, d_shadow, C, V, false);
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}
extern "C" int tn_interpolate_values_shadow(int device, uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *d_vi, const float *d_w,
                                            const float *d_shadow, float *d_out, void *stream) {
    if (!d_shadow) return tn::fail(TN_ERR_ARG, "tn_interpolate_values_shadow: null shadow");
    if (N == 0 || C == 0) return TN_OK;
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    switch (D) {  // py_binding.cpp:258-276
        case 2: tn::interp_fwd<2>(N, C, d_vi, d_w, d_shadow, d_out, s); break;
        case 3: tn::interp_fwd<3>(N, C, d_vi, d_w, d_shadow, d_out, s); break;
        case 4: tn::interp_fwd<4>(N, C, d_vi, d_w, d_shadow, d_out, s); break;
        case 6: tn::interp_fwd<6>(N, C, d_vi, d_w, d_shadow, d_out, s); break;
        default: return tn::fail(TN_ERR_ARG, "Unsupported interpolation dimension with value " + std::to_string(D));
    }
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

extern "C" int tn_interpolate_values_backward(int device, uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *d_vi,
                                              const float *d_w, const float *d_grad_in, float *d_grad_field, float *d_scratch, void *stream) {
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    if (N == 0 || C == 0) {
        TN_CUDA(cudaMemsetAsync(d_grad_field, 0, sizeof(float) * (size_t)C * V, s));  // py_binding.cpp:360
        return TN_OK;
    }
    int rc = TN_OK;
    switch (D) {  // py_binding.cpp:278-296
        case 2: rc = tn::interp_bwd<2>(N, C, V, d_vi, d_w, d_grad_in, d_grad_field, d_scratch, s); break;
        case 3: rc = tn::interp_bwd<3>(N, C, V, d_vi, d_w, d_grad_in, d_grad_field, d_scratch, s); break;
        case 4: rc = tn::interp_bwd<4>(N, C, V, d_vi, d_w, d_grad_in, d_grad_field, d_scratch, s); break;
        case 6: rc = tn::interp_bwd<6>(N, C, V, d_vi, d_w, d_grad_in, d_grad_field, d_scratch, s); break;
        default: return tn::fail(TN_ERR_ARG, "Unsupported interpolation dimension with value " + std::to_string(D));
    }
    if (rc) return rc;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

// workspace: keys and values of the sort (in | out), the [V,C] accumulator, CUB temporary storage; each part 256-byte aligned
extern "C" int tn_interpolate_values_backward_deterministic(int device, uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *d_vi,
                                                           const float *d_w, const float *d_grad_in, float *d_grad_field, void *d_workspace,
                                                           size_t *workspace_bytes, void *stream) {
    if (!workspace_bytes) return tn::fail(TN_ERR_ARG, "tn_interpolate_values_backward_deterministic: null workspace_bytes");
    if (D != 2 && D != 3 && D != 4 && D != 6) return tn::fail(TN_ERR_ARG, "Unsupported interpolation dimension with value " + std::to_string(D));
    const uint64_t n64 = (uint64_t)N * D;
    if (n64 > 0x7FFFFFFFull) return tn::fail(TN_ERR_ARG, "tn_interpolate_values_backward_deterministic: N * D must stay below 2^31");
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t n = (uint32_t)n64;
    const int end_bit = 32 - __builtin_clz(V | 1u);  // keys are <= V
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    size_t cub_bytes = 0;
    TN_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const uint32_t *)nullptr,
                                            (uint32_t *)nullptr, (int)n, 0, end_bit, s));
    const size_t kb = al(sizeof(uint32_t) * (size_t)n), sb = al(sizeof(float) * (size_t)V * C);
    const size_t need = 4 * kb + sb + al(cub_bytes);
    if (!d_workspace) { *workspace_bytes = need; return TN_OK; }
    if (*workspace_bytes < need) return tn::fail(TN_ERR_ARG, "tn_interpolate_values_backward_deterministic: workspace too small");
    if ((size_t)C * V == 0) return TN_OK;
    if (N == 0) {
        TN_CUDA(cudaMemsetAsync(d_grad_field, 0, sizeof(float) * (size_t)C * V, s));
        return TN_OK;
    }
    uint8_t *ws = (uint8_t *)d_workspace;
    uint32_t *k0 = (uint32_t *)ws, *k1 = (uint32_t *)(ws + kb), *v0 = (uint32_t *)(ws + 2 * kb), *v1 = (uint32_t *)(ws + 3 * kb);
    float *grow = (float *)(ws + 4 * kb);
    void *tmp = ws + 4 * kb + sb;
    tn::k_ivb_keys<<<(n + 255) / 256, 256, 0, s>>>(n, V, d_vi, k0, v0);
    TN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, cub_bytes, k0, k1, v0, v1, (int)n, 0, end_bit, s));
    const uint32_t blocks = (uint32_t)(((uint64_t)V * 32 + 255) / 256);
    switch (D) {
        case 2: tn::k_ivb_det<2><<<blocks, 256, 0, s>>>(V, C, n, k1, v1, d_w, d_grad_in, grow); break;
        case 3: tn::k_ivb_det<3><<<blocks, 256, 0, s>>>(V, C, n, k1, v1, d_w, d_grad_in, grow); break;
        case 4: tn::k_ivb_det<4><<<blocks, 256, 0, s>>>(V, C, n, k1, v1, d_w, d_grad_in, grow); break;
        default: tn::k_ivb_det<6><<<blocks, 256, 0, s>>>(V, C, n, k1, v1, d_w, d_grad_in, grow); break;
    }
    dim3 tb(32, 8), tg((V + 31) / 32, (C + 31) / 32);
    tn::k_transpose<<<tg, tb, 0, s>>>(grow, d_grad_field, V, C, true);  // [V,C] -> [C,V]
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}
