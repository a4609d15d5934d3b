// tn_normals.cu -- normal map of the fused render: the density gradient at every sample of the pass that gives the colours, by a
// reverse pass through the MLP on warpgroup MMA, composited with the render's own weights (DESIGN.md §4.7).
//
// The field is linear inside each tetrahedron, so the spatial gradient of the density pre-activation at a sample is exact:
//   f = F_v0 + sum_k b_k (F_vk - F_v0),   g = d pre / d f  (the reverse chain through mlp_base),   q_k = g . (F_vk - F_v0),
//   grad_x pre = E^-T q = cof(E) q / det(E),   E = [x_v1 - x_v0 | x_v2 - x_v0 | x_v3 - x_v0].
// The sample normal is -grad / |grad| (nerfstudio Field.get_normals: softplus' > 0, so the direction of grad sigma), the pixel normal
// sum_i w_i n_i normalised (nerfstudio NormalsRenderer(normalize=True)).
//
//   k_mlp_normals<PREC>  persistent over the samples, k_mlp's tile scheduler and pieces (tn_mlp.cuh).  Per 64-sample tile: the same
//                        gather and layers 1-3 as k_mlp (so the same activations and ReLU masks as the rendered sigma), the masks kept
//                        as bitmasks, then the reverse chain  dz3 = m3 * wd,  dz2 = m2 * (dz3 W3),  dz1 = m1 * (dz2 W2),  g = dz1 W1
//                        with B read MN-major (transpose bit) from the resident forward image, then q (the four vertex rows read
//                        again, a four-thread reduction) and the cofactor solve in float64.
//   k_composite_normals  one warp per active ray: the weights of k_composite (same weights_from_density call on the same inputs, so
//                        the same bits), N = sum w n, normalised.
#include <algorithm>

#include "tn_common.cuh"
#include "tn_composite.cuh"
#include "tn_mlp.cuh"
#include "tn_tetsolve.cuh"

namespace tn {

// Two warpgroups per CTA (at most 255 registers per thread): with k_mlp's three (168 registers) the reverse chain spills.
constexpr uint32_t NRM_WGS = 2;
constexpr uint32_t NRM_THREADS = 128 * NRM_WGS;
// shared memory: weight image L1 | L2 | L3 (160 KB), wd[128], weight barrier, tile slots [NRM_WGS][2]
constexpr uint32_t NRM_OFF_HEAD = MLP_W_COARSE;
constexpr uint32_t NRM_OFF_BARS = NRM_OFF_HEAD + 128 * 4;
constexpr uint32_t NRM_SMEM_BYTES = NRM_OFF_BARS + 8 + 8 * NRM_WGS;
static_assert(NRM_SMEM_BYTES <= 232448, "k_mlp_normals shared memory exceeds 227 KB");

struct NormalsParams {
    const uint32_t *n_active;
    uint32_t S;
    const uint4 *vi;
    const float *bary;
    const float *fshadow;
    const uint8_t *wimg;   // L1 | L2 | L3 of k_mlp's image (per 64-wide K block: hi 16 KB, lo 16 KB; K blocks 32 KB apart)
    const float *bias;     // b1 b2 b3
    const float *head;     // wd[128] ...
    const float *xyz;      // [V,3]
    float4 *grad;          // [rows]
    uint32_t *tile_ctr;
};

// the value of x, unknown to the compiler: shared-memory addresses derived from it are formed where they are used instead of being
// hoisted out of the tile loop (the ~90 loop-invariant 64-bit descriptors of the six GEMMs would otherwise be kept live and spill)
__device__ __forceinline__ uint32_t opaque(uint32_t x) {
    asm volatile("mov.b32 %0, %0;" : "+r"(x));
    return x;
}
// a packed mask, formed where it is computed: left alone, the compiler sinks the packing to the mask's use in the reverse chain and
// keeps the 64 separate bits of each layer live through the forward GEMMs (the bf16x3 kernel spilled them)
__device__ __forceinline__ unsigned long long opaque(unsigned long long x) {
    asm volatile("mov.b64 %0, %0;" : "+l"(x));
    return x;
}
// the same for a pointer, laundered after a layer's MMA wait: the 16 bias (or seed) loads of an epilogue are issued after the MMAs
// that precede it (hoisted above them, they stay live through the 128 operand and accumulator registers of the GEMM, and spill)
__device__ __forceinline__ const float *opaque(const float *x) {
    asm volatile("mov.b64 %0, %0;" : "+l"(x));
    return x;
}

// bias + ReLU epilogue of a forward layer, as k_mlp's, into the next layer's A fragments; mk bit 4j + e = (pre-activation of d[4j + e] > 0)
template <int PREC>
__device__ __forceinline__ void relu_masked(const float (&d)[64], const float *__restrict__ bias, uint32_t t, uint32_t (&ah)[32], uint32_t (&al)[32],
                                            unsigned long long &mk) {
    mk = 0ull;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2 *>(bias + 8 * j + 2 * t));
        const float v0 = d[4 * j] + b.x, v1 = d[4 * j + 1] + b.y, v2 = d[4 * j + 2] + b.x, v3 = d[4 * j + 3] + b.y;
        mk |= (unsigned long long)((v0 > 0.f ? 1u : 0u) | (v1 > 0.f ? 2u : 0u) | (v2 > 0.f ? 4u : 0u) | (v3 > 0.f ? 8u : 0u)) << (4 * j);
        const int i = 4 * (j >> 1) + 2 * (j & 1);
        to_operand<PREC>(fmaxf(v0, 0.f), fmaxf(v1, 0.f), ah[i], al[i]);
        to_operand<PREC>(fmaxf(v2, 0.f), fmaxf(v3, 0.f), ah[i + 1], al[i + 1]);
    }
    mk = opaque(mk);
}

// cotangent of a layer's pre-activation (the ReLU mask applied to the gradient at its output) -> A fragments of the next reverse GEMM
template <int PREC>
__device__ __forceinline__ void mask_to_operand(const float (&d)[64], unsigned long long mk, uint32_t (&ah)[32], uint32_t (&al)[32]) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint32_t m = (uint32_t)(mk >> (4 * j)) & 15u;
        const int i = 4 * (j >> 1) + 2 * (j & 1);
        to_operand<PREC>((m & 1u) ? d[4 * j] : 0.f, (m & 2u) ? d[4 * j + 1] : 0.f, ah[i], al[i]);
        to_operand<PREC>((m & 4u) ? d[4 * j + 2] : 0.f, (m & 8u) ? d[4 * j + 3] : 0.f, ah[i + 1], al[i + 1]);
    }
}

// d = A W over K = 128 (the layer's outputs), A in registers, W = the layer's block of the forward image read MN-major: k-step kk is
// rows 16 kk.. (2048 bytes further), the next 64-wide block of the layer's inputs lies 32 KB further (LBO), the lo half 16 KB after the
// hi half.  N = 128 (hidden layers) or 64 (layer 1).
template <int PREC, int N>
__device__ __forceinline__ void reverse_mma(float (&d)[N / 2], const uint32_t (&ah)[32], const uint32_t (&al)[32], uint32_t w) {
    using namespace tc;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
        const uint64_t bh = make_desc(w + (uint32_t)kk * 2048u, 32768u, 1024u), bl = make_desc(w + 16384u + (uint32_t)kk * 2048u, 32768u, 1024u);
        const uint32_t acc = kk > 0 ? 1u : 0u;
        if constexpr (PREC == 2) {
            if constexpr (N == 128) { wgmma_rs_f16_n128<1>(d, a, bh, acc); wgmma_rs_f16_n128<1>(d, a, bl, 1u); }
            else { wgmma_rs_f16_n64<1>(d, a, bh, acc); wgmma_rs_f16_n64<1>(d, a, bl, 1u); }
        } else {
            const uint32_t b[4] = {al[4 * kk], al[4 * kk + 1], al[4 * kk + 2], al[4 * kk + 3]};
            if constexpr (N == 128) {
                wgmma_rs_bf16_n128<1>(d, a, bh, acc); wgmma_rs_bf16_n128<1>(d, b, bh, 1u); wgmma_rs_bf16_n128<1>(d, a, bl, 1u);
            } else {
                wgmma_rs_bf16_n64<1>(d, a, bh, acc); wgmma_rs_bf16_n64<1>(d, b, bh, 1u); wgmma_rs_bf16_n64<1>(d, a, bl, 1u);
            }
        }
    }
    wgmma_commit();
    wgmma_wait0();
    reg_fence(d);
}

template <int PREC>
__global__ void __launch_bounds__(NRM_THREADS, 1) k_mlp_normals(const NormalsParams p) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t tn_nrm_smem[];
    uint8_t *smem = tn_nrm_smem;
    float *wd_s = reinterpret_cast<float *>(smem + NRM_OFF_HEAD);
    uint64_t *w_bar = reinterpret_cast<uint64_t *>(smem + NRM_OFF_BARS);
    volatile uint32_t *slots = reinterpret_cast<volatile uint32_t *>(smem + NRM_OFF_BARS + 8);

    const uint32_t wg = threadIdx.x >> 7, tid = threadIdx.x & 127u;
    const uint32_t warp = tid >> 5, lane = threadIdx.x & 31u, g = lane >> 2, t = lane & 3u;
    const uint32_t n_active = *p.n_active;
    const uint64_t total_rows = (uint64_t)n_active * p.S;
    const uint32_t ntiles = (uint32_t)((total_rows + MLP_TILE - 1) / MLP_TILE);
    if (blockIdx.x * NRM_WGS >= ntiles) return;

    if (threadIdx.x == 0) {
        mbar_init(w_bar, 1);
        fence_barrier_init();
    }
    for (uint32_t i = threadIdx.x; i < 128; i += NRM_THREADS) wd_s[i] = p.head[i];
    auto draw = [&]() {  // k_mlp's scheduler
        const uint32_t nx = gridDim.x * NRM_WGS + atomicAdd(p.tile_ctr, 1u);
        // the tile count read again rather than kept live through the tile loop: at 255 registers k_mlp_normals<2> would spill it
        const uint32_t nt = (uint32_t)(((uint64_t)*p.n_active * p.S + MLP_TILE - 1) / MLP_TILE);
        return nx < nt ? nx : MLP_NO_TILE;
    };
    if (tid == 0) {
        const uint32_t first = blockIdx.x * NRM_WGS + wg;
        slots[2 * wg] = first < ntiles ? first : MLP_NO_TILE;
        slots[2 * wg + 1] = draw();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(w_bar, MLP_W_COARSE);
        for (uint32_t off = 0; off < MLP_W_COARSE; off += 16384) tma_bulk_g2s(smem + off, p.wimg + off, 16384, w_bar);
    }
    // the seed wd is scaled by a power of two that puts max |wd| in [2^7, 2^8): fp16 cotangents of f16w2 keep the small entries of
    // wd out of the subnormal range (at max |wd| ~ 1 the 1e-3-sized entries of a trained density head lose most of their bits) with
    // headroom for the growth through three layers below fp16's 65504.  The normal does not depend on the scale; the power of two is
    // undone exactly in the solve.
    float wmax = 0.f;
    for (int i = 0; i < 128; ++i) wmax = fmaxf(wmax, fabsf(wd_s[i]));
    int wexp = 0;
    frexpf(wmax, &wexp);
    wexp -= 8;
    const float seed_scale = ldexpf(1.f, -wexp);
    const uint32_t wsm = smem_u32(smem);
    bool weights_ready = false;
    const uint32_t lrow = warp * 16u + g;
    uint32_t tile = slots[2 * wg];

#pragma unroll 1
    for (uint32_t n = 0;; ++n) {
        wg_sync(wg);
        if (tile == MLP_NO_TILE) break;
        const uint32_t next = slots[2 * wg + ((n + 1u) & 1u)];
        if (tid == 0) slots[2 * wg + (n & 1u)] = draw();
        const uint64_t row0 = (uint64_t)tile * MLP_TILE + lrow, row1 = row0 + 8u;

        uint32_t ah[32], al[32];
        unsigned long long mk[3];
        {   // forward layers 1-3, exactly as k_mlp (same gather, same MMAs, same epilogue), keeping the ReLU masks
            uint32_t xh[16], xl[16];
            gather_rows<PREC>(load_gather_rows(p.vi, p.bary, row0, total_rows), p.fshadow, t, xh, xl);
            if (next != MLP_NO_TILE) prefetch_gather_rows(p.vi, p.bary, (uint64_t)next * MLP_TILE + lrow, total_rows);
            if (!weights_ready) { mbar_wait(w_bar, 0); weights_ready = true; }
            float d[64];
            layer_mma<PREC, 4>(d, xh, xl, opaque(wsm + mlp_off_layer(0)));
            relu_masked<PREC>(d, opaque(p.bias), t, ah, al, mk[0]);
        }
        {
            float d[64];
            layer_mma<PREC, 8>(d, ah, al, opaque(wsm + mlp_off_layer(1)));
            relu_masked<PREC>(d, opaque(p.bias + 128), t, ah, al, mk[1]);
        }
        {
            float d[64];
            layer_mma<PREC, 8>(d, ah, al, opaque(wsm + mlp_off_layer(2)));
            mk[2] = 0ull;  // layer 3 feeds only the density head: its mask is all the reverse chain needs
            const float *b3 = opaque(p.bias + 256);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float2 b = __ldg(reinterpret_cast<const float2 *>(b3 + 8 * j + 2 * t));
                const uint32_t m = (d[4 * j] + b.x > 0.f ? 1u : 0u) | (d[4 * j + 1] + b.y > 0.f ? 2u : 0u) | (d[4 * j + 2] + b.x > 0.f ? 4u : 0u) |
                                   (d[4 * j + 3] + b.y > 0.f ? 8u : 0u);
                mk[2] |= (unsigned long long)m << (4 * j);
            }
            mk[2] = opaque(mk[2]);
        }
        // reverse chain: seed dz3 = m3 * wd 2^-e, then dh2 = dz3 W3, dz2 = m2 * dh2, dh1 = dz2 W2, dz1 = m1 * dh1, g = dz1 W1
        const float *wd = opaque(wd_s);
        float gx[32];  // g: row g columns 8j + 2t, +1 in gx[4j], gx[4j + 1]; row g + 8 in gx[4j + 2], gx[4j + 3]
        {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint32_t c = 8u * j + 2u * t, m = (uint32_t)(mk[2] >> (4 * j)) & 15u;
                const float s0 = wd[c] * seed_scale, s1 = wd[c + 1] * seed_scale;
                const int i = 4 * (j >> 1) + 2 * (j & 1);
                to_operand<PREC>((m & 1u) ? s0 : 0.f, (m & 2u) ? s1 : 0.f, ah[i], al[i]);
                to_operand<PREC>((m & 4u) ? s0 : 0.f, (m & 8u) ? s1 : 0.f, ah[i + 1], al[i + 1]);
            }
            {
                float d[64];
                reverse_mma<PREC, 128>(d, ah, al, opaque(wsm + mlp_off_layer(2)));
                mask_to_operand<PREC>(d, mk[1], ah, al);
            }
            {
                float d[64];
                reverse_mma<PREC, 128>(d, ah, al, opaque(wsm + mlp_off_layer(1)));
                mask_to_operand<PREC>(d, mk[0], ah, al);
            }
            reverse_mma<PREC, 64>(gx, ah, al, opaque(wsm + mlp_off_layer(0)));
        }
        // q_k = g . (F_vk - F_v0): the thread's 16 columns of each row are the gather's (8c + 2t, +1), then the four threads of a row.
        // One row at a time (a loop, not unrolled), so that at most one row's 64 field values are in flight.
        float q[2][3];
#pragma unroll 1
        for (int rr = 0; rr < 2; ++rr) {
            const uint64_t row = rr ? row1 : row0;
            float gg[16];
#pragma unroll
            for (int c = 0; c < 8; ++c) { gg[2 * c] = rr ? gx[4 * c + 2] : gx[4 * c]; gg[2 * c + 1] = rr ? gx[4 * c + 3] : gx[4 * c + 1]; }
            uint4 v = row < total_rows ? __ldg(p.vi + row) : make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
            if (v.x == TN_EMPTY) v = make_uint4(0u, 0u, 0u, 0u);  // (the result of an unmatched row is discarded)
            const uint32_t vs[4] = {v.x, v.y, v.z, v.w};
            float4 a[4][4];
#pragma unroll
            for (int k = 0; k < 4; ++k) load_field_quads<false>(p.fshadow + (size_t)vs[k] * 64, t, a[k]);
            float s3[3];
#pragma unroll
            for (int k = 1; k < 4; ++k) {
                float acc = 0.f;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const float2 fk = field_pair(a[k], c), f0 = field_pair(a[0], c);
                    acc = fmaf(gg[2 * c], fk.x - f0.x, acc);
                    acc = fmaf(gg[2 * c + 1], fk.y - f0.y, acc);
                }
                s3[k - 1] = acc;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                s3[k] += __shfl_xor_sync(0xffffffffu, s3[k], 1);
                s3[k] += __shfl_xor_sync(0xffffffffu, s3[k], 2);
                if (rr == 0) q[0][k] = s3[k]; else q[1][k] = s3[k];
            }
        }
        if (t < 2) {  // thread t = 0 solves row0, t = 1 row1
            const uint64_t row = t == 0 ? row0 : row1;
            if (row < total_rows) {
                const uint4 v = __ldg(p.vi + row);
                float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
                if (v.x != TN_EMPTY) {
                    // E from the fp32 positions, cofactors and determinant in float64 (exact differences; no cancellation in slivers)
                    const uint32_t vs[4] = {v.x, v.y, v.z, v.w};
                    double cf[3][3], det;
                    tet_cofactors(p.xyz, vs, cf, det);
                    if (det != 0.0) {
                        const float q0 = t == 0 ? q[0][0] : q[1][0], q1 = t == 0 ? q[0][1] : q[1][1], q2 = t == 0 ? q[0][2] : q[1][2];
                        // undo the seed's power of two.  2^wexp is built from its bits (wexp lies in [-156, 120], well inside the
                        // normal range): the same value as ldexp(1.0, wexp), without the constants of ldexp's range checks, which the
                        // compiler would keep live through the tile loop (and spill, in k_mlp_normals<2>)
                        const double sc = __longlong_as_double((long long)(1023 + wexp) << 52) / det;
                        o.x = (float)((q0 * cf[0][0] + q1 * cf[1][0] + q2 * cf[2][0]) * sc);
                        o.y = (float)((q0 * cf[0][1] + q1 * cf[1][1] + q2 * cf[2][1]) * sc);
                        o.z = (float)((q0 * cf[0][2] + q1 * cf[1][2] + q2 * cf[2][2]) * sc);
                    }
                }
                p.grad[row] = o;
            }
        }
        tile = next;
    }
    if (!weights_ready) mbar_wait(w_bar, 0);
}

// sample normal -grad / max(|grad|, 1e-12) (0 for a zero gradient: unmatched samples, flat tetrahedra)
__device__ __forceinline__ float3 sample_normal(float4 gr) {
    const float inv = -1.f / fmaxf(norm3df(gr.x, gr.y, gr.z), 1e-12f);
    return make_float3(gr.x * inv, gr.y * inv, gr.z * inv);
}

constexpr int NRM_COMP_WARPS = 4;

__global__ void __launch_bounds__(NRM_COMP_WARPS * 32) k_composite_normals(const NormalsLaunch p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * NRM_COMP_WARPS + warp;
    if (slot >= *p.n_active) return;
    const uint32_t S = p.S;
    float *w = sm + (size_t)warp * (2 * ((size_t)S + 2)), *tr = w + S + 2;
    const uint32_t ray = p.ray_list[slot];
    const float *eb = p.ebins + (size_t)slot * (S + 1);
    const float4 *of = reinterpret_cast<const float4 *>(p.out_f) + (size_t)slot * S;
    for (uint32_t j = lane; j < S; j += 32) w[j] = (eb[j + 1] - eb[j]) * of[j].x;  // as k_composite
    __syncwarp();
    weights_from_density(w, tr, S, lane);
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (uint32_t j = lane; j < S; j += 32) {
        const float3 n = sample_normal(p.grad[(size_t)slot * S + j]);
        nx = fmaf(w[j], n.x, nx); ny = fmaf(w[j], n.y, ny); nz = fmaf(w[j], n.z, nz);
    }
    nx = warp_sum_f(nx); ny = warp_sum_f(ny); nz = warp_sum_f(nz);
    if (lane == 0) {  // NormalsRenderer(normalize=True): N / sqrt(max(|N|^2, 1e-20))
        const float inv = 1.f / sqrtf(fmaxf(nx * nx + ny * ny + nz * nz, 1e-20f));
        p.normals[3 * (size_t)ray] = nx * inv; p.normals[3 * (size_t)ray + 1] = ny * inv; p.normals[3 * (size_t)ray + 2] = nz * inv;
    }
}

int launch_normals(const NormalsLaunch &a, int sms, cudaStream_t s) {
    NormalsParams p{};
    p.n_active = a.n_active; p.S = a.S; p.vi = a.vi; p.bary = a.bary; p.fshadow = a.fshadow; p.wimg = a.wimg; p.bias = a.bias; p.head = a.head;
    p.xyz = a.xyz; p.grad = a.grad; p.tile_ctr = a.tile_ctr;
    auto k = a.prec == 2 ? k_mlp_normals<2> : k_mlp_normals<3>;
    TN_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)NRM_SMEM_BYTES));
    const uint64_t tiles = ((uint64_t)a.R * a.S + MLP_TILE - 1) / MLP_TILE;
    const uint32_t grid = (uint32_t)std::min<uint64_t>((tiles + NRM_WGS - 1) / NRM_WGS, (uint64_t)sms);
    k<<<grid, NRM_THREADS, NRM_SMEM_BYTES, s>>>(p);
    // every ray's normal: (0, 0, 0) for the empty ones, the composite for the others
    TN_CUDA(cudaMemsetAsync(a.normals, 0, sizeof(float) * 3 * (size_t)a.R, s));
    const size_t smem = NRM_COMP_WARPS * sizeof(float) * 2 * ((size_t)a.S + 2);
    TN_CUDA(cudaFuncSetAttribute(k_composite_normals, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_composite_normals<<<(a.R + NRM_COMP_WARPS - 1) / NRM_COMP_WARPS, NRM_COMP_WARPS * 32, smem, s>>>(a);
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

}  // namespace tn
