// tn_render.cu -- fused forward render: trace -> sample -> (interp+MLP on wgmma) -> PDF -> (interp+MLP) -> composite.
//
// Replaces TetrahedraNerf.get_outputs between trace_rays and the pixel (tetranerf/nerfstudio/model.py:531-662)
// in eval mode, i.e. the un-vendored nerfstudio pieces it calls (restated in oracle/oracle.py):
//   k_sample_coarse : nears/fars + ray_mask (:531-545), TetrahedraSampler / UniformSampler bins (:111-122,141-192),
//                     sample mid-points (:557) and find_visited_cells (tetrahedra_tracer.cu:115-161)
//   k_mlp<false>    : interpolate_values + mlp_base + density head (:569-581)            [tn_mlp.cuh]
//   k_sample_fine   : RaySamples.get_weights (:582), PDFSampler incl. include_original merge (:584),
//                     mid-points, find_visited_cells (:585-594), direction encoding folded into a per-ray bias (:607)
//   k_mlp<true>     : interpolate_values + mlp_base + density + mlp_head + colour head (:596-621)
//   k_composite     : get_weights, RGB / accumulation / median-depth renderers, scatter to rays (:632-662)
// Per-ray kernels use one warp per ray with the ray's segments staged in shared memory.
#include <cmath>
#include <vector>

#include <cstdlib>
#include <cub/cub.cuh>
#include "tn_common.cuh"
#include "tn_mlp.cuh"
#include "tn_mlp_bwd.cuh"
#include "tn_mlp_pack.cuh"

namespace tn {

int launch_trace_internal(tn_tracer *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells, float *bary,
                          float *dist, uint32_t *verts, int dense, cudaStream_t s);

struct RenderState {
    // field
    float *fshadow = nullptr;  // [V,64]
    uint32_t V = 0;
    // weights
    uint8_t *wimg = nullptr;   // L1 32K | L2 64K | L3 64K | L4(base part) 64K  (bf16 hi/lo)
    uint8_t *wimg16 = nullptr; // the same image with fp16 hi/lo halves (mlp_prec == 2)
    int mlp_prec = 2;          // operand precision of the inference MLP: 2 = f16w2 (default), 3 = bf16x3 (tn_mlp.cuh); training always runs 3
    float *bias = nullptr;     // b1 b2 b3 [3][128]
    float *head = nullptr;     // wd[128] wc[3][128] bd bc[3]
    float *w4dir = nullptr;    // [128][27] + b4[128]
    bool have_weights = false;
    // workspace
    size_t cap_R = 0, cap_M = 0, cap_Sc = 0, cap_S2 = 0;
    uint32_t *num = nullptr, *cells = nullptr, *verts = nullptr;
    float *bary = nullptr, *dist = nullptr;
    uint32_t *n_active = nullptr, *ray_list = nullptr;
    float *ebins_c = nullptr, *sbins_c = nullptr, *bary_c = nullptr, *dens_c = nullptr;
    uint4 *vi_c = nullptr;
    float *ebins_f = nullptr, *bary_f = nullptr, *out_f = nullptr, *dirbias = nullptr;
    uint4 *vi_f = nullptr;
    // training (tn_render_train_forward / _backward): backward weight image, per-sample head gradients, accumulators
    uint8_t *wimg_bwd = nullptr;       // 7 stages of 32 KB (tn_mlp_bwd.cuh)
    float *sbins_f = nullptr, *enc = nullptr;   // [R,S2+1] spacing bins of the fine pass, [R,27] encoded directions (per slot)
    float4 *dout = nullptr;            // [R*S2] gradients at the head pre-activations
    float *gshadow = nullptr, *gw = nullptr, *g_dirbias = nullptr;
    size_t cap_train_R = 0, cap_train_S2 = 0;
    uint32_t gshadow_V = 0;
    // what the last training forward ran with (the backward continues from its buffers)
    bool train_valid = false;
    uint32_t t_R = 0, t_M = 0, t_Sc = 0, t_Sf = 0, t_S2 = 0;
    float t_bg[3] = {1.f, 1.f, 1.f};
    // fused pixel gather (tn_render_set_gather): peer[k] = rank k's [world * rays_per_rank, 6] gathered-pixel buffer
    float *peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    uint32_t gather_world = 0, gather_rank = 0, gather_stride = 0;
    // optional per-kernel timing (bench.py roofline): events around the 6 kernels of tn_render
    bool profile = false;
    cudaEvent_t ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t evb[4] = {nullptr, nullptr, nullptr, nullptr};  // backward: start | composite_bwd | mlp_bwd | finalize
    // deterministic mode (tn_render_set_deterministic): ordered slots in the training forward, fixed-order reductions in its backward
    bool det = false;                  // mode of the next training forward (initial value: TETRANERF_B200_DETERMINISTIC)
    bool t_det = false;                // mode the last training forward ran in: its backward continues in it
    uint32_t bwd_grid = 0;             // CTAs of the backward MLP kernel (test hook; 0 = default)
    uint32_t *ray_flag = nullptr, *ray_slot = nullptr;  // [R] ray has hits, its slot (exclusive scan)
    size_t cap_slot_R = 0;
    void *cub_tmp = nullptr;           // CUB scan / sort temporary storage
    size_t cub_tmp_bytes = 0;
    float *det_part = nullptr;         // [BWD_PARTS][BWD_PART_STRIDE] per-partition dW / column sums
    float *det_gdb = nullptr;          // [4 (ntiles + R)][128] direction-bias gradient partials
    float *det_dx = nullptr;           // [R*S2,64] feature gradient per sample
    float4 *det_sums = nullptr;        // [R] head-bias gradient per slot
    float *det_dbg = nullptr;          // [R/64][128*28] partial W4dir / b4 gradients per block of k_dirbias_grads
    uint32_t *det_keys = nullptr, *det_vals = nullptr;  // [2][R*S2*4] (vertex, sample row * 4 + k) pairs, sort input | output
    size_t cap_det_R = 0, cap_det_S2 = 0;
};

static void free_ws(RenderState *r) {
    cudaFree(r->num); cudaFree(r->cells); cudaFree(r->verts); cudaFree(r->bary); cudaFree(r->dist);
    cudaFree(r->n_active); cudaFree(r->ray_list); cudaFree(r->ebins_c); cudaFree(r->sbins_c); cudaFree(r->bary_c); cudaFree(r->dens_c);
    cudaFree(r->vi_c); cudaFree(r->ebins_f); cudaFree(r->bary_f); cudaFree(r->out_f); cudaFree(r->dirbias); cudaFree(r->vi_f);
    r->num = r->cells = r->verts = nullptr; r->bary = r->dist = nullptr; r->n_active = r->ray_list = nullptr;
    r->ebins_c = r->sbins_c = r->bary_c = r->dens_c = nullptr; r->vi_c = nullptr;
    r->ebins_f = r->bary_f = r->out_f = r->dirbias = nullptr; r->vi_f = nullptr;
    r->cap_R = r->cap_M = r->cap_Sc = r->cap_S2 = 0;
}

void free_render(tn_tracer *h) {
    if (!h->render) return;
    RenderState *r = h->render;
    free_ws(r);
    cudaFree(r->fshadow); cudaFree(r->wimg); cudaFree(r->wimg16); cudaFree(r->bias); cudaFree(r->head); cudaFree(r->w4dir);
    cudaFree(r->wimg_bwd); cudaFree(r->sbins_f); cudaFree(r->enc); cudaFree(r->dout); cudaFree(r->gshadow); cudaFree(r->gw); cudaFree(r->g_dirbias);
    cudaFree(r->ray_flag); cudaFree(r->ray_slot); cudaFree(r->cub_tmp); cudaFree(r->det_part); cudaFree(r->det_gdb); cudaFree(r->det_dx);
    cudaFree(r->det_sums); cudaFree(r->det_dbg); cudaFree(r->det_keys); cudaFree(r->det_vals);
    for (auto &e : r->ev) if (e) cudaEventDestroy(e);
    for (auto &e : r->evb) if (e) cudaEventDestroy(e);
    delete r;
    h->render = nullptr;
}

static RenderState *state(tn_tracer *h) {
    if (!h->render) {
        h->render = new RenderState();
        const char *e = getenv("TETRANERF_B200_MLP_PREC");  // 2 / 3: initial operand precision of the inference MLP (tn_render_set_mlp_precision)
        if (e && (atoi(e) == 2 || atoi(e) == 3)) h->render->mlp_prec = atoi(e);
        const char *d = getenv("TETRANERF_B200_DETERMINISTIC");  // 1: initial value of tn_render_set_deterministic
        if (d && atoi(d) == 1) h->render->det = true;
    }
    return h->render;
}

// ---------------------------------------------------------------------------------------------------
__global__ void k_transpose64(const float *__restrict__ in, float *__restrict__ out, uint32_t V) {  // [64,V] -> [V,64]
    __shared__ float tile[64][33];
    const uint32_t v0 = blockIdx.x * 32;
    for (uint32_t c = threadIdx.y; c < 64; c += blockDim.y) {
        const uint32_t v = v0 + threadIdx.x;
        tile[c][threadIdx.x] = v < V ? in[(size_t)c * V + v] : 0.f;
    }
    __syncthreads();
    for (uint32_t r = threadIdx.y; r < 32; r += blockDim.y) {
        const uint32_t v = v0 + r;
        if (v < V) {
            out[(size_t)v * 64 + threadIdx.x] = tile[threadIdx.x][r];
            out[(size_t)v * 64 + 32 + threadIdx.x] = tile[32 + threadIdx.x][r];
        }
    }
}

// head/bias packing: params12 order = mlp_base.layers.{0,1,2}.{weight,bias}, mlp_head.layers.0.{weight,bias},
// field_output_color.net.{weight,bias}, field_output_density.net.{weight,bias}
__global__ void k_pack_small(const float *b1, const float *b2, const float *b3, const float *w4, const float *b4, const float *wc,
                             const float *bc, const float *wd, const float *bd, float *bias, float *head, float *w4dir) {
    const int t = threadIdx.x;  // 128 threads
    bias[t] = b1[t]; bias[128 + t] = b2[t]; bias[256 + t] = b3[t];
    head[t] = wd[t];
    head[128 + t] = wc[t]; head[256 + t] = wc[128 + t]; head[384 + t] = wc[256 + t];
    if (t == 0) { head[512] = bd[0]; head[513] = bc[0]; head[514] = bc[1]; head[515] = bc[2]; }
    for (int k = 0; k < 27; ++k) w4dir[t * 27 + k] = w4[t * 155 + k];  // mlp_out = [encoded_dir(27), base(128)] (model.py:608)
    w4dir[128 * 27 + t] = b4[t];
}

// ---------------------------------------------------------------------------------------------------
constexpr int SAMPLE_WARPS = 4;

struct SampleParams {
    uint32_t R, M, Sc, Sf, S2, biased;
    const uint32_t *num;
    const float2 *dist;
    const uint4 *verts;
    const float *bary;
    const float *o, *d;
    uint32_t *n_active, *ray_list;
    float *ebins_c, *sbins_c, *bary_c;
    uint4 *vi_c;
    const float *dens_c;
    float *ebins_f, *bary_f;
    uint4 *vi_f;
    float *dirbias;
    const float *w4dir;
    const float *out_f;
    float *rgb, *acc, *depth;
    uint8_t *mask;
    float far_plane, bg0, bg1, bg2;
    // training mode (model.py:169-174 stratified bins, PDFSampler train_stratified, RGBRenderer without nan_to_num / clamp)
    uint32_t train;
    const float *jit_c, *jit_f;   // [R,Sc+1], [R,Sf+1] uniform [0,1) draws indexed by RAY (nullptr: the eval-mode bins)
    float *sbins_f, *enc;         // saved for the backward: spacing bins of the fine pass [slot,S2+1], encoded direction [slot,27]
    // fused pixel gather: when gather_world > 0 every rendered pixel is also stored, as (r, g, b, accumulation, depth, mask), at row
    // gather_rank * gather_stride + ray of EVERY rank's gathered buffer (peer[k] is mapped peer memory: stores travel over NVLink)
    float *peer[8];
    uint32_t gather_world, gather_rank, gather_stride;
    const uint32_t *ray_slot;     // deterministic mode: slot of every ray with hits (exclusive scan of num > 0)
};

// lane 0 writes the local outputs; lanes < gather_world each post the pixel to one rank's gathered buffer (three 8-byte stores)
__device__ __forceinline__ void store_pixel(const SampleParams &p, uint32_t ray, int lane, float r, float g, float b, float a, float depth, uint8_t mask) {
    if (lane == 0) {
        p.rgb[3 * (size_t)ray] = r; p.rgb[3 * (size_t)ray + 1] = g; p.rgb[3 * (size_t)ray + 2] = b;
        p.acc[ray] = a; p.depth[ray] = depth;
        if (p.mask != nullptr) p.mask[ray] = mask;
    }
    if ((uint32_t)lane < p.gather_world) {
        float2 *dst = reinterpret_cast<float2 *>(p.peer[lane] + 6 * ((size_t)p.gather_rank * p.gather_stride + ray));
        dst[0] = make_float2(r, g); dst[1] = make_float2(b, a); dst[2] = make_float2(depth, mask ? 1.f : 0.f);
        __threadfence_system();  // the pixel is performed at the peer before this kernel can complete
    }
}

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
__device__ float smem_scan_add(float *a, uint32_t n, int lane) {
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
__device__ void smem_scan_max(const float *in, float *out, uint32_t n, int lane) {
    float carry = -3.0e38f;
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t i = base + lane;
        float v = i < n ? in[i] : -3.0e38f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v = fmaxf(v, t);
        }
        v = fmaxf(v, carry);
        if (i < n) out[i] = v;
        carry = __shfl_sync(0xffffffffu, v, 31);
    }
    __syncwarp();
}
__device__ __forceinline__ float nan_to_num_f(float x) {  // torch.nan_to_num defaults
    if (isnan(x)) return 0.f;
    if (isinf(x)) return x > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
    return x;
}
// torch.linspace(start, end, steps)[i] for float32 (symmetric fill of ATen's linspace kernel)
__device__ __forceinline__ float linspace_f(float start, float end, uint32_t steps, uint32_t i) {
    const float step = (end - start) / (float)(steps - 1);
    return i < steps / 2 ? start + step * (float)i : end - step * (float)(steps - i - 1);
}

// find_visited_cells for one sample distance d: binary search over the staged prefix-max of t_out, then the segment's own
// (t_in, t_out) from the trace output (L1: the warp has just read the row)
__device__ __forceinline__ void match_sample(float d, uint32_t n, const float2 *__restrict__ dist, const float *pm, size_t row,
                                             const uint4 *__restrict__ verts, const float *__restrict__ bary, uint4 &vi, float &b0,
                                             float &b1, float &b2) {
    vi = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
    b0 = b1 = b2 = 0.f;
    uint32_t lo = 0, hi = n;  // first p with pm[p] >= d  (== the reference's monotone pointer walk for sorted samples)
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pm[mid] < d) lo = mid + 1; else hi = mid;
    }
    if (lo >= n) return;
    const float2 h = __ldg(dist + row + lo);
    if (h.x <= d) {
        vi = __ldg(verts + row + lo);
        const float mult = __fdiv_rn(__fsub_rn(d, h.x), __fsub_rn(h.y, h.x));
        const float omm = __fsub_rn(1.0f, mult);
        const float *c = bary + 6 * (row + lo);
        b0 = __fadd_rn(__fmul_rn(omm, __ldg(c)), __fmul_rn(mult, __ldg(c + 3)));
        b1 = __fadd_rn(__fmul_rn(omm, __ldg(c + 1)), __fmul_rn(mult, __ldg(c + 4)));
        b2 = __fadd_rn(__fmul_rn(omm, __ldg(c + 2)), __fmul_rn(mult, __ldg(c + 5)));
    }
}

// shared memory per warp.  Only the prefix-max of t_out (binary-searched by every sample) is staged per segment; t_in / t_out are
// read from the trace output where needed.  Coarse pass: pm[M+2], cum[M+2] (biased sampler only), e[Sc+2] = 4.6 KB at M = 512,
// Sc = 128; fine pass: pm[M+2] and cdf / e / x / y of Smax+2 = 6.2 KB -- every ray of a 4096-ray batch is resident at once
// (28 warps per SM; round 1 staged three segment arrays and sized all bin arrays for the worst case: 14.4 / 10.3 KB per warp,
// 12 / 20 warps per SM, i.e. the coarse pass ran in 2.3 waves).
__host__ __device__ __forceinline__ size_t seg_arr(uint32_t M) { return (size_t)M + 2; }
__host__ __device__ __forceinline__ size_t coarse_floats(uint32_t M, uint32_t Sc, uint32_t biased) { return seg_arr(M) * (biased ? 2 : 1) + (size_t)Sc + 2; }
__host__ __device__ __forceinline__ size_t fine_floats(uint32_t M, uint32_t Smax) { return seg_arr(M) + 4 * ((size_t)Smax + 2); }

// ORDERED (deterministic mode): the slot of a ray is its rank among the rays with hits (p.ray_slot), so slot order = ray order;
// otherwise slots are claimed with an atomic counter
template <bool ORDERED>
__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_sample_coarse(const SampleParams p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t ray = blockIdx.x * SAMPLE_WARPS + warp;
    if (ray >= p.R) return;
    const uint32_t M = p.M, S = p.Sc;
    const size_t A = seg_arr(M);
    float *pm = sm + (size_t)warp * coarse_floats(M, S, p.biased);
    float *cum = pm + A, *e = cum + (p.biased ? A : 0);
    const uint32_t n = p.num[ray];
    if constexpr (ORDERED) {
        if (ray == p.R - 1 && lane == 0) *p.n_active = p.ray_slot[ray] + (n > 0 ? 1u : 0u);
    }
    if (n == 0) {  // model.py:640-650 : background colour, accumulation 0, depth = collider far plane
        store_pixel(p, ray, lane, p.bg0, p.bg1, p.bg2, 0.f, p.far_plane, 0);
        return;
    }
    uint32_t slot = 0;
    if constexpr (ORDERED) {
        slot = p.ray_slot[ray];
        if (lane == 0) { p.ray_list[slot] = ray; p.mask[ray] = 1; }
    } else {
        if (lane == 0) { slot = atomicAdd(p.n_active, 1u); p.ray_list[slot] = ray; p.mask[ray] = 1; }
        slot = __shfl_sync(0xffffffffu, slot, 0);
    }
    const size_t row = (size_t)ray * M;
    const float near = __ldg(&p.dist[row]).x, far = __ldg(&p.dist[row + n - 1]).y;
    for (uint32_t k = lane; k < n; k += 32) {
        const float2 h = __ldg(&p.dist[row + k]);
        pm[k] = h.y;
        if (p.biased) cum[k + 1] = fmaxf(h.y - h.x, 0.f);  // map_from_real_distances_to_biased_with_bounds, model.py:111-122
    }
    if (p.biased && lane == 0) cum[0] = near;
    __syncwarp();
    smem_scan_max(pm, pm, n, lane);  // in place
    if (p.biased) {
        // cum[k] = start + sum_{i<k} len_i : scan over [start, len_0, len_1, ...]
        smem_scan_add(cum, n + 1, lane);
    }
    for (uint32_t j = lane; j <= S; j += 32) {
        float b = linspace_f(0.f, 1.f, S + 1, j);
        if (p.jit_c != nullptr) {  // stratified training bins (model.py:169-174; nerfstudio SpacedSampler): jitter between the neighbouring bin centres
            const float lower = j == 0 ? b : (b + linspace_f(0.f, 1.f, S + 1, j - 1)) / 2.0f;
            const float upper = j == S ? b : (linspace_f(0.f, 1.f, S + 1, j + 1) + b) / 2.0f;
            b = lower + (upper - lower) * __ldg(p.jit_c + (size_t)ray * (S + 1) + j);
        }
        float eu = b * far + (1.f - b) * near;  // spacing_to_euclidean_fn (model.py:177)
        float sb = b;
        if (p.biased) {
            const float uni = (eu - near) / (far - near);
            float rest = uni * (float)n;
            float iv = fminf(floorf(rest), (float)(n - 1));
            iv = fmaxf(iv, 0.f);
            rest = rest - iv;
            const uint32_t k = (uint32_t)iv;
            const float2 hk = __ldg(&p.dist[row + k]);
            const float len = fmaxf(hk.y - hk.x, 0.f);
            eu = cum[k] + len * rest;
            sb = (eu - near) / (far - near);  // model.py:182
        }
        e[j] = eu;
        p.ebins_c[(size_t)slot * (S + 1) + j] = eu;
        p.sbins_c[(size_t)slot * (S + 1) + j] = sb;
    }
    __syncwarp();
    for (uint32_t j = lane; j < S; j += 32) {
        const float dmid = (e[j + 1] + e[j]) / 2.f;  // model.py:557
        uint4 vi; float b0, b1, b2;
        match_sample(dmid, n, p.dist, pm, row, p.verts, p.bary, vi, b0, b1, b2);
        const size_t g = (size_t)slot * S + j;
        p.vi_c[g] = vi;
        p.bary_c[3 * g] = b0; p.bary_c[3 * g + 1] = b1; p.bary_c[3 * g + 2] = b2;
    }
}

// RaySamples.get_weights on staged deltas/densities: w[j] (in place over `dd`), using `tr` as scratch
__device__ void weights_from_density(float *dd, float *tr, uint32_t S, int lane) {
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

// direction encoding folded into a per-ray bias of mlp_head (model.py:607-620): dirbias[slot] = b4 + W4[:, :27] . enc(dir)
// NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0, max_freq_exp=4, include_input=True), model.py:426-432
__device__ __forceinline__ void dir_bias(const SampleParams &p, uint32_t ray, uint32_t slot, int lane) {
    const float dx = p.d[3 * (size_t)ray], dy = p.d[3 * (size_t)ray + 1], dz = p.d[3 * (size_t)ray + 2];
    float enc[27];
    {
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
    if (p.train) {
#pragma unroll
        for (int k = 0; k < 27; ++k) if (lane == k) p.enc[(size_t)slot * 27 + k] = enc[k];
    }
    for (uint32_t o = lane; o < 128; o += 32) {
        float acc = p.w4dir[128 * 27 + o];
#pragma unroll
        for (int k = 0; k < 27; ++k) acc = fmaf(__ldg(p.w4dir + o * 27 + k), enc[k], acc);
        p.dirbias[(size_t)slot * 128 + o] = acc;
    }
}

__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_sample_fine(const SampleParams p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * SAMPLE_WARPS + warp;
    if (slot >= *p.n_active) return;
    const uint32_t M = p.M, S = p.Sc, S2 = p.S2, nb = p.Sf + 1;
    const size_t A = seg_arr(M), B = (size_t)max(p.Sc, p.S2) + 2;
    float *pm = sm + (size_t)warp * fine_floats(M, max(p.Sc, p.S2));
    float *cdf = pm + A, *e = cdf + B, *x = e + B, *y = x + B;
    const uint32_t ray = p.ray_list[slot];
    const uint32_t n = p.num[ray];
    const size_t row = (size_t)ray * M;
    const float near = __ldg(&p.dist[row]).x, far = __ldg(&p.dist[row + n - 1]).y;
    for (uint32_t k = lane; k < n; k += 32) pm[k] = __ldg(&p.dist[row + k]).y;
    __syncwarp();
    smem_scan_max(pm, pm, n, lane);  // in place
    // ---- coarse weights (model.py:581-582) ----
    const float *eb = p.ebins_c + (size_t)slot * (S + 1);
    const float *sbc = p.sbins_c + (size_t)slot * (S + 1);
    for (uint32_t j = lane; j < S; j += 32) x[j] = (eb[j + 1] - eb[j]) * p.dens_c[(size_t)slot * S + j];
    __syncwarp();
    weights_from_density(x, y, S, lane);
    // ---- PDFSampler (nerfstudio ray_samplers.py), histogram_padding 0.01, eps 1e-5, eval mode ----
    float part = 0.f;
    for (uint32_t j = lane; j < S; j += 32) { x[j] = x[j] + 0.01f; part += x[j]; }
    float wsum = warp_sum_f(part);
    const float padding = fmaxf(1e-5f - wsum, 0.f);
    wsum += padding;
    for (uint32_t j = lane; j < S; j += 32) y[j] = (x[j] + padding / (float)S) / wsum;  // pdf
    __syncwarp();
    smem_scan_add(y, S, lane);
    if (lane == 0) cdf[0] = 0.f;
    for (uint32_t j = lane; j < S; j += 32) cdf[j + 1] = fminf(1.f, y[j]);
    __syncwarp();
    // new bins -> x[0..nb)
    const float u_end = (float)(1.0 - 1.0 / (double)nb), u_off = (float)(1.0 / (2.0 * (double)nb));
    for (uint32_t i = lane; i < nb; i += 32) {
        const float u = linspace_f(0.f, u_end, nb, i) + (p.jit_f != nullptr ? __ldg(p.jit_f + (size_t)ray * nb + i) / (float)nb : u_off);  // train_stratified
        uint32_t lo = 0, hi = S + 1;  // searchsorted(cdf, u, side="right"): first idx with cdf[idx] > u
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (cdf[mid] <= u) lo = mid + 1; else hi = mid; }
        const uint32_t below = (uint32_t)min(max((int)lo - 1, 0), (int)S), above = min(lo, S);
        const float c0 = cdf[below], c1 = cdf[above];
        float t = (u - c0) / (c1 - c0);
        t = isnan(t) ? 0.f : nan_to_num_f(t);
        t = fminf(fmaxf(t, 0.f), 1.f);
        const float b0 = sbc[below], b1 = sbc[above];
        x[i] = b0 + t * (b1 - b0);
    }
    __syncwarp();
    // merge existing (S+1, sorted) with new (nb, sorted) -> e[0..S2]  (torch.sort of the concatenation)
    for (uint32_t k = lane; k <= S; k += 32) {
        const float v = sbc[k];
        uint32_t lo = 0, hi = nb;  // # new strictly less than v
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (x[mid] < v) lo = mid + 1; else hi = mid; }
        e[k + lo] = v;
    }
    for (uint32_t i = lane; i < nb; i += 32) {
        const float v = x[i];
        uint32_t lo = 0, hi = S + 1;  // # existing <= v
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (sbc[mid] <= v) lo = mid + 1; else hi = mid; }
        e[i + lo] = v;
    }
    __syncwarp();
    for (uint32_t j = lane; j <= S2; j += 32) {
        const float b = e[j];
        const float eu = b * far + (1.f - b) * near;
        y[j] = eu;
        p.ebins_f[(size_t)slot * (S2 + 1) + j] = eu;
        if (p.train) p.sbins_f[(size_t)slot * (S2 + 1) + j] = b;
    }
    __syncwarp();
    for (uint32_t j = lane; j < S2; j += 32) {
        const float dmid = (y[j + 1] + y[j]) / 2.f;  // model.py:585
        uint4 vi; float b0, b1, b2;
        match_sample(dmid, n, p.dist, pm, row, p.verts, p.bary, vi, b0, b1, b2);
        const size_t g = (size_t)slot * S2 + j;
        p.vi_f[g] = vi;
        p.bary_f[3 * g] = b0; p.bary_f[3 * g + 1] = b1; p.bary_f[3 * g + 2] = b2;
    }
    dir_bias(p, ray, slot, lane);
}

__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_composite(const SampleParams p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * SAMPLE_WARPS + warp;
    if (slot >= *p.n_active) return;
    const uint32_t S2 = p.S2;
    float *w = sm + (size_t)warp * (2 * ((size_t)S2 + 2)), *tr = w + S2 + 2;
    const uint32_t ray = p.ray_list[slot];
    const float *eb = p.ebins_f + (size_t)slot * (S2 + 1);
    const float4 *of = reinterpret_cast<const float4 *>(p.out_f) + (size_t)slot * S2;
    for (uint32_t j = lane; j < S2; j += 32) w[j] = (eb[j + 1] - eb[j]) * of[j].x;
    __syncwarp();
    weights_from_density(w, tr, S2, lane);  // model.py:632
    float r = 0.f, g = 0.f, b = 0.f, a = 0.f;
    for (uint32_t j = lane; j < S2; j += 32) {
        const float4 c = of[j];
        const float wj = w[j];
        if (p.train) { r += wj * c.y; g += wj * c.z; b += wj * c.w; a += wj; }  // RGBRenderer in training: no nan_to_num, no clamp
        else { r += wj * nan_to_num_f(c.y); g += wj * nan_to_num_f(c.z); b += wj * nan_to_num_f(c.w); a += wj; }
    }
    r = warp_sum_f(r); g = warp_sum_f(g); b = warp_sum_f(b); a = warp_sum_f(a);
    // DepthRenderer("median"): first sample whose cumulative weight reaches 0.5
    for (uint32_t j = lane; j < S2; j += 32) tr[j] = w[j];
    __syncwarp();
    smem_scan_add(tr, S2, lane);
    uint32_t first = S2;
    for (uint32_t j = lane; j < S2; j += 32) if (tr[j] >= 0.5f) { first = j; break; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    const uint32_t mi = min(first, S2 - 1);
    // RGBRenderer: comp + background * (1 - acc); clamped to [0,1] in eval mode only
    float pr = r + p.bg0 * (1.f - a), pg = g + p.bg1 * (1.f - a), pb = b + p.bg2 * (1.f - a);
    if (!p.train) { pr = fminf(fmaxf(pr, 0.f), 1.f); pg = fminf(fmaxf(pg, 0.f), 1.f); pb = fminf(fmaxf(pb, 0.f), 1.f); }
    store_pixel(p, ray, lane, pr, pg, pb, a, (eb[mi] + eb[mi + 1]) / 2.f, 1);
}

// ---- backward of the compositing + field heads of the fine pass (model.py:621-637; RaySamples.get_weights, RGBRenderer and
// AccumulationRenderer of nerfstudio, GradientScaler model.py:195-205): one warp per active ray.
//   w_j = (1 - exp(-x_j)) T_j,  x_j = delta_j sigma_j,  T_j = exp(-sum_{i<j} x_i);   rgb = sum w_j c_j + bg (1 - sum w_j),  acc = sum w_j
//   dL/dw_j = g_j = grad_rgb . (c_j - bg) + grad_acc;   dL/dx_j = g_j (T_j - w_j) - sum_{k>j} g_k w_k;   dL/dc_j = grad_rgb w_j
// then through Softplus / Sigmoid to the head PRE-activations, which is where the MLP backward kernel starts.
struct CompositeBwdParams {
    uint32_t S2, use_gradient_scaling;
    const uint32_t *n_active, *ray_list;
    const float *ebins_f, *sbins_f, *out_f;
    const float *grad_rgb, *grad_acc;  // [R,3], [R] or nullptr
    float bg0, bg1, bg2;
    float4 *dout;                      // [slot * S2 + j]
    float *sums;                       // 4 floats: sum d sigma_pre, sum d z_r, d z_g, d z_b (bias gradients of the two heads);
                                       // deterministic mode: [n_active] float4, one per slot (summed in slot order by k_det_sum_slots)
};
template <bool DET>
__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_composite_bwd(const CompositeBwdParams p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * SAMPLE_WARPS + warp;
    if (slot >= *p.n_active) return;
    const uint32_t S2 = p.S2;
    float *w = sm + (size_t)warp * (4 * ((size_t)S2 + 2)), *tr = w + S2 + 2, *gw = tr + S2 + 2, *fx = gw + S2 + 2;
    const uint32_t ray = p.ray_list[slot];
    const float *eb = p.ebins_f + (size_t)slot * (S2 + 1);
    const float4 *of = reinterpret_cast<const float4 *>(p.out_f) + (size_t)slot * S2;
    const float gr = p.grad_rgb[3 * (size_t)ray], gg = p.grad_rgb[3 * (size_t)ray + 1], gb = p.grad_rgb[3 * (size_t)ray + 2];
    const float ga = p.grad_acc != nullptr ? p.grad_acc[ray] : 0.f;
    for (uint32_t j = lane; j < S2; j += 32) tr[j] = (eb[j + 1] - eb[j]) * of[j].x;  // x_j
    __syncwarp();
    smem_scan_add(tr, S2, lane);  // inclusive cumsum of x
    for (uint32_t j = lane; j < S2; j += 32) {
        const float excl = j == 0 ? 0.f : tr[j - 1];
        const float x = (eb[j + 1] - eb[j]) * of[j].x;
        const float T = expf(-excl);
        float wj = (1.f - expf(-x)) * T;
        const bool fin = isfinite(wj);  // nan_to_num in the forward: a replaced weight carries no gradient
        wj = fin ? wj : nan_to_num_f(wj);
        const float4 c = of[j];
        const float g = fin ? (gr * (c.y - p.bg0) + gg * (c.z - p.bg1) + gb * (c.w - p.bg2) + ga) : 0.f;
        w[j] = wj;
        gw[j] = g * wj;
        fx[j] = fin ? g * (T - wj) : 0.f;  // first term of dL/dx_j
    }
    __syncwarp();
    const float total = smem_scan_add(gw, S2, lane);  // inclusive cumsum of g_k w_k -> suffix_j = total - gw[j]
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    for (uint32_t j = lane; j < S2; j += 32) {
        const float4 c = of[j];
        const float delta = eb[j + 1] - eb[j];
        float dsig = delta * (fx[j] - (total - gw[j]));
        float dr = gr * w[j], dg = gg * w[j], db = gb * w[j];
        if (p.use_gradient_scaling) {  // model.py:195-205,625-630: squared (spacing_start + spacing_end), clamped to [0,1]
            const float *sb = p.sbins_f + (size_t)slot * (S2 + 1);
            const float rd = sb[j] + sb[j + 1];
            const float sc = fminf(fmaxf(rd * rd, 0.f), 1.f);
            dsig *= sc; dr *= sc; dg *= sc; db *= sc;
        }
        const float4 o = make_float4(dsig * (-expm1f(-c.x)),      // Softplus'(s) = 1 - exp(-softplus(s))
                                     dr * c.y * (1.f - c.y), dg * c.z * (1.f - c.z), db * c.w * (1.f - c.w));  // Sigmoid' = c (1 - c)
        p.dout[(size_t)slot * S2 + j] = o;
        s0 += o.x; s1 += o.y; s2 += o.z; s3 += o.w;
    }
    s0 = warp_sum_f(s0); s1 = warp_sum_f(s1); s2 = warp_sum_f(s2); s3 = warp_sum_f(s3);
    if constexpr (DET) {
        if (lane == 0) reinterpret_cast<float4 *>(p.sums)[slot] = make_float4(s0, s1, s2, s3);
    } else {
        if (lane == 0) { atomicAdd(p.sums, s0); atomicAdd(p.sums + 1, s1); atomicAdd(p.sums + 2, s2); atomicAdd(p.sums + 3, s3); }
    }
}

// ---- after k_mlp_bwd: the direction part of mlp_head.layers.0 (W4[:, :27], b4) from the per-ray bias gradients: W4dir[k][j] =
// sum_slot g_dirbias[slot][k] enc[slot][j], b4[k] = sum_slot g_dirbias[slot][k].  One block per 64 slots, 256 threads: thread t owns
// hidden unit k = t & 127 and 14 of the 28 columns (27 encoding entries + the bias column of ones); partial sums -> atomicAdd
// (deterministic mode: -> part[block][k * 28 + column], summed in block order by k_det_reduce_dbg).
constexpr uint32_t DBG_SLOTS = 64, DBG_PART = 128 * 28;
template <bool DET>
__global__ void __launch_bounds__(256) k_dirbias_grads(const uint32_t *__restrict__ n_active, const float *__restrict__ g_dirbias, const float *__restrict__ enc,
                                                        float *__restrict__ gw, float *__restrict__ part) {
    __shared__ float s_enc[DBG_SLOTS][28];
    const uint32_t n = *n_active, s0 = blockIdx.x * DBG_SLOTS;
    if (s0 >= n) return;
    const uint32_t ns = min(DBG_SLOTS, n - s0);
    for (uint32_t i = threadIdx.x; i < ns * 28; i += 256) {
        const uint32_t s = i / 28, j = i % 28;
        s_enc[s][j] = j < 27 ? __ldg(enc + (size_t)(s0 + s) * 27 + j) : 1.0f;
    }
    __syncthreads();
    const uint32_t k = threadIdx.x & 127u, j0 = (threadIdx.x >> 7) * 14u;
    float acc[14];
#pragma unroll
    for (int j = 0; j < 14; ++j) acc[j] = 0.f;
    for (uint32_t s = 0; s < ns; ++s) {
        const float g = __ldg(g_dirbias + (size_t)(s0 + s) * 128 + k);
#pragma unroll
        for (int j = 0; j < 14; ++j) acc[j] = fmaf(g, s_enc[s][j0 + j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 14; ++j) {
        const uint32_t col = j0 + (uint32_t)j;
        if constexpr (DET) part[(size_t)blockIdx.x * DBG_PART + k * 28 + col] = acc[j];
        else atomicAdd(col < 27 ? gw + GW_W4DIR + k * 27 + col : gw + GW_B4 + k, acc[j]);
    }
}

// ---- deterministic mode: the reductions of the backward in a fixed order ----------------------------------------------------------------
// slot flags for the ordered slot assignment of the training forward
__global__ void k_ray_flags(uint32_t R, const uint32_t *__restrict__ num, uint32_t *__restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) flag[i] = num[i] > 0 ? 1u : 0u;
}
// dW and the seven column sums: the non-empty partitions in index order
__global__ void k_det_reduce_parts(const uint32_t *__restrict__ n_active, uint32_t S, const float *__restrict__ part, float *__restrict__ gw) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= BWD_PART_STRIDE) return;
    const uint32_t ntiles = (uint32_t)(((uint64_t)*n_active * S + BWD_TILE - 1) / BWD_TILE);
    float acc = 0.f;
    for (uint32_t q = 0; q < BWD_PARTS; ++q)
        if (bwd_part_lo(q, ntiles) < bwd_part_lo(q + 1, ntiles)) acc += part[(size_t)q * BWD_PART_STRIDE + e];
    gw[e] = acc;
}
// head-bias gradients: per-slot sums -> one block, strided sequential sums then a fixed tree
__global__ void __launch_bounds__(256) k_det_sum_slots(const uint32_t *__restrict__ n_active, const float4 *__restrict__ part, float *__restrict__ out) {
    __shared__ float4 s[256];
    const uint32_t n = *n_active, t = threadIdx.x;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (uint32_t i = t; i < n; i += 256) { const float4 v = part[i]; a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
    s[t] = a;
    __syncthreads();
    for (uint32_t h = 128; h > 0; h >>= 1) {
        if (t < h) { const float4 b = s[t + h]; s[t].x += b.x; s[t].y += b.y; s[t].z += b.z; s[t].w += b.w; }
        __syncthreads();
    }
    if (t == 0) { out[0] = s[0].x; out[1] = s[0].y; out[2] = s[0].z; out[3] = s[0].w; }
}
// per-ray direction-bias gradient: the partial rows of the 16-row warp blocks b that hold the ray's samples, in block order
// (k_mlp_bwd<true> wrote block b = 4 tile + warp's partial for ray `slot` to row 4 (tile + slot) + warp)
__global__ void __launch_bounds__(128) k_det_dirbias(const uint32_t *__restrict__ n_active, uint32_t S, const float *__restrict__ gdb_part,
                                                     float *__restrict__ g_dirbias) {
    const uint32_t slot = blockIdx.x, k = threadIdx.x;
    if (slot >= *n_active) return;
    const uint64_t r0 = (uint64_t)slot * S, r1 = r0 + S - 1;
    float acc = 0.f;
    for (uint64_t b = r0 / 16; b <= r1 / 16; ++b) acc += __ldg(gdb_part + (4 * (b / 4 + slot) + (b & 3)) * 128 + k);
    g_dirbias[(size_t)slot * 128 + k] = acc;
}
// W4dir / b4: the per-block partials of k_dirbias_grads<true> in block order
__global__ void k_det_reduce_dbg(const uint32_t *__restrict__ n_active, const float *__restrict__ part, float *__restrict__ gw) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;  // k * 28 + column
    if (e >= DBG_PART) return;
    const uint32_t nb = (*n_active + DBG_SLOTS - 1) / DBG_SLOTS;
    float acc = 0.f;
    for (uint32_t b = 0; b < nb; ++b) acc += part[(size_t)b * DBG_PART + e];
    const uint32_t k = e / 28, col = e % 28;
    gw[col < 27 ? GW_W4DIR + k * 27 + col : GW_B4 + k] = acc;
}
// field gradient, step 1: (vertex, entry) pairs of every sample row, entry = row * 4 + k; rows past the active samples and empty
// samples get the key V (sorted behind every vertex)
__global__ void k_det_field_keys(const uint32_t *__restrict__ n_active, uint32_t S, uint32_t n, uint32_t V, const uint4 *__restrict__ vi,
                                 uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const uint64_t row = e >> 2, total = (uint64_t)*n_active * S;
    uint32_t key = V;
    if (row < total) {
        const uint4 v = __ldg(vi + row);
        if (v.x != TN_EMPTY) { const uint32_t k = e & 3u; key = k == 0 ? v.x : (k == 1 ? v.y : (k == 2 ? v.z : v.w)); }
    }
    keys[e] = key;
    vals[e] = e;
}
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t *__restrict__ a, uint32_t n, uint32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(a + mid) < x) lo = mid + 1; else hi = mid; }
    return lo;
}
// step 2 (after the stable sort by vertex): one warp per vertex sums w_k dX[row] over its entries in sorted (= row) order -> [V,64]
__global__ void __launch_bounds__(256) k_det_field_grad(uint32_t V, uint32_t n, const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                        const float *__restrict__ bary, const float *__restrict__ dx, float *__restrict__ gshadow) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (v >= V) return;
    const uint32_t lo = lower_bound_u32(keys, n, v), hi = lower_bound_u32(keys, n, v + 1);
    float2 acc = make_float2(0.f, 0.f);
    for (uint32_t b = lo; b < hi; b += 32) {
        uint32_t e = 0;
        float w = 0.f;
        if (b + lane < hi) {  // the weight of this lane's entry: (1 - b0 - b1 - b2, b0, b1, b2)[k], as k_mlp_bwd
            e = __ldg(vals + b + lane);
            const float *c = bary + 3 * (size_t)(e >> 2);
            const float b0 = __ldg(c), b1 = __ldg(c + 1), b2 = __ldg(c + 2);
            const uint32_t k = e & 3u;
            w = k == 0 ? 1.0f - ((b0 + b1) + b2) : (k == 1 ? b0 : (k == 2 ? b1 : b2));
        }
        const uint32_t m = min(32u, hi - b);
        for (uint32_t j = 0; j < m; ++j) {
            const uint32_t ej = __shfl_sync(0xffffffffu, e, j);
            const float wj = __shfl_sync(0xffffffffu, w, j);
            const float2 x = __ldg(reinterpret_cast<const float2 *>(dx + (size_t)(ej >> 2) * 64) + lane);
            acc.x = fmaf(wj, x.x, acc.x);
            acc.y = fmaf(wj, x.y, acc.y);
        }
    }
    reinterpret_cast<float2 *>(gshadow + (size_t)v * 64)[lane] = acc;
}
struct GradOut { float *p[12]; };
__global__ void k_scatter_grads(const float *__restrict__ gw, const GradOut o) {
    // o.p: mlp_base.layers.{0,1,2}.{weight,bias}, mlp_head.layers.0.{weight,bias}, field_output_color.net.{weight,bias}, field_output_density.net.{weight,bias}
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 8192) o.p[0][i] = gw[GW_W1 + i];
    if (i < 16384) { o.p[2][i] = gw[GW_W2 + i]; o.p[4][i] = gw[GW_W3 + i]; }
    if (i < 128 * 155) {
        const uint32_t k = i / 155, j = i % 155;
        o.p[6][i] = j < 27 ? gw[GW_W4DIR + k * 27 + j] : gw[GW_W4B + k * 128 + (j - 27)];
    }
    if (i < 128) { o.p[1][i] = gw[GW_B1 + i]; o.p[3][i] = gw[GW_B2 + i]; o.p[5][i] = gw[GW_B3 + i]; o.p[7][i] = gw[GW_B4 + i]; o.p[10][i] = gw[GW_WD + i]; }
    if (i < 384) o.p[8][i] = gw[GW_WC + i];
    if (i < 3) o.p[9][i] = gw[GW_SUMS + 1 + i];
    if (i == 0) o.p[11][0] = gw[GW_SUMS];
}
__global__ void k_transpose_v64(const float *__restrict__ in, float *__restrict__ out, uint32_t V) {  // [V,64] -> [64,V]
    __shared__ float tile[32][65];
    const uint32_t v0 = blockIdx.x * 32;
    for (uint32_t r = threadIdx.y; r < 32; r += blockDim.y) {
        const uint32_t v = v0 + r;
        tile[r][threadIdx.x] = v < V ? in[(size_t)v * 64 + threadIdx.x] : 0.f;
        tile[r][threadIdx.x + 32] = v < V ? in[(size_t)v * 64 + 32 + threadIdx.x] : 0.f;
    }
    __syncthreads();
    for (uint32_t c = threadIdx.y; c < 64; c += blockDim.y) {
        const uint32_t v = v0 + threadIdx.x;
        if (v < V) out[(size_t)c * V + v] = tile[threadIdx.x][c];
    }
}

// single-pass configuration (num_fine_samples == 0, model.py:573 skipped): colours come from the first and only pass -- the
// FINE MLP runs on the coarse samples and only the per-ray direction bias is still missing
__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_dirbias_only(const SampleParams p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * SAMPLE_WARPS + warp;
    if (slot >= *p.n_active) return;
    dir_bias(p, p.ray_list[slot], slot, lane);
}

static int ensure_ws(RenderState *r, size_t R, size_t M, size_t Sc, size_t S2) {
    if (R <= r->cap_R && M <= r->cap_M && Sc <= r->cap_Sc && S2 <= r->cap_S2) return TN_OK;
    free_ws(r);
    R = std::max(R, r->cap_R); M = std::max(M, r->cap_M); Sc = std::max(Sc, r->cap_Sc); S2 = std::max(S2, r->cap_S2);
#define A(ptr, bytes) TN_CUDA(cudaMalloc((void **)&(ptr), (bytes)))
    A(r->num, 4 * R); A(r->cells, 4 * R * M); A(r->verts, 16 * R * M); A(r->bary, 24 * R * M); A(r->dist, 8 * R * M);
    A(r->n_active, 16); A(r->ray_list, 4 * R);
    A(r->ebins_c, 4 * R * (Sc + 1)); A(r->sbins_c, 4 * R * (Sc + 1)); A(r->bary_c, 12 * R * Sc); A(r->dens_c, 4 * R * Sc); A(r->vi_c, 16 * R * Sc);
    A(r->ebins_f, 4 * R * (S2 + 1)); A(r->bary_f, 12 * R * S2); A(r->out_f, 16 * R * S2); A(r->dirbias, 512 * R); A(r->vi_f, 16 * R * S2);
#undef A
    r->cap_R = R; r->cap_M = M; r->cap_Sc = Sc; r->cap_S2 = S2;
    return TN_OK;
}

static int ensure_cub_tmp(RenderState *r, size_t bytes) {
    if (bytes <= r->cub_tmp_bytes) return TN_OK;
    cudaFree(r->cub_tmp); r->cub_tmp = nullptr; r->cub_tmp_bytes = 0;
    TN_CUDA(cudaMalloc(&r->cub_tmp, bytes));
    r->cub_tmp_bytes = bytes;
    return TN_OK;
}

// deterministic mode, forward: slot of every ray = number of rays with hits before it (exclusive scan)
static int ordered_slots(RenderState *r, uint32_t R, cudaStream_t s) {
    if (R > r->cap_slot_R) {
        cudaFree(r->ray_flag); cudaFree(r->ray_slot); r->ray_flag = r->ray_slot = nullptr; r->cap_slot_R = 0;
        TN_CUDA(cudaMalloc((void **)&r->ray_flag, 4 * (size_t)R));
        TN_CUDA(cudaMalloc((void **)&r->ray_slot, 4 * (size_t)R));
        r->cap_slot_R = R;
    }
    size_t bytes = 0;
    TN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, r->ray_flag, r->ray_slot, (int)R, s));
    int rc = ensure_cub_tmp(r, bytes);
    if (rc) return rc;
    k_ray_flags<<<(R + 255) / 256, 256, 0, s>>>(R, r->num, r->ray_flag);
    TN_CUDA(cub::DeviceScan::ExclusiveSum(r->cub_tmp, bytes, r->ray_flag, r->ray_slot, (int)R, s));
    return TN_OK;
}

// deterministic mode, backward workspace for R rays of S2 fine samples
static int ensure_det_ws(RenderState *r, size_t R, size_t S2) {
    if (!r->det_part) TN_CUDA(cudaMalloc((void **)&r->det_part, sizeof(float) * BWD_PARTS * (size_t)BWD_PART_STRIDE));
    if (R <= r->cap_det_R && S2 <= r->cap_det_S2) return TN_OK;
    cudaFree(r->det_gdb); cudaFree(r->det_dx); cudaFree(r->det_sums); cudaFree(r->det_dbg); cudaFree(r->det_keys); cudaFree(r->det_vals);
    r->det_gdb = r->det_dx = r->det_dbg = nullptr; r->det_sums = nullptr; r->det_keys = r->det_vals = nullptr;
    r->cap_det_R = r->cap_det_S2 = 0;
    R = std::max(R, r->cap_det_R); S2 = std::max(S2, r->cap_det_S2);
    const size_t rows = R * S2, ntiles = (rows + BWD_TILE - 1) / BWD_TILE;
    TN_CUDA(cudaMalloc((void **)&r->det_gdb, sizeof(float) * 4 * (ntiles + R) * 128));
    TN_CUDA(cudaMalloc((void **)&r->det_dx, sizeof(float) * 64 * rows));
    TN_CUDA(cudaMalloc((void **)&r->det_sums, sizeof(float4) * R));
    TN_CUDA(cudaMalloc((void **)&r->det_dbg, sizeof(float) * DBG_PART * ((R + DBG_SLOTS - 1) / DBG_SLOTS)));
    TN_CUDA(cudaMalloc((void **)&r->det_keys, sizeof(uint32_t) * 2 * 4 * rows));
    TN_CUDA(cudaMalloc((void **)&r->det_vals, sizeof(uint32_t) * 2 * 4 * rows));
    r->cap_det_R = R; r->cap_det_S2 = S2;
    return TN_OK;
}

}  // namespace tn

using namespace tn;

extern "C" int tn_render_set_field(tn_tracer *h, const float *d_field, uint32_t C, uint32_t V, void *stream) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (C != 64) return fail(TN_ERR_ARG, "tn_render: field_dim must be 64 (model.py:81)");
    DeviceGuard g(h->device);
    RenderState *r = state(h);
    if (r->V != V) { cudaFree(r->fshadow); r->fshadow = nullptr; TN_CUDA(cudaMalloc((void **)&r->fshadow, sizeof(float) * 64 * (size_t)V)); r->V = V; }
    k_transpose64<<<(V + 31) / 32, dim3(32, 8), 0, (cudaStream_t)stream>>>(d_field, r->fshadow, V);
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

// operand precision of the inference MLP: 2 = f16w2 (default: fp16 activations, fp16 hi/lo weights; 2.6e-5 absolute on unit-scale
// density / colour, inside the 1e-4 per-sample bar; ~21 % less MLP time), 3 = bf16x3 (fp32-level).  The training forward always runs 3.
extern "C" int tn_render_set_mlp_precision(tn_tracer *h, int prec) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (prec != 2 && prec != 3) return fail(TN_ERR_ARG, "tn_render_set_mlp_precision: 2 (f16w2) or 3 (bf16x3)");
    DeviceGuard g(h->device);
    state(h)->mlp_prec = prec;
    return TN_OK;
}

extern "C" int tn_render_set_weights(tn_tracer *h, const float *const *P, void *stream) {
    if (!h || !P) return fail(TN_ERR_ARG, "null argument");
    DeviceGuard g(h->device);
    RenderState *r = state(h);
    cudaStream_t s = (cudaStream_t)stream;
    if (!r->wimg) {
        TN_CUDA(cudaMalloc((void **)&r->wimg, 32768 + 3 * 65536));
        TN_CUDA(cudaMalloc((void **)&r->wimg16, 32768 + 3 * 65536));
        TN_CUDA(cudaMalloc((void **)&r->bias, sizeof(float) * 384));
        TN_CUDA(cudaMalloc((void **)&r->head, sizeof(float) * 520));
        TN_CUDA(cudaMalloc((void **)&r->w4dir, sizeof(float) * (128 * 27 + 128)));
    }
    launch_pack_weights(P[0], 64, 0, 64, r->wimg, s);                     // mlp_base.layers.0.weight [128,64]
    launch_pack_weights(P[2], 128, 0, 128, r->wimg + 32768, s);           // mlp_base.layers.1.weight [128,128]
    launch_pack_weights(P[4], 128, 0, 128, r->wimg + 32768 + 65536, s);   // mlp_base.layers.2.weight
    launch_pack_weights(P[6], 155, 27, 128, r->wimg + 32768 + 131072, s); // mlp_head.layers.0.weight [128,155], base part
    launch_pack_weights(P[0], 64, 0, 64, r->wimg16, s, 32768u, 16384u, 1);
    launch_pack_weights(P[2], 128, 0, 128, r->wimg16 + 32768, s, 32768u, 16384u, 1);
    launch_pack_weights(P[4], 128, 0, 128, r->wimg16 + 32768 + 65536, s, 32768u, 16384u, 1);
    launch_pack_weights(P[6], 155, 27, 128, r->wimg16 + 32768 + 131072, s, 32768u, 16384u, 1);
    k_pack_small<<<1, 128, 0, s>>>(P[1], P[3], P[5], P[6], P[7], P[8], P[9], P[10], P[11], r->bias, r->head, r->w4dir);
    // backward image (tn_mlp_bwd.cuh): stage 0 = [W1 hi | W1 lo]; then per 128-wide layer [hi kb0 | hi kb1][lo kb0 | lo kb1]
    if (!r->wimg_bwd) TN_CUDA(cudaMalloc((void **)&r->wimg_bwd, BWD_WIMG_BYTES));
    launch_pack_weights(P[0], 64, 0, 64, r->wimg_bwd, s, 16384u, 16384u);
    launch_pack_weights(P[2], 128, 0, 128, r->wimg_bwd + 1 * BWD_STAGE, s, 16384u, 32768u);
    launch_pack_weights(P[4], 128, 0, 128, r->wimg_bwd + 3 * BWD_STAGE, s, 16384u, 32768u);
    launch_pack_weights(P[6], 155, 27, 128, r->wimg_bwd + 5 * BWD_STAGE, s, 16384u, 32768u);
    h->launches += 13;
    TN_CUDA(cudaGetLastError());
    r->have_weights = true;
    return TN_OK;
}

// training-mode inputs of the forward (nullptr = eval)
struct TrainFwd {
    const float *jit_c, *jit_f;
};
static int ensure_train_ws(RenderState *r, size_t R, size_t S2, uint32_t V);

static int render_impl(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                       float *d_rgb, float *d_acc, float *d_depth, uint8_t *d_mask, const TrainFwd *tf, void *stream) {
    if (!h || !cfg) return fail(TN_ERR_ARG, "null argument");
    RenderState *r = h->render;
    if (!r || !r->fshadow || !r->have_weights) return fail(TN_ERR_STATE, "tn_render: call tn_render_set_field and tn_render_set_weights first");
    if (!h->mesh.nodes) return fail(TN_ERR_STATE, "tn_render: no tetrahedra loaded");
    if (r->V != h->mesh.V) return fail(TN_ERR_ARG, "tn_render: field has a different vertex count than the mesh");
    const uint32_t M = cfg->max_ray_triangles, Sc = cfg->num_samples, Sf = cfg->num_fine_samples;
    if (Sc == 0 || Sc > 4096 || Sf > 4096) return fail(TN_ERR_ARG, "tn_render: num_samples must be in [1,4096]");
    if (tf != nullptr && Sf == 0) return fail(TN_ERR_ARG, "tn_render_train_forward: the fused training step needs num_fine_samples > 0");
    const bool det = tf != nullptr && r->det;
    if (det && (uint64_t)R * (Sc + Sf + 1) * 4 > 0x7FFFFFFFull)
        return fail(TN_ERR_ARG, "tn_render_train_forward: deterministic mode takes at most 2^29 fine samples per call (split the batch)");
    if (R == 0) return TN_OK;
    if ((uint64_t)R * (uint64_t)(Sc + Sf + 1) >= (1ull << 32)) return fail(TN_ERR_ARG, "tn_render: rays x samples must stay below 2^32 per call (split the batch)");
    const bool single = Sf == 0;                       // one pass only: the colours come from the coarse samples
    const uint32_t S2 = single ? Sc : Sc + Sf + 1;     // PDFSampler include_original (model.py:463)
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    int rc = ensure_ws(r, R, M, Sc, S2);
    if (rc) return rc;
    if (tf != nullptr) {
        rc = ensure_train_ws(r, R, S2, r->V);
        if (rc) return rc;
    }
    r->train_valid = false;
    const int prec = tf != nullptr ? 3 : r->mlp_prec;  // the training forward keeps bf16x3 (its backward recomputes in bf16x3)
    TN_CUDA(cudaMemsetAsync(r->n_active, 0, 16, s));
#define TN_EV(i) do { if (r->profile) cudaEventRecord(r->ev[i], s); } while (0)
    TN_EV(0);  // the "trace" interval includes the L2 warm-up it exists for
    {   // L2 warm-up of everything read-only that the step gathers from (mesh tables, field shadow, weight image)
        const void *extra[2] = {r->fshadow, prec == 2 ? r->wimg16 : r->wimg};
        const size_t extra_b[2] = {sizeof(float) * 64 * (size_t)r->V, 32768 + 3 * 65536};
        rc = launch_prefetch(h, extra, extra_b, 2, s);
        if (rc) return rc;
    }
    rc = launch_trace_internal(h, d_origins, d_directions, R, M, r->num, r->cells, r->bary, r->dist, r->verts, 0, s);
    if (rc) return rc;
    TN_EV(1);
    SampleParams p{};
    p.R = R; p.M = M; p.Sc = Sc; p.Sf = Sf; p.S2 = S2; p.biased = cfg->use_biased_sampler;
    p.num = r->num; p.dist = (const float2 *)r->dist; p.verts = (const uint4 *)r->verts; p.bary = r->bary;
    p.o = d_origins; p.d = d_directions; p.n_active = r->n_active; p.ray_list = r->ray_list;
    p.ebins_c = r->ebins_c; p.sbins_c = r->sbins_c; p.bary_c = r->bary_c; p.vi_c = r->vi_c; p.dens_c = r->dens_c;
    p.ebins_f = r->ebins_f; p.bary_f = r->bary_f; p.vi_f = r->vi_f; p.dirbias = r->dirbias; p.w4dir = r->w4dir; p.out_f = r->out_f;
    p.rgb = d_rgb; p.acc = d_acc; p.depth = d_depth; p.mask = d_mask;
    p.far_plane = cfg->far_plane; p.bg0 = cfg->background[0]; p.bg1 = cfg->background[1]; p.bg2 = cfg->background[2];
    if (tf != nullptr) { p.train = 1; p.jit_c = tf->jit_c; p.jit_f = tf->jit_f; p.sbins_f = r->sbins_f; p.enc = r->enc; }
    if (r->gather_world) {
        if (R > r->gather_stride) return fail(TN_ERR_ARG, "tn_render: more rays than the gathered-pixel buffers were sized for (tn_render_set_gather)");
        for (int k = 0; k < 8; ++k) p.peer[k] = r->peer[k];
        p.gather_world = r->gather_world; p.gather_rank = r->gather_rank; p.gather_stride = r->gather_stride;
    }
    const uint32_t Smax = std::max(Sc, S2);
    const size_t smem_sc = SAMPLE_WARPS * sizeof(float) * coarse_floats(M, Sc, p.biased);
    const size_t smem_sf = SAMPLE_WARPS * sizeof(float) * fine_floats(M, Smax);
    const size_t smem_c = SAMPLE_WARPS * sizeof(float) * 2 * ((size_t)S2 + 2);
    auto k_coarse_sample = det ? k_sample_coarse<true> : k_sample_coarse<false>;
    TN_CUDA(cudaFuncSetAttribute(k_coarse_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sc));
    TN_CUDA(cudaFuncSetAttribute(k_sample_fine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sf));
    TN_CUDA(cudaFuncSetAttribute(k_composite, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
    auto k_coarse = prec == 2 ? k_mlp<false, 2> : k_mlp<false, 3>;
    auto k_fine = prec == 2 ? k_mlp<true, 2> : k_mlp<true, 3>;
    TN_CUDA(cudaFuncSetAttribute(k_coarse, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MLP_SMEM_BYTES));
    TN_CUDA(cudaFuncSetAttribute(k_fine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MLP_SMEM_BYTES));
    const uint32_t gridR = (R + SAMPLE_WARPS - 1) / SAMPLE_WARPS;

    if (det) {
        rc = ordered_slots(r, R, s);
        if (rc) return rc;
        p.ray_slot = r->ray_slot;
        h->launches += 2;
    }
    k_coarse_sample<<<gridR, SAMPLE_WARPS * 32, smem_sc, s>>>(p);
    TN_EV(2);
    MlpParams mc{};
    mc.n_active = r->n_active; mc.S = Sc; mc.vi = r->vi_c; mc.bary = r->bary_c; mc.fshadow = r->fshadow; mc.wimg = prec == 2 ? r->wimg16 : r->wimg;
    mc.bias = r->bias; mc.head = r->head; mc.dirbias = nullptr; mc.out = r->dens_c;
    mc.tile_ctr = r->n_active + 1;  // words 1, 2 of the zeroed 16-byte block: tile counters of the coarse / fine pass
    // one CTA per SM at most (the weight image fills its shared memory), MLP_WGS tiles of MLP_TILE samples in flight per CTA
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    const uint64_t tiles_c = ((uint64_t)R * Sc + MLP_TILE - 1) / MLP_TILE, tiles_f = ((uint64_t)R * S2 + MLP_TILE - 1) / MLP_TILE;
    const uint32_t grid_c = (uint32_t)std::min<uint64_t>((tiles_c + MLP_WGS - 1) / MLP_WGS, (uint64_t)sms);
    const uint32_t grid_f = (uint32_t)std::min<uint64_t>((tiles_f + MLP_WGS - 1) / MLP_WGS, (uint64_t)sms);
    if (!single) k_coarse<<<grid_c, MLP_THREADS, MLP_SMEM_BYTES, s>>>(mc);
    TN_EV(3);
    if (!single) k_sample_fine<<<gridR, SAMPLE_WARPS * 32, smem_sf, s>>>(p);
    else k_dirbias_only<<<gridR, SAMPLE_WARPS * 32, 0, s>>>(p);
    TN_EV(4);
    MlpParams mf = mc;
    mf.S = S2; mf.dirbias = r->dirbias; mf.out = r->out_f;
    if (!single) { mf.vi = r->vi_f; mf.bary = r->bary_f; }
    else p.ebins_f = r->ebins_c;  // k_composite integrates over the coarse bins
    mf.tile_ctr = r->n_active + 2;
    k_fine<<<grid_f, MLP_THREADS, MLP_SMEM_BYTES, s>>>(mf);
    TN_EV(5);
    k_composite<<<gridR, SAMPLE_WARPS * 32, smem_c, s>>>(p);
    TN_EV(6);
#undef TN_EV
    h->launches += 5;
    TN_CUDA(cudaGetLastError());
    if (tf != nullptr) {
        r->train_valid = true;
        r->t_det = det;
        r->t_R = R; r->t_M = M; r->t_Sc = Sc; r->t_Sf = Sf; r->t_S2 = S2;
        r->t_bg[0] = cfg->background[0]; r->t_bg[1] = cfg->background[1]; r->t_bg[2] = cfg->background[2];
    }
    return TN_OK;
}

static int ensure_train_ws(RenderState *r, size_t R, size_t S2, uint32_t V) {
    if (R > r->cap_train_R || S2 > r->cap_train_S2) {
        cudaFree(r->sbins_f); cudaFree(r->enc); cudaFree(r->dout); cudaFree(r->g_dirbias);
        r->sbins_f = r->enc = r->g_dirbias = nullptr; r->dout = nullptr;
        R = std::max(R, r->cap_train_R); S2 = std::max(S2, r->cap_train_S2);
        TN_CUDA(cudaMalloc((void **)&r->sbins_f, 4 * R * (S2 + 1)));
        TN_CUDA(cudaMalloc((void **)&r->enc, 4 * R * 27));
        TN_CUDA(cudaMalloc((void **)&r->dout, 16 * R * S2));
        TN_CUDA(cudaMalloc((void **)&r->g_dirbias, 512 * R));
        r->cap_train_R = R; r->cap_train_S2 = S2;
    }
    if (!r->gw) TN_CUDA(cudaMalloc((void **)&r->gw, sizeof(float) * GW_TOTAL));
    if (r->gshadow_V != V) {
        cudaFree(r->gshadow); r->gshadow = nullptr;
        TN_CUDA(cudaMalloc((void **)&r->gshadow, sizeof(float) * 64 * (size_t)V));
        r->gshadow_V = V;
    }
    return TN_OK;
}

extern "C" int tn_render(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                         float *d_rgb, float *d_acc, float *d_depth, uint8_t *d_mask, void *stream) {
    return render_impl(h, cfg, d_origins, d_directions, R, d_rgb, d_acc, d_depth, d_mask, nullptr, stream);
}

// ---- fused training step (SURVEY §8f-1; model.py:520-662 in training mode + autograd) ------------------------------------------------
// forward: the fused pipeline with stratified bins (d_jitter_coarse f32[R,Sc+1], d_jitter_fine f32[R,Sf+1], uniform [0,1), indexed by
// ray; nullptr = eval bins) and the training-mode RGB renderer (no nan_to_num, no clamp).  Keeps what the backward needs.
extern "C" int tn_render_train_forward(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                                       const float *d_jitter_coarse, const float *d_jitter_fine, float *d_rgb, float *d_acc, float *d_depth,
                                       uint8_t *d_mask, void *stream) {
    TrainFwd tf{d_jitter_coarse, d_jitter_fine};
    return render_impl(h, cfg, d_origins, d_directions, R, d_rgb, d_acc, d_depth, d_mask, &tf, stream);
}

// backward of the LAST tn_render_train_forward: d_grad_rgb f32[R,3] (dL/d rgb), d_grad_acc f32[R] or NULL (dL/d accumulation) ->
// d_grad_field f32[64,V] and the twelve MLP parameter gradients (same order / layouts as tn_render_set_weights); every output element
// is written.  The coarse pass carries no gradient (PDFSampler detaches its bins).  No [samples,128] tensor touches HBM.
extern "C" int tn_render_train_backward(tn_tracer *h, const float *d_grad_rgb, const float *d_grad_acc, int use_gradient_scaling,
                                        float *d_grad_field, float *const *d_grad_params12, void *stream) {
    if (!h || !d_grad_rgb || !d_grad_field || !d_grad_params12) return fail(TN_ERR_ARG, "null argument");
    RenderState *r = h->render;
    if (!r || !r->train_valid) return fail(TN_ERR_STATE, "tn_render_train_backward: no training forward to continue from");
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    const uint32_t R = r->t_R, S2 = r->t_S2, V = r->V;
    const bool det = r->t_det;
    if (det) {
        const int rc = ensure_det_ws(r, R, S2);
        if (rc) return rc;
    }
    TN_CUDA(cudaMemsetAsync(r->gw, 0, sizeof(float) * GW_TOTAL, s));
    if (!det) {  // (deterministic mode writes every element of these)
        TN_CUDA(cudaMemsetAsync(r->gshadow, 0, sizeof(float) * 64 * (size_t)V, s));
        TN_CUDA(cudaMemsetAsync(r->g_dirbias, 0, 512 * (size_t)R, s));
        TN_CUDA(cudaMemsetAsync(r->n_active + 3, 0, 4, s));  // tile counter of the backward kernel (word 3 of the 16-byte block)
    }
    CompositeBwdParams cb{};
    cb.S2 = S2; cb.use_gradient_scaling = use_gradient_scaling ? 1u : 0u; cb.n_active = r->n_active; cb.ray_list = r->ray_list;
    cb.ebins_f = r->ebins_f; cb.sbins_f = r->sbins_f; cb.out_f = r->out_f; cb.grad_rgb = d_grad_rgb; cb.grad_acc = d_grad_acc;
    cb.bg0 = r->t_bg[0]; cb.bg1 = r->t_bg[1]; cb.bg2 = r->t_bg[2]; cb.dout = r->dout; cb.sums = det ? (float *)r->det_sums : r->gw + GW_SUMS;
    const size_t smem_cb = SAMPLE_WARPS * sizeof(float) * 4 * ((size_t)S2 + 2);
    auto k_cbwd = det ? k_composite_bwd<true> : k_composite_bwd<false>;
    TN_CUDA(cudaFuncSetAttribute(k_cbwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cb));
    const uint32_t gridR = (R + SAMPLE_WARPS - 1) / SAMPLE_WARPS;
    if (r->profile) cudaEventRecord(r->evb[0], s);
    k_cbwd<<<gridR, SAMPLE_WARPS * 32, smem_cb, s>>>(cb);
    if (r->profile) cudaEventRecord(r->evb[1], s);
    MlpBwdParams bp{};
    bp.n_active = r->n_active; bp.S = S2; bp.vi = r->vi_f; bp.bary = r->bary_f; bp.fshadow = r->fshadow; bp.wimg = r->wimg_bwd;
    bp.bias = r->bias; bp.head = r->head; bp.dirbias = r->dirbias; bp.dout = r->dout; bp.gshadow = r->gshadow;
    bp.gw = r->gw; bp.g_dirbias = r->g_dirbias; bp.tile_ctr = r->n_active + 3;
    const uint64_t tiles = ((uint64_t)R * S2 + BWD_TILE - 1) / BWD_TILE;
    if (!det) {
        TN_CUDA(cudaFuncSetAttribute(k_mlp_bwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM_BYTES));
        const uint32_t grid = r->bwd_grid ? r->bwd_grid : (uint32_t)std::min<uint64_t>(tiles, (uint64_t)sms);
        k_mlp_bwd<false><<<grid, BWD_THREADS, BWD_SMEM_BYTES, s>>>(bp);
        if (r->profile) cudaEventRecord(r->evb[2], s);
        k_dirbias_grads<false><<<(R + DBG_SLOTS - 1) / DBG_SLOTS, 256, 0, s>>>(r->n_active, r->g_dirbias, r->enc, r->gw, nullptr);
    } else {
        // the same stages with every reduction in a fixed order (header of tn_mlp_bwd.cuh); the grid only decides which CTA runs
        // which partition, never what is summed in which order
        MlpBwdDetParams dp{};
        static_cast<MlpBwdParams &>(dp) = bp;
        dp.part = r->det_part; dp.gdb_part = r->det_gdb; dp.dx = r->det_dx;
        TN_CUDA(cudaFuncSetAttribute(k_mlp_bwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_DET_SMEM_BYTES));
        const uint32_t grid = r->bwd_grid ? r->bwd_grid : std::min<uint32_t>(BWD_PARTS, (uint32_t)sms);
        k_mlp_bwd<true><<<grid, BWD_THREADS, BWD_DET_SMEM_BYTES, s>>>(dp);
        if (r->profile) cudaEventRecord(r->evb[2], s);
        k_det_reduce_parts<<<(BWD_PART_STRIDE + 255) / 256, 256, 0, s>>>(r->n_active, S2, r->det_part, r->gw);
        k_det_sum_slots<<<1, 256, 0, s>>>(r->n_active, r->det_sums, r->gw + GW_SUMS);
        k_det_dirbias<<<R, 128, 0, s>>>(r->n_active, S2, r->det_gdb, r->g_dirbias);
        k_dirbias_grads<true><<<(R + DBG_SLOTS - 1) / DBG_SLOTS, 256, 0, s>>>(r->n_active, r->g_dirbias, r->enc, r->gw, r->det_dbg);
        k_det_reduce_dbg<<<(DBG_PART + 255) / 256, 256, 0, s>>>(r->n_active, r->det_dbg, r->gw);
        // field gradient: stable sort of (vertex, row * 4 + k) by vertex, then per-vertex sums in row order
        const uint32_t n = (uint32_t)(4 * (uint64_t)R * S2);
        const int end_bit = 32 - __builtin_clz(V | 1u);  // keys are <= V
        uint32_t *k0 = r->det_keys, *k1 = r->det_keys + n, *v0 = r->det_vals, *v1 = r->det_vals + n;
        size_t bytes = 0;
        TN_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k0, k1, v0, v1, (int)n, 0, end_bit, s));
        const int rc = ensure_cub_tmp(r, bytes);
        if (rc) return rc;
        k_det_field_keys<<<(n + 255) / 256, 256, 0, s>>>(r->n_active, S2, n, V, (const uint4 *)r->vi_f, k0, v0);
        TN_CUDA(cub::DeviceRadixSort::SortPairs(r->cub_tmp, bytes, k0, k1, v0, v1, (int)n, 0, end_bit, s));
        k_det_field_grad<<<(uint32_t)(((uint64_t)V * 32 + 255) / 256), 256, 0, s>>>(V, n, k1, v1, r->bary_f, r->det_dx, r->gshadow);
        h->launches += 9;
    }
    GradOut go{};
    for (int i = 0; i < 12; ++i) {
        if (!d_grad_params12[i]) return fail(TN_ERR_ARG, "tn_render_train_backward: null parameter gradient pointer");
        go.p[i] = d_grad_params12[i];
    }
    k_scatter_grads<<<(128 * 155 + 255) / 256, 256, 0, s>>>(r->gw, go);
    k_transpose_v64<<<(V + 31) / 32, dim3(32, 8), 0, s>>>(r->gshadow, d_grad_field, V);
    if (r->profile) cudaEventRecord(r->evb[3], s);
    h->launches += 5;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

// deterministic mode of the fused training step (see the header): applies from the next tn_render_train_forward on
extern "C" int tn_render_set_deterministic(tn_tracer *h, int enable) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    DeviceGuard g(h->device);
    state(h)->det = enable != 0;
    return TN_OK;
}

// test hook: CTAs of the backward MLP kernel (0 = default: one per SM, capped by the tiles / partitions)
extern "C" int tn_render_set_backward_grid(tn_tracer *h, uint32_t ctas) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    DeviceGuard g(h->device);
    state(h)->bwd_grid = ctas;
    return TN_OK;
}

// fused pixel gather: from now on tn_render stores every pixel into all ranks' gathered buffers (peer memory) from inside its own
// kernels -- the all-gather of the rendered pixels without a collective call.  world == 0 switches it off.
extern "C" int tn_render_set_gather(tn_tracer *h, uint32_t world, uint32_t rank, void *const *d_peer_buffers, uint32_t rays_per_rank) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (world > 8 || (world && (rank >= world || !d_peer_buffers || rays_per_rank == 0))) return fail(TN_ERR_ARG, "tn_render_set_gather: world <= 8, rank < world");
    RenderState *r = state(h);
    for (uint32_t k = 0; k < 8; ++k) r->peer[k] = k < world ? (float *)d_peer_buffers[k] : nullptr;
    for (uint32_t k = 0; k < world; ++k) if (!r->peer[k]) return fail(TN_ERR_ARG, "tn_render_set_gather: null peer buffer");
    r->gather_world = world; r->gather_rank = rank; r->gather_stride = rays_per_rank;
    return TN_OK;
}

// per-kernel timing of the LAST tn_render call (trace, sample_coarse, mlp_coarse, sample_fine, mlp_fine, composite), ms.
// enable with tn_render_set_profiling(h, 1); the getter synchronises on the last event.
extern "C" int tn_render_set_profiling(tn_tracer *h, int enable) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    DeviceGuard g(h->device);
    RenderState *r = state(h);
    if (enable) for (auto &e : r->ev) if (!e) TN_CUDA(cudaEventCreate(&e));
    if (enable) for (auto &e : r->evb) if (!e) TN_CUDA(cudaEventCreate(&e));
    r->profile = enable != 0;
    return TN_OK;
}
extern "C" int tn_render_get_timings(tn_tracer *h, float *ms6) {
    if (!h || !h->render || !h->render->profile) return fail(TN_ERR_STATE, "profiling is not enabled");
    DeviceGuard g(h->device);
    RenderState *r = h->render;
    TN_CUDA(cudaEventSynchronize(r->ev[6]));
    for (int i = 0; i < 6; ++i) TN_CUDA(cudaEventElapsedTime(&ms6[i], r->ev[i], r->ev[i + 1]));
    return TN_OK;
}

// per-kernel timing of the LAST tn_render_train_backward call: ms3 = composite_bwd, mlp_bwd, finalize (memsets excluded)
extern "C" int tn_render_get_backward_timings(tn_tracer *h, float *ms3) {
    if (!h || !h->render || !h->render->profile) return fail(TN_ERR_STATE, "profiling is not enabled");
    DeviceGuard g(h->device);
    RenderState *r = h->render;
    TN_CUDA(cudaEventSynchronize(r->evb[3]));
    for (int i = 0; i < 3; ++i) TN_CUDA(cudaEventElapsedTime(&ms3[i], r->evb[i], r->evb[i + 1]));
    return TN_OK;
}

// test / debug hook: device pointers of the intermediate buffers of the last tn_render call
extern "C" int tn_render_debug_buffers(tn_tracer *h, void **ptrs16) {
    if (!h || !h->render) return fail(TN_ERR_STATE, "no render state");
    RenderState *r = h->render;
    void *v[16] = {r->num, r->dist, r->n_active, r->ray_list, r->ebins_c, r->sbins_c, r->vi_c, r->bary_c,
                   r->dens_c, r->ebins_f, r->vi_f, r->bary_f, r->out_f, r->dirbias, r->fshadow, r->wimg};
    for (int i = 0; i < 16; ++i) ptrs16[i] = v[i];
    return TN_OK;
}
