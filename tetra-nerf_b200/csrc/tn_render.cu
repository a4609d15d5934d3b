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
#include <atomic>
#include <cmath>
#include <vector>

#include <cstddef>
#include <cstdlib>
#include <cub/cub.cuh>
#include "tn_background.cuh"
#include "tn_common.cuh"
#include "tn_composite.cuh"
#include "tn_direnc.cuh"
#include "tn_mlp.cuh"
#include "tn_mlp_bwd.cuh"
#include "tn_mlp_pack.cuh"
#include "tn_sort.cuh"

namespace tn {

int launch_trace_internal(tn_tracer *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells, float *bary,
                          float *dist, uint32_t *verts, int dense, cudaStream_t s);

// the buffers a render or training forward leaves behind (and a training forward's backward continues from), laid out by saved_layout
// in a saved-state blob: the caller's (tn_render_train_forward_saved) or the tracer's own (RenderState::own)
struct TrainBufs {
    uint32_t *n_active;        // 16-byte block: active rays | tile counter of the coarse pass | of the fine pass | of the normals pass;
                               // then words 4, 5: the clip bounds of the expected depth, 6, 7: the live rows of the coarse / fine pass
                               // when the forward culled (in the slot the saved state reserves for the block)
    uint32_t *ray_list;        // [R] slot -> ray
    float *ebins_f, *sbins_f;  // [R,S2+1] euclidean / spacing bins of the fine pass
    uint4 *vi_f;               // [R*S2] matched vertices
    float *bary_f;             // [R*S2,3] their weights
    float *out_f;              // [R*S2] (sigma, r, g, b) head pre-activations
    float *dirbias, *enc;      // [R,128] direction bias, [R,27] encoded direction
    float *dirs;               // [R,3] the ray directions of a training forward with a background map (nullptr: none kept)
};

// header of a saved-state blob: what a training forward ran with, which its backward continues in
constexpr uint32_t SAVED_MAGIC = 0x53564e54u;  // "TNVS"
struct SavedHeader {
    uint32_t magic, R, M, Sc, Sf, S2, det;
    uint32_t edepth;           // 1: the forward produced the expected depth (its clip bounds are in words 4, 5 of the n_active slot)
    float bg[3];
    uint32_t pad2;
    uint64_t gen;              // RenderState::gen at the forward
    uint64_t mesh_gen;         // tn_tracer::mesh_gen at the forward (the ray gradients read the mesh positions)
    uint32_t cull;             // 1: the forward culled samples by occupancy (its culled rows are marked in vi_f, DESIGN §4.12)
    uint32_t live_c, live_f;   // culling: the live rows of its coarse / fine pass (copied on the device from the n_active slot)
    uint32_t pad3;
    uint32_t bgmap;            // 1: the forward composited over the background map (tn_render_set_background; its directions are kept)
    uint32_t bg_H, bg_W, pad4;
    uint64_t bg_gen;           // RenderState::bg_gen at the forward
};

struct RenderState {
    // field
    DevArray<float> fshadow;   // [V,64] in fragment order (field_pos)
    uint32_t V = 0;
    // weights
    DevArray<uint8_t> wimg;    // L1 32K | L2 64K | L3 64K | L4(base part) 64K  (bf16 hi/lo)
    DevArray<uint8_t> wimg16;  // the same image with fp16 hi/lo halves (mlp_prec == 2)
    int mlp_prec = 2;          // operand precision of the inference MLP: 2 = f16w2 (default), 3 = bf16x3 (tn_mlp.cuh); training always runs 3
    DevArray<float> bias;      // b1 b2 b3 [3][128]
    DevArray<float> head;      // wd[128] wc[3][128] bd bc[3]
    DevArray<float> w4dir;     // [128][27] + b4[128]
    bool have_weights = false;
    uint64_t gen = 0;          // generation of field + weights: a fresh value from next_generation() on every set_field / set_weights
    // workspace
    DevArray<uint32_t> num, cells, verts;  // trace output: [R], [R,M], [R,M,4]
    DevArray<float> bary, dist;            // [R,M,6], [R,M,2]
    DevArray<float> ebins_c, sbins_c, bary_c, dens_c;  // [R,Sc+1], [R,Sc+1], [R*Sc,3], [R*Sc]
    DevArray<uint4> vi_c;                  // [R*Sc]
    // the tracer's own fine-pass state (tn_render, tn_render_train_forward): a saved-state blob, its arrays as the last call that wrote
    // it laid them out, and the host-side header of the last tn_render_train_forward (magic 0: no forward to continue from)
    DevArray<uint8_t> own;
    TrainBufs own_b{};
    SavedHeader last{};
    // training: backward weight image, per-sample head gradients, accumulators (scratch of every backward, saved state or not)
    DevArray<uint8_t> wimg_bwd;        // 7 stages of 32 KB (tn_mlp_bwd.cuh)
    DevArray<float4> dout;             // [R*S2] gradients at the head pre-activations
    DevArray<float> gshadow, gw, g_dirbias;  // [V,64], [GW_TOTAL] + the backward kernel's tile counter, [R,128]
    // fused pixel gather (tn_render_set_gather): peer[k] = rank k's [world * rays_per_rank, 6] gathered-pixel buffer
    float *peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    uint32_t gather_world = 0, gather_rank = 0, gather_stride = 0;
    // optional per-kernel timing (bench.py roofline): events around the 6 kernels of tn_render
    bool profile = false;
    cudaEvent_t ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t evb[4] = {nullptr, nullptr, nullptr, nullptr};  // backward: start | composite_bwd | mlp_bwd | finalize
    // deterministic mode (tn_render_set_deterministic): ordered slots in the training forward, fixed-order reductions in its backward
    bool det = false;                  // mode of the next training forward (initial value: TETRANERF_B200_DETERMINISTIC)
    uint32_t bwd_grid = 0;             // CTAs of the backward MLP kernel (test hook; 0 = default)
    int smem_optin = 0;                // the device's opt-in dynamic shared memory per block (read on the first render call)
    DevArray<uint32_t> ray_flag, ray_slot;  // [R] ray has hits, its slot (exclusive scan)
    DevArray<uint8_t> cub_tmp;         // CUB scan / sort temporary storage
    DevArray<float> det_part;          // [BWD_PARTS][BWD_PART_STRIDE] per-partition dW / column sums
    DevArray<float> det_gdb;           // [4 (ntiles + R)][128] direction-bias gradient partials
    DevArray<float> det_dx;            // [R*S2,64] feature gradient per sample
    DevArray<float4> det_sums;         // [R] head-bias gradient per slot
    DevArray<float> det_dbg;           // [R/64][128*28] partial W4dir / b4 gradients per block of k_dirbias_grads
    DevArray<uint32_t> det_keys, det_vals;  // [2][R*S2*4] (vertex, sample row * 4 + k) pairs, sort input | output
    // normal map (tn_render with d_normals): density gradient per sample of the last normals render
    DevArray<float4> grad_n;
    // ray gradients (tn_render_train_backward_saved with ray or vertex outputs): dX rows of the default mode (the deterministic mode keeps them in det_dx),
    // dL/dx per sample of the last such backward
    DevArray<float> ray_dx;
    DevArray<float4> ray_gx;
    // occupancy culling (tn_render_set_occupancy; DESIGN §4.12): the borrowed per-tetrahedron field and its threshold (occ == nullptr:
    // off), the live-row flags and compact-row maps of the passes (coarse, fine, the backward's rebuilt one) and the backward's row count
    const float *occ = nullptr;
    float occ_thr = 0.f;
    bool occ_place = false;            // occupancy sampling (DESIGN §4.13): coarse bins in the kept records only
    uint32_t occ_T = 0;                // the mesh's tetrahedron count when the occupancy was set
    DevArray<uint8_t> live_flag;
    DevArray<uint32_t> rowmap_c, rowmap_f, rowmap_b, rows_b;
    // tn_occupancy_update: probe rows of one chunk of tetrahedra, their densities, the chunk's row count and tile counter
    DevArray<uint4> occ_vi;
    DevArray<float> occ_bary, occ_sig;
    DevArray<uint32_t> occ_small;
    // background map (tn_render_set_background; DESIGN §4.16): borrowed f32[H,W,3] (nullptr: the constant cfg->background), its
    // generation (bumped by every set), and the backward's per-ray grad_rgb (1 - accumulation) and deterministic sort buffers
    const float *bgmap = nullptr;
    uint32_t bg_H = 0, bg_W = 0;
    uint64_t bg_gen = 0;
    DevArray<float> bg_s;
    DevArray<uint32_t> bg_keys, bg_vals;
};

void free_render(tn_tracer *h) {
    if (!h->render) return;
    RenderState *r = h->render;
    for (auto &e : r->ev) if (e) cudaEventDestroy(e);
    for (auto &e : r->evb) if (e) cudaEventDestroy(e);
    delete r;
    h->render = nullptr;
}

// generations are unique across tracers, so a saved state recorded on one tracer never matches another tracer's field and weights
uint64_t next_generation() {
    static std::atomic<uint64_t> g{0};
    return ++g;
}

int render_inputs(tn_tracer *h, RenderInputs *out) {
    const RenderState *r = h->render;
    if (!r || !r->fshadow.p || !r->have_weights) return TN_ERR_STATE;
    *out = RenderInputs{r->fshadow.p, r->V, r->wimg.p, r->bias.p, r->head.p, r->w4dir.p, r->gen};
    return TN_OK;
}

int field_shadow(const tn_tracer *h, const float **fshadow, uint32_t *V) {
    const RenderState *r = h->render;
    if (!r || !r->fshadow.p) return TN_ERR_STATE;
    *fshadow = r->fshadow.p;
    *V = r->V;
    return TN_OK;
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
// [64,V] -> [V,64], each row in fragment order (field_pos)
__global__ void k_transpose64(const float *__restrict__ in, float *__restrict__ out, uint32_t V) {
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
            out[(size_t)v * 64 + field_pos(threadIdx.x)] = tile[threadIdx.x][r];
            out[(size_t)v * 64 + field_pos(32 + threadIdx.x)] = tile[32 + threadIdx.x][r];
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
    // expected depth (k_composite<true>): unclipped depth per active ray [R]; ordered keys of the smallest / largest sample midpoint
    // of the call (DESIGN §4.10)
    float *edepth;
    uint32_t *dbounds;
    // occupancy culling: the trace's visited cells [R,M] and the per-tetrahedron occupancy (nullptr: off) with its threshold
    const uint32_t *cells;
    const float *occ;
    float occ_thr;
    // background map (nullptr: the constant bg0..bg2)
    const float *bgmap;
    uint32_t bg_H, bg_W;
};

// a culled sample (matched to a tetrahedron whose occupancy is below the threshold): vi = (E, E, E, TN_CULLED), weights 0.  Every
// consumer that tests vi.x treats it as unmatched (no field gradient, no ray or vertex gradient, no normal); k_live_rows tells it from a
// truly unmatched sample, whose density MLP(0) is still evaluated, and gives it sigma = 0 without evaluating the MLP.  A sample matched
// to a gap record (cell E, between two hull faces of a non-convex mesh) has no tetrahedron and is never culled.
#define TN_CULLED 0xFFFFFFFEu
__device__ __forceinline__ bool cell_culled(const SampleParams &p, uint32_t cell) { return cell != TN_EMPTY && __ldg(p.occ + cell) < p.occ_thr; }
__device__ __forceinline__ void cull_sample(const SampleParams &p, size_t row, uint32_t seg, uint4 &vi, float &b0, float &b1, float &b2) {
    if (vi.x == TN_EMPTY) return;
    if (cell_culled(p, __ldg(p.cells + row + seg))) {
        vi = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_CULLED);
        b0 = b1 = b2 = 0.f;
    }
}

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
// torch.linspace(start, end, steps)[i] for float32 (symmetric fill of ATen's linspace kernel)
__device__ __forceinline__ float linspace_f(float start, float end, uint32_t steps, uint32_t i) {
    const float step = (end - start) / (float)(steps - 1);
    return i < steps / 2 ? start + step * (float)i : end - step * (float)(steps - i - 1);
}

// find_visited_cells for one sample distance d: binary search over the staged prefix-max of t_out, then the segment's own
// (t_in, t_out) from the trace output (L1: the warp has just read the row)
// returns the matched segment (meaningful when vi.x != E)
__device__ __forceinline__ uint32_t match_sample(float d, uint32_t n, const float2 *__restrict__ dist, const float *pm, size_t row,
                                                 const uint4 *__restrict__ verts, const float *__restrict__ bary, uint4 &vi, float &b0,
                                                 float &b1, float &b2) {
    vi = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
    b0 = b1 = b2 = 0.f;
    uint32_t lo = 0, hi = n;  // first p with pm[p] >= d  (== the reference's monotone pointer walk for sorted samples)
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pm[mid] < d) lo = mid + 1; else hi = mid;
    }
    if (lo >= n) return lo;
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
    return lo;
}

// shared memory per warp.  Only the prefix-max of t_out (binary-searched by every sample) is staged per segment; t_in / t_out are
// read from the trace output where needed.  Coarse pass: pm[M+2], cum[M+2] (biased sampler only), e[Sc+2] = 4.6 KB at M = 512,
// Sc = 128; fine pass: pm[M+2] and cdf / e / x / y of Smax+2 = 6.2 KB -- every ray of a 4096-ray batch is resident at once
// (28 warps per SM; round 1 staged three segment arrays and sized all bin arrays for the worst case: 14.4 / 10.3 KB per warp,
// 12 / 20 warps per SM, i.e. the coarse pass ran in 2.3 waves).
__host__ __device__ __forceinline__ size_t seg_arr(uint32_t M) { return (size_t)M + 2; }
__host__ __device__ __forceinline__ size_t coarse_floats(uint32_t M, uint32_t Sc, uint32_t biased) { return seg_arr(M) * (biased ? 2 : 1) + (size_t)Sc + 2; }
__host__ __device__ __forceinline__ size_t fine_floats(uint32_t M, uint32_t Smax) { return seg_arr(M) + 4 * ((size_t)Smax + 2); }
// occupancy sampling (PLACE): pm, cum, the kept records' indices kix, e -- either sampler; at most 160 KB per block (M = 2048,
// Sc = 4096), so every accepted setting fits
__host__ __device__ __forceinline__ size_t place_floats(uint32_t M, uint32_t Sc) { return 3 * seg_arr(M) + (size_t)Sc + 2; }

// ORDERED (deterministic mode): the slot of a ray is its rank among the rays with hits (p.ray_slot), so slot order = ray order;
// otherwise slots are claimed with an atomic counter.
// PLACE (occupancy sampling, DESIGN §4.13; needs p.occ): a ray with both skipped records (a tetrahedron below the threshold) and kept
// ones places its bins in the kept records only: the biased sampler gives each kept record an equal share of [0, 1], the uniform one
// spreads them uniformly over the kept length.  near / far and the spacing bins' definition stay as they are.  A ray with no skipped or
// no kept record takes the code path of !PLACE, so its bins are the same bits.
template <bool ORDERED, bool PLACE = false>
__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_sample_coarse(const SampleParams p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t ray = blockIdx.x * SAMPLE_WARPS + warp;
    if (ray >= p.R) return;
    const uint32_t M = p.M, S = p.Sc;
    const size_t A = seg_arr(M);
    float *pm = sm + (size_t)warp * (PLACE ? place_floats(M, S) : coarse_floats(M, S, p.biased));
    float *cum = pm + A, *e = PLACE ? cum + 2 * A : cum + (p.biased ? A : 0);
    const uint32_t n = p.num[ray];
    if constexpr (ORDERED) {
        if (ray == p.R - 1 && lane == 0) *p.n_active = p.ray_slot[ray] + (n > 0 ? 1u : 0u);
    }
    if (n == 0) {  // model.py:640-650 : background colour, accumulation 0, depth = collider far plane
        float b0 = p.bg0, b1 = p.bg1, b2 = p.bg2;
        if (p.bgmap != nullptr) {  // bg(d), clamped to [0,1] in eval mode as every other pixel
            bg_lookup(p.bgmap, p.bg_H, p.bg_W, p.d[3 * (size_t)ray], p.d[3 * (size_t)ray + 1], p.d[3 * (size_t)ray + 2], b0, b1, b2);
            if (!p.train) { b0 = fminf(fmaxf(b0, 0.f), 1.f); b1 = fminf(fmaxf(b1, 0.f), 1.f); b2 = fminf(fmaxf(b2, 0.f), 1.f); }
        }
        store_pixel(p, ray, lane, b0, b1, b2, 0.f, p.far_plane, 0);
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
    bool placed = false;
    uint32_t nk = 0;  // PLACE: the kept records, their indices in kix[0..nk) in ray order
    uint32_t *kix = reinterpret_cast<uint32_t *>(cum + A);
    if constexpr (PLACE) {
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t k = base + lane;
            const bool kept = k < n && !cell_culled(p, __ldg(p.cells + row + k));
            const uint32_t bal = __ballot_sync(0xffffffffu, kept);
            if (kept) kix[nk + __popc(bal & ((1u << lane) - 1u))] = k;
            nk += __popc(bal);
        }
        placed = nk > 0 && nk < n;  // (warp-uniform)
    }
    for (uint32_t k = lane; k < n; k += 32) {
        const float2 h = __ldg(&p.dist[row + k]);
        pm[k] = h.y;
        if (p.biased && !placed) cum[k + 1] = fmaxf(h.y - h.x, 0.f);  // map_from_real_distances_to_biased_with_bounds, model.py:111-122
    }
    if (p.biased && !placed && lane == 0) cum[0] = near;
    if (placed && !p.biased) {  // cum[i] = the kept length before the i-th kept record, cum[nk] = all of it
        __syncwarp();
        for (uint32_t i = lane; i < nk; i += 32) {
            const float2 h = __ldg(&p.dist[row + kix[i]]);
            cum[i + 1] = fmaxf(h.y - h.x, 0.f);
        }
        if (lane == 0) cum[0] = 0.f;
    }
    __syncwarp();
    smem_scan_max(pm, pm, n, lane);  // in place
    if (p.biased && !placed) {
        // cum[k] = start + sum_{i<k} len_i : scan over [start, len_0, len_1, ...]
        smem_scan_add(cum, n + 1, lane);
    }
    if (placed) {
        if (!p.biased) smem_scan_add(cum, nk + 1, lane);
        for (uint32_t j = lane; j <= S; j += 32) {
            float b = linspace_f(0.f, 1.f, S + 1, j);
            if (p.jit_c != nullptr) {  // the same stratified jitter as below
                const float lower = j == 0 ? b : (b + linspace_f(0.f, 1.f, S + 1, j - 1)) / 2.0f;
                const float upper = j == S ? b : (linspace_f(0.f, 1.f, S + 1, j + 1) + b) / 2.0f;
                b = lower + (upper - lower) * __ldg(p.jit_c + (size_t)ray * (S + 1) + j);
            }
            uint32_t i;
            float off;
            if (p.biased) {  // map_from_real_distances_to_biased_with_bounds over the kept records
                const float uni = (b * far + (1.f - b) * near - near) / (far - near);
                float rest = uni * (float)nk;
                float iv = fminf(floorf(rest), (float)(nk - 1));
                iv = fmaxf(iv, 0.f);
                rest = rest - iv;
                i = (uint32_t)iv;
                const float2 hk = __ldg(&p.dist[row + kix[i]]);
                off = fmaxf(hk.y - hk.x, 0.f) * rest;
            } else {  // x = b L: the last kept record whose cumulative start is <= x
                const float x = b * cum[nk];
                uint32_t lo = 1, hi = nk;
                while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (cum[mid] <= x) lo = mid + 1; else hi = mid; }
                i = lo - 1;
                off = x - cum[i];
            }
            const float2 h = __ldg(&p.dist[row + kix[i]]);
            e[j] = fminf(h.x + off, fmaxf(h.x, h.y));  // (rounding never leaves the record)
        }
        __syncwarp();
        smem_scan_max(e, e, S + 1, lane);  // sorted bins even where two records overlap by a rounding
        for (uint32_t j = lane; j <= S; j += 32) {
            p.ebins_c[(size_t)slot * (S + 1) + j] = e[j];
            p.sbins_c[(size_t)slot * (S + 1) + j] = (e[j] - near) / (far - near);  // model.py:182
        }
    } else {
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
    }
    __syncwarp();
    for (uint32_t j = lane; j < S; j += 32) {
        const float dmid = (e[j + 1] + e[j]) / 2.f;  // model.py:557
        uint4 vi; float b0, b1, b2;
        const uint32_t seg = match_sample(dmid, n, p.dist, pm, row, p.verts, p.bary, vi, b0, b1, b2);
        if (p.occ != nullptr) cull_sample(p, row, seg, vi, b0, b1, b2);
        const size_t g = (size_t)slot * S + j;
        p.vi_c[g] = vi;
        p.bary_c[3 * g] = b0; p.bary_c[3 * g + 1] = b1; p.bary_c[3 * g + 2] = b2;
    }
}

// direction encoding folded into a per-ray bias of mlp_head (model.py:607-620): dirbias[slot] = b4 + W4[:, :27] . enc(dir)
// NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0, max_freq_exp=4, include_input=True), model.py:426-432
__device__ __forceinline__ void dir_bias(const SampleParams &p, uint32_t ray, uint32_t slot, int lane) {
    const float dx = p.d[3 * (size_t)ray], dy = p.d[3 * (size_t)ray + 1], dz = p.d[3 * (size_t)ray + 2];
    float enc[27];
    encode_direction(dx, dy, dz, enc);
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
        const uint32_t seg = match_sample(dmid, n, p.dist, pm, row, p.verts, p.bary, vi, b0, b1, b2);
        if (p.occ != nullptr) cull_sample(p, row, seg, vi, b0, b1, b2);
        const size_t g = (size_t)slot * S2 + j;
        p.vi_f[g] = vi;
        p.bary_f[3 * g] = b0; p.bary_f[3 * g + 1] = b1; p.bary_f[3 * g + 2] = b2;
    }
    dir_bias(p, ray, slot, lane);
}

// expected depth (DESIGN §4.10): the clip bounds are the smallest / largest sample midpoint over every active ray of the call, reduced
// with atomicMin / atomicMax on an order-preserving unsigned key of the float (exact and order-independent)
__device__ __forceinline__ uint32_t depth_key(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float depth_unkey(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// DEPTH: also the unclipped expected depth sum_j w_j t_j / (sum_j w_j + 1e-10) of the ray (-> p.edepth) and its midpoints' share of the
// call's clip bounds (-> p.dbounds); k_expected_depth_finalize clips.  The other outputs are the same bits either way.
template <bool DEPTH>
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
    float dt = 0.f, tlo = 3.4028234663852886e38f, thi = -3.4028234663852886e38f;  // (DEPTH only)
    for (uint32_t j = lane; j < S2; j += 32) {
        const float4 c = of[j];
        const float wj = w[j];
        if (p.train) { r += wj * c.y; g += wj * c.z; b += wj * c.w; a += wj; }  // RGBRenderer in training: no nan_to_num, no clamp
        else { r += wj * nan_to_num_f(c.y); g += wj * nan_to_num_f(c.z); b += wj * nan_to_num_f(c.w); a += wj; }
        if constexpr (DEPTH) {  // DepthRenderer("expected"): steps = (starts + ends) / 2
            const float t = (eb[j] + eb[j + 1]) / 2.f;
            dt += wj * t;
            tlo = fminf(tlo, t); thi = fmaxf(thi, t);
        }
    }
    r = warp_sum_f(r); g = warp_sum_f(g); b = warp_sum_f(b); a = warp_sum_f(a);
    if constexpr (DEPTH) {
        dt = warp_sum_f(dt);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            tlo = fminf(tlo, __shfl_xor_sync(0xffffffffu, tlo, o));
            thi = fmaxf(thi, __shfl_xor_sync(0xffffffffu, thi, o));
        }
        if (lane == 0) {
            p.edepth[ray] = dt / (a + 1e-10f);
            atomicMin(p.dbounds, depth_key(tlo));
            atomicMax(p.dbounds + 1, depth_key(thi));
        }
    }
    // DepthRenderer("median"): first sample whose cumulative weight reaches 0.5
    for (uint32_t j = lane; j < S2; j += 32) tr[j] = w[j];
    __syncwarp();
    smem_scan_add(tr, S2, lane);
    uint32_t first = S2;
    for (uint32_t j = lane; j < S2; j += 32) if (tr[j] >= 0.5f) { first = j; break; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    const uint32_t mi = min(first, S2 - 1);
    // RGBRenderer: comp + background * (1 - acc); clamped to [0,1] in eval mode only.  The background is bg(d) with a map
    float b0 = p.bg0, b1 = p.bg1, b2 = p.bg2;
    if (p.bgmap != nullptr) bg_lookup(p.bgmap, p.bg_H, p.bg_W, p.d[3 * (size_t)ray], p.d[3 * (size_t)ray + 1], p.d[3 * (size_t)ray + 2], b0, b1, b2);
    float pr = r + b0 * (1.f - a), pg = g + b1 * (1.f - a), pb = b + b2 * (1.f - a);
    if (!p.train) { pr = fminf(fmaxf(pr, 0.f), 1.f); pg = fminf(fmaxf(pg, 0.f), 1.f); pb = fminf(fmaxf(pb, 0.f), 1.f); }
    store_pixel(p, ray, lane, pr, pg, pb, a, (eb[mi] + eb[mi + 1]) / 2.f, 1);
}

// after k_composite<true>: D = clip(D_raw, t_min, t_max) on active rays (NaN passes through, as torch.clip), far_plane on empty ones
__global__ void k_expected_depth_finalize(uint32_t R, const uint32_t *__restrict__ num, const uint32_t *__restrict__ dbounds, float far_plane,
                                          float *__restrict__ edepth) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    if (num[i] == 0) { edepth[i] = far_plane; return; }
    const float lo = depth_unkey(dbounds[0]), hi = depth_unkey(dbounds[1]), x = edepth[i];
    edepth[i] = x < lo ? lo : (x > hi ? hi : x);
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
    const float *grad_ed;              // DEPTH: [R] dL/d expected depth
    const uint32_t *dbounds;           // DEPTH: the forward's clip bounds (ordered keys, k_composite<true>)
    const float *grad_dist;            // DIST: [R] dL/d distortion
    const float *bgmap;                // background map [H,W,3] (nullptr: the constant bg0..bg2); then bg(d) of the saved directions, and
    uint32_t bg_H, bg_W;               //   bg_s[ray] = grad_rgb (1 - accumulation), the map's and the directions' per-ray weight
    const float *dirs;
    float *bg_s;
};

// ---- distortion loss (DESIGN §4.11; mip-NeRF 360, nerfstudio losses.distortion_loss) over the fine pass of one ray: spacing bins s_0..s_S2,
// u_i = (s_i + s_{i+1}) / 2, delta_i = s_{i+1} - s_i, w_i the weights of rgb:
//   d = sum_i sum_j w_i w_j |u_i - u_j| + 1/3 sum_i w_i^2 delta_i = 2 sum_j w_j (u_j W_<j - P_<j) + 1/3 sum_j w_j^2 delta_j
// with W, P the prefix sums of w and w u (the bins are sorted), in one pass of warp scans.
struct DistortionParams {
    uint32_t S2;
    const uint32_t *n_active, *ray_list;
    const float *ebins_f, *sbins_f, *out_f;
    float *dist;                       // [R], zeroed by the caller (empty rays stay 0)
};
__global__ void __launch_bounds__(SAMPLE_WARPS * 32) k_distortion(const DistortionParams p) {
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot = blockIdx.x * SAMPLE_WARPS + warp;
    if (slot >= *p.n_active) return;
    const uint32_t S2 = p.S2;
    float *w = sm + (size_t)warp * (2 * ((size_t)S2 + 2)), *tr = w + S2 + 2;
    const float *eb = p.ebins_f + (size_t)slot * (S2 + 1);
    const float *sb = p.sbins_f + (size_t)slot * (S2 + 1);
    const float4 *of = reinterpret_cast<const float4 *>(p.out_f) + (size_t)slot * S2;
    for (uint32_t j = lane; j < S2; j += 32) w[j] = (eb[j + 1] - eb[j]) * of[j].x;
    __syncwarp();
    weights_from_density(w, tr, S2, lane);  // the weights k_composite composites rgb with
    float cw = 0.f, cp = 0.f, inter = 0.f, intra = 0.f;  // carries of W and P from the previous 32 samples
    for (uint32_t base = 0; base < S2; base += 32) {
        const uint32_t j = base + lane;
        const float wj = j < S2 ? w[j] : 0.f;
        const float uj = j < S2 ? (sb[j] + sb[j + 1]) / 2.f : 0.f, dj = j < S2 ? sb[j + 1] - sb[j] : 0.f;
        const float iw = warp_incl_scan_f(wj, lane), ip = warp_incl_scan_f(wj * uj, lane);
        float ew = __shfl_up_sync(0xffffffffu, iw, 1), ep = __shfl_up_sync(0xffffffffu, ip, 1);
        if (lane == 0) ew = ep = 0.f;
        inter += wj * (uj * (cw + ew) - (cp + ep));
        intra += wj * wj * dj;
        cw += __shfl_sync(0xffffffffu, iw, 31); cp += __shfl_sync(0xffffffffu, ip, 31);
    }
    inter = warp_sum_f(inter); intra = warp_sum_f(intra);
    if (lane == 0) p.dist[p.ray_list[slot]] = 2.f * inter + intra / 3.f;
}

// DEPTH: g_j also gets the expected depth's term grad_ed (t_j - D_raw) / (A + 1e-10), 0 where the forward's clip binds (DESIGN §4.10);
// A and D_raw are recomputed from the saved bins and densities exactly as k_composite<true> formed them.
// DIST: g_j also gets the distortion's term grad_dist (2 sum_i w_i |u_j - u_i| + 2/3 w_j delta_j) (DESIGN §4.11), with
// sum_i w_i |u_j - u_i| = u_j W_<j - P_<j + (P - P_<=j) - u_j (W - W_<=j) from two scans.  It is staged in fx[j], which the same lane
// overwrites only after reading it, so the shared memory per block stays 64 (S2 + 2) bytes.
template <bool DET, bool DEPTH = false, bool DIST = false>
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
    float bg0 = p.bg0, bg1 = p.bg1, bg2 = p.bg2;
    if (p.bgmap != nullptr) bg_lookup(p.bgmap, p.bg_H, p.bg_W, p.dirs[3 * (size_t)ray], p.dirs[3 * (size_t)ray + 1], p.dirs[3 * (size_t)ray + 2], bg0, bg1, bg2);
    for (uint32_t j = lane; j < S2; j += 32) tr[j] = (eb[j + 1] - eb[j]) * of[j].x;  // x_j
    __syncwarp();
    smem_scan_add(tr, S2, lane);  // inclusive cumsum of x
    float gd = 0.f, draw = 0.f, den = 1.f;
    if constexpr (DEPTH) {
        float a = 0.f, dt = 0.f;
        for (uint32_t j = lane; j < S2; j += 32) {
            const float excl = j == 0 ? 0.f : tr[j - 1];
            const float x = (eb[j + 1] - eb[j]) * of[j].x;
            const float wj = nan_to_num_f((1.f - expf(-x)) * expf(-excl));
            a += wj;
            dt += wj * ((eb[j] + eb[j + 1]) / 2.f);
        }
        a = warp_sum_f(a); dt = warp_sum_f(dt);
        den = a + 1e-10f;
        draw = dt / den;
        const float lo = depth_unkey(p.dbounds[0]), hi = depth_unkey(p.dbounds[1]);
        gd = (draw >= lo && draw <= hi) ? p.grad_ed[ray] : 0.f;  // torch.clip's backward: inclusive bounds
    }
    if constexpr (DIST) {
        const float *sb = p.sbins_f + (size_t)slot * (S2 + 1);
        const float gdist = p.grad_dist[ray];
        float tw = 0.f, tp = 0.f;  // W, P
        for (uint32_t j = lane; j < S2; j += 32) {
            const float excl = j == 0 ? 0.f : tr[j - 1];
            const float x = (eb[j + 1] - eb[j]) * of[j].x;
            const float wj = nan_to_num_f((1.f - expf(-x)) * expf(-excl));  // the forward's weights
            w[j] = wj;
            tw += wj; tp += wj * ((sb[j] + sb[j + 1]) / 2.f);
        }
        tw = warp_sum_f(tw); tp = warp_sum_f(tp);
        float cw = 0.f, cp = 0.f;  // carries of W and P from the previous 32 samples
        for (uint32_t base = 0; base < S2; base += 32) {
            const uint32_t j = base + lane;
            const float wj = j < S2 ? w[j] : 0.f;
            const float uj = j < S2 ? (sb[j] + sb[j + 1]) / 2.f : 0.f, dj = j < S2 ? sb[j + 1] - sb[j] : 0.f;
            const float iw = warp_incl_scan_f(wj, lane), ip = warp_incl_scan_f(wj * uj, lane);
            float ew = __shfl_up_sync(0xffffffffu, iw, 1), ep = __shfl_up_sync(0xffffffffu, ip, 1);
            if (lane == 0) ew = ep = 0.f;
            const float wl = cw + ew, pl = cp + ep, wle = cw + iw, ple = cp + ip;  // W_<j, P_<j, W_<=j, P_<=j
            if (j < S2) fx[j] = gdist * (2.f * (uj * wl - pl + (tp - ple) - uj * (tw - wle)) + (2.f / 3.f) * wj * dj);
            cw += __shfl_sync(0xffffffffu, iw, 31); cp += __shfl_sync(0xffffffffu, ip, 31);
        }
    }
    float acc = 0.f;  // (background map only)
    for (uint32_t j = lane; j < S2; j += 32) {
        const float excl = j == 0 ? 0.f : tr[j - 1];
        const float x = (eb[j + 1] - eb[j]) * of[j].x;
        const float T = expf(-excl);
        float wj = (1.f - expf(-x)) * T;
        const bool fin = isfinite(wj);  // nan_to_num in the forward: a replaced weight carries no gradient
        wj = fin ? wj : nan_to_num_f(wj);
        const float4 c = of[j];
        float g;
        if constexpr (DEPTH) g = fin ? (gr * (c.y - bg0) + gg * (c.z - bg1) + gb * (c.w - bg2) + ga + gd * (((eb[j] + eb[j + 1]) / 2.f - draw) / den)) : 0.f;
        else g = fin ? (gr * (c.y - bg0) + gg * (c.z - bg1) + gb * (c.w - bg2) + ga) : 0.f;
        if constexpr (DIST) g = fin ? g + fx[j] : 0.f;  // (read before this lane overwrites fx[j] below)
        w[j] = wj;
        gw[j] = g * wj;
        fx[j] = fin ? g * (T - wj) : 0.f;  // first term of dL/dx_j
        acc += wj;
    }
    if (p.bgmap != nullptr) {  // the forward's accumulation: the same weights, summed in k_composite's order
        const float oma = 1.f - warp_sum_f(acc);
        if (lane == 0) { p.bg_s[3 * (size_t)ray] = gr * oma; p.bg_s[3 * (size_t)ray + 1] = gg * oma; p.bg_s[3 * (size_t)ray + 2] = gb * oma; }
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
// (n_rows != nullptr: the tiles of the compact rows of occupancy culling)
__global__ void k_det_reduce_parts(const uint32_t *__restrict__ n_active, uint32_t S, const uint32_t *__restrict__ n_rows, const float *__restrict__ part,
                                   float *__restrict__ gw) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= BWD_PART_STRIDE) return;
    const uint64_t rows = n_rows != nullptr ? (uint64_t)*n_rows : (uint64_t)*n_active * S;
    const uint32_t ntiles = (uint32_t)((rows + BWD_TILE - 1) / BWD_TILE);
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
// (k_mlp_bwd<true> wrote block b = 4 tile + warp's partial for ray `slot` to row 4 (tile + slot) + warp).  rowmap != nullptr: the
// ray's rows are its compact rows, found by binary search of the ascending map (none: a zero gradient)
__global__ void __launch_bounds__(128) k_det_dirbias(const uint32_t *__restrict__ n_active, uint32_t S, const uint32_t *__restrict__ rowmap,
                                                     const uint32_t *__restrict__ n_rows, const float *__restrict__ gdb_part, float *__restrict__ g_dirbias) {
    const uint32_t slot = blockIdx.x, k = threadIdx.x;
    if (slot >= *n_active) return;
    uint64_t r0 = (uint64_t)slot * S, r1 = r0 + S;  // [r0, r1)
    if (rowmap != nullptr) {
        const uint32_t n = *n_rows;
        r0 = lower_bound_u32(rowmap, n, slot * S);
        r1 = lower_bound_u32(rowmap, n, (slot + 1) * S);
    }
    float acc = 0.f;
    if (r1 > r0)
        for (uint64_t b = r0 / 16; b <= (r1 - 1) / 16; ++b) acc += __ldg(gdb_part + (4 * (b / 4 + slot) + (b & 3)) * 128 + k);
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

// ---- occupancy culling (DESIGN §4.12) ---------------------------------------------------------------------------------------------
// live rows of one pass: flag[g] = 1 for every sample row g < n_active * S that is not culled (matched to an occupied tetrahedron, or
// unmatched), 0 for culled rows and rows past the active ones.  outw 1 / 4: a culled row's output (density, or sigma and colour) is
// set to 0 here, since k_mlp skips it; outw 0: flags only (the backward's rebuild of its forward's map).
__global__ void k_live_rows(const uint32_t *__restrict__ n_active, uint32_t S, uint64_t n, const uint4 *__restrict__ vi, uint32_t outw,
                            uint8_t *__restrict__ flag, float *__restrict__ out) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    uint8_t live = 0;
    if (g < (uint64_t)*n_active * S) {
        const uint4 v = __ldg(vi + g);
        live = (v.x == TN_EMPTY && v.w == TN_CULLED) ? 0 : 1;
        if (!live && outw == 1) out[g] = 0.f;
        if (!live && outw == 4) reinterpret_cast<float4 *>(out)[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    flag[g] = live;
}

// compact-row map of one pass: map[c] = the c-th live sample row in row order (so each ray's live rows stay contiguous, in slot order),
// *n_rows = their number; all on the device
static int compact_rows(tn_tracer *h, RenderState *r, const uint32_t *n_active, uint32_t S, size_t R, const uint4 *vi, float *out, uint32_t outw,
                        DevArray<uint32_t> &map, uint32_t *n_rows, cudaStream_t s) {
    const size_t n = R * S;
    TN_TRY(r->live_flag.grow(n)); TN_TRY(map.grow(n));
    k_live_rows<<<(uint32_t)((n + 255) / 256), 256, 0, s>>>(n_active, S, n, vi, outw, r->live_flag.p, out);
    cub::CountingInputIterator<uint32_t> it(0u);
    TN_TRY(cub_run(r->cub_tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceSelect::Flagged(t, bytes, it, r->live_flag.p, map.p, n_rows, (int64_t)n, s);
    }));
    h->launches += 2;
    return TN_OK;
}

// ---- tn_occupancy_update: 11 probes per tetrahedron (4 vertices, 6 edge midpoints, centroid), as barycentric weights of the cell's
// vertices 1..3 (vertex 0 gets 1 - b0 - b1 - b2, as the interpolation forms it); every weight is exact in float
__constant__ float c_probe[11][3] = {{0.f, 0.f, 0.f},    {1.f, 0.f, 0.f},    {0.f, 1.f, 0.f},     {0.f, 0.f, 1.f},
                                     {0.5f, 0.f, 0.f},   {0.f, 0.5f, 0.f},   {0.f, 0.f, 0.5f},    {0.5f, 0.5f, 0.f},
                                     {0.5f, 0.f, 0.5f},  {0.f, 0.5f, 0.5f},  {0.25f, 0.25f, 0.25f}};
constexpr uint32_t OCC_PROBES = 11;
constexpr uint32_t OCC_CHUNK = 1u << 19;  // tetrahedra per k_mlp launch (5.8 M probe rows, 176 MB of rows and densities)

// probe rows of tetrahedra t0 .. t0 + nt - 1 (vi = the cell, one row per probe); count[0] = nt (k_mlp's "rays" of S = 11), count[1] = 0
// (its tile counter)
__global__ void k_occ_rows(uint32_t t0, uint32_t nt, const uint32_t *__restrict__ cells, uint4 *__restrict__ vi, float *__restrict__ bary,
                           uint32_t *__restrict__ count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) { count[0] = nt; count[1] = 0; }
    if (i >= nt * OCC_PROBES) return;
    const uint32_t t = t0 + i / OCC_PROBES, k = i % OCC_PROBES;
    vi[i] = __ldg(reinterpret_cast<const uint4 *>(cells) + t);
    bary[3 * (size_t)i] = c_probe[k][0]; bary[3 * (size_t)i + 1] = c_probe[k][1]; bary[3 * (size_t)i + 2] = c_probe[k][2];
}
// one thread per tetrahedron, no atomics: occ = max(decay occ, max of the probe densities); decay 0 replaces it
__global__ void k_occ_reduce(uint32_t t0, uint32_t nt, const float *__restrict__ sig, float decay, float *__restrict__ occ) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nt) return;
    float m = sig[(size_t)i * OCC_PROBES];
#pragma unroll
    for (uint32_t k = 1; k < OCC_PROBES; ++k) m = fmaxf(m, sig[(size_t)i * OCC_PROBES + k]);
    occ[t0 + i] = decay == 0.f ? m : fmaxf(decay * occ[t0 + i], m);
}

// trace and coarse pass (the fine pass writes into a saved-state layout)
static int ensure_ws(RenderState *r, size_t R, size_t M, size_t Sc) {
    TN_TRY(r->num.grow(R)); TN_TRY(r->cells.grow(R * M)); TN_TRY(r->verts.grow(4 * R * M)); TN_TRY(r->bary.grow(6 * R * M));
    TN_TRY(r->dist.grow(2 * R * M));
    TN_TRY(r->ebins_c.grow(R * (Sc + 1))); TN_TRY(r->sbins_c.grow(R * (Sc + 1))); TN_TRY(r->bary_c.grow(3 * R * Sc));
    TN_TRY(r->dens_c.grow(R * Sc)); TN_TRY(r->vi_c.grow(R * Sc));
    return TN_OK;
}

// training forward: the gradient scratch of every backward
static int ensure_train_ws(RenderState *r, size_t R, size_t S2, uint32_t V) {
    TN_TRY(r->dout.grow(R * S2)); TN_TRY(r->g_dirbias.grow(128 * R));
    TN_TRY(r->gw.grow(GW_TOTAL + 1));
    TN_TRY(r->gshadow.grow(64 * (size_t)V));
    return TN_OK;
}

// deterministic mode, forward: slot of every ray = number of rays with hits before it (exclusive scan)
static int ordered_slots(RenderState *r, uint32_t R, cudaStream_t s) {
    TN_TRY(r->ray_flag.grow(R)); TN_TRY(r->ray_slot.grow(R));
    k_ray_flags<<<(R + 255) / 256, 256, 0, s>>>(R, r->num.p, r->ray_flag.p);
    TN_TRY(cub_run(r->cub_tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceScan::ExclusiveSum(t, bytes, r->ray_flag.p, r->ray_slot.p, (int)R, s);
    }));
    return TN_OK;
}

// deterministic mode, backward workspace for R rays of S2 fine samples
static int ensure_det_ws(RenderState *r, size_t R, size_t S2) {
    const size_t rows = R * S2, ntiles = (rows + BWD_TILE - 1) / BWD_TILE;
    TN_TRY(r->det_part.grow((size_t)BWD_PARTS * BWD_PART_STRIDE));
    TN_TRY(r->det_gdb.grow(4 * (ntiles + R) * 128));
    TN_TRY(r->det_dx.grow(64 * rows));
    TN_TRY(r->det_sums.grow(R));
    TN_TRY(r->det_dbg.grow((size_t)DBG_PART * ((R + DBG_SLOTS - 1) / DBG_SLOTS)));
    TN_TRY(r->det_keys.grow(2 * 4 * rows));
    TN_TRY(r->det_vals.grow(2 * 4 * rows));
    return TN_OK;
}

}  // namespace tn

using namespace tn;

extern "C" int tn_render_set_field(tn_tracer *h, const float *d_field, uint32_t C, uint32_t V, void *stream) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (C != 64) return fail(TN_ERR_ARG, "tn_render: field_dim must be 64 (model.py:81)");
    DeviceGuard g(h->device);
    RenderState *r = state(h);
    TN_TRY(r->fshadow.grow(64 * (size_t)V));
    r->V = V;
    k_transpose64<<<(V + 31) / 32, dim3(32, 8), 0, (cudaStream_t)stream>>>(d_field, r->fshadow.p, V);
    h->launches += 1;
    r->gen = next_generation();
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
    TN_TRY(r->wimg.grow(32768 + 3 * 65536)); TN_TRY(r->wimg16.grow(32768 + 3 * 65536));
    TN_TRY(r->bias.grow(384)); TN_TRY(r->head.grow(520)); TN_TRY(r->w4dir.grow(128 * 27 + 128));
    TN_TRY(r->wimg_bwd.grow(BWD_WIMG_BYTES));
    launch_pack_weights(P[0], 64, 0, 64, r->wimg.p, s);                     // mlp_base.layers.0.weight [128,64]
    launch_pack_weights(P[2], 128, 0, 128, r->wimg.p + 32768, s);           // mlp_base.layers.1.weight [128,128]
    launch_pack_weights(P[4], 128, 0, 128, r->wimg.p + 32768 + 65536, s);   // mlp_base.layers.2.weight
    launch_pack_weights(P[6], 155, 27, 128, r->wimg.p + 32768 + 131072, s); // mlp_head.layers.0.weight [128,155], base part
    launch_pack_weights(P[0], 64, 0, 64, r->wimg16.p, s, 32768u, 16384u, 1);
    launch_pack_weights(P[2], 128, 0, 128, r->wimg16.p + 32768, s, 32768u, 16384u, 1);
    launch_pack_weights(P[4], 128, 0, 128, r->wimg16.p + 32768 + 65536, s, 32768u, 16384u, 1);
    launch_pack_weights(P[6], 155, 27, 128, r->wimg16.p + 32768 + 131072, s, 32768u, 16384u, 1);
    k_pack_small<<<1, 128, 0, s>>>(P[1], P[3], P[5], P[6], P[7], P[8], P[9], P[10], P[11], r->bias.p, r->head.p, r->w4dir.p);
    // backward image (tn_mlp_bwd.cuh): stage 0 = [W1 hi | W1 lo]; then per 128-wide layer [hi kb0 | hi kb1][lo kb0 | lo kb1]
    launch_pack_weights(P[0], 64, 0, 64, r->wimg_bwd.p, s, 16384u, 16384u);
    launch_pack_weights(P[2], 128, 0, 128, r->wimg_bwd.p + 1 * BWD_STAGE, s, 16384u, 32768u);
    launch_pack_weights(P[4], 128, 0, 128, r->wimg_bwd.p + 3 * BWD_STAGE, s, 16384u, 32768u);
    launch_pack_weights(P[6], 155, 27, 128, r->wimg_bwd.p + 5 * BWD_STAGE, s, 16384u, 32768u);
    h->launches += 13;
    r->gen = next_generation();
    TN_CUDA(cudaGetLastError());
    r->have_weights = true;
    return TN_OK;
}

// saved-state blob: the SavedHeader, then the TrainBufs arrays, each 256-byte aligned
constexpr size_t SAVED_ALIGN = 256;
static_assert(sizeof(SavedHeader) <= SAVED_ALIGN, "saved-state header exceeds its slot");
// bytes of the blob for R rays of S2 fine samples; with base != nullptr also the array pointers inside it.  eval: no spacing bins or
// encodings (nullptr, 0 bytes), which only the backward reads -- the layout of the eval render in the tracer's own blob.  dirs: a
// training forward over a background map also keeps its ray directions, last (12 bytes per ray; the other arrays stay where they are)
static size_t saved_layout(size_t R, size_t S2, uint8_t *base, TrainBufs *b, bool eval = false, bool dirs = false) {
    size_t off = SAVED_ALIGN;  // header
    auto take = [&](size_t bytes) { uint8_t *p = base ? base + off : nullptr; off += (bytes + SAVED_ALIGN - 1) / SAVED_ALIGN * SAVED_ALIGN; return p; };
    TrainBufs t{};
    t.n_active = (uint32_t *)take(32);  // (one 256-byte slot either way)
    t.ray_list = (uint32_t *)take(4 * R);
    t.ebins_f = (float *)take(4 * R * (S2 + 1));
    if (!eval) t.sbins_f = (float *)take(4 * R * (S2 + 1));
    t.vi_f = (uint4 *)take(16 * R * S2);
    t.bary_f = (float *)take(12 * R * S2);
    t.out_f = (float *)take(16 * R * S2);
    t.dirbias = (float *)take(512 * R);
    if (!eval) t.enc = (float *)take(4 * 27 * R);
    if (dirs) t.dirs = (float *)take(12 * R);
    if (b) *b = t;
    return off;
}

// training-mode inputs of the forward (nullptr = eval); saved == nullptr: the tracer's own blob
struct TrainFwd {
    const float *jit_c, *jit_f;
    void *saved;
};

static int render_impl(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                       float *d_rgb, float *d_acc, float *d_depth, uint8_t *d_mask, const TrainFwd *tf, float *d_normals, float *d_edepth,
                       void *stream) {
    if (!h || !cfg) return fail(TN_ERR_ARG, "null argument");
    RenderState *r = h->render;
    if (r && r->gather_world && d_edepth != nullptr)
        return fail(TN_ERR_ARG, "tn_render: the fused pixel gather (tn_render_set_gather) carries no expected depth; switch it off first");
    if (r && r->gather_world && d_normals != nullptr)
        return fail(TN_ERR_ARG, "tn_render: the fused pixel gather (tn_render_set_gather) carries no normals; switch it off first");
    if (!r || !r->fshadow.p || !r->have_weights) return fail(TN_ERR_STATE, "tn_render: call tn_render_set_field and tn_render_set_weights first");
    if (!h->mesh.nodes.p) return fail(TN_ERR_STATE, "tn_render: no tetrahedra loaded");
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
    const bool cull = r->occ != nullptr;               // occupancy culling (DESIGN §4.12)
    if (cull && r->occ_T != h->mesh.T)
        return fail(TN_ERR_STATE, "tn_render: the occupancy was set for a mesh with another number of tetrahedra (tn_render_set_occupancy)");
    const uint32_t S2 = single ? Sc : Sc + Sf + 1;     // PDFSampler include_original (model.py:463)
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    // dynamic shared memory of the per-ray kernels (4 warps per block, one ray per warp): checked before anything is allocated or
    // launched, so a setting that cannot run fails as an argument error and leaves no CUDA error behind
    const bool place = cull && r->occ_place;           // occupancy sampling (DESIGN §4.13)
    const size_t smem_sc = SAMPLE_WARPS * sizeof(float) * (place ? place_floats(M, Sc) : coarse_floats(M, Sc, cfg->use_biased_sampler));
    const size_t smem_sf = SAMPLE_WARPS * sizeof(float) * fine_floats(M, std::max(Sc, S2));
    const size_t smem_c = SAMPLE_WARPS * sizeof(float) * 2 * ((size_t)S2 + 2);
    const size_t smem_cb = SAMPLE_WARPS * sizeof(float) * 4 * ((size_t)S2 + 2);  // k_composite_bwd, which the backward launches
    if (!r->smem_optin) TN_CUDA(cudaDeviceGetAttribute(&r->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
    {
        size_t need = std::max(smem_sc, smem_c);
        const char *kern = smem_sc >= smem_c ? "k_sample_coarse" : "k_composite";
        if (!single && smem_sf > need) { need = smem_sf; kern = "k_sample_fine"; }
        if (tf != nullptr && smem_cb > need) { need = smem_cb; kern = "k_composite_bwd"; }
        if (need > (size_t)r->smem_optin)
            return fail(TN_ERR_ARG, "tn_render: num_samples + num_fine_samples = " + std::to_string(Sc + Sf) + " at max_ray_triangles = " +
                                        std::to_string(M) + " needs " + std::to_string(need) + " bytes of shared memory per block in " + kern +
                                        ", above the device's shared-memory limit of " + std::to_string(r->smem_optin) +
                                        " bytes (fewer samples or a smaller max_ray_triangles)");
    }
    TN_TRY(ensure_ws(r, R, M, Sc));
    const bool own = tf == nullptr || tf->saved == nullptr;  // the fine pass writes into the tracer's own blob
    const bool keep_dirs = tf != nullptr && r->bgmap != nullptr;  // the backward looks the background up again
    if (own) TN_TRY(r->own.grow(saved_layout(R, S2, nullptr, nullptr, tf == nullptr, keep_dirs)));
    if (d_normals != nullptr) TN_TRY(r->grad_n.grow((size_t)R * S2));
    if (tf != nullptr) TN_TRY(ensure_train_ws(r, R, S2, r->V));
    r->last = SavedHeader{};
    TrainBufs b{};
    saved_layout(R, S2, own ? r->own.p : (uint8_t *)tf->saved, &b, tf == nullptr, keep_dirs);
    if (own) r->own_b = b;
    const int prec = tf != nullptr ? 3 : r->mlp_prec;  // the training forward keeps bf16x3 (its backward recomputes in bf16x3)
    TN_CUDA(cudaMemsetAsync(b.n_active, 0, 16, s));
    if (d_edepth != nullptr) {  // clip bounds: min starts at the largest key, max at the smallest
        TN_CUDA(cudaMemsetAsync(b.n_active + 4, 0xff, 4, s));
        TN_CUDA(cudaMemsetAsync(b.n_active + 5, 0, 4, s));
    }
#define TN_EV(i) do { if (r->profile) cudaEventRecord(r->ev[i], s); } while (0)
    TN_EV(0);  // the "trace" interval includes the L2 warm-up it exists for
    {   // L2 warm-up of everything read-only that the step gathers from (mesh tables, field shadow, weight image)
        const void *extra[2] = {r->fshadow.p, prec == 2 ? r->wimg16.p : r->wimg.p};
        const size_t extra_b[2] = {sizeof(float) * 64 * (size_t)r->V, 32768 + 3 * 65536};
        const int rc = launch_prefetch(h, extra, extra_b, 2, s);
        if (rc) return rc;
    }
    int rc = launch_trace_internal(h, d_origins, d_directions, R, M, r->num.p, r->cells.p, r->bary.p, r->dist.p, r->verts.p, 0, s);
    if (rc) return rc;
    TN_EV(1);
    SampleParams p{};
    p.R = R; p.M = M; p.Sc = Sc; p.Sf = Sf; p.S2 = S2; p.biased = cfg->use_biased_sampler;
    p.num = r->num.p; p.dist = (const float2 *)r->dist.p; p.verts = (const uint4 *)r->verts.p; p.bary = r->bary.p;
    p.o = d_origins; p.d = d_directions; p.n_active = b.n_active; p.ray_list = b.ray_list;
    p.ebins_c = r->ebins_c.p; p.sbins_c = r->sbins_c.p; p.bary_c = r->bary_c.p; p.vi_c = r->vi_c.p; p.dens_c = r->dens_c.p;
    p.ebins_f = b.ebins_f; p.bary_f = b.bary_f; p.vi_f = b.vi_f; p.dirbias = b.dirbias; p.w4dir = r->w4dir.p; p.out_f = b.out_f;
    p.rgb = d_rgb; p.acc = d_acc; p.depth = d_depth; p.mask = d_mask;
    p.far_plane = cfg->far_plane; p.bg0 = cfg->background[0]; p.bg1 = cfg->background[1]; p.bg2 = cfg->background[2];
    if (tf != nullptr) { p.train = 1; p.jit_c = tf->jit_c; p.jit_f = tf->jit_f; p.sbins_f = b.sbins_f; p.enc = b.enc; }
    p.edepth = d_edepth; p.dbounds = b.n_active + 4;
    if (cull) { p.cells = r->cells.p; p.occ = r->occ; p.occ_thr = r->occ_thr; }
    if (r->bgmap != nullptr) { p.bgmap = r->bgmap; p.bg_H = r->bg_H; p.bg_W = r->bg_W; }
    if (keep_dirs) TN_CUDA(cudaMemcpyAsync(b.dirs, d_directions, 12 * (size_t)R, cudaMemcpyDeviceToDevice, s));
    if (r->gather_world) {
        if (R > r->gather_stride) return fail(TN_ERR_ARG, "tn_render: more rays than the gathered-pixel buffers were sized for (tn_render_set_gather)");
        for (int k = 0; k < 8; ++k) p.peer[k] = r->peer[k];
        p.gather_world = r->gather_world; p.gather_rank = r->gather_rank; p.gather_stride = r->gather_stride;
    }
    auto k_coarse_sample = place ? (det ? k_sample_coarse<true, true> : k_sample_coarse<false, true>) : (det ? k_sample_coarse<true> : k_sample_coarse<false>);
    TN_CUDA(cudaFuncSetAttribute(k_coarse_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sc));
    // (single pass: k_sample_fine is not launched, and its staging at S2 = Sc can exceed the limit where the call itself fits)
    if (!single) TN_CUDA(cudaFuncSetAttribute(k_sample_fine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sf));
    auto k_comp = d_edepth != nullptr ? k_composite<true> : k_composite<false>;
    TN_CUDA(cudaFuncSetAttribute(k_comp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
    auto launch_coarse = cull ? (prec == 2 ? launch_mlp<false, 2, true> : launch_mlp<false, 3, true>) : (prec == 2 ? launch_mlp<false, 2> : launch_mlp<false, 3>);
    auto launch_fine = cull ? (prec == 2 ? launch_mlp<true, 2, true> : launch_mlp<true, 3, true>) : (prec == 2 ? launch_mlp<true, 2> : launch_mlp<true, 3>);
    const uint32_t gridR = (R + SAMPLE_WARPS - 1) / SAMPLE_WARPS;

    if (det) {
        rc = ordered_slots(r, R, s);
        if (rc) return rc;
        p.ray_slot = r->ray_slot.p;
        h->launches += 2;
    }
    k_coarse_sample<<<gridR, SAMPLE_WARPS * 32, smem_sc, s>>>(p);
    TN_EV(2);
    MlpParams mc{};
    mc.n_active = b.n_active; mc.S = Sc; mc.vi = r->vi_c.p; mc.bary = r->bary_c.p; mc.fshadow = r->fshadow.p; mc.wimg = prec == 2 ? r->wimg16.p : r->wimg.p;
    mc.bias = r->bias.p; mc.head = r->head.p; mc.dirbias = nullptr; mc.out = r->dens_c.p;
    mc.tile_ctr = b.n_active + 1;  // words 1, 2 of the zeroed 16-byte block: tile counters of the coarse / fine pass
    // one CTA per SM at most (the weight image fills its shared memory), MLP_WGS tiles of MLP_TILE samples in flight per CTA
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    const uint64_t tiles_c = ((uint64_t)R * Sc + MLP_TILE - 1) / MLP_TILE, tiles_f = ((uint64_t)R * S2 + MLP_TILE - 1) / MLP_TILE;
    const uint32_t grid_c = (uint32_t)std::min<uint64_t>((tiles_c + MLP_WGS - 1) / MLP_WGS, (uint64_t)sms);
    const uint32_t grid_f = (uint32_t)std::min<uint64_t>((tiles_f + MLP_WGS - 1) / MLP_WGS, (uint64_t)sms);
    if (!single) {
        if (cull) {  // the coarse pass's MLP runs on its live rows only; culled rows get density 0
            TN_TRY(compact_rows(h, r, b.n_active, Sc, R, r->vi_c.p, r->dens_c.p, 1, r->rowmap_c, b.n_active + 6, s));
            mc.rowmap = r->rowmap_c.p; mc.n_rows = b.n_active + 6;
        }
        rc = launch_coarse(mc, grid_c, s);
        if (rc) return rc;
    }
    TN_EV(3);
    if (!single) k_sample_fine<<<gridR, SAMPLE_WARPS * 32, smem_sf, s>>>(p);
    else k_dirbias_only<<<gridR, SAMPLE_WARPS * 32, 0, s>>>(p);
    TN_EV(4);
    MlpParams mf = mc;
    mf.S = S2; mf.dirbias = b.dirbias; mf.out = b.out_f;
    if (!single) { mf.vi = b.vi_f; mf.bary = b.bary_f; }
    else p.ebins_f = r->ebins_c.p;  // k_composite integrates over the coarse bins
    mf.tile_ctr = b.n_active + 2;
    if (cull) {  // the same for the pass that gives the colours: culled rows get (sigma, r, g, b) = 0
        TN_TRY(compact_rows(h, r, b.n_active, S2, R, mf.vi, b.out_f, 4, r->rowmap_f, b.n_active + 7, s));
        mf.rowmap = r->rowmap_f.p; mf.n_rows = b.n_active + 7;
    }
    rc = launch_fine(mf, grid_f, s);
    if (rc) return rc;
    TN_EV(5);
    k_comp<<<gridR, SAMPLE_WARPS * 32, smem_c, s>>>(p);
    TN_EV(6);
#undef TN_EV
    h->launches += 5;
    TN_CUDA(cudaGetLastError());
    if (d_edepth != nullptr) {  // after the six timed intervals, as the normals
        k_expected_depth_finalize<<<(R + 255) / 256, 256, 0, s>>>(R, r->num.p, p.dbounds, cfg->far_plane, d_edepth);
        h->launches += 1;
        TN_CUDA(cudaGetLastError());
    }
    if (d_normals != nullptr) {  // after the six timed intervals: the density gradient at the samples that give the colours, composited
        NormalsLaunch nl{};
        nl.n_active = b.n_active; nl.ray_list = b.ray_list; nl.tile_ctr = b.n_active + 3;  // word 3 of the zeroed block
        nl.S = S2; nl.R = R; nl.prec = (uint32_t)prec; nl.vi = mf.vi; nl.bary = mf.bary; nl.ebins = p.ebins_f; nl.out_f = b.out_f;
        nl.fshadow = r->fshadow.p; nl.wimg = mf.wimg; nl.bias = r->bias.p; nl.head = r->head.p; nl.xyz = h->mesh.xyz; nl.grad = r->grad_n.p;
        nl.normals = d_normals;
        rc = launch_normals(nl, sms, s);
        if (rc) return rc;
        h->launches += 2;
    }
    if (tf != nullptr) {  // what the backward continues with: kept on the host for the tracer's own blob, in the caller's blob otherwise
        SavedHeader hd{SAVED_MAGIC, R, M, Sc, Sf, S2, det ? 1u : 0u, d_edepth != nullptr ? 1u : 0u,
                       {cfg->background[0], cfg->background[1], cfg->background[2]}, 0, r->gen, h->mesh_gen, cull ? 1u : 0u, 0, 0, 0};
        if (keep_dirs) { hd.bgmap = 1; hd.bg_H = r->bg_H; hd.bg_W = r->bg_W; hd.bg_gen = r->bg_gen; }
        if (own) {
            r->last = hd;
        } else {
            // pageable source: staged before the call returns, so `hd` may go out of scope
            TN_CUDA(cudaMemcpyAsync(tf->saved, &hd, sizeof(hd), cudaMemcpyHostToDevice, s));
            if (cull)  // the live-row counts, from words 6, 7 of the forward's n_active slot
                TN_CUDA(cudaMemcpyAsync((uint8_t *)tf->saved + offsetof(SavedHeader, live_c), b.n_active + 6, 8, cudaMemcpyDeviceToDevice, s));
        }
    }
    return TN_OK;
}

// optional outputs: the expected depth d_expected_depth f32[R] (DESIGN.md §4.10) and the normal map d_normals f32[R,3] (§4.7;
// tn_normals.cu)
extern "C" int tn_render(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                         float *d_rgb, float *d_acc, float *d_depth, uint8_t *d_mask, float *d_expected_depth, float *d_normals, void *stream) {
    return render_impl(h, cfg, d_origins, d_directions, R, d_rgb, d_acc, d_depth, d_mask, nullptr, d_normals, d_expected_depth, stream);
}

// ---- fused training step (SURVEY §8f-1; model.py:520-662 in training mode + autograd) ------------------------------------------------
// forward: the fused pipeline with stratified bins (d_jitter_coarse f32[R,Sc+1], d_jitter_fine f32[R,Sf+1], uniform [0,1), indexed by
// ray; nullptr = eval bins) and the training-mode RGB renderer (no nan_to_num, no clamp).  Keeps what the backward needs.
extern "C" int tn_render_train_forward(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                                       const float *d_jitter_coarse, const float *d_jitter_fine, float *d_rgb, float *d_acc, float *d_depth,
                                       uint8_t *d_mask, void *stream) {
    TrainFwd tf{d_jitter_coarse, d_jitter_fine, nullptr};
    return render_impl(h, cfg, d_origins, d_directions, R, d_rgb, d_acc, d_depth, d_mask, &tf, nullptr, nullptr, stream);
}

// backward of the training forward whose buffers are `b` and whose header is `hd` (R rays x S2 fine samples, continued in the forward's
// mode and with its background): d_grad_rgb f32[R,3] (dL/d rgb), d_grad_acc f32[R] or NULL (dL/d accumulation) -> d_grad_field
// f32[64,V] and the twelve MLP parameter gradients (same order / layouts as tn_render_set_weights); every output element is written.
// Reads `b` and the field / weights; writes only the tracer's gradient scratch.  The coarse pass carries no gradient (PDFSampler
// detaches its bins).  No [samples,128] tensor touches HBM.
// d_grad_ed != nullptr: dL/d expected depth f32[R] of a forward that produced it (its clip bounds in b.n_active[4, 5]).
// d_grad_dist != nullptr: dL/d distortion f32[R] (k_distortion).
// Any of d_grad_o / d_grad_d / d_grad_xyz != nullptr: also the gradients at the ray origins / directions (tn_ray_grads.cu) and at the
// mesh vertex positions (tn_vertex_grads.cu), into the non-null ones.
// hd.cull: the forward culled by occupancy; its map of live fine rows is rebuilt from the culled marks in b.vi_f (never from the
// occupancy, which may have changed since)
// hd.bgmap: the forward composited over the background map, which has the same generation (the caller checked): g_j takes bg(d) of
// the saved directions, and the map gradient (d_grad_bg f32[H,W,3], or NULL) and the directions' background term follow (DESIGN §4.16)
static int train_backward_impl(tn_tracer *h, const TrainBufs &b, const SavedHeader &hd, const float *d_grad_rgb, const float *d_grad_acc,
                               const float *d_grad_ed, const float *d_grad_dist, int use_gradient_scaling, float *d_grad_field,
                               float *const *d_grad_params12, float *d_grad_o, float *d_grad_d, float *d_grad_xyz, float *d_grad_bg,
                               cudaStream_t s) {
    RenderState *r = h->render;
    if (hd.bgmap && r->bg_gen != hd.bg_gen)
        return fail(TN_ERR_STATE, "tn_render_train_backward: the background map changed (tn_render_set_background) since the forward");
    if (d_grad_bg != nullptr && !hd.bgmap)
        return fail(TN_ERR_STATE, "tn_render_train_backward_saved3: the forward composited over no background map (tn_render_set_background)");
    const uint32_t R = hd.R, S2 = hd.S2;
    const bool det = hd.det != 0, cull = hd.cull != 0;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    const uint32_t V = r->V;
    if (det) TN_TRY(ensure_det_ws(r, R, S2));
    const bool rays = d_grad_o != nullptr || d_grad_d != nullptr || d_grad_xyz != nullptr;
    const size_t rows = (size_t)R * S2;
    if (rays) {
        if (!det) TN_TRY(r->ray_dx.grow(64 * rows));
        TN_TRY(r->ray_gx.grow(rows));
    }
    TN_CUDA(cudaMemsetAsync(r->gw.p, 0, sizeof(float) * (GW_TOTAL + 1), s));  // the accumulators and the tile counter after them
    if (!det) {  // (deterministic mode writes every element of these)
        TN_CUDA(cudaMemsetAsync(r->gshadow.p, 0, sizeof(float) * 64 * (size_t)V, s));
        TN_CUDA(cudaMemsetAsync(r->g_dirbias.p, 0, 512 * (size_t)R, s));
    }
    CompositeBwdParams cb{};
    cb.S2 = S2; cb.use_gradient_scaling = use_gradient_scaling ? 1u : 0u; cb.n_active = b.n_active; cb.ray_list = b.ray_list;
    cb.ebins_f = b.ebins_f; cb.sbins_f = b.sbins_f; cb.out_f = b.out_f; cb.grad_rgb = d_grad_rgb; cb.grad_acc = d_grad_acc;
    cb.bg0 = hd.bg[0]; cb.bg1 = hd.bg[1]; cb.bg2 = hd.bg[2]; cb.dout = r->dout.p; cb.sums = det ? (float *)r->det_sums.p : r->gw.p + GW_SUMS;
    cb.grad_ed = d_grad_ed; cb.dbounds = b.n_active + 4; cb.grad_dist = d_grad_dist;
    const bool bg_grads = hd.bgmap && (d_grad_bg != nullptr || d_grad_d != nullptr);
    if (hd.bgmap) {
        TN_TRY(r->bg_s.grow(3 * (size_t)R));
        cb.bgmap = r->bgmap; cb.bg_H = hd.bg_H; cb.bg_W = hd.bg_W; cb.dirs = b.dirs; cb.bg_s = r->bg_s.p;
        // s = grad_rgb on the empty rays; k_composite_bwd writes grad_rgb (1 - accumulation) over the active ones
        if (bg_grads) TN_CUDA(cudaMemcpyAsync(r->bg_s.p, d_grad_rgb, 12 * (size_t)R, cudaMemcpyDeviceToDevice, s));
    }
    const size_t smem_cb = SAMPLE_WARPS * sizeof(float) * 4 * ((size_t)S2 + 2);
    auto k_cbwd = d_grad_dist != nullptr
                      ? (d_grad_ed != nullptr ? (det ? k_composite_bwd<true, true, true> : k_composite_bwd<false, true, true>)
                                              : (det ? k_composite_bwd<true, false, true> : k_composite_bwd<false, false, true>))
                      : (d_grad_ed != nullptr ? (det ? k_composite_bwd<true, true> : k_composite_bwd<false, true>)
                                              : (det ? k_composite_bwd<true> : k_composite_bwd<false>));
    TN_CUDA(cudaFuncSetAttribute(k_cbwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cb));
    const uint32_t gridR = (R + SAMPLE_WARPS - 1) / SAMPLE_WARPS;
    if (r->profile) cudaEventRecord(r->evb[0], s);
    k_cbwd<<<gridR, SAMPLE_WARPS * 32, smem_cb, s>>>(cb);
    if (r->profile) cudaEventRecord(r->evb[1], s);
    MlpBwdParams bp{};
    bp.n_active = b.n_active; bp.S = S2; bp.vi = b.vi_f; bp.bary = b.bary_f; bp.fshadow = r->fshadow.p; bp.wimg = r->wimg_bwd.p;
    bp.bias = r->bias.p; bp.head = r->head.p; bp.dirbias = b.dirbias; bp.dout = r->dout.p; bp.gshadow = r->gshadow.p;
    bp.gw = r->gw.p; bp.g_dirbias = r->g_dirbias.p;
    bp.tile_ctr = reinterpret_cast<uint32_t *>(r->gw.p + GW_TOTAL);  // (default mode only: the deterministic kernel has no tile counter)
    if (cull) {
        TN_TRY(r->rows_b.grow(1));
        TN_TRY(compact_rows(h, r, b.n_active, S2, R, b.vi_f, nullptr, 0, r->rowmap_b, r->rows_b.p, s));
        bp.rowmap = r->rowmap_b.p; bp.n_rows = r->rows_b.p;
    }
    const uint64_t tiles = ((uint64_t)R * S2 + BWD_TILE - 1) / BWD_TILE;
    if (!det) {
        const uint32_t grid = r->bwd_grid ? r->bwd_grid : (uint32_t)std::min<uint64_t>(tiles, (uint64_t)sms);
        if (!rays) {
            auto k = cull ? k_mlp_bwd<false, false, true> : k_mlp_bwd<false>;
            TN_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM_BYTES));
            k<<<grid, BWD_THREADS, BWD_SMEM_BYTES, s>>>(bp);
        } else {  // the same backward, storing the dX rows for k_ray_grads as well
            MlpBwdDxParams xp{};
            static_cast<MlpBwdParams &>(xp) = bp;
            xp.dx = r->ray_dx.p;
            auto k = cull ? k_mlp_bwd<false, true, true> : k_mlp_bwd<false, true>;
            TN_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM_BYTES));
            k<<<grid, BWD_THREADS, BWD_SMEM_BYTES, s>>>(xp);
        }
        if (r->profile) cudaEventRecord(r->evb[2], s);
        k_dirbias_grads<false><<<(R + DBG_SLOTS - 1) / DBG_SLOTS, 256, 0, s>>>(b.n_active, r->g_dirbias.p, b.enc, r->gw.p, nullptr);
    } else {
        // the same stages with every reduction in a fixed order (header of tn_mlp_bwd.cuh); the grid only decides which CTA runs
        // which partition, never what is summed in which order
        MlpBwdDetParams dp{};
        static_cast<MlpBwdParams &>(dp) = bp;
        dp.part = r->det_part.p; dp.gdb_part = r->det_gdb.p; dp.dx = r->det_dx.p;
        auto kd = cull ? k_mlp_bwd<true, true, true> : k_mlp_bwd<true>;
        TN_CUDA(cudaFuncSetAttribute(kd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_DET_SMEM_BYTES));
        const uint32_t grid = r->bwd_grid ? r->bwd_grid : std::min<uint32_t>(BWD_PARTS, (uint32_t)sms);
        kd<<<grid, BWD_THREADS, BWD_DET_SMEM_BYTES, s>>>(dp);
        if (r->profile) cudaEventRecord(r->evb[2], s);
        k_det_reduce_parts<<<(BWD_PART_STRIDE + 255) / 256, 256, 0, s>>>(b.n_active, S2, bp.n_rows, r->det_part.p, r->gw.p);
        k_det_sum_slots<<<1, 256, 0, s>>>(b.n_active, r->det_sums.p, r->gw.p + GW_SUMS);
        k_det_dirbias<<<R, 128, 0, s>>>(b.n_active, S2, bp.rowmap, bp.n_rows, r->det_gdb.p, r->g_dirbias.p);
        k_dirbias_grads<true><<<(R + DBG_SLOTS - 1) / DBG_SLOTS, 256, 0, s>>>(b.n_active, r->g_dirbias.p, b.enc, r->gw.p, r->det_dbg.p);
        k_det_reduce_dbg<<<(DBG_PART + 255) / 256, 256, 0, s>>>(b.n_active, r->det_dbg.p, r->gw.p);
        // field gradient: stable sort of (vertex, row * 4 + k) by vertex, then per-vertex sums in row order
        const uint32_t n = (uint32_t)(4 * (uint64_t)R * S2);
        const int end_bit = radix_end_bit(V);  // keys are <= V
        uint32_t *k0 = r->det_keys.p, *k1 = r->det_keys.p + n, *v0 = r->det_vals.p, *v1 = r->det_vals.p + n;
        k_det_field_keys<<<(n + 255) / 256, 256, 0, s>>>(b.n_active, S2, n, V, b.vi_f, k0, v0);
        TN_TRY(cub_run(r->cub_tmp, [&](void *t, size_t &bytes) {
            return cub::DeviceRadixSort::SortPairs(t, bytes, k0, k1, v0, v1, (int)n, 0, end_bit, s);
        }));
        k_det_field_grad<<<(uint32_t)(((uint64_t)V * 32 + 255) / 256), 256, 0, s>>>(V, n, k1, v1, b.bary_f, r->det_dx.p, r->gshadow.p);
        h->launches += 9;
    }
    const uint32_t *sorted_keys = nullptr, *sorted_vals = nullptr;  // deterministic mode: the field gradient's sorted pairs
    const uint32_t npairs = (uint32_t)(4 * (uint64_t)R * S2);
    if (det) { sorted_keys = r->det_keys.p + npairs; sorted_vals = r->det_vals.p + npairs; }
    GradOut go{};
    for (int i = 0; i < 12; ++i) {
        if (!d_grad_params12[i]) return fail(TN_ERR_ARG, "tn_render_train_backward: null parameter gradient pointer");
        go.p[i] = d_grad_params12[i];
    }
    if (rays) {  // after the direction-bias gradient is complete
        RayGradsLaunch rl{};
        rl.n_active = b.n_active; rl.ray_list = b.ray_list; rl.S = S2; rl.R = R; rl.ebins = b.ebins_f; rl.vi = b.vi_f;
        rl.dx = det ? r->det_dx.p : r->ray_dx.p; rl.fshadow = r->fshadow.p; rl.xyz = h->mesh.xyz; rl.enc = b.enc; rl.g_dirbias = r->g_dirbias.p;
        rl.w4dir = r->w4dir.p; rl.gx = r->ray_gx.p; rl.grad_o = d_grad_o; rl.grad_d = d_grad_d;
        int rc = launch_ray_grads(rl, s);
        if (rc) return rc;
        h->launches += 1;
        if (d_grad_xyz != nullptr) {  // after the per-sample dL/dx is complete
            VertexGradsLaunch vl{};
            vl.n_active = b.n_active; vl.S = S2; vl.R = R; vl.V = h->mesh.V; vl.vi = b.vi_f; vl.bary = b.bary_f; vl.gx = r->ray_gx.p;
            vl.keys = sorted_keys; vl.vals = sorted_vals; vl.n = npairs; vl.grad_xyz = d_grad_xyz;
            rc = launch_vertex_grads(vl, s);
            if (rc) return rc;
            h->launches += 1;
        }
    }
    if (bg_grads) {  // after k_ray_grads: its direction gradients gain the background's term
        BackgroundGradsLaunch bl{};
        bl.R = R; bl.H = hd.bg_H; bl.W = hd.bg_W; bl.map = r->bgmap; bl.dirs = b.dirs; bl.s = r->bg_s.p; bl.det = det;
        bl.grad_map = d_grad_bg; bl.grad_d = d_grad_d;
        if (det && d_grad_bg != nullptr) {
            TN_TRY(r->bg_keys.grow(8 * (size_t)R)); TN_TRY(r->bg_vals.grow(8 * (size_t)R));
            bl.keys = r->bg_keys.p; bl.vals = r->bg_vals.p;
        }
        TN_TRY(launch_background_grads(bl, r->cub_tmp, s));
        h->launches += det && d_grad_bg != nullptr ? 3 : 1;
    }
    k_scatter_grads<<<(128 * 155 + 255) / 256, 256, 0, s>>>(r->gw.p, go);
    k_transpose_v64<<<(V + 31) / 32, dim3(32, 8), 0, s>>>(r->gshadow.p, d_grad_field, V);
    if (r->profile) cudaEventRecord(r->evb[3], s);
    h->launches += 5;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

// backward of the LAST tn_render_train_forward
extern "C" int tn_render_train_backward(tn_tracer *h, const float *d_grad_rgb, const float *d_grad_acc, int use_gradient_scaling,
                                        float *d_grad_field, float *const *d_grad_params12, void *stream) {
    if (!h || !d_grad_rgb || !d_grad_field || !d_grad_params12) return fail(TN_ERR_ARG, "null argument");
    RenderState *r = h->render;
    if (!r || r->last.magic != SAVED_MAGIC) return fail(TN_ERR_STATE, "tn_render_train_backward: no training forward to continue from");
    DeviceGuard g(h->device);
    return train_backward_impl(h, r->own_b, r->last, d_grad_rgb, d_grad_acc, nullptr, nullptr, use_gradient_scaling, d_grad_field, d_grad_params12,
                               nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

// ---- the training pair with per-call saved state: everything the backward reads that a later call could overwrite goes to the
// caller's blob (header + TrainBufs, saved_layout), so any number of forwards can be in flight and each backward continues from its
// own.  The gradient scratch (dout, accumulators, deterministic-mode buffers) stays in the tracer: it is dead once a backward returns.
static int saved_shape(const tn_render_config *cfg, uint32_t R, uint32_t *S2) {
    if (!cfg) return fail(TN_ERR_ARG, "null argument");
    if (R == 0) return fail(TN_ERR_ARG, "tn_render_train_forward_saved: no rays");
    if (cfg->num_fine_samples == 0) return fail(TN_ERR_ARG, "tn_render_train_forward: the fused training step needs num_fine_samples > 0");
    *S2 = cfg->num_samples + cfg->num_fine_samples + 1;
    return TN_OK;
}

extern "C" int tn_render_train_saved_bytes(tn_tracer *h, const tn_render_config *cfg, uint32_t R, size_t *bytes) {
    if (!h || !bytes) return fail(TN_ERR_ARG, "null argument");
    uint32_t S2 = 0;
    const int rc = saved_shape(cfg, R, &S2);
    if (rc) return rc;
    *bytes = saved_layout(R, S2, nullptr, nullptr, false, h->render != nullptr && h->render->bgmap != nullptr);
    return TN_OK;
}

// optional output: the expected depth d_expected_depth f32[R] (DESIGN.md §4.10)
extern "C" int tn_render_train_forward_saved(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions,
                                             uint32_t R, const float *d_jitter_coarse, const float *d_jitter_fine, float *d_rgb, float *d_acc,
                                             float *d_depth, uint8_t *d_mask, float *d_expected_depth, void *d_saved, size_t saved_bytes,
                                             void *stream) {
    if (!h || !d_saved) return fail(TN_ERR_ARG, "null argument");
    uint32_t S2 = 0;
    int rc = saved_shape(cfg, R, &S2);
    if (rc) return rc;
    if ((uintptr_t)d_saved % SAVED_ALIGN) return fail(TN_ERR_ARG, "tn_render_train_forward_saved: d_saved must be 256-byte aligned");
    if (saved_bytes < saved_layout(R, S2, nullptr, nullptr, false, h->render != nullptr && h->render->bgmap != nullptr))
        return fail(TN_ERR_ARG, "tn_render_train_forward_saved: saved_bytes is smaller than tn_render_train_saved_bytes");
    TrainFwd tf{d_jitter_coarse, d_jitter_fine, d_saved};
    return render_impl(h, cfg, d_origins, d_directions, R, d_rgb, d_acc, d_depth, d_mask, &tf, nullptr, d_expected_depth, stream);
}

// the header of a saved state, read back to the host (waits until the stream has reached the caller), if it belongs to the current
// field and weights of this tracer; `what` names the caller in the errors
static int read_saved_header(tn_tracer *h, const void *d_saved, cudaStream_t s, const char *what, SavedHeader *hd) {
    RenderState *r = h->render;
    if (!r || !r->gw.p) return fail(TN_ERR_STATE, std::string(what) + ": no training forward on this tracer");
    TN_CUDA(cudaMemcpyAsync(hd, d_saved, sizeof(*hd), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (hd->magic != SAVED_MAGIC) return fail(TN_ERR_STATE, std::string(what) + ": d_saved holds no training forward");
    if (hd->gen != r->gen)
        return fail(TN_ERR_STATE, std::string(what) + ": the field or the weights changed (tn_render_set_field / "
                                  "tn_render_set_weights) since the forward, or the forward ran on another tracer");
    return TN_OK;
}

// optional inputs: the gradients of the expected depth d_grad_expected_depth f32[R] (DESIGN.md §4.10) and of the distortion
// d_grad_distortion f32[R] (§4.11); optional outputs: the gradients at the ray origins / directions of the forward, f32[R,3] each (0 on
// empty rays; §4.8), and at the mesh vertex positions, f32[V,3] (§4.9)
// optional output of saved3: the gradient at the background map of a forward that composited over one, f32[H,W,3] (DESIGN.md §4.16)
extern "C" int tn_render_train_backward_saved3(tn_tracer *h, const void *d_saved, const float *d_grad_rgb, const float *d_grad_acc,
                                               const float *d_grad_expected_depth, const float *d_grad_distortion, int use_gradient_scaling,
                                               float *d_grad_field, float *const *d_grad_params12, float *d_grad_origins,
                                               float *d_grad_directions, float *d_grad_xyz, float *d_grad_background, void *stream) {
    if (!h || !d_saved || !d_grad_rgb || !d_grad_field || !d_grad_params12) return fail(TN_ERR_ARG, "null argument");
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    // the launch shapes depend on the call's R and S2: read the header back (waits until the stream has reached this backward)
    SavedHeader hd{};
    TN_TRY(read_saved_header(h, d_saved, s, "tn_render_train_backward_saved", &hd));
    const bool rays = d_grad_origins != nullptr || d_grad_directions != nullptr || d_grad_xyz != nullptr;
    if (rays && hd.mesh_gen != h->mesh_gen)
        return fail(TN_ERR_STATE, "tn_render_train_backward_saved: tn_load_tetrahedra or tn_update_vertices ran since the forward "
                                  "(the ray and vertex gradients read the mesh positions)");
    if (d_grad_expected_depth != nullptr && hd.edepth == 0)
        return fail(TN_ERR_STATE, "tn_render_train_backward_saved: the forward produced no expected depth (pass d_expected_depth to "
                                  "tn_render_train_forward_saved)");
    TrainBufs b{};
    saved_layout(hd.R, hd.S2, (uint8_t *)d_saved, &b, false, hd.bgmap != 0);
    return train_backward_impl(h, b, hd, d_grad_rgb, d_grad_acc, d_grad_expected_depth, d_grad_distortion, use_gradient_scaling, d_grad_field,
                               d_grad_params12, d_grad_origins, d_grad_directions, d_grad_xyz, d_grad_background, s);
}

extern "C" int tn_render_train_backward_saved2(tn_tracer *h, const void *d_saved, const float *d_grad_rgb, const float *d_grad_acc,
                                               const float *d_grad_expected_depth, const float *d_grad_distortion, int use_gradient_scaling,
                                               float *d_grad_field, float *const *d_grad_params12, float *d_grad_origins,
                                               float *d_grad_directions, float *d_grad_xyz, void *stream) {
    return tn_render_train_backward_saved3(h, d_saved, d_grad_rgb, d_grad_acc, d_grad_expected_depth, d_grad_distortion, use_gradient_scaling,
                                           d_grad_field, d_grad_params12, d_grad_origins, d_grad_directions, d_grad_xyz, nullptr, stream);
}

extern "C" int tn_render_train_backward_saved(tn_tracer *h, const void *d_saved, const float *d_grad_rgb, const float *d_grad_acc,
                                              const float *d_grad_expected_depth, int use_gradient_scaling, float *d_grad_field,
                                              float *const *d_grad_params12, float *d_grad_origins, float *d_grad_directions, float *d_grad_xyz,
                                              void *stream) {
    return tn_render_train_backward_saved2(h, d_saved, d_grad_rgb, d_grad_acc, d_grad_expected_depth, nullptr, use_gradient_scaling, d_grad_field,
                                           d_grad_params12, d_grad_origins, d_grad_directions, d_grad_xyz, stream);
}

// the distortion loss of every ray of a saved training forward (DESIGN.md §4.11): d_distortion f32[R], 0 on empty rays
extern "C" int tn_render_train_distortion(tn_tracer *h, const void *d_saved, float *d_distortion, void *stream) {
    if (!h || !d_saved || !d_distortion) return fail(TN_ERR_ARG, "null argument");
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    SavedHeader hd{};
    TN_TRY(read_saved_header(h, d_saved, s, "tn_render_train_distortion", &hd));
    TrainBufs b{};
    saved_layout(hd.R, hd.S2, (uint8_t *)d_saved, &b, false, hd.bgmap != 0);
    DistortionParams p{hd.S2, b.n_active, b.ray_list, b.ebins_f, b.sbins_f, b.out_f, d_distortion};
    // the same staging as k_composite, below k_composite_bwd's, which the forward has checked against the device's limit
    const size_t smem = SAMPLE_WARPS * sizeof(float) * 2 * ((size_t)hd.S2 + 2);
    TN_CUDA(cudaFuncSetAttribute(k_distortion, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    TN_CUDA(cudaMemsetAsync(d_distortion, 0, sizeof(float) * (size_t)hd.R, s));
    k_distortion<<<(hd.R + SAMPLE_WARPS - 1) / SAMPLE_WARPS, SAMPLE_WARPS * 32, smem, s>>>(p);
    h->launches += 1;
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

// occupancy culling (see the header; DESIGN §4.12): borrowed f32[T]; NULL switches it off.  place_samples: occupancy sampling
// (DESIGN §4.13), which needs an occupancy
extern "C" int tn_render_set_occupancy2(tn_tracer *h, const float *d_occ, float threshold, int place_samples) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (!std::isfinite(threshold) || threshold < 0.f)
        return fail(TN_ERR_ARG, "tn_render_set_occupancy: the threshold must be finite and >= 0");
    if (place_samples && d_occ == nullptr)
        return fail(TN_ERR_ARG, "tn_render_set_occupancy2: placing the samples by occupancy needs an occupancy (d_occ is NULL)");
    DeviceGuard g(h->device);
    RenderState *r = state(h);
    r->occ = d_occ;
    r->occ_thr = threshold;
    r->occ_place = place_samples != 0;
    r->occ_T = h->mesh.T;
    return TN_OK;
}

extern "C" int tn_render_set_occupancy(tn_tracer *h, const float *d_occ, float threshold) {
    return tn_render_set_occupancy2(h, d_occ, threshold, 0);
}

// background map (see the header; DESIGN §4.16): borrowed f32[H,W,3], W = 2H; NULL switches back to cfg->background.  Every call starts a
// new generation, so the backward of a forward before it returns TN_ERR_STATE
extern "C" int tn_render_set_background(tn_tracer *h, const float *d_map, uint32_t H, uint32_t W) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (d_map != nullptr && (H == 0 || H > 16384 || W != 2 * H))
        return fail(TN_ERR_ARG, "tn_render_set_background: the map must be [H, 2H, 3] with 1 <= H <= 16384");
    DeviceGuard g(h->device);
    RenderState *r = state(h);
    r->bgmap = d_map;
    r->bg_H = d_map != nullptr ? H : 0;
    r->bg_W = d_map != nullptr ? W : 0;
    r->bg_gen = next_generation();
    return TN_OK;
}

// d_occ f32[T] <- max(decay * d_occ, the largest probe density of each tetrahedron): probe rows in chunks of OCC_CHUNK tetrahedra
// through k_mlp<false, 3> (the density the renderer uses, bf16x3), then one thread per tetrahedron
extern "C" int tn_occupancy_update(tn_tracer *h, float *d_occ, float decay, void *stream) {
    if (!h || !d_occ) return fail(TN_ERR_ARG, "null argument");
    if (!std::isfinite(decay) || decay < 0.f) return fail(TN_ERR_ARG, "tn_occupancy_update: the decay must be finite and >= 0");
    if (!h->mesh.nodes.p) return fail(TN_ERR_STATE, "tn_occupancy_update: no tetrahedra loaded");
    RenderInputs in{};
    if (render_inputs(h, &in) != TN_OK) return fail(TN_ERR_STATE, "tn_occupancy_update: call tn_render_set_field and tn_render_set_weights first");
    if (in.V != h->mesh.V) return fail(TN_ERR_ARG, "tn_occupancy_update: field has a different vertex count than the mesh");
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    RenderState *r = h->render;
    const uint32_t T = h->mesh.T;
    const uint32_t chunk = std::min(T, OCC_CHUNK);
    if (chunk == 0) return TN_OK;
    const size_t rows = (size_t)chunk * OCC_PROBES;
    TN_TRY(r->occ_vi.grow(rows)); TN_TRY(r->occ_bary.grow(3 * rows)); TN_TRY(r->occ_sig.grow(rows)); TN_TRY(r->occ_small.grow(2));
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    for (uint32_t t0 = 0; t0 < T; t0 += chunk) {
        const uint32_t nt = std::min(chunk, T - t0);
        const uint64_t n = (uint64_t)nt * OCC_PROBES;
        k_occ_rows<<<(uint32_t)((n + 255) / 256), 256, 0, s>>>(t0, nt, h->mesh.cells, r->occ_vi.p, r->occ_bary.p, r->occ_small.p);
        MlpParams mp{};
        mp.n_active = r->occ_small.p; mp.S = OCC_PROBES; mp.vi = r->occ_vi.p; mp.bary = r->occ_bary.p; mp.fshadow = in.fshadow;
        mp.wimg = in.wimg; mp.bias = in.bias; mp.head = in.head; mp.out = r->occ_sig.p; mp.tile_ctr = r->occ_small.p + 1;
        const uint64_t tiles = (n + MLP_TILE - 1) / MLP_TILE;
        const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((tiles + MLP_WGS - 1) / MLP_WGS, (uint64_t)sms));
        TN_TRY(launch_mlp<false, 3>(mp, grid, s));
        k_occ_reduce<<<(nt + 255) / 256, 256, 0, s>>>(t0, nt, r->occ_sig.p, decay, d_occ);
        h->launches += 3;
    }
    TN_CUDA(cudaGetLastError());
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

// per-kernel timing of the LAST tn_render_train_backward or tn_render_train_backward_saved call: ms3 = composite_bwd, mlp_bwd, finalize (memsets excluded)
extern "C" int tn_render_get_backward_timings(tn_tracer *h, float *ms3) {
    if (!h || !h->render || !h->render->profile) return fail(TN_ERR_STATE, "profiling is not enabled");
    DeviceGuard g(h->device);
    RenderState *r = h->render;
    TN_CUDA(cudaEventSynchronize(r->evb[3]));
    for (int i = 0; i < 3; ++i) TN_CUDA(cudaEventElapsedTime(&ms3[i], r->evb[i], r->evb[i + 1]));
    return TN_OK;
}

// test / debug hook: device pointers of the intermediate buffers of the last tn_render call (the fine pass's: of the last call that wrote
// the tracer's own blob)
extern "C" int tn_render_debug_buffers(tn_tracer *h, void **ptrs16) {
    if (!h || !h->render) return fail(TN_ERR_STATE, "no render state");
    RenderState *r = h->render;
    const TrainBufs &b = r->own_b;
    void *v[16] = {r->num.p, r->dist.p, b.n_active, b.ray_list, r->ebins_c.p, r->sbins_c.p, r->vi_c.p, r->bary_c.p,
                   r->dens_c.p, b.ebins_f, b.vi_f, b.bary_f, b.out_f, b.dirbias, r->fshadow.p, r->wimg.p};
    for (int i = 0; i < 16; ++i) ptrs16[i] = v[i];
    return TN_OK;
}

// test hook: device pointer of the per-sample density gradient of the last tn_render call with normals, float4 (x, y, z, 0) per sample in
// the slot order of the pass that gives the colours (vi_f / bary_f, or vi_c / bary_c in single-pass configurations)
extern "C" int tn_render_debug_normals_grad(tn_tracer *h, void **ptr) {
    if (!h || !h->render || !h->render->grad_n.p) return fail(TN_ERR_STATE, "no normals render");
    *ptr = h->render->grad_n.p;
    return TN_OK;
}

// test hook: device pointer of dL/dx per fine sample of the last tn_render_train_backward_saved call with ray or vertex gradients, float4 (x, y, z, 0) per sample
// in the slot order of that call's forward (0 for unmatched samples and flat tetrahedra)
extern "C" int tn_render_debug_ray_grads(tn_tracer *h, void **ptr) {
    if (!h || !h->render || !h->render->ray_gx.p) return fail(TN_ERR_STATE, "no backward with ray gradients");
    *ptr = h->render->ray_gx.p;
    return TN_OK;
}
