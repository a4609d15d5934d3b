// tn_mlp_bwd.cuh -- fused backward of the interpolate -> MLP fine pass on warpgroup MMA (wgmma, sm_90a): the training half of the
// hot path.
//
// Replaces, for the n_active*S2 samples of the fine pass of one training step, what autograd runs in the reference as ~40 torch
// kernels over [R*S,128] fp32 activations in HBM:
//   backward of RGBFieldHead / DensityFieldHead / mlp_head / mlp_base (tetranerf/nerfstudio/model.py:596-621, nerfstudio MLP)
//   and interpolate_values_backward (src/tetrahedra_tracer.cu:223-248, tetranerf/utils/extension/__init__.py:36-42).
// Nothing of size [samples,128] ever reaches HBM: per 64-sample tile the forward activations are RECOMPUTED (4 GEMMs), the
// input-gradient chain (4 GEMMs) and the weight-gradient GEMMs (4) run on the tensor cores with bf16x3 products (fp32-level
// accuracy), and the feature gradient goes to the [V,64] field-gradient shadow with vector reductions.
//
// One warpgroup per CTA, one 64-sample tile at a time (rows = samples):
//   forward   L1: D = X  W1^T     L2: D = H1 W2^T     L3: D = H2 W3^T     L4: D = H3 W4b^T      A in registers, B = W K-major
//   dX chain  dH3 = dA4 W4b       dH2 = dA3 W3        dH1 = dA2 W2        dX = dA1 W1           A in registers, B = W MN-major
//   dW        dW4b += dA4^T H3    dW3 += dA3^T H2     dW2 += dA2^T H1     dW1 += dA1^T X        A, B from shared memory, MN-major
// X = interpolated features, H_l = relu(.) activations, dA_l = dH_l * (H_l > 0).  Every operand kept in shared memory is bf16 hi|lo
// in one layout ([row][64-column block], 128-byte rows, 128-byte swizzle); the dW GEMMs read the same bytes MN-major (K along the
// rows) through the descriptors' transpose bits, so no transposed copy is ever made.  The accumulators live in registers: the
// weight gradients of a tile (two M = 64 halves per layer) are added to the global accumulators with vector reductions.
// The weights stream through a two-stage TMA ring in the fixed order of the 14 stages a tile consumes.
// Shared memory: ring 2 x 32 KB | X 16 KB | H1, H2, H3, dA 32 KB each | heads, column sums, barriers.
//
// Deterministic mode (k_mlp_bwd<true>, tn_render_set_deterministic): the same arithmetic per tile, but no reduction whose order depends
// on scheduling.  The tiles are split statically into BWD_PARTS contiguous partitions (independent of the grid size); a CTA takes
// partitions blockIdx.x, blockIdx.x + gridDim.x, ... and their tiles in order, and accumulates dW and the column sums of each partition
// in a partition-private slice of `part` with plain read-modify-write.  The four warps keep separate column sums, combined in warp
// order when a partition ends.  The per-ray direction-bias gradient goes to one partial row per (tile, ray, warp) and dX rows are
// stored to `dx`; tn_render.cu reduces all of these in a fixed order.
#pragma once
#include <type_traits>

#include "tn_common.cuh"
#include "tn_mlp.cuh"
#include "tn_tc.cuh"

namespace tn {

constexpr uint32_t BWD_THREADS = 128;                 // one warpgroup
constexpr uint32_t BWD_TILE = 64;
constexpr uint32_t BWD_STAGE = 32768;
constexpr uint32_t BWD_OFF_RING = 0;                  // 2 stages
constexpr uint32_t BWD_OFF_X = 65536;                 // hi 8 KB | lo 8 KB
constexpr uint32_t BWD_OFF_H = 81920;                 // H1, H2, H3: each hi blk0 | hi blk1 | lo blk0 | lo blk1 (8 KB each)
constexpr uint32_t BWD_OFF_DA = BWD_OFF_H + 3 * 32768;
constexpr uint32_t BWD_OFF_HEAD = BWD_OFF_DA + 32768; // wd[128] wc[3][128]
constexpr uint32_t BWD_OFF_SUMS = BWD_OFF_HEAD + 2048;  // column sums [7][128]: b1 b2 b3 wd wc0 wc1 wc2
constexpr uint32_t BWD_OFF_BARS = BWD_OFF_SUMS + 7 * 512;  // ring_full[2], tile slots[2]
constexpr uint32_t BWD_SMEM_BYTES = BWD_OFF_BARS + 32;
static_assert(BWD_SMEM_BYTES <= 232448, "k_mlp_bwd shared memory exceeds 227 KB");
static_assert(BWD_OFF_X % 1024 == 0 && BWD_OFF_H % 1024 == 0 && BWD_OFF_DA % 1024 == 0, "swizzled operands need 1024-byte alignment");
constexpr uint32_t BWD_WIMG_BYTES = 7 * BWD_STAGE;    // [L1 hi|lo][L2 HI][L2 LO][L3 HI][L3 LO][L4 HI][L4 LO]
constexpr uint32_t BWD_NSEQ = 14;                     // weight stages consumed per tile

struct MlpBwdParams {
    const uint32_t *n_active;
    uint32_t S;                 // samples per ray of the fine pass (S2)
    const uint4 *vi;            // [rows] matched vertex ids
    const float *bary;          // [rows,3]
    const float *fshadow;       // [V,64]
    const uint8_t *wimg;        // backward weight image (7 stages of 32 KB, see tn_render_set_weights)
    const float *bias;          // b1 b2 b3 [3][128]
    const float *head;          // wd[128] wc[3][128] ...
    const float *dirbias;       // [n_active,128]
    const float4 *dout;         // [rows] (d sigma_pre, d z_r, d z_g, d z_b): gradients at the head pre-activations
    float *gshadow;             // [V,64] field gradient accumulator (zeroed by the caller)
    float *gw;                  // packed MLP gradient accumulators (zeroed by the caller), see GW_* offsets
    float *g_dirbias;           // [n_active,128] gradient at the per-ray direction bias (zeroed by the caller)
    uint32_t *tile_ctr;
};
// deterministic mode (k_mlp_bwd<true>): gw, g_dirbias, gshadow and tile_ctr are not used
struct MlpBwdDetParams : MlpBwdParams {
    float *part;                // [BWD_PARTS][BWD_PART_STRIDE] per-partition dW and column sums (GW_* offsets)
    float *gdb_part;            // [4 (ntiles + n_active)][128] direction-bias gradient partials, row 4 (tile + slot) + warp
    float *dx;                  // [rows,64] gradient at the interpolated features
};
template <bool DET>
using MlpBwdParamsT = typename std::conditional<DET, MlpBwdDetParams, MlpBwdParams>::type;
// offsets (floats) inside gw
constexpr uint32_t GW_W1 = 0, GW_W2 = 8192, GW_W3 = 24576, GW_W4B = 40960, GW_B1 = 57344, GW_B2 = 57472, GW_B3 = 57600, GW_WD = 57728, GW_WC = 57856,
                   GW_SUMS = 58240 /* sum ds, sum dz_r, dz_g, dz_b */, GW_W4DIR = 58244 /* [128][27] */, GW_B4 = 61700, GW_TOTAL = 61828;

// deterministic mode: fixed tile partitions; a partition's slice holds gw[0, GW_SUMS): dW1..dW4b and the 7 column sums (b1 b2 b3 wd wc)
constexpr uint32_t BWD_PARTS = 256;
constexpr uint32_t BWD_PART_STRIDE = GW_SUMS;
constexpr uint32_t BWD_DET_OFF_BARS = BWD_OFF_SUMS + 4 * 7 * 512;  // column sums per warp [4][7][128]
constexpr uint32_t BWD_DET_SMEM_BYTES = BWD_DET_OFF_BARS + 32;
static_assert(BWD_DET_SMEM_BYTES <= 232448, "k_mlp_bwd<true> shared memory exceeds 227 KB");
// partition q holds tiles [part_lo(q), part_lo(q + 1))
__host__ __device__ __forceinline__ uint32_t bwd_part_lo(uint32_t q, uint32_t ntiles) { return (uint32_t)(((uint64_t)q * ntiles) / BWD_PARTS); }
__host__ __device__ __forceinline__ uint32_t bwd_part_of(uint32_t tile, uint32_t ntiles) {
    return (uint32_t)((((uint64_t)tile + 1) * BWD_PARTS - 1) / ntiles);
}
// first tile of the first non-empty partition q0, q0 + step, ... (MLP_NO_TILE: none)
__device__ __forceinline__ uint32_t bwd_det_first(uint32_t q, uint32_t step, uint32_t ntiles) {
    for (; q < BWD_PARTS; q += step)
        if (bwd_part_lo(q, ntiles) < bwd_part_lo(q + 1, ntiles)) return bwd_part_lo(q, ntiles);
    return MLP_NO_TILE;
}

__device__ __forceinline__ void red_add_v2(float *dst, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add_v4(float *dst, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// accumulator columns 8j + 2t, +1 of rows g (p0) and g + 8 (p1) -> four consecutive columns 8j + 4 (t >> 1) .. +3 of ONE row: row g
// for even t, row g + 8 for odd t (one shuffle with the neighbour t ^ 1), so that each thread issues one 16-byte reduction per j
__device__ __forceinline__ float4 quad_of_row(float2 p0, float2 p1, uint32_t t) {
    const bool odd = (t & 1u) != 0u;
    const float2 send = odd ? p0 : p1;
    float2 recv;
    recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
    recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
    return odd ? make_float4(recv.x, recv.y, p1.x, p1.y) : make_float4(p0.x, p0.y, recv.x, recv.y);
}

// one bf16 hi/lo pair (columns c = 8j + 2t, c+1 of row R) into a [row][64-column block] operand buffer of 64 rows (8 KB per block);
// the lo half sits lo_off bytes further.  The swizzled address is formed inside the asm: computed in C++, the loop-invariant
// addresses of every (buffer, row, j) were hoisted out of the tile loop and spilled to local memory.
__device__ __forceinline__ void st_pair(uint32_t base, uint32_t R, uint32_t j, uint32_t t, uint32_t lo_off, uint32_t h, uint32_t l) {
    const uint32_t rowoff = (R >> 3) * 1024u + (R & 7u) * 128u + 4u * t;
    asm volatile(
        "{\n\t.reg .b32 a, x, y;\n\t"
        "and.b32 x, %2, 7;\n\txor.b32 x, x, %3;\n\tshl.b32 x, x, 4;\n\t"   // 16-byte chunk ((c mod 64) / 8) ^ (R mod 8)
        "shr.b32 y, %2, 3;\n\tshl.b32 y, y, 13;\n\t"                          // 64-column block c / 64, 8 KB apart
        "add.u32 a, %0, %1;\n\tadd.u32 a, a, x;\n\tadd.u32 a, a, y;\n\t"
        "st.shared.b32 [a], %5;\n\tadd.u32 a, a, %4;\n\tst.shared.b32 [a], %6;\n\t}" ::"r"(base),
        "r"(rowoff), "r"(j), "r"(R & 7u), "r"(lo_off), "r"(h), "r"(l)
        : "memory");
}

// sum over the 64 rows of the tile of (s0, s1) = this thread's two-row partial sums of columns c, c+1: reduced over the eight
// threads of a warp that share t, then added into the shared-memory column sums (four warps)
// (deterministic mode: into the warp's own copy of the sums, [warp][7][128], without atomics)
template <bool DET = false>
__device__ __forceinline__ void colsum2(float *dst, uint32_t c, float s0, float s1, uint32_t lane, uint32_t warp = 0) {
#pragma unroll
    for (int m = 4; m <= 16; m <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, m);
        s1 += __shfl_xor_sync(0xffffffffu, s1, m);
    }
    if constexpr (DET) {
        if (lane < 4) { float *w = dst + warp * (7u * 128u); w[c] += s0; w[c + 1] += s1; }
    } else {
        if (lane < 4) { atomicAdd(dst + c, s0); atomicAdd(dst + c + 1, s1); }
    }
}

// dW (+)= dA^T H for one M = 64 half of the output features: A = dA (MN-major, half mh of its columns), B = H (MN-major, NB
// 64-column blocks), K = the tile's 64 rows; bf16x3.  Result added to gw[dst + out * (64 NB) + in] (deterministic mode: every
// thread owns its addresses, plain read-modify-write, or a store for the first tile of a partition).
template <int NB, bool DET = false>
__device__ __forceinline__ void dw_half(uint32_t sDA, uint32_t sHb, uint32_t h_lo_off, uint32_t mh, float *dst, uint32_t warp, uint32_t g, uint32_t t,
                                        bool first = false) {
    using namespace tc;
    float d[32 * NB];
#pragma unroll
    for (int i = 0; i < 32 * NB; ++i) d[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int term = 0; term < 3; ++term) {  // (dA_hi, H_hi) (dA_lo, H_hi) (dA_hi, H_lo)
        const uint32_t ao = term == 1 ? 16384u : 0u, bo = term == 2 ? h_lo_off : 0u;
#pragma unroll
        for (uint32_t kk = 0; kk < 4; ++kk) {
            const uint64_t da = make_desc(sDA + ao + mh * 8192u + kk * 2048u, 8192u, 1024u);
            const uint64_t db = make_desc(sHb + bo + kk * 2048u, 8192u, 1024u);
            if constexpr (NB == 2) wgmma_ss_bf16_n128<1, 1>(d, da, db, 1u);
            else wgmma_ss_bf16_n64<1, 1>(d, da, db, 1u);
        }
    }
    wgmma_commit();
    wgmma_wait0();
    reg_fence(d);
    const uint32_t o = mh * 64u + warp * 16u + g + 8u * (t & 1u);  // the row this thread reduces (quad_of_row)
#pragma unroll
    for (int j = 0; j < 4 * NB * 2; ++j) {
        const float4 q = quad_of_row(make_float2(d[4 * j], d[4 * j + 1]), make_float2(d[4 * j + 2], d[4 * j + 3]), t);
        if constexpr (DET) {
            float4 *a = reinterpret_cast<float4 *>(dst + (size_t)o * (64u * NB) + 8u * j + 4u * (t >> 1));
            float4 r = q;
            if (!first) { const float4 b = *a; r = make_float4(b.x + q.x, b.y + q.y, b.z + q.z, b.w + q.w); }
            *a = r;
        } else {
            red_add_v4(dst + (size_t)o * (64u * NB) + 8u * j + 4u * (t >> 1), q.x, q.y, q.z, q.w);
        }
    }
}

template <int N>
__device__ __forceinline__ void zero(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) d[i] = 0.f;
}

// A fragments (hi / lo) of a 64 x 128 operand held as an accumulator-layout array
__device__ __forceinline__ void frag_pair(float x0, float x1, float y0, float y1, int j, uint32_t (&ah)[32], uint32_t (&al)[32]) {
    const int i = 4 * (j >> 1) + 2 * (j & 1);
    tc::split_pack2(x0, x1, ah[i], al[i]);
    tc::split_pack2(y0, y1, ah[i + 1], al[i + 1]);
}

template <bool DET>
__global__ void __launch_bounds__(BWD_THREADS, 1) k_mlp_bwd(const MlpBwdParamsT<DET> p) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t tn_bwd_smem[];
    constexpr uint32_t OFF_BARS = DET ? BWD_DET_OFF_BARS : BWD_OFF_BARS;
    uint8_t *smem = tn_bwd_smem;
    float *head_s = reinterpret_cast<float *>(smem + BWD_OFF_HEAD);  // wd[128], wc[3][128]
    float *sums = reinterpret_cast<float *>(smem + BWD_OFF_SUMS);
    uint64_t *ring_full = reinterpret_cast<uint64_t *>(smem + OFF_BARS);
    volatile uint32_t *slots = reinterpret_cast<volatile uint32_t *>(smem + OFF_BARS + 16);

    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u, g = lane >> 2, t = lane & 3u;
    const uint32_t n_active = *p.n_active;
    const uint64_t total_rows = (uint64_t)n_active * p.S;
    const uint32_t ntiles = (uint32_t)((total_rows + BWD_TILE - 1) / BWD_TILE);
    uint32_t first_tile = blockIdx.x;
    if constexpr (DET) {
        if (ntiles == 0) return;
        first_tile = bwd_det_first(blockIdx.x, gridDim.x, ntiles);
        if (first_tile == MLP_NO_TILE) return;
    } else {
        if (blockIdx.x >= ntiles) return;
    }

    if (tid == 0) {
        mbar_init(&ring_full[0], 1); mbar_init(&ring_full[1], 1);
        fence_barrier_init();
        slots[0] = first_tile;
    }
    for (uint32_t i = tid; i < 512; i += BWD_THREADS) head_s[i] = p.head[i];
    for (uint32_t i = tid; i < (DET ? 4u : 1u) * 7 * 128; i += BWD_THREADS) sums[i] = 0.f;
    __syncthreads();
    const uint32_t sR = smem_u32(smem + BWD_OFF_RING), sX = smem_u32(smem + BWD_OFF_X), sH = smem_u32(smem + BWD_OFF_H), sDA = smem_u32(smem + BWD_OFF_DA);
    const float *wd = head_s, *wc = head_s + 128;

    // weight ring: stage sequence number i -> buffer i & 1; image stage of position q = i % 14 of a tile:
    // forward L1, L2 HI, L2 LO, L3 HI, L3 LO, L4 HI, L4 LO; backward W4 HI, W4 LO, W3 HI, W3 LO, W2 HI, W2 LO, W1
    auto ring_issue = [&](uint32_t i) {
        const uint32_t q = i % BWD_NSEQ;
        const uint32_t img = q < 7u ? q : (q == 13u ? 0u : (q & 1u ? 12u - q : 14u - q));
        uint64_t *bar = &ring_full[i & 1u];
        mbar_arrive_expect_tx(bar, BWD_STAGE);
        tma_bulk_g2s(smem + BWD_OFF_RING + (i & 1u) * BWD_STAGE, p.wimg + img * BWD_STAGE, 16384, bar);
        tma_bulk_g2s(smem + BWD_OFF_RING + (i & 1u) * BWD_STAGE + 16384u, p.wimg + img * BWD_STAGE + 16384u, 16384, bar);
    };
    if (tid == 0) ring_issue(0);
    uint32_t seq = 0;
    // stage `seq` (advances it): every warp is done with the previous stage, whose buffer now receives the next one
    auto ring_acquire = [&](bool more) -> uint32_t {
        wg_sync(0);
        if (tid == 0 && more) ring_issue(seq + 1u);
        mbar_wait(&ring_full[seq & 1u], (seq >> 1) & 1u);
        const uint32_t w = sR + (seq & 1u) * BWD_STAGE;
        ++seq;
        return w;
    };
    // an operand buffer written by the generic proxy is read by the next wgmma: fence + barrier
    auto publish = [&]() {
        fence_proxy_async();
        wg_sync(0);
    };

#pragma unroll 1
    for (uint32_t n = 0;; ++n) {
        wg_sync(0);
        const uint32_t tile = slots[n & 1u];
        if (tile == MLP_NO_TILE) break;
        // deterministic mode: the partition of the tile, and whether the tile opens / closes it
        uint32_t part_q = 0;
        bool part_first = false, part_last = false;
        if constexpr (DET) {
            part_q = bwd_part_of(tile, ntiles);
            part_first = tile == bwd_part_lo(part_q, ntiles);
            part_last = tile + 1u == bwd_part_lo(part_q + 1u, ntiles);
        }
        float *gw = p.gw;
        if constexpr (DET) gw = p.part + (size_t)part_q * BWD_PART_STRIDE;
        if (tid == 0) {
            if constexpr (DET) {
                slots[(n + 1u) & 1u] = part_last ? bwd_det_first(part_q + gridDim.x, gridDim.x, ntiles) : tile + 1u;
            } else {
                const uint32_t nx = gridDim.x + atomicAdd(p.tile_ctr, 1u);
                slots[(n + 1u) & 1u] = nx < ntiles ? nx : MLP_NO_TILE;
            }
        }
        const uint32_t R0 = warp * 16u + g, R1 = R0 + 8u;
        const uint64_t row0 = (uint64_t)tile * BWD_TILE + R0, row1 = row0 + 8u;
        const bool valid0 = row0 < total_rows, valid1 = row1 < total_rows;
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 g0 = valid0 ? __ldg(p.dout + row0) : z4, g1 = valid1 ? __ldg(p.dout + row1) : z4;

        uint32_t ah[32], al[32];
        unsigned long long mask[3];
        float d[64];
        const bool more_tiles = slots[(n + 1u) & 1u] != MLP_NO_TILE;  // (tid 0 wrote it above; only tid 0 uses it)
        // ---------- forward layer 1; X also goes to shared memory for dW1 ----------
        {
            uint32_t xh[16], xl[16];
            gather_rows<3>(p.vi, p.bary, p.fshadow, row0, total_rows, t, xh, xl);
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int i = 4 * (c >> 1) + 2 * (c & 1);
                st_pair(sX, R0, (uint32_t)c, t, 8192u, xh[i], xl[i]);
                st_pair(sX, R1, (uint32_t)c, t, 8192u, xh[i + 1], xl[i + 1]);
            }
            const uint32_t w = ring_acquire(true);
            zero(d);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a[4] = {xh[4 * kk], xh[4 * kk + 1], xh[4 * kk + 2], xh[4 * kk + 3]};
                const uint32_t b[4] = {xl[4 * kk], xl[4 * kk + 1], xl[4 * kk + 2], xl[4 * kk + 3]};
                wgmma_rs_bf16_n128<0>(d, a, make_desc(w + kk * 32u), kk > 0 ? 1u : 0u);
                wgmma_rs_bf16_n128<0>(d, b, make_desc(w + kk * 32u), 1u);
                wgmma_rs_bf16_n128<0>(d, a, make_desc(w + 16384u + kk * 32u), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            reg_fence(d);
        }
        // ---------- epilogues of forward layers 1..3 (H_l -> shared memory, A fragments, sign masks) and layers 2..3 ----------
#pragma unroll
        for (int l = 0; l < 3; ++l) {
            if (l > 0) {
                uint32_t w = ring_acquire(true);
                zero(d);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) {
                    const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                    const uint32_t b[4] = {al[4 * kk], al[4 * kk + 1], al[4 * kk + 2], al[4 * kk + 3]};
                    const uint32_t wo = (uint32_t)(kk >> 2) * 16384u + (uint32_t)(kk & 3) * 32u;
                    wgmma_rs_bf16_n128<0>(d, a, make_desc(w + wo), kk > 0 ? 1u : 0u);
                    wgmma_rs_bf16_n128<0>(d, b, make_desc(w + wo), 1u);
                }
                wgmma_commit();
                wgmma_wait0();
                w = ring_acquire(true);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) {
                    const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                    wgmma_rs_bf16_n128<0>(d, a, make_desc(w + (uint32_t)(kk >> 2) * 16384u + (uint32_t)(kk & 3) * 32u), 1u);
                }
                wgmma_commit();
                wgmma_wait0();
                reg_fence(d);
            }
            const float *bias = p.bias + 128 * l;
            const uint32_t hb = sH + 32768u * l;
            unsigned long long mk = 0ull;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint32_t c = 8u * j + 2u * t;
                const float2 b = __ldg(reinterpret_cast<const float2 *>(bias + c));
                const float v0 = d[4 * j] + b.x, v1 = d[4 * j + 1] + b.y, v2 = d[4 * j + 2] + b.x, v3 = d[4 * j + 3] + b.y;
                mk |= (unsigned long long)((v0 > 0.f ? 1u : 0u) | (v1 > 0.f ? 2u : 0u) | (v2 > 0.f ? 4u : 0u) | (v3 > 0.f ? 8u : 0u)) << (4 * j);
                const float x0 = fmaxf(v0, 0.f), x1 = fmaxf(v1, 0.f), y0 = fmaxf(v2, 0.f), y1 = fmaxf(v3, 0.f);
                frag_pair(x0, x1, y0, y1, j, ah, al);
                const int i = 4 * (j >> 1) + 2 * (j & 1);
                st_pair(hb, R0, (uint32_t)j, t, 16384u, ah[i], al[i]);
                st_pair(hb, R1, (uint32_t)j, t, 16384u, ah[i + 1], al[i + 1]);
                if (l == 2)  // d wd[k] = sum_s d sigma_pre[s] H3[s,k]
                    colsum2<DET>(sums + 3 * 128, c, g0.x * x0 + g1.x * y0, g0.x * x1 + g1.x * y1, lane, warp);
            }
            mask[l] = mk;
        }
        // ---------- forward layer 4 (H4 = relu(D + per-ray direction bias)) -> head weight gradients, dA4 ----------
        {
            uint32_t w = ring_acquire(true);
            zero(d);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                const uint32_t b[4] = {al[4 * kk], al[4 * kk + 1], al[4 * kk + 2], al[4 * kk + 3]};
                const uint32_t wo = (uint32_t)(kk >> 2) * 16384u + (uint32_t)(kk & 3) * 32u;
                wgmma_rs_bf16_n128<0>(d, a, make_desc(w + wo), kk > 0 ? 1u : 0u);
                wgmma_rs_bf16_n128<0>(d, b, make_desc(w + wo), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            w = ring_acquire(true);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                wgmma_rs_bf16_n128<0>(d, a, make_desc(w + (uint32_t)(kk >> 2) * 16384u + (uint32_t)(kk & 3) * 32u), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            reg_fence(d);
            const uint32_t ray0 = (uint32_t)(min(row0, total_rows - 1) / p.S), ray1 = (uint32_t)(min(row1, total_rows - 1) / p.S);
            const float *db0 = p.dirbias + (size_t)ray0 * 128, *db1 = p.dirbias + (size_t)ray1 * 128;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint32_t c = 8u * j + 2u * t;
                const float2 b0 = __ldg(reinterpret_cast<const float2 *>(db0 + c)), b1 = __ldg(reinterpret_cast<const float2 *>(db1 + c));
                const float v0 = d[4 * j] + b0.x, v1 = d[4 * j + 1] + b0.y, v2 = d[4 * j + 2] + b1.x, v3 = d[4 * j + 3] + b1.y;
                const float x0 = fmaxf(v0, 0.f), x1 = fmaxf(v1, 0.f), y0 = fmaxf(v2, 0.f), y1 = fmaxf(v3, 0.f);  // H4
                // d wc[ch][k] = sum_s d z_ch[s] H4[s,k]
                colsum2<DET>(sums + 4 * 128, c, g0.y * x0 + g1.y * y0, g0.y * x1 + g1.y * y1, lane, warp);
                colsum2<DET>(sums + 5 * 128, c, g0.z * x0 + g1.z * y0, g0.z * x1 + g1.z * y1, lane, warp);
                colsum2<DET>(sums + 6 * 128, c, g0.w * x0 + g1.w * y0, g0.w * x1 + g1.w * y1, lane, warp);
                // dA4 = (d z . wc) * (H4 > 0)
                const float wa0 = wc[c], wa1 = wc[c + 1], wb0 = wc[128 + c], wb1 = wc[128 + c + 1], wc0 = wc[256 + c], wc1 = wc[256 + c + 1];
                d[4 * j] = v0 > 0.f ? fmaf(g0.w, wc0, fmaf(g0.z, wb0, g0.y * wa0)) : 0.f;
                d[4 * j + 1] = v1 > 0.f ? fmaf(g0.w, wc1, fmaf(g0.z, wb1, g0.y * wa1)) : 0.f;
                d[4 * j + 2] = v2 > 0.f ? fmaf(g1.w, wc0, fmaf(g1.z, wb0, g1.y * wa0)) : 0.f;
                d[4 * j + 3] = v3 > 0.f ? fmaf(g1.w, wc1, fmaf(g1.z, wb1, g1.y * wa1)) : 0.f;
                frag_pair(d[4 * j], d[4 * j + 1], d[4 * j + 2], d[4 * j + 3], j, ah, al);
                const int i = 4 * (j >> 1) + 2 * (j & 1);
                st_pair(sDA, R0, (uint32_t)j, t, 16384u, ah[i], al[i]);
                st_pair(sDA, R1, (uint32_t)j, t, 16384u, ah[i + 1], al[i + 1]);
            }
            // gradient at the per-ray direction bias (-> b4 and W4[:, :27] in k_dirbias_grads): column sums per ray.  The warp's rows
            // belong to rays ray_lo .. ray_hi (usually one, two at a ray boundary).
            const uint32_t ray_lo = __shfl_sync(0xffffffffu, ray0, 0), ray_hi = __shfl_sync(0xffffffffu, ray1, 28);
#pragma unroll 1
            for (uint32_t sl = ray_lo; sl <= ray_hi; ++sl) {
                const bool in0 = valid0 && ray0 == sl, in1 = valid1 && ray1 == sl;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    float s0 = (in0 ? d[4 * j] : 0.f) + (in1 ? d[4 * j + 2] : 0.f);
                    float s1 = (in0 ? d[4 * j + 1] : 0.f) + (in1 ? d[4 * j + 3] : 0.f);
#pragma unroll
                    for (int m = 4; m <= 16; m <<= 1) {
                        s0 += __shfl_xor_sync(0xffffffffu, s0, m);
                        s1 += __shfl_xor_sync(0xffffffffu, s1, m);
                    }
                    if constexpr (DET) {
                        if (lane < 4) *reinterpret_cast<float2 *>(p.gdb_part + (4 * ((size_t)tile + sl) + warp) * 128 + 8u * j + 2u * t) = make_float2(s0, s1);
                    } else {
                        if (lane < 4) red_add_v2(p.g_dirbias + (size_t)sl * 128 + 8u * j + 2u * t, s0, s1);
                    }
                }
            }
            publish();
        }
        // ---------- layers 4, 3, 2: dW_l += dA_l^T H_{l-1}; dH_{l-1} = dA_l W_l; dA_{l-1} = dH_{l-1} * (H_{l-1} > 0) ----------
#pragma unroll 1
        for (int l = 2; l >= 0; --l) {
            float *gdst = gw + (l == 2 ? GW_W4B : (l == 1 ? GW_W3 : GW_W2));
            const uint32_t hb = sH + 32768u * (uint32_t)l;  // H3, H2, H1
            dw_half<2, DET>(sDA, hb, 16384u, 0, gdst, warp, g, t, part_first);
            dw_half<2, DET>(sDA, hb, 16384u, 1, gdst, warp, g, t, part_first);
            uint32_t w = ring_acquire(true);
            zero(d);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                const uint32_t b[4] = {al[4 * kk], al[4 * kk + 1], al[4 * kk + 2], al[4 * kk + 3]};
                wgmma_rs_bf16_n128<1>(d, a, make_desc(w + kk * 2048u, 16384u, 1024u), kk > 0 ? 1u : 0u);
                wgmma_rs_bf16_n128<1>(d, b, make_desc(w + kk * 2048u, 16384u, 1024u), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            w = ring_acquire(true);  // (its barrier also orders the dW reads of dA before the stores below)
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                wgmma_rs_bf16_n128<1>(d, a, make_desc(w + kk * 2048u, 16384u, 1024u), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            reg_fence(d);
            const unsigned long long mk = l == 2 ? mask[2] : (l == 1 ? mask[1] : mask[0]);
            float *bsum = sums + 128 * l;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint32_t c = 8u * j + 2u * t;
                float e0 = d[4 * j], e1 = d[4 * j + 1], e2 = d[4 * j + 2], e3 = d[4 * j + 3];
                if (l == 2) {  // the density head reads H3 as well
                    e0 = fmaf(g0.x, wd[c], e0); e1 = fmaf(g0.x, wd[c + 1], e1);
                    e2 = fmaf(g1.x, wd[c], e2); e3 = fmaf(g1.x, wd[c + 1], e3);
                }
                const uint32_t m = (uint32_t)(mk >> (4 * j)) & 15u;
                e0 = (m & 1u) ? e0 : 0.f; e1 = (m & 2u) ? e1 : 0.f; e2 = (m & 4u) ? e2 : 0.f; e3 = (m & 8u) ? e3 : 0.f;
                colsum2<DET>(bsum, c, e0 + e2, e1 + e3, lane, warp);
                frag_pair(e0, e1, e2, e3, j, ah, al);
                const int i = 4 * (j >> 1) + 2 * (j & 1);
                st_pair(sDA, R0, (uint32_t)j, t, 16384u, ah[i], al[i]);
                st_pair(sDA, R1, (uint32_t)j, t, 16384u, ah[i + 1], al[i + 1]);
            }
            publish();
        }
        // ---------- layer 1: dW1 += dA1^T X; dX = dA1 W1 -> field gradient (interpolate_values_backward, tetrahedra_tracer.cu:231-247) ----------
        dw_half<1, DET>(sDA, sX, 8192u, 0, gw + GW_W1, warp, g, t, part_first);
        dw_half<1, DET>(sDA, sX, 8192u, 1, gw + GW_W1, warp, g, t, part_first);
        {
            const uint32_t w = ring_acquire(more_tiles);  // the last stage of the tile: the next one is the next tile's layer 1
            float dx[32];
            zero(dx);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
                const uint32_t b[4] = {al[4 * kk], al[4 * kk + 1], al[4 * kk + 2], al[4 * kk + 3]};
                wgmma_rs_bf16_n64<1>(dx, a, make_desc(w + kk * 2048u, 16384u, 1024u), kk > 0 ? 1u : 0u);
                wgmma_rs_bf16_n64<1>(dx, b, make_desc(w + kk * 2048u, 16384u, 1024u), 1u);
                wgmma_rs_bf16_n64<1>(dx, a, make_desc(w + 16384u + kk * 2048u, 16384u, 1024u), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            reg_fence(dx);
            float4 q[8];  // this thread's row (row0 for even t, row1 for odd t), columns 8j + 4 (t >> 1) .. +3
#pragma unroll
            for (int j = 0; j < 8; ++j) q[j] = quad_of_row(make_float2(dx[4 * j], dx[4 * j + 1]), make_float2(dx[4 * j + 2], dx[4 * j + 3]), t);
            const uint64_t row = (t & 1u) ? row1 : row0;
            if constexpr (DET) {  // dX rows to HBM; the field gradient is summed per vertex in a fixed order afterwards
                if (row < total_rows) {
                    float4 *dst = reinterpret_cast<float4 *>(p.dx + row * 64 + 4u * (t >> 1));
#pragma unroll
                    for (int j = 0; j < 8; ++j) dst[2 * j] = q[j];
                }
            } else if (row < total_rows) {
                const uint4 v = __ldg(p.vi + row);
                if (v.x != TN_EMPTY) {
                    const float b0 = __ldg(p.bary + 3 * row), b1 = __ldg(p.bary + 3 * row + 1), b2 = __ldg(p.bary + 3 * row + 2);
                    const float w0 = 1.0f - ((b0 + b1) + b2);
                    const uint32_t vs[4] = {v.x, v.y, v.z, v.w};
                    const float ws[4] = {w0, b0, b1, b2};
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float *dst = p.gshadow + (size_t)vs[k] * 64 + 4u * (t >> 1);
#pragma unroll
                        for (int j = 0; j < 8; ++j) red_add_v4(dst + 8 * j, ws[k] * q[j].x, ws[k] * q[j].y, ws[k] * q[j].z, ws[k] * q[j].w);
                    }
                }
            }
        }
        if constexpr (DET) {
            // the partition is complete: its column sums (all written before the barrier of the last publish()) -> its slice, the
            // four warps in order; each thread owns one column and clears it for the next partition
            if (part_last) {
                const uint32_t c = tid;
#pragma unroll 1
                for (uint32_t k = 0; k < 7; ++k) {
                    float *s = sums + k * 128 + c;
                    gw[GW_B1 + k * 128 + c] = ((s[0] + s[896]) + s[1792]) + s[2688];
                    s[0] = 0.f; s[896] = 0.f; s[1792] = 0.f; s[2688] = 0.f;
                }
            }
        }
    }
    if constexpr (DET) return;
    // ---------- flush the column sums ----------
    __syncthreads();
    for (uint32_t c = tid; c < 128; c += BWD_THREADS) {
        atomicAdd(p.gw + GW_B1 + c, sums[c]);
        atomicAdd(p.gw + GW_B2 + c, sums[128 + c]);
        atomicAdd(p.gw + GW_B3 + c, sums[256 + c]);
        atomicAdd(p.gw + GW_WD + c, sums[384 + c]);
        atomicAdd(p.gw + GW_WC + c, sums[512 + c]);
        atomicAdd(p.gw + GW_WC + 128 + c, sums[640 + c]);
        atomicAdd(p.gw + GW_WC + 256 + c, sums[768 + c]);
    }
}

}  // namespace tn
