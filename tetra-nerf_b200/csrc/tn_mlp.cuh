// tn_mlp.cuh -- the fused interpolate -> MLP kernel on warpgroup MMA (wgmma, sm_90a).
//
// Replaces, for one pass over n_active*S samples, the chain
//   interpolate_values (src/tetrahedra_tracer.cu:195-221)  ->  mlp_base (3x Linear+ReLU, model.py:433-438)
//   -> DensityFieldHead (Linear+Softplus, :455) [-> mlp_head (Linear+ReLU, :447-452) -> RGBFieldHead
//   (Linear+Sigmoid, :454)]                                               (call sites model.py:569-621)
// which the reference runs as ~10 torch kernels with [R*S,128] fp32 activations round-tripping HBM.
//
// One persistent CTA per SM with MLP_WGS warpgroups.  The whole weight image (224 KB: four layers, bf16 or fp16 hi/lo halves)
// is staged into shared memory once per CTA by TMA bulk copies and stays resident.  Each warpgroup then works through 64-sample
// tiles on its own, entirely in registers:
//   gather    the four vertex rows of each of its two samples per thread are read from the [V,64] field shadow (stored in fragment
//             order, so a thread reads its 16 features of a row as four 16-byte loads), interpolated with
//             the reference's FMA order and converted straight into the layer-0 A fragments (see tn_tc.cuh for the layout);
//   layers    every Linear is a chain of wgmma m64n128k16 with A from registers and B = the resident weight block; the epilogue
//             (bias + ReLU) turns the fp32 accumulator into the next layer's A fragments in place -- activations never touch
//             shared or global memory;
//   heads     the density / colour dot products are formed in the epilogue of the layer that feeds them and reduced across the
//             four threads that share a row.
// While one warpgroup waits for its gather loads the others keep the tensor cores busy (three warpgroups: 168 registers per thread
// at most, no spills; on an H100 the fine pass took 0.57 ms with three against 0.74 ms with two, bench.py's 4096-ray workload).
// Products: two operand precisions, template parameter PREC:
//   PREC 3 "bf16x3": a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo, bf16 halves, fp32 accumulation (tests/test_gpu_mlp.py bounds the
//           error at 2e-5 relative) -- the reference computes in fp32 and the parity bar is 1e-4 absolute on colour/density, which
//           single-pass bf16/tf32 cannot hold.  Training forward.
//   PREC 2 "f16w2":  a*(w_hi + w_lo) with ONE fp16 activation value and fp16 hi/lo weights, 2 MMAs per K step instead of 3
//           (~2^-12 relative per activation: 2.6e-5 absolute on density / colour of unit scale, tools/split_accuracy.py) -- the
//           inference default.
#pragma once
#include "tn_common.cuh"
#include "tn_tc.cuh"

namespace tn {

#ifndef TN_MLP_WGS
#define TN_MLP_WGS 3
#endif
constexpr uint32_t MLP_WGS = TN_MLP_WGS;                   // warpgroups per CTA (each owns one 64-sample tile at a time)
constexpr uint32_t MLP_THREADS = 128 * MLP_WGS;
constexpr uint32_t MLP_TILE = 64;                          // samples per tile
constexpr uint32_t MLP_W_BYTES = 32768 + 3 * 65536;        // weight image: L1 32K | L2 64K | L3 64K | L4 (base part) 64K
constexpr uint32_t MLP_W_COARSE = 32768 + 2 * 65536;       // the coarse pass stops after L3
// shared memory of one pass: its own weight bytes, then wd[128] wc[3][128] bd bc[3], the weight barrier and the per-warpgroup
// tile slots [MLP_WGS][2].  The coarse pass asks for only what it uses (162 KB), which leaves its SM ~92 KB of L1 for the
// gathered field rows instead of the fine pass's ~28 KB.
__host__ __device__ constexpr uint32_t mlp_off_head(bool fine) { return fine ? MLP_W_BYTES : MLP_W_COARSE; }
__host__ __device__ constexpr uint32_t mlp_off_bars(bool fine) { return mlp_off_head(fine) + 520 * 4; }
__host__ __device__ constexpr uint32_t mlp_smem_bytes(bool fine) { return mlp_off_bars(fine) + 8 + 8 * MLP_WGS; }
static_assert(mlp_smem_bytes(true) <= 232448, "k_mlp shared memory exceeds 227 KB");
__host__ __device__ constexpr uint32_t mlp_off_layer(int l) { return l == 0 ? 0u : 32768u + 65536u * (uint32_t)(l - 1); }

struct MlpParams {
    const uint32_t *n_active;  // device scalar: number of non-empty rays
    uint32_t S;                // samples per ray in this pass
    const uint4 *vi;           // [n_active*S] matched vertex ids (E = unmatched)
    const float *bary;         // [n_active*S,3]
    const float *fshadow;      // [V,64] field, one row per vertex in fragment order (field_pos)
    const uint8_t *wimg;       // weight image: L1 | L2 | L3 | L4(base part), see tn_mlp_pack.cuh
    const float *bias;         // b1,b2,b3 [3][128]
    const float *head;         // wd[128], wc[3][128], bd, bc[3]
    const float *dirbias;      // FINE: [n_active,128]  = b4 + W4[:, :27] . enc(dir)
    float *out;                // COARSE: density [rows] ; FINE: (sigma,r,g,b) [rows,4]
    uint32_t *tile_ctr;        // device counter (zeroed before the launch): dynamic tile scheduler
    // MAP (occupancy culling, DESIGN §4.12): the tiles cover the compact rows 0 .. *n_rows - 1, and compact row c is sample row
    // rowmap[c] of vi / bary / out / the per-ray bias (ascending, so a ray's rows stay contiguous and in slot order)
    const uint32_t *rowmap;
    const uint32_t *n_rows;
};

constexpr uint32_t MLP_NO_TILE = 0xFFFFFFFFu;  // sentinel: the scheduler has run dry

__device__ __forceinline__ float softplus_f(float x) { return x > 20.0f ? x : log1pf(expf(x)); }  // torch Softplus(beta=1, threshold=20)
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// 16-byte read-only load that does not allocate in L1 (the gathered field rows stream through; L1 is left to the biases)
__device__ __forceinline__ float4 ldg_stream(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
// 16-byte read-only load that allocates in L1
__device__ __forceinline__ float4 ldg_l1(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// the 16 features of one field-shadow row that thread t of a fragment row needs, as four 16-byte loads: q[kk] holds column pairs
// 2kk (features 16kk + 2t, +1) and 2kk + 1 (16kk + 8 + 2t, +1) -- one load per k-step, since the shadow is in fragment order (field_pos)
template <bool ALLOC_L1>
__device__ __forceinline__ void load_field_quads(const float *__restrict__ row, uint32_t t, float4 (&q)[4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const float4 *p = reinterpret_cast<const float4 *>(row + field_pos(16u * kk + 2u * t));
        q[kk] = ALLOC_L1 ? ldg_l1(p) : ldg_stream(p);
    }
}
// column pair c (features 8c + 2t, +1) of the quads load_field_quads returned
__device__ __forceinline__ float2 field_pair(const float4 (&q)[4], int c) {
    const float4 v = q[c >> 1];
    return (c & 1) ? make_float2(v.z, v.w) : make_float2(v.x, v.y);
}

// named barrier of one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(uint32_t wg) { asm volatile("bar.sync %0, 128;" ::"r"(1u + wg) : "memory"); }

// packs a pair (low half first) in the operand precision of PREC: bf16 hi [+ lo] (3) or one fp16 value (2)
template <int PREC>
__device__ __forceinline__ void to_operand(float e0, float e1, uint32_t &hi, uint32_t &lo) {
    if (PREC == 2) hi = tc::pack2_f16(e0, e1);
    else tc::split_pack2(e0, e1, hi, lo);
}

// the sample indices of the thread's two rows (row0, row0 + 8): matched vertex ids and barycentric weights.  A row at or past
// total_rows reads as unmatched.
struct GatherRows {
    uint4 v[2];
    float b[2][3];
};
__device__ __forceinline__ GatherRows load_gather_rows(const uint4 *__restrict__ vi, const float *__restrict__ bary, uint64_t row0, uint64_t total_rows) {
    GatherRows r;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const uint64_t row = row0 + 8u * rr;
        r.v[rr] = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
        r.b[rr][0] = r.b[rr][1] = r.b[rr][2] = 0.f;
        if (row < total_rows) {
            r.v[rr] = __ldg(vi + row);
            r.b[rr][0] = __ldg(bary + 3 * row); r.b[rr][1] = __ldg(bary + 3 * row + 1); r.b[rr][2] = __ldg(bary + 3 * row + 2);
        }
    }
    return r;
}
// the same through a compact-row map: compact rows at or past total_rows read as unmatched
__device__ __forceinline__ GatherRows load_gather_rows_mapped(const uint4 *__restrict__ vi, const float *__restrict__ bary, const uint32_t *__restrict__ rowmap,
                                                          uint64_t row0, uint64_t total_rows) {
    GatherRows r;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const uint64_t row = row0 + 8u * rr;
        r.v[rr] = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
        r.b[rr][0] = r.b[rr][1] = r.b[rr][2] = 0.f;
        if (row < total_rows) {
            const size_t s = __ldg(rowmap + row);
            r.v[rr] = __ldg(vi + s);
            r.b[rr][0] = __ldg(bary + 3 * s); r.b[rr][1] = __ldg(bary + 3 * s + 1); r.b[rr][2] = __ldg(bary + 3 * s + 2);
        }
    }
    return r;
}
// brings the 128-byte line of p into L1 (no register is written, nothing waits for it)
__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// the lines load_gather_rows will read for the same rows
__device__ __forceinline__ void prefetch_gather_rows(const uint4 *vi, const float *bary, uint64_t row0, uint64_t total_rows) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const uint64_t row = row0 + 8u * rr;
        if (row < total_rows) {
            prefetch_l1(vi + row);
            prefetch_l1(bary + 3 * row);
        }
    }
}

// the interpolated features of the thread's two rows, as the layer-0 A fragments (K = 64: 4 k-steps x 4 registers).
// tetrahedra_tracer.cu:203-220: v1*b0, + v2*b1, + v3*b2, + v0*w0 (fused multiply-adds), per feature.
// All 32 field loads of the two rows (16 bytes each: one per row, vertex and k-step, see field_pos) are issued before the first one
// is consumed, so a thread has its whole gather in flight at once instead of one L2 round trip per k-step.  The loads are
// unconditional: an unmatched row reads vertex 0's features and its result is replaced by 0 (a branch around the loads would keep
// the compiler from hoisting them over the FMAs).
// ALLOC_L1: the loads allocate in L1 (k_mlp).  Samples next to each other along a ray lie in the same or adjacent tetrahedra, so
// most of a row's four vertices are among its neighbours' and the repeats of a field row, within a warp and across the warpgroups
// of an SM, are served from L1 instead of L2.  Otherwise they stream past L1 (k_mlp_bwd, k_mlp_normals).
template <int PREC, bool ALLOC_L1 = false>
__device__ __forceinline__ void gather_rows(const GatherRows &r, const float *__restrict__ fshadow, uint32_t t, uint32_t (&xh)[16], uint32_t (&xl)[16]) {
    float4 a[2][4][4];  // [row][vertex][k-step]
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const uint4 v = r.v[rr].x != TN_EMPTY ? r.v[rr] : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) load_field_quads<ALLOC_L1>(fshadow + (size_t)vs[k] * 64, t, a[rr][k]);
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const bool m = r.v[rr].x != TN_EMPTY;
        const float b0 = r.b[rr][0], b1 = r.b[rr][1], b2 = r.b[rr][2];
        const float w0 = __fsub_rn(1.0f, __fadd_rn(__fadd_rn(b0, b1), b2));
#pragma unroll
        for (int c = 0; c < 8; ++c) {  // column pair 8c + 2t, +1  ->  k-step c / 2, register 2 (c & 1) + rr
            const float2 a0 = field_pair(a[rr][0], c), a1 = field_pair(a[rr][1], c), a2 = field_pair(a[rr][2], c), a3 = field_pair(a[rr][3], c);
            float2 o;
            o.x = __fmaf_rn(b0, a1.x, 0.f); o.y = __fmaf_rn(b0, a1.y, 0.f);
            o.x = __fmaf_rn(b1, a2.x, o.x); o.y = __fmaf_rn(b1, a2.y, o.y);
            o.x = __fmaf_rn(b2, a3.x, o.x); o.y = __fmaf_rn(b2, a3.y, o.y);
            o.x = __fmaf_rn(w0, a0.x, o.x); o.y = __fmaf_rn(w0, a0.y, o.y);
            if (!m) o = make_float2(0.f, 0.f);
            const int i = 4 * (c >> 1) + 2 * (c & 1) + rr;
            to_operand<PREC>(o.x, o.y, xh[i], xl[i]);
        }
    }
}

// one Linear with a 128-wide output: d = A W^T over K = 16 * KSTEPS, A in registers (hi / lo fragments), W from the resident image
// (per 64-wide K block: hi block, lo block 16 KB further)
template <int PREC, int KSTEPS>
__device__ __forceinline__ void layer_mma(float (&d)[64], const uint32_t (&ah)[4 * KSTEPS], const uint32_t (&al)[4 * KSTEPS], uint32_t w) {
    using namespace tc;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) {
        const uint32_t wb = w + (uint32_t)(kk >> 2) * 32768u + (uint32_t)(kk & 3) * 32u;
        const uint32_t a[4] = {ah[4 * kk], ah[4 * kk + 1], ah[4 * kk + 2], ah[4 * kk + 3]};
        if (PREC == 2) {
            wgmma_rs_f16_n128<0>(d, a, make_desc(wb), kk > 0 ? 1u : 0u);
            wgmma_rs_f16_n128<0>(d, a, make_desc(wb + 16384u), 1u);
        } else {
            const uint32_t b[4] = {al[4 * kk], al[4 * kk + 1], al[4 * kk + 2], al[4 * kk + 3]};
            wgmma_rs_bf16_n128<0>(d, a, make_desc(wb), kk > 0 ? 1u : 0u);
            wgmma_rs_bf16_n128<0>(d, b, make_desc(wb), 1u);
            wgmma_rs_bf16_n128<0>(d, a, make_desc(wb + 16384u), 1u);
        }
    }
    wgmma_commit();
    wgmma_wait0();
    reg_fence(d);
}

// MAP: the tiles run over the compact rows of p.rowmap (occupancy culling); otherwise over every row
template <bool FINE, int PREC, bool MAP = false>
__global__ void __launch_bounds__(MLP_THREADS, 1) k_mlp(const MlpParams p) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t tn_mlp_smem[];
    uint8_t *smem = tn_mlp_smem;
    const float *head_s = reinterpret_cast<const float *>(smem + mlp_off_head(FINE));
    uint64_t *w_bar = reinterpret_cast<uint64_t *>(smem + mlp_off_bars(FINE));
    volatile uint32_t *slots = reinterpret_cast<volatile uint32_t *>(smem + mlp_off_bars(FINE) + 8);  // [wg][2] tile of the next / this round

    constexpr int L = FINE ? 4 : 3;
    constexpr uint32_t WBYTES = FINE ? MLP_W_BYTES : MLP_W_COARSE;
    const uint32_t wg = threadIdx.x >> 7, tid = threadIdx.x & 127u;
    const uint32_t warp = tid >> 5, lane = threadIdx.x & 31u, g = lane >> 2, t = lane & 3u;
    const uint32_t n_active = *p.n_active;
    const uint64_t total_rows = MAP ? (uint64_t)*p.n_rows : (uint64_t)n_active * p.S;
    const uint32_t ntiles = (uint32_t)((total_rows + MLP_TILE - 1) / MLP_TILE);
    if (blockIdx.x * MLP_WGS >= ntiles) return;  // (uniform over the CTA)
    auto sample_row = [&](uint64_t row) -> uint64_t { return MAP ? (uint64_t)__ldg(p.rowmap + row) : row; };

    if (threadIdx.x == 0) {
        mbar_init(w_bar, 1);
        fence_barrier_init();
    }
    for (uint32_t i = threadIdx.x; i < 516; i += MLP_THREADS) const_cast<float *>(head_s)[i] = p.head[i];
    // tile scheduler: the tile of round n sits in slots[2 wg + (n & 1)] from round n - 1 on, so a warpgroup knows its next tile for
    // the whole of the current round.  The first tile of each warpgroup is static, the following ones come from the global counter.
    auto draw = [&]() {
        const uint32_t nx = gridDim.x * MLP_WGS + atomicAdd(p.tile_ctr, 1u);
        return nx < ntiles ? nx : MLP_NO_TILE;
    };
    if (tid == 0) {
        const uint32_t first = blockIdx.x * MLP_WGS + wg;
        slots[2 * wg] = first < ntiles ? first : MLP_NO_TILE;
        slots[2 * wg + 1] = draw();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(w_bar, WBYTES);
        for (uint32_t off = 0; off < WBYTES; off += 16384) tma_bulk_g2s(smem + off, p.wimg + off, 16384, w_bar);
    }
    const uint32_t wsm = smem_u32(smem);
    const float *wd = head_s, *wc = head_s + 128;
    bool weights_ready = false;
    const uint32_t lrow = warp * 16u + g;  // the thread's first row within a tile
    uint32_t tile = slots[2 * wg];

#pragma unroll 1
    for (uint32_t n = 0;; ++n) {
        wg_sync(wg);
        if (tile == MLP_NO_TILE) break;
        const uint32_t next = slots[2 * wg + ((n + 1u) & 1u)];
        // draw the tile of round n + 2 into this round's slot (every thread read it in round n - 1, before the barrier above)
        if (tid == 0) slots[2 * wg + (n & 1u)] = draw();
        const uint64_t row0 = (uint64_t)tile * MLP_TILE + lrow, row1 = row0 + 8u;
        const float *db0 = nullptr, *db1 = nullptr;  // FINE: the per-ray bias rows of layer 4

        uint32_t ah[32], al[32];
        {
            uint32_t xh[16], xl[16];
            if constexpr (MAP) gather_rows<PREC, true>(load_gather_rows_mapped(p.vi, p.bary, p.rowmap, row0, total_rows), p.fshadow, t, xh, xl);
            else gather_rows<PREC, true>(load_gather_rows(p.vi, p.bary, row0, total_rows), p.fshadow, t, xh, xl);
            // Into L1 while this tile's MMAs run: the next tile's indices, so its gather starts with the field loads, and (FINE) this
            // tile's bias rows of layer 4, read right after that layer's MMA wait.  Prefetches hold no registers: keeping the 14
            // index words of the next tile in registers instead spills k_mlp<true, 3> at its 168-register limit.
            // (MAP: the next tile's map entries, whose loads are the first step of its gather)
            if constexpr (MAP) { if (next != MLP_NO_TILE && lrow == warp * 16u) prefetch_l1(p.rowmap + (uint64_t)next * MLP_TILE + lrow); }
            else if (next != MLP_NO_TILE) prefetch_gather_rows(p.vi, p.bary, (uint64_t)next * MLP_TILE + lrow, total_rows);
            if (FINE) {
                db0 = p.dirbias + (size_t)((uint32_t)sample_row(min(row0, total_rows - 1)) / p.S) * 128;
                db1 = p.dirbias + (size_t)((uint32_t)sample_row(min(row1, total_rows - 1)) / p.S) * 128;
                prefetch_l1(db0 + 32 * t);  // the four threads of a row cover its four 128-byte lines
                prefetch_l1(db1 + 32 * t);
            }
            if (!weights_ready) { mbar_wait(w_bar, 0); weights_ready = true; }
            float d[64];
            layer_mma<PREC, 4>(d, xh, xl, wsm + mlp_off_layer(0));
            // epilogue of layer 1 -> A fragments of layer 2
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float2 b = __ldg(reinterpret_cast<const float2 *>(p.bias + 8 * j + 2 * t));
                const int i = 4 * (j >> 1) + 2 * (j & 1);
                to_operand<PREC>(fmaxf(d[4 * j] + b.x, 0.f), fmaxf(d[4 * j + 1] + b.y, 0.f), ah[i], al[i]);
                to_operand<PREC>(fmaxf(d[4 * j + 2] + b.x, 0.f), fmaxf(d[4 * j + 3] + b.y, 0.f), ah[i + 1], al[i + 1]);
            }
        }
        float dens0 = 0.f, dens1 = 0.f;
        // hidden layers 2 and 3 (the third one also feeds the density head)
#pragma unroll
        for (int l = 1; l < 3; ++l) {
            float d[64];
            layer_mma<PREC, 8>(d, ah, al, wsm + mlp_off_layer(l));
            const float *bias = p.bias + 128 * l;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * (int)t;
                const float2 b = __ldg(reinterpret_cast<const float2 *>(bias + c));
                const float x0 = fmaxf(d[4 * j] + b.x, 0.f), x1 = fmaxf(d[4 * j + 1] + b.y, 0.f);
                const float y0 = fmaxf(d[4 * j + 2] + b.x, 0.f), y1 = fmaxf(d[4 * j + 3] + b.y, 0.f);
                if (l == 2) {
                    dens0 = fmaf(x0, wd[c], dens0); dens0 = fmaf(x1, wd[c + 1], dens0);
                    dens1 = fmaf(y0, wd[c], dens1); dens1 = fmaf(y1, wd[c + 1], dens1);
                }
                if (l < L - 1) {
                    const int i = 4 * (j >> 1) + 2 * (j & 1);
                    to_operand<PREC>(x0, x1, ah[i], al[i]);
                    to_operand<PREC>(y0, y1, ah[i + 1], al[i + 1]);
                }
            }
        }
        float col0[3] = {0.f, 0.f, 0.f}, col1[3] = {0.f, 0.f, 0.f};
        if (FINE) {
            // layer 4: per-ray bias (b4 + the direction part of W4), ReLU, colour-head partial dot products
            float d[64];
            layer_mma<PREC, 8>(d, ah, al, wsm + mlp_off_layer(3));
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * (int)t;
                const float2 b0 = __ldg(reinterpret_cast<const float2 *>(db0 + c)), b1 = __ldg(reinterpret_cast<const float2 *>(db1 + c));
                const float x0 = fmaxf(d[4 * j] + b0.x, 0.f), x1 = fmaxf(d[4 * j + 1] + b0.y, 0.f);
                const float y0 = fmaxf(d[4 * j + 2] + b1.x, 0.f), y1 = fmaxf(d[4 * j + 3] + b1.y, 0.f);
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const float *w = wc + 128 * ch;
                    col0[ch] = fmaf(x1, w[c + 1], fmaf(x0, w[c], col0[ch]));
                    col1[ch] = fmaf(y1, w[c + 1], fmaf(y0, w[c], col1[ch]));
                }
            }
        }
        // heads: the four threads of a row (t = 0..3) hold disjoint column subsets
#pragma unroll
        for (int s = 1; s <= 2; s <<= 1) {
            dens0 += __shfl_xor_sync(0xffffffffu, dens0, s);
            dens1 += __shfl_xor_sync(0xffffffffu, dens1, s);
            if (FINE) {
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    col0[ch] += __shfl_xor_sync(0xffffffffu, col0[ch], s);
                    col1[ch] += __shfl_xor_sync(0xffffffffu, col1[ch], s);
                }
            }
        }
        if (t < 2) {
            const uint64_t row = t == 0 ? row0 : row1;
            const float dn = t == 0 ? dens0 : dens1;
            if (row < total_rows) {
                const uint64_t orow = sample_row(row);
                const float sigma = softplus_f(dn + head_s[512]);
                if (FINE) {
                    const float c0 = t == 0 ? col0[0] : col1[0], c1 = t == 0 ? col0[1] : col1[1], c2 = t == 0 ? col0[2] : col1[2];
                    reinterpret_cast<float4 *>(p.out)[orow] =
                        make_float4(sigma, sigmoid_f(c0 + head_s[513]), sigmoid_f(c1 + head_s[514]), sigmoid_f(c2 + head_s[515]));
                } else {
                    p.out[orow] = sigma;
                }
            }
        }
        tile = next;
    }
    if (!weights_ready) mbar_wait(w_bar, 0);  // a warpgroup without a tile still lets the weight copy land before the CTA exits
}

// launches one k_mlp pass with the shared memory of that pass
template <bool FINE, int PREC, bool MAP = false>
inline int launch_mlp(const MlpParams &p, uint32_t grid, cudaStream_t s) {
    auto k = k_mlp<FINE, PREC, MAP>;
    TN_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mlp_smem_bytes(FINE)));
    k<<<grid, MLP_THREADS, mlp_smem_bytes(FINE), s>>>(p);
    return TN_OK;
}

}  // namespace tn
