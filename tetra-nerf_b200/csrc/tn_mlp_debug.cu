// tn_mlp_debug.cu -- one-tile bf16x3 GEMMs on wgmma used by tests to validate, in isolation, the pieces the fused MLP kernels rely
// on: the weight image (hi/lo bf16, 128-byte swizzle) staged by TMA bulk copy, A fragments in registers (thread layout of
// tn_tc.cuh), and the K-major / MN-major shared-memory descriptors of the backward kernel.
#include "tn_common.cuh"
#include "tn_mlp_pack.cuh"
#include "tn_tc.cuh"

namespace tn {
using namespace tc;

// out[128,128] = A[128,K] * W[128,K]^T: two warpgroups of 64 rows, A split into bf16 hi/lo register fragments, W from the forward
// weight image (per 64-wide K block: hi 16 KB, lo 16 KB)
__global__ void __launch_bounds__(256, 1) k_debug_gemm(const float *__restrict__ A, const uint8_t *__restrict__ wimg, uint32_t K,
                                                        float *__restrict__ out) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + 65536);
    const uint32_t wbytes = (K / 64) * 32768u;
    const uint32_t wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3u, lane = threadIdx.x & 31u, g = lane >> 2, t = lane & 3u;
    if (threadIdx.x == 0) { mbar_init(bar, 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(bar, wbytes);
        for (uint32_t off = 0; off < wbytes; off += 16384) tma_bulk_g2s(smem + off, wimg + off, 16384, bar);
    }
    const uint32_t r0 = wg * 64u + warp * 16u + g;
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    mbar_wait(bar, 0);
    const uint32_t ws = smem_u32(smem);
    for (uint32_t kk = 0; kk < K / 16; ++kk) {
        uint32_t ah[4], al[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t row = r0 + 8u * (i & 1), col = kk * 16u + 8u * (i >> 1) + 2u * t;
            split_pack2(A[row * K + col], A[row * K + col + 1], ah[i], al[i]);
        }
        const uint32_t wb = ws + (kk >> 2) * 32768u + (kk & 3u) * 32u;
        wgmma_fence();
        wgmma_rs_bf16_n128<0>(d, ah, make_desc(wb), 1u);
        wgmma_rs_bf16_n128<0>(d, al, make_desc(wb), 1u);
        wgmma_rs_bf16_n128<0>(d, ah, make_desc(wb + 16384u), 1u);
        wgmma_commit();
        wgmma_wait0();
    }
    reg_fence(d);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint32_t c = 8u * j + 2u * t;
        out[r0 * 128 + c] = d[4 * j]; out[r0 * 128 + c + 1] = d[4 * j + 1];
        out[(r0 + 8) * 128 + c] = d[4 * j + 2]; out[(r0 + 8) * 128 + c + 1] = d[4 * j + 3];
    }
}

}  // namespace tn

// test hook (not part of the reference surface): d_A f32[128,K], d_W f32[128,K] (nn.Linear layout), K in {64,128}
extern "C" int tn_debug_gemm_bf16x3(int device, const float *d_A, const float *d_W, uint32_t K, float *d_out, void *stream) {
    if (K != 64 && K != 128) return tn::fail(TN_ERR_ARG, "tn_debug_gemm_bf16x3: K must be 64 or 128");
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    tn::DevArray<uint8_t> img;
    TN_TRY(img.grow((K / 64) * 32768));
    tn::launch_pack_weights(d_W, K, 0, K, img.p, s);
    const int smem = 65536 + 128;
    TN_CUDA(cudaFuncSetAttribute(tn::k_debug_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    tn::k_debug_gemm<<<1, 256, smem, s>>>(d_A, img.p, K, d_out);
    TN_CUDA(cudaGetLastError());
    TN_CUDA(cudaStreamSynchronize(s));
    return TN_OK;
}

// ---- the three operand forms of the fused MLP backward, from shared memory: ------------------------------------------------------
// mode 0: out = P Q^T (A, B K-major)   mode 1: out = P Q (A K-major, B MN-major)   mode 2: out = P^T Q (A, B MN-major)
// P, Q f32[128,128] are stored as bf16 hi/lo [row][64-column block] images (block stride 32 KB, lo 16 KB after hi); two
// warpgroups own output rows 0..63 / 64..127.
namespace tn {
template <int MODE, int N>
__device__ __forceinline__ void gemm_modes_body(uint32_t pa, uint32_t qa, uint32_t wg, uint32_t lbo, uint32_t sbo, uint32_t kstep, float (&d)[N / 2]) {
    constexpr int TA = MODE == 2 ? 1 : 0, TB = MODE >= 1 ? 1 : 0;
    wgmma_fence();
    for (int term = 0; term < 3; ++term) {  // (P_hi,Q_hi) (P_lo,Q_hi) (P_hi,Q_lo)
        const uint32_t po = term == 1 ? 16384u : 0u, qo = term == 2 ? 16384u : 0u;
        for (uint32_t j = 0; j < 8; ++j) {  // 8 k-steps of 16
            // K-major: k-step j lives in column block j/4 at byte 32 (j%4) of every row; MN-major: rows 16j.. of every block
            const uint64_t da = TA ? make_desc(pa + po + wg * 32768u + j * kstep, lbo, sbo)
                                   : make_desc(pa + po + (j >> 2) * 32768u + wg * 8192u + (j & 3u) * 32u);
            const uint64_t db = TB ? make_desc(qa + qo + j * kstep, lbo, sbo) : make_desc(qa + qo + (j >> 2) * 32768u + (j & 3u) * 32u);
            if constexpr (N == 128) wgmma_ss_bf16_n128<TA, TB>(d, da, db, 1u);
            else wgmma_ss_bf16_n64<TA, TB>(d, da, db, 1u);
        }
    }
    wgmma_commit();
    wgmma_wait0();
    reg_fence(d);
}

template <int N>
__global__ void __launch_bounds__(256, 1) k_debug_gemm2(const float *__restrict__ P, const float *__restrict__ Q, int mode, uint32_t lbo, uint32_t sbo,
                                                         uint32_t kstep, float *__restrict__ out) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *p_s = smem, *q_s = smem + 65536;
    const uint32_t wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3u, lane = threadIdx.x & 31u, g = lane >> 2, t = lane & 3u;
    if (threadIdx.x < 128) {
        const uint32_t row = threadIdx.x;
        for (uint32_t k = 0; k < 128; k += 2) {
            uint32_t hi, lo;
            const uint32_t off = (k >> 6) * 32768u + sw128_offset(row, k & 63u);
            split_pack2(P[row * 128 + k], P[row * 128 + k + 1], hi, lo);
            *reinterpret_cast<uint32_t *>(p_s + off) = hi;
            *reinterpret_cast<uint32_t *>(p_s + off + 16384u) = lo;
            split_pack2(Q[row * 128 + k], Q[row * 128 + k + 1], hi, lo);
            *reinterpret_cast<uint32_t *>(q_s + off) = hi;
            *reinterpret_cast<uint32_t *>(q_s + off + 16384u) = lo;
        }
        fence_proxy_async();
    }
    __syncthreads();
    const uint32_t pa = smem_u32(p_s), qa = smem_u32(q_s);
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    if (mode == 0) gemm_modes_body<0, N>(pa, qa, wg, lbo, sbo, kstep, d);
    else if (mode == 1) gemm_modes_body<1, N>(pa, qa, wg, lbo, sbo, kstep, d);
    else gemm_modes_body<2, N>(pa, qa, wg, lbo, sbo, kstep, d);
    const uint32_t r0 = wg * 64u + warp * 16u + g;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
        const uint32_t c = 8u * j + 2u * t;
        out[r0 * 128 + c] = d[4 * j]; out[r0 * 128 + c + 1] = d[4 * j + 1];
        out[(r0 + 8) * 128 + c] = d[4 * j + 2]; out[(r0 + 8) * 128 + c + 1] = d[4 * j + 3];
    }
}
}  // namespace tn

// test hook: d_P, d_Q f32[128,128], d_out f32[128,128] (first N columns written); lbo / sbo / kstep in bytes describe the
// MN-major operands (the test uses lbo = 32768 (next 64-column block), sbo = 1024 (next 8 rows), kstep = 2048 (16 rows))
extern "C" int tn_debug_gemm_modes(int device, int mode, uint32_t N, uint32_t lbo, uint32_t sbo, uint32_t kstep, const float *d_P,
                                   const float *d_Q, float *d_out, void *stream) {
    if (mode < 0 || mode > 2 || (N != 64 && N != 128)) return tn::fail(TN_ERR_ARG, "tn_debug_gemm_modes: mode in 0..2, N in {64,128}");
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    const int smem = 131072;
    auto k = N == 128 ? tn::k_debug_gemm2<128> : tn::k_debug_gemm2<64>;
    TN_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k<<<1, 256, smem, s>>>(d_P, d_Q, mode, lbo, sbo, kstep, d_out);
    TN_CUDA(cudaGetLastError());
    TN_CUDA(cudaStreamSynchronize(s));
    return TN_OK;
}
