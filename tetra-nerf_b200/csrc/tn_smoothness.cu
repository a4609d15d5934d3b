// tn_smoothness.cu -- the field's smoothness along the mesh edges (tn_field_smoothness, DESIGN.md §4.15).
//
// S = sum over the unique undirected edges {i, j} of sum_c (f[c,i] - f[c,j])^2, and dS/df[c,i] = 2 sum_{j in N(i)} (f[c,i] - f[c,j]).
// The vertex adjacency is a CSR built once per loaded mesh from the 12 directed vertex pairs of every tetrahedron (a radix sort and a
// unique pass).  One pass over it then gives both: a half-warp per vertex sums its neighbours' differences in CSR order in fp32, and S is
// reduced in double in a shape that depends on V only.  No float atomics anywhere, so every call gives the same bits.
#include <cub/cub.cuh>

#include <cmath>

#include "tn_common.cuh"
#include "tn_edges.cuh"
#include "tn_sort.cuh"

namespace tn {

constexpr uint32_t SM_VERTS = 32;              // vertices per block of k_smoothness, one per half-warp
constexpr uint32_t SM_THREADS = 16 * SM_VERTS;
constexpr unsigned long long NO_PAIR = ~0ull;  // a repeated vertex of a degenerate cell: no edge (a real pair has both ends < 2^32 - 1)

// the 12 directed vertex pairs (a << 32) | b of every tetrahedron; flags[0] |= 1 on a vertex index >= V
__global__ void k_adj_pairs(uint32_t T, uint32_t V, const uint4 *__restrict__ cells, unsigned long long *__restrict__ pairs,
                            uint32_t *__restrict__ flags) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    TN_TET_EDGES;
    const uint4 c = cells[t];
    const uint32_t v[4] = {c.x, c.y, c.z, c.w};
    if (v[0] >= V || v[1] >= V || v[2] >= V || v[3] >= V) atomicOr(flags, 1u);
#pragma unroll
    for (int e = 0; e < 6; ++e) {
        const unsigned long long k = edge_key(v[EA[e]], v[EB[e]]);
        const bool self = v[EA[e]] == v[EB[e]];
        pairs[12 * (size_t)t + 2 * e] = self ? NO_PAIR : k;
        pairs[12 * (size_t)t + 2 * e + 1] = self ? NO_PAIR : (k << 32) | (k >> 32);
    }
}

// CSR from the n sorted distinct pairs P: thread p writes off[v] = p for the rows v that start at p (rows without pairs included), and
// nbr[p]; thread n writes the offsets of the rows after the last pair
__global__ void k_adj_rows(uint32_t n, uint32_t V, const unsigned long long *__restrict__ P, uint32_t *__restrict__ off,
                           uint32_t *__restrict__ nbr) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n) return;
    const uint32_t r = p < n ? (uint32_t)(P[p] >> 32) : V;
    const uint32_t r0 = p > 0 ? (uint32_t)(P[p - 1] >> 32) + 1 : 0;
    for (uint32_t v = r0; v <= r; ++v) off[v] = p;
    if (p < n) nbr[p] = (uint32_t)P[p];
}

__device__ __forceinline__ void acc_diff(const float4 fi, const float4 fj, float4 &g, float &s) {
    const float dx = fi.x - fj.x, dy = fi.y - fj.y, dz = fi.z - fj.z, dw = fi.w - fj.w;
    g.x += dx; g.y += dy; g.z += dz; g.w += dw;
    s = fmaf(dx, dx, s); s = fmaf(dy, dy, s); s = fmaf(dz, dz, s); s = fmaf(dw, dw, s);
}

// One half-warp per vertex i; lane l holds positions 4l .. 4l + 3 of the fragment-ordered shadow row (one 16-byte load per row).  The
// neighbours are summed in CSR order, four rows loaded ahead.  grad (optional) [64,V] = scale * sum_j (f_i - f_j), transposed through
// shared memory so each feature row is stored as 32 consecutive vertices.  part[block] = the block's sum over its vertices of
// sum_j sum_c (f_i - f_j)^2 in double, each vertex's own sum in fp32.
__global__ void __launch_bounds__(SM_THREADS) k_smoothness(uint32_t V, const uint32_t *__restrict__ off, const uint32_t *__restrict__ nbr,
                                                           const float4 *__restrict__ shadow, float scale, float *__restrict__ grad,
                                                           double *__restrict__ part) {
    __shared__ float tile[64][SM_VERTS + 1];
    __shared__ double vsum[SM_VERTS];
    const uint32_t hw = threadIdx.x >> 4, l = threadIdx.x & 15;
    const uint32_t v0 = blockIdx.x * SM_VERTS, i = v0 + hw;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    float s = 0.f;
    if (i < V) {
        const float4 fi = shadow[(size_t)i * 16 + l];
        const uint32_t e = off[i + 1];
        uint32_t k = off[i];
        for (; k + 4 <= e; k += 4) {
            const uint32_t j0 = nbr[k], j1 = nbr[k + 1], j2 = nbr[k + 2], j3 = nbr[k + 3];
            const float4 f0 = shadow[(size_t)j0 * 16 + l], f1 = shadow[(size_t)j1 * 16 + l];
            const float4 f2 = shadow[(size_t)j2 * 16 + l], f3 = shadow[(size_t)j3 * 16 + l];
            acc_diff(fi, f0, g, s); acc_diff(fi, f1, g, s); acc_diff(fi, f2, g, s); acc_diff(fi, f3, g, s);
        }
        for (; k < e; ++k) acc_diff(fi, shadow[(size_t)nbr[k] * 16 + l], g, s);
    }
#pragma unroll
    for (int o = 8; o; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);  // (a butterfly: every lane of the half-warp gets the same sum)
    if (l == 0) vsum[hw] = (double)s;
    if (grad) {
        tile[4 * l][hw] = g.x * scale;
        tile[4 * l + 1][hw] = g.y * scale;
        tile[4 * l + 2][hw] = g.z * scale;
        tile[4 * l + 3][hw] = g.w * scale;
    }
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (grad && v0 + lane < V) {
        for (uint32_t c = warp; c < 64; c += SM_THREADS / 32) grad[(size_t)c * V + v0 + lane] = tile[field_pos(c)][lane];
    }
    if (warp == 0) {
        double t = vsum[lane];
#pragma unroll
        for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xFFFFFFFFu, t, o);
        if (lane == 0) part[blockIdx.x] = t;
    }
}

// *out = S = half the sum of the n block partials (every edge was seen from both ends), in a fixed order: 256 strided running sums, then
// a fixed tree
__global__ void __launch_bounds__(256) k_smoothness_sum(uint32_t n, const double *__restrict__ part, double *__restrict__ out) {
    __shared__ double red[256];
    double t = 0.0;
    for (uint32_t b = threadIdx.x; b < n; b += 256) t += part[b];
    red[threadIdx.x] = t;
    __syncthreads();
    for (uint32_t w = 128; w; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = 0.5 * red[0];
}

// the CSR of the loaded mesh, into the tracer's adj_* buffers; synchronises once (to size the neighbour array)
static int build_adjacency(tn_tracer *h, cudaStream_t s) {
    const uint32_t V = h->mesh.V, T = h->mesh.T;
    const size_t n = 12 * (size_t)T;
    if (n > 0x7FFFFFFFu) return fail(TN_ERR_ARG, "tn_field_smoothness: 12 T must stay below 2^31");
    DevArray<unsigned long long> a, b;  // the pairs and the sort's second buffer, freed on return
    DevArray<uint32_t> ctr;             // [0] flags, [1] distinct pairs
    DevArray<uint8_t> tmp;
    TN_TRY(a.grow(n));
    TN_TRY(b.grow(n));
    TN_TRY(ctr.grow(2));
    cub::DoubleBuffer<unsigned long long> keys(a.p, b.p);
    TN_CUDA(cudaMemsetAsync(ctr.p, 0, 2 * sizeof(uint32_t), s));
    if (T > 0) {
        k_adj_pairs<<<(T + 255) / 256, 256, 0, s>>>(T, V, (const uint4 *)h->mesh.cells, a.p, ctr.p);
        h->launches += 1;
        TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) { return cub::DeviceRadixSort::SortKeys(t, bytes, keys, (int)n, 0, 64, s); }));
        TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
            return cub::DeviceSelect::Unique(t, bytes, keys.Current(), keys.Alternate(), ctr.p + 1, (int)n, s);
        }));
    }
    uint32_t hc[2];
    TN_CUDA(cudaMemcpyAsync(hc, ctr.p, sizeof(hc), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (hc[0] & 1u) return fail(TN_ERR_ARG, "tn_field_smoothness: a cell holds a vertex index >= V");
    const uint32_t np = hc[1] & ~1u;  // the real pairs come in mirrored twos: an odd count is the sentinel, which sorts last
    TN_TRY(h->adj_off.grow((size_t)V + 1));
    TN_TRY(h->adj_nbr.grow(std::max(np, 1u)));
    TN_TRY(h->adj_part.grow(std::max((V + SM_VERTS - 1) / SM_VERTS, 1u)));
    k_adj_rows<<<(np + 1 + 255) / 256, 256, 0, s>>>(np, V, keys.Alternate(), h->adj_off.p, h->adj_nbr.p);
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    h->adj_E = np / 2;
    h->adj_valid = true;
    return TN_OK;  // (a and b are freed here; cudaFree waits for the work queued on them)
}

}  // namespace tn

extern "C" int tn_field_smoothness(tn_tracer *h, float mult, double *d_sum, float *d_grad_field, uint32_t *n_edges, void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (!d_sum) return tn::fail(TN_ERR_ARG, "tn_field_smoothness: null d_sum");
    if (!std::isfinite(mult)) return tn::fail(TN_ERR_ARG, "tn_field_smoothness: mult must be finite");
    if (!h->mesh.nodes.p) return tn::fail(TN_ERR_STATE, "tn_field_smoothness: no tetrahedra loaded");
    const float *shadow = nullptr;
    uint32_t fV = 0;
    if (tn::field_shadow(h, &shadow, &fV) != TN_OK)
        return tn::fail(TN_ERR_STATE, "tn_field_smoothness: no field set (call tn_render_set_field first)");
    const uint32_t V = h->mesh.V;
    if (fV != V)
        return tn::fail(TN_ERR_STATE, "tn_field_smoothness: the field has " + std::to_string(fV) + " vertices, the mesh " + std::to_string(V));
    tn::DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (!h->adj_valid) TN_TRY(tn::build_adjacency(h, s));
    const uint32_t E = h->adj_E;
    // d loss / df for loss = mult S / (E 64): scale * sum_j (f_i - f_j)
    const float scale = E > 0 ? (float)((double)mult * 2.0 / ((double)E * 64.0)) : 0.f;
    const uint32_t blocks = (V + tn::SM_VERTS - 1) / tn::SM_VERTS;
    if (blocks > 0)
        tn::k_smoothness<<<blocks, tn::SM_THREADS, 0, s>>>(V, h->adj_off.p, h->adj_nbr.p, (const float4 *)shadow, scale, d_grad_field,
                                                           h->adj_part.p);
    tn::k_smoothness_sum<<<1, 256, 0, s>>>(blocks, h->adj_part.p, d_sum);
    h->launches += 2;
    TN_CUDA(cudaGetLastError());
    if (n_edges) *n_edges = E;
    return TN_OK;
}
