// tn_refine.cu -- one pass of longest-edge bisection of a tetrahedral mesh (tn_refine_edges, DESIGN.md §4.14).
//
// Candidates propose their longest edge; every tetrahedron votes for its highest-priority proposed edge; an edge is accepted when all
// the tetrahedra around it voted for it (so accepted edges share no tetrahedron and the top proposal is always accepted).  Each accepted
// edge (a, b) gets a new vertex m; each tetrahedron around it keeps its slot with b -> m and appends a child with a -> m.  Every step
// is a pure function of the inputs (integer atomics only, sorts and scans in fixed order), so the output is bitwise reproducible and
// oracle/refine.py restates it bit for bit.
#include <cub/cub.cuh>

#include "tn_common.cuh"
#include "tn_edges.cuh"

namespace tn {

constexpr unsigned long long NO_EDGE = ~0ull;  // no proposal (a real key has a < b <= 0xFFFFFFFE)

// squared length in float64 from the fp32 coordinates, every operation rounded on its own: ((dx^2 + dy^2) + dz^2)
__device__ __forceinline__ double edge_len2(const float *__restrict__ xyz, uint32_t a, uint32_t b) {
    const double dx = __dsub_rn((double)xyz[3 * (size_t)a], (double)xyz[3 * (size_t)b]);
    const double dy = __dsub_rn((double)xyz[3 * (size_t)a + 1], (double)xyz[3 * (size_t)b + 1]);
    const double dz = __dsub_rn((double)xyz[3 * (size_t)a + 2], (double)xyz[3 * (size_t)b + 2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
// priority: the larger squared length, ties to the smaller key
__device__ __forceinline__ bool higher(double l, unsigned long long k, double lo, unsigned long long ko) {
    return l > lo || (l == lo && k < ko);
}
__device__ __forceinline__ uint32_t find_key(const unsigned long long *__restrict__ P, uint32_t n, unsigned long long k) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (P[mid] < k) lo = mid + 1; else hi = mid; }
    return lo < n && P[lo] == k ? lo : TN_EMPTY;
}

// every candidate proposes its longest edge when that is at least min_length long; flags[0] |= 1 on a vertex index >= V
__global__ void k_ref_propose(uint32_t T, uint32_t V, const float *__restrict__ xyz, const uint4 *__restrict__ cells,
                              const uint8_t *__restrict__ cand, double min_len2, unsigned long long *__restrict__ prop, uint32_t *__restrict__ flags) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    TN_TET_EDGES;
    const uint4 c = cells[t];
    const uint32_t v[4] = {c.x, c.y, c.z, c.w};
    if (v[0] >= V || v[1] >= V || v[2] >= V || v[3] >= V) {
        atomicOr(flags, 1u);
        prop[t] = NO_EDGE;
        return;
    }
    unsigned long long out = NO_EDGE;
    if (cand[t]) {
        unsigned long long bk = NO_EDGE;
        double bl = -1.0;
#pragma unroll
        for (int e = 0; e < 6; ++e) {
            const unsigned long long k = edge_key(v[EA[e]], v[EB[e]]);
            const double l = edge_len2(xyz, v[EA[e]], v[EB[e]]);
            if (higher(l, k, bl, bk)) { bl = l; bk = k; }
        }
        if (bl >= min_len2) out = bk;
    }
    prop[t] = out;
}

// every tetrahedron with an edge in P counts itself on each of them and votes for the highest-priority one; voted[t] = its index in P
__global__ void k_ref_vote(uint32_t T, const float *__restrict__ xyz, const uint4 *__restrict__ cells, const unsigned long long *__restrict__ P,
                           const uint32_t *__restrict__ nP, uint32_t *__restrict__ incident, uint32_t *__restrict__ votes, uint32_t *__restrict__ voted) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    TN_TET_EDGES;
    const uint32_t n = *nP;
    const uint4 c = cells[t];
    const uint32_t v[4] = {c.x, c.y, c.z, c.w};
    uint32_t best = TN_EMPTY;
    unsigned long long bk = NO_EDGE;
    double bl = -1.0;
#pragma unroll
    for (int e = 0; e < 6; ++e) {
        const unsigned long long k = edge_key(v[EA[e]], v[EB[e]]);
        const uint32_t i = find_key(P, n, k);
        if (i == TN_EMPTY) continue;
        atomicAdd(incident + i, 1u);
        const double l = edge_len2(xyz, v[EA[e]], v[EB[e]]);
        if (best == TN_EMPTY || higher(l, k, bl, bk)) { best = i; bl = l; bk = k; }
    }
    if (best != TN_EMPTY) atomicAdd(votes + best, 1u);
    voted[t] = best;
}

// accepted[i] = every tetrahedron around edge i voted for it; sort keys for the cap: descending length (a stable sort keeps the
// ascending key order among equal lengths) in [0, 2^63), non-accepted edges behind every accepted one
__global__ void k_ref_accept(uint32_t n, const float *__restrict__ xyz, const unsigned long long *__restrict__ P, const uint32_t *__restrict__ incident,
                             const uint32_t *__restrict__ votes, uint32_t *__restrict__ accepted, unsigned long long *__restrict__ order_key,
                             uint32_t *__restrict__ order_val) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool acc = votes[i] == incident[i];
    accepted[i] = acc;
    const unsigned long long k = P[i];
    const double l = edge_len2(xyz, (uint32_t)(k >> 32), (uint32_t)k);
    // l >= +0: its bits order like its value and leave the top bit clear
    order_key[i] = acc ? (unsigned long long)__double_as_longlong(l) ^ 0x7FFFFFFFFFFFFFFFull : NO_EDGE;
    order_val[i] = i;
}
__global__ void k_ref_cap(uint32_t n, uint32_t keep, const uint32_t *__restrict__ order_val, uint32_t *__restrict__ accepted) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n && j >= keep) accepted[order_val[j]] = 0;  // only accepted edges sort before position n_accepted >= keep
}
// vertex V + vid[i] for each kept edge, in ascending key order; parent_edge rows
__global__ void k_ref_edges(uint32_t n, const unsigned long long *__restrict__ P, const uint32_t *__restrict__ accepted,
                            const uint32_t *__restrict__ vid, uint2 *__restrict__ parent_edge) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !accepted[i]) return;
    parent_edge[vid[i]] = make_uint2((uint32_t)(P[i] >> 32), (uint32_t)P[i]);
}
__global__ void k_ref_split_flags(uint32_t T, const uint32_t *__restrict__ voted, const uint32_t *__restrict__ accepted, uint32_t *__restrict__ split) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t i = voted[t];
    split[t] = i != TN_EMPTY && accepted[i];  // a tetrahedron around a kept edge voted for it
}
__global__ void k_ref_write(uint32_t T, uint32_t V, const uint4 *__restrict__ cells, const unsigned long long *__restrict__ P,
                            const uint32_t *__restrict__ voted, const uint32_t *__restrict__ split, const uint32_t *__restrict__ rank,
                            const uint32_t *__restrict__ vid, uint4 *__restrict__ cells_out, uint32_t *__restrict__ parent_cell) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint4 c = cells[t];
    parent_cell[t] = t;
    if (!split || !split[t]) { cells_out[t] = c; return; }
    const uint32_t i = voted[t];
    const uint32_t a = (uint32_t)(P[i] >> 32), b = (uint32_t)P[i], m = V + vid[i];
    uint32_t s[4] = {c.x, c.y, c.z, c.w}, ch[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (s[j] == b) s[j] = m;
        if (ch[j] == a) ch[j] = m;
    }
    cells_out[t] = make_uint4(s[0], s[1], s[2], s[3]);
    cells_out[T + rank[t]] = make_uint4(ch[0], ch[1], ch[2], ch[3]);
    parent_cell[T + rank[t]] = t;
}

}  // namespace tn

// workspace (each part 256-byte aligned): proposals and their sorted copy u64[T] x 2 (reused as the cap's sort keys), P u64[T],
// seven u32[T] arrays (incident, votes, voted, accepted, vid, split, rank; vid / rank hold the cap's sort values before they are
// computed), 16 counter words and the largest CUB temporary storage of the pass
extern "C" int tn_refine_edges(int device, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, const uint8_t *d_candidates,
                               float min_length, uint32_t max_new_vertices, uint32_t *d_cells_out, uint32_t *d_parent_edge,
                               uint32_t *d_parent_cell, uint32_t *counts3, void *d_workspace, size_t *workspace_bytes, void *stream) {
    if (!workspace_bytes) return tn::fail(TN_ERR_ARG, "tn_refine_edges: null workspace_bytes");
    if ((uint64_t)V + max_new_vertices > 0xFFFFFFFFull)
        return tn::fail(TN_ERR_ARG, "tn_refine_edges: V + max_new_vertices overflows uint32");
    if (T > 0x7FFFFFFFu) return tn::fail(TN_ERR_ARG, "tn_refine_edges: T must stay below 2^31");
    if (!(min_length >= 0.f)) return tn::fail(TN_ERR_ARG, "tn_refine_edges: min_length must be >= 0");
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const int n = (int)T;
    // every CUB algorithm of the pass, written once: with null buffers and all T items for the workspace size, with the workspace's
    // buffers in the runs
    using u64 = unsigned long long;
    auto sort_keys = [&](void *t, size_t &bytes, const u64 *in, u64 *out) { return cub::DeviceRadixSort::SortKeys(t, bytes, in, out, n, 0, 64, s); };
    auto unique = [&](void *t, size_t &bytes, u64 *in, u64 *out, uint32_t *count) { return cub::DeviceSelect::Unique(t, bytes, in, out, count, n, s); };
    auto scan = [&](void *t, size_t &bytes, uint32_t *in, uint32_t *out, int m) { return cub::DeviceScan::ExclusiveSum(t, bytes, in, out, m, s); };
    auto sort_pairs = [&](void *t, size_t &bytes, const u64 *kin, u64 *kout, const uint32_t *vin, uint32_t *vout, int m) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kin, kout, vin, vout, m, 0, 64, s);
    };
    auto sum = [&](void *t, size_t &bytes, uint32_t *in, uint32_t *out, int m) { return cub::DeviceReduce::Sum(t, bytes, in, out, m, s); };
    size_t c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0;
    TN_CUDA(sort_keys(nullptr, c0, nullptr, nullptr));
    TN_CUDA(unique(nullptr, c1, nullptr, nullptr, nullptr));
    TN_CUDA(scan(nullptr, c2, nullptr, nullptr, n));
    TN_CUDA(sort_pairs(nullptr, c3, nullptr, nullptr, nullptr, nullptr, n));
    TN_CUDA(sum(nullptr, c4, nullptr, nullptr, n));
    size_t cub_bytes = std::max(std::max(std::max(c0, c1), std::max(c2, c3)), c4);
    const size_t kb = al(sizeof(unsigned long long) * (size_t)T), ub = al(sizeof(uint32_t) * (size_t)T), cb = al(16 * sizeof(uint32_t));
    const size_t need = 3 * kb + 7 * ub + cb + al(cub_bytes);
    if (!d_workspace) { *workspace_bytes = need; return TN_OK; }
    if (*workspace_bytes < need) return tn::fail(TN_ERR_ARG, "tn_refine_edges: workspace too small");
    if (!counts3) return tn::fail(TN_ERR_ARG, "tn_refine_edges: null counts3");
    counts3[0] = counts3[1] = counts3[2] = 0;
    if (T == 0) return TN_OK;
    uint8_t *ws = (uint8_t *)d_workspace;
    unsigned long long *prop = (unsigned long long *)ws, *sorted = (unsigned long long *)(ws + kb), *P = (unsigned long long *)(ws + 2 * kb);
    uint32_t *u = (uint32_t *)(ws + 3 * kb);
    uint32_t *incident = u, *votes = (uint32_t *)((uint8_t *)u + ub), *voted = (uint32_t *)((uint8_t *)u + 2 * ub),
             *accepted = (uint32_t *)((uint8_t *)u + 3 * ub), *vid = (uint32_t *)((uint8_t *)u + 4 * ub), *split = (uint32_t *)((uint8_t *)u + 5 * ub),
             *rank = (uint32_t *)((uint8_t *)u + 6 * ub);
    uint32_t *ctr = (uint32_t *)(ws + 3 * kb + 7 * ub);  // [0] flags, [1] unique count, [2] accepted count, [3] last vid, [4] last rank
    void *tmp = ws + 3 * kb + 7 * ub + cb;
    const uint32_t blocks = (T + 255) / 256;
    const double ml = (double)min_length;
    TN_CUDA(cudaMemsetAsync(ctr, 0, 16 * sizeof(uint32_t), s));
    tn::k_ref_propose<<<blocks, 256, 0, s>>>(T, V, d_xyz, (const uint4 *)d_cells, d_candidates, ml * ml, prop, ctr);
    TN_CUDA(sort_keys(tmp, cub_bytes, prop, sorted));
    TN_CUDA(unique(tmp, cub_bytes, sorted, P, ctr + 1));
    uint32_t h[2];
    TN_CUDA(cudaMemcpyAsync(h, ctr, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    unsigned long long last = 0;
    TN_CUDA(cudaMemcpyAsync(&last, sorted + (T - 1), sizeof(last), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (h[0] & 1u) return tn::fail(TN_ERR_ARG, "tn_refine_edges: a cell holds a vertex index >= V");
    const uint32_t nP = h[1] - (last == tn::NO_EDGE ? 1u : 0u);  // the sentinel sorts last
    counts3[0] = nP;
    if (nP == 0) {  // nothing proposed: the input mesh unchanged
        tn::k_ref_write<<<blocks, 256, 0, s>>>(T, V, (const uint4 *)d_cells, P, voted, nullptr, rank, vid, (uint4 *)d_cells_out, d_parent_cell);
        TN_CUDA(cudaGetLastError());
        TN_CUDA(cudaStreamSynchronize(s));
        return TN_OK;
    }
    TN_CUDA(cudaMemcpyAsync(ctr + 1, &nP, sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    TN_CUDA(cudaMemsetAsync(incident, 0, 2 * ub, s));  // incident and votes are adjacent
    tn::k_ref_vote<<<blocks, 256, 0, s>>>(T, d_xyz, (const uint4 *)d_cells, P, ctr + 1, incident, votes, voted);
    const uint32_t pblocks = (nP + 255) / 256;
    tn::k_ref_accept<<<pblocks, 256, 0, s>>>(nP, d_xyz, P, incident, votes, accepted, prop, vid);
    TN_CUDA(sum(tmp, cub_bytes, accepted, ctr + 2, (int)nP));
    uint32_t nacc = 0;
    TN_CUDA(cudaMemcpyAsync(&nacc, ctr + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (nacc > max_new_vertices) {  // keep the highest-priority ones
        TN_CUDA(sort_pairs(tmp, cub_bytes, prop, sorted, vid, rank, (int)nP));
        tn::k_ref_cap<<<pblocks, 256, 0, s>>>(nP, max_new_vertices, rank, accepted);
        nacc = max_new_vertices;
    }
    counts3[1] = nacc;
    TN_CUDA(scan(tmp, cub_bytes, accepted, vid, (int)nP));
    tn::k_ref_edges<<<pblocks, 256, 0, s>>>(nP, P, accepted, vid, (uint2 *)d_parent_edge);
    tn::k_ref_split_flags<<<blocks, 256, 0, s>>>(T, voted, accepted, split);
    TN_CUDA(scan(tmp, cub_bytes, split, rank, n));
    tn::k_ref_write<<<blocks, 256, 0, s>>>(T, V, (const uint4 *)d_cells, P, voted, split, rank, vid, (uint4 *)d_cells_out, d_parent_cell);
    TN_CUDA(cudaGetLastError());
    uint32_t hs[2];
    TN_CUDA(cudaMemcpyAsync(hs, rank + (T - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaMemcpyAsync(hs + 1, split + (T - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    counts3[2] = hs[0] + hs[1];
    return TN_OK;
}
