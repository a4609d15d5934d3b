// tn_coarsen.cu -- one pass of empty-space vertex removal by edge collapse (tn_coarsen_vertices, DESIGN.md §4.18).
//
// A non-hull vertex a whose tetrahedra are all flagged empty proposes to collapse into its nearest neighbour b whose cones keep the
// certified orientation of every tetrahedron they replace; every tetrahedron votes for the highest-priority proposing vertex among its
// four; a proposal is accepted when its whole star voted for it (so accepted vertices share no tetrahedron, and the top proposal is always
// accepted).  The star cells of an accepted a that hold b are removed, the others take b in a's slot, and cells and vertices are compacted
// stably.  Every step is a pure function of the inputs (integer atomics only, sorts and scans in fixed order), so the output is bitwise
// reproducible and oracle/coarsen.py restates it bit for bit.
#include <cub/cub.cuh>

#include "tn_common.cuh"
#include "tn_predicates.cuh"
#include "tn_sort.cuh"

namespace tn {

// squared length in float64 from the fp32 coordinates, every operation rounded on its own (tn_refine.cu's edge length)
__device__ __forceinline__ double co_len2(const float *__restrict__ xyz, uint32_t a, uint32_t b) {
    const double dx = __dsub_rn((double)xyz[3 * (size_t)a], (double)xyz[3 * (size_t)b]);
    const double dy = __dsub_rn((double)xyz[3 * (size_t)a + 1], (double)xyz[3 * (size_t)b + 1]);
    const double dz = __dsub_rn((double)xyz[3 * (size_t)a + 2], (double)xyz[3 * (size_t)b + 2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
// (l, k) comes before (lo, ko): the smaller squared length, ties to the smaller vertex id
__device__ __forceinline__ bool before(double l, uint32_t k, double lo, uint32_t ko) { return l < lo || (l == lo && k < ko); }
__device__ __forceinline__ bool has(const uint4 c, uint32_t v) { return c.x == v || c.y == v || c.z == v || c.w == v; }
__device__ __forceinline__ uint4 with(uint4 c, uint32_t from, uint32_t to) {
    if (c.x == from) c.x = to;
    if (c.y == from) c.y = to;
    if (c.z == from) c.z = to;
    if (c.w == from) c.w = to;
    return c;
}
__device__ __forceinline__ int cell_sign(const float *__restrict__ xyz, const uint4 c) {
    int s = 0;
    orient3d_sign(xyz, c.x, c.y, c.z, c.w, s);
    return s;
}

// the (vertex, cell) pairs: the keys are the cells array itself, the values the cell of each slot; flags[0] |= 1 on a vertex index >= V
__global__ void k_co_pairs(uint32_t n4, uint32_t V, const uint32_t *__restrict__ cells, uint32_t *__restrict__ cell_of, uint32_t *__restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    if (cells[i] >= V) atomicOr(flags, 1u);
    cell_of[i] = i >> 2;
}
// CSR row offsets of the vertex -> cells incidence: off[v] = the first sorted pair of vertex v
__global__ void k_co_offsets(uint32_t V, uint32_t n4, const uint32_t *__restrict__ skeys, uint32_t *__restrict__ off) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v <= V) off[v] = v == V ? n4 : lower_bound_u32(skeys, n4, v);
}

// one thread per vertex a: its collapse target (TN_EMPTY: no proposal) and that edge's squared length
__global__ void k_co_propose(uint32_t V, const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint8_t *__restrict__ empty,
                             const uint32_t *__restrict__ off, const uint32_t *__restrict__ star, uint32_t *__restrict__ target,
                             double *__restrict__ prio, uint32_t *__restrict__ n_proposed) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    target[a] = TN_EMPTY;
    const uint32_t beg = off[a], end = off[a + 1];
    if (beg == end) return;
    for (uint32_t i = beg; i < end; ++i)  // every tetrahedron of the star empty, with a certified orientation
        if (!empty[star[i]] || cell_sign(xyz, cells[star[i]]) == 0) return;
    // a hull vertex: some face (a, x, y) of its star has no second owner (the owners of a face through a all lie in a's star)
    for (uint32_t i = beg; i < end; ++i) {
        const uint4 c = cells[star[i]];
        const uint32_t v[4] = {c.x, c.y, c.z, c.w};
        for (int p = 0; p < 4; ++p) {
            if (v[p] == a) continue;
            for (int q = p + 1; q < 4; ++q) {
                if (v[q] == a) continue;
                bool shared = false;
                for (uint32_t j = beg; j < end && !shared; ++j)
                    if (j != i) { const uint4 d = cells[star[j]]; shared = has(d, v[p]) && has(d, v[q]); }
                if (!shared) return;
            }
        }
    }
    // the neighbours in ascending (squared length, id); the first whose cones keep every orientation is the target
    double lc = -1.0;
    uint32_t bc = 0;
    for (;;) {
        double lb = 0.0;
        uint32_t b = TN_EMPTY;
        for (uint32_t i = beg; i < end; ++i) {
            const uint4 c = cells[star[i]];
            const uint32_t v[4] = {c.x, c.y, c.z, c.w};
            for (int p = 0; p < 4; ++p) {
                if (v[p] == a) continue;
                const double l = co_len2(xyz, a, v[p]);
                if (before(lc, bc, l, v[p]) && (b == TN_EMPTY || before(l, v[p], lb, b))) { lb = l; b = v[p]; }
            }
        }
        if (b == TN_EMPTY) return;  // no valid neighbour: no proposal
        bool ok = true;
        for (uint32_t i = beg; i < end && ok; ++i) {
            const uint4 c = cells[star[i]];
            if (has(c, b)) continue;  // removed by the collapse
            ok = cell_sign(xyz, with(c, a, b)) == cell_sign(xyz, c);
        }
        if (ok) {
            target[a] = b;
            prio[a] = lb;
            atomicAdd(n_proposed, 1u);
            return;
        }
        lc = lb;
        bc = b;
    }
}

// every tetrahedron with a proposing vertex votes for the highest-priority one of its four
__global__ void k_co_vote(uint32_t T, const uint4 *__restrict__ cells, const uint32_t *__restrict__ target, const double *__restrict__ prio,
                          uint32_t *__restrict__ votes) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint4 c = cells[t];
    const uint32_t v[4] = {c.x, c.y, c.z, c.w};
    uint32_t best = TN_EMPTY;
    double bl = 0.0;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        if (target[v[p]] == TN_EMPTY) continue;
        const double l = prio[v[p]];
        if (best == TN_EMPTY || before(l, v[p], bl, best)) { best = v[p]; bl = l; }
    }
    if (best != TN_EMPTY) atomicAdd(votes + best, 1u);
}

// accepted[a] = a proposed and its whole star voted for it; sort keys for the cap: ascending length (a stable sort keeps ascending ids
// among equal lengths) in [0, 2^63), the others behind every accepted vertex
__global__ void k_co_accept(uint32_t V, const uint32_t *__restrict__ off, const uint32_t *__restrict__ target, const double *__restrict__ prio,
                            const uint32_t *__restrict__ votes, uint32_t *__restrict__ accepted, unsigned long long *__restrict__ order_key,
                            uint32_t *__restrict__ order_val) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    const bool acc = target[a] != TN_EMPTY && votes[a] == off[a + 1] - off[a];
    accepted[a] = acc;
    order_key[a] = acc ? (unsigned long long)__double_as_longlong(prio[a]) : ~0ull;  // l >= +0: its bits order like its value
    order_val[a] = a;
}
__global__ void k_co_cap(uint32_t V, uint32_t keep, const uint32_t *__restrict__ order_val, uint32_t *__restrict__ accepted) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < V && j >= keep) accepted[order_val[j]] = 0;  // only accepted vertices sort before position n_accepted >= keep
}
__global__ void k_co_keep_vertices(uint32_t V, const uint32_t *__restrict__ accepted, uint32_t *__restrict__ keepv) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < V) keepv[v] = !accepted[v];
}
// a tetrahedron with a removed vertex a (at most one: accepted vertices share no tetrahedron) is removed if it holds a's target
__global__ void k_co_keep_cells(uint32_t T, const uint4 *__restrict__ cells, const uint32_t *__restrict__ accepted, const uint32_t *__restrict__ target,
                                uint32_t *__restrict__ keepc) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint4 c = cells[t];
    const uint32_t v[4] = {c.x, c.y, c.z, c.w};
    uint32_t k = 1;
#pragma unroll
    for (int p = 0; p < 4; ++p)
        if (accepted[v[p]] && has(c, target[v[p]])) k = 0;
    keepc[t] = k;
}
__global__ void k_co_write(uint32_t T, const uint4 *__restrict__ cells, const uint32_t *__restrict__ accepted, const uint32_t *__restrict__ target,
                           const uint32_t *__restrict__ keepc, const uint32_t *__restrict__ rank, const uint32_t *__restrict__ newid,
                           uint4 *__restrict__ cells_out, uint32_t *__restrict__ parent_cell) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T || !keepc[t]) return;
    const uint4 c = cells[t];
    uint32_t v[4] = {c.x, c.y, c.z, c.w};
    uint32_t a = TN_EMPTY;
#pragma unroll
    for (int p = 0; p < 4; ++p)
        if (accepted[v[p]]) a = v[p];
#pragma unroll
    for (int p = 0; p < 4; ++p) v[p] = newid[v[p] == a ? target[a] : v[p]];
    cells_out[rank[t]] = make_uint4(v[0], v[1], v[2], v[3]);
    parent_cell[rank[t]] = t;
}
__global__ void k_co_kept(uint32_t V, const uint32_t *__restrict__ keepv, const uint32_t *__restrict__ newid, uint32_t *__restrict__ kept) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < V && (!keepv || keepv[v])) kept[keepv ? newid[v] : v] = v;  // no masks: every vertex kept
}

}  // namespace tn

// workspace (each part 256-byte aligned): the (vertex, cell) pairs u32[4T] x 3 (cell of each slot, sorted vertices, sorted cells), the
// CSR offsets u32[V+1], the proposals' lengths f64[V] and the cap's sort keys u64[V] x 2, seven u32[V] arrays (target, votes, accepted,
// kept, new id, the cap's sort values x 2), two u32[T] arrays (kept, rank), 16 counter words and the largest CUB temporary storage
extern "C" int tn_coarsen_vertices(int device, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, const uint8_t *d_empty,
                                   uint32_t max_removed, uint32_t *d_cells_out, uint32_t *d_kept_vertex, uint32_t *d_parent_cell,
                                   uint32_t *counts3, void *d_workspace, size_t *workspace_bytes, void *stream) {
    if (!workspace_bytes) return tn::fail(TN_ERR_ARG, "tn_coarsen_vertices: null workspace_bytes");
    if (T > 0x1FFFFFFFu) return tn::fail(TN_ERR_ARG, "tn_coarsen_vertices: T must stay below 2^29");
    if (V > 0x7FFFFFFFu) return tn::fail(TN_ERR_ARG, "tn_coarsen_vertices: V must stay below 2^31");
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const int n4 = (int)(4 * T), nv = (int)V, nt = (int)T;
    const int end_bit = tn::radix_end_bit(V > 0 ? V - 1 : 0);
    // every CUB algorithm of the pass, written once: with null buffers for the workspace size, with the workspace's buffers in the runs
    using u64 = unsigned long long;
    auto sort_star = [&](void *t, size_t &bytes, const uint32_t *kin, uint32_t *kout, const uint32_t *vin, uint32_t *vout) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kin, kout, vin, vout, n4, 0, end_bit, s);
    };
    auto scan = [&](void *t, size_t &bytes, uint32_t *in, uint32_t *out, int m) { return cub::DeviceScan::ExclusiveSum(t, bytes, in, out, m, s); };
    auto sum = [&](void *t, size_t &bytes, uint32_t *in, uint32_t *out) { return cub::DeviceReduce::Sum(t, bytes, in, out, nv, s); };
    auto sort_cap = [&](void *t, size_t &bytes, const u64 *kin, u64 *kout, const uint32_t *vin, uint32_t *vout) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kin, kout, vin, vout, nv, 0, 64, s);
    };
    size_t c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0;
    TN_CUDA(sort_star(nullptr, c0, nullptr, nullptr, nullptr, nullptr));
    TN_CUDA(scan(nullptr, c1, nullptr, nullptr, nv));
    TN_CUDA(scan(nullptr, c2, nullptr, nullptr, nt));
    TN_CUDA(sum(nullptr, c3, nullptr, nullptr));
    TN_CUDA(sort_cap(nullptr, c4, nullptr, nullptr, nullptr, nullptr));
    size_t cub_bytes = std::max(std::max(std::max(c0, c1), std::max(c2, c3)), c4);
    const size_t pb = al(sizeof(uint32_t) * 4 * (size_t)T), ob = al(sizeof(uint32_t) * ((size_t)V + 1)), db = al(sizeof(double) * (size_t)V),
                 vb = al(sizeof(uint32_t) * (size_t)V), tb = al(sizeof(uint32_t) * (size_t)T), cb = al(16 * sizeof(uint32_t));
    const size_t need = 3 * pb + ob + 3 * db + 7 * vb + 2 * tb + cb + al(cub_bytes);
    if (!d_workspace) { *workspace_bytes = need; return TN_OK; }
    if (*workspace_bytes < need) return tn::fail(TN_ERR_ARG, "tn_coarsen_vertices: workspace too small");
    if (!counts3) return tn::fail(TN_ERR_ARG, "tn_coarsen_vertices: null counts3");
    counts3[0] = counts3[1] = counts3[2] = 0;
    if (T == 0) {  // no cell: nothing to remove, every vertex kept
        if (V) tn::k_co_kept<<<(V + 255) / 256, 256, 0, s>>>(V, nullptr, nullptr, d_kept_vertex);
        TN_CUDA(cudaGetLastError());
        TN_CUDA(cudaStreamSynchronize(s));
        return TN_OK;
    }
    uint8_t *p = (uint8_t *)d_workspace;
    auto take = [&](size_t b) { uint8_t *q = p; p += b; return q; };
    uint32_t *cell_of = (uint32_t *)take(pb), *skeys = (uint32_t *)take(pb), *star = (uint32_t *)take(pb), *off = (uint32_t *)take(ob);
    double *prio = (double *)take(db);
    u64 *okey = (u64 *)take(db), *okey_sorted = (u64 *)take(db);
    uint32_t *target = (uint32_t *)take(vb), *votes = (uint32_t *)take(vb), *accepted = (uint32_t *)take(vb), *keepv = (uint32_t *)take(vb),
             *newid = (uint32_t *)take(vb), *oval = (uint32_t *)take(vb), *oval_sorted = (uint32_t *)take(vb);
    uint32_t *keepc = (uint32_t *)take(tb), *rank = (uint32_t *)take(tb);
    uint32_t *ctr = (uint32_t *)take(cb);  // [0] flags, [1] proposals, [2] accepted
    void *tmp = take(al(cub_bytes));
    const uint32_t vblocks = (V + 255) / 256, tblocks = (T + 255) / 256;
    TN_CUDA(cudaMemsetAsync(ctr, 0, 16 * sizeof(uint32_t), s));
    tn::k_co_pairs<<<(4 * T + 255) / 256, 256, 0, s>>>(4 * T, V, d_cells, cell_of, ctr);
    uint32_t flags = 0;
    TN_CUDA(cudaMemcpyAsync(&flags, ctr, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (flags & 1u) return tn::fail(TN_ERR_ARG, "tn_coarsen_vertices: a cell holds a vertex index >= V");
    TN_CUDA(sort_star(tmp, cub_bytes, d_cells, skeys, cell_of, star));
    tn::k_co_offsets<<<(V + 1 + 255) / 256, 256, 0, s>>>(V, 4 * T, skeys, off);
    const uint4 *cells = (const uint4 *)d_cells;
    tn::k_co_propose<<<(V + 127) / 128, 128, 0, s>>>(V, d_xyz, cells, d_empty, off, star, target, prio, ctr + 1);
    TN_CUDA(cudaMemsetAsync(votes, 0, vb, s));
    tn::k_co_vote<<<tblocks, 256, 0, s>>>(T, cells, target, prio, votes);
    tn::k_co_accept<<<vblocks, 256, 0, s>>>(V, off, target, prio, votes, accepted, okey, oval);
    TN_CUDA(sum(tmp, cub_bytes, accepted, ctr + 2));
    uint32_t h[2];
    TN_CUDA(cudaMemcpyAsync(h, ctr + 1, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    counts3[0] = h[0];
    uint32_t nacc = h[1];
    if (nacc > max_removed) {  // keep the highest-priority ones
        TN_CUDA(sort_cap(tmp, cub_bytes, okey, okey_sorted, oval, oval_sorted));
        tn::k_co_cap<<<vblocks, 256, 0, s>>>(V, max_removed, oval_sorted, accepted);
        nacc = max_removed;
    }
    counts3[1] = nacc;
    tn::k_co_keep_vertices<<<vblocks, 256, 0, s>>>(V, accepted, keepv);
    tn::k_co_keep_cells<<<tblocks, 256, 0, s>>>(T, cells, accepted, target, keepc);
    TN_CUDA(scan(tmp, cub_bytes, keepv, newid, nv));
    TN_CUDA(scan(tmp, cub_bytes, keepc, rank, nt));
    tn::k_co_write<<<tblocks, 256, 0, s>>>(T, cells, accepted, target, keepc, rank, newid, (uint4 *)d_cells_out, d_parent_cell);
    tn::k_co_kept<<<vblocks, 256, 0, s>>>(V, keepv, newid, d_kept_vertex);
    TN_CUDA(cudaGetLastError());
    uint32_t hs[2];
    TN_CUDA(cudaMemcpyAsync(hs, rank + (T - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaMemcpyAsync(hs + 1, keepc + (T - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    counts3[2] = T - (hs[0] + hs[1]);
    return TN_OK;
}
