// tn_flip.cu -- one pass of Delaunay flips (tn_flip_delaunay, DESIGN.md §4.19).
//
// Every interior face whose opposite vertex e lies strictly inside the circumsphere of its other owner (certified insphere_sign) and whose
// two or three cells can be re-triangulated with certified orientations proposes a 2-3 or a 3-2 flip; every cell votes for the
// highest-priority proposal touching it (the priority is the face's position in the sorted face table); a proposal is accepted when all of
// its cells voted for it (so accepted flips share no cell, and the top proposal is always accepted).  The flips write their new cells into
// their old slots, a 2-3 flip's third cell is appended, a 3-2 flip's third slot is removed, and the cells are compacted stably.  Every
// step is a pure function of the inputs (integer atomics only, sorts and scans in fixed order), so the output is bitwise reproducible and
// oracle/flip.py restates it bit for bit.
#include <cub/cub.cuh>

#include "tn_common.cuh"
#include "tn_predicates.cuh"
#include "tn_sort.cuh"

namespace tn {

__device__ __forceinline__ uint32_t fl_at(const uint4 c, int k) { return k == 0 ? c.x : k == 1 ? c.y : k == 2 ? c.z : c.w; }
__device__ __forceinline__ void fl_sort3(uint32_t &a, uint32_t &b, uint32_t &c) {
    if (a > b) { const uint32_t t = a; a = b; b = t; }
    if (b > c) { const uint32_t t = b; b = c; c = t; }
    if (a > b) { const uint32_t t = a; a = b; b = t; }
}
// the ascending vertex triple of face slot i: the face of cell i >> 2 opposite its vertex i & 3
__device__ __forceinline__ void fl_face(const uint4 *__restrict__ cells, uint32_t i, uint32_t &a, uint32_t &b, uint32_t &c) {
    const uint4 t = cells[i >> 2];
    const int k = i & 3;
    a = fl_at(t, k == 0 ? 1 : 0);
    b = fl_at(t, k <= 1 ? 2 : 1);
    c = fl_at(t, k <= 2 ? 3 : 2);
    fl_sort3(a, b, c);
}
__device__ __forceinline__ int fl_o3(const float *__restrict__ xyz, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    int s = 0;
    orient3d_sign(xyz, a, b, c, d, s);
    return s;
}
__device__ __forceinline__ int fl_cell_sign(const float *__restrict__ xyz, const uint4 c) { return fl_o3(xyz, c.x, c.y, c.z, c.w); }

// the sorted face table: keys (a << 32 | b, c) ascending at positions [0, n4), slots in ascending order within a face
struct FaceTable {
    const unsigned long long *ab;
    const uint32_t *c, *slot;
    uint32_t n4;
    __device__ __forceinline__ bool same(uint32_t p, uint32_t q) const { return ab[p] == ab[q] && c[p] == c[q]; }
    // the first position of the face (x, y, w), n4 if it is not a face of the mesh
    __device__ uint32_t find(uint32_t x, uint32_t y, uint32_t w) const {
        fl_sort3(x, y, w);
        const unsigned long long kab = ((unsigned long long)x << 32) | y;
        uint32_t lo = 0, hi = n4;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (ab[mid] < kab || (ab[mid] == kab && c[mid] < w)) lo = mid + 1; else hi = mid;
        }
        return lo < n4 && ab[lo] == kab && c[lo] == w ? lo : n4;
    }
    // the owner other than t of the interior face (x, y, w), TN_EMPTY if the face is absent or a hull face
    __device__ uint32_t other_owner(uint32_t x, uint32_t y, uint32_t w, uint32_t t) const {
        const uint32_t lo = find(x, y, w);
        if (lo + 1 >= n4 || !same(lo, lo + 1)) return TN_EMPTY;
        const uint32_t u = slot[lo] >> 2, v = slot[lo + 1] >> 2;
        return u == t ? v : u;
    }
};

// what the interior face at sorted position p proposes (kind 0: nothing, 2: a 2-3 flip, 3: a 3-2 flip), its cells t0 < t1 (and t2) and
// its new cells in their written order; `illegal`: the face is certified non-Delaunay
struct Flip {
    int kind;
    uint32_t t0, t1, t2;
    uint4 n[3];
};
__device__ __forceinline__ uint4 fl_cell(uint32_t a, uint32_t b, uint32_t c, uint32_t d, int s, int ref) {
    return s == ref ? make_uint4(a, b, c, d) : make_uint4(a, b, d, c);
}
__device__ void fl_propose(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const FaceTable &ft, uint32_t p, Flip &f,
                           bool &illegal) {
    f.kind = 0;
    illegal = false;
    const uint32_t i0 = ft.slot[p], i1 = ft.slot[p + 1];
    f.t0 = i0 >> 2;
    f.t1 = i1 >> 2;
    f.t2 = TN_EMPTY;
    const uint4 c0 = cells[f.t0], c1 = cells[f.t1];
    const uint32_t d = fl_at(c0, i0 & 3), e = fl_at(c1, i1 & 3);
    const uint32_t a = (uint32_t)(ft.ab[p] >> 32), b = (uint32_t)ft.ab[p], c = ft.c[p];
    const int s0 = fl_cell_sign(xyz, c0);
    if (s0 == 0 || fl_cell_sign(xyz, c1) == 0) return;
    int ins = 0;
    insphere_sign(xyz, c0.x, c0.y, c0.z, c0.w, e, ins);
    if (ins == 0 || ins != s0) return;
    illegal = true;
    const int sd = fl_o3(xyz, a, b, c, d), se = fl_o3(xyz, a, b, c, e);
    if (sd == 0 || se == 0 || sd != -se) return;
    const int o[3] = {fl_o3(xyz, a, b, d, e), fl_o3(xyz, b, c, d, e), fl_o3(xyz, c, a, d, e)};
    if (o[0] == 0 || o[1] == 0 || o[2] == 0) return;
    const int nopp = (o[0] != se) + (o[1] != se) + (o[2] != se);
    if (nopp == 0) {  // d-e crosses the open triangle abc; none of the new interior faces may exist already (next to a flat cell)
        if (ft.find(a, d, e) < ft.n4 || ft.find(b, d, e) < ft.n4 || ft.find(c, d, e) < ft.n4) return;
        f.kind = 2;
        f.n[0] = fl_cell(a, b, d, e, o[0], s0);
        f.n[1] = fl_cell(b, c, d, e, o[1], s0);
        f.n[2] = fl_cell(c, a, d, e, o[2], s0);
        return;
    }
    if (nopp != 1) return;
    // the reflex edge (x, y) and the face's third vertex z
    const int j = o[0] != se ? 0 : (o[1] != se ? 1 : 2);
    const uint32_t x = j == 0 ? a : (j == 1 ? b : c), y = j == 0 ? b : (j == 1 ? c : a), z = j == 0 ? c : (j == 1 ? a : b);
    const uint32_t ta = ft.other_owner(x, y, d, f.t0), tb = ft.other_owner(x, y, e, f.t1);
    if (ta == TN_EMPTY || ta != tb) return;
    const int s2 = fl_cell_sign(xyz, cells[ta]);
    if (s2 == 0) return;
    uint32_t pp = z, qq = d, rr = e;
    fl_sort3(pp, qq, rr);
    const int oa = fl_o3(xyz, pp, qq, rr, x), ob = fl_o3(xyz, pp, qq, rr, y);
    if (oa == 0 || ob == 0 || oa != -ob) return;
    const int l0 = fl_o3(xyz, x, y, pp, qq), l1 = fl_o3(xyz, x, y, qq, rr), l2 = fl_o3(xyz, x, y, rr, pp);
    if (l0 == 0 || l0 != l1 || l1 != l2) return;
    if (ft.find(pp, qq, rr) < ft.n4) return;  // the new interior face exists already
    const int ref = ta < f.t0 ? s2 : s0;  // the lowest-slot cell's sign (t0 < t1 always)
    f.kind = 3;
    f.t2 = ta;
    f.n[0] = fl_cell(pp, qq, rr, x, oa, ref);
    f.n[1] = fl_cell(pp, qq, rr, y, ob, ref);
}
// the interior face starting at sorted position p, or none
__device__ __forceinline__ bool fl_interior(const FaceTable &ft, uint32_t p) {
    return (p == 0 || !ft.same(p - 1, p)) && p + 1 < ft.n4 && ft.same(p, p + 1);
}

// slot i: val = i, key = its face's largest vertex; flags[0] |= 1 on a vertex index >= V
__global__ void k_fl_slots(uint32_t n4, uint32_t V, const uint4 *__restrict__ cells, uint32_t *__restrict__ key_c, uint32_t *__restrict__ val,
                           uint32_t *__restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    if (((const uint32_t *)cells)[i] >= V) atomicOr(flags, 1u);
    uint32_t a, b, c;
    fl_face(cells, i, a, b, c);
    key_c[i] = c;
    val[i] = i;
}
__global__ void k_fl_keys_ab(uint32_t n4, const uint4 *__restrict__ cells, const uint32_t *__restrict__ val, unsigned long long *__restrict__ kab) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n4) return;
    uint32_t a, b, c;
    fl_face(cells, val[p], a, b, c);
    kab[p] = ((unsigned long long)a << 32) | b;
}
// kc[p] = the largest vertex of the face at position p; flags[0] |= 2 on a face with more than two owners
__global__ void k_fl_runs(uint32_t n4, const uint4 *__restrict__ cells, const unsigned long long *__restrict__ kab, const uint32_t *__restrict__ val,
                          uint32_t *__restrict__ kc, uint32_t *__restrict__ flags) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n4) return;
    uint32_t a, b, c;
    fl_face(cells, val[p], a, b, c);
    kc[p] = c;
    if (p + 2 < n4 && kab[p + 2] == kab[p]) {
        uint32_t a2, b2, c2;
        fl_face(cells, val[p + 2], a2, b2, c2);
        if (c2 == c) atomicOr(flags, 2u);
    }
}

__global__ void k_fl_propose(const float *__restrict__ xyz, const uint4 *__restrict__ cells, FaceTable ft, uint32_t *__restrict__ kind,
                             uint32_t *__restrict__ t2, uint32_t *__restrict__ ctr) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= ft.n4) return;
    kind[p] = 0;
    if (!fl_interior(ft, p)) return;
    Flip f;
    bool illegal;
    fl_propose(xyz, cells, ft, p, f, illegal);
    if (illegal) atomicAdd(ctr + 1, 1u);
    if (!f.kind) return;
    kind[p] = f.kind;
    t2[p] = f.t2;
    atomicAdd(ctr + 2, 1u);
}
// every cell keeps the smallest position of a proposal touching it
__global__ void k_fl_vote(FaceTable ft, const uint32_t *__restrict__ kind, const uint32_t *__restrict__ t2, uint32_t *__restrict__ vote) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= ft.n4 || !kind[p]) return;
    atomicMin(vote + (ft.slot[p] >> 2), p);
    atomicMin(vote + (ft.slot[p + 1] >> 2), p);
    if (kind[p] == 3) atomicMin(vote + t2[p], p);
}
__global__ void k_fl_accept(FaceTable ft, const uint32_t *__restrict__ kind, const uint32_t *__restrict__ t2, const uint32_t *__restrict__ vote,
                            uint32_t *__restrict__ acc) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= ft.n4) return;
    acc[p] = kind[p] && vote[ft.slot[p] >> 2] == p && vote[ft.slot[p + 1] >> 2] == p && (kind[p] != 3 || vote[t2[p]] == p);
}
// the kept flips (accepted and among the first max_flips accepted in priority order): their cells are marked, a 3-2 flip's highest slot
// removed; ctr[3] / ctr[4] count the 2-3 / 3-2 flips
__global__ void k_fl_mark(FaceTable ft, uint32_t max_flips, const uint32_t *__restrict__ kind, const uint32_t *__restrict__ t2,
                          const uint32_t *__restrict__ acc, const uint32_t *__restrict__ arank, uint32_t *__restrict__ k23,
                          uint32_t *__restrict__ touched, uint32_t *__restrict__ removed, uint32_t *__restrict__ ctr) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= ft.n4) return;
    const bool kept = acc[p] && arank[p] < max_flips;
    k23[p] = kept && kind[p] == 2;
    if (!kept) return;
    const uint32_t t0 = ft.slot[p] >> 2, t1 = ft.slot[p + 1] >> 2;
    touched[t0] = touched[t1] = 1;
    if (kind[p] == 3) {
        touched[t2[p]] = 1;
        removed[max(t1, t2[p])] = 1;  // t0 < t1
        atomicAdd(ctr + 4, 1u);
    } else {
        atomicAdd(ctr + 3, 1u);
    }
}
// a cell no kept flip touches: copied to its compacted slot with sources (t, E, E)
__global__ void k_fl_copy(uint32_t T, const uint4 *__restrict__ cells, const uint32_t *__restrict__ touched, const uint32_t *__restrict__ rpre,
                          uint4 *__restrict__ out, uint32_t *__restrict__ src) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T || touched[t]) return;
    const uint32_t o = t - rpre[t];
    out[o] = cells[t];
    src[3 * (size_t)o] = t;
    src[3 * (size_t)o + 1] = src[3 * (size_t)o + 2] = TN_EMPTY;
}
// a kept flip writes its new cells into its lowest two slots (compacted) and, for a 2-3 flip, the appended slot T - n32 + its rank
__global__ void k_fl_apply(const float *__restrict__ xyz, const uint4 *__restrict__ cells, FaceTable ft, uint32_t T, uint32_t max_flips,
                           const uint32_t *__restrict__ acc, const uint32_t *__restrict__ arank, const uint32_t *__restrict__ r23,
                           const uint32_t *__restrict__ rpre, const uint32_t *__restrict__ ctr, uint4 *__restrict__ out, uint32_t *__restrict__ src) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= ft.n4 || !acc[p] || arank[p] >= max_flips) return;
    Flip f;
    bool illegal;
    fl_propose(xyz, cells, ft, p, f, illegal);
    uint32_t s[3] = {f.t0, f.t1, f.t2};  // ascending: t0 < t1, t2 placed
    if (f.kind == 3) {
        if (f.t2 < s[0]) { s[2] = s[1]; s[1] = s[0]; s[0] = f.t2; }
        else if (f.t2 < s[1]) { s[2] = s[1]; s[1] = f.t2; }
    }
    uint32_t dst[3] = {s[0] - rpre[s[0]], s[1] - rpre[s[1]], T - ctr[4] + r23[p]};
    const int m = f.kind == 2 ? 3 : 2;
    for (int j = 0; j < m; ++j) {
        out[dst[j]] = f.n[j];
        src[3 * (size_t)dst[j]] = s[0];
        src[3 * (size_t)dst[j] + 1] = s[1];
        src[3 * (size_t)dst[j] + 2] = f.kind == 3 ? s[2] : TN_EMPTY;
    }
}

}  // namespace tn

// workspace (each part 256-byte aligned): the face slots u32[4T] x 4 (slot, sorted slot / 3-2 partner cell, largest vertex, its sorted copy
// / proposal kind), the (a, b) keys u64[4T] x 2 (the unsorted one reused for the accepted flags and their ranks), the kept 2-3 flags and
// their ranks u32[4T] x 2, four u32[T] arrays (vote, touched, removed, removed-before), 8 counter words and the largest CUB temporary
extern "C" int tn_flip_delaunay(int device, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, uint32_t max_flips,
                                uint32_t *d_cells_out, uint32_t *d_sources, uint32_t *counts4, void *d_workspace, size_t *workspace_bytes,
                                void *stream) {
    if (!workspace_bytes) return tn::fail(TN_ERR_ARG, "tn_flip_delaunay: null workspace_bytes");
    if (T > 0x1FFFFFFFu) return tn::fail(TN_ERR_ARG, "tn_flip_delaunay: T must stay below 2^29");
    tn::DeviceGuard g(device);
    cudaStream_t s = (cudaStream_t)stream;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    using u64 = unsigned long long;
    const int n4 = (int)(4 * T), nt = (int)T;
    const int vbits = tn::radix_end_bit(V > 0 ? V - 1 : 0);
    auto sort_c = [&](void *t, size_t &bytes, const uint32_t *kin, uint32_t *kout, const uint32_t *vin, uint32_t *vout) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kin, kout, vin, vout, n4, 0, vbits, s);
    };
    auto sort_ab = [&](void *t, size_t &bytes, const u64 *kin, u64 *kout, const uint32_t *vin, uint32_t *vout) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kin, kout, vin, vout, n4, 0, 32 + vbits, s);
    };
    auto scan = [&](void *t, size_t &bytes, uint32_t *in, uint32_t *out, int m) { return cub::DeviceScan::ExclusiveSum(t, bytes, in, out, m, s); };
    size_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
    TN_CUDA(sort_c(nullptr, c0, nullptr, nullptr, nullptr, nullptr));
    TN_CUDA(sort_ab(nullptr, c1, nullptr, nullptr, nullptr, nullptr));
    TN_CUDA(scan(nullptr, c2, nullptr, nullptr, n4));
    TN_CUDA(scan(nullptr, c3, nullptr, nullptr, nt));
    size_t cub_bytes = std::max(std::max(c0, c1), std::max(c2, c3));
    const size_t pb = al(sizeof(uint32_t) * 4 * (size_t)T), kb = al(sizeof(u64) * 4 * (size_t)T), tb = al(sizeof(uint32_t) * (size_t)T),
                 cb = al(8 * sizeof(uint32_t));
    const size_t need = 6 * pb + 2 * kb + 4 * tb + cb + al(cub_bytes);
    if (!d_workspace) { *workspace_bytes = need; return TN_OK; }
    if (*workspace_bytes < need) return tn::fail(TN_ERR_ARG, "tn_flip_delaunay: workspace too small");
    if (!counts4) return tn::fail(TN_ERR_ARG, "tn_flip_delaunay: null counts4");
    counts4[0] = counts4[1] = counts4[2] = counts4[3] = 0;
    if (T == 0) return TN_OK;  // no cell: nothing to flip
    uint8_t *p = (uint8_t *)d_workspace;
    auto take = [&](size_t b) { uint8_t *q = p; p += b; return q; };
    uint32_t *val = (uint32_t *)take(pb), *val2 = (uint32_t *)take(pb), *key_c = (uint32_t *)take(pb), *key_c2 = (uint32_t *)take(pb);
    uint32_t *k23 = (uint32_t *)take(pb), *r23 = (uint32_t *)take(pb);
    u64 *kab = (u64 *)take(kb), *kab2 = (u64 *)take(kb);
    uint32_t *vote = (uint32_t *)take(tb), *touched = (uint32_t *)take(tb), *removed = (uint32_t *)take(tb), *rpre = (uint32_t *)take(tb);
    uint32_t *ctr = (uint32_t *)take(cb);  // [0] flags, [1] illegal, [2] proposals, [3] 2-3 flips, [4] 3-2 flips
    void *tmp = take(al(cub_bytes));
    uint32_t *kc = key_c, *kind = key_c2, *t2 = val2;        // free once the sorts ran
    uint32_t *acc = (uint32_t *)kab, *arank = acc + 4 * (size_t)T;
    const uint32_t pblocks = (4 * T + 255) / 256, tblocks = (T + 255) / 256;
    const uint4 *cells = (const uint4 *)d_cells;
    TN_CUDA(cudaMemsetAsync(ctr, 0, 8 * sizeof(uint32_t), s));
    tn::k_fl_slots<<<pblocks, 256, 0, s>>>(4 * T, V, cells, key_c, val, ctr);
    TN_CUDA(sort_c(tmp, cub_bytes, key_c, key_c2, val, val2));
    tn::k_fl_keys_ab<<<pblocks, 256, 0, s>>>(4 * T, cells, val2, kab);
    TN_CUDA(sort_ab(tmp, cub_bytes, kab, kab2, val2, val));
    tn::k_fl_runs<<<pblocks, 256, 0, s>>>(4 * T, cells, kab2, val, kc, ctr);
    uint32_t flags = 0;
    TN_CUDA(cudaMemcpyAsync(&flags, ctr, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (flags & 1u) return tn::fail(TN_ERR_ARG, "tn_flip_delaunay: a cell holds a vertex index >= V");
    if (flags & 2u) return tn::fail(TN_ERR_MESH, "tn_flip_delaunay: a triangle is shared by more than two tetrahedra");
    const tn::FaceTable ft{kab2, kc, val, 4 * T};
    tn::k_fl_propose<<<(4 * T + 127) / 128, 128, 0, s>>>(d_xyz, cells, ft, kind, t2, ctr);
    TN_CUDA(cudaMemsetAsync(vote, 0xFF, tb, s));
    tn::k_fl_vote<<<pblocks, 256, 0, s>>>(ft, kind, t2, vote);
    tn::k_fl_accept<<<pblocks, 256, 0, s>>>(ft, kind, t2, vote, acc);
    TN_CUDA(scan(tmp, cub_bytes, acc, arank, n4));
    TN_CUDA(cudaMemsetAsync(touched, 0, tb, s));
    TN_CUDA(cudaMemsetAsync(removed, 0, tb, s));
    tn::k_fl_mark<<<pblocks, 256, 0, s>>>(ft, max_flips, kind, t2, acc, arank, k23, touched, removed, ctr);
    TN_CUDA(scan(tmp, cub_bytes, k23, r23, n4));
    TN_CUDA(scan(tmp, cub_bytes, removed, rpre, nt));
    tn::k_fl_copy<<<tblocks, 256, 0, s>>>(T, cells, touched, rpre, (uint4 *)d_cells_out, d_sources);
    tn::k_fl_apply<<<(4 * T + 127) / 128, 128, 0, s>>>(d_xyz, cells, ft, T, max_flips, acc, arank, r23, rpre, ctr, (uint4 *)d_cells_out, d_sources);
    TN_CUDA(cudaGetLastError());
    uint32_t h[4];
    TN_CUDA(cudaMemcpyAsync(h, ctr + 1, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    for (int i = 0; i < 4; ++i) counts4[i] = h[i];
    return TN_OK;
}
