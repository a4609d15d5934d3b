// tn_faces.cu -- unique-face tables, adjacency tables and the hull convexity test, built on the device.
//
// Replaces the host loop of the reference (convert_tetrahedra_to_triangles, src/tetrahedra_tracer.cpp:21-71: an
// std::unordered_map over the 4T face slots, scanned in order) with sort + scan, reproducing its numbering exactly:
//   * slot i = 4*tet + j is the face opposite local vertex j, in the rotation (c[j+1], c[j+2], c[j+3])        (:51-53)
//   * a face's id is its rank among the FIRST appearances in slot order, its stored winding is the first
//     appearance's rotation, tt = (first tetrahedron, second tetrahedron or E)                                (:54-63)
//   * a face with a third owner is an error                                                                   (:64-66)
// The 4T slots are sorted by their sorted vertex triple with two stable radix passes (largest vertex first, then the
// 64-bit (smallest, middle) key), so that the slots of one face end up adjacent AND in slot order; the first of each run
// is the first appearance.  A flag per slot + exclusive scan gives the reference's face ids.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include "tn_common.cuh"
#include "tn_predicates.cuh"
#include "tn_sort.cuh"

namespace tn {

struct Tri3 {
    uint32_t a, b, c;
};
__device__ __forceinline__ void slot_vertices(const uint32_t *__restrict__ cells, uint32_t slot, uint32_t &x, uint32_t &y, uint32_t &z) {
    const uint4 c = reinterpret_cast<const uint4 *>(cells)[slot >> 2];
    const uint32_t v[4] = {c.x, c.y, c.z, c.w};
    const uint32_t j = slot & 3u;
    x = v[(j + 1) & 3]; y = v[(j + 2) & 3]; z = v[(j + 3) & 3];
}
__device__ __forceinline__ Tri3 slot_triple(const uint32_t *__restrict__ cells, uint32_t slot) {
    uint32_t x, y, z;
    slot_vertices(cells, slot, x, y, z);
    uint32_t t;
    if (x > y) { t = x; x = y; y = t; }
    if (y > z) { t = y; y = z; z = t; }
    if (x > y) { t = x; x = y; y = t; }
    return Tri3{x, y, z};
}
__device__ __forceinline__ bool same3(const Tri3 &p, const Tri3 &q) { return p.a == q.a && p.b == q.b && p.c == q.c; }

// err bits: 1 = vertex index out of range, 2 = a face with more than two owners, 4 = hull not a closed convex surface
__global__ void k_face_slots(const uint32_t *__restrict__ cells, uint32_t n, uint32_t V, uint32_t *__restrict__ key_c, uint32_t *__restrict__ val,
                             uint32_t *__restrict__ err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Tri3 t = slot_triple(cells, i);
    if (cells[i] >= V) atomicOr(err, 1u);
    key_c[i] = t.c;
    val[i] = i;
}
__global__ void k_face_keys2(const uint32_t *__restrict__ cells, const uint32_t *__restrict__ val, uint32_t n, unsigned long long *__restrict__ key_ab) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const Tri3 t = slot_triple(cells, val[p]);
    key_ab[p] = ((unsigned long long)t.a << 32) | t.b;
}
__global__ void k_face_heads(const uint32_t *__restrict__ cells, const uint32_t *__restrict__ val, uint32_t n, uint32_t *__restrict__ first_flag,
                             uint32_t *__restrict__ err) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const Tri3 t = slot_triple(cells, val[p]);
    const bool head = p == 0 || !same3(t, slot_triple(cells, val[p - 1]));
    if (!head && p >= 2 && same3(t, slot_triple(cells, val[p - 2]))) atomicOr(err, 2u);  // tetrahedra_tracer.cpp:64-66
    first_flag[val[p]] = head ? 1u : 0u;
}
__global__ void k_face_assign(const uint32_t *__restrict__ cells, const uint32_t *__restrict__ val, const uint32_t *__restrict__ first_flag,
                              const uint32_t *__restrict__ fid_first, uint32_t n, uint4 *__restrict__ tri, uint2 *__restrict__ tt,
                              uint32_t *__restrict__ tet_faces) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t i = val[p];
    if (!first_flag[i]) return;
    const uint32_t id = fid_first[i];
    uint32_t x, y, z;
    slot_vertices(cells, i, x, y, z);
    tri[id] = make_uint4(x, y, z, 0u);
    uint32_t second = TN_EMPTY;
    if (p + 1 < n) {
        const uint32_t i2 = val[p + 1];
        if (!first_flag[i2]) { second = i2 >> 2; tet_faces[i2] = id; }
    }
    tt[id] = make_uint2(i >> 2, second);
    tet_faces[i] = id | TN_FACE_OWNER;  // first owner: the stored winding is this rotation
}

// adjacency tables for the walk: neighbour across each face, stored winding as local vertex indices, hull flags
__global__ void k_walk_tables(const uint4 *__restrict__ cells, const uint4 *__restrict__ tri, const uint2 *__restrict__ tt, uint4 *__restrict__ tet_faces,
                              uint32_t T, uint4 *__restrict__ nbr, uint32_t *__restrict__ wind, uint8_t *__restrict__ hull_flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    const uint4 c4 = cells[i];
    const uint32_t c[4] = {c4.x, c4.y, c4.z, c4.w};
    const uint4 f4 = tet_faces[i];
    uint32_t fw[4] = {f4.x, f4.y, f4.z, f4.w}, nb[4];
    uint32_t w = 0;
    bool hull = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t f = fw[j] & TN_FACE_MASK;
        const uint2 o = tt[f];
        nb[j] = (o.x == i) ? o.y : o.x;
        if (o.y == TN_EMPTY) { fw[j] |= TN_FACE_HULL; hull = true; }
        const uint4 g4 = tri[f];
        const uint32_t g[3] = {g4.x, g4.y, g4.z};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            uint32_t loc = 0;
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q)
                if (c[q] == g[k]) loc = q;
            w |= loc << (6 * j + 2 * k);
        }
    }
    tet_faces[i] = make_uint4(fw[0], fw[1], fw[2], fw[3]);
    nbr[i] = make_uint4(nb[0], nb[1], nb[2], nb[3]);
    wind[i] = w;
    hull_flag[i] = hull ? 1 : 0;
}

// ---- hull convexity: every hull edge is shared by exactly two hull faces, and across it no vertex of one face lies above
// the plane of the other ----
__global__ void k_hull_face_flags(const uint2 *__restrict__ tt, uint32_t F, uint8_t *__restrict__ flag) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F) flag[f] = tt[f].y == TN_EMPTY ? 1 : 0;
}
__global__ void k_hull_edges(const uint4 *__restrict__ tri, const uint32_t *__restrict__ hull_faces, uint32_t Hf, unsigned long long *__restrict__ ekey,
                             uint32_t *__restrict__ eface) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * Hf) return;
    const uint32_t f = hull_faces[e / 3], k = e % 3;
    const uint4 t = tri[f];
    const uint32_t v[3] = {t.x, t.y, t.z};
    uint32_t a = v[k], b = v[(k + 1) % 3];
    if (a > b) { const uint32_t s = a; a = b; b = s; }
    ekey[e] = ((unsigned long long)a << 32) | b;
    eface[e] = f;
}
__global__ void k_hull_check(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint4 *__restrict__ tri, const uint2 *__restrict__ tt,
                             const unsigned long long *__restrict__ ekey, const uint32_t *__restrict__ eface, uint32_t n, uint32_t *__restrict__ err) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const bool same_prev = p > 0 && ekey[p - 1] == ekey[p], same_next = p + 1 < n && ekey[p + 1] == ekey[p];
    if (same_prev == same_next) { atomicOr(err, 4u); return; }  // open edge, or an edge shared by more than two hull faces
    if (same_next && (!hull_pair_ok(xyz, cells, tri, tt, eface[p], eface[p + 1]) || !hull_pair_ok(xyz, cells, tri, tt, eface[p + 1], eface[p])))
        atomicOr(err, 4u);
}
__global__ void k_iota(uint32_t *__restrict__ v, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
}

// ---- fold test of a refit: for every interior face (a, b, c), the opposite vertices p, q of its two tetrahedra must lie strictly on
// opposite sides of its plane (face_unfolded, tn_predicates.cuh) ----
__global__ void k_fold_faces(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint4 *__restrict__ tri, const uint2 *__restrict__ tt,
                             uint32_t F, uint32_t *__restrict__ folded) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const uint2 o = tt[f];
    if (o.y == TN_EMPTY) return;
    const uint4 t = tri[f];
    if (!face_unfolded(xyz, t.x, t.y, t.z, opposite_vertex(cells[o.x], t), opposite_vertex(cells[o.y], t))) atomicAdd(folded, 1u);
}

int launch_refit_checks(const tn_tracer *h, const float *d_xyz, uint32_t *d_counts, cudaStream_t s) {
    const Mesh &m = h->mesh;
    if (m.hull_ne > 0)
        k_hull_check<<<(m.hull_ne + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)m.cells, m.tri.p, m.tt.p, m.hull_ekey.p, m.hull_eface.p,
                                                            m.hull_ne, d_counts);
    k_fold_faces<<<(m.F + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)m.cells, m.tri.p, m.tt.p, m.F, d_counts + 1);
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

// Builds the face / adjacency tables of the mesh on the device into `out` (tri, tt, hull_ekey, hull_eface go into the Mesh; tet_faces,
// nbr, wind, hull_list are build-time temporaries).  On an error `out` holds whatever was built so far, freed with it.
int build_faces_device(const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, cudaStream_t s, FaceTables &out, int *launches) {
    const uint32_t n = 4 * T;
    DevArray<uint32_t> key_c, key_c2, val, val2, flag, fid, d_small, iota, hull_faces, eface, eface2;
    DevArray<unsigned long long> kab, kab2;
    DevArray<uint8_t> bflag, tmp;
    const uint32_t nb = (n + 255) / 256;
    TN_TRY(key_c.grow(n)); TN_TRY(key_c2.grow(n));
    TN_TRY(val.grow(n)); TN_TRY(val2.grow(n));
    TN_TRY(kab.grow(n)); TN_TRY(kab2.grow(n));
    TN_TRY(flag.grow(n)); TN_TRY(fid.grow(n));
    TN_TRY(d_small.grow(4));  // [0] err, [1] selected count, [2] hull faces, [3] folded faces
    TN_CUDA(cudaMemsetAsync(d_small.p, 0, 16, s));
    // val: slots grouped by face, slot order inside.  The largest CUB request of the build: the scratch is sized for it up front, so the
    // calls below run without freeing and reallocating it in between
    auto sort_faces = [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kab.p, kab2.p, val2.p, val.p, (int)n, 0, 64, s);
    };
    size_t largest = 0;
    TN_CUDA(sort_faces(nullptr, largest));
    TN_TRY(tmp.grow(largest));
    k_face_slots<<<nb, 256, 0, s>>>(d_cells, n, V, key_c.p, val.p, d_small.p);
    TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, key_c.p, key_c2.p, val.p, val2.p, (int)n, 0, 32, s);
    }));
    k_face_keys2<<<nb, 256, 0, s>>>(d_cells, val2.p, n, kab.p);
    TN_TRY(cub_run(tmp, sort_faces));
    k_face_heads<<<nb, 256, 0, s>>>(d_cells, val.p, n, flag.p, d_small.p);
    TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) { return cub::DeviceScan::ExclusiveSum(t, bytes, flag.p, fid.p, (int)n, s); }));
    uint32_t h_small[4] = {0, 0, 0, 0}, last[2] = {0, 0};
    TN_CUDA(cudaMemcpyAsync(h_small, d_small.p, 4, cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaMemcpyAsync(&last[0], flag.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaMemcpyAsync(&last[1], fid.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if (h_small[0] & 1u) return fail(TN_ERR_ARG, "load_tetrahedra: cell index out of range");
    if (h_small[0] & 2u) return fail(TN_ERR_MESH, "A triangle is shared by more than two tetrahedra!");  // tetrahedra_tracer.cpp:64-66
    const uint32_t F = last[0] + last[1];
    out.F = F;
    TN_TRY(out.tri.grow(F));
    TN_TRY(out.tt.grow(F));
    TN_TRY(out.tet_faces.grow(T));
    TN_TRY(out.nbr.grow(T));
    TN_TRY(out.wind.grow(T));
    k_face_assign<<<nb, 256, 0, s>>>(d_cells, val.p, flag.p, fid.p, n, out.tri.p, out.tt.p, reinterpret_cast<uint32_t *>(out.tet_faces.p));
    TN_TRY(bflag.grow(std::max(T, F)));
    TN_TRY(iota.grow(std::max(T, F)));
    k_walk_tables<<<(T + 127) / 128, 128, 0, s>>>((const uint4 *)d_cells, out.tri.p, out.tt.p, out.tet_faces.p, T, out.nbr.p, out.wind.p, bflag.p);
    k_iota<<<(std::max(T, F) + 255) / 256, 256, 0, s>>>(iota.p, std::max(T, F));
    // tetrahedra owning a hull face, in tetrahedron order
    TN_TRY(out.hull_list.grow(T));
    TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceSelect::Flagged(t, bytes, iota.p, bflag.p, out.hull_list.p, d_small.p + 1, (int)T, s);
    }));
    uint32_t H = 0, Hf = 0;
    TN_CUDA(cudaMemcpyAsync(&H, d_small.p + 1, 4, cudaMemcpyDeviceToHost, s));
    // hull faces -> edges -> sorted -> pair checks
    k_hull_face_flags<<<(F + 255) / 256, 256, 0, s>>>(out.tt.p, F, bflag.p);
    TN_TRY(hull_faces.grow(F));
    TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceSelect::Flagged(t, bytes, iota.p, bflag.p, hull_faces.p, d_small.p + 2, (int)F, s);
    }));
    TN_CUDA(cudaMemcpyAsync(&Hf, d_small.p + 2, 4, cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    out.H = H;
    bool walkable = H > 0 && Hf > 0 && 3 * (size_t)Hf <= n;
    if (walkable) {
        const uint32_t ne = 3 * Hf;
        TN_TRY(eface.grow(ne)); TN_TRY(eface2.grow(ne));
        k_hull_edges<<<(ne + 255) / 256, 256, 0, s>>>(out.tri.p, hull_faces.p, Hf, kab.p, eface.p);
        TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
            return cub::DeviceRadixSort::SortPairs(t, bytes, kab.p, kab2.p, eface.p, eface2.p, (int)ne, 0, 64, s);
        }));
        k_hull_check<<<(ne + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)d_cells, out.tri.p, out.tt.p, kab2.p, eface2.p, ne, d_small.p);
        // the refit's fold test on the load's tables: the walk sees only the chain of tetrahedra from the hull entry, and on a folded mesh
        // a line also crosses faces off that chain (DESIGN §4.9), so a mesh with an uncertified face loads with the walk off
        k_fold_faces<<<(F + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)d_cells, out.tri.p, out.tt.p, F, d_small.p + 3);
        TN_CUDA(cudaMemcpyAsync(h_small, d_small.p, 16, cudaMemcpyDeviceToHost, s));
        TN_CUDA(cudaStreamSynchronize(s));
        walkable = (h_small[0] & 4u) == 0;
        out.folded = h_small[3];
        if (launches) *launches += 3;
        if (walkable) {  // kept for the convexity test of a refit (tn_update_vertices)
            TN_TRY(out.hull_ekey.grow(ne)); TN_TRY(out.hull_eface.grow(ne));
            TN_CUDA(cudaMemcpyAsync(out.hull_ekey.p, kab2.p, 8 * (size_t)ne, cudaMemcpyDeviceToDevice, s));
            TN_CUDA(cudaMemcpyAsync(out.hull_eface.p, eface2.p, 4 * (size_t)ne, cudaMemcpyDeviceToDevice, s));
            out.hull_ne = ne;
        }
    }
    out.walkable = walkable;
    if (launches) *launches += 8;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

}  // namespace tn
