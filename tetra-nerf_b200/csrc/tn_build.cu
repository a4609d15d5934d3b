// tn_build.cu -- load_tetrahedra: unique-face tables + on-device Morton-ordered 8-ary BVH.
//
// Replaces TetrahedraStructure::build (src/tetrahedra_tracer.cpp:244-340): the reference converts the
// 4T faces into unique triangles on the host (:45-71) and hands them to optixAccelBuild (:285-332).
// Here the face numbering / stored windings are reproduced exactly (they define the meaning of the
// barycentrics and of vertex_indices' slot order) and the acceleration structure is ours.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <utility>
#include <vector>

#include "tn_common.cuh"
#include "tn_sort.cuh"

namespace tn {

// ---- device kernels --------------------------------------------------------------------------
__device__ __forceinline__ int f2ord(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF); }

// bounds[0..2] = min, [3..5] = max (ordered-int encoded)
__global__ void k_bounds(const float *__restrict__ xyz, uint32_t V, int *__restrict__ bounds) {
    float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float x = xyz[3 * (size_t)i + a];
            lo[a] = fminf(lo[a], x);
            hi[a] = fmaxf(hi[a], x);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(&bounds[a], f2ord(lo[a]));
            atomicMax(&bounds[3 + a], f2ord(hi[a]));
        }
    }
}

__device__ __forceinline__ uint32_t expand10(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

__global__ void k_morton(const float *__restrict__ xyz, const uint4 *__restrict__ cells, uint32_t T, const int *__restrict__ bounds,
                         uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    const uint4 c = cells[i];
    const uint32_t id[4] = {c.x, c.y, c.z, c.w};
    float cen[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) cen[a] += 0.25f * xyz[3 * (size_t)id[k] + a];
    uint32_t q[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float lo = ord2f(bounds[a]), hi = ord2f(bounds[3 + a]);
        const float ext = fmaxf(hi - lo, 1e-30f);
        const float u = fminf(fmaxf((cen[a] - lo) / ext, 0.f), 1.f);
        q[a] = min(1023u, (uint32_t)(u * 1024.f));
    }
    keys[i] = (expand10(q[0]) << 2) | (expand10(q[1]) << 1) | expand10(q[2]);
    vals[i] = i;
}

__global__ void k_morton_subset(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint32_t *__restrict__ list, uint32_t n,
                                const int *__restrict__ bounds, uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t tet = list[i];
    const uint4 c = cells[tet];
    const uint32_t id[4] = {c.x, c.y, c.z, c.w};
    float cen[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) cen[a] += 0.25f * xyz[3 * (size_t)id[k] + a];
    uint32_t q[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float lo = ord2f(bounds[a]), hi = ord2f(bounds[3 + a]);
        const float u = fminf(fmaxf((cen[a] - lo) / fmaxf(hi - lo, 1e-30f), 0.f), 1.f);
        q[a] = min(1023u, (uint32_t)(u * 1024.f));
    }
    keys[i] = (expand10(q[0]) << 2) | (expand10(q[1]) << 1) | expand10(q[2]);
    vals[i] = tet;
}

__global__ void k_walk_records(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint4 *__restrict__ tet_faces,
                               const uint4 *__restrict__ nbr, const uint32_t *__restrict__ wind, uint32_t T, WalkRec *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    const uint4 c = cells[i], f = tet_faces[i], nb = nbr[i];
    const uint32_t id[4] = {c.x, c.y, c.z, c.w}, fi[4] = {f.x, f.y, f.z, f.w};
    WalkRec r;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        r.v[k] = make_float4(xyz[3 * (size_t)id[k]], xyz[3 * (size_t)id[k] + 1], xyz[3 * (size_t)id[k] + 2], __uint_as_float(fi[k]));
    r.nbr[0] = nb.x; r.nbr[1] = nb.y; r.nbr[2] = nb.z; r.nbr[3] = nb.w;
    r.vid[0] = c.x; r.vid[1] = c.y; r.vid[2] = c.z; r.vid[3] = c.w;
    const uint32_t w = wind[i];
    r.wind = w;
    uint32_t perm = 0;
#pragma unroll
    for (uint32_t jin = 0; jin < 4; ++jin) {
        const uint32_t wi = (w >> (6 * jin)) & 63u;
        const uint32_t ia[3] = {wi & 3u, (wi >> 2) & 3u, (wi >> 4) & 3u};
        perm |= (jin | (ia[0] << 2) | (ia[1] << 4) | (ia[2] << 6)) << (8 * jin);
        uint32_t m = 0;
#pragma unroll
        for (uint32_t jout = 0; jout < 4; ++jout) {
            const uint32_t wo = (w >> (6 * jout)) & 63u;
            const uint32_t oa[3] = {wo & 3u, (wo >> 2) & 3u, (wo >> 4) & 3u};
#pragma unroll
            for (uint32_t q = 0; q < 3; ++q) {
                uint32_t code = 3u;  // entry-face vertex q is not on the exit face
#pragma unroll
                for (uint32_t k = 0; k < 3; ++k)
                    if (ia[q] == oa[k]) code = k;
                m |= code << (6 * jout + 2 * q);
            }
        }
        r.map[jin] = m;
    }
    r.perm = perm;
    r.pad[0] = r.pad[1] = 0;
    out[i] = r;
}

// sorted position p -> leaf record + level-0 node
__global__ void k_leaves(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint4 *__restrict__ tet_faces,
                         const uint32_t *__restrict__ order, uint32_t T, LeafRec *__restrict__ leaves, float4 *__restrict__ nodes0) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= T) return;
    const uint32_t tet = order[p];
    const uint4 c = cells[tet];
    const uint4 f = tet_faces[tet];
    const uint32_t id[4] = {c.x, c.y, c.z, c.w};
    const uint32_t fi[4] = {f.x, f.y, f.z, f.w};
    float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
    LeafRec rec;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float x = xyz[3 * (size_t)id[k]], y = xyz[3 * (size_t)id[k] + 1], z = xyz[3 * (size_t)id[k] + 2];
        rec.v[k] = make_float4(x, y, z, __uint_as_float(fi[k]));
        lo[0] = fminf(lo[0], x); hi[0] = fmaxf(hi[0], x);
        lo[1] = fminf(lo[1], y); hi[1] = fmaxf(hi[1], y);
        lo[2] = fminf(lo[2], z); hi[2] = fmaxf(hi[2], z);
    }
    leaves[p] = rec;
    nodes0[2 * (size_t)p] = make_float4(lo[0], lo[1], lo[2], hi[0]);
    nodes0[2 * (size_t)p + 1] = make_float4(hi[1], hi[2], 0.f, 0.f);
}

__global__ void k_level(const float4 *__restrict__ child, uint32_t nchild, float4 *__restrict__ parent, uint32_t nparent) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nparent) return;
    float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
    for (uint32_t c = TN_FAN * i; c < min(TN_FAN * i + TN_FAN, nchild); ++c) {
        const float4 a = child[2 * (size_t)c], b = child[2 * (size_t)c + 1];
        lo[0] = fminf(lo[0], a.x); lo[1] = fminf(lo[1], a.y); lo[2] = fminf(lo[2], a.z);
        hi[0] = fmaxf(hi[0], a.w); hi[1] = fmaxf(hi[1], b.x); hi[2] = fmaxf(hi[2], b.y);
    }
    parent[2 * (size_t)i] = make_float4(lo[0], lo[1], lo[2], hi[0]);
    parent[2 * (size_t)i + 1] = make_float4(hi[1], hi[2], 0.f, 0.f);
}

// ---- refit (tn_update_vertices): the position fields of the records, rewritten in place --------------------------------------------
__global__ void k_nonfinite(const float *__restrict__ xyz, uint32_t n, uint32_t *__restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !isfinite(xyz[i])) atomicOr(flag, 1u);
}
// sorted position p -> leaf record positions + level-0 node (the face bits in .w are topological and stay); the boxes as k_leaves.
// Nothing is written while *bad is set (non-finite input): k_level then recomputes the unchanged boxes, so the tracer stays as it was.
__global__ void k_refit_leaves(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint32_t *__restrict__ order, uint32_t T,
                               const uint32_t *__restrict__ bad, LeafRec *__restrict__ leaves, float4 *__restrict__ nodes0) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= T || *bad) return;
    const uint4 c = cells[order[p]];
    const uint32_t id[4] = {c.x, c.y, c.z, c.w};
    float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
    LeafRec rec = leaves[p];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float x = xyz[3 * (size_t)id[k]], y = xyz[3 * (size_t)id[k] + 1], z = xyz[3 * (size_t)id[k] + 2];
        rec.v[k] = make_float4(x, y, z, rec.v[k].w);
        lo[0] = fminf(lo[0], x); hi[0] = fmaxf(hi[0], x);
        lo[1] = fminf(lo[1], y); hi[1] = fmaxf(hi[1], y);
        lo[2] = fminf(lo[2], z); hi[2] = fmaxf(hi[2], z);
    }
    leaves[p] = rec;
    nodes0[2 * (size_t)p] = make_float4(lo[0], lo[1], lo[2], hi[0]);
    nodes0[2 * (size_t)p + 1] = make_float4(hi[1], hi[2], 0.f, 0.f);
}
// WalkRec v[k].xyz of tetrahedron i (nbr, vid, map, wind, perm and the face bits are topological and stay); nothing while *bad is set
__global__ void k_refit_walk(const float *__restrict__ xyz, const uint4 *__restrict__ cells, uint32_t T, const uint32_t *__restrict__ bad,
                             WalkRec *__restrict__ walk) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T || *bad) return;
    const uint4 c = cells[i];
    const uint32_t id[4] = {c.x, c.y, c.z, c.w};
    float4 *v = walk[i].v;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        v[k] = make_float4(xyz[3 * (size_t)id[k]], xyz[3 * (size_t)id[k] + 1], xyz[3 * (size_t)id[k] + 2], v[k].w);
}

static float absmax_of(const int *hbounds) {  // max |coordinate| from the ordered-int bounds of k_bounds
    float amax = 0.f;
    for (int a = 0; a < 6; ++a) {
        int i = hbounds[a];
        i = i >= 0 ? i : i ^ 0x7FFFFFFF;
        float f;
        memcpy(&f, &i, 4);
        amax = std::max(amax, std::fabs(f));
    }
    return amax;
}

int build_mesh(tn_tracer *h, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, cudaStream_t s) {
    h->mesh = Mesh();  // the old mesh goes first (it is not needed to build the new one), and a failed load leaves none
    if (T == 0 || V == 0) return fail(TN_ERR_ARG, "load_tetrahedra: empty mesh");
    if (T >= (1u << 28)) return fail(TN_ERR_ARG, "load_tetrahedra: more than 2^28 tetrahedra are not supported");
    Mesh m;  // moved into h->mesh once complete

    // ---- faces, adjacency tables, hull convexity: all on the device (tn_faces.cu) ----
    FaceTables ft;
    {
        int extra = 0;
        TN_TRY(build_faces_device(d_xyz, V, d_cells, T, s, ft, &extra));
        h->launches += extra;
    }
    const uint32_t F = ft.F, H = ft.H;
    const bool walkable = ft.walkable;
    m.tri = std::move(ft.tri); m.tt = std::move(ft.tt);
    m.hull_ekey = std::move(ft.hull_ekey); m.hull_eface = std::move(ft.hull_eface); m.hull_ne = ft.hull_ne;
    const uint4 *d_tet_faces = ft.tet_faces.p, *d_nbr = ft.nbr.p;
    const uint32_t *d_wind = ft.wind.p, *d_hull_list = ft.hull_list.p;
    DevArray<uint32_t> keys, keys2, vals;
    DevArray<int> bounds;
    DevArray<uint8_t> tmp;

    // ---- levels ----
    BvhLevels lv{};
    uint32_t cnt = T, off = 0;
    int L = 0;
    for (;;) {
        if (L >= TN_MAX_LEVELS) return fail(TN_ERR_ARG, "load_tetrahedra: too many BVH levels");
        lv.count[L] = cnt; lv.offset[L] = off;
        off += (cnt + TN_FAN - 1) & ~(TN_FAN - 1);  // keep every level's base a multiple of TN_FAN nodes (256 B)
        ++L;
        if (cnt == 1) break;
        cnt = (cnt + TN_FAN - 1) / TN_FAN;
    }
    if (L == 1) {  // a single tetrahedron: add a root above it so that traversal always starts at level >= 1
        lv.count[1] = 1; lv.offset[1] = off; off += TN_FAN; L = 2;
    }
    lv.nlevels = L;
    const uint32_t total_nodes = off;

    TN_TRY(m.nodes.grow(2 * (size_t)total_nodes));
    TN_TRY(m.leaves.grow(T));
    TN_TRY(m.leaf_tet.grow(T));
    TN_TRY(keys.grow(T));
    TN_TRY(keys2.grow(T));
    TN_TRY(vals.grow(T));
    TN_TRY(bounds.grow(6));

    // ordered-int encodings (f2ord) of +FLT_MAX for the min slots and -FLT_MAX for the max slots
    const int hb_enc[6] = {0x7F7FFFFF, 0x7F7FFFFF, 0x7F7FFFFF, (int)0x80800000, (int)0x80800000, (int)0x80800000};
    TN_CUDA(cudaMemcpyAsync(bounds.p, hb_enc, sizeof(hb_enc), cudaMemcpyHostToDevice, s));
    k_bounds<<<std::min<uint32_t>((V + 255) / 256, 1184u), 256, 0, s>>>(d_xyz, V, bounds.p);
    k_morton<<<(T + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)d_cells, T, bounds.p, keys.p, vals.p);
    TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, keys.p, keys2.p, vals.p, m.leaf_tet.p, (int)T, 0, 30, s);
    }));
    k_leaves<<<(T + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)d_cells, d_tet_faces, m.leaf_tet.p, T, m.leaves.p, m.nodes.p);
    for (int l = 1; l < L; ++l) {
        const uint32_t np = lv.count[l], nc = lv.count[l - 1];
        k_level<<<(np + 127) / 128, 128, 0, s>>>(m.nodes.p + 2 * (size_t)lv.offset[l - 1], nc, m.nodes.p + 2 * (size_t)lv.offset[l], np);
    }
    h->launches += 4 + (L - 1);
    TN_CUDA(cudaGetLastError());

    // ---- adjacency walk: per-tetrahedron records + a small BVH over the tetrahedra that own a hull face ----
    BvhLevels hlv{};
    if (walkable) {
        TN_TRY(m.walk.grow(T));
        k_walk_records<<<(T + 127) / 128, 128, 0, s>>>(d_xyz, (const uint4 *)d_cells, d_tet_faces, d_nbr, d_wind, T, m.walk.p);
        uint32_t hc_ = H, hoff = 0;
        int HL = 0;
        for (;;) {
            hlv.count[HL] = hc_; hlv.offset[HL] = hoff;
            hoff += (hc_ + TN_FAN - 1) & ~(TN_FAN - 1);
            ++HL;
            if (hc_ == 1) break;
            hc_ = (hc_ + TN_FAN - 1) / TN_FAN;
        }
        if (HL == 1) { hlv.count[1] = 1; hlv.offset[1] = hoff; hoff += TN_FAN; HL = 2; }
        hlv.nlevels = HL;
        TN_TRY(m.hull_nodes.grow(2 * (size_t)hoff));
        TN_TRY(m.hull_leaves.grow(H));
        TN_TRY(m.hull_tet.grow(H));
        k_morton_subset<<<(H + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)d_cells, d_hull_list, H, bounds.p, keys.p, vals.p);
        TN_TRY(cub_run(tmp, [&](void *t, size_t &bytes) {
            return cub::DeviceRadixSort::SortPairs(t, bytes, keys.p, keys2.p, vals.p, m.hull_tet.p, (int)H, 0, 30, s);
        }));
        k_leaves<<<(H + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)d_cells, d_tet_faces, m.hull_tet.p, H, m.hull_leaves.p, m.hull_nodes.p);
        for (int l = 1; l < HL; ++l) {
            const uint32_t np = hlv.count[l], nc = hlv.count[l - 1];
            k_level<<<(np + 127) / 128, 128, 0, s>>>(m.hull_nodes.p + 2 * (size_t)hlv.offset[l - 1], nc, m.hull_nodes.p + 2 * (size_t)hlv.offset[l], np);
        }
        h->launches += 3 + HL;
        TN_CUDA(cudaGetLastError());
    }
    int hbounds[6];
    TN_CUDA(cudaMemcpyAsync(hbounds, bounds.p, sizeof(hbounds), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    m.xyz = d_xyz; m.cells = d_cells; m.V = V; m.T = T; m.F = F; m.lv = lv; m.absmax = absmax_of(hbounds);
    // the walk records are built for every convex hull, so that a refit which unfolds the mesh turns the walk on again
    m.walkable = walkable && ft.folded == 0; m.H = walkable ? H : 0; m.hull_lv = hlv;
    h->mesh = std::move(m);
    return TN_OK;
}

// Moves the vertices of the loaded mesh to d_xyz and rewrites every position-dependent field in place (same cells, same Morton order):
// leaf records and level-0 boxes of both BVHs, the upper levels by k_level, the walk records, absmax; then the hull convexity test on the
// load's hull edges and the fold test.  The non-finite check runs first on the device and the record kernels skip their writes when it
// fires, so non-finite input leaves the tracer unchanged with a single read-back at the end.
int refit_mesh(tn_tracer *h, const float *d_xyz, uint32_t V, cudaStream_t s, uint32_t *folded_faces, int *walkable) {
    Mesh &m = h->mesh;
    if (!m.nodes.p) return fail(TN_ERR_STATE, "update_vertices: no tetrahedra loaded");
    if (V != m.V) return fail(TN_ERR_ARG, "update_vertices: " + std::to_string(V) + " vertices, the loaded mesh has " + std::to_string(m.V));
    TN_TRY(h->d_refit.grow(16));
    uint32_t *d_small = h->d_refit.p;  // [0] non-finite flag, [2] hull error bits, [3] folded faces, [4..9] bounds (ordered ints)
    int *bounds = reinterpret_cast<int *>(d_small + 4);
    // ordered-int encodings (f2ord) of +FLT_MAX for the min slots and -FLT_MAX for the max slots, after four zeroed words
    const int init[10] = {0, 0, 0, 0, 0x7F7FFFFF, 0x7F7FFFFF, 0x7F7FFFFF, (int)0x80800000, (int)0x80800000, (int)0x80800000};
    TN_CUDA(cudaMemcpyAsync(d_small, init, sizeof(init), cudaMemcpyHostToDevice, s));
    const uint32_t n = 3 * V;
    k_nonfinite<<<(n + 255) / 256, 256, 0, s>>>(d_xyz, n, d_small);
    k_bounds<<<std::min<uint32_t>((V + 255) / 256, 1184u), 256, 0, s>>>(d_xyz, V, bounds);
    const uint32_t T = m.T;
    k_refit_leaves<<<(T + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)m.cells, m.leaf_tet.p, T, d_small, m.leaves.p, m.nodes.p);
    for (int l = 1; l < m.lv.nlevels; ++l)
        k_level<<<(m.lv.count[l] + 127) / 128, 128, 0, s>>>(m.nodes.p + 2 * (size_t)m.lv.offset[l - 1], m.lv.count[l - 1],
                                                             m.nodes.p + 2 * (size_t)m.lv.offset[l], m.lv.count[l]);
    h->launches += 3 + (m.lv.nlevels - 1);
    if (m.walk.p) {
        k_refit_walk<<<(T + 127) / 128, 128, 0, s>>>(d_xyz, (const uint4 *)m.cells, T, d_small, m.walk.p);
        const uint32_t H = m.hull_lv.count[0];
        k_refit_leaves<<<(H + 255) / 256, 256, 0, s>>>(d_xyz, (const uint4 *)m.cells, m.hull_tet.p, H, d_small, m.hull_leaves.p, m.hull_nodes.p);
        for (int l = 1; l < m.hull_lv.nlevels; ++l)
            k_level<<<(m.hull_lv.count[l] + 127) / 128, 128, 0, s>>>(m.hull_nodes.p + 2 * (size_t)m.hull_lv.offset[l - 1], m.hull_lv.count[l - 1],
                                                                      m.hull_nodes.p + 2 * (size_t)m.hull_lv.offset[l], m.hull_lv.count[l]);
        h->launches += 2 + (m.hull_lv.nlevels - 1);
    }
    int rc = launch_refit_checks(h, d_xyz, d_small + 2, s);
    if (rc) return rc;
    h->launches += 2;
    uint32_t hs[10];
    TN_CUDA(cudaMemcpyAsync(hs, d_small, sizeof(hs), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    TN_CUDA(cudaGetLastError());
    if (hs[0]) return fail(TN_ERR_ARG, "update_vertices: a vertex coordinate is not finite");
    h->mesh_gen = next_generation();  // the positions changed
    m.xyz = d_xyz;
    m.absmax = absmax_of(reinterpret_cast<const int *>(hs + 4));
    m.walkable = m.walk.p != nullptr && (hs[2] & 4u) == 0 && hs[3] == 0;
    if (folded_faces) *folded_faces = hs[3];
    if (walkable) *walkable = m.walkable ? 1 : 0;
    return TN_OK;
}

}  // namespace tn
