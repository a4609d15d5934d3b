// =============================================================================
// tetra_oracle.cpp -- TEST INFRASTRUCTURE ONLY.  NOT PART OF THE PRODUCT.
//
// CPU restatement of the Tetra-NeRF ray-sampling hot path (jkulhanek/tetra-nerf
// @1ea894d).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may load this library; the product path (the CUDA
// library behind include/tetranerf_b200.h) never does.
//
// PARITY STATUS: "parity unpinned" for trace_rays -- the reference's tracer is
// OptiX-only (src/py_binding.cpp:30-33), cannot be built here (no optix.h) and
// its own tests hold no golden values for trace_rays
// (tests/test_tetrahedra_tracer.py:267 "# TODO: check results").  This file is
// pinned instead against (i) the float64 known-answer crossing list derived in
// SURVEY.md §8c, (ii) an independent per-tetrahedron plane-clipping oracle
// (oracle/intervals.py), (iii) for find_matched_cells / interpolate_values the
// reference's real CUDA kernels compiled from /root/reference by
// oracle/Makefile into oracle/_ref/ (GPU box only).
//
// What follows which reference lines:
//   build_faces            src/tetrahedra_tracer.cpp:21-71
//   ray/face all-hit gather src/optix/optix_trace_rays.cu:268-294,310-331
//                          (the intersector itself is OptiX hardware, not
//                          bit-specified; restated as the fp32 watertight test
//                          of Woop/Benthin/Wald 2013, see ray_tri())
//   bitonic_sort           src/optix/optix_trace_rays.cu:78-108
//   get_common_tetrahedra  src/optix/optix_trace_rays.cu:22-37
//   combine_indices        src/optix/optix_trace_rays.cu:39-75
//   post_process           src/optix/optix_trace_rays.cu:110-266
//   find_matched_cells     src/tetrahedra_tracer.cu:115-161
//   interpolate_values     src/tetrahedra_tracer.cu:195-221
//   interpolate_backward   src/tetrahedra_tracer.cu:223-248
//   trace_rays_triangles   src/optix/optix_trace_rays_triangles.cu:49-114
//   find_tetrahedra        src/optix/optix_find_tetrahedra.cu:84-213
//
// Pinned choices where the reference leaves behaviour undefined:
//   * sort ties: reference compares t only on an undefined (OptiX traversal)
//     input order; here the key is (t, face id) -- a total order.
//   * hit cap: reference keeps whichever M-1 hits OptiX reports first; here the
//     M-1 smallest keys are kept.
//   * OOB read of triangle_tetrahedra[0xFFFFFFFF] (optix_trace_rays.cu:131-134)
//     is not reproduced (value is never used).
//   * tails of hit_distances / barycentric_coordinates beyond num_visited hold
//     sort scratch in the reference; here they are zero.
//
// Compile: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math -shared -fPIC
// (-ffp-contract=off is REQUIRED: the CUDA side uses __fmul_rn/__fadd_rn.)
// =============================================================================
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

constexpr uint32_t EMPTY = 0xFFFFFFFFu;
constexpr float EPS = 1e-6;  // optix_trace_rays.cu:8 (double literal -> float)

struct U3 { uint32_t x, y, z; };
struct U2 { uint32_t x, y; };
struct F2 { float x, y; };
struct F3 { float x, y, z; };
struct U4 { uint32_t x, y, z, w; };

// ---- src/tetrahedra_tracer.cpp:21-33 ---------------------------------------
static U3 order_faces(U3 f) {
    if (f.x > f.y) std::swap(f.x, f.y);
    if (f.y > f.z) std::swap(f.y, f.z);
    if (f.x > f.y) std::swap(f.x, f.y);
    return f;
}
struct U3Hash {
    size_t operator()(const U3 &k) const {
        // any hash works: the map is only used for membership (tracer.cpp:35-43)
        uint64_t h = k.x * 0x9E3779B97F4A7C15ull;
        h ^= (uint64_t)k.y * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2);
        h ^= (uint64_t)k.z * 0x165667B19E3779F9ull + (h << 6) + (h >> 2);
        return (size_t)h;
    }
};
struct U3Eq { bool operator()(const U3 &a, const U3 &b) const { return a.x == b.x && a.y == b.y && a.z == b.z; } };

// ---- src/tetrahedra_tracer.cpp:45-71 ---------------------------------------
// returns 0, or -1 if a face has more than two owners (reference throws).
static int build_faces(const uint32_t *cells, uint32_t T, std::vector<U3> &tri, std::vector<U2> &tt) {
    std::unordered_map<U3, uint32_t, U3Hash, U3Eq> known;
    known.reserve((size_t)T * 2 + 16);
    for (uint32_t i = 0; i < T; ++i) {
        for (int j = 0; j < 4; ++j) {
            const uint32_t *c = cells + 4 * (size_t)i;
            U3 t{c[(j + 1) % 4], c[(j + 2) % 4], c[(j + 3) % 4]};
            U3 key = order_faces(t);
            auto it = known.find(key);
            if (it == known.end()) {
                known.emplace(key, (uint32_t)tt.size());
                tri.push_back(t);
                tt.push_back(U2{i, EMPTY});
            } else {
                if (tt[it->second].y != EMPTY) return -1;
                tt[it->second].y = i;
            }
        }
    }
    return 0;
}

// ---- ray setup + watertight fp32 ray/triangle test --------------------------
// Stand-in for optixTrace's built-in triangle intersector (call site
// optix_trace_rays.cu:280-292).  Woop, Benthin, Wald: "Watertight Ray/Triangle
// Intersection", JCGT 2013, fp32 with the double fallback on zero edge
// functions.  Every operation is individually rounded (no FMA); the CUDA
// kernel performs the same sequence with __f*_rn intrinsics.
struct RaySetup {
    int kx, ky, kz;
    float Sx, Sy, Sz;
    float o[3];
    bool valid;
};
static RaySetup ray_setup(const float *o, const float *d) {
    RaySetup r;
    r.o[0] = o[0]; r.o[1] = o[1]; r.o[2] = o[2];
    int kz = 0;
    if (std::fabs(d[1]) > std::fabs(d[kz])) kz = 1;
    if (std::fabs(d[2]) > std::fabs(d[kz])) kz = 2;
    int kx = (kz + 1) % 3, ky = (kx + 1) % 3;
    if (d[kz] < 0.0f) std::swap(kx, ky);
    r.kx = kx; r.ky = ky; r.kz = kz;
    r.valid = (d[kz] != 0.0f) && std::isfinite(d[0]) && std::isfinite(d[1]) && std::isfinite(d[2]);
    r.Sx = d[kx] / d[kz];
    r.Sy = d[ky] / d[kz];
    r.Sz = 1.0f / d[kz];
    return r;
}
// returns true on hit with 0 < t < 1e16; (u,v) follow optixGetTriangleBarycentrics:
// hit = (1-u-v) p0 + u p1 + v p2.
static bool ray_tri(const RaySetup &r, const float *p0, const float *p1, const float *p2, float &t, float &u, float &v) {
    const float A0 = p0[0] - r.o[0], A1 = p0[1] - r.o[1], A2 = p0[2] - r.o[2];
    const float B0 = p1[0] - r.o[0], B1 = p1[1] - r.o[1], B2 = p1[2] - r.o[2];
    const float C0 = p2[0] - r.o[0], C1 = p2[1] - r.o[1], C2 = p2[2] - r.o[2];
    const float A[3] = {A0, A1, A2}, B[3] = {B0, B1, B2}, C[3] = {C0, C1, C2};
    const float Ax = A[r.kx] - r.Sx * A[r.kz];
    const float Ay = A[r.ky] - r.Sy * A[r.kz];
    const float Bx = B[r.kx] - r.Sx * B[r.kz];
    const float By = B[r.ky] - r.Sy * B[r.kz];
    const float Cx = C[r.kx] - r.Sx * C[r.kz];
    const float Cy = C[r.ky] - r.Sy * C[r.kz];
    float U = Cx * By - Cy * Bx;
    float V = Ax * Cy - Ay * Cx;
    float W = Bx * Ay - By * Ax;
    if (U == 0.0f || V == 0.0f || W == 0.0f) {
        const double CxBy = (double)Cx * (double)By, CyBx = (double)Cy * (double)Bx;
        U = (float)(CxBy - CyBx);
        const double AxCy = (double)Ax * (double)Cy, AyCx = (double)Ay * (double)Cx;
        V = (float)(AxCy - AyCx);
        const double BxAy = (double)Bx * (double)Ay, ByAx = (double)By * (double)Ax;
        W = (float)(BxAy - ByAx);
    }
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return false;
    const float det = (U + V) + W;
    if (det == 0.0f) return false;
    const float Az = r.Sz * A[r.kz];
    const float Bz = r.Sz * B[r.kz];
    const float Cz = r.Sz * C[r.kz];
    const float Tn = (U * Az + V * Bz) + W * Cz;
    const float rcp = 1.0f / det;
    t = Tn * rcp;
    u = V * rcp;
    v = W * rcp;
    if (!(t > 0.0f && t < 1e16f)) return false;  // tmin=0, tmax=1e16 (optix_trace_rays.cu:284-285)
    return true;
}

// ---- mesh + a plain CPU BVH over the unique faces ---------------------------
// The BVH is NOT a restatement of anything in the reference (OptiX's GAS is
// opaque, tetrahedra_tracer.cpp:285-332); it only prunes the all-hits gather
// and is validated against brute force (accel=0) in tests/test_oracle.py.
struct BNode { float lo[3], hi[3]; uint32_t left, right, first, count; };
struct Mesh {
    uint32_t V = 0, T = 0, F = 0;
    std::vector<float> xyz;
    std::vector<uint32_t> cells;
    std::vector<U3> tri;
    std::vector<U2> tt;
    std::vector<BNode> nodes;
    std::vector<uint32_t> order;  // face ids in leaf order
    float absmax = 0.f;
};

static void face_bounds(const Mesh &m, uint32_t f, float *lo, float *hi) {
    const uint32_t ids[3] = {m.tri[f].x, m.tri[f].y, m.tri[f].z};
    for (int a = 0; a < 3; ++a) { lo[a] = 1e30f; hi[a] = -1e30f; }
    for (int k = 0; k < 3; ++k)
        for (int a = 0; a < 3; ++a) {
            float x = m.xyz[3 * (size_t)ids[k] + a];
            lo[a] = std::min(lo[a], x); hi[a] = std::max(hi[a], x);
        }
}
static uint32_t build_bvh(Mesh &m, std::vector<F3> &cent, uint32_t first, uint32_t count) {
    BNode n{};
    for (int a = 0; a < 3; ++a) { n.lo[a] = 1e30f; n.hi[a] = -1e30f; }
    float clo[3] = {1e30f, 1e30f, 1e30f}, chi[3] = {-1e30f, -1e30f, -1e30f};
    for (uint32_t i = first; i < first + count; ++i) {
        float lo[3], hi[3];
        face_bounds(m, m.order[i], lo, hi);
        const float c[3] = {cent[m.order[i]].x, cent[m.order[i]].y, cent[m.order[i]].z};
        for (int a = 0; a < 3; ++a) {
            n.lo[a] = std::min(n.lo[a], lo[a]); n.hi[a] = std::max(n.hi[a], hi[a]);
            clo[a] = std::min(clo[a], c[a]); chi[a] = std::max(chi[a], c[a]);
        }
    }
    n.first = first; n.count = count; n.left = n.right = EMPTY;
    const uint32_t id = (uint32_t)m.nodes.size();
    m.nodes.push_back(n);
    if (count > 4) {
        int ax = 0;
        if (chi[1] - clo[1] > chi[ax] - clo[ax]) ax = 1;
        if (chi[2] - clo[2] > chi[ax] - clo[ax]) ax = 2;
        const uint32_t mid = first + count / 2;
        std::nth_element(m.order.begin() + first, m.order.begin() + mid, m.order.begin() + first + count,
                         [&](uint32_t a, uint32_t b) { return (&cent[a].x)[ax] < (&cent[b].x)[ax]; });
        const uint32_t l = build_bvh(m, cent, first, mid - first);
        const uint32_t r = build_bvh(m, cent, mid, first + count - mid);
        m.nodes[id].left = l; m.nodes[id].right = r; m.nodes[id].count = 0;
    }
    return id;
}

struct Hit { float t; uint32_t face; float u, v; };
static inline bool hit_less(const Hit &a, const Hit &b) { return a.t < b.t || (a.t == b.t && a.face < b.face); }

static inline bool slab(const BNode &n, const float *o, const float *d, float pad) {
    float tn = 0.f, tf = 3.0e38f;
    for (int a = 0; a < 3; ++a) {
        const float lo = n.lo[a] - pad, hi = n.hi[a] + pad;
        if (d[a] == 0.0f) { if (o[a] < lo || o[a] > hi) return false; continue; }
        const double inv = 1.0 / (double)d[a];
        double t0 = ((double)lo - o[a]) * inv, t1 = ((double)hi - o[a]) * inv;
        if (t0 > t1) std::swap(t0, t1);
        if (t0 > tn) tn = (float)std::nextafter((float)t0, -3e38f);
        if (t1 < tf) tf = (float)std::nextafter((float)t1, 3e38f);
    }
    return tn <= tf;
}

static void gather_hits(const Mesh &m, const float *o, const float *d, int accel, std::vector<Hit> &hits) {
    hits.clear();
    const RaySetup rs = ray_setup(o, d);
    if (!rs.valid) return;
    auto test = [&](uint32_t f) {
        Hit h; h.face = f;
        if (ray_tri(rs, &m.xyz[3 * (size_t)m.tri[f].x], &m.xyz[3 * (size_t)m.tri[f].y], &m.xyz[3 * (size_t)m.tri[f].z], h.t, h.u, h.v))
            hits.push_back(h);
    };
    if (!accel || m.nodes.empty()) {
        for (uint32_t f = 0; f < m.F; ++f) test(f);
        return;
    }
    const float omax = std::max(std::fabs(o[0]), std::max(std::fabs(o[1]), std::fabs(o[2])));
    const float pad = 1e-4f * (omax + m.absmax);
    uint32_t stack[128]; int sp = 0; stack[sp++] = 0;
    while (sp) {
        const BNode &n = m.nodes[stack[--sp]];
        if (!slab(n, o, d, pad)) continue;
        if (n.left == EMPTY) { for (uint32_t i = 0; i < n.count; ++i) test(m.order[n.first + i]); }
        else { stack[sp++] = n.left; stack[sp++] = n.right; }
    }
}

// ---- optix_trace_rays.cu:22-37 ---------------------------------------------
static bool get_common_tetrahedra(const U2 &a, const U2 &b, uint32_t &tet) {
    if (a.x == b.x) { tet = a.x; return true; }
    else if (a.x == b.y) { tet = a.x; return true; }
    else if (a.y == b.x) { tet = a.y; return true; }
    else if (a.y == b.y) { tet = a.y; return true; }
    return false;
}
// ---- optix_trace_rays.cu:39-75 ---------------------------------------------
static U4 combine_indices(const U3 &id1, const U3 &id2, const F2 &in1, const F2 &in2, F3 &out1, F3 &out2) {
    U4 result{0, id1.x, id1.y, id1.z};
    out1 = F3{1.0f - in1.x - in1.y, in1.x, in1.y};
    const F3 out2_ref{1.0f - in2.x - in2.y, in2.x, in2.y};
    out2 = F3{0, 0, 0};
    const uint32_t a1[3] = {id1.x, id1.y, id1.z}, a2[3] = {id2.x, id2.y, id2.z};
    const float r2[3] = {out2_ref.x, out2_ref.y, out2_ref.z};
    float *o2 = &out2.x;
    for (int i = 0; i < 3; ++i) {
        bool was_break = false;
        for (int j = 0; j < 3; ++j) {
            if (a1[j] == a2[i]) { o2[j] = r2[i]; was_break = true; break; }
        }
        if (!was_break) result.x = a2[i];
    }
    return result;
}

// ---- optix_trace_rays.cu:78-108 (key widened to (t, face id), see header) ---
static void bitonic_sort(uint32_t N, F2 *dist, uint32_t *v1, F3 *v2 /* pairs: 2 per entry */) {
    uint32_t Nup2 = 1;
    while (Nup2 < N) Nup2 <<= 1;
    for (uint32_t i = N; i < Nup2; i++) { dist[i].x = 1e20f; v1[i] = EMPTY; }
    N = Nup2;
    auto greater = [&](uint32_t a, uint32_t b) {  // dist[a] > dist[b] in (t, face) order
        return dist[a].x > dist[b].x || (dist[a].x == dist[b].x && v1[a] > v1[b]);
    };
    for (uint32_t k = 2; k <= N; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1)
            for (uint32_t i = 0; i < N; i++) {
                const uint32_t ij = i ^ j;
                if (ij > i) {
                    const uint32_t ik = i & k;
                    if ((ik == 0 && greater(i, ij)) || (ik != 0 && greater(ij, i))) {
                        std::swap(dist[i], dist[ij]);
                        std::swap(v1[i], v1[ij]);
                        std::swap(v2[2 * i], v2[2 * ij]);
                        std::swap(v2[2 * i + 1], v2[2 * ij + 1]);
                    }
                }
            }
}

// ---- optix_trace_rays.cu:110-266 -------------------------------------------
// Operates in place on one ray's slice of the output buffers, like the reference.
static uint32_t post_process(const Mesh &m, uint32_t ray_len, uint32_t M, uint32_t *t, F2 *dl, F3 *bcs, U4 *vertex_indices) {
    size_t jc = 0;
    for (size_t j = 0; j + 1 < ray_len; ++j) {
        if (t[j] == EMPTY) continue;
        float dn = dl[j].x;
        bool clear_self = false;
        for (size_t offset = 1; j + offset < ray_len && (t[j + offset] == EMPTY || std::fabs(dl[j + offset].x - dn) < EPS); offset++) {
            uint32_t cell;
            if (t[j + offset] != EMPTY && get_common_tetrahedra(m.tt[t[j]], m.tt[t[j + offset]], cell)) {
                if (t[j] != t[j + offset]) clear_self = true;
                if (dl[j + offset].y > 0.0f) t[j + offset] = EMPTY;
                else dl[j + offset].y = 1.0f;
            }
        }
        if (clear_self) {
            if (dl[j].y > 0.0f) t[j] = EMPTY;
        }
        dl[j].y = 0.0f;
    }
    for (size_t j = 0; j < ray_len; ++j) {
        if (t[j] == EMPTY) continue;
        const U2 orig_tj = m.tt[t[j]];
        float dn = dl[j].x;
        size_t real_offset = 1;
        for (size_t offset = 1;
             j + offset < ray_len && (real_offset < 3 || t[j + offset] == EMPTY || std::fabs(dl[j + offset].x - dn) < EPS);
             offset++) {
            if (t[j + offset] == EMPTY) continue;
            uint32_t cell;
            if (get_common_tetrahedra(orig_tj, m.tt[t[j + offset]], cell)) {
                if (std::fabs(dl[j].x - dl[j + offset].x) >= EPS) {
                    const F2 coords0{bcs[2 * j].x, bcs[2 * j].y};
                    const F2 coords1{bcs[2 * (j + offset)].x, bcs[2 * (j + offset)].y};
                    const U3 tri0 = m.tri[t[j]], tri1 = m.tri[t[j + offset]];
                    const F2 d_out{dl[j].x, dl[j + offset].x};
                    F3 bc0, bc1;
                    const U4 vi = combine_indices(tri0, tri1, coords0, coords1, bc0, bc1);
                    bcs[2 * jc] = bc0;
                    bcs[2 * jc + 1] = bc1;
                    vertex_indices[jc] = vi;
                    dl[jc] = d_out;
                    t[jc] = cell;
                    jc++;
                }
                if (offset > 1) {
                    std::swap(dl[j + offset], dl[j + 1]);
                    std::swap(bcs[(j + offset) * 2], bcs[(j + 1) * 2]);
                    std::swap(t[j + offset], t[j + 1]);
                }
                break;
            }
            dn = dl[j + offset].x;
            real_offset++;
        }
    }
    for (size_t j = jc; j < M; ++j) {
        t[j] = EMPTY;
        vertex_indices[j] = U4{EMPTY, EMPTY, EMPTY, EMPTY};
        dl[j] = F2{0.f, 0.f};                       // pinned: reference leaves scratch here
        bcs[2 * j] = F3{0, 0, 0}; bcs[2 * j + 1] = F3{0, 0, 0};
    }
    return (uint32_t)jc;
}

template <class Fn>
static void parallel_for(uint32_t n, int nthreads, Fn fn) {
    if (nthreads <= 0) nthreads = (int)std::thread::hardware_concurrency();
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
    std::atomic<uint32_t> next{0};
    auto worker = [&]() {
        for (;;) {
            const uint32_t lo = next.fetch_add(16);
            if (lo >= n) break;
            const uint32_t hi = std::min(n, lo + 16);
            for (uint32_t i = lo; i < hi; ++i) fn(i);
        }
    };
    if (nthreads == 1) { worker(); return; }
    std::vector<std::thread> th;
    for (int i = 0; i < nthreads; ++i) th.emplace_back(worker);
    for (auto &x : th) x.join();
}

}  // namespace

extern "C" {

int orc_hardware_threads() { return (int)std::thread::hardware_concurrency(); }

void *orc_mesh_create(const float *xyz, uint32_t V, const uint32_t *cells, uint32_t T, int build_accel, int *err) {
    Mesh *m = new Mesh();
    m->V = V; m->T = T;
    m->xyz.assign(xyz, xyz + 3 * (size_t)V);
    m->cells.assign(cells, cells + 4 * (size_t)T);
    *err = build_faces(cells, T, m->tri, m->tt);
    if (*err) { delete m; return nullptr; }
    m->F = (uint32_t)m->tri.size();
    for (size_t i = 0; i < 3 * (size_t)V; ++i) m->absmax = std::max(m->absmax, std::fabs(xyz[i]));
    if (build_accel && m->F) {
        std::vector<F3> cent(m->F);
        m->order.resize(m->F);
        for (uint32_t f = 0; f < m->F; ++f) {
            float lo[3], hi[3];
            face_bounds(*m, f, lo, hi);
            cent[f] = F3{0.5f * (lo[0] + hi[0]), 0.5f * (lo[1] + hi[1]), 0.5f * (lo[2] + hi[2])};
            m->order[f] = f;
        }
        m->nodes.reserve(m->F);
        build_bvh(*m, cent, 0, m->F);
    }
    return m;
}
void orc_mesh_destroy(void *h) { delete (Mesh *)h; }
uint32_t orc_mesh_num_faces(void *h) { return ((Mesh *)h)->F; }
void orc_mesh_faces(void *h, uint32_t *tri, uint32_t *tt) {
    Mesh *m = (Mesh *)h;
    std::memcpy(tri, m->tri.data(), sizeof(U3) * m->F);
    std::memcpy(tt, m->tt.data(), sizeof(U2) * m->F);
}

// single ray/triangle test, exposed for the arithmetic-parity test of the CUDA kernel
int orc_ray_tri(const float *o, const float *d, const float *p0, const float *p1, const float *p2, float *tuv) {
    RaySetup rs = ray_setup(o, d);
    if (!rs.valid) return 0;
    return ray_tri(rs, p0, p1, p2, tuv[0], tuv[1], tuv[2]) ? 1 : 0;
}
// orc_ray_tri over n (ray, triangle) pairs: pair i tests ray ray[i] of o / d against the triangle with vertex ids tri[3i..3i+2] of xyz,
// in that winding; hit[i] = 0 / 1, tuv[3i..3i+2] = (t, u, v) on a hit.  The step loop of oracle/walk.py.
void orc_ray_tri_pairs(const float *xyz, const float *o, const float *d, uint32_t n, const uint32_t *ray, const uint32_t *tri, uint8_t *hit,
                       float *tuv, int nthreads) {
    parallel_for(n, nthreads, [&](uint32_t i) {
        const RaySetup rs = ray_setup(o + 3 * (size_t)ray[i], d + 3 * (size_t)ray[i]);
        float t = 0.f, u = 0.f, v = 0.f;
        hit[i] = rs.valid && ray_tri(rs, xyz + 3 * (size_t)tri[3 * (size_t)i], xyz + 3 * (size_t)tri[3 * (size_t)i + 1],
                                     xyz + 3 * (size_t)tri[3 * (size_t)i + 2], t, u, v) ? 1 : 0;
        tuv[3 * (size_t)i] = t; tuv[3 * (size_t)i + 1] = u; tuv[3 * (size_t)i + 2] = v;
    });
}

// raw sorted face hits (reference: trace_rays_triangles, optix_trace_rays_triangles.cu:49-114)
// outputs: num[R], faces[R,M], bary[R,M,2], dist[R,M], verts[R,M,3]; tails zero (py_binding.cpp:90-94)
int orc_trace_triangles(void *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *faces,
                        float *bary, float *dist, uint32_t *verts, int accel, int nthreads) {
    Mesh *m = (Mesh *)h;
    if (M == 0 || (M & (M - 1))) return -2;
    parallel_for(R, nthreads, [&](uint32_t i) {
        std::vector<Hit> hits;
        gather_hits(*m, o + 3 * (size_t)i, d + 3 * (size_t)i, accel, hits);
        std::sort(hits.begin(), hits.end(), hit_less);
        if (hits.size() > M - 1) hits.resize(M - 1);
        num[i] = (uint32_t)hits.size();
        for (uint32_t j = 0; j < M; ++j) {
            const size_t g = (size_t)i * M + j;
            if (j < hits.size()) {
                faces[g] = hits[j].face; dist[g] = hits[j].t; bary[2 * g] = hits[j].u; bary[2 * g + 1] = hits[j].v;
                verts[3 * g] = m->tri[hits[j].face].x; verts[3 * g + 1] = m->tri[hits[j].face].y; verts[3 * g + 2] = m->tri[hits[j].face].z;
            } else {
                faces[g] = 0; dist[g] = 0; bary[2 * g] = bary[2 * g + 1] = 0; verts[3 * g] = verts[3 * g + 1] = verts[3 * g + 2] = 0;
            }
        }
    });
    return 0;
}

// post-process alone on caller-supplied (unsorted) face hits of ONE ray: used to stress the
// pairing logic with ties/duplicates.  hits_* have n entries (n <= M-1).
int orc_post_process_one(void *h, uint32_t n, uint32_t M, const uint32_t *hit_face, const float *hit_t, const float *hit_uv,
                         uint32_t *num, uint32_t *cells, float *bary, float *dist, uint32_t *verts) {
    Mesh *m = (Mesh *)h;
    if (M == 0 || (M & (M - 1)) || n > M - 1) return -2;
    F2 *dl = (F2 *)dist; F3 *bcs = (F3 *)bary; U4 *vi = (U4 *)verts;
    std::memset(cells, 0, 4 * (size_t)M); std::memset(dist, 0, 8 * (size_t)M); std::memset(bary, 0, 24 * (size_t)M); std::memset(verts, 0, 16 * (size_t)M);
    for (uint32_t j = 0; j < n; ++j) { cells[j] = hit_face[j]; dl[j] = F2{hit_t[j], 0.f}; bcs[2 * j] = F3{hit_uv[2 * j], hit_uv[2 * j + 1], 0.f}; }
    bitonic_sort(n, dl, cells, bcs);
    *num = post_process(*m, n, M, cells, dl, bcs, vi);
    return 0;
}

// trace_rays (py_binding.cpp:41-76 -> tetrahedra_tracer.cpp:137-176 -> optix_trace_rays.cu:268-331)
// outputs: num[R] u32, cells[R,M] u32, bary[R,M,2,3] f32, dist[R,M,2] f32, verts[R,M,4] u32
int orc_trace(void *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells, float *bary,
              float *dist, uint32_t *verts, int accel, int nthreads) {
    Mesh *m = (Mesh *)h;
    if (M == 0 || (M & (M - 1))) return -2;  // py_binding.cpp:44-47
    parallel_for(R, nthreads, [&](uint32_t i) {
        std::vector<Hit> hits;
        gather_hits(*m, o + 3 * (size_t)i, d + 3 * (size_t)i, accel, hits);
        if (hits.size() > M - 1) {  // pinned cap: M-1 smallest keys (optix_trace_rays.cu:312-315 keeps an arbitrary M-1)
            std::partial_sort(hits.begin(), hits.begin() + (M - 1), hits.end(), hit_less);
            hits.resize(M - 1);
        }
        uint32_t *t = cells + (size_t)i * M;
        F2 *dl = (F2 *)dist + (size_t)i * M;
        F3 *bcs = (F3 *)bary + (size_t)i * M * 2;
        U4 *vi = (U4 *)verts + (size_t)i * M;
        std::memset(t, 0, 4 * (size_t)M); std::memset(dl, 0, 8 * (size_t)M); std::memset(bcs, 0, 24 * (size_t)M); std::memset(vi, 0, 16 * (size_t)M);
        const uint32_t p0 = (uint32_t)hits.size();
        for (uint32_t j = 0; j < p0; ++j) {  // __anyhit__ms, optix_trace_rays.cu:323-326
            t[j] = hits[j].face; dl[j] = F2{hits[j].t, 0.f}; bcs[2 * j] = F3{hits[j].u, hits[j].v, 0.f};
        }
        bitonic_sort(p0, dl, t, bcs);
        num[i] = post_process(*m, p0, M, t, dl, bcs, vi);
    });
    return 0;
}

// find_matched_cells (tetrahedra_tracer.cu:115-161) + defaults of py_binding.cpp:188-191
// mask is uint8 (torch bool).  IEEE arithmetic, individually rounded ops (the reference is
// compiled --use_fast_math, cmake/FindTorch.cmake:33; differences are <= a few ulp).
void orc_match(uint32_t R, uint32_t S, uint32_t M, const uint32_t *num, const uint32_t *cells, const float *dist_in,
               const float *bary_in, const float *sample_d, const uint32_t *verts_in, uint32_t *cell_out, uint32_t *verts_out,
               uint8_t *mask_out, float *bary_out, int nthreads) {
    parallel_for(R, nthreads, [&](uint32_t i) {
        for (uint32_t j = 0; j < S; ++j) {
            const size_t g = (size_t)i * S + j;
            mask_out[g] = 0; cell_out[g] = EMPTY;
            for (int k = 0; k < 4; ++k) verts_out[4 * g + k] = EMPTY;
            for (int k = 0; k < 3; ++k) bary_out[3 * g + k] = 0.f;
        }
        uint32_t p = 0;
        const F2 *hd = (const F2 *)dist_in + (size_t)i * M;
        for (uint32_t j = 0; j < S; ++j) {
            const size_t g = (size_t)i * S + j;
            const float cd = sample_d[g];
            while (p < num[i] && hd[p].y < cd) p++;
            if (p >= num[i]) break;
            const F2 h = hd[p];
            if (h.x <= cd) {
                mask_out[g] = 1;
                cell_out[g] = cells[(size_t)i * M + p];
                for (int k = 0; k < 4; ++k) verts_out[4 * g + k] = verts_in[((size_t)i * M + p) * 4 + k];
                const float mult = (cd - h.x) / (h.y - h.x);
                const float om = 1.0f - mult;
                const float *c1 = bary_in + ((size_t)i * M + p) * 6, *c2 = c1 + 3;
                for (int k = 0; k < 3; ++k) bary_out[3 * g + k] = om * c1[k] + mult * c2[k];
            }
        }
    });
}

// interpolate_values<D> (tetrahedra_tracer.cu:195-221); result laid out [N, C] (the value the
// reference returns after .moveaxis(0,-1), py_binding.cpp:330).  field is [C, V].
// "out += w * f" is an FFMA in the reference SASS (nvcc -fmad default) -> fmaf here.
void orc_interp_fwd(uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *vi, const float *w, const float *field,
                    float *out, int nthreads) {
    parallel_for(N, nthreads, [&](uint32_t i) {
        for (uint32_t j = 0; j < C; ++j) {
            float o = 0.f, weight = 0.f;
            for (uint32_t k = 0; k + 1 < D; ++k) {
                const float wk = w[(size_t)i * (D - 1) + k];
                const uint32_t v = vi[(size_t)i * D + k + 1];
                if (v != EMPTY) o = std::fmaf(wk, field[(size_t)j * V + v], o);
                weight += wk;
            }
            if (vi[(size_t)i * D] != EMPTY) o = std::fmaf(1.0f - weight, field[(size_t)j * V + vi[(size_t)i * D]], o);
            out[(size_t)i * C + j] = o;
        }
    });
}
// interpolate_values_backward<D> (tetrahedra_tracer.cu:223-248); grad_in [N, C]; out [C, V] zero-init
// (py_binding.cpp:360).  Serial accumulation in sample order (the reference's atomics are unordered).
void orc_interp_bwd(uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *vi, const float *w, const float *grad_in,
                    float *grad_field) {
    std::memset(grad_field, 0, sizeof(float) * (size_t)C * V);
    for (uint32_t i = 0; i < N; ++i)
        for (uint32_t j = 0; j < C; ++j) {
            const float g = grad_in[(size_t)i * C + j];
            float weight = 0.f;
            for (uint32_t k = 0; k + 1 < D; ++k) {
                const float wk = w[(size_t)i * (D - 1) + k];
                const uint32_t v = vi[(size_t)i * D + k + 1];
                if (v != EMPTY) grad_field[(size_t)j * V + v] += wk * g;
                weight += wk;
            }
            if (vi[(size_t)i * D] != EMPTY) grad_field[(size_t)j * V + vi[(size_t)i * D]] += (1.0f - weight) * g;
        }
}

// find_tetrahedra (optix_find_tetrahedra.cu:84-213): two closest-hit rays +x / -x.
// outputs: tet[N] u32 (EMPTY if none), bary[N,3], verts[N,4] (zero when not found, py_binding.cpp:121-128)
void orc_find_tetrahedra(void *h, const float *pos, uint32_t N, uint32_t *tet, float *bary, uint32_t *verts, int accel, int nthreads) {
    Mesh *m = (Mesh *)h;
    parallel_for(N, nthreads, [&](uint32_t i) {
        const float *o = pos + 3 * (size_t)i;
        const float dp[3] = {1.f, 0.f, 0.f}, dm[3] = {-1.f, 0.f, 0.f};
        std::vector<Hit> hp, hm;
        gather_hits(*m, o, dp, accel, hp);
        gather_hits(*m, o, dm, accel, hm);
        tet[i] = EMPTY;
        for (int k = 0; k < 3; ++k) bary[3 * (size_t)i + k] = 0.f;
        for (int k = 0; k < 4; ++k) verts[4 * (size_t)i + k] = 0;
        if (hp.empty() || hm.empty()) return;
        const Hit a = *std::min_element(hp.begin(), hp.end(), hit_less);
        const Hit b = *std::min_element(hm.begin(), hm.end(), hit_less);
        uint32_t cell;
        if (get_common_tetrahedra(m->tt[a.face], m->tt[b.face], cell)) {
            F3 c0, c1;
            const U4 vi = combine_indices(m->tri[a.face], m->tri[b.face], F2{a.u, a.v}, F2{b.u, b.v}, c0, c1);
            const float mm = b.t / (a.t + b.t);
            const float om = 1.0f - mm;
            bary[3 * (size_t)i + 0] = c0.x * mm + c1.x * om;
            bary[3 * (size_t)i + 1] = c0.y * mm + c1.y * om;
            bary[3 * (size_t)i + 2] = c0.z * mm + c1.z * om;
            verts[4 * (size_t)i + 0] = vi.x; verts[4 * (size_t)i + 1] = vi.y; verts[4 * (size_t)i + 2] = vi.z; verts[4 * (size_t)i + 3] = vi.w;
            tet[i] = cell;
        }
    });
}

}  // extern "C"
