// tn_common.cuh -- shared declarations of the H100-native Tetra-NeRF hot path (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>

#include "../../include/tetranerf_b200.h"

#define TN_EMPTY 0xFFFFFFFFu

namespace tn {

void set_error(const std::string &msg);
int fail(int code, const std::string &msg);

#define TN_CUDA(expr)                                                                                       \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e != cudaSuccess)                                                                              \
            return tn::fail(TN_ERR_CUDA, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + \
                                             __FILE__ + ":" + std::to_string(__LINE__) + ")");              \
    } while (0)

// returns a non-zero TN_* code of expr to the caller
#define TN_TRY(...)                              \
    do {                                         \
        const int _rc = (__VA_ARGS__);           \
        if (_rc != TN_OK) return _rc;            \
    } while (0)

// bytes held by every DevArray of the process (tn_debug_device_bytes)
inline std::atomic<uint64_t> g_device_bytes{0};

// The owner of every device buffer of the library (DESIGN.md §3): grow-only, freed by its destructor.  `cap` (elements) is set only
// after a successful allocation, so a failed grow leaves {nullptr, 0} and the next call allocates again.  No device is recorded: every
// owner is destroyed, and every grow runs, under the tracer's DeviceGuard.  No conversion to T *: call sites write `.p`.
template <typename T>
struct DevArray {
    T *p = nullptr;
    size_t cap = 0;

    DevArray() = default;
    DevArray(const DevArray &) = delete;
    DevArray &operator=(const DevArray &) = delete;
    DevArray(DevArray &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevArray &operator=(DevArray &&o) noexcept {
        if (this != &o) {
            release();
            p = o.p; cap = o.cap;
            o.p = nullptr; o.cap = 0;
        }
        return *this;
    }
    ~DevArray() { release(); }

    // at least n elements (rounded up to 256 bytes); the contents are not kept.  The old allocation is freed first, so the peak is the
    // larger of the two, never their sum.
    int grow(size_t n) {
        if (n <= cap) return TN_OK;
        release();
        const size_t bytes = (n * sizeof(T) + 255) / 256 * 256;
        void *q = nullptr;
        TN_CUDA(cudaMalloc(&q, bytes));
        p = static_cast<T *>(q);
        cap = bytes / sizeof(T);
        g_device_bytes += cap * sizeof(T);
        return TN_OK;
    }

  private:
    void release() {
        if (!p) return;
        cudaFree(p);
        g_device_bytes -= cap * sizeof(T);
        p = nullptr; cap = 0;
    }
};

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// ---- acceleration structure: implicit 8-ary BVH over Morton-sorted tetrahedra ----------------
// Level 0 = one node per tetrahedron (sorted order); node i of level l+1 bounds nodes 8i..8i+7 of
// level l (256 contiguous bytes).  A node is 32 bytes: (lo.x lo.y lo.z hi.x)(hi.y hi.z - -).
// All levels live in one array.
constexpr int TN_MAX_LEVELS = 16;
constexpr uint32_t TN_FAN = 8, TN_FAN_LOG2 = 3;
struct BvhLevels {
    uint32_t count[TN_MAX_LEVELS];
    uint32_t offset[TN_MAX_LEVELS];  // in nodes
    int nlevels;                     // top level (nlevels-1) has exactly 1 node
};

// 64-byte leaf record of one tetrahedron, in sorted (Morton) order:
//   v[j] = (x, y, z, bits(face_id_j | hull<<30 | owner<<31)) ; face j is opposite vertex j and is stored in the
//   reference winding (v[(j+1)%4], v[(j+2)%4], v[(j+3)%4]) (src/tetrahedra_tracer.cpp:54-57) iff this
//   tetrahedron is the face's first owner.  hull = the face has a single owner.
struct LeafRec {
    float4 v[4];
};
#define TN_FACE_MASK 0x3FFFFFFFu
#define TN_FACE_HULL 0x40000000u
#define TN_FACE_OWNER 0x80000000u

// 128-byte (one cache line) record of one tetrahedron, indexed by tetrahedron id, for the adjacency walk:
struct WalkRec {
    float4 v[4];       // as LeafRec
    uint32_t nbr[4];   // tetrahedron across face j (TN_EMPTY on the hull)
    uint32_t vid[4];   // the cell's vertex ids
    uint32_t map[4];   // map[jin]: for each exit face jout 6 bits = three 2-bit codes: which exit barycentric (0: 1-u-v, 1: u, 2: v,
                       // 3: none -> 0) belongs to slot q of the ENTRY face's winding (combine_indices, optix_trace_rays.cu:39-75)
    uint32_t wind;     // 4 x 6 bits: stored winding of face j as three local vertex indices (2 bits each, a | b<<2 | c<<4)
    uint32_t perm;     // 4 x 8 bits: record vertex order when entering through face jin: (jin, wind[jin].a, .b, .c) as local indices
    uint32_t pad[2];
};
static_assert(sizeof(WalkRec) == 128, "WalkRec is one 128-byte line");

struct Mesh {
    const float *xyz = nullptr;      // borrowed, [V,3]
    const uint32_t *cells = nullptr; // borrowed, [T,4]
    uint32_t V = 0, T = 0, F = 0;
    DevArray<uint4> tri;             // [F]: stored winding (v0,v1,v2, 0)   (triangle_indices)
    DevArray<uint2> tt;              // [F]: (first owner, second owner|E)   (triangle_tetrahedra)
    DevArray<float4> nodes;          // BVH nodes, 2 float4 per node
    DevArray<LeafRec> leaves;        // [T]
    DevArray<uint32_t> leaf_tet;     // [T] sorted position -> tetrahedron id
    // adjacency walk (fast path of trace_rays): valid when `walkable`
    DevArray<WalkRec> walk;          // [T]
    DevArray<float4> hull_nodes;     // BVH over the tetrahedra that own a hull face
    DevArray<LeafRec> hull_leaves;   // [H]
    DevArray<uint32_t> hull_tet;     // [H] sorted position -> tetrahedron id
    BvhLevels hull_lv{};
    uint32_t H = 0;
    bool walkable = false;           // conforming mesh with a convex hull (always true for a Delaunay triangulation), and after a
                                     // refit (tn_update_vertices) still convex and unfolded
    // hull edges of a mesh that was walkable at load (walk.p != nullptr), sorted by (a, b): what the convexity test of a refit reads
    DevArray<unsigned long long> hull_ekey;  // [hull_ne] (a << 32 | b), a < b
    DevArray<uint32_t> hull_eface;           // [hull_ne] the hull face of each edge entry
    uint32_t hull_ne = 0;
    BvhLevels lv{};
    float absmax = 0.f;              // max |coordinate| over the vertices
};

struct RenderState;
struct SurfaceState;

}  // namespace tn

struct tn_tracer {
    int device = 0;
    tn::Mesh mesh;
    tn::DevArray<int> d_flags;  // [0] traversal-stack overflow count, [2] number of rays deferred to the large-buffer pass
    tn::DevArray<uint32_t> d_ovf_list;  // rays deferred by phase 1 of trace_rays / listed by the walk for the exact stage
    tn::DevArray<unsigned long long> d_walk_keys;  // [R, M] (t, face) keys written by the adjacency walk
    // trace_rays picks between bit-identical implementations by batch size:
    //   warp-per-ray all-hits BVH gather   <- below walk_quad_min_rays (latency of the few rays in flight dominates)
    //   walk, 8 rays per warp ("quad")     <- [walk_quad_min_rays, walk_min_rays)  (speculative record loads up to walk_quad_spec_max_rays,
    //                                         prefetches above)
    //   walk, 1 ray per warp ("solo")      (the quad walk launched with one quad per warp; range empty by default, for tests)
    //   walk, 32 rays per warp             <- >= walk_min_rays (fewest instructions per ray: only pays off once the machine is full
    //                                         several times over)
    uint32_t walk_min_rays = 1u << 20;
    uint32_t walk_solo_min_rays = 1, walk_solo_max_rays = 0;
    uint32_t walk_quad_min_rays = 3584, walk_quad_max_rays = 0xFFFFFFFFu;
    uint32_t walk_quad_spec_max_rays = 65536;  // quad and solo walks: batches up to this size load the candidate next records speculatively (tn_walk.cu)
    uint64_t launches = 0;
    uint64_t mesh_gen = 0;  // a fresh next_generation() on every tn_load_tetrahedra / tn_update_vertices (a surface extraction records it)
    tn::DevArray<uint32_t> d_refit;  // 16 words of tn_update_vertices scratch: flags, counts and bounds, read back once per refit
    tn::RenderState *render = nullptr;
    tn::SurfaceState *surface = nullptr;
    // vertex adjacency of the loaded mesh (tn_field_smoothness, tn_smoothness.cu): built on the first call after a tn_load_tetrahedra,
    // kept by tn_update_vertices (same cells); nothing is allocated before that first call
    bool adj_valid = false;
    uint32_t adj_E = 0;                    // unique undirected edges
    tn::DevArray<uint32_t> adj_off;        // [V+1] CSR row offsets
    tn::DevArray<uint32_t> adj_nbr;        // [2E] neighbours, each row ascending
    tn::DevArray<double> adj_part;         // one partial sum per block of the smoothness kernel
    // scratch of tn_guard_vertex_step (tn_fold_guard.cu), grown on its first call and kept
    tn::DevArray<uint4> guard_face;        // [F] per interior face certified at P0: (a, b, c, p); a = TN_EMPTY otherwise
    tn::DevArray<uint32_t> guard_faceq;    // [F] its other opposite vertex q
    tn::DevArray<float> guard_p1;          // [3V] the proposed positions
    tn::DevArray<uint8_t> guard_vtx;       // [3V] per vertex: exponent state, failure mark, changed in the last round
    tn::DevArray<uint32_t> guard_counts;   // [8] flags and counters, read back once per round
};

namespace tn {
int build_mesh(tn_tracer *h, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, cudaStream_t s);
// device-built face / adjacency tables (tn_faces.cu)
struct FaceTables {
    DevArray<uint4> tri;         // [F] stored winding (reference numbering), padded
    DevArray<uint2> tt;          // [F] (first owner, second owner or TN_EMPTY)
    DevArray<uint4> tet_faces;   // [T] face id | TN_FACE_OWNER | TN_FACE_HULL of the face opposite local vertex j
    DevArray<uint4> nbr;         // [T] neighbour across each face
    DevArray<uint32_t> wind;     // [T] stored windings as local vertex indices (2 bits x 3 x 4)
    DevArray<uint32_t> hull_list;  // [H] tetrahedra owning a hull face, ascending
    uint32_t F = 0, H = 0;
    bool walkable = false;       // the hull is a closed convex surface
    uint32_t folded = 0;         // walkable: interior faces the fold test (k_fold_faces) does not certify unfolded
    DevArray<unsigned long long> hull_ekey;  // walkable: the sorted hull edges (Mesh::hull_ekey / hull_eface)
    DevArray<uint32_t> hull_eface;
    uint32_t hull_ne = 0;
};
int build_faces_device(const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, cudaStream_t s, FaceTables &out, int *launches);
// position-dependent tests of a refit (tn_faces.cu), on the loaded mesh's kept tables at positions d_xyz; stream-ordered.
// d_counts[0] |= 4 if the hull is not convex (the load's test, on its sorted hull edges); d_counts[1] += number of folded interior faces
int launch_refit_checks(const tn_tracer *h, const float *d_xyz, uint32_t *d_counts, cudaStream_t s);
// tn_update_vertices (tn_build.cu)
int refit_mesh(tn_tracer *h, const float *d_xyz, uint32_t V, cudaStream_t s, uint32_t *folded_faces, int *walkable);
void free_render(tn_tracer *h);
void free_surface(tn_tracer *h);
// a value no earlier call returned (tn_render.cu): the generation of a field, weights or mesh
uint64_t next_generation();
// The field shadow `fshadow` [V,64] (tn_render_set_field) keeps one 256-byte row per vertex with its features in fragment order: in
// each 16-feature block b (one k-step of the MLP's layer 0), feature 16b + 8h + 2t + e (h, e in {0, 1}, t in 0..3) is stored at
// 16b + 4t + 2h + e.  The four features thread t of a wgmma A fragment row needs in k-step b, the column pairs 2t and 8 + 2t, are then
// one 16-byte load at 16b + 4t, and column pairs stay adjacent.  This is the only statement of the layout: the writer and every
// reader of the shadow go through it.  (The gradient shadow `gshadow` keeps the canonical order.)
__host__ __device__ constexpr uint32_t field_pos(uint32_t f) { return (f & ~15u) | ((f & 6u) << 1) | ((f >> 2) & 2u) | (f & 1u); }
// the field and weights of the fused render as the surface extraction reads them; TN_ERR_STATE unless both were set
struct RenderInputs {
    const float *fshadow;   // [V,64] in fragment order (field_pos)
    uint32_t V;
    const uint8_t *wimg;    // bf16 hi/lo weight image of k_mlp<*, 3>
    const float *bias, *head, *w4dir;
    uint64_t gen;           // generation of field + weights
};
int render_inputs(tn_tracer *h, RenderInputs *out);
// the fused render's field shadow [V,64] (fragment order, field_pos) and its V; TN_ERR_STATE if tn_render_set_field never ran
int field_shadow(const tn_tracer *h, const float **fshadow, uint32_t *V);
// the normal map of a fused render (tn_normals.cu), launched after its composite on the render's own buffers
struct NormalsLaunch {
    const uint32_t *n_active, *ray_list;  // active rays, slot -> ray
    uint32_t *tile_ctr;                   // zeroed device counter
    uint32_t S, R, prec;                  // samples per ray of the pass that gives the colours, rays, operand precision (2 / 3)
    const uint4 *vi;                      // [n_active*S] matched vertex ids of that pass
    const float *bary;                    // [n_active*S,3]
    const float *ebins;                   // [n_active,S+1] its euclidean bin edges
    const float *out_f;                   // [n_active*S] (sigma, r, g, b)
    const float *fshadow;                 // [V,64] in fragment order (field_pos)
    const uint8_t *wimg;                  // weight image of k_mlp<*, prec>
    const float *bias, *head;
    const float *xyz;                     // [V,3] mesh vertex positions
    float4 *grad;                         // out: [n_active*S] density gradient (x, y, z, 0)
    float *normals;                       // out: [R,3]
};
int launch_normals(const NormalsLaunch &a, int sms, cudaStream_t s);
// gradients of a training step at the ray origins and directions (tn_ray_grads.cu), launched at the end of its backward
struct RayGradsLaunch {
    const uint32_t *n_active, *ray_list;  // active rays, slot -> ray
    uint32_t S, R;                        // fine samples per ray, rays of the forward
    const float *ebins;                   // [n_active,S+1] euclidean bin edges of the fine pass
    const uint4 *vi;                      // [n_active*S] matched vertex ids
    const float *dx;                      // [n_active*S,64] gradient at the interpolated features
    const float *fshadow;                 // [V,64] in fragment order (field_pos)
    const float *xyz;                     // [V,3] mesh vertex positions
    const float *enc;                     // [n_active,27] encoded directions (entries 24..26: the direction itself)
    const float *g_dirbias;               // [n_active,128] gradient at the per-ray direction bias
    const float *w4dir;                   // [128][27] W4[:, :27]
    float4 *gx;                           // out: [n_active*S] dL/dx per sample (x, y, z, 0)
    float *grad_o, *grad_d;               // out: [R,3] each, or nullptr
};
int launch_ray_grads(const RayGradsLaunch &a, cudaStream_t s);
// gradient of a training step at the mesh vertex positions (tn_vertex_grads.cu), launched after k_ray_grads on its per-sample dL/dx
struct VertexGradsLaunch {
    const uint32_t *n_active;             // active rays
    uint32_t S, R, V;                     // fine samples per ray, rays of the forward, mesh vertices
    const uint4 *vi;                      // [n_active*S] matched vertex ids
    const float *bary;                    // [n_active*S,3] their weights on v1..v3
    const float4 *gx;                     // [n_active*S] dL/dx per sample (k_ray_grads)
    const uint32_t *keys, *vals;          // deterministic mode: the (vertex, row * 4 + k) pairs stably sorted by vertex, n of them;
    uint32_t n;                           //   nullptr = default mode (float reductions)
    float *grad_xyz;                      // out: [V,3]
};
int launch_vertex_grads(const VertexGradsLaunch &a, cudaStream_t s);
// gradients of a training step at the background map and, through it, at the ray directions (tn_background.cu; DESIGN §4.16), launched
// after k_ray_grads, whose direction gradients it adds to
struct BackgroundGradsLaunch {
    uint32_t R, H, W;                     // rays of the forward, map rows / columns
    const float *map;                     // [H,W,3]
    const float *dirs;                    // [R,3] the forward's ray directions
    const float *s;                       // [R,3] grad_rgb (1 - accumulation) per ray (grad_rgb on empty rays)
    bool det;                             // deterministic mode: a stable sort by texel and per-texel sums in ray order
    uint32_t *keys, *vals;                // deterministic mode: [2][4R] sort buffers
    float *grad_map;                      // out: [H,W,3], or nullptr
    float *grad_d;                        // in / out: [R,3] += (d bg / d d)^T s, or nullptr
};
// tmp: the temporary storage of the deterministic mode's sort, grown as it needs
int launch_background_grads(const BackgroundGradsLaunch &a, DevArray<uint8_t> &tmp, cudaStream_t s);
int launch_walk(tn_tracer *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells, float *bary,
                float *dist, uint32_t *verts, unsigned long long *keys, uint32_t *list, uint32_t *list_count, int kind, cudaStream_t s);
int launch_tail_fill(tn_tracer *h, uint32_t R, uint32_t M, const uint32_t *num, uint32_t *cells, float *bary, float *dist, uint32_t *verts,
                     cudaStream_t s);
int launch_prefetch(tn_tracer *h, const void *const *extra, const size_t *extra_bytes, int nextra, cudaStream_t s);
}  // namespace tn

// =================================================================================================
// Device arithmetic shared by every kernel that intersects rays with faces.  The op sequence is
// the contract with oracle/tetra_oracle.cpp (ray_setup / ray_tri): every operation individually
// rounded to nearest-even, no FMA contraction -> bit-identical t,u,v on CPU and GPU.
// =================================================================================================
#ifdef __CUDACC__
namespace tn {

struct RaySetup {
    float ox, oy, oz;
    float Sx, Sy, Sz;
    int kx, ky, kz;
    bool valid;
};

// branch-free 3-way select (k is a per-ray constant; nested ternaries on floats tend to become divergent branches)
__device__ __forceinline__ float sel3(int k, float x, float y, float z) {
    float r;
    asm("{\n\t.reg .pred p1, p2;\n\tsetp.eq.s32 p1, %4, 1;\n\tsetp.eq.s32 p2, %4, 2;\n\tselp.f32 %0, %2, %1, p1;\n\tselp.f32 %0, %3, %0, p2;\n\t}"
        : "=&f"(r) : "f"(x), "f"(y), "f"(z), "r"(k));
    return r;
}

__device__ __forceinline__ RaySetup ray_setup(float ox, float oy, float oz, float dx, float dy, float dz) {
    RaySetup r;
    r.ox = ox; r.oy = oy; r.oz = oz;
    int kz = 0;
    float m = fabsf(dx);
    if (fabsf(dy) > m) { kz = 1; m = fabsf(dy); }
    if (fabsf(dz) > m) { kz = 2; }
    int kx = (kz + 1) % 3, ky = (kx + 1) % 3;
    const float dk = sel3(kz, dx, dy, dz);
    if (dk < 0.0f) { int t = kx; kx = ky; ky = t; }
    r.kx = kx; r.ky = ky; r.kz = kz;
    r.valid = (dk != 0.0f) && isfinite(dx) && isfinite(dy) && isfinite(dz);
    r.Sx = __fdiv_rn(sel3(kx, dx, dy, dz), dk);
    r.Sy = __fdiv_rn(sel3(ky, dx, dy, dz), dk);
    r.Sz = __fdiv_rn(1.0f, dk);
    return r;
}

// sheared coordinates of one vertex relative to the ray (x, y in the projection plane, z along the ray)
struct Sheared { float x, y, z; };
__device__ __forceinline__ Sheared shear(const RaySetup &r, float px, float py, float pz) {
    const float a0 = __fsub_rn(px, r.ox), a1 = __fsub_rn(py, r.oy), a2 = __fsub_rn(pz, r.oz);
    const float ax = sel3(r.kx, a0, a1, a2), ay = sel3(r.ky, a0, a1, a2), az = sel3(r.kz, a0, a1, a2);
    Sheared s;
    s.x = __fsub_rn(ax, __fmul_rn(r.Sx, az));
    s.y = __fsub_rn(ay, __fmul_rn(r.Sy, az));
    s.z = __fmul_rn(r.Sz, az);
    return s;
}

// watertight ray/triangle test on sheared vertices A,B,C (stored winding).  (u,v) as
// optixGetTriangleBarycentrics: hit = (1-u-v) A + u B + v C.  Accepts 0 < t < 1e16.
__device__ __forceinline__ bool tri_test(const Sheared &A, const Sheared &B, const Sheared &C, float &t, float &u, float &v) {
    float U = __fsub_rn(__fmul_rn(C.x, B.y), __fmul_rn(C.y, B.x));
    float V = __fsub_rn(__fmul_rn(A.x, C.y), __fmul_rn(A.y, C.x));
    float W = __fsub_rn(__fmul_rn(B.x, A.y), __fmul_rn(B.y, A.x));
    if (U == 0.0f || V == 0.0f || W == 0.0f) {
        U = __double2float_rn(__dsub_rn(__dmul_rn((double)C.x, (double)B.y), __dmul_rn((double)C.y, (double)B.x)));
        V = __double2float_rn(__dsub_rn(__dmul_rn((double)A.x, (double)C.y), __dmul_rn((double)A.y, (double)C.x)));
        W = __double2float_rn(__dsub_rn(__dmul_rn((double)B.x, (double)A.y), __dmul_rn((double)B.y, (double)A.x)));
    }
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return false;
    const float det = __fadd_rn(__fadd_rn(U, V), W);
    if (det == 0.0f) return false;
    const float Tn = __fadd_rn(__fadd_rn(__fmul_rn(U, A.z), __fmul_rn(V, B.z)), __fmul_rn(W, C.z));
    const float rcp = __fdiv_rn(1.0f, det);
    t = __fmul_rn(Tn, rcp);
    u = __fmul_rn(V, rcp);
    v = __fmul_rn(W, rcp);
    return (t > 0.0f && t < 1e16f);
}

// The same test without early exits (identical operation sequence for every value that is returned when the result is `true`):
// eight rays share a warp in the quad walk, where every data-dependent branch costs a divergence / reconvergence pair per step.
// The double-precision recomputation of zero edge functions stays a (rare) branch.
__device__ __forceinline__ bool tri_test_nobranch(const Sheared &A, const Sheared &B, const Sheared &C, float &t, float &u, float &v) {
    float U = __fsub_rn(__fmul_rn(C.x, B.y), __fmul_rn(C.y, B.x));
    float V = __fsub_rn(__fmul_rn(A.x, C.y), __fmul_rn(A.y, C.x));
    float W = __fsub_rn(__fmul_rn(B.x, A.y), __fmul_rn(B.y, A.x));
    if (U == 0.0f || V == 0.0f || W == 0.0f) {
        U = __double2float_rn(__dsub_rn(__dmul_rn((double)C.x, (double)B.y), __dmul_rn((double)C.y, (double)B.x)));
        V = __double2float_rn(__dsub_rn(__dmul_rn((double)A.x, (double)C.y), __dmul_rn((double)A.y, (double)C.x)));
        W = __double2float_rn(__dsub_rn(__dmul_rn((double)B.x, (double)A.y), __dmul_rn((double)B.y, (double)A.x)));
    }
    const bool mixed = (U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f);
    const float det = __fadd_rn(__fadd_rn(U, V), W);
    const float Tn = __fadd_rn(__fadd_rn(__fmul_rn(U, A.z), __fmul_rn(V, B.z)), __fmul_rn(W, C.z));
    const float rcp = __fdiv_rn(1.0f, det);
    t = __fmul_rn(Tn, rcp);
    u = __fmul_rn(V, rcp);
    v = __fmul_rn(W, rcp);
    return !mixed && det != 0.0f && t > 0.0f && t < 1e16f;
}

// conservative ray/AABB slab test on a 32-byte BVH node (a = lo.xyz hi.x, b = hi.yz); NaN-safe via fminf/fmaxf
__device__ __forceinline__ bool slab(const float4 a, const float4 b, float ox, float oy, float oz, float ix, float iy, float iz,
                                     float pad) {
    const float t0x = (a.x - pad - ox) * ix, t1x = (a.w + pad - ox) * ix;
    const float t0y = (a.y - pad - oy) * iy, t1y = (b.x + pad - oy) * iy;
    const float t0z = (a.z - pad - oz) * iz, t1z = (b.y + pad - oz) * iz;
    const float tn = fmaxf(fmaxf(fminf(t0x, t1x), fminf(t0y, t1y)), fmaxf(fminf(t0z, t1z), 0.0f));
    const float tf = fminf(fminf(fmaxf(t0x, t1x), fmaxf(t0y, t1y)), fmaxf(t0z, t1z));
    return tn <= tf;
}

// optix_trace_rays.cu:22-37
__device__ __forceinline__ bool common_tet(const uint2 a, const uint2 b, uint32_t &tet) {
    if (a.x == b.x) { tet = a.x; return true; }
    if (a.x == b.y) { tet = a.x; return true; }
    if (a.y == b.x) { tet = a.y; return true; }
    if (a.y == b.y) { tet = a.y; return true; }
    return false;
}

}  // namespace tn
#endif
