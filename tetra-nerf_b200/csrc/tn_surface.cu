// tn_surface.cu -- the density iso-surface {sigma = level} of the field as a triangle mesh, by marching tetrahedra on the tracer's own
// Delaunay mesh (DESIGN.md §4.6).  The field is linear inside each tetrahedron, so the surface needs no grid: one output vertex per
// mesh edge whose endpoints lie on different sides of the level, one or two triangles per tetrahedron with mixed vertices.
//   vertex densities   k_mlp<false,3> over the V vertices (S = 1, vi = (v,v,v,v), weights 0)
//   cases / faces      k_tet_case -> exclusive scan of (edges, triangles) per tetrahedron -> k_tet_edges -> radix sort + unique of
//                      the crossing-edge keys (= the output vertices, in key order) -> k_faces (binary search of each corner's edge)
//   refinement         two rounds of k_mlp<false,3> with one 64-sample tile per crossing edge (vi = (a,b,b,b), weights (s,0,0)),
//                      each followed by k_bracket; the second one places the vertex by linear interpolation in a 1/4096 bracket
//   normals            face normals, stable radix sort of (vertex, face) pairs, per-vertex sums in face order (k_vertex_normals)
//   colours            direction bias b4 + W4[:, :27] enc(-n) per vertex, then k_mlp<true,3> at the vertex's features (S = 1)
// Every MLP evaluation is bf16x3, whatever tn_render_set_mlp_precision says.  No atomics decide anything that is stored: the
// output is bitwise reproducible.  The extraction reads the field, the weights and the mesh and writes only its own workspace.
#include <algorithm>
#include <cmath>

#include <cub/cub.cuh>
#include "tn_common.cuh"
#include "tn_direnc.cuh"
#include "tn_mlp.cuh"
#include "tn_sort.cuh"

namespace tn {

constexpr uint32_t EDGE_SAMPLES = 64;  // samples per edge and refinement round: one k_mlp tile

struct SurfaceState {
    // the last extraction: counts and the generations of what it read (tn_surface_copy refuses a stale result)
    bool valid = false;
    uint32_t N = 0, F = 0;
    uint64_t gen = 0, mesh_gen = 0;
    // workspace, grown on demand and kept
    DevArray<uint32_t> small;                  // [8]: tile counters of the four k_mlp launches | V | E
    DevArray<uint4> vvi;                       // [V] (v,v,v,v)
    DevArray<float> vbary, vsig;               // [V,3] zeros, [V] vertex densities
    DevArray<unsigned long long> tcnt, toff;   // [T+1] (edges << 32 | triangles) per tetrahedron, its exclusive scan
    DevArray<unsigned long long> keys, skeys;  // [crossing-edge slots]: keys a * V + b as emitted, sorted; `keys` then holds the unique ones
    DevArray<uint4> evi;                       // [64 E] rows of a refinement round (the colour pass reuses the first E rows)
    DevArray<float> ebary, eout;               // [64 E,3], [64 E] (the colour pass: eout as float4 [E])
    DevArray<float4> br;                       // [E]: (s_lo, sigma_lo, sigma_hi, s) bracket of each edge, final parameter
    DevArray<float> pos, nrm, dirbias;         // [E,3], [E,3], [E,128]
    DevArray<uint32_t> faces, ftet;            // [F,3], [F]
    DevArray<float> fnrm;                      // [F,3]
    DevArray<uint32_t> nk0, nk1, nv0, nv1;     // [3F] (vertex, face) pairs and their sorted copies
    DevArray<uint8_t> cub;
};

void free_surface(tn_tracer *h) {
    delete h->surface;
    h->surface = nullptr;
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------------
__global__ void k_vertex_rows(uint32_t V, uint4 *__restrict__ vi, uint32_t *__restrict__ count) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v == 0) *count = V;
    if (v < V) vi[v] = make_uint4(v, v, v, v);
}

// the inside (sigma >= level) and outside vertex ids of one tetrahedron, each list ascending
struct TetCase {
    uint32_t in[4], out[4];
    uint32_t nin, nout;
};
__device__ __forceinline__ TetCase tet_case(const uint32_t *__restrict__ cells, uint32_t t, const float *__restrict__ vsig, float level) {
    const uint4 c = __ldg(reinterpret_cast<const uint4 *>(cells) + t);
    uint32_t v[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int i = 1; i < 4; ++i)  // insertion sort of four ids
#pragma unroll
        for (int j = i; j > 0; --j)
            if (v[j] < v[j - 1]) { const uint32_t x = v[j]; v[j] = v[j - 1]; v[j - 1] = x; }
    TetCase k{};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (__ldg(vsig + v[i]) >= level) k.in[k.nin++] = v[i];
        else k.out[k.nout++] = v[i];
    }
    return k;
}

// (crossing edges << 32) | triangles of every tetrahedron; slot T is 0, so that the exclusive scan's last entry is the total
__global__ void k_tet_case(uint32_t T, const uint32_t *__restrict__ cells, const float *__restrict__ vsig, float level,
                           unsigned long long *__restrict__ cnt) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > T) return;
    unsigned long long c = 0;
    if (t < T) {
        const TetCase k = tet_case(cells, t, vsig, level);
        if (k.nin == 1 || k.nin == 3) c = (3ull << 32) | 1ull;
        else if (k.nin == 2) c = (4ull << 32) | 2ull;
    }
    cnt[t] = c;
}

__device__ __forceinline__ unsigned long long edge_key(uint32_t x, uint32_t y, uint32_t V) {
    return x < y ? (unsigned long long)x * V + y : (unsigned long long)y * V + x;
}

// the crossing edges of every tetrahedron, at its scanned offset (an edge shared by several tetrahedra appears once per tetrahedron)
__global__ void k_tet_edges(uint32_t T, uint32_t V, const uint32_t *__restrict__ cells, const float *__restrict__ vsig, float level,
                            const unsigned long long *__restrict__ off, unsigned long long *__restrict__ keys) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const TetCase k = tet_case(cells, t, vsig, level);
    if (k.nin == 0 || k.nin == 4) return;
    unsigned long long *o = keys + (off[t] >> 32);
    uint32_t n = 0;
    for (uint32_t i = 0; i < k.nin; ++i)
        for (uint32_t j = 0; j < k.nout; ++j) o[n++] = edge_key(k.in[i], k.out[j], V);
}

__device__ __forceinline__ uint32_t find_key(const unsigned long long *__restrict__ ukeys, uint32_t E, unsigned long long key) {
    uint32_t lo = 0, hi = E;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(ukeys + mid) < key) lo = mid + 1; else hi = mid; }
    return lo;
}

// det(q1 - q0, q2 - q0, q3 - q0) in double, every operation rounded on its own (no contraction): oracle/surface.py repeats it
__device__ __forceinline__ double orient(const float *__restrict__ xyz, uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
    const double x0 = xyz[3 * (size_t)q0], y0 = xyz[3 * (size_t)q0 + 1], z0 = xyz[3 * (size_t)q0 + 2];
    const double ax = __dsub_rn(xyz[3 * (size_t)q1], x0), ay = __dsub_rn(xyz[3 * (size_t)q1 + 1], y0), az = __dsub_rn(xyz[3 * (size_t)q1 + 2], z0);
    const double bx = __dsub_rn(xyz[3 * (size_t)q2], x0), by = __dsub_rn(xyz[3 * (size_t)q2 + 1], y0), bz = __dsub_rn(xyz[3 * (size_t)q2 + 2], z0);
    const double cx = __dsub_rn(xyz[3 * (size_t)q3], x0), cy = __dsub_rn(xyz[3 * (size_t)q3 + 1], y0), cz = __dsub_rn(xyz[3 * (size_t)q3 + 2], z0);
    const double t1 = __dsub_rn(__dmul_rn(by, cz), __dmul_rn(bz, cy));
    const double t2 = __dsub_rn(__dmul_rn(bx, cz), __dmul_rn(bz, cx));
    const double t3 = __dsub_rn(__dmul_rn(bx, cy), __dmul_rn(by, cx));
    return __dadd_rn(__dsub_rn(__dmul_rn(ax, t1), __dmul_rn(ay, t2)), __dmul_rn(az, t3));
}

// marching tetrahedra, with inside ids i0 < i1 < .. and outside ids o0 < o1 < .. (e(x, y) = the output vertex on edge {x, y}):
//   1 inside : (e(i,o0), e(i,o1), e(i,o2)),                 flipped iff det(o0-i, o1-i, o2-i) < 0
//   3 inside : (e(i0,o), e(i1,o), e(i2,o)),                 flipped iff det(i0-o, i1-o, i2-o) > 0
//   2 inside : (e(i0,o0), e(i0,o1), e(i1,o1)), (e(i0,o0), e(i1,o1), e(i1,o0)) -- the quad split along e(i0,o0) - e(i1,o1) --
//              flipped iff det(i1-i0, o0-i0, o1-i0) < 0
// "flipped" swaps the last two corners.  With these signs every normal points from the inside vertices to the outside ones for any
// crossing positions strictly inside their edges (the triple products are affine invariant); a flat tetrahedron (det 0) keeps the order.
__global__ void k_faces(uint32_t T, uint32_t V, uint32_t E, const uint32_t *__restrict__ cells, const float *__restrict__ xyz,
                        const float *__restrict__ vsig, float level, const unsigned long long *__restrict__ off,
                        const unsigned long long *__restrict__ ukeys, uint32_t *__restrict__ faces, uint32_t *__restrict__ ftet) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const TetCase k = tet_case(cells, t, vsig, level);
    if (k.nin == 0 || k.nin == 4) return;
    const uint32_t f0 = (uint32_t)(off[t] & 0xFFFFFFFFull);
    auto e = [&](uint32_t x, uint32_t y) { return find_key(ukeys, E, edge_key(x, y, V)); };
    uint32_t tri[2][3];
    uint32_t ntri = 1;
    bool flip;
    if (k.nin == 1) {
        const uint32_t i = k.in[0];
        tri[0][0] = e(i, k.out[0]); tri[0][1] = e(i, k.out[1]); tri[0][2] = e(i, k.out[2]);
        flip = orient(xyz, i, k.out[0], k.out[1], k.out[2]) < 0.0;
    } else if (k.nin == 3) {
        const uint32_t o = k.out[0];
        tri[0][0] = e(k.in[0], o); tri[0][1] = e(k.in[1], o); tri[0][2] = e(k.in[2], o);
        flip = orient(xyz, o, k.in[0], k.in[1], k.in[2]) > 0.0;
    } else {
        const uint32_t a = e(k.in[0], k.out[0]), b = e(k.in[0], k.out[1]), c = e(k.in[1], k.out[1]), d = e(k.in[1], k.out[0]);
        tri[0][0] = a; tri[0][1] = b; tri[0][2] = c;
        tri[1][0] = a; tri[1][1] = c; tri[1][2] = d;
        ntri = 2;
        flip = orient(xyz, k.in[0], k.in[1], k.out[0], k.out[1]) < 0.0;
    }
    for (uint32_t q = 0; q < ntri; ++q) {
        uint32_t *o = faces + 3 * (size_t)(f0 + q);
        o[0] = tri[q][0];
        o[1] = flip ? tri[q][2] : tri[q][1];
        o[2] = flip ? tri[q][1] : tri[q][2];
        ftet[f0 + q] = t;
    }
}

// the rows of one refinement round: edge e, sample j at s = s0 + (j + 1) step, with s0 = 0 (round 1) or the edge's bracket start
__global__ void k_edge_rows(uint32_t E, uint32_t V, const unsigned long long *__restrict__ ukeys, const float4 *__restrict__ br, float step,
                            uint4 *__restrict__ vi, float *__restrict__ bary) {
    const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= (uint64_t)E * EDGE_SAMPLES) return;
    const uint32_t e = (uint32_t)(row / EDGE_SAMPLES), j = (uint32_t)(row % EDGE_SAMPLES);
    const unsigned long long key = __ldg(ukeys + e);
    const uint32_t a = (uint32_t)(key / V), b = (uint32_t)(key % V);
    const float s = (br != nullptr ? br[e].x : 0.f) + (float)(j + 1) * step;
    vi[row] = make_uint4(a, b, b, b);
    bary[3 * row] = s; bary[3 * row + 1] = 0.f; bary[3 * row + 2] = 0.f;
}

// one warp per crossing edge (a, b): sample i = 1..64 of the round has sigma out[64 e + i - 1] (i < 64) or the known value at the
// bracket's end (i = 64), sample 0 the known value at its start; the new bracket is [i - 1, i] for the smallest i whose side differs
// from a's.  Round 2 (final) places the vertex: s = s_lo + (level - sigma_lo) / (sigma_hi - sigma_lo) step, the point (1-s) x_a + s x_b,
// and writes the colour pass's row e.
__global__ void __launch_bounds__(256) k_bracket(uint32_t E, uint32_t V, const unsigned long long *__restrict__ ukeys, const float *__restrict__ vsig,
                                                 float level, const float *__restrict__ out, float step, int final_round, float4 *__restrict__ br,
                                                 const float *__restrict__ xyz, float *__restrict__ pos, uint4 *__restrict__ cvi,
                                                 float *__restrict__ cbary) {
    const uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (e >= E) return;
    const unsigned long long key = __ldg(ukeys + e);
    const uint32_t a = (uint32_t)(key / V), b = (uint32_t)(key % V);
    const float sig_a = __ldg(vsig + a);
    const bool ins_a = sig_a >= level;
    float s0 = 0.f, lo0 = sig_a, hi = __ldg(vsig + b);
    if (final_round) { const float4 q = br[e]; s0 = q.x; lo0 = q.y; hi = q.z; }
    const float *o = out + (size_t)e * EDGE_SAMPLES;
    const float x1 = o[lane], x2 = lane + 33 < 64 ? o[lane + 32] : hi;  // samples i = lane + 1, lane + 33
    const uint32_t m1 = __ballot_sync(0xffffffffu, (x1 >= level) != ins_a), m2 = __ballot_sync(0xffffffffu, (x2 >= level) != ins_a);
    const uint32_t i = m1 ? (uint32_t)__ffs(m1) : 32u + (uint32_t)__ffs(m2);  // >= 1; sample 64 always differs
    if (lane != 0) return;
    const float sig_hi = i < 64 ? o[i - 1] : hi, sig_lo = i > 1 ? o[i - 2] : lo0;
    const float s_lo = s0 + (float)(i - 1) * step;
    if (!final_round) { br[e] = make_float4(s_lo, sig_lo, sig_hi, 0.f); return; }
    float t = (level - sig_lo) / (sig_hi - sig_lo);
    t = fminf(fmaxf(t, 0.f), 1.f);  // (also maps a NaN to 0)
    const float s = s_lo + t * step;
    br[e] = make_float4(s_lo, sig_lo, sig_hi, s);
    for (int c = 0; c < 3; ++c) pos[3 * (size_t)e + c] = (1.f - s) * __ldg(xyz + 3 * (size_t)a + c) + s * __ldg(xyz + 3 * (size_t)b + c);
    cvi[e] = make_uint4(a, b, b, b);
    cbary[3 * (size_t)e] = s; cbary[3 * (size_t)e + 1] = 0.f; cbary[3 * (size_t)e + 2] = 0.f;
}

// unnormalised face normals (p1 - p0) x (p2 - p0) and the (vertex, face) pairs of the segmented sum
__global__ void k_face_normals(uint32_t F, const uint32_t *__restrict__ faces, const float *__restrict__ pos, float *__restrict__ fnrm,
                               uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const uint32_t v0 = faces[3 * (size_t)f], v1 = faces[3 * (size_t)f + 1], v2 = faces[3 * (size_t)f + 2];
    const float *p0 = pos + 3 * (size_t)v0, *p1 = pos + 3 * (size_t)v1, *p2 = pos + 3 * (size_t)v2;
    const float ux = p1[0] - p0[0], uy = p1[1] - p0[1], uz = p1[2] - p0[2];
    const float wx = p2[0] - p0[0], wy = p2[1] - p0[1], wz = p2[2] - p0[2];
    fnrm[3 * (size_t)f] = uy * wz - uz * wy;
    fnrm[3 * (size_t)f + 1] = uz * wx - ux * wz;
    fnrm[3 * (size_t)f + 2] = ux * wy - uy * wx;
    for (int k = 0; k < 3; ++k) { keys[3 * (size_t)f + k] = faces[3 * (size_t)f + k]; vals[3 * (size_t)f + k] = f; }
}

// one warp per vertex: lane 0 sums the normals of the vertex's faces in face order (the stable sort kept it), the warp then forms the
// direction bias of the colour pass, b4 + W4[:, :27] enc(-n), as k_sample_fine does per ray
__global__ void __launch_bounds__(256) k_vertex_normals(uint32_t N, uint32_t n, const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                        const float *__restrict__ fnrm, const float *__restrict__ w4dir, float *__restrict__ nrm,
                                                        float *__restrict__ dirbias) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (v >= N) return;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (lane == 0) {
        const uint32_t lo = lower_bound_u32(keys, n, v), hi = lower_bound_u32(keys, n, v + 1);
        for (uint32_t q = lo; q < hi; ++q) {
            const float *fn = fnrm + 3 * (size_t)__ldg(vals + q);
            nx += fn[0]; ny += fn[1]; nz += fn[2];
        }
        const float len = sqrtf(nx * nx + ny * ny + nz * nz);
        if (len > 0.f) { nx /= len; ny /= len; nz /= len; }
        else { nx = ny = nz = 0.f; }
        nrm[3 * (size_t)v] = nx; nrm[3 * (size_t)v + 1] = ny; nrm[3 * (size_t)v + 2] = nz;
    }
    nx = __shfl_sync(0xffffffffu, nx, 0); ny = __shfl_sync(0xffffffffu, ny, 0); nz = __shfl_sync(0xffffffffu, nz, 0);
    float enc[27];
    encode_direction(-nx, -ny, -nz, enc);
    for (uint32_t o = lane; o < 128; o += 32) {
        float acc = w4dir[128 * 27 + o];
#pragma unroll
        for (int k = 0; k < 27; ++k) acc = fmaf(__ldg(w4dir + o * 27 + k), enc[k], acc);
        dirbias[(size_t)v * 128 + o] = acc;
    }
}

__global__ void k_surface_copy(uint32_t N, const float *__restrict__ pos, const float *__restrict__ nrm, const float4 *__restrict__ cout,
                               float *__restrict__ d_pos, float *__restrict__ d_nrm, float *__restrict__ d_col) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * N) return;
    if (d_pos) d_pos[i] = pos[i];
    if (d_nrm) d_nrm[i] = nrm[i];
    if (d_col) { const float4 c = cout[i / 3]; const uint32_t k = i % 3; d_col[i] = k == 0 ? c.y : (k == 1 ? c.z : c.w); }
}

}  // namespace tn

using namespace tn;

namespace {
// one k_mlp<FINE, 3> pass over n_active * S rows (count on the device, n_host on the host for the grid)
template <bool FINE>
int run_mlp(tn_tracer *h, const RenderInputs &in, const uint32_t *d_count, uint64_t rows, uint32_t S, const uint4 *vi, const float *bary,
            const float *dirbias, float *out, uint32_t *tile_ctr, cudaStream_t s) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    MlpParams p{};
    p.n_active = d_count; p.S = S; p.vi = vi; p.bary = bary; p.fshadow = in.fshadow; p.wimg = in.wimg; p.bias = in.bias;
    p.head = in.head; p.dirbias = dirbias; p.out = out; p.tile_ctr = tile_ctr;
    const uint64_t tiles = (rows + MLP_TILE - 1) / MLP_TILE;
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((tiles + MLP_WGS - 1) / MLP_WGS, (uint64_t)sms));
    h->launches += 1;
    return launch_mlp<FINE, 3>(p, grid, s);
}

uint32_t blocks(uint64_t n, uint32_t per) { return (uint32_t)((n + per - 1) / per); }
}  // namespace

extern "C" int tn_surface_extract(tn_tracer *h, float level, uint32_t *n_vertices, uint32_t *n_faces, void *stream) {
    if (!h || !n_vertices || !n_faces) return fail(TN_ERR_ARG, "null argument");
    if (!h->mesh.nodes.p) return fail(TN_ERR_STATE, "tn_surface_extract: no tetrahedra loaded");
    RenderInputs in{};
    if (render_inputs(h, &in) != TN_OK) return fail(TN_ERR_STATE, "tn_surface_extract: call tn_render_set_field and tn_render_set_weights first");
    if (!(level > 0.f) || !std::isfinite(level)) return fail(TN_ERR_ARG, "tn_surface_extract: the level must be finite and greater than 0");
    if (in.V != h->mesh.V) return fail(TN_ERR_ARG, "tn_surface_extract: field has a different vertex count than the mesh");
    const uint32_t V = h->mesh.V, T = h->mesh.T;
    if ((uint64_t)V * V >= (1ull << 63)) return fail(TN_ERR_ARG, "tn_surface_extract: too many vertices");
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (!h->surface) h->surface = new SurfaceState();
    SurfaceState &S = *h->surface;
    S.valid = false;
    *n_vertices = *n_faces = 0;
    TN_TRY(S.small.grow(8));
    uint32_t *small = S.small.p, *d_V = small + 4, *d_E = small + 5;
    TN_CUDA(cudaMemsetAsync(small, 0, 8 * sizeof(uint32_t), s));
    // ---- vertex densities ----
    TN_TRY(S.vvi.grow(V)); TN_TRY(S.vbary.grow(3 * (size_t)V)); TN_TRY(S.vsig.grow(V));
    const float *vsig = S.vsig.p;
    TN_CUDA(cudaMemsetAsync(S.vbary.p, 0, 12 * (size_t)V, s));
    k_vertex_rows<<<blocks(V, 256), 256, 0, s>>>(V, S.vvi.p, d_V);
    h->launches += 1;
    TN_TRY(run_mlp<false>(h, in, d_V, V, 1, S.vvi.p, S.vbary.p, nullptr, S.vsig.p, small + 0, s));
    // ---- cases, crossing edges, faces ----
    TN_TRY(S.tcnt.grow((size_t)T + 1)); TN_TRY(S.toff.grow((size_t)T + 1));
    unsigned long long *tcnt = S.tcnt.p, *toff = S.toff.p;
    k_tet_case<<<blocks((uint64_t)T + 1, 256), 256, 0, s>>>(T, h->mesh.cells, vsig, level, tcnt);
    TN_TRY(cub_run(S.cub, [&](void *t, size_t &bytes) { return cub::DeviceScan::ExclusiveSum(t, bytes, tcnt, toff, (int64_t)T + 1, s); }));
    h->launches += 2;
    unsigned long long total = 0;
    TN_CUDA(cudaMemcpyAsync(&total, toff + T, sizeof(total), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    const uint64_t nslots = total >> 32, F = total & 0xFFFFFFFFull;
    if (F == 0) {  // the level lies above or below every vertex density: an empty surface
        S.N = S.F = 0; S.gen = in.gen; S.mesh_gen = h->mesh_gen; S.valid = true;
        TN_CUDA(cudaGetLastError());
        return TN_OK;
    }
    if (nslots >= (1ull << 31)) return fail(TN_ERR_ARG, "tn_surface_extract: too many crossing tetrahedra");
    TN_TRY(S.keys.grow(nslots)); TN_TRY(S.skeys.grow(nslots));
    unsigned long long *keys = S.keys.p, *skeys = S.skeys.p;
    k_tet_edges<<<blocks(T, 256), 256, 0, s>>>(T, V, h->mesh.cells, vsig, level, toff, keys);
    const int end_bit = radix_end_bit((uint64_t)V * V);
    TN_TRY(cub_run(S.cub, [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortKeys(t, bytes, keys, skeys, (int64_t)nslots, 0, end_bit, s);
    }));
    TN_TRY(cub_run(S.cub, [&](void *t, size_t &bytes) { return cub::DeviceSelect::Unique(t, bytes, skeys, keys, d_E, (int64_t)nslots, s); }));
    h->launches += 3;
    uint32_t E = 0;
    TN_CUDA(cudaMemcpyAsync(&E, d_E, sizeof(E), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    if ((uint64_t)E * EDGE_SAMPLES >= (1ull << 32)) return fail(TN_ERR_ARG, "tn_surface_extract: more than 2^26 crossing edges");
    const unsigned long long *ukeys = keys;
    TN_TRY(S.faces.grow(3 * F)); TN_TRY(S.ftet.grow(F));
    k_faces<<<blocks(T, 256), 256, 0, s>>>(T, V, E, h->mesh.cells, h->mesh.xyz, vsig, level, toff, ukeys, S.faces.p, S.ftet.p);
    h->launches += 1;
    // ---- refinement: two rounds of 64 samples per edge ----
    const uint64_t rows = (uint64_t)E * EDGE_SAMPLES;
    TN_TRY(S.evi.grow(rows)); TN_TRY(S.ebary.grow(3 * rows)); TN_TRY(S.eout.grow(rows)); TN_TRY(S.br.grow(E)); TN_TRY(S.pos.grow(3 * (size_t)E));
    uint4 *evi = S.evi.p;
    float *ebary = S.ebary.p, *eout = S.eout.p, *pos = S.pos.p;
    float4 *br = S.br.p;
    for (int round = 0; round < 2; ++round) {
        const float step = round == 0 ? 1.f / 64.f : 1.f / 4096.f;
        k_edge_rows<<<blocks(rows, 256), 256, 0, s>>>(E, V, ukeys, round == 0 ? nullptr : br, step, evi, ebary);
        TN_TRY(run_mlp<false>(h, in, d_E, rows, EDGE_SAMPLES, evi, ebary, nullptr, eout, small + 1 + round, s));
        k_bracket<<<blocks((uint64_t)E * 32, 256), 256, 0, s>>>(E, V, ukeys, vsig, level, eout, step, round, br, h->mesh.xyz, pos, evi, ebary);
        h->launches += 2;
    }
    // ---- normals (deterministic segmented sum) and the colour pass's direction bias ----
    const uint64_t n3 = 3 * F;
    TN_TRY(S.fnrm.grow(3 * F)); TN_TRY(S.nk0.grow(n3)); TN_TRY(S.nk1.grow(n3)); TN_TRY(S.nv0.grow(n3)); TN_TRY(S.nv1.grow(n3));
    TN_TRY(S.nrm.grow(3 * (size_t)E)); TN_TRY(S.dirbias.grow(128 * (size_t)E));
    uint32_t *nk0 = S.nk0.p, *nk1 = S.nk1.p, *nv0 = S.nv0.p, *nv1 = S.nv1.p;
    k_face_normals<<<blocks(F, 256), 256, 0, s>>>((uint32_t)F, S.faces.p, pos, S.fnrm.p, nk0, nv0);
    const int vbits = radix_end_bit(E);
    TN_TRY(cub_run(S.cub, [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, nk0, nk1, nv0, nv1, (int64_t)n3, 0, vbits, s);
    }));
    k_vertex_normals<<<blocks((uint64_t)E * 32, 256), 256, 0, s>>>(E, (uint32_t)n3, nk1, nv1, S.fnrm.p, in.w4dir, S.nrm.p, S.dirbias.p);
    h->launches += 3;
    // ---- colours: the colour head at the vertex's features, seen along -n ----
    TN_TRY(run_mlp<true>(h, in, d_E, E, 1, evi, ebary, S.dirbias.p, eout, small + 3, s));
    TN_CUDA(cudaGetLastError());
    S.N = E; S.F = (uint32_t)F; S.gen = in.gen; S.mesh_gen = h->mesh_gen; S.valid = true;
    *n_vertices = E; *n_faces = (uint32_t)F;
    return TN_OK;
}

extern "C" int tn_surface_copy(tn_tracer *h, float *d_vertices, float *d_normals, float *d_colors, uint32_t *d_faces, uint32_t *d_face_tet,
                               void *stream) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    SurfaceState *S = h->surface;
    if (!S || !S->valid) return fail(TN_ERR_STATE, "tn_surface_copy: no surface extraction to copy from");
    RenderInputs in{};
    if (render_inputs(h, &in) != TN_OK || in.gen != S->gen || h->mesh_gen != S->mesh_gen)
        return fail(TN_ERR_STATE, "tn_surface_copy: the field, the weights or the mesh changed (tn_render_set_field / tn_render_set_weights / "
                                  "tn_load_tetrahedra) since the extraction");
    DeviceGuard g(h->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (S->N > 0 && (d_vertices || d_normals || d_colors)) {
        k_surface_copy<<<blocks(3 * (uint64_t)S->N, 256), 256, 0, s>>>(S->N, S->pos.p, S->nrm.p, reinterpret_cast<const float4 *>(S->eout.p),
                                                                        d_vertices, d_normals, d_colors);
        h->launches += 1;
    }
    if (S->F > 0 && d_faces) TN_CUDA(cudaMemcpyAsync(d_faces, S->faces.p, 12 * (size_t)S->F, cudaMemcpyDeviceToDevice, s));
    if (S->F > 0 && d_face_tet) TN_CUDA(cudaMemcpyAsync(d_face_tet, S->ftet.p, 4 * (size_t)S->F, cudaMemcpyDeviceToDevice, s));
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}
