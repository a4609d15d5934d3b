// tn_fold_guard.cu -- the fold guard of a vertex step (tn_guard_vertex_step, DESIGN.md §4.17): scales back, per vertex, the part of a
// proposed move P0 -> P1 that would fold a face the refit's fold test certifies at P0, or break a hull edge the convexity test accepts.
//
// Each moving vertex (a P1 row that differs bitwise from its P0 row) holds an exponent k: 0 = P1, 1..K = P0 + 2^-k (P1 - P0), FROZEN = P0.
// Round r tests every guarded item at the current positions; the moving, not yet frozen vertices of a failing item get k = r + 1, or
// FROZEN from round K on, until a round finds nothing failing.  An item is retested only when one of its vertices changed in the round
// before: an item none of whose vertices moved sits where it was last tested.  Every update is "this vertex fails in round r", set by plain
// stores, and the new exponent depends only on r, so the result is a function of (P0, P1, cells) alone, whatever the scheduling.
#include "tn_common.cuh"
#include "tn_predicates.cuh"

namespace tn {

constexpr uint8_t GUARD_STILL = 0xFF;   // not moving: P1 row == P0 row, never marked
constexpr uint8_t GUARD_FROZEN = 0xFE;  // back at P0
constexpr uint32_t GUARD_MAX_HALVINGS = 23;

// counters (tracer scratch guard_counts): [0] non-finite input, [1] interior faces uncertified at P0, [2] hull edges rejected at P0,
// [3] items failing this round, [4] vertices changed this round, [5] vertices limited (1 <= k <= K), [6] vertices frozen
__global__ void k_guard_init(const float *__restrict__ p0, const float *__restrict__ p1, uint32_t V, float *__restrict__ p1_copy,
                             uint8_t *__restrict__ kexp, uint8_t *__restrict__ mark, uint8_t *__restrict__ changed, uint32_t *__restrict__ counts) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    bool moving = false, finite = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float x0 = p0[3 * (size_t)v + a], x1 = p1[3 * (size_t)v + a];
        moving |= __float_as_uint(x0) != __float_as_uint(x1);
        finite &= isfinite(x0) && isfinite(x1);
        p1_copy[3 * (size_t)v + a] = x1;
    }
    if (!finite) atomicOr(counts, 1u);
    kexp[v] = moving ? 0 : GUARD_STILL;
    mark[v] = 0;
    changed[v] = moving ? 1 : 0;
}

// the guarded faces: every interior face certified unfolded at P0, as (a, b, c, p) + q; the others get a = TN_EMPTY
__global__ void k_guard_faces_p0(const float *__restrict__ p0, const uint4 *__restrict__ cells, const uint4 *__restrict__ tri, const uint2 *__restrict__ tt,
                                 uint32_t F, uint4 *__restrict__ rec, uint32_t *__restrict__ recq, uint32_t *__restrict__ counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const uint2 o = tt[f];
    uint4 r = make_uint4(TN_EMPTY, 0u, 0u, 0u);
    uint32_t q = 0;
    if (o.y != TN_EMPTY) {
        const uint4 t = tri[f];
        const uint32_t p = opposite_vertex(cells[o.x], t);
        q = opposite_vertex(cells[o.y], t);
        if (face_unfolded(p0, t.x, t.y, t.z, p, q)) r = make_uint4(t.x, t.y, t.z, p);
        else atomicAdd(counts + 1, 1u);
    }
    rec[f] = r;
    recq[f] = q;
}

__device__ __forceinline__ void guard_mark(uint32_t v, const uint8_t *__restrict__ kexp, uint8_t *__restrict__ mark) {
    const uint8_t k = kexp[v];
    if (k != GUARD_STILL && k != GUARD_FROZEN) mark[v] = 1;
}

__global__ void k_guard_faces_round(const float *__restrict__ xyz, const uint4 *__restrict__ rec, const uint32_t *__restrict__ recq, uint32_t F,
                                    const uint8_t *__restrict__ kexp, uint8_t *__restrict__ mark, const uint8_t *__restrict__ changed,
                                    uint32_t *__restrict__ counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const uint4 r = rec[f];
    if (r.x == TN_EMPTY) return;
    const uint32_t q = recq[f];
    if (!(changed[r.x] | changed[r.y] | changed[r.z] | changed[r.w] | changed[q])) return;
    if (face_unfolded(xyz, r.x, r.y, r.z, r.w, q)) return;
    guard_mark(r.x, kexp, mark); guard_mark(r.y, kexp, mark); guard_mark(r.z, kexp, mark); guard_mark(r.w, kexp, mark); guard_mark(q, kexp, mark);
    atomicAdd(counts + 3, 1u);
}

// hull edges of a walkable load: sorted (a, b) keys, each edge's two hull faces at entries 2i and 2i + 1.  p0: count the rejected ones at
// the positions (counts[2]); otherwise a round: retest the edges with a changed vertex and mark a failing one's moving vertices, the 4th
// vertices of both faces' tetrahedra included (hull_pair_ok reads them)
__global__ void k_guard_hull(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint4 *__restrict__ tri, const uint2 *__restrict__ tt,
                             const uint32_t *__restrict__ eface, uint32_t npairs, int p0, const uint8_t *__restrict__ kexp, uint8_t *__restrict__ mark,
                             const uint8_t *__restrict__ changed, uint32_t *__restrict__ counts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const uint32_t f = eface[2 * i], g = eface[2 * i + 1];
    const uint4 ft = tri[f], gt = tri[g];
    const uint32_t vs[8] = {ft.x, ft.y, ft.z, gt.x, gt.y, gt.z, opposite_vertex(cells[tt[f].x], ft), opposite_vertex(cells[tt[g].x], gt)};
    if (!p0) {
        uint8_t any = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) any |= changed[vs[j]];
        if (!any) return;
    }
    if (hull_pair_ok(xyz, cells, tri, tt, f, g) && hull_pair_ok(xyz, cells, tri, tt, g, f)) return;
    if (p0) { atomicAdd(counts + 2, 1u); return; }
#pragma unroll
    for (int j = 0; j < 8; ++j) guard_mark(vs[j], kexp, mark);
    atomicAdd(counts + 3, 1u);
}

// the marked vertices take exponent knew (r + 1, or GUARD_FROZEN from round K on) and their new position:
// x = p0 + (p1 - p0) * 2^-k, each operation rounded to fp32 in this order (no FMA); x = p0 when frozen
__global__ void k_guard_apply(const float *__restrict__ p0, const float *__restrict__ p1, float *__restrict__ xyz, uint32_t V, uint8_t knew,
                              uint32_t K, uint8_t *__restrict__ kexp, uint8_t *__restrict__ mark, uint8_t *__restrict__ changed,
                              uint32_t *__restrict__ counts) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    if (!mark[v]) { changed[v] = 0; return; }
    const uint8_t kold = kexp[v];
    kexp[v] = knew;
    mark[v] = 0;
    changed[v] = 1;
    const float scale = __uint_as_float((127u - knew) << 23);  // 2^-knew, knew <= 23
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float x0 = p0[3 * (size_t)v + a];
        xyz[3 * (size_t)v + a] = knew == GUARD_FROZEN ? x0 : __fadd_rn(x0, __fmul_rn(__fsub_rn(p1[3 * (size_t)v + a], x0), scale));
    }
    atomicAdd(counts + 4, 1u);
    const bool was_limited = kold >= 1 && kold <= K;
    if (knew == GUARD_FROZEN) {
        atomicAdd(counts + 6, 1u);
        if (was_limited) atomicSub(counts + 5, 1u);
    } else if (!was_limited) {
        atomicAdd(counts + 5, 1u);
    }
}

int guard_vertex_step(tn_tracer *h, const float *d_old, float *d_new, uint32_t V, uint32_t K, uint32_t *counts3, cudaStream_t s) {
    const Mesh &m = h->mesh;
    if (!m.nodes.p) return fail(TN_ERR_STATE, "guard_vertex_step: no tetrahedra loaded");
    if (V != m.V) return fail(TN_ERR_ARG, "guard_vertex_step: " + std::to_string(V) + " vertices, the loaded mesh has " + std::to_string(m.V));
    if (K > GUARD_MAX_HALVINGS) return fail(TN_ERR_ARG, "guard_vertex_step: max_halvings " + std::to_string(K) + " > 23");
    const uint32_t F = m.F;
    TN_TRY(h->guard_face.grow(F)); TN_TRY(h->guard_faceq.grow(F));
    TN_TRY(h->guard_p1.grow(3 * (size_t)V)); TN_TRY(h->guard_vtx.grow(3 * (size_t)V));
    TN_TRY(h->guard_counts.grow(8));
    uint32_t *d_cnt = h->guard_counts.p;
    uint8_t *kexp = h->guard_vtx.p, *mark = kexp + V, *changed = mark + V;
    const uint4 *cells = (const uint4 *)m.cells;
    TN_CUDA(cudaMemsetAsync(d_cnt, 0, 8 * sizeof(uint32_t), s));
    const uint32_t vb = (V + 255) / 256, fb = (F + 255) / 256;
    // round 0 of the masks: moving vertices, the faces certified at P0, the hull edges accepted at P0
    k_guard_init<<<vb, 256, 0, s>>>(d_old, d_new, V, h->guard_p1.p, kexp, mark, changed, d_cnt);
    k_guard_faces_p0<<<fb, 256, 0, s>>>(d_old, cells, m.tri.p, m.tt.p, F, h->guard_face.p, h->guard_faceq.p, d_cnt);
    const uint32_t npairs = m.walk.p ? m.hull_ne / 2 : 0;
    if (npairs)
        k_guard_hull<<<(npairs + 255) / 256, 256, 0, s>>>(d_old, cells, m.tri.p, m.tt.p, m.hull_eface.p, npairs, 1, kexp, mark, changed, d_cnt);
    h->launches += 2 + (npairs ? 1 : 0);
    uint32_t hc[8];
    TN_CUDA(cudaMemcpyAsync(hc, d_cnt, sizeof(hc), cudaMemcpyDeviceToHost, s));
    TN_CUDA(cudaStreamSynchronize(s));
    TN_CUDA(cudaGetLastError());
    if (hc[0]) return fail(TN_ERR_ARG, "guard_vertex_step: a vertex coordinate is not finite");
    // the hull edges are guarded only if the mesh is walkable at P0: every hull edge accepted and no interior face uncertified
    const bool guard_hull = npairs > 0 && hc[1] == 0 && hc[2] == 0;
    uint32_t rounds = 0;
    for (uint32_t r = 0;; ++r) {
        TN_CUDA(cudaMemsetAsync(d_cnt + 3, 0, 2 * sizeof(uint32_t), s));
        k_guard_faces_round<<<fb, 256, 0, s>>>(d_new, h->guard_face.p, h->guard_faceq.p, F, kexp, mark, changed, d_cnt);
        if (guard_hull)
            k_guard_hull<<<(npairs + 255) / 256, 256, 0, s>>>(d_new, cells, m.tri.p, m.tt.p, m.hull_eface.p, npairs, 0, kexp, mark, changed, d_cnt);
        const uint8_t knew = r < K ? (uint8_t)(r + 1) : GUARD_FROZEN;
        k_guard_apply<<<vb, 256, 0, s>>>(d_old, h->guard_p1.p, d_new, V, knew, K, kexp, mark, changed, d_cnt);
        h->launches += 2 + (guard_hull ? 1 : 0);
        TN_CUDA(cudaMemcpyAsync(hc, d_cnt, sizeof(hc), cudaMemcpyDeviceToHost, s));
        TN_CUDA(cudaStreamSynchronize(s));
        TN_CUDA(cudaGetLastError());
        rounds = r + 1;
        if (hc[3] == 0) break;
        // a failing item has a moving vertex that is not frozen (one at P0 throughout passes), so every freeze round freezes one more
        if (hc[4] == 0) return fail(TN_ERR_STATE, "guard_vertex_step: a failing item with no vertex left to move back");
    }
    if (counts3) { counts3[0] = hc[5]; counts3[1] = hc[6]; counts3[2] = rounds; }
    return TN_OK;
}

}  // namespace tn

extern "C" int tn_guard_vertex_step(tn_tracer *h, const float *d_xyz_old, float *d_xyz_new, uint32_t V, uint32_t max_halvings, uint32_t *counts3,
                                    void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (!d_xyz_old || !d_xyz_new) return tn::fail(TN_ERR_ARG, "guard_vertex_step: null pointer");
    tn::DeviceGuard g(h->device);
    return tn::guard_vertex_step(h, d_xyz_old, d_xyz_new, V, max_halvings, counts3, (cudaStream_t)stream);
}
