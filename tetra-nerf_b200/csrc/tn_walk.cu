// tn_walk.cu -- fast path of trace_rays: adjacency walk through the tetrahedral mesh.
// Two kernels with the same semantics: k_walk, one thread per ray, 32 rays per warp (throughput: large batches), and k_walk_quad,
// four cooperating lanes per ray (latency: 4 lanes shear the 4 vertices and test the candidate exit faces at once, so a step is
// one L2/L1 round trip plus ~150 dependent instructions, with no lane divergence and no 32-way scattered loads and stores), with
// 8 rays per warp or, launched with one ray per warp, only the first quad of each warp walking.
//
// The reference gathers every face hit of a ray with an OptiX any-hit program, sorts them and pairs consecutive
// faces (src/optix/optix_trace_rays.cu:268-331).  In a conforming mesh with a convex hull (every Delaunay
// triangulation) the hit faces of a generic ray are exactly the faces crossed when walking tetrahedron to
// tetrahedron from the hull entry face, already in order -- ~40x fewer instructions per ray than the all-hits BVH
// gather of tn_trace.cu.  Bit-exactness with the oracle is kept by construction and by classification:
//   * every face is tested in its stored winding (WalkRec::wind) with the same watertight fp32 test, so (t,u,v) are
//     the bits the exact path computes;
//   * a ray is emitted directly ("generic") only if every step found exactly ONE exit face and consecutive hits
//     are >= eps apart -- then the reference's dedupe phase is a no-op and its pairing is the identity;
//   * a ray that met a crossing shorter than eps keeps its (t, face) key list; the exact sort + literal pairing
//     stage of tn_trace.cu runs on that list (mode "keys provided");
//   * anything else (zero or several exit faces: edge/vertex hits; origin inside the mesh) is re-traced by the
//     exact all-hits path.  Meshes that are not walkable (non-convex hull) never take this path.
#include "tn_common.cuh"

namespace tn {
typedef unsigned long long u64;
#define TN_EPS 1e-6f

struct WalkParams {
    const float *o, *d;
    uint32_t R, M;
    uint32_t *num, *cells;
    float *bary, *dist;
    uint32_t *verts;
    const WalkRec *walk;
    const float4 *hull_nodes;
    const LeafRec *hull_leaves;
    const uint32_t *hull_tet;
    BvhLevels hlv;
    float absmax;
    u64 *keys;              // [R, M] (t bits << 32 | face) in walk order
    uint32_t *list, *list_count;  // rays for the exact stage: ray | 0x80000000 = keys provided
};

constexpr int WALK_THREADS = 32;
__device__ __forceinline__ uint32_t sel4u(uint32_t k, uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return k == 0 ? a : (k == 1 ? b : (k == 2 ? c : d)); }

// a ray the walk cannot certify is re-traced from scratch by the exact all-hits stage of tn_trace.cu
__device__ __forceinline__ void list_exact(const WalkParams &p, uint32_t ray) {
    p.list[atomicAdd(p.list_count, 1u)] = ray;
    atomicAdd(p.list_count + 1, 1u);  // diagnostics: rays that need the all-hits gather
    p.num[ray] = 0;
}
// end of a walk: exact -> re-traced from scratch; not generic -> the exact stage sorts and pairs the nfaces keys the walk wrote;
// otherwise the nrec records the walk wrote are the result
__device__ __forceinline__ void finish_walk(const WalkParams &p, uint32_t ray, bool exact, bool generic, uint32_t nfaces, uint32_t nrec) {
    if (exact) {
        list_exact(p, ray);
    } else if (!generic) {
        p.list[atomicAdd(p.list_count, 1u)] = ray | 0x80000000u;
        p.num[ray] = nfaces;  // number of keys; the pairing stage replaces it by the number of records
    } else {
        p.num[ray] = nrec;
    }
}

__global__ void __launch_bounds__(WALK_THREADS) k_walk(const WalkParams p) {
    // sheared vertices of the current tetrahedron, one column per thread: the stored winding of a face selects three of
    // the four vertices at run time, which would force a register array into local memory; shared memory indexes freely
    __shared__ float ssm[12][WALK_THREADS];
    const int tid = threadIdx.x;
    const uint32_t ray = blockIdx.x * blockDim.x + threadIdx.x;
    if (ray >= p.R) return;
    const float ox = p.o[3 * (size_t)ray], oy = p.o[3 * (size_t)ray + 1], oz = p.o[3 * (size_t)ray + 2];
    const float dx = p.d[3 * (size_t)ray], dy = p.d[3 * (size_t)ray + 1], dz = p.d[3 * (size_t)ray + 2];
    const RaySetup rs = ray_setup(ox, oy, oz, dx, dy, dz);
    if (!rs.valid) { p.num[ray] = 0; return; }
    const size_t row = (size_t)ray * p.M;

    // ---- hull entry: closest hit over the hull faces (smallest (t, face id) key) ----
    u64 best = ~0ull;
    float bu = 0.f, bv = 0.f;
    uint32_t btet = TN_EMPTY, bj = 0, hullhits = 0;
    {
        const float ix = __fdiv_rn(1.0f, dx), iy = __fdiv_rn(1.0f, dy), iz = __fdiv_rn(1.0f, dz);
        const float pad = 4e-6f * (fmaxf(fabsf(ox), fmaxf(fabsf(oy), fabsf(oz))) + p.absmax);
        uint32_t stack[7 * TN_MAX_LEVELS + 8];
        int sp = 0;
        stack[sp++] = (uint32_t)(p.hlv.nlevels - 1) << 28;
        while (sp) {
            const uint32_t e = stack[--sp];
            const uint32_t cl = (e >> 28) - 1u, cbase = (e & 0x0FFFFFFFu) << TN_FAN_LOG2;
            const uint32_t nc = min(TN_FAN, p.hlv.count[cl] - cbase);
            for (uint32_t c = 0; c < nc; ++c) {
                const float4 *np = p.hull_nodes + 2 * (size_t)(p.hlv.offset[cl] + cbase + c);
                if (!slab(__ldg(np), __ldg(np + 1), ox, oy, oz, ix, iy, iz, pad)) continue;
                if (cl != 0) { stack[sp++] = (cl << 28) | (cbase + c); continue; }
                const float4 *lp = reinterpret_cast<const float4 *>(p.hull_leaves + cbase + c);
                const float4 v0 = __ldg(lp), v1 = __ldg(lp + 1), v2 = __ldg(lp + 2), v3 = __ldg(lp + 3);
                const uint32_t f[4] = {__float_as_uint(v0.w), __float_as_uint(v1.w), __float_as_uint(v2.w), __float_as_uint(v3.w)};
                if (!((f[0] | f[1] | f[2] | f[3]) & TN_FACE_HULL)) continue;
                const Sheared s[4] = {shear(rs, v0.x, v0.y, v0.z), shear(rs, v1.x, v1.y, v1.z), shear(rs, v2.x, v2.y, v2.z), shear(rs, v3.x, v3.y, v3.z)};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (!(f[j] & TN_FACE_HULL)) continue;
                    float t, u, v;  // a hull face is always owned: its stored winding is this rotation
                    if (tri_test(s[(j + 1) & 3], s[(j + 2) & 3], s[(j + 3) & 3], t, u, v)) {
                        const u64 k = ((u64)__float_as_uint(t) << 32) | (f[j] & TN_FACE_MASK);
                        hullhits++;
                        if (k < best) { best = k; bu = u; bv = v; btet = p.hull_tet[cbase + c]; bj = (uint32_t)j; }
                    }
                }
            }
        }
    }
    if (btet == TN_EMPTY) { p.num[ray] = 0; return; }  // the ray misses the mesh
    // A ray the walk may certify crosses the (closed, convex) hull exactly twice: once in, once out.  One hull hit = the origin is
    // inside the mesh (the "entry" is the exit face: the walk would run backwards); more than two = the ray passes through a hull
    // edge or vertex, where the all-hits gather reports the extra hull faces -- they count towards the M-1 hit cap
    // (optix_trace_rays.cu:312-315) although pairing drops them again.  Both go to the exact all-hits stage at once.
    if (hullhits != 2) { list_exact(p, ray); return; }

    // ---- walk ----
    uint32_t c = btet, jin = bj, fin = (uint32_t)best, nfaces = 1, nrec = 0;
    float t_in = __uint_as_float((uint32_t)(best >> 32)), u_in = bu, v_in = bv;
    bool generic = true, exact = false, prev_small = false;
    p.keys[row] = best;
    for (;;) {
        const float4 *wp = reinterpret_cast<const float4 *>(p.walk + c);
        const float4 v0 = __ldg(wp), v1 = __ldg(wp + 1), v2 = __ldg(wp + 2), v3 = __ldg(wp + 3);
        const uint4 nb = __ldg(reinterpret_cast<const uint4 *>(wp + 4));
        const uint4 vid = __ldg(reinterpret_cast<const uint4 *>(wp + 5));
        const uint4 map = __ldg(reinterpret_cast<const uint4 *>(wp + 6));
        const uint2 wp2 = __ldg(reinterpret_cast<const uint2 *>(wp + 7));
        const uint32_t wind = wp2.x, perm = wp2.y;
        // the next record is one of the neighbours: start fetching all of them while this tetrahedron is intersected
        if (nb.x != TN_EMPTY) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.walk + nb.x));
        if (nb.y != TN_EMPTY) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.walk + nb.y));
        if (nb.z != TN_EMPTY) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.walk + nb.z));
        if (nb.w != TN_EMPTY) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.walk + nb.w));
        const uint32_t fw0 = __float_as_uint(v0.w), fw1 = __float_as_uint(v1.w), fw2 = __float_as_uint(v2.w), fw3 = __float_as_uint(v3.w);
        // locate the entry face inside this tetrahedron (after the first step it is the face shared with the previous one)
        jin = (fw0 & TN_FACE_MASK) == fin ? 0u : ((fw1 & TN_FACE_MASK) == fin ? 1u : ((fw2 & TN_FACE_MASK) == fin ? 2u : 3u));
        {
            const Sheared s0 = shear(rs, v0.x, v0.y, v0.z), s1 = shear(rs, v1.x, v1.y, v1.z), s2 = shear(rs, v2.x, v2.y, v2.z), s3 = shear(rs, v3.x, v3.y, v3.z);
            ssm[0][tid] = s0.x; ssm[1][tid] = s0.y; ssm[2][tid] = s0.z; ssm[3][tid] = s1.x; ssm[4][tid] = s1.y; ssm[5][tid] = s1.z;
            ssm[6][tid] = s2.x; ssm[7][tid] = s2.y; ssm[8][tid] = s2.z; ssm[9][tid] = s3.x; ssm[10][tid] = s3.y; ssm[11][tid] = s3.z;
        }
        uint32_t hits = 0, jout = 0;
        float t_out = 0.f, u_out = 0.f, v_out = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if ((uint32_t)j == jin) continue;
            const uint32_t w = (wind >> (6 * j)) & 63u;
            const uint32_t a = (w & 3u) * 3u, b = ((w >> 2) & 3u) * 3u, cc = ((w >> 4) & 3u) * 3u;
            Sheared A, B, Cv;
            A.x = ssm[a][tid]; A.y = ssm[a + 1][tid]; A.z = ssm[a + 2][tid];
            B.x = ssm[b][tid]; B.y = ssm[b + 1][tid]; B.z = ssm[b + 2][tid];
            Cv.x = ssm[cc][tid]; Cv.y = ssm[cc + 1][tid]; Cv.z = ssm[cc + 2][tid];
            float t, u, v;
            if (tri_test(A, B, Cv, t, u, v)) { hits++; jout = (uint32_t)j; t_out = t; u_out = u; v_out = v; }
        }
        if (hits != 1) { exact = true; break; }
        const uint32_t fout = sel4u(jout, fw0, fw1, fw2, fw3) & TN_FACE_MASK;
        // An ISOLATED crossing shorter than eps (strictly increasing t, both neighbouring crossings >= eps) leaves the
        // reference's dedupe phase without effect (optix_trace_rays.cu:124-159: the two faces share the sliver, nothing was
        // marked before, the mark is cleared again) and its pairing phase just skips that record (:208).  Anything else
        // within eps (ties, inversions, two short crossings in a row) goes to the literal implementation.
        const bool small = fabsf(__fsub_rn(t_out, t_in)) < TN_EPS;
        if (!(t_out > t_in) || (small && prev_small)) generic = false;
        prev_small = small;
        if (generic && !small) {
            // record (optix_trace_rays.cu:216-225 with combine_indices :39-75), expressed in local vertex indices
            // (the vertex order and the slot of every exit barycentric come from the tables built with the record)
            const uint32_t pm = perm >> (8 * jin), mc = sel4u(jin, map.x, map.y, map.z, map.w) >> (6 * jout);
            const float r0 = __fsub_rn(__fsub_rn(1.0f, u_out), v_out);
            float o2[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const uint32_t code = (mc >> (2 * q)) & 3u;
                o2[q] = code == 0 ? r0 : (code == 1 ? u_out : (code == 2 ? v_out : 0.f));
            }
            const size_t g = row + nrec;
            p.cells[g] = c;
            reinterpret_cast<uint4 *>(p.verts)[g] = make_uint4(sel4u(pm & 3u, vid.x, vid.y, vid.z, vid.w), sel4u((pm >> 2) & 3u, vid.x, vid.y, vid.z, vid.w),
                                                               sel4u((pm >> 4) & 3u, vid.x, vid.y, vid.z, vid.w), sel4u((pm >> 6) & 3u, vid.x, vid.y, vid.z, vid.w));
            float2 *bp = reinterpret_cast<float2 *>(p.bary + 6 * g);
            bp[0] = make_float2(__fsub_rn(__fsub_rn(1.0f, u_in), v_in), u_in);
            bp[1] = make_float2(v_in, o2[0]);
            bp[2] = make_float2(o2[1], o2[2]);
            reinterpret_cast<float2 *>(p.dist)[g] = make_float2(t_in, t_out);
            nrec++;
        }
        p.keys[row + nfaces] = ((u64)__float_as_uint(t_out) << 32) | fout;
        nfaces++;
        const uint32_t next = sel4u(jout, nb.x, nb.y, nb.z, nb.w);
        if (next == TN_EMPTY) break;  // left the mesh
        // Hit cap (optix_trace_rays.cu:312-315; pinned: the M-1 smallest (t, face id) keys survive).  The first M-1 faces in WALK order
        // are those only if nothing behind them ties with or precedes the last one (a zero-length tetrahedron at the cut sorts its
        // exit face first when that face has the smaller id) -- the walk cannot know without going on, so a ray that really is
        // truncated goes to the exact all-hits stage and its rank selection.  M = 512 never truncates on the meshes of SURVEY §8d.
        if (nfaces >= p.M - 1) { exact = true; break; }
        c = next; fin = fout; t_in = t_out; u_in = u_out; v_in = v_out;
    }
    finish_walk(p, ray, exact, generic, nfaces, nrec);
}

// ---- four cooperating lanes per ray ("quad"), eight rays per warp -----------------------------------------------------------------
// Same outputs, classification and fallbacks as k_walk (the same algorithm).  A 4096-ray batch is 512 warps = 3.5 per SM: the walk is
// a serial chain of L2 round trips per ray, so what matters at this size is how many instructions are issued per step and how many
// chains are in flight per scheduler.  One ray per warp issues a full warp instruction stream per ray (28 warps per SM fight for
// issue slots); 32 rays per warp (k_walk) leaves 128 warps for 132 SMs.  Here a warp instruction stream serves 8 rays: lane j of a
// quad owns vertex j and the face opposite to it.
// RPW: rays per warp, 8 or 1 (the "solo" form trace_rays can be set to use): with 1, only quad 0 of each warp carries a ray; the
// other quads take part in the warp-wide shuffles, ballots and barriers only, as they do for rays past the end of the batch.
// SPEC: the records of all candidate next tetrahedra (the neighbours across the three faces the ray did not enter through) are LOADED
// while the current one is intersected and the right one is selected afterwards, instead of prefetched into L1: ncu (round 2) put 25 %
// of the walk's stall samples on the first use of the next record although it had been prefetched a step earlier.  Three times the L2
// traffic of the walk, which is irrelevant while the walk is latency-bound (batches that do not fill the machine); large batches keep
// the prefetch.
constexpr int QUAD_WARPS = 2;  // 64 threads = 16 rays per block: 256 blocks for 4096 rays, spread over all SMs
template <bool SPEC, int RPW>
__global__ void __launch_bounds__(QUAD_WARPS * 32) k_walk_quad(const WalkParams p) {
    static_assert(RPW == 8 || RPW == 1, "a warp walks 8 rays (one per quad) or one");
    __shared__ uint32_t s_stack[QUAD_WARPS * RPW][8 * TN_MAX_LEVELS + 8];
    constexpr unsigned FULLM = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t lq = lane & 3u, gbase = lane & ~3u, grp = lane >> 2;  // lane inside the quad, first lane of the quad, quad inside the warp
    const uint32_t ray = (blockIdx.x * QUAD_WARPS + warp) * (uint32_t)RPW + grp;
    const bool in_range = (RPW == 8 || grp == 0) && ray < p.R;
    const uint32_t rr = in_range ? ray : 0u;
    uint32_t *stack = s_stack[warp * RPW + (RPW == 8 ? grp : 0u)];
    const float ox = p.o[3 * (size_t)rr], oy = p.o[3 * (size_t)rr + 1], oz = p.o[3 * (size_t)rr + 2];
    const float dx = p.d[3 * (size_t)rr], dy = p.d[3 * (size_t)rr + 1], dz = p.d[3 * (size_t)rr + 2];
    const RaySetup rs = ray_setup(ox, oy, oz, dx, dy, dz);
    const size_t row = (size_t)rr * p.M;
    bool live = in_range && rs.valid;  // quad-uniform
    if (in_range && !rs.valid && lq == 0) p.num[ray] = 0;

    // ---- hull entry: closest hit over the hull faces; lane lq takes children lq and lq + 4 of the popped node ----
    u64 best = ~0ull;
    float bu = 0.f, bv = 0.f;
    uint32_t btet = TN_EMPTY, bj = 0, hullhits = 0;
    {
        const float ix = __fdiv_rn(1.0f, dx), iy = __fdiv_rn(1.0f, dy), iz = __fdiv_rn(1.0f, dz);
        const float pad = 4e-6f * (fmaxf(fabsf(ox), fmaxf(fabsf(oy), fabsf(oz))) + p.absmax);
        int sp = live ? 1 : 0;
        if (live && lq == 0) stack[0] = (uint32_t)(p.hlv.nlevels - 1) << 28;
        __syncwarp();
        while (__any_sync(FULLM, sp > 0)) {
            const bool act = sp > 0;
            uint32_t e = 0;
            if (act) e = stack[--sp];
            __syncwarp();  // every lane of the quad has read the entry before it can be overwritten
            const uint32_t cl = act ? (e >> 28) - 1u : 0u, cbase = (e & 0x0FFFFFFFu) << TN_FAN_LOG2;
            const uint32_t nc = act ? min(TN_FAN, p.hlv.count[cl] - cbase) : 0u;
            bool hit[2] = {false, false};
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const uint32_t c = lq + 4u * (uint32_t)k;
                if (c < nc) {
                    const float4 *np = p.hull_nodes + 2 * (size_t)(p.hlv.offset[cl] + cbase + c);
                    hit[k] = slab(__ldg(np), __ldg(np + 1), ox, oy, oz, ix, iy, iz, pad);
                }
            }
            const uint32_t m0 = (__ballot_sync(FULLM, hit[0]) >> gbase) & 0xFu, m1 = (__ballot_sync(FULLM, hit[1]) >> gbase) & 0xFu;
            if (act && cl != 0) {
                if (hit[0]) stack[sp + __popc(m0 & ((1u << lq) - 1u))] = (cl << 28) | (cbase + lq);
                if (hit[1]) stack[sp + __popc(m0) + __popc(m1 & ((1u << lq) - 1u))] = (cl << 28) | (cbase + lq + 4u);
                sp += __popc(m0) + __popc(m1);
            } else if (act) {
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    if (!hit[k]) continue;  // a hull tetrahedron: its hull faces are owned, their stored winding is this rotation
                    const uint32_t c = lq + 4u * (uint32_t)k;
                    const float4 *lp = reinterpret_cast<const float4 *>(p.hull_leaves + cbase + c);
                    const float4 v0 = __ldg(lp), v1 = __ldg(lp + 1), v2 = __ldg(lp + 2), v3 = __ldg(lp + 3);
                    const uint32_t f[4] = {__float_as_uint(v0.w), __float_as_uint(v1.w), __float_as_uint(v2.w), __float_as_uint(v3.w)};
                    const Sheared sv[4] = {shear(rs, v0.x, v0.y, v0.z), shear(rs, v1.x, v1.y, v1.z), shear(rs, v2.x, v2.y, v2.z), shear(rs, v3.x, v3.y, v3.z)};
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (!(f[j] & TN_FACE_HULL)) continue;
                        float t, u, v;
                        if (tri_test(sv[(j + 1) & 3], sv[(j + 2) & 3], sv[(j + 3) & 3], t, u, v)) {
                            const u64 key = ((u64)__float_as_uint(t) << 32) | (f[j] & TN_FACE_MASK);
                            hullhits++;
                            if (key < best) { best = key; bu = u; bv = v; btet = p.hull_tet[cbase + c]; bj = (uint32_t)j; }
                        }
                    }
                }
            }
            __syncwarp();
        }
        // the smallest key over the quad wins (keys are unique: a face is tested by one lane only)
        u64 m = best;
#pragma unroll
        for (int o = 2; o >= 1; o >>= 1) {
            const u64 other = __shfl_xor_sync(FULLM, m, o);
            m = other < m ? other : m;
            hullhits += __shfl_xor_sync(FULLM, hullhits, o);
        }
        const uint32_t winm = (__ballot_sync(FULLM, best == m) >> gbase) & 0xFu;
        const uint32_t win = gbase + (winm ? (uint32_t)__ffs(winm) - 1u : 0u);
        best = m;
        bu = __shfl_sync(FULLM, bu, win); bv = __shfl_sync(FULLM, bv, win);
        btet = __shfl_sync(FULLM, btet, win); bj = __shfl_sync(FULLM, bj, win);
    }
    if (live && btet == TN_EMPTY) { if (lq == 0) p.num[ray] = 0; live = false; }  // the ray misses the mesh
    if (live && hullhits != 2) {  // origin inside the mesh, or a hull edge / vertex hit: exact all-hits stage (see k_walk)
        if (lq == 0) list_exact(p, ray);
        live = false;
    }

    // ---- walk: lane lq owns vertex lq / the face opposite to it; every lane of the quad keeps the (quad-uniform) bookkeeping ----
    uint32_t c = live ? btet : 0u, jin = bj, fin = (uint32_t)best, nfaces = 1, nrec = 0;
    float t_in = __uint_as_float((uint32_t)(best >> 32)), u_in = bu, v_in = bv;
    bool generic = true, exact = false, prev_small = false, walking = live;
    if (live && lq == 0) p.keys[row] = best;
    // this lane's part of the current tetrahedron's record (SPEC: carried from the previous step's speculative loads)
    float4 vj = make_float4(0.f, 0.f, 0.f, 0.f);
    uint32_t nbj = TN_EMPTY, vidj = 0;
    uint2 wp2 = make_uint2(0u, 0u);
    auto load_rec = [&](uint32_t tet, float4 &v, uint32_t &nb, uint32_t &vid, uint2 &w2) {
        const float4 *wp = reinterpret_cast<const float4 *>(p.walk + tet);
        const uint32_t *wq = reinterpret_cast<const uint32_t *>(wp);
        v = __ldg(wp + lq);                  // vertex lq + the face id opposite to it
        nb = __ldg(wq + 16 + lq);            // neighbour across my face
        vid = __ldg(wq + 20 + lq);           // my vertex id
        w2 = __ldg(reinterpret_cast<const uint2 *>(wp + 7));
    };
    if (SPEC && walking) load_rec(c, vj, nbj, vidj, wp2);
    while (__any_sync(FULLM, walking)) {
        const uint32_t *wq = reinterpret_cast<const uint32_t *>(p.walk + c);
        if (!SPEC) {
            vj = make_float4(0.f, 0.f, 0.f, 0.f); nbj = TN_EMPTY; vidj = 0; wp2 = make_uint2(0u, 0u);
            if (walking) {
                load_rec(c, vj, nbj, vidj, wp2);
                if (nbj != TN_EMPTY) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.walk + nbj));  // the next record is one of the neighbours
            }
        }
        const uint32_t wind = wp2.x, perm = wp2.y;
        const uint32_t fwj = __float_as_uint(vj.w);
        const uint32_t inm = (__ballot_sync(FULLM, walking && (fwj & TN_FACE_MASK) == fin) >> gbase) & 0xFu;  // entry face
        jin = inm ? (uint32_t)__ffs(inm) - 1u : 3u;
        // SPEC: this lane's part of every candidate next record, in flight while the faces are tested
        float4 cv[4];
        uint32_t cnb[4], cvid[4];
        uint2 cw[4];
        if (SPEC) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t nk = __shfl_sync(FULLM, nbj, gbase + k);
                cv[k] = make_float4(0.f, 0.f, 0.f, 0.f); cnb[k] = TN_EMPTY; cvid[k] = 0; cw[k] = make_uint2(0u, 0u);
                if (walking && (uint32_t)k != jin && nk != TN_EMPTY) load_rec(nk, cv[k], cnb[k], cvid[k], cw[k]);
            }
        }
        const Sheared sj = shear(rs, vj.x, vj.y, vj.z);
        const uint32_t w = (wind >> (6 * lq)) & 63u;  // stored winding of my face as local vertex indices
        const uint32_t a = gbase + (w & 3u), b = gbase + ((w >> 2) & 3u), cc = gbase + ((w >> 4) & 3u);
        Sheared A, B, Cv;
        A.x = __shfl_sync(FULLM, sj.x, a); A.y = __shfl_sync(FULLM, sj.y, a); A.z = __shfl_sync(FULLM, sj.z, a);
        B.x = __shfl_sync(FULLM, sj.x, b); B.y = __shfl_sync(FULLM, sj.y, b); B.z = __shfl_sync(FULLM, sj.z, b);
        Cv.x = __shfl_sync(FULLM, sj.x, cc); Cv.y = __shfl_sync(FULLM, sj.y, cc); Cv.z = __shfl_sync(FULLM, sj.z, cc);
        float t = 0.f, u = 0.f, v = 0.f;
        const bool tri = tri_test_nobranch(A, B, Cv, t, u, v);
        const bool hit = walking && lq != jin && tri;
        const uint32_t hm = (__ballot_sync(FULLM, hit) >> gbase) & 0xFu;
        const bool one = __popc(hm) == 1;
        const uint32_t jout = hm ? (uint32_t)__ffs(hm) - 1u : 0u;
        const float t_out = __shfl_sync(FULLM, t, gbase + jout), u_out = __shfl_sync(FULLM, u, gbase + jout), v_out = __shfl_sync(FULLM, v, gbase + jout);
        const uint32_t fout = __shfl_sync(FULLM, fwj, gbase + jout) & TN_FACE_MASK;
        const uint32_t next = __shfl_sync(FULLM, nbj, gbase + jout);
        const uint32_t vq = __shfl_sync(FULLM, vidj, gbase + ((perm >> (8 * jin + 2 * lq)) & 3u));
        if (walking) {
            if (!one) { exact = true; walking = false; }
            else {
                // isolated sub-eps crossings: see k_walk
                const bool small = fabsf(__fsub_rn(t_out, t_in)) < TN_EPS;
                if (!(t_out > t_in) || (small && prev_small)) generic = false;
                prev_small = small;
                // record (optix_trace_rays.cu:216-225 with combine_indices :39-75): lane q writes slot q of every field
                if (generic && !small) {
                    const size_t g = row + nrec;
                    const uint32_t code = (__ldg(wq + 24 + jin) >> (6 * jout + 2 * lq)) & 3u;  // map[jin]: same line, L1 hit
                    const float r0 = __fsub_rn(__fsub_rn(1.0f, u_out), v_out), e0 = __fsub_rn(__fsub_rn(1.0f, u_in), v_in);
                    const float ev = sel3((int)lq, e0, u_in, v_in);
                    float xv = sel3((int)code, r0, u_out, v_out);
                    xv = code == 3u ? 0.f : xv;
                    p.verts[4 * g + lq] = vq;
                    if (lq < 3u) {
                        p.bary[6 * g + lq] = ev;
                        p.bary[6 * g + 3 + lq] = xv;
                    } else {
                        p.cells[g] = c;
                        reinterpret_cast<float2 *>(p.dist)[g] = make_float2(t_in, t_out);
                    }
                    nrec++;
                }
                if (lq == 0) p.keys[row + nfaces] = ((u64)__float_as_uint(t_out) << 32) | fout;
                nfaces++;
                if (next == TN_EMPTY) walking = false;                              // left the mesh
                else if (nfaces >= p.M - 1) { exact = true; walking = false; }      // truncated by the hit cap: exact stage (see k_walk)
                else {
                    c = next; fin = fout; t_in = t_out; u_in = u_out; v_in = v_out;
                    if (SPEC) {  // the record of the tetrahedron behind the exit face has been loaded already
                        vj = jout == 0u ? cv[0] : (jout == 1u ? cv[1] : (jout == 2u ? cv[2] : cv[3]));
                        nbj = jout == 0u ? cnb[0] : (jout == 1u ? cnb[1] : (jout == 2u ? cnb[2] : cnb[3]));
                        vidj = jout == 0u ? cvid[0] : (jout == 1u ? cvid[1] : (jout == 2u ? cvid[2] : cvid[3]));
                        wp2 = jout == 0u ? cw[0] : (jout == 1u ? cw[1] : (jout == 2u ? cw[2] : cw[3]));
                    }
                }
            }
        }
    }
    if (!live || lq != 0) return;
    finish_walk(p, ray, exact, generic, nfaces, nrec);
}

// dense API tails (optix_trace_rays.cu:260-265 + the zeroed scratch tails pinned by the oracle): one warp per ray
__global__ void k_tail_fill(uint32_t R, uint32_t M, const uint32_t *__restrict__ num, uint32_t *__restrict__ cells, float *__restrict__ bary,
                            float *__restrict__ dist, uint32_t *__restrict__ verts) {
    const uint32_t ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (ray >= R) return;
    const size_t row = (size_t)ray * M;
    for (uint32_t j = num[ray] + lane; j < M; j += 32) {
        const size_t g = row + j;
        cells[g] = TN_EMPTY;
        reinterpret_cast<uint4 *>(verts)[g] = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
        float2 *bp = reinterpret_cast<float2 *>(bary + 6 * g);
        bp[0] = make_float2(0.f, 0.f); bp[1] = make_float2(0.f, 0.f); bp[2] = make_float2(0.f, 0.f);
        reinterpret_cast<float2 *>(dist)[g] = make_float2(0.f, 0.f);
    }
}

int launch_walk(tn_tracer *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells, float *bary,
                float *dist, uint32_t *verts, u64 *keys, uint32_t *list, uint32_t *list_count, int kind, cudaStream_t s) {
    WalkParams p{};
    p.o = o; p.d = d; p.R = R; p.M = M; p.num = num; p.cells = cells; p.bary = bary; p.dist = dist; p.verts = verts;
    p.walk = h->mesh.walk.p; p.hull_nodes = h->mesh.hull_nodes.p; p.hull_leaves = h->mesh.hull_leaves.p; p.hull_tet = h->mesh.hull_tet.p;
    p.hlv = h->mesh.hull_lv; p.absmax = h->mesh.absmax; p.keys = keys; p.list = list; p.list_count = list_count;
    if (kind == 1 || kind == 2) {  // 4 lanes per ray: kind 2 = 8 rays per warp, kind 1 = one ray per warp
        const bool spec = R <= h->walk_quad_spec_max_rays;  // speculative record loads, else prefetched
        const uint32_t rpw = kind == 2 ? 8u : 1u;
        auto kern = kind == 2 ? (spec ? k_walk_quad<true, 8> : k_walk_quad<false, 8>) : (spec ? k_walk_quad<true, 1> : k_walk_quad<false, 1>);
        kern<<<(R + QUAD_WARPS * rpw - 1) / (QUAD_WARPS * rpw), QUAD_WARPS * 32, 0, s>>>(p);
    } else {
        k_walk<<<(R + WALK_THREADS - 1) / WALK_THREADS, WALK_THREADS, 0, s>>>(p);  // 32 rays per warp
    }
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}
int launch_tail_fill(tn_tracer *h, uint32_t R, uint32_t M, const uint32_t *num, uint32_t *cells, float *bary, float *dist, uint32_t *verts,
                     cudaStream_t s) {
    k_tail_fill<<<(uint32_t)(((size_t)R * 32 + 255) / 256), 256, 0, s>>>(R, M, num, cells, bary, dist, verts);
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}
}  // namespace tn
