// tn_trace.cu -- trace_rays / trace_rays_triangles on sm_90a without OptiX.
//
// Replaces src/optix/optix_trace_rays.cu (+ the OptiX host runtime in src/tetrahedra_tracer.cpp:137-176,
// 342-587).  One WARP per ray:
//   1. all-hits gather (semantics of __anyhit__ms, optix_trace_rays.cu:310-331): the warp walks the
//      implicit 4-ary BVH with a shared LIFO work list -- every lane pops a different node, tests its
//      4 children, and the survivors are re-packed with a warp scan (order is irrelevant because ALL
//      hits are wanted, so the frontier is embarrassingly parallel).  Leaves are tetrahedra; a lane
//      tests only the faces its tetrahedron OWNS (first owner in reference numbering), so each unique
//      face is tested once, in the reference's stored winding, by the watertight fp32 test of
//      tn_common.cuh (bit-identical to oracle/tetra_oracle.cpp).
//   2. hits live in shared memory as 64-bit keys (t bits << 32 | face id): a bitonic sort of the keys
//      is the reference's bitonic_sort (optix_trace_rays.cu:78-108) with ties pinned by face id.
//      (u,v) are not carried through the sort; they are recomputed for the <= 2 faces of each emitted
//      record (same function, same inputs -> same bits).
//   3. post_process_tetrahedra (optix_trace_rays.cu:110-266): if no two consecutive hits are within
//      eps and every consecutive pair shares a tetrahedron (the generic case) the pairing is the
//      identity and all lanes emit records in parallel; otherwise lane 0 runs the literal three-phase
//      algorithm on the shared-memory keys and the lanes emit from its result.
// More than M-1 hits: the M-1 smallest keys are kept (the reference keeps an arbitrary M-1).
#include <algorithm>
#include <cstdlib>

#include "tn_common.cuh"
#include "tn_pairing.cuh"

namespace tn {

using namespace pairing;  // key_t, key_face, face_hit, the key sorts, pair_and_emit, FULL
constexpr int TRACE_WARPS = 4;

struct TraceParams {
    const float *o, *d;
    uint32_t R, M;
    uint32_t *num, *cells;
    float *bary, *dist;
    uint32_t *verts;
    const float4 *nodes;
    const LeafRec *leaves;
    const uint4 *tri;
    const uint2 *tt;
    const float *xyz;
    BvhLevels lv;
    float absmax;
    int dense;
    int *flags;
    uint32_t hcap, scap, lcap;
    // two-phase launch: phase 1 (small hit buffer, high occupancy) appends rays whose hits do not fit to
    // `ovf_list` (count in ovf_count); phase 2 (ray_list != nullptr) re-traces exactly those with the full buffer
    uint32_t *ovf_count, *ovf_list;
    const uint32_t *ray_count, *ray_list;
    // list entries with bit 31 set carry their face hits already (written by the adjacency walk, tn_walk.cu):
    // num[ray] keys at keys_in[ray*M ..]; the gather is skipped and only sort + pairing + emit run
    const u64 *keys_in;
};

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += t;
    }
    return v;
}
// keep the `keep` smallest of hits[0..nh) (keys are distinct), compacting in place; returns the
// largest kept key.  Rare path (ray with more than M-1 face hits).
__device__ u64 rank_select(u64 *hits, uint32_t &nh, uint32_t keep, int lane) {
    u64 f0 = 0, f1 = 0;
    for (uint32_t k = 0; lane + 32 * k < nh; ++k) {
        const u64 key = hits[lane + 32 * k];
        uint32_t rank = 0;
        for (uint32_t j = 0; j < nh; ++j) rank += (hits[j] < key) ? 1u : 0u;
        if (rank < keep) { if (k < 64) f0 |= 1ull << k; else f1 |= 1ull << (k - 64); }
    }
    __syncwarp();
    uint32_t base = 0;
    u64 mx = 0;
    for (uint32_t k = 0; 32 * k < nh; ++k) {
        const uint32_t i = lane + 32 * k;
        const bool kp = i < nh && (((k < 64) ? (f0 >> k) : (f1 >> (k - 64))) & 1ull);
        const u64 key = kp ? hits[i] : 0ull;
        const uint32_t mask = __ballot_sync(FULL, kp);
        __syncwarp();
        if (kp) { hits[base + __popc(mask & ((1u << lane) - 1u))] = key; mx = key > mx ? key : mx; }
        base += __popc(mask);
        __syncwarp();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const u64 t = __shfl_xor_sync(FULL, mx, o); mx = t > mx ? t : mx; }
    nh = base;
    return mx;
}

template <int MODE>  // 0: trace_rays (tetrahedra), 1: trace_rays_triangles (sorted raw face hits)
__global__ void __launch_bounds__(TRACE_WARPS * 32, 7) k_trace(const TraceParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ uint32_t s_count[TN_MAX_LEVELS], s_offset[TN_MAX_LEVELS];
    if (threadIdx.x < TN_MAX_LEVELS) { s_count[threadIdx.x] = p.lv.count[threadIdx.x]; s_offset[threadIdx.x] = p.lv.offset[threadIdx.x]; }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t per_warp = (size_t)p.hcap * 8 + (size_t)p.scap * 4 + (size_t)p.lcap * 4;
    unsigned char *base = smem_raw + (size_t)warp * per_warp;
    u64 *hits = reinterpret_cast<u64 *>(base);
    uint32_t *stack = reinterpret_cast<uint32_t *>(base + (size_t)p.hcap * 8);
    uint32_t *leafq = stack + p.scap;
    const uint32_t M = p.M;

    const uint32_t nwork = p.ray_list ? *p.ray_count : p.R;
    for (uint32_t wi = blockIdx.x * TRACE_WARPS + warp; wi < nwork; wi += gridDim.x * TRACE_WARPS) {
        const uint32_t entry = p.ray_list ? p.ray_list[wi] : wi;
        const uint32_t ray = entry & 0x7FFFFFFFu;
        const bool provided = p.keys_in != nullptr && (entry >> 31) != 0u;
        const float ox = p.o[3 * (size_t)ray], oy = p.o[3 * (size_t)ray + 1], oz = p.o[3 * (size_t)ray + 2];
        const float dx = p.d[3 * (size_t)ray], dy = p.d[3 * (size_t)ray + 1], dz = p.d[3 * (size_t)ray + 2];
        const RaySetup rs = ray_setup(ox, oy, oz, dx, dy, dz);
        const float ix = __fdiv_rn(1.0f, dx), iy = __fdiv_rn(1.0f, dy), iz = __fdiv_rn(1.0f, dz);
        const float pad = 4e-6f * (fmaxf(fabsf(ox), fmaxf(fabsf(oy), fabsf(oz))) + p.absmax);

        uint32_t sc = 0, lc = 0, nh = 0;
        u64 cutoff = ~0ull;
        bool overflow = false, deferred = false;
        if (provided) {
            nh = p.num[ray];
            for (uint32_t i = lane; i < nh; i += 32) hits[i] = p.keys_in[(size_t)ray * M + i];
        } else if (rs.valid) {
            if (lane == 0) stack[0] = (uint32_t)(p.lv.nlevels - 1) << 28;
            sc = 1;
        }
        __syncwarp();

        // ---------------- 1. all-hits gather ----------------
        while (sc | lc) {
            if (lc >= 32 || sc == 0) {
                const uint32_t room = (p.hcap - nh) >> 2;
                const uint32_t n = min(min(lc, 32u), room);
                if (n == 0) {
                    if (p.ovf_list != nullptr) { deferred = true; break; }  // phase 1: this ray needs the large buffer
                    // hit buffer full: nh > M-1 for sure, drop everything beyond the M-1 nearest
                    cutoff = rank_select(hits, nh, M - 1, lane);
                    continue;
                }
                u64 k0 = 0, k1 = 0, k2 = 0, k3 = 0;
                uint32_t fl = 0;
                if (lane < n) {
                    const uint32_t pos = leafq[lc - 1 - lane];
                    const float4 *lp = reinterpret_cast<const float4 *>(p.leaves + pos);
                    const float4 v0 = __ldg(lp), v1 = __ldg(lp + 1), v2 = __ldg(lp + 2), v3 = __ldg(lp + 3);
                    const Sheared s0 = shear(rs, v0.x, v0.y, v0.z), s1 = shear(rs, v1.x, v1.y, v1.z);
                    const Sheared s2 = shear(rs, v2.x, v2.y, v2.z), s3 = shear(rs, v3.x, v3.y, v3.z);
                    const uint32_t f0 = __float_as_uint(v0.w), f1 = __float_as_uint(v1.w), f2 = __float_as_uint(v2.w), f3 = __float_as_uint(v3.w);
                    float t, u, v;
                    // face j = (v[(j+1)&3], v[(j+2)&3], v[(j+3)&3])   (src/tetrahedra_tracer.cpp:54-57)
                    if ((f0 >> 31) && tri_test(s1, s2, s3, t, u, v)) { k0 = ((u64)__float_as_uint(t) << 32) | (f0 & TN_FACE_MASK); if (k0 < cutoff) fl |= 1u; }
                    if ((f1 >> 31) && tri_test(s2, s3, s0, t, u, v)) { k1 = ((u64)__float_as_uint(t) << 32) | (f1 & TN_FACE_MASK); if (k1 < cutoff) fl |= 2u; }
                    if ((f2 >> 31) && tri_test(s3, s0, s1, t, u, v)) { k2 = ((u64)__float_as_uint(t) << 32) | (f2 & TN_FACE_MASK); if (k2 < cutoff) fl |= 4u; }
                    if ((f3 >> 31) && tri_test(s0, s1, s2, t, u, v)) { k3 = ((u64)__float_as_uint(t) << 32) | (f3 & TN_FACE_MASK); if (k3 < cutoff) fl |= 8u; }
                }
                const uint32_t c = __popc(fl);
                const uint32_t incl = warp_incl_scan(c, lane);
                const uint32_t total = __shfl_sync(FULL, incl, 31);
                uint32_t w = nh + incl - c;
                if (fl & 1u) hits[w++] = k0;
                if (fl & 2u) hits[w++] = k1;
                if (fl & 4u) hits[w++] = k2;
                if (fl & 8u) hits[w++] = k3;
                nh += total;
                lc -= n;
                __syncwarp();
            } else {
                const uint32_t n = min(min(sc, 32u), (p.scap - sc) / (TN_FAN - 1u));
                if (n == 0) { if (p.ovf_list != nullptr) deferred = true; else overflow = true; break; }
                uint32_t hm = 0, cl = 1, cbase = 0;
                if (lane < n) {
                    const uint32_t e = stack[sc - 1 - lane];
                    cl = (e >> 28) - 1u;
                    cbase = (e & 0x0FFFFFFFu) << TN_FAN_LOG2;
                    const uint32_t nc = min(TN_FAN, s_count[cl] - cbase);
                    const float4 *np = p.nodes + 2 * (size_t)(s_offset[cl] + cbase);
#pragma unroll
                    for (uint32_t c = 0; c < TN_FAN; ++c) {
                        if (c < nc) {
                            const float4 a = __ldg(np + 2 * c), b = __ldg(np + 2 * c + 1);
                            if (slab(a, b, ox, oy, oz, ix, iy, iz, pad)) hm |= 1u << c;
                        }
                    }
                }
                __syncwarp();  // all pops are done before anything is pushed over them
                const uint32_t k = __popc(hm);
                const uint32_t packed = (cl == 0) ? (k << 16) : k;
                const uint32_t incl = warp_incl_scan(packed, lane);
                const uint32_t total = __shfl_sync(FULL, incl, 31);
                const uint32_t excl = incl - packed;
                uint32_t sb = sc - n + (excl & 0xFFFFu), lb = lc + (excl >> 16);
#pragma unroll
                for (uint32_t c = 0; c < TN_FAN; ++c) {
                    if (hm & (1u << c)) {
                        if (cl == 0) leafq[lb++] = cbase + c;
                        else stack[sb++] = (cl << 28) | (cbase + c);
                    }
                }
                sc = sc - n + (total & 0xFFFFu);
                lc += total >> 16;
                __syncwarp();
            }
        }
        // pairing stage: tts[] (8 bytes per hit) is staged over the work list ONLY (scap * 4 bytes); emit[] lives in leafq
        if (p.ovf_list != nullptr && nh > (p.scap >> 1)) deferred = true;
        if (deferred) {  // uniform per warp
            if (lane == 0) p.ovf_list[atomicAdd(p.ovf_count, 1u)] = ray;
            __syncwarp();
            continue;
        }
        if (overflow) {
            if (lane == 0) atomicAdd(p.flags, 1);
            nh = 0;
        }
        if (nh > M - 1) rank_select(hits, nh, M - 1, lane);  // (phase 1 never gets here with nh > hcap - 4 >= ... it defers first)

        // ---------------- 2. sort by (t, face id) ----------------
        if (nh > 1) {
            if (provided) sort_nearly_sorted(hits, nh, lane);
            else bitonic_sort_keys(hits, nh, lane);
        }
        __syncwarp();

        const size_t row = (size_t)ray * M;
        uint32_t jc = 0;
        if (MODE == 1) {
            // optix_trace_rays_triangles.cu:70-84 : sorted hits + their vertex ids
            for (uint32_t j = lane; j < nh; j += 32) {
                const uint32_t f = key_face(hits[j]);
                const uint4 tr = __ldg(p.tri + f);
                float t, u, v;
                face_hit(rs, p.xyz, tr, t, u, v);
                p.cells[row + j] = f;
                p.dist[row + j] = t;
                reinterpret_cast<float2 *>(p.bary)[row + j] = make_float2(u, v);
                p.verts[3 * (row + j)] = tr.x; p.verts[3 * (row + j) + 1] = tr.y; p.verts[3 * (row + j) + 2] = tr.z;
            }
            jc = nh;
            if (p.dense) {
                for (uint32_t j = nh + lane; j < M; j += 32) {
                    p.cells[row + j] = 0; p.dist[row + j] = 0.f;
                    reinterpret_cast<float2 *>(p.bary)[row + j] = make_float2(0.f, 0.f);
                    p.verts[3 * (row + j)] = 0; p.verts[3 * (row + j) + 1] = 0; p.verts[3 * (row + j) + 2] = 0;
                }
            }
        } else {
            // ---------------- 3. face pairing ----------------
            uint2 *tts = reinterpret_cast<uint2 *>(stack);
            uint16_t *emit = reinterpret_cast<uint16_t *>(leafq);
            const uint32_t nw = (nh + 31u) >> 5;  // mask words of the windowed pairing: behind tts[] in the work-list region when it has room
            uint32_t *mask = (size_t)nh * 8 + (size_t)nw * 12 <= (size_t)p.scap * 4 ? reinterpret_cast<uint32_t *>(tts + nh) : nullptr;
            const pairing::PairOut po{p.cells, p.verts, p.bary, p.dist};
            jc = pairing::pair_and_emit(hits, tts, emit, mask, nh, p.tt, p.tri, p.xyz, rs, row, po, lane);
            if (p.dense) {
                // phase 3 (optix_trace_rays.cu:260-265) + zeroed scratch tails (pinned, see oracle header)
                for (uint32_t j = jc + lane; j < M; j += 32) {
                    const size_t g = row + j;
                    p.cells[g] = TN_EMPTY;
                    reinterpret_cast<uint4 *>(p.verts)[g] = make_uint4(TN_EMPTY, TN_EMPTY, TN_EMPTY, TN_EMPTY);
                    float2 *bp = reinterpret_cast<float2 *>(p.bary + 6 * g);
                    bp[0] = make_float2(0.f, 0.f); bp[1] = make_float2(0.f, 0.f); bp[2] = make_float2(0.f, 0.f);
                    reinterpret_cast<float2 *>(p.dist)[g] = make_float2(0.f, 0.f);
                }
            }
        }
        if (lane == 0) p.num[ray] = jc;
        __syncwarp();
    }
}

// warm L2 with the read-only working set (BVH nodes, leaf records, face tables, vertices, ...): one bulk
// prefetch instruction per 16 KB instead of thousands of latency-bound first-touch misses inside k_trace.
struct PrefetchArgs {
    const void *ptr[8];
    unsigned long long bytes[8];
    int n;
};
__global__ void k_l2_prefetch(const PrefetchArgs a) {
    const unsigned long long CH = 16384ull;
    unsigned long long base = 0;
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (unsigned long long)gridDim.x * blockDim.x;
    for (int i = 0; i < a.n; ++i) {
        const unsigned long long nch = (a.bytes[i] + CH - 1) / CH;
        for (unsigned long long c = (tid + nth - base % nth) % nth; c < nch; c += nth) {
            const unsigned long long off = c * CH;
            const unsigned int sz = (unsigned int)min(CH, a.bytes[i] - off) & ~15u;
            if (sz) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"((const char *)a.ptr[i] + off), "r"(sz) : "memory");
        }
        base += nch;
    }
}

int launch_prefetch(tn_tracer *h, const void *const *extra, const size_t *extra_bytes, int nextra, cudaStream_t s) {
    const Mesh &m = h->mesh;
    PrefetchArgs a{};
    int n = 0;
    auto add = [&](const void *p, size_t b) { if (p && b && n < 8 && ((uintptr_t)p & 15) == 0) { a.ptr[n] = p; a.bytes[n] = b; ++n; } };
    if (m.walkable) {  // the walk touches one 128-byte record per crossed tetrahedron; the big BVH is only the rare exact path's
        add(m.walk.p, sizeof(WalkRec) * (size_t)m.T);
        add(m.hull_leaves.p, sizeof(LeafRec) * (size_t)m.H);
        add(m.hull_nodes.p, sizeof(float4) * 2 * (size_t)(m.hull_lv.offset[m.hull_lv.nlevels - 1] + TN_FAN));
    } else {
        const uint32_t total_nodes = m.lv.offset[m.lv.nlevels - 1] + TN_FAN;
        add(m.nodes.p, sizeof(float4) * 2 * (size_t)total_nodes);
        add(m.leaves.p, sizeof(LeafRec) * (size_t)m.T);
    }
    add(m.tri.p, sizeof(uint4) * (size_t)m.F);
    add(m.tt.p, sizeof(uint2) * (size_t)m.F);
    add(m.xyz, sizeof(float) * 3 * (size_t)m.V);
    for (int i = 0; i < nextra; ++i) add(extra[i], extra_bytes[i]);
    a.n = n;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    k_l2_prefetch<<<sms, 128, 0, s>>>(a);
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

static int launch_trace(tn_tracer *h, int mode, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells,
                        float *bary, float *dist, uint32_t *verts, int dense, cudaStream_t s) {
    if (!h) return fail(TN_ERR_ARG, "null tracer");
    if (M == 0 || (M & (M - 1)) != 0) return fail(TN_ERR_ARG, "max_ray_triangles must be a power of 2.");  // py_binding.cpp:44-47
    if (M < 2 || M > 2048) return fail(TN_ERR_ARG, "max_ray_triangles must be in [2, 2048]");
    if (!h->mesh.nodes.p) return fail(TN_ERR_STATE, "trace_rays: no tetrahedra loaded (call load_tetrahedra first)");
    if (R == 0) return TN_OK;
    DeviceGuard g(h->device);
    TraceParams p{};
    p.o = o; p.d = d; p.R = R; p.M = M; p.num = num; p.cells = cells; p.bary = bary; p.dist = dist; p.verts = verts;
    p.nodes = h->mesh.nodes.p; p.leaves = h->mesh.leaves.p; p.tri = h->mesh.tri.p; p.tt = h->mesh.tt.p;
    p.xyz = h->mesh.xyz; p.lv = h->mesh.lv; p.absmax = h->mesh.absmax; p.dense = dense; p.flags = h->d_flags.p;
    auto kern = mode == 0 ? k_trace<0> : k_trace<1>;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    auto launch = [&](uint32_t nblocks_wanted) -> int {
        const size_t smem = (size_t)TRACE_WARPS * ((size_t)p.hcap * 8 + (size_t)p.scap * 4 + (size_t)p.lcap * 4);
        TN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 1;
        TN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, TRACE_WARPS * 32, smem));
        if (occ < 1) occ = 1;
        const uint32_t grid = std::min<uint32_t>(nblocks_wanted, (uint32_t)(sms * occ));
        kern<<<grid, TRACE_WARPS * 32, smem, s>>>(p);
        h->launches += 1;
        TN_CUDA(cudaGetLastError());
        return TN_OK;
    };
    const uint32_t want = (R + TRACE_WARPS - 1) / TRACE_WARPS;
    // path choice.  The adjacency walk needs ~40x fewer instructions per ray than the all-hits gather but is a serial chain
    // of L2 round trips per ray: with >= walk_min_rays rays it runs 32 rays per warp (throughput); smaller batches in the quad
    // range run 4 lanes per ray, 8 rays per warp (latency: no divergence, no scattered 32-way accesses), and those in the solo
    // range 4 lanes per ray, one ray per warp; anything else, and meshes that cannot be walked, take the warp-per-ray BVH gather.
    const bool thread_walk = R >= h->walk_min_rays;
    const bool quad_walk = !thread_walk && R >= h->walk_quad_min_rays && R <= h->walk_quad_max_rays;
    const bool solo_walk = !thread_walk && !quad_walk && R >= h->walk_solo_min_rays && R <= h->walk_solo_max_rays;
    if (mode == 0 && h->mesh.walkable && M >= 4 && (thread_walk || solo_walk || quad_walk)) {
        // fast path: adjacency walk (tn_walk.cu); rays it cannot certify are listed for the exact stage below
        const size_t need = (size_t)R * M;
        TN_TRY(h->d_walk_keys.grow(need));
        TN_TRY(h->d_ovf_list.grow(R));
        uint32_t *list_count = reinterpret_cast<uint32_t *>(h->d_flags.p + 2);
        TN_CUDA(cudaMemsetAsync(list_count, 0, 2 * sizeof(uint32_t), s));
        int rc = launch_walk(h, o, d, R, M, num, cells, bary, dist, verts, h->d_walk_keys.p, h->d_ovf_list.p, list_count, thread_walk ? 0 : (quad_walk ? 2 : 1), s);
        if (rc) return rc;
        p.dense = 0;
        p.hcap = M + 128; p.scap = 4096; p.lcap = M > 512 ? M / 2 : 320;
        p.ray_count = list_count; p.ray_list = h->d_ovf_list.p; p.keys_in = h->d_walk_keys.p;
        rc = launch((uint32_t)sms);
        if (rc) return rc;
        if (dense) return launch_tail_fill(h, R, M, num, cells, bary, dist, verts, s);
        return TN_OK;
    }
    // phase 1: min(M + 128, 512) keys per ray (7.75 KB of shared memory per ray at M = 512 -> 28 rays per SM); rays whose hits
    // or work list do not fit are deferred to phase 2 (never dropped)
    TN_TRY(h->d_ovf_list.grow(R));
    uint32_t *ovf_count = reinterpret_cast<uint32_t *>(h->d_flags.p + 2);
    TN_CUDA(cudaMemsetAsync(ovf_count, 0, sizeof(uint32_t), s));
    p.hcap = M <= 256 ? M + 128 : M; p.scap = 640; p.lcap = 320; p.ovf_count = ovf_count; p.ovf_list = h->d_ovf_list.p;
    int rc = launch(want);
    if (rc) return rc;
    // phase 2: the deferred rays with the full streaming buffer (M + 128 keys) and a 4096-entry work list; exits at once
    // when there are none.  A work list overflow HERE is counted in d_flags[0] and reported by tn_synchronize.
    p.hcap = M + 128; p.scap = 4096; p.lcap = M > 512 ? M / 2 : 320;
    p.ovf_count = nullptr; p.ovf_list = nullptr; p.ray_count = ovf_count; p.ray_list = h->d_ovf_list.p;
    return launch((uint32_t)sms);
}

int launch_trace_internal(tn_tracer *h, const float *o, const float *d, uint32_t R, uint32_t M, uint32_t *num, uint32_t *cells, float *bary,
                          float *dist, uint32_t *verts, int dense, cudaStream_t s) {
    return launch_trace(h, 0, o, d, R, M, num, cells, bary, dist, verts, dense, s);
}

}  // namespace tn

extern "C" int tn_trace_rays(tn_tracer *h, const float *d_origins, const float *d_directions, uint32_t R, uint32_t M, uint32_t *d_num,
                             uint32_t *d_cells, float *d_bary, float *d_dist, uint32_t *d_verts, int dense, void *stream) {
    return tn::launch_trace(h, 0, d_origins, d_directions, R, M, d_num, d_cells, d_bary, d_dist, d_verts, dense, (cudaStream_t)stream);
}

extern "C" int tn_trace_rays_triangles(tn_tracer *h, const float *d_origins, const float *d_directions, uint32_t R, uint32_t M,
                                       uint32_t *d_num, uint32_t *d_faces, float *d_bary, float *d_dist, uint32_t *d_verts, void *stream) {
    return tn::launch_trace(h, 1, d_origins, d_directions, R, M, d_num, d_faces, d_bary, d_dist, d_verts, 1, (cudaStream_t)stream);
}
