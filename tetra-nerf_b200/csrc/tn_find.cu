// tn_find.cu -- find_tetrahedra: point location by two closest-hit rays (+x / -x).
// Replaces src/optix/optix_find_tetrahedra.cu:84-213 (+ FindTetrahedraPipeline, tetrahedra_tracer.cpp:589-853).
// One thread per query point, depth-first walk of the 8-ary BVH with t-max shrinking; the closest hit
// is the smallest (t, face id) key, as in oracle/tetra_oracle.cpp:orc_find_tetrahedra.
#include "tn_common.cuh"

namespace tn {
typedef unsigned long long u64;

struct FindParams {
    const float *pos;
    uint32_t N;
    uint32_t *tet;
    float *bary;
    uint32_t *verts;
    const float4 *nodes;
    const LeafRec *leaves;
    const uint4 *tri;
    const uint2 *tt;
    BvhLevels lv;
    float absmax;
};

__device__ bool closest_hit(const FindParams &p, float ox, float oy, float oz, float dx, uint32_t &face, float &t, float &u, float &v) {
    const RaySetup rs = ray_setup(ox, oy, oz, dx, 0.f, 0.f);
    const float ix = __fdiv_rn(1.0f, dx), iy = __fdiv_rn(1.0f, 0.0f), iz = iy;
    const float pad = 4e-6f * (fmaxf(fabsf(ox), fmaxf(fabsf(oy), fabsf(oz))) + p.absmax);
    uint32_t stack[7 * TN_MAX_LEVELS + 8];
    int sp = 0;
    stack[sp++] = (uint32_t)(p.lv.nlevels - 1) << 28;
    u64 best = ~0ull;
    float bu = 0.f, bv = 0.f;
    while (sp) {
        const uint32_t e = stack[--sp];
        const uint32_t cl = (e >> 28) - 1u, cbase = (e & 0x0FFFFFFFu) << TN_FAN_LOG2;
        const uint32_t nc = min(TN_FAN, p.lv.count[cl] - cbase);
        for (uint32_t c = 0; c < nc; ++c) {
            const float4 *np = p.nodes + 2 * (size_t)(p.lv.offset[cl] + cbase + c);
            if (!slab(__ldg(np), __ldg(np + 1), ox, oy, oz, ix, iy, iz, pad)) continue;
            if (cl != 0) { stack[sp++] = (cl << 28) | (cbase + c); continue; }
            const float4 *lp = reinterpret_cast<const float4 *>(p.leaves + cbase + c);
            const float4 v0 = __ldg(lp), v1 = __ldg(lp + 1), v2 = __ldg(lp + 2), v3 = __ldg(lp + 3);
            const Sheared s0 = shear(rs, v0.x, v0.y, v0.z), s1 = shear(rs, v1.x, v1.y, v1.z);
            const Sheared s2 = shear(rs, v2.x, v2.y, v2.z), s3 = shear(rs, v3.x, v3.y, v3.z);
            const uint32_t f[4] = {__float_as_uint(v0.w), __float_as_uint(v1.w), __float_as_uint(v2.w), __float_as_uint(v3.w)};
            float tt_, uu, vv;
            u64 k;
            if ((f[0] >> 31) && tri_test(s1, s2, s3, tt_, uu, vv)) { k = ((u64)__float_as_uint(tt_) << 32) | (f[0] & TN_FACE_MASK); if (k < best) { best = k; bu = uu; bv = vv; } }
            if ((f[1] >> 31) && tri_test(s2, s3, s0, tt_, uu, vv)) { k = ((u64)__float_as_uint(tt_) << 32) | (f[1] & TN_FACE_MASK); if (k < best) { best = k; bu = uu; bv = vv; } }
            if ((f[2] >> 31) && tri_test(s3, s0, s1, tt_, uu, vv)) { k = ((u64)__float_as_uint(tt_) << 32) | (f[2] & TN_FACE_MASK); if (k < best) { best = k; bu = uu; bv = vv; } }
            if ((f[3] >> 31) && tri_test(s0, s1, s2, tt_, uu, vv)) { k = ((u64)__float_as_uint(tt_) << 32) | (f[3] & TN_FACE_MASK); if (k < best) { best = k; bu = uu; bv = vv; } }
        }
    }
    if (best == ~0ull) return false;
    face = (uint32_t)best; t = __uint_as_float((uint32_t)(best >> 32)); u = bu; v = bv;
    return true;
}

__global__ void k_find(const FindParams p) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    const float ox = p.pos[3 * (size_t)i], oy = p.pos[3 * (size_t)i + 1], oz = p.pos[3 * (size_t)i + 2];
    uint32_t f0 = 0, f1 = 0, cell = TN_EMPTY;
    float t0, u0, v0, t1, u1, v1;
    float c[3] = {0.f, 0.f, 0.f};
    uint4 vi = make_uint4(0, 0, 0, 0);
    const bool h0 = closest_hit(p, ox, oy, oz, 1.0f, f0, t0, u0, v0);
    const bool h1 = closest_hit(p, ox, oy, oz, -1.0f, f1, t1, u1, v1);
    if (h0 && h1 && common_tet(__ldg(p.tt + f0), __ldg(p.tt + f1), cell)) {
        const uint4 tr0 = __ldg(p.tri + f0), tr1 = __ldg(p.tri + f1);
        const float c0[3] = {__fsub_rn(__fsub_rn(1.0f, u0), v0), u0, v0};
        const float r2[3] = {__fsub_rn(__fsub_rn(1.0f, u1), v1), u1, v1};
        const uint32_t id1[3] = {tr0.x, tr0.y, tr0.z}, id2[3] = {tr1.x, tr1.y, tr1.z};
        float c1[3] = {0.f, 0.f, 0.f};  // NOTE: the reference leaves coords_out2 uninitialised here (optix_find_tetrahedra.cu:57); 0 is pinned
        uint32_t newv = 0;
        for (int a = 0; a < 3; ++a) {
            bool was = false;
            for (int q = 0; q < 3; ++q)
                if (!was && id1[q] == id2[a]) { c1[q] = r2[a]; was = true; }
            if (!was) newv = id2[a];
        }
        const float m = __fdiv_rn(t1, __fadd_rn(t0, t1));  // optix_find_tetrahedra.cu:175
        const float om = __fsub_rn(1.0f, m);
        for (int a = 0; a < 3; ++a) c[a] = __fadd_rn(__fmul_rn(c0[a], m), __fmul_rn(c1[a], om));
        vi = make_uint4(newv, tr0.x, tr0.y, tr0.z);
    } else {
        cell = TN_EMPTY;
    }
    p.tet[i] = cell;
    p.bary[3 * (size_t)i] = c[0]; p.bary[3 * (size_t)i + 1] = c[1]; p.bary[3 * (size_t)i + 2] = c[2];
    reinterpret_cast<uint4 *>(p.verts)[i] = vi;
}
}  // namespace tn

extern "C" int tn_find_tetrahedra(tn_tracer *h, const float *d_positions, uint32_t N, uint32_t *d_tet, float *d_bary, uint32_t *d_verts,
                                  void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (!h->mesh.nodes.p) return tn::fail(TN_ERR_STATE, "find_tetrahedra: no tetrahedra loaded");
    if (N == 0) return TN_OK;
    tn::DeviceGuard g(h->device);
    tn::FindParams p;
    p.pos = d_positions; p.N = N; p.tet = d_tet; p.bary = d_bary; p.verts = d_verts;
    p.nodes = h->mesh.nodes.p; p.leaves = h->mesh.leaves.p; p.tri = h->mesh.tri.p; p.tt = h->mesh.tt.p;
    p.lv = h->mesh.lv; p.absmax = h->mesh.absmax;
    tn::k_find<<<(N + 63) / 64, 64, 0, (cudaStream_t)stream>>>(p);
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}
