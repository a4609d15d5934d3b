// tn_predicates.cuh -- the geometric certificates of a refit, shared by the load / refit checks (tn_faces.cu) and the fold guard of a
// vertex step (tn_fold_guard.cu), so the two certify every face and hull edge with the same bits.
#pragma once
#include "tn_common.cuh"

namespace tn {

// fold test of one interior face (a, b, c): orient3d(a, b, c, x) = det[a - x; b - x; c - x] in float64 on the fp32 positions, with every
// operation rounded individually (no FMA contraction, the op order of oracle/vertex_grads.py's restatement) and Shewchuk's forward error
// bound (7 + 56 eps) eps * permanent, eps = 2^-53: a sign the bound cannot certify counts as folded, so rounding can only turn the walk off.
__device__ __forceinline__ bool orient3d_sign(const float *__restrict__ xyz, uint32_t ia, uint32_t ib, uint32_t ic, uint32_t ix, int &sign) {
    auto P = [&](uint32_t v, int a) { return (double)__ldg(xyz + 3 * (size_t)v + a); };
    const double adx = __dsub_rn(P(ia, 0), P(ix, 0)), ady = __dsub_rn(P(ia, 1), P(ix, 1)), adz = __dsub_rn(P(ia, 2), P(ix, 2));
    const double bdx = __dsub_rn(P(ib, 0), P(ix, 0)), bdy = __dsub_rn(P(ib, 1), P(ix, 1)), bdz = __dsub_rn(P(ib, 2), P(ix, 2));
    const double cdx = __dsub_rn(P(ic, 0), P(ix, 0)), cdy = __dsub_rn(P(ic, 1), P(ix, 1)), cdz = __dsub_rn(P(ic, 2), P(ix, 2));
    const double bdxcdy = __dmul_rn(bdx, cdy), cdxbdy = __dmul_rn(cdx, bdy);
    const double cdxady = __dmul_rn(cdx, ady), adxcdy = __dmul_rn(adx, cdy);
    const double adxbdy = __dmul_rn(adx, bdy), bdxady = __dmul_rn(bdx, ady);
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(adz, __dsub_rn(bdxcdy, cdxbdy)), __dmul_rn(bdz, __dsub_rn(cdxady, adxcdy))),
                                 __dmul_rn(cdz, __dsub_rn(adxbdy, bdxady)));
    const double perm = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(fabs(bdxcdy), fabs(cdxbdy)), fabs(adz)),
                                            __dmul_rn(__dadd_rn(fabs(cdxady), fabs(adxcdy)), fabs(bdz))),
                                  __dmul_rn(__dadd_rn(fabs(adxbdy), fabs(bdxady)), fabs(cdz)));
    const double eps = 1.1102230246251565e-16;  // 2^-53
    const double bound = __dmul_rn(__dmul_rn(__dadd_rn(7.0, __dmul_rn(56.0, eps)), eps), perm);
    sign = det > bound ? 1 : (-det > bound ? -1 : 0);
    return sign != 0;
}

// insphere(a, b, c, d, e): Shewchuk's insphere determinant in float64 on the fp32 positions, positive when e lies inside the sphere
// through a, b, c, d and orient3d(a, b, c, d) > 0 (the sign flips with that orientation).  Every operation rounded individually, in his
// order (oracle/flip.py restates it), with his forward error bound (16 + 224 eps) eps * permanent: a sign the bound cannot certify is 0.
__device__ __forceinline__ bool insphere_sign(const float *__restrict__ xyz, uint32_t ia, uint32_t ib, uint32_t ic, uint32_t id, uint32_t ie,
                                              int &sign) {
    auto P = [&](uint32_t v, int a) { return (double)__ldg(xyz + 3 * (size_t)v + a); };
    const double aex = __dsub_rn(P(ia, 0), P(ie, 0)), aey = __dsub_rn(P(ia, 1), P(ie, 1)), aez = __dsub_rn(P(ia, 2), P(ie, 2));
    const double bex = __dsub_rn(P(ib, 0), P(ie, 0)), bey = __dsub_rn(P(ib, 1), P(ie, 1)), bez = __dsub_rn(P(ib, 2), P(ie, 2));
    const double cex = __dsub_rn(P(ic, 0), P(ie, 0)), cey = __dsub_rn(P(ic, 1), P(ie, 1)), cez = __dsub_rn(P(ic, 2), P(ie, 2));
    const double dex = __dsub_rn(P(id, 0), P(ie, 0)), dey = __dsub_rn(P(id, 1), P(ie, 1)), dez = __dsub_rn(P(id, 2), P(ie, 2));
    const double aexbey = __dmul_rn(aex, bey), bexaey = __dmul_rn(bex, aey), ab = __dsub_rn(aexbey, bexaey);
    const double bexcey = __dmul_rn(bex, cey), cexbey = __dmul_rn(cex, bey), bc = __dsub_rn(bexcey, cexbey);
    const double cexdey = __dmul_rn(cex, dey), dexcey = __dmul_rn(dex, cey), cd = __dsub_rn(cexdey, dexcey);
    const double dexaey = __dmul_rn(dex, aey), aexdey = __dmul_rn(aex, dey), da = __dsub_rn(dexaey, aexdey);
    const double aexcey = __dmul_rn(aex, cey), cexaey = __dmul_rn(cex, aey), ac = __dsub_rn(aexcey, cexaey);
    const double bexdey = __dmul_rn(bex, dey), dexbey = __dmul_rn(dex, bey), bd = __dsub_rn(bexdey, dexbey);
    const double abc = __dadd_rn(__dsub_rn(__dmul_rn(aez, bc), __dmul_rn(bez, ac)), __dmul_rn(cez, ab));
    const double bcd = __dadd_rn(__dsub_rn(__dmul_rn(bez, cd), __dmul_rn(cez, bd)), __dmul_rn(dez, bc));
    const double cda = __dadd_rn(__dadd_rn(__dmul_rn(cez, da), __dmul_rn(dez, ac)), __dmul_rn(aez, cd));
    const double dab = __dadd_rn(__dadd_rn(__dmul_rn(dez, ab), __dmul_rn(aez, bd)), __dmul_rn(bez, da));
    auto lift = [](double x, double y, double z) { return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)); };
    const double alift = lift(aex, aey, aez), blift = lift(bex, bey, bez), clift = lift(cex, cey, cez), dlift = lift(dex, dey, dez);
    const double det = __dadd_rn(__dsub_rn(__dmul_rn(dlift, abc), __dmul_rn(clift, dab)), __dsub_rn(__dmul_rn(blift, cda), __dmul_rn(alift, bcd)));
    const double az = fabs(aez), bz = fabs(bez), cz = fabs(cez), dz = fabs(dez);
    const double ab_ = __dadd_rn(fabs(aexbey), fabs(bexaey)), bc_ = __dadd_rn(fabs(bexcey), fabs(cexbey));
    const double cd_ = __dadd_rn(fabs(cexdey), fabs(dexcey)), da_ = __dadd_rn(fabs(dexaey), fabs(aexdey));
    const double ac_ = __dadd_rn(fabs(aexcey), fabs(cexaey)), bd_ = __dadd_rn(fabs(bexdey), fabs(dexbey));
    auto t3 = [](double p, double x, double q, double y, double r, double z) {
        return __dadd_rn(__dadd_rn(__dmul_rn(p, x), __dmul_rn(q, y)), __dmul_rn(r, z));
    };
    const double perm = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(t3(cd_, bz, bd_, cz, bc_, dz), alift), __dmul_rn(t3(da_, cz, ac_, dz, cd_, az), blift)),
                                            __dmul_rn(t3(ab_, dz, bd_, az, da_, bz), clift)),
                                  __dmul_rn(t3(bc_, az, ac_, bz, ab_, cz), dlift));
    const double eps = 1.1102230246251565e-16;  // 2^-53
    const double bound = __dmul_rn(__dmul_rn(__dadd_rn(16.0, __dmul_rn(224.0, eps)), eps), perm);
    sign = det > bound ? 1 : (-det > bound ? -1 : 0);
    return sign != 0;
}

// the vertex of cell c that is not on face f
__device__ __forceinline__ uint32_t opposite_vertex(const uint4 c, const uint4 f) {
    const uint32_t cv[4] = {c.x, c.y, c.z, c.w};
    uint32_t o = cv[0];
    for (int q = 0; q < 4; ++q)
        if (cv[q] != f.x && cv[q] != f.y && cv[q] != f.z) o = cv[q];
    return o;
}

// interior face (a, b, c) with opposite vertices p, q: certified unfolded iff both signs are certified and opposite
__device__ __forceinline__ bool face_unfolded(const float *__restrict__ xyz, uint32_t a, uint32_t b, uint32_t c, uint32_t p, uint32_t q) {
    int sp = 0, sq = 0;
    const bool cp = orient3d_sign(xyz, a, b, c, p, sp);
    const bool cq = orient3d_sign(xyz, a, b, c, q, sq);
    return cp && cq && sp == -sq;
}

// hull convexity across one hull edge: no vertex of hull face g lies above the plane of hull face f, the plane's outward side being away
// from the 4th vertex of f's tetrahedron (`inner`, which the test therefore reads too).  float64 on the fp32 positions, every operation
// rounded individually in this order (oracle/fold_guard.py restates it), with a relative tolerance of 1e-9.
__device__ __forceinline__ bool hull_pair_ok(const float *__restrict__ xyz, const uint4 *__restrict__ cells, const uint4 *__restrict__ tri,
                                             const uint2 *__restrict__ tt, uint32_t f, uint32_t g) {
    const uint4 ft = tri[f], gt = tri[g];
    const uint32_t inner = opposite_vertex(cells[tt[f].x], ft);
    const uint32_t fv[3] = {ft.x, ft.y, ft.z}, gv[3] = {gt.x, gt.y, gt.z};
    auto P = [&](uint32_t v, int a) { return (double)xyz[3 * (size_t)v + a]; };
    double e1[3], e2[3], n[3];
    for (int a = 0; a < 3; ++a) { e1[a] = __dsub_rn(P(fv[1], a), P(fv[0], a)); e2[a] = __dsub_rn(P(fv[2], a), P(fv[0], a)); }
    n[0] = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
    n[1] = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
    n[2] = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
    double si = 0, nn = 0;
    for (int a = 0; a < 3; ++a) {
        si = __dadd_rn(si, __dmul_rn(n[a], __dsub_rn(P(inner, a), P(fv[0], a))));
        nn = __dadd_rn(nn, __dmul_rn(n[a], n[a]));
    }
    if (si > 0) for (int a = 0; a < 3; ++a) n[a] = -n[a];
    for (int k = 0; k < 3; ++k) {
        double sd = 0, dd = 0;
        for (int a = 0; a < 3; ++a) {
            const double d = __dsub_rn(P(gv[k], a), P(fv[0], a));
            sd = __dadd_rn(sd, __dmul_rn(n[a], d));
            dd = __dadd_rn(dd, __dmul_rn(d, d));
        }
        if (sd > __dadd_rn(__dmul_rn(1e-9, __dsqrt_rn(__dmul_rn(nn, dd))), 1e-30)) return false;  // a vertex of g lies outside
    }
    return true;
}

}  // namespace tn
