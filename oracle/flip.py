"""Oracle of one Delaunay flip pass (tn_flip_delaunay, DESIGN.md §4.19) -- TEST INFRASTRUCTURE ONLY.

A numpy restatement of the pass that matches the CUDA one bit for bit:
  * face table: face slot 4t + k is the face of cell t opposite its vertex k, keyed by its ascending vertex triple (a, b, c); the slots
    sorted by (a, b, c, slot).  A face with one slot is a hull face, with three or more an error.  An interior face's priority is the
    position of its first slot in that order (the smaller goes first); t0 is the owner of its first slot, t1 the other, d / e their
    vertices off the face;
  * predicates: `_orient3d` (oracle/vertex_grads.py, tn_predicates.cuh orient3d_sign) and `_insphere`, Shewchuk's insphere determinant in
    float64 on the fp32 positions with his bound (16 + 224 eps) eps * permanent; numpy rounds every operation on its own, in the order
    written, as the kernel does.  0 = not certified;
  * illegal: t0, t1 certified and insphere(t0 in cell order, e) certified with t0's sign (e strictly inside t0's circumsphere);
  * proposal: an illegal face whose d and e are certified on opposite sides of it (sigma = orient3d(a, b, c, e)) and whose orient3d(a,b,d,e),
    (b,c,d,e), (c,a,d,e) are certified.  None differs from sigma: a 2-3 flip to (a,b,d,e), (b,c,d,e), (c,a,d,e).  Exactly one, for edge
    (x, y) of (a,b), (b,c), (c,a) with z the third face vertex: a 3-2 flip when the faces (x,y,d) of t0 and (x,y,e) of t1 are both interior
    with the same other owner t2 (certified), and with the link p < q < r of {z, d, e}, orient3d(p,q,r,x) and (p,q,r,y) certified and
    opposite and orient3d(x,y,p,q), (x,y,q,r), (x,y,r,p) certified and equal (the segment x-y crosses the open triangle pqr); it gives
    (p,q,r,x), (p,q,r,y).  Neither kind proposes when one of its new interior faces ((a,d,e), (b,d,e), (c,d,e) / (p,q,r)) is already a
    face of the mesh, as it can be next to a flat cell.  A new cell is written with its last two entries swapped when its sign differs from the flip's lowest-slot cell's;
  * vote / accept / cap: every cell votes for the highest-priority proposal touching it; a proposal is accepted when all its cells voted
    for it; beyond max_flips the highest-priority accepted ones are kept;
  * apply: old slots s0 < s1 (< s2); the new cells go to s0, s1 and, for a 2-3 flip, T + its rank among the kept 2-3 flips; s2 of a 3-2
    flip is removed by a stable compaction.  sources[i] = the old slots cell i came from, ascending, padded with -1.

`check_flipped` is an independent validity check of any flipped mesh that looks only at the input and output meshes."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from .vertex_grads import _orient3d

FACES = ((1, 2, 3), (0, 2, 3), (0, 1, 3), (0, 1, 2))
EPS = 1.1102230246251565e-16  # 2^-53


def _insphere(pa, pb, pc, pd, pe):
    """Shewchuk's insphere(a, b, c, d, e) in float64 with his forward error bound -> sign (0 = not certified): +1 when e lies inside the
    sphere through a, b, c, d and orient3d(a, b, c, d) > 0 (the sign flips with that orientation)"""
    aex, aey, aez = pa[:, 0] - pe[:, 0], pa[:, 1] - pe[:, 1], pa[:, 2] - pe[:, 2]
    bex, bey, bez = pb[:, 0] - pe[:, 0], pb[:, 1] - pe[:, 1], pb[:, 2] - pe[:, 2]
    cex, cey, cez = pc[:, 0] - pe[:, 0], pc[:, 1] - pe[:, 1], pc[:, 2] - pe[:, 2]
    dex, dey, dez = pd[:, 0] - pe[:, 0], pd[:, 1] - pe[:, 1], pd[:, 2] - pe[:, 2]
    aexbey, bexaey = aex * bey, bex * aey
    ab = aexbey - bexaey
    bexcey, cexbey = bex * cey, cex * bey
    bc = bexcey - cexbey
    cexdey, dexcey = cex * dey, dex * cey
    cd = cexdey - dexcey
    dexaey, aexdey = dex * aey, aex * dey
    da = dexaey - aexdey
    aexcey, cexaey = aex * cey, cex * aey
    ac = aexcey - cexaey
    bexdey, dexbey = bex * dey, dex * bey
    bd = bexdey - dexbey
    abc = (aez * bc - bez * ac) + cez * ab
    bcd = (bez * cd - cez * bd) + dez * bc
    cda = (cez * da + dez * ac) + aez * cd
    dab = (dez * ab + aez * bd) + bez * da
    alift = (aex * aex + aey * aey) + aez * aez
    blift = (bex * bex + bey * bey) + bez * bez
    clift = (cex * cex + cey * cey) + cez * cez
    dlift = (dex * dex + dey * dey) + dez * dez
    det = (dlift * abc - clift * dab) + (blift * cda - alift * bcd)
    A = np.abs
    az, bz, cz, dz = A(aez), A(bez), A(cez), A(dez)
    ab_, ba_, bc_, cb_, cd_, dc_ = A(aexbey), A(bexaey), A(bexcey), A(cexbey), A(cexdey), A(dexcey)
    da_, ad_, ac_, ca_, bd_, db_ = A(dexaey), A(aexdey), A(aexcey), A(cexaey), A(bexdey), A(dexbey)
    perm = ((((((cd_ + dc_) * bz + (db_ + bd_) * cz) + (bc_ + cb_) * dz) * alift
              + (((da_ + ad_) * cz + (ac_ + ca_) * dz) + (cd_ + dc_) * az) * blift)
             + (((ab_ + ba_) * dz + (bd_ + db_) * az) + (da_ + ad_) * bz) * clift)
            + (((bc_ + cb_) * az + (ca_ + ac_) * bz) + (ab_ + ba_) * cz) * dlift)
    bound = ((16.0 + 224.0 * EPS) * EPS) * perm
    return np.where(det > bound, 1, np.where(-det > bound, -1, 0))


def _o3(X, a, b, c, d):
    return _orient3d(X[a], X[b], X[c], X[d])


def face_table(cells):
    """-> (F i64[4T,3] the sorted face triples, slot i64[4T] the face slot at each sorted position)"""
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    T = len(c)
    f = np.sort(np.stack([c[:, list(q)] for q in FACES], 1).reshape(-1, 3), 1)  # slot 4t + k: the face opposite vertex k
    slot = np.arange(4 * T)
    order = np.lexsort((slot, f[:, 2], f[:, 1], f[:, 0]))
    return f[order], slot[order]


def _runs(F):
    n = len(F)
    first = np.ones(n, bool)
    first[1:] = (F[1:] != F[:-1]).any(1)
    start = np.nonzero(first)[0]
    length = np.diff(np.append(start, n))
    return start, length


def proposals(xyz, cells) -> Dict[str, np.ndarray]:
    """every interior face and what it proposes: positions `p` (priority), t0, t1, t2 (-1 unless 3-2), kind (0 none, 2, 3), `illegal`,
    the new cells `new` i64[n, 3, 4] (already in their written order; the third row only for 2-3) and `ref` (the lowest-slot cell's
    sign).  Raises ValueError on a face with more than two owners."""
    X = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    F, slot = face_table(c)
    start, length = _runs(F)
    if (length > 2).any():
        raise ValueError("a face has more than two owners")
    p = start[length == 2]
    t0, t1 = slot[p] // 4, slot[p + 1] // 4
    d, e = c[t0, slot[p] % 4], c[t1, slot[p + 1] % 4]
    a, b, cc = F[p, 0], F[p, 1], F[p, 2]
    sign = _orient3d(X[c[:, 0]], X[c[:, 1]], X[c[:, 2]], X[c[:, 3]])
    s0, s1 = sign[t0], sign[t1]
    ins = _insphere(X[c[t0, 0]], X[c[t0, 1]], X[c[t0, 2]], X[c[t0, 3]], X[e])
    illegal = (s0 != 0) & (s1 != 0) & (ins != 0) & (ins == s0)
    sd, se = _o3(X, a, b, cc, d), _o3(X, a, b, cc, e)
    o = np.stack([_o3(X, a, b, d, e), _o3(X, b, cc, d, e), _o3(X, cc, a, d, e)], 1)
    cand = illegal & (sd != 0) & (se != 0) & (sd == -se) & (o != 0).all(1)
    nopp = (o != se[:, None]).sum(1)
    n = len(p)
    kind = np.zeros(n, np.int64)
    t2 = np.full(n, -1, np.int64)
    new = np.full((n, 3, 4), -1, np.int64)
    ref = s0.copy()
    F64 = (F[:, 0] << 42) | (F[:, 1] << 21) | F[:, 2]
    assert len(X) < (1 << 21)

    def exists(x, y, w):
        k = np.sort(np.stack([x, y, w], 1), 1)
        key = (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]
        return F64[np.minimum(np.searchsorted(F64, key), len(F64) - 1)] == key

    # 2-3: none of its new interior faces (a,d,e), (b,d,e), (c,d,e) is already a face of the mesh
    m = cand & (nopp == 0)
    m &= ~exists(a, d, e) & ~exists(b, d, e) & ~exists(cc, d, e)
    kind[m] = 2
    rows = [(a, b, d, e), (b, cc, d, e), (cc, a, d, e)]
    for j, r in enumerate(rows):
        new[:, j] = np.stack(r, 1)
        sw = m & (o[:, j] != ref)
        new[sw, j, 2], new[sw, j, 3] = new[sw, j, 3], new[sw, j, 2].copy()
    # 3-2

    def other_owner(x, y, w, t):
        k = np.sort(np.stack([x, y, w], 1), 1)
        q = np.searchsorted(F64, (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2])
        q = np.minimum(q, len(F64) - 1)
        found = F64[q] == ((k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2])
        two = found & (q + 1 < len(F64)) & (F64[np.minimum(q + 1, len(F64) - 1)] == F64[q])
        u, v = slot[q] // 4, slot[np.minimum(q + 1, len(F64) - 1)] // 4
        return np.where(two, np.where(u == t, v, u), -1)

    j = np.argmax(o != se[:, None], 1)
    x = np.choose(j, [a, b, cc])
    y = np.choose(j, [b, cc, a])
    z = np.choose(j, [cc, a, b])
    m3 = cand & (nopp == 1)
    ta, tb = other_owner(x, y, d, t0), other_owner(x, y, e, t1)
    m3 &= (ta >= 0) & (ta == tb)
    t2c = np.maximum(ta, 0)
    m3 &= sign[t2c] != 0
    lk = np.sort(np.stack([z, d, e], 1), 1)
    pp, qq, rr = lk[:, 0], lk[:, 1], lk[:, 2]
    oa, ob = _o3(X, pp, qq, rr, x), _o3(X, pp, qq, rr, y)
    l0, l1, l2 = _o3(X, x, y, pp, qq), _o3(X, x, y, qq, rr), _o3(X, x, y, rr, pp)
    m3 &= (oa != 0) & (ob != 0) & (oa == -ob) & (l0 != 0) & (l0 == l1) & (l1 == l2)
    m3 &= ~exists(pp, qq, rr)  # its new interior face is not already a face of the mesh
    kind[m3] = 3
    t2[m3] = ta[m3]
    lo = np.minimum(np.minimum(t0, t1), t2c)
    ref = np.where(m3, sign[lo], ref)
    for jj, (w, s) in enumerate(((x, oa), (y, ob))):
        rowv = np.stack([pp, qq, rr, w], 1)
        sw = s != ref
        rowv[sw, 2], rowv[sw, 3] = rowv[sw, 3], rowv[sw, 2].copy()
        new[m3, jj] = rowv[m3]
    return {"p": p, "t0": t0, "t1": t1, "t2": t2, "kind": kind, "illegal": illegal, "new": new, "ref": ref}


def flip_delaunay(xyz, cells, max_flips: Optional[int] = None) -> Dict[str, object]:
    """the outputs of tn_flip_delaunay as numpy arrays: cells i32[T', 4], sources i32[T', 3] (-1 = none), n_illegal, n_proposed, n_23,
    n_32, and `prop` (proposals()), `accepted_all` / `kept` (indices into prop's faces, ascending priority)"""
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    T = len(c)
    pr = proposals(xyz, c)
    idx = np.nonzero(pr["kind"] > 0)[0]
    owners = [np.stack([pr["t0"][i], pr["t1"][i]] + ([pr["t2"][i]] if pr["kind"][i] == 3 else [])) for i in idx]
    vote = np.full(T, np.iinfo(np.int64).max)
    for i, ow in zip(idx, owners):
        vote[ow] = np.minimum(vote[ow], pr["p"][i])
    acc = np.array([i for i, ow in zip(idx, owners) if (vote[ow] == pr["p"][i]).all()], np.int64)
    kept = acc if max_flips is None else acc[:max_flips]
    n_ext = T + int((pr["kind"][kept] == 2).sum())
    out = np.zeros((n_ext, 4), np.int64)
    out[:T] = c
    src = np.full((n_ext, 3), -1, np.int64)
    src[:T, 0] = np.arange(T)
    removed = np.zeros(n_ext, bool)
    r23 = 0
    for i in kept:
        s = np.sort(np.array([pr["t0"][i], pr["t1"][i]] + ([pr["t2"][i]] if pr["kind"][i] == 3 else [])))
        src_row = np.full(3, -1, np.int64)
        src_row[: len(s)] = s
        if pr["kind"][i] == 2:
            dst = [s[0], s[1], T + r23]
            r23 += 1
        else:
            dst = [s[0], s[1]]
            removed[s[2]] = True
        for j, t in enumerate(dst):
            out[t] = pr["new"][i, j]
            src[t] = src_row
    n23 = r23
    n32 = int(removed.sum())
    return {"cells": out[~removed].astype(np.int32), "sources": src[~removed].astype(np.int32), "n_illegal": int(pr["illegal"].sum()),
            "n_proposed": len(idx), "n_23": n23, "n_32": n32, "prop": pr, "accepted_all": acc, "kept": kept}


def _abs_det_sum(X, cells):
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    e = X[c[:, 1:]] - X[c[:, :1]]
    det = (e[:, 0, 0] * (e[:, 1, 1] * e[:, 2, 2] - e[:, 1, 2] * e[:, 2, 1]) - e[:, 0, 1] * (e[:, 1, 0] * e[:, 2, 2] - e[:, 1, 2] * e[:, 2, 0])
           + e[:, 0, 2] * (e[:, 1, 0] * e[:, 2, 1] - e[:, 1, 1] * e[:, 2, 0]))
    return float(np.abs(det).sum())


def _faces(c):
    return np.sort(np.concatenate([c[:, list(q)] for q in FACES], 0), 1)


def check_flipped(xyz, cells, new_cells) -> Dict[str, object]:
    """validity of a re-triangulation of the mesh (xyz, cells) over the same vertices, from the two meshes alone: no face has more than
    two owners; the hull faces are the same; the cells use the same vertex set; every output cell that is not an input cell has a certified
    non-zero orientation;
    the sum of |det| over the cells is unchanged to 1e-12 relative.  Raises AssertionError naming the first property that fails; -> the
    measured quantities"""
    X = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    n = np.asarray(new_cells).astype(np.int64).reshape(-1, 4)
    u1, k1 = np.unique(_faces(n), axis=0, return_counts=True)
    assert k1.max(initial=0) <= 2, "a face has more than two owners"
    u0, k0 = np.unique(_faces(c), axis=0, return_counts=True)
    assert np.array_equal(u0[k0 == 1], u1[k1 == 1]), "the hull faces changed"
    assert np.array_equal(np.unique(c), np.unique(n)), "the vertex set changed"
    s = _orient3d(X[n[:, 0]], X[n[:, 1]], X[n[:, 2]], X[n[:, 3]])
    old_rows = {tuple(r) for r in c.tolist()}
    new_cell = np.array([tuple(r) not in old_rows for r in n.tolist()], bool)
    assert (s[new_cell] != 0).all(), "a new cell's orientation is not certified"
    v0, v1 = _abs_det_sum(X, c), _abs_det_sum(X, n)
    assert abs(v1 - v0) <= 1e-12 * v0, f"sum |det| changed: {v0!r} -> {v1!r}"
    return {"hull_faces": int((k1 == 1).sum()), "cells": (len(c), len(n)), "new_cells": int(new_cell.sum()), "abs_det_sum": (v0, v1)}


def illegal_faces(xyz, cells) -> Dict[str, int]:
    """certified-illegal interior faces and, of them, the ones that propose a flip"""
    pr = proposals(xyz, cells)
    return {"illegal": int(pr["illegal"].sum()), "proposed": int((pr["kind"] > 0).sum())}
