"""Oracle of the fold guard of a vertex step (tn_guard_vertex_step, tn_fold_guard.cu; DESIGN.md §4.17) -- TEST INFRASTRUCTURE ONLY.

Definition.  P0 f32[V,3] are the positions at the last load or refit, P1 f32[V,3] the proposed ones.  A vertex is moving if its P1 row
differs bitwise from its P0 row.  The guarded items are fixed at P0:
  * every interior face the refit's fold test certifies unfolded at P0 (vertex_grads.fold_count's predicate), with its five vertices;
  * if the mesh is walkable at P0 -- its hull is closed and every hull edge passes the convexity test at P0 (`hull_pair_ok` both ways, the
    load's test) and no interior face is uncertified -- every hull edge, with the six vertices the test reads: the two faces' four and
    the fourth vertex of each face's tetrahedron.
Every moving vertex starts at k = 0 (P1).  Round r = 0, 1, ... tests every guarded item at the current positions; the moving, not frozen
vertices of a failing item get k = r + 1 while r < K, and are frozen (back at P0) from round K on; the rounds stop when nothing fails.
A vertex at 1 <= k <= K sits at P0 + (P1 - P0) * 2^-k, each operation rounded to fp32 in that order.  The CUDA rounds retest only the
items with a vertex that changed in the round before; an item whose vertices did not change passed its last test (a failing item moves a
vertex, unless all its moving vertices are frozen, and then it is at P0 and passes), so testing every item every round, as here, gives
the same result.

`hull_pair_ok` restates tn_predicates.cuh's hull convexity test with the same operations in the same order, each rounded to float64, so
its decisions equal the kernel's."""
from __future__ import annotations

from typing import Dict

import numpy as np

from .vertex_grads import _orient3d, face_tables

FROZEN = -2  # exponent of a vertex moved back to P0 (non-moving vertices: -1)


def _opposite(cells, tri, t):
    cv = cells[t]
    out = cv[:, 0].copy()
    for q in range(4):
        other = (cv[:, q] != tri[:, 0]) & (cv[:, q] != tri[:, 1]) & (cv[:, q] != tri[:, 2])
        out = np.where(other, cv[:, q], out)
    return out


def hull_pairs(tri, tt):
    """the hull edges as the load sorts them: hull faces in face order, their edges (v[k], v[k+1]) keyed by the sorted vertex pair, stably
    sorted -> (f [n], g [n]) the two hull faces of each edge, closed: whether every hull edge has exactly two hull faces"""
    tri, tt = np.asarray(tri, np.int64), np.asarray(tt, np.int64)
    hf = np.nonzero(tt[:, 1] < 0)[0]
    if len(hf) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), False
    a = np.stack([tri[hf, k] for k in range(3)], 1).reshape(-1)
    b = np.stack([tri[hf, (k + 1) % 3] for k in range(3)], 1).reshape(-1)
    key = np.minimum(a, b) * (1 << 32) + np.maximum(a, b)
    face = np.repeat(hf, 3)
    order = np.argsort(key, kind="stable")
    key, face = key[order], face[order]
    _, counts = np.unique(key, return_counts=True)
    closed = bool(np.all(counts == 2))
    if not closed:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), False
    return face[0::2], face[1::2], True


def hull_pair_ok(X, cells, tri, tt, f, g):
    """tn_predicates.cuh hull_pair_ok for arrays of face pairs: no vertex of hull face g above the outward plane of hull face f, in float64
    on the float32 positions X, every operation rounded in the kernel's order -> bool [n]"""
    X = np.asarray(X, np.float32).astype(np.float64)
    c, tri, tt = np.asarray(cells, np.int64), np.asarray(tri, np.int64), np.asarray(tt, np.int64)
    ft, gt = tri[f], tri[g]
    inner = _opposite(c, ft, tt[f, 0])
    F0 = X[ft[:, 0]]
    e1, e2 = X[ft[:, 1]] - F0, X[ft[:, 2]] - F0
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    di = X[inner] - F0
    si = np.zeros(len(f))
    nn = np.zeros(len(f))
    for a in range(3):
        si = si + n[:, a] * di[:, a]
        nn = nn + n[:, a] * n[:, a]
    n = np.where((si > 0)[:, None], -n, n)
    ok = np.ones(len(f), bool)
    for k in range(3):
        d = X[gt[:, k]] - F0
        sd = np.zeros(len(f))
        dd = np.zeros(len(f))
        for a in range(3):
            sd = sd + n[:, a] * d[:, a]
            dd = dd + d[:, a] * d[:, a]
        ok &= ~(sd > 1e-9 * np.sqrt(nn * dd) + 1e-30)
    return ok


def _items(cells, tri, tt):
    """interior faces (a, b, c, p, q) [n,5] and hull edges (f, g, closed)"""
    c, tri, tt = np.asarray(cells, np.int64), np.asarray(tri, np.int64), np.asarray(tt, np.int64)
    inner = tt[:, 1] >= 0
    ti, tti = tri[inner], tt[inner]
    faces = np.concatenate([ti, _opposite(c, ti, tti[:, 0])[:, None], _opposite(c, ti, tti[:, 1])[:, None]], 1)
    return faces, hull_pairs(tri, tt)


def _faces_ok(X, faces):
    A, B, Cc = X[faces[:, 0]], X[faces[:, 1]], X[faces[:, 2]]
    sp, sq = _orient3d(A, B, Cc, X[faces[:, 3]]), _orient3d(A, B, Cc, X[faces[:, 4]])
    return (sp != 0) & (sq != 0) & (sp == -sq)


def _hull_ok(X, cells, tri, tt, f, g):
    return hull_pair_ok(X, cells, tri, tt, f, g) & hull_pair_ok(X, cells, tri, tt, g, f)


def _hull_vertices(cells, tri, tt, f, g):
    c, tri, tt = np.asarray(cells, np.int64), np.asarray(tri, np.int64), np.asarray(tt, np.int64)
    return np.concatenate([tri[f], tri[g], _opposite(c, tri[f], tt[f, 0])[:, None], _opposite(c, tri[g], tt[g, 0])[:, None]], 1)


def step_position(p0, p1, k):
    """P0 + (P1 - P0) * 2^-k in float32, each operation rounded in this order; k >= 1"""
    p0, p1 = np.asarray(p0, np.float32), np.asarray(p1, np.float32)
    return p0 + (p1 - p0) * np.float32(2.0 ** -k)


def guard(p0, p1, cells, max_halvings: int, tri=None, tt=None) -> Dict[str, object]:
    """the guarded positions of the move p0 -> p1 (both f32[V,3]) on the mesh `cells` -> {"xyz" f32[V,3], "k" i64[V] (-1 not moving, 0..K,
    FROZEN), "limited", "frozen", "rounds", "folded_p0" (interior faces uncertified at P0), "hull_guarded" (walkable at P0)}"""
    K = int(max_halvings)
    P0 = np.ascontiguousarray(p0, np.float32)
    P1 = np.ascontiguousarray(p1, np.float32)
    if tri is None:
        tri, tt = face_tables(cells)
    faces, (hf, hg, closed) = _items(cells, tri, tt)
    X0 = P0.astype(np.float64)
    ok0 = _faces_ok(X0, faces)
    faces = faces[ok0]
    folded_p0 = int(np.sum(~ok0))
    hull_guarded = closed and len(hf) > 0 and folded_p0 == 0 and bool(np.all(_hull_ok(P0, cells, tri, tt, hf, hg)))
    if not hull_guarded:
        hf, hg = hf[:0], hg[:0]
    hv = _hull_vertices(cells, tri, tt, hf, hg)
    moving = np.any(P0.view(np.uint32) != P1.view(np.uint32), axis=1)
    k = np.where(moving, 0, -1).astype(np.int64)
    X = P1.copy()
    r = 0
    while True:
        Xd = X.astype(np.float64)
        bad_f = ~_faces_ok(Xd, faces)
        bad_h = ~_hull_ok(X, cells, tri, tt, hf, hg) if len(hf) else np.zeros(0, bool)
        mark = np.zeros(len(X), bool)
        mark[faces[bad_f].reshape(-1)] = True
        mark[hv[bad_h].reshape(-1)] = True
        mark &= moving & (k != FROZEN)
        rounds = r + 1
        if not (bad_f.any() or bad_h.any()):
            break
        assert mark.any(), "a failing item with no vertex left to move back"
        if r < K:
            k[mark] = r + 1
            X[mark] = step_position(P0[mark], P1[mark], r + 1)
        else:
            k[mark] = FROZEN
            X[mark] = P0[mark]
        r += 1
    return {"xyz": X, "k": k, "limited": int(np.sum((k >= 1) & (k <= K))), "frozen": int(np.sum(k == FROZEN)), "rounds": rounds,
            "folded_p0": folded_p0, "hull_guarded": hull_guarded}
