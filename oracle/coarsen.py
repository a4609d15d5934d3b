"""Oracle of one empty-space vertex-removal pass (tn_coarsen_vertices, DESIGN.md §4.18) -- TEST INFRASTRUCTURE ONLY.

A numpy restatement of the pass that matches the CUDA one bit for bit:
  * star of a vertex: the cells that hold it, in ascending cell order; hull faces: the faces with one owner, as exact vertex triples;
  * candidates: a vertex with a non-empty star of empty cells, no hull face through it and every star cell's orient3d sign certified
    (`_orient3d`, the float64 restatement of tn_predicates.cuh orient3d_sign);
  * target: the neighbours b in ascending (squared length, id), the squared length ((xa-xb)^2 + (ya-yb)^2) + (za-zb)^2 in float64 from the
    fp32 coordinates (numpy float64 arithmetic rounds each operation on its own); the first b for which every star cell without b, with b
    in a's slot, keeps its certified sign.  Priority: the smaller squared length, ties to the smaller a;
  * vote / accept / cap: every cell votes for its highest-priority proposing vertex; accepted when the whole star voted for it; beyond
    max_removed the highest-priority accepted vertices are kept;
  * apply: star cells holding b go, the others take b in a's slot; stable compaction of cells and vertices.

`check_coarsened` is an independent validity check of any coarsened mesh that looks only at the input and output meshes."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from .vertex_grads import _orient3d

FACES = ((1, 2, 3), (0, 2, 3), (0, 1, 3), (0, 1, 2))


def _len2(X, a, b):
    d = X[a] - X[b]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def cell_signs(X, cells):
    """certified orient3d sign (0 = not certified) of every cell (v0, v1, v2, v3), X the float64 image of the fp32 positions"""
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    return _orient3d(X[c[:, 0]], X[c[:, 1]], X[c[:, 2]], X[c[:, 3]])


def hull_faces(cells):
    """the faces with a single owner, as ascending vertex triples i64[F,3], in lexicographic order"""
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    f = np.sort(np.concatenate([c[:, list(q)] for q in FACES], 0), 1)
    u, n = np.unique(f, axis=0, return_counts=True)
    return u[n == 1]


def stars(cells, V):
    """vertex -> cells CSR: (offsets i64[V+1], cells of each vertex ascending i64[4T])"""
    flat = np.asarray(cells).astype(np.int64).reshape(-1)
    order = np.argsort(flat, kind="stable")
    off = np.searchsorted(flat[order], np.arange(V + 1))
    return off, order // 4


def proposals(xyz, cells, empty):
    """-> (target i64[V], -1 for no proposal; squared length f64[V] of the proposed edge)"""
    X = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    V = len(X)
    empty = np.asarray(empty).astype(bool)
    off, star = stars(c, V)
    deg = np.diff(off)
    sign = cell_signs(X, c)
    bad = np.zeros(V, bool)  # a non-empty or uncertified cell in the star
    np.logical_or.at(bad, c[~empty | (sign == 0)].reshape(-1), True)
    hull = np.zeros(V, bool)
    hull[hull_faces(c).reshape(-1)] = True
    target = np.full(V, -1, dtype=np.int64)
    prio = np.zeros(V)
    for a in np.nonzero((deg > 0) & ~bad & ~hull)[0]:
        sc = star[off[a]:off[a + 1]]
        cs = c[sc]
        nb = np.unique(cs[cs != a])
        ln = _len2(X, np.full(len(nb), a), nb)
        for j in np.lexsort((nb, ln)):
            b = nb[j]
            keep = ~(cs == b).any(1)
            moved = np.where(cs[keep] == a, b, cs[keep])
            if np.array_equal(cell_signs(X, moved), sign[sc[keep]]):
                target[a], prio[a] = b, ln[j]
                break
    return target, prio


def coarsen_vertices(xyz, cells, empty, max_removed: Optional[int] = None) -> Dict[str, object]:
    """the outputs of tn_coarsen_vertices as numpy arrays: cells i32[T', 4], kept_vertex i32[V'], parent_cell i32[T'], n_proposed,
    n_removed, n_cells_removed, and `target` i64[V] (every proposal, -1 for none), `accepted_all` (the vertices accepted before the
    cap, ascending) and `removed` (the kept ones, ascending)"""
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    T, V = len(c), len(xyz)
    target, prio = proposals(xyz, c, empty)
    prop = target >= 0
    # vote: each cell for its highest-priority proposing vertex (the smaller squared length, then the smaller id)
    best = np.full(T, -1, dtype=np.int64)
    bl = np.full(T, np.inf)
    for q in range(4):
        v = c[:, q]
        ok = prop[v]
        better = ok & ((best < 0) | (prio[v] < bl) | ((prio[v] == bl) & (v < best)))
        best = np.where(better, v, best)
        bl = np.where(better, prio[v], bl)
    votes = np.bincount(best[best >= 0], minlength=V)
    deg = np.bincount(c.reshape(-1), minlength=V)
    accepted = prop & (votes == deg)
    acc = np.nonzero(accepted)[0]
    keep = accepted.copy()
    if max_removed is not None and len(acc) > max_removed:
        order = np.lexsort((acc, prio[acc]))  # ascending length, then ascending id
        keep[:] = False
        keep[acc[order[:max_removed]]] = True
    # apply: at most one removed vertex per cell
    rem = keep[c]
    has = rem.any(1)
    a = np.where(has, c[np.arange(T), rem.argmax(1)], -1)
    b = np.where(has, target[np.maximum(a, 0)], -1)
    gone = has & (c == b[:, None]).any(1)
    moved = np.where(has[:, None] & (c == a[:, None]), b[:, None], c)
    keepv = ~keep
    newid = np.cumsum(keepv) - keepv
    out = newid[moved[~gone]]
    return {"cells": out.astype(np.int32).reshape(-1, 4), "kept_vertex": np.nonzero(keepv)[0].astype(np.int32),
            "parent_cell": np.nonzero(~gone)[0].astype(np.int32), "n_proposed": int(prop.sum()), "n_removed": int(keep.sum()),
            "n_cells_removed": int(gone.sum()), "target": target, "accepted_all": acc, "removed": np.nonzero(keep)[0]}


def _abs_det_sum(X, cells):
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    e = X[c[:, 1:]] - X[c[:, :1]]
    det = (e[:, 0, 0] * (e[:, 1, 1] * e[:, 2, 2] - e[:, 1, 2] * e[:, 2, 1]) - e[:, 0, 1] * (e[:, 1, 0] * e[:, 2, 2] - e[:, 1, 2] * e[:, 2, 0])
           + e[:, 0, 2] * (e[:, 1, 0] * e[:, 2, 1] - e[:, 1, 1] * e[:, 2, 0]))
    return float(np.abs(det).sum())


def check_coarsened(xyz, cells, new_cells, kept_vertex, parent_cell) -> Dict[str, object]:
    """validity of a coarsened mesh from the input mesh (xyz, cells) and the output (new_cells over the vertices kept_vertex, each cell
    with its parent): no face has more than two owners; the hull faces, mapped to the input's ids, are the input's; every output cell has
    its parent's orient3d sign, certified wherever the cell changed; the sum of |det| over the cells is unchanged to 1e-12 relative.
    Raises AssertionError naming the first property that fails; -> the measured quantities"""
    X = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    kv = np.asarray(kept_vertex).astype(np.int64)
    n = kv[np.asarray(new_cells).astype(np.int64).reshape(-1, 4)]  # the output cells in the input's vertex ids
    pc = np.asarray(parent_cell).astype(np.int64)
    f = np.sort(np.concatenate([n[:, list(q)] for q in FACES], 0), 1)
    _, owners = np.unique(f, axis=0, return_counts=True)
    assert owners.max(initial=0) <= 2, "a face has more than two owners"
    h0, h1 = hull_faces(c), hull_faces(n)
    assert np.array_equal(h0, h1), "the hull faces changed"
    s_old, s_new = cell_signs(X, c)[pc], cell_signs(X, n)
    changed = (n != c[pc]).any(1)
    assert np.array_equal(s_new, s_old), "a cell's orientation differs from its parent's"
    assert (s_new[changed] != 0).all(), "a changed cell's orientation is not certified"
    v0, v1 = _abs_det_sum(X, c), _abs_det_sum(X, n)
    assert abs(v1 - v0) <= 1e-12 * v0, f"sum |det| changed: {v0!r} -> {v1!r}"
    return {"hull_faces": len(h0), "changed_cells": int(changed.sum()), "abs_det_sum": (v0, v1)}
