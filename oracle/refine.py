"""Oracle of one longest-edge bisection pass (tn_refine_edges, DESIGN.md §4.14) -- TEST INFRASTRUCTURE ONLY.

A numpy restatement of the pass that matches the CUDA one bit for bit:
  * edge {a, b}: key (min << 32) | max; squared length ((xa-xb)^2 + (ya-yb)^2) + (za-zb)^2 in float64 from the fp32 coordinates, each
    operation rounded on its own (numpy float64 arithmetic is exactly that); priority: larger squared length, ties to the smaller key;
  * propose: each candidate's highest-priority edge, when its squared length >= float64(float32(min_length))^2; P = sorted distinct proposals;
  * vote: each tetrahedron with an edge in P votes for its highest-priority one; accept: every tetrahedron around the edge voted for it;
    beyond max_new_vertices keep the highest-priority accepted edges;
  * split: kept edges in ascending key order become V, V+1, ...; a tetrahedron around kept edge (a, b) keeps its slot with b -> m and
    appends a child at T + rank with a -> m.

Also the mesh properties the tests check: faces and their owners, hull area, signed volumes."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

EDGES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


def edge_table(xyz, cells):
    """-> keys u64[T,6], squared lengths f64[T,6] of every tetrahedron's six edges"""
    xyz = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cells).astype(np.int64)
    a = np.stack([c[:, i] for i, _ in EDGES], 1)
    b = np.stack([c[:, j] for _, j in EDGES], 1)
    lo, hi = np.minimum(a, b).astype(np.uint64), np.maximum(a, b).astype(np.uint64)
    keys = (lo << np.uint64(32)) | hi
    d = xyz[a] - xyz[b]
    len2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    return keys, len2


def _best(keys, len2, valid):
    """per row, the column of the highest-priority edge among `valid` ones (-1 if none)"""
    T = keys.shape[0]
    best = np.full(T, -1, dtype=np.int64)
    bl = np.full(T, -np.inf)
    bk = np.full(T, np.iinfo(np.uint64).max, dtype=np.uint64)
    for e in range(6):
        l, k, ok = len2[:, e], keys[:, e], valid[:, e]
        better = ok & ((best < 0) | (l > bl) | ((l == bl) & (k < bk)))
        best = np.where(better, e, best)
        bl = np.where(better, l, bl)
        bk = np.where(better, k, bk)
    return best


def refine_edges(xyz, cells, candidates, min_length: float = 0.0, max_new_vertices: Optional[int] = None) -> Dict[str, object]:
    """the outputs of tn_refine_edges as numpy arrays: cells i32[T + n_split, 4], parent_edge i32[n_new, 2], parent_cell i32[T + n_split],
    n_proposed, n_accepted (= n_new), n_split, and `accepted_all` (the keys accepted before the cap, ascending)"""
    cells = np.asarray(cells).astype(np.int64)
    T, V = len(cells), len(xyz)
    keys, len2 = edge_table(xyz, cells)
    cand = np.asarray(candidates).astype(bool)
    allv = np.ones((T, 6), dtype=bool)
    longest = _best(keys, len2, allv)
    rows = np.arange(T)
    ml = np.float64(np.float32(min_length))  # the C ABI takes it as a float
    min2 = ml * ml
    propose = cand & (len2[rows, longest] >= min2)
    P = np.unique(keys[rows[propose], longest[propose]])
    in_p = np.isin(keys, P)
    vote_col = _best(keys, len2, in_p)
    voters = vote_col >= 0
    incident = np.zeros(len(P), dtype=np.int64)
    np.add.at(incident, np.searchsorted(P, keys[in_p]), 1)
    votes = np.zeros(len(P), dtype=np.int64)
    voted_idx = np.full(T, -1, dtype=np.int64)
    voted_idx[voters] = np.searchsorted(P, keys[rows[voters], vote_col[voters]])
    np.add.at(votes, voted_idx[voters], 1)
    accepted = (votes == incident) & (incident > 0)
    acc_idx = np.nonzero(accepted)[0]
    if max_new_vertices is not None and len(acc_idx) > max_new_vertices:
        a, b = (P[acc_idx] >> np.uint64(32)).astype(np.int64), (P[acc_idx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        x = np.asarray(xyz, dtype=np.float32).astype(np.float64)
        d = x[a] - x[b]
        l2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        order = np.lexsort((P[acc_idx], -l2))  # descending length, then ascending key
        keep = np.zeros(len(P), dtype=bool)
        keep[acc_idx[order[:max_new_vertices]]] = True
    else:
        keep = accepted
    vid = np.cumsum(keep) - keep  # exclusive scan
    kept = P[keep]
    parent_edge = np.stack([(kept >> np.uint64(32)).astype(np.int64), (kept & np.uint64(0xFFFFFFFF)).astype(np.int64)], 1).reshape(-1, 2)
    split = voters.copy()
    split[voters] = keep[voted_idx[voters]]
    out = cells.copy()
    children, parents = [], []
    for t in np.nonzero(split)[0]:
        i = voted_idx[t]
        a, b, m = int(P[i] >> np.uint64(32)), int(P[i] & np.uint64(0xFFFFFFFF)), V + int(vid[i])
        child = cells[t].copy()
        out[t][out[t] == b] = m
        child[child == a] = m
        children.append(child)
        parents.append(t)
    new_cells = np.concatenate([out, np.asarray(children, dtype=np.int64).reshape(-1, 4)], 0)
    parent_cell = np.concatenate([np.arange(T), np.asarray(parents, dtype=np.int64)])
    return {"cells": new_cells.astype(np.int32), "parent_edge": parent_edge.astype(np.int32), "parent_cell": parent_cell.astype(np.int32),
            "n_proposed": int(len(P)), "n_accepted": int(keep.sum()), "n_split": int(split.sum()), "accepted_all": P[accepted]}


def migrate_vertices(x, parent_edge, axis: int = 0):
    """(x[a] + x[b]) * 0.5 appended along `axis`, in the dtype of x"""
    x = np.asarray(x)
    pe = np.asarray(parent_edge).astype(np.int64).reshape(-1, 2)
    new = (np.take(x, pe[:, 0], axis) + np.take(x, pe[:, 1], axis)) * x.dtype.type(0.5)
    return np.concatenate([x, new.astype(x.dtype)], axis)


def signed_volumes(xyz, cells):
    """float64 signed volume of every tetrahedron: det(x1-x0, x2-x0, x3-x0) / 6"""
    x = np.asarray(xyz, dtype=np.float64)[np.asarray(cells).astype(np.int64)]
    return np.linalg.det(x[:, 1:] - x[:, :1]) / 6.0


def face_owners(cells):
    """-> (sorted faces i64[F,3], owner counts i64[F])"""
    c = np.asarray(cells).astype(np.int64)
    faces = np.sort(np.concatenate([c[:, [1, 2, 3]], c[:, [0, 2, 3]], c[:, [0, 1, 3]], c[:, [0, 1, 2]]], 0), 1)
    return np.unique(faces, axis=0, return_counts=True)


def hull_area(xyz, cells):
    """float64 total area of the faces with a single owner"""
    faces, counts = face_owners(cells)
    f = faces[counts == 1]
    x = np.asarray(xyz, dtype=np.float64)
    return float(0.5 * np.linalg.norm(np.cross(x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]]), axis=1).sum())
