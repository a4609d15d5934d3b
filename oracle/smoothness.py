"""Oracle of the field smoothness loss (tn_field_smoothness, DESIGN.md §4.15) -- TEST INFRASTRUCTURE ONLY.

In float64 numpy, straight from the definition: over the unique undirected edges {i, j} (i < j) of the mesh, two distinct vertices of one
cell, with E their number and C the number of features,
    S = sum_{i,j} sum_c (f[c,i] - f[c,j])^2,   loss = mult * S / (E * C),
    d loss / d f[c,i] = mult * 2 / (E * C) * sum_{j in N(i)} (f[c,i] - f[c,j])."""
from __future__ import annotations

import numpy as np

PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


def edges(cells) -> np.ndarray:
    """the unique undirected edges of the cells -> int64[E,2], each row (i, j) with i < j, rows ascending"""
    c = np.asarray(cells).astype(np.int64).reshape(-1, 4)
    a = np.concatenate([c[:, i] for i, _ in PAIRS])
    b = np.concatenate([c[:, j] for _, j in PAIRS])
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    keep = lo != hi
    n = int(c.max()) + 1 if c.size else 1
    key = np.unique(lo[keep] * n + hi[keep])  # sorted pairs as one integer each
    return np.stack([key // n, key % n], 1)


def smoothness(field, cells):
    """-> (S, E) for field [C,V]"""
    f = np.asarray(field, dtype=np.float64)
    e = edges(cells)
    S = 0.0
    for c in range(f.shape[0]):  # one feature at a time: the [C,E] differences of a 2 M-tetrahedra mesh would take 1.2 GB
        d = f[c, e[:, 0]] - f[c, e[:, 1]]
        S += float(np.dot(d, d))
    return S, len(e)


def loss(field, cells, mult: float = 1.0) -> float:
    S, E = smoothness(field, cells)
    C = np.asarray(field).shape[0]
    return mult * S / (E * C) if E else 0.0


def _per_vertex(field, cells, fn):
    """[C,V]: sum over the neighbours j of i of fn(f[c,i] - f[c,j]) -> (it, edges)"""
    f = np.asarray(field, dtype=np.float64)
    e = edges(cells)
    C, V = f.shape
    out = np.zeros((C, V))
    for c in range(C):
        d = f[c, e[:, 0]] - f[c, e[:, 1]]
        out[c] = np.bincount(e[:, 0], weights=fn(d), minlength=V) + np.bincount(e[:, 1], weights=fn(-d), minlength=V)
    return out, e


def gradient(field, cells, mult: float = 1.0) -> np.ndarray:
    """d loss / d field, float64 [C,V]"""
    g, e = _per_vertex(field, cells, lambda d: d)
    return g * (mult * 2.0 / (len(e) * g.shape[0])) if len(e) else g


def neighbour_abs_sum(field, cells) -> tuple:
    """-> (sum_{j in N(i)} |f[c,i] - f[c,j]| float64 [C,V], degree int64[V]): what the per-element error bound of an fp32 evaluation
    of the gradient is made of"""
    a, e = _per_vertex(field, cells, np.abs)
    return a, np.bincount(e.ravel(), minlength=a.shape[1])
