"""Second, independent float64 restatement of the expected depth and its gradient -- TEST INFRASTRUCTURE ONLY.

oracle/expected_depth.py writes DepthRenderer(method="expected") in torch and lets autograd differentiate it.  This module computes the
same quantities from the definition in DESIGN.md §4.10 with plain per-ray loops in Python floats, in the style of second_opinion.py, and
never imports torch or oracle.py:
  * w_i = (1 - exp(-delta_i sigma_i)) * prod_{k<i} exp(-delta_k sigma_k), A = sum_i w_i, t_i = the bin midpoints;
  * D_raw = sum_i w_i t_i / (A + 1e-10); D = min(max(D_raw, t_min), t_max) with t_min / t_max over every sample of every active ray;
    empty rays: far_plane;
  * dD/dw_i = (t_i - D_raw) / (A + 1e-10) where t_min <= D_raw <= t_max, else 0; then, x_j = delta_j sigma_j,
    dD/dx_j = dD/dw_j exp(-x_j) prod_{k<j} exp(-x_k) - sum_{i>j} dD/dw_i w_i, and dD/dsigma_j = delta_j dD/dx_j.
tests/test_expected_depth_cpu.py holds the two against each other."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

EPS = 1e-10


def _weights(deltas: Sequence[float], sigmas: Sequence[float]) -> List[float]:
    w, trans = [], 1.0
    for dl, s in zip(deltas, sigmas):
        x = dl * s
        w.append((1.0 - math.exp(-x)) * trans)
        trans *= math.exp(-x)
    return w


def expected_depth(edges: Sequence[Optional[Sequence[float]]], sigmas: Sequence[Optional[Sequence[float]]], far_plane: float,
                   grad_out: Optional[Sequence[float]] = None, midpoints: Optional[Sequence[Optional[Sequence[float]]]] = None
                   ) -> Tuple[List[float], List[Optional[List[float]]]]:
    """per ray: bin edges (None for an empty ray) and densities; grad_out[r] = dL/dD_r.  midpoints: the t_i per ray when the caller
    forms them itself (float32 midpoints of float32 edges, as the renderers do); else (e_i + e_{i+1}) / 2 here.
    -> (D per ray, dL/dsigma per ray (None for empty rays))"""
    steps = []
    for r, e in enumerate(edges):
        if e is None:
            steps.append(None)
        elif midpoints is not None:
            steps.append([float(t) for t in midpoints[r]])
        else:
            steps.append([(float(e[i]) + float(e[i + 1])) / 2.0 for i in range(len(e) - 1)])
    lo = min(t for s in steps if s is not None for t in s)
    hi = max(t for s in steps if s is not None for t in s)
    depth, grads = [], []
    for r, e in enumerate(edges):
        if e is None:
            depth.append(far_plane)
            grads.append(None)
            continue
        deltas = [float(e[i + 1]) - float(e[i]) for i in range(len(e) - 1)]
        sg = [float(s) for s in sigmas[r]]
        w = _weights(deltas, sg)
        a = 0.0
        num = 0.0
        for wi, ti in zip(w, steps[r]):
            a += wi
            num += wi * ti
        d_raw = num / (a + EPS)
        depth.append(min(max(d_raw, lo), hi))
        g = 0.0 if grad_out is None else float(grad_out[r])
        inside = lo <= d_raw <= hi
        dw = [g * (ti - d_raw) / (a + EPS) if inside else 0.0 for ti in steps[r]]
        gs = []
        for j in range(len(w)):
            trans = 1.0
            for k in range(j):
                trans *= math.exp(-deltas[k] * sg[k])
            dx = dw[j] * math.exp(-deltas[j] * sg[j]) * trans
            for i in range(j + 1, len(w)):
                dx -= dw[i] * w[i]
            gs.append(deltas[j] * dx)
        grads.append(gs)
    return depth, grads
