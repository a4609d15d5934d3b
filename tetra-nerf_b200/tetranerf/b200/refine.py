"""Mesh refinement by longest-edge bisection (DESIGN §4.14).

`refine_edges` runs one pass of tn_refine_edges on the GPU.  A new vertex m on edge (a, b) takes the value (x_a + x_b) * 0.5 of every
per-vertex tensor (an fp32 add, then a multiply), and each tetrahedron around the edge is split in two halves that interpolate exactly
the linear function of their parent, so the field is unchanged by a pass.  `migrate_vertices` / `migrate_cells` carry per-vertex and
per-tetrahedron tensors (positions, field, optimizer moments, occupancy) over to the refined mesh.  `select_candidates` is the model's
choice of the tetrahedra to refine (TetrahedraNerf.refine)."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from ..utils.extension import tetranerf_cpp_extension as ext

_lib = ext._lib
MAX_VERTICES = 0xFFFFFFFF  # vertex ids are uint32


def refine_edges(xyz: torch.Tensor, cells: torch.Tensor, candidates: torch.Tensor, min_length: float = 0.0,
                 max_new_vertices: int | None = None) -> Dict[str, object]:
    """one bisection pass on the mesh (xyz f32[V,3], cells i32[T,4]) with candidate mask `candidates` bool / u8 [T], all on one CUDA
    device.  Every candidate whose longest edge is at least min_length long proposes it; an edge is split when every tetrahedron around
    it voted for it; at most max_new_vertices edges (the highest-priority ones; None: no cap) are split.  -> {"cells" i32[T + n_split, 4],
    "parent_edge" i32[n_new, 2] (a < b: the edge of vertex V + i), "parent_cell" i32[T + n_split] (the identity on the first T, the split
    parent after), "n_proposed", "n_accepted" (= n_new), "n_split"}.  Raises RuntimeError on a vertex index out of range or an overflow
    of the uint32 vertex ids.  Waits until the stream has reached it."""
    for x, n in ((xyz, "xyz"), (cells, "cells"), (candidates, "candidates")):
        ext._check_input(x, n)
    ext._require(xyz.dtype == torch.float32 and xyz.dim() == 2 and xyz.size(1) == 3, "xyz must be float32 [V,3]")
    ext._require(cells.dtype == torch.int32 and cells.dim() == 2 and cells.size(1) == 4, "cells must be int32 [T,4]")
    ext._require(candidates.dim() == 1 and candidates.numel() == cells.size(0), "candidates must have one entry per tetrahedron")
    ext._require(xyz.device == cells.device == candidates.device, "xyz, cells and candidates must be on the same device")
    V, T, dev = xyz.size(0), cells.size(0), xyz.device
    cand = candidates.to(torch.uint8).contiguous()
    max_new = MAX_VERTICES - V if max_new_vertices is None else int(max_new_vertices)
    ext._require(max_new >= 0, "max_new_vertices must be >= 0")
    cells_out = torch.empty((2 * T, 4), dtype=torch.int32, device=dev)
    parent_cell = torch.empty((2 * T,), dtype=torch.int32, device=dev)
    parent_edge = torch.empty((max(min(T, max_new), 1), 2), dtype=torch.int32, device=dev)
    counts = (C.c_uint32 * 3)()
    nbytes = C.c_size_t(0)
    s = ext._stream(dev)
    args = (dev.index, xyz.data_ptr(), V, cells.data_ptr(), T, cand.data_ptr(), float(min_length), max_new & 0xFFFFFFFF, cells_out.data_ptr(),
            parent_edge.data_ptr(), parent_cell.data_ptr(), counts)
    with torch.cuda.device(dev):
        ext._check(_lib.tn_refine_edges(*args, None, C.byref(nbytes), s))
        workspace = torch.empty((max(int(nbytes.value), 1),), dtype=torch.uint8, device=dev)
        ext._check(_lib.tn_refine_edges(*args, workspace.data_ptr(), C.byref(nbytes), s))
    n_prop, n_new, n_split = int(counts[0]), int(counts[1]), int(counts[2])
    return {"cells": cells_out[: T + n_split], "parent_edge": parent_edge[:n_new], "parent_cell": parent_cell[: T + n_split],
            "n_proposed": n_prop, "n_accepted": n_new, "n_split": n_split}


def migrate_vertices(t: torch.Tensor, parent_edge: torch.Tensor, dim: int) -> torch.Tensor:
    """`t` with one entry per new vertex appended along `dim`: (t[a] + t[b]) * 0.5 for its parent edge (a, b), rounded as the fp32 add
    and multiply it is (so a linear field stays exactly linear on the split tetrahedra up to that one rounding)"""
    if parent_edge.numel() == 0:
        return t
    pe = parent_edge.to(t.device).long()
    new = (t.index_select(dim, pe[:, 0]) + t.index_select(dim, pe[:, 1])) * 0.5
    return torch.cat((t, new.to(t.dtype)), dim)


def migrate_cells(t: torch.Tensor, parent_cell: torch.Tensor) -> torch.Tensor:
    """per-tetrahedron `t` [T, ...] on the refined mesh: each tetrahedron holds its parent's entry (children copy their parent)"""
    return t.index_select(0, parent_cell.to(t.device).long())


def select_candidates(vertex_score: torch.Tensor, cells: torch.Tensor, fraction: float) -> torch.Tensor:
    """the model's refinement candidates: a tetrahedron scores the mean of its four vertices' scores (((s0 + s1) + s2) + s3) * 0.25; the floor(fraction * T)
    highest-scoring tetrahedra with a score > 0 are candidates, ties going to the smaller index.  -> bool [T]"""
    T = cells.size(0)
    k = min(T, max(0, int(fraction * T)))
    mask = torch.zeros((T,), dtype=torch.bool, device=cells.device)
    if k == 0:
        return mask
    sc = vertex_score[cells.long()]
    score = (((sc[:, 0] + sc[:, 1]) + sc[:, 2]) + sc[:, 3]) * 0.25
    _, order = torch.sort(score, descending=True, stable=True)
    top = order[:k]
    mask[top[score[top] > 0]] = True
    return mask
