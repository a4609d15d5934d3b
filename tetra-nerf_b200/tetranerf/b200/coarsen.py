"""Mesh coarsening by empty-space vertex removal (DESIGN §4.18).

`coarsen_vertices` runs one pass of tn_coarsen_vertices on the GPU: a non-hull vertex whose tetrahedra are all empty is collapsed into a
neighbour, the tetrahedra around the collapsed edge disappear and the others of its star take the neighbour in its slot.  Removed
vertices take nothing with them: `compact_vertices` keeps the surviving entries of a per-vertex tensor (positions, field, optimizer
moments) and `refine.migrate_cells` carries a per-tetrahedron tensor (occupancy) over, each cell keeping its parent's entry.  The model's
driver is TetrahedraNerf.coarsen."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from ..utils.extension import tetranerf_cpp_extension as ext

_lib = ext._lib


def coarsen_vertices(xyz: torch.Tensor, cells: torch.Tensor, empty: torch.Tensor, max_removed: int | None = None) -> Dict[str, object]:
    """one collapse pass on the mesh (xyz f32[V,3], cells i32[T,4]) with the per-tetrahedron mask `empty` bool / u8 [T], all on one
    CUDA device.  Every non-hull vertex whose tetrahedra are all empty proposes its nearest neighbour whose cones keep every orientation;
    a proposal is accepted when every tetrahedron of its star voted for it; at most max_removed vertices (the highest-priority ones:
    shortest edge first; None: no cap) are removed.  -> {"cells" i32[T', 4], "kept_vertex" i32[V'] (the old id of each new vertex,
    ascending), "parent_cell" i32[T'] (the old index of each new tetrahedron, ascending), "n_proposed", "n_removed" (= V - V'),
    "n_cells_removed" (= T - T')}.  Raises RuntimeError on a vertex index out of range.  Waits until the stream has reached it."""
    for x, n in ((xyz, "xyz"), (cells, "cells"), (empty, "empty")):
        ext._check_input(x, n)
    ext._require(xyz.dtype == torch.float32 and xyz.dim() == 2 and xyz.size(1) == 3, "xyz must be float32 [V,3]")
    ext._require(cells.dtype == torch.int32 and cells.dim() == 2 and cells.size(1) == 4, "cells must be int32 [T,4]")
    ext._require(empty.dim() == 1 and empty.numel() == cells.size(0), "empty must have one entry per tetrahedron")
    ext._require(xyz.device == cells.device == empty.device, "xyz, cells and empty must be on the same device")
    V, T, dev = xyz.size(0), cells.size(0), xyz.device
    mask = empty.to(torch.uint8).contiguous()
    cap = V if max_removed is None else int(max_removed)
    ext._require(cap >= 0, "max_removed must be >= 0")
    cells_out = torch.empty((max(T, 1), 4), dtype=torch.int32, device=dev)
    parent_cell = torch.empty((max(T, 1),), dtype=torch.int32, device=dev)
    kept_vertex = torch.empty((max(V, 1),), dtype=torch.int32, device=dev)
    counts = (C.c_uint32 * 3)()
    nbytes = C.c_size_t(0)
    s = ext._stream(dev)
    args = (dev.index, xyz.data_ptr(), V, cells.data_ptr(), T, mask.data_ptr(), min(cap, V), cells_out.data_ptr(), kept_vertex.data_ptr(),
            parent_cell.data_ptr(), counts)
    with torch.cuda.device(dev):
        ext._check(_lib.tn_coarsen_vertices(*args, None, C.byref(nbytes), s))
        workspace = torch.empty((max(int(nbytes.value), 1),), dtype=torch.uint8, device=dev)
        ext._check(_lib.tn_coarsen_vertices(*args, workspace.data_ptr(), C.byref(nbytes), s))
    n_prop, n_rem, n_cells = int(counts[0]), int(counts[1]), int(counts[2])
    return {"cells": cells_out[: T - n_cells], "kept_vertex": kept_vertex[: V - n_rem], "parent_cell": parent_cell[: T - n_cells],
            "n_proposed": n_prop, "n_removed": n_rem, "n_cells_removed": n_cells}


def compact_vertices(t: torch.Tensor, kept_vertex: torch.Tensor, dim: int) -> torch.Tensor:
    """per-vertex `t` on the coarsened mesh: the entries of the kept vertices along `dim`, in their order"""
    return t.index_select(dim, kept_vertex.to(t.device).long())
