"""Restoring the Delaunay property of a mesh by flips (DESIGN §4.19).

`flip_delaunay` runs one pass of tn_flip_delaunay on the GPU: every interior face whose opposite vertex lies strictly inside the other
owner's circumsphere (certified in float64) and whose cells can be re-triangulated with certified orientations proposes a 2-3 or a 3-2
flip, and the flips that share no cell are applied.  The vertices do not move, so every per-vertex tensor (positions, field, optimizer
moments) stays as it is; `migrate_cells_max` carries a per-tetrahedron tensor (occupancy) over as the maximum over each new cell's
sources.  The model's driver is TetrahedraNerf.flip_delaunay."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from ..utils.extension import tetranerf_cpp_extension as ext

_lib = ext._lib


def flip_delaunay(xyz: torch.Tensor, cells: torch.Tensor, max_flips: int | None = None) -> Dict[str, object]:
    """one flip pass on the mesh (xyz f32[V,3], cells i32[T,4]), both on one CUDA device; at most max_flips flips (the highest-priority
    ones; None: no cap).  -> {"cells" i32[T', 4], "sources" i32[T', 3] (the old tetrahedra each new one's region came from, ascending,
    padded with -1), "n_illegal" (interior faces certified non-Delaunay), "n_proposed", "n_23", "n_32" (flips applied; T' = T + n_23 -
    n_32)}.  Raises RuntimeError on a vertex index out of range or a face with more than two owners.  Waits until the stream has reached
    it."""
    for x, n in ((xyz, "xyz"), (cells, "cells")):
        ext._check_input(x, n)
    ext._require(xyz.dtype == torch.float32 and xyz.dim() == 2 and xyz.size(1) == 3, "xyz must be float32 [V,3]")
    ext._require(cells.dtype == torch.int32 and cells.dim() == 2 and cells.size(1) == 4, "cells must be int32 [T,4]")
    ext._require(xyz.device == cells.device, "xyz and cells must be on the same device")
    V, T, dev = xyz.size(0), cells.size(0), xyz.device
    cap = 0xFFFFFFFF if max_flips is None else int(max_flips)
    ext._require(0 <= cap <= 0xFFFFFFFF, "max_flips must be >= 0")
    n_out = max(T + T // 2, 1)
    cells_out = torch.empty((n_out, 4), dtype=torch.int32, device=dev)
    sources = torch.empty((n_out, 3), dtype=torch.int32, device=dev)
    counts = (C.c_uint32 * 4)()
    nbytes = C.c_size_t(0)
    s = ext._stream(dev)
    args = (dev.index, xyz.data_ptr(), V, cells.data_ptr(), T, cap, cells_out.data_ptr(), sources.data_ptr(), counts)
    with torch.cuda.device(dev):
        ext._check(_lib.tn_flip_delaunay(*args, None, C.byref(nbytes), s))
        workspace = torch.empty((max(int(nbytes.value), 1),), dtype=torch.uint8, device=dev)
        ext._check(_lib.tn_flip_delaunay(*args, workspace.data_ptr(), C.byref(nbytes), s))
    n_illegal, n_prop, n23, n32 = (int(counts[i]) for i in range(4))
    T1 = T + n23 - n32
    if T1 < n_out:  # own storage of the result's size, so a kept or saved result does not hold the T + T/2 capacity
        cells_out, sources = cells_out[:T1].clone(), sources[:T1].clone()
    return {"cells": cells_out, "sources": sources, "n_illegal": n_illegal, "n_proposed": n_prop, "n_23": n23, "n_32": n32}


def migrate_cells_max(t: torch.Tensor, sources: torch.Tensor) -> torch.Tensor:
    """per-tetrahedron `t` [T, ...] on the flipped cells: each new cell's entry is the maximum over its sources (i32[T', 3], -1 = none;
    the first always set), so a value like occupancy never drops where a flip moved a cell's region"""
    src = sources.to(t.device).long()
    first = t.index_select(0, src[:, 0])
    out = first
    for j in (1, 2):
        s = src[:, j]
        v = t.index_select(0, s.clamp_min(0))
        keep = (s >= 0).view(-1, *([1] * (t.dim() - 1)))
        out = torch.where(keep, torch.maximum(out, v), out)
    return out
