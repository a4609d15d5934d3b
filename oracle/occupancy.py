"""Oracle of the occupancy field and of occupancy culling on the fused paths -- TEST INFRASTRUCTURE ONLY.

Definition (DESIGN.md §4.12).
  * occupancy(t) = max of sigma over 11 barycentric probes of tetrahedron t -- its 4 vertices, 6 edge midpoints and centroid --
    sigma = softplus(density head(mlp_base(interpolated field))), no GradientScaler.  An update is occ <- max(decay occ, probe max);
    decay = 0 recomputes.
  * culling: a sample matched to tetrahedron t with occ[t] < threshold gets sigma := 0 as a constant (no MLP, no gradient, weight 0).
    Unmatched samples keep sigma = MLP(0).  It applies to both passes, so the PDF sampler sees the culled coarse weights.

`render` / `render_train` are oracle.render / oracle.render_train with `occupancy=(occ f32[T], threshold)`; None gives their results
(they call them).  Both return aux["culled"]: the culled mask of the pass that gives rgb, in the ray order of the non-empty rays, and
`render` also aux["coarse_culled"]."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from . import oracle as orc

# the probes as weights of the cell's vertices 1..3 (vertex 0 gets the rest), in the order of tn_occupancy_update
PROBES = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5], [0.5, 0.5, 0], [0.5, 0, 0.5],
                   [0, 0.5, 0.5], [0.25, 0.25, 0.25]], dtype=np.float64)


def probe_sigmas(field, params: Dict[str, torch.Tensor], cells, dtype=torch.float64) -> torch.Tensor:
    """sigma at the 11 probes of every tetrahedron -> [T, 11], in `dtype`"""
    F = torch.as_tensor(np.asarray(field)).to(dtype).t()  # [V, C]
    c = torch.as_tensor(np.asarray(cells)).long()
    b = torch.as_tensor(PROBES, dtype=dtype)
    w = torch.cat([(1 - b.sum(-1))[:, None], b], -1)  # [11, 4]
    x = torch.einsum("pk,tkc->tpc", w, F[c])  # [T, 11, C]
    p = {k: v.detach().to(dtype) for k, v in params.items()}
    return orc.density_head(p, orc.mlp_base(p, x))[..., 0]


def occupancy(field, params: Dict[str, torch.Tensor], cells, decay: float = 0.0, previous=None) -> torch.Tensor:
    """the float64 occupancy update: max(decay * previous, probe max) (decay 0 or no previous: the probe max) -> [T]"""
    m = probe_sigmas(field, params, cells).amax(-1)
    if decay == 0.0 or previous is None:
        return m
    return torch.maximum(decay * torch.as_tensor(previous).to(m.dtype), m)


def culled_mask(matched, occupancy) -> torch.Tensor:
    """matched: find_visited_cells output; occupancy: (occ [T], threshold) -> bool [R', S]"""
    occ, thr = occupancy
    occ = torch.as_tensor(np.asarray(occ.cpu() if torch.is_tensor(occ) else occ), dtype=torch.float32)
    cell = torch.as_tensor(matched["cell_indices"]).long()
    hit = cell >= 0
    return hit & (occ[cell.clamp_min(0)] < float(thr))


def _cull_sigma(sig, culled):
    return torch.where(culled[..., None], torch.zeros_like(sig).detach(), sig)


class _Patch:
    """runs an oracle render with density_head replaced by one that zeroes the culled samples of each call in turn (the coarse pass,
    then the fine pass), so that the pipeline itself stays the oracle's own"""

    def __init__(self, masks):
        self.masks, self.calls = masks, 0

    def __enter__(self):
        self.orig = orc.density_head

        def head(p, x):
            sig = self.orig(p, x)
            m = self.masks(self.calls)
            self.calls += 1
            return _cull_sigma(sig, m) if m is not None else sig

        orc.density_head = head
        return self

    def __exit__(self, *a):
        orc.density_head = self.orig


def _with_matching(fn, occupancy):
    """runs fn() with orc.find_visited_cells recording each call's culled mask and density_head applying it"""
    if occupancy is None:
        return fn(), []
    masks = []
    orig_match = orc.find_visited_cells

    def match(*a, **k):
        tc = orig_match(*a, **k)
        masks.append(culled_mask(tc, occupancy))
        return tc

    orc.find_visited_cells = match
    try:
        with _Patch(lambda i: masks[i] if i < len(masks) else None):
            out = fn()
    finally:
        orc.find_visited_cells = orig_match
    return out, masks


def render(mesh, field, params, origins, directions, cfg, occupancy=None, fine_euclid=None, nthreads: int = 0):
    """oracle.render (eval mode) with culling; aux as there plus "culled" (and "coarse_culled" when a coarse pass ran)"""
    out, masks = _with_matching(lambda: orc.render(mesh, field, params, origins, directions, cfg, nthreads=nthreads, return_aux=True,
                                                   fine_euclid=fine_euclid), occupancy)
    if masks:
        out["aux"]["culled"] = masks[-1]
        if len(masks) == 2:
            out["aux"]["coarse_culled"] = masks[0]
    return out


def render_train(mesh, field, params, origins, directions, cfg, jitter_coarse=None, jitter_fine=None, use_gradient_scaling: bool = False,
                 occupancy=None, fine_euclid=None, nthreads: int = 0):
    """oracle.render_train with culling (differentiable; culled samples carry no gradient); aux as there plus "culled"."""
    out, masks = _with_matching(lambda: orc.render_train(mesh, field, params, origins, directions, cfg, jitter_coarse, jitter_fine,
                                                         use_gradient_scaling=use_gradient_scaling, nthreads=nthreads,
                                                         fine_euclid=fine_euclid), occupancy)
    if masks:
        out["aux"]["culled"] = masks[-1]
    return out
