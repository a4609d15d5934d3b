"""Oracle of the fused training step with differentiable mesh vertices, and of the fold test of a refit -- TEST INFRASTRUCTURE ONLY.

`render_train_geometry` is `ray_grads.render_train_rays` with one more differentiable input: the vertex positions `xyz`, a torch tensor
that may require grad.  Definition (DESIGN.md §4.9), in the convention of §4.8: the sample distances are constants (coarse bins, PDF
bins, the trace's t_in / t_out detached) and so is the tetrahedron each fine sample was matched to.  The matched weights
b = E^-1 (x_i - x_v0) then depend on the sample position AND on the four vertices; they go through the reference's add_barycentrics_grad,
whose vertex half (grad_vertices = -b_full (x) E^-T q, tetranerf/utils/extension/__init__.py) routes to `xyz` because the tetrahedra's
corners are gathered from it.  exact_bary=True recomputes b from the positions in the working dtype instead (plain autograd), a function
of (o, d, xyz) for finite differences, with `matched` and `fine_euclid` from an earlier call holding the tetrahedra and bins fixed.  The
trace itself always runs on `mesh` (the positions it was built with).

`fold_count` restates the fold test of tn_update_vertices (tn_faces.cu k_fold_faces) in numpy: the same operations in the same order,
each rounded to float64 (numpy does not contract to FMA), and the same error bound, so its count equals the kernel's."""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from . import oracle as orc
from . import ray_grads as rg


def tet_edges(vertex_indices, xyz, dtype):
    """ray_grads.tet_edges with `xyz` either float32 positions or a torch tensor (gathered from, so that gradients reach it)"""
    vi = torch.as_tensor(vertex_indices).long()
    if isinstance(xyz, torch.Tensor):
        X = xyz.to(dtype).reshape(-1, 3)
    else:
        X = torch.as_tensor(np.asarray(xyz, dtype=np.float32)).to(dtype).reshape(-1, 3)
    verts = X[vi.clamp_min(0)]
    E = verts[..., 1:, :] - verts[..., :1, :]
    good = (vi[..., 0] >= 0) & (torch.linalg.det(E.detach()) != 0)
    unit = torch.cat([torch.zeros((1, 3), dtype=dtype), torch.eye(3, dtype=dtype)])
    return torch.where(good[..., None, None], verts, unit), good


def differentiable_bary(vertex_indices, bary, xyz, points, exact: bool = False):
    """ray_grads.differentiable_bary with differentiable vertex positions (`xyz` a torch tensor)"""
    from tetranerf.utils.extension import add_barycentrics_grad

    b = torch.as_tensor(bary).to(points.dtype)
    verts, good = tet_edges(vertex_indices, xyz, points.dtype)
    if exact:
        E = (verts[..., 1:, :] - verts[..., :1, :]).transpose(-1, -2)
        bx = torch.linalg.solve(E, points - verts[..., 0, :])
    else:
        bx = add_barycentrics_grad(b, verts, points)
    return torch.where(good[..., None], bx, b)


def render_train_geometry(mesh: "orc.OracleMesh", field: torch.Tensor, params: Dict[str, torch.Tensor], origins: torch.Tensor,
                          directions: torch.Tensor, xyz, cfg: "orc.RenderConfig", jitter_coarse=None, jitter_fine=None,
                          use_gradient_scaling: bool = False, nthreads: int = 0, fine_euclid=None, matched=None, exact_bary: bool = False):
    """ray_grads.render_train_rays with the matched weights a function of the vertex positions `xyz` [V,3] (a torch tensor that may require
    grad) as well: the same stages in the same order, only the weights are gathered from `xyz`; the same outputs (the CPU tests compare
    the two renders)"""
    o = origins.reshape(-1, 3)
    d = directions.reshape(-1, 3)
    R = o.shape[0]
    assert cfg.num_fine_samples > 0
    tr = mesh.trace_rays(o.detach().float().numpy(), d.detach().float().numpy(), cfg.max_intersected_triangles, nthreads=nthreads)
    num_visited = torch.from_numpy(tr["num_visited_cells"])
    hd = torch.from_numpy(tr["hit_distances"])
    nears = hd[:, 0, 0][:, None]
    fars = torch.gather(hd[:, :, 1], 1, (num_visited[:, None].long() - 1).clamp_min(0))
    ray_mask = num_visited > 0
    m = ray_mask.numpy()
    nears_r, fars_r = nears[ray_mask], fars[ray_mask]
    trm = {k: v[m] for k, v in tr.items()}
    jc = torch.as_tensor(jitter_coarse)[ray_mask] if jitter_coarse is not None else None
    jf = torch.as_tensor(jitter_fine)[ray_mask] if jitter_fine is not None else None

    def match(euclid_bins):
        dist = ((euclid_bins[:, 1:] + euclid_bins[:, :-1]) / 2).contiguous()
        return orc.find_visited_cells(trm["num_visited_cells"], trm["visited_cells"], trm["barycentric_coordinates"], trm["hit_distances"],
                                      trm["vertex_indices"], dist.detach().numpy(), nthreads=nthreads)

    if fine_euclid is not None:
        euclid = torch.as_tensor(fine_euclid, dtype=torch.float32)
        sbins = (euclid - nears_r) / (fars_r - nears_r)
    else:
        with torch.no_grad():  # the coarse pass only feeds the (detached) PDF bins
            euclid, sbins = orc.coarse_bins(cfg, nears_r, fars_r, num_visited[ray_mask], hd[ray_mask], jc)
            tc = match(euclid)
            fv = orc.interpolate_torch(tc["vertex_indices"], tc["barycentric_coordinates"], field.detach())
            density_coarse = orc.density_head(params, orc.mlp_base(params, fv))
            weights = orc.get_weights((euclid[:, 1:] - euclid[:, :-1])[..., None], density_coarse)
            euclid, sbins = orc.pdf_bins(cfg, sbins, weights, nears_r, fars_r, u_rand=jf)
    tc = match(euclid) if matched is None else matched
    t = ((euclid[:, 1:] + euclid[:, :-1]) / 2).detach().to(o.dtype)
    idx = torch.nonzero(ray_mask).flatten()
    pos = o[idx][:, None, :] + t[..., None] * d[idx][:, None, :]
    bary = differentiable_bary(tc["vertex_indices"], tc["barycentric_coordinates"], xyz, pos, exact=exact_bary).to(field.dtype)
    fv = rg.interpolate_with_weights(tc["vertex_indices"], bary, field)
    for x in (pos, fv):
        if x.requires_grad:
            x.retain_grad()
    base = orc.mlp_base(params, fv)
    sigmas = orc.density_head(params, base)
    enc = orc.nerf_encoding_dirs(d[idx].to(base.dtype))[:, None, :].expand(-1, base.shape[1], -1)
    colors = orc.color_head(params, base, enc)
    if use_gradient_scaling:
        ray_dist = (sbins[:, 1:] + sbins[:, :-1])[..., None]
        colors, sigmas, _ = orc._GradientScaler.apply(colors, sigmas, ray_dist)
    deltas = (euclid[:, 1:] - euclid[:, :-1])[..., None]
    weights = orc.get_weights(deltas, sigmas)
    comp = torch.sum(weights * colors, dim=-2)
    accum = torch.sum(weights, dim=-2)
    bg = torch.tensor(cfg.background, dtype=comp.dtype)
    rgb_r = comp + bg * (1.0 - accum)
    steps = (euclid[:, 1:] + euclid[:, :-1]) / 2
    cumw = torch.cumsum(weights[..., 0].detach(), dim=-1)
    mi = torch.clamp(torch.searchsorted(cumw, torch.ones((weights.shape[0], 1)) * 0.5, side="left"), 0, steps.shape[-1] - 1)
    depth_r = torch.gather(steps, dim=-1, index=mi)
    rgb = bg.expand(R, 3).clone().index_copy(0, idx, rgb_r)
    acc = torch.zeros((R, 1), dtype=rgb_r.dtype).index_copy(0, idx, accum)
    depth = torch.full((R, 1), cfg.far_plane, dtype=depth_r.dtype).index_copy(0, idx, depth_r)
    return {"rgb": rgb, "accumulation": acc, "depth": depth, "ray_mask": ray_mask,
            "aux": {"fine_euclid": euclid.detach(), "sigmas": sigmas.detach(), "colors": colors.detach(), "weights": weights.detach(), "matched": tc,
                    "positions": pos, "features": fv}}


def scatter_vertex_grads(vertex_indices, bary, m, V):
    """float64 restatement of the kernel's scatter: dL/dx_vj += -b_j m_i with b = (1 - b1 - b2 - b3, b1, b2, b3) in float32 as the
    kernel forms b_0; vertex_indices [N,4] (-1 = unmatched), bary [N,3] float32, m [N,3] (the per-sample dL/dx) -> [V,3] float64"""
    vi = np.asarray(vertex_indices, dtype=np.int64).reshape(-1, 4)
    b = np.asarray(bary, dtype=np.float32).reshape(-1, 3)
    b0 = np.float32(1.0) - ((b[:, 0] + b[:, 1]) + b[:, 2])
    w = np.concatenate([b0[:, None], b], 1).astype(np.float64)
    m = np.asarray(m, dtype=np.float64).reshape(-1, 3)
    ok = vi[:, 0] >= 0
    out = np.zeros((V, 3), np.float64)
    for k in range(4):
        np.add.at(out, vi[ok, k], -w[ok, k:k + 1] * m[ok])
    return out


def face_tables(cells):
    """the unique faces in the reference's numbering (src/tetrahedra_tracer.cpp:45-71): slot 4 t + j is the face opposite local vertex j in
    the rotation (c[j+1], c[j+2], c[j+3]); a face's id and stored winding come from its first slot -> (tri [F,3], tt [F,2], -1 = none)"""
    c = np.asarray(cells, dtype=np.int64)
    T = len(c)
    rot = np.stack([c[:, [(j + 1) % 4, (j + 2) % 4, (j + 3) % 4]] for j in range(4)], 1).reshape(-1, 3)  # slot order
    key = np.sort(rot, 1)
    _, first, inv = np.unique(key, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(first, kind="stable")  # face ids by first appearance
    fid = np.empty_like(order)
    fid[order] = np.arange(len(order))
    slot_face = fid[inv]
    F = len(order)
    head = first[order]  # first slot of each face, by face id
    tri = rot[head]
    tt = np.full((F, 2), -1, np.int64)
    tt[:, 0] = head // 4
    slots = np.arange(4 * T)
    second = slots[slots != head[slot_face]]
    tt[slot_face[second], 1] = second // 4
    return tri, tt


def _orient3d(a, b, c, d):
    """float64 orient3d det[a - d; b - d; c - d] and Shewchuk's bound, the op order of tn_faces.cu orient3d_sign -> sign (0 = uncertified)"""
    adx, ady, adz = a[:, 0] - d[:, 0], a[:, 1] - d[:, 1], a[:, 2] - d[:, 2]
    bdx, bdy, bdz = b[:, 0] - d[:, 0], b[:, 1] - d[:, 1], b[:, 2] - d[:, 2]
    cdx, cdy, cdz = c[:, 0] - d[:, 0], c[:, 1] - d[:, 1], c[:, 2] - d[:, 2]
    bdxcdy, cdxbdy = bdx * cdy, cdx * bdy
    cdxady, adxcdy = cdx * ady, adx * cdy
    adxbdy, bdxady = adx * bdy, bdx * ady
    det = (adz * (bdxcdy - cdxbdy) + bdz * (cdxady - adxcdy)) + cdz * (adxbdy - bdxady)
    perm = ((np.abs(bdxcdy) + np.abs(cdxbdy)) * np.abs(adz) + (np.abs(cdxady) + np.abs(adxcdy)) * np.abs(bdz)) \
        + (np.abs(adxbdy) + np.abs(bdxady)) * np.abs(cdz)
    eps = 1.1102230246251565e-16  # 2^-53
    bound = ((7.0 + 56.0 * eps) * eps) * perm
    return np.where(det > bound, 1, np.where(-det > bound, -1, 0))


def fold_count(xyz, cells, tri=None, tt=None, return_faces: bool = False):
    """number of interior faces whose two opposite vertices are not certified to lie strictly on opposite sides of the face's plane, at
    the float32 positions `xyz` [V,3]; tri / tt: the tracer's face tables (face_tables(cells) when omitted); return_faces: the vertex
    triples [n,3] of those faces instead"""
    if tri is None:
        tri, tt = face_tables(cells)
    X = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cells, dtype=np.int64)
    tri, tt = np.asarray(tri, dtype=np.int64), np.asarray(tt, dtype=np.int64)
    inner = tt[:, 1] >= 0
    tri, tt = tri[inner], tt[inner]

    def opposite(t):
        cv = c[t]
        out = cv[:, 0].copy()
        for q in range(4):
            other = (cv[:, q] != tri[:, 0]) & (cv[:, q] != tri[:, 1]) & (cv[:, q] != tri[:, 2])
            out = np.where(other, cv[:, q], out)
        return out

    A, B, Cc = X[tri[:, 0]], X[tri[:, 1]], X[tri[:, 2]]
    sp = _orient3d(A, B, Cc, X[opposite(tt[:, 0])])
    sq = _orient3d(A, B, Cc, X[opposite(tt[:, 1])])
    folded = ~((sp != 0) & (sq != 0) & (sp == -sq))
    return tri[folded] if return_faces else int(np.sum(folded))
