"""Oracle of the fused training step with differentiable rays -- TEST INFRASTRUCTURE ONLY.

`render_train_rays` is `oracle.render_train` with `origins` / `directions` kept as torch tensors that may require grad (the same outputs
up to rounding: the direction encoding's argument is formed in the rays' dtype).  Definition (DESIGN.md §4.8): the sample distances are constants (the coarse bins, the PDF bins and the trace's t_in /
t_out are detached), and a fine sample i sits at x_i = o + t_i d, t_i the midpoint of its bin (the distance the matcher uses).  It is
matched to the tetrahedron (v0, v1, v2, v3) with weights (b1, b2, b3); the feature is the tetrahedron's affine function
f(x) = F_v0 + sum_k b_k(x) (F_vk - F_v0), b(x) = E^-1 (x - x_v0), E = [x_v1 - x_v0 | x_v2 - x_v0 | x_v3 - x_v0].  Its value is the tracer's
interpolated feature; only its derivative is new:
  * the matched weights go through the reference's add_barycentrics_grad (identity forward, E^-T backward to the points), and
  * the interpolation differentiates its weights (interpolate_torch detaches them).
The direction also enters through the direction encoding of the colour head.  Unmatched samples and det E = 0 carry no ray gradient.

exact_bary=True instead recomputes b = E^-1 (x - x_v0) from the positions in the working dtype (plain autograd, no add_barycentrics_grad):
a function of (o, d) for finite differences, with `matched` (the aux["matched"] of an earlier call) holding the tetrahedra fixed."""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from . import oracle as orc


def interpolate_with_weights(vertex_indices, bary, field):
    """interpolate_torch with the weights differentiable: the same formula (so the same values), d f / d b_k = F_vk - F_v0"""
    vi = torch.as_tensor(vertex_indices).long()
    w = bary
    ok = (vi >= 0).to(field.dtype)
    F = field.t()
    safe = vi.clamp_min(0)
    w0 = 1.0 - w.sum(-1)
    return (w[..., 0:1] * ok[..., 1:2]) * F[safe[..., 1]] + (w[..., 1:2] * ok[..., 2:3]) * F[safe[..., 2]] + (w[..., 2:3] * ok[..., 3:4]) * F[safe[..., 3]] \
        + (w0[..., None] * ok[..., 0:1]) * F[safe[..., 0]]


def tet_edges(vertex_indices, xyz, dtype):
    """vertex positions [...,4,3] of the matched tetrahedra (float32 positions, exact in `dtype`), a mask of the samples that carry a ray
    gradient (matched, det E != 0) and the positions with a unit tetrahedron in place of the others (so that every solve is regular)"""
    vi = torch.as_tensor(vertex_indices).long()
    X = torch.as_tensor(np.asarray(xyz, dtype=np.float32)).to(dtype).reshape(-1, 3)
    verts = X[vi.clamp_min(0)]
    E = verts[..., 1:, :] - verts[..., :1, :]  # rows e_k
    good = (vi[..., 0] >= 0) & (torch.linalg.det(E) != 0)
    unit = torch.cat([torch.zeros((1, 3), dtype=dtype), torch.eye(3, dtype=dtype)])
    return torch.where(good[..., None, None], verts, unit), good


def differentiable_bary(vertex_indices, bary, xyz, points, exact: bool = False):
    """the matched weights as a function of the sample positions `points` [...,3]: their values (exact=False: add_barycentrics_grad, the
    values unchanged) or E^-1 (x - x_v0) recomputed (exact=True); unmatched samples and det E = 0 keep the constant weights"""
    from tetranerf.utils.extension import add_barycentrics_grad

    b = torch.as_tensor(bary).to(points.dtype)
    verts, good = tet_edges(vertex_indices, xyz, points.dtype)
    if exact:
        E = (verts[..., 1:, :] - verts[..., :1, :]).transpose(-1, -2)  # columns e_k
        bx = torch.linalg.solve(E, points - verts[..., 0, :])
    else:
        bx = add_barycentrics_grad(b, verts, points)
    return torch.where(good[..., None], bx, b)


def render_train_rays(mesh: "orc.OracleMesh", field: torch.Tensor, params: Dict[str, torch.Tensor], origins: torch.Tensor,
                      directions: torch.Tensor, cfg: "orc.RenderConfig", jitter_coarse=None, jitter_fine=None, use_gradient_scaling: bool = False,
                      nthreads: int = 0, fine_euclid=None, matched=None, exact_bary: bool = False):
    """oracle.render_train with gradients to `origins` / `directions` ([R,3] tensors; the trace and the samplers see their float32
    values).  aux adds `positions` (the fine sample positions x_i, [R',S2,3] for the non-empty rays) and `features` (f_i, [R',S2,64]); when
    they require grad their .grad after a backward holds dL/dx_i and dL/df_i."""
    o = origins.reshape(-1, 3)
    d = directions.reshape(-1, 3)
    R = o.shape[0]
    assert cfg.num_fine_samples > 0
    o32, d32 = o.detach().float().numpy(), d.detach().float().numpy()
    tr = mesh.trace_rays(o32, d32, cfg.max_intersected_triangles, nthreads=nthreads)
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
    # the fine samples' positions: the matcher's distances (float32, constants) along the differentiable rays
    t = ((euclid[:, 1:] + euclid[:, :-1]) / 2).detach().to(o.dtype)
    idx = torch.nonzero(ray_mask).flatten()
    pos = o[idx][:, None, :] + t[..., None] * d[idx][:, None, :]
    bary = differentiable_bary(tc["vertex_indices"], tc["barycentric_coordinates"], mesh.xyz, pos, exact=exact_bary).to(field.dtype)
    fv = interpolate_with_weights(tc["vertex_indices"], bary, field)
    for x in (pos, fv):  # per-sample dL/dx and dL/df for the tests, after backward
        if x.requires_grad:
            x.retain_grad()
    base = orc.mlp_base(params, fv)
    sigmas = orc.density_head(params, base)
    enc = orc.nerf_encoding_dirs(d[idx].to(base.dtype))[:, None, :].expand(-1, base.shape[1], -1)
    colors = orc.color_head(params, base, enc)
    if use_gradient_scaling:
        ray_dist = (sbins[:, 1:] + sbins[:, :-1])[..., None]  # spacing_ends + spacing_starts (model.py:629)
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
