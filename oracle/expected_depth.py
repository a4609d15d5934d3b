"""Oracle of the expected depth of the fused render and training step -- TEST INFRASTRUCTURE ONLY.

Definition (DESIGN.md §4.10; nerfstudio 0.3.x DepthRenderer(method="expected"), which is not installed here, so this restatement is
the contract).  For the active rays of one call, over the bins and weights that give rgb (the fine bins; the coarse ones when
num_fine_samples = 0), with t_i = (e_i + e_{i+1}) / 2 the bin midpoints (formed in float32, as the bins are), w_i the weights of
get_weights and A = sum_i w_i:
  * D_raw = sum_i w_i t_i / (A + 1e-10);
  * D = clip(D_raw, t_min, t_max), t_min / t_max the smallest / largest midpoint over ALL samples of ALL active rays of the call (as
    nerfstudio's steps.min() / steps.max() of the batch); the clip only binds when A is tiny;
  * empty rays: D = far_plane, no gradient; training mode: no nan_to_num or clamp.
Gradient, in the conventions of §4.5 / §4.8 / §4.9: bins and midpoints are constants; where t_min <= D_raw <= t_max (inclusive, as
torch.clip's backward) dD/dw_i = (t_i - D_raw) / (A + 1e-10), else 0.  It joins dL/dw_i before the transmittance sums, so GradientScaler
(which scales dL/dsigma) applies to it as to the colour term.

`expected_depth` is that formula in torch (autograd gives the gradient above); `render_train_depth` is
vertex_grads.render_train_geometry (hence ray_grads.render_train_rays and oracle.render_train when nothing but the field and the MLP
require grad) with `expected_depth` added, so one call differentiates a depth loss to the field, the MLP, the rays and the vertices.
`depth_at_bins` evaluates D at given bins (an implementation's own) with the eval-mode network, for single-pass configurations too."""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from . import oracle as orc
from . import ray_grads as rg
from . import vertex_grads as vg

EPS = 1e-10


def expected_depth(weights: torch.Tensor, euclid: torch.Tensor, ray_mask: torch.Tensor, far_plane: float) -> torch.Tensor:
    """weights [R',S,1] (differentiable), euclid [R',S+1] bin edges of the active rays in ray order, ray_mask bool[R] -> D [R,1]"""
    steps = ((euclid[:, 1:] + euclid[:, :-1]) / 2).detach().to(weights.dtype)  # float32 midpoints, as the renderers form them
    w = weights[..., 0]
    d_raw = torch.sum(w * steps, dim=-1) / (torch.sum(w, dim=-1) + EPS)
    d = torch.clip(d_raw, steps.min(), steps.max()) if steps.numel() else d_raw
    idx = torch.nonzero(ray_mask).flatten()
    return torch.full((ray_mask.shape[0], 1), far_plane, dtype=weights.dtype).index_copy(0, idx, d[:, None])


def render_train_depth(mesh: "orc.OracleMesh", field: torch.Tensor, params: Dict[str, torch.Tensor], origins: torch.Tensor,
                       directions: torch.Tensor, xyz, cfg: "orc.RenderConfig", jitter_coarse=None, jitter_fine=None,
                       use_gradient_scaling: bool = False, fine_euclid=None):
    """vertex_grads.render_train_geometry plus `expected_depth` [R,1]; `xyz` is the float32 positions (no vertex gradient) or a torch
    tensor that may require grad.  The same stages in the same order; aux as there."""
    o = origins.reshape(-1, 3)
    d = directions.reshape(-1, 3)
    R = o.shape[0]
    assert cfg.num_fine_samples > 0
    tr = mesh.trace_rays(o.detach().float().numpy(), d.detach().float().numpy(), cfg.max_intersected_triangles)
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
                                      trm["vertex_indices"], dist.detach().numpy())

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
    tc = match(euclid)
    t = ((euclid[:, 1:] + euclid[:, :-1]) / 2).detach().to(o.dtype)
    idx = torch.nonzero(ray_mask).flatten()
    pos = o[idx][:, None, :] + t[..., None] * d[idx][:, None, :]
    bary = vg.differentiable_bary(tc["vertex_indices"], tc["barycentric_coordinates"], xyz, pos).to(field.dtype)
    fv = rg.interpolate_with_weights(tc["vertex_indices"], bary, field)
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
    rgb = bg.expand(R, 3).clone().index_copy(0, idx, rgb_r)
    acc = torch.zeros((R, 1), dtype=rgb_r.dtype).index_copy(0, idx, accum)
    ed = expected_depth(weights, euclid, ray_mask, cfg.far_plane)
    return {"rgb": rgb, "accumulation": acc, "expected_depth": ed, "ray_mask": ray_mask,
            "aux": {"fine_euclid": euclid.detach(), "weights": weights.detach(), "matched": tc}}


def depth_at_bins(mesh: "orc.OracleMesh", field, params: Dict[str, torch.Tensor], origins, directions, cfg: "orc.RenderConfig", euclid,
                  dtype=torch.float64) -> Dict[str, torch.Tensor]:
    """D of the eval render at the bins `euclid` f32[R',S+1] (the active rays in ray order: the fine bins, or the coarse ones when
    num_fine_samples = 0), the network evaluated in `dtype` -> {"expected_depth" [R,1], "accumulation" [R,1], "ray_mask"}"""
    o = np.asarray(origins, dtype=np.float32).reshape(-1, 3)
    d = np.asarray(directions, dtype=np.float32).reshape(-1, 3)
    tr = mesh.trace_rays(o, d, cfg.max_intersected_triangles)
    ray_mask = torch.from_numpy(tr["num_visited_cells"]) > 0
    m = ray_mask.numpy()
    euclid = torch.as_tensor(euclid, dtype=torch.float32)
    dist = ((euclid[:, 1:] + euclid[:, :-1]) / 2).contiguous()
    tc = orc.find_visited_cells(tr["num_visited_cells"][m], tr["visited_cells"][m], tr["barycentric_coordinates"][m], tr["hit_distances"][m],
                                tr["vertex_indices"][m], dist.numpy())
    p = {k: torch.as_tensor(v).detach().to(dtype) for k, v in params.items()}
    fv = orc.interpolate_torch(tc["vertex_indices"], tc["barycentric_coordinates"], torch.as_tensor(np.asarray(field)).to(dtype))
    sigmas = orc.density_head(p, orc.mlp_base(p, fv))
    weights = orc.get_weights((euclid[:, 1:] - euclid[:, :-1]).to(dtype)[..., None], sigmas)
    idx = torch.nonzero(ray_mask).flatten()
    acc = torch.zeros((len(o), 1), dtype=dtype).index_copy(0, idx, weights.sum(-2))
    return {"expected_depth": expected_depth(weights, euclid, ray_mask, cfg.far_plane), "accumulation": acc, "ray_mask": ray_mask}
