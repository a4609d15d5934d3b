"""Oracle of the distortion loss of the fused training step -- TEST INFRASTRUCTURE ONLY.

Definition (DESIGN.md §4.11; mip-NeRF 360, nerfstudio 0.3.x losses.distortion_loss, which is not installed here, so this restatement is
the contract).  For one active ray, over the samples that give rgb (the fine pass), with s_0 ... s_S the spacing bins
(ray_samples_to_sdist: spacing_starts plus the last spacing_end), u_i = (s_i + s_{i+1}) / 2, delta_i = s_{i+1} - s_i and w_i the weights
of get_weights:
  d = sum_i sum_j w_i w_j |u_i - u_j| + 1/3 sum_i w_i^2 delta_i,       dd/dw_j = 2 sum_i w_i |u_j - u_i| + 2/3 w_j delta_j;
empty rays: d = 0, no gradient.  The bins are constants (the PDF sampler detaches them; the ray and vertex gradients hold the sample
distances fixed).  The gradient joins dL/dw_j before the transmittance sums, so GradientScaler applies to it as to the colour term.

`distortion` is the literal double sum, evaluated in chunks of rays so that its [rays, S, S] terms stay small, with the closed-form
gradient above as its backward; `render_train_distortion` is expected_depth.render_train_depth (the same stages in the same order) with
`distortion` added, so one call differentiates a distortion loss to the field, the MLP, the rays and the vertices."""
from __future__ import annotations

from typing import Dict

import torch

from . import expected_depth as edo
from . import oracle as orc
from . import ray_grads as rg
from . import vertex_grads as vg

CHUNK = 16  # rays per [CHUNK, S, S] block


class _Definition(torch.autograd.Function):
    """w [R,S] (differentiable), u / delta [R,S] constants -> d [R]"""

    @staticmethod
    def forward(ctx, w, u, delta):
        ctx.save_for_backward(w, u, delta)
        out = w.new_zeros(w.shape[0])
        for a in range(0, w.shape[0], CHUNK):
            wc, uc = w[a:a + CHUNK], u[a:a + CHUNK]
            dist = (uc[:, :, None] - uc[:, None, :]).abs()
            out[a:a + CHUNK] = torch.einsum("ri,rij,rj->r", wc, dist, wc) + (wc * wc * delta[a:a + CHUNK]).sum(-1) / 3
        return out

    @staticmethod
    def backward(ctx, g):
        w, u, delta = ctx.saved_tensors
        gw = torch.zeros_like(w)
        for a in range(0, w.shape[0], CHUNK):
            wc, uc = w[a:a + CHUNK], u[a:a + CHUNK]
            dist = (uc[:, :, None] - uc[:, None, :]).abs()
            gw[a:a + CHUNK] = g[a:a + CHUNK, None] * (2 * torch.einsum("rij,ri->rj", dist, wc) + 2.0 / 3.0 * wc * delta[a:a + CHUNK])
        return gw, None, None


def distortion(weights: torch.Tensor, sdist: torch.Tensor) -> torch.Tensor:
    """weights [R',S,1] (differentiable), sdist [R',S+1] spacing bins of the same rays -> d [R',1], in the weights' dtype"""
    s = sdist.detach().to(weights.dtype)
    u = (s[:, 1:] + s[:, :-1]) / 2
    delta = s[:, 1:] - s[:, :-1]
    return _Definition.apply(weights[..., 0], u, delta)[:, None]


def render_train_distortion(mesh: "orc.OracleMesh", field: torch.Tensor, params: Dict[str, torch.Tensor], origins: torch.Tensor,
                            directions: torch.Tensor, xyz, cfg: "orc.RenderConfig", jitter_coarse=None, jitter_fine=None,
                            use_gradient_scaling: bool = False, fine_euclid=None, fine_sbins=None, exact_bary: bool = False):
    """expected_depth.render_train_depth plus `distortion` [R,1] (0 on empty rays).  fine_euclid: the fine bins to use instead of the
    sampler's (ray order of the non-empty rays); fine_sbins: their spacing bins (default: mapped back from fine_euclid with the ray's
    near / far).  exact_bary: the sample weights solved from the positions in the forward too (vertex_grads.differentiable_bary), so
    that finite differences see the ray and vertex gradients.  aux as there, plus "sbins"."""
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
        sbins = torch.as_tensor(fine_sbins, dtype=torch.float32) if fine_sbins is not None else (euclid - nears_r) / (fars_r - nears_r)
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
    bary = vg.differentiable_bary(tc["vertex_indices"], tc["barycentric_coordinates"], xyz, pos, exact=exact_bary).to(field.dtype)
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
    ed = edo.expected_depth(weights, euclid, ray_mask, cfg.far_plane)
    dist = torch.zeros((R, 1), dtype=rgb_r.dtype).index_copy(0, idx, distortion(weights, sbins))
    return {"rgb": rgb, "accumulation": acc, "expected_depth": ed, "distortion": dist, "ray_mask": ray_mask,
            "aux": {"fine_euclid": euclid.detach(), "sbins": sbins.detach(), "weights": weights.detach(), "matched": tc}}
