"""Host-side mirror of the reference's nerfstudio plug-in for the ray-sampling hot path.

Same public names, constructor arguments, config fields, state-dict keys/shapes and output dictionary as
the reference `tetranerf/nerfstudio/model.py` (TetrahedraNerfConfig :70-107, TetrahedraSampler :125-192,
TetrahedraNerf :209-662), so `ns-train tetra-nerf` can import this module unchanged.  What differs is where
the work happens:

  * inference (`not self.training` and no autograd): the whole body of `get_outputs` after the ray bundle --
    trace, sampling, matching, interpolation, both MLP passes, PDF resampling and compositing
    (reference :526-662) -- is ONE call into the fused CUDA pipeline (`tetranerf.b200.render.FusedRenderer`);
  * training: the reference's own sequence of calls (trace_rays -> sampler -> find_visited_cells ->
    interpolate_values -> torch MLPs -> renderers) is kept, on top of our CUDA ops, so that autograd
    reaches `tetrahedra_field` and the MLP weights exactly as it does upstream.

Evaluation images / metrics (`get_image_metrics_and_images`, reference :676-713) are provided with PSNR and SSIM computed in torch
(torchmetrics / LPIPS are used when nerfstudio and its dependencies are installed); appearance embeddings (reference :440-446,
608-620) run on the unfused path.  The occupancy field the reference declares but never reads (:98,256-265) culls empty tetrahedra on the
fused paths here (DESIGN §4.12).  nerfstudio itself is imported when it is installed; otherwise the minimal look-alikes of `_ns_compat`
are used.
"""
from __future__ import annotations

import dataclasses
import os
import warnings
from dataclasses import dataclass
from pathlib import Path
from typing import Any, Dict, List, Literal, Optional

import torch
from torch import nn
from torch.nn import Parameter

try:  # the real thing when available (reference model.py:10-28)
    from nerfstudio.cameras.rays import RayBundle, RaySamples
    from nerfstudio.engine.callbacks import TrainingCallback, TrainingCallbackAttributes, TrainingCallbackLocation
    from nerfstudio.field_components.encodings import NeRFEncoding
    from nerfstudio.field_components.field_heads import DensityFieldHead, FieldHeadNames, RGBFieldHead
    from nerfstudio.field_components.mlp import MLP
    from nerfstudio.model_components.losses import MSELoss
    from nerfstudio.model_components.ray_samplers import PDFSampler, Sampler, UniformSampler
    from nerfstudio.model_components.renderers import AccumulationRenderer, DepthRenderer, RGBRenderer
    from nerfstudio.models.base_model import Model, ModelConfig
    from nerfstudio.utils.misc import scale_dict

    HAVE_NERFSTUDIO = True
except ImportError:
    from ._ns_compat import (AccumulationRenderer, DensityFieldHead, DepthRenderer, FieldHeadNames, MLP, MSELoss, Model, ModelConfig,
                             NeRFEncoding, PDFSampler, RayBundle, RaySamples, RGBFieldHead, RGBRenderer, Sampler, TrainingCallback,
                             TrainingCallbackAttributes, TrainingCallbackLocation, UniformSampler, scale_dict)

    HAVE_NERFSTUDIO = False

from ..utils.extension import TetrahedraTracer, interpolate_values, triangulate


VERTEX_FOLD_GUARD_MAX_HALVINGS = 8
"""vertex_fold_guard: the most times a vertex's step is halved before the vertex is held at its old position instead (2^-8 of the step)"""


@dataclass
class TetrahedraNerfConfig(ModelConfig):
    """Field-for-field the reference config (model.py:70-107)."""

    _target: Any = dataclasses.field(default_factory=lambda: TetrahedraNerf)
    tetrahedra_path: Optional[Path] = None
    num_tetrahedra_vertices: Optional[int] = None
    num_tetrahedra_cells: Optional[int] = None
    max_intersected_triangles: int = 512
    num_samples: int = 256
    num_fine_samples: int = 256
    use_biased_sampler: bool = False
    field_dim: int = 64
    num_color_layers: int = 1
    num_density_layers: int = 3
    hidden_size: int = 128
    input_fourier_frequencies: int = 0
    initialize_colors: bool = True
    use_gradient_scaling: bool = False
    background_color: Literal["random", "last_sample", "black", "white"] = "white"
    appearance_embed_dim: int = 0
    use_occupancy_field: bool = False
    """register the reference's `tetrahedra_occupancy` f32[T] buffer and cull, on the fused render and training paths, the samples that
    fall in a tetrahedron whose occupancy (the largest density over its vertices, edge midpoints and centroid) is below
    occupancy_threshold: their density is 0 and their MLP is skipped (DESIGN §4.12).  Needs the fused pipeline (RuntimeError otherwise)"""
    occupancy_threshold: float = 0.01
    """density below which a tetrahedron is culled: a culled cell removes at most 1 - exp(-0.01 l) of opacity over a chord of length l"""
    occupancy_update_interval: int = 16
    """training steps between two occupancy updates (the first one at occupancy_warmup_steps)"""
    occupancy_decay: float = 0.95
    """an update sets occupancy = max(occupancy_decay * occupancy, the new probe maximum), so a cell that empties out is culled after a
    few updates rather than at once"""
    occupancy_warmup_steps: int = 256
    """training steps without culling at the start, so the randomly initialised field is not culled away"""
    occupancy_sampling: bool = False
    """also place each ray's coarse samples in its tetrahedra at or above occupancy_threshold only, so the num_samples /
    num_fine_samples budget is not spent on culled empty space (DESIGN §4.13); applies exactly when culling does.  Needs
    use_occupancy_field (RuntimeError otherwise)"""
    render_normals: bool = False
    """eval renders also return "normals" f32[R,3], the composited normal of the density field (fused path only; training ignores it)"""
    optimize_vertices: bool = False
    """train the mesh vertex positions too: `tetrahedra_vertices` becomes a parameter in its own param group "vertices" (same state-dict
    key and shape), the tracer is refit after every optimizer step (topology fixed), training runs on the fused path only (DESIGN §4.9)"""
    vertex_fold_guard: bool = False
    """with optimize_vertices: before each refit, scale back per vertex the part of the optimizer's step that would fold the mesh
    (TetrahedraTracer.guard_vertex_step, DESIGN §4.17): every interior face certified unfolded at the last load or refit stays so, and
    a mesh the adjacency walk ran on keeps it.  A vertex of a face the step would fold moves 2^-k of its step, k the round in
    1..VERTEX_FOLD_GUARD_MAX_HALVINGS after which none of its faces fails, or stays where it was.  The optimizer state is not touched.  A different
    policy from the default (where a folding step is taken, warned about once, and the walk turns off), hence an option.  Needs
    optimize_vertices (RuntimeError otherwise).  False changes nothing"""
    render_expected_depth: bool = False
    """every path (fused eval, fused training, unfused) also returns "expected_depth" f32[R,1], nerfstudio's
    DepthRenderer(method="expected") clipped to the batch's smallest / largest sample midpoint, far plane on empty rays (DESIGN §4.10);
    differentiable in training"""
    depth_loss_mult: float = 0.0
    """> 0: implies render_expected_depth and adds depth_loss = depth_loss_mult * mean over rays with hits and a finite target > 0 of
    (expected_depth - target)^2, the target batch["depth_image"] [R,1] in the model's frame"""
    is_euclidean_depth: bool = False
    """the depth target is the distance along the ray; False: z-depth, multiplied by the ray bundle's metadata["directions_norm"]"""
    distortion_loss_mult: float = 0.0
    """> 0: training outputs also hold "distortion" f32[R,1], mip-NeRF 360's distortion of each ray's weights over its spacing bins (0 on
    empty rays; DESIGN §4.11), and the loss dict gains distortion_loss = distortion_loss_mult * its mean over the rays with hits, as
    nerfacto's distortion_loss_mult.  Training only; 0 changes nothing"""
    field_smoothness_mult: float = 0.0
    """> 0: the loss dict gains field_smoothness_loss = field_smoothness_mult * S / (E * field_dim), S the sum over the mesh's E unique
    undirected edges {i, j} of sum_c (F[c,i] - F[c,j])^2: a uniform-weight neighbour-difference regulariser on tetrahedra_field, as
    explicit-feature radiance fields use, that keeps the vertices few rays see from drifting (DESIGN §4.15).  It does not depend on the
    vertex positions.  After refine() the next loss is taken on the refined mesh, and the refinement score then sees the sum of both field
    gradients (rendering and smoothness).  Needs the fused pipeline (RuntimeError otherwise).  Training only; 0 changes nothing"""
    refine_every: int = 0
    """> 0: refine the mesh during training every refine_every steps in [refine_start, refine_stop) (TetrahedraNerf.refine, DESIGN §4.14):
    the tetrahedra whose field gradient stays large have their longest edges bisected, the new vertices taking the mean of their edge's
    endpoints, so the field is unchanged and the optimizer gains degrees of freedom where the images need them.  0 = off, nothing
    changes.  With use_biased_sampler a refined ray shares its samples over more records, so renders are not preserved at the moment of
    refinement (by design; the uniform sampler preserves them).  Refinement raises the number of tetrahedra per ray: watch that
    max_intersected_triangles still covers the rays.  The refined mesh is no longer Delaunay, which nothing downstream requires;
    delaunay_flip_every > 0 flips it back towards Delaunay at the end of every refinement"""
    refine_start: int = 500
    """first training step at which the mesh may be refined"""
    refine_stop: int = 15000
    """no refinement from this training step on"""
    refine_fraction: float = 0.05
    """share of the tetrahedra that are candidates in one refinement: the highest-scoring ones with a score > 0, a tetrahedron scoring the
    mean over its vertices of the mean per-step gradient norm of their field column since the last refinement"""
    refine_passes: int = 3
    """bisection passes per refinement; a tetrahedron split in one pass, and its children, are not candidates again in the same one"""
    refine_min_edge_length: float = 0.0
    """a candidate proposes its longest edge only when that is at least this long"""
    refine_max_vertices: Optional[int] = None
    """refinement stops adding vertices at this many mesh vertices (None: no limit)"""
    coarsen_every: int = 0
    """> 0: coarsen the mesh in empty space during training every coarsen_every steps in [coarsen_start, coarsen_stop)
    (TetrahedraNerf.coarsen, DESIGN §4.18): a non-hull vertex whose tetrahedra all have tetrahedra_occupancy < occupancy_threshold is
    collapsed into its nearest neighbour that keeps every tetrahedron's orientation, so empty space stops costing trace steps, samples,
    records and memory.  The hull and the occupied tetrahedra are untouched.  0 = off, nothing changes.  Needs use_occupancy_field and
    the fused pipeline (RuntimeError at construction otherwise).  It never runs before occupancy_warmup_steps training steps or on an
    occupancy buffer that was never computed.  When a refinement is due on the same step, coarsening runs first"""
    coarsen_start: int = 1000
    """first training step at which the mesh may be coarsened"""
    coarsen_stop: int = 15000
    """no coarsening from this training step on"""
    coarsen_passes: int = 3
    """collapse passes per coarsening; a pass removes vertices that share no tetrahedron, so later passes reach the neighbours of
    vertices an earlier pass kept"""
    delaunay_flip_every: int = 0
    """> 0: restore the Delaunay property of the mesh as far as flips can (TetrahedraNerf.flip_delaunay, DESIGN §4.19) every
    delaunay_flip_every training steps and at the end of every refine() and coarsen() that changed the mesh: 2-3 and 3-2 flips of the
    faces whose opposite vertex lies inside the other tetrahedron's circumsphere, until a pass proposes nothing.  The vertices, the field
    and the optimizer state do not change; only the tetrahedra do, each new one taking the maximum occupancy of the ones it replaced.
    Refinement, coarsening and trained vertex positions all leave non-Delaunay faces behind.  0 = off, nothing changes"""
    delaunay_flip_max_passes: int = 64
    """flip passes per flip_delaunay at most; a pass applies flips that share no tetrahedron, so later passes reach the faces an earlier
    pass created or left.  Meshes refined three times took 29 to 47 passes to the fixed point (DESIGN §4.19); when the limit stops the
    loop first, flip_delaunay's "illegal_left" counts what was not reached, and the next flip continues from there"""
    background_envmap_height: int = 0
    """> 0: learn the light that leaves the mesh as an environment map: the parameter `background_envmap` f32[H, 2H, 3] (H this value;
    "fields" group, in the state dict only when enabled) in the model's frame, z up, equal-area in latitude, initialised to
    background_color (white or black; RuntimeError otherwise), so the first render is the constant-background render bit for bit.
    Every path composites rgb = sum_j w_j c_j + (1 - accumulation) bg(d), and rgb = bg(d) on rays that miss the mesh (DESIGN §4.16).
    0 = off, nothing changes"""

    def __post_init__(self):
        if self.tetrahedra_path is not None and self.num_tetrahedra_vertices is None:
            if not Path(self.tetrahedra_path).exists():
                raise RuntimeError(f"Tetrahedra path {self.tetrahedra_path} does not exist")
            th = torch.load(self.tetrahedra_path)
            self.num_tetrahedra_vertices = len(th["vertices"])
            self.num_tetrahedra_cells = len(th["cells"])


def map_from_real_distances_to_biased_with_bounds(num_bounds, bounds, samples):
    """Every visited tetrahedron receives the same share of the unit interval (reference model.py:111-122).

    num_bounds i64[R]; bounds f32[R,M,2] = (t_in, t_out) per visited cell; samples f32[R,S] euclidean distances in
    [first t_in, last t_out].  Returns the samples re-mapped onto the concatenated cell intervals."""
    seg_len = (bounds[..., 1] - bounds[..., 0]).clamp_min(0)
    first = bounds[:, 0, 0]
    last = torch.gather(bounds[..., 1], 1, (num_bounds[:, None] - 1).clamp_min(0)).squeeze(-1)
    pos = (samples - first[:, None]) / (last - first)[:, None] * num_bounds[:, None]
    cell = torch.minimum(pos.floor(), (num_bounds[:, None] - 1).to(pos.dtype)).clamp_min(0)
    frac = pos - cell
    cell = cell.long()
    starts = torch.cumsum(torch.cat((first[:, None], seg_len), 1), 1)
    return torch.gather(starts, 1, cell) + torch.gather(seg_len, 1, cell) * frac


class TetrahedraSampler(Sampler):
    """Biased sampler: an equal number of bins per visited tetrahedron (reference model.py:125-192)."""

    def __init__(self, num_samples: Optional[int] = None, train_stratified=True) -> None:
        super().__init__(num_samples=num_samples)
        self.train_stratified = train_stratified

    def generate_ray_samples(self, ray_bundle: Optional[RayBundle] = None, num_samples: Optional[int] = None, *, num_visited_cells, hit_distances) -> RaySamples:
        assert ray_bundle is not None and ray_bundle.nears is not None and ray_bundle.fars is not None
        num_samples = num_samples or self.num_samples
        assert num_samples is not None
        dev = ray_bundle.origins.device
        bins = torch.linspace(0.0, 1.0, num_samples + 1).to(dev)[None, ...]
        if self.train_stratified and self.training:  # per-bin jitter, as nerfstudio's SpacedSampler
            jitter = torch.rand((ray_bundle.origins.shape[0], num_samples + 1), dtype=bins.dtype, device=dev)
            mids = (bins[..., 1:] + bins[..., :-1]) / 2.0
            hi = torch.cat([mids, bins[..., -1:]], -1)
            lo = torch.cat([bins[..., :1], mids], -1)
            bins = lo + (hi - lo) * jitter
        near, far = ray_bundle.nears, ray_bundle.fars

        def to_euclidean(x):
            return x * far + (1 - x) * near

        euclid = map_from_real_distances_to_biased_with_bounds(num_visited_cells.long(), hit_distances, to_euclidean(bins))
        bins = (euclid - near) / (far - near)
        return ray_bundle.get_ray_samples(bin_starts=euclid[..., :-1, None], bin_ends=euclid[..., 1:, None], spacing_starts=bins[..., :-1, None],
                                          spacing_ends=bins[..., 1:, None], spacing_to_euclidean_fn=to_euclidean)


class GradientScaler(torch.autograd.Function):
    """Near-camera gradient damping, squared ray distance clamped to [0,1] (reference model.py:195-205)."""

    @staticmethod
    def forward(ctx, colors, sigmas, ray_dist):
        ctx.save_for_backward(ray_dist)
        return colors, sigmas, ray_dist

    @staticmethod
    def backward(ctx, g_colors, g_sigmas, g_dist):
        (ray_dist,) = ctx.saved_tensors
        s = torch.square(ray_dist).clamp(0, 1)
        return g_colors * s, g_sigmas * s, g_dist


def distortion_per_ray(weights: torch.Tensor, sdist: torch.Tensor) -> torch.Tensor:
    """mip-NeRF 360's distortion of each ray (nerfstudio's losses.distortion_loss before its mean), in O(S) per ray: weights [R,S,1],
    sdist [R,S+1] sorted spacing bins -> [R,1].  With u the bin midpoints, delta their widths and W_<j, P_<j the exclusive prefix sums of
    w and w u, sum_i sum_j w_i w_j |u_i - u_j| = 2 sum_j w_j (u_j W_<j - P_<j), so no [R,S,S] tensor is formed; autograd gives
    dd/dw_j = 2 sum_i w_i |u_j - u_i| + 2/3 w_j delta_j"""
    w = weights[..., 0]
    u = (sdist[..., 1:] + sdist[..., :-1]) / 2
    delta = sdist[..., 1:] - sdist[..., :-1]
    zero = torch.zeros_like(w[..., :1])
    w_excl = torch.cumsum(torch.cat((zero, w[..., :-1]), -1), -1)
    p_excl = torch.cumsum(torch.cat((zero, (w * u)[..., :-1]), -1), -1)
    inter = 2 * torch.sum(w * (u * w_excl - p_excl), -1, keepdim=True)
    intra = torch.sum(w**2 * delta, -1, keepdim=True) / 3
    return inter + intra


class TetrahedraNerf(Model):
    """Tetra-NeRF model on the H100-native tracer.  Buffers `tetrahedra_vertices` f32[V,3], `tetrahedra_cells`
    i32[T,4] and parameter `tetrahedra_field` f32[field_dim,V] keep the reference's names and shapes
    (model.py:239-255) so checkpoints interchange."""

    config: TetrahedraNerfConfig

    def __init__(self, config: TetrahedraNerfConfig, dataparser_transform=None, dataparser_scale=None, metadata=None, **kwargs) -> None:
        super().__init__(config=config, **kwargs)
        self.dataparser_transform = dataparser_transform
        self.dataparser_scale = dataparser_scale
        self._tetrahedra_tracer = None
        self._fused = None
        self._fused_versions = None
        self._grad_acc = self._grad_cnt = None  # refinement statistics (refine_every > 0): not part of the state dict
        self._guard_start = None  # vertex_fold_guard: device copy of the positions the tracer was last loaded or refit at
        if self.config.tetrahedra_path is None and metadata is not None and "points3D_xyz" in metadata:
            self._load_points_from_metadata(**metadata)
        else:
            if self.config.num_tetrahedra_vertices is None or self.config.num_tetrahedra_cells is None:
                raise RuntimeError("The tetrahedra_path must be specified.")
            V, T = self.config.num_tetrahedra_vertices, self.config.num_tetrahedra_cells
            self._register_vertices(torch.empty((V, 3), dtype=torch.float32))
            self.register_buffer("tetrahedra_cells", torch.empty((T, 4), dtype=torch.int32))
            self.register_parameter("tetrahedra_field", nn.Parameter(torch.empty((self.config.field_dim, V), dtype=torch.float32)))
            self._register_occupancy(T)
            self._tetrahedra_initialized = False

    # ---- initialisation (reference :268-392) --------------------------------------------------------
    @staticmethod
    def _init_tetrahedra_field(tetrahedra_field):
        tetrahedra_field.uniform_(-1e-4, 1e-4)

    def _register_occupancy(self, T: int):
        """`tetrahedra_occupancy` f32[T] of zeros (the reference's key, shape and dtype, model.py:256-265), with use_occupancy_field.  All
        zeros means "never computed": it is recomputed before its first use"""
        self._occ_ready = False
        self._occ_step = 0
        if self.config.use_occupancy_field:
            self.register_buffer("tetrahedra_occupancy", torch.zeros((T,), dtype=torch.float32))

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        complete = all(f"{prefix}{k}" in state_dict for k in ("tetrahedra_vertices", "tetrahedra_cells", "tetrahedra_field"))
        self._occ_ready = False  # a loaded buffer is checked for zeros again
        # a refined checkpoint holds more vertices and tetrahedra than the config the model was built from: take its sizes in place,
        # through .data, so the Parameter objects an optimizer built before the load holds stay the model's (DESIGN §4.14)
        resized = False
        for name in ("tetrahedra_vertices", "tetrahedra_cells", "tetrahedra_field", "tetrahedra_occupancy"):
            cur, new = getattr(self, name, None), state_dict.get(prefix + name)
            if isinstance(cur, torch.Tensor) and isinstance(new, torch.Tensor) and new.shape != cur.shape:
                _set_data(cur, torch.empty(new.shape, dtype=cur.dtype, device=cur.device))
                resized = True
        if resized:
            self.config.num_tetrahedra_vertices, self.config.num_tetrahedra_cells = len(self.tetrahedra_vertices), len(self.tetrahedra_cells)
            self._tetrahedra_tracer = self._fused = self._fused_versions = None
            self._grad_acc = self._grad_cnt = None
        self._guard_start = None  # the loaded positions are not a step: the next refit takes them as they are
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
        if complete:
            self._tetrahedra_initialized = True

    def _register_vertices(self, vertices: torch.Tensor):
        """`tetrahedra_vertices`: a buffer, or with optimize_vertices a parameter (the same state-dict key either way)"""
        if self.config.optimize_vertices:
            self.register_parameter("tetrahedra_vertices", nn.Parameter(vertices))
        else:
            self.register_buffer("tetrahedra_vertices", vertices)

    def _install_mesh(self, vertices: torch.Tensor, cells: torch.Tensor, colors: Optional[torch.Tensor], alpha: Optional[torch.Tensor]):
        V = len(vertices)
        self.config.num_tetrahedra_vertices, self.config.num_tetrahedra_cells = V, len(cells)
        if hasattr(self, "tetrahedra_vertices"):
            with torch.no_grad():
                self.tetrahedra_vertices.copy_(vertices.to(self.tetrahedra_vertices.device))
            self.tetrahedra_cells.copy_(cells.to(torch.int32).to(self.tetrahedra_cells.device))
            if self.config.use_occupancy_field:
                self.tetrahedra_occupancy.zero_()
                self._occ_ready = False
        else:
            self._register_vertices(vertices.float())
            self.register_buffer("tetrahedra_cells", cells.to(torch.int32))
            self.register_parameter("tetrahedra_field", nn.Parameter(torch.empty((self.config.field_dim, V), dtype=torch.float32)))
            self._register_occupancy(len(cells))
        self._init_tetrahedra_field(self.tetrahedra_field.data)
        if self.config.initialize_colors:
            assert colors is not None and colors.dtype == torch.uint8
            rgb = colors.float().to(self.tetrahedra_field.device) * 2.0 / 255.0 - 1.0
            self.tetrahedra_field.data[1:4, :] = rgb[:, :3].T
            self.tetrahedra_field.data[0, :] = 1.0 if alpha is None else alpha.float().to(self.tetrahedra_field.device) * 2.0 / 255.0 - 1.0
        self._tetrahedra_initialized = True

    def _load_points_from_metadata(self, points3D_xyz, points3D_rgb=None, **kwargs):
        cells = triangulate(points3D_xyz).int()
        self._install_mesh(points3D_xyz, cells, points3D_rgb, None)

    def _init_tetrahedra(self):
        if self.config.tetrahedra_path is None:
            raise RuntimeError("The tetrahedra_path must be specified.")
        path = Path(self.config.tetrahedra_path)
        if not path.exists():
            raise RuntimeError(f"Specified tetrahedra path {path} does not exist")
        if self.dataparser_scale is None:
            raise RuntimeError("Could not read the dataparser_scale and dataparser_transform parameters."
                               "Make sure you are using the TetrahedraNerfPipeline with the model.")
        th = torch.load(str(path), map_location=torch.device("cpu"))  # {"vertices", "cells", "colors"} (scripts/triangulate.py:68-75)
        verts = th["vertices"].float()
        verts = torch.cat((verts, torch.ones_like(verts[..., :1])), -1) @ self.dataparser_transform.T
        verts = verts * self.dataparser_scale
        colors = th.get("colors")
        self._install_mesh(verts, th["cells"].int(), colors, colors[:, 3] if colors is not None else None)

    def get_tetrahedra_tracer(self):
        device = self.tetrahedra_field.device
        if device.type != "cuda":
            raise RuntimeError("Tetrahedra tracer is only supported on a CUDA device")  # reference :396-397
        if self._tetrahedra_tracer is not None and self._tetrahedra_tracer.device != device:
            self._tetrahedra_tracer = self._fused = self._fused_versions = None
        xyz = self.tetrahedra_vertices.detach()
        if self._tetrahedra_tracer is not None and self.config.optimize_vertices:
            ptr, V, version = self._tracer_vertices
            if (xyz.data_ptr(), len(xyz)) != (ptr, V):  # another tensor: a fresh load
                self._tetrahedra_tracer.load_tetrahedra(xyz, self.tetrahedra_cells)
                self._keep_guard_start(xyz)
            elif self.tetrahedra_vertices._version != version:  # moved in place (an optimizer step): refit, same topology
                if self._guard_start is not None:  # vertex_fold_guard: scale the step back where it would fold the mesh
                    self._tetrahedra_tracer.guard_vertex_step(self._guard_start, xyz, VERTEX_FOLD_GUARD_MAX_HALVINGS)
                folded, _ = self._tetrahedra_tracer.update_vertices(xyz)
                if folded and not self._fold_warned:
                    warnings.warn(f"optimize_vertices: {folded} mesh faces are folded; tracing continues on the all-hits gather (exact, slower)")
                    self._fold_warned = True
                self._keep_guard_start(xyz)
            self._tracer_vertices = (xyz.data_ptr(), len(xyz), self.tetrahedra_vertices._version)
        if self._tetrahedra_tracer is None:
            if not self._tetrahedra_initialized:
                self._init_tetrahedra()
            xyz = self.tetrahedra_vertices.detach()
            self._tetrahedra_tracer = TetrahedraTracer(device)
            self._tetrahedra_tracer.load_tetrahedra(xyz, self.tetrahedra_cells)
            self._tracer_vertices = (xyz.data_ptr(), len(xyz), self.tetrahedra_vertices._version)
            self._keep_guard_start(xyz)
            self._fold_warned = False
        return self._tetrahedra_tracer

    def _keep_guard_start(self, xyz: torch.Tensor) -> None:
        """vertex_fold_guard: the positions the tracer now holds are where the next step starts from"""
        if not (self.config.optimize_vertices and self.config.vertex_fold_guard):
            return
        if self._guard_start is not None and self._guard_start.shape == xyz.shape and self._guard_start.device == xyz.device:
            self._guard_start.copy_(xyz)
        else:
            self._guard_start = xyz.clone()

    # ---- modules (reference :409-477) ----------------------------------------------------------------
    def populate_modules(self):
        super().populate_modules()
        in_dim = self.config.field_dim
        if self.config.input_fourier_frequencies > 0:
            self.position_encoding = NeRFEncoding(in_dim=in_dim, num_frequencies=self.config.input_fourier_frequencies, min_freq_exp=0.0,
                                                  max_freq_exp=float(self.config.input_fourier_frequencies), include_input=True)
            in_dim += self.position_encoding.get_out_dim()
        else:
            self.position_encoding = lambda x: x
        self.direction_encoding = NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0.0, max_freq_exp=4.0, include_input=True)
        self.mlp_base = MLP(in_dim=in_dim, num_layers=self.config.num_density_layers, layer_width=self.config.hidden_size, out_activation=nn.ReLU())
        head_in = self.mlp_base.get_out_dim() + self.direction_encoding.get_out_dim()
        if self.config.appearance_embed_dim > 0:  # reference :440-446
            self.appearance_embedding = nn.Embedding(self.num_train_data, self.config.appearance_embed_dim)
            head_in += self.config.appearance_embed_dim
        self.mlp_head = MLP(in_dim=head_in, num_layers=self.config.num_color_layers, layer_width=self.config.hidden_size, out_activation=nn.ReLU())
        self.field_output_color = RGBFieldHead(in_dim=self.mlp_head.get_out_dim())
        self.field_output_density = DensityFieldHead(in_dim=self.mlp_base.get_out_dim())
        if self.config.use_biased_sampler:
            self.sampler_uniform = TetrahedraSampler(num_samples=self.config.num_samples)
        else:
            self.sampler_uniform = UniformSampler(num_samples=self.config.num_samples)
        if self.config.num_fine_samples > 0:
            self.sampler_pdf = PDFSampler(num_samples=self.config.num_fine_samples)
        self.renderer_rgb = RGBRenderer(background_color=self.config.background_color)
        self.renderer_accumulation = AccumulationRenderer()
        self.renderer_depth = DepthRenderer()
        self.renderer_expected_depth = DepthRenderer(method="expected")
        self.rgb_loss = MSELoss()
        if self.config.vertex_fold_guard and not self.config.optimize_vertices:
            raise RuntimeError("vertex_fold_guard guards the steps of the vertex positions: it needs optimize_vertices=True")
        if self.config.coarsen_every > 0:
            if not self.config.use_occupancy_field:
                raise RuntimeError("coarsen_every > 0 removes vertices in empty space as the occupancy field sees it: it needs use_occupancy_field=True")
            if self._fused_unsupported():
                raise RuntimeError(f"coarsen_every > 0 reads the occupancy field of the fused CUDA pipeline, which does not support "
                                   f"{', '.join(self._fused_unsupported())}")
        H = self.config.background_envmap_height
        if H > 0:
            if self.config.background_color not in ("white", "black"):
                raise RuntimeError(f"background_envmap_height > 0 starts the map at background_color, which must be 'white' or 'black', "
                                   f"got {self.config.background_color!r}")
            init = 1.0 if self.config.background_color == "white" else 0.0
            self.register_parameter("background_envmap", nn.Parameter(torch.full((H, 2 * H, 3), init, dtype=torch.float32)))

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        if not self.config.optimize_vertices:
            return {"fields": list(self.parameters())}
        return {"fields": [p for n, p in self.named_parameters() if n != "tetrahedra_vertices"], "vertices": [self.tetrahedra_vertices]}

    def get_background_color(self, shape, device):
        return self.renderer_rgb.get_background_color(self.renderer_rgb.background_color, shape, device)

    # ---- fused inference path ---------------------------------------------------------------------------
    def _fused_unsupported(self) -> List[str]:
        """the config options, as `name=value`, that keep this model off the fused CUDA pipeline"""
        c = self.config
        want = {"field_dim": (64,), "hidden_size": (128,), "num_density_layers": (3,), "num_color_layers": (1,), "input_fourier_frequencies": (0,),
                "appearance_embed_dim": (0,), "background_color": ("white", "black")}
        return [f"{k}={getattr(c, k)!r}" for k, ok in want.items() if getattr(c, k) not in ok]

    def _fused_supported(self) -> bool:
        return not self._fused_unsupported()

    def _fused_renderer(self):
        from ..b200.render import FusedRenderer

        tracer = self.get_tetrahedra_tracer()
        if self._fused is None:
            self._fused = FusedRenderer(tracer)
        names = ["mlp_base.layers.0", "mlp_base.layers.1", "mlp_base.layers.2", "mlp_head.layers.0", "field_output_color.net", "field_output_density.net"]
        mods = [self.mlp_base.layers[0], self.mlp_base.layers[1], self.mlp_base.layers[2], self.mlp_head.layers[0], self.field_output_color.net,
                self.field_output_density.net]
        versions = (self.tetrahedra_field._version, self.tetrahedra_field.data_ptr()) + tuple(p._version for m in mods for p in (m.weight, m.bias))
        if versions != self._fused_versions:  # refresh the [V,64] shadow / packed weights only when a parameter changed
            self._fused.set_field(self.tetrahedra_field.detach().contiguous())
            self._fused.set_weights({f"{n}.{k}": getattr(m, k) for n, m in zip(names, mods) for k in ("weight", "bias")})
            self._fused_versions = versions
        return self._fused

    def _apply_occupancy(self, fr, training: bool) -> None:
        """sets (or clears) the culling of the fused renderer `fr` for the next call.  Training: no culling before
        occupancy_warmup_steps, then an update every occupancy_update_interval steps, at the start of the step (so after the previous
        optimizer step, as the vertex refit).  A buffer that was never computed (all zeros) is recomputed with decay 0 first."""
        c = self.config
        if not c.use_occupancy_field:
            fr.set_occupancy(None)
            return
        occ = self.tetrahedra_occupancy
        step = self._occ_step
        if training:
            self._occ_step += 1
            if step < c.occupancy_warmup_steps:
                fr.set_occupancy(None)
                return
        fresh = False
        if not self._occ_ready:
            if not bool(occ.any()):
                fr.update_occupancy(occ, 0.0)
                fresh = True
            self._occ_ready = True
        if training and not fresh and (step - c.occupancy_warmup_steps) % max(1, c.occupancy_update_interval) == 0:
            fr.update_occupancy(occ, c.occupancy_decay)
        if c.occupancy_sampling:
            fr.set_occupancy(occ, c.occupancy_threshold, place_samples=True)
        else:
            fr.set_occupancy(occ, c.occupancy_threshold)

    def _apply_background(self, fr) -> None:
        """points the fused renderer `fr` at background_envmap, or at the constant background when it is off.  The renderer is set again
        only when the map's storage changed, so a training forward's backward stays valid across other renders"""
        m = self.background_envmap.detach() if self.config.background_envmap_height > 0 else None
        cur = fr._bg
        if m is None:
            if cur is not None:
                fr.set_background(None)
        elif cur is None or cur.data_ptr() != m.data_ptr() or cur.shape != m.shape:
            fr.set_background(m)

    # ---- forward (reference :520-662) ---------------------------------------------------------------------
    def _expected_depth_on(self) -> bool:
        return self.config.render_expected_depth or self.config.depth_loss_mult > 0

    def _distortion_on(self) -> bool:
        return self.config.distortion_loss_mult > 0 and self.training

    def get_outputs(self, ray_bundle: RayBundle):
        outputs = self._get_outputs(ray_bundle)
        # the z-depth target's conversion to a distance along the ray, for get_loss_dict only: in training, and in nerfstudio's eval
        # loss (get_eval_loss_dict renders in eval mode and calls get_loss_dict too)
        if self.config.depth_loss_mult > 0 and not self.config.is_euclidean_depth:
            dn = (getattr(ray_bundle, "metadata", None) or {}).get("directions_norm")
            if dn is not None:
                outputs["directions_norm"] = dn
        return outputs

    def _get_outputs(self, ray_bundle: RayBundle):
        assert self.collider is not None
        origins, directions = ray_bundle.origins.contiguous(), ray_bundle.directions.contiguous()
        normals = self.config.render_normals and not self.training
        if self.config.occupancy_sampling and not self.config.use_occupancy_field:
            raise RuntimeError("occupancy_sampling places the samples by the occupancy field: it needs use_occupancy_field=True")
        if self.config.use_occupancy_field and self._fused_unsupported():
            raise RuntimeError(f"use_occupancy_field culls on the fused CUDA pipeline, which does not support {', '.join(self._fused_unsupported())}")
        if normals and self._fused_unsupported():
            raise RuntimeError(f"render_normals runs on the fused CUDA pipeline, which does not support {', '.join(self._fused_unsupported())}")
        if normals or (not self.training and not torch.is_grad_enabled() and self._fused_supported()):
            from ..b200.render import RenderSettings

            bg = (1.0, 1.0, 1.0) if self.config.background_color == "white" else (0.0, 0.0, 0.0)
            st = RenderSettings(self.config.max_intersected_triangles, self.config.num_samples, self.config.num_fine_samples,
                                self.config.use_biased_sampler, float(self.collider.far_plane), bg)
            with torch.no_grad():
                fr = self._fused_renderer()
                self._apply_occupancy(fr, training=False)
                self._apply_background(fr)
                return fr.render(origins, directions, st, normals=normals, expected_depth=self._expected_depth_on())
        unfused_train = os.environ.get("TETRANERF_B200_UNFUSED_TRAIN", "0") == "1"
        if self.training and torch.is_grad_enabled() and self.config.optimize_vertices:
            causes = self._fused_unsupported() + (["num_fine_samples=0"] if self.config.num_fine_samples == 0 else []) \
                + (["TETRANERF_B200_UNFUSED_TRAIN=1"] if unfused_train else [])
            if causes:
                raise RuntimeError(f"optimize_vertices trains on the fused CUDA pipeline, which does not support {', '.join(causes)}")
        if self.training and torch.is_grad_enabled() and self._fused_supported() and self.config.num_fine_samples > 0 and not unfused_train:
            return self._get_outputs_fused_train(origins, directions)
        return self._get_outputs_unfused(ray_bundle, origins, directions)

    def _get_outputs_fused_train(self, origins, directions):
        """training step on the fused CUDA pipeline: ONE differentiable op (forward + wgmma backward) instead of the reference's op
        sequence; the stratified draws are the same two torch.rand calls the reference makes (model.py:169-174, PDFSampler)."""
        from ..b200.render import PARAM_ORDER, FusedTrainRender, FusedTrainRenderDepth, FusedTrainRenderDistortion, RenderSettings

        c = self.config
        bg = (1.0, 1.0, 1.0) if c.background_color == "white" else (0.0, 0.0, 0.0)
        st = RenderSettings(c.max_intersected_triangles, c.num_samples, c.num_fine_samples, c.use_biased_sampler, float(self.collider.far_plane), bg)
        fr = self._fused_renderer()
        with torch.no_grad():
            self._apply_occupancy(fr, training=True)
        self._apply_background(fr)
        R, dev = origins.shape[0], origins.device
        jc = torch.rand((R, c.num_samples + 1), dtype=torch.float32, device=dev) if getattr(self.sampler_uniform, "train_stratified", True) else None
        jf = torch.rand((R, c.num_fine_samples + 1), dtype=torch.float32, device=dev) if getattr(self.sampler_pdf, "train_stratified", True) else None
        named = dict(self.named_parameters())
        xyz = (self.tetrahedra_vertices,) if c.optimize_vertices else ()  # the tensor the tracer borrowed (get_tetrahedra_tracer)
        bg = (self.background_envmap,) if c.background_envmap_height > 0 else ()  # the tensor the renderer holds (_apply_background)
        args = (fr, st, c.use_gradient_scaling, origins, directions, jc, jf, self.tetrahedra_field, *[named[n] for n in PARAM_ORDER], *xyz, *bg)
        if self._distortion_on():
            res = FusedTrainRenderDistortion.apply(*args[:3], self._expected_depth_on(), *args[3:])
            keys = ["rgb", "accumulation", "depth"] + (["expected_depth"] if self._expected_depth_on() else []) + ["distortion", "ray_mask"]
            return dict(zip(keys, res))
        if self._expected_depth_on():
            rgb, acc, depth, ed, mask = FusedTrainRenderDepth.apply(*args)
            return {"rgb": rgb, "accumulation": acc, "depth": depth, "expected_depth": ed, "ray_mask": mask}
        rgb, acc, depth, mask = FusedTrainRender.apply(*args)
        return {"rgb": rgb, "accumulation": acc, "depth": depth, "ray_mask": mask}

    def _field_at(self, tracer, traced, ray_mask, distances):
        matched = tracer.find_visited_cells(traced["num_visited_cells"][ray_mask], traced["visited_cells"][ray_mask],
                                            traced["barycentric_coordinates"][ray_mask], traced["hit_distances"][ray_mask],
                                            traced["vertex_indices"][ray_mask], distances.squeeze(-1).contiguous())
        return interpolate_values(matched["vertex_indices"], matched["barycentric_coordinates"], self.tetrahedra_field)

    def _get_outputs_unfused(self, ray_bundle, origins, directions):
        tracer = self.get_tetrahedra_tracer()
        traced = tracer.trace_rays(origins, directions, self.config.max_intersected_triangles)
        count = traced["num_visited_cells"]
        nears = traced["hit_distances"][:, 0, 0][:, None]
        fars = torch.gather(traced["hit_distances"][:, :, 1], 1, (count[:, None].long() - 1).clamp_min(0))
        ray_mask = count > 0
        device = ray_mask.device
        R = ray_mask.shape[0]
        envmap = self.config.background_envmap_height > 0
        if envmap:  # bg(d) on every ray (the torch restatement of the fused lookup), clamped in eval mode as every pixel
            from ..b200.render import background_lookup

            bg = background_lookup(self.background_envmap, directions)
            rgb = bg if self.training else bg.clamp(0.0, 1.0)
        else:
            rgb = self.get_background_color((R, 3), device=device)
        accumulation = torch.zeros((R, 1), dtype=torch.float32, device=device)
        depth = torch.full((R, 1), self.collider.far_plane, dtype=torch.float32, device=device)
        outputs = {"rgb": rgb, "accumulation": accumulation, "depth": depth, "ray_mask": ray_mask}
        if self._expected_depth_on():
            outputs["expected_depth"] = depth.clone()
        if self._distortion_on():
            outputs["distortion"] = torch.zeros((R, 1), dtype=torch.float32, device=device)
        if bool(ray_mask.any()):
            bundle = dataclasses.replace(ray_bundle[ray_mask], nears=nears[ray_mask], fars=fars[ray_mask])
            if isinstance(self.sampler_uniform, TetrahedraSampler):
                samples = self.sampler_uniform(bundle, num_visited_cells=count[ray_mask], hit_distances=traced["hit_distances"][ray_mask])
            else:
                samples = self.sampler_uniform(bundle)
            features = self._field_at(tracer, traced, ray_mask, (samples.frustums.ends + samples.frustums.starts) / 2)
            if self.config.num_fine_samples > 0:
                coarse_density = self.field_output_density(self.mlp_base(self.position_encoding(features)))
                samples = self.sampler_pdf(bundle, samples, samples.get_weights(coarse_density))
                features = self._field_at(tracer, traced, ray_mask, (samples.frustums.ends + samples.frustums.starts) / 2)
            base = self.mlp_base(self.position_encoding(features))
            sigmas = self.field_output_density(base)
            head_in = [self.direction_encoding(samples.frustums.directions), base]
            if self.config.appearance_embed_dim > 0:  # reference :608-620
                if self.training:
                    assert samples.camera_indices is not None
                    head_in.append(self.appearance_embedding(samples.camera_indices.squeeze()))
                else:
                    head_in.append(torch.ones((*base.shape[:-1], self.config.appearance_embed_dim), device=base.device) * self.appearance_embedding.weight.mean(dim=0))
            colors = self.field_output_color(self.mlp_head(torch.cat(head_in, dim=-1)))
            if self.config.use_gradient_scaling:
                colors, sigmas, _ = GradientScaler.apply(colors, sigmas, samples.spacing_ends + samples.spacing_starts)
            weights = samples.get_weights(sigmas)
            if envmap:  # RGBRenderer over the per-ray background
                if not self.training:
                    colors = torch.nan_to_num(colors)
                comp = torch.sum(weights * colors, dim=-2) + bg[ray_mask] * (1.0 - torch.sum(weights, dim=-2))
                rgb = rgb.clone()
                rgb[ray_mask] = comp if self.training else comp.clamp(0.0, 1.0)
                outputs["rgb"] = rgb
            else:
                rgb[ray_mask] = self.renderer_rgb(rgb=colors, weights=weights)
            accumulation[ray_mask] = self.renderer_accumulation(weights)
            depth[ray_mask] = self.renderer_depth(weights, samples)
            if self._expected_depth_on():
                outputs["expected_depth"][ray_mask] = self.renderer_expected_depth(weights, samples)
            if self._distortion_on():  # over the spacing bins of the samples that give rgb (nerfstudio's ray_samples_to_sdist)
                sdist = torch.cat((samples.spacing_starts[..., 0], samples.spacing_ends[..., -1:, 0]), -1)
                outputs["distortion"][ray_mask] = distortion_per_ray(weights, sdist)
        return outputs

    # ---- mesh refinement (DESIGN §4.14) ------------------------------------------------------------------------------------------------
    def get_training_callbacks(self, training_callback_attributes: TrainingCallbackAttributes) -> List[TrainingCallback]:
        """with refine_every > 0: after every training iteration, the field-gradient statistics; every refine_every steps in
        [refine_start, refine_stop), `refine` with the trainer's optimizers.  With coarsen_every > 0: every coarsen_every steps in
        [coarsen_start, coarsen_stop), `coarsen` with them, after the statistics and before a refinement of the same step.  With
        delaunay_flip_every > 0: every delaunay_flip_every steps, `flip_delaunay`, after all of those.  None otherwise"""
        c = self.config
        if c.refine_every <= 0 and c.coarsen_every <= 0 and c.delaunay_flip_every <= 0:
            return []
        optimizers = training_callback_attributes.optimizers

        def refine(step: int):
            if c.refine_start <= step < c.refine_stop and step % c.refine_every == 0:
                self.refine(optimizers)

        def coarsen(step: int):
            if c.coarsen_start <= step < c.coarsen_stop and step % c.coarsen_every == 0:
                self.coarsen(optimizers)

        def flip(step: int):
            if step > 0 and step % c.delaunay_flip_every == 0:
                self.flip_delaunay(optimizers)

        after = [TrainingCallbackLocation.AFTER_TRAIN_ITERATION]
        cbs = [TrainingCallback(after, lambda step: self.accumulate_refine_statistics())] if c.refine_every > 0 else []
        if c.coarsen_every > 0:
            cbs.append(TrainingCallback(after, coarsen))
        if c.refine_every > 0:
            cbs.append(TrainingCallback(after, refine))
        if c.delaunay_flip_every > 0:
            cbs.append(TrainingCallback(after, flip))
        return cbs

    def accumulate_refine_statistics(self) -> None:
        """acc_v += ||dL/dF[:, v]||_2 and cnt_v += 1 where that column is non-zero, from the field gradient of the step that just ran
        (before it is zeroed; under DDP the all-reduced one, so every rank decides alike).  No gradient: nothing happens"""
        g = self.tetrahedra_field.grad
        if g is None:
            return
        with torch.no_grad():
            norm = torch.linalg.vector_norm(g, dim=0)
            if self._grad_acc is None or self._grad_acc.shape != norm.shape or self._grad_acc.device != norm.device:
                self._grad_acc = torch.zeros_like(norm)
                self._grad_cnt = torch.zeros(norm.shape, dtype=torch.int32, device=norm.device)
            self._grad_acc += norm
            self._grad_cnt += (norm > 0).to(torch.int32)

    def refine(self, optimizers=None) -> Dict[str, Any]:
        """bisects the longest edges of the tetrahedra whose field gradient stayed large since the last call: up to refine_passes
        passes of `tetranerf.b200.refine.refine_edges` over the refine_fraction highest-scoring tetrahedra (score: the mean over its
        vertices of acc_v / max(cnt_v, 1)), stopping at refine_max_vertices.  The field, the positions, the occupancy and, in
        `optimizers` (nerfstudio's Optimizers, a dict of torch optimizers or one optimizer), every per-vertex state tensor of the field
        and vertex parameters (RAdam's exp_avg / exp_avg_sq; `step` is kept) are carried over: new vertices take their edge's
        endpoint average, new tetrahedra their parent's occupancy.  The Parameter objects stay the same; their .grad is cleared.  The
        tracer is reloaded and the statistics reset.  -> counts before / after, per-pass proposals and acceptances, seconds taken"""
        import time

        from ..b200 import refine as rf

        c = self.config
        t0 = time.perf_counter()
        V0, T0 = len(self.tetrahedra_vertices), len(self.tetrahedra_cells)
        res: Dict[str, Any] = {"vertices_before": V0, "tetrahedra_before": T0, "passes": []}
        field = self.tetrahedra_field
        dev = field.device
        if self._grad_acc is not None and len(self._grad_acc) == V0:
            score = self._grad_acc / self._grad_cnt.clamp_min(1).to(self._grad_acc.dtype)
        else:
            score = torch.zeros((V0,), dtype=torch.float32, device=dev)
        with torch.no_grad():
            xyz, cells = self.tetrahedra_vertices.detach(), self.tetrahedra_cells
            cand = rf.select_candidates(score.to(dev), cells, c.refine_fraction)
            parent_edges, parent_cells = [], []
            for _ in range(max(0, c.refine_passes)):
                room = None if c.refine_max_vertices is None else c.refine_max_vertices - len(xyz)
                if (room is not None and room <= 0) or not bool(cand.any()):
                    break
                out = rf.refine_edges(xyz, cells, cand, c.refine_min_edge_length, room)
                res["passes"].append({"proposed": out["n_proposed"], "accepted": out["n_accepted"], "split": out["n_split"]})
                if out["n_accepted"] == 0:
                    break
                T = len(cells)
                split = torch.zeros((T,), dtype=torch.bool, device=dev)
                split[out["parent_cell"][T:].long()] = True
                cand = torch.cat((cand & ~split, torch.zeros((out["n_split"],), dtype=torch.bool, device=dev)))
                xyz, cells = rf.migrate_vertices(xyz, out["parent_edge"], 0), out["cells"]
                parent_edges.append(out["parent_edge"])
                parent_cells.append(out["parent_cell"])
            if parent_edges:
                self._apply_refinement(parent_edges, parent_cells, xyz, cells, optimizers)
                if c.delaunay_flip_every > 0:
                    res["flip"] = self.flip_delaunay(optimizers)
        res["vertices_after"], res["tetrahedra_after"] = len(self.tetrahedra_vertices), len(self.tetrahedra_cells)
        self._grad_acc = self._grad_cnt = None
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        res["seconds"] = time.perf_counter() - t0
        return res

    def _apply_refinement(self, parent_edges, parent_cells, xyz, cells, optimizers) -> None:
        """installs the refined mesh (xyz, cells) after the passes given by their parent_edge / parent_cell tables"""
        from ..b200 import refine as rf

        def per_vertex(t, dim):
            for pe in parent_edges:
                t = rf.migrate_vertices(t, pe, dim)
            return t

        params = [(self.tetrahedra_field, 1)] + ([(self.tetrahedra_vertices, 0)] if self.config.optimize_vertices else [])
        opts = getattr(optimizers, "optimizers", optimizers)
        opts = list(opts.values()) if isinstance(opts, dict) else ([] if opts is None else [opts])
        for p, dim in params:
            old_shape = p.shape
            for opt in opts:
                st = opt.state.get(p)
                for k, v in (st or {}).items():
                    if isinstance(v, torch.Tensor) and v.shape == old_shape:  # exp_avg, exp_avg_sq (not the scalar step)
                        st[k] = per_vertex(v, dim)
        _set_data(self.tetrahedra_field, per_vertex(self.tetrahedra_field.data, 1))
        self.tetrahedra_field.grad = None
        _set_data(self.tetrahedra_vertices, xyz)
        self.tetrahedra_vertices.grad = None
        if self.config.use_occupancy_field:
            occ = self.tetrahedra_occupancy.data
            for pc in parent_cells:
                occ = rf.migrate_cells(occ, pc)
            self.tetrahedra_occupancy.data = occ
        self.tetrahedra_cells.data = cells.contiguous()
        self.config.num_tetrahedra_vertices, self.config.num_tetrahedra_cells = len(xyz), len(cells)
        if self._tetrahedra_tracer is not None:
            self._tetrahedra_tracer.load_tetrahedra(self.tetrahedra_vertices.detach(), self.tetrahedra_cells)
            self._tracer_vertices = (self.tetrahedra_vertices.data_ptr(), len(xyz), self.tetrahedra_vertices._version)
            self._keep_guard_start(self.tetrahedra_vertices.detach())

    # ---- mesh coarsening (DESIGN §4.18) --------------------------------------------------------------------------------------------------
    def coarsen_ready(self) -> bool:
        """the occupancy buffer describes the field: training has passed occupancy_warmup_steps and the buffer was computed (an all-zero
        buffer would mark every tetrahedron empty)"""
        c = self.config
        return (c.use_occupancy_field and self._occ_ready and self._occ_step > c.occupancy_warmup_steps
                and bool(self.tetrahedra_occupancy.any()))

    def coarsen(self, optimizers=None) -> Dict[str, Any]:
        """removes vertices in empty space: up to coarsen_passes passes of `tetranerf.b200.coarsen.coarsen_vertices`, a tetrahedron
        being empty when its tetrahedra_occupancy is below occupancy_threshold.  Nothing happens until `coarsen_ready()`.  The field, the
        positions, the occupancy (each tetrahedron keeps its parent's), the refinement statistics and, in `optimizers` (as `refine`),
        every per-vertex state tensor of the field and vertex parameters (`step` is kept) keep the entries of the surviving vertices.
        The Parameter objects stay the same; their .grad is cleared; the tracer is reloaded.  -> counts before / after, per-pass
        proposals and removals, seconds taken ("ready": False when nothing could run), and over all the passes "kept_vertex" / "parent_cell"
        (the old index of each new vertex / tetrahedron; None when nothing was removed), to carry other per-vertex or per-tetrahedron
        tensors over.  With delaunay_flip_every > 0 the coarsened mesh is then flipped ("flip": flip_delaunay's result); "parent_cell"
        describes the coarsened tetrahedra before that flip, and the installed ones only when "flip" made no change"""
        import time

        from ..b200 import coarsen as cv
        from ..b200 import refine as rf

        c = self.config
        if not c.use_occupancy_field:
            raise RuntimeError("coarsen removes vertices in empty space as the occupancy field sees it: it needs use_occupancy_field=True")
        t0 = time.perf_counter()
        V0, T0 = len(self.tetrahedra_vertices), len(self.tetrahedra_cells)
        res: Dict[str, Any] = {"vertices_before": V0, "tetrahedra_before": T0, "passes": [], "ready": self.coarsen_ready()}
        dev = self.tetrahedra_field.device
        if res["ready"]:
            with torch.no_grad():
                xyz, cells, occ = self.tetrahedra_vertices.detach(), self.tetrahedra_cells, self.tetrahedra_occupancy
                kept = parent = None
                for _ in range(max(0, c.coarsen_passes)):
                    out = cv.coarsen_vertices(xyz, cells, occ < c.occupancy_threshold)
                    res["passes"].append({"proposed": out["n_proposed"], "removed": out["n_removed"], "cells_removed": out["n_cells_removed"]})
                    if out["n_removed"] == 0:
                        break
                    k, p = out["kept_vertex"].long(), out["parent_cell"].long()
                    kept, parent = (k, p) if kept is None else (kept[k], parent[p])
                    xyz, cells, occ = cv.compact_vertices(xyz, k, 0), out["cells"], rf.migrate_cells(occ, p)
                if kept is not None:
                    self._apply_coarsening(kept, parent, xyz, cells, optimizers)
                    if c.delaunay_flip_every > 0:
                        res["flip"] = self.flip_delaunay(optimizers)
                res["kept_vertex"], res["parent_cell"] = kept, parent
        res["vertices_after"], res["tetrahedra_after"] = len(self.tetrahedra_vertices), len(self.tetrahedra_cells)
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        res["seconds"] = time.perf_counter() - t0
        return res

    def _apply_coarsening(self, kept_vertex, parent_cell, xyz, cells, optimizers) -> None:
        """installs the coarsened mesh (xyz, cells): kept_vertex / parent_cell give the old vertex of each new one and the old tetrahedron
        of each new one over all the passes"""
        from ..b200 import coarsen as cv
        from ..b200 import refine as rf

        params = [(self.tetrahedra_field, 1)] + ([(self.tetrahedra_vertices, 0)] if self.config.optimize_vertices else [])
        opts = getattr(optimizers, "optimizers", optimizers)
        opts = list(opts.values()) if isinstance(opts, dict) else ([] if opts is None else [opts])
        for p, dim in params:
            old_shape = p.shape
            for opt in opts:
                st = opt.state.get(p)
                for k, v in (st or {}).items():
                    if isinstance(v, torch.Tensor) and v.shape == old_shape:  # exp_avg, exp_avg_sq (not the scalar step)
                        st[k] = cv.compact_vertices(v, kept_vertex, dim)
        V0 = len(self.tetrahedra_vertices)
        _set_data(self.tetrahedra_field, cv.compact_vertices(self.tetrahedra_field.data, kept_vertex, 1))
        self.tetrahedra_field.grad = None
        _set_data(self.tetrahedra_vertices, xyz)
        self.tetrahedra_vertices.grad = None
        self.tetrahedra_occupancy.data = rf.migrate_cells(self.tetrahedra_occupancy.data, parent_cell)
        self.tetrahedra_cells.data = cells.contiguous()
        if self._grad_acc is not None and len(self._grad_acc) == V0:
            self._grad_acc = cv.compact_vertices(self._grad_acc, kept_vertex, 0)
            self._grad_cnt = cv.compact_vertices(self._grad_cnt, kept_vertex, 0)
        self.config.num_tetrahedra_vertices, self.config.num_tetrahedra_cells = len(xyz), len(cells)
        if self._tetrahedra_tracer is not None:
            self._tetrahedra_tracer.load_tetrahedra(self.tetrahedra_vertices.detach(), self.tetrahedra_cells)
            self._tracer_vertices = (self.tetrahedra_vertices.data_ptr(), len(xyz), self.tetrahedra_vertices._version)
            self._keep_guard_start(self.tetrahedra_vertices.detach())

    # ---- Delaunay flips (DESIGN §4.19) ---------------------------------------------------------------------------------------------------
    def flip_delaunay(self, optimizers=None) -> Dict[str, Any]:
        """flips the mesh towards Delaunay: passes of `tetranerf.b200.flip.flip_delaunay` until one proposes nothing, at most
        delaunay_flip_max_passes.  Only the tetrahedra change: the occupancy of each new one is the maximum over the ones its region came
        from, the tracer is reloaded and the fold guard restarts from the current positions; the positions, the field, the optimizer state
        (`optimizers` is accepted for the callbacks' sake and left alone) and the refinement statistics are untouched.  When the first
        pass proposes nothing, nothing is installed.  With optimize_vertices, a vertex step the tracer has not refit yet (an optimizer
        step since the last forward) first goes through the refit and, with vertex_fold_guard, its guard, so the flips see the positions
        the next forward would trace and the guard's start is never skipped.  -> counts before / after, per-pass counts (illegal faces,
        proposals, 2-3 and 3-2 flips), "illegal_left" (faces still certified illegal at the end: stuck ones that no flip of the definition
        removes, or not yet reached when the pass limit stopped the loop) and the seconds taken"""
        import time

        from ..b200 import flip as fl

        c = self.config
        t0 = time.perf_counter()
        T0 = len(self.tetrahedra_cells)
        res: Dict[str, Any] = {"tetrahedra_before": T0, "passes": []}
        dev = self.tetrahedra_field.device
        if self._tetrahedra_tracer is not None and c.optimize_vertices:
            self.get_tetrahedra_tracer()  # guard and refit a pending vertex step before flipping on its positions
        with torch.no_grad():
            xyz, cells = self.tetrahedra_vertices.detach().contiguous(), self.tetrahedra_cells
            occ = self.tetrahedra_occupancy.data if c.use_occupancy_field else None
            changed = False
            left = None
            for _ in range(max(0, c.delaunay_flip_max_passes)):
                out = fl.flip_delaunay(xyz, cells)
                res["passes"].append({"illegal": out["n_illegal"], "proposed": out["n_proposed"], "flips_23": out["n_23"], "flips_32": out["n_32"]})
                if out["n_proposed"] == 0:
                    left = out["n_illegal"]
                    break
                changed = True
                cells = out["cells"]
                if occ is not None:
                    occ = fl.migrate_cells_max(occ, out["sources"])
            if left is None and changed:  # stopped by the pass limit: count what is left without flipping
                left = fl.flip_delaunay(xyz, cells, max_flips=0)["n_illegal"]
            if changed:
                self._apply_flips(cells, occ)
        res["illegal_left"] = left if left is not None else 0
        res["tetrahedra_after"] = len(self.tetrahedra_cells)
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        res["seconds"] = time.perf_counter() - t0
        return res

    def _apply_flips(self, cells, occupancy=None) -> None:
        """installs the flipped cells over the same vertices, with the migrated occupancy (None: without the occupancy field)"""
        if occupancy is not None:
            self.tetrahedra_occupancy.data = occupancy
        self.tetrahedra_cells.data = cells.contiguous()
        self.config.num_tetrahedra_cells = len(cells)
        if self._tetrahedra_tracer is not None:
            self._tetrahedra_tracer.load_tetrahedra(self.tetrahedra_vertices.detach(), self.tetrahedra_cells)
            self._tracer_vertices = (self.tetrahedra_vertices.data_ptr(), len(self.tetrahedra_vertices), self.tetrahedra_vertices._version)
            self._keep_guard_start(self.tetrahedra_vertices.detach())

    # ---- geometry export -----------------------------------------------------------------------------------------------------------------
    def extract_surface(self, level: float) -> Dict[str, torch.Tensor]:
        """the density iso-surface sigma = level of the trained field as a triangle mesh, by marching tetrahedra on the model's own
        tetrahedra (FusedRenderer.extract_surface): device tensors `vertices`, `normals`, `colors` f32[N,3], `faces` i32[F,3],
        `face_tetrahedra` i32[F], in the model's (nerfstudio) frame, the one the renders use.  `tetranerf.b200.surface.write_ply` writes
        it out.  Needs the fused pipeline: raises RuntimeError naming the options that rule it out."""
        bad = self._fused_unsupported()
        if bad:
            raise RuntimeError(f"extract_surface runs on the fused CUDA pipeline, which does not support {', '.join(bad)}")
        with torch.no_grad():
            return self._fused_renderer().extract_surface(level)

    def get_loss_dict(self, outputs, batch, metrics_dict=None) -> Dict[str, torch.Tensor]:
        image = batch["image"].to(outputs["rgb"].device)
        losses = {"rgb_loss": self.rgb_loss(image, outputs["rgb"])}
        if self.config.depth_loss_mult > 0:
            losses["depth_loss"] = self.config.depth_loss_mult * self._depth_loss(outputs, batch)
        if self._distortion_on():  # mean over the rays with hits (empty rays hold 0)
            n = outputs["ray_mask"].sum().clamp_min(1)
            losses["distortion_loss"] = self.config.distortion_loss_mult * outputs["distortion"].sum() / n
        if self.config.field_smoothness_mult > 0 and self.training:
            losses["field_smoothness_loss"] = self._field_smoothness_loss()
        return scale_dict(losses, self.config.loss_coefficients)

    def _field_smoothness_loss(self) -> torch.Tensor:
        """field_smoothness_mult * S / (E * 64) on the current field and mesh (FieldSmoothness), differentiable to tetrahedra_field"""
        bad = self._fused_unsupported()
        if bad:
            raise RuntimeError(f"field_smoothness_mult runs on the fused CUDA pipeline, which does not support {', '.join(bad)}")
        from ..b200.render import FieldSmoothness

        fr = self._fused_renderer()  # refreshes the field shadow the kernel reads, whichever path rendered the step
        return FieldSmoothness.apply(fr, self.config.field_smoothness_mult, self.tetrahedra_field)

    def _depth_loss(self, outputs, batch) -> torch.Tensor:
        """mean over rays with hits and a finite target > 0 of (expected_depth - target)^2; the target batch["depth_image"] [R,1] is a
        distance along the ray (is_euclidean_depth) or a z-depth, converted with outputs["directions_norm"]"""
        ed = outputs["expected_depth"]
        target = batch["depth_image"].to(ed.device).reshape(ed.shape).to(ed.dtype)
        if not self.config.is_euclidean_depth:
            if "directions_norm" not in outputs:
                raise RuntimeError("depth_loss_mult > 0 with a z-depth target (is_euclidean_depth=False) needs the ray bundle's "
                                   'metadata["directions_norm"] to turn z-depth into a distance along the ray')
            target = target * outputs["directions_norm"].to(ed.device).reshape(ed.shape)
        valid = outputs["ray_mask"].reshape(-1, 1) & torch.isfinite(target) & (target > 0)
        sq = torch.where(valid, ed - torch.where(valid, target, torch.zeros_like(target)), torch.zeros_like(ed)) ** 2
        return sq.sum() / valid.sum().clamp_min(1)

    # ---- evaluation images and metrics (reference :676-713) --------------------------------------------------------------------------
    def get_image_metrics_and_images(self, outputs: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor]):
        image = batch["image"].to(outputs["rgb"].device)
        rgb = outputs["rgb"]
        acc = _apply_colormap(outputs["accumulation"])
        depth = _apply_depth_colormap(outputs["depth"], accumulation=outputs["accumulation"])
        images = {"img": torch.cat([image, rgb], dim=1), "accumulation": torch.cat([acc], dim=1), "depth": torch.cat([depth], dim=1)}
        if "expected_depth" in outputs:
            images["expected_depth"] = _apply_depth_colormap(outputs["expected_depth"], accumulation=outputs["accumulation"])
        if "normals" in outputs:  # unit normals in [-1, 1] shown as colours in [0, 1]
            images["normals"] = (outputs["normals"] + 1.0) / 2.0
        # [H, W, C] -> [1, C, H, W]
        im, pr = torch.moveaxis(image, -1, 0)[None, ...], torch.moveaxis(rgb, -1, 0)[None, ...]
        metrics = {"psnr": float(_psnr(im, pr)), "nerfstudio_ssim": float(_ssim(im, pr))}
        lp = _lpips(im, pr)
        if lp is not None:
            metrics["lpips"] = float(lp)
        return metrics, images


def _set_data(t: torch.Tensor, new: torch.Tensor) -> None:
    """t.data = new for a `new` of another shape.  Autograd caches a leaf's gradient accumulator, with the leaf's shape, for as long as
    a graph that reaches it is alive (the previous step's loss usually is), and `.data =` drops that cache only on a dtype or device
    change: so the data passes through an empty tensor of another dtype first, and the next graph gets an accumulator of the new shape"""
    t.data = torch.empty(0, dtype=torch.float64 if new.dtype != torch.float64 else torch.float32, device=new.device)
    t.data = new


def _psnr(a: torch.Tensor, b: torch.Tensor, data_range: float = 1.0) -> torch.Tensor:
    """torchmetrics PeakSignalNoiseRatio(data_range=1.0) (reference :470)"""
    mse = torch.mean((a - b) ** 2)
    return 10.0 * torch.log10(data_range**2 / mse)


def _ssim(a: torch.Tensor, b: torch.Tensor, data_range: float = 1.0, kernel: int = 11, sigma: float = 1.5, k1: float = 0.01, k2: float = 0.03) -> torch.Tensor:
    """torchmetrics.functional.structural_similarity_index_measure with its defaults (Gaussian 11x11, sigma 1.5), [N,C,H,W] in [0,1]"""
    c = a.shape[1]
    x = torch.arange(kernel, dtype=a.dtype, device=a.device) - (kernel - 1) / 2
    g = torch.exp(-(x**2) / (2 * sigma**2))
    g = (g / g.sum())[:, None] * (g / g.sum())[None, :]
    w = g.expand(c, 1, kernel, kernel).contiguous()
    pad = (kernel - 1) // 2
    ap, bp = (torch.nn.functional.pad(t, (pad, pad, pad, pad), mode="reflect") for t in (a, b))

    def f(t):
        return torch.nn.functional.conv2d(t, w, groups=c)

    mu_a, mu_b = f(ap), f(bp)
    s_aa, s_bb, s_ab = f(ap * ap) - mu_a**2, f(bp * bp) - mu_b**2, f(ap * bp) - mu_a * mu_b
    c1, c2 = (k1 * data_range) ** 2, (k2 * data_range) ** 2
    ssim = ((2 * mu_a * mu_b + c1) * (2 * s_ab + c2)) / ((mu_a**2 + mu_b**2 + c1) * (s_aa + s_bb + c2))
    return ssim.mean()


_LPIPS = None


def _lpips(a, b):
    """LearnedPerceptualImagePatchSimilarity (reference :474) when torchmetrics + its weights are available; None otherwise"""
    global _LPIPS
    if _LPIPS is False:
        return None
    try:
        if _LPIPS is None:
            from torchmetrics.image.lpip import LearnedPerceptualImagePatchSimilarity

            _LPIPS = LearnedPerceptualImagePatchSimilarity().to(a.device)
        return _LPIPS(a, b)
    except Exception:  # not installed / no pretrained weights offline
        _LPIPS = False
        return None


def _apply_colormap(x: torch.Tensor) -> torch.Tensor:
    try:
        from nerfstudio.utils import colormaps

        return colormaps.apply_colormap(x)
    except ImportError:
        return torch.nan_to_num(x, 0.0).clamp(0, 1).expand(*x.shape[:-1], 3)


def _apply_depth_colormap(depth: torch.Tensor, accumulation: Optional[torch.Tensor] = None) -> torch.Tensor:
    try:
        from nerfstudio.utils import colormaps

        return colormaps.apply_depth_colormap(depth, accumulation=accumulation)
    except ImportError:
        near, far = float(depth.min()), float(depth.max())
        d = ((depth - near) / (far - near + 1e-10)).clamp(0, 1)
        img = torch.nan_to_num(d, 0.0).expand(*d.shape[:-1], 3)
        return img * accumulation + (1 - accumulation) if accumulation is not None else img
