"""Minimal stand-ins for the nerfstudio (0.3.x) classes the Tetra-NeRF model touches on its hot path.

nerfstudio is an un-vendored dependency of the reference (setup.py:133) and is not installed in this
environment; `model.py` imports the real package when it is available and falls back to these look-alikes
otherwise, so that the drop-in `TetrahedraNerf` / `TetrahedraSampler` API can be exercised (tests, bench).
Only what model.py imports is provided (plus `Optimizers`, what the training callbacks receive), with the arithmetic of nerfstudio 0.3.x restated (same
restatement as oracle/oracle.py, which is the parity reference for these pieces).
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from enum import Enum, auto
from typing import Any, Callable, Dict, List, Optional, Tuple, Type

import torch
from torch import nn


# ---- cameras/rays.py -------------------------------------------------------------------------------
@dataclass
class Frustums:
    origins: torch.Tensor
    directions: torch.Tensor
    starts: torch.Tensor
    ends: torch.Tensor
    pixel_area: Optional[torch.Tensor] = None


@dataclass
class RaySamples:
    frustums: Frustums
    camera_indices: Optional[torch.Tensor] = None
    deltas: Optional[torch.Tensor] = None
    spacing_starts: Optional[torch.Tensor] = None
    spacing_ends: Optional[torch.Tensor] = None
    spacing_to_euclidean_fn: Optional[Callable] = None
    metadata: Optional[Dict[str, torch.Tensor]] = None
    times: Optional[torch.Tensor] = None

    def get_weights(self, densities: torch.Tensor) -> torch.Tensor:
        delta_density = self.deltas * densities
        alphas = 1 - torch.exp(-delta_density)
        transmittance = torch.cumsum(delta_density[..., :-1, :], dim=-2)
        transmittance = torch.cat([torch.zeros((*transmittance.shape[:1], 1, 1), device=densities.device), transmittance], dim=-2)
        transmittance = torch.exp(-transmittance)
        return torch.nan_to_num(alphas * transmittance)


@dataclass
class RayBundle:
    origins: torch.Tensor
    directions: torch.Tensor
    pixel_area: Optional[torch.Tensor] = None
    camera_indices: Optional[torch.Tensor] = None
    nears: Optional[torch.Tensor] = None
    fars: Optional[torch.Tensor] = None
    metadata: Dict[str, torch.Tensor] = field(default_factory=dict)
    times: Optional[torch.Tensor] = None

    def __len__(self):
        return self.origins.shape[0]

    def __getitem__(self, idx):
        def sel(x):
            return x[idx] if isinstance(x, torch.Tensor) else x

        return RayBundle(**{f.name: (sel(getattr(self, f.name)) if f.name != "metadata" else {k: sel(v) for k, v in self.metadata.items()})
                            for f in dataclasses.fields(self)})

    def get_ray_samples(self, bin_starts, bin_ends, spacing_starts=None, spacing_ends=None, spacing_to_euclidean_fn=None) -> RaySamples:
        deltas = bin_ends - bin_starts
        camera_indices = self.camera_indices[..., None] if self.camera_indices is not None else None
        frustums = Frustums(
            origins=self.origins[..., None, :].expand(*bin_starts.shape[:-1], 3),
            directions=self.directions[..., None, :].expand(*bin_starts.shape[:-1], 3),
            starts=bin_starts, ends=bin_ends,
            pixel_area=self.pixel_area[..., None, :] if self.pixel_area is not None else None,
        )
        return RaySamples(frustums=frustums, camera_indices=camera_indices, deltas=deltas, spacing_starts=spacing_starts,
                          spacing_ends=spacing_ends, spacing_to_euclidean_fn=spacing_to_euclidean_fn, metadata=self.metadata, times=self.times)


# ---- field components ------------------------------------------------------------------------------
class FieldHeadNames(Enum):
    RGB = "rgb"
    DENSITY = "density"


class NeRFEncoding(nn.Module):
    def __init__(self, in_dim: int, num_frequencies: int, min_freq_exp: float, max_freq_exp: float, include_input: bool = False):
        super().__init__()
        self.in_dim, self.num_frequencies, self.min_freq, self.max_freq, self.include_input = in_dim, num_frequencies, min_freq_exp, max_freq_exp, include_input

    def get_out_dim(self) -> int:
        return self.in_dim * self.num_frequencies * 2 + (self.in_dim if self.include_input else 0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        scaled = 2 * torch.pi * x
        freqs = 2 ** torch.linspace(self.min_freq, self.max_freq, self.num_frequencies, device=x.device)
        s = (scaled[..., None] * freqs).reshape(*scaled.shape[:-1], -1)
        enc = torch.sin(torch.cat([s, s + torch.pi / 2.0], dim=-1))
        return torch.cat([enc, x], dim=-1) if self.include_input else enc


class MLP(nn.Module):
    def __init__(self, in_dim: int, num_layers: int, layer_width: int, out_dim: Optional[int] = None, activation=nn.ReLU(), out_activation=None):
        super().__init__()
        self.out_dim = out_dim if out_dim is not None else layer_width
        dims = [in_dim] + [layer_width] * (num_layers - 1) + [self.out_dim]
        self.layers = nn.ModuleList([nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])])
        self.activation, self.out_activation = activation, out_activation

    def get_out_dim(self) -> int:
        return self.out_dim

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = layer(x)
            if self.activation is not None and i < len(self.layers) - 1:
                x = self.activation(x)
        return self.out_activation(x) if self.out_activation is not None else x


class _Head(nn.Module):
    def __init__(self, in_dim, out_dim, name, act):
        super().__init__()
        self.net, self.field_head_name, self.activation = nn.Linear(in_dim, out_dim), name, act

    def forward(self, x):
        return self.activation(self.net(x))


class DensityFieldHead(_Head):
    def __init__(self, in_dim: int):
        super().__init__(in_dim, 1, FieldHeadNames.DENSITY, nn.Softplus())


class RGBFieldHead(_Head):
    def __init__(self, in_dim: int):
        super().__init__(in_dim, 3, FieldHeadNames.RGB, nn.Sigmoid())


# ---- samplers ---------------------------------------------------------------------------------------
class Sampler(nn.Module):
    def __init__(self, num_samples: Optional[int] = None):
        super().__init__()
        self.num_samples = num_samples

    def generate_ray_samples(self, *a, **k):
        raise NotImplementedError

    def forward(self, *args, **kwargs):
        return self.generate_ray_samples(*args, **kwargs)


class UniformSampler(Sampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False):
        super().__init__(num_samples)
        self.train_stratified, self.single_jitter = train_stratified, single_jitter

    def generate_ray_samples(self, ray_bundle=None, num_samples=None):
        num_samples = num_samples or self.num_samples
        n = ray_bundle.origins.shape[0]
        bins = torch.linspace(0.0, 1.0, num_samples + 1, device=ray_bundle.origins.device)[None, ...]
        if self.train_stratified and self.training:
            t_rand = torch.rand((n, 1 if self.single_jitter else num_samples + 1), dtype=bins.dtype, device=bins.device)
            centers = (bins[..., 1:] + bins[..., :-1]) / 2.0
            upper = torch.cat([centers, bins[..., -1:]], -1)
            lower = torch.cat([bins[..., :1], centers], -1)
            bins = lower + (upper - lower) * t_rand
        s_near, s_far = ray_bundle.nears, ray_bundle.fars
        fn = lambda x: x * s_far + (1 - x) * s_near  # noqa: E731
        eb = fn(bins)
        return ray_bundle.get_ray_samples(bin_starts=eb[..., :-1, None], bin_ends=eb[..., 1:, None], spacing_starts=bins[..., :-1, None].expand(n, -1, 1),
                                          spacing_ends=bins[..., 1:, None].expand(n, -1, 1), spacing_to_euclidean_fn=fn)


class PDFSampler(Sampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False, include_original=True, histogram_padding=0.01):
        super().__init__(num_samples)
        self.train_stratified, self.single_jitter, self.include_original, self.histogram_padding = train_stratified, single_jitter, include_original, histogram_padding

    def generate_ray_samples(self, ray_bundle=None, ray_samples=None, weights=None, num_samples=None, eps=1e-5):
        num_samples = num_samples or self.num_samples
        num_bins = num_samples + 1
        weights = weights[..., 0] + self.histogram_padding
        weights_sum = torch.sum(weights, dim=-1, keepdim=True)
        padding = torch.relu(eps - weights_sum)
        weights = weights + padding / weights.shape[-1]
        weights_sum = weights_sum + padding
        pdf = weights / weights_sum
        cdf = torch.min(torch.ones_like(pdf), torch.cumsum(pdf, dim=-1))
        cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
        if self.train_stratified and self.training:
            u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins, device=cdf.device).expand(size=(*cdf.shape[:-1], num_bins))
            rand = torch.rand((*cdf.shape[:-1], 1 if self.single_jitter else num_samples + 1), device=cdf.device) / num_bins
            u = u + rand
        else:
            u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins, device=cdf.device) + 1.0 / (2 * num_bins)
            u = u.expand(size=(*cdf.shape[:-1], num_bins))
        u = u.contiguous()
        existing = torch.cat([ray_samples.spacing_starts[..., 0], ray_samples.spacing_ends[..., -1:, 0]], dim=-1)
        inds = torch.searchsorted(cdf, u, side="right")
        below = torch.clamp(inds - 1, 0, existing.shape[-1] - 1)
        above = torch.clamp(inds, 0, existing.shape[-1] - 1)
        cdf0, b0 = torch.gather(cdf, -1, below), torch.gather(existing, -1, below)
        cdf1, b1 = torch.gather(cdf, -1, above), torch.gather(existing, -1, above)
        t = torch.clip(torch.nan_to_num((u - cdf0) / (cdf1 - cdf0), 0), 0, 1)
        bins = b0 + t * (b1 - b0)
        if self.include_original:
            bins, _ = torch.sort(torch.cat([existing, bins], -1), -1)
        bins = bins.detach()
        eb = ray_samples.spacing_to_euclidean_fn(bins)
        return ray_bundle.get_ray_samples(bin_starts=eb[..., :-1, None], bin_ends=eb[..., 1:, None], spacing_starts=bins[..., :-1, None],
                                          spacing_ends=bins[..., 1:, None], spacing_to_euclidean_fn=ray_samples.spacing_to_euclidean_fn)


# ---- renderers --------------------------------------------------------------------------------------
COLORS_DICT = {"white": torch.tensor([1.0, 1.0, 1.0]), "black": torch.tensor([0.0, 0.0, 0.0])}


class RGBRenderer(nn.Module):
    def __init__(self, background_color="random"):
        super().__init__()
        self.background_color = background_color

    def get_background_color(self, background_color, shape, device):
        if background_color == "random":
            return torch.rand(shape, dtype=torch.float32, device=device)
        return COLORS_DICT[background_color].expand(shape).to(device).contiguous()

    def forward(self, rgb, weights):
        if not self.training:
            rgb = torch.nan_to_num(rgb)
        comp = torch.sum(weights * rgb, dim=-2)
        acc = torch.sum(weights, dim=-2)
        out = comp + self.get_background_color(self.background_color, comp.shape, comp.device) * (1.0 - acc)
        if not self.training:
            out = torch.clamp(out, min=0.0, max=1.0)
        return out


class AccumulationRenderer(nn.Module):
    def forward(self, weights):
        return torch.sum(weights, dim=-2)


class DepthRenderer(nn.Module):
    def __init__(self, method="median"):
        super().__init__()
        if method not in ("median", "expected"):
            raise NotImplementedError(f"DepthRenderer method {method!r}")
        self.method = method

    def forward(self, weights, ray_samples):
        steps = (ray_samples.frustums.starts + ray_samples.frustums.ends) / 2
        if self.method == "expected":  # clipped to the smallest / largest midpoint of the whole batch (DESIGN §4.10)
            eps = 1e-10
            depth = torch.sum(weights * steps, dim=-2) / (torch.sum(weights, -2) + eps)
            return torch.clip(depth, steps.min(), steps.max())
        cum = torch.cumsum(weights[..., 0], dim=-1)
        split = torch.ones((*weights.shape[:-2], 1), device=weights.device) * 0.5
        idx = torch.clamp(torch.searchsorted(cum, split, side="left"), 0, steps.shape[-2] - 1)
        return torch.gather(steps[..., 0], dim=-1, index=idx)


class MSELoss(nn.MSELoss):
    pass


# ---- models/base_model.py -----------------------------------------------------------------------------
class NearFarCollider(nn.Module):
    def __init__(self, near_plane: float, far_plane: float):
        super().__init__()
        self.near_plane, self.far_plane = near_plane, far_plane

    def forward(self, ray_bundle: RayBundle) -> RayBundle:
        ones = torch.ones_like(ray_bundle.origins[..., 0:1])
        ray_bundle.nears, ray_bundle.fars = ones * self.near_plane, ones * self.far_plane
        return ray_bundle


@dataclass
class ModelConfig:
    _target: Any = None
    enable_collider: bool = True
    collider_params: Optional[Dict[str, float]] = field(default_factory=lambda: {"near_plane": 2.0, "far_plane": 6.0})
    loss_coefficients: Dict[str, float] = field(default_factory=lambda: {"rgb_loss_coarse": 1.0, "rgb_loss_fine": 1.0})
    eval_num_rays_per_chunk: int = 4096

    def setup(self, **kwargs):
        return self._target(self, **kwargs)


class Model(nn.Module):
    config: ModelConfig

    def __init__(self, config, scene_box=None, num_train_data: int = 1, **kwargs):
        super().__init__()
        self.config, self.scene_box, self.num_train_data, self.kwargs = config, scene_box, num_train_data, kwargs
        self.collider = None
        self.populate_modules()
        self.device_indicator_param = nn.Parameter(torch.empty(0))

    @property
    def device(self):
        return self.device_indicator_param.device

    def populate_modules(self):
        if self.config.enable_collider:
            self.collider = NearFarCollider(near_plane=self.config.collider_params["near_plane"], far_plane=self.config.collider_params["far_plane"])

    def forward(self, ray_bundle: RayBundle):
        if self.collider is not None:
            ray_bundle = self.collider(ray_bundle)
        return self.get_outputs(ray_bundle)


def scale_dict(d: Dict[str, torch.Tensor], coefficients: Dict[str, float]) -> Dict[str, torch.Tensor]:
    return {k: (v * coefficients[k] if k in coefficients else v) for k, v in d.items()}


# ---- engine/callbacks.py, engine/optimizers.py --------------------------------------------------------
class TrainingCallbackLocation(Enum):
    BEFORE_TRAIN_ITERATION = auto()
    AFTER_TRAIN_ITERATION = auto()


@dataclass
class TrainingCallbackAttributes:
    optimizers: Optional["Optimizers"] = None
    grad_scaler: Optional[Any] = None
    pipeline: Optional[Any] = None


class TrainingCallback:
    """func(*args, **kwargs, step=step) at the locations in where_to_run, every update_every_num_iters steps or at the listed iters"""

    def __init__(self, where_to_run: List[TrainingCallbackLocation], func: Callable, update_every_num_iters: Optional[int] = None,
                 iters: Optional[Tuple[int, ...]] = None, args: Optional[List] = None, kwargs: Optional[Dict] = None):
        assert update_every_num_iters is None or iters is None, "only one of update_every_num_iters and iters"
        self.where_to_run, self.func, self.update_every_num_iters, self.iters = where_to_run, func, update_every_num_iters, iters
        self.args, self.kwargs = args or [], kwargs or {}

    def run_callback(self, step: int) -> None:
        if self.update_every_num_iters is not None:
            if step % self.update_every_num_iters == 0:
                self.func(*self.args, **self.kwargs, step=step)
        elif self.iters is not None:
            if step in self.iters:
                self.func(*self.args, **self.kwargs, step=step)
        else:
            self.func(*self.args, **self.kwargs, step=step)

    def run_callback_at_location(self, step: int, location: TrainingCallbackLocation) -> None:
        if location in self.where_to_run:
            self.run_callback(step=step)


class Optimizers:
    """one torch optimizer per param group: `config` maps a group name to {"optimizer": factory(params) -> torch.optim.Optimizer}"""

    def __init__(self, config: Dict[str, Dict[str, Callable]], param_groups: Dict[str, List[nn.Parameter]]):
        self.config = config
        self.optimizers = {name: config[name]["optimizer"](params) for name, params in param_groups.items()}
        self.parameters = {name: params for name, params in param_groups.items()}

    def zero_grad_all(self) -> None:
        for opt in self.optimizers.values():
            opt.zero_grad()

    def optimizer_step_all(self) -> None:
        for opt in self.optimizers.values():
            opt.step()

    def load_optimizers(self, loaded_state: Dict[str, Any]) -> None:
        for k, v in loaded_state.items():
            self.optimizers[k].load_state_dict(v)
