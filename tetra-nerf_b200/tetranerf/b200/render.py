"""Fused forward render (trace -> sample -> interp+MLP -> PDF -> interp+MLP -> composite) through the C ABI.

`FusedRenderer` is what `TetrahedraNerf.get_outputs` (tetranerf/nerfstudio/model.py:520-662) calls in eval mode;
it needs the CUDA library -- there is no PyTorch fallback."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from ..utils.extension import tetranerf_cpp_extension as ext

_lib = ext._lib
_vp = C.c_void_p

KERNEL_NAMES = ["trace", "sample_coarse", "mlp_coarse", "sample_fine", "mlp_fine", "composite"]

PARAM_ORDER = [
    "mlp_base.layers.0.weight", "mlp_base.layers.0.bias", "mlp_base.layers.1.weight", "mlp_base.layers.1.bias",
    "mlp_base.layers.2.weight", "mlp_base.layers.2.bias", "mlp_head.layers.0.weight", "mlp_head.layers.0.bias",
    "field_output_color.net.weight", "field_output_color.net.bias", "field_output_density.net.weight", "field_output_density.net.bias",
]
_SHAPES = [(128, 64), (128,), (128, 128), (128,), (128, 128), (128,), (128, 155), (128,), (3, 128), (3,), (1, 128), (1,)]


@dataclass
class RenderSettings:
    """hot-path subset of TetrahedraNerfConfig (model.py:70-107)"""

    max_intersected_triangles: int = 512
    num_samples: int = 256
    num_fine_samples: int = 256
    use_biased_sampler: bool = False
    far_plane: float = 6.0
    background: tuple = (1.0, 1.0, 1.0)

    @staticmethod
    def tetra_nerf():  # registration.py:48-61
        return RenderSettings(num_samples=128, num_fine_samples=128, use_biased_sampler=True)

    @staticmethod
    def tetra_nerf_original():  # registration.py:20-46
        return RenderSettings()


def _config(settings: RenderSettings) -> "ext._Cfg":
    return ext._Cfg(settings.max_intersected_triangles, settings.num_samples, settings.num_fine_samples, int(settings.use_biased_sampler),
                    float(settings.far_plane), (C.c_float * 3)(*settings.background))


class FusedRenderer:
    def __init__(self, tracer: "ext.TetrahedraTracer"):
        self.tracer = tracer
        self.device = tracer.device
        self._keep = None

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def set_field(self, field: torch.Tensor) -> None:
        """field: f32[64, V] feature-major (`tetrahedra_field`, model.py:247-255)."""
        if field.device != self.device or field.dtype != torch.float32 or not field.is_contiguous() or field.dim() != 2:
            raise RuntimeError("field must be a contiguous float32 [64, V] tensor on the tracer's device")
        ext._check(_lib.tn_render_set_field(self.tracer.handle, field.data_ptr(), field.shape[0], field.shape[1], self._stream()))

    def set_weights(self, params: Dict[str, torch.Tensor]) -> None:
        """params: nerfstudio state-dict names (PARAM_ORDER) -> tensors."""
        ts = []
        for name, shape in zip(PARAM_ORDER, _SHAPES):
            t = params[name].detach().to(device=self.device, dtype=torch.float32).contiguous()
            if tuple(t.shape) != shape:
                raise RuntimeError(f"{name} must have shape {shape}, got {tuple(t.shape)}")
            ts.append(t)
        arr = (_vp * 12)(*[t.data_ptr() for t in ts])
        ext._check(_lib.tn_render_set_weights(self.tracer.handle, arr, self._stream()))
        self._keep = ts  # repacked on the stream; keep sources alive until then

    def render(self, origins: torch.Tensor, directions: torch.Tensor, settings: RenderSettings, out: Optional[dict] = None):
        tr = self.tracer
        tr._check_float_dim3(origins, "ray_origins")
        tr._check_float_dim3(directions, "ray_directions")
        R = origins.numel() // 3
        dev = self.device
        if out is None:
            out = {
                "rgb": torch.empty((R, 3), dtype=torch.float32, device=dev),
                "accumulation": torch.empty((R, 1), dtype=torch.float32, device=dev),
                "depth": torch.empty((R, 1), dtype=torch.float32, device=dev),
                "ray_mask": torch.empty((R,), dtype=torch.bool, device=dev),
            }
        cfg = _config(settings)
        ext._check(_lib.tn_render(tr.handle, C.byref(cfg), origins.data_ptr(), directions.data_ptr(), R, out["rgb"].data_ptr(),
                                  out["accumulation"].data_ptr(), out["depth"].data_ptr(), out["ray_mask"].data_ptr(), self._stream()))
        return out

    # ---- fused training step ------------------------------------------------------------------------------------------------------
    def train_forward(self, origins: torch.Tensor, directions: torch.Tensor, settings: RenderSettings, jitter_coarse: Optional[torch.Tensor] = None,
                      jitter_fine: Optional[torch.Tensor] = None):
        """training-mode forward (stratified bins from the given uniform draws f32[R,S_c+1] / f32[R,S_f+1]; None = eval bins; RGB renderer
        without clamp).  Keeps the per-sample buffers the backward continues from.  Runs in deterministic mode (bitwise reproducible
        outputs and gradients, see tn_render_set_deterministic) when `torch.are_deterministic_algorithms_enabled()` or
        TETRANERF_B200_DETERMINISTIC=1; the backward continues in the mode of its forward."""
        tr = self.tracer
        tr._check_float_dim3(origins, "ray_origins")
        tr._check_float_dim3(directions, "ray_directions")
        R = origins.numel() // 3
        dev = self.device
        for t, n, w in ((jitter_coarse, "jitter_coarse", settings.num_samples + 1), (jitter_fine, "jitter_fine", settings.num_fine_samples + 1)):
            if t is not None and (t.device != dev or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != (R, w)):
                raise RuntimeError(f"{n} must be a contiguous float32 [{R}, {w}] tensor on the tracer's device")
        out = {"rgb": torch.empty((R, 3), dtype=torch.float32, device=dev), "accumulation": torch.empty((R, 1), dtype=torch.float32, device=dev),
               "depth": torch.empty((R, 1), dtype=torch.float32, device=dev), "ray_mask": torch.empty((R,), dtype=torch.bool, device=dev)}
        cfg = _config(settings)
        ext._check(_lib.tn_render_set_deterministic(tr.handle, int(ext.deterministic_enabled())))
        ext._check(_lib.tn_render_train_forward(tr.handle, C.byref(cfg), origins.data_ptr(), directions.data_ptr(), R,
                                                jitter_coarse.data_ptr() if jitter_coarse is not None else None,
                                                jitter_fine.data_ptr() if jitter_fine is not None else None, out["rgb"].data_ptr(),
                                                out["accumulation"].data_ptr(), out["depth"].data_ptr(), out["ray_mask"].data_ptr(), self._stream()))
        return out

    def train_backward(self, grad_rgb: torch.Tensor, grad_acc: Optional[torch.Tensor], num_vertices: int, use_gradient_scaling: bool = False):
        """backward of the last train_forward: -> (grad_field f32[64,V], {state-dict name: gradient} for the twelve MLP parameters)"""
        dev = self.device
        grad_rgb = grad_rgb.contiguous()
        if grad_acc is not None:
            grad_acc = grad_acc.contiguous()
        gfield = torch.empty((64, num_vertices), dtype=torch.float32, device=dev)
        gps = [torch.empty(sh, dtype=torch.float32, device=dev) for sh in _SHAPES]
        arr = (_vp * 12)(*[t.data_ptr() for t in gps])
        ext._check(_lib.tn_render_train_backward(self.tracer.handle, grad_rgb.data_ptr(), grad_acc.data_ptr() if grad_acc is not None else None,
                                                 int(use_gradient_scaling), gfield.data_ptr(), arr, self._stream()))
        return gfield, dict(zip(PARAM_ORDER, gps))

    def set_mlp_precision(self, prec: int) -> None:
        """operand precision of the inference MLP: 2 = f16w2 (default: fp16 activations x fp16 hi/lo weights, ~2.6e-5 absolute on
        unit-scale density / colour, inside the 1e-4 per-sample bar), 3 = bf16x3 (fp32-level, ~5e-7).  Training always runs bf16x3."""
        ext._check(_lib.tn_render_set_mlp_precision(self.tracer.handle, int(prec)))

    def set_backward_grid(self, ctas: int) -> None:
        """test hook: CTAs of the backward MLP kernel (0 = default, one per SM)"""
        ext._check(_lib.tn_render_set_backward_grid(self.tracer.handle, int(ctas)))

    def set_profiling(self, enable: bool) -> None:
        ext._check(_lib.tn_render_set_profiling(self.tracer.handle, int(enable)))

    def kernel_timings_ms(self) -> Dict[str, float]:
        """CUDA-event durations of the six kernels of the last render() (profiling must be enabled)."""
        arr = (C.c_float * 6)()
        ext._check(_lib.tn_render_get_timings(self.tracer.handle, arr))
        return {n: float(arr[i]) for i, n in enumerate(KERNEL_NAMES)}

    def backward_timings_ms(self) -> Dict[str, float]:
        """CUDA-event durations of the kernels of the last train_backward() (profiling must be enabled)"""
        arr = (C.c_float * 3)()
        ext._check(_lib.tn_render_get_backward_timings(self.tracer.handle, arr))
        return {n: float(arr[i]) for i, n in enumerate(["composite_bwd", "mlp_bwd", "finalize"])}

    def debug_buffers(self):
        arr = (_vp * 16)()
        ext._check(_lib.tn_render_debug_buffers(self.tracer.handle, arr))
        names = ["num", "dist", "n_active", "ray_list", "ebins_c", "sbins_c", "vi_c", "bary_c", "dens_c", "ebins_f", "vi_f", "bary_f",
                 "out_f", "dirbias", "fshadow", "wimg"]
        return {n: arr[i] for i, n in enumerate(names)}


class FusedTrainRender(torch.autograd.Function):
    """TetrahedraNerf.get_outputs in training mode as ONE differentiable op: forward = tn_render_train_forward, backward =
    tn_render_train_backward (gradients for `tetrahedra_field` and the twelve MLP parameters; none for rays or jitter).
    The renderer must already hold the current field / weights (FusedRenderer.set_field / set_weights)."""

    @staticmethod
    def forward(ctx, fr, settings, use_gradient_scaling, origins, directions, jitter_coarse, jitter_fine, field, *params):
        out = fr.train_forward(origins, directions, settings, jitter_coarse, jitter_fine)
        ctx.fr, ctx.nv, ctx.gs = fr, field.shape[1], bool(use_gradient_scaling)
        ctx.mark_non_differentiable(out["depth"], out["ray_mask"])
        return out["rgb"], out["accumulation"], out["depth"], out["ray_mask"]

    @staticmethod
    def backward(ctx, g_rgb, g_acc, _g_depth, _g_mask):
        if g_rgb is None:
            g_rgb = torch.zeros((g_acc.shape[0], 3), dtype=torch.float32, device=g_acc.device)
        gfield, gp = ctx.fr.train_backward(g_rgb, g_acc.reshape(-1) if g_acc is not None else None, ctx.nv, ctx.gs)
        return (None, None, None, None, None, None, None, gfield) + tuple(gp[n] for n in PARAM_ORDER)
