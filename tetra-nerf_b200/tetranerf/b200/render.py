"""Fused forward render (trace -> sample -> interp+MLP -> PDF -> interp+MLP -> composite) through the C ABI.

`FusedRenderer` is what `TetrahedraNerf.get_outputs` (tetranerf/nerfstudio/model.py:520-662) calls in eval mode;
it needs the CUDA library -- there is no PyTorch fallback."""
from __future__ import annotations

import ctypes as C
import math
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
    """hot-path subset of TetrahedraNerfConfig (model.py:70-107).  max_intersected_triangles (M) is a power of two in [2, 2048],
    num_samples in [1, 4096], num_fine_samples in [0, 4096] (0 = single pass).  Two-pass settings must also fit the per-ray kernels'
    shared memory: 16 (M + 4 S2 + 10) bytes per block with S2 = num_samples + num_fine_samples + 1, at most the device's opt-in limit
    (232,448 B on an H100: num_samples + num_fine_samples <= 3500 at M = 512, <= 3116 at M = 2048); beyond it render and the
    training forwards raise RuntimeError before anything runs.  Occupancy sampling (set_occupancy(..., place_samples=True)) adds
    32 (M + 2) bytes per block to the coarse sampler only, at most 164 KB in all: every setting above still runs with it."""

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


def _ptr(t: Optional[torch.Tensor]):
    """device pointer of an optional tensor (None: NULL)"""
    return t.data_ptr() if t is not None else None


BACKGROUND_POLE_EPS = 1e-8  # BG_POLE_EPS of csrc/tn_background.cuh


def background_lookup(bg_map: torch.Tensor, directions: torch.Tensor) -> torch.Tensor:
    """bg(d) of the background map f32[H,2H,3] for directions [..., 3] -> [..., 3], in torch (differentiable to both), the lookup the
    fused kernels make (csrc/tn_background.cuh; DESIGN §4.16): n = d / |d|, u = W (atan2(n_y, n_x) / 2 pi + 1/2) - 1/2 with columns
    modulo W, v = H (1 - n_z) / 2 - 1/2 clamped to [0, H - 1], bilinear in the lerp form, so a constant map returns its constant
    exactly.  No grid_sample: its CUDA backward is not deterministic.  As the fused backward, the u-derivative is 0 where
    n_x^2 + n_y^2 < BACKGROUND_POLE_EPS (near the poles, where atan2's derivative is unbounded, and 0/0 at the poles themselves)."""
    H, W = int(bg_map.shape[0]), int(bg_map.shape[1])
    n = directions / torch.linalg.vector_norm(directions, dim=-1, keepdim=True)
    pole = (n[..., 0] * n[..., 0] + n[..., 1] * n[..., 1] < BACKGROUND_POLE_EPS)[..., None]
    nxy = torch.where(pole, n[..., :2].detach(), n[..., :2])  # (where's backward drops the detached branch's NaN at the pole)
    u = W * (torch.atan2(nxy[..., 1], nxy[..., 0]) / (2 * math.pi) + 0.5) - 0.5
    v = (H * (1 - n[..., 2]) / 2 - 0.5).clamp(0, H - 1)
    fi, fj = torch.floor(u), torch.floor(v)
    fu, fv = (u - fi)[..., None], (v - fj)[..., None]
    i0 = torch.remainder(fi.long(), W)
    i1 = torch.remainder(i0 + 1, W)
    j0 = fj.long().clamp(0, H - 1)
    j1 = (j0 + 1).clamp(max=H - 1)
    flat = bg_map.reshape(-1, 3)

    def lerp(a, b, t):
        return a + t * (b - a)

    top = lerp(flat[j0 * W + i0], flat[j0 * W + i1], fu)
    bot = lerp(flat[j1 * W + i0], flat[j1 * W + i1], fu)
    return lerp(top, bot, fv)


def _config(settings: RenderSettings) -> "ext._Cfg":
    return ext._Cfg(settings.max_intersected_triangles, settings.num_samples, settings.num_fine_samples, int(settings.use_biased_sampler),
                    float(settings.far_plane), (C.c_float * 3)(*settings.background))


@dataclass
class TrainState:
    """what one FusedRenderer.train_forward_saved call keeps for its backward: the saved-state blob (device memory from torch's
    allocator, freed with this object whether or not the backward ever runs) and the call's ray count"""

    blob: torch.Tensor
    R: int


class FusedRenderer:
    def __init__(self, tracer: "ext.TetrahedraTracer"):
        self.tracer = tracer
        self.device = tracer.device
        self._keep = None
        self._bg = None

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

    def render(self, origins: torch.Tensor, directions: torch.Tensor, settings: RenderSettings, out: Optional[dict] = None, normals: bool = False,
               expected_depth: bool = False):
        """eval-mode render -> `rgb` f32[R,3], `accumulation` / `depth` f32[R,1], `ray_mask` bool[R]; normals=True adds `normals`
        f32[R,3]: the composited unit normal of the density field (nerfstudio's "normals" output, (0, 0, 0) on empty rays; DESIGN §4.7).
        expected_depth=True adds `expected_depth` f32[R,1]: nerfstudio's DepthRenderer(method="expected"), clipped to the call's smallest
        and largest sample midpoint, far_plane on empty rays (DESIGN §4.10).  The two combine; the other outputs are the same bits as
        without them.  Neither is available while a fused pixel gather is set."""
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
        if normals and "normals" not in out:
            out["normals"] = torch.empty((R, 3), dtype=torch.float32, device=dev)
        if expected_depth and "expected_depth" not in out:
            out["expected_depth"] = torch.empty((R, 1), dtype=torch.float32, device=dev)
        ext._check(_lib.tn_render(tr.handle, C.byref(_config(settings)), origins.data_ptr(), directions.data_ptr(), R, out["rgb"].data_ptr(),
                                  out["accumulation"].data_ptr(), out["depth"].data_ptr(), out["ray_mask"].data_ptr(),
                                  out["expected_depth"].data_ptr() if expected_depth else None, out["normals"].data_ptr() if normals else None,
                                  self._stream()))
        return out

    def set_background(self, bg_map: Optional[torch.Tensor]) -> None:
        """composite, in every later render and training forward, over the background map bg_map f32[H,2H,3] (borrowed, kept alive
        here; None: back to the settings' constant background): rgb = sum_j w_j c_j + (1 - accumulation) bg(d) on rays with hits,
        rgb = bg(d) on empty ones (background_lookup; DESIGN §4.16).  Every call starts a new generation: the backward of a training
        forward before it raises RuntimeError.  A training forward over a map keeps its directions, 12 more bytes per ray."""
        if bg_map is not None:
            if (bg_map.device != self.device or bg_map.dtype != torch.float32 or not bg_map.is_contiguous() or bg_map.dim() != 3
                    or bg_map.shape[2] != 3 or bg_map.shape[1] != 2 * bg_map.shape[0]):
                raise RuntimeError("the background map must be a contiguous float32 [H, 2H, 3] tensor on the tracer's device, got "
                                   f"{tuple(bg_map.shape)}")
            H, W = bg_map.shape[0], bg_map.shape[1]
        else:
            H = W = 0
        ext._check(_lib.tn_render_set_background(self.tracer.handle, _ptr(bg_map), H, W))
        self._bg = bg_map

    # ---- fused training step ------------------------------------------------------------------------------------------------------
    def _train_args(self, origins, directions, settings, jitter_coarse, jitter_fine):
        """checks the inputs of a training forward, allocates its outputs and sets the mode of the call -> (R, outputs, C arguments)"""
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
        ext._check(_lib.tn_render_set_deterministic(tr.handle, int(ext.deterministic_enabled())))
        args = [tr.handle, C.byref(_config(settings)), origins.data_ptr(), directions.data_ptr(), R,
                jitter_coarse.data_ptr() if jitter_coarse is not None else None, jitter_fine.data_ptr() if jitter_fine is not None else None,
                out["rgb"].data_ptr(), out["accumulation"].data_ptr(), out["depth"].data_ptr(), out["ray_mask"].data_ptr()]
        return R, out, args

    def _grad_outputs(self, num_vertices):
        """the outputs of a training backward -> (grad_field f32[64,V], {state-dict name: gradient} for the twelve MLP parameters, the
        twelve as the C pointer array the backward writes through)"""
        gfield = torch.empty((64, num_vertices), dtype=torch.float32, device=self.device)
        gps = [torch.empty(sh, dtype=torch.float32, device=self.device) for sh in _SHAPES]
        return gfield, dict(zip(PARAM_ORDER, gps)), (_vp * 12)(*[t.data_ptr() for t in gps])

    def train_forward(self, origins: torch.Tensor, directions: torch.Tensor, settings: RenderSettings, jitter_coarse: Optional[torch.Tensor] = None,
                      jitter_fine: Optional[torch.Tensor] = None):
        """training-mode forward (stratified bins from the given uniform draws f32[R,S_c+1] / f32[R,S_f+1]; None = eval bins; RGB renderer
        without clamp).  Keeps the per-sample buffers the backward continues from in the tracer, until the next render call (see
        train_forward_saved for a forward with its own saved state).  Runs in deterministic mode (bitwise reproducible outputs and
        gradients, see tn_render_set_deterministic) when `torch.are_deterministic_algorithms_enabled()` or TETRANERF_B200_DETERMINISTIC=1;
        the backward continues in the mode of its forward."""
        _, out, args = self._train_args(origins, directions, settings, jitter_coarse, jitter_fine)
        ext._check(_lib.tn_render_train_forward(*args, self._stream()))
        return out

    def train_backward(self, grad_rgb: torch.Tensor, grad_acc: Optional[torch.Tensor], num_vertices: int, use_gradient_scaling: bool = False):
        """backward of the last train_forward: -> (grad_field f32[64,V], {state-dict name: gradient} for the twelve MLP parameters)"""
        grad_rgb = grad_rgb.contiguous()
        grad_acc = grad_acc.contiguous() if grad_acc is not None else None
        gfield, gp, arr = self._grad_outputs(num_vertices)
        ext._check(_lib.tn_render_train_backward(self.tracer.handle, grad_rgb.data_ptr(), _ptr(grad_acc), int(use_gradient_scaling),
                                                 gfield.data_ptr(), arr, self._stream()))
        return gfield, gp

    def train_saved_bytes(self, R: int, settings: RenderSettings) -> int:
        """device bytes of the saved state of one training forward of R rays, for the renderer's state now: with a background map set
        (set_background) the forward also keeps its ray directions, 12 bytes per ray more.  A blob sized before a set_background that
        adds a map is too small for the forwards after it (they raise RuntimeError); train_forward_saved sizes its blob on every call"""
        n = C.c_size_t()
        ext._check(_lib.tn_render_train_saved_bytes(self.tracer.handle, C.byref(_config(settings)), int(R), C.byref(n)))
        return n.value

    def train_forward_saved(self, origins: torch.Tensor, directions: torch.Tensor, settings: RenderSettings,
                            jitter_coarse: Optional[torch.Tensor] = None, jitter_fine: Optional[torch.Tensor] = None, expected_depth: bool = False):
        """train_forward whose backward state goes to a blob of its own instead of the tracer -> (outputs, TrainState).  Any number of
        these can be in flight; train_backward_saved(state, ...) continues from the one it is given.  expected_depth=True adds
        `expected_depth` f32[R,1] to the outputs (as render's, in training mode; DESIGN §4.10), and its backward then accepts a gradient
        for it; the other outputs are the same bits either way."""
        R, out, args = self._train_args(origins, directions, settings, jitter_coarse, jitter_fine)
        blob = torch.empty((self.train_saved_bytes(R, settings),), dtype=torch.uint8, device=self.device)
        if expected_depth:
            out["expected_depth"] = torch.empty((R, 1), dtype=torch.float32, device=self.device)
        ext._check(_lib.tn_render_train_forward_saved(*args, _ptr(out.get("expected_depth")), blob.data_ptr(), blob.numel(), self._stream()))
        return out, TrainState(blob, R)

    def train_backward_saved(self, state: "TrainState", grad_rgb: torch.Tensor, grad_acc: Optional[torch.Tensor], num_vertices: int,
                             use_gradient_scaling: bool = False, grad_origins: bool = False, grad_directions: bool = False,
                             grad_vertices: bool = False, grad_expected_depth: Optional[torch.Tensor] = None,
                             grad_distortion: Optional[torch.Tensor] = None, grad_background: bool = False):
        """backward of the train_forward_saved call that returned `state`; outputs as train_backward.  Raises RuntimeError if
        set_field / set_weights ran since that forward.  Waits until the stream has reached it (it reads the call's shape back).
        grad_origins / grad_directions: also the gradients at the forward's ray origins / directions (the sample distances held fixed;
        DESIGN §4.8) -> (grad_field, grads, grad_origins f32[R,3] or None, grad_directions f32[R,3] or None), 0 on empty rays; then it
        also raises RuntimeError if load_tetrahedra ran since that forward.  grad_vertices: also the gradient at the mesh vertex positions
        (the matched tetrahedra held fixed as well; DESIGN §4.9) -> (grad_field, grads, grad_origins or None, grad_directions or None,
        grad_vertices f32[V,3]); then it raises RuntimeError if load_tetrahedra or update_vertices ran since that forward.
        grad_expected_depth f32[R] or [R,1]: dL/d expected_depth of a forward with expected_depth=True (RuntimeError otherwise); the
        outputs keep the form above.  grad_distortion f32[R] or [R,1]: dL/d distortion (train_distortion; DESIGN §4.11), for any forward;
        None runs the same kernels as before it existed.  grad_background: also the gradient at the background map of a forward over
        one (set_background; DESIGN §4.16; RuntimeError otherwise, or after another set_background) -> always the 6-tuple (grad_field,
        grads, grad_origins or None, grad_directions or None, grad_vertices or None, grad_background f32[H,2H,3]).  With a map the
        direction gradients also hold the background's term, on every ray."""
        if tuple(grad_rgb.shape) != (state.R, 3) or (grad_acc is not None and grad_acc.numel() != state.R):
            raise RuntimeError(f"the forward rendered {state.R} rays: grad_rgb must be [{state.R}, 3] and grad_acc [{state.R}], got "
                               f"{tuple(grad_rgb.shape)} and {None if grad_acc is None else tuple(grad_acc.shape)}")
        g_ed, g_dist = grad_expected_depth, grad_distortion
        for name, t in (("grad_expected_depth", g_ed), ("grad_distortion", g_dist)):
            if t is not None and (t.numel() != state.R or t.device != self.device or t.dtype != torch.float32):
                raise RuntimeError(f"{name} must be a float32 [{state.R}] tensor on the tracer's device, got {tuple(t.shape)}")
        g_ed = g_ed.reshape(-1).contiguous() if g_ed is not None else None
        g_dist = g_dist.reshape(-1).contiguous() if g_dist is not None else None
        grad_rgb = grad_rgb.contiguous()
        grad_acc = grad_acc.contiguous() if grad_acc is not None else None
        go = torch.empty((state.R, 3), dtype=torch.float32, device=self.device) if grad_origins else None
        gd = torch.empty((state.R, 3), dtype=torch.float32, device=self.device) if grad_directions else None
        gv = torch.empty((num_vertices, 3), dtype=torch.float32, device=self.device) if grad_vertices else None
        gbg = None
        if grad_background:
            if self._bg is None:
                raise RuntimeError("grad_background: no background map is set (set_background)")
            gbg = torch.empty_like(self._bg)
        gfield, gp, arr = self._grad_outputs(num_vertices)
        ext._check(_lib.tn_render_train_backward_saved3(self.tracer.handle, state.blob.data_ptr(), grad_rgb.data_ptr(), _ptr(grad_acc),
                                                        _ptr(g_ed), _ptr(g_dist), int(use_gradient_scaling), gfield.data_ptr(), arr, _ptr(go),
                                                        _ptr(gd), _ptr(gv), _ptr(gbg), self._stream()))
        if grad_background:
            return gfield, gp, go, gd, gv, gbg
        if grad_vertices:
            return gfield, gp, go, gd, gv
        return (gfield, gp, go, gd) if grad_origins or grad_directions else (gfield, gp)

    def train_distortion(self, state: "TrainState") -> torch.Tensor:
        """the distortion loss per ray of the train_forward_saved call that returned `state` -> f32[R,1], 0 on empty rays: mip-NeRF 360's
        sum_i sum_j w_i w_j |u_i - u_j| + 1/3 sum_i w_i^2 delta_i over the fine samples, u / delta the midpoints / widths of the spacing
        bins, w the weights of rgb (nerfstudio's distortion_loss per ray; DESIGN §4.11).  Raises RuntimeError if set_field / set_weights
        ran since that forward.  Waits until the stream has reached it (it reads the call's shape back)."""
        out = torch.empty((state.R, 1), dtype=torch.float32, device=self.device)
        ext._check(_lib.tn_render_train_distortion(self.tracer.handle, state.blob.data_ptr(), out.data_ptr(), self._stream()))
        return out

    # ---- occupancy culling (DESIGN §4.12) -------------------------------------------------------------------------------------------
    def _check_occupancy(self, occ: torch.Tensor) -> None:
        T = self.tracer._cells.numel() // 4 if self.tracer._cells is not None else 0
        if occ.device != self.device or occ.dtype != torch.float32 or not occ.is_contiguous() or tuple(occ.shape) != (T,):
            raise RuntimeError(f"the occupancy must be a contiguous float32 [{T}] tensor (one entry per tetrahedron) on the tracer's device")

    def set_occupancy(self, occ: Optional[torch.Tensor], threshold: float = 0.0, place_samples: bool = False) -> None:
        """cull, in every later render and training forward, the samples matched to a tetrahedron t with occ[t] < threshold: their
        density is the constant 0 and their MLP is not evaluated (unmatched samples are evaluated as before).  occ f32[T] is borrowed
        (kept alive here); None switches culling off.  A saved training forward's backward does not read occ again.
        place_samples (needs occ): also place each ray's coarse bins in its records outside those tetrahedra only, so the sample budget
        lands where the density can be non-zero (DESIGN §4.13)."""
        if occ is not None:
            self._check_occupancy(occ)
        ext._check(_lib.tn_render_set_occupancy2(self.tracer.handle, _ptr(occ), C.c_float(float(threshold)), 1 if place_samples else 0))
        self._occ = occ

    def update_occupancy(self, occ: torch.Tensor, decay: float = 0.0) -> torch.Tensor:
        """occ f32[T] <- max(decay * occ, the largest density over the 4 vertices, 6 edge midpoints and centroid of each tetrahedron),
        in place, with the current field and weights (decay 0: recomputed; bitwise reproducible) -> occ"""
        self._check_occupancy(occ)
        ext._check(_lib.tn_occupancy_update(self.tracer.handle, occ.data_ptr(), C.c_float(float(decay)), self._stream()))
        return occ

    # ---- field smoothness (DESIGN §4.15) ------------------------------------------------------------------------------------------
    def field_smoothness(self, mult: float = 1.0, grad: bool = False):
        """the field's smoothness along the mesh edges, for the field of the last set_field on the tracer's mesh -> (S f64[] on the
        device, E, grad_field f32[64,V] or None): S = sum over the E unique undirected edges {i, j} of sum_c (F[c,i] - F[c,j])^2, and
        with grad=True the gradient of mult * S / (E * 64), 0 for a vertex no cell uses.  The first call after load_tetrahedra builds
        the vertex adjacency and waits for the stream once; later calls do not wait.  Bitwise reproducible in every mode."""
        S = torch.empty((), dtype=torch.float64, device=self.device)
        V = self.tracer._vertices.shape[0] if self.tracer._vertices is not None else 0
        g = torch.empty((64, V), dtype=torch.float32, device=self.device) if grad else None
        E = C.c_uint32(0)
        ext._check(_lib.tn_field_smoothness(self.tracer.handle, C.c_float(float(mult)), S.data_ptr(), _ptr(g), C.byref(E), self._stream()))
        return S, int(E.value), g

    # ---- surface extraction ---------------------------------------------------------------------------------------------------------
    def extract_surface(self, level: float) -> Dict[str, torch.Tensor]:
        """the density iso-surface sigma = level (finite, > 0) of the current field and weights, by marching tetrahedra on the tracer's
        mesh (tn_surface_extract; DESIGN §4.6) -> device tensors `vertices`, `normals`, `colors` f32[N,3], `faces` i32[F,3] and
        `face_tetrahedra` i32[F], in the mesh's frame.  Empty tensors when the level lies above or below every vertex density.  Waits
        until the stream has reached it (the counts are read back)."""
        tr, dev = self.tracer, self.device
        n, f = C.c_uint32(0), C.c_uint32(0)
        with torch.cuda.device(dev):
            ext._check(_lib.tn_surface_extract(tr.handle, C.c_float(float(level)), C.byref(n), C.byref(f), self._stream()))
            N, F = int(n.value), int(f.value)
            out = {"vertices": torch.empty((N, 3), dtype=torch.float32, device=dev), "normals": torch.empty((N, 3), dtype=torch.float32, device=dev),
                   "colors": torch.empty((N, 3), dtype=torch.float32, device=dev), "faces": torch.empty((F, 3), dtype=torch.int32, device=dev),
                   "face_tetrahedra": torch.empty((F,), dtype=torch.int32, device=dev)}
            self.copy_surface(out)
        return out

    def copy_surface(self, out: Dict[str, torch.Tensor]) -> None:
        """copies the last extraction into `out` (the tensors extract_surface allocates); raises RuntimeError if set_field, set_weights or
        load_tetrahedra ran since it"""
        ext._check(_lib.tn_surface_copy(self.tracer.handle, out["vertices"].data_ptr(), out["normals"].data_ptr(), out["colors"].data_ptr(),
                                        out["faces"].data_ptr(), out["face_tetrahedra"].data_ptr(), self._stream()))

    def set_mlp_precision(self, prec: int) -> None:
        """operand precision of the inference MLP: 2 = f16w2 (default: fp16 activations x fp16 hi/lo weights; per-sample error relative
        to the activations -- ~2.6e-5 absolute on unit-scale density / colour, ~4.9e-4 relative on large densities -- pixels within
        1e-4), 3 = bf16x3 (fp32-level, ~5e-7).  Training always runs bf16x3."""
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

    def debug_normals_grad(self) -> int:
        """test hook: device pointer of the per-sample density gradient (float4 per sample, slot order) of the last normals render"""
        ptr = _vp()
        ext._check(_lib.tn_render_debug_normals_grad(self.tracer.handle, C.byref(ptr)))
        return ptr.value

    def debug_ray_grads(self) -> int:
        """test hook: device pointer of dL/dx per fine sample (float4 per sample, slot order) of the last backward with ray gradients"""
        ptr = _vp()
        ext._check(_lib.tn_render_debug_ray_grads(self.tracer.handle, C.byref(ptr)))
        return ptr.value

    def debug_buffers(self):
        """test hook: device pointers of the intermediate buffers of the last render, by name.  "fshadow" is the field as the fused
        MLP reads it, f32[V,64] with each vertex's row in fragment order: within each 16-feature block b, feature
        16b + 8h + 2t + e (h, e in {0, 1}, t in 0..3) sits at position 16b + 4t + 2h + e, so one 16-byte load gives a thread of
        a wgmma A fragment row the four features it needs in one k-step (csrc/tn_common.cuh, field_pos)."""
        arr = (_vp * 16)()
        ext._check(_lib.tn_render_debug_buffers(self.tracer.handle, arr))
        names = ["num", "dist", "n_active", "ray_list", "ebins_c", "sbins_c", "vi_c", "bary_c", "dens_c", "ebins_f", "vi_f", "bary_f",
                 "out_f", "dirbias", "fshadow", "wimg"]
        return {n: arr[i] for i, n in enumerate(names)}


class FusedTrainRender(torch.autograd.Function):
    """TetrahedraNerf.get_outputs in training mode as ONE differentiable op: forward = tn_render_train_forward_saved, backward =
    tn_render_train_backward_saved (gradients for `tetrahedra_field` and the twelve MLP parameters; none for the jitter).  When
    `origins` / `directions` require grad, the backward also returns their gradients (tn_render_train_backward_saved, DESIGN §4.8:
    the sample distances held fixed, as nerfstudio's samplers feed a camera optimizer), so a pose correction upstream of the rays learns.
    The renderer must already hold the current field / weights (FusedRenderer.set_field / set_weights).  Every call keeps its own
    saved state (~115 MB at 8192 rays x 257 fine samples, freed with the graph), so calls compose like any autograd op: several
    forwards before one backward, other renders in between, retain_graph.  A backward after an in-place change of the field or a
    parameter, or after set_field / set_weights on the renderer, raises RuntimeError.

    An optional 13th tensor after the twelve parameters is the mesh's vertex positions f32[V,3], the very tensor the tracer borrowed
    (load_tetrahedra / update_vertices); when it requires grad the backward returns its gradient too (DESIGN §4.9: the sample distances
    and the matched tetrahedra held fixed), so an optimizer can move the points.  It raises if the tensor changed in place since the
    tracer was loaded or refit (the trace would be stale), and an in-place change of it before the backward raises, as for the field.

    An optional last tensor, after the vertex positions when they are given, is the background map f32[H,2H,3] the renderer holds
    (set_background; DESIGN §4.16); when it requires grad the backward returns its gradient too, and an in-place change of it before the
    backward raises.  The same trailing tensors, and the same rules, apply to FusedTrainRenderDepth and FusedTrainRenderDistortion."""

    @staticmethod
    def forward(ctx, fr, settings, use_gradient_scaling, origins, directions, jitter_coarse, jitter_fine, field, *params):
        out = _fused_forward(ctx, "FusedTrainRender", False, fr, settings, use_gradient_scaling, origins, directions, jitter_coarse,
                             jitter_fine, field, params)
        return out["rgb"], out["accumulation"], out["depth"], out["ray_mask"]

    @staticmethod
    def backward(ctx, g_rgb, g_acc, _g_depth, _g_mask):
        return _fused_backward(ctx, g_rgb, g_acc, None)


class FusedTrainRenderDepth(torch.autograd.Function):
    """FusedTrainRender with the expected depth (DESIGN §4.10): the same arguments (the optional vertex positions included), outputs
    (rgb, accumulation, depth, expected_depth, ray_mask) with expected_depth f32[R,1] nerfstudio's DepthRenderer(method="expected") over
    the fine samples (clipped to the call's smallest / largest sample midpoint, far_plane on empty rays).  rgb, accumulation and
    expected_depth are differentiable: a depth loss reaches the field, the MLP and, when they require grad, the ray origins / directions
    and the vertex positions (tn_render_train_forward_saved / tn_render_train_backward_saved).  The other outputs are the
    same bits as FusedTrainRender's."""

    @staticmethod
    def forward(ctx, fr, settings, use_gradient_scaling, origins, directions, jitter_coarse, jitter_fine, field, *params):
        out = _fused_forward(ctx, "FusedTrainRenderDepth", True, fr, settings, use_gradient_scaling, origins, directions, jitter_coarse,
                             jitter_fine, field, params)
        return out["rgb"], out["accumulation"], out["depth"], out["expected_depth"], out["ray_mask"]

    @staticmethod
    def backward(ctx, g_rgb, g_acc, _g_depth, g_ed, _g_mask):
        return _fused_backward(ctx, g_rgb, g_acc, g_ed)


class FusedTrainRenderDistortion(torch.autograd.Function):
    """FusedTrainRender with the distortion loss per ray (DESIGN §4.11), and the expected depth when asked.  Arguments: those of
    FusedTrainRender (the optional vertex positions included) with a flag `expected_depth` after use_gradient_scaling.  Outputs
    (rgb, accumulation, depth, distortion, ray_mask), or (rgb, accumulation, depth, expected_depth, distortion, ray_mask) with
    expected_depth=True; distortion f32[R,1] is FusedRenderer.train_distortion, 0 on empty rays.  rgb, accumulation, expected_depth and
    distortion are differentiable: a distortion loss reaches the field, the MLP and, when they require grad, the ray origins / directions
    and the vertex positions, with the spacing bins held fixed.  The other outputs are the same bits as FusedTrainRender's."""

    @staticmethod
    def forward(ctx, fr, settings, use_gradient_scaling, expected_depth, origins, directions, jitter_coarse, jitter_fine, field, *params):
        out = _fused_forward(ctx, "FusedTrainRenderDistortion", expected_depth, fr, settings, use_gradient_scaling, origins, directions,
                             jitter_coarse, jitter_fine, field, params, first=4)
        dist = fr.train_distortion(ctx.state)
        ctx.ed = bool(expected_depth)
        ed = (out["expected_depth"],) if expected_depth else ()
        return (out["rgb"], out["accumulation"], out["depth"], *ed, dist, out["ray_mask"])

    @staticmethod
    def backward(ctx, g_rgb, g_acc, _g_depth, *rest):
        g_ed, g_dist = (rest[0], rest[1]) if ctx.ed else (None, rest[0])
        return _fused_backward(ctx, g_rgb, g_acc, g_ed, g_dist)


class FieldSmoothness(torch.autograd.Function):
    """mult * S / (E * 64) as one differentiable op (FusedRenderer.field_smoothness; DESIGN §4.15), a float32 scalar: S the sum over the
    mesh's unique undirected edges of the squared feature differences, E their number.  Arguments (fr, mult, field): the renderer must
    already hold `field` as its current field (set_field), which is what the kernel reads; `field` is passed so that autograd routes the
    gradient to it.  The forward computes the gradient in the same pass; the backward scales it by the incoming scalar.  An in-place
    change of `field` before the backward raises RuntimeError."""

    @staticmethod
    def forward(ctx, fr, mult, field):
        if tuple(field.shape) != (64, fr.tracer._vertices.shape[0] if fr.tracer._vertices is not None else -1):
            raise RuntimeError(f"FieldSmoothness: the field must be [64, V] for the tracer's V vertices, got {tuple(field.shape)}")
        S, E, g = fr.field_smoothness(mult, grad=ctx.needs_input_grad[2])
        ctx.g = g
        ctx.save_for_backward(field)  # its version counter rejects a backward after an in-place change
        return (S * (float(mult) / (E * 64) if E > 0 else 0.0)).to(torch.float32)

    @staticmethod
    def backward(ctx, g_loss):
        _ = ctx.saved_tensors  # raises if the field changed in place since the forward
        return None, None, ctx.g * g_loss


def _fused_forward(ctx, name, expected_depth, fr, settings, use_gradient_scaling, origins, directions, jitter_coarse, jitter_fine, field, params,
                   first=3):
    """forward of FusedTrainRender / FusedTrainRenderDepth / FusedTrainRenderDistortion: checks the optional vertex positions, runs the
    saved training forward and keeps what the backward needs in ctx -> the forward's outputs.  `first`: the index of `origins` among the
    op's arguments"""
    bg = None
    if len(params) > len(PARAM_ORDER) and params[-1].dim() == 3:  # the background map
        bg, params = params[-1], params[:-1]
        if fr._bg is None or bg.data_ptr() != fr._bg.data_ptr() or bg.shape != fr._bg.shape:
            raise RuntimeError(f"{name}: the background map must be the tensor the renderer holds (set_background)")
    if len(params) == len(PARAM_ORDER) + 1:
        xyz, borrowed = params[-1], fr.tracer._vertices
        if borrowed is None or xyz.data_ptr() != borrowed.data_ptr() or xyz.shape != borrowed.shape:
            raise RuntimeError(f"{name}: the vertex positions must be the tensor the tracer borrowed (load_tetrahedra / "
                               "update_vertices), with the same number of vertices")
        if xyz._version != fr.tracer._vertices_version:  # (a detached view shares the parameter's version counter)
            raise RuntimeError(f"{name}: the vertex positions changed in place since the tracer was loaded or refit; call "
                               "update_vertices first")
    elif len(params) != len(PARAM_ORDER):
        raise RuntimeError(f"{name} takes the {len(PARAM_ORDER)} MLP parameters and optionally the vertex positions and the background map")
    out, state = fr.train_forward_saved(origins, directions, settings, jitter_coarse, jitter_fine, expected_depth=expected_depth)
    ctx.fr, ctx.state, ctx.gs, ctx.first = fr, state, bool(use_gradient_scaling), first
    ctx.ray_shapes = (origins.shape, directions.shape)
    ctx.has_xyz, ctx.has_bg = len(params) == len(PARAM_ORDER) + 1, bg is not None
    ctx.save_for_backward(field, *params, *((bg,) if bg is not None else ()))  # their version counters reject a backward after an in-place change
    ctx.mark_non_differentiable(out["depth"], out["ray_mask"])
    return out


def _fused_backward(ctx, g_rgb, g_acc, g_ed, g_dist=None):
    """backward of FusedTrainRender / FusedTrainRenderDepth / FusedTrainRenderDistortion (g_ed, g_dist: the expected depth's and the
    distortion's gradients, or None)"""
    field = ctx.saved_tensors[0]
    if g_rgb is None:
        g_rgb = torch.zeros((ctx.state.R, 3), dtype=torch.float32, device=field.device)
    first = ctx.first
    want_o, want_d = ctx.needs_input_grad[first], ctx.needs_input_grad[first + 1]
    has_xyz, has_bg = ctx.has_xyz, ctx.has_bg
    want_v = has_xyz and ctx.needs_input_grad[first + 5 + len(PARAM_ORDER)]
    want_bg = has_bg and ctx.needs_input_grad[-1]
    g_acc = g_acc.reshape(-1) if g_acc is not None else None
    g_ed = g_ed.reshape(-1) if g_ed is not None else None
    g_dist = g_dist.reshape(-1) if g_dist is not None else None
    res = ctx.fr.train_backward_saved(ctx.state, g_rgb, g_acc, field.shape[1], ctx.gs, grad_origins=want_o, grad_directions=want_d,
                                      grad_vertices=want_v, grad_expected_depth=g_ed, grad_distortion=g_dist, grad_background=want_bg)
    gfield, gp, go, gd, gv, gbg = res + (None,) * (6 - len(res))
    go = go.reshape(ctx.ray_shapes[0]) if go is not None else None
    gd = gd.reshape(ctx.ray_shapes[1]) if gd is not None else None
    return (None,) * first + (go, gd, None, None, gfield) + tuple(gp[n] for n in PARAM_ORDER) + ((gv,) if has_xyz else ()) \
        + ((gbg,) if has_bg else ())
