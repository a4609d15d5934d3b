"""`tetranerf_cpp_extension` -- the reference's pybind surface (src/py_binding.cpp:433-449) as a thin
ctypes shim over the C ABI of include/tetranerf_b200.h (csrc/libtetranerf_b200.so).

Same class / function names, argument checks and error behaviour (RuntimeError) as the reference
binding; tensors in, tensors out.  All device work is hand-written CUDA in the shared library, launched
on torch's current stream; there is no CPU fallback (importing this module without the built library
raises, and a non-CUDA device raises exactly like py_binding.cpp:31-33).

This module is where the package declares the C ABI to ctypes: the signatures of every entry point it calls, including the
fused-render ones that tetranerf.b200.render calls through `_lib`.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parents[3]  # .../tetra-nerf_b200
_LIB_PATH = Path(os.environ.get("TETRANERF_B200_LIB", _PKG / "csrc" / "libtetranerf_b200.so"))
if not _LIB_PATH.exists():
    raise ImportError(f"{_LIB_PATH} not found: run `python tetra-nerf_b200/build.py` (nvcc, sm_90a)")
_lib = C.CDLL(str(_LIB_PATH))

_vp, _u32, _i = C.c_void_p, C.c_uint32, C.c_int
_lib.tn_last_error.restype = C.c_char_p
_lib.tn_create.argtypes = [_i, C.POINTER(_vp)]
_lib.tn_destroy.argtypes = [_vp]
_lib.tn_synchronize.argtypes = [_vp, _vp]
_lib.tn_load_tetrahedra.argtypes = [_vp, _vp, _u32, _vp, _u32, _vp]
_lib.tn_update_vertices.argtypes = [_vp, _vp, _u32, C.POINTER(_u32), C.POINTER(_i), _vp]
_lib.tn_guard_vertex_step.argtypes = [_vp, _vp, _vp, _u32, _u32, C.POINTER(_u32 * 3), _vp]
_lib.tn_num_faces.argtypes = [_vp, C.POINTER(_u32)]
_lib.tn_get_faces.argtypes = [_vp, _vp, _vp, _vp]
_lib.tn_trace_rays.argtypes = [_vp, _vp, _vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _i, _vp]
_lib.tn_trace_rays_triangles.argtypes = [_vp, _vp, _vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp]
_lib.tn_find_tetrahedra.argtypes = [_vp, _vp, _u32, _vp, _vp, _vp, _vp]
_lib.tn_find_visited_cells.argtypes = [_vp, _u32, _u32, _u32] + [_vp] * 11
_lib.tn_interpolate_values_backward.argtypes = [_i, _u32, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp]
_lib.tn_interpolate_values_backward_deterministic.argtypes = [_i, _u32, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp, C.POINTER(C.c_size_t), _vp]
_lib.tn_make_field_shadow.argtypes = [_i, _u32, _u32, _vp, _vp, _vp]
_lib.tn_interpolate_values_shadow.argtypes = [_i, _u32, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp]
_lib.tn_debug_trace_stats.argtypes = [_vp, C.POINTER(_u32)]
_lib.tn_set_walk_min_rays.argtypes = [_vp, _u32]
_lib.tn_set_walk_solo_range.argtypes = [_vp, _u32, _u32]
_lib.tn_set_walk_quad_range.argtypes = [_vp, _u32, _u32]
_lib.tn_set_walk_quad_spec_max_rays.argtypes = [_vp, _u32]
_lib.tn_launch_count.restype = C.c_uint64
_lib.tn_launch_count.argtypes = [_vp]
_lib.tn_debug_device_bytes.restype = C.c_uint64


class _Cfg(C.Structure):  # tn_render_config
    _fields_ = [("max_ray_triangles", C.c_uint32), ("num_samples", C.c_uint32), ("num_fine_samples", C.c_uint32),
                ("use_biased_sampler", C.c_uint32), ("far_plane", C.c_float), ("background", C.c_float * 3)]


_lib.tn_render_set_field.argtypes = [_vp, _vp, _u32, _u32, _vp]
_lib.tn_render_set_weights.argtypes = [_vp, C.POINTER(_vp), _vp]
_lib.tn_render.argtypes = [_vp, C.POINTER(_Cfg), _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
_lib.tn_render_debug_normals_grad.argtypes = [_vp, C.POINTER(_vp)]
_lib.tn_render_debug_ray_grads.argtypes = [_vp, C.POINTER(_vp)]
_lib.tn_render_train_forward.argtypes = [_vp, C.POINTER(_Cfg), _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
_lib.tn_render_train_backward.argtypes = [_vp, _vp, _vp, _i, _vp, C.POINTER(_vp), _vp]
_lib.tn_render_train_saved_bytes.argtypes = [_vp, C.POINTER(_Cfg), _u32, C.POINTER(C.c_size_t)]
_lib.tn_render_train_forward_saved.argtypes = [_vp, C.POINTER(_Cfg), _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t, _vp]
_lib.tn_render_train_backward_saved.argtypes = [_vp, _vp, _vp, _vp, _vp, _i, _vp, C.POINTER(_vp), _vp, _vp, _vp, _vp]
_lib.tn_render_train_backward_saved2.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, C.POINTER(_vp), _vp, _vp, _vp, _vp]
_lib.tn_render_train_distortion.argtypes = [_vp, _vp, _vp, _vp]
_lib.tn_render_train_backward_saved3.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, C.POINTER(_vp), _vp, _vp, _vp, _vp, _vp]
_lib.tn_render_set_background.argtypes = [_vp, _vp, _u32, _u32]
_lib.tn_render_debug_buffers.argtypes = [_vp, C.POINTER(_vp)]
_lib.tn_render_set_profiling.argtypes = [_vp, _i]
_lib.tn_render_set_mlp_precision.argtypes = [_vp, _i]
_lib.tn_render_get_timings.argtypes = [_vp, C.POINTER(C.c_float)]
_lib.tn_render_get_backward_timings.argtypes = [_vp, C.POINTER(C.c_float)]
_lib.tn_render_set_deterministic.argtypes = [_vp, _i]
_lib.tn_render_set_backward_grid.argtypes = [_vp, _u32]
_lib.tn_surface_extract.argtypes = [_vp, C.c_float, C.POINTER(_u32), C.POINTER(_u32), _vp]
_lib.tn_surface_copy.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp]
_lib.tn_occupancy_update.argtypes = [_vp, _vp, C.c_float, _vp]
_lib.tn_render_set_occupancy.argtypes = [_vp, _vp, C.c_float]
_lib.tn_render_set_occupancy2.argtypes = [_vp, _vp, C.c_float, _i]
_lib.tn_field_smoothness.argtypes = [_vp, C.c_float, _vp, _vp, C.POINTER(_u32), _vp]
_lib.tn_refine_edges.argtypes = [_i, _vp, _u32, _vp, _u32, _vp, C.c_float, _u32, _vp, _vp, _vp, C.POINTER(_u32), _vp, C.POINTER(C.c_size_t), _vp]
_lib.tn_coarsen_vertices.argtypes = [_i, _vp, _u32, _vp, _u32, _vp, _u32, _vp, _vp, _vp, C.POINTER(_u32), _vp, C.POINTER(C.c_size_t), _vp]
_lib.tn_flip_delaunay.argtypes = [_i, _vp, _u32, _vp, _u32, _u32, _vp, _vp, C.POINTER(_u32), _vp, C.POINTER(C.c_size_t), _vp]

LIBRARY_PATH = str(_LIB_PATH)


def _check(rc: int):
    if rc != 0:
        raise RuntimeError(_lib.tn_last_error().decode("utf-8", "replace"))


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def deterministic_enabled() -> bool:
    """Whether the custom ops run in their bitwise-reproducible mode: `torch.use_deterministic_algorithms(True)` or the environment
    variable TETRANERF_B200_DETERMINISTIC=1.  Read on every call."""
    return torch.are_deterministic_algorithms_enabled() or os.environ.get("TETRANERF_B200_DETERMINISTIC", "0") == "1"


def _require(cond: bool, msg: str):
    if not cond:
        raise RuntimeError(msg)


def _check_input(x: torch.Tensor, name: str):  # CHECK_INPUT, py_binding.cpp:15-21
    _require(x.device.type == "cuda", f"{name} must be a CUDA tensor")
    _require(x.is_contiguous(), f"{name} must be contiguous")


class TetrahedraTracer:
    """py_binding.cpp:28-227."""

    def __init__(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("The device argument must be a CUDA device.")  # py_binding.cpp:31-33
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self._device = device
        self._h = _vp()
        self._vertices = None
        self._vertices_version = None
        self._cells = None
        _check(_lib.tn_create(device.index, C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value and _lib is not None:
            try:
                _lib.tn_destroy(h)
            except Exception:
                pass
            self._h = None
        self._vertices = None
        self._cells = None

    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def handle(self) -> int:
        """Raw tn_tracer* (for the fused-render API in tetranerf.b200)."""
        return self._h.value

    def _check_float_dim3(self, x: torch.Tensor, name: str):  # CHECK_FLOAT_DIM3, py_binding.cpp:22-26
        _check_input(x, name)
        _require(x.device == self._device, f"{name} must be on the same device")
        _require(x.dtype == torch.float32, f"{name} must have float32 type")
        _require(x.size(-1) == 3, f"{name} must have last dimension with size 3")

    def _on_device(self, x: torch.Tensor, name: str):
        _check_input(x, name)
        _require(x.device == self._device, f"{name} must be on the same device")

    # ---- load_tetrahedra (py_binding.cpp:144-161) ------------------------------------------------
    def load_tetrahedra(self, xyz: torch.Tensor, cells: torch.Tensor) -> None:
        self._check_float_dim3(xyz, "xyz")
        self._on_device(cells, "cells")
        _require(cells.size(-1) == 4, "indices must have last dimension with size 4")
        _require(cells.dtype == torch.int32, "indices must have int32 type")
        self._cells, self._vertices = cells, xyz  # borrowed by the tracer: keep them alive (:154-155)
        self._vertices_version = xyz._version  # the positions the tracer holds (FusedTrainRender rejects a stale tracer)
        with torch.cuda.device(self._device):
            _check(_lib.tn_load_tetrahedra(self._h, xyz.data_ptr(), xyz.numel() // 3, cells.data_ptr(), cells.numel() // 4,
                                           _stream(self._device)))

    def update_vertices(self, xyz: torch.Tensor):
        """moves the loaded mesh's vertices to `xyz` f32[V,3] (same V; borrowed like load_tetrahedra's) and refits the tracer in place:
        every trace afterwards equals one after a fresh load_tetrahedra(xyz, cells).  -> (folded_faces, walkable): the number of interior
        faces that are folded or not certified unfolded, and whether the adjacency walk stays on (otherwise every trace takes the
        all-hits gather).  Raises RuntimeError on a different V or a non-finite coordinate (the tracer is then unchanged).  Waits until the
        stream has reached it.  DESIGN §4.9"""
        self._check_float_dim3(xyz, "xyz")
        _require(self._cells is not None, "load_tetrahedra must be called first")
        folded, walkable = _u32(0), _i(0)
        with torch.cuda.device(self._device):
            _check(_lib.tn_update_vertices(self._h, xyz.data_ptr(), xyz.numel() // 3, C.byref(folded), C.byref(walkable), _stream(self._device)))
        self._vertices, self._vertices_version = xyz, xyz._version
        return int(folded.value), bool(walkable.value)

    def guard_vertex_step(self, old: torch.Tensor, new: torch.Tensor, max_halvings: int = 8):
        """the fold guard of a vertex step (DESIGN §4.17): scales back, in place in `new` f32[V,3], each vertex's move from `old` f32[V,3]
        (the positions the tracer was last loaded or refit at, typically) that would fold an interior face certified unfolded at `old`, or,
        on a mesh walkable at `old`, break the hull's convexity.  A moving vertex ends at `new` (bitwise), at old + (new - old) * 2^-k for
        some 1 <= k <= max_halvings, or back at `old` (bitwise); if nothing would fold, `new` is unchanged.  update_vertices(new) then
        reports only the faces already uncertified at `old`, and the walk stays on if it was on at `old`.  Uses the loaded mesh's topology;
        nothing is borrowed.  -> (limited, frozen, rounds): vertices scaled back, vertices moved back to `old`, rounds run.  Raises
        RuntimeError without a loaded mesh, on another V, a non-finite coordinate (`new` is then unchanged) or max_halvings > 23.  Waits
        until the stream has reached it; bumps `new`'s version counter when it changed it."""
        self._check_float_dim3(old, "old")
        self._check_float_dim3(new, "new")
        _require(self._cells is not None, "load_tetrahedra must be called first")
        _require(old.numel() == new.numel(), "old and new must have the same shape")
        counts = (_u32 * 3)()
        with torch.cuda.device(self._device):
            _check(_lib.tn_guard_vertex_step(self._h, old.data_ptr(), new.data_ptr(), new.numel() // 3, int(max_halvings), C.byref(counts),
                                             _stream(self._device)))
        limited, frozen, rounds = (int(x) for x in counts)
        if limited or frozen:
            torch.autograd.graph.increment_version(new)
        return limited, frozen, rounds

    def num_faces(self) -> int:
        n = _u32(0)
        _check(_lib.tn_num_faces(self._h, C.byref(n)))
        return int(n.value)

    def get_faces(self):
        """(triangle_indices i32[F,3], triangle_tetrahedra i32[F,2]) in reference numbering
        (src/tetrahedra_tracer.cpp:45-71); exposed for parity tests."""
        F = self.num_faces()
        tri = torch.empty((F, 3), dtype=torch.int32, device=self._device)
        tt = torch.empty((F, 2), dtype=torch.int32, device=self._device)
        _check(_lib.tn_get_faces(self._h, tri.data_ptr(), tt.data_ptr(), _stream(self._device)))
        return tri, tt

    def synchronize(self) -> None:
        """Stream sync + deferred device-side error check (the reference syncs on every call,
        src/tetrahedra_tracer.cpp:173-174; here it is explicit)."""
        _check(_lib.tn_synchronize(self._h, _stream(self._device)))

    def set_walk_min_rays(self, n: int) -> None:
        """batches of >= n rays use the adjacency-walk implementation of trace_rays (0 = always, 2**32-1 = never)"""
        _check(_lib.tn_set_walk_min_rays(self._h, int(n)))

    def set_walk_solo_range(self, lo: int, hi: int) -> None:
        """batches below walk_min_rays with lo <= rays <= hi use the one-ray-per-warp form of the walk (lo > hi = never)"""
        _check(_lib.tn_set_walk_solo_range(self._h, int(lo), int(hi)))

    def set_walk_quad_range(self, lo: int, hi: int) -> None:
        """batches below walk_min_rays with lo <= rays <= hi use the 8-rays-per-warp form of the walk (lo > hi = never); checked before the solo range"""
        _check(_lib.tn_set_walk_quad_range(self._h, int(lo), int(hi)))

    def set_walk_quad_spec_max_rays(self, n: int) -> None:
        """quad and solo walks: batches of up to n rays load all candidate next records speculatively instead of prefetching them (0 = never)"""
        _check(_lib.tn_set_walk_quad_spec_max_rays(self._h, int(n)))

    def trace_stats(self):
        """(walkable mesh?, rays of the last trace_rays that took the exact stage) -- test/diagnostic hook"""
        out = (_u32 * 2)()
        _check(_lib.tn_debug_trace_stats(self._h, out))
        return bool(out[0]), int(out[1])

    def launch_count(self) -> int:
        return int(_lib.tn_launch_count(self._h))

    # ---- trace_rays (py_binding.cpp:41-76) ------------------------------------------------------
    def trace_rays(self, ray_origins: torch.Tensor, ray_directions: torch.Tensor, max_ray_triangles: int):
        M = int(max_ray_triangles)
        if M <= 0 or (M & (M - 1)) != 0:
            raise RuntimeError("max_ray_triangles must be a power of 2.")
        self._check_float_dim3(ray_origins, "ray_origins")
        self._check_float_dim3(ray_directions, "ray_directions")
        R = ray_origins.numel() // 3
        dev = self._device
        with torch.no_grad():
            num = torch.empty((R,), dtype=torch.int32, device=dev)
            cells = torch.empty((R, M), dtype=torch.int32, device=dev)
            bary = torch.empty((R, M, 2, 3), dtype=torch.float32, device=dev)
            dist = torch.empty((R, M, 2), dtype=torch.float32, device=dev)
            verts = torch.empty((R, M, 4), dtype=torch.int32, device=dev)
            _check(_lib.tn_trace_rays(self._h, ray_origins.data_ptr(), ray_directions.data_ptr(), R, M, num.data_ptr(), cells.data_ptr(),
                                      bary.data_ptr(), dist.data_ptr(), verts.data_ptr(), 1, _stream(dev)))
        return {
            "num_visited_cells": num,
            "visited_cells": cells,
            "barycentric_coordinates": bary,
            "vertex_indices": verts,
            "hit_distances": dist,
        }

    def trace_rays_into(self, ray_origins, ray_directions, max_ray_triangles: int, out: dict, dense: bool = False):
        """trace_rays into caller-provided tensors (same keys/shapes as trace_rays); dense=False skips the tail fill
        (entries >= num_visited_cells are left untouched) -- the form the fused renderer uses; for benchmarking."""
        M = int(max_ray_triangles)
        R = ray_origins.numel() // 3
        _check(_lib.tn_trace_rays(self._h, ray_origins.data_ptr(), ray_directions.data_ptr(), R, M, out["num_visited_cells"].data_ptr(),
                                  out["visited_cells"].data_ptr(), out["barycentric_coordinates"].data_ptr(), out["hit_distances"].data_ptr(),
                                  out["vertex_indices"].data_ptr(), int(dense), _stream(self._device)))
        return out

    # ---- trace_rays_triangles (py_binding.cpp:78-113) --------------------------------------------
    def trace_rays_triangles(self, ray_origins: torch.Tensor, ray_directions: torch.Tensor, max_ray_triangles: int):
        M = int(max_ray_triangles)
        if M <= 0 or (M & (M - 1)) != 0:
            raise RuntimeError("max_ray_triangles must be a power of 2.")
        self._check_float_dim3(ray_origins, "ray_origins")
        self._check_float_dim3(ray_directions, "ray_directions")
        R = ray_origins.numel() // 3
        dev = self._device
        with torch.no_grad():
            num = torch.empty((R,), dtype=torch.int32, device=dev)
            faces = torch.empty((R, M), dtype=torch.int32, device=dev)
            bary = torch.empty((R, M, 2), dtype=torch.float32, device=dev)
            dist = torch.empty((R, M), dtype=torch.float32, device=dev)
            verts = torch.empty((R, M, 3), dtype=torch.int32, device=dev)
            _check(_lib.tn_trace_rays_triangles(self._h, ray_origins.data_ptr(), ray_directions.data_ptr(), R, M, num.data_ptr(),
                                                faces.data_ptr(), bary.data_ptr(), dist.data_ptr(), verts.data_ptr(), _stream(dev)))
        return {
            "num_visited_triangles": num,
            "visited_triangles": faces,
            "barycentric_coordinates": bary,
            "vertex_indices": verts,
            "hit_distances": dist,
        }

    # ---- find_tetrahedra (py_binding.cpp:115-142) ------------------------------------------------
    def find_tetrahedra(self, positions: torch.Tensor):
        self._check_float_dim3(positions, "positions")
        N = positions.numel() // 3
        shape = list(positions.shape)
        dev = self._device
        with torch.no_grad():
            bary = torch.empty(shape, dtype=torch.float32, device=dev)
            verts = torch.empty(shape[:-1] + [4], dtype=torch.int32, device=dev)
            tet = torch.empty(shape[:-1], dtype=torch.int32, device=dev)
            _check(_lib.tn_find_tetrahedra(self._h, positions.data_ptr(), N, tet.data_ptr(), bary.data_ptr(), verts.data_ptr(), _stream(dev)))
        return {"tetrahedra": tet, "barycentric_coordinates": bary, "vertex_indices": verts, "valid_mask": tet != -1}

    # ---- find_visited_cells (py_binding.cpp:163-216) ---------------------------------------------
    def find_visited_cells(self, num_visited_cells, visited_cells, barycentric_coordinates, hit_distances, vertex_indices, distances):
        for x, n in ((num_visited_cells, "num_visited_cells"), (visited_cells, "visited_cells"),
                     (barycentric_coordinates, "barycentric_coordinates"), (hit_distances, "hit_distances"),
                     (distances, "distances"), (vertex_indices, "vertex_indices")):
            self._on_device(x, n)
        _require(distances.dtype == torch.float32, "distances must have float32 type")
        R = num_visited_cells.size(0)
        _require(distances.dim() == 2 and distances.size(0) == R, "distances must be of [num_rays, num_samples_per_ray] shape")
        _require(vertex_indices.size(-1) == 4, "vertex_indices must have last dimension with size 4")
        _require(self._vertices is not None, "load_tetrahedra must be called first")
        S = distances.size(-1)
        M = visited_cells.size(1)
        dev = self._device
        mask = torch.empty((R, S), dtype=torch.bool, device=dev)
        matched = torch.empty((R, S), dtype=torch.int32, device=dev)
        bary_out = torch.empty((R, S, 3), dtype=torch.float32, device=dev)
        verts_out = torch.empty((R, S, 4), dtype=torch.int32, device=dev)
        _check(_lib.tn_find_visited_cells(self._h, R, S, M, num_visited_cells.data_ptr(), visited_cells.data_ptr(),
                                          barycentric_coordinates.data_ptr(), hit_distances.data_ptr(), vertex_indices.data_ptr(),
                                          distances.data_ptr(), matched.data_ptr(), verts_out.data_ptr(), mask.data_ptr(),
                                          bary_out.data_ptr(), _stream(dev)))
        return {"cell_indices": matched, "vertex_indices": verts_out, "mask": mask, "barycentric_coordinates": bary_out}


# ---- interpolate_values (py_binding.cpp:298-339) ----------------------------------------------------
def interpolate_values(vertex_indices: torch.Tensor, barycentric_coordinates: torch.Tensor, field: torch.Tensor) -> torch.Tensor:
    _check_input(vertex_indices, "vertex_indices")
    _check_input(barycentric_coordinates, "barycentric_coordinates")
    _check_input(field, "field")
    _require(vertex_indices.dtype == torch.int32, "vertex_indices must be a tensor of type int32")
    _require(barycentric_coordinates.dtype == torch.float32, "barycentric_coordinates must be a tensor of type float32")
    _require(barycentric_coordinates.size(-1) + 1 == vertex_indices.size(-1),
             "barycentric_coordinates must have the same last dimension as vertex_indices - 1")
    _require(field.dtype == torch.float32, "field must be a tensor of type float32")
    D = vertex_indices.size(-1)
    if D not in (2, 3, 4, 6):
        raise RuntimeError(f"Unsupported interpolation dimension with value {D}")  # py_binding.cpp:273-275
    N = vertex_indices.numel() // D
    Cdim, V = field.size(0), field.size(-1)
    dev = field.device
    out = torch.empty(list(vertex_indices.shape[:-1]) + [Cdim], dtype=torch.float32, device=dev)
    shadow = _field_shadow(field)
    _check(_lib.tn_interpolate_values_shadow(dev.index, D, N, Cdim, V, vertex_indices.data_ptr(), barycentric_coordinates.data_ptr(),
                                             shadow.data_ptr(), out.data_ptr(), _stream(dev)))
    return out


_SHADOW = {}  # device -> (key, [V,C] shadow): one entry per device, rebuilt when the field's storage, shape or version changes


def _field_shadow(field: torch.Tensor) -> torch.Tensor:
    """[V,C] row-major shadow of the feature-major field, cached by (storage, shape, version): the two interpolations of a
    training step (coarse + fine pass) and repeated evaluation calls share one transposition."""
    dev = field.device
    key = (field.data_ptr(), tuple(field.shape), field._version)
    hit = _SHADOW.get(dev)
    if hit is not None and hit[0] == key:
        return hit[1]
    Cdim, V = field.size(0), field.size(-1)
    shadow = hit[1] if hit is not None and hit[1].shape == (V, Cdim) else torch.empty((V, Cdim), dtype=torch.float32, device=dev)
    _check(_lib.tn_make_field_shadow(dev.index, Cdim, V, field.data_ptr(), shadow.data_ptr(), _stream(dev)))
    _SHADOW[dev] = (key, shadow)
    return shadow


# ---- interpolate_values_backward (py_binding.cpp:341-372) -------------------------------------------
def interpolate_values_backward(vertex_indices, barycentric_coordinates, field, grad_in) -> torch.Tensor:
    for x, n in ((vertex_indices, "vertex_indices"), (barycentric_coordinates, "barycentric_coordinates"), (field, "field"), (grad_in, "grad_in")):
        _check_input(x, n)
    _require(vertex_indices.dtype == torch.int32, "vertex_indices must be a tensor of type int32")
    _require(barycentric_coordinates.dtype == torch.float32, "barycentric_coordinates must be a tensor of type float32")
    _require(field.dtype == torch.float32, "field must be a tensor of type float32")
    _require(grad_in.dtype == torch.float32, "grad_in must be a tensor of type float32")
    _require(barycentric_coordinates.size(-1) + 1 == vertex_indices.size(-1),
             "barycentric_coordinates must have the same last dimension as vertex_indices - 1")
    D = vertex_indices.size(-1)
    if D not in (2, 3, 4, 6):
        raise RuntimeError(f"Unsupported interpolation dimension with value {D}")
    N = vertex_indices.numel() // D
    Cdim, V = field.size(0), field.size(-1)
    _require(grad_in.size(-1) == Cdim, "grad_in must have shape [..., field_dim]")
    dev = grad_in.device
    grad_field = torch.empty((Cdim, V), dtype=torch.float32, device=dev)
    grad_in = grad_in.contiguous()
    if deterministic_enabled():  # sorted by vertex, summed in input order: bitwise reproducible
        nbytes = C.c_size_t(0)
        args = (dev.index, D, N, Cdim, V, vertex_indices.data_ptr(), barycentric_coordinates.data_ptr(), grad_in.data_ptr(), grad_field.data_ptr())
        _check(_lib.tn_interpolate_values_backward_deterministic(*args, None, C.byref(nbytes), _stream(dev)))
        workspace = torch.empty((max(int(nbytes.value), 1),), dtype=torch.uint8, device=dev)
        _check(_lib.tn_interpolate_values_backward_deterministic(*args, workspace.data_ptr(), C.byref(nbytes), _stream(dev)))
        return grad_field
    # row-major [V,C] accumulator for the vector-reduction path (worth it once there is more than a handful of samples)
    scratch = torch.empty((V, Cdim), dtype=torch.float32, device=dev) if (Cdim % 4 == 0 and N >= 1024) else None
    _check(_lib.tn_interpolate_values_backward(dev.index, D, N, Cdim, V, vertex_indices.data_ptr(), barycentric_coordinates.data_ptr(),
                                               grad_in.data_ptr(), grad_field.data_ptr(), scratch.data_ptr() if scratch is not None else None,
                                               _stream(dev)))
    return grad_field


# ---- out of the hot-path scope (SURVEY.md §2): CGAL preprocessing and the unused occupancy remnants ----
def triangulate(points: torch.Tensor) -> torch.Tensor:
    """The reference calls CGAL (src/triangulation.cpp:34-75), offline preprocessing outside this path.
    Provided through scipy's Qhull Delaunay so that `_load_points_from_metadata` (model.py:302-306) works."""
    _require(points.dim() == 2 and points.size(1) == 3, "points must have shape [num_points, 3]")
    from scipy.spatial import Delaunay

    cells = Delaunay(points.detach().cpu().double().numpy()).simplices
    return torch.from_numpy(cells).to(torch.int32).to(points.device)


def find_average_spacing(points: torch.Tensor) -> float:
    raise RuntimeError("find_average_spacing (CGAL, src/triangulation.cpp:121-134) is outside this project's hot-path scope")


def gather_uint32(self: torch.Tensor, dim: int, index: torch.Tensor) -> torch.Tensor:
    raise RuntimeError("gather_uint32 (occupancy-field remnant, unused by the model) is outside this project's hot-path scope")


def scatter_ema_uint32(self, dim, index, decay, values) -> None:
    raise RuntimeError("scatter_ema_uint32 (occupancy-field remnant, unused by the model) is outside this project's hot-path scope")
