"""CPU oracle for the Tetra-NeRF ray-sampling hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product (tetra-nerf_b200/) never does.

Two halves:
  * ctypes bindings onto oracle/_build/liboracle.so (tetra_oracle.cpp): faces, trace_rays,
    find_visited_cells, interpolate_values(+backward), trace_rays_triangles, find_tetrahedra.
  * a torch-CPU fp32 restatement of the Python/nerfstudio part of the path
    (tetranerf/nerfstudio/model.py:111-122,141-192,520-662 plus the un-vendored nerfstudio 0.3.x
    pieces it calls: MLP, NeRFEncoding, DensityFieldHead, RGBFieldHead, UniformSampler, PDFSampler,
    RaySamples.get_weights, RGB/Accumulation/DepthRenderer).  nerfstudio is NOT in /root/reference
    (setup.py:133 dependency, Dockerfile:10 pins dromni/nerfstudio:0.3.4); those pieces are
    restated from the published 0.3.x sources and are "parity unpinned" (no reference test covers
    them, SURVEY.md §8c).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass
from pathlib import Path
from typing import Dict, Optional

import numpy as np
import torch

_HERE = Path(__file__).resolve().parent
_LIB: Optional[C.CDLL] = None

u32p = C.POINTER(C.c_uint32)
f32p = C.POINTER(C.c_float)
u8p = C.POINTER(C.c_uint8)


def build(force: bool = False) -> Path:
    """Compile the C++ restatement (and, if /root/reference exists, oracle/_ref)."""
    so = _HERE / "_build" / "liboracle.so"
    src = _HERE / "tetra_oracle.cpp"
    if force or not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(["make", "-C", str(_HERE), "_build/liboracle.so"], check=True, capture_output=True)
    return so


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(str(build()))
        _LIB.orc_mesh_create.restype = C.c_void_p
        _LIB.orc_mesh_create.argtypes = [f32p, C.c_uint32, u32p, C.c_uint32, C.c_int, C.POINTER(C.c_int)]
        _LIB.orc_mesh_destroy.argtypes = [C.c_void_p]
        _LIB.orc_mesh_num_faces.restype = C.c_uint32
        _LIB.orc_mesh_num_faces.argtypes = [C.c_void_p]
        _LIB.orc_mesh_faces.argtypes = [C.c_void_p, u32p, u32p]
        _LIB.orc_ray_tri.argtypes = [f32p] * 6
        _LIB.orc_trace.argtypes = [C.c_void_p, f32p, f32p, C.c_uint32, C.c_uint32, u32p, u32p, f32p, f32p, u32p, C.c_int, C.c_int]
        _LIB.orc_trace_triangles.argtypes = [C.c_void_p, f32p, f32p, C.c_uint32, C.c_uint32, u32p, u32p, f32p, f32p, u32p, C.c_int, C.c_int]
        _LIB.orc_post_process_one.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, u32p, f32p, f32p, u32p, u32p, f32p, f32p, u32p]
        _LIB.orc_match.argtypes = [C.c_uint32] * 3 + [u32p, u32p, f32p, f32p, f32p, u32p, u32p, u32p, u8p, f32p, C.c_int]
        _LIB.orc_match.restype = None
        _LIB.orc_interp_fwd.argtypes = [C.c_uint32] * 4 + [u32p, f32p, f32p, f32p, C.c_int]
        _LIB.orc_interp_fwd.restype = None
        _LIB.orc_interp_bwd.argtypes = [C.c_uint32] * 4 + [u32p, f32p, f32p, f32p]
        _LIB.orc_interp_bwd.restype = None
        _LIB.orc_find_tetrahedra.argtypes = [C.c_void_p, f32p, C.c_uint32, u32p, f32p, u32p, C.c_int, C.c_int]
        _LIB.orc_find_tetrahedra.restype = None
    return _LIB


def _f(a):
    return a.ctypes.data_as(f32p)


def _u(a):
    return a.ctypes.data_as(u32p)


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def hardware_threads() -> int:
    return int(lib().orc_hardware_threads())


class OracleMesh:
    """load_tetrahedra (py_binding.cpp:144-161 -> tetrahedra_tracer.cpp:244-281)."""

    def __init__(self, xyz, cells, accel: bool = True):
        self.xyz = _c(xyz, np.float32).reshape(-1, 3)
        self.cells = _c(cells, np.int32).reshape(-1, 4)
        err = C.c_int(0)
        self.h = lib().orc_mesh_create(_f(self.xyz), len(self.xyz), _u(self.cells.view(np.uint32)), len(self.cells), int(accel), C.byref(err))
        if err.value != 0 or not self.h:
            raise RuntimeError("A triangle is shared by more than two tetrahedra!")  # tetrahedra_tracer.cpp:64-66
        self.accel = accel

    def __del__(self):
        try:
            if getattr(self, "h", None) and _LIB is not None:
                _LIB.orc_mesh_destroy(self.h)
        except Exception:  # interpreter shutdown
            pass
        self.h = None

    @property
    def num_faces(self) -> int:
        return int(lib().orc_mesh_num_faces(self.h))

    def faces(self):
        F = self.num_faces
        tri = np.empty((F, 3), np.uint32)
        tt = np.empty((F, 2), np.uint32)
        lib().orc_mesh_faces(self.h, _u(tri), _u(tt))
        return tri, tt

    def trace_rays(self, origins, directions, M: int, accel: Optional[bool] = None, nthreads: int = 0) -> Dict[str, np.ndarray]:
        o = _c(origins, np.float32).reshape(-1, 3)
        d = _c(directions, np.float32).reshape(-1, 3)
        R = len(o)
        num = np.zeros((R,), np.uint32)
        cells = np.zeros((R, M), np.uint32)
        bary = np.zeros((R, M, 2, 3), np.float32)
        dist = np.zeros((R, M, 2), np.float32)
        verts = np.zeros((R, M, 4), np.uint32)
        rc = lib().orc_trace(self.h, _f(o), _f(d), R, M, _u(num), _u(cells), _f(bary), _f(dist), _u(verts),
                             int(self.accel if accel is None else accel), nthreads)
        if rc != 0:
            raise RuntimeError("max_ray_triangles must be a power of 2.")  # py_binding.cpp:44-47
        return {
            "num_visited_cells": num.view(np.int32),
            "visited_cells": cells.view(np.int32),
            "barycentric_coordinates": bary,
            "vertex_indices": verts.view(np.int32),
            "hit_distances": dist,
        }

    def trace_rays_triangles(self, origins, directions, M: int, accel: Optional[bool] = None, nthreads: int = 0):
        o = _c(origins, np.float32).reshape(-1, 3)
        d = _c(directions, np.float32).reshape(-1, 3)
        R = len(o)
        num = np.zeros((R,), np.uint32)
        faces = np.zeros((R, M), np.uint32)
        bary = np.zeros((R, M, 2), np.float32)
        dist = np.zeros((R, M), np.float32)
        verts = np.zeros((R, M, 3), np.uint32)
        rc = lib().orc_trace_triangles(self.h, _f(o), _f(d), R, M, _u(num), _u(faces), _f(bary), _f(dist), _u(verts),
                                       int(self.accel if accel is None else accel), nthreads)
        if rc != 0:
            raise RuntimeError("max_ray_triangles must be a power of 2.")
        return {
            "num_visited_triangles": num.view(np.int32),
            "visited_triangles": faces.view(np.int32),
            "barycentric_coordinates": bary,
            "vertex_indices": verts.view(np.int32),
            "hit_distances": dist,
        }

    def post_process_one(self, hit_face, hit_t, hit_uv, M: int):
        hf = _c(hit_face, np.uint32)
        ht = _c(hit_t, np.float32)
        huv = _c(hit_uv, np.float32).reshape(-1, 2)
        num = np.zeros((1,), np.uint32)
        cells = np.zeros((M,), np.uint32)
        bary = np.zeros((M, 2, 3), np.float32)
        dist = np.zeros((M, 2), np.float32)
        verts = np.zeros((M, 4), np.uint32)
        rc = lib().orc_post_process_one(self.h, len(hf), M, _u(hf), _f(ht), _f(huv), _u(num), _u(cells), _f(bary), _f(dist), _u(verts))
        assert rc == 0
        return int(num[0]), cells.view(np.int32), bary, dist, verts.view(np.int32)

    def find_tetrahedra(self, positions, accel: Optional[bool] = None, nthreads: int = 0):
        p = _c(positions, np.float32).reshape(-1, 3)
        N = len(p)
        tet = np.zeros((N,), np.uint32)
        bary = np.zeros((N, 3), np.float32)
        verts = np.zeros((N, 4), np.uint32)
        lib().orc_find_tetrahedra(self.h, _f(p), N, _u(tet), _f(bary), _u(verts), int(self.accel if accel is None else accel), nthreads)
        t = tet.view(np.int32)
        return {"tetrahedra": t, "barycentric_coordinates": bary, "vertex_indices": verts.view(np.int32), "valid_mask": t != -1}


def find_visited_cells(num_visited_cells, visited_cells, barycentric_coordinates, hit_distances, vertex_indices, distances, nthreads: int = 0):
    """py_binding.cpp:163-216 -> tetrahedra_tracer.cu:115-161."""
    num = _c(num_visited_cells, np.int32).view(np.uint32)
    cells = _c(visited_cells, np.int32).view(np.uint32)
    bary = _c(barycentric_coordinates, np.float32)
    hd = _c(hit_distances, np.float32)
    vi = _c(vertex_indices, np.int32).view(np.uint32)
    d = _c(distances, np.float32)
    R, S = d.shape
    M = cells.shape[1]
    cell_out = np.empty((R, S), np.uint32)
    verts_out = np.empty((R, S, 4), np.uint32)
    mask = np.empty((R, S), np.uint8)
    bary_out = np.empty((R, S, 3), np.float32)
    lib().orc_match(R, S, M, _u(num), _u(cells), _f(hd), _f(bary), _f(d), _u(vi), _u(cell_out), _u(verts_out),
                    mask.ctypes.data_as(u8p), _f(bary_out), nthreads)
    return {
        "cell_indices": cell_out.view(np.int32),
        "vertex_indices": verts_out.view(np.int32),
        "mask": mask.astype(bool),
        "barycentric_coordinates": bary_out,
    }


def interpolate_values(vertex_indices, barycentric_coordinates, field, nthreads: int = 0) -> np.ndarray:
    """py_binding.cpp:298-339 -> tetrahedra_tracer.cu:195-221.  field is [C, V]; result [..., C]."""
    vi = _c(vertex_indices, np.int32).view(np.uint32)
    w = _c(barycentric_coordinates, np.float32)
    fld = _c(field, np.float32)
    D = vi.shape[-1]
    assert w.shape[-1] + 1 == D
    N = vi.size // D
    Cdim, V = fld.shape
    out = np.empty((N, Cdim), np.float32)
    lib().orc_interp_fwd(D, N, Cdim, V, _u(vi), _f(w), _f(fld), _f(out), nthreads)
    return out.reshape(*vi.shape[:-1], Cdim)


def interpolate_values_backward(vertex_indices, barycentric_coordinates, field_shape, grad_in) -> np.ndarray:
    """py_binding.cpp:341-372 -> tetrahedra_tracer.cu:223-248.  returns [C, V]."""
    vi = _c(vertex_indices, np.int32).view(np.uint32)
    w = _c(barycentric_coordinates, np.float32)
    g = _c(grad_in, np.float32)
    D = vi.shape[-1]
    N = vi.size // D
    Cdim, V = field_shape
    out = np.zeros((Cdim, V), np.float32)
    lib().orc_interp_bwd(D, N, Cdim, V, _u(vi), _f(w), _f(g), _f(out))
    return out


def ray_tri(o, d, p0, p1, p2):
    a = [_c(x, np.float32) for x in (o, d, p0, p1, p2)]
    tuv = np.zeros(3, np.float32)
    hit = lib().orc_ray_tri(*[_f(x) for x in a], _f(tuv))
    return bool(hit), tuv


# =====================================================================================
# torch-CPU restatement of the Python / nerfstudio half of the path
# =====================================================================================


@dataclass
class RenderConfig:
    """The hot-path subset of TetrahedraNerfConfig (model.py:70-107) + collider far plane."""

    max_intersected_triangles: int = 512
    num_samples: int = 256
    num_fine_samples: int = 256
    use_biased_sampler: bool = False
    field_dim: int = 64
    hidden_size: int = 128
    far_plane: float = 6.0  # nerfstudio ModelConfig.collider_params default {"near_plane": 2.0, "far_plane": 6.0}
    background: tuple = (1.0, 1.0, 1.0)  # RGBRenderer background colour (model.py:258): "white" = (1, 1, 1), "black" = (0, 0, 0)

    @staticmethod
    def tetra_nerf():  # registration.py:48-61
        return RenderConfig(num_samples=128, num_fine_samples=128, use_biased_sampler=True)

    @staticmethod
    def tetra_nerf_original():  # registration.py:20-46
        return RenderConfig()


def init_mlp_params(seed: int = 0, field_dim: int = 64, hidden: int = 128) -> Dict[str, torch.Tensor]:
    """torch default nn.Linear init under torch.manual_seed(seed), in module construction order of
    populate_modules (model.py:433-455): mlp_base (3 layers), mlp_head (1 layer), colour head, density head."""
    g = torch.Generator().manual_seed(seed)

    def lin(i, o):
        k = 1.0 / (i**0.5)
        w = (torch.rand((o, i), generator=g) * 2 - 1) * k
        b = (torch.rand((o,), generator=g) * 2 - 1) * k
        return w.float(), b.float()

    p = {}
    p["mlp_base.layers.0.weight"], p["mlp_base.layers.0.bias"] = lin(field_dim, hidden)
    p["mlp_base.layers.1.weight"], p["mlp_base.layers.1.bias"] = lin(hidden, hidden)
    p["mlp_base.layers.2.weight"], p["mlp_base.layers.2.bias"] = lin(hidden, hidden)
    p["mlp_head.layers.0.weight"], p["mlp_head.layers.0.bias"] = lin(hidden + 27, hidden)
    p["field_output_color.net.weight"], p["field_output_color.net.bias"] = lin(hidden, 3)
    p["field_output_density.net.weight"], p["field_output_density.net.bias"] = lin(hidden, 1)
    return p


def nerf_encoding_dirs(dirs: torch.Tensor) -> torch.Tensor:
    """NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0, max_freq_exp=4, include_input=True)
    (model.py:426-432; nerfstudio 0.3.x field_components/encodings.py NeRFEncoding.pytorch_fwd) -> [...,27]."""
    scaled = 2 * torch.pi * dirs
    freqs = 2 ** torch.linspace(0.0, 4.0, 4)
    si = scaled[..., None] * freqs
    si = si.reshape(*si.shape[:-2], -1)
    enc = torch.sin(torch.cat([si, si + torch.pi / 2.0], dim=-1))
    return torch.cat([enc, dirs], dim=-1)


def mlp_base(p, x):  # nerfstudio MLP(in, num_layers=3, width=128, out_activation=ReLU) (model.py:433-438)
    x = torch.relu(torch.nn.functional.linear(x, p["mlp_base.layers.0.weight"], p["mlp_base.layers.0.bias"]))
    x = torch.relu(torch.nn.functional.linear(x, p["mlp_base.layers.1.weight"], p["mlp_base.layers.1.bias"]))
    x = torch.relu(torch.nn.functional.linear(x, p["mlp_base.layers.2.weight"], p["mlp_base.layers.2.bias"]))
    return x


def density_head(p, x):  # DensityFieldHead: Linear(128,1) + Softplus (model.py:455)
    return torch.nn.functional.softplus(torch.nn.functional.linear(x, p["field_output_density.net.weight"], p["field_output_density.net.bias"]))


def color_head(p, base, enc_dir):  # mlp_head (1 layer + ReLU) + RGBFieldHead (Linear+Sigmoid) (model.py:447-454,607-621)
    h = torch.relu(torch.nn.functional.linear(torch.cat([enc_dir, base], dim=-1), p["mlp_head.layers.0.weight"], p["mlp_head.layers.0.bias"]))
    return torch.sigmoid(torch.nn.functional.linear(h, p["field_output_color.net.weight"], p["field_output_color.net.bias"]))


def get_weights(deltas, densities):
    """RaySamples.get_weights (nerfstudio 0.3.x cameras/rays.py).  deltas, densities: [R,S,1]."""
    delta_density = deltas * densities
    alphas = 1 - torch.exp(-delta_density)
    transmittance = torch.cumsum(delta_density[..., :-1, :], dim=-2)
    transmittance = torch.cat([torch.zeros((*transmittance.shape[:1], 1, 1)), transmittance], dim=-2)
    transmittance = torch.exp(-transmittance)
    weights = alphas * transmittance
    return torch.nan_to_num(weights)


def map_from_real_distances_to_biased_with_bounds(num_bounds, bounds, samples):
    """model.py:111-122, literal (out-of-place where the in-place form would alias)."""
    lengths = (bounds[..., 1] - bounds[..., 0]).clamp_min(0)
    bounds_start = bounds[..., 0, 0]
    bounds_end = torch.gather(bounds[..., 1], 1, (num_bounds[:, None] - 1).clamp_min(0)).squeeze(-1)
    unisamples = (samples - bounds_start[..., None]) / (bounds_end - bounds_start)[..., None]
    rest = unisamples * num_bounds[..., None]
    intervals = torch.minimum(rest.floor(), (num_bounds[..., None] - 1).to(rest.dtype)).clamp_min(0)
    rest = rest - intervals
    intervals = intervals.long()
    cum_lengths = torch.cumsum(torch.cat((bounds_start[:, None], lengths), 1), 1)
    return torch.gather(cum_lengths, 1, intervals) + torch.gather(lengths, 1, intervals) * rest


def coarse_bins(cfg: RenderConfig, nears, fars, num_visited, hit_distances, t_rand=None):
    """TetrahedraSampler.generate_ray_samples (model.py:141-192) or nerfstudio UniformSampler.  t_rand = None: eval mode (no
    jitter); t_rand f32[R,S+1] uniform in [0,1): the stratified training bins (model.py:169-174 -- the reference draws it with
    torch.rand; here it is an input so that kernel and oracle consume the same numbers).
    Returns (euclidean_bins [R,S+1], spacing_bins [R,S+1])."""
    S = cfg.num_samples
    bins = torch.linspace(0.0, 1.0, S + 1)[None, ...]
    if t_rand is not None:
        bin_centers = (bins[..., 1:] + bins[..., :-1]) / 2.0
        bin_upper = torch.cat([bin_centers, bins[..., -1:]], -1)
        bin_lower = torch.cat([bins[..., :1], bin_centers], -1)
        bins = bin_lower + (bin_upper - bin_lower) * t_rand
    euclid = bins * fars + (1 - bins) * nears
    if cfg.use_biased_sampler:
        euclid = map_from_real_distances_to_biased_with_bounds(num_visited.long(), hit_distances, euclid)
        bins = (euclid - nears) / (fars - nears)
    else:
        bins = bins.expand(nears.shape[0], -1)
    return euclid, bins


def pdf_bins(cfg: RenderConfig, spacing_bins, weights, nears, fars, histogram_padding=0.01, eps=1e-5, u_rand=None):
    """PDFSampler.generate_ray_samples(include_original=True) (nerfstudio 0.3.x model_components/ray_samplers.py).
    weights [R,S,1].  u_rand = None: eval mode (bin mid-points); u_rand f32[R,Sf+1] uniform in [0,1): train_stratified
    (u = linspace + rand / num_bins).  Returns (euclidean_bins, spacing_bins) [R,S+Sf+2], detached like upstream."""
    num_bins = cfg.num_fine_samples + 1
    w = weights[..., 0] + histogram_padding
    weights_sum = torch.sum(w, dim=-1, keepdim=True)
    padding = torch.relu(eps - weights_sum)
    w = w + padding / w.shape[-1]
    weights_sum = weights_sum + padding
    pdf = w / weights_sum
    cdf = torch.min(torch.ones_like(pdf), torch.cumsum(pdf, dim=-1))
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins)
    if u_rand is not None:
        u = u.expand(size=(*cdf.shape[:-1], num_bins)) + u_rand / num_bins
    else:
        u = (u + 1.0 / (2 * num_bins)).expand(size=(*cdf.shape[:-1], num_bins))
    u = u.contiguous()
    existing_bins = spacing_bins
    inds = torch.searchsorted(cdf, u, side="right")
    below = torch.clamp(inds - 1, 0, existing_bins.shape[-1] - 1)
    above = torch.clamp(inds, 0, existing_bins.shape[-1] - 1)
    cdf_g0 = torch.gather(cdf, -1, below)
    bins_g0 = torch.gather(existing_bins, -1, below)
    cdf_g1 = torch.gather(cdf, -1, above)
    bins_g1 = torch.gather(existing_bins, -1, above)
    t = torch.clip(torch.nan_to_num((u - cdf_g0) / (cdf_g1 - cdf_g0), 0), 0, 1)
    bins = bins_g0 + t * (bins_g1 - bins_g0)
    bins, _ = torch.sort(torch.cat([existing_bins, bins], -1), -1)
    bins = bins.detach()  # "Stop gradients"
    euclid = bins * fars + (1 - bins) * nears
    return euclid, bins


def render(mesh: OracleMesh, field: torch.Tensor, params: Dict[str, torch.Tensor], origins, directions, cfg: RenderConfig,
           nthreads: int = 0, return_aux: bool = False, fine_euclid=None):
    """TetrahedraNerf.get_outputs in eval mode, background cfg.background (model.py:520-662).  fine_euclid f32[R',S2+1] (non-empty
    rays, in ray order): evaluate the fine pass at THESE bin edges instead of the coarse pass + PDF sampler, as render_train does --
    so that per-sample values can be compared at an implementation's own sample positions."""
    o = torch.as_tensor(np.asarray(origins), dtype=torch.float32).reshape(-1, 3)
    d = torch.as_tensor(np.asarray(directions), dtype=torch.float32).reshape(-1, 3)
    R = o.shape[0]
    tr = mesh.trace_rays(o.numpy(), d.numpy(), cfg.max_intersected_triangles, nthreads=nthreads)
    num_visited = torch.from_numpy(tr["num_visited_cells"])
    hd = torch.from_numpy(tr["hit_distances"])
    nears = hd[:, 0, 0][:, None]
    fars = torch.gather(hd[:, :, 1], 1, (num_visited[:, None].long() - 1).clamp_min(0))
    ray_mask = num_visited > 0
    bg = torch.tensor(cfg.background, dtype=torch.float32)
    rgb = bg.expand(R, 3).clone()
    acc = torch.zeros((R, 1), dtype=torch.float32)
    depth = torch.full((R, 1), cfg.far_plane, dtype=torch.float32)
    aux = {"trace": tr}
    if int(ray_mask.sum()) > 0:
        m = ray_mask.numpy()
        nears_r, fars_r = nears[ray_mask], fars[ray_mask]
        trm = {k: v[m] for k, v in tr.items()}
        dirs_r = d[ray_mask]
        euclid, sbins = coarse_bins(cfg, nears_r, fars_r, num_visited[ray_mask], hd[ray_mask])
        fld = field.detach().float().numpy()

        def field_at(euclid_bins):
            dist = ((euclid_bins[:, 1:] + euclid_bins[:, :-1]) / 2).contiguous()
            tc = find_visited_cells(trm["num_visited_cells"], trm["visited_cells"], trm["barycentric_coordinates"],
                                    trm["hit_distances"], trm["vertex_indices"], dist.numpy(), nthreads=nthreads)
            fv = interpolate_values(tc["vertex_indices"], tc["barycentric_coordinates"], fld, nthreads=nthreads)
            return torch.from_numpy(fv), tc

        if fine_euclid is not None:
            euclid = torch.as_tensor(fine_euclid, dtype=torch.float32)
        elif cfg.num_fine_samples > 0:
            fv, tc = field_at(euclid)
            base = mlp_base(params, fv)
            density_coarse = density_head(params, base)
            deltas = (euclid[:, 1:] - euclid[:, :-1])[..., None]
            weights = get_weights(deltas, density_coarse)
            aux.update(coarse_euclid=euclid, coarse_density=density_coarse, coarse_weights=weights)
            euclid, sbins = pdf_bins(cfg, sbins, weights, nears_r, fars_r)
        fv, tc = field_at(euclid)
        base = mlp_base(params, fv)
        sigmas = density_head(params, base)
        enc = nerf_encoding_dirs(dirs_r)[:, None, :].expand(-1, base.shape[1], -1)
        colors = color_head(params, base, enc)
        deltas = (euclid[:, 1:] - euclid[:, :-1])[..., None]
        weights = get_weights(deltas, sigmas)
        # RGBRenderer (eval: nan_to_num, background, clamp), AccumulationRenderer, DepthRenderer("median")
        comp = torch.sum(weights * torch.nan_to_num(colors), dim=-2)
        accum = torch.sum(weights, dim=-2)
        rgb_r = torch.clamp(comp + bg * (1.0 - accum), 0.0, 1.0)
        steps = (euclid[:, 1:] + euclid[:, :-1]) / 2
        cumw = torch.cumsum(weights[..., 0], dim=-1)
        split = torch.ones((weights.shape[0], 1)) * 0.5
        mi = torch.clamp(torch.searchsorted(cumw, split, side="left"), 0, steps.shape[-1] - 1)
        depth_r = torch.gather(steps, dim=-1, index=mi)
        rgb[ray_mask] = rgb_r
        acc[ray_mask] = accum
        depth[ray_mask] = depth_r
        aux.update(fine_euclid=euclid, sigmas=sigmas, colors=colors, weights=weights, matched=tc)
    out = {"rgb": rgb, "accumulation": acc, "depth": depth, "ray_mask": ray_mask}
    if return_aux:
        out["aux"] = aux
    return out


# =====================================================================================
# training mode with autograd: the oracle of the fused training step
# =====================================================================================
class _GradientScaler(torch.autograd.Function):
    """model.py:195-205"""

    @staticmethod
    def forward(ctx, colors, sigmas, ray_dist):
        ctx.save_for_backward(ray_dist)
        return colors, sigmas, ray_dist

    @staticmethod
    def backward(ctx, g_colors, g_sigmas, g_dist):
        (ray_dist,) = ctx.saved_tensors
        scaling = torch.square(ray_dist).clamp(0, 1)
        return g_colors * scaling, g_sigmas * scaling, g_dist


def interpolate_torch(vertex_indices, bary, field):
    """interpolate_values (tetrahedra_tracer.cu:203-220) in differentiable torch: vertex_indices i64[...,4] (-1 = empty), bary f32[...,3],
    field f32[C,V] -> [...,C]; the gradient w.r.t. the field is interpolate_values_backward (:231-247); none flows to the weights
    (tetranerf/utils/extension/__init__.py:36-42 returns None for them)."""
    vi = torch.as_tensor(vertex_indices).long()
    w = torch.as_tensor(bary).detach()
    ok = (vi >= 0).to(field.dtype)
    F = field.t()  # [V,C]
    safe = vi.clamp_min(0)
    w0 = 1.0 - w.sum(-1)
    out = (w[..., 0:1] * ok[..., 1:2]) * F[safe[..., 1]] + (w[..., 1:2] * ok[..., 2:3]) * F[safe[..., 2]] + (w[..., 2:3] * ok[..., 3:4]) * F[safe[..., 3]] \
        + (w0[..., None] * ok[..., 0:1]) * F[safe[..., 0]]
    return out


def render_train(mesh: OracleMesh, field: torch.Tensor, params: Dict[str, torch.Tensor], origins, directions, cfg: RenderConfig,
                 jitter_coarse=None, jitter_fine=None, use_gradient_scaling: bool = False, nthreads: int = 0, fine_euclid=None):
    """TetrahedraNerf.get_outputs in TRAINING mode (model.py:520-662) in differentiable torch-CPU fp32: `field` and the entries of `params`
    may require grad.  jitter_coarse f32[R,S_c+1] / jitter_fine f32[R,S_f+1] are the uniform draws of the two stratified samplers, indexed by
    RAY (the reference draws them with torch.rand on the non-empty rays).  Training-mode renderer: background cfg.background, no nan_to_num /
    clamp.
    fine_euclid f32[R',S2+1] (non-empty rays, in ray order): use THESE fine-pass bin edges instead of running the coarse pass and the PDF
    sampler -- the bins are detached (non-differentiable) in the reference, so the gradient arithmetic of an implementation can be checked
    at the implementation's own sample positions, which move by ~1e-6 between any two fp32 PDF inversions."""
    o = torch.as_tensor(np.asarray(origins), dtype=torch.float32).reshape(-1, 3)
    d = torch.as_tensor(np.asarray(directions), dtype=torch.float32).reshape(-1, 3)
    R = o.shape[0]
    assert cfg.num_fine_samples > 0
    tr = mesh.trace_rays(o.numpy(), d.numpy(), cfg.max_intersected_triangles, nthreads=nthreads)
    num_visited = torch.from_numpy(tr["num_visited_cells"])
    hd = torch.from_numpy(tr["hit_distances"])
    nears = hd[:, 0, 0][:, None]
    fars = torch.gather(hd[:, :, 1], 1, (num_visited[:, None].long() - 1).clamp_min(0))
    ray_mask = num_visited > 0
    m = ray_mask.numpy()
    nears_r, fars_r = nears[ray_mask], fars[ray_mask]
    trm = {k: v[m] for k, v in tr.items()}
    dirs_r = d[ray_mask]
    jc = torch.as_tensor(jitter_coarse)[ray_mask] if jitter_coarse is not None else None
    jf = torch.as_tensor(jitter_fine)[ray_mask] if jitter_fine is not None else None

    def match(euclid_bins):
        dist = ((euclid_bins[:, 1:] + euclid_bins[:, :-1]) / 2).contiguous()
        return find_visited_cells(trm["num_visited_cells"], trm["visited_cells"], trm["barycentric_coordinates"], trm["hit_distances"],
                                  trm["vertex_indices"], dist.detach().numpy(), nthreads=nthreads)

    if fine_euclid is not None:
        euclid = torch.as_tensor(fine_euclid, dtype=torch.float32)
        sbins = (euclid - nears_r) / (fars_r - nears_r)
    else:
      with torch.no_grad():  # the coarse pass only feeds the (detached) PDF bins
        euclid, sbins = coarse_bins(cfg, nears_r, fars_r, num_visited[ray_mask], hd[ray_mask], jc)
        tc = match(euclid)
        fv = interpolate_torch(tc["vertex_indices"], tc["barycentric_coordinates"], field.detach())
        density_coarse = density_head(params, mlp_base(params, fv))
        weights = get_weights((euclid[:, 1:] - euclid[:, :-1])[..., None], density_coarse)
        euclid, sbins = pdf_bins(cfg, sbins, weights, nears_r, fars_r, u_rand=jf)
    tc = match(euclid)
    fv = interpolate_torch(tc["vertex_indices"], tc["barycentric_coordinates"], field)
    base = mlp_base(params, fv)
    sigmas = density_head(params, base)
    enc = nerf_encoding_dirs(dirs_r)[:, None, :].expand(-1, base.shape[1], -1)
    colors = color_head(params, base, enc)
    if use_gradient_scaling:
        ray_dist = (sbins[:, 1:] + sbins[:, :-1])[..., None]  # spacing_ends + spacing_starts (model.py:629)
        colors, sigmas, _ = _GradientScaler.apply(colors, sigmas, ray_dist)
    deltas = (euclid[:, 1:] - euclid[:, :-1])[..., None]
    weights = get_weights(deltas, sigmas)
    comp = torch.sum(weights * colors, dim=-2)
    accum = torch.sum(weights, dim=-2)
    bg = torch.tensor(cfg.background, dtype=comp.dtype)
    rgb_r = comp + bg * (1.0 - accum)  # RGBRenderer in training: no nan_to_num, no clamp
    steps = (euclid[:, 1:] + euclid[:, :-1]) / 2
    cumw = torch.cumsum(weights[..., 0].detach(), dim=-1)
    mi = torch.clamp(torch.searchsorted(cumw, torch.ones((weights.shape[0], 1)) * 0.5, side="left"), 0, steps.shape[-1] - 1)
    depth_r = torch.gather(steps, dim=-1, index=mi)
    idx = torch.nonzero(ray_mask).flatten()
    rgb = bg.expand(R, 3).clone().index_copy(0, idx, rgb_r)  # (dtype follows the inputs: tests also run this in float64)
    acc = torch.zeros((R, 1), dtype=rgb_r.dtype).index_copy(0, idx, accum)
    depth = torch.full((R, 1), cfg.far_plane, dtype=depth_r.dtype).index_copy(0, idx, depth_r)
    return {"rgb": rgb, "accumulation": acc, "depth": depth, "ray_mask": ray_mask,
            "aux": {"fine_euclid": euclid.detach(), "sigmas": sigmas.detach(), "colors": colors.detach(), "weights": weights.detach(), "matched": tc}}
