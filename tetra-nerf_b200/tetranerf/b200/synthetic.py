"""Deterministic synthetic inputs for the ray-sampling hot path (no datasets are available offline).

Meshes follow SURVEY.md §8d: uniform random points in the unit cube -> scipy Delaunay (the reference
uses CGAL, src/triangulation.cpp:34-75; cell order/orientation is irrelevant once the mesh is an
input).  Rays: camera-like coherent bundle, or incoherent (origins on a radius-2 sphere)."""
from __future__ import annotations

import numpy as np

CUBE_VERTICES = np.array(
    [[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1], [1, 0, 1], [0, 1, 1], [1, 1, 1], [0.5, 0.5, 0.5]], dtype=np.float32
)
# the 12-tetrahedra cube of the reference's tests/test_tetrahedra_tracer.py:231-253
CUBE_CELLS = np.array(
    [[0, 1, 2, 8], [2, 1, 3, 8], [0, 1, 4, 8], [4, 1, 5, 8], [0, 2, 4, 8], [4, 2, 6, 8],
     [4, 5, 6, 8], [5, 6, 7, 8], [2, 3, 6, 8], [3, 6, 7, 8], [1, 3, 5, 8], [3, 5, 7, 8]], dtype=np.int32
)


def delaunay_mesh(num_points: int, seed: int = 0):
    """-> (vertices f32[V,3], cells i32[T,4]).  45_000 points -> 302,024 tets; 150_000 -> 1,009,158."""
    from scipy.spatial import Delaunay

    pts = np.random.default_rng(seed).random((num_points, 3), dtype=np.float32)
    cells = Delaunay(pts.astype(np.float64)).simplices.astype(np.int32)
    return pts, np.ascontiguousarray(cells)


def camera_rays(num_rays: int, seed: int = 1):
    """Coherent bundle: origins (0.5,-1.5,0.5)+N(0,0.05^2), targets uniform in [0.2,0.8]^3, unit directions."""
    rng = np.random.default_rng(seed)
    o = (np.array([0.5, -1.5, 0.5]) + 0.05 * rng.standard_normal((num_rays, 3))).astype(np.float32)
    tgt = (0.2 + 0.6 * rng.random((num_rays, 3))).astype(np.float32)
    d = tgt - o
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    return o, d


def sphere_rays(num_rays: int, seed: int = 2, radius: float = 2.0):
    """Incoherent: origins uniform on a sphere of given radius around the cube centre, random targets inside."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((num_rays, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    o = (0.5 + radius * v).astype(np.float32)
    tgt = (0.1 + 0.8 * rng.random((num_rays, 3))).astype(np.float32)
    d = tgt - o
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    return o, d


def random_field(num_vertices: int, field_dim: int = 64, seed: int = 3, kind: str = "normal"):
    """tetrahedra_field [field_dim, V] (feature-major, model.py:247-255).  kind "init" = U(-1e-4,1e-4)
    as model.py:268-271; "normal" = N(0,1) so that parity is not vacuous."""
    rng = np.random.default_rng(seed)
    if kind == "init":
        return ((rng.random((field_dim, num_vertices)) * 2 - 1) * 1e-4).astype(np.float32)
    return rng.standard_normal((field_dim, num_vertices)).astype(np.float32)


# the two spheres of surface_scene: (centre, radius).  Camera rays (camera_rays) look along +y: the small sphere sits behind the
# right edge of the large one, so some rays cross both surfaces, some one, and many none.
SURFACE_SPHERES = (((0.5, 0.42, 0.5), 0.3), ((0.75, 0.82, 0.5), 0.12))
SURFACE_TRUNCATION = 0.25  # feature 0 saturates at +-this distance
SURFACE_EDGE = 0.02        # ... after this many units of signed distance (the smoothed step's width at the surface)


def sphere_sdf(points):
    """signed distance to the union of SURFACE_SPHERES, positive inside, in float64: points [..., 3] -> [...]"""
    p = np.asarray(points, dtype=np.float64)
    return np.max([r - np.linalg.norm(p - np.asarray(c), axis=-1) for c, r in SURFACE_SPHERES], axis=0)


def sphere_hits(origins, directions):
    """analytic ray-sphere intersections with SURFACE_SPHERES in float64: -> f64[R, len(SURFACE_SPHERES), 2] (entry, exit distance along
    the normalised direction; NaN where the ray's line misses the sphere or the sphere lies behind the origin; entry clamped to 0 for
    an origin inside)"""
    o = np.asarray(origins, dtype=np.float64).reshape(-1, 3)
    d = np.asarray(directions, dtype=np.float64).reshape(-1, 3)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    out = np.full((len(o), len(SURFACE_SPHERES), 2), np.nan)
    for i, (c, r) in enumerate(SURFACE_SPHERES):
        oc = o - np.asarray(c)
        b = np.sum(oc * d, axis=1)
        disc = b * b - (np.sum(oc * oc, axis=1) - r * r)
        hit = disc > 0
        h = np.sqrt(np.where(hit, disc, 0.0))
        t0, t1 = -b - h, -b + h
        hit &= t1 > 0
        out[hit, i, 0], out[hit, i, 1] = np.maximum(t0[hit], 0.0), t1[hit]
    return out


def surface_scene(vertices, sharpness: float, params, seed: int = 0, noise: float = 1.0):
    """A hand-built opaque scene: a field on the mesh vertices and MLP parameters under which the fused render sees what a trained
    Tetra-NeRF shows it -- densities that jump from ~0 to ~sharpness/4 at two sphere surfaces, opaque rays whose weights are one narrow
    peak, empty rays, rays that cross two surfaces -- instead of the almost transparent field of the torch-default network.
    -> (field f32[64, V], {PARAM_ORDER name: tensor}).

    Field: feature 0 is a smoothly truncated signed distance to SURFACE_SPHERES (positive inside), T tanh(sdf / SURFACE_EDGE) with
    T = SURFACE_TRUNCATION; features 1-3 are colour logits sin(7 p); features 4-63 N(0, noise^2) as the "normal" field.
    Network: `params` ({PARAM_ORDER name: tensor}, left unchanged; the tests pass the torch-default init of oracle.init_mlp_params)
    with a few entries overwritten, so that every other row and column of each GEMM stays random:
    units 0-7 of mlp_base.layers.0 carry +-feature 0..3 through the ReLU, layers 1 and 2 pass units 0-7 on unchanged, the density
    head has weight `sharpness` on unit 0 and -`sharpness` on unit 1 (its other entries scaled by 1e-2): sigma ~ softplus(k T tanh(.)).
    mlp_head units 0-5 carry +-logits (their 27 direction columns stay random) and the colour head reads them with gain 3."""
    import torch

    xyz = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    V = len(xyz)
    rng = np.random.default_rng(seed)
    field = np.empty((64, V), np.float64)
    field[0] = SURFACE_TRUNCATION * np.tanh(sphere_sdf(xyz) / SURFACE_EDGE)
    field[1:4] = np.sin(7.0 * xyz.T)
    field[4:] = noise * rng.standard_normal((60, V))
    p = {k: v.detach().to(torch.float32).clone() for k, v in params.items()}
    w0, b0 = p["mlp_base.layers.0.weight"], p["mlp_base.layers.0.bias"]
    w0[:8] = 0.0
    b0[:8] = 0.0
    for f in range(4):
        w0[2 * f, f], w0[2 * f + 1, f] = 1.0, -1.0
    for layer in (1, 2):
        w, b = p[f"mlp_base.layers.{layer}.weight"], p[f"mlp_base.layers.{layer}.bias"]
        w[:8] = 0.0
        b[:8] = 0.0
        w[:8, :8] = torch.eye(8)
    wd, bd = p["field_output_density.net.weight"], p["field_output_density.net.bias"]
    wd *= 1e-2
    bd *= 1e-2
    wd[0, 0], wd[0, 1] = float(sharpness), -float(sharpness)
    w4, b4 = p["mlp_head.layers.0.weight"], p["mlp_head.layers.0.bias"]  # input: 27 direction encodings, then the 128 base units
    w4[:6, 27:] = 0.0
    b4[:6] = 0.0
    for c in range(3):
        w4[2 * c, 27 + 2 + 2 * c] = 1.0                   # +logit c = relu(u_{2+2c}) - relu(u_{3+2c}) ...
        w4[2 * c, 27 + 3 + 2 * c] = -1.0
        w4[2 * c + 1, 27 + 2 + 2 * c] = -1.0              # ... and -logit c
        w4[2 * c + 1, 27 + 3 + 2 * c] = 1.0
    wc, bc = p["field_output_color.net.weight"], p["field_output_color.net.bias"]
    wc *= 1e-2
    bc *= 1e-2
    for c in range(3):
        wc[c, 2 * c], wc[c, 2 * c + 1] = 3.0, -3.0
    return field.astype(np.float32), {k: v.contiguous() for k, v in p.items()}
