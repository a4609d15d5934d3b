"""Capture-like scenes for the fused paths, and the checks of them that the CPU oracle can make (GPU parity: test_gpu_scene_geometry.py).

Every other parity test renders uniform points in the unit cube seen from outside.  A Tetra-NeRF scene is a COLMAP cloud of a 360°
capture instead: the cameras sit inside the cloud's hull (so every ray of every call takes the trace's exact all-hits stage), a dense
centre is surrounded by sparse background points far out (tetrahedra whose sizes differ by orders of magnitude on one ray, long ray
distances), coordinates are centred on the origin, and the scene's scale is arbitrary while the pairing epsilon TN_EPS = 1e-6 is
absolute.  The scenes here, all deterministic:

  * capture: 3000 points in the unit ball around the origin, radius (0.05 + 0.95 u)^2 (dense towards the centre), plus 300 background
    points on a shell of radius 6 ... 20, triangulated by scipy (convex hull, no gap records); 256 cameras at radius 1.3 ... 1.6, inside
    the hull: the even rays look at the centre through the dense ball, the odd ones outward into the background tetrahedra;
  * capture_2^-6 / capture_2^6: every coordinate and origin times 2^-6 / 2^6 (exact in fp32), the same cells;
  * offset: the capture scene translated by OFFSET (|OFFSET| ~ 41, mixed signs; the fp32 ulp of a coordinate is 2^-19 ... 2^-18
    instead of ~2^-24 near the origin), re-triangulated.

Density: the field of synthetic.surface_scene evaluated at the scene's canonical (unscaled, untranslated) coordinates mapped into its
unit-cube frame (u = 0.5 + 0.5 x: two spheres of radius 0.6 and 0.24 in the dense ball), with the density head set so that sigma is
SIGMA_IN / s inside the spheres and softplus(-12) / s ~ 6e-6 / s outside, s the scene's scale: the optical depth along a ray is the same at
every scale, so every scene keeps rays that are neither clear nor opaque.

At this size no ray crosses more than ~150 tetrahedra, so M = 512 truncates nothing; the fused checks run at M = CAP = 64, which
truncates the inward rays through the centre and none of the outward ones."""
import functools

import numpy as np
import pytest
import torch
from scipy.spatial import Delaunay

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn

OFFSET = np.array([23.5, -27.25, 19.75], np.float32)
SCENES = {"capture": (1.0, None), "capture_2^-6": (2.0**-6, None), "capture_2^6": (2.0**6, None), "offset": (1.0, OFFSET)}
CAP = 64
SIGMA_IN = 2.0      # density inside the spheres, per canonical unit of length
Z_OUT = -12.0       # density head pre-activation outside the spheres
EPS = 1e-6          # TN_EPS of the trace's pairing (tn_pairing.cuh)
KEYS = ["num_visited_cells", "visited_cells", "vertex_indices", "barycentric_coordinates", "hit_distances"]


def _unit(rng, n):
    u = rng.standard_normal((n, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


@functools.lru_cache(maxsize=None)
def canonical(seed=0, n_dense=3000, n_bg=300, n_cam=256):
    """-> (points f32[V,3], cells i32[T,4], origins f32[R,3], unit directions f32[R,3]) of the capture scene at scale 1"""
    rng = np.random.default_rng(seed)
    dense = _unit(rng, n_dense) * ((0.05 + 0.95 * rng.random(n_dense)) ** 2)[:, None]
    bg = _unit(rng, n_bg) * (6.0 + 14.0 * rng.random(n_bg))[:, None]
    P = np.concatenate([dense, bg]).astype(np.float32)
    cells = Delaunay(P.astype(np.float64)).simplices.astype(np.int32)
    o = _unit(rng, n_cam) * (1.3 + 0.3 * rng.random(n_cam))[:, None]
    inward = (np.arange(n_cam) % 2 == 0)[:, None]
    tgt = np.where(inward, 0.3 * rng.standard_normal((n_cam, 3)), 3.0 * o + 2.0 * rng.standard_normal((n_cam, 3)))
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return P, np.ascontiguousarray(cells), o.astype(np.float32), d.astype(np.float32)


def density_params(s):
    """(k, density bias) for surface_scene's head, sigma ~ softplus(k f0 + b) with f0 in [-T, T]: SIGMA_IN / s inside, Z_OUT outside"""
    z_in = float(np.log(np.expm1(SIGMA_IN / s)))  # softplus^-1
    a = (z_in - Z_OUT) / 2
    return a / syn.SURFACE_TRUNCATION, z_in - a


@functools.lru_cache(maxsize=None)
def scene(name):
    """-> dict V, C, o, d (fp32 numpy), scale s, field f32[64,V], params (PARAM_ORDER name -> tensor)"""
    s, off = SCENES[name]
    P, cells, o, d = canonical()
    if off is None:
        V, C, oo = P * np.float32(s), cells, o * np.float32(s)
    else:
        V, oo = P + off, o + off
        C = np.ascontiguousarray(Delaunay(V.astype(np.float64)).simplices.astype(np.int32))
    k, b = density_params(s)
    field, params = syn.surface_scene(0.5 + 0.5 * P.astype(np.float64), k, orc.init_mlp_params(0))
    params["field_output_density.net.bias"] += b
    return {"V": V, "C": C, "o": oo, "d": d.copy(), "s": s, "field": field, "params": params}


@functools.lru_cache(maxsize=None)
def oracle_mesh(name):
    sc = scene(name)
    return orc.OracleMesh(sc["V"], sc["C"])


def truncated(mesh, o, d, M):
    """bool[R]: rays with more cells than the cap M keeps"""
    return mesh.trace_rays(o, d, 4 * M)["num_visited_cells"] > mesh.trace_rays(o, d, M)["num_visited_cells"]


def tie_rays(mesh, o, d, thr):
    """bool[R]: rays with two face crossings closer than thr (the sorted t of every hit face of the all-hits trace)"""
    tri = mesh.trace_rays_triangles(o, d, 2048)
    n, t = tri["num_visited_triangles"], tri["hit_distances"]
    assert int(n.max()) < 2048
    return np.array([bool(np.any(np.diff(np.sort(t[r, :n[r]].astype(np.float64))) < thr)) for r in range(len(o))])


def equivariance(ref, got, s):
    """bool[R]: rays whose trace at scale s is not the scale-1 trace with every hit distance times s, bit for bit"""
    R = len(ref["num_visited_cells"])
    bad = np.zeros(R, bool)
    for key in KEYS:
        a = np.asarray(ref[key] * np.float32(s) if key == "hit_distances" else ref[key])
        bad |= ~np.all((np.asarray(got[key]).view(np.uint32) == a.view(np.uint32)).reshape(R, -1), axis=1)
    return bad


def exempt_rays(k):
    """the rays of the scale-2^k capture scene that may break equivariance: two crossings of the scale-1 key list closer than
    EPS max(1, 2^-k), where the absolute epsilon can decide differently at the two scales"""
    sc = scene("capture")
    return tie_rays(oracle_mesh("capture"), sc["o"], sc["d"], EPS * max(1.0, 2.0**-k))


def test_scenes_are_deterministic():
    P, C, o, d = canonical()
    canonical.cache_clear()
    P2, C2, o2, d2 = canonical()
    assert all(np.array_equal(x, y) for x, y in ((P, P2), (C, C2), (o, o2), (d, d2)))
    assert len(P) == 3300 and len(o) == 256
    assert np.allclose(np.linalg.norm(d.astype(np.float64), axis=1), 1.0, atol=1e-6)
    for name, (s, off) in SCENES.items():
        sc = scene(name)
        if off is None:  # a power of two times an fp32 number: exact
            assert np.array_equal(sc["V"].astype(np.float64), P.astype(np.float64) * s)
            assert np.array_equal(sc["o"].astype(np.float64), o.astype(np.float64) * s)
        assert sc["V"].dtype == np.float32 and sc["C"].dtype == np.int32 and len(np.unique(sc["C"])) == len(P)


@pytest.mark.parametrize("name", list(SCENES))
def test_cameras_inside_and_cells_of_every_size(name):
    """every origin lies inside the mesh; the tetrahedra on one ray differ in size by orders of magnitude"""
    sc = scene(name)
    mesh = oracle_mesh(name)
    assert bool(mesh.find_tetrahedra(sc["o"])["valid_mask"].all())
    tr = mesh.trace_rays(sc["o"], sc["d"], 512)
    n, hd = tr["num_visited_cells"], tr["hit_distances"].astype(np.float64) / sc["s"]
    assert bool((n > 0).all())
    seg = hd[..., 1] - hd[..., 0]
    ratio = [seg[r, :n[r]].max() / seg[r, :n[r]][seg[r, :n[r]] > 0].min() for r in range(len(n))]
    far = np.array([hd[r, n[r] - 1, 1] for r in range(len(n))])
    print(f"{name}: cells per ray {n.min()} ... {n.max()}; near (scale 1) median {np.median(hd[:, 0, 0]):.3f}; far (scale 1) up to "
          f"{far.max():.1f}; longest / shortest segment on a ray: median {np.median(ratio):.1e}")
    assert np.median(ratio) > 100 and far.max() > 5


@pytest.mark.parametrize("name", list(SCENES))
def test_cap_truncates_some_rays(name):
    sc = scene(name)
    mesh = oracle_mesh(name)
    cut = truncated(mesh, sc["o"], sc["d"], CAP)
    print(f"{name}: truncated at M = {CAP}: {cut.mean():.3f} (inward {cut[0::2].mean():.3f}, outward {cut[1::2].mean():.3f}); "
          f"at M = 512: {truncated(mesh, sc['o'], sc['d'], 512).mean():.3f}")
    assert 0.0 < cut.mean() < 1.0


@pytest.mark.parametrize("k", [-6, 6])
def test_oracle_trace_is_scale_equivariant(k):
    """scaling every coordinate by 2^k scales every hit distance by 2^k and leaves cells, vertices and barycentrics bitwise unchanged,
    except on rays where the absolute epsilon can decide differently (exempt_rays): the watertight test is a chain of individually
    rounded products and differences, each of which scales exactly"""
    name = f"capture_2^{k}"
    sc0, sc = scene("capture"), scene(name)
    ex = exempt_rays(k)
    for M in (CAP, 512):
        ref = oracle_mesh("capture").trace_rays(sc0["o"], sc0["d"], M)
        got = oracle_mesh(name).trace_rays(sc["o"], sc["d"], M)
        bad = equivariance(ref, got, 2.0**k)
        print(f"2^{k}, M = {M}: {int(ex.sum())} exempt rays of {len(ex)}, {int(bad.sum())} not equivariant, "
              f"{int((bad & ~ex).sum())} of them not exempt")
        assert not np.any(bad & ~ex), np.nonzero(bad & ~ex)[0]
    assert ex.mean() < 0.5


def test_eps_ties_at_the_small_scale():
    """at scale 2^-6, crossings closer than TN_EPS (the literal dedupe / pairing) happen on some rays"""
    sc = scene("capture_2^-6")
    ties = tie_rays(oracle_mesh("capture_2^-6"), sc["o"], sc["d"], EPS)
    print(f"capture_2^-6: {int(ties.sum())} of {len(ties)} rays with eps-ties; capture: "
          f"{int(tie_rays(oracle_mesh('capture'), scene('capture')['o'], scene('capture')['d'], EPS).sum())}")
    assert ties.any()


@pytest.mark.parametrize("name", list(SCENES))
def test_accumulation_regime(name):
    """the oracle's eval render (tetra_nerf at M = CAP): at least 20 % of the rays end with accumulation in (0.05, 0.95)"""
    sc = scene(name)
    oc = orc.RenderConfig.tetra_nerf()
    oc.max_intersected_triangles = CAP
    ref = orc.render(oracle_mesh(name), torch.from_numpy(sc["field"]), sc["params"], sc["o"], sc["d"], oc)
    acc = ref["accumulation"][:, 0]
    mid = ((acc > 0.05) & (acc < 0.95)).float().mean().item()
    print(f"{name}: accumulation in (0.05, 0.95) on {mid:.2f} of the rays, > 0.95 on {(acc >= 0.95).float().mean().item():.2f}")
    assert bool(ref["ray_mask"].all())
    assert mid >= 0.2
