"""GPU: trace_rays on folded meshes after a fresh load, as refinement and a checkpoint resume load them (DESIGN §4.9).

The folded meshes of test_walk_cpu.py (one vertex moved through a face at three depths, a dozen folds far apart, a smooth displacement
that folds a few faces, the sliver mesh after two bisection passes) keep the clean mesh's convex hull, so only the load's fold test keeps
the adjacency walk off them; on those meshes the walk misses the crossings off its chain of tetrahedra (test_walk_cpu.py counts them).
  * a fresh load traces bit for bit as the oracle: every implementation of trace_rays, the default choice for 4096 rays,
    trace_rays_triangles and find_tetrahedra at points in the folded region; a fused render equals the render on a refit tracer;
  * wherever the walk is on, every walk implementation equals oracle/walk.py on every ray, and the tracer's exact-stage counts equal
    the restatement's routes, so the CPU finding carries over to the GPU;
  * the model: optimize_vertices moved in place to a folded state (the refit warns and turns the walk off), then refine(): the reloaded
    tracer traces as the oracle and as a refit; a checkpoint of the folded model, loaded into a model built from the original config,
    traces and renders bit for bit as the uninterrupted model."""
import copy
import functools

import numpy as np
import pytest
import torch

from conftest import TRACE_IMPLS, force_trace_impl
from oracle import oracle as orc
from oracle import vertex_grads as vg
from oracle import walk as W
from tetranerf.b200 import synthetic as syn
from test_gpu_slivers import sliver_mesh
from test_walk_cpu import FOLDED, M, N_RAYS, folded_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ["num_visited_cells", "visited_cells", "vertex_indices", "hit_distances", "barycentric_coordinates"]
WALKS = [k for k in TRACE_IMPLS if k.startswith("walk")]


@functools.lru_cache(maxsize=None)
def _case(name):
    small = syn.delaunay_mesh(3000, seed=0)
    if name in ("small", "cube", "slivers"):
        V, C = {"small": small, "cube": (syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()), "slivers": sliver_mesh()}[name]
        oc, dc = syn.camera_rays(N_RAYS // 2, seed=3)
        os_, ds = syn.sphere_rays(N_RAYS // 2, seed=4)
        return V, C, V, np.concatenate([oc, os_]), np.concatenate([dc, ds]), np.zeros(0, np.int64), np.zeros(0, np.int64)
    V, C, P, o, d, inv, near, _ = folded_case(name, small)
    return V, C, P, o, d, inv, near


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _same(got, want, what):
    for k in want:
        a, b = got[k].cpu().numpy() if torch.is_tensor(got[k]) else got[k], np.asarray(want[k])
        if a.dtype.kind == "f":
            a, b = a.view(np.uint32), b.astype(a.dtype).view(np.uint32)
        else:
            b = b.astype(a.dtype)
        bad = np.unique(np.nonzero(a != b)[0])
        assert len(bad) == 0, f"{what}: {k} differs on {len(bad)} rays / points, e.g. {bad[:8]}"


def _load(P, C):
    from tetranerf import cpp

    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(_t(P), _t(C))
    return tr


@pytest.mark.parametrize("name", FOLDED)
def test_fresh_load_is_exact(name):
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    V, C, P, o, d, inv, near = _case(name)
    folded = vg.fold_count(P, C)
    tr = _load(P, C)
    walkable, _ = tr.trace_stats()
    print(f"{name}: {folded} folded faces, walk {'on' if walkable else 'off'} after a fresh load")
    assert not walkable  # every construction leaves faces the fold test does not certify
    mesh = orc.OracleMesh(P, C)
    ref = mesh.trace_rays(o, d, M)
    ot, dt = _t(o), _t(d)
    out = tr.trace_rays(ot, dt, M)  # the default choice for this batch size
    tr.synchronize()
    _same(out, ref, f"{name} default")
    for impl in TRACE_IMPLS:
        force_trace_impl(tr, impl)
        out = tr.trace_rays(ot, dt, M)
        tr.synchronize()
        _same(out, ref, f"{name} {impl}")
    _same(tr.trace_rays_triangles(ot, dt, M), mesh.trace_rays_triangles(o, d, M), f"{name} trace_rays_triangles")
    rng = np.random.default_rng(2)
    region = near if len(near) else np.arange(len(C))
    pts = (P[C[region[rng.integers(0, len(region), 2000)]]].mean(1) + 0.002 * rng.standard_normal((2000, 3))).astype(np.float32)
    found = tr.find_tetrahedra(_t(pts))
    _same({k: v for k, v in found.items() if k != "valid_mask"}, {k: v for k, v in mesh.find_tetrahedra(pts).items() if k != "valid_mask"},
          f"{name} find_tetrahedra")
    # a fused eval render on the fresh load against the same render on a tracer refit to the same positions (walk off by the fold test)
    refit = _load(V, C)
    nf, walk_on = refit.update_vertices(_t(P))
    assert nf == folded and not walk_on
    field, params = syn.surface_scene(P, 60, orc.init_mlp_params(0), noise=0.3)
    st = RenderSettings(max_intersected_triangles=M, num_samples=48, num_fine_samples=32, use_biased_sampler=True)
    res = []
    for t in (tr, refit):
        force_trace_impl(t, "walk_quad")
        fr = FusedRenderer(t)
        fr.set_field(_t(field))
        fr.set_weights(params)
        res.append(fr.render(ot, dt, st))
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", ["small", "cube", "slivers"] + FOLDED)
def test_gpu_walk_equals_restatement(name):
    """wherever a load leaves the walk on, every walk implementation gives the restatement's bits on every ray and the restatement's
    routes: listed rays (keys provided + exact) and all-hits rays"""
    from tetranerf.utils.extension import tetranerf_cpp_extension as ext

    V, C, P, o, d, _, _ = _case(name)
    tr = _load(P, C)
    walkable, _ = tr.trace_stats()
    if walkable:  # (a folded mesh walks only without the load's fold test; test_fresh_load_is_exact holds it to the oracle)
        want = W.walk_trace(P, C, o, d, M)
        routes = np.bincount(want["route"], minlength=4)
        ot, dt = _t(o), _t(d)
        for impl in WALKS:
            force_trace_impl(tr, impl)
            out = tr.trace_rays(ot, dt, M)
            _, listed = tr.trace_stats()
            exact = ext._lib.tn_debug_last_exact_count()
            print(f"{name} {impl}: listed {listed}, all-hits {exact}; restatement {dict(zip(W.ROUTES, routes.tolist()))}")
            _same(out, {k: want[k] for k in KEYS}, f"{name} {impl}")
            assert listed == routes[W.KEYS] + routes[W.EXACT] and exact == routes[W.EXACT]
    folded = vg.fold_count(P, C)
    assert walkable == (folded == 0), (walkable, folded)


# ---- the model ---------------------------------------------------------------------------------------------------------------------------
def _folded_model(**cfg):
    """a TetrahedraNerf with optimize_vertices on the small mesh whose vertices are then moved in place to the scattered folds: the refit
    warns and turns the walk off"""
    from test_gpu_refine import _model

    V, C, P, o, d, _, _ = _case("scattered")
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, Mod, original = _model(V, C, field, params, optimize_vertices=True, **cfg)
    assert m.get_tetrahedra_tracer().trace_stats()[0]
    with torch.no_grad():
        m.tetrahedra_vertices.copy_(_t(P))
    with pytest.warns(UserWarning, match="folded"):
        tr = m.get_tetrahedra_tracer()
    assert not tr.trace_stats()[0]
    return m, Mod, original, o, d


def test_refine_after_folding_reloads_an_exact_tracer():
    m, _, _, o, d = _folded_model(refine_every=1, refine_fraction=0.1, refine_passes=2)
    g = torch.Generator().manual_seed(4)
    V0 = len(m.tetrahedra_vertices)
    m._grad_acc = torch.rand(V0, generator=g).to(DEV)
    m._grad_cnt = torch.randint(0, 3, (V0,), generator=g, dtype=torch.int32).to(DEV)
    res = m.refine()
    assert res["vertices_after"] > res["vertices_before"]
    P1, C1 = m.tetrahedra_vertices.detach().cpu().numpy(), m.tetrahedra_cells.cpu().numpy()
    folded = vg.fold_count(P1, C1)
    tr = m.get_tetrahedra_tracer()
    print(f"refined {res['vertices_before']} -> {res['vertices_after']} vertices: {folded} folded faces, walk "
          f"{'on' if tr.trace_stats()[0] else 'off'}")
    assert folded > 0 and not tr.trace_stats()[0]
    ref = orc.OracleMesh(P1, C1).trace_rays(o, d, M)
    refit = _load(P1, C1)
    refit.update_vertices(_t(P1))
    ot, dt = _t(o), _t(d)
    a, b = tr.trace_rays(ot, dt, M), refit.trace_rays(ot, dt, M)
    _same(a, ref, "reloaded after refine")
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k


def test_checkpoint_of_a_folded_model_resumes_exactly():
    from tetranerf.nerfstudio import model as Mod

    m, _, original, o, d = _folded_model()
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    m2 = Mod.TetrahedraNerf(copy.deepcopy(original)).to(DEV)  # nerfstudio on resume: the model from config.yml, then the checkpoint
    m2.load_state_dict(sd, strict=True)
    ot, dt = _t(o), _t(d)
    tr1, tr2 = m.get_tetrahedra_tracer(), m2.get_tetrahedra_tracer()
    assert not tr2.trace_stats()[0]
    a, b = tr1.trace_rays(ot, dt, 1024), tr2.trace_rays(ot, dt, 1024)
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k
    P = m.tetrahedra_vertices.detach().cpu().numpy()
    _same(b, orc.OracleMesh(P, m.tetrahedra_cells.cpu().numpy()).trace_rays(o, d, 1024), "resumed")
    bundle = Mod.RayBundle(origins=ot[:1024], directions=dt[:1024])
    m.eval()
    m2.eval()
    with torch.no_grad():
        want, got = m(bundle), m2(bundle)
    for k in ("rgb", "accumulation", "depth", "ray_mask"):
        assert torch.equal(got[k], want[k]), k
