"""GPU: mesh refinement by longest-edge bisection (DESIGN §4.14).
  * tn_refine_edges equals the numpy oracle (oracle/refine.py) bit for bit on the small, bottle and sliver meshes with random masks,
    the max_new_vertices cap included, and two runs are bitwise equal;
  * the field is preserved: find_tetrahedra + interpolate_values at 1e4 random interior points agree before and after a refinement
    within 1e-5 of the N(0,1) field's largest magnitude;
  * the render is preserved: the fused eval render (uniform sampler, no ray truncated) agrees in rgb, accumulation and expected depth
    within 1e-4 in both MLP precisions (median depth jumps with the weights and is not compared);
  * the rest of the path accepts the refined mesh: every trace implementation is bit-exact against the oracle, and one fused training
    step passes the float64 bar of test_gpu_train.py;
  * the model through a RAdam loop driven by its callbacks (with and without optimize_vertices), and a checkpoint of a refined model
    loaded into a model built from the original config with its optimizer built first."""
import copy
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import TRACE_IMPLS, force_trace_impl
from oracle import oracle as orc
from oracle import refine as orf
from tetranerf.b200 import synthetic as syn
from test_gpu_slivers import sliver_mesh
from test_gpu_train import DEV, _run

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
TRACE_KEYS = ["num_visited_cells", "visited_cells", "vertex_indices", "hit_distances", "barycentric_coordinates"]


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _gpu_pass(V, C, cand, min_length=0.0, max_new=None):
    from tetranerf.b200.refine import refine_edges

    return refine_edges(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV), torch.from_numpy(cand).to(DEV), min_length, max_new)


def _refined(V, C, frac=0.2, seed=0, passes=1):
    """(V', C') after `passes` GPU passes over a random mask, positions migrated as the model does"""
    from tetranerf.b200.refine import migrate_vertices

    rng = np.random.default_rng(seed)
    for _ in range(passes):
        out = _gpu_pass(V, C, rng.random(len(C)) < frac)
        V = migrate_vertices(torch.from_numpy(V).to(DEV), out["parent_edge"], 0).cpu().numpy()
        C = out["cells"].cpu().numpy()
    return V, C


@pytest.mark.parametrize("mesh", ["small", "bottle", "sliver"])
def test_refine_edges_vs_oracle(small_mesh, mesh):
    V, C = {"small": lambda: small_mesh, "bottle": _bottle, "sliver": lambda: sliver_mesh(300)}[mesh]()
    rng = np.random.default_rng(3)
    for frac, min_length, cap in ((0.05, 0.0, None), (0.5, 0.0, None), (1.0, 0.0, 7), (0.3, 0.05, None), (0.0, 0.0, None)):
        cand = rng.random(len(C)) < frac
        want = orf.refine_edges(V, C, cand, min_length, cap)
        got = _gpu_pass(V, C, cand, min_length, cap)
        again = _gpu_pass(V, C, cand, min_length, cap)
        for k in ("n_proposed", "n_accepted", "n_split"):
            assert got[k] == want[k] == again[k], (k, got[k], want[k])
        for k in ("cells", "parent_edge", "parent_cell"):
            assert np.array_equal(got[k].cpu().numpy(), want[k]), k
            assert torch.equal(got[k], again[k]), k
        print(f"{mesh} frac {frac} min_length {min_length} cap {cap}: proposed {got['n_proposed']} accepted {got['n_accepted']} split {got['n_split']}")


def test_refine_edges_rejects_bad_input():
    from tetranerf.b200.refine import refine_edges

    V, C = syn.delaunay_mesh(200, seed=0)
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV)
    cand = torch.ones(len(C), dtype=torch.bool, device=DEV)
    bad = cells.clone()
    bad[5, 2] = len(V)
    with pytest.raises(RuntimeError, match="vertex index"):
        refine_edges(xyz, bad, cand)
    with pytest.raises(RuntimeError, match="overflows"):
        refine_edges(xyz, cells, cand, 0.0, 2**32 - len(V))


def test_field_is_preserved(small_mesh):
    from tetranerf import cpp
    from tetranerf.utils.extension import interpolate_values
    from tetranerf.b200.refine import migrate_vertices

    V, C = small_mesh
    rng = np.random.default_rng(0)
    out = _gpu_pass(V, C, rng.random(len(C)) < 0.3)
    field = torch.from_numpy(rng.standard_normal((64, len(V))).astype(np.float32)).to(DEV)
    xyz = torch.from_numpy(V).to(DEV)
    V1, F1 = migrate_vertices(xyz, out["parent_edge"], 0), migrate_vertices(field, out["parent_edge"], 1)
    pts = torch.from_numpy((0.1 + 0.8 * rng.random((10_000, 3))).astype(np.float32)).to(DEV)
    vals = []
    for x, c, f in ((xyz, torch.from_numpy(C).to(DEV), field), (V1, out["cells"], F1)):
        tr = cpp.TetrahedraTracer(DEV)
        tr.load_tetrahedra(x, c)
        found = tr.find_tetrahedra(pts)
        assert bool(found["valid_mask"].all())
        vals.append(interpolate_values(found["vertex_indices"], found["barycentric_coordinates"], f))
    err = (vals[0] - vals[1]).abs().max().item()
    scale = field.abs().max().item()
    print(f"refined {len(C)} -> {len(out['cells'])} tetrahedra: max |field before - after| at 1e4 points = {err:.2e} (max |F| {scale:.2f})")
    # both sides carry fp32 barycentrics (find_tetrahedra) and the new vertices one fp32 rounding of their midpoint
    assert err < 1e-5 * scale


@pytest.mark.parametrize("prec", [2, 3])
def test_render_is_preserved(small_mesh, prec):
    from tetranerf import cpp
    from tetranerf.b200.refine import migrate_vertices
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    V, C = small_mesh
    rng = np.random.default_rng(1)
    out = _gpu_pass(V, C, rng.random(len(C)) < 0.5)
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    field = torch.from_numpy(field).to(DEV)
    xyz = torch.from_numpy(V).to(DEV)
    meshes = [(xyz, torch.from_numpy(C).to(DEV), field),
              (migrate_vertices(xyz, out["parent_edge"], 0), out["cells"], migrate_vertices(field, out["parent_edge"], 1))]
    o, d = syn.camera_rays(2000, seed=4)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    st = RenderSettings(max_intersected_triangles=1024, num_samples=64, num_fine_samples=64, use_biased_sampler=False)
    res = []
    for x, c, f in meshes:
        tr = cpp.TetrahedraTracer(DEV)
        tr.load_tetrahedra(x, c)
        assert int(tr.trace_rays(o, d, 1024)["num_visited_cells"].max()) < 1024  # no ray truncated
        fr = FusedRenderer(tr)
        fr.set_field(f)
        fr.set_weights(params)
        fr.set_mlp_precision(prec)
        res.append(fr.render(o, d, st, expected_depth=True))
    assert torch.equal(res[0]["ray_mask"], res[1]["ray_mask"])
    for k in ("rgb", "accumulation", "expected_depth"):
        err = (res[0][k] - res[1][k]).abs().max().item()
        print(f"precision {prec}: max |{k} before - after| = {err:.2e}")
        assert err < 1e-4, k


@pytest.mark.parametrize("mesh", ["small", "bottle"])
def test_trace_on_refined_mesh_is_bit_exact(small_mesh, mesh):
    from tetranerf import cpp

    V, C = small_mesh if mesh == "small" else _bottle()
    V1, C1 = _refined(V, C, frac=0.3, passes=2)
    rng = np.random.default_rng(6)  # rays from outside the mesh's box towards random vertices
    lo, hi = V.min(0), V.max(0)
    tgt = V[rng.integers(0, len(V), 512)]
    u = rng.standard_normal((512, 3))
    o = (tgt + 2.0 * np.linalg.norm(hi - lo) * u / np.linalg.norm(u, axis=1, keepdims=True)).astype(np.float32)
    d = tgt - o
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    ref = orc.OracleMesh(V1, C1).trace_rays(o, d, 512)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V1).to(DEV), torch.from_numpy(C1).to(DEV))
    for impl in TRACE_IMPLS:
        force_trace_impl(tr, impl)
        out = tr.trace_rays(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), 512)
        tr.synchronize()
        for k in TRACE_KEYS:
            assert np.array_equal(out[k].cpu().numpy().view(np.uint32), ref[k].view(np.uint32)), (impl, k)


def test_fused_train_step_on_refined_mesh(small_mesh):
    from tetranerf.b200.render import RenderSettings

    V1, C1 = _refined(*small_mesh, frac=0.3, passes=2)
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    _run(V1, C1, o, d, RenderSettings(num_samples=48, num_fine_samples=33), orc.RenderConfig(num_samples=48, num_fine_samples=33), False, seed=5)


# ---- the model --------------------------------------------------------------------------------------------------------------------
def _model(V, C, field, params, **cfg):
    from tetranerf.nerfstudio import model as M

    config = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=48, num_fine_samples=32,
                                    max_intersected_triangles=1024, **cfg)
    original = copy.deepcopy(config)
    m = M.TetrahedraNerf(config)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(params)
    if config.use_occupancy_field:
        sd["tetrahedra_occupancy"] = torch.zeros(len(C))
    m.load_state_dict(sd, strict=False)
    return m.to(DEV), M, original


def _optimizers(m, M):
    from tetranerf.nerfstudio._ns_compat import Optimizers

    cfg = {k: {"optimizer": (lambda ps, lr=(1e-4 if k == "vertices" else 1e-2): torch.optim.RAdam(ps, lr=lr))} for k in m.get_param_groups()}
    return Optimizers(cfg, m.get_param_groups())


@pytest.mark.parametrize("optimize_vertices", [False, True])
def test_model_refines_through_callbacks(small_mesh, optimize_vertices):
    from tetranerf import cpp

    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    cap = len(V) + 600
    m, M, _ = _model(V, C, field, params, refine_every=3, refine_start=3, refine_stop=9, refine_fraction=0.05, refine_passes=2,
                     refine_max_vertices=cap, use_occupancy_field=True, occupancy_warmup_steps=1000, optimize_vertices=optimize_vertices)
    opts = _optimizers(m, M)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers=opts))
    assert len(cbs) == 2
    o, d = syn.camera_rays(1024, seed=2)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(0)).to(DEV)}
    field_p, xyz_p = m.tetrahedra_field, m.tetrahedra_vertices
    m.train()
    m.tetrahedra_occupancy.uniform_(0.5, 1.0)
    sizes = []
    for step in range(1, 13):
        opts.zero_grad_all()
        loss = sum(m.get_loss_dict(m(bundle), target).values())
        loss.backward()
        opts.optimizer_step_all()
        refine_now = 3 <= step < 9 and step % 3 == 0
        snap = None
        if refine_now:
            st = opts.optimizers["fields"].state[field_p]
            snap = {"field": field_p.detach().clone(), "xyz": xyz_p.detach().clone(), "occ": m.tetrahedra_occupancy.clone(),
                    "cells": m.tetrahedra_cells.clone(), "exp_avg": st["exp_avg"].clone(), "exp_avg_sq": st["exp_avg_sq"].clone(),
                    "step": st["step"].clone()}
            if optimize_vertices:
                snap["v_exp_avg"] = opts.optimizers["vertices"].state[xyz_p]["exp_avg"].clone()
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
        sizes.append(len(m.tetrahedra_vertices))
        assert m.tetrahedra_field is field_p and m.tetrahedra_vertices is xyz_p
        assert torch.isfinite(field_p).all() and torch.isfinite(loss)
        if snap is None:
            continue
        V0, nV = snap["field"].shape[1], field_p.shape[1]
        assert V0 < nV <= cap and field_p.grad is None
        assert torch.equal(field_p[:, :V0], snap["field"]) and torch.equal(xyz_p[:V0], snap["xyz"])
        st = opts.optimizers["fields"].state[field_p]
        assert torch.equal(st["step"], snap["step"])
        for k in ("exp_avg", "exp_avg_sq"):
            assert st[k].shape == field_p.shape and torch.equal(st[k][:, :V0], snap[k])
        if optimize_vertices:
            assert torch.equal(opts.optimizers["vertices"].state[xyz_p]["exp_avg"][:V0], snap["v_exp_avg"])
        # new columns: endpoint averages, pass after pass (the parent edges read back from the mesh growth)
        cells, T0 = m.tetrahedra_cells, len(snap["cells"])
        assert len(m.tetrahedra_occupancy) == len(cells) > T0
        assert torch.equal(m.tetrahedra_occupancy[:T0], snap["occ"])
        assert bool(((m.tetrahedra_occupancy[T0:] >= 0.5) & (m.tetrahedra_occupancy[T0:] <= 1.0)).all())
        # the reloaded tracer traces like a fresh load
        fresh = cpp.TetrahedraTracer(DEV)
        fresh.load_tetrahedra(xyz_p.detach(), cells)
        a = m._tetrahedra_tracer.trace_rays(bundle.origins, bundle.directions, 1024)
        b = fresh.trace_rays(bundle.origins, bundle.directions, 1024)
        for k in TRACE_KEYS:
            assert torch.equal(a[k], b[k]), k
    grew = [b for a, b in zip(sizes, sizes[1:]) if b != a]
    print(f"optimize_vertices={optimize_vertices}: vertices per step {sizes}")
    assert len(grew) >= 1 and sizes[-1] == sizes[6 - 1] and sizes[-1] <= cap  # refinements at steps 3 and 6 only (refine_stop = 9)


def test_model_refine_matches_oracle_and_is_an_endpoint_average(small_mesh):
    """one refine() on a fixed statistic, replayed with the oracle: the same mesh, and new columns equal to endpoint averages"""
    from tetranerf.b200.refine import select_candidates

    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, _ = _model(V, C, field, params, refine_every=1, refine_fraction=0.1, refine_passes=2)
    g = torch.Generator().manual_seed(4)
    m._grad_acc = torch.rand(len(V), generator=g).to(DEV)
    m._grad_cnt = torch.randint(0, 3, (len(V),), generator=g, dtype=torch.int32).to(DEV)
    score = (m._grad_acc / m._grad_cnt.clamp_min(1).float()).cpu()
    cand = select_candidates(score, torch.from_numpy(C), 0.1).numpy()
    res = m.refine()
    Vo, Co, Fo = V, C, field
    for p in res["passes"]:
        out = orf.refine_edges(Vo, Co, cand)
        assert (out["n_proposed"], out["n_accepted"], out["n_split"]) == (p["proposed"], p["accepted"], p["split"])
        split = np.zeros(len(Co), bool)
        split[out["parent_cell"][len(Co):]] = True
        cand = np.concatenate([cand & ~split, np.zeros(out["n_split"], bool)])
        Vo, Fo, Co = orf.migrate_vertices(Vo, out["parent_edge"], 0), orf.migrate_vertices(Fo, out["parent_edge"], 1), out["cells"]
    assert np.array_equal(m.tetrahedra_cells.cpu().numpy(), Co)
    assert np.array_equal(m.tetrahedra_vertices.cpu().numpy(), Vo)
    assert np.array_equal(m.tetrahedra_field.detach().cpu().numpy(), Fo)
    assert res["vertices_before"] == len(V) and res["vertices_after"] == len(Vo) and res["tetrahedra_after"] == len(Co)
    print(res)


def test_refined_checkpoint_loads_into_the_original_config(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, original = _model(V, C, field, params, refine_every=1, refine_fraction=0.1, refine_passes=2, use_occupancy_field=True)
    opts = _optimizers(m, M)
    o, d = syn.camera_rays(512, seed=9)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    m.train()
    for step in range(2):
        opts.zero_grad_all()
        sum(m.get_loss_dict(m(bundle), {"image": torch.full((512, 3), 0.5, device=DEV)}).values()).backward()
        opts.optimizer_step_all()
        m.accumulate_refine_statistics()
    res = m.refine(opts)
    assert res["vertices_after"] > res["vertices_before"]
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    osd = {k: copy.deepcopy(o.state_dict()) for k, o in opts.optimizers.items()}
    m.eval()
    with torch.no_grad():
        want = m(bundle)
    # nerfstudio on resume: the model from config.yml (the original sizes), its optimizers, then the checkpoint
    m2 = M.TetrahedraNerf(copy.deepcopy(original)).to(DEV)
    opts2 = _optimizers(m2, M)
    m2.load_state_dict(sd, strict=True)
    opts2.load_optimizers(osd)
    assert m2.tetrahedra_field.shape == m.tetrahedra_field.shape and m2.tetrahedra_occupancy.shape == m.tetrahedra_occupancy.shape
    m2.eval()
    with torch.no_grad():
        got = m2(bundle)
    for k in ("rgb", "accumulation", "depth", "ray_mask"):
        assert torch.equal(got[k], want[k]), k
    m2.train()
    opts2.zero_grad_all()
    sum(m2.get_loss_dict(m2(bundle), {"image": torch.full((512, 3), 0.5, device=DEV)}).values()).backward()
    opts2.optimizer_step_all()
    assert torch.isfinite(m2.tetrahedra_field).all()
