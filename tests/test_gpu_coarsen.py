"""GPU: mesh coarsening by empty-space vertex removal (DESIGN §4.18).
  * tn_coarsen_vertices equals the numpy oracle (oracle/coarsen.py) bit for bit on the 3000-point, bottle and sliver meshes with random
    empty masks, the max_removed cap included, and two runs are bitwise equal; bad input raises;
  * the trace accepts the coarsened mesh: the walk stays on, every trace implementation is bit-exact against the oracle, and every record
    in a tetrahedron the pass left alone and that shares no face with a changed one is the pre-coarsening record, bit for bit (next to
    a changed one: the same vertices and, within rounding, the same values);
  * the render is preserved: with occupancy culling on and the uniform sampler, the fused eval render in both MLP precisions equals the
    pre-coarsening render (rgb, accumulation, expected depth) within 1e-5;
  * one fused training step on a coarsened mesh passes the float64 bar of test_gpu_train.py;
  * the model: callbacks coarsen, parameters keep their identity, moments and statistics are compacted, nothing happens on a buffer that
    was never computed, a coarsened checkpoint loads into the original config and renders the same bits, and a short run with
    refinement and coarsening both on keeps the walk;
  * the 2.02 M-tetrahedra mesh: counts, validity and the walk."""
import copy
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import TRACE_IMPLS, force_trace_impl
from oracle import coarsen as oco
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_slivers import sliver_mesh
from test_gpu_train import DEV, _run

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
TRACE_KEYS = ["num_visited_cells", "visited_cells", "vertex_indices", "hit_distances", "barycentric_coordinates"]


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _gpu_pass(V, C, empty, cap=None):
    from tetranerf.b200.coarsen import coarsen_vertices

    return coarsen_vertices(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV), torch.from_numpy(empty).to(DEV), cap)


def _coarsened(V, C, frac=1.0, seed=0, passes=2):
    """(V', C', kept_vertex, parent_cell) after `passes` GPU passes over random masks, composed over the passes"""
    rng = np.random.default_rng(seed)
    kept, parent = np.arange(len(V)), np.arange(len(C))
    for _ in range(passes):
        out = _gpu_pass(V, C, rng.random(len(C)) < frac)
        k, p = out["kept_vertex"].cpu().numpy(), out["parent_cell"].cpu().numpy()
        V, C = V[k], out["cells"].cpu().numpy()
        kept, parent = kept[k], parent[p]
    return V, C, kept, parent


@pytest.mark.parametrize("mesh", ["small", "bottle", "sliver"])
def test_coarsen_vertices_vs_oracle(small_mesh, mesh):
    V, C = {"small": lambda: small_mesh, "bottle": _bottle, "sliver": lambda: sliver_mesh(300)}[mesh]()
    rng = np.random.default_rng(3)
    for frac, cap in ((1.0, None), (0.95, None), (0.8, None), (1.0, 5), (1.0, 0), (0.0, None)):
        empty = rng.random(len(C)) < frac
        want = oco.coarsen_vertices(V, C, empty, cap)
        got = _gpu_pass(V, C, empty, cap)
        again = _gpu_pass(V, C, empty, cap)
        for k in ("n_proposed", "n_removed", "n_cells_removed"):
            assert got[k] == want[k] == again[k], (k, got[k], want[k])
        for k in ("cells", "kept_vertex", "parent_cell"):
            assert np.array_equal(got[k].cpu().numpy(), want[k]), k
            assert torch.equal(got[k], again[k]), k
        if got["n_removed"]:
            oco.check_coarsened(V, C, want["cells"], want["kept_vertex"], want["parent_cell"])
        print(f"{mesh} empty {frac} cap {cap}: proposed {got['n_proposed']} removed {got['n_removed']} cells removed {got['n_cells_removed']}")


def test_coarsen_vertices_rejects_bad_input():
    from tetranerf.b200.coarsen import coarsen_vertices

    V, C = syn.delaunay_mesh(200, seed=0)
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV)
    empty = torch.ones(len(C), dtype=torch.bool, device=DEV)
    bad = cells.clone()
    bad[5, 2] = len(V)
    with pytest.raises(RuntimeError, match="vertex index"):
        coarsen_vertices(xyz, bad, empty)
    with pytest.raises(RuntimeError, match="one entry per tetrahedron"):
        coarsen_vertices(xyz, cells, empty[1:])
    with pytest.raises(RuntimeError, match="max_removed"):
        coarsen_vertices(xyz, cells, empty, -1)
    with pytest.raises(RuntimeError, match="CUDA"):
        coarsen_vertices(xyz.cpu(), cells, empty)
    out = coarsen_vertices(xyz, cells[:0], empty[:0])  # no cell: nothing to remove
    assert out["n_removed"] == 0 and torch.equal(out["kept_vertex"].long().cpu(), torch.arange(len(V)))


def _outside_rays(V, C, n, seed):
    # rays from outside the mesh's box towards the centroids of random tetrahedra: generic rays, which pass through no vertex or edge,
    # so the tetrahedra a ray crosses do not depend on how the trace breaks the ties of a degenerate crossing
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    tgt = V[C[rng.integers(0, len(C), n)]].astype(np.float64).mean(1)
    u = rng.standard_normal((n, 3))
    o = (tgt + 2.0 * np.linalg.norm(hi - lo) * u / np.linalg.norm(u, axis=1, keepdims=True)).astype(np.float32)
    d = tgt - o
    return o, (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("mesh", ["small", "bottle"])
def test_trace_on_coarsened_mesh(small_mesh, mesh):
    from tetranerf import cpp

    V, C = small_mesh if mesh == "small" else _bottle()
    V1, C1, kept, parent = _coarsened(V, C, frac=1.0, passes=2)
    assert len(V1) < len(V)
    o, d = _outside_rays(V, C, 512, 6)
    do, dd = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    tr0 = cpp.TetrahedraTracer(DEV)
    tr0.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    before = {k: v.cpu().numpy() for k, v in tr0.trace_rays(do, dd, 1024).items()}
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V1).to(DEV), torch.from_numpy(C1).to(DEV))
    assert tr.trace_stats()[0] == tr0.trace_stats()[0], "the coarsened mesh lost the adjacency walk"
    ref = orc.OracleMesh(V1, C1).trace_rays(o, d, 1024)
    for impl in TRACE_IMPLS:
        force_trace_impl(tr, impl)
        out = tr.trace_rays(do, dd, 1024)
        tr.synchronize()
        for k in TRACE_KEYS:
            assert np.array_equal(out[k].cpu().numpy().view(np.uint32), ref[k].view(np.uint32)), (impl, k)
    # property 4: a record in a tetrahedron the passes left alone, none of whose faces it shared with a tetrahedron they changed or
    # removed, is the old record bit for bit (vertex ids renumbered).  Next to a changed tetrahedron the face table may take a face's
    # stored winding from another first owner, so there the record holds the same vertices and, within rounding, the same values.
    unchanged = (kept[C1] == C[parent]).all(1)
    touched = np.ones(len(C), bool)
    touched[parent[unchanged]] = False  # changed or removed
    faces = np.sort(np.concatenate([C[:, q] for q in ([1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2])], 0), 1)
    _, fid = np.unique(faces, axis=0, return_inverse=True)
    fid = fid.reshape(4, -1).T
    near = np.zeros(fid.max() + 1, bool)
    np.logical_or.at(near, fid[touched].reshape(-1), True)
    clean = ~touched & ~near[fid].any(1)  # old ids
    n0, n1 = before["num_visited_cells"], ref["num_visited_cells"]
    exact = border = border_bitwise = 0
    for r in range(len(o)):
        old = {int(t): j for j, t in enumerate(before["visited_cells"][r, : n0[r]])}
        for j in range(n1[r]):
            t = int(ref["visited_cells"][r, j])
            if t < 0 or not unchanged[t]:  # a gap record between two hull faces of a non-convex mesh (the bottle) has no cell
                continue
            i = old.get(int(parent[t]))
            assert i is not None, (r, j, "the ray no longer crosses an unchanged tetrahedron it crossed before")
            vi_new, vi_old = kept[ref["vertex_indices"][r, j]], before["vertex_indices"][r, i]
            same = np.array_equal(vi_new, vi_old) and all(np.array_equal(ref[k][r, j].view(np.uint32), before[k][r, i].view(np.uint32))
                                                          for k in ("hit_distances", "barycentric_coordinates"))
            if clean[parent[t]]:
                assert same, (r, j)
                exact += 1
                continue
            border += 1
            border_bitwise += same
            assert np.array_equal(np.sort(vi_new), np.sort(vi_old)), (r, j)
            np.testing.assert_allclose(ref["hit_distances"][r, j], before["hit_distances"][r, i], rtol=1e-5, atol=1e-6)
            # entry and exit barycentrics, each over its face's vertices in the stored rotation
            np.testing.assert_allclose(np.sort(ref["barycentric_coordinates"][r, j], 1), np.sort(before["barycentric_coordinates"][r, i], 1),
                                       rtol=0, atol=1e-5)
    print(f"{mesh}: {len(V)} -> {len(V1)} vertices, {len(C)} -> {len(C1)} tetrahedra; mean records per ray "
          f"{n0.mean():.1f} -> {n1.mean():.1f}; {exact} records in unchanged tetrahedra away from the changes bitwise equal; "
          f"next to them {border_bitwise} of {border} bitwise equal")
    assert exact > 0


def _occupied_scene(V, C, prec=3):
    """surface_scene's field and weights on (V, C) and its occupancy f32[T] (decay 0)"""
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(DEV))
    fr.set_weights(params)
    occ = fr.update_occupancy(torch.zeros(len(C), device=DEV), 0.0).clone()
    return field, params, occ


@pytest.mark.parametrize("prec", [2, 3])
def test_render_is_preserved(small_mesh, prec):
    from tetranerf import cpp
    from tetranerf.b200.coarsen import compact_vertices, coarsen_vertices
    from tetranerf.b200.refine import migrate_cells
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    V, C = small_mesh
    thr = 0.01
    field, params, occ = _occupied_scene(V, C)
    xyz, cells, f, o_ = torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV), torch.from_numpy(field).to(DEV), occ
    meshes = [(xyz, cells, f, o_)]
    for _ in range(2):
        out = coarsen_vertices(xyz, cells, o_ < thr)
        xyz, f = compact_vertices(xyz, out["kept_vertex"], 0), compact_vertices(f, out["kept_vertex"], 1)
        cells, o_ = out["cells"], migrate_cells(o_, out["parent_cell"])
    meshes.append((xyz, cells, f.contiguous(), o_))
    assert len(cells) < len(C)
    o, d = syn.camera_rays(2000, seed=4)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    st = RenderSettings(max_intersected_triangles=1024, num_samples=64, num_fine_samples=64, use_biased_sampler=False)
    res = []
    for x, c, fi, oc in meshes:
        tr = cpp.TetrahedraTracer(DEV)
        tr.load_tetrahedra(x, c)
        assert int(tr.trace_rays(o, d, 1024)["num_visited_cells"].max()) < 1024  # no ray truncated
        fr = FusedRenderer(tr)
        fr.set_field(fi)
        fr.set_weights(params)
        fr.set_mlp_precision(prec)
        fr.set_occupancy(oc, thr)
        res.append(fr.render(o, d, st, expected_depth=True))
    assert torch.equal(res[0]["ray_mask"], res[1]["ray_mask"])
    for k in ("rgb", "accumulation", "expected_depth"):
        err = (res[0][k] - res[1][k]).abs().max().item()
        print(f"precision {prec}: {len(C)} -> {len(cells)} tetrahedra; max |{k} before - after| = {err:.2e}, bitwise {torch.equal(res[0][k], res[1][k])}")
        assert err < 1e-5, k


def test_fused_train_step_on_coarsened_mesh(small_mesh):
    from tetranerf.b200.render import RenderSettings

    V1, C1, _, _ = _coarsened(*small_mesh, frac=1.0, passes=2)
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    _run(V1, C1, o, d, RenderSettings(num_samples=48, num_fine_samples=33), orc.RenderConfig(num_samples=48, num_fine_samples=33), False, seed=5)


# ---- the model --------------------------------------------------------------------------------------------------------------------
def _model(V, C, field, params, **cfg):
    from tetranerf.nerfstudio import model as M

    config = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=48, num_fine_samples=32,
                                    max_intersected_triangles=1024, use_occupancy_field=True, **cfg)
    original = copy.deepcopy(config)
    m = M.TetrahedraNerf(config)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field),
          "tetrahedra_occupancy": torch.zeros(len(C))}
    sd.update(params)
    m.load_state_dict(sd, strict=False)
    return m.to(DEV), M, original


def _optimizers(m):
    from tetranerf.nerfstudio._ns_compat import Optimizers

    cfg = {k: {"optimizer": (lambda ps, lr=(1e-5 if k == "vertices" else 1e-3): torch.optim.RAdam(ps, lr=lr))} for k in m.get_param_groups()}
    return Optimizers(cfg, m.get_param_groups())


def _bundle(M, n, seed):
    o, d = syn.camera_rays(n, seed=seed)
    return M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))


@pytest.mark.parametrize("optimize_vertices", [False, True])
def test_model_coarsens_through_callbacks(small_mesh, optimize_vertices):
    from tetranerf import cpp

    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, _ = _model(V, C, field, params, coarsen_every=2, coarsen_start=2, coarsen_stop=5, coarsen_passes=2, occupancy_warmup_steps=0,
                     optimize_vertices=optimize_vertices)
    opts = _optimizers(m)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers=opts))
    assert len(cbs) == 1
    bundle = _bundle(M, 1024, 2)
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(0)).to(DEV)}
    field_p, xyz_p = m.tetrahedra_field, m.tetrahedra_vertices
    m.train()
    sizes = []
    for step in range(1, 8):
        opts.zero_grad_all()
        loss = sum(m.get_loss_dict(m(bundle), target).values())
        loss.backward()
        opts.optimizer_step_all()
        due = step in (2, 4)
        if due:
            st = opts.optimizers["fields"].state[field_p]
            snap = {"field": field_p.detach().clone(), "xyz": xyz_p.detach().clone(), "occ": m.tetrahedra_occupancy.clone(),
                    "cells": m.tetrahedra_cells.clone(), "exp_avg": st["exp_avg"].clone(), "exp_avg_sq": st["exp_avg_sq"].clone(),
                    "step": st["step"].clone()}
            if optimize_vertices:
                snap["v_exp_avg"] = opts.optimizers["vertices"].state[xyz_p]["exp_avg"].clone()
            nV = len(m.tetrahedra_vertices)
            m._grad_acc = torch.rand(nV, device=DEV)
            m._grad_cnt = torch.randint(0, 4, (nV,), dtype=torch.int32, device=DEV)
            snap["acc"], snap["cnt"] = m._grad_acc.clone(), m._grad_cnt.clone()
            calls = []
            coarsen = m.coarsen
            m.coarsen = lambda optimizers=None: calls.append(coarsen(optimizers)) or calls[-1]
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
        sizes.append(len(m.tetrahedra_vertices))
        assert m.tetrahedra_field is field_p and m.tetrahedra_vertices is xyz_p
        assert torch.isfinite(field_p).all() and torch.isfinite(loss)
        if not due:
            continue
        del m.coarsen
        assert len(calls) == 1
        res = calls[0]
        assert res["ready"] and res["vertices_after"] < res["vertices_before"], res
        kv, pc = res["kept_vertex"], res["parent_cell"]
        assert field_p.grad is None and torch.equal(field_p, snap["field"][:, kv]) and torch.equal(xyz_p, snap["xyz"][kv])
        st = opts.optimizers["fields"].state[field_p]
        assert torch.equal(st["step"], snap["step"])
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(st[k], snap[k].index_select(1, kv))
        if optimize_vertices:
            assert torch.equal(opts.optimizers["vertices"].state[xyz_p]["exp_avg"], snap["v_exp_avg"].index_select(0, kv))
        assert torch.equal(m._grad_acc, snap["acc"][kv]) and torch.equal(m._grad_cnt, snap["cnt"][kv])
        assert torch.equal(m.tetrahedra_occupancy, snap["occ"][pc])
        oco.check_coarsened(snap["xyz"].cpu().numpy(), snap["cells"].cpu().numpy(), m.tetrahedra_cells.cpu().numpy(), kv.cpu().numpy(),
                            pc.cpu().numpy())
        # the reloaded tracer traces like a fresh load, on the walk
        fresh = cpp.TetrahedraTracer(DEV)
        fresh.load_tetrahedra(xyz_p.detach(), m.tetrahedra_cells)
        assert m._tetrahedra_tracer.trace_stats()[0]
        a = m._tetrahedra_tracer.trace_rays(bundle.origins, bundle.directions, 1024)
        b = fresh.trace_rays(bundle.origins, bundle.directions, 1024)
        for k in TRACE_KEYS:
            assert torch.equal(a[k], b[k]), k
        print(f"optimize_vertices={optimize_vertices} step {step}: {res['passes']}")
    print(f"optimize_vertices={optimize_vertices}: vertices per step {sizes}")
    assert sizes[0] > sizes[1] >= sizes[3] and sizes[3] == sizes[-1]  # coarsenings at steps 2 and 4 only (coarsen_stop = 5)


def test_model_without_occupancy_field_raises(small_mesh):
    from tetranerf.nerfstudio import model as M

    V, C = small_mesh
    with pytest.raises(RuntimeError, match="use_occupancy_field"):
        M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), coarsen_every=1))


def test_no_coarsening_on_a_never_computed_buffer(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, _ = _model(V, C, field, params, coarsen_every=1, coarsen_start=0, occupancy_warmup_steps=100)
    opts = _optimizers(m)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers=opts))
    bundle = _bundle(M, 512, 3)
    m.train()
    cells = m.tetrahedra_cells.clone()
    for step in range(1, 4):
        opts.zero_grad_all()
        sum(m.get_loss_dict(m(bundle), {"image": torch.full((512, 3), 0.5, device=DEV)}).values()).backward()
        opts.optimizer_step_all()
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
    assert not bool(m.tetrahedra_occupancy.any())  # still in the warmup: never computed
    assert not m.coarsen(opts)["ready"] and torch.equal(m.tetrahedra_cells, cells)


def test_coarsened_checkpoint_loads_into_the_original_config(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, original = _model(V, C, field, params, coarsen_every=1, occupancy_warmup_steps=0)
    opts = _optimizers(m)
    bundle = _bundle(M, 512, 9)
    m.train()
    for _ in range(2):
        opts.zero_grad_all()
        sum(m.get_loss_dict(m(bundle), {"image": torch.full((512, 3), 0.5, device=DEV)}).values()).backward()
        opts.optimizer_step_all()
    res = m.coarsen(opts)
    assert res["vertices_after"] < res["vertices_before"]
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    osd = {k: copy.deepcopy(o.state_dict()) for k, o in opts.optimizers.items()}
    m.eval()
    with torch.no_grad():
        want = m(bundle)
    m2 = M.TetrahedraNerf(copy.deepcopy(original)).to(DEV)
    opts2 = _optimizers(m2)
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


def test_refine_and_coarsen_keep_the_walk(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, _ = _model(V, C, field, params, coarsen_every=2, coarsen_start=2, coarsen_stop=100, refine_every=2, refine_start=2,
                     refine_stop=100, refine_fraction=0.05, refine_passes=2, occupancy_warmup_steps=0)
    opts = _optimizers(m)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers=opts))
    assert len(cbs) == 3
    bundle = _bundle(M, 1024, 4)
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(1)).to(DEV)}
    m.train()
    sizes = []
    for step in range(1, 9):
        opts.zero_grad_all()
        sum(m.get_loss_dict(m(bundle), target).values()).backward()
        opts.optimizer_step_all()
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
        assert m.get_tetrahedra_tracer().trace_stats()[0], step
        sizes.append((len(m.tetrahedra_vertices), len(m.tetrahedra_cells)))
    print(f"(vertices, tetrahedra) per step: {sizes}")
    assert len(set(sizes)) > 1


def test_full_size_mesh():
    from tetranerf import cpp

    V, C = syn.delaunay_mesh(300_000, seed=0)
    assert 2_000_000 < len(C) < 2_050_000
    empty = np.random.default_rng(0).random(len(C)) < 0.98
    out = _gpu_pass(V, C, empty)
    kv, pc, C1 = (out[k].cpu().numpy() for k in ("kept_vertex", "parent_cell", "cells"))
    assert out["n_removed"] > 0 and len(kv) == len(V) - out["n_removed"] and len(C1) == len(C) - out["n_cells_removed"]
    info = oco.check_coarsened(V, C, C1, kv, pc)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V[kv]).to(DEV), out["cells"])
    assert tr.trace_stats()[0]
    print(f"2.02 M mesh, 98 % empty: proposed {out['n_proposed']}, removed {out['n_removed']} vertices and {out['n_cells_removed']} "
          f"tetrahedra; {info}")
