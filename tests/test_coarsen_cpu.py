"""CPU: the oracle of one empty-space vertex-removal pass (oracle/coarsen.py, DESIGN §4.18) and the model's host side of coarsening.
  * properties of the pass on Delaunay meshes and the bottle mesh with random empty masks: the output passes the independent validity
    check (conforming, same hull, every cell with its parent's orientation, the same volume); accepted vertices share no cell; the top
    proposal is removed; no hull vertex and no vertex with an occupied cell is removed; the cap; determinism; no-op cases;
  * the model: the options it refuses, its callbacks, the migration of parameters, optimizer moments, statistics and occupancy, the
    guard against a never-computed occupancy buffer, and a coarsened checkpoint loaded into the original config."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import coarsen as oco
from tetranerf.b200 import synthetic as syn

ROOT = Path(__file__).resolve().parents[1]


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _meshes():
    yield "delaunay", *syn.delaunay_mesh(800, seed=4)
    yield "bottle", *_bottle()


def _check_pass(V, C, empty, out, max_removed=None):
    oco.check_coarsened(V, C, out["cells"], out["kept_vertex"], out["parent_cell"])
    # accepted vertices share no input cell
    acc = out["accepted_all"]
    seen = set()
    for a in acc:
        ts = set(np.nonzero((C == a).any(1))[0].tolist())
        assert not (ts & seen)
        seen |= ts
    # the top proposal is removed
    tgt = out["target"]
    prop = np.nonzero(tgt >= 0)[0]
    assert out["n_proposed"] == len(prop)
    if len(prop):
        X = V.astype(np.float64)
        d = X[prop] - X[tgt[prop]]
        l2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        top = prop[np.lexsort((prop, l2))[0]]
        if max_removed is None or max_removed > 0:
            assert top in out["removed"]
    # no hull vertex, no vertex with an occupied (or no) cell
    hull = np.unique(oco.hull_faces(C))
    occupied = np.unique(C[~empty])
    removed = out["removed"]
    assert not np.isin(removed, hull).any() and not np.isin(removed, occupied).any()
    assert np.isin(removed, C).all()
    assert out["n_removed"] == len(removed) == len(V) - len(out["kept_vertex"])
    assert out["n_cells_removed"] == len(C) - len(out["cells"])
    if max_removed is not None:
        assert out["n_removed"] == min(max_removed, len(acc))
    assert set(removed.tolist()) <= set(acc.tolist())
    # kept vertices and parent cells ascending; unchanged cells renumbered only
    assert (np.diff(out["kept_vertex"]) > 0).all() and (np.diff(out["parent_cell"]) > 0).all()


@pytest.mark.parametrize("name,V,C", list(_meshes()), ids=lambda x: x if isinstance(x, str) else "")
def test_pass_properties(name, V, C):
    rng = np.random.default_rng(11)
    for frac in (1.0, 0.97, 0.8):
        empty = rng.random(len(C)) < frac
        out = oco.coarsen_vertices(V, C, empty)
        _check_pass(V, C, empty, out)
        print(f"{name} empty {frac}: proposed {out['n_proposed']} removed {out['n_removed']} cells removed {out['n_cells_removed']}")
    empty = np.ones(len(C), bool)
    full = oco.coarsen_vertices(V, C, empty)
    assert full["n_removed"] > 0
    capped = oco.coarsen_vertices(V, C, empty, max_removed=3)
    _check_pass(V, C, empty, capped, max_removed=3)
    # the cap keeps the highest-priority accepted vertices
    acc = full["removed"]
    X = V.astype(np.float64)
    d = X[acc] - X[full["target"][acc]]
    l2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    assert np.array_equal(capped["removed"], np.sort(acc[np.lexsort((acc, l2))[:3]]))


def test_repeated_passes_stay_valid():
    V, C = syn.delaunay_mesh(500, seed=2)
    X, cells = V, C
    kept, parent = np.arange(len(V)), np.arange(len(C))
    for _ in range(3):
        empty = np.ones(len(cells), bool)
        out = oco.coarsen_vertices(X, cells, empty)
        _check_pass(X, cells, empty, out)
        X, cells = X[out["kept_vertex"]], out["cells"]
        kept, parent = kept[out["kept_vertex"]], parent[out["parent_cell"]]
    oco.check_coarsened(V, C, cells, kept, parent)  # the three passes together, against the original mesh
    assert len(X) < len(V)


def test_cap_zero_and_occupied_mesh_change_nothing():
    V, C = syn.delaunay_mesh(300, seed=1)
    for empty, cap in ((np.ones(len(C), bool), 0), (np.zeros(len(C), bool), None)):
        out = oco.coarsen_vertices(V, C, empty, max_removed=cap)
        assert out["n_removed"] == out["n_cells_removed"] == 0
        assert np.array_equal(out["cells"], C) and np.array_equal(out["parent_cell"], np.arange(len(C)))
        assert np.array_equal(out["kept_vertex"], np.arange(len(V)))
    assert oco.coarsen_vertices(V, C, np.zeros(len(C), bool))["n_proposed"] == 0


def test_deterministic():
    V, C = syn.delaunay_mesh(400, seed=6)
    empty = np.random.default_rng(0).random(len(C)) < 0.95
    a, b = oco.coarsen_vertices(V, C, empty), oco.coarsen_vertices(V, C, empty)
    for k in ("cells", "kept_vertex", "parent_cell", "target"):
        assert np.array_equal(a[k], b[k]), k


def test_no_interior_vertex_removes_nothing():
    # the cube's five tetrahedra and a single tetrahedron: every vertex is on the hull
    for V, C in ((syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()),
                 (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32), np.array([[0, 1, 2, 3]], np.int32))):
        out = oco.coarsen_vertices(V, C, np.ones(len(C), bool))
        assert out["n_proposed"] == out["n_removed"] == 0 and np.array_equal(out["cells"], C)


def test_single_interior_vertex_collapses_into_its_nearest_valid_neighbour():
    # an octahedron around a centre vertex 0 slightly off the middle: 8 cells, 0 collapses into its nearest vertex (+x), which removes the
    # 4 cells around the edge and leaves 4 cones from that vertex; the hull (the 8 octahedron faces) is kept
    V = np.array([[0.1, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    C = []
    for x in (1, 2):
        for y in (3, 4):
            for z in (5, 6):
                c = [0, x, y, z]
                s = oco.cell_signs(V.astype(np.float64), np.array([c]))[0]
                C.append(c if s > 0 else [0, x, z, y])
    C = np.array(C, np.int32)
    out = oco.coarsen_vertices(V, C, np.ones(len(C), bool))
    assert out["n_proposed"] == out["n_removed"] == 1 and out["target"][0] == 1 and out["n_cells_removed"] == 4
    assert np.array_equal(out["kept_vertex"], np.arange(1, 7))
    _check_pass(V, C, np.ones(len(C), bool), out)
    # one occupied cell keeps the centre
    empty = np.ones(len(C), bool)
    empty[5] = False
    assert oco.coarsen_vertices(V, C, empty)["n_removed"] == 0


def test_checker_catches_a_fold():
    V, C = syn.delaunay_mesh(200, seed=3)
    out = oco.coarsen_vertices(V, C, np.ones(len(C), bool))
    bad = out["cells"].copy()
    bad[0, [0, 1]] = bad[0, [1, 0]]  # flip one cell's orientation
    with pytest.raises(AssertionError, match="orientation"):
        oco.check_coarsened(V, C, bad, out["kept_vertex"], out["parent_cell"])
    with pytest.raises(AssertionError):  # drop a cell: a hole in the domain
        oco.check_coarsened(V, C, out["cells"][1:], out["kept_vertex"], out["parent_cell"][1:])


# ---- the model's host side --------------------------------------------------------------------------------------------------------
def _model(V, C, **kw):
    from tetranerf.nerfstudio import model as M

    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), **kw))
    m.load_state_dict({"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C),
                       "tetrahedra_field": torch.randn(64, len(V), generator=torch.Generator().manual_seed(0))}, strict=False)
    return m, M


def test_requires_the_occupancy_field_and_the_fused_pipeline():
    V, C = syn.delaunay_mesh(100, seed=0)
    with pytest.raises(RuntimeError, match="use_occupancy_field"):
        _model(V, C, coarsen_every=10)
    with pytest.raises(RuntimeError, match="hidden_size"):
        _model(V, C, coarsen_every=10, use_occupancy_field=True, hidden_size=64)
    m, _ = _model(V, C, use_occupancy_field=True)
    assert m.config.coarsen_every == 0
    m, _ = _model(V, C)
    with pytest.raises(RuntimeError, match="use_occupancy_field"):
        m.coarsen()


def test_callbacks():
    V, C = syn.delaunay_mesh(100, seed=0)
    m, M = _model(V, C, coarsen_every=10, use_occupancy_field=True)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes())
    assert len(cbs) == 1 and M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION in cbs[0].where_to_run
    m, M = _model(V, C, coarsen_every=10, refine_every=10, use_occupancy_field=True)
    calls = []
    m.coarsen = lambda optimizers=None: calls.append("coarsen")
    m.refine = lambda optimizers=None: calls.append("refine")
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes())
    assert len(cbs) == 3
    for step in (995, 1000, 1001, 1010):
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
    assert calls == ["coarsen", "refine", "coarsen", "refine"]  # both due at 1000 and 1010: coarsening first


def test_never_computed_occupancy_is_not_coarsened():
    V, C = syn.delaunay_mesh(200, seed=3)
    m, _ = _model(V, C, coarsen_every=1, use_occupancy_field=True, occupancy_warmup_steps=0)
    cells = m.tetrahedra_cells.clone()
    m._occ_step = 5
    m._occ_ready = True  # the buffer is all zeros: never computed, although flagged
    res = m.coarsen()
    assert not res["ready"] and res["passes"] == [] and torch.equal(m.tetrahedra_cells, cells)
    m.tetrahedra_occupancy.fill_(1.0)
    m._occ_ready = False
    assert not m.coarsen()["ready"]
    m._occ_ready, m._occ_step = True, 0  # before the warmup has passed
    m.config.occupancy_warmup_steps = 3
    assert not m.coarsen()["ready"]
    m._occ_step = 4
    assert m.coarsen_ready()


@pytest.mark.parametrize("optimize_vertices", [False, True])
def test_apply_coarsening_migrates_parameters_moments_and_statistics(optimize_vertices):
    V, C = syn.delaunay_mesh(300, seed=3)
    m, M = _model(V, C, coarsen_every=1, use_occupancy_field=True, optimize_vertices=optimize_vertices)
    occ = torch.rand(len(C), generator=torch.Generator().manual_seed(1))
    m.tetrahedra_occupancy.copy_(occ)
    opts = {k: torch.optim.RAdam(v, lr=1e-3) for k, v in m.get_param_groups().items()}
    for _ in range(2):
        for p in m.parameters():
            p.grad = torch.randn_like(p)
        for o in opts.values():
            o.step()
    m._grad_acc = torch.rand(len(V))
    m._grad_cnt = torch.randint(0, 5, (len(V),), dtype=torch.int32)
    acc0, cnt0 = m._grad_acc.clone(), m._grad_cnt.clone()
    field, xyz = m.tetrahedra_field, m.tetrahedra_vertices
    f0, x0 = field.detach().clone(), xyz.detach().clone()
    st0 = {g: {k: v.clone() for k, v in o.state[p].items()} for g, o in opts.items() for p in o.param_groups[0]["params"] if p is field or p is xyz}
    alive = (field * 2).sum() + (xyz * 2).sum()
    alive.backward()
    out = oco.coarsen_vertices(x0.numpy(), C, occ.numpy() < 0.9)
    assert out["n_removed"] > 0
    kv, pc = torch.from_numpy(out["kept_vertex"]).long(), torch.from_numpy(out["parent_cell"]).long()
    m._apply_coarsening(kv, pc, x0[kv], torch.from_numpy(out["cells"]), opts)
    assert m.tetrahedra_field is field and m.tetrahedra_vertices is xyz and field.grad is None
    assert torch.equal(field, f0[:, kv]) and torch.equal(xyz, x0[kv]) and torch.equal(m.tetrahedra_cells, torch.from_numpy(out["cells"]))
    assert m.config.num_tetrahedra_vertices == len(kv) and m.config.num_tetrahedra_cells == len(pc)
    assert torch.equal(m.tetrahedra_occupancy, occ[pc])
    assert torch.equal(m._grad_acc, acc0[kv]) and torch.equal(m._grad_cnt, cnt0[kv])
    st = opts["fields"].state[field]
    for k in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(st[k], st0["fields"][k].index_select(1, kv))
    assert torch.equal(st["step"], st0["fields"]["step"])
    if optimize_vertices:
        vs = opts["vertices"].state[xyz]
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(vs[k], st0["vertices"][k].index_select(0, kv))
    ((field * 3).sum() + (xyz * 3).sum()).backward()
    assert field.grad.shape == field.shape
    for o in opts.values():
        o.step()
    assert torch.isfinite(field).all()


def test_coarsened_checkpoint_loads_into_the_original_config():
    V, C = syn.delaunay_mesh(300, seed=3)
    m, M = _model(V, C, coarsen_every=1, use_occupancy_field=True, optimize_vertices=True)
    out = oco.coarsen_vertices(V, C, np.ones(len(C), bool))
    kv, pc = torch.from_numpy(out["kept_vertex"]).long(), torch.from_numpy(out["parent_cell"]).long()
    m._apply_coarsening(kv, pc, torch.from_numpy(V)[kv], torch.from_numpy(out["cells"]), None)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m2, _ = _model(V, C, coarsen_every=1, use_occupancy_field=True, optimize_vertices=True)
    opt = torch.optim.RAdam(m2.get_param_groups()["fields"], lr=1e-3)
    field, xyz = m2.tetrahedra_field, m2.tetrahedra_vertices
    m2.load_state_dict(sd, strict=True)
    assert m2.tetrahedra_field is field and m2.tetrahedra_vertices is xyz and len(xyz) < len(V)
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert m2.config.num_tetrahedra_vertices == len(kv) and m2.config.num_tetrahedra_cells == len(pc)
    field.grad = torch.randn_like(field)
    opt.step()
