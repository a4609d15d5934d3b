"""CPU: the oracle of one longest-edge bisection pass (oracle/refine.py, DESIGN §4.14) and the model's host side of refinement.
  * properties of the pass on Delaunay meshes, the bottle mesh and hand-made cases: accepted edges share no tetrahedron and include the
    top proposal; the refined mesh is conforming (no face with more than two owners, the hull area unchanged); every child has half its
    parent's signed volume and its orientation; an empty mask is a bitwise no-op; the cap keeps the highest-priority edges;
  * the model's candidate selection (top fraction, ties, score > 0), its statistics, the migration of parameters, optimizer moments and
    occupancy, and the in-place resize of a checkpoint load."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import refine as orf
from tetranerf.b200 import synthetic as syn

ROOT = Path(__file__).resolve().parents[1]


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _meshes():
    V, C = syn.delaunay_mesh(600, seed=4)
    yield "delaunay", V, C
    yield "bottle", *_bottle()
    yield "cube", syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()


def _tets_of(cells, key):
    a, b = int(key >> np.uint64(32)), int(key & np.uint64(0xFFFFFFFF))
    return set(np.nonzero((cells == a).any(1) & (cells == b).any(1))[0].tolist())


def _check_pass(V, C, cand, out, max_new=None):
    T = len(C)
    keys, len2 = orf.edge_table(V, C)
    # accepted edges are tetrahedron-disjoint, and the top proposal is among them
    acc = out["accepted_all"]
    seen = set()
    for k in acc:
        ts = _tets_of(C, k)
        assert not (ts & seen)
        seen |= ts
    if out["n_proposed"]:
        rows = np.nonzero(cand)[0]
        best = orf._best(keys[rows], len2[rows], np.ones((len(rows), 6), bool))
        pk, pl = keys[rows, best], len2[rows, best]
        top = pk[np.lexsort((pk, -pl))[0]]
        assert top in acc
        assert out["n_accepted"] >= 1
    if max_new is not None:
        assert out["n_accepted"] == min(max_new, len(acc))
    # children: half the parent's signed volume, same orientation; the parent slot is the other half (with the exact, float64
    # midpoints: the model's fp32 midpoints move them by one rounding)
    newV = orf.migrate_vertices(V, out["parent_edge"], 0)
    exact = orf.migrate_vertices(V.astype(np.float64), out["parent_edge"], 0)
    vol0 = orf.signed_volumes(V, C)
    vol1 = orf.signed_volumes(exact, out["cells"])
    pc = out["parent_cell"]
    assert np.array_equal(pc[:T], np.arange(T))
    assert len(out["cells"]) == T + out["n_split"]
    split = np.zeros(T, bool)
    split[pc[T:]] = True
    np.testing.assert_array_equal(out["cells"][:T][~split], C[~split])
    scale = np.abs(vol0).max()
    np.testing.assert_allclose(vol1[:T][split], vol0[split] / 2, rtol=0, atol=1e-12 * scale)
    np.testing.assert_allclose(vol1[T:], vol0[pc[T:]] / 2, rtol=0, atol=1e-12 * scale)
    solid = np.abs(vol0[pc[T:]]) > 1e-9 * scale  # (the bottle has flat tetrahedra)
    assert (np.sign(vol1[T:]) == np.sign(vol0[pc[T:]]))[solid].all()
    # conforming: no face has more than two owners, and the hull keeps its area
    _, counts = orf.face_owners(out["cells"])
    assert counts.max() <= 2
    assert orf.hull_area(exact, out["cells"]) == pytest.approx(orf.hull_area(V, C), rel=1e-12)
    # new vertices: ids V.. in ascending key order, at their edge's midpoint
    pe = out["parent_edge"].astype(np.int64)
    assert (pe[:, 0] < pe[:, 1]).all()
    k = (pe[:, 0].astype(np.uint64) << np.uint64(32)) | pe[:, 1].astype(np.uint64)
    assert (np.diff(k.astype(np.float64)) > 0).all() if len(k) > 1 else True
    return newV


@pytest.mark.parametrize("name,V,C", list(_meshes()), ids=lambda x: x if isinstance(x, str) else "")
def test_pass_properties(name, V, C):
    rng = np.random.default_rng(7)
    for frac in (0.05, 0.3, 1.0):
        cand = rng.random(len(C)) < frac
        out = orf.refine_edges(V, C, cand)
        assert out["n_accepted"] == len(out["accepted_all"])
        _check_pass(V, C, cand, out)
    # every tetrahedron a candidate, and the cap
    cand = np.ones(len(C), bool)
    out = orf.refine_edges(V, C, cand)
    _check_pass(V, C, cand, out)
    if out["n_accepted"] > 2:
        capped = orf.refine_edges(V, C, cand, max_new_vertices=2)
        _check_pass(V, C, cand, capped, max_new=2)
        kept = (capped["parent_edge"][:, 0].astype(np.uint64) << np.uint64(32)) | capped["parent_edge"][:, 1].astype(np.uint64)
        assert set(kept.tolist()) <= set(out["accepted_all"].tolist())


def test_empty_mask_is_a_noop():
    V, C = syn.delaunay_mesh(300, seed=1)
    out = orf.refine_edges(V, C, np.zeros(len(C), bool))
    assert out["n_proposed"] == out["n_accepted"] == out["n_split"] == 0
    assert np.array_equal(out["cells"], C) and np.array_equal(out["parent_cell"], np.arange(len(C))) and out["parent_edge"].shape == (0, 2)


def test_min_length():
    V, C = syn.delaunay_mesh(300, seed=2)
    keys, len2 = orf.edge_table(V, C)
    longest = np.sqrt(len2.max(1))
    ml = float(np.median(longest))
    out = orf.refine_edges(V, C, np.ones(len(C), bool), min_length=ml)
    rows = np.arange(len(C))
    best = orf._best(keys, len2, np.ones_like(keys, bool))
    prop = len2[rows, best] >= np.float64(np.float32(ml)) ** 2
    assert out["n_proposed"] == len(np.unique(keys[rows[prop], best[prop]]))
    assert orf.refine_edges(V, C, np.ones(len(C), bool), min_length=1e9)["n_proposed"] == 0


def test_boundary_edge_and_shared_edge():
    # a single tetrahedron: its longest edge lies on the hull and is accepted
    V = np.array([[0, 0, 0], [3, 0, 0], [1.5, 1, 0], [1.5, 0, 1]], np.float32)
    C = np.array([[0, 1, 2, 3]], np.int32)
    out = orf.refine_edges(V, C, np.ones(1, bool))
    assert out["n_accepted"] == 1 and out["parent_edge"].tolist() == [[0, 1]]
    assert out["cells"].tolist() == [[0, 4, 2, 3], [4, 1, 2, 3]]
    _check_pass(V, C, np.ones(1, bool), out)
    # eight tetrahedra around one long axis edge (0, 1): one candidate proposes it, all eight vote for it, all eight split
    n = 8
    ring = [[np.cos(2 * np.pi * i / n) * 0.3, np.sin(2 * np.pi * i / n) * 0.3, 0.5] for i in range(n)]
    V = np.array([[0, 0, -1], [0, 0, 2]] + ring, np.float32)
    C = np.array([[0, 1, 2 + i, 2 + (i + 1) % n] for i in range(n)], np.int32)
    cand = np.zeros(n, bool)
    cand[3] = True
    out = orf.refine_edges(V, C, cand)
    assert out["n_proposed"] == 1 and out["n_accepted"] == 1 and out["n_split"] == n
    assert out["parent_cell"][n:].tolist() == list(range(n))
    _check_pass(V, C, cand, out)
    # an edge not every neighbour votes for is refused: tetrahedron 0 gets a longer edge of its own proposed too
    V2 = V.copy()
    V2[2] = [3.0, 0.0, 0.5]
    out = orf.refine_edges(V2, C, np.ones(n, bool))
    _check_pass(V2, C, np.ones(n, bool), out)


# ---- the model's host side --------------------------------------------------------------------------------------------------------
def test_select_candidates():
    from tetranerf.b200.refine import select_candidates

    cells = torch.tensor([[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 5], [0, 0, 0, 0], [5, 5, 5, 5]], dtype=torch.int32)
    score = torch.tensor([0.0, 0.0, 0.0, 0.0, 4.0, 4.0])  # tet scores: 0, 1, 2, 0, 4
    assert select_candidates(score, cells, 0.4).tolist() == [False, False, True, False, True]
    assert select_candidates(score, cells, 1.0).tolist() == [False, True, True, False, True]  # score 0 never a candidate
    assert select_candidates(score, cells, 0.1).tolist() == [False] * 5  # floor(0.5) = 0
    tie = torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, 1.0])  # every tetrahedron scores 1: ties go to the smaller index
    assert select_candidates(tie, cells, 0.4).tolist() == [True, True, False, False, False]


def _model(V, C, **kw):
    from tetranerf.nerfstudio import model as M

    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), **kw))
    m.load_state_dict({"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C),
                       "tetrahedra_field": torch.randn(64, len(V), generator=torch.Generator().manual_seed(0))}, strict=False)
    return m, M


def test_callbacks_off_by_default():
    V, C = syn.delaunay_mesh(100, seed=0)
    m, M = _model(V, C)
    assert m.get_training_callbacks(M.TrainingCallbackAttributes()) == []


def test_statistics():
    V, C = syn.delaunay_mesh(100, seed=0)
    m, M = _model(V, C, refine_every=10)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes())
    assert len(cbs) == 2 and all(M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION in cb.where_to_run for cb in cbs)
    g = torch.zeros(64, len(V))
    g[:, 3] = 2.0
    g[5, 7] = -3.0
    m.tetrahedra_field.grad = g
    cbs[0].run_callback_at_location(1, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
    g2 = torch.zeros(64, len(V))
    g2[0, 3] = 1.0
    m.tetrahedra_field.grad = g2
    cbs[0].run_callback_at_location(2, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
    assert m._grad_acc[3].item() == pytest.approx(16.0 + 1.0) and m._grad_cnt[3].item() == 2
    assert m._grad_acc[7].item() == pytest.approx(3.0) and m._grad_cnt[7].item() == 1
    assert m._grad_cnt.sum().item() == 3
    assert "_grad_acc" not in str(list(m.state_dict()))


@pytest.mark.parametrize("optimize_vertices", [False, True])
def test_apply_refinement_migrates_parameters_and_moments(optimize_vertices):
    V, C = syn.delaunay_mesh(200, seed=3)
    m, M = _model(V, C, refine_every=1, use_occupancy_field=True, optimize_vertices=optimize_vertices)
    m.tetrahedra_occupancy.copy_(torch.rand(len(C), generator=torch.Generator().manual_seed(1)))
    groups = m.get_param_groups()
    opts = {k: torch.optim.RAdam(v, lr=1e-3) for k, v in groups.items()}
    for _ in range(2):
        for p in m.parameters():
            p.grad = torch.randn_like(p)
        for o in opts.values():
            o.step()
    field, xyz, occ = m.tetrahedra_field, m.tetrahedra_vertices, m.tetrahedra_occupancy.clone()
    before = {k: v.clone() for k, v in opts["fields"].state[field].items() if isinstance(v, torch.Tensor)}
    f0, x0 = field.detach().clone(), xyz.detach().clone()
    V = x0.numpy()  # the positions the optimizer moved
    alive = (field * 2).sum() + (xyz * 2).sum()  # a graph that outlives the refinement, as the trainer's last loss does
    alive.backward()
    cand = np.zeros(len(C), bool)
    cand[::7] = True
    o1 = orf.refine_edges(V, C, cand)
    V1 = orf.migrate_vertices(V, o1["parent_edge"], 0)
    o2 = orf.refine_edges(V1, o1["cells"], np.zeros(len(o1["cells"]), bool) | (np.arange(len(o1["cells"])) % 5 == 0))
    V2 = orf.migrate_vertices(V1, o2["parent_edge"], 0)
    pes = [torch.from_numpy(o["parent_edge"]) for o in (o1, o2)]
    pcs = [torch.from_numpy(o["parent_cell"]) for o in (o1, o2)]
    m._apply_refinement(pes, pcs, torch.from_numpy(V2), torch.from_numpy(o2["cells"]), opts)
    assert m.tetrahedra_field is field and m.tetrahedra_vertices is xyz and field.grad is None
    nV = len(V2)
    assert field.shape == (64, nV) and xyz.shape == (nV, 3) and m.tetrahedra_cells.shape == (len(o2["cells"]), 4)
    assert m.config.num_tetrahedra_vertices == nV and m.config.num_tetrahedra_cells == len(o2["cells"])
    assert torch.equal(field[:, : len(V)], f0) and torch.equal(xyz[: len(V)], x0)
    want = orf.migrate_vertices(orf.migrate_vertices(f0.numpy(), o1["parent_edge"], 1), o2["parent_edge"], 1)
    assert np.array_equal(field.detach().numpy(), want)
    st = opts["fields"].state[field]
    for k in ("exp_avg", "exp_avg_sq"):
        assert st[k].shape == field.shape and torch.equal(st[k][:, : len(V)], before[k][:, : len(V)])
        w = orf.migrate_vertices(orf.migrate_vertices(before[k].numpy(), o1["parent_edge"], 1), o2["parent_edge"], 1)
        assert np.array_equal(st[k].numpy(), w)
    assert torch.equal(st["step"], before["step"])
    if optimize_vertices:
        assert opts["vertices"].state[xyz]["exp_avg"].shape == (nV, 3)
    want_occ = occ[torch.from_numpy(o1["parent_cell"]).long()][torch.from_numpy(o2["parent_cell"]).long()]
    assert torch.equal(m.tetrahedra_occupancy, want_occ)
    # a new graph differentiates the resized parameters, and an optimizer step runs on the new shapes
    ((field * 3).sum() + (xyz * 3).sum()).backward()
    assert field.grad.shape == field.shape and alive is not None
    for p in m.parameters():
        p.grad = torch.randn_like(p)
    for o in opts.values():
        o.step()
    assert torch.isfinite(field).all()


def test_checkpoint_resize_keeps_parameters():
    V, C = syn.delaunay_mesh(200, seed=3)
    m, M = _model(V, C, refine_every=1, use_occupancy_field=True, optimize_vertices=True)
    o = orf.refine_edges(V, C, np.arange(len(C)) % 3 == 0)
    m._apply_refinement([torch.from_numpy(o["parent_edge"])], [torch.from_numpy(o["parent_cell"])],
                        torch.from_numpy(orf.migrate_vertices(V, o["parent_edge"], 0)), torch.from_numpy(o["cells"]), None)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m2, _ = _model(V, C, refine_every=1, use_occupancy_field=True, optimize_vertices=True)
    groups = m2.get_param_groups()
    opt = torch.optim.RAdam(groups["fields"], lr=1e-3)
    field, xyz = m2.tetrahedra_field, m2.tetrahedra_vertices
    m2.load_state_dict(sd, strict=True)
    assert m2.tetrahedra_field is field and m2.tetrahedra_vertices is xyz
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert m2.config.num_tetrahedra_vertices == len(sd["tetrahedra_vertices"])
    field.grad = torch.randn_like(field)
    opt.step()
