"""CPU: the oracle of one Delaunay flip pass (oracle/flip.py, DESIGN §4.19) and the model's host side of flipping.
  * the insphere predicate: wherever the float64 restatement certifies a sign, it is the exact sign (Python integers on the fp32
    positions, which are dyadic rationals), on Delaunay, bottle and sliver meshes and on them after refinement, coarsening and a jitter;
  * properties of the pass on those meshes: the output passes the independent validity check (conforming, same hull, same vertices,
    certified orientations, the same volume); accepted flips share no cell; the top proposal is applied; every applied flip's face is
    illegal in exact arithmetic; the cap; determinism; a mesh with no certified illegal face comes back unchanged;
  * the fixed point: repeated passes terminate, every face still certified illegal then proposes nothing, and the illegal count fell;
  * the model: the callback schedule, the flip at the end of refine() and coarsen(), occupancy as the maximum over the sources, the
    untouched per-vertex state, and a flipped checkpoint loaded into the original config."""
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import coarsen as oco
from oracle import flip as ofl
from oracle import refine as ore
from tetranerf.b200 import synthetic as syn
from test_gpu_slivers import sliver_mesh

ROOT = Path(__file__).resolve().parents[1]


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _refined(V, C, passes=3, frac=0.2, seed=0):
    rng = np.random.default_rng(seed)
    for _ in range(passes):
        out = ore.refine_edges(V, C, rng.random(len(C)) < frac)
        V, C = ore.migrate_vertices(V, out["parent_edge"]).astype(np.float32), out["cells"]
    return V, C


def _coarsened(V, C, passes=3, frac=0.9, seed=0):
    rng = np.random.default_rng(seed)
    for _ in range(passes):
        out = oco.coarsen_vertices(V, C, rng.random(len(C)) < frac)
        V, C = V[out["kept_vertex"]], out["cells"]
    return V, C


def _jittered(V, C, rel=0.003, seed=0, keep_hull=False):
    """every vertex (keep_hull: every vertex off the hull) moved by rel times the box diagonal, then the vertices of any cell whose
    certified orientation changed put back, until none does: a moved mesh that is still a valid tetrahedralisation, as the fold guard
    keeps a trained one"""
    rng = np.random.default_rng(seed)
    scale = float(np.linalg.norm(V.max(0) - V.min(0)))
    X = (V + rel * scale * rng.standard_normal(V.shape)).astype(np.float32)
    if keep_hull:
        hull = np.unique(oco.hull_faces(C))
        X[hull] = V[hull]
    s0 = oco.cell_signs(V.astype(np.float64), C)
    while True:
        bad = oco.cell_signs(X.astype(np.float64), C) != s0
        if not bad.any():
            return X, C
        X[np.unique(C[bad])] = V[np.unique(C[bad])]


def base_meshes():
    return {"delaunay": syn.delaunay_mesh(800, seed=4), "bottle": _bottle(), "sliver": sliver_mesh(300)}


def flip_meshes(names=("delaunay", "bottle", "sliver")):
    """name -> (V f32, C i32): each base mesh as it is and after three refine passes, three coarsen passes and an unfolded 0.3 % jitter"""
    out = {}
    for name, (V, C) in base_meshes().items():
        if name not in names:
            continue
        out[name] = (V, C)
        out[name + "+refined"] = _refined(V, C)
        out[name + "+coarsened"] = _coarsened(V, C)
        out[name + "+jittered"] = _jittered(V, C)
    return out


MESHES = flip_meshes()


# ---- exact arithmetic ----------------------------------------------------------------------------------------------------------------
def _exact_points(V):
    """the fp32 positions as Python integers over one common power-of-two denominator (insphere / orient3d signs are scale-invariant)"""
    fr = [Fraction(float(x)) for x in np.asarray(V, np.float32).reshape(-1)]
    den = max(f.denominator for f in fr)
    ints = [int(f * den) for f in fr]
    return [tuple(ints[3 * i:3 * i + 3]) for i in range(len(V))]


def _exact_insphere(P, a, b, c, d, e):
    pe = P[e]
    r = [[P[v][k] - pe[k] for k in range(3)] for v in (a, b, c, d)]
    rows = [x + [x[0] * x[0] + x[1] * x[1] + x[2] * x[2]] for x in r]

    def det3(m):
        return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
                + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))

    det = 0
    for j in range(4):  # det [x_i - e, |x_i - e|^2] (rows a, b, c, d) by Laplace along the lift column: Shewchuk's insphere
        minor = [[row[k] for k in range(3)] for i, row in enumerate(rows) if i != j]
        det += (-1) ** (j + 3) * rows[j][3] * det3(minor)
    return (det > 0) - (det < 0)


def _exact_orient(P, a, b, c, d):
    m = [[P[v][k] - P[d][k] for k in range(3)] for v in (a, b, c)]
    det = (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
           + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))
    return (det > 0) - (det < 0)


def _exact_illegal(P, C, t0, e):
    c0 = [int(v) for v in C[t0]]
    return _exact_insphere(P, *c0, int(e)) * _exact_orient(P, *c0)


def test_exact_insphere_convention():
    # the unit tetrahedron, positively oriented, and a point inside / outside its circumsphere
    X = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [0.25, 0.25, 0.25], [2, 2, 2]], np.float32)
    P = _exact_points(X)
    a, b, c, d = 0, 1, 2, 3
    if _exact_orient(P, a, b, c, d) < 0:
        b, c = c, b
    assert _exact_orient(P, a, b, c, d) > 0
    assert _exact_insphere(P, a, b, c, d, 4) == 1 and _exact_insphere(P, a, b, c, d, 5) == -1
    Xd = X.astype(np.float64)
    s = ofl._insphere(Xd[[a, a]], Xd[[b, b]], Xd[[c, c]], Xd[[d, d]], Xd[[4, 5]])
    assert s.tolist() == [1, -1]


@pytest.mark.parametrize("name", list(MESHES))
def test_insphere_certified_sign_is_exact(name):
    V, C = MESHES[name]
    X = V.astype(np.float64)
    c = C.astype(np.int64)
    F, slot = ofl.face_table(c)
    start, length = ofl._runs(F)
    p = start[length == 2]
    t0, t1 = slot[p] // 4, slot[p + 1] // 4
    e = c[t1, slot[p + 1] % 4]
    got = ofl._insphere(X[c[t0, 0]], X[c[t0, 1]], X[c[t0, 2]], X[c[t0, 3]], X[e])
    P = _exact_points(V)
    wrong = 0
    for i in np.nonzero(got)[0]:
        wrong += _exact_insphere(P, *(int(v) for v in c[t0[i]]), int(e[i])) != got[i]
    print(f"{name}: {len(p)} interior faces, {(got == 0).sum()} uncertified insphere signs")
    assert wrong == 0


def _check_pass(V, C, out, max_flips=None):
    info = ofl.check_flipped(V, C, out["cells"])
    pr = out["prop"]
    T = len(C)
    # accepted flips share no cell
    owners = lambda i: {int(pr["t0"][i]), int(pr["t1"][i])} | ({int(pr["t2"][i])} if pr["kind"][i] == 3 else set())
    seen = set()
    for i in out["accepted_all"]:
        assert not (owners(i) & seen)
        seen |= owners(i)
    # the top proposal is applied (unless the cap is 0)
    prop = np.nonzero(pr["kind"] > 0)[0]
    assert out["n_proposed"] == len(prop)
    if len(prop) and (max_flips is None or max_flips > 0):
        assert prop[0] in out["kept"]
    # every applied flip's face is illegal in exact arithmetic
    P = _exact_points(V)
    c = C.astype(np.int64)
    for i in out["kept"]:
        t0 = int(pr["t0"][i])
        tt1 = int(pr["t1"][i])
        e = [v for v in c[tt1] if v not in c[t0]]
        assert len(e) == 1 and _exact_illegal(P, c, t0, e[0]) > 0
    n = len(out["kept"])
    assert out["n_23"] + out["n_32"] == n and len(out["cells"]) == T + out["n_23"] - out["n_32"]
    if max_flips is not None:
        assert n == min(max_flips, len(out["accepted_all"]))
    # sources: ascending, padded with -1; an unchanged cell keeps its own cell
    src = out["sources"]
    plain = src[:, 1] < 0
    assert np.array_equal(out["cells"][plain], C[src[plain, 0]])
    assert (plain.sum() == T - 2 * out["n_23"] - 3 * out["n_32"])
    return info


@pytest.mark.parametrize("name", list(MESHES))
def test_pass_properties(name):
    V, C = MESHES[name]
    out = ofl.flip_delaunay(V, C)
    info = _check_pass(V, C, out)
    print(f"{name}: T {len(C)} illegal {out['n_illegal']} proposed {out['n_proposed']} 2-3 {out['n_23']} 3-2 {out['n_32']}; {info}")
    if out["n_proposed"] > 3:
        for cap in (0, 1, 3):
            _check_pass(V, C, ofl.flip_delaunay(V, C, max_flips=cap), max_flips=cap)
    again = ofl.flip_delaunay(V, C)
    for k in ("cells", "sources"):
        assert np.array_equal(out[k], again[k]), k


def test_refined_meshes_propose_flips():
    for name in ("delaunay+refined", "bottle+refined", "delaunay+jittered"):
        assert ofl.flip_delaunay(*MESHES[name])["n_proposed"] > 0, name


@pytest.mark.parametrize("name", ["delaunay+refined", "bottle+refined", "sliver+refined"])
def test_both_flip_kinds_apply(name):
    """the 2-3 and the 3-2 path both run (the 3-2 path: the t2 lookup, the ordering of three slots, the removal and the compaction), and
    a 3-2 flip's output is what the definition writes: two cells on its three old slots' lowest two, the highest one gone"""
    V, C = MESHES[name]
    cells, n23, n32, checked = C, 0, 0, 0
    for _ in range(80):
        out = ofl.flip_delaunay(V, cells)
        n23, n32 = n23 + out["n_23"], n32 + out["n_32"]
        pr, T = out["prop"], len(cells)
        removed = np.zeros(T, bool)
        for i in out["kept"]:
            if pr["kind"][i] == 3:
                removed[max(pr["t0"][i], pr["t1"][i], pr["t2"][i])] = True
        rank = np.cumsum(~removed) - 1  # new slot of each kept old slot
        for i in out["kept"]:
            if pr["kind"][i] != 3:
                continue
            s = np.sort([pr["t0"][i], pr["t1"][i], pr["t2"][i]])
            for j in (0, 1):
                assert np.array_equal(out["cells"][rank[s[j]]], pr["new"][i, j])
                assert out["sources"][rank[s[j]]].tolist() == s.tolist()
            assert set(cells[s].reshape(-1).tolist()) == set(out["cells"][rank[s[:2]]].reshape(-1).tolist())  # the same five vertices
            checked += 1
        if out["n_proposed"] == 0:
            break
        cells = out["cells"]
    print(f"{name}: {n23} 2-3 flips, {n32} 3-2 flips to the fixed point")
    assert n23 > 0 and n32 > 0 and checked == n32


def test_delaunay_mesh_comes_back_unchanged():
    V, C = MESHES["delaunay"]
    out = ofl.flip_delaunay(V, C)
    assert out["n_illegal"] == out["n_proposed"] == 0
    assert np.array_equal(out["cells"], C)
    assert np.array_equal(out["sources"][:, 0], np.arange(len(C))) and (out["sources"][:, 1:] == -1).all()


def test_three_owners_raise():
    V, C = syn.delaunay_mesh(100, seed=0)
    bad = np.concatenate([C, C[:1]], 0)
    with pytest.raises(ValueError, match="more than two owners"):
        ofl.flip_delaunay(V, bad)


@pytest.mark.parametrize("name", [n for n in MESHES if "+" in n])
def test_fixed_point(name):
    V, C = MESHES[name]
    cells = C
    counts = []
    for _ in range(80):
        out = ofl.flip_delaunay(V, cells)
        counts.append((out["n_illegal"], out["n_proposed"], out["n_23"], out["n_32"]))
        if out["n_proposed"] == 0:
            break
        cells = out["cells"]
    assert counts[-1][1] == 0, "the passes did not reach a fixed point"
    ofl.check_flipped(V, C, cells)  # all the passes together, against the original mesh
    pr = ofl.proposals(V, cells)
    assert not (pr["kind"] > 0).any()  # every face still certified illegal is unflippable by the definition
    if counts[0][0]:
        assert counts[-1][0] < counts[0][0]
    print(f"{name}: {len(counts)} passes; illegal {counts[0][0]} -> {counts[-1][0]} (stuck); per pass {counts}")


# ---- the model's host side --------------------------------------------------------------------------------------------------------
def _model(V, C, **kw):
    from tetranerf.nerfstudio import model as M

    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), **kw))
    m.load_state_dict({"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C),
                       "tetrahedra_field": torch.randn(64, len(V), generator=torch.Generator().manual_seed(0))}, strict=False)
    return m, M


def test_off_by_default():
    V, C = syn.delaunay_mesh(100, seed=0)
    m, M = _model(V, C)
    assert m.config.delaunay_flip_every == 0
    assert m.get_training_callbacks(M.TrainingCallbackAttributes()) == []


def test_callbacks():
    V, C = syn.delaunay_mesh(100, seed=0)
    m, M = _model(V, C, delaunay_flip_every=5)
    calls = []
    m.flip_delaunay = lambda optimizers=None: calls.append("flip")
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes())
    assert len(cbs) == 1 and M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION in cbs[0].where_to_run
    for step in range(0, 16):
        cbs[0].run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
    assert calls == ["flip"] * 3  # steps 5, 10, 15
    m, M = _model(V, C, delaunay_flip_every=10, coarsen_every=10, refine_every=10, use_occupancy_field=True)
    calls = []
    m.coarsen = lambda optimizers=None: calls.append("coarsen")
    m.refine = lambda optimizers=None: calls.append("refine")
    m.flip_delaunay = lambda optimizers=None: calls.append("flip")
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes())
    assert len(cbs) == 4
    for step in (995, 1000, 1001, 1010):
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
    assert calls == ["coarsen", "refine", "flip", "coarsen", "refine", "flip"]


def _oracle_backends(monkeypatch):
    """the GPU passes the model drives, replaced by their numpy oracles on CPU tensors"""
    from tetranerf.b200 import coarsen as cv
    from tetranerf.b200 import flip as fl
    from tetranerf.b200 import refine as rf

    def refine_edges(xyz, cells, cand, min_length=0.0, room=None):
        o = ore.refine_edges(xyz.numpy(), cells.numpy(), cand.numpy(), min_length, room)
        return {k: torch.from_numpy(v) if isinstance(v, np.ndarray) else v for k, v in o.items()}

    def coarsen_vertices(xyz, cells, empty, max_removed=None):
        o = oco.coarsen_vertices(xyz.numpy(), cells.numpy(), empty.numpy(), max_removed)
        return {k: torch.from_numpy(v) if isinstance(v, np.ndarray) else v for k, v in o.items()}

    def flip_delaunay(xyz, cells, max_flips=None):
        o = ofl.flip_delaunay(xyz.numpy(), cells.numpy(), max_flips)
        return {k: (torch.from_numpy(o[k]) if isinstance(o[k], np.ndarray) else o[k])
                for k in ("cells", "sources", "n_illegal", "n_proposed", "n_23", "n_32")}

    monkeypatch.setattr(rf, "refine_edges", refine_edges)
    monkeypatch.setattr(cv, "coarsen_vertices", coarsen_vertices)
    monkeypatch.setattr(fl, "flip_delaunay", flip_delaunay)


def test_refine_and_coarsen_end_with_a_flip(monkeypatch):
    _oracle_backends(monkeypatch)
    V, C = syn.delaunay_mesh(300, seed=3)
    m, _ = _model(V, C, delaunay_flip_every=100, refine_every=100, refine_fraction=0.3, refine_passes=2)
    m._grad_acc, m._grad_cnt = torch.rand(len(V)), torch.ones(len(V), dtype=torch.int32)
    res = m.refine()
    assert res["vertices_after"] > res["vertices_before"] and "flip" in res
    fl = res["flip"]
    assert fl["passes"][0]["illegal"] > 0 and fl["passes"][-1]["proposed"] == 0
    assert ofl.illegal_faces(m.tetrahedra_vertices.numpy(), m.tetrahedra_cells.numpy())["proposed"] == 0
    assert m.config.num_tetrahedra_cells == len(m.tetrahedra_cells) == fl["tetrahedra_after"]
    # without the option refine() leaves the mesh as it bisected it
    m2, _ = _model(V, C, refine_every=100, refine_fraction=0.3, refine_passes=2)
    m2._grad_acc, m2._grad_cnt = torch.rand(len(V)), torch.ones(len(V), dtype=torch.int32)
    assert "flip" not in m2.refine()
    # coarsen()
    m3, _ = _model(V, C, delaunay_flip_every=100, coarsen_every=100, use_occupancy_field=True, occupancy_warmup_steps=0)
    m3.tetrahedra_occupancy.fill_(1e-6)
    m3._occ_ready, m3._occ_step = True, 1
    res = m3.coarsen()
    assert res["vertices_after"] < res["vertices_before"] and "flip" in res
    assert ofl.illegal_faces(m3.tetrahedra_vertices.numpy(), m3.tetrahedra_cells.numpy())["proposed"] == 0
    assert len(m3.tetrahedra_occupancy) == len(m3.tetrahedra_cells)


def test_flip_delaunay_installs_and_migrates(monkeypatch):
    _oracle_backends(monkeypatch)
    V, C = _refined(*syn.delaunay_mesh(300, seed=3), passes=2)
    m, M = _model(V, C, delaunay_flip_every=1, use_occupancy_field=True, optimize_vertices=True)
    occ = torch.rand(len(C), generator=torch.Generator().manual_seed(1))
    m.tetrahedra_occupancy.copy_(occ)
    opts = {k: torch.optim.RAdam(v, lr=1e-3) for k, v in m.get_param_groups().items()}
    for _ in range(2):
        for p in m.parameters():
            p.grad = torch.randn_like(p)
        for o in opts.values():
            o.step()
    m._grad_acc, m._grad_cnt = torch.rand(len(V)), torch.randint(0, 5, (len(V),), dtype=torch.int32)
    field, xyz = m.tetrahedra_field, m.tetrahedra_vertices
    snap = {"field": field.detach().clone(), "xyz": xyz.detach().clone(), "acc": m._grad_acc.clone(), "cnt": m._grad_cnt.clone()}
    st0 = {(g, i): {k: v.clone() for k, v in o.state[p].items()} for g, o in opts.items() for i, p in enumerate(o.param_groups[0]["params"])}
    # the expected occupancy: pass by pass, the maximum over the sources
    want_occ, cells = occ.clone(), C
    while True:
        o = ofl.flip_delaunay(snap["xyz"].numpy(), cells)
        if o["n_proposed"] == 0:
            break
        s = torch.from_numpy(o["sources"]).long()
        vals = torch.where(s >= 0, want_occ[s.clamp_min(0)], torch.full(s.shape, -1.0))
        want_occ, cells = vals.amax(1), o["cells"]
    res = m.flip_delaunay(opts)
    assert res["tetrahedra_before"] == len(C) and res["passes"][0]["proposed"] > 0 and res["passes"][-1]["proposed"] == 0
    assert res["illegal_left"] == res["passes"][-1]["illegal"]
    assert torch.equal(m.tetrahedra_cells, torch.from_numpy(cells)) and m.config.num_tetrahedra_cells == len(cells)
    assert torch.equal(m.tetrahedra_occupancy, want_occ)
    assert m.tetrahedra_field is field and m.tetrahedra_vertices is xyz
    assert torch.equal(field, snap["field"]) and torch.equal(xyz, snap["xyz"])
    assert torch.equal(m._grad_acc, snap["acc"]) and torch.equal(m._grad_cnt, snap["cnt"])
    for g, o in opts.items():
        for i, p in enumerate(o.param_groups[0]["params"]):
            for k, v in o.state[p].items():
                assert torch.equal(v, st0[g, i][k]), (g, i, k)
    # a mesh with nothing to flip installs nothing
    cells_before = m.tetrahedra_cells
    res = m.flip_delaunay(opts)
    assert len(res["passes"]) == 1 and res["passes"][0]["proposed"] == 0 and m.tetrahedra_cells is cells_before


def test_migrate_cells_max():
    from tetranerf.b200.flip import migrate_cells_max

    t = torch.tensor([0.1, 0.5, 0.2, 0.9])
    src = torch.tensor([[0, -1, -1], [1, 2, -1], [0, 3, -1], [1, 2, 3], [2, -1, -1]], dtype=torch.int32)
    assert torch.equal(migrate_cells_max(t, src), torch.tensor([0.1, 0.5, 0.9, 0.9, 0.2]))
    t2 = torch.stack([t, -t], 1)
    assert torch.equal(migrate_cells_max(t2, src)[:, 1], torch.tensor([-0.1, -0.2, -0.1, -0.2, -0.2]))


def test_flipped_checkpoint_loads_into_the_original_config(monkeypatch):
    _oracle_backends(monkeypatch)
    V, C = _refined(*syn.delaunay_mesh(300, seed=3), passes=2)
    m, M = _model(V, C, delaunay_flip_every=1, use_occupancy_field=True)
    m.flip_delaunay()
    assert len(m.tetrahedra_cells) != len(C)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m2, _ = _model(V, C, delaunay_flip_every=1, use_occupancy_field=True)
    m2.load_state_dict(sd, strict=True)
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert m2.config.num_tetrahedra_cells == len(m.tetrahedra_cells)
