"""CPU: the fold guard's oracle (oracle/fold_guard.py, DESIGN §4.17) has the properties its definition promises, and the model option
is validated.
  * a step that folds nothing comes back bitwise;
  * every output row is P1, P0 + 2^-k (P1 - P0) for its reported k, or P0, and the counts agree with the exponents;
  * afterwards every face certified at P0 is certified, and on a mesh walkable at P0 every hull edge passes the convexity test;
  * one vertex pushed through its opposite face ends at the smallest exponent that certifies its faces: one halving fewer folds;
  * max_halvings = 0 leaves only P1 and P0 rows;
  * vertex_fold_guard without optimize_vertices raises."""
import numpy as np
import pytest

from oracle import fold_guard as fg
from oracle import vertex_grads as vg
from tetranerf.b200 import synthetic as syn


@pytest.fixture(scope="module")
def mesh():
    V, C = syn.delaunay_mesh(1500, seed=2)
    tri, tt = vg.face_tables(C)
    edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
    return V, C, tri, tt, edge


def _noise(V, edge, amount, seed, smooth=False):
    if smooth:
        X = V.astype(np.float64)
        d = np.stack([np.sin(6.0 * X[:, 1] + 1.0), np.sin(6.0 * X[:, 2] + 2.0), np.sin(6.0 * X[:, 0] + 3.0)], -1)
    else:
        d = np.random.default_rng(seed).standard_normal(V.shape)
    return (V + amount * edge * d).astype(np.float32)


def _certified(P, C, tri, tt, res):
    """every face certified at P0 is certified at P; with the hull guarded, every hull edge passes"""
    assert vg.fold_count(P, C, tri, tt) == res["folded_p0"]
    if res["hull_guarded"]:
        f, g, closed = fg.hull_pairs(tri, tt)
        assert closed and fg.hull_pair_ok(P, C, tri, tt, f, g).all() and fg.hull_pair_ok(P, C, tri, tt, g, f).all()


def _rows_are_defined(P0, P1, res, K):
    out, k = res["xyz"], res["k"]
    bits = lambda a: np.asarray(a, np.float32).view(np.uint32)
    moving = (bits(P0) != bits(P1)).any(1)
    assert np.array_equal(moving, k != -1)
    at1, at0 = (k == 0) | (k == -1), k == fg.FROZEN
    assert np.array_equal(bits(out[at1]), bits(P1[at1]))
    assert np.array_equal(bits(out[at0]), bits(P0[at0]))
    for j in range(1, K + 1):
        s = k == j
        assert np.array_equal(bits(out[s]), bits(fg.step_position(P0[s], P1[s], j)))
    assert res["limited"] == int(((k >= 1) & (k <= K)).sum()) and res["frozen"] == int(at0.sum())


def test_no_fold_is_bitwise(mesh):
    V, C, tri, tt, edge = mesh
    A = np.array([[1.01, 0.01, 0.0], [0.0, 0.99, 0.01], [0.01, 0.0, 1.0]])  # an affine motion: no tetrahedron turns, the hull stays convex
    P1 = (V.astype(np.float64) @ A.T + 0.05).astype(np.float32)
    assert vg.fold_count(P1, C, tri, tt) == 0
    res = fg.guard(V, P1, C, 8, tri, tt)
    assert np.array_equal(res["xyz"].view(np.uint32), P1.view(np.uint32))
    assert (res["limited"], res["frozen"], res["rounds"]) == (0, 0, 1) and res["hull_guarded"]


@pytest.mark.parametrize("amount,smooth,K", [(0.15, False, 8), (0.6, False, 8), (2.0, False, 8), (0.6, True, 8), (0.6, False, 0), (0.6, False, 2)])
def test_guarded_step_is_certified_and_well_formed(mesh, amount, smooth, K):
    V, C, tri, tt, edge = mesh
    P1 = _noise(V, edge, amount, 3, smooth)
    unguarded = vg.fold_count(P1, C, tri, tt)
    res = fg.guard(V, P1, C, K, tri, tt)
    print(f"  {amount} x edge ({'smooth' if smooth else 'independent'}), K={K}: {unguarded} faces folded unguarded; limited "
          f"{res['limited']}, frozen {res['frozen']}, rounds {res['rounds']}")
    assert unguarded > 0 and res["hull_guarded"]
    _rows_are_defined(V, P1, res, K)
    _certified(res["xyz"], C, tri, tt, res)
    if K == 0:
        assert res["limited"] == 0 and res["frozen"] > 0


def test_hull_convexity_is_kept(mesh):
    """hull vertices pulled inwards make the hull non-convex without folding an interior face: the guard holds the hull edges"""
    V, C, tri, tt, edge = mesh
    hull = np.unique(tri[tt[:, 1] < 0])
    c = V.mean(0)
    P1 = V.copy()
    P1[hull] = (V[hull] + 0.3 * (c - V[hull]) * np.random.default_rng(4).random((len(hull), 1))).astype(np.float32)
    f, g, _ = fg.hull_pairs(tri, tt)
    assert not (fg.hull_pair_ok(P1, C, tri, tt, f, g) & fg.hull_pair_ok(P1, C, tri, tt, g, f)).all()
    res = fg.guard(V, P1, C, 8, tri, tt)
    assert res["hull_guarded"] and res["limited"] + res["frozen"] > 0
    _rows_are_defined(V, P1, res, 8)
    _certified(res["xyz"], C, tri, tt, res)


def test_single_vertex_takes_the_smallest_certifying_exponent(mesh):
    V, C, tri, tt, edge = mesh
    hull = set(np.unique(tri[tt[:, 1] < 0]).tolist())
    tried = 0
    for v in (i for i in range(len(V)) if i not in hull):
        t = int(np.nonzero((C == v).any(1))[0][0])
        others = [u for u in C[t] if u != v]
        P1 = V.copy()
        P1[v] = (V[v] + 2.0 * (V[others].mean(0) - V[v])).astype(np.float32)  # through the opposite face, as far again beyond it
        assert vg.fold_count(P1, C, tri, tt) > 0
        res = fg.guard(V, P1, C, 8, tri, tt)
        k = int(res["k"][v])
        assert res["frozen"] + res["limited"] == 1 and 1 <= k <= 8, k
        P = V.copy()
        P[v] = fg.step_position(V[v], P1[v], k)
        assert np.array_equal(P, res["xyz"])
        assert vg.fold_count(P, C, tri, tt) == 0
        P[v] = P1[v] if k == 1 else fg.step_position(V[v], P1[v], k - 1)
        assert vg.fold_count(P, C, tri, tt) > 0
        assert res["rounds"] == k + 1
        tried += 1
        if tried == 5:
            break


def test_hull_pair_ok_agrees_with_the_hull_shape():
    """the restated convexity test accepts a convex hull and rejects one with a vertex pushed in"""
    V, C = syn.delaunay_mesh(400, seed=9)
    tri, tt = vg.face_tables(C)
    f, g, closed = fg.hull_pairs(tri, tt)
    assert closed and len(f) > 0
    ok = fg.hull_pair_ok(V, C, tri, tt, f, g) & fg.hull_pair_ok(V, C, tri, tt, g, f)
    assert ok.all()
    hv = int(tri[f[0], 0])
    P = V.copy()
    P[hv] = (V[hv] + 0.5 * (V.mean(0) - V[hv])).astype(np.float32)
    assert not (fg.hull_pair_ok(P, C, tri, tt, f, g) & fg.hull_pair_ok(P, C, tri, tt, g, f)).all()


def test_guard_needs_optimize_vertices():
    from tetranerf.nerfstudio.model import TetrahedraNerf, TetrahedraNerfConfig

    cfg = TetrahedraNerfConfig(num_tetrahedra_vertices=8, num_tetrahedra_cells=4, vertex_fold_guard=True)
    with pytest.raises(RuntimeError, match="vertex_fold_guard"):
        TetrahedraNerf(cfg)
    m = TetrahedraNerf(TetrahedraNerfConfig(num_tetrahedra_vertices=8, num_tetrahedra_cells=4, vertex_fold_guard=True, optimize_vertices=True))
    assert m._guard_start is None
