"""CPU: the adjacency walk of trace_rays (csrc/tn_walk.cu) restated in numpy (oracle/walk.py), against the oracle's all-hits trace.

  * on clean meshes (the small Delaunay mesh, the cube, the sliver mesh of test_gpu_slivers.py) the restatement equals
    OracleMesh.trace_rays on every ray: the walk's chain from the hull entry is every face the line crosses;
  * on folded meshes with an unchanged (convex) hull -- one vertex moved through the opposite face of a tetrahedron of its star, a dozen
    such folds far apart, a smooth displacement that folds a few faces, the sliver mesh after two bisection passes -- the line also
    crosses tetrahedra off that chain (a region covered more than once), and the restatement counts the rays on which the walk path
    would differ from the all-hits gather.  That is why a load runs the fold test and takes the walk only on an unfolded mesh
    (DESIGN §4.9); tests/test_gpu_folded_meshes.py checks the GPU against the same meshes;
  * a ray with exactly one hull hit starts inside the mesh, and walked anyway it ends on the exact stage (DESIGN §2, mutation (d)).
"""
import numpy as np
import pytest

from oracle import intervals
from oracle import oracle as orc
from oracle import refine as orf
from oracle import vertex_grads as vg
from oracle import walk as W
from tetranerf.b200 import synthetic as syn
from test_gpu_slivers import sliver_mesh

M = 256
N_RAYS = 4096  # trace_rays picks the quad walk for a batch of this size by default


# ---- folded meshes: the hull keeps its vertices, so a fresh load finds it convex --------------------------------------------------------
def signed_volumes(X, C):
    X = np.asarray(X, np.float64)
    a, b, c, d = (X[C[:, k]] for k in range(4))
    return np.einsum("ij,ij->i", np.cross(b - a, c - a), d - a)


def hull_vertices(C):
    tri, tt = vg.face_tables(C)
    return np.unique(tri[tt[:, 1] < 0])


def fold_vertex(V, C, P, v, t, depth):
    """moves vertex v (in P) through the face of tetrahedron t opposite to it, to `depth` times its distance to that face beyond it"""
    A, B, Cc = (V[u].astype(np.float64) for u in C[t] if u != v)
    n = np.cross(B - A, Cc - A)
    n /= np.linalg.norm(n)
    h = float(np.dot(V[v] - A, n))
    P[v] = (V[v] - (1.0 + depth) * h * n).astype(np.float32)


def _interior_star_vertex(V, C, hull, rng, away_from=()):
    """an interior vertex none of whose neighbours is a hull vertex, at least 0.15 from every point of `away_from`"""
    inner = np.setdiff1d(np.arange(len(V)), hull)
    for v in rng.permutation(inner):
        star = C[(C == v).any(1)]
        if np.isin(star, hull).any():
            continue
        if len(away_from) and np.linalg.norm(np.asarray(away_from) - V[v], axis=1).min() < 0.15:
            continue
        return int(v)
    raise AssertionError("no interior vertex left")


def one_fold(V, C, depth, seed=0):
    rng = np.random.default_rng(seed)
    v = _interior_star_vertex(V, C, hull_vertices(C), rng)
    star = np.nonzero((C == v).any(1))[0]
    P = V.copy()
    fold_vertex(V, C, P, v, int(rng.choice(star)), depth)
    return P, [v]


def scattered_folds(V, C, n=12, depth=0.3, seed=1):
    rng = np.random.default_rng(seed)
    hull = hull_vertices(C)
    P, moved = V.copy(), []
    for _ in range(n):
        v = _interior_star_vertex(V, C, hull, rng, V[moved])
        fold_vertex(V, C, P, v, int(rng.choice(np.nonzero((C == v).any(1))[0])), depth)
        moved.append(v)
    return P, moved


def smooth_fold(V, C, amplitude=0.03):
    """test_vertex_recovery_through_the_fused_op's smooth displacement of the interior vertices at 0.03 edge lengths, without its freezing:
    it folds a few of the mesh's slivers (32 of 39k faces)"""
    tri, tt = vg.face_tables(C)
    edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
    X = V.astype(np.float64)
    noise = amplitude * edge * np.stack([np.sin(6.0 * X[:, 1] + 1.0), np.sin(6.0 * X[:, 2] + 2.0), np.sin(6.0 * X[:, 0] + 3.0)], -1)
    noise[np.unique(C[tt[tt[:, 1] < 0, 0]])] = 0  # the tetrahedra on the hull keep their shape: the hull stays certified convex
    P = (X + noise).astype(np.float32)
    moved = np.unique(vg.fold_count(P, C, tri, tt, return_faces=True))
    return P, moved


def refined_slivers(passes=2, frac=0.3, seed=0):
    """the sliver mesh after `passes` bisection passes over random masks, positions migrated as the model does (fp32 midpoints)"""
    V, C = sliver_mesh(300)
    rng = np.random.default_rng(seed)
    for _ in range(passes):
        out = orf.refine_edges(V, C, rng.random(len(C)) < frac)
        V, C = orf.migrate_vertices(V, out["parent_edge"], 0), out["cells"]
    return V, C


FOLDED = ["fold-0.05", "fold-0.3", "fold-1.0", "scattered", "smooth", "refined-slivers"]


def folded_mesh(name, small):
    """-> (V, C, P, moved vertices): the mesh, its folded positions P and the vertices that were moved (refined: none)"""
    V, C = small
    if name.startswith("fold-"):
        return (V, C) + one_fold(V, C, float(name[5:]))
    if name == "scattered":
        return (V, C) + scattered_folds(V, C)
    if name == "smooth":
        return (V, C) + smooth_fold(V, C)
    V1, C1 = refined_slivers()
    return V1, C1, V1, []


def aimed_rays(P, C, cells, n, seed):
    """rays from 2 units away towards uniform random points inside the given tetrahedra (at positions P)"""
    rng = np.random.default_rng(seed)
    t = cells[rng.integers(0, len(cells), n)]
    tgt = np.einsum("nk,nkd->nd", rng.dirichlet(np.ones(4), n), P[C[t]].astype(np.float64))
    u = rng.standard_normal((n, 3))
    o = tgt + 2.0 * u / np.linalg.norm(u, axis=1, keepdims=True)
    d = tgt - o
    return o.astype(np.float32), (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def folded_case(name, small):
    """(V, C, P, o, d, inverted tetrahedra, tetrahedra near the folds, moved vertices) with N_RAYS rays: 3/4 aimed into the inverted tetrahedra (or the
    star of the folded faces), 1/4 camera rays"""
    V, C, P, moved = folded_mesh(name, small)
    inv = np.nonzero(np.sign(signed_volumes(P, C)) != np.sign(signed_volumes(V, C)))[0]
    faces = vg.fold_count(P, C, return_faces=True)
    near_v = np.unique(np.concatenate([np.asarray(moved, np.int64).reshape(-1), faces.reshape(-1)]))
    near = np.nonzero(np.isin(C, near_v).any(1))[0]
    target = inv if len(inv) else near
    na = 3 * N_RAYS // 4
    if len(target):
        oa, da = aimed_rays(P, C, target, na, seed=5)
    else:
        oa, da = syn.sphere_rays(na, seed=5)
    oc, dc = syn.camera_rays(N_RAYS - na, seed=6)
    return V, C, P, np.concatenate([oa, oc]), np.concatenate([da, dc]), inv, near, moved


def multiply_covered(P, C, near, o, d):
    """rays whose float64 intervals in the tetrahedra `near` overlap beyond endpoint contact (a region covered more than once)"""
    out = np.zeros(len(o), bool)
    if len(near) == 0:
        return out
    for r in range(len(o)):
        _, t0, t1 = intervals.tet_intervals(P, C[near], o[r], d[r])
        if len(t0) > 1:
            reach = np.maximum.accumulate(t1)[:-1]
            out[r] = bool((t0[1:] < reach - 1e-9 * np.maximum(1.0, np.abs(reach))).any())
    return out


# ---- clean meshes: the restatement is the all-hits trace ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small", "cube", "slivers"])
def test_walk_equals_oracle_on_clean_meshes(small_mesh, cube_mesh, name):
    V, C = {"small": small_mesh, "cube": cube_mesh, "slivers": sliver_mesh()}[name]
    assert vg.fold_count(V, C) == 0
    oc, dc = syn.camera_rays(N_RAYS // 2, seed=3)
    os_, ds = syn.sphere_rays(N_RAYS // 2, seed=4)
    o, d = np.concatenate([oc, os_]), np.concatenate([dc, ds])
    mesh = orc.OracleMesh(V, C)
    w = W.walk_trace(V, C, o, d, M, mesh=mesh)
    ref = mesh.trace_rays(o, d, M)
    routes = np.bincount(w["route"], minlength=4)
    print(f"{name}: routes {dict(zip(W.ROUTES, routes.tolist()))}")
    if name == "slivers":  # most rays cross several short slivers in a row: the sort + pairing of the walk's keys
        assert routes[W.KEYS] > N_RAYS // 2 and routes[W.GENERIC] > 50
    else:
        assert routes[W.GENERIC] > N_RAYS // 2
    bad = W.differing_rays(w, ref)
    assert len(bad) == 0, f"the walk restatement differs from the oracle on rays {bad[:10]}"


# ---- folded meshes: the guards, and the finding -----------------------------------------------------------------------------------------
EXPECTED_FOLDS = {"fold-0.05": (1, 60), "fold-0.3": (1, 60), "fold-1.0": (1, 60), "scattered": (12, 600), "smooth": (10, 80),
                  "refined-slivers": (0, None)}


# measured: 325, 539, 1073, 408 and 8 rays of 4096
MIN_DIFFERING = {"fold-0.05": 150, "fold-0.3": 250, "fold-1.0": 500, "scattered": 200, "smooth": 4}


@pytest.mark.parametrize("name", FOLDED)
def test_walk_on_folded_meshes(small_mesh, name):
    V, C, P, o, d, inv, near, moved = folded_case(name, small_mesh)
    tri, tt = vg.face_tables(C)
    folded = vg.fold_count(P, C, tri, tt)
    faces = vg.fold_count(P, C, tri, tt, return_faces=True)
    hull = hull_vertices(C)
    assert np.array_equal(P[hull], V[hull])  # the hull is the clean mesh's: a fresh load finds it convex
    lo, hi = EXPECTED_FOLDS[name]
    assert folded >= lo and (hi is None or folded <= hi), folded
    if name != "refined-slivers":
        # every folded face lies in the star of a moved vertex: the folds are the constructed ones and nothing else
        star = np.unique(C[np.isin(C, moved).any(1)])
        assert np.isin(faces, star).all() and len(inv) > 0
    mesh = orc.OracleMesh(P, C)
    w = W.walk_trace(P, C, o, d, M, mesh=mesh)
    ref = mesh.trace_rays(o, d, M)
    bad = W.differing_rays(w, ref)
    cover = multiply_covered(P, C, near, o, d)
    gen = w["route"] == W.GENERIC
    routes = np.bincount(w["route"], minlength=4)
    print(f"{name}: {folded} folded faces, {len(inv)} inverted tetrahedra; {int(cover.sum())} of {len(o)} rays cross a region covered more "
          f"than once, {int((cover & gen).sum())} of them generic; routes {dict(zip(W.ROUTES, routes.tolist()))}; the walk path differs from "
          f"the all-hits gather on {len(bad)} rays ({int(gen[bad].sum())} generic)")
    if name == "refined-slivers":
        # fp32 midpoints leave a few faces of near-flat tetrahedra uncertified, but none turns over: the walk path is still exact there
        assert len(inv) == 0 and len(bad) == 0
        return
    assert cover.sum() >= 2000 and (cover & gen).sum() >= 2
    # the finding: the walk misses the crossings off its chain, on generic rays through the folds as on rays whose keys it pairs; a
    # generic ray it gets wrong always crosses a region covered more than once
    assert len(bad) >= MIN_DIFFERING[name] and np.all(cover[bad] | ~gen[bad])


# ---- DESIGN §2, mutation (d): one hull hit -------------------------------------------------------------------------------------------------
def test_one_hull_hit_means_the_origin_is_inside(small_mesh):
    """A ray with exactly one hull hit starts inside the (convex) mesh.  Walked anyway (`hullhits > 2` in place of `!= 2`), it walks
    backwards from the exit face: its first step has t_out < t_in, so it is no longer generic and writes no record, and it stops in the
    tetrahedron that holds the origin, whose other crossing lies behind the origin (no exit face), which sends it to the exact stage.  So
    the mutant traces every ray as the kernel does: it is equivalent, which is why no trace test can catch it."""
    V, C = small_mesh
    rng = np.random.default_rng(8)
    n = 1024
    inside = (0.05 + 0.9 * rng.random((n, 3))).astype(np.float32)  # origins inside the mesh, random directions
    u = rng.standard_normal((n, 3))
    tri, tt = vg.face_tables(C)
    hf = tri[tt[:, 1] < 0]
    on = V[hf[rng.integers(0, len(hf), n)]].mean(1).astype(np.float32)  # origins on hull faces (to fp32 rounding), towards the centre
    o = np.concatenate([inside, on, syn.camera_rays(n, seed=9)[0]])
    d = np.concatenate([u, 0.5 - on + 0.3 * rng.standard_normal((n, 3)), syn.camera_rays(n, seed=9)[1]])
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    mesh = orc.OracleMesh(V, C)
    ref = mesh.trace_rays(o, d, M)
    kernel = W.walk_trace(V, C, o, d, M, mesh=mesh)
    mutant = W.walk_trace(V, C, o, d, M, mesh=mesh, walk_one_hull_hit=True)
    one = kernel["hull_hits"] == 1
    print(f"hull hits per ray: {dict(zip(*np.unique(kernel['hull_hits'], return_counts=True)))}")
    assert one[:n].sum() == n and one.sum() >= n + n // 4  # every inside origin, and the origins a hull face rounds to its inner side
    # one hull hit: the origin is inside the hull or on it (float64: nowhere more than 1e-6 outside the plane of a hull face)
    X = V.astype(np.float64)
    a, b, c = X[hf[:, 0]], X[hf[:, 1]], X[hf[:, 2]]
    nrm = np.cross(b - a, c - a)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm *= np.sign(np.einsum("ij,ij->i", nrm, a - 0.5))[:, None]  # outwards: the hull holds the centre of the cube
    out = np.einsum("fk,rfk->rf", nrm, o[one].astype(np.float64)[:, None, :] - a[None])
    assert out.max() < 1e-6
    assert np.all(mutant["route"][one] == W.EXACT)
    assert np.array_equal(mutant["route"], kernel["route"])
    assert len(W.differing_rays(mutant, ref)) == 0 and len(W.differing_rays(kernel, ref)) == 0
