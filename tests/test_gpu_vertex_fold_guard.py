"""GPU: the fold guard of a vertex step (TetrahedraTracer.guard_vertex_step, tn_fold_guard.cu; DESIGN §4.17).
  * kernel against oracle/fold_guard.py, positions and counts bitwise, on the small Delaunay mesh, the bottle (not walkable at load, so no
    hull edge is guarded) and the sliver mesh, for independent and smooth steps of 0.01 .. 2 median edge lengths, a single vertex pushed
    through its opposite face and max_halvings = 0;
  * after the guard a refit reports no face beyond those uncertified at P0 (none on the clean meshes), the walk stays as it was, and
    traces equal a fresh load;
  * on the 2.02 M-tetrahedra mesh, noise that folds thousands of faces unguarded folds none guarded, and repeated runs are bitwise equal;
  * the error codes;
  * the model option: an aggressive vertex learning rate folds the unguarded model; with vertex_fold_guard the same run never warns, keeps
    the walk on and lowers the loss;
  * the vertex recovery scenario of test_gpu_vertex_grads without freezing vertices by hand, at a learning rate that folds unguarded."""
import warnings

import numpy as np
import pytest
import torch

from oracle import fold_guard as fg
from oracle import oracle as orc
from oracle import vertex_grads as vg
from tetranerf.b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _bottle():
    from test_bottle import GOLD

    z = np.load(GOLD)
    return np.ascontiguousarray(z["vertices"], dtype=np.float32), np.ascontiguousarray(z["cells"], dtype=np.int32)


def _sliver():
    from test_gpu_slivers import sliver_mesh

    V, C = sliver_mesh()
    return V.astype(np.float32), C.astype(np.int32)


MESHES = {"small": lambda: syn.delaunay_mesh(3000, seed=0), "bottle": _bottle, "sliver": _sliver}
STEPS = [(a, s) for a in (0.01, 0.15, 0.6, 2.0) for s in (False, True)]
_cache = {}


def _mesh(name):
    if name not in _cache:
        V, C = MESHES[name]()
        tri, tt = vg.face_tables(C)
        edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
        _cache[name] = (V, C, tri, tt, edge)
    return _cache[name]


def _step(V, edge, amount, smooth, seed=3):
    if smooth:
        X = V.astype(np.float64)
        lo, hi = X.min(0), X.max(0)
        U = (X - lo) / np.maximum(hi - lo, 1e-30)
        d = np.stack([np.sin(6.0 * U[:, 1] + 1.0), np.sin(6.0 * U[:, 2] + 2.0), np.sin(6.0 * U[:, 0] + 3.0)], -1)
    else:
        d = np.random.default_rng(seed).standard_normal(V.shape)
    return (V + amount * edge * d).astype(np.float32)


def _single_fold(V, C, tri, tt):
    """one interior vertex pushed through its opposite face, as test_model_optimize_vertices_steps does"""
    hull = set(np.unique(tri[tt[:, 1] < 0]).tolist())
    v = next(i for i in range(len(V)) if i not in hull)
    t = int(np.nonzero((C == v).any(1))[0][0])
    others = [u for u in C[t] if u != v]
    P = V.copy()
    P[v] = P[v] + 2.0 * (P[others].mean(0) - P[v])
    return P


def _tracer(V, C):
    from tetranerf import cpp

    tr = cpp.TetrahedraTracer(DEV)
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV)
    tr.load_tetrahedra(xyz, cells)
    return tr, xyz, cells


def _run_case(name, P1, K, trace_check=False):
    from tetranerf import cpp

    V, C, tri, tt, edge = _mesh(name)
    tr, xyz, cells = _tracer(V, C)
    walk0, _ = tr.trace_stats()
    old = xyz.clone()
    new = torch.from_numpy(P1).to(DEV)
    limited, frozen, rounds = tr.guard_vertex_step(old, new, K)
    ref = fg.guard(V, P1, C, K, tri, tt)
    got = new.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), ref["xyz"].view(np.uint32)), f"{int((got != ref['xyz']).any(1).sum())} rows differ"
    assert (limited, frozen, rounds) == (ref["limited"], ref["frozen"], ref["rounds"])
    assert ref["hull_guarded"] == walk0  # (the tracer was loaded at P0: walkable there iff walkable at load)
    folded, walkable = tr.update_vertices(new)
    assert walkable == walk0
    # the faces uncertified afterwards are among those uncertified at P0 (all of them on a clean mesh); an exempt one may unfold
    after = vg.fold_count(got, C, tri, tt, return_faces=True)
    at_p0 = vg.fold_count(V, C, tri, tt, return_faces=True)
    assert folded == len(after) and len(at_p0) == ref["folded_p0"]
    assert set(map(tuple, after.tolist())) <= set(map(tuple, at_p0.tolist()))
    if trace_check:
        fresh = cpp.TetrahedraTracer(DEV)
        fresh.load_tetrahedra(new.clone(), cells)
        o, d = (torch.from_numpy(x).to(DEV) for x in syn.camera_rays(2000, seed=3))
        if name == "bottle":
            c, r = V.mean(0), float(np.linalg.norm(V - V.mean(0), axis=1).max())
            o = (torch.from_numpy(c).to(DEV) + (o - 0.5) * 2.0 * r).contiguous()
        a, b = tr.trace_rays(o, d, 256), fresh.trace_rays(o, d, 256)
        for k in a:
            assert torch.equal(a[k], b[k]), k
        tr.synchronize()
    return (limited, frozen, rounds), ref


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("amount,smooth", STEPS, ids=[f"{a}-{'smooth' if s else 'independent'}" for a, s in STEPS])
def test_kernel_equals_oracle(name, amount, smooth):
    V, C, tri, tt, edge = _mesh(name)
    P1 = _step(V, edge, amount, smooth)
    unguarded = vg.fold_count(P1, C, tri, tt)
    counts, ref = _run_case(name, P1, 8, trace_check=amount in (0.15, 2.0))
    print(f"  {name} {amount} x edge {'smooth' if smooth else 'independent'}: folded at P0 {ref['folded_p0']}, unguarded {unguarded}, "
          f"limited / frozen / rounds {counts}")


@pytest.mark.parametrize("name", list(MESHES))
def test_single_vertex_fold_and_no_halvings(name):
    V, C, tri, tt, edge = _mesh(name)
    P1 = _single_fold(V, C, tri, tt)
    counts, _ = _run_case(name, P1, 8, trace_check=True)
    assert counts[0] + counts[1] >= 1
    counts0, _ = _run_case(name, _step(V, edge, 0.6, False), 0)
    assert counts0[0] == 0 and counts0[1] > 0
    print(f"  {name}: single vertex {counts}, max_halvings 0 at 0.6 x edge {counts0}")


def test_no_fold_leaves_the_step_alone():
    V, C, tri, tt, edge = _mesh("small")
    A = np.array([[1.01, 0.01, 0.0], [0.0, 0.99, 0.01], [0.01, 0.0, 1.0]])
    P1 = (V.astype(np.float64) @ A.T + 0.05).astype(np.float32)
    tr, xyz, _ = _tracer(V, C)
    new = torch.from_numpy(P1).to(DEV)
    v0 = new._version
    assert tr.guard_vertex_step(xyz, new, 8) == (0, 0, 1)
    assert torch.equal(new.cpu(), torch.from_numpy(P1)) and new._version == v0


def test_at_size_and_repeatable():
    """the 300k-point Delaunay mesh (2.02 M tetrahedra): independent noise of 0.15 edge lengths folds thousands of faces; guarded, none,
    the walk stays on, and two runs give the same bits"""
    V, C = syn.delaunay_mesh(300_000, seed=0)
    edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
    P1 = _step(V, edge, 0.15, False)
    tr, xyz, _ = _tracer(V, C)
    assert tr.trace_stats()[0]
    unguarded, walk_u = tr.update_vertices(torch.from_numpy(P1).to(DEV))
    tr.update_vertices(xyz)
    outs = []
    for _ in range(2):
        new = torch.from_numpy(P1).to(DEV)
        counts = tr.guard_vertex_step(xyz, new, 8)
        outs.append((new, counts))
    assert torch.equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1]
    folded, walkable = tr.update_vertices(outs[0][0])
    print(f"  {len(C)} tetrahedra, 0.15 x edge: unguarded {unguarded} folded (walk {walk_u}); guarded {folded} folded, walk {walkable}, "
          f"limited / frozen / rounds {outs[0][1]}")
    assert unguarded > 1000 and not walk_u
    assert folded == 0 and walkable


def test_errors():
    """TN_ERR_STATE without a mesh; TN_ERR_ARG for another V, max_halvings > 23 and a non-finite coordinate in either array, which leaves
    the proposed positions unchanged"""
    import ctypes

    from tetranerf import cpp
    from tetranerf.utils.extension.tetranerf_cpp_extension import _lib

    V, C, tri, tt, edge = _mesh("small")
    stream = torch.cuda.current_stream(DEV).cuda_stream
    counts = (ctypes.c_uint32 * 3)()

    def rc(tr, old, new, n, K):
        return _lib.tn_guard_vertex_step(tr.handle, old.data_ptr(), new.data_ptr(), n, K, ctypes.byref(counts), stream)

    x = torch.from_numpy(V).to(DEV)
    assert rc(cpp.TetrahedraTracer(DEV), x, x.clone(), len(V), 8) == 4  # TN_ERR_STATE
    tr, xyz, _ = _tracer(V, C)
    y = xyz + 1e-3
    assert rc(tr, xyz, y, len(V) - 1, 8) == 1
    assert rc(tr, xyz, y, len(V), 24) == 1
    assert rc(tr, xyz, y, len(V), 23) == 0
    with pytest.raises(RuntimeError, match="vertices"):
        tr.guard_vertex_step(xyz[:-1].contiguous(), xyz[:-1].contiguous().add(1e-3))
    with pytest.raises(RuntimeError, match="23"):
        tr.guard_vertex_step(xyz, xyz + 1e-3, 24)
    for which in ("new", "old"):
        old, new = xyz.clone(), torch.from_numpy(_step(V, edge, 0.6, False)).to(DEV)
        (new if which == "new" else old)[5, 2] = float("inf") if which == "new" else float("nan")
        keep = new.clone()
        with pytest.raises(RuntimeError, match="finite"):
            tr.guard_vertex_step(old, new)
        assert torch.equal(new.isnan(), keep.isnan()) and torch.equal(new.nan_to_num(), keep.nan_to_num()), which


def _model_run(small_mesh, guard, lr_scale, steps):
    from tetranerf.nerfstudio import model as M
    from test_gpu_model import build_model

    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    m, _ = build_model(V, C, field, num_samples=48, num_fine_samples=33, use_biased_sampler=True, optimize_vertices=True,
                       vertex_fold_guard=guard)
    m.train()
    edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
    groups = m.get_param_groups()
    opt = torch.optim.Adam([{"params": groups["fields"], "lr": 5e-3}, {"params": groups["vertices"], "lr": lr_scale * edge}])
    o, d = (torch.from_numpy(x).to(DEV) for x in syn.camera_rays(2048, seed=21))
    target = torch.rand((2048, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    tri, tt = vg.face_tables(C)
    losses, folds, walks = [], [], []
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        for _ in range(steps):
            opt.zero_grad()
            out = m(M.RayBundle(origins=o, directions=d))
            loss = m.get_loss_dict(out, {"image": target})["rgb_loss"]
            loss.backward()
            opt.step()
            tr = m.get_tetrahedra_tracer()  # the refit (and with the option, the guard) of this step
            losses.append(loss.item())
            folds.append(vg.fold_count(m.tetrahedra_vertices.detach().cpu().numpy(), C, tri, tt))
            walks.append(tr.trace_stats()[0])
    fold_warnings = [w for w in caught if "folded" in str(w.message)]
    return losses, folds, walks, fold_warnings, m


def test_model_vertex_fold_guard(small_mesh):
    steps = 12
    losses_u, folds_u, walks_u, warn_u, _ = _model_run(small_mesh, False, 0.3, steps)
    print(f"  unguarded: folded faces per step {folds_u}, loss {losses_u[0]:.4f} -> {losses_u[-1]:.4f}")
    assert max(folds_u) > 0 and len(warn_u) == 1 and not all(walks_u)  # the scenario is real: this rate folds the mesh
    losses, folds, walks, warn, m = _model_run(small_mesh, True, 0.3, steps)
    print(f"  guarded: folded faces per step {folds}, loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert not warn and max(folds) == 0 and all(walks)
    assert min(losses[-3:]) < losses[0]
    # the tracer holds exactly the parameter's positions, as after a fresh load
    from tetranerf import cpp

    tr = m.get_tetrahedra_tracer()
    fresh = cpp.TetrahedraTracer(DEV)
    fresh.load_tetrahedra(m.tetrahedra_vertices.detach().clone(), m.tetrahedra_cells)
    o, d = (torch.from_numpy(x).to(DEV) for x in syn.camera_rays(1000, seed=4))
    a, b = tr.trace_rays(o, d, 64), fresh.trace_rays(o, d, 64)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # a checkpoint resume starts from the loaded positions, unguarded: a folding state loads as it is
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    V, C = small_mesh
    sd["tetrahedra_vertices"] = torch.from_numpy(_single_fold(V, C, *vg.face_tables(C))).to(DEV)
    m.load_state_dict(sd)
    with pytest.warns(UserWarning, match="folded"):
        m.get_tetrahedra_tracer()
    assert torch.equal(m.tetrahedra_vertices.detach(), sd["tetrahedra_vertices"])


def _recovery_setup(small_mesh):
    from tetranerf.b200.render import PARAM_ORDER, FusedTrainRender
    from test_gpu_ray_grads import _settings
    from test_gpu_train import _setup

    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    st, _ = _settings("tetra_nerf")
    tr, fr, params = _setup(V, C, field, params)
    f = torch.from_numpy(field).to(DEV)
    ps = [params[n].to(DEV) for n in PARAM_ORDER]
    n = 48
    u = torch.linspace(-0.25, 0.25, n, device=DEV)
    uu, vv = torch.meshgrid(u, u, indexing="xy")
    rays_o, rays_d = [], []
    for k in range(8):
        a = 2 * np.pi * k / 8
        cam = torch.tensor([0.5 + 1.6 * np.cos(a), 0.5 + 1.6 * np.sin(a), 0.5 + 0.3 * (-1) ** k], device=DEV, dtype=torch.float32)
        fwd = torch.tensor([0.5, 0.5, 0.5], device=DEV) - cam
        fwd = fwd / fwd.norm()
        right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0], device=DEV))
        right = right / right.norm()
        up = torch.linalg.cross(right, fwd)
        dirs = fwd + uu.reshape(-1, 1) * right + vv.reshape(-1, 1) * up
        rays_o.append(cam.expand(n * n, 3))
        rays_d.append(dirs / dirs.norm(dim=-1, keepdim=True))
    o, d = torch.cat(rays_o).contiguous(), torch.cat(rays_d).contiguous()
    with torch.no_grad():
        target = FusedTrainRender.apply(fr, st, False, o, d, None, None, f, *ps)[0].clone()
    render = lambda xyz: FusedTrainRender.apply(fr, st, False, o, d, None, None, f, *ps, xyz)[0]
    return tr, render, target


def test_vertex_recovery_with_the_guard(small_mesh):
    """test_vertex_recovery_through_the_fused_op's scenario (surface_scene, 8 cameras, only the vertices train through FusedTrainRender)
    with the guard in place of freezing vertices by hand: the start displacement (smooth, 0.1 edge lengths on the interior vertices) is
    itself a guarded step from the true positions, and every Adam step is guarded before the refit, at 5x the learning rate of that test,
    which folds the unguarded run"""
    V, C = small_mesh
    tri, tt = vg.face_tables(C)
    hull = np.unique(tri[tt[:, 1] < 0])
    edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
    X = torch.from_numpy(V).double()
    noise = 0.1 * edge * torch.stack([torch.sin(6.0 * X[:, 1] + 1.0), torch.sin(6.0 * X[:, 2] + 2.0), torch.sin(6.0 * X[:, 0] + 3.0)], -1).float()
    noise[torch.from_numpy(hull).long()] = 0
    true = torch.from_numpy(V).to(DEV)
    near = torch.from_numpy(np.abs(syn.sphere_sdf(V.astype(np.float64))) < edge).to(DEV) & (noise.abs().sum(-1).to(DEV) > 0)
    lr = 0.01 * edge
    results = {}
    for guard in (False, True):
        tr, render, target = _recovery_setup(small_mesh)
        start = true + noise.to(DEV)
        if guard:
            print(f"  start displacement guarded: limited / frozen / rounds {tr.guard_vertex_step(true, start)}")
        folded0, walk0 = tr.update_vertices(start)
        xyz = torch.nn.Parameter(start.clone())
        tr.update_vertices(xyz.detach())
        prev = xyz.detach().clone()
        opt = torch.optim.Adam([xyz], lr=lr)
        err0 = (xyz.detach() - true)[near].norm(dim=-1).mean().item()
        losses, folds = [], []
        for it in range(200):
            opt.zero_grad()
            loss = torch.nn.functional.mse_loss(render(xyz), target)
            loss.backward()
            opt.step()
            if guard:
                tr.guard_vertex_step(prev, xyz.detach())
            folded, walkable = tr.update_vertices(xyz.detach())
            prev.copy_(xyz.detach())
            losses.append(loss.item())
            folds.append(folded)
        err = (xyz.detach() - true)[near].norm(dim=-1).mean().item()
        results[guard] = (folded0, walk0, losses, folds, err0, err)
        print(f"  guard {guard}: start folded {folded0}; loss {losses[0]:.3e} -> {min(losses[-5:]):.3e} ({losses[0] / min(losses[-5:]):.1f}x); "
              f"most folded faces in a step {max(folds)}; mean position error {err0:.3e} -> {err:.3e} ({err0 / err:.2f}x)")
    assert results[False][0] > 0 or max(results[False][3]) > 0  # unguarded, the start or the steps fold
    folded0, walk0, losses, folds, err0, err = results[True]
    assert folded0 == 0 and walk0 and max(folds) == 0
    # measured on an H100: the loss falls about 130x and the error 1.41x (1.01e-2 -> 7.2e-3); unguarded, the start folds 234 faces and
    # the steps up to 2036, and the error grows (0.60x)
    assert losses[0] / min(losses[-5:]) > 50.0
    assert err0 / err > 1.2
