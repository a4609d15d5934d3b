"""GPU: Delaunay flips (DESIGN §4.19).
  * tn_flip_delaunay equals the numpy oracle (oracle/flip.py) bit for bit on the Delaunay, bottle and sliver meshes and on them after
    refinement, coarsening and a jitter, with and without the max_flips cap, pass after pass to the fixed point, and two runs are bitwise
    equal; the workspace query, TN_ERR_ARG and TN_ERR_MESH;
  * a flipped mesh that was walkable before keeps the adjacency walk and every trace implementation gives the oracle's all-hits bits;
  * same domain, same interpolant class: with every field channel affine in the position, linear interpolation reproduces it on any
    tetrahedralisation of the domain, so the fused eval render before and after flipping agrees to rounding;
  * the model: a short training run with refinement and flips every few steps keeps every loss and gradient finite, and its flips
    install as specified (fixed point, occupancy, tracer)."""
import ctypes as C
import copy

import numpy as np
import pytest
import torch

from conftest import TRACE_IMPLS, force_trace_impl
from oracle import flip as ofl
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_flip_cpu import _coarsened, _jittered, _refined, flip_meshes
from test_gpu_train import DEV

pytestmark = pytest.mark.gpu
TRACE_KEYS = ["num_visited_cells", "visited_cells", "vertex_indices", "hit_distances", "barycentric_coordinates"]
MESHES = flip_meshes()


def _gpu_pass(V, C_, cap=None):
    from tetranerf.b200.flip import flip_delaunay

    return flip_delaunay(torch.from_numpy(V).to(DEV), torch.from_numpy(np.ascontiguousarray(C_)).to(DEV), cap)


def _same(got, want):
    for k in ("n_illegal", "n_proposed", "n_23", "n_32"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert np.array_equal(got["cells"].cpu().numpy(), want["cells"]), "cells"
    assert np.array_equal(got["sources"].cpu().numpy(), want["sources"]), "sources"


@pytest.mark.parametrize("name", list(MESHES))
def test_flip_delaunay_vs_oracle(name):
    V, C0 = MESHES[name]
    for cap in (None, 1, 7):
        want = ofl.flip_delaunay(V, C0, cap)
        got, again = _gpu_pass(V, C0, cap), _gpu_pass(V, C0, cap)
        _same(got, want)
        assert torch.equal(got["cells"], again["cells"]) and torch.equal(got["sources"], again["sources"])
    # pass after pass to the fixed point, each pass against the oracle
    cells, n, n23, n32 = C0, 0, 0, 0
    for n in range(1, 81):
        got = _gpu_pass(V, cells)
        want = ofl.flip_delaunay(V, cells)
        _same(got, want)
        n23, n32 = n23 + got["n_23"], n32 + got["n_32"]
        if got["n_proposed"] == 0:
            break
        cells = want["cells"]
    assert got["n_proposed"] == 0
    if name.endswith("+refined"):  # both kinds of flip ran through the kernel
        assert n23 > 0 and n32 > 0, (n23, n32)
    ofl.check_flipped(V, C0, cells)
    print(f"{name}: T {len(C0)} -> {len(cells)}, {n} passes, illegal left {got['n_illegal']}")


def test_flip_delaunay_errors_and_workspace():
    from tetranerf.b200.flip import flip_delaunay
    from tetranerf.utils.extension import tetranerf_cpp_extension as ext

    V, C0 = syn.delaunay_mesh(200, seed=0)
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(C0).to(DEV)
    bad = cells.clone()
    bad[5, 2] = len(V)
    with pytest.raises(RuntimeError, match="vertex index"):
        flip_delaunay(xyz, bad)
    with pytest.raises(RuntimeError, match="more than two"):
        flip_delaunay(xyz, torch.cat([cells, cells[:1]]))
    with pytest.raises(RuntimeError, match="max_flips"):
        flip_delaunay(xyz, cells, -1)
    with pytest.raises(RuntimeError, match="CUDA"):
        flip_delaunay(xyz.cpu(), cells)
    out = flip_delaunay(xyz, cells[:0])
    assert len(out["cells"]) == 0 and out["n_proposed"] == 0
    # the workspace query writes the size and nothing else; a smaller workspace is refused
    T = len(C0)
    cells_out = torch.empty((T + T // 2, 4), dtype=torch.int32, device=DEV)
    src = torch.empty((T + T // 2, 3), dtype=torch.int32, device=DEV)
    counts = (C.c_uint32 * 4)(7, 7, 7, 7)
    nbytes = C.c_size_t(0)
    s = ext._stream(DEV)
    args = (DEV.index, xyz.data_ptr(), len(V), cells.data_ptr(), T, 0xFFFFFFFF, cells_out.data_ptr(), src.data_ptr(), counts)
    assert ext._lib.tn_flip_delaunay(*args, None, C.byref(nbytes), s) == 0
    assert nbytes.value > 0 and list(counts) == [7, 7, 7, 7]
    ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=DEV)
    small = C.c_size_t(nbytes.value - 1)
    assert ext._lib.tn_flip_delaunay(*args, ws.data_ptr(), C.byref(small), s) == 1  # TN_ERR_ARG
    assert ext._lib.tn_flip_delaunay(*args, ws.data_ptr(), C.byref(nbytes), s) == 0
    bad3 = torch.cat([cells, cells[:1]])
    args3 = (DEV.index, xyz.data_ptr(), len(V), bad3.data_ptr(), T + 1, 0xFFFFFFFF, cells_out.data_ptr(), src.data_ptr(), counts)
    n3 = C.c_size_t(0)
    assert ext._lib.tn_flip_delaunay(*args3, None, C.byref(n3), s) == 0
    ws3 = torch.empty((n3.value,), dtype=torch.uint8, device=DEV)
    assert ext._lib.tn_flip_delaunay(*args3, ws3.data_ptr(), C.byref(n3), s) == 3  # TN_ERR_MESH


def _fixed_point(V, C0, max_passes=80):
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(C0).to(DEV)
    for _ in range(max_passes):
        out = _gpu_pass(V, cells.cpu().numpy())
        if out["n_proposed"] == 0:
            return cells
        cells = out["cells"]
    raise AssertionError("no fixed point")


def _outside_rays(V, C0, n, seed):
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    tgt = V[C0[rng.integers(0, len(C0), n)]].astype(np.float64).mean(1)
    u = rng.standard_normal((n, 3))
    o = (tgt + 2.0 * np.linalg.norm(hi - lo) * u / np.linalg.norm(u, axis=1, keepdims=True)).astype(np.float32)
    d = tgt - o
    return o, (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("kind", ["coarsened", "jittered"])
def test_flipped_mesh_keeps_the_walk(small_mesh, kind):
    """refinement splits hull faces into nearly coplanar ones, which turns the walk off before any flip; coarsening and a move of the
    interior vertices keep the hull, so those meshes are walkable before flipping"""
    from tetranerf import cpp

    V, C0 = _coarsened(*small_mesh) if kind == "coarsened" else _jittered(*small_mesh, keep_hull=True)
    assert ofl.flip_delaunay(V, C0)["n_proposed"] > 0
    tr0 = cpp.TetrahedraTracer(DEV)
    tr0.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C0).to(DEV))
    assert tr0.trace_stats()[0] == 1, "the refined mesh is not walkable to begin with"
    C1 = _fixed_point(V, C0).cpu().numpy()
    assert len(C1) != len(C0) or not np.array_equal(C1, C0)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C1).to(DEV))
    assert tr.trace_stats()[0] == 1, "the flipped mesh lost the adjacency walk"
    o, d = _outside_rays(V, C1, 512, 6)
    ref = orc.OracleMesh(V, C1).trace_rays(o, d, 1024)
    do, dd = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    for impl in TRACE_IMPLS:
        force_trace_impl(tr, impl)
        out = tr.trace_rays(do, dd, 1024)
        tr.synchronize()
        for k in TRACE_KEYS:
            assert np.array_equal(out[k].cpu().numpy().view(np.uint32), ref[k].view(np.uint32)), (impl, k)


def test_affine_field_renders_the_same(small_mesh):
    """an affine field f_c(x) = A_c . (x - m) + b_c is reproduced exactly by linear interpolation on any tetrahedralisation of the same
    domain, so the fused render before and after flipping differs by rounding only.  Bound: the interpolated field differs by a few fp32
    ulps (|f| < 4, barycentric weights in [0, 1]: about 1e-6 absolute); the MLP in bf16x3 keeps fp32-level accuracy, and the uniform
    sampler puts the samples at the same distances because the hull is the same, so each sample's colour and density move by ~1e-6
    relative and the composite by at most that times the sample count's weight sum: 1e-4 on rgb / accumulation, 1e-4 of the far
    bound on depth, with two orders of margin."""
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    V, C0 = _refined(*small_mesh, passes=3, frac=0.05)
    C1 = _fixed_point(V, C0)
    assert len(C1) != len(C0) or not torch.equal(C1.cpu(), torch.from_numpy(C0))
    g = np.random.default_rng(0)
    A, b = g.standard_normal((64, 3)).astype(np.float32), (0.1 * g.standard_normal(64)).astype(np.float32)
    m = V.mean(0)
    field = (A @ (V - m).T + b[:, None]).astype(np.float32)  # [64, V]
    params = orc.init_mlp_params(0)
    o, d = syn.camera_rays(2000, seed=4)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    st = RenderSettings(max_intersected_triangles=1024, num_samples=64, num_fine_samples=64, use_biased_sampler=False)
    res = []
    for cells in (torch.from_numpy(C0).to(DEV), C1):
        tr = cpp.TetrahedraTracer(DEV)
        tr.load_tetrahedra(torch.from_numpy(V).to(DEV), cells)
        assert int(tr.trace_rays(o, d, 1024)["num_visited_cells"].max()) < 1024
        fr = FusedRenderer(tr)
        fr.set_field(torch.from_numpy(field).to(DEV))
        fr.set_weights(params)
        fr.set_mlp_precision(3)
        res.append(fr.render(o, d, st, expected_depth=True))
    assert torch.equal(res[0]["ray_mask"], res[1]["ray_mask"])
    far = float(np.linalg.norm(V.max(0) - V.min(0))) + 10.0
    for k, tol in (("rgb", 1e-4), ("accumulation", 1e-4), ("expected_depth", 1e-4 * far)):
        err = (res[0][k] - res[1][k]).abs().max().item()
        print(f"{len(C0)} -> {len(C1)} tetrahedra: max |{k} before - after| = {err:.2e} (tolerance {tol:.1e})")
        assert err < tol, k


def _model(V, C0, field, params, **cfg):
    from tetranerf.nerfstudio import model as M

    config = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C0), num_samples=48, num_fine_samples=32,
                                    max_intersected_triangles=1024, use_occupancy_field=True, **cfg)
    m = M.TetrahedraNerf(config)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C0), "tetrahedra_field": torch.from_numpy(field),
          "tetrahedra_occupancy": torch.zeros(len(C0))}
    sd.update(params)
    m.load_state_dict(sd, strict=False)
    return m.to(DEV), M, copy.deepcopy(config)


def _optimizers(m):
    from tetranerf.nerfstudio._ns_compat import Optimizers

    cfg = {k: {"optimizer": (lambda ps, lr=(1e-5 if k == "vertices" else 1e-3): torch.optim.RAdam(ps, lr=lr))} for k in m.get_param_groups()}
    return Optimizers(cfg, m.get_param_groups())


def test_model_trains_with_refinement_and_flips(small_mesh):
    from tetranerf import cpp
    from tetranerf.b200.flip import flip_delaunay

    V, C0 = small_mesh
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    m, M, original = _model(V, C0, field, params, refine_every=2, refine_start=2, refine_stop=100, refine_fraction=0.05,
                            refine_passes=2, delaunay_flip_every=3, occupancy_warmup_steps=0)
    opts = _optimizers(m)
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers=opts))
    assert len(cbs) == 3
    o, d = syn.camera_rays(1024, seed=4)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(1)).to(DEV)}
    m.train()
    flips = []
    flip = m.flip_delaunay
    m.flip_delaunay = lambda optimizers=None: flips.append(flip(optimizers)) or flips[-1]
    for step in range(1, 9):
        opts.zero_grad_all()
        losses = m.get_loss_dict(m(bundle), target)
        assert all(torch.isfinite(v).all() for v in losses.values()), step
        sum(losses.values()).backward()
        for p in m.parameters():
            assert p.grad is None or torch.isfinite(p.grad).all(), step
        opts.optimizer_step_all()
        n0 = len(flips)
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
        if len(flips) > n0:
            res = flips[-1]
            xyz, cells = m.tetrahedra_vertices.detach(), m.tetrahedra_cells
            if res["passes"][-1]["proposed"] == 0:  # a fixed point: nothing left to propose, and the left count is the pass's
                again = flip_delaunay(xyz, cells)
                assert again["n_proposed"] == 0 and again["n_illegal"] == res["illegal_left"]
            assert len(m.tetrahedra_occupancy) == len(cells) == m.config.num_tetrahedra_cells
            fresh = cpp.TetrahedraTracer(DEV)
            fresh.load_tetrahedra(xyz, cells)
            a = m._tetrahedra_tracer.trace_rays(bundle.origins, bundle.directions, 1024)
            b = fresh.trace_rays(bundle.origins, bundle.directions, 1024)
            for k in TRACE_KEYS:
                assert torch.equal(a[k], b[k]), k
            print(f"step {step}: {len(res['passes'])} passes, {res['tetrahedra_before']} -> {res['tetrahedra_after']} tetrahedra, "
                  f"illegal left {res['illegal_left']}, {res['seconds'] * 1e3:.1f} ms")
    assert flips and any(r["passes"][0]["proposed"] > 0 for r in flips)
    # the flipped checkpoint loads into the original config and renders the same bits
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    m.eval()
    with torch.no_grad():
        want = m(bundle)
    m2 = M.TetrahedraNerf(copy.deepcopy(original)).to(DEV)
    m2.load_state_dict(sd, strict=True)
    m2.eval()
    with torch.no_grad():
        got = m2(bundle)
    for k in ("rgb", "accumulation", "depth"):
        assert torch.equal(got[k], want[k]), k


def test_flips_keep_the_vertex_fold_guard(small_mesh):
    """with optimize_vertices and vertex_fold_guard, the flip callback runs after the optimizer step and before the forward that would
    guard and refit it: flip_delaunay must bring that step through the guard first, so no flip installs unguarded positions.  At a vertex
    rate whose raw steps fold the mesh, every step's flip leaves a mesh with no folded face and the walk on"""
    from tetranerf.nerfstudio import model as M
    from oracle import vertex_grads as vg
    from test_gpu_model import build_model

    V, C0 = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    m, _ = build_model(V, C0, field, num_samples=48, num_fine_samples=33, use_biased_sampler=True, optimize_vertices=True,
                       vertex_fold_guard=True, delaunay_flip_every=1)
    m.train()
    edge = float(np.median(np.linalg.norm(V[C0[:, 1]] - V[C0[:, 0]], axis=-1)))
    groups = m.get_param_groups()
    opt = torch.optim.Adam([{"params": groups["fields"], "lr": 5e-3}, {"params": groups["vertices"], "lr": 0.3 * edge}])
    cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers=opt))
    assert len(cbs) == 1
    o, d = (torch.from_numpy(x).to(DEV) for x in syn.camera_rays(2048, seed=21))
    target = torch.rand((2048, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    raw_folds, changed = [], 0
    for step in range(1, 11):
        opt.zero_grad()
        loss = m.get_loss_dict(m(M.RayBundle(origins=o, directions=d)), {"image": target})["rgb_loss"]
        assert torch.isfinite(loss)
        loss.backward()
        opt.step()
        cells = m.tetrahedra_cells.clone()
        raw_folds.append(vg.fold_count(m.tetrahedra_vertices.detach().cpu().numpy(), cells.cpu().numpy()))  # the step as taken
        for cb in cbs:
            cb.run_callback_at_location(step, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
        changed += not torch.equal(cells, m.tetrahedra_cells)
        tr = m.get_tetrahedra_tracer()
        assert tr.trace_stats()[0], f"step {step}: the walk is off after the flip"
        assert vg.fold_count(m.tetrahedra_vertices.detach().cpu().numpy(), m.tetrahedra_cells.cpu().numpy()) == 0, step
    print(f"folded faces of each raw step {raw_folds}; {changed} of 10 flips changed the mesh")
    assert max(raw_folds) > 0, "the vertex rate never folds the mesh: the scenario is not exercised"
    assert changed > 0
