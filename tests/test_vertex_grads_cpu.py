"""CPU: the float64 oracle of the vertex gradient of the training step (oracle/vertex_grads.py, DESIGN §4.9) against central finite
differences in the vertex positions and against translation invariance; the numpy fold test; the optimize_vertices option of the model
(param groups, state dict, checkpoints); and the DDP gradient average of a vertex gradient."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import oracle as orc
from oracle import vertex_grads as vg
from tetranerf.b200 import synthetic as syn
from tetranerf.nerfstudio import model as M

ROOT = Path(__file__).resolve().parents[1]


def _loss(out, target):
    return torch.nn.functional.mse_loss(out["rgb"], target) + 0.05 * out["accumulation"].mean()


@pytest.fixture(scope="module")
def scene():
    V, C = syn.delaunay_mesh(3000, seed=0)
    field = torch.from_numpy(syn.random_field(len(V), 64, seed=3)).double()
    params = {k: v.double() for k, v in orc.init_mlp_params(0).items()}
    o, d = syn.camera_rays(24, seed=11)
    o[3] = [5, 5, 5]; d[3] = [1, 0, 0]  # empty ray
    return orc.OracleMesh(V, C), V, C, field, params, o, d


def _render(scene, xyz, ot, dt, **kw):
    mesh, _, _, field, params, _, _ = scene
    cfg = orc.RenderConfig(num_samples=24, num_fine_samples=23, use_biased_sampler=True)
    R = len(ot)
    g = torch.Generator().manual_seed(4)
    jc, jf, target = torch.rand((R, 25), generator=g), torch.rand((R, 24), generator=g), torch.rand((R, 3), generator=g).double()
    return vg.render_train_geometry(mesh, field, params, ot, dt, xyz, cfg, jc, jf, **kw), target


def test_vertex_gradient_matches_finite_differences(scene):
    """dL/dx_v of the add_barycentrics_grad oracle against central differences of the same render with b = E^-1 (x - x_v0) recomputed
    from the positions, the fine bins and the matched tetrahedra held fixed"""
    _, V, _, _, _, o, d = scene
    torch.set_default_dtype(torch.float64)
    try:
        xyz = torch.from_numpy(V).double().requires_grad_(True)
        ot, dt = torch.from_numpy(o).double(), torch.from_numpy(d).double()
        out, target = _render(scene, xyz, ot, dt)
        _loss(out, target).backward()
        gv = xyz.grad.clone()
        assert gv.abs().max() > 0
        fixed = dict(fine_euclid=out["aux"]["fine_euclid"], matched=out["aux"]["matched"], exact_bary=True)
        x2 = xyz.detach().clone().requires_grad_(True)
        out2, _ = _render(scene, x2, ot, dt, **fixed)
        _loss(out2, target).backward()
        rel = (gv - x2.grad).abs().max().item() / x2.grad.abs().max().item()
        # (3.3e-3: a vertex entry sums the few samples around the vertex, so where the tracer's float32 weights of one sample differ from
        # the recomputed ones -- samples on a face, thin tetrahedra -- it shows undiluted, unlike the ray sums of test_ray_grads_cpu.py)
        print(f"  add_barycentrics_grad vs recomputed weights: {rel:.2e} of the largest entry")
        assert rel < 1e-2
        g = x2.grad

        def L(x):
            with torch.no_grad():
                return _loss(_render(scene, x, ot, dt, **fixed)[0], target).item()

        h = 1e-8
        scale = g.abs().max().item()
        worst = 0.0
        for v in torch.argsort(g.abs().sum(-1), descending=True)[:4].tolist() + [int(torch.nonzero(g.abs().sum(-1) > 0)[0])]:
            for c in range(3):
                u = torch.zeros_like(xyz)
                u[v, c] = 1.0
                fd = (L(xyz.detach() + h * u) - L(xyz.detach() - h * u)) / (2 * h)
                worst = max(worst, abs(fd - g[v, c].item()) / scale)
                assert abs(fd - g[v, c].item()) <= 1e-5 * scale, (v, c, g[v, c].item(), fd)
        print(f"  max |finite differences - analytic| / max |g|: {worst:.2e}")
    finally:
        torch.set_default_dtype(torch.float32)


def test_translation_invariance(scene):
    """moving the rays and the mesh together changes nothing: sum_v dL/dx_v + sum_r dL/do_r = 0"""
    _, V, _, _, _, o, d = scene
    torch.set_default_dtype(torch.float64)
    try:
        xyz = torch.from_numpy(V).double().requires_grad_(True)
        ot, dt = torch.from_numpy(o).double().requires_grad_(True), torch.from_numpy(d).double()
        out, target = _render(scene, xyz, ot, dt)
        _loss(out, target).backward()
        total = xyz.grad.sum(0) + ot.grad.sum(0)
        rel = total.abs().max().item() / xyz.grad.abs().sum().item()
        print(f"  |sum g_v + sum g_o| / sum |g_v| = {rel:.2e}")
        assert rel < 1e-12
    finally:
        torch.set_default_dtype(torch.float32)


def test_geometry_render_restates_the_ray_render(scene):
    """render_train_geometry is render_train_rays with a vertex input: the same outputs and the same ray gradient"""
    from oracle import ray_grads as rg

    mesh, V, _, field, params, o, d = scene
    cfg = orc.RenderConfig(num_samples=24, num_fine_samples=23, use_biased_sampler=True)
    g = torch.Generator().manual_seed(4)
    jc, jf = torch.rand((len(o), 25), generator=g), torch.rand((len(o), 24), generator=g)
    torch.set_default_dtype(torch.float64)
    try:
        res = []
        for geo in (False, True):
            ot = torch.from_numpy(o).double().requires_grad_(True)
            dt = torch.from_numpy(d).double()
            if geo:
                out = vg.render_train_geometry(mesh, field, params, ot, dt, torch.from_numpy(V).double(), cfg, jc, jf)
            else:
                out = rg.render_train_rays(mesh, field, params, ot, dt, cfg, jc, jf)
            (out["rgb"].sum() + out["accumulation"].sum()).backward()
            res.append((out, ot.grad))
        (a, ga), (b, gb) = res
        for k in ("rgb", "accumulation", "depth", "ray_mask"):
            assert torch.equal(a[k], b[k]), k
        assert torch.equal(ga, gb)
    finally:
        torch.set_default_dtype(torch.float32)


@pytest.mark.parametrize("cause", ["hidden_size", "single_pass", "unfused_env"])
def test_optimize_vertices_outside_the_fused_path_raises(monkeypatch, cause):
    """optimize_vertices trains on the fused pipeline only: an unsupported configuration, num_fine_samples = 0 or
    TETRANERF_B200_UNFUSED_TRAIN=1 raises in training before any device work, naming the cause"""
    cfg = dict(num_tetrahedra_vertices=10, num_tetrahedra_cells=5, optimize_vertices=True)
    want = {"hidden_size": "hidden_size=64", "single_pass": "num_fine_samples=0", "unfused_env": "TETRANERF_B200_UNFUSED_TRAIN=1"}[cause]
    if cause == "hidden_size":
        cfg["hidden_size"] = 64
    elif cause == "single_pass":
        cfg["num_fine_samples"] = 0
    else:
        monkeypatch.setenv("TETRANERF_B200_UNFUSED_TRAIN", "1")
    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(**cfg))
    m.train()
    bundle = M.RayBundle(origins=torch.zeros((4, 3)), directions=torch.tensor([[0.0, 1.0, 0.0]]).expand(4, 3).contiguous())
    with pytest.raises(RuntimeError, match=want):
        m.get_outputs(bundle)


def test_scatter_restatement_sums_to_minus_m():
    """the float64 scatter of the kernel's per-sample vectors: the four terms of a sample sum to -m (b_0 = 1 - b_1 - b_2 - b_3)"""
    g = np.random.default_rng(0)
    vi = np.array([[0, 1, 2, 3], [-1, -1, -1, -1], [4, 2, 1, 0]])
    bary = g.random((3, 3)).astype(np.float32) / 3
    m = g.standard_normal((3, 3))
    out = vg.scatter_vertex_grads(vi, bary, m, 5)
    assert np.allclose(out.sum(0), -(m[0] + m[2]), rtol=1e-6, atol=1e-7)
    assert np.allclose(out[3], -bary[0, 2] * m[0], rtol=1e-6)  # vertex 3 is v3 of sample 0 only


def test_fold_count(scene):
    """0 on the Delaunay mesh; an interior vertex pushed through the opposite face of one of its tetrahedra folds faces"""
    _, V, C, _, _, _, _ = scene
    tri, tt = vg.face_tables(C)
    assert len(tri) == len(np.unique(np.sort(tri, 1), axis=0)) and np.all(tt[:, 0] >= 0)
    assert vg.fold_count(V, C, tri, tt) == 0
    X = V.copy()
    hull = set(tri[tt[:, 1] < 0].reshape(-1).tolist())
    v = next(i for i in range(len(V)) if i not in hull)
    t = int(np.nonzero((C == v).any(1))[0][0])
    others = [u for u in C[t] if u != v]
    X[v] = X[v] + 2.0 * (X[others].mean(0) - X[v])  # reflected through the centroid of the opposite face
    n = vg.fold_count(X, C, tri, tt)
    print(f"  folded faces after pushing one vertex through its opposite face: {n}")
    assert n > 0
    # the face tables are the reference's: a tetrahedron's first face (opposite local vertex 0) is (c1, c2, c3) as stored
    assert list(tri[0]) == list(C[0][[1, 2, 3]])


def _model(on, V=7, T=3):
    return M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=V, num_tetrahedra_cells=T, optimize_vertices=on))


def test_optimize_vertices_param_groups_and_checkpoints():
    off, on = _model(False), _model(True)
    assert not M.TetrahedraNerfConfig(num_tetrahedra_vertices=7, num_tetrahedra_cells=3).optimize_vertices
    assert set(off.get_param_groups()) == {"fields"}
    assert all(p is not off.tetrahedra_vertices for p in off.get_param_groups()["fields"])
    groups = on.get_param_groups()
    assert set(groups) == {"fields", "vertices"}
    assert len(groups["vertices"]) == 1 and groups["vertices"][0] is on.tetrahedra_vertices and on.tetrahedra_vertices.requires_grad
    assert all(p is not on.tetrahedra_vertices for p in groups["fields"])
    assert len(groups["fields"]) == len(off.get_param_groups()["fields"])
    assert isinstance(on.tetrahedra_vertices, torch.nn.Parameter) and not isinstance(off.tetrahedra_vertices, torch.nn.Parameter)
    assert set(on.state_dict()) == set(off.state_dict())
    assert on.state_dict()["tetrahedra_vertices"].shape == (7, 3)
    # checkpoints go both ways
    g = torch.Generator().manual_seed(0)
    for src, dst in ((on, _model(False)), (off, _model(True))):
        with torch.no_grad():
            src.tetrahedra_vertices.copy_(torch.rand((7, 3), generator=g))
            src.tetrahedra_field.copy_(torch.rand((64, 7), generator=g))
        dst.load_state_dict(src.state_dict())
        assert torch.equal(dst.tetrahedra_vertices, src.tetrahedra_vertices) and torch.equal(dst.tetrahedra_field, src.tetrahedra_field)
        assert dst._tetrahedra_initialized


def test_optimize_vertices_install_mesh_under_no_grad():
    """_install_mesh writes the parameter in place without recording it in a graph"""
    V, C = syn.delaunay_mesh(50, seed=1)
    m = _model(True, len(V), len(C))
    rgb = np.full((len(V), 3), 128, np.uint8)
    m._install_mesh(torch.from_numpy(V), torch.from_numpy(C), torch.from_numpy(rgb), None)
    assert isinstance(m.tetrahedra_vertices, torch.nn.Parameter) and m.tetrahedra_vertices.grad_fn is None
    assert torch.equal(m.tetrahedra_vertices.detach(), torch.from_numpy(V))


# ---- DDP: average_gradients averages the vertex gradient like any other ----------------------------------------------------------------
def _grad_worker(rank, world, port, out_dir):
    for p in (str(ROOT), str(ROOT / "tetra-nerf_b200")):
        sys.path.insert(0, p)
    from oracle import oracle as orc
    from oracle import vertex_grads as vg
    from tetranerf.b200 import synthetic as syn
    from tetranerf.b200.distributed import average_gradients, shard_bounds

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    V, C = syn.delaunay_mesh(800, seed=2)
    mesh = orc.OracleMesh(V, C)
    cfg = orc.RenderConfig(num_samples=16, num_fine_samples=16, use_biased_sampler=True)
    R = 32
    o, d = syn.camera_rays(R, seed=3)
    g = torch.Generator().manual_seed(4)
    jc, jf, tgt = torch.rand((R, 17), generator=g), torch.rand((R, 17), generator=g), torch.rand((R, 3), generator=g)

    def grads(lo, hi):
        f = torch.from_numpy(syn.random_field(len(V), 64, seed=3)).requires_grad_(True)
        x = torch.from_numpy(V).clone().requires_grad_(True)
        p = {k: v.clone() for k, v in orc.init_mlp_params(0).items()}
        out = vg.render_train_geometry(mesh, f, p, torch.from_numpy(o[lo:hi]), torch.from_numpy(d[lo:hi]), x, cfg, jc[lo:hi], jf[lo:hi],
                                       nthreads=1)
        torch.nn.functional.mse_loss(out["rgb"], tgt[lo:hi]).backward()
        return [f, x]

    lo, hi = shard_bounds(R, rank, world)
    mine = grads(lo, hi)
    average_gradients(mine)
    whole = grads(0, R)
    err = max(((a.grad - b.grad).abs().max() / b.grad.abs().max().clamp_min(1e-30)).item() for a, b in zip(mine, whole))
    torch.save({"err": err, "nonzero": bool(whole[1].grad.abs().max() > 0)}, os.path.join(out_dir, f"g{rank}.pt"))
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_ddp_average_of_vertex_gradients(tmp_path):
    """two ranks, each differentiating its half of the batch; after average_gradients the vertex gradient is the whole batch's"""
    world = 2
    mp.spawn(_grad_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"g{r}.pt") for r in range(world)]
    assert all(r["nonzero"] for r in res)
    assert max(r["err"] for r in res) < 1e-5, res
