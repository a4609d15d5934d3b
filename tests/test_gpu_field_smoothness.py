"""GPU: the field smoothness loss (tn_field_smoothness, FieldSmoothness, the model's field_smoothness_mult; DESIGN §4.15) against the
float64 oracle (oracle/smoothness.py).
  * the kernel on the 12-tetrahedra cube, the bottle mesh, a small Delaunay mesh, a refined mesh, a mesh with a vertex no cell uses and
    the 301,875- and 2,020,866-tetrahedra meshes: S within 1e-5 relative, E exact, the gradient within the per-element bound below;
  * repeated calls and the default / deterministic modes give the same bits;
  * lifecycle: another mesh of other V and T (a stale adjacency would show), update_vertices (same bits), set_field (a stale shadow would
    show), and the errors without a field or with a field of another V;
  * the model: mult = 0 changes nothing, mult > 0 adds mult * the oracle's loss and the oracle's gradient to the field gradient, two
    deterministic steps are bitwise equal, refine / optimize_vertices / occupancy / distortion compose, eval adds no key, the unfused
    training path gets the loss too.
Gradient bound: the kernel forms each difference d_k = f_i - f_j with one fp32 rounding, sums the deg_i of them in CSR order in fp32
and multiplies by an fp32 scale kappa = mult 2 / (E 64), so per element |g - g64| <= kappa (deg_i + 3) 2^-24 sum_k |d_k| (to first
order; 1 % slack on top).  A vertex without neighbours has the bound 0: its gradient must be exactly 0."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import smoothness as osm
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _deterministic
from test_gpu_refine import _model, _optimizers, _refined
from test_gpu_train import DEV

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
U = 2.0**-24


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _unused():
    V, C = syn.delaunay_mesh(300, seed=6)
    V = np.insert(V, 150, np.float32([0.5, 0.5, 0.5]), axis=0)
    return V, np.where(C >= 150, C + 1, C).astype(np.int32)


MESHES = {
    "cube": lambda: (syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()),
    "bottle": _bottle,
    "small": lambda: syn.delaunay_mesh(3000, seed=0),
    "refined": lambda: _refined(*syn.delaunay_mesh(3000, seed=0), frac=0.3, passes=2),
    "unused_vertex": _unused,
    "45k": lambda: syn.delaunay_mesh(45_000, seed=0),
    "300k": lambda: syn.delaunay_mesh(300_000, seed=0),
}


def _load(V, C, field):
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    tr = cpp.TetrahedraTracer(DEV)
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV)
    tr.load_tetrahedra(xyz, cells)
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(DEV))
    return tr, fr


def _field(n, seed=1):
    return np.random.default_rng(seed).standard_normal((64, n)).astype(np.float32)


def _check(fr, V, C, field, mult, what, grad=True):
    """the kernel's S, E and gradient against the oracle -> (S, gradient) as the kernel gave them"""
    S, E, g = fr.field_smoothness(mult, grad=grad)
    torch.cuda.synchronize()
    S64, E64 = osm.smoothness(field, C)
    assert E == E64, (what, E, E64)
    rel = abs(S.item() - S64) / max(S64, 1e-300)
    msg = f"{what}: V {len(V)}, T {len(C)}, E {E}; |S - S64| / S64 = {rel:.2e}"
    assert rel <= 1e-5 or S64 == S.item() == 0.0, msg
    if grad:
        g64 = osm.gradient(field, C, mult)
        a, deg = osm.neighbour_abs_sum(field, C)
        kappa = mult * 2.0 / (E * 64) if E else 0.0
        bound = 1.01 * kappa * (deg[None, :] + 3) * U * a
        err = np.abs(g.cpu().numpy().astype(np.float64) - g64)
        msg += f"; max |g - g64| / bound = {(err / np.where(bound > 0, bound, 1)).max():.3f}"
        assert np.all(err <= bound), msg
    print(msg)
    return S, g


@pytest.mark.parametrize("mesh", list(MESHES))
def test_kernel_against_oracle(mesh):
    V, C = MESHES[mesh]()
    field = _field(len(V))
    tr, fr = _load(V, C, field)
    S, g = _check(fr, V, C, field, 0.5, mesh)
    if mesh == "unused_vertex":
        assert torch.all(g[:, 150] == 0)
    # without the gradient: the same S
    S2, _, none = fr.field_smoothness(0.5)
    assert none is None and torch.equal(S, S2)


def test_reproducible_and_mode_independent():
    V, C = syn.delaunay_mesh(45_000, seed=0)
    field = _field(len(V), seed=4)
    tr, fr = _load(V, C, field)
    runs = []
    for det in (False, True, False, True):
        with _deterministic(det):
            S, E, g = fr.field_smoothness(2.0, grad=True)
            runs.append((S.clone(), g.clone()))
    for S, g in runs[1:]:
        assert torch.equal(S, runs[0][0]) and torch.equal(g, runs[0][1])


def test_lifecycle():
    V1, C1 = syn.delaunay_mesh(3000, seed=0)
    V2, C2 = _refined(*syn.delaunay_mesh(2000, seed=7), frac=0.4, passes=1)
    f1, f2 = _field(len(V1), 1), _field(len(V2), 2)
    tr, fr = _load(V1, C1, f1)
    _check(fr, V1, C1, f1, 1.0, "first mesh")
    # another mesh with a field of the old V: an error, not a stale read
    xyz2, cells2 = torch.from_numpy(V2).to(DEV), torch.from_numpy(C2).to(DEV)
    tr.load_tetrahedra(xyz2, cells2)
    with pytest.raises(RuntimeError, match="vertices"):
        fr.field_smoothness(1.0, grad=True)
    fr.set_field(torch.from_numpy(f2).to(DEV))
    S2, g2 = _check(fr, V2, C2, f2, 1.0, "second mesh")
    # moving the vertices keeps the adjacency and the bits
    moved = (xyz2 + 1e-4 * torch.randn_like(xyz2)).contiguous()
    tr.update_vertices(moved)
    S3, _, g3 = fr.field_smoothness(1.0, grad=True)
    assert torch.equal(S2, S3) and torch.equal(g2, g3)
    # a new field is read
    f3 = _field(len(V2), 3)
    fr.set_field(torch.from_numpy(f3).to(DEV))
    _check(fr, V2, C2, f3, 1.0, "new field")


def test_errors():
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    V, C = syn.delaunay_mesh(500, seed=0)
    tr = cpp.TetrahedraTracer(DEV)
    fr = FusedRenderer(tr)
    with pytest.raises(RuntimeError, match="no tetrahedra"):
        fr.field_smoothness()
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    with pytest.raises(RuntimeError, match="no field"):
        fr.field_smoothness()
    fr.set_field(torch.from_numpy(_field(len(V))).to(DEV))
    with pytest.raises(RuntimeError, match="finite"):
        fr.field_smoothness(float("nan"))


def test_autograd_function():
    from tetranerf.b200.render import FieldSmoothness

    V, C = syn.delaunay_mesh(3000, seed=0)
    field = _field(len(V))
    tr, fr = _load(V, C, field)
    f = torch.from_numpy(field).to(DEV).requires_grad_(True)
    loss = FieldSmoothness.apply(fr, 0.3, f)
    assert loss.dtype == torch.float32 and loss.shape == ()
    assert loss.item() == pytest.approx(osm.loss(field, C, 0.3), rel=1e-5)
    (3.0 * loss).backward()
    _, _, g = fr.field_smoothness(0.3, grad=True)
    assert torch.equal(f.grad, g * 3.0)


# ---- the model --------------------------------------------------------------------------------------------------------------------
MULT = 0.05


def _bundle(M, R=1024, seed=2):
    o, d = syn.camera_rays(R, seed=seed)
    return M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))


def _step(m, M, bundle, target, seed=0):
    """one training forward + loss + backward from a fixed seed -> (loss dict, {parameter name: gradient})"""
    m.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    losses = m.get_loss_dict(m(bundle), target)
    sum(losses.values()).backward()
    return {k: v.detach().clone() for k, v in losses.items()}, {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


def _scene(small=True):
    V, C = syn.delaunay_mesh(3000, seed=0)
    field, params = syn.surface_scene(V, 60, orc.init_mlp_params(0), noise=0.3)
    return V, C, field, params


def test_model_mult_zero_changes_nothing():
    V, C, field, params = _scene()
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(0)).to(DEV)}
    res = []
    for cfg in ({}, {"field_smoothness_mult": 0.0}):
        m, M, _ = _model(V, C, field, params, **cfg)
        m.train()
        with _deterministic():
            res.append(_step(m, M, _bundle(M), target))
    assert res[0][0].keys() == res[1][0].keys() and "field_smoothness_loss" not in res[1][0]
    for k in res[0][0]:
        assert torch.equal(res[0][0][k], res[1][0][k]), k
    assert res[0][1].keys() == res[1][1].keys()
    for k in res[0][1]:
        assert torch.equal(res[0][1][k], res[1][1][k]), k


@pytest.mark.parametrize("extra", [{}, {"optimize_vertices": True, "use_occupancy_field": True, "occupancy_warmup_steps": 0,
                                       "distortion_loss_mult": 0.01}], ids=["plain", "vertices+occupancy+distortion"])
def test_model_loss_and_gradient(extra):
    V, C, field, params = _scene()
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(0)).to(DEV)}
    m0, M, _ = _model(V, C, field, params, **extra)
    m1, _, _ = _model(V, C, field, params, field_smoothness_mult=MULT, **extra)
    m0.train(); m1.train()
    if extra.get("use_occupancy_field"):
        for m in (m0, m1):
            m.tetrahedra_occupancy.uniform_(0.5, 1.0)
    with _deterministic():
        l0, g0 = _step(m0, M, _bundle(M), target)
        l1, g1 = _step(m1, M, _bundle(M), target)
        l1b, g1b = _step(m1, M, _bundle(M), target)
    want = MULT * osm.smoothness(field, C)[0] / (osm.smoothness(field, C)[1] * 64)
    assert l1["field_smoothness_loss"].item() == pytest.approx(want, rel=1e-5)
    for k in l0:
        assert torch.equal(l0[k], l1[k]), k
    # two deterministic steps: the same bits
    for k in l1:
        assert torch.equal(l1[k], l1b[k]), k
    for k in g1:
        assert torch.equal(g1[k], g1b[k]), k
    # the other parameters see nothing of the loss; the field gains the oracle's gradient
    for k in g0:
        if k != "tetrahedra_field":
            assert torch.equal(g0[k], g1[k]), k
    g64 = osm.gradient(field, C, MULT)
    a, deg = osm.neighbour_abs_sum(field, C)
    E = osm.smoothness(field, C)[1]
    got = g1["tetrahedra_field"].cpu().numpy().astype(np.float64) - g0["tetrahedra_field"].cpu().numpy().astype(np.float64)
    bound = 1.01 * (MULT * 2.0 / (E * 64) * (deg[None, :] + 3) * U * a + U * np.abs(g1["tetrahedra_field"].cpu().numpy()))
    assert np.all(np.abs(got - g64) <= bound), np.abs(got - g64).max()


def test_model_after_refine():
    V, C, field, params = _scene()
    m, M, _ = _model(V, C, field, params, field_smoothness_mult=MULT, refine_fraction=0.1, refine_passes=2)
    opts = _optimizers(m, M)
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(0)).to(DEV)}
    m.train()
    for _ in range(2):
        opts.zero_grad_all()
        sum(m.get_loss_dict(m(_bundle(M)), target).values()).backward()
        opts.optimizer_step_all()
        m.accumulate_refine_statistics()
    res = m.refine(opts)
    assert res["tetrahedra_after"] > res["tetrahedra_before"]
    losses = m.get_loss_dict(m(_bundle(M)), target)
    F, cells = m.tetrahedra_field.detach().cpu().numpy(), m.tetrahedra_cells.cpu().numpy()
    assert losses["field_smoothness_loss"].item() == pytest.approx(MULT * osm.loss(F, cells), rel=1e-5)
    sum(losses.values()).backward()
    assert m.tetrahedra_field.grad.shape == F.shape


def test_model_eval_and_unfused_train():
    import os

    V, C, field, params = _scene()
    m, M, _ = _model(V, C, field, params, field_smoothness_mult=MULT)
    target = {"image": torch.rand((1024, 3), generator=torch.Generator().manual_seed(0)).to(DEV)}
    m.eval()
    with torch.no_grad():
        assert "field_smoothness_loss" not in m.get_loss_dict(m(_bundle(M)), target)
    # the unfused training path still gets the loss, on a fresh shadow
    m.train()
    os.environ["TETRANERF_B200_UNFUSED_TRAIN"] = "1"
    try:
        with torch.no_grad():
            m.tetrahedra_field.mul_(0.5)
        losses = m.get_loss_dict(m(_bundle(M)), target)
    finally:
        del os.environ["TETRANERF_B200_UNFUSED_TRAIN"]
    F = m.tetrahedra_field.detach().cpu().numpy()
    assert losses["field_smoothness_loss"].item() == pytest.approx(MULT * osm.loss(F, C), rel=1e-5)

