"""GPU: deterministic mode of the fused training step and of interpolate_values_backward (torch.use_deterministic_algorithms(True) or
TETRANERF_B200_DETERMINISTIC=1).  With identical inputs the outputs and every gradient are bitwise identical from run to run, whatever
the backward grid size; the forward outputs equal the default mode's bit for bit; the gradients meet the same float64 bar as the
default mode (tests/test_gpu_train.py)."""
import contextlib
import os
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_train import DEV, _run, _setup

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


@contextlib.contextmanager
def _deterministic(on: bool = True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _settings(name):
    from tetranerf.b200.render import RenderSettings

    if name == "tetra_nerf":
        return RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    return RenderSettings.tetra_nerf_original(), orc.RenderConfig.tetra_nerf_original()


def _inputs(o, d, st, seed):
    g = torch.Generator().manual_seed(seed)
    R = len(o)
    jc = torch.rand((R, st.num_samples + 1), generator=g).to(DEV)
    jf = torch.rand((R, st.num_fine_samples + 1), generator=g).to(DEV)
    target = torch.rand((R, 3), generator=g).to(DEV)
    return torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), jc, jf, target


def _step(fr, tr, nv, st, inp, gs, det=True):
    """one fused training step; -> (forward outputs, field gradient, {name: MLP gradient}), cloned"""
    o, d, jc, jf, target = inp
    R = o.shape[0]
    with _deterministic(det):
        out = fr.train_forward(o, d, st, jc, jf)
        g_rgb = (2.0 * (out["rgb"] - target) / (3 * R)).contiguous()
        g_acc = torch.full((R,), 0.05 / R, device=DEV)
        gf, gp = fr.train_backward(g_rgb, g_acc, nv, use_gradient_scaling=gs)
    tr.synchronize()
    return {k: v.clone() for k, v in out.items()}, gf.clone(), {k: v.clone() for k, v in gp.items()}


def _assert_bitwise(a, b, what):
    assert torch.equal(a[0]["rgb"], b[0]["rgb"]), f"{what}: rgb"
    assert torch.equal(a[1], b[1]), f"{what}: tetrahedra_field gradient"
    assert len(a[2]) == 12
    for k in a[2]:
        assert torch.equal(a[2][k], b[2][k]), f"{what}: {k}"


def _differs(a, b):
    return (not torch.equal(a[1], b[1])) or any(not torch.equal(a[2][k], b[2][k]) for k in a[2])


@pytest.mark.parametrize("cfgname,gs", [("tetra_nerf", False), ("tetra_nerf_original", True)])
def test_deterministic_step_is_bitwise_repeatable(medium_mesh, cfgname, gs):
    """1200 rays: many tiles per CTA of the backward, every partition busy"""
    V, C = medium_mesh
    st, _ = _settings(cfgname)
    tr, fr, _ = _setup(V, C, syn.random_field(len(V), 64, seed=3))
    inp = _inputs(*syn.camera_rays(1200, seed=12), st, seed=6)
    a = _step(fr, tr, len(V), st, inp, gs)
    b = _step(fr, tr, len(V), st, inp, gs)
    _assert_bitwise(a, b, "two deterministic runs")
    assert all(torch.isfinite(t).all() for t in [a[1]] + list(a[2].values()))


def test_deterministic_gradients_do_not_depend_on_the_grid(medium_mesh):
    V, C = medium_mesh
    st, _ = _settings("tetra_nerf")
    tr, fr, _ = _setup(V, C, syn.random_field(len(V), 64, seed=3))
    inp = _inputs(*syn.camera_rays(1200, seed=12), st, seed=6)
    runs = {}
    for ctas in (1, 3, 0):  # 0: the default grid (one CTA per SM)
        fr.set_backward_grid(ctas)
        runs[ctas] = _step(fr, tr, len(V), st, inp, False)
    fr.set_backward_grid(0)
    _assert_bitwise(runs[1], runs[0], "grid 1 vs default grid")
    _assert_bitwise(runs[3], runs[0], "grid 3 vs default grid")


def test_deterministic_hot_vertices(cube_mesh):
    """the 12-tetrahedra cube: ~1000 rays x 257 samples land on nine vertices, so the order of the field-gradient sums matters"""
    V, C = cube_mesh
    st, _ = _settings("tetra_nerf")
    tr, fr, _ = _setup(V, C, syn.random_field(len(V), 64, seed=3))
    inp = _inputs(*syn.camera_rays(1000, seed=21), st, seed=8)
    a = _step(fr, tr, len(V), st, inp, True)
    b = _step(fr, tr, len(V), st, inp, True)
    _assert_bitwise(a, b, "hot vertices, two deterministic runs")
    x = _step(fr, tr, len(V), st, inp, True, det=False)
    y = _step(fr, tr, len(V), st, inp, True, det=False)
    print(f"default mode: two identical steps gave {'different' if _differs(x, y) else 'identical'} gradients")


@pytest.mark.parametrize("cfgname,gs", [("tetra_nerf", False), ("tetra_nerf_original", True)])
def test_deterministic_gradients_meet_the_float64_bar(small_mesh, cfgname, gs):
    """the bar of test_fused_train_step_gradients: max|g - g_f64| <= max(2e-4, 6 max|g_torch_f32 - g_f64|), per tensor"""
    V, C = small_mesh
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    st, oc = _settings(cfgname)
    with _deterministic():
        _run(V, C, o, d, st, oc, gs, seed=5)


def test_deterministic_forward_equals_default(medium_mesh):
    V, C = medium_mesh
    st, _ = _settings("tetra_nerf")
    tr, fr, _ = _setup(V, C, syn.random_field(len(V), 64, seed=3))
    o, d = syn.camera_rays(1200, seed=12)
    o[7] = [5, 5, 5]; d[7] = [1, 0, 0]  # empty ray: slots shift
    inp = _inputs(o, d, st, seed=6)
    a = _step(fr, tr, len(V), st, inp, False, det=False)
    b = _step(fr, tr, len(V), st, inp, False, det=True)
    for k in ("rgb", "accumulation", "depth", "ray_mask"):
        assert torch.equal(a[0][k], b[0][k]), k
    # the modes only sum in another order: the gradients agree to rounding
    for k in a[2]:
        s = a[2][k].abs().max().item()
        assert (a[2][k] - b[2][k]).abs().max().item() <= 1e-4 * s + 1e-12, k


@pytest.mark.parametrize("D", [2, 3, 4, 6])
@pytest.mark.parametrize("C", [3, 5, 64])
def test_deterministic_interpolate_values_backward(D, C):
    from tetranerf import cpp

    V, N = 97, 6000  # ~60 samples per vertex slot: the summation order matters
    rng = np.random.default_rng(100 * D + C)
    vi = rng.integers(0, V, size=(N, D)).astype(np.int32)
    vi[rng.random(N) < 0.05, 0] = -1  # empty slots
    w = rng.random((N, D - 1)).astype(np.float32) / D
    g = rng.standard_normal((N, C)).astype(np.float32)
    field = torch.zeros((C, V), dtype=torch.float32, device=DEV)
    args = (torch.from_numpy(vi).to(DEV), torch.from_numpy(w).to(DEV), field, torch.from_numpy(g).to(DEV))
    with _deterministic():
        a = cpp.interpolate_values_backward(*args)
        b = cpp.interpolate_values_backward(*args)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    # float64 truth: slot k >= 1 carries w[k-1], slot 0 the rest; empty slots contribute nothing
    w64 = torch.from_numpy(w).double()
    wk = torch.cat([1.0 - w64.sum(1, keepdim=True), w64], 1)
    ref = torch.zeros((V + 1, C), dtype=torch.float64)
    idx = torch.from_numpy(vi).long().where(torch.from_numpy(vi) >= 0, torch.tensor(V))
    for k in range(D):
        ref.index_add_(0, idx[:, k], wk[:, k:k + 1] * torch.from_numpy(g).double())
    ref = ref[:V].T
    err = (a.cpu().double() - ref).abs().max().item()
    assert err <= 1e-5 * ref.abs().max().item(), err


_MODEL_STEP = textwrap.dedent("""
    import os, sys
    sys.path[:0] = [{root!r}, {pkg!r}]
    import torch
    from oracle import oracle as orc
    from tetranerf.b200 import synthetic as syn
    from tetranerf.nerfstudio import model as M

    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    V, C = syn.delaunay_mesh(3000, seed=0)
    field = syn.random_field(len(V), 64, seed=3)
    o, d = syn.camera_rays(256, seed=14)
    target = torch.rand((256, 3), generator=torch.Generator().manual_seed(3)).to(dev)
    grads = []
    for _ in range(2):
        torch.manual_seed(0)  # the stratified draws
        cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=64, num_fine_samples=64,
                                     use_biased_sampler=True, use_gradient_scaling=True)
        m = M.TetrahedraNerf(cfg)
        sd = {{"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}}
        sd.update(orc.init_mlp_params(0))
        m.load_state_dict(sd, strict=False)
        m = m.to(dev).train()
        out = m(M.RayBundle(origins=torch.from_numpy(o).to(dev), directions=torch.from_numpy(d).to(dev)))
        m.get_loss_dict(out, {{"image": target}})["rgb_loss"].backward()
        grads.append({{n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}})
    assert "tetrahedra_field" in grads[0] and len(grads[0]) == 13, sorted(grads[0])
    bad = [n for n in grads[0] if not torch.equal(grads[0][n], grads[1][n])]
    assert not bad, bad
    print("bitwise-equal gradients:", len(grads[0]))
""")


@pytest.mark.parametrize("unfused", ["0", "1"])
def test_model_training_step_is_bitwise_repeatable(unfused):
    """TetrahedraNerf under torch.use_deterministic_algorithms(True), fused and unfused training path, in a subprocess (cuBLAS needs
    CUBLAS_WORKSPACE_CONFIG under that flag, and the flag must not leak into other tests)"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", TETRANERF_B200_UNFUSED_TRAIN=unfused)
    env.pop("TETRANERF_B200_DETERMINISTIC", None)
    code = _MODEL_STEP.format(root=str(ROOT), pkg=str(ROOT / "tetra-nerf_b200"))
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    print(p.stdout[-2000:])
    assert p.returncode == 0, p.stderr[-4000:]
