"""GPU parity of the fused TRAINING step (tn_render_train_forward / _backward: stratified bins, training-mode renderer, wgmma MLP
backward, field-gradient scatter) against torch-CPU autograd through the oracle (oracle.render_train = model.py:520-662 in training
mode).  Forward pixels within 1e-4 absolute.  Gradients: the oracle is differentiated twice, in float32 (what the reference computes)
and in float64 (the truth); the fine-pass sample positions come out of an fp32 PDF inversion and move by ~1e-6 between any two
implementations, so torch's own fp32 gradient already differs from the float64 one by up to ~6e-4 of the tensor's largest entry.
Measured with the oracle alone: the gradient itself is ill-conditioned in fp32 -- sums over ~10^5 samples with cancelling
terms -- so torch's OWN fp32 autograd differs from the float64 gradient by 1e-6 (heads) ... 8e-5 (third layer) ... 6e-4
(tetrahedra_field) of the tensor's largest entry, even at identical sample positions; an rtol of 1e-4 against an fp32 reference is
not a meaningful bar for the early layers.  The kernel computes with bf16x3 products (2^-17 operands instead of 2^-24).  Bars, per tensor (tetrahedra_field and each of the twelve MLP parameters), in units of the tensor's largest entry:
  (A) gradient arithmetic only: the float64 oracle evaluated AT THE KERNEL'S OWN fine-pass bins (detached in the reference, so this
      isolates everything that is differentiated: interpolation, MLP, heads, compositing, gradient scaling);
  (B) end to end, every stage independent (the oracle's own bins);
  both:  max |g_kernel - g_f64|  <=  max(2e-4, 6 x max |g_torch_f32 - g_f64|)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GRAD_TOL = 1e-4


def _setup(V, C, field, params=None):
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    params = orc.init_mlp_params(0) if params is None else params
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(DEV))
    fr.set_weights(params)
    return tr, fr, params


def _oracle_grads(V, C, field, params, o, d, oc, jc, jf, target, gs, mesh=None, dtype=torch.float32, fine_euclid=None):
    f = torch.from_numpy(field).to(dtype).requires_grad_(True)
    p = {k: v.clone().to(dtype).requires_grad_(True) for k, v in params.items()}
    torch.set_default_dtype(dtype)
    try:
        out = orc.render_train(mesh or orc.OracleMesh(V, C), f, p, o, d, oc, jc, jf, use_gradient_scaling=gs, fine_euclid=fine_euclid)
    finally:
        torch.set_default_dtype(torch.float32)
    loss = torch.nn.functional.mse_loss(out["rgb"], target.to(out["rgb"].dtype)) + 0.05 * out["accumulation"].mean()  # the accumulation path carries gradient too
    loss.backward()
    return out, f.grad, {k: v.grad for k, v in p.items()}


def _from_ptr(ptr, shape, dtype):
    import ctypes

    t = torch.empty(shape, dtype=dtype, device=DEV)
    ctypes.CDLL("libcudart.so").cudaMemcpy(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(ptr), ctypes.c_size_t(t.numel() * t.element_size()), ctypes.c_int(3))
    return t


def _check(name, got, f32, f64, f64_same_bins, failures):
    got, f32, f64, fsb = (t.detach().cpu().double() for t in (got, f32, f64, f64_same_bins))
    assert got.shape == f64.shape, (name, got.shape, f64.shape)
    assert torch.isfinite(got).all(), name
    scale = f64.abs().max().item()
    arith = (got - fsb).abs().max().item() / fsb.abs().max().item()   # (A) same sample positions: pure gradient arithmetic
    noise = (f32 - f64).abs().max().item() / scale                      # torch fp32 autograd against the float64 truth
    err = (got - f64).abs().max().item() / scale                        # (B) every stage independent
    print(f"  {name:34s} max|g| {scale:.3e}  (A) kernel vs f64 at the kernel's bins: {arith:.2e}   (B) kernel vs f64: {err:.2e}   torch-f32 vs f64: {noise:.2e}")
    if not (arith <= max(2 * GRAD_TOL, 6 * noise) and err <= max(2 * GRAD_TOL, 6 * noise)):
        failures.append((name, arith, err, noise))


def _run(V, C, o, d, st, oc, gs, seed, field_kind="normal", mesh=None, field=None, params=None, details=None):
    """field / params default to syn.random_field(kind=field_kind) and the torch-default network; the background is st's / oc's.
    details (a dict), if given, receives the kernel's gradients ("gfield", "gp") and the float64 oracle at the kernel's own fine bins
    ("gfield_f64", "gp_f64", "out_f64": its forward, with the per-sample aux)."""
    from tetranerf.b200.render import PARAM_ORDER

    field = syn.random_field(len(V), 64, seed=3, kind=field_kind) if field is None else field
    tr, fr, params = _setup(V, C, field, params)
    g = torch.Generator().manual_seed(seed)
    R = len(o)
    jc = torch.rand((R, st.num_samples + 1), generator=g)
    jf = torch.rand((R, st.num_fine_samples + 1), generator=g)
    target = torch.rand((R, 3), generator=g)
    mesh = mesh or orc.OracleMesh(V, C)
    ref, gf32, gp32 = _oracle_grads(V, C, field, params, o, d, oc, jc, jf, target, gs, mesh)
    _, gf64, gp64 = _oracle_grads(V, C, field, params, o, d, oc, jc, jf, target, gs, mesh, dtype=torch.float64)
    out = fr.train_forward(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    tr.synchronize()
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    e_rgb = (out["rgb"].cpu() - ref["rgb"].detach()).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"].detach()).abs().max().item()
    print(f"forward (training mode): max|rgb| {e_rgb:.2e} max|acc| {e_acc:.2e}")
    assert e_rgb < 1e-4 and e_acc < 1e-4
    # the same loss, differentiated by hand at the pixels: dL/drgb, dL/dacc
    g_rgb = (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
    g_acc = torch.full((R,), 0.05 / R, device=DEV)
    gfield, gp = fr.train_backward(g_rgb, g_acc, len(V), use_gradient_scaling=gs)
    tr.synchronize()
    # (A): the float64 oracle at the kernel's own fine bins (slot order -> order of the non-empty rays)
    bufs = fr.debug_buffers()
    n_act = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    S2 = st.num_samples + st.num_fine_samples + 1
    ray_list = _from_ptr(bufs["ray_list"], (n_act,), torch.int32).cpu().long()
    eb = _from_ptr(bufs["ebins_f"], (n_act, S2 + 1), torch.float32).cpu()
    fine = eb[torch.argsort(ray_list)]
    out_sb, gfsb, gpsb = _oracle_grads(V, C, field, params, o, d, oc, jc, jf, target, gs, mesh, dtype=torch.float64, fine_euclid=fine)
    if details is not None:
        details.update(gfield=gfield, gp=gp, gfield_f64=gfsb, gp_f64=gpsb, out_f64=out_sb)
    failures = []
    _check("tetrahedra_field", gfield, gf32, gf64, gfsb, failures)
    for n in PARAM_ORDER:
        _check(n, gp[n], gp32[n], gp64[n], gpsb[n], failures)
    assert not failures, failures
    return fr, tr


@pytest.mark.parametrize("cfgname,gs", [("tetra_nerf", False), ("tetra_nerf", True), ("small_uniform", False), ("tetra_nerf_original", True)])
def test_fused_train_step_gradients(small_mesh, cfgname, gs):
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    if cfgname == "tetra_nerf":
        st, oc = RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    elif cfgname == "tetra_nerf_original":
        st, oc = RenderSettings.tetra_nerf_original(), orc.RenderConfig.tetra_nerf_original()
    else:
        st, oc = RenderSettings(num_samples=48, num_fine_samples=33), orc.RenderConfig(num_samples=48, num_fine_samples=33)
    print(f"--- {cfgname}, gradient scaling {gs}")
    _run(V, C, o, d, st, oc, gs, seed=5)


def test_fused_train_step_is_repeatable_and_many_tiles(medium_mesh):
    """more tiles than SMs (dynamic tile scheduler, several tiles per CTA, dW reductions from every tile) and a second call on the
    same renderer (workspace reuse, counters reset)"""
    from tetranerf.b200.render import RenderSettings

    V, C = medium_mesh
    o, d = syn.camera_rays(1200, seed=12)
    st, oc = RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    fr, tr = _run(V, C, o, d, st, oc, False, seed=6)
    g = torch.Generator().manual_seed(6)
    R = len(o)
    jc, jf = torch.rand((R, 129), generator=g).to(DEV), torch.rand((R, 129), generator=g).to(DEV)
    outs = []
    for _ in range(2):
        out = fr.train_forward(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc, jf)
        gf, gp = fr.train_backward(torch.ones((R, 3), device=DEV) / R, None, len(V))
        tr.synchronize()
        outs.append((out["rgb"].clone(), gf.clone(), {k: v.clone() for k, v in gp.items()}))
    assert torch.equal(outs[0][0], outs[1][0])
    for k in outs[0][2]:  # atomics reorder the sums: equal to rounding, not bitwise
        s = outs[0][2][k].abs().max().item()
        assert (outs[0][2][k] - outs[1][2][k]).abs().max().item() <= 1e-5 * s + 1e-12, k
    assert (outs[0][1] - outs[1][1]).abs().max().item() <= 1e-5 * outs[0][1].abs().max().item()


def test_fused_train_step_on_2m_tetrahedra():
    """BASELINE configs[2] mesh size (300k points -> ~2.0 M tetrahedra), a ray subset the CPU oracle differentiates in seconds"""
    from tetranerf.b200.render import RenderSettings

    V, C = syn.delaunay_mesh(300_000, seed=0)
    assert len(C) > 1.9e6
    o, d = syn.camera_rays(96, seed=13)
    _run(V, C, o, d, RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf(), True, seed=7, field_kind="normal")


def test_model_training_path_fused_vs_unfused(small_mesh, monkeypatch):
    """TetrahedraNerf in training mode: the fused differentiable op against the reference's op sequence on the unfused CUDA ops + torch
    autograd (stratified draws switched off so that both consume the same bins)"""
    from tetranerf.nerfstudio import model as M

    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    o, d = syn.camera_rays(256, seed=14)
    target = torch.rand((256, 3), generator=torch.Generator().manual_seed(3)).to(DEV)
    grads = {}
    for mode in ("fused", "unfused"):
        monkeypatch.setenv("TETRANERF_B200_UNFUSED_TRAIN", "1" if mode == "unfused" else "0")
        cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=64, num_fine_samples=64,
                                     use_biased_sampler=True, use_gradient_scaling=True)
        m = M.TetrahedraNerf(cfg)
        sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
        sd.update(orc.init_mlp_params(0))
        m.load_state_dict(sd, strict=False)
        m = m.to(DEV).train()
        m.sampler_uniform.train_stratified = False
        m.sampler_pdf.train_stratified = False
        out = m(M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV)))
        loss = m.get_loss_dict(out, {"image": target})["rgb_loss"]
        loss.backward()
        grads[mode] = (out["rgb"].detach().clone(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    assert (grads["fused"][0] - grads["unfused"][0]).abs().max().item() < 1e-4
    assert set(grads["fused"][1]) == set(grads["unfused"][1]) and "tetrahedra_field" in grads["fused"][1]
    worst = 0.0
    for n, g in grads["unfused"][1].items():
        a = grads["fused"][1][n]
        rel = ((a - g).abs().max() / g.abs().max().clamp_min(1e-30)).item()
        l2 = ((a - g).norm() / g.norm().clamp_min(1e-30)).item()
        print(f"  {n:34s} fused vs unfused(torch fp32 autograd): max {rel:.2e}  L2 {l2:.2e}")
        assert torch.isfinite(a).all()
        worst = max(worst, l2)
        assert rel < 5e-3 and l2 < 1e-3, (n, rel, l2)  # two fp32 pipelines with independently rounded sample positions (see the module docstring)
