"""GPU: the fused render and training step on opaque surfaces and non-white backgrounds, against the float32 / float64 oracles.

Every other parity test renders the torch-default network, which is almost transparent (accumulation ~0.5 on every ray, flat coarse
weights), on a white background.  Here synthetic.surface_scene puts two spheres into the field, with densities up to sharpness / 4
(sharpness k = 10, 100, 1000; ~250 at k = 1000, the order a trained NeRF reaches): rays turn opaque within a few samples, the median
depth is found by a crossing instead of the fall-through default, the PDF sampler inverts steep CDFs, the composite backward forms its
suffix sums behind a surface, and the f16w2 MLP meets densities two orders of magnitude above unit scale.  Regime guards
(test_surface_scene.assert_regime) keep each case from silently turning vacuous.

Bars: pixels (rgb, accumulation) 1e-4 absolute end to end for both MLP precisions.  Per sample, at the kernel's own fine bins (so that
PDF-inversion drift is not charged to the MLP): bf16x3 colour 1e-4 and density 1e-4 + 2e-5 |sigma|.  f16w2 carries the activations
as fp16 (11 significant bits), so its per-sample error is relative to the activations and grows with the gain behind them: density
1e-4 + 1e-3 |sigma| (measured on an H100: 4.9e-4 |sigma|), colour 3e-4 (measured 1.8e-4: unit-scale logits through the colour head's
gain of 3; 2.6e-5 on the torch-default network).  The pixel bar stays 1e-4 for both.  Gradients: the (A)/(B) bar of test_gpu_train.py."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _assert_bitwise, _deterministic, _inputs, _step
from test_gpu_render import _from_ptr, setup
from test_gpu_train import _run
from test_surface_scene import assert_regime, regime, scene_rays

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ASYM = (0.1, 0.6, 0.3)


def _settings(cfgname, background=(1.0, 1.0, 1.0)):
    from tetranerf.b200.render import RenderSettings

    if cfgname == "tetra_nerf":
        st, oc = RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    else:
        st, oc = RenderSettings.tetra_nerf_original(), orc.RenderConfig.tetra_nerf_original()
    st.background = oc.background = tuple(background)
    return st, oc


def _scene(V, k):
    """k = None: the random "normal" field with the torch-default network"""
    if k is None:
        return syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)
    return syn.surface_scene(V, k, orc.init_mlp_params(0))


def _render_parity(V, C, o, d, field, params, st, oc, prec, label):
    """fused render vs oracle.render: ray mask, empty rays, pixels, per-sample values at the kernel's fine bins, median depth.
    -> (fused outputs, oracle render with aux, kernel fine bins in ray order of the non-empty rays)"""
    tr, fr, _, _ = setup(V, C, prec=prec, field=field, params=params)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    tr.synchronize()
    mesh = orc.OracleMesh(V, C)
    ref = orc.render(mesh, torch.from_numpy(field), params, o, d, oc, return_aux=True)
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    empty = ~ref["ray_mask"]
    assert bool(empty.any())
    assert torch.equal(out["rgb"].cpu()[empty], torch.tensor(st.background, dtype=torch.float32).expand(int(empty.sum()), 3)), label
    assert bool((out["depth"].cpu()[empty] == st.far_plane).all()) and bool((out["accumulation"].cpu()[empty] == 0).all())
    # ---- per sample, at the kernel's own fine bins ----
    bufs = fr.debug_buffers()
    n_act = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    ray_list = _from_ptr(bufs["ray_list"], (n_act,), torch.int32).cpu().long()
    S2 = st.num_samples + st.num_fine_samples + 1
    eb = _from_ptr(bufs["ebins_f"], (n_act, S2 + 1), torch.float32).cpu()
    outf = _from_ptr(bufs["out_f"], (n_act, S2, 4), torch.float32).cpu()
    vi_gpu = _from_ptr(bufs["vi_f"], (n_act, S2, 4), torch.int32).cpu()
    back = torch.argsort(ray_list)  # slot -> order of the non-empty rays
    fine = eb[back]
    at = orc.render(mesh, torch.from_numpy(field), params, o, d, oc, return_aux=True, fine_euclid=fine)["aux"]
    sig_ref, col_ref = at["sigmas"][..., 0], at["colors"]
    sig, col = outf[back][..., 0], outf[back][..., 1:]
    flipped = (vi_gpu[back] != torch.from_numpy(at["matched"]["vertex_indices"])).any(-1)
    assert flipped.float().mean().item() < 2e-3
    sig_err, col_err = (sig - sig_ref).abs()[~flipped], (col - col_ref).abs().amax(-1)[~flipped]
    sref = sig_ref[~flipped].abs()
    big = sref > 1.0
    rel = (sig_err[big] / sref[big]).max().item() if bool(big.any()) else 0.0
    slope, col_bar = (2e-5, 1e-4) if prec == 3 else (1e-3, 3e-4)
    # ---- pixels, end to end ----
    e_rgb = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"]).abs().max().item()
    opaque = ref["accumulation"][:, 0] > 0.5
    e_dep = (out["depth"].cpu() - ref["depth"])[:, 0].abs()[opaque]
    print(f"{label}: max sigma {sig_ref.max().item():.1f}  sigma err max {sig_err.max().item():.2e}  max rel (sigma > 1) {rel:.2e}  colour err "
          f"{col_err.max().item():.2e}  |  max|rgb| {e_rgb:.2e}  max|acc| {e_acc:.2e}  depth > 1e-4 on {int((e_dep > 1e-4).sum())} of "
          f"{int(opaque.sum())} opaque rays  | flipped {int(flipped.sum())}")
    assert bool((sig_err <= 1e-4 + slope * sref).all()), (label, (sig_err - slope * sref).max().item())
    assert col_err.max().item() <= col_bar, (label, col_err.max().item())
    assert e_rgb < 1e-4 and e_acc < 1e-4, (label, e_rgb, e_acc)
    assert int((e_dep > 1e-4).sum()) <= max(1, int(opaque.sum()) // 100), label
    return out, ref, fine


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("cfgname", ["tetra_nerf", "tetra_nerf_original"])
@pytest.mark.parametrize("k", [10, 100, 1000])
def test_opaque_render_vs_oracle(small_mesh, k, cfgname, prec):
    V, C = small_mesh
    o, d = scene_rays(300)
    field, params = _scene(V, k)
    st, oc = _settings(cfgname)
    out, ref, fine = _render_parity(V, C, o, d, field, params, st, oc, prec, f"k={k} {cfgname} prec={prec}")
    if k >= 100:
        stats = regime(ref, o, d, oc)
        print(f"  regime: {stats}")
        assert_regime(stats, k, oc)
    if k == 1000:
        # independent of the oracle: the median depth of an opaque ray lies at the analytic first sphere crossing, up to one fine bin
        # plus the size of the tetrahedron there (the field is interpolated linearly over it, so the surface moves inside it)
        acc = out["accumulation"].cpu()[:, 0].numpy()
        dep = out["depth"].cpu()[:, 0].numpy().astype(np.float64)
        first = np.min(np.where(np.isfinite(syn.sphere_hits(o, d)[:, :, 0]), syn.sphere_hits(o, d)[:, :, 0], np.inf), axis=1)
        sel = np.nonzero((acc > 0.99) & np.isfinite(first))[0]
        assert len(sel) >= 50
        dn = d.astype(np.float64) / np.linalg.norm(d.astype(np.float64), axis=1, keepdims=True)
        hit = o[sel].astype(np.float64) + first[sel, None] * dn[sel]
        cell = orc.OracleMesh(V, C).find_tetrahedra(hit.astype(np.float32))["tetrahedra"]
        assert bool((cell >= 0).all())
        P = V[C[cell]].astype(np.float64)
        size = np.max([np.linalg.norm(P[:, i] - P[:, j], axis=1) for i in range(4) for j in range(i + 1, 4)], axis=0)
        row = np.cumsum(out["ray_mask"].cpu().numpy()) - 1  # ray -> row of the non-empty rays
        fe = fine.numpy().astype(np.float64)
        width = np.array([np.diff(fe[row[r]])[min(max(np.searchsorted(fe[row[r]], dep[r]) - 1, 0), fe.shape[1] - 2)] for r in sel])
        res = np.abs(dep[sel] - first[sel])
        print(f"  depth vs analytic sphere crossing on {len(sel)} rays: max {res.max():.3e}, max residual / (bin + tetrahedron) "
              f"{(res / (width + size)).max():.3f}")
        assert bool((res <= width + size).all())


def _occluded_vertex_check(details, V, label, min_count):
    """vertices touched only by samples whose float64 transmittance is < 1e-20: the float64 gradient there is ~0, the kernel's must be
    <= 1e-6 of the tensor's largest entry (the composite backward's suffix sums behind an opaque surface).  At k = 100 the densities
    (<= 25) cannot reach an optical depth of 46 inside the spheres, so only k = 1000 has such vertices."""
    aux = details["out_f64"]["aux"]
    fe, sig = aux["fine_euclid"].double(), aux["sigmas"][..., 0].double()
    x = (fe[:, 1:] - fe[:, :-1]) * sig
    T = torch.exp(-(torch.cumsum(x, -1) - x))
    vi = torch.from_numpy(aux["matched"]["vertex_indices"]).long()
    seen = torch.zeros(len(V), dtype=torch.bool)
    lit = vi[(T >= 1e-20)[..., None].expand_as(vi) & (vi >= 0)]
    seen[lit] = True
    dark = torch.zeros(len(V), dtype=torch.bool)
    dark[vi[(T < 1e-20)[..., None].expand_as(vi) & (vi >= 0)]] = True
    occluded = dark & ~seen
    g, g64 = details["gfield"].cpu().double(), details["gfield_f64"].double()
    scale = g.abs().max().item()
    worst = g[:, occluded].abs().max().item() if bool(occluded.any()) else 0.0
    worst64 = g64[:, occluded].abs().max().item() if bool(occluded.any()) else 0.0
    print(f"  {label}: {int(occluded.sum())} occluded vertices; kernel max |g| there {worst:.3e} = {worst / scale:.2e} of max |g| "
          f"(float64: {worst64 / scale:.2e})")
    assert int(occluded.sum()) >= min_count, int(occluded.sum())
    assert worst <= 1e-6 * scale, (label, worst / scale)


@pytest.mark.parametrize("gs", [False, True])
@pytest.mark.parametrize("k", [100, 1000])
def test_opaque_train_step_gradients(small_mesh, k, gs):
    V, C = small_mesh
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]
    field, params = _scene(V, k)
    st, oc = _settings("tetra_nerf")
    print(f"--- k={k}, gradient scaling {gs}")
    details = {}
    _run(V, C, o, d, st, oc, gs, seed=5, field=field, params=params, details=details)
    _occluded_vertex_check(details, V, f"k={k} gs={gs}", 20 if k == 1000 else 0)


def test_opaque_deterministic_and_saved_state(small_mesh):
    """k = 1000: deterministic mode gives bitwise-equal gradients twice, and one FusedTrainRender forward + backward (its own saved
    state) equals FusedRenderer.train_forward + train_backward bit for bit"""
    from tetranerf.b200.render import PARAM_ORDER, FusedTrainRender
    from test_gpu_train import _setup

    V, C = small_mesh
    o, d = scene_rays(300)
    field, params = _scene(V, 1000)
    st, _ = _settings("tetra_nerf")
    tr, fr, _ = _setup(V, C, field, params)
    inp = _inputs(o, d, st, seed=8)
    a = _step(fr, tr, len(V), st, inp, gs=True)
    b = _step(fr, tr, len(V), st, inp, gs=True)
    _assert_bitwise(a, b, "deterministic, k=1000")
    ro, rd, jc, jf, target = inp
    R = ro.shape[0]
    f = torch.from_numpy(field).to(DEV).requires_grad_(True)
    ps = [params[n].detach().to(DEV).clone().requires_grad_(True) for n in PARAM_ORDER]
    with _deterministic(True):
        rgb, acc, _, _ = FusedTrainRender.apply(fr, st, True, ro, rd, jc, jf, f, *ps)
        g_rgb = (2.0 * (rgb.detach() - target) / (3 * R)).contiguous()
        torch.autograd.backward([rgb, acc], [g_rgb, torch.full((R, 1), 0.05 / R, device=DEV)])
    tr.synchronize()
    assert torch.equal(rgb.detach(), a[0]["rgb"]) and torch.equal(acc.detach(), a[0]["accumulation"])
    assert torch.equal(f.grad, a[1])
    for n, p in zip(PARAM_ORDER, ps):
        assert torch.equal(p.grad, a[2][n]), n


@pytest.mark.parametrize("bg", [(0.0, 0.0, 0.0), ASYM], ids=["black", "asym"])
@pytest.mark.parametrize("k", [100, None], ids=["k100", "init"])
def test_background_render_and_gradients(small_mesh, k, bg):
    """a background other than white, through FusedRenderer: empty rays, bg (1 - acc) in the composite, (c - bg) in its backward"""
    V, C = small_mesh
    field, params = _scene(V, k)
    st, oc = _settings("tetra_nerf", bg)
    o, d = scene_rays(300)
    _render_parity(V, C, o, d, field, params, st, oc, 3, f"background {bg} k={k}")
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]
    _run(V, C, o, d, st, oc, False, seed=5, field=field, params=params)


def test_model_black_background_fused_vs_unfused(small_mesh, monkeypatch):
    """TetrahedraNerf(background_color="black"): the fused eval render against the unfused op sequence and the oracle; the fused
    training step against unfused training (pixels) and against the float64 oracle differentiated with the black background (gradients,
    the (B) bar of test_gpu_train.py: the unfused path is itself a torch fp32 pipeline whose field gradient already differs from the
    float64 one by ~1e-3 L2)"""
    from tetranerf.nerfstudio import model as M
    from test_gpu_train import _check

    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    params = orc.init_mlp_params(0)
    o, d = scene_rays(256)
    target = torch.rand((256, 3), generator=torch.Generator().manual_seed(3))
    bundle = lambda: M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))  # noqa: E731
    res = {}
    for mode in ("fused", "unfused"):
        monkeypatch.setenv("TETRANERF_B200_UNFUSED_TRAIN", "1" if mode == "unfused" else "0")
        cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=64, num_fine_samples=64,
                                     use_biased_sampler=True, use_gradient_scaling=True, background_color="black")
        m = M.TetrahedraNerf(cfg)
        sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
        sd.update(params)
        m.load_state_dict(sd, strict=False)
        m = m.to(DEV).eval()
        if mode == "fused":
            with torch.no_grad():
                ev = m(bundle())
            assert m._fused is not None
        else:
            ev = {k: v.detach() for k, v in m(bundle()).items()}  # autograd on: the unfused op sequence
        m.train()
        m.sampler_uniform.train_stratified = False
        m.sampler_pdf.train_stratified = False
        out = m(bundle())
        m.get_loss_dict(out, {"image": target.to(DEV)})["rgb_loss"].backward()
        res[mode] = (ev["rgb"].cpu(), out["rgb"].detach().cpu(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    oc = orc.RenderConfig(num_samples=64, num_fine_samples=64, use_biased_sampler=True, background=(0.0, 0.0, 0.0))
    ref = orc.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, oc)
    assert res["fused"][0][5].tolist() == [0.0, 0.0, 0.0] and res["unfused"][0][5].tolist() == [0.0, 0.0, 0.0]
    assert (res["fused"][0] - ref["rgb"]).abs().max().item() < 1e-4
    assert (res["fused"][0] - res["unfused"][0]).abs().max().item() < 1e-4
    assert (res["fused"][1] - res["unfused"][1]).abs().max().item() < 1e-4
    assert set(res["fused"][2]) == set(res["unfused"][2]) and "tetrahedra_field" in res["fused"][2]
    grads = {}
    for dtype in (torch.float32, torch.float64):  # the model's loss (MSE) through the oracle, eval-mode bins as the stratification is off
        f = torch.from_numpy(field).to(dtype).requires_grad_(True)
        p = {k: v.clone().to(dtype).requires_grad_(True) for k, v in params.items()}
        torch.set_default_dtype(dtype)
        try:
            r = orc.render_train(orc.OracleMesh(V, C), f, p, o, d, oc, use_gradient_scaling=True)
        finally:
            torch.set_default_dtype(torch.float32)
        torch.nn.functional.mse_loss(r["rgb"], target.to(dtype)).backward()
        assert (r["rgb"].detach().float() - res["fused"][1]).abs().max().item() < 1e-4
        grads[dtype] = {"tetrahedra_field": f.grad, **{k: v.grad for k, v in p.items()}}
    failures = []
    for n, g in res["fused"][2].items():
        assert torch.isfinite(g).all(), n
        _check(n, g, grads[torch.float32][n], grads[torch.float64][n], grads[torch.float64][n], failures)
    assert not failures, failures
