"""GPU: the expected depth of the fused render and training step (DESIGN §4.10) against the float64 oracle (oracle/expected_depth.py).
  * no regression: the other outputs are the same bits with the expected depth requested, and a depth backward without a depth gradient
    gives the existing entry points' bits;
  * forward: D at the kernel's own bins against float64, per MLP precision;
  * gradients of a loss on D (alone and with rgb / accumulation) to the field, the twelve MLP tensors, origins / directions and vertex
    positions, (A) at the kernel's bins and (B) end to end, with the bar of test_gpu_train.py;
  * the batch-wide clip and its gradient mask on rays where the clip binds;
  * determinism, the analytic sphere crossing of surface_scene, the model's fused and unfused training paths, and learning from depth
    alone."""
import numpy as np
import pytest
import torch

from oracle import expected_depth as edo
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_ray_grads import _blob_arrays, _inputs, _settings
from test_gpu_train import DEV, _check, _from_ptr, _setup
from tetranerf.b200.render import _lib

pytestmark = pytest.mark.gpu
# rays whose accumulation A is below this carry a 1/(A + 1e-10) that no fp32 implementation resolves: excluded from the depth loss of the
# gradient checks and from the forward bar, and counted
A_MIN = 1e-3
# forward bar, |D - D64| over rays with A >= A_MIN, in units of the call's depth range t_max - t_min (measured maxima: DESIGN §4.10)
FWD_BAR = {3: 3e-5, 2: 1e-4}


def _single():
    from tetranerf.b200.render import RenderSettings

    return RenderSettings(num_samples=96, num_fine_samples=0), orc.RenderConfig(num_samples=96, num_fine_samples=0)


def _field(V, k):
    return (syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)) if k is None else syn.surface_scene(V, k, orc.init_mlp_params(0))


def _rays(R=300, seed=11):
    o, d = syn.camera_rays(R, seed=seed)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    return o, d


@pytest.mark.parametrize("prec", [3, 2], ids=["bf16x3", "f16w2"])
def test_eval_outputs_unchanged(small_mesh, prec):
    """render with expected_depth (and normals) gives the same bits for every other output"""
    V, C = small_mesh
    field, params = _field(V, 100)
    _, fr, _ = _setup(V, C, field, params)
    fr.set_mlp_precision(prec)
    o, d = (torch.from_numpy(x).to(DEV) for x in _rays())
    for st, _ in (_settings("tetra_nerf"), _single()):
        for normals in (False, True):
            a = fr.render(o, d, st, normals=normals)
            b = fr.render(o, d, st, normals=normals, expected_depth=True)
            torch.cuda.synchronize()
            for key in a:
                assert torch.equal(a[key], b[key]), (key, normals)
            assert b["expected_depth"].shape == (len(o), 1) and torch.isfinite(b["expected_depth"]).all()
            assert b["expected_depth"][5, 0].item() == st.far_plane


def test_training_outputs_and_gradients_unchanged_by_expected_depth(small_mesh, monkeypatch):
    """deterministic mode: a forward with the expected depth gives the same rgb / accumulation / depth / mask, and its backward without
    a depth gradient the same gradients as a forward without it, with and without the ray and vertex gradients"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = small_mesh
    field, params = _field(V, None)
    st, _ = _settings("tetra_nerf")
    o, d = _rays(400, 21)
    jc, jf, target = _inputs(len(o), st, 7)
    _, fr, _ = _setup(V, C, field, params)
    args = (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    a, sa = fr.train_forward_saved(*args)
    b, sb = fr.train_forward_saved(*args, expected_depth=True)
    for key in a:
        assert torch.equal(a[key], b[key]), key
    g_rgb = (2.0 * (a["rgb"] - target.to(DEV)) / (3 * len(o))).contiguous()
    g_acc = torch.full((len(o),), 0.05 / len(o), device=DEV)
    for kw in ({}, {"grad_origins": True, "grad_directions": True, "grad_vertices": True}):
        ra = fr.train_backward_saved(sa, g_rgb, g_acc, len(V), True, **kw)
        rb = fr.train_backward_saved(sb, g_rgb, g_acc, len(V), True, **kw)
        # the backward entry point itself with a NULL depth gradient
        outs = [torch.empty((n, 3), device=DEV) if kw else None for n in (len(o), len(o), len(V))]
        rc = fr._grad_outputs(len(V))
        assert _lib.tn_render_train_backward_saved(fr.tracer.handle, sb.blob.data_ptr(), g_rgb.data_ptr(), g_acc.data_ptr(), None, 1,
                                                   rc[0].data_ptr(), rc[2], *(t.data_ptr() if t is not None else None for t in outs),
                                                   fr._stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(ra[0], rb[0])
        for n in ra[1]:
            assert torch.equal(ra[1][n], rb[1][n]), n
        for x, y in zip(ra[2:], rb[2:]):
            assert torch.equal(x, y)
        assert torch.equal(ra[0], rc[0]) and all(torch.equal(ra[1][n], rc[1][n]) for n in ra[1])
        for x, y in zip(ra[2:], outs if kw else ()):
            assert torch.equal(x, y)
    # a depth gradient on a forward that produced no expected depth is refused
    with pytest.raises(RuntimeError, match="no expected depth"):
        fr.train_backward_saved(sa, g_rgb, g_acc, len(V), True, grad_expected_depth=torch.ones(len(o), device=DEV))
    torch.cuda.synchronize()


def _kernel_bins_eval(fr, n_S, single):
    bufs = fr.debug_buffers()
    n = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    ray_list = _from_ptr(bufs["ray_list"], (n,), torch.int32).cpu().long()
    eb = _from_ptr(bufs["ebins_c" if single else "ebins_f"], (n, n_S + 1), torch.float32).cpu()
    return eb[torch.argsort(ray_list)]


FWD_CASES = [("tetra_nerf", None), ("tetra_nerf_original", None), ("single", None), ("tetra_nerf", 10), ("tetra_nerf", 100),
             ("tetra_nerf", 1000)]


@pytest.mark.parametrize("prec", [3, 2], ids=["bf16x3", "f16w2"])
@pytest.mark.parametrize("cfgname,k", FWD_CASES, ids=[f"{c}-{'random' if k is None else f'k{k}'}" for c, k in FWD_CASES])
def test_forward_against_float64(small_mesh, cfgname, k, prec):
    V, C = small_mesh
    field, params = _field(V, k)
    _, fr, params = _setup(V, C, field, params)
    fr.set_mlp_precision(prec)
    st, oc = _single() if cfgname == "single" else _settings(cfgname)
    o, d = _rays()
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, expected_depth=True)
    S = st.num_samples if st.num_fine_samples == 0 else st.num_samples + st.num_fine_samples + 1
    eb = _kernel_bins_eval(fr, S, st.num_fine_samples == 0)
    torch.cuda.synchronize()
    ref = edo.depth_at_bins(orc.OracleMesh(V, C), field, params, o, d, oc, eb)
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    got = out["expected_depth"].cpu().double()[:, 0]
    want = ref["expected_depth"][:, 0]
    mids = (eb[:, 1:] + eb[:, :-1]) / 2
    span = float(mids.max() - mids.min())
    keep = ref["accumulation"][:, 0] >= A_MIN
    keep |= ~ref["ray_mask"]
    err = ((got - want).abs() / span)[keep]
    print(f"--- {cfgname}, {'random' if k is None else f'k = {k}'}, prec {prec}: max |D - D64| / (t_max - t_min) = {err.max().item():.2e} "
          f"over {int(keep.sum())} rays ({int((~keep).sum())} with A < {A_MIN} excluded)")
    assert got[5].item() == oc.far_plane
    assert err.max().item() <= FWD_BAR[prec]


def _depth_grad(A, R):
    """dL/dD of L = sum_r D_r / R over the rays with A >= A_MIN (the others get 0)"""
    return (A >= A_MIN).to(torch.float64) / R


def _oracle_depth(mesh, V, field, params, o, d, oc, jc, jf, target, gs, dtype, loss, fine=None, gdep=None):
    torch.set_default_dtype(dtype)
    try:
        ot = torch.from_numpy(o).to(dtype).requires_grad_(True)
        dt = torch.from_numpy(d).to(dtype).requires_grad_(True)
        xyz = torch.from_numpy(V).to(dtype).requires_grad_(True)
        f = torch.from_numpy(field).to(dtype).requires_grad_(True)
        p = {k: v.detach().to(dtype).requires_grad_(True) for k, v in params.items()}
        out = edo.render_train_depth(mesh, f, p, ot, dt, xyz, oc, jc, jf, use_gradient_scaling=gs, fine_euclid=fine)
        R = len(o)
        if gdep is None:
            gdep = _depth_grad(out["accumulation"][:, 0].detach(), R)
        L = (out["expected_depth"][:, 0] * gdep.to(dtype)).sum()
        if loss == "rgb+depth":
            L = L + torch.nn.functional.mse_loss(out["rgb"], target.to(dtype)) + 0.05 * out["accumulation"].mean()
        L.backward()
    finally:
        torch.set_default_dtype(torch.float32)
    return out, gdep, {"tetrahedra_field": f.grad, **{n: v.grad for n, v in p.items()}, "origins": ot.grad, "directions": dt.grad,
                       "vertices": xyz.grad}


GRAD_CASES = [("tetra_nerf", False, None, "depth"), ("tetra_nerf", True, None, "rgb+depth"), ("small_uniform", True, None, "depth"),
              ("tetra_nerf", True, 100, "rgb+depth"), ("tetra_nerf", False, 1000, "depth")]


@pytest.mark.parametrize("cfgname,gs,k,loss", GRAD_CASES,
                         ids=[f"{c}-gs{int(g)}-{'random' if k is None else f'k{k}'}-{l}" for c, g, k, l in GRAD_CASES])
def test_gradients_against_float64(small_mesh, cfgname, gs, k, loss):
    V, C = small_mesh
    field, params = _field(V, k)
    st, oc = _settings(cfgname)
    o, d = _rays()
    R = len(o)
    jc, jf, target = _inputs(R, st, 5)
    tr, fr, params = _setup(V, C, field, params)
    mesh = orc.OracleMesh(V, C)
    # the depth loss's weights come from the float64 oracle's accumulation, so that kernel and oracle differentiate the same loss
    ref64, gdep, g64 = _oracle_depth(mesh, V, field, params, o, d, oc, jc, jf, target, gs, torch.float64, loss)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV),
                                        expected_depth=True)
    if loss == "rgb+depth":
        g_rgb = (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
        g_acc = torch.full((R,), 0.05 / R, device=DEV)
    else:
        g_rgb, g_acc = torch.zeros((R, 3), device=DEV), None
    gfield, gp, go, gd, gv = fr.train_backward_saved(state, g_rgb, g_acc, len(V), gs, grad_origins=True, grad_directions=True,
                                                     grad_vertices=True, grad_expected_depth=gdep.float().to(DEV))
    S2 = st.num_samples + st.num_fine_samples + 1
    n, ray_list, eb, _ = _blob_arrays(state, S2)
    torch.cuda.synchronize()
    _, _, g32 = _oracle_depth(mesh, V, field, params, o, d, oc, jc, jf, target, gs, torch.float32, loss, gdep=gdep)
    _, _, gsb = _oracle_depth(mesh, V, field, params, o, d, oc, jc, jf, target, gs, torch.float64, loss, fine=eb[torch.argsort(ray_list)],
                              gdep=gdep)
    e_d = (out["expected_depth"].cpu().double() - ref64["expected_depth"].detach()).abs()[gdep > 0].max().item()
    print(f"--- {cfgname}, gradient scaling {gs}, {'random field' if k is None else f'k = {k}'}, loss on {loss}: "
          f"{int((gdep == 0).sum()) - int((~ref64['ray_mask']).sum())} rays with A < {A_MIN} left out of the depth loss; "
          f"forward max |D - D64| {e_d:.2e}")
    got = {"tetrahedra_field": gfield, **gp, "origins": go, "directions": gd, "vertices": gv}
    failures = []
    for name in got:
        if g64[name] is None or g64[name].abs().max() == 0:  # a loss on D alone does not reach the colour heads: the kernel gives 0
            assert torch.all(got[name] == 0), name
            continue
        _check(name, got[name], g32[name], g64[name], gsb[name], failures)
    assert not failures, failures


def _depth_step(fr, V, st, batch, gs=True):
    o, d, jc, jf = batch
    out, state = fr.train_forward_saved(o, d, st, jc, jf, expected_depth=True)
    g_ed = (out["expected_depth"][:, 0] - 1.0) * 2.0 / len(o)
    res = fr.train_backward_saved(state, torch.zeros_like(out["rgb"]), None, len(V), gs, grad_origins=True, grad_directions=True,
                                  grad_vertices=True, grad_expected_depth=g_ed.contiguous())
    torch.cuda.synchronize()
    return out, res


def test_deterministic_depth_steps(small_mesh, monkeypatch):
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = small_mesh
    field, params = _field(V, 100)
    st, _ = _settings("tetra_nerf")
    o, d = _rays(400, 21)
    jc, jf, _ = _inputs(len(o), st, 7)
    _, fr, _ = _setup(V, C, field, params)
    batch = (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), jc.to(DEV), jf.to(DEV))
    a_out, a = _depth_step(fr, V, st, batch)
    b_out, b = _depth_step(fr, V, st, batch)
    for key in a_out:
        assert torch.equal(a_out[key], b_out[key]), key
    assert torch.equal(a[0], b[0])
    for n in a[1]:
        assert torch.equal(a[1][n], b[1][n]), n
    for x, y in zip(a[2:], b[2:]):
        assert torch.equal(x, y)
    assert a[0].abs().max() > 0 and a[4].abs().max() > 0


@pytest.mark.parametrize("path", ["eval", "train"])
def test_batch_wide_clip_on_transparent_rays(small_mesh, monkeypatch, path):
    """surface_scene at k = 1000: rays that cross the mesh but miss both spheres keep A ~ 1e-20, so D_raw = sum w t / (A + 1e-10) lies far
    below every midpoint and the clip binds.  Their D must be exactly the smallest midpoint of the whole call (the kernel's own bins),
    not the ray's own.  Training (deterministic mode): a depth gradient placed only on those rays must leave every gradient bitwise equal
    to the backward without a depth gradient, since the clip mask zeroes it."""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = small_mesh
    field, params = _field(V, 1000)
    st, _ = _settings("tetra_nerf")
    o, d = _rays()
    R = len(o)
    _, fr, _ = _setup(V, C, field, params)
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    S2 = st.num_samples + st.num_fine_samples + 1
    if path == "eval":
        out = fr.render(ot, dt, st, expected_depth=True)
        eb = _kernel_bins_eval(fr, S2, False)
    else:
        jc, jf, target = _inputs(R, st, 7)
        out, state = fr.train_forward_saved(ot, dt, st, jc.to(DEV), jf.to(DEV), expected_depth=True)
        _, ray_list, eb, _ = _blob_arrays(state, S2)
        eb = eb[torch.argsort(ray_list)]
    torch.cuda.synchronize()
    act = torch.nonzero(out["ray_mask"].cpu()).flatten()
    acc = out["accumulation"].cpu()[act, 0].double()
    D = out["expected_depth"].cpu()[act, 0]
    mids = (eb[:, 1:] + eb[:, :-1]) / 2  # float32, as the kernels form them
    t_min, t_max = mids.min(), mids.max()
    # D_raw <= t_max A / (A + 1e-10): below half of t_min for these rays, so the clip binds with a wide margin
    bare = t_max.double() * acc / (acc + 1e-10) < 0.5 * t_min.double()
    own = mids.min(1).values
    print(f"{path}: {int(bare.sum())} of {len(act)} active rays with a binding clip; batch t_min {t_min.item():.6f}, their own smallest "
          f"midpoints {own[bare].min().item():.6f} ... {own[bare].max().item():.6f}")
    assert int(bare.sum()) >= 10
    assert torch.all(D[bare] == t_min)
    assert torch.any(own[bare] > t_min)  # a per-ray clip would give these rays another value
    if path == "eval":
        return
    g_rgb = (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
    g_acc = torch.full((R,), 0.05 / R, device=DEV)
    kw = dict(grad_origins=True, grad_directions=True, grad_vertices=True)
    ref = fr.train_backward_saved(state, g_rgb, g_acc, len(V), True, **kw)
    g_ed = torch.zeros(R, dtype=torch.float32)
    g_ed[act[bare]] = 1.0 / int(bare.sum())
    got = fr.train_backward_saved(state, g_rgb, g_acc, len(V), True, grad_expected_depth=g_ed.to(DEV), **kw)
    torch.cuda.synchronize()
    assert torch.equal(ref[0], got[0])
    for n in ref[1]:
        assert torch.equal(ref[1][n], got[1][n]), n
    for x, y in zip(ref[2:], got[2:]):
        assert torch.equal(x, y)


def test_opaque_rays_meet_the_analytic_sphere(small_mesh):
    """surface_scene at k = 1000: D of opaque rays lies within one fine bin plus the local tetrahedron size of the first analytic
    ray-sphere crossing.  The field is the truncated distance interpolated linearly on the tetrahedra, so its zero crossing sits within
    about one tetrahedron of the sphere along the normal, i.e. size / cos(incidence) along the ray; rays meeting the sphere at more than
    70 degrees from its normal are left out and counted"""
    from scipy.spatial import Delaunay

    V, C = small_mesh
    field, params = _field(V, 1000)
    _, fr, _ = _setup(V, C, field, params)
    st, _ = _settings("tetra_nerf")
    o, d = syn.camera_rays(2000, seed=5)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, expected_depth=True)
    S2 = st.num_samples + st.num_fine_samples + 1
    eb = _kernel_bins_eval(fr, S2, False).double().numpy()
    torch.cuda.synchronize()
    D = out["expected_depth"].cpu().double().numpy()[:, 0]
    acc = out["accumulation"].cpu().double().numpy()[:, 0]
    act = np.nonzero(out["ray_mask"].cpu().numpy())[0]
    hits = syn.sphere_hits(o, d)[:, :, 0]
    t_hit = np.where(np.isnan(hits), np.inf, hits).min(1)
    first = np.where(np.isnan(hits), np.inf, hits).argmin(1)
    dn_all = d / np.linalg.norm(d, axis=1, keepdims=True)
    ph = o + np.where(np.isfinite(t_hit), t_hit, 0.0)[:, None] * dn_all
    ctr = np.asarray([syn.SURFACE_SPHERES[i][0] for i in first])
    nrm = (ph - ctr) / np.linalg.norm(ph - ctr, axis=1, keepdims=True)
    cosi = np.abs(np.sum(nrm * dn_all, axis=1))
    opaque = (acc[act] > 0.99) & np.isfinite(t_hit[act]) & (cosi[act] >= np.cos(np.deg2rad(70)))
    n_grazing = int(((acc[act] > 0.99) & np.isfinite(t_hit[act])).sum() - opaque.sum())
    rays = act[opaque]
    e = eb[opaque]
    k = np.clip(np.array([np.searchsorted(e[i], D[r]) for i, r in enumerate(rays)]), 1, S2)
    bin_w = e[np.arange(len(rays)), k] - e[np.arange(len(rays)), k - 1]
    dn = d[rays] / np.linalg.norm(d[rays], axis=1, keepdims=True)
    p = o[rays] + t_hit[rays, None] * dn
    tri = Delaunay(V.astype(np.float64))
    simp = tri.simplices[tri.find_simplex(p)]
    X = V.astype(np.float64)[simp]
    size = np.max([np.linalg.norm(X[:, i] - X[:, j], axis=-1) for i in range(4) for j in range(i + 1, 4)], axis=0)
    bound = bin_w + size / cosi[rays]
    excess = np.abs(D[rays] - t_hit[rays]) - bound
    print(f"{len(rays)} opaque rays ({n_grazing} grazing ones left out): max |D - t_hit| {np.abs(D[rays] - t_hit[rays]).max():.3e}, "
          f"max over the bound {excess.max():.3e} (bound: median {np.median(bound):.3e}), max |D - t_hit| / bound "
          f"{(np.abs(D[rays] - t_hit[rays]) / bound).max():.2f}")
    assert len(rays) > 200
    assert excess.max() <= 0


def _model_run(V, C, field, mode, o, d, target_rgb, target_depth, monkeypatch):
    from tetranerf.nerfstudio import model as M

    monkeypatch.setenv("TETRANERF_B200_UNFUSED_TRAIN", "1" if mode == "unfused" else "0")
    cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=64, num_fine_samples=64,
                                 use_biased_sampler=True, use_gradient_scaling=True, depth_loss_mult=0.1)
    m = M.TetrahedraNerf(cfg)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(orc.init_mlp_params(0))
    m.load_state_dict(sd, strict=False)
    m = m.to(DEV).train()
    m.sampler_uniform.train_stratified = False
    m.sampler_pdf.train_stratified = False
    dn = 1.0 + 0.1 * torch.arange(len(o), device=DEV, dtype=torch.float32)[:, None] / len(o)
    out = m(M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV), metadata={"directions_norm": dn}))
    losses = m.get_loss_dict(out, {"image": target_rgb, "depth_image": target_depth})
    (losses["rgb_loss"] + losses["depth_loss"]).backward()
    return out, losses, {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


def test_model_training_paths_agree_with_a_depth_loss(small_mesh, monkeypatch):
    """TetrahedraNerf with depth_loss_mult > 0 and a z-depth target: the fused op and the unfused op sequence (torch autograd through
    DepthRenderer("expected")) agree, as test_gpu_train.test_model_training_path_fused_vs_unfused"""
    V, C = small_mesh
    field, _ = _field(V, None)
    o, d = syn.camera_rays(256, seed=14)
    g = torch.Generator().manual_seed(3)
    target = torch.rand((256, 3), generator=g).to(DEV)
    target_depth = (1.0 + torch.rand((256, 1), generator=g)).to(DEV)
    res = {mode: _model_run(V, C, field, mode, o, d, target, target_depth, monkeypatch) for mode in ("fused", "unfused")}
    (of, lf, gf), (ou, lu, gu) = res["fused"], res["unfused"]
    assert (of["expected_depth"] - ou["expected_depth"]).abs().max().item() < 1e-4
    assert abs(lf["depth_loss"].item() - lu["depth_loss"].item()) <= 1e-4 * lu["depth_loss"].item()
    assert set(gf) == set(gu)
    for n, gg in gu.items():
        a = gf[n]
        rel = ((a - gg).abs().max() / gg.abs().max().clamp_min(1e-30)).item()
        l2 = ((a - gg).norm() / gg.norm().clamp_min(1e-30)).item()
        print(f"  {n:34s} fused vs unfused: max {rel:.2e}  L2 {l2:.2e}")
        assert torch.isfinite(a).all()
        assert rel < 5e-3 and l2 < 1e-3, (n, rel, l2)


@pytest.mark.parametrize("vertices", [False, True], ids=["field-mlp", "vertices"])
def test_depth_only_supervision_learns(small_mesh, monkeypatch, vertices):
    """surface_scene (k = 100) rendered at the truth gives the target depth; a perturbed start (field feature 0 shifted, or the vertices
    moved) trained on the expected depth alone must cut the median depth error of the opaque rays by the stated factor (the median: the
    mean is carried by a few silhouette rays and moves with rounding-level changes of the gradient).  Deterministic mode, so
    that the result repeats run to run (the vertex run is sensitive to the float-atomic order of the default mode)"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    from tetranerf.b200.render import PARAM_ORDER, FusedTrainRenderDepth

    V, C = small_mesh
    field, params = _field(V, 100)
    st, _ = _settings("tetra_nerf")
    tr, fr, params = _setup(V, C, field, params)
    o, d = syn.camera_rays(2048, seed=9)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    with torch.no_grad():
        ref = fr.render(o, d, st, expected_depth=True)
    opaque = ref["accumulation"][:, 0] > 0.99
    target = ref["expected_depth"].clone()
    ps = [params[n].to(DEV).clone().requires_grad_(not vertices) for n in PARAM_ORDER]
    f = torch.from_numpy(field).to(DEV).clone()
    xyz = torch.from_numpy(V).to(DEV).clone()
    g = torch.Generator().manual_seed(0)
    if vertices:
        xyz += (0.01 * torch.randn(xyz.shape, generator=g)).to(DEV)
        tr.load_tetrahedra(xyz, torch.from_numpy(C).to(DEV))
        xyz.requires_grad_(True)
        opt = torch.optim.Adam([xyz], lr=3e-4)
    else:
        f[0] -= 0.1  # moves the zero crossing of the truncated distance, i.e. the surfaces, inwards
        f.requires_grad_(True)
        opt = torch.optim.Adam([f] + ps, lr=2e-3)

    def err():
        with torch.no_grad():
            fr.set_field(f.detach())
            fr.set_weights({n: p.detach() for n, p in zip(PARAM_ORDER, ps)})
            out = fr.render(o, d, st, expected_depth=True)
        return (out["expected_depth"] - target)[opaque].abs().median().item()

    e0 = err()
    for it in range(80 if vertices else 60):
        fr.set_field(f.detach())
        fr.set_weights({n: p.detach() for n, p in zip(PARAM_ORDER, ps)})
        opt.zero_grad()
        extra = (xyz,) if vertices else ()
        _, _, _, ed, _ = FusedTrainRenderDepth.apply(fr, st, False, o, d, None, None, f, *ps, *extra)
        loss = ((ed - target)[opaque] ** 2).mean()
        loss.backward()
        opt.step()
        if vertices:
            with torch.no_grad():
                tr.update_vertices(xyz.detach())
    e1 = err()
    print(f"{'vertices' if vertices else 'field + MLP'}: median |D - D*| on {int(opaque.sum())} opaque rays {e0:.3e} -> {e1:.3e} "
          f"({e0 / e1:.1f}x)")
    assert e0 / e1 > 2.0
