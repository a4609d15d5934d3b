"""GPU: the normal map of the fused render (tn_render's d_normals, DESIGN §4.7) against the float64 oracle (oracle/normals.py).

Per sample, at the kernel's own samples: |grad_kernel - grad_64| <= tol |cof E|_F |q_64| / |det E|, tol = 1e-3 (bf16x3) and 5e-2
(f16w2).  The operand-rounding emulation of the reverse chain (oracle.normals.emulate_grad_pre) puts the maximum of this measure in a
heavy tail that grows with the number of samples (q = g . (F_vk - F_v0) cancels): on the 3000-point mesh 9.0e-5 / 3.7e-3 over 4000
samples, 2.6e-4 / 2.4e-2 over 80,000 (its 99.9th percentile stays at 3-6e-5 / 2-5e-3).  These cases check ~35-140k samples each; an
H100 measured at most 6.0e-4 and 2.4e-2.  Samples with a hidden pre-activation inside the
mask-ambiguity band (kappa = 2^-14 bf16x3, 2^-11 f16w2: the relative precision of the activations) are excluded, counted and bounded.
Pixels: rgb / accumulation / depth / ray_mask equal a plain render's bit for bit; sum w n against the oracle at the kernel's bins;
k_composite_normals' output against the normalised sum of the kernel's own sample normals and weights.
Analytic: on the 45k-point mesh at k = 1000 the opaque rays' normals against the normal of the sphere they hit first."""
import numpy as np
import pytest
import torch

from oracle import normals as onm
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_render import _from_ptr, setup

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = {3: 1e-3, 2: 5e-2}
KAPPA = {3: 2.0**-14, 2: 2.0**-11}
AMB = {3: 0.15, 2: 0.6}  # bound on the excluded share
# unnormalised sum w n against the oracle: 2e-3 (bf16x3), 1e-2 (f16w2); an H100 measured at most 8.0e-4 and 6.0e-3 (both on the
# torch-default network, whose flat weights spread each pixel over many samples near a mask boundary)
PIX = {3: 2e-3, 2: 1e-2}


def _settings(cfgname):
    from tetranerf.b200.render import RenderSettings

    if cfgname == "tetra_nerf":
        return RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    if cfgname == "tetra_nerf_original":
        return RenderSettings.tetra_nerf_original(), orc.RenderConfig.tetra_nerf_original()
    st, oc = RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()  # single pass
    st.num_fine_samples = oc.num_fine_samples = 0
    return st, oc


def _scene(V, k):
    if k is None:
        return syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)
    return syn.surface_scene(V, k, orc.init_mlp_params(0))


def _rays(n):
    o, d = syn.camera_rays(n)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]
    o[17] = [0.5, 0.5, 0.5]
    return o, d


def _kernel_samples(fr, st):
    """(slot -> ray, vi [n_act,S,4], bary [n_act,S,3], ebins [n_act,S+1], out_f, grad [n_act,S,4]) of the last normals render"""
    b = fr.debug_buffers()
    n_act = int(_from_ptr(b["n_active"], (1,), torch.int32)[0])
    single = st.num_fine_samples == 0
    S = st.num_samples if single else st.num_samples + st.num_fine_samples + 1
    ray_list = _from_ptr(b["ray_list"], (n_act,), torch.int32).cpu().long()
    vi = _from_ptr(b["vi_c" if single else "vi_f"], (n_act, S, 4), torch.int32).cpu().numpy()
    bary = _from_ptr(b["bary_c" if single else "bary_f"], (n_act, S, 3), torch.float32).cpu().numpy()
    eb = _from_ptr(b["ebins_c" if single else "ebins_f"], (n_act, S + 1), torch.float32).cpu()
    out_f = _from_ptr(b["out_f"], (n_act, S, 4), torch.float32).cpu()
    grad = _from_ptr(fr.debug_normals_grad(), (n_act, S, 4), torch.float32).cpu().numpy()
    return ray_list, vi, bary, eb, out_f, grad


def _check_samples(V, field, params, vi, bary, grad, prec, label):
    ref = onm.grad_pre(vi.reshape(-1, 4), bary.reshape(-1, 3), V, field, params, kappa=KAPPA[prec])
    g = grad.reshape(-1, 4)
    assert np.all(g[:, 3] == 0.0)
    unmatched = ~ref["matched"]
    assert np.all(g[unmatched, :3] == 0.0), label
    err = onm.error_measure(g[:, :3], ref)
    amb = ref["ambiguous"] & ref["matched"]
    keep = ref["matched"] & ~amb
    rate = amb.sum() / max(ref["matched"].sum(), 1)
    print(f"{label}: {keep.sum()} samples, max err {err[keep].max():.2e} (bar {TOL[prec]:.0e}), median {np.median(err[keep]):.2e}, "
          f"mask-ambiguous {amb.sum()} ({100 * rate:.3f} %)")
    assert keep.sum() > 1000, label
    assert rate < AMB[prec], (label, rate)
    assert err[keep].max() <= TOL[prec], (label, err[keep].max())
    return ref


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("case", [("tetra_nerf", None), ("tetra_nerf", 10), ("tetra_nerf", 100), ("tetra_nerf", 1000),
                                  ("tetra_nerf_original", 100), ("single", 100)])
def test_normals_per_sample_and_pixels(small_mesh, case, prec):
    cfgname, k = case
    V, C = small_mesh
    field, params = _scene(V, k)
    st, oc = _settings(cfgname)
    tr, fr, _, _ = setup(V, C, prec=prec, field=field, params=params)
    o, d = _rays(300)
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    plain = fr.render(ot, dt, st)
    plain = {kk: v.clone() for kk, v in plain.items()}
    out = fr.render(ot, dt, st, normals=True)
    tr.synchronize()
    label = f"{cfgname} k={k} prec={prec}"
    for key in ("rgb", "accumulation", "depth", "ray_mask"):  # the same bits as a plain render
        assert torch.equal(plain[key], out[key]), (label, key)
    assert set(out) == {"rgb", "accumulation", "depth", "ray_mask", "normals"}
    ray_list, vi, bary, eb, out_f, grad = _kernel_samples(fr, st)
    ref = _check_samples(V, field, params, vi, bary, grad, prec, label)
    # ---- pixels: sum w n at the kernel's bins against the oracle ----
    N = out["normals"].cpu().numpy()
    empty = ~out["ray_mask"].cpu().numpy()
    assert np.all(N[empty] == 0.0)
    back = torch.argsort(ray_list)
    mesh = orc.OracleMesh(V, C)
    at = orc.render(mesh, torch.from_numpy(field), params, o, d, oc, return_aux=True, fine_euclid=eb[back])["aux"]
    vi_ref = at["matched"]["vertex_indices"]
    flipped = (vi[back.numpy()] != vi_ref).any(-1)
    ok_rays = ~flipped.any(-1)
    w_ref = at["weights"][..., 0].numpy().astype(np.float64)
    n_ref = onm.sample_normals(onm.grad_pre(vi_ref.reshape(-1, 4), at["matched"]["barycentric_coordinates"].reshape(-1, 3), V, field,
                                            params)["grad"]).reshape(*vi_ref.shape[:2], 3)
    sum_ref, unit_ref = onm.composite(w_ref, n_ref)
    # the kernel's unnormalised sum from its own per-sample gradients and weights (its pixel = that sum normalised)
    n_k = onm.sample_normals(grad[..., :3].astype(np.float64))[back.numpy()]
    rays = np.nonzero(~empty)[0]
    sum_k, unit_k = onm.composite(w_ref, n_k)
    e_sum = np.abs(sum_k - sum_ref).max(-1)[ok_rays]
    print(f"{label}: pixel |sum w n - oracle| max {e_sum.max():.2e} (bar {PIX[prec]:.0e}) over {ok_rays.sum()} rays, "
          f"{(~ok_rays).sum()} with flipped samples excluded")
    assert ok_rays.mean() > 0.8
    assert e_sum.max() <= PIX[prec], (label, e_sum.max())
    # k_composite_normals itself: its pixels against the normalised sum of the kernel's own sample normals, weighted with the
    # weights of the kernel's own densities and bins (get_weights in float64; k_composite_normals forms them in fp32)
    x = (eb[:, 1:] - eb[:, :-1]).double().numpy() * out_f[..., 0].double().numpy()
    w_k = (1.0 - np.exp(-x)) * np.exp(-np.concatenate([np.zeros((len(x), 1)), np.cumsum(x, -1)[:, :-1]], -1))
    s_own, u_own = onm.composite(w_k, onm.sample_normals(grad[..., :3].astype(np.float64)))
    N_slot = N[ray_list.numpy()]
    mag = np.linalg.norm(s_own, axis=-1)
    live = mag > 1e-3
    dev_own = np.linalg.norm(N_slot - u_own, axis=-1)[live]
    print(f"{label}: composite vs its own samples: max |N - unit(sum w n)| {dev_own.max():.2e} over {live.sum()} rays "
          f"(max x |sum w n| {(dev_own * mag[live]).max():.2e})")
    assert np.all(dev_own <= 2e-5 / mag[live] + 1e-6), (label, dev_own.max())
    # the kernel's pixel: its normalised sum (weights of k_composite = the oracle's within fp32 rounding)
    Nk = N[rays]
    strong = np.linalg.norm(sum_ref, axis=-1) > 0.1
    sel = ok_rays & strong
    cos = np.sum(Nk[sel] * unit_ref[sel], -1)
    print(f"{label}: pixel normals vs oracle: min cos {cos.min():.6f} over {sel.sum()} rays with |sum w n| > 0.1")
    assert cos.min() > 1 - 10 * PIX[prec]
    assert np.allclose(np.linalg.norm(N[~empty], axis=-1)[np.linalg.norm(sum_ref, axis=-1) > 1e-6], 1.0, atol=1e-5)


def test_normals_of_analytic_spheres():
    """45k-point mesh, surface_scene at k = 1000: opaque rays whose first analytic hit is on one sphere; rendered normal vs the sphere's"""
    V, C = syn.delaunay_mesh(45000, seed=0)
    field, params = syn.surface_scene(V, 1000, orc.init_mlp_params(0))
    st, _ = _settings("tetra_nerf")
    o, d = syn.camera_rays(4096)
    for prec in (2, 3):
        tr, fr, _, _ = setup(V, C, prec=prec, field=field, params=params)
        out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, normals=True)
        tr.synchronize()
        acc = out["accumulation"][:, 0].cpu().numpy()
        N = out["normals"].cpu().numpy().astype(np.float64)
        hits = syn.sphere_hits(o, d)
        entry = hits[:, :, 0]
        first = np.where(np.isfinite(entry), entry, np.inf)
        s = np.argmin(first, 1)
        t = first[np.arange(len(o)), s]
        sel = (acc > 0.999) & np.isfinite(t) & (t > 0)
        p = o.astype(np.float64) + t[:, None] * (d / np.linalg.norm(d, axis=1, keepdims=True))
        centres = np.array([c for c, _ in syn.SURFACE_SPHERES])
        n_true = p - centres[s]
        n_true /= np.maximum(np.linalg.norm(n_true, axis=1, keepdims=True), 1e-300)  # (rays that miss both spheres are not selected)
        dot = np.sum(N[sel] * n_true[sel], -1)
        ang = np.arccos(np.clip(dot, -1, 1))
        print(f"prec={prec}: {sel.sum()} opaque rays on a sphere: dot > 0 for {100 * np.mean(dot > 0):.2f} %, angle median "
              f"{np.median(ang):.4f} p90 {np.percentile(ang, 90):.4f} p99 {np.percentile(ang, 99):.4f} max {ang.max():.4f} rad")
        assert sel.sum() > 500
        assert np.mean(dot > 0) >= 0.99
        assert np.median(ang) <= 0.25


def test_normals_render_is_deterministic_and_isolated(small_mesh):
    V, C = small_mesh
    field, params = _scene(V, 100)
    st, _ = _settings("tetra_nerf")
    tr, fr, _, _ = setup(V, C, prec=2, field=field, params=params)
    o, d = _rays(300)
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    a = {k: v.clone() for k, v in fr.render(ot, dt, st, normals=True).items()}
    b = fr.render(ot, dt, st, normals=True)
    tr.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # the fused pixel gather has no room for normals
    buf = torch.zeros((300, 6), device=DEV)
    from tetranerf.b200.render import _lib

    import ctypes as C_

    arr = (C_.c_void_p * 1)(buf.data_ptr())
    assert _lib.tn_render_set_gather(tr.handle, 1, 0, arr, 300) == 0
    with pytest.raises(RuntimeError, match="gather"):
        fr.render(ot, dt, st, normals=True)
    assert _lib.tn_render_set_gather(tr.handle, 0, 0, None, 0) == 0
    fr.render(ot, dt, st, normals=True)
    tr.synchronize()


def test_normals_render_between_training_forward_and_backward(small_mesh, monkeypatch):
    """in deterministic mode a normals render between a saved training forward and its backward leaves the gradients unchanged"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = small_mesh
    field, params = _scene(V, 100)
    st, _ = _settings("tetra_nerf")
    tr, fr, _, _ = setup(V, C, prec=3, field=field, params=params)
    o, d = _rays(256)
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    g = torch.Generator(device="cpu").manual_seed(4)
    jc = torch.rand((256, st.num_samples + 1), generator=g).to(DEV)
    jf = torch.rand((256, st.num_fine_samples + 1), generator=g).to(DEV)
    grad_rgb = torch.randn((256, 3), generator=g).to(DEV)

    def run(with_normals):
        out, state = fr.train_forward_saved(ot, dt, st, jc, jf)
        if with_normals:
            fr.render(ot, dt, st, normals=True)
        gf, gp = fr.train_backward_saved(state, grad_rgb, None, len(V))
        tr.synchronize()
        return [gf.clone()] + [gp[n].clone() for n in sorted(gp)]

    base, mixed = run(False), run(True)
    for x, y in zip(base, mixed):
        assert torch.equal(x, y)


def test_model_render_normals(small_mesh):
    """TetrahedraNerf(render_normals=True) in eval returns the renderer's normals; with the flag off the outputs keep today's keys"""
    from test_gpu_model import build_model
    from tetranerf.nerfstudio import model as M

    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    o, d = _rays(200)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    m, params = build_model(V, C, field, num_samples=128, num_fine_samples=128, use_biased_sampler=True)
    m.eval()
    with torch.no_grad():
        plain = m(bundle)
    assert set(plain) == {"rgb", "accumulation", "depth", "ray_mask"}
    m.config.render_normals = True
    with torch.no_grad():
        out = m(bundle)
    assert set(out) == {"rgb", "accumulation", "depth", "ray_mask", "normals"}
    st, _ = _settings("tetra_nerf")
    tr, fr, _, _ = setup(V, C, prec=2, field=field, params=params)
    want = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, normals=True)
    for k in out:
        assert torch.equal(out[k], want[k]), k
    m.train()  # training ignores the flag
    out_t = m(bundle)
    assert "normals" not in out_t
