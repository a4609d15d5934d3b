"""GPU: gradients of the fused training step at the ray origins and directions (tn_render_train_backward_saved, DESIGN §4.8) against
float64 autograd of oracle/ray_grads.render_train_rays, with the bars of test_gpu_train.py: (A) at the kernel's own fine bins and (B) end to
end, max |g - g64| <= max(2e-4, 6 max |g_torch_f32 - g64|) in units of the largest entry.  Also: dL/dx per sample against float64 at the
kernel's positions, isolation of the other outputs and gradients, determinism, saved state, the autograd op, and recovery of a perturbed
camera pose through FusedTrainRender."""
import numpy as np
import pytest
import torch

from oracle import normals as nrm
from oracle import oracle as orc
from oracle import ray_grads as rg
from tetranerf.b200 import synthetic as syn
from test_gpu_train import DEV, _check, _from_ptr, _setup

pytestmark = pytest.mark.gpu
# per-sample dL/dx: max over samples of |g - g64| / (the largest |cof E| |(|dL/df| |F_vk - F_v0|)_k| / |det E| on the sample's ray)
# (_sample_error): at most 1.1e-2 measured on an H100 (surface scene, k = 1000), 7.2e-3 on the random fields
SAMPLE_BAR = 2e-2


def _settings(cfgname):
    from tetranerf.b200.render import RenderSettings

    if cfgname == "tetra_nerf":
        return RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    if cfgname == "tetra_nerf_original":
        return RenderSettings.tetra_nerf_original(), orc.RenderConfig.tetra_nerf_original()
    return RenderSettings(num_samples=48, num_fine_samples=33), orc.RenderConfig(num_samples=48, num_fine_samples=33)


def _inputs(R, st, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((R, st.num_samples + 1), generator=g), torch.rand((R, st.num_fine_samples + 1), generator=g), torch.rand((R, 3), generator=g)


def _blob_arrays(state, S2):
    """n_active, ray_list, fine bins and matched vertices of a saved state (the layout of saved_layout in tn_render.cu)"""
    R, base = state.R, state.blob.data_ptr()
    off = [256]

    def take(nbytes):
        p = base + off[0]
        off[0] += (nbytes + 255) // 256 * 256
        return p

    p_n, p_list, p_eb = take(16), take(4 * R), take(4 * R * (S2 + 1))
    take(4 * R * (S2 + 1))
    p_vi = take(16 * R * S2)
    n = int(_from_ptr(p_n, (1,), torch.int32)[0])
    ray_list = _from_ptr(p_list, (n,), torch.int32).cpu().long()
    eb = _from_ptr(p_eb, (n, S2 + 1), torch.float32).cpu()
    vi = _from_ptr(p_vi, (n, S2, 4), torch.int32).cpu()
    return n, ray_list, eb, vi


def _loss_grads(out, target, R):
    return (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous(), torch.full((R,), 0.05 / R, device=DEV)


def _oracle(mesh, field, params, o, d, oc, jc, jf, target, gs, dtype, fine=None):
    torch.set_default_dtype(dtype)
    try:
        ot = torch.from_numpy(o).to(dtype).requires_grad_(True)
        dt = torch.from_numpy(d).to(dtype).requires_grad_(True)
        f = torch.from_numpy(field).to(dtype)
        p = {k: v.detach().to(dtype) for k, v in params.items()}
        out = rg.render_train_rays(mesh, f, p, ot, dt, oc, jc, jf, use_gradient_scaling=gs, fine_euclid=fine)
        loss = torch.nn.functional.mse_loss(out["rgb"], target.to(dtype)) + 0.05 * out["accumulation"].mean()
        loss.backward()
    finally:
        torch.set_default_dtype(torch.float32)
    return out, ot.grad, dt.grad


def _sample_error(gx, sol, vi, g, field):
    """per-sample |dL/dx - ref| / (|cof E| |(|g| |F_vk - F_v0|)_k| / |det E|): the error relative to what a relative error of the
    feature gradient g can become through q and the solve (q itself cancels, so a bound by |q| as for the normals does not hold here);
    -> (measure, bound)"""
    F = np.asarray(field, dtype=np.float64).T
    v = np.where(vi[:, :1] >= 0, vi, 0)
    gn = np.linalg.norm(g, axis=-1)
    a = np.stack([gn * np.linalg.norm(F[v[:, k]] - F[v[:, 0]], axis=-1) for k in (1, 2, 3)], -1)
    bound = np.linalg.norm(sol["cof"], axis=(-2, -1)) * np.linalg.norm(a, axis=-1) / np.where(sol["det"] != 0, np.abs(sol["det"]), 1.0)
    bound = np.where((vi[:, 0] >= 0) & (sol["det"] != 0), bound, 0.0)
    diff = np.linalg.norm(np.asarray(gx, dtype=np.float64) - sol["grad"], axis=-1)
    return diff / np.where(bound > 0, bound, 1.0), bound


CASES = [("tetra_nerf", False, None), ("tetra_nerf", True, None), ("small_uniform", False, None), ("tetra_nerf_original", True, None),
         ("tetra_nerf", True, 100), ("tetra_nerf", True, 1000)]


@pytest.mark.parametrize("cfgname,gs,k", CASES, ids=[f"{c}-gs{int(g)}-{'random' if k is None else f'k{k}'}" for c, g, k in CASES])
def test_ray_gradients_against_float64(small_mesh, cfgname, gs, k):
    """k = None: the random field; k = 100 / 1000: synthetic.surface_scene (opaque spheres).  The torch-default network throughout."""
    V, C = small_mesh
    field, params = (syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)) if k is None else syn.surface_scene(V, k, orc.init_mlp_params(0))
    st, oc = _settings(cfgname)
    o, d = syn.camera_rays(300, seed=11)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    R = len(o)
    jc, jf, target = _inputs(R, st, 5)
    tr, fr, params = _setup(V, C, field, params)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    g_rgb, g_acc = _loss_grads(out, target, R)
    _, _, go, gd = fr.train_backward_saved(state, g_rgb, g_acc, len(V), gs, grad_origins=True, grad_directions=True)
    S2 = st.num_samples + st.num_fine_samples + 1
    n, ray_list, eb, vi_k = _blob_arrays(state, S2)
    gx = _from_ptr(fr.debug_ray_grads(), (n, S2, 4), torch.float32).cpu()[..., :3]
    torch.cuda.synchronize()
    assert torch.all(go[5] == 0) and torch.all(gd[5] == 0)
    mesh = orc.OracleMesh(V, C)
    _, go32, gd32 = _oracle(mesh, field, params, o, d, oc, jc, jf, target, gs, torch.float32)
    _, go64, gd64 = _oracle(mesh, field, params, o, d, oc, jc, jf, target, gs, torch.float64)
    order = torch.argsort(ray_list)  # slot order -> order of the non-empty rays
    ref, gosb, gdsb = _oracle(mesh, field, params, o, d, oc, jc, jf, target, gs, torch.float64, fine=eb[order])
    print(f"--- {cfgname}, gradient scaling {gs}, {'random field' if k is None else f'surface scene k = {k}'}")
    failures = []
    _check("grad_origins", go, go32, go64, gosb, failures)
    _check("grad_directions", gd, gd32, gd64, gdsb, failures)
    # per sample, at the kernel's positions and matched tetrahedra
    vi_o = torch.as_tensor(ref["aux"]["matched"]["vertex_indices"]).reshape(-1, 4)
    vi_k = vi_k[order].reshape(-1, 4).long()
    same = torch.all(vi_o == vi_k, -1).numpy()
    assert same.mean() > 0.999, same.mean()
    g_f = ref["aux"]["features"].grad.reshape(-1, 64).numpy()
    sol = nrm.solve(vi_o.numpy(), g_f, field, V)
    want = ref["aux"]["positions"].grad.reshape(-1, 3).numpy()
    assert np.allclose(sol["grad"], want, rtol=1e-6, atol=1e-9 * np.abs(want).max())  # the oracle's E^-T q is autograd's dL/dx
    meas, bound = _sample_error(gx[order].reshape(-1, 3).numpy(), sol, vi_o.numpy(), g_f, field)
    # the same error relative to the largest bound on the sample's ray: what the sample's error does to the ray's sum
    ray_bound = np.repeat(bound.reshape(n, S2).max(-1), S2)
    diff = meas * bound
    per_ray = (diff / np.where(ray_bound > 0, ray_bound, 1.0))[same]
    meas = meas[same & (bound > 0)]
    print(f"  per-sample dL/dx: {len(meas)} samples, own bound: 99.9th percentile {np.quantile(meas, 0.999):.2e}, max {meas.max():.2e};"
          f"  ray's bound: 99.9th percentile {np.quantile(per_ray, 0.999):.2e}, max {per_ray.max():.2e}")
    assert not failures, failures
    assert per_ray.max() <= SAMPLE_BAR


def _scene(small_mesh, R=400, seed=21):
    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    st, _ = _settings("tetra_nerf")
    o, d = syn.camera_rays(R, seed=seed)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]
    jc, jf, target = _inputs(R, st, 7)
    return V, C, field, st, (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), jc.to(DEV), jf.to(DEV), target.to(DEV))


def _step(fr, st, batch, nv, rays=(True, True), gs=True):
    o, d, jc, jf, target = batch
    out, state = fr.train_forward_saved(o, d, st, jc, jf)
    g_rgb, g_acc = _loss_grads(out, target, len(o))
    if rays == (False, False):
        gf, gp = fr.train_backward_saved(state, g_rgb, g_acc, nv, gs)
        go = gd = None
    else:
        gf, gp, go, gd = fr.train_backward_saved(state, g_rgb, g_acc, nv, gs, grad_origins=rays[0], grad_directions=rays[1])
    torch.cuda.synchronize()
    return out, gf, gp, go, gd


@pytest.mark.parametrize("det", [True, False], ids=["deterministic", "default"])
def test_other_outputs_and_gradients_unchanged(small_mesh, monkeypatch, det):
    """rgb / accumulation / depth / mask and the field and MLP gradients with and without the ray gradients: bitwise in deterministic
    mode; in the default mode the pixels are bitwise and the gradients within the run-to-run spread of its float atomics (1e-5)"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1" if det else "0")
    V, C, field, st, batch = _scene(small_mesh)
    _, fr, _ = _setup(V, C, field)
    a = _step(fr, st, batch, len(V), rays=(False, False))
    b = _step(fr, st, batch, len(V))
    for key in ("rgb", "accumulation", "depth", "ray_mask"):
        assert torch.equal(a[0][key], b[0][key]), key
    for name, x, y in [("tetrahedra_field", a[1], b[1])] + [(n, a[2][n], b[2][n]) for n in a[2]]:
        if det:
            assert torch.equal(x, y), name
        else:
            assert (x - y).abs().max().item() <= 1e-5 * x.abs().max().item(), name


def test_deterministic_ray_gradients(small_mesh, monkeypatch):
    """deterministic mode: two runs give bitwise-equal ray gradients; the empty ray gets exactly 0; asking for one of the two gives that
    one, the same bits, and None for the other"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C, field, st, batch = _scene(small_mesh)
    _, fr, _ = _setup(V, C, field)
    _, _, _, go1, gd1 = _step(fr, st, batch, len(V))
    _, _, _, go2, gd2 = _step(fr, st, batch, len(V))
    assert torch.equal(go1, go2) and torch.equal(gd1, gd2)
    assert torch.all(go1[5] == 0) and torch.all(gd1[5] == 0)
    assert go1.abs().max() > 0 and gd1.abs().max() > 0
    _, _, _, go, gd = _step(fr, st, batch, len(V), rays=(True, False))
    assert gd is None and torch.equal(go, go1)
    _, _, _, go, gd = _step(fr, st, batch, len(V), rays=(False, True))
    assert go is None and torch.equal(gd, gd1)


def test_default_mode_origins_are_reproducible(small_mesh, monkeypatch):
    """default mode: dL/do depends only on the per-tile dX rows and a fixed-order sum, so it is bitwise reproducible as well"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "0")
    V, C, field, st, batch = _scene(small_mesh)
    _, fr, _ = _setup(V, C, field)
    _, _, _, go1, gd1 = _step(fr, st, batch, len(V))
    _, _, _, go2, gd2 = _step(fr, st, batch, len(V))
    assert torch.equal(go1, go2)
    assert (gd1 - gd2).abs().max().item() <= 1e-5 * gd1.abs().max().item()


def test_saved_state_reverse_order_and_mesh_reload(small_mesh, monkeypatch):
    """two forwards, then their backwards in reverse order: bitwise the separate runs; load_tetrahedra between a forward and its backward
    makes the ray gradients raise (they read the mesh positions)"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C, field, st, a = _scene(small_mesh, 400, 21)
    _, _, _, _, b = _scene(small_mesh, 250, 22)
    tr, fr, _ = _setup(V, C, field)
    ra = _step(fr, st, a, len(V))
    rb = _step(fr, st, b, len(V))
    outs = []
    for batch in (a, b):
        o, d, jc, jf, target = batch
        out, state = fr.train_forward_saved(o, d, st, jc, jf)
        outs.append((out, state, target))
    res = {}
    for key, (out, state, target) in reversed(list(zip("ab", outs))):
        g_rgb, g_acc = _loss_grads(out, target, state.R)
        res[key] = fr.train_backward_saved(state, g_rgb, g_acc, len(V), True, grad_origins=True, grad_directions=True)
    torch.cuda.synchronize()
    for key, sep in (("a", ra), ("b", rb)):
        assert torch.equal(res[key][2], sep[3]) and torch.equal(res[key][3], sep[4]), key
        assert torch.equal(res[key][0], sep[1]), key
    o, d, jc, jf, target = a
    out, state = fr.train_forward_saved(o, d, st, jc, jf)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    g_rgb, g_acc = _loss_grads(out, target, state.R)
    with pytest.raises(RuntimeError, match="tn_load_tetrahedra"):
        fr.train_backward_saved(state, g_rgb, g_acc, len(V), True, grad_origins=True)
    torch.cuda.synchronize()


def test_autograd_op_returns_ray_gradients(small_mesh, monkeypatch):
    """FusedTrainRender: origins / directions that require grad get the gradients of train_backward_saved; rays that do not require
    grad get none"""
    from tetranerf.b200.render import PARAM_ORDER, FusedTrainRender

    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C, field, st, batch = _scene(small_mesh)
    _, fr, params = _setup(V, C, field)
    f = torch.from_numpy(field).to(DEV)
    ps = [params[n].to(DEV) for n in PARAM_ORDER]
    _, _, _, go, gd = _step(fr, st, batch, len(V))
    o, d, jc, jf, target = batch
    for want in ((True, True), (False, True)):
        ot, dt = o.clone().requires_grad_(want[0]), d.clone().requires_grad_(want[1])
        rgb, acc, _, _ = FusedTrainRender.apply(fr, st, True, ot, dt, jc, jf, f, *ps)
        (torch.nn.functional.mse_loss(rgb, target) + 0.05 * acc.mean()).backward()
        # (torch's MSE backward may round dL/drgb differently from _loss_grads: equal to rounding)
        assert (dt.grad - gd).abs().max().item() <= 1e-5 * gd.abs().max().item()
        if want[0]:
            assert (ot.grad - go).abs().max().item() <= 1e-5 * go.abs().max().item()
        else:
            assert ot.grad is None


def _rotation(w):
    K = torch.zeros((3, 3), dtype=w.dtype, device=w.device)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -w[2], w[1], w[2], -w[0], -w[1], w[0]
    return torch.linalg.matrix_exp(K)


class _PoseCorrection(torch.nn.Module):
    """a per-camera SE(3) correction, as nerfstudio's camera optimizer (SO3xR3) applies it: o' = o + t, d' = R(w) d"""

    def __init__(self, w0, t0):
        super().__init__()
        self.w = torch.nn.Parameter(w0.clone())
        self.t = torch.nn.Parameter(t0.clone())

    def forward(self, o, d):
        return (o + self.t).contiguous(), (d @ _rotation(self.w).T).contiguous()


def test_pose_recovery_through_the_fused_op(small_mesh):
    """surface_scene (k = 100), a 48 x 48 pinhole camera, a target rendered at the true pose.  A pose correction starting 1 % of the
    camera distance and 0.5 degrees off, trained through FusedTrainRender with eval bins (field and MLP frozen), must shrink the
    translation and rotation errors"""
    from tetranerf.b200.render import PARAM_ORDER, FusedTrainRender

    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    st, _ = _settings("tetra_nerf")
    _, fr, params = _setup(V, C, field, params)
    f = torch.from_numpy(field).to(DEV)
    ps = [params[n].to(DEV) for n in PARAM_ORDER]
    n = 48
    u = torch.linspace(-0.2, 0.2, n, device=DEV)
    uu, vv = torch.meshgrid(u, u, indexing="xy")
    dirs = torch.stack([uu.reshape(-1), torch.ones(n * n, device=DEV), vv.reshape(-1)], -1)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    cam = torch.tensor([0.5, -1.5, 0.5], device=DEV)
    origins = cam.expand(n * n, 3)

    def render(o, d):
        rgb, acc, _, _ = FusedTrainRender.apply(fr, st, False, o, d, None, None, f, *ps)
        return rgb

    with torch.no_grad():
        target = render(origins.contiguous(), dirs.contiguous()).clone()
    dist = cam.norm().item()
    g = torch.Generator().manual_seed(0)
    t_err = torch.randn(3, generator=g)
    t_err = (0.01 * dist * t_err / t_err.norm()).to(DEV)
    w_err = torch.randn(3, generator=g)
    w_err = (np.deg2rad(0.5) * w_err / w_err.norm()).to(DEV)
    pose = _PoseCorrection(w_err, t_err)
    opt = torch.optim.Adam(pose.parameters(), lr=1e-3)
    e_t0, e_w0 = pose.t.norm().item(), pose.w.norm().item()
    for it in range(150):
        opt.zero_grad()
        o, d = pose(origins, dirs)
        loss = torch.nn.functional.mse_loss(render(o, d), target)
        loss.backward()
        opt.step()
        if it % 30 == 0:
            print(f"  step {it}: loss {loss.item():.3e}  |t err| {pose.t.norm().item():.2e}  |w err| {pose.w.norm().item():.2e}")
    e_t, e_w = pose.t.norm().item(), pose.w.norm().item()
    print(f"translation error {e_t0:.3e} -> {e_t:.3e} ({e_t0 / e_t:.1f}x), rotation error {e_w0:.3e} -> {e_w:.3e} ({e_w0 / e_w:.1f}x)")
    assert e_t0 / e_t > 2.0 and e_w0 / e_w > 2.0
