"""GPU: the distortion loss of the fused training step (DESIGN §4.11) against the float64 oracle (oracle/distortion.py).
  * forward: d per ray (tn_render_train_distortion) at the kernel's own fine bins against float64;
  * gradients of L = sum_r d_r / R_active, alone and with an rgb / accumulation loss and an expected-depth loss, to the field, the twelve
    MLP tensors, origins / directions and vertex positions, (A) at the kernel's bins and (B) end to end;
  * no regression: a backward without a distortion gradient, and the old entry point, give the same bits;
  * determinism, the settings edges of test_gpu_settings_edges.py, errors, the model's fused and unfused training paths, and that
    distortion-only steps concentrate the weights of a hazy scene.
Bars, as test_gpu_train.py derives its own: the truth is float64 autograd through the oracle; torch's own float32 run of the same oracle
differs from it by a noise floor (sums over ~10^5 samples with cancelling terms), so per tensor, in units of its largest entry,
max |g_kernel - g_f64| <= max(2e-4, 6 x max |g_torch_f32 - g_f64|), both at the kernel's own bins (A) and end to end (B).  The forward
d is held to the same rule with d in place of g: max |d - d64| / D <= max(2e-4, 6 x max |d_torch_f32 - d64| / D), D = max(max d64,
D_UNIT_MIN), with d_torch_f32 the oracle in float32 at the kernel's bins.  GradientScaler changes only the backward, so the forward runs once per setting."""
import numpy as np
import pytest
import torch

from oracle import distortion as dso
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _deterministic
from test_gpu_expected_depth import A_MIN, _depth_grad
from test_gpu_ray_grads import _inputs, _settings
from test_gpu_settings_edges import CASES as EDGE_CASES
from test_gpu_settings_edges import _empty_batch, _s2_max
from test_gpu_settings_edges import _settings as _edge_settings
from test_gpu_train import DEV, GRAD_TOL, _check, _from_ptr, _setup
from tetranerf.b200.render import _lib

pytestmark = pytest.mark.gpu
# the forward bar's unit is the largest d, or this when every ray is almost transparent (cap4's truncated rays: d <= 6e-6, as d is at most
# about A^2 for weights summing to A); an error of 1e-9 on such a loss is far below anything a training step resolves
D_UNIT_MIN = 1e-3
_MESH = {}


def _mesh(V, C):
    if "small" not in _MESH:
        _MESH["small"] = orc.OracleMesh(V, C)
    return _MESH["small"]


def _field(V, k):
    return (syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)) if k is None else syn.surface_scene(V, k, orc.init_mlp_params(0))


def _rays(R=300, seed=11):
    o, d = syn.camera_rays(R, seed=seed)
    if R >= 8:
        o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    return o, d


def _blob(state, S2):
    """n_active, ray_list, fine bins, spacing bins and (sigma, rgb) per sample of a saved state (saved_layout in tn_render.cu)"""
    R, base = state.R, state.blob.data_ptr()
    off = [256]

    def take(nbytes):
        p = base + off[0]
        off[0] += (nbytes + 255) // 256 * 256
        return p

    p_n, p_list, p_eb, p_sb = take(16), take(4 * R), take(4 * R * (S2 + 1)), take(4 * R * (S2 + 1))
    take(16 * R * S2)
    take(12 * R * S2)
    p_out = take(16 * R * S2)
    n = int(_from_ptr(p_n, (1,), torch.int32)[0])
    ray_list = _from_ptr(p_list, (n,), torch.int32).long()
    eb = _from_ptr(p_eb, (n, S2 + 1), torch.float32)
    sb = _from_ptr(p_sb, (n, S2 + 1), torch.float32)
    out = _from_ptr(p_out, (n, S2, 4), torch.float32)
    return n, ray_list, eb, sb, out


def _ray_order(state, S2):
    """the kernel's fine bins and spacing bins in the ray order of the non-empty rays (the oracle's order), on the CPU"""
    _, ray_list, eb, sb, _ = _blob(state, S2)
    order = torch.argsort(ray_list.cpu())
    return eb.cpu()[order], sb.cpu()[order]


def _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, gs, dtype, loss, fine=None, sbins=None, gdep=None, cdist=None):
    """float64 / float32 autograd of the loss through oracle.render_train_distortion -> (outputs, dL/dD used, gradients); the distortion
    term is sum_r d_r / R_active, or sum_r cdist_r d_r"""
    torch.set_default_dtype(dtype)
    try:
        ot = torch.from_numpy(o).to(dtype).requires_grad_(True)
        dt = torch.from_numpy(d).to(dtype).requires_grad_(True)
        xyz = torch.from_numpy(V).to(dtype).requires_grad_(True)
        f = torch.from_numpy(field).to(dtype).requires_grad_(True)
        p = {k: v.detach().to(dtype).requires_grad_(True) for k, v in params.items()}
        out = dso.render_train_distortion(mesh, f, p, ot, dt, xyz, oc, jc, jf, use_gradient_scaling=gs, fine_euclid=fine, fine_sbins=sbins)
        R = len(o)
        n_act = max(1, int(out["ray_mask"].sum()))
        if "dist" in loss:
            L = out["distortion"].sum() / n_act if cdist is None else (out["distortion"][:, 0] * cdist.to(dtype)).sum()
        else:
            L = 0.0
        if "rgb" in loss:
            L = L + torch.nn.functional.mse_loss(out["rgb"], target.to(dtype)) + 0.05 * out["accumulation"].mean()
        if "depth" in loss:
            if gdep is None:
                gdep = _depth_grad(out["accumulation"][:, 0].detach().double(), R)
            L = L + (out["expected_depth"][:, 0] * gdep.to(dtype)).sum()
        L.backward()
    finally:
        torch.set_default_dtype(torch.float32)
    return out, gdep, {"tetrahedra_field": f.grad, **{n: v.grad for n, v in p.items()}, "origins": ot.grad, "directions": dt.grad,
                       "vertices": xyz.grad}


def _kernel_step(fr, st, V, o, d, jc, jf, target, gs, loss, gdep=None, cdist=None):
    """forward (+ expected depth when the loss has it), d, and the backward of the same loss -> (outputs, d, state, gradients)"""
    R = len(o)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV),
                                        expected_depth="depth" in loss)
    dist = fr.train_distortion(state)
    n_act = max(1, int(out["ray_mask"].sum()))
    g_dist = (torch.full((R,), 1.0 / n_act, device=DEV) if cdist is None else cdist.float().to(DEV)) if "dist" in loss else None
    if "rgb" in loss:
        g_rgb = (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
        g_acc = torch.full((R,), 0.05 / R, device=DEV)
    else:
        g_rgb, g_acc = torch.zeros((R, 3), device=DEV), None
    g_ed = gdep.float().to(DEV) if "depth" in loss else None
    gfield, gp, go, gd, gv = fr.train_backward_saved(state, g_rgb, g_acc, len(V), gs, grad_origins=True, grad_directions=True,
                                                     grad_vertices=True, grad_expected_depth=g_ed, grad_distortion=g_dist)
    torch.cuda.synchronize()
    return out, dist, state, {"tetrahedra_field": gfield, **gp, "origins": go, "directions": gd, "vertices": gv}


def _forward_check(fr, state, st, oc, V, C, field, params, o, d, dist, what, keep=None):
    """d of the kernel against float64 at the kernel's own bins, with the float32 oracle as the noise floor (over the rays `keep`, if
    given)"""
    S2 = st.num_samples + st.num_fine_samples + 1
    eb, sb = _ray_order(state, S2)
    mesh = _mesh(V, C)
    res = {}
    for dtype in (torch.float64, torch.float32):
        torch.set_default_dtype(dtype)
        try:
            with torch.no_grad():
                f = torch.from_numpy(field).to(dtype)
                p = {k: v.detach().to(dtype) for k, v in params.items()}
                res[dtype] = dso.render_train_distortion(mesh, f, p, torch.from_numpy(o).to(dtype), torch.from_numpy(d).to(dtype), V, oc,
                                                         fine_euclid=eb, fine_sbins=sb)
        finally:
            torch.set_default_dtype(torch.float32)
    d64 = res[torch.float64]["distortion"][:, 0]
    d32 = res[torch.float32]["distortion"][:, 0].double()
    got = dist.cpu().double()[:, 0]
    mask = res[torch.float64]["ray_mask"]
    sel = torch.ones_like(mask) if keep is None else keep
    scale = max(d64[sel].abs().max().item(), D_UNIT_MIN)
    err = (got - d64)[sel].abs().max().item() / scale
    noise = (d32 - d64)[sel].abs().max().item() / scale
    print(f"--- {what}: max d {scale:.3e}, mean d {d64[mask].mean().item():.3e}; max |d - d64| / max d64 = {err:.2e}, "
          f"torch-f32 vs f64 {noise:.2e}")
    assert torch.all(got[~mask] == 0)
    assert torch.isfinite(got).all() and bool((got >= 0).all())
    assert err <= max(2 * GRAD_TOL, 6 * noise), (what, err, noise)


FWD_CASES = [("tetra_nerf", None), ("tetra_nerf", 100), ("tetra_nerf_original", None), ("small_uniform", 1000)]


@pytest.mark.parametrize("cfgname,k", FWD_CASES, ids=[f"{c}-{'random' if k is None else f'k{k}'}" for c, k in FWD_CASES])
def test_forward_against_float64(small_mesh, cfgname, k):
    V, C = small_mesh
    field, params = _field(V, k)
    _, fr, params = _setup(V, C, field, params)
    st, oc = _settings(cfgname)
    o, d = _rays()
    jc, jf, _ = _inputs(len(o), st, 5)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    dist = fr.train_distortion(state)
    torch.cuda.synchronize()
    assert dist.shape == (len(o), 1) and dist[5, 0].item() == 0.0
    _forward_check(fr, state, st, oc, V, C, field, params, o, d, dist, f"{cfgname}, {'random' if k is None else f'k = {k}'}")


GRAD_CASES = [("tetra_nerf", False, None, "dist"), ("tetra_nerf", True, None, "rgb+dist"), ("tetra_nerf", True, 100, "rgb+depth+dist"),
              ("tetra_nerf_original", True, None, "dist"), ("small_uniform", False, 1000, "rgb+dist")]


@pytest.mark.parametrize("cfgname,gs,k,loss", GRAD_CASES,
                         ids=[f"{c}-gs{int(g)}-{'random' if k is None else f'k{k}'}-{l}" for c, g, k, l in GRAD_CASES])
def test_gradients_against_float64(small_mesh, cfgname, gs, k, loss):
    V, C = small_mesh
    field, params = _field(V, k)
    st, oc = _settings(cfgname)
    o, d = _rays()
    R = len(o)
    jc, jf, target = _inputs(R, st, 5)
    _, fr, params = _setup(V, C, field, params)
    mesh = _mesh(V, C)
    ref64, gdep, g64 = _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, gs, torch.float64, loss)
    out, dist, state, got = _kernel_step(fr, st, V, o, d, jc, jf, target, gs, loss, gdep)
    S2 = st.num_samples + st.num_fine_samples + 1
    eb, sb = _ray_order(state, S2)
    _, _, g32 = _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, gs, torch.float32, loss, gdep=gdep)
    _, _, gsb = _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, gs, torch.float64, loss, fine=eb, sbins=sb, gdep=gdep)
    e_d = (dist.cpu().double() - ref64["distortion"].detach()).abs().max().item() / ref64["distortion"].abs().max().item()
    print(f"--- {cfgname}, gradient scaling {gs}, {'random field' if k is None else f'k = {k}'}, loss on {loss}: end-to-end max |d - d64| "
          f"/ max d64 {e_d:.2e}")
    failures = []
    for name in got:
        if g64[name] is None or g64[name].abs().max() == 0:  # a loss on the weights alone does not reach the colour heads
            assert torch.all(got[name] == 0), name
            continue
        _check(name, got[name], g32[name], g64[name], gsb[name], failures)
    assert not failures, failures


def test_null_distortion_gradient_and_old_entry_point_unchanged(small_mesh, monkeypatch):
    """deterministic mode: d is computed from the saved state alone, so the forward's outputs are the same bits with or without it;
    a backward with grad_distortion=None, and the old tn_render_train_backward_saved symbol, give the same gradients bit for bit, with
    and without the expected depth's gradient and the ray and vertex gradients"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = small_mesh
    field, params = _field(V, None)
    st, _ = _settings("tetra_nerf")
    o, d = _rays(400, 21)
    jc, jf, target = _inputs(len(o), st, 7)
    _, fr, _ = _setup(V, C, field, params)
    args = (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    a, sa = fr.train_forward_saved(*args, expected_depth=True)
    b, sb = fr.train_forward_saved(*args, expected_depth=True)
    fr.train_distortion(sb)
    for key in a:
        assert torch.equal(a[key], b[key]), key
    R = len(o)
    g_rgb = (2.0 * (a["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
    g_acc = torch.full((R,), 0.05 / R, device=DEV)
    g_ed = torch.full((R,), 0.5 / R, device=DEV)
    for ged in (None, g_ed):
        for kw in ({}, {"grad_origins": True, "grad_directions": True, "grad_vertices": True}):
            ra = fr.train_backward_saved(sa, g_rgb, g_acc, len(V), True, grad_expected_depth=ged, **kw)
            rb = fr.train_backward_saved(sb, g_rgb, g_acc, len(V), True, grad_expected_depth=ged, grad_distortion=None, **kw)
            outs = [torch.empty((n, 3), device=DEV) if kw else None for n in (R, R, len(V))]
            rc = fr._grad_outputs(len(V))
            assert _lib.tn_render_train_backward_saved(fr.tracer.handle, sb.blob.data_ptr(), g_rgb.data_ptr(), g_acc.data_ptr(),
                                                       ged.data_ptr() if ged is not None else None, 1, rc[0].data_ptr(), rc[2],
                                                       *(t.data_ptr() if t is not None else None for t in outs), fr._stream()) == 0
            torch.cuda.synchronize()
            assert torch.equal(ra[0], rb[0]) and torch.equal(ra[0], rc[0])
            for n in ra[1]:
                assert torch.equal(ra[1][n], rb[1][n]) and torch.equal(ra[1][n], rc[1][n]), n
            for x, y in zip(ra[2:], rb[2:]):
                assert torch.equal(x, y)
            for x, y in zip(ra[2:], outs if kw else ()):
                assert torch.equal(x, y)
    # and a distortion gradient does change them
    rd = fr.train_backward_saved(sb, g_rgb, g_acc, len(V), True, grad_distortion=torch.full((R,), 1.0 / R, device=DEV))
    torch.cuda.synchronize()
    assert not torch.equal(rd[0], ra[0])


def _dist_step(fr, V, st, batch, gs=True):
    o, d, jc, jf = batch
    out, state = fr.train_forward_saved(o, d, st, jc, jf)
    dist = fr.train_distortion(state)
    g_rgb = (2.0 * (out["rgb"] - 0.5) / (3 * len(o))).contiguous()
    res = fr.train_backward_saved(state, g_rgb, None, len(V), gs, grad_origins=True, grad_directions=True, grad_vertices=True,
                                  grad_distortion=torch.full((len(o),), 1.0 / len(o), device=DEV))
    torch.cuda.synchronize()
    return out, dist, state, res


@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
def test_repeatability(small_mesh, monkeypatch, det):
    """d of one saved state is the same bits every time in both modes; in the deterministic mode two whole steps with a distortion
    gradient are the same bits"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1" if det else "0")
    V, C = small_mesh
    field, params = _field(V, 100)
    st, _ = _settings("tetra_nerf")
    o, d = _rays(400, 21)
    jc, jf, _ = _inputs(len(o), st, 7)
    _, fr, _ = _setup(V, C, field, params)
    batch = (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), jc.to(DEV), jf.to(DEV))
    a_out, a_d, a_state, a = _dist_step(fr, V, st, batch)
    again = fr.train_distortion(a_state)
    torch.cuda.synchronize()
    assert torch.equal(a_d, again)
    assert a_d.abs().max() > 0
    if not det:
        return
    b_out, b_d, _, b = _dist_step(fr, V, st, batch)
    for key in a_out:
        assert torch.equal(a_out[key], b_out[key]), key
    assert torch.equal(a_d, b_d)
    assert torch.equal(a[0], b[0])
    for n in a[1]:
        assert torch.equal(a[1][n], b[1][n]), n
    for x, y in zip(a[2:], b[2:]):
        assert torch.equal(x, y)


EDGES = ["s2_3", "s2_64", "cap4", "large", "ceiling", "tiny_r1", "tiny_r5"]


@pytest.mark.parametrize("case", EDGES)
def test_settings_edges(small_mesh, case):
    """the per-ray kernels at the edges of the settings: d against float64 at the kernel's bins, and the gradients of the distortion
    loss (default mode, GradientScaler on) with the bars above; the ceiling case (the largest S2 at M = 512) runs with the distortion.
    Rays with a sample that the kernel and the oracle match to different tetrahedra (a sample on a face; frequent with cap4's
    truncated rays, where a flipped sample turns a density on or off) are left out of both checks and counted: the float32 oracle has
    the oracle's match, so its noise floor does not cover them."""
    V, C = small_mesh
    Sc, Sf, M, biased, R = EDGE_CASES[case]
    S2 = Sc + Sf + 1
    st, oc = _edge_settings(Sc, Sf, M, biased)
    o, d = _rays(R)
    if case == "ceiling":
        optin = torch.cuda.get_device_properties(DEV).shared_memory_per_block_optin
        assert S2 == _s2_max(M, optin)
    field, params = _field(V, None)
    _, fr, params = _setup(V, C, field, params)
    jc, jf, target = _inputs(R, st, 5)
    mesh = _mesh(V, C)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    n, ray_list, _, _, _ = _blob(state, S2)
    eb, sb = _ray_order(state, S2)
    # matched vertices: after the header, the active-count slot, ray_list and the two bin arrays (saved_layout in tn_render.cu)
    vi_off = 256 + 256 + 256 * ((4 * R + 255) // 256) + 2 * 256 * ((4 * R * (S2 + 1) + 255) // 256)
    vi_k = _from_ptr(state.blob.data_ptr() + vi_off, (n, S2, 4), torch.int32).cpu()[torch.argsort(ray_list.cpu())]
    with torch.no_grad():
        ref = dso.render_train_distortion(mesh, torch.from_numpy(field), params, torch.from_numpy(o), torch.from_numpy(d), V, oc,
                                          fine_euclid=eb, fine_sbins=sb)
    vi_o = torch.from_numpy(ref["aux"]["matched"]["vertex_indices"])
    mask = ref["ray_mask"]
    keep = mask.clone()
    keep[torch.nonzero(mask).flatten()[(vi_k != vi_o).any(-1).any(-1)]] = False
    print(f"--- {case}: {int(mask.sum() - keep.sum())} of {int(mask.sum())} active rays with a flipped sample left out")
    assert int(keep.sum()) >= max(1, int(mask.sum()) // 2)
    dist = fr.train_distortion(state)
    _forward_check(fr, state, st, oc, V, C, field, params, o, d, dist, case, keep=keep)
    cdist = keep.double() / int(keep.sum())
    loss = "dist"
    _, _, g64 = _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, True, torch.float64, loss, cdist=cdist)
    got = _kernel_step(fr, st, V, o, d, jc, jf, target, True, loss, cdist=cdist)[3]  # (the same jitter: the same bins)
    _, _, g32 = _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, True, torch.float32, loss, cdist=cdist)
    _, _, gsb = _oracle(mesh, field, params, o, d, V, oc, jc, jf, target, True, torch.float64, loss, fine=eb, sbins=sb, cdist=cdist)
    # cap4's truncated rays are almost transparent (x = delta sigma ~ 1e-4 per sample): their weights, 1 - expf(-x) times T as the
    # forward forms them, carry a relative error of ~ulp(1) / x from the device expf, uniform over every tensor (6.2e-4 measured on an
    # H100), where torch's correctly rounded float32 exp gives a floor about 6x lower; that case's floor is 1e-3 instead of 2e-4
    floor = 1e-3 if case == "cap4" else 2 * GRAD_TOL
    failures = []
    for name in got:
        if g64[name] is None or g64[name].abs().max() == 0:  # a loss on the weights alone does not reach the colour heads
            assert torch.all(got[name] == 0), name
            continue
        g, f32, f64, fsb = (t.detach().cpu().double() for t in (got[name], g32[name], g64[name], gsb[name]))
        assert torch.isfinite(g).all(), name
        arith = (g - fsb).abs().max().item() / fsb.abs().max().item()
        noise = (f32 - f64).abs().max().item() / f64.abs().max().item()
        err = (g - f64).abs().max().item() / f64.abs().max().item()
        print(f"  {name:34s} (A) {arith:.2e}  (B) {err:.2e}  torch-f32 vs f64 {noise:.2e}")
        if not (arith <= max(floor, 6 * noise) and err <= max(floor, 6 * noise)):
            failures.append((name, arith, err, noise))
    assert not failures, failures


def test_all_empty_batch(small_mesh):
    """M = 2: every ray crosses the mesh and keeps no tetrahedron; d is 0 and every gradient 0, in both modes"""
    V, C = small_mesh
    st, o, d = _empty_batch("cap2")
    R = len(o)
    _, fr, _ = _setup(V, C, *_field(V, None))
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    for det in (False, True):
        g = torch.Generator().manual_seed(2)
        jc = torch.rand((R, st.num_samples + 1), generator=g).to(DEV)
        jf = torch.rand((R, st.num_fine_samples + 1), generator=g).to(DEV)
        with _deterministic(det):
            out, state = fr.train_forward_saved(ot, dt, st, jc, jf)
            dist = fr.train_distortion(state)
            grads = fr.train_backward_saved(state, torch.zeros((R, 3), device=DEV), None, len(V), True, grad_origins=True,
                                            grad_directions=True, grad_vertices=True, grad_distortion=torch.ones((R,), device=DEV))
        torch.cuda.synchronize()
        assert not bool(out["ray_mask"].any())
        assert bool((dist == 0).all())
        gfield, gp, go, gd, gv = grads
        for n, t in {"tetrahedra_field": gfield, **gp, "origins": go, "directions": gd, "vertices": gv}.items():
            assert bool((t == 0).all()), f"deterministic {det}: {n}"


def test_errors(small_mesh):
    V, C = small_mesh
    field, params = _field(V, None)
    st, _ = _settings("tetra_nerf")
    o, d = _rays(64)
    R = len(o)
    _, fr, params = _setup(V, C, field, params)
    args = (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    out, state = fr.train_forward_saved(*args)
    g_rgb = torch.zeros((R, 3), device=DEV)
    for bad in (torch.ones((R + 1,), device=DEV), torch.ones((R,), device=DEV, dtype=torch.float64), torch.ones((R,)),
                torch.ones((R, 2), device=DEV)):
        with pytest.raises(RuntimeError, match="grad_distortion"):
            fr.train_backward_saved(state, g_rgb, None, len(V), grad_distortion=bad)
    fr.train_distortion(state)
    fr.train_backward_saved(state, g_rgb, None, len(V), grad_distortion=torch.ones((R, 1), device=DEV))  # [R,1] is accepted
    for change in ("field", "weights"):
        out, state = fr.train_forward_saved(*args)
        if change == "field":
            fr.set_field(torch.from_numpy(field).to(DEV))
        else:
            fr.set_weights(params)
        with pytest.raises(RuntimeError, match="changed"):
            fr.train_distortion(state)
        with pytest.raises(RuntimeError, match="changed"):
            fr.train_backward_saved(state, g_rgb, None, len(V), grad_distortion=torch.ones((R,), device=DEV))
    torch.cuda.synchronize()


def _model_run(V, C, field, mode, o, d, target_rgb, target_depth, monkeypatch, det=False):
    from tetranerf.nerfstudio import model as M

    monkeypatch.setenv("TETRANERF_B200_UNFUSED_TRAIN", "1" if mode == "unfused" else "0")
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1" if det else "0")
    cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=64, num_fine_samples=64,
                                 use_biased_sampler=True, use_gradient_scaling=True, depth_loss_mult=0.1, distortion_loss_mult=0.5)
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
    sum(losses.values()).backward()
    return out, losses, {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


def test_model_training_paths_agree_with_a_distortion_loss(small_mesh, monkeypatch):
    """TetrahedraNerf with distortion_loss_mult > 0 (and a depth loss): the fused op and the unfused op sequence (the O(S) torch form
    under autograd) give the same outputs, losses and gradients, as test_model_training_paths_agree_with_a_depth_loss"""
    V, C = small_mesh
    field, _ = _field(V, None)
    o, d = syn.camera_rays(256, seed=14)
    g = torch.Generator().manual_seed(3)
    target = torch.rand((256, 3), generator=g).to(DEV)
    target_depth = (1.0 + torch.rand((256, 1), generator=g)).to(DEV)
    res = {mode: _model_run(V, C, field, mode, o, d, target, target_depth, monkeypatch) for mode in ("fused", "unfused")}
    (of, lf, gf), (ou, lu, gu) = res["fused"], res["unfused"]
    assert set(lf) == set(lu) == {"rgb_loss", "depth_loss", "distortion_loss"}
    assert of["distortion"].shape == ou["distortion"].shape == (256, 1)
    assert (of["distortion"] - ou["distortion"]).abs().max().item() <= 1e-4 * ou["distortion"].abs().max().item() + 1e-7
    assert abs(lf["distortion_loss"].item() - lu["distortion_loss"].item()) <= 1e-4 * lu["distortion_loss"].item()
    assert set(gf) == set(gu)
    for n, gg in gu.items():
        a = gf[n]
        rel = ((a - gg).abs().max() / gg.abs().max().clamp_min(1e-30)).item()
        l2 = ((a - gg).norm() / gg.norm().clamp_min(1e-30)).item()
        print(f"  {n:34s} fused vs unfused: max {rel:.2e}  L2 {l2:.2e}")
        assert torch.isfinite(a).all()
        assert rel < 5e-3 and l2 < 1e-3, (n, rel, l2)
    # the deterministic mode and the vertex parameters compose with it
    out, losses, grads = _model_run(V, C, field, "fused", o, d, target, target_depth, monkeypatch, det=True)
    assert abs(losses["distortion_loss"].item() - lf["distortion_loss"].item()) <= 1e-5 * lf["distortion_loss"].item()


def test_distortion_only_steps_concentrate_the_weights(small_mesh, monkeypatch):
    """surface_scene (k = 100) with a diffuse haze (feature 0 raised to at least 0, i.e. sigma ~ softplus(0) everywhere outside the
    spheres): a few Adam steps on the field with the distortion loss alone lower the mean d of the active rays at every step and raise
    their mean peak weight.  Deterministic mode, so that the run repeats."""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    from tetranerf.b200.render import PARAM_ORDER, FusedTrainRenderDistortion

    V, C = small_mesh
    field, params = _field(V, 100)
    field = field.copy()
    field[0] = np.maximum(field[0], 0.0)  # the haze
    st, _ = _settings("tetra_nerf")
    _, fr, params = _setup(V, C, field, params)
    o, d = syn.camera_rays(1024, seed=9)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    ps = [params[n].to(DEV) for n in PARAM_ORDER]
    f = torch.from_numpy(field).to(DEV).clone().requires_grad_(True)
    opt = torch.optim.Adam([f], lr=1e-2)
    S2 = st.num_samples + st.num_fine_samples + 1
    means, peaks = [], []
    for it in range(8):
        fr.set_field(f.detach())
        opt.zero_grad()
        _, _, _, dist, mask = FusedTrainRenderDistortion.apply(fr, st, False, False, o, d, None, None, f, *ps)
        with torch.no_grad():  # the peak weight per active ray, from this forward's own saved state
            out, state = fr.train_forward_saved(o, d, st)
            _, _, eb, _, of = _blob(state, S2)
            x = (eb[:, 1:] - eb[:, :-1]) * of[..., 0]
            w = (1 - torch.exp(-x)) * torch.exp(-torch.cumsum(x, -1) + x)
            peaks.append(w.max(-1).values.mean().item())
        loss = dist.sum() / mask.sum()
        means.append(loss.item())
        loss.backward()
        opt.step()
    print("mean d per step: " + " ".join(f"{m:.4e}" for m in means) + f"; mean peak weight {peaks[0]:.4f} -> {peaks[-1]:.4f}")
    assert all(b < a for a, b in zip(means, means[1:])), means
    assert peaks[-1] > peaks[0]
