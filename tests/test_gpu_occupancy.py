"""GPU: occupancy culling on the fused paths (DESIGN §4.12) against the oracle (oracle/occupancy.py).
  * tn_occupancy_update against the float64 probe maximum (the bf16x3 per-sample bar 1e-4 + 2e-5 |sigma|), bitwise on a second call, decay;
  * an occupancy where nothing is culled gives the bits of no occupancy: eval render in both precisions (expected depth and normals too),
    training step with expected depth, distortion, ray and vertex gradients in the deterministic mode (the default mode's float
    reductions are not reproducible run to run, so there its forward is compared bitwise and its gradients at 1e-5 of their scale);
  * partial culling of surface_scene: render against the oracle at the pixel bar, training gradients against float64 autograd at the
    bar of test_gpu_train.py, with the GPU's own occupancy in the oracle; the culled fraction of both passes is strictly inside (0, 1);
  * deterministic mode with culling is bitwise repeatable, and an occupancy change between a saved forward and its backward changes
    nothing;
  * the model: strict loading of the reference's buffer, the recompute of a zero buffer, update interval and warm-up, unsupported configs."""
import numpy as np
import pytest
import torch

from oracle import occupancy as ocu
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _deterministic
from test_gpu_train import DEV, _check, _from_ptr, _setup

pytestmark = pytest.mark.gpu
THR = 0.01  # the model's default threshold
CULLED = -2  # vi.w of a culled sample (0xFFFFFFFE), with vi.x = -1


def _settings(cfgname):
    from tetranerf.b200.render import RenderSettings

    if cfgname == "tetra_nerf":
        return RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    return RenderSettings(num_samples=48, num_fine_samples=64), orc.RenderConfig(num_samples=48, num_fine_samples=64)


def _rays(R=300, seed=11):
    o, d = syn.camera_rays(R, seed=seed)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    return o, d


def _occ(fr, T, decay=0.0, occ=None):
    occ = torch.zeros((T,), dtype=torch.float32, device=DEV) if occ is None else occ
    fr.update_occupancy(occ, decay)
    torch.cuda.synchronize()
    return occ


def _culled_fraction(fr, st):
    """culled share of the active samples of each pass of the last render (debug buffers)"""
    bufs = fr.debug_buffers()
    n = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    S2 = st.num_samples + st.num_fine_samples + 1
    vc = _from_ptr(bufs["vi_c"], (n, st.num_samples, 4), torch.int32)
    vf = _from_ptr(bufs["vi_f"], (n, S2, 4), torch.int32)
    return [((v[..., 0] == -1) & (v[..., 3] == CULLED)).float().mean().item() for v in (vc, vf)]


def _blob_culled(fr, state, st):
    """culled share of the active samples of the coarse pass (the tracer's buffers) and the fine pass (vi_f in the saved state;
    saved_layout in tn_render.cu) of the last saved training forward"""
    R, S2 = state.R, st.num_samples + st.num_fine_samples + 1
    up = lambda b: (b + 255) // 256 * 256
    base = state.blob.data_ptr()
    n = int(_from_ptr(base + 256, (1,), torch.int32)[0])
    off = 512 + up(4 * R) + 2 * up(4 * R * (S2 + 1))
    vf = _from_ptr(base + off, (n, S2, 4), torch.int32)
    vc = _from_ptr(fr.debug_buffers()["vi_c"], (n, st.num_samples, 4), torch.int32)
    return [((v[..., 0] == -1) & (v[..., 3] == CULLED)).float().mean().item() for v in (vc, vf)]


def test_occupancy_update_vs_oracle(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    occ = _occ(fr, len(C))
    ref = ocu.occupancy(field, params, C)
    err = (occ.cpu().double() - ref).abs()
    print(f"occupancy: max {ref.max().item():.3f}, max err {err.max().item():.2e}")
    assert bool((err <= 1e-4 + 2e-5 * ref.abs()).all())
    assert torch.equal(_occ(fr, len(C)), occ)  # bitwise on a second call
    # decay: max(decay occ, probe max); with a large previous value the decayed one wins
    prev = torch.full((len(C),), 50.0, device=DEV)
    prev[::2] = 0.0
    got = _occ(fr, len(C), 0.5, prev.clone())
    assert torch.equal(got, torch.maximum(0.5 * prev, occ))
    assert torch.equal(_occ(fr, len(C), 0.0, torch.full((len(C),), float("nan"), device=DEV)), occ)  # decay 0 never reads it
    with pytest.raises(RuntimeError):
        fr.update_occupancy(occ, -1.0)
    with pytest.raises(RuntimeError):
        fr.set_occupancy(occ, float("inf"))


def _render(fr, o, d, st, normals=False, ed=False):
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, normals=normals, expected_depth=ed)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


@pytest.mark.parametrize("prec", [2, 3])
def test_all_occupied_render_bitwise(small_mesh, prec):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    fr.set_mlp_precision(prec)
    o, d = _rays()
    for cfg in ("tetra_nerf", "small"):
        st, _ = _settings(cfg)
        base = _render(fr, o, d, st, normals=True, ed=True)
        occ = _occ(fr, len(C))
        fr.set_occupancy(occ, 0.0)  # sigma >= 0: nothing is below 0
        got = _render(fr, o, d, st, normals=True, ed=True)
        assert _culled_fraction(fr, st) == [0.0, 0.0]
        fr.set_occupancy(None)
        for k in base:
            assert torch.equal(base[k], got[k]), (cfg, k)


def _train(fr, o, d, st, jc, jf, g, V, gs=False):
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc, jf, expected_depth=True)
    dist = fr.train_distortion(state)
    R = len(o)
    res = fr.train_backward_saved(state, g[:, :3].contiguous(), g[:, 3].contiguous(), len(V), gs, grad_origins=True, grad_directions=True,
                                  grad_vertices=True, grad_expected_depth=g[:, 4].contiguous(), grad_distortion=g[:, 5].contiguous())
    torch.cuda.synchronize()
    gfield, gp, go, gd, gv = res
    outs = {k: v.clone() for k, v in out.items()}
    outs["distortion"] = dist.clone()
    grads = {"field": gfield, "origins": go, "directions": gd, "vertices": gv, **gp}
    assert R == state.R
    return outs, grads, state


def _train_inputs(o, st, seed=5):
    gen = torch.Generator().manual_seed(seed)
    R = len(o)
    jc = torch.rand((R, st.num_samples + 1), generator=gen).to(DEV)
    jf = torch.rand((R, st.num_fine_samples + 1), generator=gen).to(DEV)
    g = (torch.randn((R, 6), generator=gen) * 1e-2).to(DEV)
    return jc, jf, g


@pytest.mark.parametrize("det", [True, False])
def test_all_occupied_train_bitwise(small_mesh, det):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    o, d = _rays()
    st, _ = _settings("tetra_nerf")
    jc, jf, g = _train_inputs(o, st)
    with _deterministic(det):
        out0, g0, _ = _train(fr, o, d, st, jc, jf, g, V, gs=True)
        fr.set_occupancy(_occ(fr, len(C)), 0.0)
        out1, g1, _ = _train(fr, o, d, st, jc, jf, g, V, gs=True)
        fr.set_occupancy(None)
    for k in out0:
        assert torch.equal(out0[k], out1[k]), k
    for k in g0:
        if det:
            assert torch.equal(g0[k], g1[k]), k
        else:
            scale = g0[k].abs().max().item()
            assert (g0[k] - g1[k]).abs().max().item() <= 1e-5 * scale, k


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("cfgname", ["tetra_nerf", "small"])
def test_partial_culling_render_vs_oracle(small_mesh, cfgname, prec):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    fr.set_mlp_precision(prec)
    occ = _occ(fr, len(C))
    fr.set_occupancy(occ, THR)
    o, d = _rays()
    st, oc = _settings(cfgname)
    out = _render(fr, o, d, st)
    frac = _culled_fraction(fr, st)
    ref = ocu.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, oc, occupancy=(occ.cpu(), THR))
    ref_frac = [ref["aux"]["coarse_culled"].float().mean().item(), ref["aux"]["culled"].float().mean().item()]
    e_rgb = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"]).abs().max().item()
    print(f"{cfgname} prec={prec}: culled (coarse, fine) {frac} oracle {ref_frac}  max|rgb| {e_rgb:.2e} max|acc| {e_acc:.2e}")
    assert all(0.0 < f < 1.0 for f in frac), frac
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    assert e_rgb < 1e-4 and e_acc < 1e-4


@pytest.mark.parametrize("gs", [False, True])
def test_partial_culling_train_gradients(small_mesh, gs):
    from tetranerf.b200.render import PARAM_ORDER
    from test_gpu_distortion import _ray_order

    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    occ = _occ(fr, len(C))
    fr.set_occupancy(occ, THR)
    o, d = _rays()
    st, oc = _settings("tetra_nerf")
    R = len(o)
    gen = torch.Generator().manual_seed(7)
    jc, jf = torch.rand((R, st.num_samples + 1), generator=gen), torch.rand((R, st.num_fine_samples + 1), generator=gen)
    target = torch.rand((R, 3), generator=gen)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    torch.cuda.synchronize()
    frac = _blob_culled(fr, state, st)
    g_rgb = (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
    g_acc = torch.full((R,), 0.05 / R, device=DEV)
    gfield, gp = fr.train_backward_saved(state, g_rgb, g_acc, len(V), gs)
    torch.cuda.synchronize()
    S2 = st.num_samples + st.num_fine_samples + 1
    fine, _ = _ray_order(state, S2)
    mesh = orc.OracleMesh(V, C)

    def oracle(dtype, fine_euclid=None):
        f = torch.from_numpy(field).to(dtype).requires_grad_(True)
        p = {k: v.clone().to(dtype).requires_grad_(True) for k, v in params.items()}
        torch.set_default_dtype(dtype)
        try:
            r = ocu.render_train(mesh, f, p, o, d, oc, jc, jf, use_gradient_scaling=gs, occupancy=(occ.cpu(), THR), fine_euclid=fine_euclid)
        finally:
            torch.set_default_dtype(torch.float32)
        loss = torch.nn.functional.mse_loss(r["rgb"], target.to(r["rgb"].dtype)) + 0.05 * r["accumulation"].mean()
        loss.backward()
        return r, f.grad, {k: v.grad for k, v in p.items()}

    ref, gf32, gp32 = oracle(torch.float32)
    _, gf64, gp64 = oracle(torch.float64)
    rsb, gfsb, gpsb = oracle(torch.float64, fine)
    print(f"gs={gs}: culled (coarse, fine) {frac}, oracle fine {rsb['aux']['culled'].float().mean().item():.3f}")
    assert all(0.0 < f < 1.0 for f in frac), frac
    assert (out["rgb"].cpu() - ref["rgb"].detach()).abs().max().item() < 1e-4
    failures = []
    _check("tetrahedra_field", gfield, gf32, gf64, gfsb, failures)
    for n in PARAM_ORDER:
        _check(n, gp[n], gp32[n], gp64[n], gpsb[n], failures)
    assert not failures, failures


def test_culling_deterministic_and_independent_of_later_updates(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    occ = _occ(fr, len(C))
    fr.set_occupancy(occ, THR)
    o, d = _rays()
    st, _ = _settings("tetra_nerf")
    jc, jf, g = _train_inputs(o, st)
    with _deterministic(True):
        out0, g0, state = _train(fr, o, d, st, jc, jf, g, V)
        out1, g1, _ = _train(fr, o, d, st, jc, jf, g, V)
        assert _blob_culled(fr, state, st)[1] > 0.0
        for k in out0:
            assert torch.equal(out0[k], out1[k]), k
        for k in g0:
            assert torch.equal(g0[k], g1[k]), k
        # a different occupancy between the saved forward and its backward: the backward reads only its own state
        occ.fill_(0.0)
        fr.set_occupancy(None)
        res = fr.train_backward_saved(state, g[:, :3].contiguous(), g[:, 3].contiguous(), len(V), False, grad_origins=True,
                                      grad_directions=True, grad_vertices=True, grad_expected_depth=g[:, 4].contiguous(),
                                      grad_distortion=g[:, 5].contiguous())
        torch.cuda.synchronize()
    gfield, gp, go, gd, gv = res
    again = {"field": gfield, "origins": go, "directions": gd, "vertices": gv, **gp}
    for k in g0:
        assert torch.equal(g0[k], again[k]), k


# ---- model ------------------------------------------------------------------------------------------------------------------------------
def _model(V, C, field, params, **cfg):
    from tetranerf.nerfstudio import model as M

    config = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=48, num_fine_samples=64,
                                    use_occupancy_field=True, **cfg)
    m = M.TetrahedraNerf(config)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field),
          "tetrahedra_occupancy": torch.zeros(len(C))}
    sd.update(params)
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and "tetrahedra_occupancy" not in res.missing_keys
    return m.to(DEV), M


def test_model_occupancy(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    m, M = _model(V, C, field, params, occupancy_warmup_steps=2, occupancy_update_interval=3)
    assert m.tetrahedra_occupancy.shape == (len(C),) and m.tetrahedra_occupancy.dtype == torch.float32
    # a reference checkpoint (the buffer present, all zeros) loads strictly
    m2 = M.TetrahedraNerf(m.config)
    m2.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    o, d = _rays(200)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    # eval: the zero buffer is computed before the first render, which then culls
    m.eval()
    with torch.no_grad():
        out = m(bundle)
    fr = m._fused
    ref = torch.zeros(len(C), device=DEV)
    fr.update_occupancy(ref, 0.0)
    assert torch.equal(m.tetrahedra_occupancy, ref)
    fr.set_occupancy(None)
    with torch.no_grad():
        plain = fr.render(bundle.origins, bundle.directions, fr_settings(m))
    st = fr_settings(m)
    assert (out["rgb"] - plain["rgb"]).abs().max().item() < 1e-2  # culling changes little on this scene
    # training: no culling for the warm-up steps, then an update every interval
    calls = []
    orig = fr.update_occupancy
    fr.update_occupancy = lambda occ, decay=0.0: (calls.append(decay), orig(occ, decay))[1]
    sets = []
    orig_set = fr.set_occupancy
    fr.set_occupancy = lambda occ, thr=0.0: (sets.append(occ is not None), orig_set(occ, thr))[1]
    m.train()
    m._occ_step = 0
    for _ in range(8):
        r = m(bundle)
        (r["rgb"].sum() * 0).backward()
    assert sets == [False, False, True, True, True, True, True, True], sets
    assert calls == [m.config.occupancy_decay] * 2, calls  # steps 2 and 5 (step 8 is not reached)
    assert st.num_samples == 48
    # an unsupported config raises and names the option
    bad, _ = _model(V, C, field, params, background_color="random")
    with pytest.raises(RuntimeError, match="background_color"):
        with torch.no_grad():
            bad.eval()(bundle)


def fr_settings(m):
    from tetranerf.b200.render import RenderSettings

    c = m.config
    return RenderSettings(c.max_intersected_triangles, c.num_samples, c.num_fine_samples, c.use_biased_sampler, float(m.collider.far_plane))
