"""GPU: occupancy sampling on the fused paths (DESIGN §4.13) against the oracle (oracle/placement.py).
  * coarse bins of the placed rays against the oracle's float32 restatement, both samplers, eval and training jitter;
  * the eval render in both MLP precisions against the oracle at the 1e-4 pixel bar; the training gradients (field and MLP) against
    float64 autograd at the bar of test_gpu_train.py, with and without GradientScaler;
  * with nothing skipped (threshold 0) the outputs and gradients are the bits of culling only; the option off is culling only;
  * the deterministic mode is bitwise repeatable with it (expected depth, distortion, ray and vertex gradients included);
  * the settings edges; the model hooks and the RuntimeError;
  * on surface_scene at 64 + 64 samples, placement renders closer to a converged dense render than culling only, for both samplers."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import placement as pl
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _deterministic
from test_gpu_occupancy import THR, _culled_fraction, _occ, _render, _train, _train_inputs
from test_gpu_train import DEV, _check, _from_ptr, _setup

pytestmark = pytest.mark.gpu


def _st(Sc, Sf, biased, M=512):
    from tetranerf.b200.render import RenderSettings

    kw = dict(num_samples=Sc, num_fine_samples=Sf, use_biased_sampler=biased, max_intersected_triangles=M)
    return RenderSettings(**kw), orc.RenderConfig(**kw)


def _rays(R=300, seed=11):
    o, d = syn.camera_rays(R, seed=seed)
    if R > 5:
        o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    return o, d


def _scene(small_mesh):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    return V, C, field, params, fr, _occ(fr, len(C))


def _coarse_bins(fr, st, state=None):
    """the last call's coarse euclidean bins in the ray order of the non-empty rays (a saved training forward keeps its active-ray count
    and slot -> ray map in its own state: saved_layout in tn_render.cu)"""
    bufs = fr.debug_buffers()
    n_ptr, rl_ptr = (bufs["n_active"], bufs["ray_list"]) if state is None else (state.blob.data_ptr() + 256, state.blob.data_ptr() + 512)
    n = int(_from_ptr(n_ptr, (1,), torch.int32)[0])
    rl = _from_ptr(rl_ptr, (n,), torch.int32).cpu()
    eb = _from_ptr(bufs["ebins_c"], (n, st.num_samples + 1), torch.float32).cpu()
    return eb[torch.argsort(rl)]


@pytest.mark.parametrize("biased", [True, False])
@pytest.mark.parametrize("train", [False, True])
def test_coarse_bins_vs_oracle(small_mesh, biased, train):
    V, C, field, params, fr, occ = _scene(small_mesh)
    fr.set_occupancy(occ, THR, place_samples=True)
    o, d = _rays()
    st, oc = _st(64, 64, biased)
    mesh = orc.OracleMesh(V, C)
    tr = mesh.trace_rays(o, d, oc.max_intersected_triangles)
    m = tr["num_visited_cells"] > 0
    hd = torch.from_numpy(tr["hit_distances"][m])
    nv = torch.from_numpy(tr["num_visited_cells"][m])
    nears = hd[:, 0, 0][:, None]
    fars = torch.gather(hd[:, :, 1], 1, (nv[:, None].long() - 1).clamp_min(0))
    kept = pl.kept_records(tr["num_visited_cells"][m], tr["visited_cells"][m], occ.cpu(), THR)
    jc, state = None, None
    if train:
        jc, jf, _ = _train_inputs(o, st)
        _, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc, jf)
        jc = jc.cpu()[torch.from_numpy(m)]
    else:
        _render(fr, o, d, st)
    torch.cuda.synchronize()
    got = _coarse_bins(fr, st, state)
    ref, _ = pl.place_coarse_bins(oc, nears, fars, nv, hd, kept, jc)
    placed = torch.from_numpy((kept.sum(1) > 0) & (kept.sum(1) < nv.numpy()))
    ulp = (torch.nextafter(fars, torch.full_like(fars, np.inf)) - fars)
    err = (got - ref).abs() / ulp
    far_off = err > 8
    print(f"biased={biased} train={train}: {int(placed.sum())} of {len(got)} rays placed; bitwise {torch.equal(got, ref)}, "
          f"{int(far_off.sum())} of {got.numel()} edges more than 8 ulp(far) apart, the rest within {err[~far_off].max().item():.0f}")
    assert int(placed.sum()) > len(got) // 4
    # The spacing edges (linspace, jitter, the biased sampler's u) are nvcc's float arithmetic, with fused multiply-adds, against
    # torch's: a few ulp.  Where u n_kept lands within that of an integer, floor() picks the neighbouring kept record in one of the two
    # and the edge sits at the end of one record instead of the start of the next -- a rare jump across a skipped run, biased only.
    assert int(far_off.sum()) <= (0.002 * got.numel() if biased else 0), int(far_off.sum())
    for r, j in torch.nonzero(far_off).tolist():
        k = np.nonzero(kept[r])[0]
        ends, starts = hd[r, k[:-1], 1].numpy(), hd[r, k[1:], 0].numpy()
        a, b = sorted((float(got[r, j]), float(ref[r, j])))
        assert np.any(np.isclose(ends, a, rtol=0, atol=1e-5) & np.isclose(starts, b, rtol=0, atol=1e-5)), (r, j, a, b)
    # every placed edge lies in a kept record
    for r in torch.nonzero(placed).flatten().tolist()[:60]:
        k = np.nonzero(kept[r])[0]
        e = got[r].numpy()
        assert all(np.any((hd[r, k, 0].numpy() <= x) & (x <= hd[r, k, 1].numpy())) for x in e), r


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("biased", [True, False])
def test_render_vs_oracle(small_mesh, biased, prec):
    V, C, field, params, fr, occ = _scene(small_mesh)
    fr.set_mlp_precision(prec)
    fr.set_occupancy(occ, THR, place_samples=True)
    o, d = _rays()
    st, oc = _st(64, 64, biased)
    out = _render(fr, o, d, st, normals=True, ed=True)
    frac = _culled_fraction(fr, st)
    ref = pl.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, oc, occupancy=(occ.cpu(), THR))
    e_rgb = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"]).abs().max().item()
    print(f"biased={biased} prec={prec}: culled (coarse, fine) {frac}  max|rgb| {e_rgb:.2e} max|acc| {e_acc:.2e}")
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    assert e_rgb < 1e-4 and e_acc < 1e-4
    assert torch.isfinite(out["expected_depth"]).all() and torch.isfinite(out["normals"]).all()
    fr.set_occupancy(occ, THR)  # fewer coarse samples culled than with culling only
    _render(fr, o, d, st)
    assert frac[0] < _culled_fraction(fr, st)[0]


@pytest.mark.parametrize("gs", [False, True])
@pytest.mark.parametrize("biased", [True, False])
def test_train_gradients_vs_float64(small_mesh, biased, gs):
    from tetranerf.b200.render import PARAM_ORDER
    from test_gpu_distortion import _ray_order

    V, C, field, params, fr, occ = _scene(small_mesh)
    fr.set_occupancy(occ, THR, place_samples=True)
    o, d = _rays()
    st, oc = _st(64, 64, biased)
    R = len(o)
    gen = torch.Generator().manual_seed(7)
    jc, jf = torch.rand((R, st.num_samples + 1), generator=gen), torch.rand((R, st.num_fine_samples + 1), generator=gen)
    target = torch.rand((R, 3), generator=gen)
    out, state = fr.train_forward_saved(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st, jc.to(DEV), jf.to(DEV))
    g_rgb = (2.0 * (out["rgb"] - target.to(DEV)) / (3 * R)).contiguous()
    g_acc = torch.full((R,), 0.05 / R, device=DEV)
    gfield, gp = fr.train_backward_saved(state, g_rgb, g_acc, len(V), gs)
    torch.cuda.synchronize()
    fine, _ = _ray_order(state, st.num_samples + st.num_fine_samples + 1)
    mesh = orc.OracleMesh(V, C)

    def oracle(dtype, fine_euclid=None):
        f = torch.from_numpy(field).to(dtype).requires_grad_(True)
        p = {k: v.clone().to(dtype).requires_grad_(True) for k, v in params.items()}
        torch.set_default_dtype(dtype)
        try:
            r = pl.render_train(mesh, f, p, o, d, oc, jc, jf, use_gradient_scaling=gs, occupancy=(occ.cpu(), THR), fine_euclid=fine_euclid)
        finally:
            torch.set_default_dtype(torch.float32)
        loss = torch.nn.functional.mse_loss(r["rgb"], target.to(r["rgb"].dtype)) + 0.05 * r["accumulation"].mean()
        loss.backward()
        return r, f.grad, {k: v.grad for k, v in p.items()}

    ref, gf32, gp32 = oracle(torch.float32)
    _, gf64, gp64 = oracle(torch.float64)
    _, gfsb, gpsb = oracle(torch.float64, fine)
    assert (out["rgb"].cpu() - ref["rgb"].detach()).abs().max().item() < 1e-4
    failures = []
    _check("tetrahedra_field", gfield, gf32, gf64, gfsb, failures)
    for n in PARAM_ORDER:
        _check(n, gp[n], gp32[n], gp64[n], gpsb[n], failures)
    assert not failures, failures


@pytest.mark.parametrize("biased", [True, False])
def test_nothing_skipped_or_off_is_culling_only(small_mesh, biased):
    V, C, field, params, fr, occ = _scene(small_mesh)
    o, d = _rays()
    st, _ = _st(64, 64, biased)
    for prec in (2, 3):
        fr.set_mlp_precision(prec)
        fr.set_occupancy(occ, 0.0)
        base = _render(fr, o, d, st, normals=True, ed=True)
        fr.set_occupancy(occ, 0.0, place_samples=True)
        got = _render(fr, o, d, st, normals=True, ed=True)
        for k in base:
            assert torch.equal(base[k], got[k]), (prec, k)
    fr.set_occupancy(occ, THR)  # the option off: culling only, whatever was set before
    a = _render(fr, o, d, st)
    fr.set_occupancy(occ, THR, place_samples=True)
    fr.set_occupancy(occ, THR)
    b = _render(fr, o, d, st)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    jc, jf, g = _train_inputs(o, st)
    with _deterministic(True):
        fr.set_occupancy(occ, 0.0)
        out0, g0, _ = _train(fr, o, d, st, jc, jf, g, V, gs=True)
        fr.set_occupancy(occ, 0.0, place_samples=True)
        out1, g1, _ = _train(fr, o, d, st, jc, jf, g, V, gs=True)
    for k in out0:
        assert torch.equal(out0[k], out1[k]), k
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_deterministic_repeatable(small_mesh):
    V, C, field, params, fr, occ = _scene(small_mesh)
    fr.set_occupancy(occ, THR, place_samples=True)
    o, d = _rays()
    st, _ = _st(64, 64, True)
    jc, jf, g = _train_inputs(o, st)
    with _deterministic(True):
        out0, g0, _ = _train(fr, o, d, st, jc, jf, g, V)
        out1, g1, _ = _train(fr, o, d, st, jc, jf, g, V)
    for k in out0:
        assert torch.equal(out0[k], out1[k]), k
    for k in g0:
        assert torch.isfinite(g0[k]).all() and torch.equal(g0[k], g1[k]), k


# name: (num_samples, num_fine_samples, max_intersected_triangles, biased, rays)
EDGES = {"cap4": (24, 23, 4, True, 300), "cap2048": (64, 64, 2048, False, 300), "ceiling": (1750, 1750, 512, True, 8),
         "single_max": (4096, 0, 512, False, 8), "single_max_2048": (4096, 0, 2048, True, 8), "tiny_r1": (8, 8, 512, False, 1)}


@pytest.mark.parametrize("case", list(EDGES))
def test_settings_edges(small_mesh, case):
    Sc, Sf, M, biased, R = EDGES[case]
    V, C, field, params, fr, occ = _scene(small_mesh)
    fr.set_occupancy(occ, THR, place_samples=True)
    o, d = _rays(R)
    st, oc = _st(Sc, Sf, biased, M)
    out = _render(fr, o, d, st)
    ref = pl.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, oc, occupancy=(occ.cpu(), THR))
    e = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    print(f"{case}: max|rgb - oracle| {e:.2e}")
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"]) and e < 1e-4
    if Sf > 0:
        jc, jf, g = _train_inputs(o, st)
        outs, grads, _ = _train(fr, o, d, st, jc, jf, g, V)
        assert all(torch.isfinite(v).all() for v in grads.values())


def test_all_miss_batch_and_errors(small_mesh):
    V, C, field, params, fr, occ = _scene(small_mesh)
    fr.set_occupancy(occ, THR, place_samples=True)
    o = np.tile(np.array([[5, 5, 5]], np.float32), (16, 1))
    d = np.tile(np.array([[1, 0, 0]], np.float32), (16, 1))
    st, _ = _st(64, 64, True)
    out = _render(fr, o, d, st)
    assert not out["ray_mask"].any() and torch.equal(out["rgb"].cpu(), torch.ones(16, 3))
    with pytest.raises(RuntimeError, match="needs an occupancy"):
        fr.set_occupancy(None, THR, place_samples=True)


def test_model_occupancy_sampling(small_mesh):
    from test_gpu_occupancy import _model

    V, C = small_mesh
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    m, M = _model(V, C, field, params, occupancy_sampling=True, occupancy_warmup_steps=1)
    o, d = _rays(200)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    m.eval()
    with torch.no_grad():
        out = m(bundle)
    fr = m._fused
    st = fr_settings(m)
    want = fr.render(bundle.origins, bundle.directions, st)
    torch.cuda.synchronize()
    assert torch.equal(out["rgb"], want["rgb"])  # the model left placement on
    fr.set_occupancy(m.tetrahedra_occupancy, m.config.occupancy_threshold)
    plain = fr.render(bundle.origins, bundle.directions, st)
    assert not torch.equal(out["rgb"], plain["rgb"])
    sets = []
    orig_set = fr.set_occupancy
    fr.set_occupancy = lambda occ, thr=0.0, place_samples=False: (sets.append((occ is not None, place_samples)), orig_set(occ, thr, place_samples))[1]
    m.train()
    m._occ_step = 0
    for _ in range(3):
        r = m(bundle)
        (r["rgb"].sum() * 0).backward()
    assert sets == [(False, False), (True, True), (True, True)], sets
    bad = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), occupancy_sampling=True))
    with pytest.raises(RuntimeError, match="occupancy_sampling.*use_occupancy_field"):
        bad.eval().to(DEV)(bundle)


def fr_settings(m):
    from tetranerf.b200.render import RenderSettings

    c = m.config
    return RenderSettings(c.max_intersected_triangles, c.num_samples, c.num_fine_samples, c.use_biased_sampler, float(m.collider.far_plane))


@pytest.mark.parametrize("biased", [True, False])
def test_placement_beats_culling_at_64_64(biased):
    """the point of the feature: on surface_scene (k = 100), at 64 + 64 samples, mean |rgb - converged| is lower with placement than with
    culling only.  The converged reference is the culled single pass at 4096 samples; its distance to 2048 shows it has converged."""
    V, C = syn.delaunay_mesh(20000, seed=0)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr, fr, params = _setup(V, C, field, params)
    fr.set_mlp_precision(3)
    occ = _occ(fr, len(C))
    o, d = syn.camera_rays(2048, seed=5)
    fr.set_occupancy(occ, THR)
    ref = _render(fr, o, d, _st(4096, 0, biased)[0])["rgb"]
    half = _render(fr, o, d, _st(2048, 0, biased)[0])["rgb"]
    st = _st(64, 64, biased)[0]
    cull = _render(fr, o, d, st)["rgb"]
    fr.set_occupancy(occ, THR, place_samples=True)
    place = _render(fr, o, d, st)["rgb"]
    conv = (half - ref).abs().mean().item()
    e_cull, e_place = (cull - ref).abs().mean().item(), (place - ref).abs().mean().item()
    print(f"biased={biased}: mean|rgb - ref| culling {e_cull:.3e}, placement {e_place:.3e}; |Sc 2048 - Sc 4096| {conv:.3e}")
    assert conv < 0.2 * e_cull
    assert e_place < e_cull
