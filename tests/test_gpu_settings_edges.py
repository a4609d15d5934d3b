"""GPU parity of the fused render and training step at the edges of the settings the C ABI accepts: num_samples 1 ... 4096,
num_fine_samples 0 ... 4096, max_ray_triangles (M) 2 ... 2048, tiny batches.  The other parity tests run S2 = Sc + Sf + 1 (fine samples
per ray) between 41 and 513 and M in {128, 256, 512}; the per-ray kernels and the MLP kernels branch on these sizes:

* S2 < 16: one 16-row warp block of the MLP backward holds several rays, so its per-ray direction-bias sums run over more than the two
  rays at a boundary (default mode), and the deterministic mode writes several partial rows per block (k_det_dirbias);
* S2 >> 64: one ray spans dozens of 64-row tiles;
* M = 4 truncates almost every ray (the exact trace stage); M = 2048 is the largest staging of the biased coarse sampler;
* S2 at the shared-memory ceiling of k_sample_fine (16 (M + 4 S2 + 10) bytes per 4-warp block), and one past it, where the call must
  fail as an argument error and leave the tracer usable;
* M = 2 keeps no tetrahedron on any ray: an all-empty batch through every kernel of both modes;
* R = 1 and batches that are not multiples of the 4-warp per-ray blocks or of the quad walk's 8 rays per warp.

Bars are those of test_gpu_render.py / test_gpu_train.py, and the pixels are also held against the float64 oracle at the kernel's own
fine bins."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _assert_bitwise, _deterministic, _inputs, _step
from test_gpu_render import _from_ptr, setup
from test_gpu_train import _run

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BG = (0.1, 0.6, 0.3)

# name: (num_samples, num_fine_samples, max_intersected_triangles, biased sampler, rays)
CASES = {
    "one_sample": (1, 0, 512, False, 300),    # single pass, 64 rays per MLP tile
    "s2_3": (1, 1, 512, True, 300),           # linspace with 2 steps, a PDF over one bin, 5-6 rays per 16-row block
    "s2_16": (7, 8, 512, False, 300),         # one ray per 16-row block exactly
    "s2_64": (31, 32, 256, True, 300),        # each 64-row tile is exactly one ray
    "cap4": (24, 23, 4, True, 300),           # at most 2 cells per ray: truncation on nearly every ray
    "cap2048": (64, 64, 2048, True, 300),     # largest per-segment staging
    "large": (1024, 1024, 512, False, 24),    # S2 = 2049: one ray spans 33 tiles
    "ceiling": (1750, 1750, 512, True, 8),    # S2 = 3501: the largest k_sample_fine fits at M = 512 on an H100 (232,448 B per block)
    "single_max": (4096, 0, 512, True, 8),    # largest single pass
    "tiny_r1": (8, 8, 512, False, 1),         # S2 = 17: the whole call sits in one partly filled 64-row tile
    "tiny_r3": (8, 8, 512, False, 3),
    "tiny_r5": (8, 8, 512, False, 5),         # not a multiple of the 4-warp per-ray blocks
}
_MESH = {}
_ORACLE = {}


def _mesh(V, C):
    if "small" not in _MESH:
        _MESH["small"] = orc.OracleMesh(V, C)
    return _MESH["small"]


def _settings(Sc, Sf, M, biased, bg=(1.0, 1.0, 1.0)):
    from tetranerf.b200.render import RenderSettings

    kw = dict(num_samples=Sc, num_fine_samples=Sf, max_intersected_triangles=M, use_biased_sampler=biased, background=bg)
    return RenderSettings(**kw), orc.RenderConfig(**kw)


def _rays(R, seed=11):
    o, d = syn.camera_rays(R, seed=seed)
    if R >= 8:
        o[5] = [5, 5, 5]; d[5] = [1, 0, 0]  # empty ray
    return o, d


def _s2_max(M, optin):
    """largest S2 whose per-ray kernels fit the opt-in shared memory: k_sample_fine (16 (M + 4 S2 + 10) bytes) and k_composite_bwd
    (64 (S2 + 2) bytes)"""
    return min((optin // 16 - M - 10) // 4, optin // 64 - 2)


def _render_parity(V, C, field, params, o, d, st, oc, out, bufs, what, oracle_key=None):
    """the bars of test_fused_render_vs_oracle, plus the pixels against the float64 oracle at the kernel's own fine bins (two-pass)"""
    single = st.num_fine_samples == 0
    if oracle_key is not None and oracle_key in _ORACLE:
        ref = _ORACLE[oracle_key]
    else:
        ref = orc.render(_mesh(V, C), torch.from_numpy(field), params, o, d, oc, return_aux=True)
        if oracle_key is not None:
            _ORACLE[oracle_key] = ref
    R = len(o)
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"]), what
    n_act = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    assert n_act == int(ref["ray_mask"].sum()) and n_act > 0
    ray_list = _from_ptr(bufs["ray_list"], (n_act,), torch.int32).cpu().long()
    active = torch.nonzero(ref["ray_mask"]).flatten()
    inv = torch.empty(R, dtype=torch.long)
    inv[active] = torch.arange(n_act)
    order = inv[ray_list]  # row of the oracle's compacted arrays for each slot
    Sc = st.num_samples
    S2 = Sc if single else Sc + st.num_fine_samples + 1
    aux = ref["aux"]
    eb_c = _from_ptr(bufs["ebins_c"], (n_act, Sc + 1), torch.float32).cpu()
    torch.testing.assert_close(eb_c, (aux["fine_euclid"] if single else aux["coarse_euclid"])[order], rtol=2e-6, atol=2e-6)
    if not single:
        dens = _from_ptr(bufs["dens_c"], (n_act, Sc), torch.float32).cpu()
        assert (dens - aux["coarse_density"][order][..., 0]).abs().max().item() < 1e-4
        eb_f = _from_ptr(bufs["ebins_f"], (n_act, S2 + 1), torch.float32).cpu()
        torch.testing.assert_close(eb_f, aux["fine_euclid"][order], rtol=1e-4, atol=1e-4)
    outf = _from_ptr(bufs["out_f"], (n_act, S2, 4), torch.float32).cpu()
    vi_gpu = _from_ptr(bufs["vi_c" if single else "vi_f"], (n_act, S2, 4), torch.int32).cpu()
    vi_ref = torch.from_numpy(aux["matched"]["vertex_indices"])[order]
    flipped = (vi_gpu != vi_ref).any(-1)
    sig_ref = aux["sigmas"][order][..., 0]
    sig_err = (outf[..., 0] - sig_ref).abs()
    col_err = (outf[..., 1:] - aux["colors"][order]).abs().amax(-1)
    flip_rate = flipped.float().mean().item()
    ok = ~flipped
    e_sig = sig_err[ok].max().item()
    e_col = col_err[ok].max().item()
    assert flip_rate < 2e-3, (what, flip_rate, int(flipped.sum()))
    assert bool((sig_err[ok] <= 1e-4 + 2e-5 * sig_ref[ok].abs()).all()), (what, e_sig)
    assert e_col <= 1e-4, (what, e_col)
    e_rgb = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"]).abs().max().item()
    e_dep = (out["depth"].cpu() - ref["depth"]).abs()
    msg = (f"{what}: per sample sigma {e_sig:.2e} colour {e_col:.2e} flipped {int(flipped.sum())}/{flipped.numel()}  pixels rgb {e_rgb:.2e} "
           f"acc {e_acc:.2e} depth > 1e-4: {int((e_dep > 1e-4).sum())}")
    assert e_rgb < 1e-4 and e_acc < 1e-4, msg
    assert (e_dep.flatten() > 1e-4).sum().item() <= max(2, R // 100), msg
    if not single:  # float64 at the kernel's own fine bins (ray order of the non-empty rays)
        fine = eb_f[torch.argsort(ray_list)]
        torch.set_default_dtype(torch.float64)
        try:
            r64 = orc.render_train(_mesh(V, C), torch.from_numpy(field).double(), {k: v.double() for k, v in params.items()}, o, d, oc,
                                   fine_euclid=fine)
        finally:
            torch.set_default_dtype(torch.float32)
        e64_rgb = (out["rgb"].cpu().double() - r64["rgb"]).abs().max().item()
        e64_acc = (out["accumulation"].cpu().double() - r64["accumulation"]).abs().max().item()
        msg += f"  vs float64 at the kernel's bins: rgb {e64_rgb:.2e} acc {e64_acc:.2e}"
        assert e64_rgb < 1e-4 and e64_acc < 1e-4, msg
    print(msg)


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("case", list(CASES))
def test_render_vs_oracle_at_the_edges(small_mesh, case, prec):
    V, C = small_mesh
    Sc, Sf, M, biased, R = CASES[case]
    st, oc = _settings(Sc, Sf, M, biased)
    o, d = _rays(R)
    tr, fr, field, params = setup(V, C, prec=prec)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    tr.synchronize()
    _render_parity(V, C, field, params, o, d, st, oc, out, fr.debug_buffers(), f"{case}/prec={prec}", oracle_key=case)
    if case == "cap4":  # n <= M - 2 = 2 cells on every ray, and most rays cross more
        num = tr.trace_rays(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), 512)["num_visited_cells"]
        tr.synchronize()
        assert (num > 2).float().mean().item() > 0.9


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("case,gs", [("s2_3", False), ("s2_16", True), ("cap4", False), ("large", True), ("ceiling", False), ("tiny_r3", True)])
def test_train_step_at_the_edges(small_mesh, case, gs, det):
    """the bar of test_fused_train_step_gradients per tensor; mlp_head.layers.0.{weight,bias} is fed by the per-ray direction-bias
    gradient (k_mlp_bwd's per-ray sums, k_det_dirbias)"""
    V, C = small_mesh
    Sc, Sf, M, biased, R = CASES[case]
    st, oc = _settings(Sc, Sf, M, biased)
    o, d = _rays(R)
    print(f"--- {case}, deterministic {det}, gradient scaling {gs}")
    with _deterministic(det):
        fr, tr = _run(V, C, o, d, st, oc, gs, seed=5, mesh=_mesh(V, C))
    if det and case in ("s2_3", "large"):
        inp = _inputs(o, d, st, seed=6)
        a = _step(fr, tr, len(V), st, inp, gs)
        _assert_bitwise(a, _step(fr, tr, len(V), st, inp, gs), f"{case}: two deterministic runs")
        for ctas in (1, 7):
            fr.set_backward_grid(ctas)
            _assert_bitwise(a, _step(fr, tr, len(V), st, inp, gs), f"{case}: backward grid {ctas} vs default grid")
        fr.set_backward_grid(0)


def _empty_batch(kind):
    """cap2: camera rays that cross the mesh with max_intersected_triangles = 2 (no ray keeps a tetrahedron); miss: rays that all
    miss the mesh, default settings"""
    from tetranerf.b200.render import RenderSettings

    if kind == "cap2":
        st, _ = _settings(32, 32, 2, True, BG)
        o, d = syn.camera_rays(37, seed=3)
    else:
        st = RenderSettings.tetra_nerf()
        st.background = BG
        rng = np.random.default_rng(5)
        o = (np.array([5.0, 5.0, 5.0]) + rng.random((37, 3))).astype(np.float32)
        d = np.tile(np.array([[1.0, 0.0, 0.0]], np.float32), (37, 1))
    return st, o, d


@pytest.mark.parametrize("kind", ["cap2", "miss"])
def test_all_empty_batch(small_mesh, kind):
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    st, o, d = _empty_batch(kind)
    R = len(o)
    tr, fr, field, params = setup(V, C)
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    num = tr.trace_rays(ot, dt, 512)["num_visited_cells"]
    tr.synchronize()
    if kind == "cap2":
        assert bool((num > 0).all())  # every ray really crosses the mesh
    else:
        assert bool((num == 0).all())
    bg = torch.tensor(BG, dtype=torch.float32, device=DEV).expand(R, 3)
    far = torch.full((R, 1), st.far_plane, dtype=torch.float32, device=DEV)

    def assert_empty(out, what):
        assert torch.equal(out["rgb"], bg), what
        assert bool((out["accumulation"] == 0).all()), what
        assert torch.equal(out["depth"], far), what
        assert not bool(out["ray_mask"].any()), what
        if "expected_depth" in out:
            assert torch.equal(out["expected_depth"], far), what
        if "normals" in out:
            assert bool((out["normals"] == 0).all()), what

    out = fr.render(ot, dt, st, normals=True, expected_depth=True)
    tr.synchronize()
    assert_empty(out, "eval")
    xyz = tr._vertices
    for det in (False, True):
        g = torch.Generator().manual_seed(2)
        jc = torch.rand((R, st.num_samples + 1), generator=g).to(DEV)
        jf = torch.rand((R, st.num_fine_samples + 1), generator=g).to(DEV)
        with _deterministic(det):
            out, state = fr.train_forward_saved(ot, dt, st, jc, jf, expected_depth=True)
            grads = fr.train_backward_saved(state, torch.rand((R, 3), generator=g).to(DEV), torch.rand((R,), generator=g).to(DEV), len(V),
                                            use_gradient_scaling=True, grad_origins=True, grad_directions=True, grad_vertices=True,
                                            grad_expected_depth=torch.rand((R,), generator=g).to(DEV))
        tr.synchronize()
        assert_empty(out, f"training forward, deterministic {det}")
        gfield, gp, go, gd, gv = grads
        named = {"tetrahedra_field": gfield, **gp, "origins": go, "directions": gd, "vertices": gv}
        assert len(named) == 16 and gv.shape == xyz.shape
        for n, t in named.items():
            assert bool(torch.isfinite(t).all()) and bool((t == 0).all()), f"deterministic {det}: {n} gradient is not 0"
    # the tracer is as good as a fresh one afterwards
    st_r = RenderSettings.tetra_nerf()
    st_r.background = BG
    o2, d2 = _rays(300, seed=12)
    inp = _inputs(o2, d2, st_r, seed=6)
    results = []
    for t, f in ((tr, fr), setup(V, C)[:2]):
        out = f.render(inp[0], inp[1], st_r, normals=True, expected_depth=True)
        out = {k: v.clone() for k, v in out.items()}
        t.synchronize()
        results.append((out, _step(f, t, len(V), st_r, inp, True)))
    for k in results[0][0]:
        assert torch.equal(results[0][0][k], results[1][0][k]), k
    assert bool(results[0][0]["ray_mask"].any())
    _assert_bitwise(results[0][1], results[1][1], "after an all-empty batch vs a fresh tracer")


@pytest.mark.parametrize("M", [512, 2048])
def test_shared_memory_ceiling(small_mesh, M):
    """the largest S2 that fits the device's opt-in shared memory runs (M = 512 is the "ceiling" parity case above; M = 2048 is held to
    the same bars here); one past it the eval render, the training forward and the saved-state forward raise an argument error, and
    the tracer's next call is exactly a fresh tracer's"""
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    optin = torch.cuda.get_device_properties(DEV).shared_memory_per_block_optin
    s2 = _s2_max(M, optin)
    Sc = (s2 - 1) // 2
    Sf = s2 - 1 - Sc
    print(f"opt-in shared memory {optin} B: S2 <= {s2} at M = {M} (num_samples {Sc} + num_fine_samples {Sf})")
    o, d = _rays(8, seed=13)
    if M == 2048:
        st, oc = _settings(Sc, Sf, M, True)
        tr, fr, field, params = setup(V, C)
        out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
        tr.synchronize()
        _render_parity(V, C, field, params, o, d, st, oc, out, fr.debug_buffers(), f"S2 = {s2} at M = {M}")
        _run(V, C, o, d, st, oc, False, seed=7, mesh=_mesh(V, C))
    over = RenderSettings(num_samples=Sc + 1, num_fine_samples=Sf, max_intersected_triangles=M, use_biased_sampler=True)
    ok = RenderSettings(num_samples=64, num_fine_samples=64, max_intersected_triangles=M, use_biased_sampler=True)
    tr, fr, _, _ = setup(V, C)
    ot, dt = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    with pytest.raises(RuntimeError, match="shared-memory limit"):
        fr.render(ot, dt, over)
    with pytest.raises(RuntimeError, match="shared-memory limit"):
        fr.train_forward(ot, dt, over)
    with pytest.raises(RuntimeError, match="shared-memory limit"):
        fr.train_forward_saved(ot, dt, over)
    a = fr.render(ot, dt, ok)
    tr.synchronize()
    tr2, fr2, _, _ = setup(V, C)
    b = fr2.render(ot, dt, ok)
    tr2.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k
