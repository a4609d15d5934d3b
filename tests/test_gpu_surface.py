"""GPU: the density iso-surface by marching tetrahedra (tn_surface_extract / FusedRenderer.extract_surface / TetrahedraNerf.extract_surface)
against the float64 oracle (oracle/surface.py), the analytic spheres of synthetic.surface_scene, the fused render, and itself."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import surface as osf
from tetranerf.b200 import synthetic as syn
from test_gpu_deterministic import _deterministic, _inputs, _step
from test_gpu_render import _from_ptr, setup

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LN2 = float(np.log(2.0))
KEYS = ("vertices", "normals", "colors", "faces", "face_tetrahedra")


def _host(surf):
    return {k: surf[k].cpu().numpy() for k in KEYS}


def _scene(V, k):
    if k is None:
        return syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)
    return syn.surface_scene(V, k, orc.init_mlp_params(0))


def _median_level(V, field, params):
    """a level at the median vertex density: the middle of the widest gap between the vertex densities around the median, so that no
    vertex sits on the level"""
    sig = np.sort(osf.network(params)[0](field.astype(np.float64).T))
    m = len(sig) // 2
    w = sig[m - 50:m + 51]
    i = int(np.argmax(np.diff(w)))
    return float((w[i] + w[i + 1]) / 2)


@pytest.mark.parametrize("k", [10, 100, 1000, None], ids=["k10", "k100", "k1000", "init"])
def test_surface_vs_oracle(small_mesh, k):
    """faces, face tetrahedra and vertex edges identical; positions within |edge| / 4096, normals 1e-4 rad, colours 1e-4 (at the kernel's
    positions and normals).  The torch-default network (k None) puts every vertex density into [0.63, 0.74]: on the 3000 points of
    small_mesh neighbouring densities near the median are ~2e-5 apart, less than the 1.4e-4 wide band around the level that must stay
    empty, so that case runs on 1000 points (widest gap near the median 1.6e-4)."""
    V, C = small_mesh if k is not None else syn.delaunay_mesh(1000, seed=0)
    field, params = _scene(V, k)
    level = LN2 if k is not None else _median_level(V, field, params)
    tr, fr, _, _ = setup(V, C, prec=2, field=field, params=params)  # the extraction runs bf16x3 whatever the render precision
    got = _host(fr.extract_surface(level))
    tr.synchronize()
    ref = osf.extract(V, C, field, params, level)
    near = np.abs(ref["vertex_sigma"] - level) <= 1e-4 * level
    assert not near.any(), f"{int(near.sum())} vertex densities within 1e-4 level of the level: the comparison would be ambiguous"
    assert len(ref["faces"]) > 100
    assert np.array_equal(got["faces"], ref["faces"]) and np.array_equal(got["face_tetrahedra"], ref["face_tetrahedra"])
    assert len(got["vertices"]) == len(ref["edges"])
    xa, xb = V[ref["edges"][:, 0]].astype(np.float64), V[ref["edges"][:, 1]].astype(np.float64)
    elen = np.linalg.norm(xb - xa, axis=1)
    p = got["vertices"].astype(np.float64)
    off_line = np.linalg.norm(np.cross(p - xa, xb - xa), axis=1) / elen**2  # each vertex sits on the oracle's edge of the same index
    assert off_line.max() < 1e-5, off_line.max()
    pos_err = np.linalg.norm(p - ref["vertices"], axis=1) / elen
    # normals and colours at the kernel's own positions (and normals), as the render tests compare at the kernel's own bins: a flat
    # density (the torch-default network) turns the bf16x3 density error into position error, which tilts small faces
    at = osf.extract(V, C, field, params, level, positions=got["vertices"], normals=got["normals"])
    ok = at["area"] >= 1e-12
    n = got["normals"].astype(np.float64)

    def angle(nr):
        return np.arctan2(np.linalg.norm(np.cross(n, nr), axis=1), np.sum(n * nr, axis=1))[ok]

    ang, ang_own = angle(at["normals"]), angle(ref["normals"])
    col_err = np.abs(got["colors"] - at["colors"]).max()
    print(f"k={k} level={level:.6f}: {len(p)} vertices, {len(got['faces'])} faces; max position error {pos_err.max():.3e} |edge| "
          f"(bound 1/4096 = {1 / 4096:.3e}); max normal angle {ang.max():.2e} rad at the kernel's positions, {ang_own.max():.2e} rad to "
          f"the oracle's own normals ({int((~ok).sum())} vertices with area < 1e-12 excluded); max colour error {col_err:.2e}")
    assert pos_err.max() <= 1 / 4096
    assert ang.max() <= 1e-4
    assert col_err <= 1e-4


@pytest.fixture(scope="module")
def cube45k():
    V, C = syn.delaunay_mesh(45_000, seed=0)
    field, params = syn.surface_scene(V, 1000, orc.init_mlp_params(0))
    tr, fr, _, _ = setup(V, C, field=field, params=params)
    surf = fr.extract_surface(LN2)
    tr.synchronize()
    return V, C, tr, fr, surf, field, params


def _check_closed_spheres(V, surf, label):
    """closed, consistently oriented, two components of Euler characteristic 2, on the spheres, outward"""
    s = _host(surf)
    top = osf.topology(s["faces"], len(s["vertices"]))
    print(f"{label}: {len(s['vertices'])} vertices, {len(s['faces'])} faces, components (V, E, F, chi) {top['components']}")
    assert top["directed_once"]
    assert len(top["components"]) == 2 and all(c[3] == 2 for c in top["components"])
    return s


def test_surface_analytic_spheres(cube45k):
    V, C, tr, fr, surf, field, params = cube45k
    s = _check_closed_spheres(V, surf, "45k points, k=1000")
    # every vertex within its edge's length of the analytic surface (the edge of a vertex: the shortest edge of its faces' tetrahedra
    # through it is not known here, so the bound is the longest edge of the tetrahedra around it)
    p = s["vertices"].astype(np.float64)
    tets = V[C[s["face_tetrahedra"]]].astype(np.float64)
    tsize = np.max([np.linalg.norm(tets[:, i] - tets[:, j], axis=1) for i in range(4) for j in range(i + 1, 4)], axis=0)
    vsize = np.zeros(len(p))
    for k in range(3):
        np.maximum.at(vsize, s["faces"][:, k], tsize)
    sdf = np.abs(syn.sphere_sdf(p))
    print(f"  max |sdf| {sdf.max():.3e}, max |sdf| / local edge length {(sdf / vsize).max():.3f}")
    assert (sdf <= vsize).all()
    # every face normal points from its tetrahedron's inside vertices to its outside ones (the winding rule)
    tri = p[s["faces"]]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    cells = C[s["face_tetrahedra"]]
    ins = (osf.network(params)[0](field.astype(np.float64).T) >= LN2)[cells]
    x = V[cells].astype(np.float64)
    c_in = np.sum(x * ins[..., None], 1) / ins.sum(1, keepdims=True)
    c_out = np.sum(x * ~ins[..., None], 1) / (~ins).sum(1, keepdims=True)
    assert (np.sum(n * (c_out - c_in), axis=1) > 0).all()
    # and outward from the spheres, away from the centre of the sphere whose surface is nearest, for all but a few faces: those lie in
    # sliver tetrahedra of the Delaunay mesh, where the inside -> outside direction runs almost tangent to the sphere and a small face
    # whose corners all lie within a few hundredths of an edge of the sphere can tilt past 90 degrees (the float64 oracle gives the same
    # faces: 30 of 16,514 = 0.18 % here; flat tetrahedra are counted)
    c = tri.mean(1)
    centres = np.array([cc for cc, _ in syn.SURFACE_SPHERES])
    radii = np.array([r for _, r in syn.SURFACE_SPHERES])
    which = np.argmin(np.abs(np.linalg.norm(c[:, None] - centres[None], axis=2) - radii), axis=1)
    outward = np.sum(n * (c - centres[which]), axis=1) > 0
    print(f"  outward faces {outward.mean() * 100:.3f} % ({int((~outward).sum())} of {len(outward)} not)")
    assert outward.mean() >= 0.995


def test_surface_agrees_with_render(cube45k):
    """rays from outside along -n at 200 surface vertices: the fused render's median depth is the vertex's distance up to one fine bin
    plus the local tetrahedron size (the bound of test_gpu_opaque.py)"""
    from tetranerf.b200.render import RenderSettings

    V, C, tr, fr, surf, _, _ = cube45k
    s = _host(surf)
    p, n =s["vertices"].astype(np.float64), s["normals"].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):  # origins just outside the unit cube (the mesh), on the vertex's normal line
        t_exit = np.nanmin(np.where(n > 0, (1.0 - p) / n, np.where(n < 0, -p / n, np.inf)), axis=1)
    L = t_exit + 0.05
    o = (p + L[:, None] * n).astype(np.float32)
    d = (-n).astype(np.float32)
    hits = syn.sphere_hits(o, d)[:, :, 0]
    first = np.min(np.where(np.isfinite(hits), hits, np.inf), axis=1)
    cand = np.nonzero(np.isfinite(first) & (np.abs(first - L) < 0.02) & (np.linalg.norm(n, axis=1) > 0.99))[0]  # nothing in front of it
    assert len(cand) >= 200
    sel = np.random.default_rng(0).choice(cand, 200, replace=False)
    L = L[sel]
    st = RenderSettings.tetra_nerf()
    fr.set_mlp_precision(3)
    out = fr.render(torch.from_numpy(o[sel]).to(DEV), torch.from_numpy(d[sel]).to(DEV), st)
    tr.synchronize()
    acc = out["accumulation"].cpu()[:, 0].numpy()
    dep = out["depth"].cpu()[:, 0].numpy().astype(np.float64)
    bufs = fr.debug_buffers()
    n_act = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    ray_list = _from_ptr(bufs["ray_list"], (n_act,), torch.int32).cpu().numpy()
    S2 = st.num_samples + st.num_fine_samples + 1
    eb = _from_ptr(bufs["ebins_f"], (n_act, S2 + 1), torch.float32).cpu().numpy().astype(np.float64)
    slot = np.full(len(sel), -1)
    slot[ray_list] = np.arange(n_act)
    assert (slot >= 0).all() and (acc > 0.5).all()
    width = np.array([np.diff(eb[slot[r]])[min(max(np.searchsorted(eb[slot[r]], dep[r]) - 1, 0), S2 - 1)] for r in range(len(sel))])
    tets = V[C[s["face_tetrahedra"]]].astype(np.float64)
    tsize = np.max([np.linalg.norm(tets[:, i] - tets[:, j], axis=1) for i in range(4) for j in range(i + 1, 4)], axis=0)
    vsize = np.zeros(len(s["vertices"]))
    for k in range(3):
        np.maximum.at(vsize, s["faces"][:, k], tsize)
    res = np.abs(dep - L)
    print(f"  median depth vs vertex distance on 200 rays: max {res.max():.3e}, max residual / (bin + tetrahedron) "
          f"{(res / (width + vsize[sel])).max():.3f}")
    assert (res <= width + vsize[sel]).all()


def test_surface_scale_closed():
    """the 2.02 M-tetrahedra mesh of bench.py --mode train: the extraction runs and the surface is closed"""
    V, C = syn.delaunay_mesh(300_000, seed=0)
    field, params = syn.surface_scene(V, 1000, orc.init_mlp_params(0))
    tr, fr, _, _ = setup(V, C, field=field, params=params)
    surf = fr.extract_surface(LN2)
    tr.synchronize()
    _check_closed_spheres(V, surf, f"{len(C)} tetrahedra, k=1000")


def test_surface_deterministic(small_mesh):
    V, C = small_mesh
    field, params = _scene(V, 100)
    tr, fr, _, _ = setup(V, C, field=field, params=params)
    a, b = fr.extract_surface(LN2), fr.extract_surface(LN2)
    tr.synchronize()
    for k in KEYS:
        assert a[k].shape == b[k].shape and a[k].numel() > 0
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


def test_surface_leaves_training_backward_alone(small_mesh):
    """deterministic mode: an extraction between a training forward and its backward leaves the gradients bitwise equal to a run
    without it, for the tracer-held state and the saved state"""
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    field, params = _scene(V, 100)
    st = RenderSettings.tetra_nerf()
    o, d = syn.camera_rays(256, seed=11)
    inp = _inputs(o, d, st, seed=8)
    tr, fr, _, _ = setup(V, C, field=field, params=params)
    ref = _step(fr, tr, len(V), st, inp, gs=True)
    ro, rd, jc, jf, target = inp
    R = ro.shape[0]
    with _deterministic(True):
        out = fr.train_forward(ro, rd, st, jc, jf)
        surf = fr.extract_surface(LN2)
        g_rgb = (2.0 * (out["rgb"] - target) / (3 * R)).contiguous()
        gf, gp = fr.train_backward(g_rgb, torch.full((R,), 0.05 / R, device=DEV), len(V), use_gradient_scaling=True)
        tr.synchronize()
        assert surf["faces"].shape[0] > 0
        assert torch.equal(out["rgb"], ref[0]["rgb"]) and torch.equal(gf, ref[1])
        for n in gp:
            assert torch.equal(gp[n], ref[2][n]), n
        # saved state: two forwards in flight, an extraction, then both backwards
        out1, s1 = fr.train_forward_saved(ro, rd, st, jc, jf)
        out2, s2 = fr.train_forward_saved(ro, rd, st, jc, jf)
        fr.extract_surface(LN2)
        for outk, sk in ((out2, s2), (out1, s1)):
            g = (2.0 * (outk["rgb"] - target) / (3 * R)).contiguous()
            gfk, gpk = fr.train_backward_saved(sk, g, torch.full((R,), 0.05 / R, device=DEV), len(V), use_gradient_scaling=True)
            tr.synchronize()
            assert torch.equal(gfk, ref[1])
            for n in gpk:
                assert torch.equal(gpk[n], ref[2][n]), n


def test_surface_errors_and_empty(small_mesh):
    V, C = small_mesh
    field, params = _scene(V, 100)
    tr, fr, _, _ = setup(V, C, field=field, params=params)
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="level"):
            fr.extract_surface(bad)
    sig = osf.network(params)[0](field.astype(np.float64).T)
    for level in (float(sig.max()) * 2.0, float(sig.min()) / 2.0):
        s = fr.extract_surface(level)
        assert all(s[k].shape[0] == 0 for k in KEYS), level
        assert s["faces"].shape == (0, 3) and s["faces"].dtype == torch.int32
    s = fr.extract_surface(LN2)
    assert s["faces"].shape[0] > 0
    fr.set_weights(params)
    with pytest.raises(RuntimeError, match="changed"):
        fr.copy_surface(s)
    fr.extract_surface(LN2)
    fr.set_field(torch.from_numpy(field).to(DEV))
    with pytest.raises(RuntimeError, match="changed"):
        fr.copy_surface(s)
    fr.extract_surface(LN2)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    with pytest.raises(RuntimeError, match="changed"):
        fr.copy_surface(s)
    tr.synchronize()


def test_model_extract_surface(small_mesh):
    """TetrahedraNerf.extract_surface: the fused renderer's extraction of the model's field and weights; a config off the fused path
    raises naming the option"""
    from tetranerf.b200.render import FusedRenderer
    from tetranerf.nerfstudio import model as M

    V, C = small_mesh
    field, params = _scene(V, 1000)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(params)
    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C)))
    m.load_state_dict(sd, strict=False)
    m = m.to(DEV)
    got = m.extract_surface(LN2)
    assert not any(t.requires_grad for t in got.values())
    tr, fr, _, _ = setup(V, C, field=field, params=params)
    want = fr.extract_surface(LN2)
    tr.synchronize()
    for k in KEYS:
        assert torch.equal(got[k], want[k]), k
    bad = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), hidden_size=64)).to(DEV)
    with pytest.raises(RuntimeError, match="hidden_size=64"):
        bad.extract_surface(LN2)
    assert isinstance(m._fused, FusedRenderer)
