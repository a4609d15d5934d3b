"""CPU: the float64 normal-map oracle (oracle/normals.py) against finite differences of the density, the NormalsRenderer restatement,
the config default and the "normals" metrics image, and the operand-rounding emulation that predicts the kernel's per-sample error."""
import numpy as np
import pytest
import torch

from oracle import normals as onm
from oracle import oracle as orc
from oracle import second_opinion as so
from tetranerf.b200 import synthetic as syn
from tetranerf.nerfstudio import model as M


def _inside_samples(V, C, n, seed=0, margin=0.1):
    """n samples strictly inside random tetrahedra (every weight >= margin): (vi [n,4], bary [n,3] on v1..v3, points [n,3] float64)"""
    rng = np.random.default_rng(seed)
    cells = C[rng.integers(0, len(C), n)]
    w = margin + (1 - 4 * margin) * rng.dirichlet(np.ones(4), n)
    X = V.astype(np.float64)
    pts = np.einsum("nk,nkc->nc", w, X[cells])
    return cells.astype(np.int64), w[:, 1:], pts


def _sigma_plain(params, field, V, cell, x):
    """sigma at point x of tetrahedron `cell`, from the definition: barycentric solve in float64, interpolation, plain-loop MLP"""
    X = V.astype(np.float64)[cell]
    b = np.linalg.solve((X[1:] - X[0]).T, x - X[0])
    F = field.astype(np.float64)[:, cell].T
    f = F[0] + b @ (F[1:] - F[0])
    return so.mlp_forward(params, f[None], [0.0] * 27)[0][0]


@pytest.mark.parametrize("scene", ["default", "surface100"])
def test_gradient_matches_finite_differences(small_mesh, scene):
    V, C = small_mesh
    if scene == "default":
        field, params = syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)
    else:
        field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    vi, bary, pts = _inside_samples(V, C, 60)
    ref = onm.grad_pre(vi, bary, V, field, params, kappa=1e-6)
    sig = lambda z: 1.0 / (1.0 + np.exp(-z))  # noqa: E731  softplus'
    checked = 0
    for i in range(len(vi)):
        if ref["ambiguous"][i]:  # a ReLU kink within reach of the difference step
            continue
        h = 1e-6 * np.abs(ref["det"][i]) ** (1 / 3)
        fd = np.array([(_sigma_plain(params, field, V, vi[i], pts[i] + h * e) - _sigma_plain(params, field, V, vi[i], pts[i] - h * e)) / (2 * h)
                       for e in np.eye(3)])
        want = sig(ref["pre"][i]) * ref["grad"][i]
        assert np.linalg.norm(fd - want) <= 1e-5 * np.linalg.norm(want) + 1e-9, (i, fd, want)
        checked += 1
    assert checked >= 50


def test_oracle_is_the_inverse_transpose_and_handles_degenerate_samples():
    V, C = syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()
    field, params = syn.random_field(len(V), 64, seed=1), orc.init_mlp_params(0)
    vi = np.array([C[0], C[3], [-1, -1, -1, -1], [0, 1, 2, 3]])  # the last: four coplanar cube corners (det 0)
    bary = np.full((4, 3), 0.2)
    r = onm.grad_pre(vi, bary, V, field, params)
    E = np.stack([V[vi[0, k]].astype(np.float64) - V[vi[0, 0]] for k in (1, 2, 3)], -1)
    assert np.allclose(r["grad"][0], np.linalg.solve(E.T, r["q"][0]))
    assert not np.allclose(r["grad"][0], np.linalg.solve(E, r["q"][0]))  # E^-1 q is another vector
    assert np.all(r["grad"][2] == 0) and np.all(r["grad"][3] == 0) and r["det"][3] == 0
    n = onm.sample_normals(r["grad"])
    assert np.allclose(np.linalg.norm(n[:2], axis=-1), 1) and np.all(n[2:] == 0)
    assert np.allclose(n[0], -r["grad"][0] / np.linalg.norm(r["grad"][0]))


def test_normals_renderer_restatement():
    """NormalsRenderer(normalize=True): sum w n, then n / sqrt(max(|n|^2, 1e-20)); empty rays and |N| -> 0 stay finite"""
    w = np.array([[0.5, 0.5, 0.0], [0.0, 0.0, 0.0], [0.5, 0.5, 0.0], [0.2, 0.1, 0.0]])
    n = np.zeros((4, 3, 3))
    n[0, 0], n[0, 1] = [1, 0, 0], [0, 1, 0]
    n[2, 0], n[2, 1] = [0, 0, 1], [0, 0, -1]   # opposite normals: |N| = 0
    n[3, 0], n[3, 1] = [0, 1, 0], [0, 1, 0]
    s, u = onm.composite(w, n)
    assert np.allclose(s[0], [0.5, 0.5, 0]) and np.allclose(u[0], [2**-0.5, 2**-0.5, 0])
    assert np.all(s[1] == 0) and np.all(u[1] == 0)
    assert np.all(np.isfinite(u)) and np.all(u[2] == 0)
    assert np.allclose(u[3], [0, 1, 0])
    t = torch.from_numpy(s)  # nerfstudio's safe_normalize
    assert np.allclose(u, (t / torch.sqrt(torch.clamp(torch.sum(t * t, -1, keepdim=True), min=1e-20))).numpy())


def test_config_default_and_metrics_image():
    c = M.TetrahedraNerfConfig(num_tetrahedra_vertices=10, num_tetrahedra_cells=5)
    assert c.render_normals is False
    m = M.TetrahedraNerf(c)
    img = torch.rand((32, 32, 3))
    out = {"rgb": img, "accumulation": torch.ones((32, 32, 1)), "depth": torch.ones((32, 32, 1))}
    _, images = m.get_image_metrics_and_images(out, {"image": img})
    assert "normals" not in images
    nrm = torch.nn.functional.normalize(torch.randn((32, 32, 3)), dim=-1)
    _, images = m.get_image_metrics_and_images({**out, "normals": nrm}, {"image": img})
    assert torch.allclose(images["normals"], (nrm + 1) / 2) and images["normals"].min() >= 0 and images["normals"].max() <= 1


def test_render_normals_on_an_unsupported_configuration_raises():
    """render_normals needs the fused pipeline: in eval an unsupported configuration raises before any device work, naming the option"""
    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=10, num_tetrahedra_cells=5, hidden_size=64, render_normals=True))
    m.eval()
    bundle = M.RayBundle(origins=torch.zeros((4, 3)), directions=torch.tensor([[0.0, 1.0, 0.0]]).expand(4, 3).contiguous())
    with pytest.raises(RuntimeError, match="hidden_size=64"):
        with torch.no_grad():
            m.get_outputs(bundle)


@pytest.mark.parametrize("scene", ["default", "surface10", "surface1000"])
def test_operand_rounding_predicts_the_per_sample_error(small_mesh, scene):
    """the reverse chain with the kernel's operand rounding: the predicted per-sample error of each precision lies inside the GPU
    test's bars (1e-3 bf16x3, 5e-2 f16w2), on samples outside the mask-ambiguity band.  Over these 4000 samples the maxima are ~1e-4 and
    ~4e-3 (asserted below 3e-4 and 2e-2); the maximum is a heavy tail that grows with the sample count (2.6e-4 and 2.4e-2 over 80,000),
    because q = g . (F_vk - F_v0) cancels.  f16w2 rounds each cotangent to fp16 (2^-11 relative)."""
    V, C = small_mesh
    if scene == "default":
        field, params = syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0)
    else:
        field, params = syn.surface_scene(V, int(scene[7:]), orc.init_mlp_params(0))
    vi, bary, _ = _inside_samples(V, C, 4000, seed=2, margin=0.0)
    for prec, bar, kappa in ((3, 3e-4, 2.0**-14), (2, 2e-2, 2.0**-11)):
        ref = onm.grad_pre(vi, bary, V, field, params, kappa=kappa)
        err = onm.error_measure(onm.emulate_grad_pre(vi, bary, V, field, params, prec), ref)[~ref["ambiguous"]]
        print(f"{scene} prec={prec}: predicted error max {err.max():.2e} p99 {np.percentile(err, 99):.2e} median {np.median(err):.2e}, "
              f"ambiguous {ref['ambiguous'].mean() * 100:.2f} %")
        assert err.max() <= bar, (prec, err.max())
