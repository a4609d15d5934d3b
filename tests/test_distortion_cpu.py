"""CPU: the distortion loss (DESIGN §4.11).  The model's O(S) prefix-sum form (model.distortion_per_ray, the unfused path) against the
literal O(S^2) double sum in float64 (oracle/distortion.py), its autograd gradient against the closed form, the oracle's training
render against central differences on a tiny mesh, and the model's distortion_loss."""
import math

import numpy as np
import pytest
import torch

from oracle import distortion as dso
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from tetranerf.nerfstudio import model as M


def _case(R, S2, seed, kind="random"):
    """weights [R,S2,1] float64 (get_weights-like: sum <= 1) and sorted spacing bins [R,S2+1] in [0,1]"""
    g = torch.Generator().manual_seed(seed)
    s = torch.sort(torch.rand((R, S2 + 1), generator=g, dtype=torch.float64), -1)[0]
    s[:, 0], s[:, -1] = 0.0, 1.0
    if kind == "zero":
        w = torch.zeros((R, S2), dtype=torch.float64)
    elif kind == "onehot":
        w = torch.zeros((R, S2), dtype=torch.float64)
        w[torch.arange(R), torch.randint(0, S2, (R,), generator=g)] = torch.rand(R, generator=g, dtype=torch.float64)
    else:
        w = torch.rand((R, S2), generator=g, dtype=torch.float64) ** 4
        w = w / w.sum(-1, keepdim=True) * torch.rand((R, 1), generator=g, dtype=torch.float64)
    return w[..., None], s


def _closed_form(w, s):
    """2 sum_i w_i |u_j - u_i| + 2/3 w_j delta_j, by the O(S^2) sum"""
    w = w[..., 0]
    u = (s[:, 1:] + s[:, :-1]) / 2
    delta = s[:, 1:] - s[:, :-1]
    return 2 * torch.einsum("rij,ri->rj", (u[:, :, None] - u[:, None, :]).abs(), w) + 2.0 / 3.0 * w * delta


@pytest.mark.parametrize("kind", ["random", "zero", "onehot"])
@pytest.mark.parametrize("S2", [1, 2, 3, 17, 257, 3501])
def test_prefix_sum_form_equals_the_definition(S2, kind):
    R = 4 if S2 > 1000 else 24
    w, s = _case(R, S2, seed=S2, kind=kind)
    want = dso.distortion(w, s)
    got64 = M.distortion_per_ray(w, s)
    # the float32 form against the definition at its own (float32-rounded) inputs: the arithmetic alone
    want32 = dso.distortion(w.float().double(), s.float().double())
    got32 = M.distortion_per_ray(w.float(), s.float()).double()
    scale = max(want.abs().max().item(), 1e-30)
    print(f"S2 {S2} {kind}: max d {want.max().item():.3e}, float64 form {((got64 - want).abs().max() / scale).item():.1e}, "
          f"float32 form {((got32 - want32).abs().max() / scale).item():.1e} of the largest d")
    assert got64.shape == (R, 1)
    if kind == "zero":
        assert torch.all(got64 == 0) and torch.all(got32 == 0) and torch.all(want == 0)
        return
    assert torch.all(want >= 0)
    torch.testing.assert_close(got64, want, rtol=1e-12, atol=1e-14 * scale)
    assert ((got32 - want32).abs() <= 2e-5 * scale + 1e-6 * want32.abs()).all()
    if kind == "onehot":  # only the sample's own term: w^2 delta / 3
        wk = w[..., 0].sum(-1)
        k = w[..., 0].argmax(-1)
        delta = (s[:, 1:] - s[:, :-1])[torch.arange(R), k]
        torch.testing.assert_close(want[:, 0], wk * wk * delta / 3, rtol=1e-12, atol=0.0)


@pytest.mark.parametrize("S2", [1, 3, 17, 257])
def test_prefix_sum_gradient_equals_the_closed_form(S2):
    w, s = _case(16, S2, seed=100 + S2)
    g_out = torch.linspace(0.5, 2.0, 16, dtype=torch.float64)[:, None]
    wr = w.clone().requires_grad_(True)
    (M.distortion_per_ray(wr, s) * g_out).sum().backward()
    want = g_out * _closed_form(w, s)
    torch.testing.assert_close(wr.grad[..., 0], want, rtol=1e-11, atol=1e-14)
    # the oracle's backward is the same closed form
    wo = w.clone().requires_grad_(True)
    (dso.distortion(wo, s) * g_out).sum().backward()
    torch.testing.assert_close(wo.grad[..., 0], want, rtol=1e-12, atol=1e-15)
    # and a central difference of the definition agrees with it
    h = 1e-7
    for j in range(0, S2, max(1, S2 // 5)):
        e = torch.zeros_like(w)
        e[:, j] = h
        fd = ((dso.distortion(w + e, s) - dso.distortion(w - e, s)) * g_out).sum() / (2 * h)
        assert abs(fd.item() - want[:, j].sum().item()) <= 1e-6 * max(1.0, abs(fd.item())), j


def test_render_train_distortion_matches_central_differences():
    """float64 training render on a tiny mesh at fixed fine bins: d(sum_r c_r d_r) by autograd against central differences in the field,
    an MLP weight, the ray origins / directions and the vertex positions"""
    V, C = syn.delaunay_mesh(200, seed=1)
    mesh = orc.OracleMesh(V, C)
    field = torch.from_numpy(syn.random_field(len(V), 64, seed=3)).double()
    params = {k: v.double() for k, v in orc.init_mlp_params(0).items()}
    o, d = syn.camera_rays(12, seed=11)
    o[2] = [5, 5, 5]; d[2] = [1, 0, 0]  # empty ray
    cfg = orc.RenderConfig(num_samples=16, num_fine_samples=15, use_biased_sampler=True)
    g = torch.Generator().manual_seed(4)
    jc, jf = torch.rand((12, 17), generator=g), torch.rand((12, 16), generator=g)
    cw = torch.linspace(0.5, 1.5, 12, dtype=torch.float64)[:, None]
    torch.set_default_dtype(torch.float64)
    try:
        ot, dt = torch.from_numpy(o).double(), torch.from_numpy(d).double()
        first = dso.render_train_distortion(mesh, field, params, ot, dt, V, cfg, jc, jf)
        fine, sb = first["aux"]["fine_euclid"], first["aux"]["sbins"]

        def loss(f, p, oo, dd, xyz):
            out = dso.render_train_distortion(mesh, f, p, oo, dd, xyz, cfg, fine_euclid=fine, fine_sbins=sb, exact_bary=True)
            return (out["distortion"] * cw).sum(), out

        leaves = {"field": field.clone().requires_grad_(True), "w1": params["mlp_base.layers.0.weight"].clone().requires_grad_(True),
                  "origins": ot.clone().requires_grad_(True), "directions": dt.clone().requires_grad_(True),
                  "vertices": torch.from_numpy(V).double().requires_grad_(True)}

        def run(lv):
            p = dict(params)
            p["mlp_base.layers.0.weight"] = lv["w1"]
            return loss(lv["field"], p, lv["origins"], lv["directions"], lv["vertices"])

        L, out = run(leaves)
        L.backward()
        assert out["distortion"][2, 0].item() == 0.0 and L.item() > 0
        worst = 0.0
        for name, t in leaves.items():
            # a ray or a vertex moves many samples at once: steps of 1e-8, as larger ones move some hidden pre-activations across the
            # ReLU kink (test_ray_grads_cpu.py)
            h = 1e-6 if name in ("field", "w1") else 1e-8
            grad = t.grad
            flat = grad.abs().flatten()
            picks = torch.argsort(flat, descending=True)[:4].tolist()
            for i in picks:
                plus = {k: v.detach().clone() for k, v in leaves.items()}
                minus = {k: v.detach().clone() for k, v in leaves.items()}
                plus[name].view(-1)[i] += h
                minus[name].view(-1)[i] -= h
                fd = (run(plus)[0].item() - run(minus)[0].item()) / (2 * h)
                err = abs(fd - grad.view(-1)[i].item())
                worst = max(worst, err / flat.max().item())
                assert err <= 2e-5 * flat.max().item(), (name, i, fd, grad.view(-1)[i].item())
    finally:
        torch.set_default_dtype(torch.float32)
    print(f"  max |central differences - autograd| / max |g|: {worst:.2e}")


def _model(**kw):
    return M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=10, num_tetrahedra_cells=5, **kw))


def test_distortion_loss_is_the_mean_over_rays_with_hits():
    R = 32
    g = torch.Generator().manual_seed(1)
    dist = torch.rand((R, 1), generator=g).requires_grad_(True)
    mask = torch.rand(R, generator=g) > 0.3
    with torch.no_grad():
        dist[~mask] = 0.0
    outputs = {"rgb": torch.rand((R, 3), generator=g), "accumulation": torch.ones((R, 1)), "depth": torch.ones((R, 1)),
               "distortion": dist, "ray_mask": mask}
    batch = {"image": torch.rand((R, 3), generator=g)}
    m = _model(distortion_loss_mult=0.01).train()
    loss = m.get_loss_dict(outputs, batch)
    assert math.isclose(loss["distortion_loss"].item(), 0.01 * dist[mask].mean().item(), rel_tol=1e-6)
    # only while training, and not at all at distortion_loss_mult = 0
    assert "distortion_loss" not in _model(distortion_loss_mult=0.01).eval().get_loss_dict(outputs, batch)
    assert set(_model().train().get_loss_dict(outputs, batch)) == {"rgb_loss"}
    # an all-empty batch gives 0, not NaN
    empty = {**outputs, "distortion": torch.zeros((R, 1)), "ray_mask": torch.zeros(R, dtype=torch.bool)}
    assert m.get_loss_dict(empty, batch)["distortion_loss"].item() == 0.0
    assert not np.isnan(m.get_loss_dict(empty, batch)["distortion_loss"].item())
