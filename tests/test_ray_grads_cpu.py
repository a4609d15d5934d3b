"""CPU: the float64 oracle of the ray gradients of the training step (oracle/ray_grads.py, DESIGN §4.8) against central finite differences
in the ray origins and directions, and against a closed form that tells E^-T from E^-1."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import ray_grads as rg
from tetranerf.b200 import synthetic as syn


def _loss(out, target):
    return torch.nn.functional.mse_loss(out["rgb"], target) + 0.05 * out["accumulation"].mean()


@pytest.fixture(scope="module")
def scene():
    V, C = syn.delaunay_mesh(3000, seed=0)
    field = torch.from_numpy(syn.random_field(len(V), 64, seed=3)).double()
    params = {k: v.double() for k, v in orc.init_mlp_params(0).items()}
    o, d = syn.camera_rays(24, seed=11)
    o[3] = [5, 5, 5]; d[3] = [1, 0, 0]  # empty ray
    return orc.OracleMesh(V, C), V, field, params, o, d


def test_oracle_matches_finite_differences(scene):
    """dL/do, dL/dd of the add_barycentrics_grad oracle against central differences of the same render with b = E^-1 (x - x_v0)
    recomputed from the positions, the fine bins and the matched tetrahedra held fixed (the steps keep every sample in its tetrahedron)"""
    mesh, V, field, params, o, d = scene
    gs = False  # (GradientScaler changes the backward only: no finite difference sees it)
    cfg = orc.RenderConfig(num_samples=24, num_fine_samples=23, use_biased_sampler=True)
    R = len(o)
    g = torch.Generator().manual_seed(4)
    jc, jf, target = torch.rand((R, 25), generator=g), torch.rand((R, 24), generator=g), torch.rand((R, 3), generator=g).double()
    torch.set_default_dtype(torch.float64)
    try:
        ot = torch.from_numpy(o).double().requires_grad_(True)
        dt = torch.from_numpy(d).double().requires_grad_(True)
        out = rg.render_train_rays(mesh, field, params, ot, dt, cfg, jc, jf, use_gradient_scaling=gs)
        ref = orc.render_train(mesh, field, params, o, d, cfg, jc, jf, use_gradient_scaling=gs)
        # the values are render_train's (only the encoding's argument is formed in float64 instead of float32 here)
        assert torch.equal(out["ray_mask"], ref["ray_mask"])
        assert (out["rgb"] - ref["rgb"]).abs().max().item() < 1e-6
        _loss(out, target).backward()
        go, gd = ot.grad.clone(), dt.grad.clone()
        assert torch.all(go[3] == 0) and torch.all(gd[3] == 0)  # the empty ray
        assert go.abs().max() > 0 and gd.abs().max() > 0
        fixed = dict(fine_euclid=out["aux"]["fine_euclid"], matched=out["aux"]["matched"], exact_bary=True)

        def L(oo, dd):
            with torch.no_grad():
                return _loss(rg.render_train_rays(mesh, field, params, oo, dd, cfg, jc, jf, use_gradient_scaling=gs, **fixed), target).item()

        # plain autograd through the recomputed weights: the same gradient up to the features' float32 weights (the recomputed ones
        # differ from the tracer's by ~1e-7, which moves the gradient by second-order terms)
        o2, d2 = ot.detach().clone().requires_grad_(True), dt.detach().clone().requires_grad_(True)
        _loss(rg.render_train_rays(mesh, field, params, o2, d2, cfg, jc, jf, use_gradient_scaling=gs, **fixed), target).backward()
        for a, b in ((go, o2.grad), (gd, d2.grad)):
            rel = (a - b).abs().max().item() / b.abs().max().item()
            print(f"  add_barycentrics_grad vs recomputed weights: {rel:.2e} of the largest entry")
            assert rel < 1e-3
        go, gd = o2.grad, d2.grad  # the finite differences below are of exactly this function
        # steps of 1e-8: a step of 1e-6 along every ray at once already moves a few of the ~4e5 hidden pre-activations across 0
        h = 1e-8
        scale = max(go.abs().max().item(), gd.abs().max().item())
        worst = 0.0
        for r in (0, 7, 12, 20):
            for c in range(3):
                for which in ("o", "d"):
                    u = torch.zeros((R, 3))
                    u[r, c] = 1.0
                    uo, ud = (u, 0 * u) if which == "o" else (0 * u, u)
                    fd = (L(ot.detach() + h * uo, dt.detach() + h * ud) - L(ot.detach() - h * uo, dt.detach() - h * ud)) / (2 * h)
                    an = (go if which == "o" else gd)[r, c].item()
                    worst = max(worst, abs(fd - an) / scale)
                    assert abs(fd - an) <= 1e-5 * scale, (r, c, which, an, fd)
        print(f"  max |finite differences - analytic| / max |g|: {worst:.2e}")
    finally:
        torch.set_default_dtype(torch.float32)


def test_affine_field_gives_a_transpose(scene):
    """a field affine in position, F_v = A x_v + c, is reproduced exactly by every tetrahedron: f(x) = A x + c, so dL/dx = A^T dL/df
    whatever the mesh.  With E^-1 in place of E^-T the result would be E^-1 E^-T A^T dL/df instead."""
    mesh, V, _, _, _, _ = scene
    g = torch.Generator().manual_seed(9)
    A = torch.randn((64, 3), generator=g, dtype=torch.float64)
    c = torch.randn((64,), generator=g, dtype=torch.float64)
    X = torch.from_numpy(V).double()
    field = (X @ A.T + c).T.contiguous()  # [64,V]
    # 500 points inside random tetrahedra of the mesh
    cells = np.asarray(syn.delaunay_mesh(3000, seed=0)[1], dtype=np.int64)
    pick = torch.randint(0, len(cells), (500,), generator=g)
    vi = torch.from_numpy(cells)[pick]
    w = torch.rand((500, 4), generator=g, dtype=torch.float64)
    w = w / w.sum(-1, keepdim=True)
    x = (w[:, :, None] * X[vi]).sum(1).requires_grad_(True)
    bary = w[:, 1:].float()  # the tracer's weights are float32
    b = rg.differentiable_bary(vi, bary, V, x)
    f = rg.interpolate_with_weights(vi, b, field)
    gf = torch.randn((500, 64), generator=g, dtype=torch.float64)
    (f * gf).sum().backward()
    want = gf @ A
    err = (x.grad - want).abs().max().item() / want.abs().max().item()
    print(f"  max |dL/dx - A^T dL/df| / max: {err:.2e}")
    assert err < 1e-9
    # E^-1 applied instead (the mutation this catches) is far off
    verts, _ = rg.tet_edges(vi, V, torch.float64)
    E = (verts[:, 1:, :] - verts[:, :1, :]).transpose(-1, -2)
    q = torch.einsum("nc,nkc->nk", gf, field.T[vi[:, 1:]] - field.T[vi[:, :1]])
    wrong = torch.linalg.solve(E, q)
    assert (wrong - want).abs().max().item() > 0.1 * want.abs().max().item()


def test_unmatched_and_flat_samples_carry_no_ray_gradient():
    vi = torch.tensor([[0, 1, 2, 3], [-1, -1, -1, -1], [0, 1, 2, 4]])
    xyz = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0]], np.float32)  # tetrahedron 2 is flat (z = 0)
    x = torch.tensor([[0.2, 0.2, 0.2], [0.3, 0.3, 0.3], [0.3, 0.3, 0.0]], dtype=torch.float64, requires_grad=True)
    bary = torch.tensor([[0.2, 0.2, 0.2], [0.0, 0.0, 0.0], [0.1, 0.2, 0.3]])
    b = rg.differentiable_bary(vi, bary, xyz, x)
    assert torch.equal(b.detach(), bary.double())
    b.sum().backward()
    assert x.grad[0].abs().sum() > 0 and torch.all(x.grad[1:] == 0)
