"""CPU: the expected depth (DESIGN §4.10).  The torch oracle (oracle/expected_depth.py) against the plain-loop float64 restatement
(oracle/second_opinion_depth.py) and central differences, the compat DepthRenderer("expected") against the oracle, and the model's
depth loss (target mask, z-depth conversion)."""
import math

import numpy as np
import pytest
import torch

from oracle import expected_depth as edo
from oracle import oracle as orc
from oracle import second_opinion_depth as so
from tetranerf.b200 import synthetic as syn
from tetranerf.nerfstudio import model as M

FAR = 6.0


def _batch():
    """five rays: three ordinary ones, one with A tiny (sigma ~ 1e-13: the batch-wide clip binds, at another ray's midpoint), one with
    A = 0 (sigma = 0), and two empty rays in between; float32 bin edges"""
    g = torch.Generator().manual_seed(0)
    rows, sig = [], []
    for near, far, scale in ((1.0, 3.0, 1.0), (2.5, 4.0, 3.0), (2.0, 5.5, 0.3), (3.0, 4.5, 1e-13), (3.5, 5.0, 0.0)):
        u = torch.sort(torch.rand(17, generator=g))[0]
        u[0], u[-1] = 0.0, 1.0
        rows.append((near + (far - near) * u).float())
        sig.append(torch.rand(16, generator=g, dtype=torch.float64) * 4 * scale)
    mask = torch.tensor([True, False, True, True, False, True, True])
    return torch.stack(rows), torch.stack(sig), mask


def _oracle(euclid, sig, mask, grad_out=None):
    s = sig.clone().requires_grad_(True)
    w = orc.get_weights((euclid[:, 1:] - euclid[:, :-1]).double()[..., None], s[..., None])
    d = edo.expected_depth(w, euclid, mask, FAR)
    if grad_out is not None:
        (d[:, 0] * grad_out).sum().backward()
    return d.detach(), s.grad


def test_oracle_matches_second_opinion():
    euclid, sig, mask = _batch()
    go = torch.linspace(0.5, 2.0, len(mask), dtype=torch.float64)
    d, gs = _oracle(euclid, sig, mask, go)
    mids = ((euclid[:, 1:] + euclid[:, :-1]) / 2).double()
    act = torch.nonzero(mask).flatten().tolist()
    edges = [None] * len(mask)
    sigs = [None] * len(mask)
    midp = [None] * len(mask)
    for k, r in enumerate(act):
        edges[r], sigs[r], midp[r] = euclid[k].double().tolist(), sig[k].tolist(), mids[k].tolist()
    d2, g2 = so.expected_depth(edges, sigs, FAR, go.tolist(), midpoints=midp)
    assert np.allclose(d[:, 0].numpy(), d2, rtol=1e-13, atol=1e-13)
    for k, r in enumerate(act):
        assert np.allclose(gs[k].numpy(), g2[r], rtol=1e-9, atol=1e-12), r
    lo = float(mids.min())
    # the tiny-A and A = 0 rays are clipped to the BATCH's smallest midpoint (ray 0's), not their own, and carry no gradient
    assert d[5, 0].item() == lo and d[6, 0].item() == lo and mids[3].min().item() > lo + 1.0
    assert torch.all(gs[3] == 0) and torch.all(gs[4] == 0)
    assert d[1, 0].item() == FAR and d[4, 0].item() == FAR
    assert gs[:3].abs().max() > 0


def test_oracle_gradient_matches_central_differences():
    euclid, sig, mask = _batch()
    go = torch.linspace(0.5, 2.0, len(mask), dtype=torch.float64)
    _, gs = _oracle(euclid, sig, mask, go)
    h = 1e-6
    worst = 0.0
    for k in range(3):
        for j in range(0, 16, 3):
            e = torch.zeros_like(sig)
            e[k, j] = h
            fp = (_oracle(euclid, sig + e, mask)[0][:, 0] * go).sum().item()
            fm = (_oracle(euclid, sig - e, mask)[0][:, 0] * go).sum().item()
            fd = (fp - fm) / (2 * h)
            worst = max(worst, abs(fd - gs[k, j].item()))
            assert abs(fd - gs[k, j].item()) <= 1e-7 * max(1.0, abs(fd)), (k, j, fd, gs[k, j].item())
    print(f"  max |finite differences - autograd|: {worst:.2e}")


def test_compat_depth_renderer_expected_equals_oracle():
    if M.HAVE_NERFSTUDIO:
        pytest.skip("real nerfstudio present")
    euclid, sig, mask = _batch()
    w = orc.get_weights((euclid[:, 1:] - euclid[:, :-1]).double()[..., None], sig[..., None])
    bundle = M.RayBundle(origins=torch.zeros((5, 3)), directions=torch.ones((5, 3)), nears=euclid[:, :1], fars=euclid[:, -1:])
    rs = bundle.get_ray_samples(bin_starts=euclid[:, :-1, None], bin_ends=euclid[:, 1:, None], spacing_starts=euclid[:, :-1, None],
                                spacing_ends=euclid[:, 1:, None], spacing_to_euclidean_fn=lambda x: x)
    got = M.DepthRenderer(method="expected")(w, rs)
    want = edo.expected_depth(w, euclid, torch.ones(5, dtype=torch.bool), FAR)
    assert torch.equal(got, want)
    assert torch.equal(M.DepthRenderer()(w, rs), M.DepthRenderer(method="median")(w, rs))
    with pytest.raises(NotImplementedError):
        M.DepthRenderer(method="accumulation")


def _model(**kw):
    return M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=10, num_tetrahedra_cells=5, **kw))


def test_depth_loss_mask_and_z_depth_conversion():
    R = 64
    g = torch.Generator().manual_seed(1)
    ed = (2 + 3 * torch.rand((R, 1), generator=g)).requires_grad_(True)
    target = 2 + 3 * torch.rand((R, 1), generator=g)
    target[3] = 0.0
    target[4] = float("nan")
    target[5] = float("inf")
    mask = torch.ones(R, dtype=torch.bool)
    mask[6] = False
    dn = 1 + torch.rand((R, 1), generator=g)
    outputs = {"rgb": torch.rand((R, 3), generator=g), "accumulation": torch.ones((R, 1)), "depth": ed.detach(), "expected_depth": ed,
               "ray_mask": mask, "directions_norm": dn}
    batch = {"image": torch.rand((R, 3), generator=g), "depth_image": target}
    ok = torch.ones(R, dtype=torch.bool)
    ok[[3, 4, 5, 6]] = False
    # z-depth (the default): the target becomes a distance along the ray
    m = _model(depth_loss_mult=0.5)
    loss = m.get_loss_dict(outputs, batch)
    want = 0.5 * ((ed - target * dn)[ok] ** 2).mean()
    assert math.isclose(loss["depth_loss"].item(), want.item(), rel_tol=1e-6)
    loss["depth_loss"].backward()
    assert torch.all(ed.grad[~ok] == 0) and torch.all(ed.grad[ok] != 0)
    # euclidean targets are used as they are
    loss = _model(depth_loss_mult=0.5, is_euclidean_depth=True).get_loss_dict(outputs, batch)
    assert math.isclose(loss["depth_loss"].item(), 0.5 * ((ed - target)[ok] ** 2).mean().item(), rel_tol=1e-6)
    # z-depth without directions_norm is an error; depth_loss_mult = 0 adds nothing
    with pytest.raises(RuntimeError, match="directions_norm"):
        m.get_loss_dict({k: v for k, v in outputs.items() if k != "directions_norm"}, batch)
    assert set(_model().get_loss_dict(outputs, batch)) == {"rgb_loss"}
    assert _model(depth_loss_mult=0.5)._expected_depth_on() and _model(render_expected_depth=True)._expected_depth_on()
    assert not _model()._expected_depth_on()


def test_image_metrics_show_expected_depth():
    g = torch.Generator().manual_seed(0)
    img = torch.rand((16, 20, 3), generator=g)
    out = {"rgb": img, "accumulation": torch.rand((16, 20, 1), generator=g), "depth": 2 + torch.rand((16, 20, 1), generator=g)}
    _, images = _model().get_image_metrics_and_images(out, {"image": img})
    assert "expected_depth" not in images
    _, images = _model().get_image_metrics_and_images({**out, "expected_depth": out["depth"] + 0.1}, {"image": img})
    assert images["expected_depth"].shape == (16, 20, 3)


def test_render_train_depth_matches_the_geometry_oracle(small_mesh):
    """render_train_depth restates vertex_grads.render_train_geometry: the same rgb / accumulation and gradients; its expected depth
    equals expected_depth() of that oracle's weights and bins"""
    from oracle import vertex_grads as vg

    V, C = small_mesh
    mesh = orc.OracleMesh(V, C)
    field = torch.from_numpy(syn.random_field(len(V), 64, seed=3)).double()
    params = {k: v.double() for k, v in orc.init_mlp_params(0).items()}
    o, d = syn.camera_rays(16, seed=11)
    o[2] = [5, 5, 5]; d[2] = [1, 0, 0]
    cfg = orc.RenderConfig(num_samples=24, num_fine_samples=23, use_biased_sampler=True)
    g = torch.Generator().manual_seed(4)
    jc, jf = torch.rand((16, 25), generator=g), torch.rand((16, 24), generator=g)
    torch.set_default_dtype(torch.float64)
    try:
        ot, dt = torch.from_numpy(o).double(), torch.from_numpy(d).double()
        a = edo.render_train_depth(mesh, field, params, ot, dt, V, cfg, jc, jf)
        b = vg.render_train_geometry(mesh, field, params, ot, dt, V, cfg, jc, jf)
    finally:
        torch.set_default_dtype(torch.float32)
    assert torch.equal(a["rgb"], b["rgb"]) and torch.equal(a["accumulation"], b["accumulation"])
    want = edo.expected_depth(b["aux"]["weights"], b["aux"]["fine_euclid"], b["ray_mask"], cfg.far_plane)
    assert torch.equal(a["expected_depth"], want)
    assert a["expected_depth"][2, 0].item() == cfg.far_plane
