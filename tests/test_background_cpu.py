"""CPU: the oracle of the learned background (oracle/background.py, DESIGN §4.16) and its torch restatement on the unfused path
(tetranerf.b200.render.background_lookup).
  * a constant map is returned exactly, by both;
  * the lookup is continuous across the u seam (atan2's branch cut at -x) and at the v clamps (near the poles);
  * float64 central differences agree with the analytic map and direction gradients;
  * the pole convention: the u-derivative is 0 where n_x^2 + n_y^2 < POLE_EPS, and the direction gradient stays finite there;
  * the torch restatement equals the oracle, and its autograd the oracle's gradients away from the poles;
  * the model's option: a background_color other than white / black raises, naming the option; the map is initialised to the colour."""
import numpy as np
import pytest
import torch

from oracle import background as obg
from tetranerf.b200.render import background_lookup


def _dirs(R=200, seed=0):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(R, 3))
    return d * rng.uniform(0.3, 3.0, size=(R, 1))  # not unit length: the lookup normalises


def _map(H=6, seed=1):
    return np.random.default_rng(seed).normal(size=(H, 2 * H, 3))


@pytest.mark.parametrize("c", [0.0, 1.0, 0.3127])
def test_constant_map_is_returned_exactly(c):
    B = np.full((5, 10, 3), c)
    d = _dirs()
    assert np.array_equal(obg.lookup(B, d), np.full((len(d), 3), c))
    Bt = torch.full((5, 10, 3), c, dtype=torch.float32)
    got = background_lookup(Bt, torch.from_numpy(d).float())
    assert torch.equal(got, torch.full_like(got, float(np.float32(c))))


def test_continuous_across_the_u_seam():
    B = _map()
    eps = 1e-9
    for x, z in ((-1.0, 0.3), (-2.0, -0.7), (-0.5, 0.0)):  # atan2(+-0, x < 0) = +-pi: u = W - 1/2 and -1/2, the same wrapped column
        a = obg.lookup(B, [[x, eps, z]])
        b = obg.lookup(B, [[x, -eps, z]])
        assert np.abs(a - b).max() < 1e-6


def test_continuous_at_the_v_clamps():
    B = _map()
    H = B.shape[0]
    for sgn in (1.0, -1.0):  # v = -1/2 .. 0 (north) and H - 1 .. H - 1/2 (south) are clamped: bg is constant in v there
        a = obg.lookup(B, [[0.05, 0.02, sgn]])
        b = obg.lookup(B, [[0.01, 0.004, sgn]])
        assert np.abs(a - b).max() < 1e-12
        t = obg.taps(H, 2 * H, [[0.05, 0.02, sgn]])
        assert not t["v_in"][0]
    # just inside and just outside the clamp boundary agree
    for nz in (1 - 1 / H, -(1 - 1 / H)):  # v_raw = -1/2 + ... at the first / last row centre
        vz = np.array([[np.sqrt(1 - nz * nz), 0.0, nz]])
        a = obg.lookup(B, vz * (1 + 1e-9))
        b = obg.lookup(B, vz)
        assert np.abs(a - b).max() < 1e-6


def _fd_direction(B, d, s, h=1e-6):
    g = np.zeros_like(d)
    for c in range(3):
        e = np.zeros(3)
        e[c] = h
        g[:, c] = (np.sum(obg.lookup(B, d + e) * s, 1) - np.sum(obg.lookup(B, d - e) * s, 1)) / (2 * h)
    return g


def test_map_gradient_against_finite_differences():
    B = _map(H=4)
    d = _dirs(60, seed=3)
    s = np.random.default_rng(4).normal(size=(len(d), 3))
    g = obg.grad_map(4, 8, d, s)
    h = 1e-6
    fd = np.zeros_like(B)
    for idx in np.ndindex(*B.shape):
        Bp, Bm = B.copy(), B.copy()
        Bp[idx] += h
        Bm[idx] -= h
        fd[idx] = (np.sum(obg.lookup(Bp, d) * s) - np.sum(obg.lookup(Bm, d) * s)) / (2 * h)
    assert np.abs(g - fd).max() < 1e-7 * max(1.0, np.abs(fd).max())


def test_direction_gradient_against_finite_differences():
    B = _map(H=8)
    d = _dirs(300, seed=5)
    t = obg.taps(8, 16, d)
    # central differences are exact only inside one bilinear cell and away from the clamps: keep rays 1e-3 texels from every edge
    far = (np.minimum(t["fu"], 1 - t["fu"]) > 1e-3) & (np.minimum(t["fv"], 1 - t["fv"]) > 1e-3) & t["v_in"]
    d = d[far]
    s = np.random.default_rng(6).normal(size=(len(d), 3))
    g = obg.grad_direction(B, d, s)
    fd = _fd_direction(B, d, s)
    assert len(d) > 200
    assert np.abs(g - fd).max() < 1e-5 * max(1.0, np.abs(fd).max())


def test_pole_convention():
    B = _map(H=8)
    s = np.ones((4, 3))
    d = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, -2.0], [3e-5, 4e-5, 1.0], [1e-3, 0.0, 1.0]])
    t = obg.taps(8, 16, d)
    rho2 = t["n"][:, 0] ** 2 + t["n"][:, 1] ** 2
    assert (rho2[:3] < obg.POLE_EPS).all() and rho2[3] >= obg.POLE_EPS
    g = obg.grad_direction(B, d, s)
    assert np.isfinite(g).all()
    # below the epsilon the u-derivative is 0, and at the poles v is clamped, so no term is left
    assert np.array_equal(g[:3], np.zeros((3, 3)))
    assert np.abs(g[3]).max() > 0
    # the lookup itself stays finite at the exact pole direction
    assert np.isfinite(obg.lookup(B, d)).all()


def test_torch_restatement_matches_the_oracle():
    B = _map(H=8, seed=7)
    d = _dirs(500, seed=8)
    Bt = torch.from_numpy(B).requires_grad_(True)
    dt = torch.from_numpy(d).requires_grad_(True)
    out = background_lookup(Bt, dt)
    assert np.abs(out.detach().numpy() - obg.lookup(B, d)).max() < 1e-12
    s = np.random.default_rng(9).normal(size=(len(d), 3))
    (out * torch.from_numpy(s)).sum().backward()
    assert np.abs(Bt.grad.numpy() - obg.grad_map(8, 16, d, s)).max() < 1e-10
    assert np.abs(dt.grad.numpy() - obg.grad_direction(B, d, s)).max() < 1e-8 * max(1.0, np.abs(dt.grad.numpy()).max())


def test_torch_restatement_keeps_the_pole_convention():
    """the unfused path's directions get the fused path's gradient at and near the poles: finite, with the u-derivative 0"""
    B = _map(H=8, seed=7)
    d = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, -2.0], [3e-5, 4e-5, 1.0], [2e-5, -1e-5, -0.5], [1e-3, 0.0, 1.0], [0.3, 0.2, 0.7]])
    s = np.random.default_rng(2).normal(size=(len(d), 3))
    dt = torch.from_numpy(d).requires_grad_(True)
    (background_lookup(torch.from_numpy(B), dt) * torch.from_numpy(s)).sum().backward()
    g = dt.grad.numpy()
    assert np.isfinite(g).all()
    assert np.array_equal(g[:4], np.zeros((4, 3)))
    want = obg.grad_direction(B, d, s)
    assert np.abs(g - want).max() <= 1e-8 * np.abs(want).max()


def test_composite():
    B = _map(H=4)
    d = _dirs(10)
    comp = np.random.default_rng(1).uniform(size=(10, 3))
    acc = np.random.default_rng(2).uniform(size=10)
    mask = np.arange(10) % 3 != 0
    rgb = obg.composite(comp, acc, mask, B, d, train=True)
    bg = obg.lookup(B, d)
    assert np.allclose(rgb[mask], comp[mask] + (1 - acc[mask, None]) * bg[mask])
    assert np.array_equal(rgb[~mask], bg[~mask])
    assert obg.composite(comp, acc, mask, B, d, train=False).max() <= 1.0


def _model_config(**kw):
    from tetranerf.nerfstudio.model import TetrahedraNerfConfig

    return TetrahedraNerfConfig(num_tetrahedra_vertices=10, num_tetrahedra_cells=5, **kw)


def test_model_option():
    from tetranerf.nerfstudio.model import TetrahedraNerf

    with pytest.raises(RuntimeError, match="background_envmap_height"):
        TetrahedraNerf(_model_config(background_envmap_height=4, background_color="random"))
    for color, v in (("white", 1.0), ("black", 0.0)):
        m = TetrahedraNerf(_model_config(background_envmap_height=4, background_color=color))
        assert tuple(m.background_envmap.shape) == (4, 8, 3) and bool((m.background_envmap == v).all())
        assert "background_envmap" in m.state_dict()
        assert any(p is m.background_envmap for p in m.get_param_groups()["fields"])
    m = TetrahedraNerf(_model_config())
    assert "background_envmap" not in m.state_dict() and not hasattr(m, "background_envmap")
