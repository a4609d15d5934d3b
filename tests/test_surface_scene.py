"""CPU: the opaque two-sphere scene (synthetic.surface_scene) and the background colour of the oracle renders.

The scene is what makes tests/test_gpu_opaque.py meaningful: with the torch-default network every ray ends at accumulation ~0.5,
the coarse weights are nearly flat and the median-depth search rarely finds a crossing.  `regime` measures, on the oracle's render,
that the scene takes the fused kernels where that network never goes (opaque rays, empty rays, two surfaces on one ray, large
densities, a steep PDF); the GPU tests assert the same guards on their own renders so that they cannot silently become vacuous."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn


def scene_rays(n):
    """camera rays plus an empty ray (5) and an origin inside the mesh (17), as in test_gpu_render"""
    o, d = syn.camera_rays(n)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]
    o[17] = [0.5, 0.5, 0.5]
    return o, d


def regime(ref, o, d, cfg):
    """statistics of an oracle render (return_aux=True) of the surface scene -> dict"""
    acc = ref["accumulation"][:, 0].numpy()
    hits = syn.sphere_hits(o, d)
    aux = ref["aux"]
    m = ref["ray_mask"].numpy()
    ce, fe, cw = aux["coarse_euclid"].numpy(), aux["fine_euclid"].numpy(), aux["coarse_weights"][..., 0].numpy()
    # share of the PDF sampler's new bin edges within 4 coarse-bin widths of the coarse median depth, on opaque rays
    share = []
    for i in np.nonzero(acc[m] > 0.999)[0]:
        j = min(int(np.searchsorted(np.cumsum(cw[i]), 0.5)), len(cw[i]) - 1)
        t, w = (ce[i, j] + ce[i, j + 1]) / 2, ce[i, j + 1] - ce[i, j]
        share.append((np.sum(np.abs(fe[i] - t) <= 4 * w) - np.sum(np.abs(ce[i] - t) <= 4 * w)) / (cfg.num_fine_samples + 1))
    return {"opaque": float(np.mean(acc > 0.999)), "clear": float(np.mean(acc < 0.01)), "both": int(np.isfinite(hits[:, :, 0]).all(1).sum()),
            "max_sigma": aux["sigmas"].max().item(), "near_surface": float(np.median(share)) if share else 0.0}


def assert_regime(st, k, cfg):
    """the guards of a scene of sharpness k >= 100.  A flat CDF puts 8 / S of the new samples in a window of 8 coarse bins; the
    padding of 0.01 per coarse bin of the PDF sampler caps what any CDF can put there at 1 / (1 + 0.01 S) (44 % at S = 128, 28 % at
    256), so a steep CDF is asked for as 3x the flat share."""
    r = max(rad for _, rad in syn.SURFACE_SPHERES)
    assert st["opaque"] >= 0.25 and st["clear"] >= 0.10, st
    assert st["both"] >= 3, st
    assert st["max_sigma"] > 0.4 * k * r, st
    assert st["near_surface"] >= 3 * 8 / cfg.num_samples, st


def test_surface_scene_is_deterministic(small_mesh):
    V, _ = small_mesh
    base = orc.init_mlp_params(0)
    f1, p1 = syn.surface_scene(V, 100, base, seed=0)
    f2, p2 = syn.surface_scene(V, 100, orc.init_mlp_params(0), seed=0)
    f3, _ = syn.surface_scene(V, 100, base, seed=1)
    assert f1.shape == (64, len(V)) and f1.dtype == np.float32 and np.array_equal(f1, f2)
    assert not np.array_equal(f1[4:], f3[4:]) and np.array_equal(f1[:4], f3[:4])  # the seed draws the noise features only
    assert list(p1) == list(base) and all(torch.equal(p1[n], p2[n]) for n in p1)
    assert torch.equal(base["field_output_density.net.weight"], orc.init_mlp_params(0)["field_output_density.net.weight"])  # input untouched
    # random rows stay random: only units 0-7 of the base MLP are overwritten
    assert torch.equal(p1["mlp_base.layers.1.weight"][8:], base["mlp_base.layers.1.weight"][8:])
    assert torch.equal(p1["mlp_head.layers.0.weight"][:, :27], base["mlp_head.layers.0.weight"][:, :27])


def test_surface_scene_densities_follow_the_spheres():
    """the network on its own, at points with known signed distance: sigma ~ softplus(k T tanh(sdf / edge))"""
    rng = np.random.default_rng(0)
    pts = rng.random((4000, 3))
    V = pts.astype(np.float32)
    field, p = syn.surface_scene(V, 1000, orc.init_mlp_params(0))
    sigma = orc.density_head(p, orc.mlp_base(p, torch.from_numpy(field.T.copy())))[:, 0].numpy()
    sdf = syn.sphere_sdf(V)
    assert sigma[sdf > 0.05].min() > 0.9 * 1000 * syn.SURFACE_TRUNCATION
    assert sigma[sdf < -0.05].max() < 1e-3


@pytest.mark.parametrize("k", [100, 1000])
def test_surface_scene_regime(small_mesh, k):
    V, C = small_mesh
    o, d = scene_rays(150)
    field, params = syn.surface_scene(V, k, orc.init_mlp_params(0))
    cfg = orc.RenderConfig.tetra_nerf()
    st = regime(orc.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, cfg, return_aux=True), o, d, cfg)
    print(f"k={k}: {st}")
    assert_regime(st, k, cfg)


@pytest.mark.parametrize("bg", [(0.0, 0.0, 0.0), (0.1, 0.6, 0.3)])
def test_oracle_background(small_mesh, bg):
    """rgb = comp + bg (1 - acc) in eval and training mode; empty rays get bg and the far plane"""
    V, C = small_mesh
    o, d = scene_rays(60)
    field, params = syn.surface_scene(V, 10, orc.init_mlp_params(0))  # semi-transparent: 1 - acc spans (0, 1)
    mesh, f = orc.OracleMesh(V, C), torch.from_numpy(field)
    white = orc.RenderConfig(num_samples=32, num_fine_samples=32)
    cfg = orc.RenderConfig(num_samples=32, num_fine_samples=32, background=bg)
    b = torch.tensor(bg)
    for mode in ("eval", "train"):
        if mode == "eval":
            w, c = (orc.render(mesh, f, params, o, d, x) for x in (white, cfg))
        else:
            jc, jf = torch.rand((len(o), 33), generator=torch.Generator().manual_seed(0)), torch.rand((len(o), 33), generator=torch.Generator().manual_seed(1))
            w, c = (orc.render_train(mesh, f, params, o, d, x, jc, jf) for x in (white, cfg))
        acc = c["accumulation"]
        assert torch.equal(acc, w["accumulation"]) and torch.equal(c["depth"], w["depth"])
        assert 0.05 < acc[c["ray_mask"]].min() and acc.max() < 0.999
        comp = w["rgb"] - (1.0 - acc)
        torch.testing.assert_close(c["rgb"], comp + b * (1.0 - acc), rtol=0, atol=1e-6)
        assert not bool(c["ray_mask"][5]) and c["rgb"][5].tolist() == list(b.tolist()) and float(c["depth"][5]) == cfg.far_plane
        assert float(acc[5]) == 0.0


def test_oracle_render_at_given_fine_bins(small_mesh):
    """render(fine_euclid=) evaluates the fine pass at the given bins: its own bins reproduce the render"""
    V, C = small_mesh
    o, d = scene_rays(40)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    mesh, f, cfg = orc.OracleMesh(V, C), torch.from_numpy(field), orc.RenderConfig.tetra_nerf()
    ref = orc.render(mesh, f, params, o, d, cfg, return_aux=True)
    again = orc.render(mesh, f, params, o, d, cfg, return_aux=True, fine_euclid=ref["aux"]["fine_euclid"])
    for k in ("rgb", "accumulation", "depth", "ray_mask"):
        assert torch.equal(ref[k], again[k]), k
    assert torch.equal(ref["aux"]["sigmas"], again["aux"]["sigmas"])
