"""CPU: oracle/oracle.py's torch-fp32 restatement of the nerfstudio pieces against the independent float64, loop-based
oracle/second_opinion.py (encoding order, sampler mapping, get_weights, PDF inversion + include_original merge, median depth,
MLP / heads / compositing of whole rays)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import second_opinion as so2


def test_nerf_encoding_order_and_values():
    rng = np.random.default_rng(0)
    d = rng.standard_normal((50, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    got = orc.nerf_encoding_dirs(torch.from_numpy(d.astype(np.float32))).numpy()
    want = np.array([so2.nerf_encoding(x) for x in d.astype(np.float32)])
    assert got.shape == (50, 27)
    assert np.abs(got - want).max() < 2e-5  # fp32 sin of arguments up to 2 pi 16


def test_get_weights_product_form():
    rng = np.random.default_rng(1)
    deltas = rng.random((7, 40)).astype(np.float32) * 0.05
    sig = (rng.random((7, 40)).astype(np.float32) * 30) ** 2
    got = orc.get_weights(torch.from_numpy(deltas)[..., None], torch.from_numpy(sig)[..., None])[..., 0].numpy()
    for r in range(7):
        assert np.abs(got[r] - np.array(so2.weights_from_density(deltas[r], sig[r]))).max() < 2e-6


@pytest.mark.parametrize("biased", [True, False])
def test_coarse_bins(biased):
    rng = np.random.default_rng(2)
    R, M, S = 6, 32, 24
    num = rng.integers(1, 20, size=R)
    hd = np.zeros((R, M, 2), np.float32)
    for r in range(R):
        t = 1.0 + np.sort(rng.random(2 * num[r])).astype(np.float32)
        hd[r, : num[r], 0], hd[r, : num[r], 1] = t[0::2], t[1::2]  # gaps between consecutive cells on purpose
    nears = torch.from_numpy(hd[:, 0, 0])[:, None]
    fars = torch.from_numpy(np.array([hd[r, num[r] - 1, 1] for r in range(R)], np.float32))[:, None]
    cfg = orc.RenderConfig(num_samples=S, num_fine_samples=8, use_biased_sampler=biased)
    eu, sb = orc.coarse_bins(cfg, nears, fars, torch.from_numpy(num), torch.from_numpy(hd))
    for r in range(R):
        seg = [(hd[r, k, 0], hd[r, k, 1]) for k in range(num[r])] if biased else None
        e2, s2 = so2.coarse_bins(S, float(nears[r]), float(fars[r]), seg)
        assert np.abs(eu[r].numpy() - np.array(e2)).max() < 5e-6
        assert np.abs(np.broadcast_to(sb[r].numpy(), (S + 1,)) - np.array(s2)).max() < 5e-6


def test_pdf_bins_merge_and_inversion():
    rng = np.random.default_rng(3)
    R, S, Sf = 9, 31, 17
    sb = np.sort(rng.random((R, S + 1)).astype(np.float32), axis=1)
    sb[:, 0], sb[:, -1] = 0.0, 1.0
    w = (rng.random((R, S)).astype(np.float32)) ** 4
    w[3] = 0.0          # empty ray: uniform resampling through the histogram padding
    w[4, :] = 0.0
    w[4, 7] = 0.9       # one dominant bin
    cfg = orc.RenderConfig(num_samples=S, num_fine_samples=Sf)
    nears, fars = torch.full((R, 1), 2.0), torch.full((R, 1), 5.0)
    eu, bins = orc.pdf_bins(cfg, torch.from_numpy(sb), torch.from_numpy(w)[..., None], nears, fars)
    assert bins.shape == (R, S + Sf + 2)
    for r in range(R):
        want = np.array(so2.pdf_bins(sb[r], w[r], Sf))
        assert np.abs(bins[r].numpy() - want).max() < 3e-6, r
        assert np.abs(eu[r].numpy() - (want * 5.0 + (1 - want) * 2.0)).max() < 1e-5


def test_whole_ray_render_against_definitions(small_mesh):
    """oracle.render (torch fp32, upstream code order) vs per-ray float64 evaluation from the definitions: interpolation by
    explicit weights, MLP in float64, product-form weights, scan-based PDF inversion, sorted() merge, loop median depth."""
    from tetranerf.b200 import synthetic as syn

    V, _ = small_mesh
    _whole_ray_render(small_mesh, syn.random_field(len(V), 64, seed=3), orc.init_mlp_params(0), (1.0, 1.0, 1.0))


def test_whole_ray_render_with_background_on_surface_scene(small_mesh):
    """the same on the semi-transparent surface scene (1 - acc spans most of (0, 1)) and an asymmetric background colour, so that
    a swapped or dropped channel of the background shows"""
    from tetranerf.b200 import synthetic as syn

    V, _ = small_mesh
    field, params = syn.surface_scene(V, 10, orc.init_mlp_params(0))
    _whole_ray_render(small_mesh, field, params, (0.1, 0.6, 0.3))


def _whole_ray_render(small_mesh, field, params, background):
    V, C = small_mesh
    from tetranerf.b200 import synthetic as syn

    o, d = syn.camera_rays(24, seed=5)
    o[3] = [5, 5, 5]; d[3] = [1, 0, 0]  # empty ray: the background
    cfg = orc.RenderConfig(num_samples=32, num_fine_samples=24, use_biased_sampler=True, background=background)
    mesh = orc.OracleMesh(V, C)
    ref = orc.render(mesh, torch.from_numpy(field), params, o, d, cfg, return_aux=True)
    tr = ref["aux"]["trace"]
    F64 = field.astype(np.float64)

    def features_at(r, mids):
        n = int(tr["num_visited_cells"][r])
        out = np.zeros((len(mids), 64))
        for j, t in enumerate(mids):
            for k in range(n):
                t0, t1 = float(tr["hit_distances"][r, k, 0]), float(tr["hit_distances"][r, k, 1])
                if t0 <= t <= t1:
                    m = (t - t0) / (t1 - t0)
                    b = (1 - m) * tr["barycentric_coordinates"][r, k, 0].astype(np.float64) + m * tr["barycentric_coordinates"][r, k, 1].astype(np.float64)
                    vi = tr["vertex_indices"][r, k]
                    out[j] = b[0] * F64[:, vi[1]] + b[1] * F64[:, vi[2]] + b[2] * F64[:, vi[3]] + (1 - b.sum()) * F64[:, vi[0]]
                    break
        return out

    worst = 0.0
    rows = [r for r in range(len(o)) if tr["num_visited_cells"][r] > 0]
    assert ref["rgb"][3].tolist() == list(np.float32(background)) and not bool(ref["ray_mask"][3])
    for r in rows:
        n = int(tr["num_visited_cells"][r])
        seg = [(float(tr["hit_distances"][r, k, 0]), float(tr["hit_distances"][r, k, 1])) for k in range(n)]
        near, far = seg[0][0], seg[-1][1]
        eu, sb = so2.coarse_bins(cfg.num_samples, near, far, seg)
        mids = [(eu[j] + eu[j + 1]) / 2 for j in range(cfg.num_samples)]
        enc = so2.nerf_encoding(d[r])
        sig_c, _ = so2.mlp_forward(params, features_at(r, mids), enc)
        w_c = so2.weights_from_density([eu[j + 1] - eu[j] for j in range(cfg.num_samples)], sig_c)
        sb2 = so2.pdf_bins(sb, w_c, cfg.num_fine_samples)
        eu2 = [b * far + (1 - b) * near for b in sb2]
        mids2 = [(eu2[j] + eu2[j + 1]) / 2 for j in range(len(eu2) - 1)]
        sig, col = so2.mlp_forward(params, features_at(r, mids2), enc)
        rgb, acc, dep = so2.composite(eu2, sig, col, background=background)
        worst = max(worst, float(np.abs(np.array(rgb) - ref["rgb"][r].numpy()).max()), abs(acc - float(ref["accumulation"][r])))
    print("whole-ray render: fp32 restatement vs float64 definitions, max |rgb/acc| diff", worst)
    assert worst < 5e-5
