"""CPU: the occupancy oracle (oracle/occupancy.py, DESIGN §4.12) -- probes against a direct evaluation at the probe points, the decay
rule, culling against a brute-force masked pipeline, unmatched samples never culled -- and the model's buffer."""
import numpy as np
import torch

from oracle import occupancy as ocu
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn


def _scene(n=300, seed=0):
    V, C = syn.delaunay_mesh(n, seed=seed)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    return V, C, field, params


def test_probes_match_direct_evaluation():
    V, C, field, params = _scene()
    got = ocu.probe_sigmas(field, params, C)
    F = torch.from_numpy(field).double()
    p = {k: v.double() for k, v in params.items()}
    pts = [(0,), (1,), (2,), (3,), (0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3), (0, 1, 2, 3)]
    for k, verts in enumerate(pts):  # the probe as the mean of the listed vertices' features
        x = sum(F[:, torch.from_numpy(C[:, v]).long()] for v in verts).t() / len(verts)
        ref = orc.density_head(p, orc.mlp_base(p, x))[..., 0]
        assert torch.allclose(got[:, k], ref, rtol=1e-12, atol=1e-12), k
    occ = ocu.occupancy(field, params, C)
    assert torch.equal(occ, got.amax(-1))
    assert float(occ.max()) > 1.0 and float(occ.min()) < 1e-2  # the scene has occupied and empty tetrahedra


def test_decay_rule():
    V, C, field, params = _scene()
    m = ocu.occupancy(field, params, C)
    prev = torch.linspace(0, 40, len(C), dtype=torch.float64)
    assert torch.equal(ocu.occupancy(field, params, C, 0.5, prev), torch.maximum(0.5 * prev, m))
    assert torch.equal(ocu.occupancy(field, params, C, 0.0, torch.full((len(C),), float("nan"))), m)


def test_unmatched_never_culled():
    matched = {"cell_indices": np.array([[-1, 0, 1, -1]], np.int32)}
    occ = torch.tensor([0.0, 5.0])
    assert ocu.culled_mask(matched, (occ, float("inf"))).tolist() == [[False, True, True, False]]
    assert ocu.culled_mask(matched, (occ, 1.0)).tolist() == [[False, True, False, False]]
    assert ocu.culled_mask(matched, (occ, 0.0)).tolist() == [[False, False, False, False]]


def test_culling_equals_masked_pipeline():
    V, C, field, params = _scene(600, seed=1)
    mesh = orc.OracleMesh(V, C)
    o, d = syn.camera_rays(120, seed=3)
    cfg = orc.RenderConfig(num_samples=32, num_fine_samples=32)
    occ = ocu.occupancy(field, params, C).float()
    F = torch.from_numpy(field)
    # threshold 0 culls nothing: the oracle's own render, bit for bit
    base = orc.render(mesh, F, params, o, d, cfg)
    none = ocu.render(mesh, F, params, o, d, cfg, occupancy=(occ, 0.0))
    assert not bool(none["aux"]["culled"].any())
    for k in ("rgb", "accumulation", "depth"):
        assert torch.equal(base[k], none[k]), k
    thr = 0.01
    out = ocu.render(mesh, F, params, o, d, cfg, occupancy=(occ, thr))
    aux = out["aux"]
    cc, cf = aux["coarse_culled"], aux["culled"]
    assert 0 < float(cc.float().mean()) < 1 and 0 < float(cf.float().mean()) < 1
    # brute force: the coarse pass with sigma zeroed where culled, the PDF bins from its weights, the fine pass likewise
    mask = out["ray_mask"]
    tr = mesh.trace_rays(o, d, cfg.max_intersected_triangles)
    trm = {k: v[mask.numpy()] for k, v in tr.items()}
    hd = torch.from_numpy(trm["hit_distances"])
    nv = torch.from_numpy(trm["num_visited_cells"])
    nears = hd[:, 0, 0][:, None]
    fars = torch.gather(hd[:, :, 1], 1, (nv[:, None].long() - 1).clamp_min(0))

    def sig_at(euclid):
        dist = ((euclid[:, 1:] + euclid[:, :-1]) / 2).contiguous().numpy()
        tc = orc.find_visited_cells(trm["num_visited_cells"], trm["visited_cells"], trm["barycentric_coordinates"], trm["hit_distances"],
                                    trm["vertex_indices"], dist)
        cell = torch.from_numpy(tc["cell_indices"]).long()
        culled = (cell >= 0) & (occ[cell.clamp_min(0)] < thr)
        fv = torch.from_numpy(orc.interpolate_values(tc["vertex_indices"], tc["barycentric_coordinates"], field))
        base_ = orc.mlp_base(params, fv)
        sig = orc.density_head(params, base_)
        sig = torch.where(culled[..., None], torch.zeros_like(sig), sig)
        return sig, base_, culled

    euclid, sb = orc.coarse_bins(cfg, nears, fars, nv, hd)
    sig_c, _, cul_c = sig_at(euclid)
    assert torch.equal(cul_c, cc)
    w = orc.get_weights((euclid[:, 1:] - euclid[:, :-1])[..., None], sig_c)
    euclid, sb = orc.pdf_bins(cfg, sb, w, nears, fars)
    assert torch.equal(euclid, aux["fine_euclid"])
    sig, base_, cul_f = sig_at(euclid)
    assert torch.equal(cul_f, cf)
    col = orc.color_head(params, base_, orc.nerf_encoding_dirs(torch.from_numpy(d)[mask])[:, None, :].expand(-1, base_.shape[1], -1))
    w = orc.get_weights((euclid[:, 1:] - euclid[:, :-1])[..., None], sig)
    rgb = torch.clamp(torch.sum(w * col, -2) + (1.0 - torch.sum(w, -2)), 0, 1)
    assert torch.allclose(out["rgb"][mask], rgb, atol=1e-6)
    assert bool((w[..., 0][cf] == 0).all())


def test_model_registers_reference_buffer():
    from tetranerf.nerfstudio import model as M

    V, C = syn.delaunay_mesh(200, seed=0)
    cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), use_occupancy_field=True)
    m = M.TetrahedraNerf(cfg)
    assert m.tetrahedra_occupancy.shape == (len(C),) and m.tetrahedra_occupancy.dtype == torch.float32
    assert "tetrahedra_occupancy" in m.state_dict()
    off = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C)))
    assert "tetrahedra_occupancy" not in off.state_dict()
    m.load_state_dict(m.state_dict(), strict=True)
    m2 = M.TetrahedraNerf(M.TetrahedraNerfConfig(use_occupancy_field=True), metadata={"points3D_xyz": torch.from_numpy(V),
                                                                                     "points3D_rgb": torch.zeros((len(V), 3), dtype=torch.uint8)})
    assert m2.tetrahedra_occupancy.shape == (m2.tetrahedra_cells.shape[0],)
