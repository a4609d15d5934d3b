"""CPU: the oracle of the field smoothness loss (oracle/smoothness.py, DESIGN §4.15).
  * S, the loss and the gradient against float64 torch autograd of the edge-list formula, its edges collected independently (a Python set
    of vertex pairs), on the 12-tetrahedra cube, the bottle mesh, a small Delaunay mesh, a mesh after one refinement pass and a mesh with a
    vertex no cell uses (whose gradient is 0);
  * a constant field gives 0, and a field linear in position gives sum_e sum_c (a_c . (x_i - x_j))^2;
  * the model's option: a config the fused pipeline does not support raises, naming the option and the cause."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import refine as orf
from oracle import smoothness as osm
from tetranerf.b200 import synthetic as syn

ROOT = Path(__file__).resolve().parents[1]


def _bottle():
    z = np.load(ROOT / "tests" / "golden" / "bottle_mesh.npz")
    return z["vertices"].astype(np.float32), z["cells"].astype(np.int32)


def _refined():
    V, C = syn.delaunay_mesh(400, seed=2)
    out = orf.refine_edges(V, C, np.random.default_rng(0).random(len(C)) < 0.3)
    return orf.migrate_vertices(V, out["parent_edge"], 0).astype(np.float32), out["cells"].astype(np.int32)


def _unused():
    """a Delaunay mesh with one more vertex, in the middle of the index range, that no cell uses"""
    V, C = syn.delaunay_mesh(300, seed=6)
    k = 150
    V = np.insert(V, k, np.float32([0.5, 0.5, 0.5]), axis=0)
    C = np.where(C >= k, C + 1, C).astype(np.int32)
    return V, C, k


MESHES = {
    "cube": lambda: (syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()),
    "bottle": _bottle,
    "delaunay": lambda: syn.delaunay_mesh(600, seed=4),
    "refined": _refined,
    "unused_vertex": lambda: _unused()[:2],
}


def _edge_list(cells):
    pairs = set()
    for c in np.asarray(cells).tolist():
        for a in range(4):
            for b in range(a + 1, 4):
                if c[a] != c[b]:
                    pairs.add((min(c[a], c[b]), max(c[a], c[b])))
    return torch.tensor(sorted(pairs), dtype=torch.long)


@pytest.mark.parametrize("mesh", list(MESHES))
def test_oracle_matches_autograd_of_the_edge_list(mesh):
    V, C = MESHES[mesh]()
    field = np.random.default_rng(1).standard_normal((64, len(V))).astype(np.float32)
    mult = 0.37
    e = _edge_list(C)
    f = torch.from_numpy(field).double().requires_grad_(True)
    d = f[:, e[:, 0]] - f[:, e[:, 1]]
    S_t = (d * d).sum()
    loss_t = mult * S_t / (len(e) * 64)
    loss_t.backward()
    S, E = osm.smoothness(field, C)
    assert E == len(e)
    assert np.array_equal(osm.edges(C), e.numpy())
    assert S == pytest.approx(S_t.item(), rel=1e-12)
    assert osm.loss(field, C, mult) == pytest.approx(loss_t.item(), rel=1e-12)
    g = osm.gradient(field, C, mult)
    np.testing.assert_allclose(g, f.grad.numpy(), rtol=1e-11, atol=1e-15 * np.abs(g).max())
    if mesh == "unused_vertex":
        k = _unused()[2]
        assert not np.any(np.asarray(C) == k)
        assert np.all(g[:, k] == 0)
    print(f"{mesh}: V {len(V)}, T {len(C)}, E {E}, S {S:.6e}")


def test_constant_field_gives_zero():
    V, C = syn.delaunay_mesh(500, seed=1)
    field = np.tile(np.linspace(-1, 1, 64, dtype=np.float32)[:, None], (1, len(V)))
    S, E = osm.smoothness(field, C)
    assert S == 0.0 and E > 0
    assert np.all(osm.gradient(field, C, 2.0) == 0)


def test_linear_field():
    V, C = syn.delaunay_mesh(500, seed=3)
    rng = np.random.default_rng(2)
    a, b = rng.standard_normal((64, 3)), rng.standard_normal((64, 1))
    x = V.astype(np.float64)
    field = a @ x.T + b
    e = osm.edges(C)
    want = float(((a @ (x[e[:, 0]] - x[e[:, 1]]).T) ** 2).sum())
    S, _ = osm.smoothness(field, C)
    assert S == pytest.approx(want, rel=1e-9)


def test_model_option_needs_the_fused_pipeline():
    from tetranerf.nerfstudio import model as M

    m = M.TetrahedraNerf(M.TetrahedraNerfConfig(num_tetrahedra_vertices=7, num_tetrahedra_cells=3, field_dim=32, field_smoothness_mult=0.1))
    assert M.TetrahedraNerfConfig(num_tetrahedra_vertices=7, num_tetrahedra_cells=3).field_smoothness_mult == 0.0
    m.train()
    with pytest.raises(RuntimeError, match="field_smoothness_mult.*field_dim=32"):
        m.get_loss_dict({"rgb": torch.zeros((4, 3))}, {"image": torch.zeros((4, 3))})
    m.eval()
    assert "field_smoothness_loss" not in m.get_loss_dict({"rgb": torch.zeros((4, 3))}, {"image": torch.zeros((4, 3))})
