"""CPU: the float64 surface-extraction oracle (oracle/surface.py) on hand-made cases, and the PLY writer."""
import itertools

import numpy as np
import pytest

from oracle import surface as osf
from tetranerf.b200 import synthetic as syn

TET = np.array([[0.1, 0.0, 0.0], [1.0, 0.2, 0.0], [0.0, 1.0, 0.1], [0.2, 0.1, 1.0]], dtype=np.float32)


def _linear(values):
    """features [V, 1] = values, density = the feature itself (linear along every edge)"""
    return np.asarray(values, dtype=np.float64)[:, None], (lambda f: np.asarray(f)[..., 0])


@pytest.mark.parametrize("cell", [[0, 1, 2, 3], [1, 0, 2, 3]], ids=["positive", "negative"])
@pytest.mark.parametrize("pattern", [p for p in itertools.product([0, 1], repeat=4) if 0 < sum(p) < 4])
def test_one_tetrahedron_all_patterns(pattern, cell):
    """14 mixed patterns x both orientations of the tetrahedron: triangle count, the edges the vertices sit on, winding"""
    level = 1.0
    vals = np.where(np.array(pattern) == 1, 2.0, 0.25) + 0.1 * np.arange(4)  # distinct values on both sides of the level
    feats, sigma = _linear(vals)
    out = osf.surface(TET, np.array([cell]), feats, level, sigma)
    nin = sum(pattern)
    assert len(out["faces"]) == (2 if nin == 2 else 1)
    assert (out["face_tetrahedra"] == 0).all()
    want = sorted((min(i, o), max(i, o)) for i in range(4) if pattern[i] for o in range(4) if not pattern[o])
    assert [tuple(e) for e in out["edges"]] == want  # one vertex per crossing edge, in (a, b) order
    for a, b in out["edges"]:  # the vertex is where the linear density crosses the level
        s = out["s"][list(map(tuple, out["edges"])).index((a, b))]
        assert abs((1 - s) * vals[a] + s * vals[b] - level) < 1e-12
    inside = np.array(pattern, dtype=bool)
    c_in, c_out = TET[inside].astype(np.float64).mean(0), TET[~inside].astype(np.float64).mean(0)
    p = out["vertices"][out["faces"]]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (n @ (c_out - c_in) > 0).all(), (pattern, cell)
    if nin == 2:  # the quad's diagonal joins the vertices on (i0, o0) and (i1, o1)
        i0, i1 = np.nonzero(inside)[0]
        o0, o1 = np.nonzero(~inside)[0]
        e = [tuple(x) for x in out["edges"]]
        diag = {e.index((min(i0, o0), max(i0, o0))), e.index((min(i1, o1), max(i1, o1)))}
        assert all(diag <= set(f) for f in out["faces"].tolist())


def test_crossing_exact_on_linear_density():
    rng = np.random.default_rng(0)
    E = 500
    sa, sb = rng.uniform(0.0, 2.0, E), rng.uniform(0.0, 2.0, E)
    level = 1.0
    keep = (sa >= level) != (sb >= level)
    sa, sb = sa[keep], sb[keep]
    s = osf.crossing(lambda ss: (1 - ss) * sa[:, None] + ss * sb[:, None], level, sa, sb)
    root = (level - sa) / (sb - sa)
    assert np.abs(s - root).max() < 1e-12


def test_crossing_takes_the_one_nearest_a():
    """sigma crosses the level three times along the edge: the vertex is the crossing nearest a"""
    f = lambda ss: 1.0 + np.cos(5 * np.pi * ss)  # noqa: E731  (level 1: crossings at s = 0.1, 0.3, 0.5, ...; a = 2 inside, b = 0 outside)
    s = osf.crossing(f, 1.0, np.array([2.0]), np.array([f(np.array([1.0]))[0]]))
    assert abs(s[0] - 0.1) < 1e-6


def test_cube_central_vertex_closed_sphere(cube_mesh):
    V, C = cube_mesh
    vals = np.zeros(len(V))
    vals[8] = 2.0
    feats, sigma = _linear(vals)
    out = osf.surface(V, C, feats, 1.0, sigma)
    assert len(out["faces"]) == 12 and len(out["edges"]) == 8
    top = osf.topology(out["faces"], len(out["edges"]))
    assert top["directed_once"]
    assert [c[3] for c in top["components"]] == [2]
    # outward: every face normal points away from the centre
    p = out["vertices"][out["faces"]]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (np.sum(n * (p.mean(1) - 0.5), 1) > 0).all()
    assert (np.sum(out["normals"] * (out["vertices"] - 0.5), 1) > 0).all()


def test_network_oracle_on_small_mesh():
    """the network form on surface_scene: closed, oriented, every vertex next to the analytic spheres"""
    from oracle import oracle as orc

    V, C = syn.delaunay_mesh(800, seed=0)
    field, params = syn.surface_scene(V, 1000, orc.init_mlp_params(0))
    out = osf.extract(V, C, field, params, float(np.log(2.0)))
    assert len(out["faces"]) > 0
    top = osf.topology(out["faces"], len(out["edges"]))
    assert top["directed_once"]
    edge_len = np.linalg.norm(V[out["edges"][:, 1]].astype(np.float64) - V[out["edges"][:, 0]], axis=1)
    assert (np.abs(syn.sphere_sdf(out["vertices"])) <= edge_len).all()
    assert out["colors"].shape == (len(out["edges"]), 3) and (out["colors"] >= 0).all() and (out["colors"] <= 1).all()


def test_write_ply_round_trip(tmp_path):
    from tetranerf.b200.surface import read_ply, write_ply

    rng = np.random.default_rng(1)
    surf = {"vertices": rng.standard_normal((7, 3)).astype(np.float32), "normals": rng.standard_normal((7, 3)).astype(np.float32),
            "colors": rng.random((7, 3)).astype(np.float32), "faces": rng.integers(0, 7, (5, 3)).astype(np.int32),
            "face_tetrahedra": np.arange(5, dtype=np.int32)}
    path = tmp_path / "s.ply"
    write_ply(path, surf)
    back = read_ply(path)
    assert np.array_equal(back["vertices"], surf["vertices"]) and np.array_equal(back["normals"], surf["normals"])
    assert np.array_equal(back["faces"], surf["faces"])
    assert np.array_equal(back["colors"], np.rint(surf["colors"] * 255).astype(np.uint8))
    assert path.read_bytes().startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex 7\n")
    write_ply(tmp_path / "empty.ply", {k: v[:0] for k, v in surf.items()})
    assert len(read_ply(tmp_path / "empty.ply")["faces"]) == 0
