"""GPU parity: the CUDA path (through the C ABI / the tetranerf_cpp_extension shim) against the CPU oracle.
Bit-exact for ids, ordering, t and barycentrics (same fp32 op sequence on both sides)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ["num_visited_cells", "visited_cells", "vertex_indices", "hit_distances", "barycentric_coordinates"]


from conftest import TRACE_IMPLS, force_trace_impl

IMPL = "walk"  # set by the autouse fixture


@pytest.fixture(autouse=True, params=list(TRACE_IMPLS))
def trace_impl(request):
    """every test of this file runs against all four (bit-identical) implementations of trace_rays: adjacency walk with
    32 / 8 / 1 rays per warp, warp-per-ray BVH gather"""
    global IMPL
    IMPL = request.param
    yield request.param


def make_tracer(V, C):
    from tetranerf import cpp

    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    force_trace_impl(tr, IMPL)
    return tr


def gpu_trace(tr, o, d, M):
    out = tr.trace_rays(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), M)
    tr.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def assert_same(a, b, what=""):
    for k in KEYS:
        if a[k].dtype.kind == "f":
            assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), f"{what}{k} differs bitwise"
        else:
            assert np.array_equal(a[k], b[k]), f"{what}{k} differs"


def test_faces_numbering(small_mesh, cube_mesh):
    for V, C in (cube_mesh, small_mesh):
        tr = make_tracer(V, C)
        tri, tt = tr.get_faces()
        otri, ott = orc.OracleMesh(V, C).faces()
        assert np.array_equal(tri.cpu().numpy().view(np.uint32), otri)
        assert np.array_equal(tt.cpu().numpy().view(np.uint32), ott)


def test_faces_numbering_large_and_permuted():
    """The device build (sort + scan, tn_faces.cu) must reproduce the reference's first-appearance numbering
    (tetrahedra_tracer.cpp:45-63) -- which depends on the order of the tetrahedra and of the vertices inside each."""
    V, C = syn.delaunay_mesh(6000, seed=4)
    rng = np.random.default_rng(0)
    C2 = C[rng.permutation(len(C))].copy()
    for i in range(len(C2)):
        C2[i] = C2[i][rng.permutation(4)]
    for cells in (C, C2):
        tr = make_tracer(V, cells)
        tri, tt = tr.get_faces()
        otri, ott = orc.OracleMesh(V, cells).faces()
        assert tr.num_faces() == len(otri)
        assert np.array_equal(tri.cpu().numpy().view(np.uint32), otri)
        assert np.array_equal(tt.cpu().numpy().view(np.uint32), ott)


def test_face_build_errors(cube_mesh):
    """tetrahedra_tracer.cpp:64-66 (a triangle with a third owner) and an out-of-range vertex index."""
    from tetranerf import cpp
    V, C = cube_mesh
    tr = cpp.TetrahedraTracer(DEV)
    bad = np.concatenate([C, C[:1], C[:1]]).astype(C.dtype)  # the first tetrahedron three times
    with pytest.raises(Exception, match="shared by more than two"):
        tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(bad).to(DEV))
    bad2 = C.copy(); bad2[3, 2] = len(V) + 5
    with pytest.raises(Exception, match="out of range"):
        tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(bad2).to(DEV))
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))  # the tracer is still usable
    assert tr.num_faces() == 30


def test_cube_known_answer(cube_mesh):
    V, C = cube_mesh
    tr = make_tracer(V, C)
    d = np.array([1, 0.13, 0.29])
    d = (d / np.linalg.norm(d)).astype(np.float32)[None]
    o = np.array([[-0.05, 0.07, 0.21]], np.float32)
    g = gpu_trace(tr, o, d, 16)
    assert g["num_visited_cells"][0] == 4 and g["visited_cells"][0, :4].tolist() == [4, 2, 3, 10]
    assert g["vertex_indices"][0, 0].tolist() == [8, 0, 2, 4]
    assert_same(g, orc.OracleMesh(V, C).trace_rays(o, d, 16))


def test_cube_reference_degenerate_ray(cube_mesh):
    """tests/test_tetrahedra_tracer.py:228-267 (asserts nothing upstream): kernel == oracle, no OOB."""
    V, C = cube_mesh
    tr = make_tracer(V, C)
    o = np.array([[-0.05, 0.05, 0.05]], np.float32)
    d = np.array([[1.0, 0.0, 0.0]], np.float32)
    assert_same(gpu_trace(tr, o, d, 16), orc.OracleMesh(V, C).trace_rays(o, d, 16))


def test_cube_edge_and_vertex_rays(cube_mesh):
    """rays aimed exactly at mesh vertices / edge midpoints / along faces: ties, zero edge functions, duplicates"""
    V, C = cube_mesh
    tr = make_tracer(V, C)
    rng = np.random.default_rng(7)
    tg = [V[i] for i in range(9)] + [(V[a] + V[b]) / 2 for a, b in ((0, 8), (1, 8), (0, 1), (2, 3), (4, 7), (0, 3))]
    o, d = [], []
    for t in tg:
        for _ in range(8):
            src = (np.array([0.5, 0.5, 0.5]) + 3 * rng.standard_normal(3)).astype(np.float32)
            dd = np.asarray(t, np.float32) - src
            o.append(src); d.append((dd / np.linalg.norm(dd)).astype(np.float32))
    # axis-aligned rays lying in faces of the mesh
    for y in (0.0, 0.5, 1.0):
        o.append(np.array([-1, y, 0.25], np.float32)); d.append(np.array([1, 0, 0], np.float32))
        o.append(np.array([0.25, -1, y], np.float32)); d.append(np.array([0, 1, 0], np.float32))
    o, d = np.stack(o), np.stack(d)
    assert_same(gpu_trace(tr, o, d, 32), orc.OracleMesh(V, C).trace_rays(o, d, 32))


@pytest.mark.parametrize("gen,M", [(syn.camera_rays, 512), (syn.sphere_rays, 256), (syn.camera_rays, 64), (syn.camera_rays, 16),
                                   (syn.camera_rays, 2), (syn.camera_rays, 4), (syn.camera_rays, 2048)])
def test_random_mesh_bit_exact(small_mesh, gen, M):
    """M = 2 keeps no cell on any ray, M = 4 truncates nearly every ray, M = 2048 is the largest hit cap"""
    V, C = small_mesh
    tr = make_tracer(V, C)
    o, d = gen(700)
    g = gpu_trace(tr, o, d, M)
    assert_same(g, orc.OracleMesh(V, C).trace_rays(o, d, M), f"M={M} ")
    if M >= 256:
        assert g["num_visited_cells"].max() > 40
    else:
        assert g["num_visited_cells"].max() <= M - 2
    if M == 4:
        assert (g["num_visited_cells"] == 2).mean() > 0.9


@pytest.mark.parametrize("R", [1, 3, 9])
def test_tiny_batches_bit_exact(small_mesh, R):
    """batches below the 4-warp blocks and not a multiple of the quad walk's 8 rays per warp"""
    V, C = small_mesh
    tr = make_tracer(V, C)
    o, d = syn.camera_rays(R, seed=30 + R)
    g = gpu_trace(tr, o, d, 512)
    assert_same(g, orc.OracleMesh(V, C).trace_rays(o, d, 512), f"R={R} ")
    assert g["num_visited_cells"].min() > 0


def test_medium_mesh_bit_exact(medium_mesh):
    V, C = medium_mesh
    tr = make_tracer(V, C)
    for gen in (syn.camera_rays, syn.sphere_rays):
        o, d = gen(1500, seed=11)
        assert_same(gpu_trace(tr, o, d, 512), orc.OracleMesh(V, C).trace_rays(o, d, 512), gen.__name__ + " ")


def test_special_rays(small_mesh):
    """origins inside the mesh, rays that miss, zero / non-finite directions, unnormalised directions"""
    V, C = small_mesh
    tr = make_tracer(V, C)
    rng = np.random.default_rng(3)
    o = np.concatenate([0.2 + 0.6 * rng.random((64, 3)), np.full((8, 3), 5.0), 0.5 * np.ones((4, 3)), -1 + 0 * rng.random((16, 3))]).astype(np.float32)
    d = rng.standard_normal((len(o), 3)).astype(np.float32)
    d[64:72] = [1, 0, 0]
    d[72] = 0; d[73] = [np.nan, 0, 1]; d[74] = [np.inf, 0, 0]; d[75] = [0, 0, 1e-30]
    d[76:] = (np.array([1.5, 1.5, 1.5]) + rng.random((16, 3))) * 3.7  # not unit length (trace_rays does not normalise)
    g = gpu_trace(tr, o, d, 256)
    assert_same(g, orc.OracleMesh(V, C).trace_rays(o, d, 256))
    assert (g["num_visited_cells"][64:75] == 0).all() and g["num_visited_cells"][:64].min() > 0


def test_single_tetrahedron_and_tiny_meshes():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 1]], np.float32)
    for C in (np.array([[0, 1, 2, 3]], np.int32), np.array([[0, 1, 2, 3], [1, 2, 3, 4]], np.int32)):
        tr = make_tracer(V, C)
        o = np.array([[-1, 0.2, 0.2], [0.1, 0.1, -1], [2, 2, 2]], np.float32)
        d = np.array([[1, 0, 0], [0, 0, 1], [-1, -1, -1]], np.float32)
        assert_same(gpu_trace(tr, o, d, 8), orc.OracleMesh(V, C).trace_rays(o, d, 8))


def test_api_errors(cube_mesh):
    from tetranerf import cpp

    V, C = cube_mesh
    tr = cpp.TetrahedraTracer(DEV)
    o = torch.zeros((2, 3), device=DEV)
    with pytest.raises(RuntimeError, match="load_tetrahedra|loaded"):
        tr.trace_rays(o, o, 16)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    with pytest.raises(RuntimeError, match="power of 2"):  # py_binding.cpp:44-47
        tr.trace_rays(o, o, 12)
    with pytest.raises(RuntimeError, match="float32"):
        tr.trace_rays(o.double(), o.double(), 16)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        tr.trace_rays(o.cpu(), o.cpu(), 16)
    with pytest.raises(RuntimeError, match="contiguous"):
        tr.trace_rays(torch.zeros((3, 2), device=DEV).T, o, 16)
    bad = torch.tensor([[0, 1, 2, 3], [0, 1, 2, 4], [0, 1, 2, 5]], dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="more than two"):  # tetrahedra_tracer.cpp:64-66
        cpp.TetrahedraTracer(DEV).load_tetrahedra(torch.rand((6, 3), device=DEV), bad)
    assert tr.device == DEV


def test_trace_rays_triangles(small_mesh):
    V, C = small_mesh
    tr = make_tracer(V, C)
    o, d = syn.camera_rays(300)
    out = tr.trace_rays_triangles(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), 256)
    ref = orc.OracleMesh(V, C).trace_rays_triangles(o, d, 256)
    for k in ref:
        a = out[k].cpu().numpy()
        assert np.array_equal(a.view(np.uint32), ref[k].view(np.uint32)), k


def test_find_tetrahedra(cube_mesh, small_mesh):
    V, C = cube_mesh
    tr = make_tracer(V, C)

    def mix(*a):
        return sum(V[i] * w for i, w in zip(a[::2], a[1::2]))

    pts = np.stack([mix(0, 0.23, 1, 0.27, 2, 0.21, 8, 0.29), mix(2, 0.23, 4, 0.24, 6, 0.26, 8, 0.27), mix(3, 0.39, 5, 0.41, 7, 0.09, 8, 0.11)]).astype(np.float32)
    out = tr.find_tetrahedra(torch.from_numpy(pts).to(DEV))
    # golden values of the reference's tests/test_tetrahedra_tracer.py:324-344
    assert out["tetrahedra"].cpu().tolist() == [0, 5, 11]
    gt_coords = torch.tensor([[0.23, 0.27, 0.21, 0.29], [0.23, 0.24, 0.26, 0.27], [0.39, 0.41, 0.09, 0.11]])
    gt_idx = torch.tensor([[0, 1, 2, 8], [2, 4, 6, 8], [3, 5, 7, 8]], dtype=torch.int32)
    bc = out["barycentric_coordinates"].cpu()
    bc = torch.cat((1 - bc.sum(-1, keepdim=True), bc), -1)
    for i in range(3):
        idx, order = torch.sort(out["vertex_indices"][i].cpu())
        assert torch.all(idx == gt_idx[i])
        torch.testing.assert_close(bc[i][order], gt_coords[i], rtol=1.3e-6, atol=1e-5)
    # random points in a random mesh vs the oracle (bit-exact), including points outside the hull
    V, C = small_mesh
    tr = make_tracer(V, C)
    p = (np.random.default_rng(4).random((500, 3)) * 1.2 - 0.1).astype(np.float32)
    out = tr.find_tetrahedra(torch.from_numpy(p).to(DEV))
    ref = orc.OracleMesh(V, C).find_tetrahedra(p)
    assert np.array_equal(out["tetrahedra"].cpu().numpy(), ref["tetrahedra"])
    assert np.array_equal(out["vertex_indices"].cpu().numpy(), ref["vertex_indices"])
    assert np.array_equal(out["barycentric_coordinates"].cpu().numpy().view(np.uint32), ref["barycentric_coordinates"].view(np.uint32))
    assert np.array_equal(out["valid_mask"].cpu().numpy(), ref["valid_mask"])
    assert 0.3 < ref["valid_mask"].mean() < 0.9


def test_walk_fast_path_classification(small_mesh):
    """the adjacency walk certifies most rays itself; the rest (sub-eps slivers, degenerate hits) go through the exact stage"""
    V, C = small_mesh
    tr = make_tracer(V, C)
    o, d = syn.camera_rays(2000, seed=21)
    g = gpu_trace(tr, o, d, 512)
    walkable, listed = tr.trace_stats()
    assert walkable
    if IMPL != "bvh":  # any form of the walk
        assert 0 < listed < 0.15 * len(o), listed
    assert_same(g, orc.OracleMesh(V, C).trace_rays(o, d, 512))


def test_non_convex_mesh_takes_exact_path(small_mesh):
    """remove tetrahedra from the hull -> non-convex hull: rays leave and re-enter; the reference pairs the two hull
    faces of a gap into a record with cell = -1 (optix_trace_rays.cu:22-37: E == E).  Walk disabled, exact path used."""
    V, C = small_mesh
    cen = V[C].mean(1)
    keep = ~((np.abs(cen[:, 0] - 0.5) < 0.12) & (cen[:, 1] < 0.6))  # carve a slot into the cloud
    C2 = np.ascontiguousarray(C[keep])
    tr = make_tracer(V, C2)
    o, d = syn.camera_rays(600, seed=5)
    g = gpu_trace(tr, o, d, 512)
    walkable, _ = tr.trace_stats()
    assert not walkable
    ref = orc.OracleMesh(V, C2).trace_rays(o, d, 512)
    assert_same(g, ref)
    assert (ref["visited_cells"][np.arange(512)[None] < ref["num_visited_cells"][:, None]] == -1).any()  # gap records exist
