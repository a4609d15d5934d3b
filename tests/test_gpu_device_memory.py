"""GPU: ownership of the library's device memory (DESIGN.md §3), through tn_debug_device_bytes -- the bytes every library-owned buffer
of the process holds.  Each test reads only the change around its own calls, so other live tracers do not matter:

* a tracer's whole lifecycle (load, renders with every optional output, both training pairs in both modes with ray, vertex and depth
  gradients, a surface extraction) gives back every byte when the tracer is destroyed;
* repeating an identical training step or render allocates nothing;
* alternating shapes reach a fixed point once each shape has run (every buffer grows to the larger of its two needs);
* a saved training step leaves the tracer's own fine-pass state unallocated;
* calls that fail with an argument, mesh or state error allocate nothing."""
import contextlib
import gc

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LN2 = float(np.log(2.0))


def _bytes():
    """after collecting garbage, so that no tracer dropped earlier is destroyed between two readings"""
    from tetranerf.utils.extension import tetranerf_cpp_extension as ext

    gc.collect()
    torch.cuda.synchronize()
    return int(ext._lib.tn_debug_device_bytes())


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _settings(Sc=64, Sf=64, M=256):
    from tetranerf.b200.render import RenderSettings

    return RenderSettings(num_samples=Sc, num_fine_samples=Sf, max_intersected_triangles=M)


def _setup(V, C):
    """tracer and fused renderer on a field with a non-empty iso-surface at LN2"""
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(DEV))
    fr.set_weights(params)
    return tr, fr, field


def _rays(R, st, seed=11):
    o, d = syn.camera_rays(R, seed=seed)
    g = torch.Generator().manual_seed(seed)
    jc = torch.rand((R, st.num_samples + 1), generator=g).to(DEV)
    jf = torch.rand((R, st.num_fine_samples + 1), generator=g).to(DEV)
    return torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), jc, jf


def _train_step(fr, nv, st, rays, det):
    """one step of the tracer-held training pair"""
    o, d, jc, jf = rays
    R = o.shape[0]
    with _deterministic(det):
        fr.train_forward(o, d, st, jc, jf)
        fr.train_backward(torch.full((R, 3), 1.0 / R, device=DEV), torch.full((R,), 0.05 / R, device=DEV), nv)


def _saved_step(fr, nv, st, rays, det):
    """one step of the saved training pair, with every optional output and gradient"""
    o, d, jc, jf = rays
    R = o.shape[0]
    with _deterministic(det):
        _, state = fr.train_forward_saved(o, d, st, jc, jf, expected_depth=True)
        fr.train_backward_saved(state, torch.full((R, 3), 1.0 / R, device=DEV), torch.full((R,), 0.05 / R, device=DEV), nv,
                                grad_origins=True, grad_directions=True, grad_vertices=True,
                                grad_expected_depth=torch.full((R,), 0.01 / R, device=DEV))


def test_lifecycle_frees_every_byte(small_mesh):
    V, C = small_mesh
    b0 = _bytes()
    tr, fr, _ = _setup(V, C)
    st = _settings()
    rays = _rays(500, st)
    fr.render(rays[0], rays[1], st)
    fr.render(rays[0], rays[1], st, normals=True, expected_depth=True)
    for det in (False, True):
        _train_step(fr, len(V), st, rays, det)
        _saved_step(fr, len(V), st, rays, det)
    surf = fr.extract_surface(LN2)
    assert surf["faces"].shape[0] > 0
    tr.synchronize()
    assert _bytes() > b0
    del tr, fr, surf
    assert _bytes() == b0


def test_steady_state_allocates_nothing(small_mesh):
    V, C = small_mesh
    tr, fr, _ = _setup(V, C)
    st = _settings()
    rays = _rays(500, st)
    for det in (False, True):
        _saved_step(fr, len(V), st, rays, det)
        b = _bytes()
        for _ in range(3):
            _saved_step(fr, len(V), st, rays, det)
        assert _bytes() == b, f"deterministic={det}: a repeated training step allocated"
    fr.render(rays[0], rays[1], st, normals=True, expected_depth=True)
    b = _bytes()
    for _ in range(3):
        fr.render(rays[0], rays[1], st, normals=True, expected_depth=True)
    assert _bytes() == b, "a repeated render allocated"


def test_alternating_shapes_reach_a_fixed_point(small_mesh):
    """deterministic mode, (1200 rays, 64 fine samples) and (300 rays, 512 fine samples): neither shape's workspace covers the other's,
    and each buffer keeps the larger of the two"""
    V, C = small_mesh
    tr, fr, _ = _setup(V, C)
    a, b = _settings(Sf=64), _settings(Sf=512)
    ra, rb = _rays(1200, a, seed=12), _rays(300, b, seed=13)
    _train_step(fr, len(V), a, ra, det=True)
    _train_step(fr, len(V), b, rb, det=True)
    fixed = _bytes()
    for _ in range(2):
        _train_step(fr, len(V), a, ra, det=True)
        assert _bytes() == fixed
        _train_step(fr, len(V), b, rb, det=True)
        assert _bytes() == fixed


def test_saved_step_leaves_the_tracer_state_unallocated(small_mesh):
    """the fine pass of a saved training step writes into its blob only, so the first tracer-held forward after it allocates the
    tracer's own saved-state blob"""
    V, C = small_mesh
    tr, fr, _ = _setup(V, C)
    st = _settings()
    o, d, jc, jf = rays = _rays(500, st)
    _saved_step(fr, len(V), st, rays, det=False)
    b = _bytes()
    fr.train_forward(o, d, st, jc, jf)
    assert _bytes() - b >= fr.train_saved_bytes(500, st) - 256


def test_failed_calls_allocate_nothing(small_mesh, cube_mesh):
    from tetranerf import cpp

    # a triangle shared by three tetrahedra, on a fresh tracer (TN_ERR_MESH after the face build's temporaries were allocated)
    Vc, Cc = cube_mesh
    fresh = cpp.TetrahedraTracer(DEV)
    b = _bytes()
    bad = np.concatenate([Cc, Cc[:1], Cc[:1]]).astype(Cc.dtype)
    with pytest.raises(RuntimeError, match="shared by more than two"):
        fresh.load_tetrahedra(torch.from_numpy(Vc).to(DEV), torch.from_numpy(bad).to(DEV))
    assert _bytes() == b
    del fresh

    V, C = small_mesh
    tr, fr, field = _setup(V, C)
    st = _settings()
    o, d, _, _ = _rays(500, st)
    fr.render(o, d, st)
    # sample counts beyond the per-ray kernels' shared memory (TN_ERR_ARG)
    b = _bytes()
    with pytest.raises(RuntimeError, match="shared memory"):
        fr.render(o, d, _settings(Sc=4096, Sf=4096, M=512))
    assert _bytes() == b
    # a field whose vertex count differs from the mesh's (TN_ERR_ARG)
    fr.set_field(torch.from_numpy(np.ascontiguousarray(field[:, :-1])).to(DEV))
    b = _bytes()
    with pytest.raises(RuntimeError, match="different vertex count"):
        fr.render(o, d, st)
    assert _bytes() == b
    # a non-finite vertex coordinate, after a first refit (TN_ERR_ARG)
    xyz = torch.from_numpy(V).to(DEV)
    tr.update_vertices(xyz)
    b = _bytes()
    xyz = xyz.clone()
    xyz[3, 1] = float("nan")
    with pytest.raises(RuntimeError, match="finite"):
        tr.update_vertices(xyz)
    assert _bytes() == b
