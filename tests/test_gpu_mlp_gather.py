"""GPU: the two field gathers of the fused MLP passes (tn_set_mlp_gather: rows cached in L1, the default, or streamed past it)
give bit-identical pixels and per-sample values: rgb / accumulation / depth / mask, the fine pass's (sigma, r, g, b) per sample
and the coarse pass's densities."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_render import _from_ptr, setup

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _settings(cfgname, fine_samples=None):
    from tetranerf.b200.render import RenderSettings

    st = RenderSettings.tetra_nerf() if cfgname == "tetra_nerf" else RenderSettings.tetra_nerf_original()
    if fine_samples is not None:
        st.num_fine_samples = fine_samples
    return st


def _render(tr, fr, o, d, st, gather):
    tr.set_mlp_gather(gather)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    tr.synchronize()
    b = fr.debug_buffers()
    n_act = int(_from_ptr(b["n_active"], (1,), torch.int32)[0])
    single = st.num_fine_samples == 0
    S2 = st.num_samples if single else st.num_samples + st.num_fine_samples + 1
    res = {k: out[k].cpu().clone() for k in ("rgb", "accumulation", "depth", "ray_mask")}
    # per-sample buffers are in slot order, and which slot a ray gets may change between two renders: compare in ray order
    order = torch.argsort(_from_ptr(b["ray_list"], (n_act,), torch.int32).cpu().long())
    res["out_f"] = _from_ptr(b["out_f"], (n_act, S2, 4), torch.float32).cpu()[order]
    if not single:
        res["dens_c"] = _from_ptr(b["dens_c"], (n_act, st.num_samples), torch.float32).cpu()[order]
    return res, n_act * S2


def _assert_same_bits(tr, fr, o, d, st):
    new, rows = _render(tr, fr, o, d, st, 1)
    old, _ = _render(tr, fr, o, d, st, 0)
    assert rows > 0
    for k in new:
        assert torch.equal(new[k], old[k]), k
    assert bool(new["ray_mask"].any())
    return rows


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("cfgname", ["tetra_nerf", "tetra_nerf_original"])
def test_gathers_bitwise_equal(small_mesh, cfgname, prec):
    V, C = small_mesh
    tr, fr, _, _ = setup(V, C, prec=prec)
    o, d = syn.camera_rays(300)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]   # empty ray
    _assert_same_bits(tr, fr, o, d, _settings(cfgname))


@pytest.mark.parametrize("prec", [3, 2])
def test_gathers_bitwise_equal_single_pass(small_mesh, prec):
    V, C = small_mesh
    tr, fr, _, _ = setup(V, C, prec=prec)
    o, d = syn.camera_rays(300)
    _assert_same_bits(tr, fr, o, d, _settings("tetra_nerf", fine_samples=0))


def test_gathers_bitwise_equal_partial_tile(small_mesh):
    V, C = small_mesh
    tr, fr, _, _ = setup(V, C, prec=2)
    o, d = syn.camera_rays(37)
    rows = _assert_same_bits(tr, fr, o, d, _settings("tetra_nerf"))
    assert rows % 64 != 0  # the last tile of the fine pass has rows past the end


@pytest.mark.parametrize("prec", [3, 2])
def test_gathers_bitwise_equal_opaque_scene(small_mesh, prec):
    V, C = small_mesh
    field, params = syn.surface_scene(V, 40.0, orc.init_mlp_params(0))
    tr, fr, _, _ = setup(V, C, prec=prec, field=field, params=params)
    o, d = syn.camera_rays(300)
    _assert_same_bits(tr, fr, o, d, _settings("tetra_nerf"))


def test_gathers_bitwise_equal_tiny_mesh(cube_mesh):
    """a few tetrahedra: whole tiles read the same handful of field rows"""
    V, C = cube_mesh
    tr, fr, _, _ = setup(V.astype(np.float32), C.astype(np.int32), prec=2)
    o, d = syn.camera_rays(200)
    _assert_same_bits(tr, fr, o, d, _settings("tetra_nerf"))


def test_gather_setter_rejects_other_modes(small_mesh):
    V, C = small_mesh
    tr, _, _, _ = setup(V, C)
    with pytest.raises(RuntimeError):
        tr.set_mlp_gather(2)
