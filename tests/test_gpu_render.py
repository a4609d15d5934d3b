"""GPU parity of the fused render (tn_render) against the CPU oracle render (oracle.render = model.py:520-662 in
eval mode): ray_mask exact, rgb / accumulation within 1e-4 absolute (the north-star tolerance), plus the
intermediate stages (bins, matched samples, densities) so that a failure localises."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _from_ptr(ptr, shape, dtype):
    n = int(np.prod(shape))
    t = torch.empty(shape, dtype=dtype, device=DEV)
    rt = ctypes.CDLL("libcudart.so")
    rt.cudaMemcpy(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(ptr), ctypes.c_size_t(n * t.element_size()), ctypes.c_int(3))
    return t


def setup(V, C, field_kind="normal", prec=3, field=None, params=None):
    """field / params default to syn.random_field(kind=field_kind) and the torch-default network"""
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    field = syn.random_field(len(V), 64, seed=3, kind=field_kind) if field is None else field
    params = orc.init_mlp_params(0) if params is None else params
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(DEV))
    fr.set_weights(params)
    fr.set_mlp_precision(prec)
    return tr, fr, field, params


# prec: operand precision of the tensor-core MLP -- 3 = bf16x3 (fp32-level), 2 = f16w2 (fp16 activations x fp16 hi/lo weights, 2 MMAs per
# product).  On this (torch-default, unit-scale) network BOTH are held to the same bars: 1e-4 absolute per sample and per pixel.  f16w2's
# per-sample error is relative to the activations (~4.9e-4 sigma, 1.8e-4 colour on a trained-NeRF-like network: tests/test_gpu_opaque.py,
# DESIGN 4.2); its pixels stay within 1e-4 there too.
@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("cfgname", ["tetra_nerf", "tetra_nerf_original", "small_uniform", "small_biased", "tetra_nerf_cube"])
@pytest.mark.parametrize("field_kind", ["normal", "init"])
def test_fused_render_vs_oracle(small_mesh, cube_mesh, cfgname, field_kind, prec):
    from tetranerf.b200.render import RenderSettings

    # tetra_nerf_cube: the 12-tetrahedra cube, so whole MLP tiles read the same few field rows
    V, C = cube_mesh if cfgname == "tetra_nerf_cube" else small_mesh
    tr, fr, field, params = setup(V, C, field_kind, prec)
    o, d = syn.camera_rays(300)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]       # empty ray
    o[17] = [0.5, 0.5, 0.5]                   # origin inside the mesh
    if cfgname in ("tetra_nerf", "tetra_nerf_cube"):
        st, oc = RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()
    elif cfgname == "tetra_nerf_original":
        st, oc = RenderSettings.tetra_nerf_original(), orc.RenderConfig.tetra_nerf_original()
    elif cfgname == "small_uniform":
        st, oc = RenderSettings(num_samples=48, num_fine_samples=33), orc.RenderConfig(num_samples=48, num_fine_samples=33)
    else:
        st = RenderSettings(num_samples=20, num_fine_samples=20, use_biased_sampler=True, max_intersected_triangles=256)
        oc = orc.RenderConfig(num_samples=20, num_fine_samples=20, use_biased_sampler=True, max_intersected_triangles=256)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    tr.synchronize()
    ref = orc.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, oc, return_aux=True)
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    assert not bool(ref["ray_mask"][5])
    assert out["rgb"][5].cpu().tolist() == [1.0, 1.0, 1.0] and float(out["depth"][5]) == st.far_plane and float(out["accumulation"][5]) == 0

    # ---- intermediates (slot order -> ray order) ----
    bufs = fr.debug_buffers()
    n_act = int(_from_ptr(bufs["n_active"], (1,), torch.int32)[0])
    assert n_act == int(ref["ray_mask"].sum())
    ray_list = _from_ptr(bufs["ray_list"], (n_act,), torch.int32).cpu().long()
    active = torch.nonzero(ref["ray_mask"]).flatten()
    inv = torch.empty(len(o), dtype=torch.long)
    inv[active] = torch.arange(n_act)
    order = inv[ray_list]  # row of the oracle's compacted arrays for each slot
    Sc, S2 = st.num_samples, st.num_samples + st.num_fine_samples + 1
    assert (n_act * S2) % 64 != 0  # the fine pass ends in a partly filled 64-row MLP tile
    aux = ref["aux"]
    eb_c = _from_ptr(bufs["ebins_c"], (n_act, Sc + 1), torch.float32).cpu()
    torch.testing.assert_close(eb_c, aux["coarse_euclid"][order], rtol=2e-6, atol=2e-6)
    dens = _from_ptr(bufs["dens_c"], (n_act, Sc), torch.float32).cpu()
    dref = aux["coarse_density"][order][..., 0]
    print(cfgname, field_kind, f"prec={prec}", "coarse density max abs err", (dens - dref).abs().max().item())
    assert (dens - dref).abs().max().item() < 1e-4
    eb_f = _from_ptr(bufs["ebins_f"], (n_act, S2 + 1), torch.float32).cpu()
    print("fine bins max abs err", (eb_f - aux["fine_euclid"][order]).abs().max().item())
    torch.testing.assert_close(eb_f, aux["fine_euclid"][order], rtol=1e-4, atol=1e-4)
    outf = _from_ptr(bufs["out_f"], (n_act, S2, 4), torch.float32).cpu()
    # north_star: fp32 colour/density within 1e-4 abs PER SAMPLE.  The fine sample positions agree to ~1e-7 only (PDF
    # inversion in fp32), so a sample sitting on a face may legitimately land in the neighbouring tetrahedron ("flip"):
    # those are excluded -- and counted -- everything else is asserted.
    vi_gpu = _from_ptr(bufs["vi_f"], (n_act, S2, 4), torch.int32).cpu()
    vi_ref = torch.from_numpy(aux["matched"]["vertex_indices"])[order]
    flipped = (vi_gpu != vi_ref).any(-1)
    sig_err = (outf[..., 0] - aux["sigmas"][order][..., 0]).abs()
    col_err = (outf[..., 1:] - aux["colors"][order]).abs().amax(-1)
    flip_rate = flipped.float().mean().item()
    print(f"sigma err: max {sig_err[~flipped].max().item():.2e} median {sig_err.median().item():.2e}  colour err max "
          f"{col_err[~flipped].max().item():.2e}  flipped samples {int(flipped.sum())} ({100 * flip_rate:.3f} %)")
    assert flip_rate < 2e-3, flip_rate
    # density: 1e-4 absolute, or relative where sigma is large (softplus is the identity there and fp32 itself has ~1e-6 relative)
    sig_ref = aux["sigmas"][order][..., 0]
    assert bool((sig_err[~flipped] <= 1e-4 + 2e-5 * sig_ref[~flipped].abs()).all()), sig_err[~flipped].max().item()
    assert col_err[~flipped].max().item() <= 1e-4, col_err[~flipped].max().item()
    # ---- pixels ----
    e_rgb = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"]).abs().max().item()
    e_dep = (out["depth"].cpu() - ref["depth"]).abs()
    print(f"{cfgname}/{field_kind}/prec={prec}: max|rgb| {e_rgb:.2e}  max|acc| {e_acc:.2e}  depth: max {e_dep.max().item():.2e} median {e_dep.median().item():.2e}")
    assert e_rgb < 1e-4 and e_acc < 1e-4
    # median depth is a step function of the cumulative weights: allow a handful of rays to pick the neighbouring sample
    assert (e_dep.flatten() > 1e-4).sum().item() <= max(2, len(o) // 100)


@pytest.mark.parametrize("prec", [3, 2])
@pytest.mark.parametrize("biased", [False, True])
def test_fused_render_single_pass(small_mesh, biased, prec):
    """num_fine_samples == 0 (model.py:573: the PDF pass is skipped, colours come from the first pass)"""
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    tr, fr, field, params = setup(V, C, prec=prec)
    o, d = syn.camera_rays(200, seed=9)
    o[7] = [5, 5, 5]; d[7] = [1, 0, 0]
    st = RenderSettings(num_samples=96, num_fine_samples=0, use_biased_sampler=biased)
    oc = orc.RenderConfig(num_samples=96, num_fine_samples=0, use_biased_sampler=biased)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    tr.synchronize()
    ref = orc.render(orc.OracleMesh(V, C), torch.from_numpy(field), params, o, d, oc)
    assert torch.equal(out["ray_mask"].cpu(), ref["ray_mask"])
    e_rgb = (out["rgb"].cpu() - ref["rgb"]).abs().max().item()
    e_acc = (out["accumulation"].cpu() - ref["accumulation"]).abs().max().item()
    e_dep = (out["depth"].cpu() - ref["depth"]).abs()
    print(f"single pass biased={biased}: max|rgb| {e_rgb:.2e} max|acc| {e_acc:.2e} depth max {e_dep.max().item():.2e}")
    assert e_rgb < 1e-4 and e_acc < 1e-4
    assert (e_dep.flatten() > 1e-4).sum().item() <= 2


def test_fused_render_is_deterministic_and_reusable(small_mesh):
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    tr, fr, field, params = setup(V, C)
    o, d = syn.sphere_rays(513)
    st = RenderSettings.tetra_nerf()
    a = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    a = {k: v.clone() for k, v in a.items()}
    b = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), st)
    tr.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # smaller batch afterwards reuses the workspace
    c = fr.render(torch.from_numpy(o[:100]).to(DEV), torch.from_numpy(d[:100]).to(DEV), st)
    tr.synchronize()
    assert torch.equal(c["rgb"], a["rgb"][:100])


def test_f16w2_saturates_out_of_range_activations(small_mesh):
    """the f16w2 mode carries activations as fp16: features beyond +-65504 must saturate (not turn into inf / NaN pixels);
    bf16x3 covers the fp32 range and stays the reference for such fields"""
    from tetranerf.b200.render import RenderSettings

    V, C = small_mesh
    tr, fr, field, params = setup(V, C, prec=2)
    fr.set_field(torch.from_numpy(field * 3.0e5).to(DEV))
    o, d = syn.camera_rays(128, seed=4)
    out = fr.render(torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), RenderSettings.tetra_nerf())
    tr.synchronize()
    for k in ("rgb", "accumulation", "depth"):
        assert bool(torch.isfinite(out[k]).all()), k
