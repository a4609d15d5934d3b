"""GPU: the fused path's field shadow (tn_render_set_field) is stored in fragment order.  Within each 16-feature block b, feature
16b + 8h + 2t + e (h, e in {0, 1}, t in 0..3) sits at position 16b + 4t + 2h + e of the vertex's 256-byte row, so one 16-byte load gives a
thread of a wgmma A fragment row its four features of one k-step (DESIGN §3).  Checked here: the shadow read back against that
permutation, and that every kernel that reads the shadow (both MLP passes in both precisions, the normals, the training backward, the
ray and vertex gradients) gives the same bits after the shadow is rewritten from the same field.  Their values against the oracle and
float64 are checked by the tests of each path."""
import ctypes

import numpy as np
import pytest
import torch

from tetranerf.b200 import synthetic as syn
from test_gpu_train import DEV, _setup

pytestmark = pytest.mark.gpu


def _fragment_pos(f):
    """position of feature f in a shadow row, written out independently of the library's field_pos"""
    b, r = divmod(f, 16)
    h, q = divmod(r, 8)
    t, e = divmod(q, 2)
    return 16 * b + 4 * t + 2 * h + e


def _shadow(fr, V):
    torch.cuda.synchronize()
    t = torch.empty((V, 64), dtype=torch.float32, device=DEV)
    rc = ctypes.CDLL("libcudart.so").cudaMemcpy(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(fr.debug_buffers()["fshadow"]),
                                                ctypes.c_size_t(t.numel() * 4), ctypes.c_int(3))
    assert rc == 0
    return t.cpu().numpy()


def test_shadow_is_in_fragment_order(small_mesh):
    V, C = small_mesh
    nv = len(V)
    # distinct values, exact in float32: feature f of vertex v = 64 v + f
    field = (np.arange(nv, dtype=np.float64)[None, :] * 64 + np.arange(64, dtype=np.float64)[:, None]).astype(np.float32)
    assert np.unique(field).size == field.size
    _, fr, _ = _setup(V, C, field)
    got = _shadow(fr, nv)
    want = np.empty((nv, 64), dtype=np.float32)
    want[:, [_fragment_pos(f) for f in range(64)]] = field.T
    assert np.array_equal(got, want)


def _scene(small_mesh, R=400):
    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    other = syn.random_field(len(V), 64, seed=11)
    o, d = syn.camera_rays(R, seed=21)
    g = torch.Generator().manual_seed(7)
    return V, C, field, other, torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), g


def _all_paths(fr, nv, o, d, jc, jf, target):
    """every call that reads the field shadow -> {name: tensor}, cloned"""
    from tetranerf.b200.render import RenderSettings

    st = RenderSettings.tetra_nerf()
    res = {}
    for prec in (2, 3):
        fr.set_mlp_precision(prec)
        out = fr.render(o, d, st, normals=True, expected_depth=True)
        res.update({f"render{prec}/{k}": v.clone() for k, v in out.items()})
    out, state = fr.train_forward_saved(o, d, st, jc, jf)
    R = o.shape[0]
    g_rgb = (2.0 * (out["rgb"] - target) / (3 * R)).contiguous()
    g_acc = torch.full((R,), 0.05 / R, device=DEV)
    gf, gp, go, gd, gv = fr.train_backward_saved(state, g_rgb, g_acc, nv, True, grad_origins=True, grad_directions=True, grad_vertices=True)
    torch.cuda.synchronize()
    res.update({f"train/{k}": v.clone() for k, v in out.items()})
    res.update({"grad/field": gf.clone(), "grad/origins": go.clone(), "grad/directions": gd.clone(), "grad/vertices": gv.clone()})
    res.update({f"grad/{k}": v.clone() for k, v in gp.items()})
    return res


def test_rewritten_shadow_gives_the_same_bits(small_mesh, monkeypatch):
    """the same calls before and after the shadow is rewritten from the same field (with another field set in between): bitwise equal
    in deterministic mode, on the render in both precisions with normals and expected depth, and on the training step with ray and
    vertex gradients"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C, field, other, o, d, g = _scene(small_mesh)
    _, fr, _ = _setup(V, C, field)
    from tetranerf.b200.render import RenderSettings

    st = RenderSettings.tetra_nerf()
    R = o.shape[0]
    jc = torch.rand((R, st.num_samples + 1), generator=g).to(DEV)
    jf = torch.rand((R, st.num_fine_samples + 1), generator=g).to(DEV)
    target = torch.rand((R, 3), generator=g).to(DEV)
    a = _all_paths(fr, len(V), o, d, jc, jf, target)
    assert a["render2/ray_mask"].any() and a["grad/vertices"].abs().max() > 0
    fr.set_field(torch.from_numpy(other).to(DEV))
    c = _all_paths(fr, len(V), o, d, jc, jf, target)
    assert not torch.equal(a["render2/rgb"], c["render2/rgb"])  # the second field reaches the outputs
    fr.set_field(torch.from_numpy(field).to(DEV))
    b = _all_paths(fr, len(V), o, d, jc, jf, target)
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k
