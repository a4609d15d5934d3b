"""Generates tests/golden/ref_kernels.npz on a GPU -- run from the repo root after build() has compiled the reference's own
kernels into oracle/_ref (oracle/Makefile, needs the reference sources at build time):

    python tests/golden/make_ref_kernels.py

The reference's find_matched_cells / interpolate_values / interpolate_values_backward (src/tetrahedra_tracer.cu) run on the
inputs of tests/test_gpu_ops.py::test_against_reference_kernels; a fixed sample of their outputs is stored (the full outputs are
tens of MB), so that the test compares against the reference without its sources."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path[:0] = [str(ROOT), str(ROOT / "tetra-nerf_b200"), str(ROOT / "tests")]

import test_gpu_ops as t  # noqa: E402
from tetranerf.b200 import synthetic as syn  # noqa: E402

DEV = t.DEV


def main():
    ref = ctypes.CDLL(str(ROOT / "oracle" / "_ref" / "libref_kernels.so"))
    V, C = syn.delaunay_mesh(3000, seed=0)  # the small_mesh fixture
    traced = t.make_traced(V, C)
    tr, out, dist, V, C = traced
    srt, g, field, gin, _, _ = t.ref_kernel_case(traced)
    R, S = srt.shape
    M = out["visited_cells"].shape[1]
    mask = torch.zeros((R, S), dtype=torch.bool, device=DEV)
    cell = torch.full((R, S), -1, dtype=torch.int32, device=DEV)
    bary = torch.zeros((R, S, 3), dtype=torch.float32, device=DEV)
    verts = torch.full((R, S, 4), -1, dtype=torch.int32, device=DEV)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    torch.cuda.synchronize()
    rc = ref.ref_find_matched_cells(ctypes.c_size_t(R), ctypes.c_size_t(S), ctypes.c_size_t(M), p(torch.from_numpy(C).to(DEV)),
                                    p(out["num_visited_cells"]), p(out["visited_cells"]), p(out["hit_distances"]),
                                    p(out["barycentric_coordinates"]), p(srt), p(out["vertex_indices"]), p(cell), p(verts), p(mask), p(bary))
    assert rc == 0
    N = R * S
    res = torch.empty((64, N), dtype=torch.float32, device=DEV)
    # the interpolation kernels see the same matched vertices / weights as this repo's (from its matcher, as in the test)
    vi, bw = g["vertex_indices"], g["barycentric_coordinates"]
    rc = ref.ref_interpolate_values4(ctypes.c_uint32(len(V)), ctypes.c_uint32(N), ctypes.c_uint32(64), p(vi), p(bw), p(field), p(res))
    assert rc == 0
    gref = torch.zeros((64, len(V)), device=DEV)
    rc = ref.ref_interpolate_values_backward4(ctypes.c_uint32(len(V)), ctypes.c_uint32(N), ctypes.c_uint32(64), p(vi), p(bw),
                                              p(gin.T.contiguous()), p(gref))
    assert rc == 0
    idx, vidx = t.ref_kernel_sample(N, len(V))
    np.savez_compressed(ROOT / "tests" / "golden" / "ref_kernels.npz", idx=idx, vidx=vidx,
                        mask=mask.reshape(N).cpu().numpy()[idx], cell=cell.reshape(N).cpu().numpy()[idx],
                        verts=verts.reshape(N, 4).cpu().numpy()[idx], bary=bary.reshape(N, 3).cpu().numpy()[idx],
                        interp=res.T.contiguous().cpu().numpy()[idx], grad=gref.cpu().numpy()[:, vidx])
    print("wrote tests/golden/ref_kernels.npz")


if __name__ == "__main__":
    main()
