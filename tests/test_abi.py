"""CPU: the C-ABI library loads and exports every symbol include/tetranerf_b200.h declares; without a CUDA
device the product fails loudly (no fallback)."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "tetra-nerf_b200" / "csrc" / "libtetranerf_b200.so"


def _declared():
    text = (ROOT / "include" / "tetranerf_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tn_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    assert LIB.exists(), "run python tetra-nerf_b200/build.py"
    lib = ctypes.CDLL(str(LIB))
    names = _declared()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/tetranerf_b200.h but not exported"


def test_shim_surface_matches_reference_pybind():
    """src/py_binding.cpp:433-449"""
    from tetranerf import cpp
    from tetranerf.utils import extension

    for n in ("trace_rays", "trace_rays_triangles", "find_visited_cells", "find_tetrahedra", "load_tetrahedra", "device"):
        assert hasattr(cpp.TetrahedraTracer, n)
    for n in ("triangulate", "find_average_spacing", "interpolate_values", "interpolate_values_backward", "gather_uint32", "scatter_ema_uint32"):
        assert callable(getattr(cpp, n))
    for n in ("TetrahedraTracer", "triangulate", "gather_uint32", "scatter_ema_uint32_", "interpolate_values", "add_barycentrics_grad"):
        assert hasattr(extension, n)


def test_non_cuda_device_raises():
    from tetranerf import cpp

    with pytest.raises(RuntimeError, match="CUDA device"):  # py_binding.cpp:31-33
        cpp.TetrahedraTracer(torch.device("cpu"))


@pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without GPU")
def test_no_silent_cpu_fallback():
    from tetranerf import cpp

    with pytest.raises(RuntimeError):
        cpp.TetrahedraTracer(torch.device("cuda:0"))
    with pytest.raises(RuntimeError):
        cpp.interpolate_values(torch.zeros((1, 4), dtype=torch.int32), torch.zeros((1, 3)), torch.zeros((2, 3)))


def test_out_of_scope_ops_raise():
    """the occupancy-field remnants and the CGAL spacing query exist by name but raise RuntimeError instead of computing"""
    from tetranerf import cpp

    with pytest.raises(RuntimeError):
        cpp.gather_uint32(torch.zeros(1), 0, torch.zeros(1, dtype=torch.int32))
    with pytest.raises(RuntimeError):
        cpp.scatter_ema_uint32(torch.zeros(1), 0, torch.zeros(1, dtype=torch.int32), 0.5, torch.zeros(1))
    with pytest.raises(RuntimeError):
        cpp.find_average_spacing(torch.zeros((4, 3)))
