import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "tetra-nerf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def cube_mesh():
    from tetranerf.b200 import synthetic as syn

    return syn.CUBE_VERTICES.copy(), syn.CUBE_CELLS.copy()


@pytest.fixture(scope="session")
def small_mesh():
    from tetranerf.b200 import synthetic as syn

    return syn.delaunay_mesh(3000, seed=0)


@pytest.fixture(scope="session")
def medium_mesh():
    from tetranerf.b200 import synthetic as syn

    return syn.delaunay_mesh(20000, seed=5)


# the bit-identical implementations of trace_rays and how to force each one: (walk_min_rays, solo range, quad range)
TRACE_IMPLS = {
    "walk": (0, (1, 0), (1, 0)),                                  # adjacency walk, 32 rays per warp
    "walk_solo": (2**32 - 1, (0, 2**32 - 1), (1, 0)),             # adjacency walk, one ray per warp
    "walk_quad": (2**32 - 1, (1, 0), (0, 2**32 - 1)),             # adjacency walk, 8 rays per warp (4 lanes per ray), speculative record loads
    "walk_quad_pf": (2**32 - 1, (1, 0), (0, 2**32 - 1), 0),       # the same with prefetches instead (the form large batches take)
    "bvh": (2**32 - 1, (1, 0), (1, 0)),                           # warp-per-ray all-hits BVH gather
}


def force_trace_impl(tracer, name):
    w = TRACE_IMPLS[name]
    tracer.set_walk_min_rays(w[0])
    tracer.set_walk_solo_range(*w[1])
    tracer.set_walk_quad_range(*w[2])
    tracer.set_walk_quad_spec_max_rays(w[3] if len(w) > 3 else 2**32 - 1)
