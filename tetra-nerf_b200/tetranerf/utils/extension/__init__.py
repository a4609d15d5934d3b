"""Public Python surface of the native extension.

Same names as the reference module (tetranerf/utils/extension/__init__.py): `cpp`, `TetrahedraTracer`,
`triangulate`, `gather_uint32`, `scatter_ema_uint32_`, `interpolate_values` (differentiable w.r.t. the
field, reference :29-43,72-73) and `add_barycentrics_grad` (reference :45-68).  The native module here
is a ctypes shim over the C ABI in include/tetranerf_b200.h; when the shared library is missing every
use raises RuntimeError (the reference defers its ImportError the same way, :3-21) -- there is no CPU
or PyTorch fallback.
"""
import torch

_LOAD_ERROR = None
try:
    from . import tetranerf_cpp_extension as cpp
except (ImportError, OSError) as _e:  # library not built
    _LOAD_ERROR = _e

    class _Unavailable:
        """Stands in for the native module; any attribute is a callable that raises."""

        def __getattr__(self, name):
            def _raise(*_a, **_k):
                raise RuntimeError(
                    "ERROR: Tetra-NeRF could not load cpp extension. Please build the project first "
                    f"(python tetra-nerf_b200/build.py): {_LOAD_ERROR}"
                ) from _LOAD_ERROR

            return _raise

    cpp = _Unavailable()

TetrahedraTracer = cpp.TetrahedraTracer
triangulate = cpp.triangulate
gather_uint32 = cpp.gather_uint32
scatter_ema_uint32_ = cpp.scatter_ema_uint32


class _Interpolate(torch.autograd.Function):
    """interpolate_values with the field gradient of interpolate_values_backward (no gradient flows to
    the indices or the barycentric weights, as in the reference)."""

    @staticmethod
    def forward(ctx, vertex_indices, barycentric_coordinates, field):
        ctx.save_for_backward(vertex_indices, barycentric_coordinates, field)
        return cpp.interpolate_values(vertex_indices, barycentric_coordinates, field)

    @staticmethod
    def backward(ctx, grad_out):
        vi, w, field = ctx.saved_tensors
        return None, None, cpp.interpolate_values_backward(vi, w, field, grad_out.contiguous())


def interpolate_values(vertex_indices, barycentric_coordinates, field):
    return _Interpolate.apply(vertex_indices, barycentric_coordinates, field)


class _BaryGrad(torch.autograd.Function):
    """Identity on the barycentrics that back-propagates to tetrahedron vertices / query points
    (pose-optimisation stub of the reference; not used by the model)."""

    @staticmethod
    def forward(ctx, barycentrics, vertices, points):
        ctx.save_for_backward(barycentrics, vertices)
        return barycentrics

    @staticmethod
    def backward(ctx, g):
        bary, verts = ctx.saved_tensors
        need_v, need_p = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        gv = gp = None
        if need_v or need_p:
            edges = verts[..., 1:, :] - verts[..., :1, :]
            m = torch.linalg.solve(edges, g)
            if need_p:
                gp = m
            if need_v:
                full = torch.cat([1.0 - bary.sum(-1, keepdim=True), bary], -1)
                gv = -(full.unsqueeze(-1) * m.unsqueeze(-2))
        return g, gv, gp


def add_barycentrics_grad(barycentrics, vertices, points):
    return _BaryGrad.apply(barycentrics, vertices, points)
