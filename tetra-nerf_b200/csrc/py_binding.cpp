// py_binding.cpp -- the pybind11 module `tetranerf_cpp_extension` (reference: src/py_binding.cpp:433-449) over the C ABI of
// include/tetranerf_b200.h.  Same class / function names, argument checks and error behaviour as the reference binding
// (std::runtime_error -> Python RuntimeError); tensors in, tensors out; every device call is hand-written CUDA inside
// libtetranerf_b200.so, launched on torch's current stream (the reference uses a private stream and a device-wide sync per
// call, src/tetrahedra_tracer.cpp:173-174).  Built in-tree by tetra-nerf_b200/build.py (INTEGRATION.md, option B); the ctypes
// shim next to it (tetranerf_cpp_extension.py) exposes the identical surface without a compile step.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <stdexcept>
#include <string>

#include "../../include/tetranerf_b200.h"

namespace py = pybind11;

namespace {

void check(int rc) {
    if (rc != 0) throw std::runtime_error(tn_last_error());
}
void require(bool cond, const std::string &msg) {
    if (!cond) throw std::runtime_error(msg);
}
void check_input(const torch::Tensor &x, const char *name) {  // CHECK_INPUT, py_binding.cpp:15-21
    require(x.is_cuda(), std::string(name) + " must be a CUDA tensor");
    require(x.is_contiguous(), std::string(name) + " must be contiguous");
}
void *stream_of(const torch::Device &d) { return (void *)at::cuda::getCurrentCUDAStream(d.index()).stream(); }
template <typename T> T *ptr(const torch::Tensor &t) { return reinterpret_cast<T *>(t.data_ptr()); }

class PyTetrahedraTracer {  // py_binding.cpp:28-227
   public:
    explicit PyTetrahedraTracer(const torch::Device &device) : device_(device) {
        if (!device.is_cuda()) throw std::runtime_error("The device argument must be a CUDA device.");  // py_binding.cpp:31-33
        if (!device_.has_index()) device_ = torch::Device(torch::kCUDA, (c10::DeviceIndex)at::cuda::current_device());
        check(tn_create(device_.index(), &h_));
    }
    ~PyTetrahedraTracer() {
        if (h_) tn_destroy(h_);
        h_ = nullptr;
    }
    PyTetrahedraTracer(const PyTetrahedraTracer &) = delete;
    PyTetrahedraTracer &operator=(const PyTetrahedraTracer &) = delete;

    torch::Device device() const { return device_; }
    uintptr_t handle() const { return reinterpret_cast<uintptr_t>(h_); }

    void check_float_dim3(const torch::Tensor &x, const char *name) const {  // CHECK_FLOAT_DIM3, py_binding.cpp:22-26
        check_input(x, name);
        require(x.device() == device_, std::string(name) + " must be on the same device");
        require(x.dtype() == torch::kFloat32, std::string(name) + " must have float32 type");
        require(x.size(-1) == 3, std::string(name) + " must have last dimension with size 3");
    }
    void on_device(const torch::Tensor &x, const char *name) const {
        check_input(x, name);
        require(x.device() == device_, std::string(name) + " must be on the same device");
    }

    void load_tetrahedra(const torch::Tensor &xyz, const torch::Tensor &cells) {  // py_binding.cpp:144-161
        check_float_dim3(xyz, "xyz");
        on_device(cells, "cells");
        require(cells.size(-1) == 4, "indices must have last dimension with size 4");
        require(cells.dtype() == torch::kInt32, "indices must have int32 type");
        vertices_ = xyz;  // borrowed by the tracer: keep them alive (:154-155)
        cells_ = cells;
        c10::cuda::CUDAGuard guard(device_);
        check(tn_load_tetrahedra(h_, ptr<float>(xyz), (uint32_t)(xyz.numel() / 3), ptr<uint32_t>(cells), (uint32_t)(cells.numel() / 4), stream_of(device_)));
    }

    py::dict trace_rays(const torch::Tensor &o, const torch::Tensor &d, unsigned long M) {  // py_binding.cpp:41-76
        if (M == 0 || (M & (M - 1)) != 0) throw std::runtime_error("max_ray_triangles must be a power of 2.");
        check_float_dim3(o, "ray_origins");
        check_float_dim3(d, "ray_directions");
        torch::NoGradGuard no_grad;
        const int64_t R = o.numel() / 3, m = (int64_t)M;
        auto fo = torch::TensorOptions().device(device_);
        auto num = torch::empty({R}, fo.dtype(torch::kInt32));
        auto cells = torch::empty({R, m}, fo.dtype(torch::kInt32));
        auto bary = torch::empty({R, m, 2, 3}, fo.dtype(torch::kFloat32));
        auto dist = torch::empty({R, m, 2}, fo.dtype(torch::kFloat32));
        auto verts = torch::empty({R, m, 4}, fo.dtype(torch::kInt32));
        check(tn_trace_rays(h_, ptr<float>(o), ptr<float>(d), (uint32_t)R, (uint32_t)M, ptr<uint32_t>(num), ptr<uint32_t>(cells), ptr<float>(bary),
                            ptr<float>(dist), ptr<uint32_t>(verts), 1, stream_of(device_)));
        py::dict out;
        out["num_visited_cells"] = num;
        out["visited_cells"] = cells;
        out["barycentric_coordinates"] = bary;
        out["vertex_indices"] = verts;
        out["hit_distances"] = dist;
        return out;
    }

    py::dict trace_rays_into(const torch::Tensor &o, const torch::Tensor &d, unsigned long M, py::dict out, bool dense) {
        const int64_t R = o.numel() / 3;
        auto T = [&](const char *k) { return out[k].cast<torch::Tensor>(); };
        check(tn_trace_rays(h_, ptr<float>(o), ptr<float>(d), (uint32_t)R, (uint32_t)M, ptr<uint32_t>(T("num_visited_cells")), ptr<uint32_t>(T("visited_cells")),
                            ptr<float>(T("barycentric_coordinates")), ptr<float>(T("hit_distances")), ptr<uint32_t>(T("vertex_indices")), dense ? 1 : 0,
                            stream_of(device_)));
        return out;
    }

    py::dict trace_rays_triangles(const torch::Tensor &o, const torch::Tensor &d, unsigned long M) {  // py_binding.cpp:78-113
        if (M == 0 || (M & (M - 1)) != 0) throw std::runtime_error("max_ray_triangles must be a power of 2.");
        check_float_dim3(o, "ray_origins");
        check_float_dim3(d, "ray_directions");
        torch::NoGradGuard no_grad;
        const int64_t R = o.numel() / 3, m = (int64_t)M;
        auto fo = torch::TensorOptions().device(device_);
        auto num = torch::empty({R}, fo.dtype(torch::kInt32));
        auto faces = torch::empty({R, m}, fo.dtype(torch::kInt32));
        auto bary = torch::empty({R, m, 2}, fo.dtype(torch::kFloat32));
        auto dist = torch::empty({R, m}, fo.dtype(torch::kFloat32));
        auto verts = torch::empty({R, m, 3}, fo.dtype(torch::kInt32));
        check(tn_trace_rays_triangles(h_, ptr<float>(o), ptr<float>(d), (uint32_t)R, (uint32_t)M, ptr<uint32_t>(num), ptr<uint32_t>(faces), ptr<float>(bary),
                                      ptr<float>(dist), ptr<uint32_t>(verts), stream_of(device_)));
        py::dict out;
        out["num_visited_triangles"] = num;
        out["visited_triangles"] = faces;
        out["barycentric_coordinates"] = bary;
        out["vertex_indices"] = verts;
        out["hit_distances"] = dist;
        return out;
    }

    py::dict find_tetrahedra(const torch::Tensor &positions) {  // py_binding.cpp:115-142
        check_float_dim3(positions, "positions");
        torch::NoGradGuard no_grad;
        const int64_t N = positions.numel() / 3;
        auto shape = positions.sizes().vec();
        auto fo = torch::TensorOptions().device(device_);
        auto bary = torch::empty(shape, fo.dtype(torch::kFloat32));
        auto vshape = shape;
        vshape.back() = 4;
        auto verts = torch::empty(vshape, fo.dtype(torch::kInt32));
        shape.pop_back();
        auto tet = torch::empty(shape, fo.dtype(torch::kInt32));
        check(tn_find_tetrahedra(h_, ptr<float>(positions), (uint32_t)N, ptr<uint32_t>(tet), ptr<float>(bary), ptr<uint32_t>(verts), stream_of(device_)));
        py::dict out;
        out["tetrahedra"] = tet;
        out["barycentric_coordinates"] = bary;
        out["vertex_indices"] = verts;
        out["valid_mask"] = tet.ne(-1);
        return out;
    }

    py::dict find_visited_cells(const torch::Tensor &num, const torch::Tensor &cells, const torch::Tensor &bary, const torch::Tensor &dist,
                                const torch::Tensor &verts, const torch::Tensor &distances) {  // py_binding.cpp:163-216
        on_device(num, "num_visited_cells");
        on_device(cells, "visited_cells");
        on_device(bary, "barycentric_coordinates");
        on_device(dist, "hit_distances");
        on_device(distances, "distances");
        on_device(verts, "vertex_indices");
        require(distances.dtype() == torch::kFloat32, "distances must have float32 type");
        const int64_t R = num.size(0);
        require(distances.dim() == 2 && distances.size(0) == R, "distances must be of [num_rays, num_samples_per_ray] shape");
        require(verts.size(-1) == 4, "vertex_indices must have last dimension with size 4");
        require(vertices_.defined(), "load_tetrahedra must be called first");
        const int64_t S = distances.size(-1), M = cells.size(1);
        auto fo = torch::TensorOptions().device(device_);
        auto mask = torch::empty({R, S}, fo.dtype(torch::kBool));
        auto matched = torch::empty({R, S}, fo.dtype(torch::kInt32));
        auto bary_out = torch::empty({R, S, 3}, fo.dtype(torch::kFloat32));
        auto verts_out = torch::empty({R, S, 4}, fo.dtype(torch::kInt32));
        check(tn_find_visited_cells(h_, (uint32_t)R, (uint32_t)S, (uint32_t)M, ptr<uint32_t>(num), ptr<uint32_t>(cells), ptr<float>(bary), ptr<float>(dist),
                                    ptr<uint32_t>(verts), ptr<float>(distances), ptr<uint32_t>(matched), ptr<uint32_t>(verts_out), ptr<uint8_t>(mask),
                                    ptr<float>(bary_out), stream_of(device_)));
        py::dict out;
        out["cell_indices"] = matched;
        out["vertex_indices"] = verts_out;
        out["mask"] = mask;
        out["barycentric_coordinates"] = bary_out;
        return out;
    }

    // ---- additions over the reference surface (same as the ctypes shim) ----
    int64_t num_faces() const {
        uint32_t n = 0;
        check(tn_num_faces(h_, &n));
        return n;
    }
    py::tuple get_faces() {
        const int64_t F = num_faces();
        auto fo = torch::TensorOptions().device(device_).dtype(torch::kInt32);
        auto tri = torch::empty({F, 3}, fo), tt = torch::empty({F, 2}, fo);
        check(tn_get_faces(h_, ptr<uint32_t>(tri), ptr<uint32_t>(tt), stream_of(device_)));
        return py::make_tuple(tri, tt);
    }
    void synchronize() { check(tn_synchronize(h_, stream_of(device_))); }
    void set_walk_min_rays(uint64_t n) { check(tn_set_walk_min_rays(h_, (uint32_t)n)); }
    void set_walk_solo_range(uint64_t lo, uint64_t hi) { check(tn_set_walk_solo_range(h_, (uint32_t)lo, (uint32_t)hi)); }
    void set_walk_quad_range(uint64_t lo, uint64_t hi) { check(tn_set_walk_quad_range(h_, (uint32_t)lo, (uint32_t)hi)); }
    void set_walk_quad_spec_max_rays(uint64_t n) { check(tn_set_walk_quad_spec_max_rays(h_, (uint32_t)n)); }
    py::tuple trace_stats() {
        uint32_t o2[2] = {0, 0};
        check(tn_debug_trace_stats(h_, o2));
        return py::make_tuple(o2[0] != 0, (int64_t)o2[1]);
    }
    uint64_t launch_count() const { return tn_launch_count(h_); }

   private:
    tn_tracer *h_ = nullptr;
    torch::Device device_;
    torch::Tensor vertices_, cells_;
};

void check_interp_args(const torch::Tensor &vi, const torch::Tensor &w, const torch::Tensor &field) {
    check_input(vi, "vertex_indices");
    check_input(w, "barycentric_coordinates");
    check_input(field, "field");
    require(vi.dtype() == torch::kInt32, "vertex_indices must be a tensor of type int32");
    require(w.dtype() == torch::kFloat32, "barycentric_coordinates must be a tensor of type float32");
    require(w.size(-1) + 1 == vi.size(-1), "barycentric_coordinates must have the same last dimension as vertex_indices - 1");
    require(field.dtype() == torch::kFloat32, "field must be a tensor of type float32");
    const int64_t D = vi.size(-1);
    if (D != 2 && D != 3 && D != 4 && D != 6) throw std::runtime_error("Unsupported interpolation dimension with value " + std::to_string(D));  // :273-275
}

torch::Tensor interpolate_values(const torch::Tensor &vi, const torch::Tensor &w, const torch::Tensor &field) {  // py_binding.cpp:298-339
    check_interp_args(vi, w, field);
    const int64_t D = vi.size(-1), N = vi.numel() / D, C = field.size(0), V = field.size(-1);
    auto shape = vi.sizes().vec();
    shape.back() = C;
    auto fo = torch::TensorOptions().device(field.device()).dtype(torch::kFloat32);
    auto out = torch::empty(shape, fo);
    auto scratch = torch::empty({V, C}, fo);  // [V,C] shadow of the feature-major field
    check(tn_interpolate_values(field.device().index(), (uint32_t)D, (uint32_t)N, (uint32_t)C, (uint32_t)V, ptr<uint32_t>(vi), ptr<float>(w), ptr<float>(field),
                                ptr<float>(out), ptr<float>(scratch), stream_of(field.device())));
    return out;
}

torch::Tensor interpolate_values_backward(const torch::Tensor &vi, const torch::Tensor &w, const torch::Tensor &field, const torch::Tensor &grad_in_) {  // :341-372
    check_interp_args(vi, w, field);
    check_input(grad_in_, "grad_in");
    require(grad_in_.dtype() == torch::kFloat32, "grad_in must be a tensor of type float32");
    const int64_t D = vi.size(-1), N = vi.numel() / D, C = field.size(0), V = field.size(-1);
    require(grad_in_.size(-1) == C, "grad_in must have shape [..., field_dim]");
    auto grad_in = grad_in_.contiguous();
    auto fo = torch::TensorOptions().device(grad_in.device()).dtype(torch::kFloat32);
    auto grad_field = torch::empty({C, V}, fo);
    torch::Tensor scratch;
    if (C % 4 == 0 && N >= 1024) scratch = torch::empty({V, C}, fo);  // row-major accumulator for the vector-reduction path
    check(tn_interpolate_values_backward(grad_in.device().index(), (uint32_t)D, (uint32_t)N, (uint32_t)C, (uint32_t)V, ptr<uint32_t>(vi), ptr<float>(w),
                                         ptr<float>(grad_in), ptr<float>(grad_field), scratch.defined() ? ptr<float>(scratch) : nullptr,
                                         stream_of(grad_in.device())));
    return grad_field;
}

torch::Tensor triangulate(const torch::Tensor &points) {  // src/triangulation.cpp:34-75 (CGAL) is offline preprocessing: served by scipy's Qhull
    require(points.dim() == 2 && points.size(1) == 3, "points must have shape [num_points, 3]");
    py::object delaunay = py::module_::import("scipy.spatial").attr("Delaunay");
    py::object np_pts = py::cast(points.detach().cpu().to(torch::kFloat64)).attr("numpy")();
    py::object simplices = delaunay(np_pts).attr("simplices");
    torch::Tensor cells = py::module_::import("torch").attr("from_numpy")(simplices).cast<torch::Tensor>();
    return cells.to(torch::kInt32).to(points.device());
}
float find_average_spacing(const torch::Tensor &) {
    throw std::runtime_error("find_average_spacing (CGAL, src/triangulation.cpp:121-134) is outside this project's hot-path scope");
}
torch::Tensor gather_uint32(const torch::Tensor &, int64_t, const torch::Tensor &) {
    throw std::runtime_error("gather_uint32 (occupancy-field remnant, unused by the model) is outside this project's hot-path scope");
}
void scatter_ema_uint32(const torch::Tensor &, int64_t, const torch::Tensor &, float, const torch::Tensor &) {
    throw std::runtime_error("scatter_ema_uint32 (occupancy-field remnant, unused by the model) is outside this project's hot-path scope");
}

}  // namespace

PYBIND11_MODULE(tetranerf_cpp_extension, m) {  // py_binding.cpp:433-449
    py::class_<PyTetrahedraTracer>(m, "TetrahedraTracer")
        .def(py::init([](py::object device) { return new PyTetrahedraTracer(torch::python::detail::py_object_to_device(device)); }))
        .def_property_readonly("device", [](const PyTetrahedraTracer &t) { return py::reinterpret_steal<py::object>(THPDevice_New(t.device())); })
        .def_property_readonly("handle", &PyTetrahedraTracer::handle)
        .def("trace_rays", &PyTetrahedraTracer::trace_rays)
        .def("trace_rays_into", &PyTetrahedraTracer::trace_rays_into, py::arg("ray_origins"), py::arg("ray_directions"), py::arg("max_ray_triangles"),
             py::arg("out"), py::arg("dense") = false)
        .def("trace_rays_triangles", &PyTetrahedraTracer::trace_rays_triangles)
        .def("find_visited_cells", &PyTetrahedraTracer::find_visited_cells)
        .def("find_tetrahedra", &PyTetrahedraTracer::find_tetrahedra)
        .def("load_tetrahedra", &PyTetrahedraTracer::load_tetrahedra)
        .def("num_faces", &PyTetrahedraTracer::num_faces)
        .def("get_faces", &PyTetrahedraTracer::get_faces)
        .def("synchronize", &PyTetrahedraTracer::synchronize)
        .def("set_walk_min_rays", &PyTetrahedraTracer::set_walk_min_rays)
        .def("set_walk_solo_range", &PyTetrahedraTracer::set_walk_solo_range)
        .def("set_walk_quad_range", &PyTetrahedraTracer::set_walk_quad_range)
        .def("set_walk_quad_spec_max_rays", &PyTetrahedraTracer::set_walk_quad_spec_max_rays)
        .def("trace_stats", &PyTetrahedraTracer::trace_stats)
        .def("launch_count", &PyTetrahedraTracer::launch_count)
        .def("_check_float_dim3", &PyTetrahedraTracer::check_float_dim3);
    m.def("triangulate", &triangulate);
    m.def("find_average_spacing", &find_average_spacing);
    m.def("interpolate_values", &interpolate_values);
    m.def("interpolate_values_backward", &interpolate_values_backward);
    m.def("gather_uint32", &gather_uint32);
    m.def("scatter_ema_uint32", &scatter_ema_uint32);
    m.attr("BINDING") = "pybind11";
}
