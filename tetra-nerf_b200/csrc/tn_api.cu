// tn_api.cu -- C-ABI entry points: tracer lifetime, errors, mesh load, face export, sync.
#include <cstring>
#include <memory>

#include "tn_common.cuh"

namespace tn {
static thread_local std::string g_last_error;
void set_error(const std::string &msg) { g_last_error = msg; }
int fail(int code, const std::string &msg) {
    g_last_error = msg;
    return code;
}

__global__ void k_export_faces(const uint4 *__restrict__ tri4, const uint2 *__restrict__ tt, uint32_t F, uint32_t *__restrict__ tri_out,
                               uint32_t *__restrict__ tt_out) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const uint4 t = tri4[f];
    tri_out[3 * (size_t)f] = t.x; tri_out[3 * (size_t)f + 1] = t.y; tri_out[3 * (size_t)f + 2] = t.z;
    const uint2 o = tt[f];
    tt_out[2 * (size_t)f] = o.x; tt_out[2 * (size_t)f + 1] = o.y;
}
}  // namespace tn

extern "C" {

const char *tn_last_error(void) { return tn::g_last_error.c_str(); }
int tn_version(void) { return 100; }

int tn_create(int device, tn_tracer **out) {
    if (!out) return tn::fail(TN_ERR_ARG, "tn_create: null output pointer");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
        return tn::fail(TN_ERR_CUDA, "The device argument must be a CUDA device (no CUDA device is available).");  // py_binding.cpp:31-33
    if (device < 0 || device >= ndev) return tn::fail(TN_ERR_ARG, "tn_create: invalid CUDA device index " + std::to_string(device));
    tn::DeviceGuard g(device);
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device);
    if (major != 9 || minor != 0)
        return tn::fail(TN_ERR_CUDA, "tetranerf_b200 is built for sm_90a (H100) only; device has compute capability " + std::to_string(major) + "." +
                                         std::to_string(minor));
    std::unique_ptr<tn_tracer> h(new tn_tracer());
    h->device = device;
    TN_TRY(h->d_flags.grow(4));
    TN_CUDA(cudaMemset(h->d_flags.p, 0, sizeof(int) * 4));
    *out = h.release();
    return TN_OK;
}

int tn_destroy(tn_tracer *h) {
    if (!h) return TN_OK;
    tn::DeviceGuard g(h->device);
    cudaDeviceSynchronize();
    tn::free_render(h);
    tn::free_surface(h);
    delete h;
    return TN_OK;
}

int tn_synchronize(tn_tracer *h, void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    tn::DeviceGuard g(h->device);
    TN_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    int flags[4] = {0, 0, 0, 0};
    TN_CUDA(cudaMemcpy(flags, h->d_flags.p, sizeof(flags), cudaMemcpyDeviceToHost));
    if (flags[0] != 0) {
        cudaMemset(h->d_flags.p, 0, sizeof(flags));
        return tn::fail(TN_ERR_OVERFLOW, "trace_rays: BVH work list overflow on " + std::to_string(flags[0]) + " ray(s); their results were dropped");
    }
    return TN_OK;
}

int tn_load_tetrahedra(tn_tracer *h, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (!d_xyz || !d_cells) return tn::fail(TN_ERR_ARG, "load_tetrahedra: null pointer");
    tn::DeviceGuard g(h->device);
    h->mesh_gen = tn::next_generation();  // any earlier surface extraction is stale from here on, even if the build fails
    h->adj_valid = false;                 // the vertex adjacency of the old cells, likewise
    return tn::build_mesh(h, d_xyz, V, d_cells, T, (cudaStream_t)stream);
}

int tn_update_vertices(tn_tracer *h, const float *d_xyz, uint32_t V, uint32_t *folded_faces, int *walkable, void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (!d_xyz) return tn::fail(TN_ERR_ARG, "update_vertices: null pointer");
    tn::DeviceGuard g(h->device);
    return tn::refit_mesh(h, d_xyz, V, (cudaStream_t)stream, folded_faces, walkable);
}

int tn_num_faces(tn_tracer *h, uint32_t *F) {
    if (!h || !F) return tn::fail(TN_ERR_ARG, "null argument");
    if (!h->mesh.nodes.p) return tn::fail(TN_ERR_STATE, "no tetrahedra loaded");
    *F = h->mesh.F;
    return TN_OK;
}

int tn_get_faces(tn_tracer *h, uint32_t *d_tri, uint32_t *d_tt, void *stream) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    if (!h->mesh.nodes.p) return tn::fail(TN_ERR_STATE, "no tetrahedra loaded");
    tn::DeviceGuard g(h->device);
    const uint32_t F = h->mesh.F;
    tn::k_export_faces<<<(F + 255) / 256, 256, 0, (cudaStream_t)stream>>>(h->mesh.tri.p, h->mesh.tt.p, F, d_tri, d_tt);
    h->launches += 1;
    TN_CUDA(cudaGetLastError());
    return TN_OK;
}

uint64_t tn_launch_count(tn_tracer *h) { return h ? h->launches : 0; }

// test hook: bytes held by the library's own device buffers (every DevArray of the process; peer buffers excluded)
uint64_t tn_debug_device_bytes(void) { return tn::g_device_bytes.load(); }

// ---- peer-mapped buffers (one process per GPU): cudaMalloc + CUDA IPC, so that a kernel of rank a can store into rank b's
// memory over NVLink (fused pixel gather, tn_render_set_gather) ----
int tn_peer_alloc(int device, uint64_t bytes, void **d_ptr, unsigned char *handle64) {
    if (!d_ptr || !handle64 || bytes == 0) return tn::fail(TN_ERR_ARG, "tn_peer_alloc: null argument");
    tn::DeviceGuard g(device);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    TN_CUDA(cudaMalloc(d_ptr, bytes));
    TN_CUDA(cudaMemset(*d_ptr, 0, bytes));
    cudaIpcMemHandle_t hd;
    TN_CUDA(cudaIpcGetMemHandle(&hd, *d_ptr));
    memcpy(handle64, &hd, 64);
    return TN_OK;
}
int tn_peer_open(int device, const unsigned char *handle64, void **d_ptr) {
    if (!d_ptr || !handle64) return tn::fail(TN_ERR_ARG, "tn_peer_open: null argument");
    tn::DeviceGuard g(device);
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle64, 64);
    TN_CUDA(cudaIpcOpenMemHandle(d_ptr, hd, cudaIpcMemLazyEnablePeerAccess));
    return TN_OK;
}
int tn_peer_close(int device, void *d_ptr) {
    tn::DeviceGuard g(device);
    if (d_ptr) TN_CUDA(cudaIpcCloseMemHandle(d_ptr));
    return TN_OK;
}
int tn_peer_free(int device, void *d_ptr) {
    tn::DeviceGuard g(device);
    if (d_ptr) TN_CUDA(cudaFree(d_ptr));
    return TN_OK;
}

// batches with at least `n` rays take the adjacency-walk fast path of trace_rays (0 = always, UINT32_MAX = never);
// (the default, 2^20, leaves batches of realistic size to the quad walk)
extern "C" int tn_set_walk_min_rays(tn_tracer *h, uint32_t n) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    h->walk_min_rays = n;
    return TN_OK;
}
// batches below walk_min_rays with lo <= rays <= hi take the one-ray-per-warp form of the walk (lo > hi = never)
extern "C" int tn_set_walk_solo_range(tn_tracer *h, uint32_t lo, uint32_t hi) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    h->walk_solo_min_rays = lo;
    h->walk_solo_max_rays = hi;
    return TN_OK;
}
// batches below walk_min_rays with lo <= rays <= hi take the 8-rays-per-warp form of the walk (lo > hi = never); checked before the solo range
extern "C" int tn_set_walk_quad_range(tn_tracer *h, uint32_t lo, uint32_t hi) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    h->walk_quad_min_rays = lo;
    h->walk_quad_max_rays = hi;
    return TN_OK;
}
// quad and solo walks: batches of up to n rays load the records of all candidate next tetrahedra while the current one is intersected (0 = never)
extern "C" int tn_set_walk_quad_spec_max_rays(tn_tracer *h, uint32_t n) {
    if (!h) return tn::fail(TN_ERR_ARG, "null tracer");
    h->walk_quad_spec_max_rays = n;
    return TN_OK;
}
static uint32_t g_last_exact = 0;
extern "C" uint32_t tn_debug_last_exact_count(void) { return g_last_exact; }
// test hook: (walkable mesh?, number of rays the last trace_rays call handed to the exact stage); synchronises the device
int tn_debug_trace_stats(tn_tracer *h, uint32_t *out2) {
    if (!h || !out2) return tn::fail(TN_ERR_ARG, "null argument");
    tn::DeviceGuard g(h->device);
    TN_CUDA(cudaDeviceSynchronize());
    int flags[4];
    TN_CUDA(cudaMemcpy(flags, h->d_flags.p, sizeof(flags), cudaMemcpyDeviceToHost));
    out2[0] = h->mesh.walkable ? 1u : 0u;
    out2[1] = (uint32_t)flags[2];
    g_last_exact = (uint32_t)flags[3];
    return TN_OK;
}

}  // extern "C"
