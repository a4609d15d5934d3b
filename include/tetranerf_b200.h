/* tetranerf_b200.h -- C ABI of the H100-native Tetra-NeRF ray-sampling hot path.
 *
 * Drop-in boundary: these entry points are what the reference's pybind module
 * `tetranerf_cpp_extension` (src/py_binding.cpp:433-449) binds for this path.  Plain pointers and
 * sizes only; every pointer named d_* is a DEVICE pointer on the tracer's device; `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  All calls are stream-ordered and
 * asynchronous unless noted (the reference does cudaDeviceSynchronize per call,
 * src/tetrahedra_tracer.cpp:173-174; a caller who wants that behaviour calls tn_synchronize).
 *
 * Return value: 0 on success, non-zero on error; tn_last_error() gives the message of the last
 * failing call on the calling thread (the reference throws `Exception`, src/utils/exception.h:164-181,
 * surfacing as Python RuntimeError -- the Python shim turns non-zero into RuntimeError).
 *
 * "E" below is 0xFFFFFFFF ("empty", -1 in the int32 tensors of the reference).
 */
#ifndef TETRANERF_B200_H
#define TETRANERF_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct tn_tracer tn_tracer;

enum { TN_OK = 0, TN_ERR_ARG = 1, TN_ERR_CUDA = 2, TN_ERR_MESH = 3, TN_ERR_STATE = 4, TN_ERR_OVERFLOW = 5 };

const char *tn_last_error(void);
int tn_version(void);

/* TetrahedraTracer(device)  -- src/py_binding.cpp:30-35, src/tetrahedra_tracer.cpp:90-127 */
int tn_create(int device, tn_tracer **out);
/* ~TetrahedraTracer         -- src/tetrahedra_tracer.cpp:178-189 */
int tn_destroy(tn_tracer *h);
/* stream sync + deferred device-side error flags (traversal stack overflow) */
int tn_synchronize(tn_tracer *h, void *stream);

/* load_tetrahedra(xyz f32[V,3], cells i32[T,4]) -- src/py_binding.cpp:144-161,
 * src/tetrahedra_tracer.cpp:244-340 (unique-face build :45-71 + acceleration structure).
 * Borrows d_xyz / d_cells (caller keeps them alive, as the reference, tetrahedra_tracer.h:300-303).
 * Returns TN_ERR_MESH "A triangle is shared by more than two tetrahedra!" like :64-66.
 * Synchronous (the face table is sized on the host). */
int tn_load_tetrahedra(tn_tracer *h, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, void *stream);
int tn_num_faces(tn_tracer *h, uint32_t *F);
/* copies out the unique-face tables in reference numbering: d_tri u32[F,3], d_tt u32[F,2]
 * (triangle_indices / triangle_tetrahedra of src/optix_types.h:4-5) */
int tn_get_faces(tn_tracer *h, uint32_t *d_tri, uint32_t *d_tt, void *stream);

/* trace_rays(origins, directions, max_ray_triangles) -- src/py_binding.cpp:41-76,
 * src/tetrahedra_tracer.cpp:137-176, src/optix/optix_trace_rays.cu:268-331.
 *   d_num   u32[R]        num_visited_cells
 *   d_cells u32[R,M]      visited_cells            (tail = E)
 *   d_bary  f32[R,M,2,3]  barycentric_coordinates  (tail = 0)
 *   d_dist  f32[R,M,2]    hit_distances            (tail = 0)
 *   d_verts u32[R,M,4]    vertex_indices           (tail = E)
 * M must be a power of two (py_binding.cpp:44-47).  The kernel writes every element (no pre-zeroing
 * needed).  dense=0 skips the tail fill (entries >= num are left untouched). */
int tn_trace_rays(tn_tracer *h, const float *d_origins, const float *d_directions, uint32_t R, uint32_t M, uint32_t *d_num,
                  uint32_t *d_cells, float *d_bary, float *d_dist, uint32_t *d_verts, int dense, void *stream);

/* trace_rays_triangles -- src/py_binding.cpp:78-113, src/optix/optix_trace_rays_triangles.cu:49-114.
 *   d_num u32[R], d_faces u32[R,M], d_bary f32[R,M,2], d_dist f32[R,M], d_verts u32[R,M,3]; tails 0 */
int tn_trace_rays_triangles(tn_tracer *h, const float *d_origins, const float *d_directions, uint32_t R, uint32_t M,
                            uint32_t *d_num, uint32_t *d_faces, float *d_bary, float *d_dist, uint32_t *d_verts, void *stream);

/* find_tetrahedra(positions) -- src/py_binding.cpp:115-142, src/optix/optix_find_tetrahedra.cu:84-213.
 *   d_tet u32[N] (E if none), d_bary f32[N,3], d_verts u32[N,4] (0 when not found) */
int tn_find_tetrahedra(tn_tracer *h, const float *d_positions, uint32_t N, uint32_t *d_tet, float *d_bary, uint32_t *d_verts,
                       void *stream);

/* find_visited_cells -- src/py_binding.cpp:163-216, src/tetrahedra_tracer.cu:115-161.
 * Writes every output element (defaults: cell E, verts E, mask 0, bary 0; py_binding.cpp:188-191). */
int tn_find_visited_cells(tn_tracer *h, uint32_t R, uint32_t S, uint32_t M, const uint32_t *d_num, const uint32_t *d_cells,
                          const float *d_bary, const float *d_dist, const uint32_t *d_verts, const float *d_sample_dist,
                          uint32_t *d_cell_out, uint32_t *d_verts_out, uint8_t *d_mask_out, float *d_bary_out, void *stream);

/* interpolate_values<D> -- src/py_binding.cpp:298-339, src/tetrahedra_tracer.cu:195-221, in two steps.
 * tn_make_field_shadow: d_field f32[C,V] (feature-major, the checkpoint layout, model.py:247-255) -> d_shadow f32[V,C]
 * (row-major: one vertex = one contiguous row); built once per field, a training step interpolates the same field twice.
 * tn_interpolate_values_shadow: d_vi u32[N,D], d_w f32[N,D-1], d_shadow f32[V,C] -> d_out f32[N,C] (contiguous; the
 * reference returns the same values as a moveaxis view).  D in {2,3,4,6}. */
int tn_make_field_shadow(int device, uint32_t C, uint32_t V, const float *d_field, float *d_shadow, void *stream);
int tn_interpolate_values_shadow(int device, uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *d_vi, const float *d_w,
                                 const float *d_shadow, float *d_out, void *stream);
/* interpolate_values_backward<D> -- src/py_binding.cpp:341-372, src/tetrahedra_tracer.cu:223-248.
 *   d_grad_in f32[N,C], d_grad_field f32[C,V] (every element written by this call, py_binding.cpp:360).
 *   d_scratch: NULL (scalar atomics straight into the feature-major gradient, as the reference), or >= C*V floats for
 *   a row-major [V,C] accumulator filled with 16-byte vector reductions and transposed at the end (needs C % 4 == 0). */
int tn_interpolate_values_backward(int device, uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *d_vi,
                                   const float *d_w, const float *d_grad_in, float *d_grad_field, float *d_scratch, void *stream);
/* The same gradient, bitwise reproducible: identical inputs give identical bits on every run (same build, same GPU model), whatever
 * the scheduling.  The vertex slots are sorted by vertex (stable radix sort) and each vertex sums its contributions in input order;
 * the products are the ones above, only the summation order differs (so results differ from tn_interpolate_values_backward by
 * rounding).  Any C; N * D < 2^31.  d_workspace == NULL: *workspace_bytes receives the size the call needs and nothing else happens;
 * otherwise d_workspace holds *workspace_bytes (>= that size) bytes of device memory used only during the call (stream-ordered). */
int tn_interpolate_values_backward_deterministic(int device, uint32_t D, uint32_t N, uint32_t C, uint32_t V, const uint32_t *d_vi,
                                                 const float *d_w, const float *d_grad_in, float *d_grad_field, void *d_workspace,
                                                 size_t *workspace_bytes, void *stream);

/* ---- fused forward render (new; replaces model.py:531-662 between trace_rays and the pixel) -------
 * Weights are passed once (tn_render_set_weights) in nerfstudio state-dict layout and repacked on
 * the device.  See DESIGN.md §"fused render". */
typedef struct tn_render_config {
    uint32_t max_ray_triangles; /* M, power of two                      model.py:77  */
    uint32_t num_samples;       /* S_c                                  model.py:78  */
    uint32_t num_fine_samples;  /* S_f (0 = single pass)                model.py:79  */
    uint32_t use_biased_sampler;/*                                      model.py:80  */
    float far_plane;            /* collider far plane: depth of empty rays (model.py:645-650) */
    float background[3];        /* renderer background colour (white = 1,1,1; model.py:93) */
} tn_render_config;

/* field: f32[64,V] feature-major.  Keeps a [V,64] row-major shadow inside the tracer. */
int tn_render_set_field(tn_tracer *h, const float *d_field, uint32_t C, uint32_t V, void *stream);
/* operand precision of the inference MLP (tn_render; the training forward always uses 3):
 *   3 = "bf16x3": a*w = a_hi*w_hi + a_lo*w_hi + a_hi*w_lo in bf16 halves, 3 MMAs per K step, ~5e-7 absolute on unit-scale outputs;
 *   2 = "f16w2":  fp16 activations, fp16 hi/lo weights, 2 MMAs per K step, ~2.6e-5 absolute (inside the 1e-4 per-sample bar).
 * Initial value: environment variable TETRANERF_B200_MLP_PREC, else 2. */
int tn_render_set_mlp_precision(tn_tracer *h, int prec);
/* mlp_base.layers.{0,1,2}.{weight,bias}, mlp_head.layers.0.{weight,bias}, field_output_color.net.*,
 * field_output_density.net.* as 12 device pointers in that order (torch nn.Linear [out,in] layout). */
int tn_render_set_weights(tn_tracer *h, const float *const *d_params12, void *stream);
/* d_rgb f32[R,3], d_acc f32[R,1], d_depth f32[R,1], d_mask u8[R] */
int tn_render(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
              float *d_rgb, float *d_acc, float *d_depth, uint8_t *d_mask, void *stream);
/* ---- fused training step (SURVEY.md §8f-1): TetrahedraNerf.get_outputs in training mode (model.py:520-662) + its autograd backward.
 * Forward = the fused pipeline with the stratified bins of training (model.py:169-174 for the coarse pass, PDFSampler train_stratified
 * for the fine pass; the uniform [0,1) draws come from the caller, d_jitter_coarse f32[R,S_c+1] / d_jitter_fine f32[R,S_f+1] indexed by
 * ray, NULL = the eval-mode bins) and the training-mode RGBRenderer (no nan_to_num, no clamp).  Backward continues from the buffers of
 * the LAST training forward: d_grad_rgb f32[R,3] (+ optional d_grad_acc f32[R]) -> d_grad_field f32[64,V] (interpolate_values_backward,
 * src/tetrahedra_tracer.cu:223-248) and the twelve MLP gradients in the order / layouts of tn_render_set_weights; use_gradient_scaling =
 * GradientScaler (model.py:195-205,625-630).  Every output element is written.  The MLP backward runs on wgmma (recompute + dX + dW
 * GEMMs per 64-sample tile); no [samples,128] tensor is materialised in HBM. */
int tn_render_train_forward(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                            const float *d_jitter_coarse, const float *d_jitter_fine, float *d_rgb, float *d_acc, float *d_depth,
                            uint8_t *d_mask, void *stream);
int tn_render_train_backward(tn_tracer *h, const float *d_grad_rgb, const float *d_grad_acc, int use_gradient_scaling, float *d_grad_field,
                             float *const *d_grad_params12, void *stream);
/* Deterministic mode of the fused training step (enable != 0; initial value: 1 if the environment variable TETRANERF_B200_DETERMINISTIC
 * is 1, else 0).  Read by tn_render_train_forward; tn_render_train_backward continues in the mode of the forward it belongs to.  With
 * identical inputs, on the same build and GPU model, forward outputs and every gradient are then bitwise identical from run to run and
 * process to process, whatever the backward grid size and whatever order warps claim work in: slots go to rays in ray order (an
 * exclusive scan instead of an atomic counter), the backward assigns its 64-sample tiles to 256 fixed partitions with private
 * accumulators, and every sum (weight gradients, column sums, per-ray bias gradients, the per-vertex field gradient after a stable sort
 * by vertex) is reduced in a fixed order.  Forward outputs (rgb, accumulation, depth, ray_mask) equal those of the default mode bit for
 * bit; gradients differ from it by rounding (another summation order).  Costs extra device memory: ~0.9 GB at 8192 rays x 257 fine
 * samples (the [samples,64] feature gradient, the sort, partition partials).  The eval render (tn_render) is unaffected. */
int tn_render_set_deterministic(tn_tracer *h, int enable);
/* ---- multi-GPU: final gather of the rendered pixels (north_star; tetranerf/nerfstudio/pipeline.py:53-58 is the reference's only
 * multi-GPU mechanism).  One process per GPU; each rank owns a gathered-pixel buffer f32[world * rays_per_rank, 6]
 * (r, g, b, accumulation, depth, mask) allocated with tn_peer_alloc, whose 64-byte CUDA IPC handle the ranks exchange and map
 * with tn_peer_open.  After tn_render_set_gather the kernels of tn_render store every pixel straight into ALL ranks' buffers
 * (peer stores over NVLink, row = rank * rays_per_rank + ray): the all-gather is fused into the render, no collective call. */
int tn_peer_alloc(int device, uint64_t bytes, void **d_ptr, unsigned char *handle64);
int tn_peer_open(int device, const unsigned char *handle64, void **d_ptr);
int tn_peer_close(int device, void *d_ptr);
int tn_peer_free(int device, void *d_ptr);
int tn_render_set_gather(tn_tracer *h, uint32_t world, uint32_t rank, void *const *d_peer_buffers, uint32_t rays_per_rank);
/* per-kernel CUDA-event timing of the last tn_render call: ms6 = trace, sample_coarse, mlp_coarse, sample_fine,
 * mlp_fine, composite (used by bench.py for the roofline of the dominant kernel) */
int tn_render_set_profiling(tn_tracer *h, int enable);
int tn_render_get_timings(tn_tracer *h, float *ms6);
/* the same for the last tn_render_train_backward: ms3 = composite_bwd, mlp_bwd, finalize */
int tn_render_get_backward_timings(tn_tracer *h, float *ms3);
/* trace_rays picks between bit-identical implementations by batch size:
 * >= walk_min_rays (default 2^20): adjacency walk, 32 rays per warp (throughput);
 * solo range [lo, hi] below that (default empty): adjacency walk, one ray per warp with cooperating lanes;
 * otherwise, for meshes that cannot be walked, and as the exact stage the walks fall back to: warp-per-ray all-hits BVH gather. */
int tn_set_walk_min_rays(tn_tracer *h, uint32_t n);
int tn_set_walk_solo_range(tn_tracer *h, uint32_t lo, uint32_t hi);
/* [lo, hi] below walk_min_rays (checked before the solo range): adjacency walk with 8 rays per warp, 4 cooperating lanes per ray */
int tn_set_walk_quad_range(tn_tracer *h, uint32_t lo, uint32_t hi);
/* the quad walk of batches of up to n rays (default 65536) loads the records of all candidate next tetrahedra while the current one
 * is intersected instead of prefetching them (latency-bound regime); 0 = never.  Results are identical. */
int tn_set_walk_quad_spec_max_rays(tn_tracer *h, uint32_t n);
/* test hook: number of CTAs of the backward MLP kernel of tn_render_train_backward (0 = default, one per SM) */
int tn_render_set_backward_grid(tn_tracer *h, uint32_t ctas);
/* out2[0] = 1 if the loaded mesh takes the adjacency-walk fast path (conforming, convex hull); out2[1] = rays of the last
 * trace_rays call that needed the exact sort/pairing or all-hits stage.  Synchronises. */
int tn_debug_trace_stats(tn_tracer *h, uint32_t *out2);
/* ---- test hooks (not part of the reference surface) ------------------------------------------------
 * device pointers of the intermediate buffers of the last tn_render call, in the order
 * num, dist, n_active, ray_list, ebins_c, sbins_c, vi_c, bary_c, dens_c, ebins_f, vi_f, bary_f, out_f,
 * dirbias, field shadow, weight image */
int tn_render_debug_buffers(tn_tracer *h, void **ptrs16);
/* one 128x128 tile out = A[128,K] * W[128,K]^T through the wgmma bf16x3 path (A from registers); K in {64,128}; synchronous */
int tn_debug_gemm_bf16x3(int device, const float *d_A, const float *d_W, uint32_t K, float *d_out, void *stream);
/* probe of the shared-memory operand forms of the fused MLP backward: P, Q f32[128,128] staged as bf16 hi/lo blocks
 * ([rows][64 columns], 128-byte swizzle); mode 0: out = P Q^T (both K-major), 1: out = P Q (B MN-major), 2: out = P^T Q (both
 * MN-major); N in {64,128}; lbo / sbo / kstep (bytes) describe the MN-major descriptors; synchronous */
int tn_debug_gemm_modes(int device, int mode, uint32_t N, uint32_t lbo, uint32_t sbo, uint32_t kstep, const float *d_P,
                        const float *d_Q, float *d_out, void *stream);
/* rays of the last tn_debug_trace_stats call that needed the all-hits gather (subset of out2[1]) */
uint32_t tn_debug_last_exact_count(void);

/* number of kernels launched by this library on this tracer since creation (bench "gpu_launches") */
uint64_t tn_launch_count(tn_tracer *h);

#ifdef __cplusplus
}
#endif
#endif
