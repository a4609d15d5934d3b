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
 * The adjacency walk is on iff the hull is a closed convex surface and no interior face is folded (the fold test of
 * tn_update_vertices); otherwise every trace takes the all-hits gather.  Either way a trace gives the bits of the all-hits gather.
 * Synchronous (the face table is sized on the host). */
int tn_load_tetrahedra(tn_tracer *h, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, void *stream);
/* Moves the loaded mesh's vertices to d_xyz f32[V,3] (same V, same cells; borrowed like load_tetrahedra's) and refits the tracer in
 * place: the positions in the leaf and walk records, the boxes of both BVHs (the load's Morton order is kept) and the coordinate bound.
 * Every trace afterwards gives the same bits as the all-hits gather of a fresh tn_load_tetrahedra at d_xyz (the reference's algorithm
 * on any triangle soup), and while the walk stays on, the same bits as its walk.  The adjacency walk is on iff the hull was a closed
 * convex surface at load and still is, and no interior face is folded: *folded_faces (may be NULL) receives the number of interior
 * faces whose two opposite vertices are not certified (float64 orient3d on the fp32 positions, with a forward error bound) to lie strictly
 * on opposite sides; *walkable (may be NULL) whether the walk is on.  Otherwise every trace takes the all-hits gather.  TN_ERR_ARG if V
 * differs from the load's or a coordinate is not finite (the tracer is then unchanged).  Like tn_load_tetrahedra, it starts a new mesh
 * generation: a pending ray / vertex gradient backward returns TN_ERR_STATE and tn_surface_copy refuses an earlier extraction.
 * Synchronous (one small read-back).  DESIGN.md §4.9. */
int tn_update_vertices(tn_tracer *h, const float *d_xyz, uint32_t V, uint32_t *folded_faces, int *walkable, void *stream);
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

/* ---- mesh refinement: one pass of longest-edge bisection (DESIGN.md §4.14).  A pure function of device arrays (no tracer): d_xyz
 * f32[V,3], d_cells u32[T,4], d_candidates u8[T] (non-zero = candidate).  Edge {a, b} has key (min << 32) | max and squared length
 * ((xa-xb)^2 + (ya-yb)^2) + (za-zb)^2 in float64 from the fp32 coordinates, every operation rounded on its own; priority is the larger
 * squared length, ties to the smaller key, and a tetrahedron's longest edge is the highest-priority one of its six.
 *   propose: each candidate whose longest edge has squared length >= (double)min_length^2 proposes it; P = the sorted distinct proposals;
 *   vote:    each tetrahedron with an edge in P votes for its highest-priority such edge;
 *   accept:  an edge of P is accepted iff every tetrahedron around it voted for it (so accepted edges share no tetrahedron, and the
 *            highest-priority proposal is always accepted); beyond max_new_vertices the highest-priority accepted edges are kept;
 *   split:   kept edges in ascending key order become vertices V, V+1, ...; each tetrahedron around kept edge (a, b) keeps its slot
 *            with b replaced by the new vertex m and appends a child at T + rank (rank = its position among the split tetrahedra, in
 *            index order) with a replaced by m: each half has half the parent's signed volume and its orientation.
 * Outputs (capacities the caller provides: d_cells_out u32[2T,4], d_parent_cell u32[2T], d_parent_edge u32[min(T, max_new_vertices),2]):
 * d_cells_out[:T + n_split], d_parent_edge[:n_new] = (a, b), a < b, of vertex V + i, d_parent_cell[:T + n_split] (identity on the first
 * T, the split parent after).  counts3 (host) = n_proposed (|P|), n_new (kept edges = new vertices), n_split.  New positions and field
 * values are not computed here: (x_a + x_b) * 0.5 per vertex tensor (tetranerf/b200/refine.py).  The output depends on the inputs only,
 * bitwise.  TN_ERR_ARG for a vertex index >= V, V + max_new_vertices > 2^32 - 1 or min_length < 0.  Workspace as
 * tn_interpolate_values_backward_deterministic: d_workspace == NULL writes the size to *workspace_bytes and does nothing else (60 bytes
 * per tetrahedron plus CUB's temporary storage: 129.7 MB at 2.02 M tetrahedra on an H100).  Synchronous (three small read-backs). */
int tn_refine_edges(int device, const float *d_xyz, uint32_t V, const uint32_t *d_cells, uint32_t T, const uint8_t *d_candidates,
                    float min_length, uint32_t max_new_vertices, uint32_t *d_cells_out, uint32_t *d_parent_edge, uint32_t *d_parent_cell,
                    uint32_t *counts3, void *d_workspace, size_t *workspace_bytes, void *stream);

/* ---- fused forward render (new; replaces model.py:531-662 between trace_rays and the pixel) -------
 * Weights are passed once (tn_render_set_weights) in nerfstudio state-dict layout and repacked on
 * the device.  See DESIGN.md §"fused render". */
typedef struct tn_render_config {
    uint32_t max_ray_triangles; /* M, power of two in [2, 2048]         model.py:77  */
    uint32_t num_samples;       /* S_c in [1, 4096]                     model.py:78  */
    uint32_t num_fine_samples;  /* S_f in [0, 4096] (0 = single pass)   model.py:79  */
    /* With S_f > 0 the per-ray fine sampler stages 16 (M + 4 S2 + 10) bytes of shared memory per block, S2 = S_c + S_f + 1, and the
     * training backward's composite stage 64 (S2 + 2): a call whose largest staging exceeds the device's opt-in shared memory per
     * block (cudaDevAttrMaxSharedMemoryPerBlockOptin; 232,448 B on an H100) returns TN_ERR_ARG before anything runs.  On an H100
     * that is S_c + S_f > 3500 at M = 512 and > 3116 at M = 2048.  Single-pass settings (S_f = 0) always fit. */
    uint32_t use_biased_sampler;/*                                      model.py:80  */
    float far_plane;            /* collider far plane: depth of empty rays (model.py:645-650) */
    float background[3];        /* renderer background colour (white = 1,1,1; model.py:93) */
} tn_render_config;

/* field: f32[64,V] feature-major.  Keeps a [V,64] shadow inside the tracer, one row per vertex with its features in the order of
 * the MLP's A fragments (csrc/tn_common.cuh, field_pos). */
int tn_render_set_field(tn_tracer *h, const float *d_field, uint32_t C, uint32_t V, void *stream);
/* operand precision of the inference MLP (tn_render; the training forward always uses 3):
 *   3 = "bf16x3": a*w = a_hi*w_hi + a_lo*w_hi + a_hi*w_lo in bf16 halves, 3 MMAs per K step, ~5e-7 absolute on unit-scale outputs;
 *   2 = "f16w2":  fp16 activations, fp16 hi/lo weights, 2 MMAs per K step, ~2.6e-5 absolute (inside the 1e-4 per-sample bar).
 * Initial value: environment variable TETRANERF_B200_MLP_PREC, else 2. */
int tn_render_set_mlp_precision(tn_tracer *h, int prec);
/* mlp_base.layers.{0,1,2}.{weight,bias}, mlp_head.layers.0.{weight,bias}, field_output_color.net.*,
 * field_output_density.net.* as 12 device pointers in that order (torch nn.Linear [out,in] layout). */
int tn_render_set_weights(tn_tracer *h, const float *const *d_params12, void *stream);
/* d_rgb f32[R,3], d_acc f32[R,1], d_depth f32[R,1], d_mask u8[R].  Two optional outputs (NULL: not computed; every element of a
 * non-NULL one is written); the other outputs are the same bits with or without them:
 *   d_expected_depth f32[R], nerfstudio DepthRenderer(method="expected"): over the samples that give rgb (the fine pass; the coarse one
 *     when num_fine_samples = 0), t_i the bin midpoints and w_i the weights of rgb, A = sum w_i: D_raw = sum w_i t_i / (A + 1e-10), and
 *     D = clip(D_raw, t_min, t_max) with t_min / t_max the smallest / largest midpoint over every active ray of the call; far_plane on
 *     empty rays.  DESIGN.md §4.10.
 *   d_normals f32[R,3]: per sample the exact gradient of the density pre-activation (reverse pass through mlp_base in the render's
 *     operand precision, then grad = cof(E) q / det(E) on the matched tetrahedron), n = -grad / |grad|, composited with the weights of
 *     rgb and normalised (nerfstudio NormalsRenderer(normalize=True)); (0,0,0) on empty rays.  DESIGN.md §4.7.
 * TN_ERR_ARG if either is given while a fused pixel gather is set (tn_render_set_gather). */
int tn_render(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
              float *d_rgb, float *d_acc, float *d_depth, uint8_t *d_mask, float *d_expected_depth, float *d_normals, void *stream);
/* ---- fused training step (SURVEY.md §8f-1): TetrahedraNerf.get_outputs in training mode (model.py:520-662) + its autograd backward.
 * Forward = the fused pipeline with the stratified bins of training (model.py:169-174 for the coarse pass, PDFSampler train_stratified
 * for the fine pass; the uniform [0,1) draws come from the caller, d_jitter_coarse f32[R,S_c+1] / d_jitter_fine f32[R,S_f+1] indexed by
 * ray, NULL = the eval-mode bins) and the training-mode RGBRenderer (no nan_to_num, no clamp).  tn_render_train_backward continues from
 * the buffers of the LAST training forward (any tn_render / training forward in between invalidates them): d_grad_rgb f32[R,3] (+ optional
 * d_grad_acc f32[R]) -> d_grad_field f32[64,V] (interpolate_values_backward, src/tetrahedra_tracer.cu:223-248) and the twelve MLP
 * gradients in the order / layouts of tn_render_set_weights; use_gradient_scaling = GradientScaler (model.py:195-205,625-630).  Every
 * output element is written.  The MLP backward runs on wgmma (recompute + dX + dW GEMMs per 64-sample tile); no [samples,128] tensor is
 * materialised in HBM. */
int tn_render_train_forward(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                            const float *d_jitter_coarse, const float *d_jitter_fine, float *d_rgb, float *d_acc, float *d_depth,
                            uint8_t *d_mask, void *stream);
int tn_render_train_backward(tn_tracer *h, const float *d_grad_rgb, const float *d_grad_acc, int use_gradient_scaling, float *d_grad_field,
                             float *const *d_grad_params12, void *stream);
/* The same training step with per-call saved state in caller-owned device memory, so that several forwards can be in flight before
 * their backwards, in any order, and a backward can run more than once.  tn_render_train_saved_bytes gives the size of one call's state
 * (R >= 1 rays, cfg as for the forward; ~115 MB at 8192 rays x 257 fine samples).  tn_render_train_forward_saved takes the arguments of
 * tn_render_train_forward plus d_saved (256-byte aligned, saved_bytes >= that size) and writes into it everything its backward reads that
 * a later call could overwrite: a header (R, M, S_c, S_f, S2, background, deterministic mode, generations of field and weights and of the mesh), the
 * slot -> ray map and active count, the fine-pass samples (matched vertices, weights, (sigma, rgb) pre-activations, bins, spacing bins),
 * the per-ray direction bias and encoding.  Its optional d_expected_depth f32[R] (NULL: none) is tn_render's, in training mode (no
 * nan_to_num, no clamp); the saved state has the same size with it (the two clip bounds sit in the slot of the active count, and the
 * header records that the forward produced them).  TN_ERR_ARG if it is given while a fused pixel gather is set.
 * tn_render_train_backward_saved computes the gradients of that forward (outputs as tn_render_train_backward, d_grad_rgb f32[R,3] of the
 * forward's R).  It reads d_saved, the field and the weights, and uses the tracer's gradient scratch, so calls on one tracer must be
 * stream-ordered.  It reads the header back to the host, so it waits until the stream has reached it.  Returns TN_ERR_STATE if
 * tn_render_set_field or tn_render_set_weights ran since the forward (or the forward ran on another tracer).  The caller frees d_saved
 * whenever it likes; the library keeps no reference to it.  Optional input and outputs (NULL: none; every element of a non-NULL output
 * is written); with all four NULL the backward runs the same kernels as tn_render_train_backward, and given or not, the ray and vertex
 * gradients leave the other outputs as they are (bitwise in the deterministic mode):
 *   d_grad_expected_depth f32[R]: dL/d expected depth, for a forward that produced it (TN_ERR_STATE otherwise).  The bins and midpoints
 *     are constants; where t_min <= D_raw <= t_max, dL/dw_i gains dL/dD (t_i - D_raw) / (A + 1e-10), before the transmittance sums and
 *     GradientScaler, so the depth loss reaches the field, the MLP, the rays and the vertices.  DESIGN.md §4.10.
 *   d_grad_origins / d_grad_directions f32[R,3]: the gradients at the forward's ray origins and directions, 0 on empty rays.  The sample
 *     distances are constants: a fine sample sits at x = o + t d, t the midpoint of its bin; dL/dx = E^-T q on its tetrahedron
 *     (q_k = dL/df . (F_vk - F_v0), solved in float64 from the fp32 mesh positions), dL/do = sum dL/dx, dL/dd = sum t dL/dx + the
 *     direction encoding's term.  dL/do is bitwise reproducible in both modes, dL/dd in the deterministic mode.  DESIGN.md §4.8.
 *   d_grad_xyz f32[V,3]: the gradient at the mesh vertex positions.  The sample distances and the matched tetrahedra are held fixed; a
 *     fine sample's weights b = E^-1 (x - x_v0) move with the vertices: dL/dx_vj += -b_j dL/dx (b_0 = 1 - b_1 - b_2 - b_3), the vertex
 *     half of the reference's add_barycentrics_grad.  Default mode: float reductions; deterministic mode: per-vertex sums in a fixed
 *     order, bitwise reproducible.  DESIGN.md §4.9.
 * With any of the last three: TN_ERR_STATE if tn_load_tetrahedra or tn_update_vertices ran since the forward (they read the mesh
 * positions), and the default mode keeps the [samples,64] feature gradient for them (0.54 GB at 8192 rays x 257 fine samples).
 * tn_render_train_backward_saved2 is tn_render_train_backward_saved with one more optional input after d_grad_expected_depth:
 *   d_grad_distortion f32[R]: dL/d distortion (tn_render_train_distortion).  The spacing bins are constants; dL/dw_j gains
 *     dL/dd (2 sum_i w_i |u_j - u_i| + 2/3 w_j delta_j), before the transmittance sums and GradientScaler, so the distortion loss
 *     reaches the field, the MLP, the rays and the vertices.  NULL runs the same kernels as tn_render_train_backward_saved, which is
 *     tn_render_train_backward_saved2 with NULL here.  DESIGN.md §4.11.
 * tn_render_train_distortion writes d_distortion f32[R], the distortion loss of mip-NeRF 360 / nerfstudio's distortion_loss per ray of a
 * saved forward: over its fine samples, with s_0 ... s_S2 the spacing bins, u_i = (s_i + s_{i+1}) / 2, delta_i = s_{i+1} - s_i and w_i the
 * weights of rgb, d = sum_i sum_j w_i w_j |u_i - u_j| + 1/3 sum_i w_i^2 delta_i, in O(S2) per ray; 0 on empty rays.  It reads d_saved
 * only, so the forward and its saved state are the same with or without it; like the backward it reads the header back (waits until
 * the stream has reached it) and returns TN_ERR_STATE if the field or the weights changed since the forward. */
int tn_render_train_saved_bytes(tn_tracer *h, const tn_render_config *cfg, uint32_t R, size_t *bytes);
int tn_render_train_forward_saved(tn_tracer *h, const tn_render_config *cfg, const float *d_origins, const float *d_directions, uint32_t R,
                                  const float *d_jitter_coarse, const float *d_jitter_fine, float *d_rgb, float *d_acc, float *d_depth,
                                  uint8_t *d_mask, float *d_expected_depth, void *d_saved, size_t saved_bytes, void *stream);
int tn_render_train_backward_saved(tn_tracer *h, const void *d_saved, const float *d_grad_rgb, const float *d_grad_acc,
                                   const float *d_grad_expected_depth, int use_gradient_scaling, float *d_grad_field,
                                   float *const *d_grad_params12, float *d_grad_origins, float *d_grad_directions, float *d_grad_xyz,
                                   void *stream);
int tn_render_train_backward_saved2(tn_tracer *h, const void *d_saved, const float *d_grad_rgb, const float *d_grad_acc,
                                    const float *d_grad_expected_depth, const float *d_grad_distortion, int use_gradient_scaling,
                                    float *d_grad_field, float *const *d_grad_params12, float *d_grad_origins, float *d_grad_directions,
                                    float *d_grad_xyz, void *stream);
int tn_render_train_distortion(tn_tracer *h, const void *d_saved, float *d_distortion, void *stream);
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
/* ---- occupancy culling of the fused paths (DESIGN.md §4.12; the reference config's use_occupancy_field) -------------------------
 * tn_occupancy_update writes d_occ f32[T] (T = the loaded mesh's tetrahedra): occ[t] <- max(decay * occ[t], m_t), m_t the largest
 * density sigma (softplus of the density head, no GradientScaler, bf16x3 as tn_surface_extract) over 11 probes of tetrahedron t: its 4
 * vertices, 6 edge midpoints and centroid, as barycentric points.  decay = 0 recomputes from scratch (the old values are not read).
 * One thread writes each entry, without atomics: bitwise reproducible.  11 probe rows per tetrahedron run through the density MLP in
 * chunks of 2^19 tetrahedra (a 176 MB workspace the tracer keeps).  TN_ERR_STATE without mesh, field or weights; TN_ERR_ARG if decay is
 * not finite and >= 0.
 * tn_render_set_occupancy borrows d_occ f32[T] (NULL: culling off, every kernel runs as without it) and a threshold (TN_ERR_ARG unless
 * finite and >= 0).  While it is set, a sample of tn_render (both precisions, expected depth and normals included) or of a training
 * forward that is matched to a tetrahedron t with occ[t] < threshold is culled: its density is the constant 0 (weight 0, no gradient),
 * its MLP is not evaluated; the PDF sampler sees the resulting coarse weights.  Unmatched samples are evaluated as without culling.  The
 * MLP passes and the training backward's MLP run over the live rows only, compacted in row order.  A saved forward records its culled
 * samples in its own state, so its backward never reads d_occ again (an update in between leaves its gradients as they were); the state
 * is no larger than without culling.  With every occ[t] >= threshold, outputs and gradients are the bits of no occupancy (the default
 * mode's float reductions aside).  tn_render and the training forwards return TN_ERR_STATE if a mesh with another number of
 * tetrahedra was loaded since.  Surface extraction and the fused pixel gather are unaffected. */
int tn_occupancy_update(tn_tracer *h, float *d_occ, float decay, void *stream);
int tn_render_set_occupancy(tn_tracer *h, const float *d_occ, float threshold);
/* ---- occupancy sampling (DESIGN.md §4.13): tn_render_set_occupancy2 is tn_render_set_occupancy (which calls it with 0) plus
 * place_samples.  With place_samples != 0, tn_render and the training forwards also place each ray's coarse bins in its kept records
 * only -- a record is skipped when its cell is a tetrahedron t with occ[t] < threshold, kept otherwise (gap records between hull faces
 * included): the biased sampler gives every kept record an equal share, the uniform one samples the kept length uniformly.  near / far,
 * the spacing bins' definition, the fine pass, the composite and every backward are unchanged; a ray with no skipped record, or no kept
 * one, gets the bins of place_samples = 0.  The saved training state has the same size and layout.  Every accepted setting runs with
 * it (the coarse sampler stages 2 (M + 2) more floats per ray).  TN_ERR_ARG if place_samples is set without d_occ. */
int tn_render_set_occupancy2(tn_tracer *h, const float *d_occ, float threshold, int place_samples);
/* ---- surface extraction: the density iso-surface sigma = level of the field as a triangle mesh, by marching tetrahedra on the loaded
 * mesh (DESIGN.md §4.6).  sigma is the density the renderer uses (density head of mlp_base, no GradientScaler), always evaluated in
 * bf16x3.  A vertex is inside when sigma(F[:, v]) >= level; every mesh edge (a, b), a < b, with one end inside and one outside gives one
 * output vertex, placed on the edge by two rounds of 64 density evaluations and a linear interpolation in the last 1/4096 bracket (the
 * crossing nearest a); a tetrahedron with 1 or 3 inside vertices gives one triangle, one with 2 gives two; normals point from inside to
 * outside.  Vertex normals: normalised sums of the unnormalised face normals; vertex colours: the colour head at the vertex's features
 * seen along -normal.  Vertices are ordered by edge (a, b), faces by tetrahedron then by the case table; the output is bitwise
 * reproducible and is not cleaned up (degenerate triangles are kept, so connectivity stays exact).
 * tn_surface_extract runs the extraction into a workspace the tracer owns and keeps (2.6 KB per crossing edge, 76 bytes per face, 16 per
 * tetrahedron, 32 per mesh vertex) and returns the
 * counts: it reads them back, so it waits until the stream has reached it.  It reads the mesh, field and weights only: a pending
 * training backward (tracer-held or saved) is unaffected.  TN_ERR_STATE without mesh, field or weights; TN_ERR_ARG if level is not
 * finite and > 0 or the field's vertex count differs from the mesh's.  An empty surface (level above or below every vertex) is not an
 * error: both counts are 0.
 * tn_surface_copy copies the last extraction out: d_vertices, d_normals, d_colors f32[N,3], d_faces u32[F,3] (indices into the
 * vertices), d_face_tet u32[F] (the tetrahedron of each face); a NULL pointer skips that output.  TN_ERR_STATE if no extraction ran, or
 * tn_render_set_field, tn_render_set_weights or tn_load_tetrahedra ran since it. */
int tn_surface_extract(tn_tracer *h, float level, uint32_t *n_vertices, uint32_t *n_faces, void *stream);
int tn_surface_copy(tn_tracer *h, float *d_vertices, float *d_normals, float *d_colors, uint32_t *d_faces, uint32_t *d_face_tet, void *stream);
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
/* the same for the last tn_render_train_backward or tn_render_train_backward_saved: ms3 = composite_bwd, mlp_bwd, finalize */
int tn_render_get_backward_timings(tn_tracer *h, float *ms3);
/* trace_rays picks between bit-identical implementations by batch size:
 * >= walk_min_rays (default 2^20): adjacency walk, 32 rays per warp (throughput);
 * solo range [lo, hi] below that (default empty): adjacency walk, one ray per warp, 4 cooperating lanes (the quad walk's kernel
 * with one quad per warp);
 * otherwise, for meshes that cannot be walked, and as the exact stage the walks fall back to: warp-per-ray all-hits BVH gather. */
int tn_set_walk_min_rays(tn_tracer *h, uint32_t n);
int tn_set_walk_solo_range(tn_tracer *h, uint32_t lo, uint32_t hi);
/* [lo, hi] below walk_min_rays (checked before the solo range): adjacency walk with 8 rays per warp, 4 cooperating lanes per ray */
int tn_set_walk_quad_range(tn_tracer *h, uint32_t lo, uint32_t hi);
/* the quad and solo walks of batches of up to n rays (default 65536) load the records of all candidate next tetrahedra while the
 * current one is intersected instead of prefetching them (latency-bound regime); 0 = never.  Results are identical. */
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
/* device pointer of the per-sample density gradient of the last tn_render call with d_normals: float4 (x, y, z, 0) per sample, in the
 * slot order of the pass that gives the colours (vi_f / bary_f; vi_c / bary_c when num_fine_samples = 0) */
int tn_render_debug_normals_grad(tn_tracer *h, void **ptr);
/* device pointer of dL/dx per fine sample of the last tn_render_train_backward_saved call with ray or vertex gradients: float4
 * (x, y, z, 0) per sample, in the slot order of its forward (0 for unmatched samples and flat tetrahedra) */
int tn_render_debug_ray_grads(tn_tracer *h, void **ptr);
/* one 128x128 tile out = A[128,K] * W[128,K]^T through the wgmma bf16x3 path (A from registers); K in {64,128}; synchronous */
int tn_debug_gemm_bf16x3(int device, const float *d_A, const float *d_W, uint32_t K, float *d_out, void *stream);
/* probe of the shared-memory operand forms of the fused MLP backward: P, Q f32[128,128] staged as bf16 hi/lo blocks
 * ([rows][64 columns], 128-byte swizzle); mode 0: out = P Q^T (both K-major), 1: out = P Q (B MN-major), 2: out = P^T Q (both
 * MN-major); N in {64,128}; lbo / sbo / kstep (bytes) describe the MN-major descriptors; synchronous */
int tn_debug_gemm_modes(int device, int mode, uint32_t N, uint32_t lbo, uint32_t sbo, uint32_t kstep, const float *d_P,
                        const float *d_Q, float *d_out, void *stream);
/* rays of the last tn_debug_trace_stats call that needed the all-hits gather (subset of out2[1]) */
uint32_t tn_debug_last_exact_count(void);
/* bytes of device memory the library's own buffers hold in this process, over every tracer (peer buffers excluded) */
uint64_t tn_debug_device_bytes(void);

/* number of kernels launched by this library on this tracer since creation (bench "gpu_launches") */
uint64_t tn_launch_count(tn_tracer *h);

#ifdef __cplusplus
}
#endif
#endif
