/*
 * multiply_b200 — C ABI of the H100-native (sm_90a) MultiPly volume-rendering hot path.
 *
 * The reference (eth-ait/MultiPly) has no FFI / plugin registry: its boundary for this path
 * is the Python operator surface of code/lib/model (SURVEY.md §8b).  Each entry point below
 * names the reference function it replaces (file:line relative to /root/reference/code).
 * INTEGRATION.md shows the ctypes stub a maintainer adds on the reference side.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types.
 *   - every `const float*` / `float*` / `int*` is a CUDA DEVICE pointer owned by the caller
 *     unless the parameter name ends in `_host`.
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it and never call
 *     cudaDeviceSynchronize.
 *   - return 0 on success, negative on error; mp_last_error() gives the (thread-local) text.
 *   - fp32 row-major contiguous tensors; B = 1 (the reference indexes [0] everywhere,
 *     multiply.py:208, deformer.py:22-24).
 *   - scratch memory comes from caller-provided workspaces sized by the *_workspace_bytes calls, and persistent
 *     handles live in caller storage sized by the *_bytes calls (mp_mesh_plan's storage_bytes).  Exactly the query's
 *     bytes suffice and a call writes none beyond them; where a query answers 0 the call also takes a NULL buffer.  Every workspace, storage and scratch base
 *     (mp_mesh_plan's MP_MESH_PLAN_SCRATCH_BYTES included) must be 256-byte aligned, as every cudaMalloc and torch
 *     allocation is.  A call refuses a smaller or misaligned buffer before it enqueues anything.
 */
#ifndef MULTIPLY_B200_H
#define MULTIPLY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MP_MAX_LAYERS 12
#define MP_MAX_PERSONS 8
#define MP_NUM_JOINTS 24

/* ------------------------------------------------------------------------------------------
 * misc
 * ---------------------------------------------------------------------------------------- */
int mp_version(void);
const char* mp_last_error(void);
/* number of SMs of the current device (grid sizing) */
int mp_device_sm_count(void);
/* host helper: torch.linspace(start, end, n) in fp32, bit-exact with the ATen CPU kernel
 * (fma(step, i, start) for i < n/2, fma(-step, n-1-i, end) otherwise).  ray_sampler.py:29,167,204,215 */
int mp_linspace_host(float start, float end, int n, float* out_host);
/* total number of this library's kernels launched since the last reset (bench.py "gpu_launches") */
long long mp_launch_count(int reset);

/* ------------------------------------------------------------------------------------------
 * networks: ImplicitNet / RenderingNet  (lib/model/networks.py:7-208, 223-312)
 * ---------------------------------------------------------------------------------------- */
typedef struct mp_net mp_net_t;

/* Raw parameters of a stack of nn.Linear layers exactly as they sit in the state dict
 * (`lin{l}.weight_v`, `lin{l}.weight_g`, `lin{l}.bias`; `lin{l}.weight` when weight_g == NULL). */
typedef struct {
  int n_layers;
  const float* weight_v[MP_MAX_LAYERS]; /* [out,in] */
  const float* weight_g[MP_MAX_LAYERS]; /* [out,1] or NULL (no weight norm) */
  const float* bias[MP_MAX_LAYERS];     /* [out] */
  int in_dim[MP_MAX_LAYERS];
  int out_dim[MP_MAX_LAYERS];
} mp_linear_stack_t;

/* ImplicitNet description (networks.py:7-116). */
typedef struct {
  mp_linear_stack_t lin;   /* 9 layers for the shipped configs */
  int d_in;                /* 3 (fg) or 4 (bg) */
  int multires;            /* 6 (fg) or 10 (bg) ; embedding dim = d_in*(1+2*multires) */
  int cond_dim;            /* 69 ('smpl') or 32 ('frame'); cond is concatenated at layer 0 */
  int skip_layer;          /* 4 */
} mp_implicit_desc_t;

/* RenderingNet description (networks.py:223-262). mode 0 = 'pose_no_view', 1 = 'nerf_frame_encoding'. */
typedef struct {
  mp_linear_stack_t lin;   /* lin0..lin{n-1} */
  int mode;
  int multires_view;       /* -1 or 4 */
  const float* lin_pose_weight; /* [8,69] (mode 0) or NULL */
  const float* lin_pose_bias;   /* [8] */
} mp_render_desc_t;

/* A foreground field = ImplicitNet + RenderingNet of one person; background field = bg pair.
 * Packing folds weight-norm (networks.py:82-83), the 1/sqrt(2) of the skip layer (:166-167) and
 * lays the weights out for the kernels (fp32 transposed for the SIMT engine, fp16 hi/lo
 * swizzled K-major tiles for the tensor-core engine).  The handle is immutable afterwards.
 * mp_field_pack_bytes is the storage of exactly these two networks; it reads only the descriptors' dimensions and
 * whether lin_pose is given (no weight is dereferenced), and answers 0 for a pair mp_field_pack would refuse.  The
 * pack refuses a pair, or a short or misaligned storage, before it enqueues anything. */
size_t mp_field_pack_bytes(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, int is_background);
int mp_field_pack(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, int is_background,
                  void* storage, size_t storage_bytes, mp_net_t** out, void* stream);
void mp_field_free(mp_net_t* f);
/* Per-call conditioning: folds cond (pose[3:]/pi, multiply.py:270, or the frame code, :407-410) into
 * the layer-0 bias and lin_pose(body_pose) (networks.py:277-281) / frame code into the colour layer-0 bias. */
int mp_field_set_cond(mp_net_t* f, const float* cond /*[cond_dim]*/, void* stream);

/* engine selection: 0 = fp32 SIMT (validation engine), 1 = wgmma split-fp16 tensor-core engine */
int mp_set_engine(int engine);
int mp_get_engine(void);
/* Precision mode of the tensor-core engine: which split-precision product terms each MLP layer issues (fp16 hi/lo operand
 * pairs, fp32 accumulation).  0 = parity (default): A_hi.W_hi + A_lo.W_hi + A_hi.W_lo everywhere (RGB / SDF within 1e-4 of
 * the fp32 reference); 1 = the colour layers issue A_hi.W_hi only (SDF / normals unchanged, RGB ~2e-5); 2 = throughput:
 * every layer single-term, i.e. plain fp16 operands — outside the 1e-4 gate, reported separately. */
int mp_set_precision(int mode);
int mp_get_precision(void);
/* mp_render_rays schedule: 1 (default) = persons and background on their own streams, joined before the compositor;
 * 0 = everything on the caller's stream (used for per-kernel timing).  Environment override: MP_RENDER_STREAMS. */
int mp_set_streams(int on);

/* Per-launch timing of the tensor-core MLP kernel (CUDA events on the launching stream), by program kind:
 * [0] sdf-only, [1] forward (sdf + features), [2] full shade, [3] background.  mp_profile_read synchronises
 * on the recorded events and returns summed milliseconds, launch counts and processed points (host arrays of 4).
 * on = 2 also runs the kernel's stall-accounting build: every consumer warp (lane 0) and the weight loader sum clock64
 * intervals by step kind and phase into a per-CTA block of the MLP workspace, added after each launch into a
 * process-wide device total on the current device.  The block is part of mp_mlp_workspace_bytes (and of every query that
 * nests it) only while on = 2, so switch it on before sizing the workspaces it will run with.
 * mp_profile_read_stalls synchronises the device and copies that total out: clocks_host
 * [4 program kinds][MP_STALL_WARPS][MP_STALL_WORDS], warp 0 the loader lane, warps 1.. the consumer warps; word
 * MP_STALL_PHASES * k + ph is step kind k (0 softplus, 1 softplus saving sigma', 2 seed of the reverse sweep, 3 features,
 * 4 reverse, 5 final gradient, 6 ReLU) and phase ph (0 whole step, 1 blocked on a weight slot, 2 in wgmma waits,
 * 3 in named barriers, 4 epilogue, 5 loader blocked on a free ring position), then MP_STALL_PROLOGUE (tile
 * prologues) and MP_STALL_ELAPSED (the warp's whole run).  reset != 0 zeroes the total. */
enum { MP_STALL_KINDS = 7, MP_STALL_PHASES = 6, MP_STALL_PROLOGUE = 42, MP_STALL_ELAPSED = 43, MP_STALL_WORDS = 44,
       MP_STALL_WARPS = 9 };
int mp_profile_enable(int on);
int mp_profile_read(double* ms_host, long long* launches_host, double* points_host, int reset);
int mp_profile_read_stalls(unsigned long long* clocks_host, int reset);

/* ImplicitNet.forward (networks.py:126-208): x [N,d_in] -> out [N,257] (sdf | feature).
 * sdf / feat may be NULL.  Replaces `self.foreground_implicit_network_list[p](x_c, cond)`. */
int mp_implicit_forward(mp_net_t* f, const float* x, int N, float* sdf /*[N]*/, float* feat /*[N,256]*/,
                        void* workspace, size_t workspace_bytes, void* stream);
/* forward + d sdf / d x (replaces the autograd.grad at multiply.py:653-659) */
int mp_implicit_forward_grad(mp_net_t* f, const float* x, int N, float* sdf, float* feat, float* grad /*[N,3]*/,
                             void* workspace, size_t workspace_bytes, void* stream);
/* RenderingNet.forward 'pose_no_view' (networks.py:263-312): -> rgb [N,3] */
int mp_render_forward(mp_net_t* f, const float* points, const float* normals, const float* feat, int N,
                      float* rgb, void* workspace, size_t workspace_bytes, void* stream);
size_t mp_mlp_workspace_bytes(int N);
/* Background pair at given points (multiply.py:523-526): bg_implicit_network(pts [N,4], {'frame': code}) ->
 * sdf [N] (may be NULL) and bg_rendering_network(None, None, view_dirs [N,3], None, feature, code) -> rgb [N,3].
 * The frame code is the field's cond (mp_field_set_cond).  Workspace: mp_mlp_workspace_bytes(N). */
int mp_bg_nets_forward(mp_net_t* bg_field, const float* pts, const float* view_dirs, int N, float* sdf, float* rgb,
                       void* workspace, size_t workspace_bytes, void* stream);

/* First-order backward of the networks (DESIGN.md §3.9): layer-major wgmma GEMMs in split fp16 with fp32 accumulation,
 * every operand scaled into fp16's range by a power of two (so the accuracy does not depend on the loss's scale),
 * the forward's pre-activations recomputed in chunks of points, every sum over points bounded per tensor-core accumulator
 * and added in fp64 in a fixed order, so results are bit-identical from run to run and independent of the workspace's
 * contents.  Outputs are overwritten, not accumulated; a NULL output is not computed.  N = 0 writes zero parameter
 * gradients (the query answers 0, and a NULL workspace is accepted).  mp_set_engine does not affect these calls. */
typedef struct {             /* gradients of one linear stack; every pointer may be NULL (not wanted) */
  float* d_weight[MP_MAX_LAYERS];   /* [out,in]: dL/dW_l of the W the reference's lin{l} applies (g v/||v|| when weight-normed) */
  float* d_bias[MP_MAX_LAYERS];     /* [out] */
} mp_linear_grads_t;
/* Workspace of mp_implicit_backward over N points (either field kind). */
size_t mp_implicit_backward_workspace_bytes(int N);
/* VJP of ImplicitNet.forward (networks.py:126-208) at x [N,d_in] with the field's cond (mp_field_set_cond), for the
 * foreground (d_in 3, 'smpl' cond) and the background (d_in 4, 'frame' cond) field: d_sdf [N] and d_feat [N,256] are
 * dL/d out[:, 0] and dL/d out[:, 1:] (NULL: zero) -> d_x [N,d_in], grads (all nine layers; d_weight[0] covers the
 * cond columns, d_weight[4] is of the reference's W4, before the skip's 1/sqrt(2)) and d_cond [cond_dim]. */
int mp_implicit_backward(mp_net_t* f, const float* x, int N, const float* d_sdf /*[N] or NULL*/,
                         const float* d_feat /*[N,256] or NULL*/, float* d_x /*[N,d_in] or NULL*/,
                         mp_linear_grads_t* grads, float* d_cond /*[cond_dim] or NULL*/,
                         void* workspace, size_t workspace_bytes, void* stream);
/* Workspace of mp_render_backward over N points. */
size_t mp_render_backward_workspace_bytes(int N);
/* VJP of RenderingNet.forward 'pose_no_view' (networks.py:263-312; 270 -> 4 x 256 -> 3) with the field's cond as
 * body_pose: d_rgb [N,3] -> d_points, d_normals [N,3], d_feat [N,256], grads of lin0..lin4, lin_pose's d weight [8,69]
 * and d bias [8], d_body_pose [69].  A background field is refused before anything is enqueued. */
int mp_render_backward(mp_net_t* f, const float* points, const float* normals, const float* feat, int N,
                       const float* d_rgb /*[N,3]*/, float* d_points, float* d_normals, float* d_feat,
                       mp_linear_grads_t* grads, float* d_lin_pose_weight /*[8,69]*/, float* d_lin_pose_bias /*[8]*/,
                       float* d_body_pose /*[69]*/, void* workspace, size_t workspace_bytes, void* stream);

/* Canonical SDF on the dense lattice of lib/utils/mesh.py:generate_mesh (:78-105; the values MISE's octree queries
 * through Multiply.query_oc, multiply.py:169-172, batch by batch): values[(ix*(res+1)+iy)*(res+1)+iz] =
 * ImplicitNet(p)[0] with p = ((idx/res - 0.5) * pad) * extent + centre (fp32, rounded step by step as numpy does;
 * pad = 1.1, extent = the longest side of the SMPL bounds).  The pose conditioning is the field's cond
 * (mp_field_set_cond).  The lattice is generated on the device and streamed through the sdf-only MLP program in
 * 2^20-point slabs. */
size_t mp_sdf_grid_workspace_bytes(int res);
int mp_sdf_grid(mp_net_t* field, const float* center_host /*[3]*/, float extent, float pad, int res,
                float* values /*[(res+1)^3]*/, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * deformer: SMPLDeformer (lib/model/deformer.py:6-89)
 * ---------------------------------------------------------------------------------------- */
typedef struct mp_body mp_body_t;
size_t mp_body_bytes(int V);
/* verts_cano [V,3], weights [V,24]: SMPLDeformer.smpl_verts / smpl_weights (deformer.py:16-17).
 * Builds the canonical-space vertex grid once. */
int mp_body_create(const float* verts_cano, const float* weights, int V, float cano_cell,
                   void* storage, size_t storage_bytes, mp_body_t** out, void* stream);
void mp_body_free(mp_body_t* b);
/* per frame: posed verts [V,3] (smpl_output['smpl_verts']) and bone transforms [24,4,4] (smpl_tfs);
 * rebuilds the posed-space vertex grid (cell >= 0.1 = the outlier radius of deformer.py:49). */
int mp_body_set_pose(mp_body_t* b, const float* verts_posed, const float* tfs, void* stream);

/* SMPLDeformer.forward(x, smpl_tfs, return_weights=False, inverse=True, smpl_verts) (deformer.py:19-30):
 * x [N,3] -> x_c [N,3], outlier [N] (uint8).  exact_far != 0 also resolves the exact nearest
 * vertex of points farther than the grid radius (needed only when outliers are not pruned). */
int mp_deform_inverse(mp_body_t* b, const float* x, int N, float* x_c, uint8_t* outlier, int exact_far,
                      void* stream);
/* SMPLDeformer.forward_skinning (deformer.py:31-35) + the Jacobian the reference obtains by three
 * autograd VJPs (multiply.py:625-640): x_c [N,3] -> x_d [N,3] (may be NULL), Jinv [N,9] = inverse of
 * the upper-left 3x3 of sum_j w_j tfs_j with w from the nearest CANONICAL vertex. */
int mp_deform_forward_jac(mp_body_t* b, const float* x_c, int N, float* x_d, float* Jinv, void* stream);

/* Backward of the two deformer calls (VJPs; the weights are detached, deformer.py:47, so gradients reach the points and
 * the bone transforms only).  Both use the body's current pose (mp_body_set_pose), recompute the nearest vertex with the
 * forward's own search, and write every element of d_tfs [24,4,4] (= dL/d smpl_tfs; N = 0 gives zeros).  Sums over
 * points are per-CTA partials added in a fixed order (no float atomics): reruns are bit-identical.  Workspace:
 * mp_deform_backward_workspace_bytes(N); its contents on entry do not matter.
 *
 * mp_deform_inverse_backward: of mp_deform_inverse (skinning(inverse=True), deformer.py:72-89, weights of the nearest
 * POSED vertex).  d_x_c [N,3] required; with A = sum_j w_j tfs_j, u = A[:3,:3]^-T d_x_c: dL/dA = -[u ; -t.u/s] [x_c ; 1]^T
 * (all four rows, as torch's inverse backward gives them), d_x [N,3] = u (NULL: not written), x_c [N,3] = the recomputed
 * canonical point, bit-equal to mp_deform_inverse's (NULL: not written).  A point with no vertex within reach
 * (exact_far == 0) has x_c = x: d_x = d_x_c, nothing to the bones.  Refused while the body's root finder is on (the
 * reference has none, so that gradient has no definition to match).
 *
 * mp_deform_forward_jac_backward: of mp_deform_forward_jac (forward skinning with the weights of the nearest CANONICAL
 * vertex, deformer.py:31-35, and the inverse Jacobian of multiply.py:625-641).  d_x_d [N,3] and d_Jinv [N,9] may be NULL
 * (zero).  dL/dJ = -Jinv^T d_Jinv Jinv^T and d_x_d [x_c;1]^T go to tfs_j[:3,:]; the bottom row of d_tfs is 0.
 * d_x_c [N,3] = J^T d_x_d (NULL: not written). */
size_t mp_deform_backward_workspace_bytes(int N);
int mp_deform_inverse_backward(mp_body_t* b, const float* x, int N, int exact_far, const float* d_x_c,
                               float* d_tfs, float* d_x, float* x_c, void* workspace, size_t workspace_bytes,
                               void* stream);
int mp_deform_forward_jac_backward(mp_body_t* b, const float* x_c, int N, const float* d_x_d, const float* d_Jinv,
                                   float* d_tfs, float* d_x_c, void* workspace, size_t workspace_bytes, void* stream);

/* Optional root finder (SURVEY.md §8 row f4; BASELINE.json north_star: "Broyden-root-finds canonical points").  The
 * reference has NO such step (SURVEY.md fact 0-1: its deformer is KNN + closed-form inverse LBS, deformer.py:19-50), so
 * this is non-default and checked against its own CPU restatement (oracle/port.py:deform_broyden), not against MultiPly.
 * Solves forward_skinning(x_c) = x (deformer.py:31-35: weights of the nearest CANONICAL vertex) by Broyden's method
 * started from the closed-form inverse (weights of the nearest POSED vertex), J^-1 initialised with the inverse
 * blended 3x3 at the start point, at most max_steps rank-one updates, lowest-residual iterate returned.
 *   x [N,3] -> x_c [N,3]; residual [N] = |forward_skinning(x_c) - x| (NULL ok); converged [N] = residual <
 *   cvg_threshold (NULL ok); outlier [N] as mp_deform_inverse (NULL ok); steps [N] iterations taken (NULL ok). */
int mp_deform_broyden(mp_body_t* b, const float* x, int N, int max_steps, float cvg_threshold, float* x_c,
                      float* residual, uint8_t* converged, uint8_t* outlier, int* steps, void* stream);
/* max_steps > 0 makes every inverse-deformer call on this body (mp_deform_inverse, mp_sdf_with_deformer, the sampler
 * and the main pass of mp_render_rays) refine its non-outlier points this way; 0 (the default) = reference behaviour. */
int mp_body_set_root_finder(mp_body_t* b, int max_steps, float cvg_threshold);

/* ------------------------------------------------------------------------------------------
 * density: LaplaceDensity (lib/model/density.py:11-29)
 * ---------------------------------------------------------------------------------------- */
int mp_laplace_density(const float* sdf, int N, float beta, float* sigma, void* stream);

/* ------------------------------------------------------------------------------------------
 * rays: rend_util.get_camera_params / get_sphere_intersections (lib/utils/rend_util.py:45-87,131-147)
 * ---------------------------------------------------------------------------------------- */
int mp_camera_rays(const float* uv /*[R,2]*/, const float* pose /*[4,4]*/, const float* intrinsics /*[4,4]*/,
                   int R, float* ray_dirs /*[R,3]*/, float* cam_loc /*[R,3]*/, void* stream);
/* status_flag (device int) is set to 1 if any ray misses the sphere (the reference calls exit(), :140-142) */
int mp_sphere_intersections(const float* cam_loc, const float* ray_dirs, int R, float r,
                            float* near_far /*[R,2]*/, int* status_flag, void* stream);

/* Ray / box culling (replaces the host-side trimesh ray/triangle test on the x1.2 oriented box,
 * multiply.py:208-214, :256-263): box = centre + half extents (host doubles) + optional 3x3 rotation (device
 * doubles, rows = box axes, NULL = axis aligned).  idx_out [R] receives the hit ray ids in ascending order,
 * count_dev their number.  An empty result is the caller's to replace by ray 0 (multiply.py:262-263). */
int mp_ray_box_hits(const float* cam_loc, const float* ray_dirs, int R, const double* center_host,
                    const double* half_extent_host, const double* rot_dev, int64_t* idx_out, int* count_dev,
                    void* stream);
/* multiply.py:262-263 on the device: an empty hit list becomes the single ray 0 (idx[0] = 0, *count_dev = 1). */
int mp_hit_list_finalize(int64_t* idx, int* count_dev, void* stream);
/* Same test with the box taken from the posed vertices on the device (no host read of the vertices): centre and half
 * extents of the axis-aligned bounds of verts [V,3], inflated by `inflate` (1.2, multiply.py:212).  box_ws: >= 64 bytes
 * of device scratch. */
int mp_ray_aabb_hits(const float* cam_loc, const float* ray_dirs, int R, const float* verts, int V, double inflate,
                     int64_t* idx_out, int* count_dev, void* box_ws, void* stream);

/* ------------------------------------------------------------------------------------------
 * SMPL server: SMPLServer.forward (lib/model/smpl.py:50-95) -> SMPL.forward (lib/smpl/body_models.py:278-364)
 * -> lbs (lib/smpl/lbs.py:136-229).  Model arrays are the ones the SMPL pkl provides (device pointers, kept by
 * reference); parents is a host array of 24 ints.  The canonical pose of smpl.py:35-47 is evaluated at creation.
 * ---------------------------------------------------------------------------------------- */
typedef struct mp_smpl mp_smpl_t;
size_t mp_smpl_bytes(int V);
int mp_smpl_create(const float* v_template /*[V,3]*/, const float* shapedirs /*[V,3,10]*/,
                   const float* posedirs /*[207,V*3]*/, const float* J_regressor /*[24,V]*/,
                   const int* parents_host /*[24]*/, const float* lbs_weights /*[V,24]*/, int V,
                   const float* betas_canonical /*[10] device or NULL*/, void* storage, size_t storage_bytes,
                   mp_smpl_t** out, void* stream);
void mp_smpl_free(mp_smpl_t* s);
/* SMPLServer.verts_c [V,3] and tfs_c_inv [24,4,4] (either may be NULL) */
int mp_smpl_canonical(mp_smpl_t* s, float* verts_c, float* tfs_c_inv, void* stream);
/* scale [1], transl [3], thetas [72], betas [10] (device) -> smpl_verts [V,3], smpl_tfs [24,4,4] */
int mp_smpl_forward(mp_smpl_t* s, const float* scale, const float* transl, const float* thetas, const float* betas,
                    int absolute, float* smpl_verts, float* smpl_tfs, void* stream);
/* Backward (VJP) of mp_smpl_forward with the same inputs: d_verts [V,3] and d_tfs [24,4,4] are the upstream gradients
 * (either may be NULL: zero; the bottom row of d_tfs reaches no parameter and is ignored) -> d_scale [1], d_transl [3],
 * d_thetas [72], d_betas [10], every element written.  Reverses skinning, the pose blend (posedirs), the shape blend
 * (shapedirs), J = J_t + J_s betas, the kinematic chain, the rel_transforms correction (lbs.py:371-376), Rodrigues as
 * lbs.py:276-307 writes it (angle = |theta + 1e-8|; theta = 0 gets the finite skew-basis derivative), scale /
 * translation (smpl.py:86-88) and the tfs_c_inv product when absolute == 0.  Everything is recomputed from the inputs
 * (the handle's per-call scratch is not read); the per-joint part runs in fp64.  Sums over vertices are per-CTA partials
 * added in a fixed order: reruns are bit-identical.  A server built with v_template ignores betas (smpl.py:65-66): its
 * caller passes zero betas and discards d_betas.  Workspace: mp_smpl_backward_workspace_bytes(V), any contents. */
size_t mp_smpl_backward_workspace_bytes(int V);
int mp_smpl_backward(mp_smpl_t* s, const float* scale, const float* transl, const float* thetas, const float* betas,
                     int absolute, const float* d_verts, const float* d_tfs, float* d_scale, float* d_transl,
                     float* d_thetas, float* d_betas, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * sampler: ErrorBoundSampler (lib/model/ray_sampler.py:45-230), eval mode
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  float scene_bounding_sphere; /* 3.0 (multiply.py:85) */
  float near;                  /* 0.0 */
  int N_samples;               /* S */
  int N_samples_eval;          /* E */
  int N_samples_extra;         /* X */
  float eps;                   /* 0.1 */
  int beta_iters;              /* 10 */
  int max_total_iters;         /* 5 */
  float add_tiny;              /* 1e-6 */
  float beta_param;            /* density.beta parameter; beta = |beta_param| + beta_min */
  float beta_min;              /* 1e-4 */
} mp_sampler_cfg_t;

size_t mp_sampler_workspace_bytes(const mp_sampler_cfg_t* cfg, int R);
/* ErrorBoundSampler.get_z_vals(ray_dirs, cam_loc, model, cond, smpl_tfs, eval_mode=True, smpl_verts, person_id)
 * (ray_sampler.py:66-220).  The SDF callback of the reference (`model.sdf_func_with_smpl_deformer`)
 * is the (body, field) pair.  Outputs z_vals [R, S+X+2], z_bg [R,32] (may be NULL); trips_out (device
 * int, may be NULL) receives the number of Algorithm-1 iterations executed.  No host sync. */
int mp_sample_rays(const mp_sampler_cfg_t* cfg, mp_body_t* body, mp_net_t* field,
                   const float* ray_dirs, const float* cam_loc, int R,
                   float* z_vals, float* z_bg, int* trips_out,
                   void* workspace, size_t workspace_bytes, void* stream);

/* Training-mode get_z_vals (model.training: ray_sampler.py:32-40 stratified start samples, :171 random abscissae of the
 * final set, :202 randperm extras, :212-213 the eikonal pick, :216 jittered inverse-sphere depths; the SDF callback does
 * not clamp outliers, multiply.py:142).  Every random draw of the reference is an INPUT so that a caller can replay the
 * reference's RNG stream.  The draws made after the Algorithm-1 loop depend on the number of trips T+1 the loop took
 * (randperm((T+1) E), and the generator state after it), which only the device knows: they are passed for EVERY possible
 * T and the kernels pick the row of the trip the loop ended on.  T_max = cfg->max_total_iters. */
typedef struct {
  const float* t_rand;     /* [R, E]                      torch.rand of UniformSampler.get_z_vals */
  const float* u_final;    /* [R, S]                      torch.rand at the final inverse-CDF step */
  const int* extra_perm;   /* [T_max, T_max*E] int32      row T: torch.randperm((T+1)*E), first X entries are used */
  const int* eik_idx;      /* [T_max, R] int32            row T: torch.randint(S+X+2, (R,)) */
  const float* t_rand_bg;  /* [T_max, R, 32] or NULL      row T: torch.rand of the inverse-sphere UniformSampler */
} mp_sampler_rng_t;
/* outputs as mp_sample_rays plus z_eik [R] (z_samples_eik, may be NULL).  Requires N_samples_extra <= N_samples_eval:
 * after one trip randperm(E)[:X] has only min(X, E) entries, so a larger X is rejected with an error. */
int mp_sample_rays_train(const mp_sampler_cfg_t* cfg, mp_body_t* body, mp_net_t* field,
                         const float* ray_dirs, const float* cam_loc, int R, const mp_sampler_rng_t* rng,
                         float* z_vals, float* z_bg, float* z_eik, int* trips_out,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Multiply.sdf_func_with_smpl_deformer (multiply.py:137-151, eval): x [N,3] -> sdf [N] (4.0 on outliers),
 * x_c [N,3], feat [N,256] (may be NULL). */
size_t mp_sdf_with_deformer_workspace_bytes(int N);
int mp_sdf_with_deformer(mp_body_t* body, mp_net_t* field, const float* x, int N,
                         float* sdf, float* x_c, float* feat,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * compositing (multiply.py:427-480 with nerfacc; 682-696 background)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int n_rows;               /* rays in this person's hit list (R_p) */
  const int64_t* ray_index; /* [R_p] sorted ray ids (index_ray_box, multiply.py:256-263) */
  const float* z_vals;      /* [R_p, n+1] (last column = z_max) */
  const float* sdf;         /* [R_p, n] */
  const float* rgb;         /* [R_p, n, 3] */
  const float* normal;      /* [R_p, n, 3] */
} mp_person_samples_t;

size_t mp_composite_workspace_bytes(int R, int P);
/* outputs: fg_rgb [R,3], normal [R,3], acc [R], acc_person [R,P], bg_T [R] */
int mp_composite(const mp_person_samples_t* persons_host, int P, int R, int n, float beta,
                 float* fg_rgb, float* normal, float* acc, float* acc_person, float* bg_T,
                 void* workspace, size_t workspace_bytes, void* stream);

/* rgb_values = fg_rgb + bg_T * bg_rgb (bg_rgb NULL -> white, multiply.py:540-545), fg_rgb_values = fg_rgb + bg_T * 1
 * (multiply.py:590); fg_rgb_values may be NULL.  The last stage of Multiply.forward, exported for callers that composite
 * ray blocks themselves (person-sharded rendering, multiply_b200/parallel.py). */
int mp_final_compose(const float* fg_rgb /*[R,3]*/, const float* bg_T /*[R]*/, const float* bg_rgb /*[R,3] or NULL*/, int R,
                     float* rgb_values /*[R,3]*/, float* fg_rgb_values /*[R,3] or NULL*/, void* stream);

/* Backward of the compositing stages (multiply.py:427-480, :544-545, :590, :682-696) with torch autograd's kink
 * conventions: d sigma / d sdf = 0 at sdf == 0 (sign(0) = 0) and d|s|/ds = sign(s).  Every upstream gradient d_* may be
 * NULL, meaning zero, unless marked required.  Each output slot is written once; deterministic (no float atomics).
 *
 * mp_composite_backward: the same inputs as mp_composite plus the upstream gradients d_fg_rgb [R,3], d_normal [R,3],
 * d_acc [R], d_acc_person [R,P], d_bg_T [R]; writes per person p the sample gradients of its [R_p, n] rows and
 * d_beta (one device float, required) = dL/dbeta for beta = |beta_param| + beta_min (the chain to beta_param is the
 * caller's).  Rays no person hits contribute nothing (their bg_T = 1 is a constant). */
typedef struct {
  float* d_sdf;             /* [R_p, n] */
  float* d_rgb;             /* [R_p, n, 3] */
  float* d_normal;          /* [R_p, n, 3] */
} mp_person_sample_grads_t;

size_t mp_composite_backward_workspace_bytes(int R, int P);
int mp_composite_backward(const mp_person_samples_t* persons_host, int P, int R, int n, float beta,
                          const float* d_fg_rgb, const float* d_normal, const float* d_acc, const float* d_acc_person,
                          const float* d_bg_T, const mp_person_sample_grads_t* grads_host, float* d_beta,
                          void* workspace, size_t workspace_bytes, void* stream);
/* bg_volume_rendering + the weighted sum (multiply.py:682-696, :539): bg_sdf [R,32], bg_rgb_samples [R,32,3] in the
 * flipped depth order the networks see (the bg_sdf / bg_rgb_samples taps of mp_render_out_t); depths from bound_r and
 * t_rand_bg [R,32] (training) or NULL (eval), the last interval 1e10 long.  d_bg_rgb [R,3] (required) ->
 * d_bg_sdf [R,32], d_bg_rgb_samples [R,32,3]. */
int mp_bg_composite_backward(const float* bg_sdf, const float* bg_rgb_samples, int R, float bound_r,
                             const float* t_rand_bg_or_null, const float* d_bg_rgb, float* d_bg_sdf,
                             float* d_bg_rgb_samples, void* stream);
/* backward of mp_final_compose: d_fg_rgb = d_rgb_values + d_fg_rgb_values ; d_bg_T = sum_c (d_rgb_values_c * bg_rgb_c +
 * d_fg_rgb_values_c) (bg_rgb NULL -> white) ; d_bg_rgb = bg_T * d_rgb_values (may be NULL: not written). */
int mp_final_compose_backward(const float* bg_T /*[R]*/, const float* bg_rgb_or_null /*[R,3]*/, int R,
                              const float* d_rgb_values /*[R,3]*/, const float* d_fg_rgb_values_or_null /*[R,3]*/,
                              float* d_fg_rgb /*[R,3]*/, float* d_bg_T /*[R]*/, float* d_bg_rgb_or_null /*[R,3]*/,
                              void* stream);

/* background: inverse-sphere samples -> depth2pts_outside (multiply.py:698-726) -> bg nets -> bg_volume_rendering
 * A ray through the sphere's centre (cross(o, p_sphere) = 0) gets the limit p_sphere / |p_sphere| where the reference
 * returns NaN. */
size_t mp_background_workspace_bytes(int R);
int mp_background(mp_net_t* bg_field, const float* ray_dirs, const float* cam_loc, int R, float bound_r,
                  float* bg_rgb /*[R,3]*/, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * canonical mesh: kaolin.metrics.trianglemesh.point_to_mesh_distance and kaolin.ops.mesh.check_sign as used by
 * Multiply.check_off_in_surface_points_cano_mesh (multiply.py:153-167) and MultiplyModel.get_interpenetration_loss
 * (multiply_model.py:532).  A uniform grid of face references over the mesh's bounds; one handle per mesh, built
 * once (model build, multiply.py:118-121, and each mesh swap, multiply_model.py:504-506).
 * ---------------------------------------------------------------------------------------- */
typedef struct mp_mesh mp_mesh_t;
#define MP_MESH_PLAN_SCRATCH_BYTES 1024
typedef struct {
  int V, F;
  double lo[3];            /* grid origin (mesh bounds minus the margin) */
  double h;                /* cubic cell size */
  int dim[3];              /* cells per axis */
  long long n_refs;        /* (cell, face) references */
  size_t storage_bytes;    /* device storage mp_mesh_create needs */
} mp_mesh_plan_t;
/* verts [V,3] fp32, faces [F,3] int64 (device).  Sizes the grid over the bounds padded by `margin` and counts the
 * references each face's bounding box makes; scratch: MP_MESH_PLAN_SCRATCH_BYTES of device memory.  Synchronises
 * `stream` once (to read the sizes back). */
int mp_mesh_plan(const float* verts, int V, const int64_t* faces, int F, float margin, void* scratch,
                 mp_mesh_plan_t* plan_host, void* stream);
/* Builds the grid (count, scan, fill on the device) into caller storage of plan->storage_bytes; verts / faces must be
 * the arrays given to mp_mesh_plan.  They are copied: the caller may release them once the stream has passed. */
int mp_mesh_create(const mp_mesh_plan_t* plan_host, const float* verts, const int64_t* faces, void* storage,
                   size_t storage_bytes, mp_mesh_t** out, void* stream);
void mp_mesh_free(mp_mesh_t* mesh);
/* kaolin point_to_mesh_distance (multiply.py:155): pts [N,3] -> dist2 [N] squared distance to the nearest face,
 * face_idx [N] its index (lowest on ties), dist_type [N] where on it: 0 interior, 1/2/3 vertex 0/1/2, 4/5/6 edge
 * 01/12/20.  face_idx / dist_type may be NULL. */
int mp_mesh_distance(const mp_mesh_t* mesh, const float* pts, int N, float* dist2, int64_t* face_idx, int* dist_type,
                     void* stream);
/* kaolin check_sign (multiply.py:158, multiply_model.py:532): inside [N] = 1 iff the ray p + t (0,0,1), t > 0, crosses
 * the mesh an odd number of times (fp64 watertight crossing test).  Meaningful for watertight meshes only. */
int mp_mesh_check_sign(const mp_mesh_t* mesh, const float* pts, int N, uint8_t* inside, void* stream);
/* check_off_in_surface_points_cano_mesh (multiply.py:153-167): x_c [rows*N_samples,3] (row-major by ray) -> off [rows]
 * = min over the row's samples of the signed distance > thr, in [rows] = that minimum <= 0 (uint8).  The signed
 * distance is -sqrtf(d2) inside and +sqrtf(d2) outside, compared in fp32.  Any thr is allowed, including thr <= 0 (with
 * thr < 0 an inside sample at depth d < |thr| keeps off) and +-inf; a NaN thr is an error. */
int mp_mesh_surface_flags(const mp_mesh_t* mesh, const float* x_c, int rows, int N_samples, float thr, uint8_t* off,
                          uint8_t* in, void* stream);

/* ------------------------------------------------------------------------------------------
 * posed-mesh depth maps and the nearest partner vertex: the pytorch3d operators of opt_depth's geometric losses,
 * Renderer.render_multiple_depth_map (lib/model/render.py:135-157, layer 0 of zbuf, multiply_model.py:396-401) and
 * pytorch3d.ops.knn_points(K=1, return_nn=True) (multiply_model.py:539).  Definitions: oracle/raster.py and
 * oracle/port.py:knn_points (DESIGN §3.8).  Backward sums are stable sorts by vertex, each vertex summing its terms in
 * a fixed order in fp64 (no float atomics): reruns are bit-identical.  Every output element is written.
 * ---------------------------------------------------------------------------------------- */
/* The camera of Renderer.set_camera in OpenCV's convention (the flips of render.py:73-78 cancel): (X, Y, Z) = R v + T,
 * u = fx X / Z + cx, v = fy Y / Z + cy; fx, fy, cx, cy = K[0,0], K[1,1], K[0,2], K[1,2] of cv2's decomposition. */
typedef struct {
  float R[9];              /* world -> camera rotation, row-major */
  float T[3];
  float fx, fy, cx, cy;
} mp_camera_t;
/* verts [V,3] fp32, faces [F,3] int64 -> zbuf [H,W] (view-space depth of the nearest covering face, -1 where none) and
 * pix_to_face [H,W] int64 (its index, -1 where none).  Pixel (r, c) samples the image point (c + 0.5, r + 0.5); a face
 * covers it when the point lies in the closed projected triangle; depth z = 1 / sum_i(b_i / Z_i) (perspective-correct,
 * fp64 on the fp32 inputs, rounded to fp32 once); the nearest fp32 depth wins, then the lowest face index.  Faces with a
 * vertex at Z <= 0, of zero projected area, or with an index outside [0, V) are skipped.  Needs H, W >= 1, V, F >= 0. */
size_t mp_depth_raster_workspace_bytes(int H, int W, int F);
int mp_depth_raster(const mp_camera_t* cam_host, const float* verts, int V, const int64_t* faces, int F, int H, int W,
                    float* zbuf, int64_t* pix_to_face, void* workspace, size_t workspace_bytes, void* stream);
/* d_verts [V,3] = sum over pixels of d_zbuf [H,W] times the exact derivative of the pixel's z with respect to its face's
 * world-space vertices, the face (pix_to_face, as mp_depth_raster wrote it) held fixed; vertices no such face touches
 * get 0. */
size_t mp_depth_raster_backward_workspace_bytes(int H, int W, int V);
int mp_depth_raster_backward(const mp_camera_t* cam_host, const float* verts, int V, const int64_t* faces, int F, int H,
                             int W, const int64_t* pix_to_face, const float* d_zbuf, float* d_verts, void* workspace,
                             size_t workspace_bytes, void* stream);
/* p1 [N1,3], p2 [N2,3] fp32 (N2 >= 1) -> dists [N1] = min_j (dx*dx + dy*dy) + dz*dz (fp32, each step rounded), idx [N1]
 * int64 the arg-min (lowest index on ties), nn [N1,3] = p2[idx]; any output may be NULL (not written).  Finite inputs. */
size_t mp_knn1_workspace_bytes(int N1);
int mp_knn1(const float* p1, int N1, const float* p2, int N2, float* dists, int64_t* idx, float* nn, void* workspace,
            size_t workspace_bytes, void* stream);
/* Backward of mp_knn1 at its idx: d_dists [N1] and d_nn [N1,3] may be NULL (zero).  d_p1 [N1,3] = 2 (p1 - nn) d_dists;
 * d_p2 [N2,3] = sum over the queries i with idx[i] = j of d_nn[i] - 2 (p1 - nn) d_dists[i]. */
size_t mp_knn1_backward_workspace_bytes(int N1, int N2);
int mp_knn1_backward(const float* p1, int N1, const float* p2, int N2, const int64_t* idx, const float* d_dists,
                     const float* d_nn, float* d_p1, float* d_p2, void* workspace, size_t workspace_bytes,
                     void* stream);

/* ------------------------------------------------------------------------------------------
 * mesh extraction: lib/utils/mesh.py:generate_mesh (:78-132) — MISE, marching cubes, largest component (DESIGN §3.7).
 * Grids are [(R+1)^3] fp32, x-major: value (ix, iy, iz) at (ix*(R+1) + iy)*(R+1) + iz, as mp_sdf_grid writes them.
 * ---------------------------------------------------------------------------------------- */
/* MISE (generate_mesh :87-109 driving lib/libmise/mise.pyx, then to_dense :130-164) with R = res_init << depth in
 * [1, 1024]: starts from the (res_init+1)^3 points at stride 2^depth, evaluates every added point once through the
 * sdf-only program (points placed as mp_sdf_grid places them; the field's cond as set by mp_field_set_cond), splits
 * every leaf below depth that some known point marks both ways (value >= level and value <= level; a point marks every
 * leaf whose closed box holds it) and stops when a round adds no point.  grid receives the evaluated values, the rest
 * filled by copying forward along x, then y, then z.  evaluated [(R+1)^3] (uint8, may be NULL) = 1 where a point was
 * evaluated; *n_evaluated_host (may be NULL) their number.  Synchronises `stream` once per round (the number of
 * points to evaluate). */
size_t mp_mise_workspace_bytes(int res_init, int depth);
int mp_mise(mp_net_t* field, const float* center_host /*[3]*/, float extent, float pad, int res_init, int depth,
            double level, float* grid /*[(R+1)^3]*/, uint8_t* evaluated, long long* n_evaluated_host,
            void* workspace, size_t workspace_bytes, void* stream);
/* Marching cubes on any grid (generate_mesh :111-119; the tiling is DESIGN §3.7's, not skimage's Lewiner tables).  A
 * corner is below when (double)v < level; an edge with one end below owns one vertex at t = (level - v0) / (v1 - v0)
 * (fp64, v0 at the lower index), in world space ((p / R - 0.5) * pad) * extent + centre (fp64, rounded to fp32 once).
 * Vertices in lattice-edge order, faces in cube order, oriented so that (v1-v0) x (v2-v0) points toward increasing
 * value.  Two calls sharing one workspace: _count reads the sizes back (one synchronisation), _emit fills verts [V,3]
 * and faces [F,3] (either may be NULL: not written). */
size_t mp_marching_cubes_workspace_bytes(int res);
int mp_marching_cubes_count(const float* grid, int res, double level, long long* V_host, long long* F_host,
                            void* workspace, size_t workspace_bytes, void* stream);
int mp_marching_cubes_emit(const float* grid, int res, double level, const double* center_host /*[3]*/, double extent,
                           double pad, float* verts, int64_t* faces, void* workspace, size_t workspace_bytes,
                           void* stream);
/* The connected component of largest area (generate_mesh :122-130; faces connected through shared vertices), areas
 * summed in fp64 in a fixed order; on equal areas the component holding the lowest face index.  Its faces and vertices
 * are compacted in their order into verts_out [V,3] / faces_out [F,3] (capacity V / F) and re-indexed; the kept sizes go
 * to *V_out_host / *F_out_host (one synchronisation).  V == 0 or F == 0: an empty result, no error. */
size_t mp_largest_component_workspace_bytes(int V, int F);
int mp_largest_component(const float* verts, int V, const int64_t* faces, int F, float* verts_out, int64_t* faces_out,
                         int* V_out_host, int* F_out_host, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * the fused entry used by Multiply.forward (multiply.py:174-598, eval branch)
 * ---------------------------------------------------------------------------------------- */
/* Training-mode forward VALUES (multiply.py:174-598 with self.training, shipped loss weights, current_epoch >= 250):
 * stochastic sampling per person (mp_sampler_rng_t), no outlier clamp in the SDF callback or the main pass
 * (multiply.py:142 is eval-only), jittered inverse-sphere depths of the background pass (the second
 * inverse_sphere_sampler.get_z_vals call, :482).  The render produces no gradients itself; the backward of its
 * compositing stages is mp_composite_backward / mp_bg_composite_backward / mp_final_compose_backward on its taps. */
typedef struct {
  const mp_sampler_rng_t* rng[MP_MAX_PERSONS]; /* host structs of device pointers, one per person */
  float* z_eik[MP_MAX_PERSONS];                /* [R_p] z_samples_eik out, or NULL */
  const float* t_rand_bg;                      /* [R,32] torch.rand of the background's UniformSampler, or NULL */
  /* current_epoch < 250 (multiply.py:313-316, :549-560): when cano_mesh[k] is set, the canonical points of rendered
   * person k's main pass go through mp_mesh_surface_flags' kernel, and the per-person flags are merged into
   * index_off_surface [R] (AND over persons; rays a person does not hit count as off) and index_in_surface [R] (OR).
   * All NULL: no flags (epoch >= 250). */
  const mp_mesh_t* cano_mesh[MP_MAX_PERSONS];
  float surface_threshold;                     /* 0.05 (multiply.py:88); any value but NaN (mp_mesh_surface_flags) */
  uint8_t* index_off_surface;                  /* [R] out, required when a mesh is set */
  uint8_t* index_in_surface;                   /* [R] out, required when a mesh is set */
} mp_train_t;

typedef struct {
  mp_sampler_cfg_t sampler;
  int P;
  mp_body_t* body[MP_MAX_PERSONS];
  mp_net_t* field[MP_MAX_PERSONS];
  mp_net_t* bg_field;              /* NULL -> white background (multiply.py:540-541) */
  const int64_t* hit_index[MP_MAX_PERSONS]; /* device, sorted ray ids per person */
  int hit_count[MP_MAX_PERSONS];            /* >=1 (the reference substitutes ray 0 for an empty list) */
  /* Optional device-side row counts (GPU culling without a host round trip, mp_ray_box_hits + mp_hit_list_finalize):
   * when hit_count_dev[p] != NULL, hit_count[p] is the CAPACITY of hit_index[p] (normally R) and the number of valid
   * rows is read on the device by every kernel of person p's branch.  NULL -> hit_count[p] is exact. */
  const int* hit_count_dev[MP_MAX_PERSONS];
  const mp_train_t* train;                  /* NULL: eval mode */
} mp_scene_t;

typedef struct {
  float* rgb_values;      /* [R,3] */
  float* fg_rgb_values;   /* [R,3] */
  float* normal_values;   /* [R,3] */
  float* acc_map;         /* [R] */
  float* acc_person_list; /* [R,P] */
  /* optional debug taps (NULL to skip): per person p, [R_p, n+1], [R_p, n], [R_p,n,3], [R_p,n,3] */
  float* z_vals[MP_MAX_PERSONS];
  float* sdf[MP_MAX_PERSONS];
  float* rgb[MP_MAX_PERSONS];
  float* normals[MP_MAX_PERSONS];
  int* trips;             /* device [P] or NULL */
  float* bg_T;            /* [R] or NULL */
  int* status;            /* device int or NULL: bit 0 = some ray misses the bounding sphere (the reference prints
                             'BOUNDING SPHERE PROBLEM' and exits, rend_util.py:140-142; its pixels are undefined here) */
  /* optional background taps (NULL to skip; written only when a background is rendered), the inputs of
   * mp_bg_composite_backward: bg_rgb [R,3] (bg_rgb_values, multiply.py:539), bg_sdf [R,32] and bg_rgb_samples [R,32,3]
   * (the background networks' per-sample outputs in the flipped depth order of multiply.py:516) */
  float* bg_rgb;
  float* bg_sdf;
  float* bg_rgb_samples;
} mp_render_out_t;

size_t mp_render_workspace_bytes(const mp_scene_t* scene, int R);
/* uv [R,2], pose [4,4], intrinsics [4,4] (device).  Replaces Multiply.forward(input) in eval mode. */
int mp_render_rays(const mp_scene_t* scene, const float* uv, const float* pose, const float* intrinsics,
                   int R, const mp_render_out_t* out, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MULTIPLY_B200_H */
