/*
 * gs_b200.h — C ABI of libgs_b200.so: H100-native (sm_90a) differentiable tile rasterizer.
 *
 * This is the drop-in boundary for the hot path of WangFeng18/3d-gaussian-splatting
 * (projection + 3D->2D covariance, (tile|depth) sort, front-to-back alpha blend, and the
 * backward of all of it).  The reference exposes that path as a torch/pybind11 module
 * named `gaussian` (reference src/bindings.cpp:21-50); our pybind shim
 * (3d-gaussian-splatting_b200/csrc/bindings.cpp) keeps that Python-visible surface and
 * forwards every call to the functions below.  Everything here is plain C:
 *   - raw DEVICE pointers (unless a name ends in `_host`), explicit sizes,
 *   - a trailing `gs_stream_t` (a `cudaStream_t`; NULL = legacy default stream),
 *   - return value: 0 on success, otherwise a `cudaError_t` code (or GS_ERR_* < 0),
 *   - no function allocates or synchronises unless its comment says so.
 * All tensors are dense row-major float32 unless stated; indices int32; mask int64.
 */
#ifndef GS_B200_H
#define GS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* gs_stream_t; /* cudaStream_t */

#define GS_ERR_INVALID_ARG (-1)
#define GS_ERR_UNSUPPORTED (-2)
#define GS_ERR_NO_FORWARD (-3)

/* ABI version of this header (bumped on any signature change). */
int gs_abi_version(void);
/* Human-readable text of the last error on this host thread ("" if none). */
const char* gs_last_error(void);
/* A/B tuning knobs of the blend kernels (A/B experiments; defaults = the configuration measured fastest on the H100):
 * "fwd_kernel", "fwd_ch", "bwd_kernel", "bwd_px", "bwd_ws", "bwd_unroll", "bwd_stages", "bwd_minb"
 * (see csrc/internal.h GsTuning).  An unsupported combination makes the next backward fail with
 * cudaErrorInvalidValue.  Process-wide, not thread-safe. */
int gs_tune(const char* name, int value);
/* Number of kernels of THIS library launched by the process so far (library kernels such as CUB's are not
 * counted); bench.py reports the difference over its timed region as `gpu_launches`. */
unsigned long long gs_kernel_launches(void);

/* ---------------------------------------------------------------------------------------
 * Legacy per-stage entry points == the reference's `gaussian` module functions.
 * ------------------------------------------------------------------------------------- */

/* global_culling — reference bindings.cpp:48, gaussian.cu:1338-1369 (kernel :1182-1336).
 * quat/scale are PRE-activated (splatter.py:519-524).  res_pos[n,3]=(x/z,y/z,|p_c|),
 * res_cov[n,2,2], mask[n] int64; outputs must be zero-filled by the caller (culled rows
 * are left untouched, like the reference). */
int gs_project_fwd(const float* pos, const float* quat, const float* scale, const float* rot,
                   const float* tran, int n, float near_plane, float half_width, float half_height,
                   float* res_pos, float* res_cov, int64_t* mask, gs_stream_t stream);

/* global_culling_backward — bindings.cpp:49, gaussian.cu:1578-1609 (kernel :1371-1576).
 * The projection Jacobian is treated as constant (no d cov2d / d pos), as in the reference. */
int gs_project_bwd(const float* pos, const float* quat, const float* scale, const float* rot,
                   const float* tran, const float* gradout_pos, const float* gradout_cov,
                   const int64_t* mask, int n, float* gradin_pos, float* gradin_quat,
                   float* gradin_scale, gs_stream_t stream);

/* calc_tile_list — bindings.cpp:44, gaussian.cu:254-335.  method 0 "dist" (:101-136),
 * 1 "prob" (:138-195), 2 "prob2" (:197-250).  tile_top/bottom/left/right[n_tiles] are only
 * read by methods 0/1.  tile_n_point[T] is incremented (may exceed max_per_tile; entries
 * beyond capacity are dropped, caller clamps — splatter.py:586). */
int gs_tile_list(const float* pos /*[n,3]*/, const float* cov /*[n,4]*/, int n,
                 const float* tile_top, const float* tile_bottom, const float* tile_left,
                 const float* tile_right, int n_tiles, int* tile_n_point, int* tile_gaussian_list,
                 int max_per_tile, float thresh, int method, float tile_length_x, float tile_length_y,
                 int n_tiles_x, int n_tiles_y, float leftmost, float topmost, gs_stream_t stream);

/* gather_gaussians — bindings.cpp:45, gaussian.cu:359-381. */
int gs_gather(const int* tile_n_point_accum /*[T+1]*/, const int* tile_gaussian_list /*[T,list_stride]*/,
              int n_tiles, int list_stride, int max_points_for_tile, int* gathered_list /*[M]*/,
              int* tile_ids_for_points /*[M]*/, gs_stream_t stream);

/* Scratch bytes needed by gs_draw_fwd / gs_draw_bwd for m tile-instances with colour width
 * d (3 = RGB, 27 = SH degree 2). */
size_t gs_draw_workspace_bytes(int m, int d);

/* draw — bindings.cpp:46, gaussian.cu:973-1043 (kernel :806-970).  Inputs are the already
 * (tile, depth)-sorted per-instance tensors pos[m,3], rgb[m,d], opa[m], cov[m,2,2] and
 * tile_n_point_accum[T+1]; image[Hp,Wp,3] is fully overwritten.  d = 3 or 27
 * (use_sh_coeff).  `weight_normalize` / `sigmoid` must be 0 (GS_ERR_UNSUPPORTED
 * otherwise: the reference never enables them, splatter.py:627, train.py:377).
 * rays_o/lefttop/vec_dx/vec_dy[3] are only read when d == 27 (splatter.py:305-321). */
int gs_draw_fwd(const float* pos, const float* rgb, const float* opa, const float* cov,
                const int* tile_n_point_accum, int m, int d, int width_padded, int height_padded,
                float focal_x, float focal_y, int weight_normalize, int sigmoid,
                const float* rays_o, const float* lefttop, const float* vec_dx, const float* vec_dy,
                float* image, void* workspace, size_t workspace_bytes, gs_stream_t stream);

/* draw_backward — bindings.cpp:47, gaussian.cu:1045-1129 (kernel :440-803).
 * grad_pos[m,3] (z column untouched), grad_rgb[m,d], grad_opa[m], grad_cov[m,2,2] receive the
 * per-instance gradients (every row of the listed columns is written). */
int gs_draw_bwd(const float* pos, const float* rgb, const float* opa, const float* cov,
                const int* tile_n_point_accum, int m, int d, int width_padded, int height_padded,
                float focal_x, float focal_y, int weight_normalize, int sigmoid,
                const float* rays_o, const float* lefttop, const float* vec_dx, const float* vec_dy,
                const float* image, const float* grad_image,
                float* grad_pos, float* grad_rgb, float* grad_opa, float* grad_cov,
                void* workspace, size_t workspace_bytes, gs_stream_t stream);

/* world2camera / world2camera_backward / jacobian — bindings.cpp:24-26,
 * gaussian.cu:71-76, :95-99, :41-47 (deprecated cudaculling=0 path). */
int gs_w2c_fwd(const float* pos, const float* rot, const float* tran, int n, float* res, gs_stream_t stream);
int gs_w2c_bwd(const float* grad_out, const float* rot, int n, float* grad_in, gs_stream_t stream);
int gs_jacobian(const float* pos_cam, int n, float* jac /*[n,3,3]*/, gs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Fused frame path (additive; replaces the PyTorch glue of splatter.py:513-655 and the
 * autograd glue around it): parameters -> image, grad_image -> parameter gradients.
 * ------------------------------------------------------------------------------------- */

typedef struct gs_ctx gs_ctx; /* owns device workspaces; one per (device, in-flight frame).  NOT thread-safe:
                                 use a context from one host thread / one stream at a time; it holds the
                                 intermediate state of its LAST forward only. */

typedef struct gs_camera {
  int width, height;          /* un-padded image size; render target is padded to x16 */
  float focal_x, focal_y;     /* principal point = image centre (splatter.py:499-500)  */
  float rot[9];               /* world->camera rotation, row-major                      */
  float tran[3];
  float near_plane;           /* splatter.py: near=0.3                                   */
  float tile_thresh;          /* bbox probability threshold, train.py:310 (0.05)         */
} gs_camera;

typedef struct gs_frame_info {
  int n_gaussians;            /* N                                                       */
  int n_visible;              /* Nc: passed near + 1.2x frustum cull                     */
  long long n_instances;      /* M : tile-instances binned                               */
  long long n_instances_eff;  /* M_eff: instances actually consumed before every pixel   */
                              /*        of their tile saturated (filled by forward)      */
  int width_padded, height_padded, n_tiles;
  int max_tile_count;
  long long n_instances_eff_bwd; /* instances the last BACKWARD consumed (sub-chunk granular); -1 if none ran */
} gs_frame_info;

/* scale_activation: 0 = abs()+1e-4 (splatter.py:521), 1 = trunc_exp (splatter.py:524). */
#define GS_SCALE_ABS 0
#define GS_SCALE_EXP 1

int gs_ctx_create(gs_ctx** out);           /* binds to the current CUDA device            */
/* Optional: workspaces of this context come from the caller's allocator instead of cudaMalloc / cudaFree
 * (which synchronise the stream when a buffer has to grow, e.g. after every densification).  `alloc` returns
 * device memory usable on `stream` (NULL = out of memory), `free_fn` releases it stream-ordered (the caller's
 * allocator must keep the block alive until the work already enqueued on that stream has finished - PyTorch's
 * caching allocator does; the torch shim installs it).  Pass NULL, NULL to go back to cudaMalloc. */
typedef void* (*gs_alloc_fn)(size_t bytes, void* user, gs_stream_t stream);
typedef void (*gs_free_fn)(void* ptr, void* user);
int gs_ctx_set_allocator(gs_ctx* ctx, gs_alloc_fn alloc, gs_free_fn free_fn, void* user);
void gs_ctx_destroy(gs_ctx* ctx);          /* frees workspaces (synchronises the device)  */

/* Raw parameters (splatter.py:399-406): pos[n,3], rgb[n,d] (logits if d==3, SH coefficients
 * channel-major [c*K+k] if d==27 (K = 9) or d==48 (K = 16)), opa[n] logits, quat[n,4] wxyz un-normalised, scale[n,3]
 * raw.  Writes image[Hp,Wp,3] (un-clamped, padded; black background) and, if non-NULL,
 * culling_mask[n] int64 (train.py:150).  Performs ONE host synchronisation on `stream`
 * (reads back the instance count M to size the sort).
 * SH colour is evaluated as set by gs_ctx_set_sh_eval (below): per pixel ray by default. */
int gs_render_forward(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                      const float* quat, const float* scale, int n, int d, int scale_activation,
                      const gs_camera* cam_host, float* image, int64_t* culling_mask,
                      gs_stream_t stream);

/* Backward of the most recent gs_render_forward on `ctx` (same parameter pointers).
 * grad_image[Hp,Wp,3]; `image` is the forward output.  Writes (overwrites, all n rows)
 * grad_pos[n,3], grad_rgb[n,d], grad_opa[n], grad_quat[n,4], grad_scale[n,3]:
 * gradients wrt the RAW parameters (activation backward included).  No synchronisation. */
int gs_render_backward(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                       const float* quat, const float* scale, const float* image,
                       const float* grad_image, float* grad_pos, float* grad_rgb, float* grad_opa,
                       float* grad_quat, float* grad_scale, gs_stream_t stream);

/* Same as gs_render_forward / gs_render_backward with the post-processing of reference
 * splatter.py:652-653 fused in: forward additionally writes image_final[height,width,3] =
 * centre crop of clamp(image_raw_padded, 0, 1); backward takes grad_final[height,width,3], the
 * gradient of that final image (clamp passes gradients where 0 <= raw <= 1; padding gets none). */
int gs_render_forward_final(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                            const float* quat, const float* scale, int n, int d, int scale_activation,
                            const gs_camera* cam_host, float* image_raw_padded, float* image_final,
                            int64_t* culling_mask, gs_stream_t stream);
int gs_render_backward_final(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                             const float* quat, const float* scale, const float* image_raw_padded,
                             const float* grad_final, float* grad_pos, float* grad_rgb, float* grad_opa,
                             float* grad_quat, float* grad_scale, gs_stream_t stream);

/* Depth and alpha maps and a background colour (additive; the calls above keep the reference's black
 * background and produce no maps).  Per pixel, with instances in (tile, depth) order, w_i = alpha_i T_i as in the
 * blend and T_f the transmittance after the last live instance (the 1e-4 early stop applies):
 *   image_c = sum_i w_i c_i,c + T_f background_c        (background = 0 is the plain image, bit for bit)
 *   depth   = sum_i w_i |p_c,i|                          accumulated, NOT normalised (expected depth = depth / alpha);
 *                                                        Euclidean camera distance (the sort key), not camera z
 *   alpha   = 1 - T_f
 * The background is a constant: it has no gradient.  gs_render_backward_aux takes the gradient of
 * (depth, alpha) too; the depth gradient reaches pos through p_c / |p_c|.
 *   background : HOST float[3]; NULL = black.  Must be finite (GS_ERR_INVALID_ARG otherwise).
 *   aux        : DEVICE [Hp,Wp,2] = (depth, alpha) per padded pixel; NULL = not written.
 *   aux_final  : DEVICE [height,width,2] centre crop of aux (not clamped); needs image_final.
 * Implemented for RGB and SH colour on the default (gather) path with the shipped kernels; the packed path
 * (gs_tune("gather", 0)), the two-pixel tensor-core SH backward (sh_tc bit 2) and non-default RGB blend knobs
 * return GS_ERR_UNSUPPORTED when a map or a background is requested.  SH colour evaluated per Gaussian
 * (gs_ctx_set_sh_eval) blends on the RGB kernels and follows the RGB rules here.  Same synchronisation and launch count as gs_render_forward_final; no workspace is allocated for
 * the maps (the buffers are the caller's). */
typedef struct gs_render_aux {
  const float* background;
  float* aux;
  float* aux_final;
} gs_render_aux;
/* image_final may be NULL (then aux_final must be NULL).  aux == NULL behaves like gs_render_forward[_final]. */
int gs_render_forward_aux(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                          const float* quat, const float* scale, int n, int d, int scale_activation,
                          const gs_camera* cam_host, float* image_raw_padded, float* image_final,
                          int64_t* culling_mask, const gs_render_aux* aux, gs_stream_t stream);
/* Backward of gs_render_forward_aux.  grad_image is [Hp,Wp,3] (grad_is_final == 0) or [height,width,3] of the
 * final image (grad_is_final != 0, as gs_render_backward_final).  aux = the forward's [Hp,Wp,2] buffer;
 * grad_aux = [Hp,Wp,2] or [height,width,2] (per grad_is_final) gradient of (depth, alpha); NULL = zero, which runs
 * the plain backward kernels.  grad_aux without an aux written by the forward is GS_ERR_INVALID_ARG.  The
 * data-parallel push (gs_ctx_set_grad_push) applies as in gs_render_backward. */
int gs_render_backward_aux(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                           const float* quat, const float* scale, const float* image_raw_padded,
                           const float* grad_image, int grad_is_final, const float* aux, const float* grad_aux,
                           float* grad_pos, float* grad_rgb, float* grad_opa, float* grad_quat, float* grad_scale,
                           gs_stream_t stream);

/* 2D Gaussian surfels (additive; Huang et al., "2D Gaussian Splatting", SIGGRAPH 2024).  The five parameter tensors
 * are those of gs_render_forward; only scale columns 0 and 1 are used (grad_scale[:, 2] is written as 0).  A surfel is
 * the flat disk spanned by u = s_u R r0 and v = s_v R r1 (r0, r1, r2: the columns of the normalised quaternion's
 * rotation, s the activated scale, R the camera rotation) at p_c = R pos + tran, evaluated exactly at the ray-disk
 * intersection (a, b): rho = a^2 + b^2, or 2DGS's screen filter rho = 2 |q - centre|^2 in px^2 where that is smaller
 * (then z = the centre's camera z).  alpha = min(0.99, sigmoid(opa) exp(-rho / 2)); alpha < 1/255 is skipped, and so is a
 * hit whose depth z is not beyond the near plane (a disk whose plane crosses the camera plane can be met behind the
 * camera just past its 3-sigma edge; without this the depth and distortion of that pixel would be negative or
 * infinite); the 1e-4 early stop applies.  Culling and the 1.2x frustum test are on the centre, the sort key is the centre's camera z,
 * and the tile rectangle is the box of the projected 3-sigma disk joined with a sqrt(2)/2 px box around the centre
 * (a disk that reaches the camera plane gets no instances).  Colour: RGB logits (d = 3), or SH of degree 2 / 3
 * (d = 27 / 48) evaluated once per Gaussian, which requires GS_SH_EVAL_GAUSSIAN on the context.
 * Per pixel, with instances in (tile, depth) order and w_i = alpha_i T_i:
 *   image = sum w c + T_f background;  maps (GS_SURFEL_MAP_CH floats per pixel, in this order):
 *   0 alpha = 1 - T_f;  1 depth = sum w z (camera z; expected depth = depth / alpha);  2 median = z of the last blended
 *   instance with T > 0.5 before it (0: none);  3 distortion = sum_i w_i sum_{j<i} w_j (m_i - m_j)^2 with
 *   m(z) = far / (far - near) (1 - near / z);  4..6 normal = sum w n, n = R r2 flipped to face the camera (camera frame;
 *   the world normal is rot^T normal);  7 zero.
 *   background : HOST float[3]; NULL = black.  Must be finite.  It has no gradient.
 *   maps       : DEVICE [Hp, Wp, GS_SURFEL_MAP_CH], 16-byte aligned; NULL: no maps (the kernels that skip them run).
 *   maps_final : DEVICE [height, width, GS_SURFEL_MAP_CH] centre crop of maps (not clamped), or NULL; needs maps and
 *                image_final.
 *   dist_near, dist_far : the distortion's m(z); 0 < dist_near < dist_far, finite.
 * s == NULL: black background, no maps.  The context keeps 16 bytes per padded pixel of workspace (48 with maps).
 * Refused before any launch, GS_ERR_UNSUPPORTED: SH colour evaluated per pixel (d != 3 without GS_SH_EVAL_GAUSSIAN); a
 * lens other than the image-centre pinhole; the 2-D or 3-D filter; densification statistics; a gradient push; the
 * packed path (gs_tune("gather", 0)).  GS_ERR_INVALID_ARG: bad arguments as gs_render_forward_aux, misaligned or
 * inconsistent map pointers, a bad dist_near / dist_far.  Batched views, feature maps and camera gradients have no
 * surfel entry; every existing backward after a surfel forward is GS_ERR_INVALID_ARG, and so is
 * gs_render_backward_surfel after any other forward.  gs_frame_stats, gs_frame_visible and the stage timer report
 * surfel frames as they report 3DGS ones. */
#define GS_SURFEL_MAP_CH 8
typedef struct gs_render_surfel {
  const float* background;
  float* maps;
  float* maps_final;
  float dist_near, dist_far;
} gs_render_surfel;
int gs_render_forward_surfel(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                             const float* scale, int n, int d, int scale_activation, const gs_camera* cam_host,
                             float* image_raw_padded, float* image_final, int64_t* culling_mask,
                             const gs_render_surfel* s /* nullable */, gs_stream_t stream);
/* Backward of gs_render_forward_surfel.  grad_image is [Hp,Wp,3] (grad_is_final == 0) or [height,width,3] of the final
 * image (grad_is_final != 0: clamp mask from image_raw_padded, zero outside the crop).  grad_maps: [Hp,Wp,8] or
 * [height,width,8] (per grad_is_final; maps are not clamped, only the crop masks them), 16-byte aligned, or NULL (zero
 * map gradients, which runs the kernels without the map terms); channel 7 is ignored.  grad_maps needs a forward that
 * wrote maps (GS_ERR_INVALID_ARG).  The median's gradient reaches only the median instance's z.  Deterministic (fixed
 * order sums, no atomics).  Refused before any launch: no surfel forward on ctx (GS_ERR_INVALID_ARG after a 3DGS
 * forward, GS_ERR_NO_FORWARD without one), a gradient push or densification statistics configured
 * (GS_ERR_UNSUPPORTED). */
int gs_render_backward_surfel(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                              const float* scale, const float* image_raw_padded, const float* grad_image,
                              int grad_is_final, const float* grad_maps, float* grad_pos, float* grad_rgb,
                              float* grad_opa, float* grad_quat, float* grad_scale, gs_stream_t stream);

/* gs_render_backward_aux plus the gradient with respect to the camera of the last forward, p_c = rot p + tran (rot
 * used as given, not re-orthonormalised): grad_cam (DEVICE float[12]) receives dL/drot row-major [9], then dL/dtran [3].
 * It follows the semantics of pos: the projection Jacobian is constant, rot stays live in the 2-D covariance
 * (J rot) Sigma (J rot)^T, culling / tile rectangles / sort order have no gradient; depth gradients (grad_aux) and the
 * view direction of per-Gaussian SH (GS_SH_EVAL_GAUSSIAN) reach the pose too.  The five parameter gradients are all
 * NULL (camera only: nothing else is written) or all non-NULL (then equal to gs_render_backward_aux's); a mix, a NULL
 * grad_cam or ctx is GS_ERR_INVALID_ARG.  grad_cam is always written (zeros for an empty or fully culled frame) and
 * is bit-deterministic (fixed-order sums, fp64 across CTAs; no atomics).  RGB and per-Gaussian SH frames only: a
 * per-pixel SH frame, or a context with a gradient push configured, is GS_ERR_UNSUPPORTED.  One more launch than
 * gs_render_backward_aux; no synchronisation; a workspace of 48 bytes per 256 Gaussians is kept by the context. */
int gs_render_backward_cam(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                           const float* scale, const float* image_raw_padded, const float* grad_image,
                           int grad_is_final, const float* aux, const float* grad_aux,
                           float* grad_pos, float* grad_rgb, float* grad_opa, float* grad_quat, float* grad_scale,
                           float* grad_cam /* DEVICE [12]: dL/drot row-major [9], then dL/dtran [3] */,
                           gs_stream_t stream);

/* Feature maps (additive): per-Gaussian raw float32 features feat[n, f] (no activation), f = 8, 16 or 32, blended in
 * the same pass as the image with the image's weights w_i = alpha_i T_i:
 *   feature_k = sum_i w_i f_i,k     composited over zero (the background applies to the image only; the expected
 *                                   feature is feature / alpha).  Features are not clamped.
 * Another width: pad with zero channels.  Image, depth and alpha are bit-identical to gs_render_forward_aux's with the
 * same arguments, and the launch count is the same.
 *   feat      : DEVICE [n, f], 16-byte aligned.
 *   map       : DEVICE [Hp, Wp, f], 16-byte aligned; required (the feature backward reads it).
 *   map_final : DEVICE [height, width, f] centre crop of map, or NULL; needs image_final.
 * Frames that blend on the RGB kernels of the gather path only: RGB colour and SH with GS_SH_EVAL_GAUSSIAN, with or
 * without maps / background (aux), under any 2-D filter.  Refused before any launch: f not 8 / 16 / 32, a NULL or
 * misaligned pointer (GS_ERR_INVALID_ARG); a per-pixel SH frame, the packed path (gs_tune("gather", 0))
 * (GS_ERR_UNSUPPORTED). */
typedef struct gs_render_feat {
  int f;
  const float* feat;
  float* map;
  float* map_final;
} gs_render_feat;
int gs_render_forward_feat(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                           const float* scale, int n, int d, int scale_activation, const gs_camera* cam_host,
                           float* image_raw_padded, float* image_final, int64_t* culling_mask,
                           const gs_render_aux* aux /* nullable */, const gs_render_feat* feat, gs_stream_t stream);
/* Backward of gs_render_forward_feat: gs_render_backward_aux's arguments plus the feature terms.  grad_map is
 * [Hp, Wp, f] or [height, width, f] (per grad_is_final; only the crop masks it), 16-byte aligned; NULL = zero, which
 * runs the plain or aux backward kernels and zero-fills grad_feat.  grad_feat (DEVICE [n, f]) receives
 * dL/dfeat = sum_p w_p,i g_F(p), bit-deterministic; the other gradients gain the feature loss's terms through alpha.
 * feat must be the forward's pointer and map the forward's buffer.  After a feature forward the other backward entries
 * (plain, final, aux, cam) work unchanged and treat the feature gradient as zero.  Densification statistics
 * (gs_ctx_set_densify_stats, grad2d) include the feature loss.
 * GS_ERR_INVALID_ARG: the forward blended no features, feat differs from the forward's, NULL grad_feat (n > 0),
 * grad_map without map, misaligned map / grad_map.  GS_ERR_UNSUPPORTED, before any launch, with a non-NULL grad_map:
 * absgrad statistics set; a gradient push configured (grad_feat is not part of the bucket).
 * One more launch than gs_render_backward_aux when grad_map is set; the context keeps M * f * 4 bytes of workspace. */
int gs_render_backward_feat(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                            const float* scale, const float* image_raw_padded, const float* grad_image,
                            int grad_is_final, const float* aux, const float* grad_aux, const float* feat,
                            const float* map, const float* grad_map, float* grad_pos, float* grad_rgb,
                            float* grad_opa, float* grad_quat, float* grad_scale, float* grad_feat,
                            gs_stream_t stream);

/* A batch of B camera views rendered as one frame.  Per view, the semantics are exactly gs_render_forward_aux /
 * gs_render_backward_aux with cams_host[v]; the background is shared by all views, and the parameter gradients are the
 * SUM over the views (divide the loss by B for a mean).  The frame works on the B n (view, Gaussian) pairs j = v n + i
 * and draws the views stacked vertically: image_raw_padded [B,Hp,Wp,3] (and aux [B,Hp,Wp,2]) is byte for byte the
 * [B Hp, Wp, .] tall image; image_final [B,height,width,3] and aux_final [B,height,width,2] crop each view on its own;
 * culling_mask is [B,n].  One host synchronisation and the launch count of one gs_render_forward_aux +
 * gs_render_backward_aux frame, whatever B.  The context settings sh_eval, filter2d, densification statistics (added
 * view by view in view order) and timing apply; gs_frame_stats / gs_frame_instances / gs_frame_sorted /
 * gs_frame_tile_consumed / gs_frame_stage_ms report the batch (totals, B T tiles, pair indices j; width_padded /
 * height_padded are one view's).  With n_views == 1 the gradients are gs_render_backward_aux's bit for bit.
 * Refused before any launch:
 *   GS_ERR_INVALID_ARG: a null ctx or cams; n_views outside 1 .. GS_MAX_VIEWS; views that differ in width, height,
 *     near_plane or tile_thresh; B n >= 2^31 or B Hp / 16 > 65535; a bad camera or pointer as in gs_render_forward_aux;
 *     more than 2^31 instances (as in gs_render_forward); gs_render_backward_batch after a single-view forward, and
 *     every single-view backward entry after gs_render_forward_batch.
 *   GS_ERR_UNSUPPORTED: SH colour evaluated per pixel; the packed path (gs_tune("gather", 0)); RGB blend knobs other
 *     than the shipped ones (live-pixel repack on); a gradient push configured (gs_ctx_set_grad_push). */
#define GS_MAX_VIEWS 64
int gs_render_forward_batch(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                            const float* scale, int n, int d, int scale_activation, int n_views,
                            const gs_camera* cams_host /* [n_views] */, float* image_raw_padded /* [B,Hp,Wp,3] */,
                            float* image_final /* [B,H,W,3] | NULL */, int64_t* culling_mask /* [B,n] | NULL */,
                            const gs_render_aux* aux /* nullable */, gs_stream_t stream);
int gs_render_backward_batch(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa, const float* quat,
                             const float* scale, const float* image_raw_padded, const float* grad_image,
                             int grad_is_final, const float* aux, const float* grad_aux, float* grad_pos,
                             float* grad_rgb, float* grad_opa, float* grad_quat, float* grad_scale, gs_stream_t stream);
/* gs_render_backward_batch plus each view's camera gradient: per view v, gs_render_backward_cam's semantics with view
 * v's camera cams_host[v] of the last gs_render_forward_batch (projection Jacobian detached, rot used as given, depth
 * gradients and the per-Gaussian SH view direction reach the pose, view v's 2-D filter).  grad_cams (DEVICE
 * float[B][12]) receives per view dL/drot row-major [9], then dL/dtran [3]; it is always written (zeros for a view
 * that bins nothing) and bit-deterministic (fixed-order sums per CTA and view, fp64 across CTAs; no atomics).  The five
 * parameter gradients are all NULL (camera only: nothing else is written, the densification statistics are left
 * alone) or all non-NULL (then equal to gs_render_backward_batch's, statistics included).  With n_views == 1 the
 * single-view kernels run, so grad_cams[0] and the parameter gradients are gs_render_backward_cam's bit for bit.
 * Refused before any launch: a NULL grad_cams or ctx, or a mixed set of parameter gradients (GS_ERR_INVALID_ARG,
 * checked before the context is read); no forward (GS_ERR_NO_FORWARD); a single-view last forward
 * (GS_ERR_INVALID_ARG); a gradient push configured, or a batch the batched blend cannot run (GS_ERR_UNSUPPORTED).
 * gs_render_backward_cam after gs_render_forward_batch stays refused.  One launch more than gs_render_backward_batch,
 * whatever B; no synchronisation; the context keeps B * 48 bytes of workspace per 256 Gaussians. */
int gs_render_backward_batch_cam(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                                 const float* quat, const float* scale, const float* image_raw_padded,
                                 const float* grad_image, int grad_is_final, const float* aux,
                                 const float* grad_aux, float* grad_pos, float* grad_rgb, float* grad_opa,
                                 float* grad_quat, float* grad_scale,
                                 float* grad_cams /* DEVICE [B][12]: per view dL/drot row-major [9], dL/dtran [3] */,
                                 gs_stream_t stream);

/* Where the SH colour (d == 27 / 48) is evaluated.  Two colour MODELS, not two speeds of one: the same coefficients
 * render differently.
 *   GS_SH_EVAL_PIXEL    (default; the reference): the basis is evaluated per pixel, along the pixel's world-space ray,
 *                       inside the blend:  c_c(pixel) = sigmoid( sum_k Y_k(ray dir) rgb[c*K+k] ).
 *   GS_SH_EVAL_GAUSSIAN (the usual 3D Gaussian Splatting model): once per Gaussian, along the world-space direction
 *                       from the camera centre C = -R^T t to the mean, dir = (pos - C) / |pos - C|, in the projection;
 *                       c_c = sigmoid( sum_k Y_k(dir) rgb[c*K+k] ) then blends like an RGB colour.  The backward
 *                       includes the direction term: dL/dpos gains (I - dir dir^T) / |pos - C| dL/ddir.
 * The setting belongs to the context and applies to the forwards that follow; a backward always uses the mode of its
 * forward.  Frames with d == 3 ignore it.  In per-Gaussian mode the frame runs the RGB blend kernels, so the aux
 * calls (depth / alpha / background) and the packed path (gs_tune("gather", 0)) behave as for RGB, the per-pixel SH
 * knobs (gs_tune("sh_tc", ...)) do not apply, and the gradients keep the parameter layout grad_rgb[n,d].
 * Null ctx or an unknown mode: GS_ERR_INVALID_ARG. */
#define GS_SH_EVAL_PIXEL 0
#define GS_SH_EVAL_GAUSSIAN 1
int gs_ctx_set_sh_eval(gs_ctx* ctx, int mode);

/* Screen-space 2-D low-pass filter of the projected Gaussians (additive; default NONE, the reference, which has none).
 * With a filter variance s px^2 and the pixel pitch 1/fx by 1/fy, the 2-D covariance Sigma = (a, b, c, d) of every
 * Gaussian becomes Sigma' = (a + s/fx^2, b, c, d + s/fy^2):
 *   GS_FILTER2D_NONE      : no filter (the variance is kept but not used).
 *   GS_FILTER2D_DILATE    : the original 3D Gaussian Splatting dilation (s = 0.3): the conic, the det <= 0 test and the
 *                           tile rectangle come from Sigma'.  A Gaussian below a pixel no longer thins to a needle, and
 *                           its screen-space integral grows by sqrt(det'/det).
 *   GS_FILTER2D_ANTIALIAS : the Mip-Splatting 2-D filter (gsplat "antialiased"): as DILATE, and the opacity is scaled by
 *                           sqrt(det/det'), which keeps every Gaussian's screen-space integral unchanged.  A Gaussian
 *                           with det <= 0 gets no instances (its culling_mask entry still reports the frustum test).
 * Backward: Sigma' - Sigma is a constant; the compensation's gradient reaches the 2-D covariance and from there the
 * parameters and (gs_render_backward_cam) the camera; the opacity-logit gradient is unchanged.
 * The setting belongs to the context and applies to every fused forward that follows (plain, final, aux, the packed
 * path and gs_render_forward_backward_host); a backward (plain, final, aux, cam, with or without a gradient push) always
 * uses the filter of its forward.  Depth, sort order, colour and culling are unchanged.  No launch or synchronisation
 * is added.  The legacy per-stage API is not affected.  A scene trained under one mode renders differently under
 * another: train and render with the same one.
 * Null ctx, an unknown mode, or a variance that is not finite and > 0 (whatever the mode): GS_ERR_INVALID_ARG. */
#define GS_FILTER2D_NONE 0
#define GS_FILTER2D_DILATE 1
#define GS_FILTER2D_ANTIALIAS 2
int gs_ctx_set_filter2d(gs_ctx* ctx, int mode, float variance_px2);

/* 3-D smoothing filter of the Gaussians (additive; default off, the reference, which has none): Mip-Splatting's 3D
 * filter, which bounds every Gaussian's 3-D scale from below by the finest sampling interval any training view has at
 * it, so that a scene rendered closer or at a longer focal length than it was trained shows no needle-like artefacts.
 * With filter3d[i] = f_i >= 0 (world units) and the activated scale s (|raw| + 1e-4 or exp(raw)), every fused frame
 * uses
 *   s'_k = sqrt(s_k^2 + f_i^2)                 for the 3-D covariance (the conic, the det <= 0 test, the tile
 *                                              rectangle and the 2-D filter, if one is set, follow it);
 *   sigma' = sigma prod_k s_k / s'_k           the opacity, which keeps sigma sqrt(det Sigma3), the 3-D integral.
 * A row with f_i == 0 takes the unfiltered arithmetic by selection: a zero filter renders, and differentiates, the bits
 * of a frame without one.  A scale that underflows to 0 gets opacity 0 and zero gradients.  Backward: filter3d is a
 * constant (no gradient); dL/ds_k = dL/ds'_k s_k / s'_k + dL/dl2o f^2 / (ln 2 s_k (s_k^2 + f^2)) joins the raw-scale
 * chain; the opacity-logit gradient is unchanged; the camera gradient uses s' (f does not depend on the camera).
 * gs_ctx_set_filter3d: a context setting, like gs_ctx_set_densify_stats: the DEVICE pointer [n] is the caller's and
 * must stay alive while it is set; NULL turns the filter off.  It applies to every fused forward that follows (plain,
 * final, aux, feat, batch, the packed path, gs_render_forward_backward_host); a forward records the pointer and its
 * backward (plain, final, aux, cam, batch, batch cam, feat, with or without a gradient push, the densification
 * statistics' max_radius) uses the recorded one.  A forward whose n differs from the filter's n is refused
 * (GS_ERR_INVALID_ARG) before any launch.  No launch or synchronisation is added.  Null ctx or n < 0:
 * GS_ERR_INVALID_ARG. */
int gs_ctx_set_filter3d(gs_ctx* ctx, const float* filter3d /* DEVICE [n]; NULL: off */, int n);
/* The filter of Mip-Splatting's sampling rate over the views cams_host[n_cams] (e.g. all training views), into
 * filter3d[n] (DEVICE):  view c (W, H, fx, fy, R, t, near = near_plane) sees Gaussian i when, with p_c = R pos_i + t,
 * u = fx x / z + W / 2 and w = fy y / z + H / 2:  z > near, -margin W <= u <= (1 + margin) W and
 * -margin H <= w <= (1 + margin) H.  nu_i = max over the views that see i of fx / z (the maximal sampling rate), and
 * filter3d[i] = sqrt(variance) / nu_i.  A Gaussian no view sees gets the largest filter, that of the smallest nu over
 * the seen ones; none seen at all: 0 everywhere.  Mip-Splatting's defaults: margin 0.15, variance 0.2.  The rates are
 * fp64 divisions and max / min are order-independent: the same bits on every call and for any order of the views, so
 * data-parallel replicas agree without an exchange.  Two launches when n > 0, no host synchronisation; the context
 * keeps 112 bytes of device workspace and pinned staging per view.  Refused before any launch (GS_ERR_INVALID_ARG):
 * a null ctx or cams_host, a null pos or filter3d with n > 0; n < 0 or n_cams < 1; a variance that is not finite and > 0; a margin that is not finite and
 * >= 0; a camera whose size or focal lengths are not positive and finite, or whose near_plane is not finite and >= 0. */
int gs_filter3d_compute(gs_ctx* ctx, const float* pos /* [n,3] */, int n, const gs_camera* cams_host, int n_cams,
                        float margin, float variance, float* filter3d /* [n] */, gs_stream_t stream);

/* COLMAP camera intrinsics on the fused frame path (additive; default off: every camera is an undistorted pinhole whose
 * principal point is the image centre, as in the reference).  With (a, b) = (x/z, y/z) and rho = |(a, b)|, a lens maps
 * (a, b) to (a_d, b_d) by COLMAP's formulas:
 *   GS_LENS_PINHOLE : (a_d, b_d) = (a, b)                                               (k unused)
 *   GS_LENS_OPENCV  : a_d = a rad + 2 p1 a b + p2 (rho^2 + 2 a^2), b_d = b rad + p1 (rho^2 + 2 b^2) + 2 p2 a b,
 *                     rad = 1 + k1 rho^2 + k2 rho^4                                     (k = k1, k2, p1, p2)
 *   GS_LENS_FISHEYE : (a_d, b_d) = (theta_d / rho) (a, b), theta = atan(rho),
 *                     theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8)  (COLMAP OPENCV_FISHEYE)
 * and pixel u of the image (centre u + 0.5) sits at u + 0.5 = fx a_d + cx, v + 0.5 = fy b_d + cy, as COLMAP projects.
 * The 2-D covariance is J_D (J Sigma3 J^T) J_D^T with J_D the lens map's Jacobian.  Backward: the mean chain is live
 * through the lens; J_D, like the pinhole Jacobian, is detached in the covariance; the camera gradient uses J_D J;
 * depth, the SH view direction, the 2-D and 3-D filters and the opacity are unchanged; the intrinsics get no gradient.
 * Culling: z > near, the 1.2x frustum test on the stored (distorted, principal-point shifted) mean, and rho < rho_max,
 * where the radial polynomial folds back: OPENCV the smallest rho > 0 with 1 + 3 k1 rho^2 + 5 k2 rho^4 <= 0, FISHEYE
 * tan of the smallest theta in (0, pi/2) with d theta_d / d theta <= 0 (none: no limit).  A Gaussian past it gets no
 * instances and its culling_mask entry reports it culled.  Fields of view beyond 180 degrees are not supported.
 * gs_ctx_set_lens: a context setting, like gs_ctx_set_filter2d: it applies to every fused forward that follows (plain,
 * final, aux, feat, batch, the packed path, gs_render_forward_backward_host), and a backward (plain, final, aux, cam,
 * batch, batch cam, feat, the densification statistics' max_radius) uses the lenses its forward recorded.  n == 1: one
 * lens for every view; n == B: lens v for view v of a batched frame; any other n at a forward is GS_ERR_INVALID_ARG
 * before any launch.  A PINHOLE lens at exactly (W/2, H/2) in every view runs the kernels of a frame without a lens, so
 * it renders and differentiates the same bits.  No launch or synchronisation is added.
 * Refused:  gs_ctx_set_lens (GS_ERR_INVALID_ARG): a null ctx; n < 0 or n > GS_MAX_VIEWS; NULL lenses with n > 0; an
 * unknown model; a cx, cy or k that is not finite.  Before any launch (GS_ERR_UNSUPPORTED): a forward of SH colour
 * evaluated per pixel with any lens but a pinhole (a principal point alone is supported: its rays shift with it); a
 * backward with a gradient push configured (train data-parallel through an all-reduce instead).
 * gs_filter3d_compute uses the context's lenses too (n == 1 or n == n_cams, GS_ERR_INVALID_ARG otherwise): view c sees
 * a Gaussian when z > near, rho < rho_max and the distorted pixel position (fx a_d + cx, fy b_d + cy) lies inside the
 * widened image; the rate stays fx / z for PINHOLE and OPENCV (Mip-Splatting's rate, which ignores distortion) and is
 * fx max(theta_d'(theta), theta_d(theta) / sin theta) / |p_c| for FISHEYE (the larger of the radial and tangential
 * magnifications; fx / z on the axis), in fp64.  The legacy per-stage API is not affected. */
#define GS_LENS_PINHOLE 0
#define GS_LENS_OPENCV 1  /* k = k1, k2, p1, p2 */
#define GS_LENS_FISHEYE 2 /* k = k1, k2, k3, k4 (COLMAP OPENCV_FISHEYE) */
typedef struct gs_lens {
  int model;
  float cx, cy; /* principal point in pixels, COLMAP convention (the image centre is (W/2, H/2)) */
  float k[4];
} gs_lens;
int gs_ctx_set_lens(gs_ctx* ctx, const gs_lens* lenses /* HOST [n]; NULL: off */, int n);

/* Screen-space densification statistics (additive; default off).  While a context has them set, every backward that
 * computes parameter gradients (plain, final, aux, cam with parameter gradients, gs_render_forward_backward_host, with
 * or without a gradient push) accumulates, for every Gaussian i with count[i] > 0 in its forward (i.e. binned into at
 * least one tile):
 *   grad2d[i]    += |(gx W / (2 fx), gy H / (2 fy))|: (gx, gy) = dL/d(mean2d) in normalised image-plane units, the sum
 *                   of Gaussian i's per-instance gradients; W, H the un-padded image size, fx, fy the focal lengths in
 *                   pixels.  The scale gives the NDC convention of 3DGS's viewspace_points.grad and gsplat, so their
 *                   threshold 0.0002 means the same here for the same loss normalisation.
 *   absgrad[i]   += |(Ax W / (2 fx), Ay H / (2 fy))| with Ax = sum_p |g_x,p|, Ay = sum_p |g_y,p| over the pixels' own
 *                   contributions to (gx, gy) (AbsGS; gsplat absgrad=True), depth / alpha terms included.  NULL: off.
 *   count[i]     += 1 (the 3DGS denominator: the views in which the Gaussian got an instance).
 *   max_radius[i] = max(max_radius[i], ceil(3 sqrt(lambda_max))), lambda_max the largest eigenvalue in px^2 of the
 *                   2-D covariance the forward binned (after the 2-D filter when one is set); 3DGS's radius without its
 *                   0.1 floor.
 * A camera-only gs_render_backward_cam leaves them alone.  The caller zeroes the buffers (all device, [n]) and keeps
 * them alive while they are set; results are bit-deterministic (no atomics).  One launch per backward when n > 0,
 * timed in stage 7 of gs_frame_stage_ms.  The backward refuses, before any launch: s->n != the forward's n
 * (GS_ERR_INVALID_ARG); absgrad on a frame the shipped RGB blend backward of the gather path does not run (per-pixel SH
 * colour, the packed path, other backward blend knobs: GS_ERR_UNSUPPORTED).
 * gs_ctx_set_densify_stats: NULL turns them off; a null ctx, n < 0, or a NULL grad2d / count / max_radius with n > 0
 * is GS_ERR_INVALID_ARG.  The pointers are the caller's, as with gs_ctx_set_grad_push. */
typedef struct gs_densify_stats {
  int n;               /* must equal the n of the frame whose backward runs */
  float* grad2d;       /* [n] */
  float* absgrad;      /* [n] or NULL */
  int* count;          /* [n] */
  float* max_radius;   /* [n] */
} gs_densify_stats;
int gs_ctx_set_densify_stats(gs_ctx* ctx, const gs_densify_stats* s /* NULL: off */);

/* Per-stage device timing with CUDA events recorded on the frame's stream (off by default).
 * gs_frame_stage_ms fills out[GS_N_STAGES] with the milliseconds of the last frame's stages:
 * 0 project, 1 depth sort of Gaussians + scan + M readback, 2 key emit, 3 tile-id radix sort,
 * 4 range + pack, 5 blend forward,
 * 6 blend backward, 7 project backward (with gs_render_backward_cam: both camera-gradient kernels)
 * (-1 where not available).  Synchronises `stream`. */
#define GS_N_STAGES 8
int gs_ctx_set_timing(gs_ctx* ctx, int enable);
int gs_frame_stage_ms(gs_ctx* ctx, float* out_host, gs_stream_t stream);

/* M (tile-instances) of the last forward on ctx, -1 if none; no synchronisation (the forward
 * already read it back). */
long long gs_frame_instances(gs_ctx* ctx);

/* Statistics of the last forward on ctx (host struct; synchronises `stream` for M_eff). */
int gs_frame_stats(gs_ctx* ctx, gs_frame_info* out_host, gs_stream_t stream);

/* Exposes the last frame's sorted instance list for parity tests: copies
 * min(capacity, M) entries of the sorted Gaussian ids into gauss_idx (device int32) and
 * T+1 entries into tile_accum (device int32).  Either pointer may be NULL. */
int gs_frame_sorted(gs_ctx* ctx, int* gauss_idx, long long capacity, int* tile_accum, gs_stream_t stream);

/* Per-tile consumed instance counts of the last forward (device int32 [T]): tile t's blend stopped
 * after tile_consumed[t] of its tile_accum[t+1]-tile_accum[t] instances because every pixel had
 * saturated (M_eff = their sum).  For parity tests / roofline accounting. */
int gs_frame_tile_consumed(gs_ctx* ctx, int* tile_consumed, gs_stream_t stream);

/* Which Gaussians the last forward on ctx binned: visible[i] (DEVICE uint8 [n]) = 1 if Gaussian i got at least one
 * tile instance (for a batched forward: in any of its views), else 0.  accumulate != 0 ORs into what visible holds
 * (several frames before one optimizer step); 0 overwrites.  This is "binned", the rule the projection backward, the
 * feature gradient and the densification statistics (count += 1) use for "took part", not the frustum test that
 * culling_mask reports: a Gaussian can pass the cull and get no tile (a non-positive determinant, an ANTIALIAS
 * det <= 0).  A Gaussian that is not visible has an exactly zero gradient row.  Valid after every forward entry, on
 * the gather and the packed path, for every colour model.  One launch when n > 0, no synchronisation, no atomics.
 * GS_ERR_INVALID_ARG: a null ctx or pointer, no forward on ctx yet, n different from the last forward's. */
int gs_frame_visible(gs_ctx* ctx, unsigned char* visible, int n, int accumulate, gs_stream_t stream);

/* Blend-weight scores of the last forward on ctx (additive; for pruning a scene by contribution): for every Gaussian
 * i, with w_{i,p} = alpha_{i,p} T_{i,p} the weight the gather forward blended Gaussian i's colour with at pixel p (0
 * once T_{i,p} <= GS_T_STOP: the forward's alpha, T recurrence, instance order and early stop), over the pixels p of
 * the rendered image (the crop, not the padding) and, for a batched forward, over its views v:
 *   weight_sum[i] += sum_v sum_p w_{i,p}                        (LightGaussian / Mini-Splatting's score)
 *   weight_max[i]  = max(weight_max[i], max_v max_p w_{i,p})    (RadSplat's score)
 * The weights depend on geometry and opacity only, so RGB, per-Gaussian and per-pixel SH, feature frames, both 2-D
 * filters, the 3-D filter and lenses are all covered.  The caller zeroes the buffers (all DEVICE float32 [n]); a call
 * adds, so two calls after one forward add twice.  A batched forward adds view by view: B views give the bits of B
 * single-view forwards each followed by a call, in view order.  Bit-deterministic: one thread per Gaussian sums its
 * rows in row order, no atomics.
 * Valid after gs_render_forward, _final, _aux, _feat, _batch and gs_render_forward_backward_host; reads only what
 * that forward left in ctx and writes nothing a backward reads (forward, scores, backward gives the gradients and
 * densification statistics of forward, backward).  The per-instance rows (12 bytes per tile instance) live in a
 * workspace of their own, grown on the first call.  Two launches when n > 0, no synchronisation.
 * Refused before any launch: a null ctx, s, weight_sum or weight_max, no forward on ctx yet, s->n different from the
 * forward's n (GS_ERR_INVALID_ARG); a surfel forward, a packed-path forward (gs_tune("gather", 0)) (GS_ERR_UNSUPPORTED).
 * The struct has no typedef: its tag is also the entry's name. */
struct gs_frame_scores {
  int n;               /* must equal the n of the last forward */
  float* weight_sum;   /* [n] */
  float* weight_max;   /* [n] */
};
int gs_frame_scores(gs_ctx* ctx, const struct gs_frame_scores* s, gs_stream_t stream);

/* End-to-end convenience with HOST buffers (bench `e2e` leg and plain-C callers): copies
 * the camera + grad_image from host, runs forward + backward on device-resident parameters,
 * copies the padded image back.  Host buffers should be pinned.  Synchronises. */
int gs_render_forward_backward_host(gs_ctx* ctx, const float* pos, const float* rgb, const float* opa,
                                    const float* quat, const float* scale, int n, int d,
                                    int scale_activation, const gs_camera* cam_host,
                                    const float* grad_image_host, float* image_host,
                                    float* grad_pos, float* grad_rgb, float* grad_opa,
                                    float* grad_quat, float* grad_scale, gs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Next-row widening (SURVEY.md §8 f-2): fused Adam over the flat parameter / gradient buckets.
 * Replaces torch.optim.Adam over the five parameter groups of reference train.py:56-64 (same
 * update as torch's single-tensor Adam, no weight decay / amsgrad).  `param`, `grad`, `exp_avg`,
 * `exp_avg_sq` are flat device buffers of n floats (n % 4 == 0) split into n_seg (<= 8) segments
 * ending at seg_end_host[s] (ascending multiples of 4) with learning rate lr_host[s]; `step` is
 * the 1-based step count used for the bias corrections. */
int gs_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                 const long long* seg_end_host, const float* lr_host, int n_seg, float beta1, float beta2,
                 float eps, int step, gs_stream_t stream);

/* Adam on the rows of the visible Gaussians only (the "sparse Adam" of 3DGS, gsplat's SelectiveAdam): a different
 * optimizer from gs_adam_step, not a faster route to its numbers.  A Gaussian that is not visible is frozen: its
 * parameters and both moments keep their bits (dense Adam would let it drift on its momentum and decay the moments).
 * The flat buffers are those of gs_adam_step; segment s is the row-major [n_rows, seg_width_host[s]] array that starts
 * at float seg_start_host[s] (a multiple of 4) and has learning rate lr_host[s].  For every i with visible[i] != 0
 * (DEVICE uint8 [n_rows], e.g. from gs_frame_visible), every float of row i of every segment gets exactly
 * gs_adam_step's update: the same rounded operations, the same bias corrections from the global `step` (not from a
 * per-row count).  Nothing else in param / exp_avg / exp_avg_sq is read or written, the pad floats between segments
 * included; DRAM traffic follows the number of visible rows.  Bit-deterministic (no atomics).  One launch, no
 * synchronisation; n_rows == 0 returns 0 without a launch.
 * GS_ERR_INVALID_ARG, before any launch: step < 1; n_seg outside 1 .. 8; n_flat negative or not a multiple of 4;
 * n_rows < 0; a width outside 1 .. 2^24; starts that are not ascending multiples of 4; segments that overlap or end
 * beyond n_flat; a NULL host array; a NULL device buffer or mask with n_rows > 0. */
int gs_adam_step_visible(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n_flat,
                         const long long* seg_start_host, const int* seg_width_host, const float* lr_host, int n_seg,
                         int n_rows, const unsigned char* visible, float beta1, float beta2, float eps, int step,
                         gs_stream_t stream);

/* Densification on the device (SURVEY.md §8 f-2; reference splatter.py:122-228 `adaptive_control`, called
 * from train.py:156-172): prune Gaussians with opacity logit <= opa_logit_min or activated-scale norm >=
 * delete_thresh; of the kept ones whose aggregated |grad| (max or mean over xyz) exceeds grad_thresh, CLONE the
 * small ones (norm <= tau; the copy is moved by -grad * clone_dt) and SPLIT the large ones (scale / 1.6, or
 * - log 1.6 for the exp activation; both halves re-positioned at pos + R (s_act * z), z ~ N(0, I) supplied by the
 * caller so that data-parallel replicas draw identical samples).
 *   gs_densify_plan : code[n+1] (bit0 keep, bit1 clone, bit2 split) and dst[3][n+1] = exclusive scans of the
 *                     three flags (dst[b][n] = totals: n_keep, n_clone, n_split).  No synchronisation.
 *   gs_densify_apply: writes the n_keep + n_clone + n_split rows of the new parameter arrays, laid out like the
 *                     reference's torch.cat: kept (in order), clones (in order), second split samples (in order).
 *                     normals: [2][n_split][3].  Output arrays are caller-allocated.  grad == NULL: clones are exact
 *                     copies (3DGS; the plan of gs_densify_plan_stats). */
size_t gs_densify_workspace_bytes(int n);
int gs_densify_plan(const float* opa, const float* scale, const float* grad, int n, int scale_activation,
                    float opa_logit_min, float delete_thresh, float grad_thresh, int grad_agg_max, float tau,
                    int use_clone, int use_split, unsigned char* code, int* dst, void* workspace,
                    size_t workspace_bytes, gs_stream_t stream);
int gs_densify_apply(const float* pos, const float* rgb, const float* opa, const float* quat, const float* scale,
                     int n, int d, const unsigned char* code, const int* dst, const float* grad, float clone_dt,
                     const float* normals, int n_keep, int n_clone, int n_split, int scale_activation,
                     float* out_pos, float* out_rgb, float* out_opa, float* out_quat, float* out_scale,
                     gs_stream_t stream);
/* Another per-Gaussian row tensor src[n, w] (e.g. features) laid out like gs_densify_apply's outputs for the same
 * plan: kept rows, clones, second split samples; both split halves and clones are exact copies.  out: caller-allocated
 * [n_keep + n_clone + n_split, w].  One launch when n > 0; no synchronisation. */
int gs_densify_apply_rows(const float* src, int n, int w, const unsigned char* code, const int* dst, int n_keep,
                          int n_clone, int n_split, float* out, gs_stream_t stream);
/* gs_densify_plan from screen-space statistics (gs_ctx_set_densify_stats), as 3DGS scores them: a kept Gaussian
 * densifies when accum[i] / max(count[i], 1) >= grad_thresh (accum: the caller's grad2d or absgrad).  With a non-NULL
 * max_radius, a Gaussian whose max_radius > max_screen_px is pruned as well.  Opacity / scale-norm pruning and the
 * clone / split choice by tau are gs_densify_plan's.  Same outputs, workspace and synchronisation. */
int gs_densify_plan_stats(const float* opa, const float* scale, const float* accum, const int* count,
                          const float* max_radius /* nullable */, float max_screen_px, int n, int scale_activation,
                          float opa_logit_min, float delete_thresh, float grad_thresh, float tau, int use_clone,
                          int use_split, unsigned char* code, int* dst, void* workspace, size_t workspace_bytes,
                          gs_stream_t stream);

/* MCMC densification (3DGS-MCMC, Kheradmand et al. 2024), an opt-in alternative to prune / clone / split.  o =
 * sigmoid(opa); s = the activated scale (|raw| + 1e-4 or exp(raw)).  A draw picks source i with probability
 * proportional to its weight w_i = round(o_i 2^32) (an integer; round half to even; o below 2^-33 weighs 0): with the
 * caller's uniforms u_j in [0, 1) and C the inclusive integer prefix sum of the weights, t_j = min(floor(u_j C_{n-1}),
 * C_{n-1} - 1) (the product in fp64) and src_j = min{i : C_i > t_j}.  A source drawn r - 1 times (r clamped to 51) gets
 *   o' = 1 - (1 - o)^(1/r),  s' = o / den * s,  den = sum_{a=1..r} sum_{b=0..a-1} C(a-1, b) (-1)^b o'^(b+1) / sqrt(b+1)
 * (fp64), then o' is clamped to [min_opacity, 1 - 2^-23] and stored as its logit; s' is inverted with the activation
 * (exp: log s'; abs: sign(raw) max(s' - 1e-4, 0), sign(0) = +, so an s' below 1e-4 becomes the raw scale 0).  Every
 * destination row is a copy of its source with (o', s'), and the source takes the same (o', s').  The prefix sums and
 * the counts are integer sums, so for the same inputs every call draws the same sources and writes the same bits (on
 * every data-parallel replica too), whatever order the device adds them in.  No entry synchronises.
 *   gs_mcmc_workspace_bytes(n): a sampler over n Gaussians with up to n draws.
 *   gs_mcmc_relocate (gsplat's relocate): in place.  Dead Gaussians (o <= min_opacity) are the destinations, in
 *     ascending order, with one draw each from the alive ones (u[n]: the first k are used, k = the number of dead).
 *     With exp_avg / exp_avg_sq (flat buffers and segment table as gs_adam_step_visible takes them, rows = n; NULL =
 *     no optimizer state) the moment rows of every source and destination are zeroed in every segment: gsplat zeroes
 *     the sources only, but a relocated row is a new Gaussian that a dead one's moments must not steer.  touched
 *     (nullable uint8 [n]) gets 1 at those rows and is otherwise left alone.  *n_relocated (DEVICE int) = k, or 0
 *     when nothing is alive.  Nothing else of the parameters or moments is written.
 *   gs_mcmc_add (gsplat's sample_add): n_new draws over all n Gaussians with weights o (u[n_new]); out_* are
 *     caller-allocated [n + n_new] rows: rows 0 .. n-1 are the input with the sources' (o', s'), row n + j the copy of
 *     src_j.  Workspace: gs_mcmc_workspace_bytes(max(n, n_new)).  feat / out_feat: optional [.., f] feature rows.  When
 *     every weight is 0 (every opacity below 2^-33) there is nothing to draw from: the n_new appended rows are then
 *     copies of row 0, unchanged, and row 0 keeps its values.
 *   gs_mcmc_noise (gsplat's inject_noise_to_position): pos_i += scaler g(o_i) R diag(s^2) R^T z_i with R of the
 *     normalised quaternion and g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))); z_i = z[i] (nullable [n][3]) or three
 *     normals of the Philox4x32-10 stream (seed, subsequence i).  Writes pos only; one launch.
 * GS_ERR_INVALID_ARG, before any launch: n or n_new < 0; a NULL pointer that the call needs with n > 0; d not 3 / 27 /
 * 48; f not 8 / 16 / 32 with feat; an unknown activation; min_opacity outside (0, 1); a non-finite scaler; a short
 * workspace; one moment buffer without the other; a segment table gs_adam_step_visible would refuse.  quat (and
 * out_quat) rows are read and written as float4: the pointers must be 16-byte aligned. */
size_t gs_mcmc_workspace_bytes(int n);
int gs_mcmc_relocate(float* pos, float* rgb, float* opa, float* quat, float* scale, float* feat /* nullable */, int f,
                     int n, int d, int scale_activation, float min_opacity, const float* u, float* exp_avg,
                     float* exp_avg_sq, long long n_flat, const long long* seg_start_host, const int* seg_width_host,
                     int n_seg, unsigned char* touched /* nullable */, int* n_relocated, void* workspace,
                     size_t workspace_bytes, gs_stream_t stream);
int gs_mcmc_add(const float* pos, const float* rgb, const float* opa, const float* quat, const float* scale,
                const float* feat /* nullable */, int f, int n, int d, int scale_activation, float min_opacity,
                int n_new, const float* u, float* out_pos, float* out_rgb, float* out_opa, float* out_quat,
                float* out_scale, float* out_feat, void* workspace, size_t workspace_bytes, gs_stream_t stream);
int gs_mcmc_noise(float* pos, const float* quat, const float* scale, const float* opa, int n, int scale_activation,
                  float scaler, unsigned long long seed, const float* z /* nullable */, gs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Next-row widening (SURVEY.md §8 f-3): the training loss of reference train.py:99-107 on the device,
 * forward and backward in two kernels, producing the image gradient in the layout
 * gs_render_backward_final consumes.  image / grad_image: [height, width, 3] float32; target: same
 * shape, float32 or float16 (`target_is_half`; reference `ground_truth` is float16, splatter.py:478).
 *   L1   = mean |image - target|                                             (train.py:99)
 *   SSIM = torchmetrics StructuralSimilarityIndexMeasure(data_range=1.0): 11x11 Gaussian window,
 *          sigma 1.5, k1 0.01, k2 0.03, mean over the pixels whose window is inside the image and
 *          over channels                                                      (train.py:72,101-104)
 *   out3 (device) = { w_l1 * L1 + w_ssim * SSIM + bias,  L1,  SSIM }
 *   grad_image (nullable) = d out3[0] / d image.
 * train.py:107's loss (1 - w) l1 + w (1 - ssim) is w_l1 = 1 - w, w_ssim = -w, bias = w.
 * height and width must exceed 10.  No allocation, no synchronisation. */
size_t gs_loss_workspace_bytes(int height, int width);
int gs_loss_l1_ssim(const float* image, const void* target, int target_is_half, int height, int width,
                    float w_l1, float w_ssim, float bias, float* grad_image, float* out3, void* workspace,
                    size_t workspace_bytes, gs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Per-view bilateral grids for appearance correction (additive; Wang et al., "Bilateral Guided Radiance Field
 * Processing", SIGGRAPH Asia 2024): a rendered image is "sliced" through its training view's grid of 3x4 affine colour
 * transforms before the loss, so per-image exposure, white balance and tone end up in the grids, not in the scene.
 *   grids     : DEVICE float32 [V, GH, GW, GL, 12], one row per training view, the 12 coefficients innermost (a node's
 *               affine is three float4 loads: pointers 16-byte aligned).  Row-major affine A:
 *               out_i = sum_j A[i][j] rgb_j + A[i][3].  grid_sample's [V, 12, GL, GH, GW] is grids.permute(0, 4, 3, 1, 2).
 *               Identity initialisation: A = [I | 0] at every node.
 *   image/out : DEVICE float32 [B, H, W, 3];  view_ids_host : HOST int[B] in [0, V), repeats allowed.
 * Pixel (x, y) of image b samples row view_ids_host[b] at
 *   gx = (x + 0.5) / W (GW - 1),  gy = (y + 0.5) / H (GH - 1),  gz = clamp(z, 0, 1) (GL - 1),
 *   z  = fmaf(0.114f, b, fmaf(0.587f, g, 0.299f * r))   (fp32 luminance of the INPUT pixel)
 * trilinearly with border clamping: value and gradients equal
 *   grid_sample(grids_ncdhw[ids], coords * 2 - 1, mode="bilinear", align_corners=True, padding_mode="border")
 * followed by the affine, including grid_sample's knot convention: dz is 0 at z <= 0 and z >= 1, and an interior knot
 * takes the upper cell's slope.  The output is not clamped; inputs outside [0, 1] are accepted (only z is clamped).
 * Bounds: 2 <= GH, GW <= GS_BILAGRID_MAX_HW; 2 <= GL <= GS_BILAGRID_MAX_L (the backward keeps one accumulator per
 * z knot in registers); B <= 65535; H * W <= 2^30.
 * gs_bilagrid_slice_fwd: one kernel launch per 64 images.
 * gs_bilagrid_slice_bwd: from grad_out = dL/dout [B, H, W, 3] in one pass over the pixels,
 *   grad_image (nullable) = dL/dimage, through the affine and through the guide z;
 *   grad_grids (nullable) : the rows of the views in the batch are WRITTEN (repeated views' contributions added); the
 *               other rows are left as they are (callers zero them).
 * The grid gradient is bit-deterministic without floating-point atomics: per-CTA partials of one spatial cell, written
 * once, then summed per node in index order (images of the view ascending, adjacent cells, row slices).  Two launches
 * (one without grad_grids) after one that writes the view table into the workspace (one per 960 table entries; the
 * table has at most 2B).  No allocation, no synchronisation.
 * Refused before any launch (GS_ERR_INVALID_ARG, gs_last_error set): a null image, grids, view_ids_host, out / grad_out
 * or workspace; B, H, W or V <= 0; a grid dimension outside the bounds; a view id outside [0, V); a workspace shorter
 * than gs_bilagrid_workspace_bytes (0 for invalid shapes).  Nothing to compute (both gradients NULL) returns 0. */
#define GS_BILAGRID_MAX_HW 256
#define GS_BILAGRID_MAX_L 16
size_t gs_bilagrid_workspace_bytes(int B, int H, int W, int V, int GH, int GW, int GL);
int gs_bilagrid_slice_fwd(const float* image, const float* grids, const int* view_ids_host, int B, int H, int W,
                          int V, int GH, int GW, int GL, float* out, gs_stream_t stream);
int gs_bilagrid_slice_bwd(const float* image, const float* grids, const int* view_ids_host, int B, int H, int W,
                          int V, int GH, int GW, int GL, const float* grad_out, float* grad_image /* nullable */,
                          float* grad_grids /* nullable */, void* workspace, size_t workspace_bytes,
                          gs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Multi-GPU exchange step (SURVEY.md §8e; new - the reference is single-GPU): in-place SUM of
 * the flat gradient bucket across `world` GPUs of one NVSwitch domain through an NVLS multicast
 * mapping.  `multicast_ptr` is the multicast address of a symmetric buffer holding each rank's
 * n_floats (multiple of 4) gradients at the same offset; rank r reduces and re-broadcasts slice r
 * (multimem.ld_reduce + multimem.st).  The caller orders it between two cross-rank barriers
 * (all buckets written before; all slices visible after).  No synchronisation inside. */
int gs_allreduce_multimem_f32(void* multicast_ptr, long long n_floats, int rank, int world,
                              gs_stream_t stream);

/* The same exchange over plain peer mappings (no multicast needed): `peer_ptrs` is a HOST array
 * of `world` (2, 4 or 8) device pointers, entry p = rank p's copy of the bucket as mapped into
 * this process (entry `rank` = the local copy).  Rank r sums slice r over all copies and stores
 * the sum into all of them.  Same barrier contract as above. */
#define GS_MAX_PEERS 8
int gs_allreduce_p2p_f32(void* const* peer_ptrs, long long n_floats, int rank, int world,
                         gs_stream_t stream);

/* Exchange fused into the backward ("push"): the flat bucket is cut into `world` slices of `per`
 * floats (multiple of 4; world * per >= bucket length, < 2^32); rank r owns slice r.  While a
 * context has a push configuration, gs_render_backward, gs_render_backward_final,
 * gs_render_backward_aux and gs_render_backward_feat (without a feature-map gradient) store every
 * gradient float that belongs to ANOTHER rank's slice straight into slot `rank` of that owner's
 * staging buffer (staging[p] = rank p's [world][per] float buffer as mapped into this process)
 * from inside the projection-backward kernel, and only its own slice into `bucket` - the reduce
 * half of the exchange overlaps the kernel; the camera-gradient, feature-map-gradient and batched
 * backwards refuse a push configuration.  The five gradient pointers of the backward call must lie
 * inside [bucket, bucket + world * per) with grad_quat on a 16-byte bucket offset; a call that
 * breaks this is refused before any launch.  gs_allreduce_push_finish_f32 (after a cross-rank barrier)
 * completes it: rank r sums its own slice with the world-1 pushed contributions and stores the sum
 * into every rank's bucket (`peer_buckets`: host array of `world` device pointers); a second
 * barrier makes all slices visible.  world must be 2, 4 or 8.  NULL clears the configuration. */
typedef struct gs_grad_push {
  int world, rank;
  long long per;
  float* bucket;
  float* staging[GS_MAX_PEERS];
} gs_grad_push;
int gs_ctx_set_grad_push(gs_ctx* ctx, const gs_grad_push* push);
int gs_allreduce_push_finish_f32(void* const* peer_buckets, const float* staging_local, long long n_floats,
                                 long long per, int rank, int world, gs_stream_t stream);
/* The same second half with the broadcast done by the NVSwitch: the sum of rank r's slice is written once
 * through `bucket_multicast` (the NVLS multicast address of the symmetric bucket; `bucket_local` is this
 * rank's own mapping of it) with multimem.st and lands in all `world` buckets. */
int gs_allreduce_push_finish_mc_f32(void* bucket_multicast, const float* bucket_local, const float* staging_local,
                                    long long n_floats, long long per, int rank, int world, gs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_H */
