// Internal (non-ABI) launcher declarations shared between the translation units of libgs_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gs_b200.h"
#include "project.cuh"

// Width (floats) of one per-instance gradient record written by the blend backward:
// {d_x, d_y, d_ca, d_cb, d_cc, d_l2o, d_r, d_g, d_b} (+ 3 pad so rows are 16-byte aligned)
#define GS_GREC 12

struct GsFrameGeom {
  int width, height, wp, hp, ntx, nty, n_tiles;
  float fx, fy;
};

// Optional fused post-processing of reference splatter.py:652-653 (clamp to [0,1] + centre crop):
// forward additionally writes final[height,width,3]; backward takes the gradient of that final
// image (clamp mask from the raw padded image, zero outside the crop) instead of a padded one.
struct GsCrop {
  int left, top, width, height;
};

// Optional per-pixel outputs of the gather blend kernels (gs_render_forward_aux): the image gets T_f * bg added, and
// aux[Hp,Wp,2] / aux_final[height,width,2] (either nullable) receive (depth = sum w t, alpha = 1 - T_f) per pixel,
// t = |p_c| (GsRec c.y).  Only read by the AUX instantiations of the blend forward kernels.
struct GsAuxOut {
  float bg[3];
  float* aux;
  float* aux_final;
};

#ifdef __CUDACC__
// (depth, alpha) of padded pixel (ix, iy) to aux[Hp,Wp,2] and, inside the crop, to aux_final[height,width,2]
__device__ __forceinline__ void gs_store_aux(const GsAuxOut& ax, int ix, int iy, int wp, const GsCrop& crop,
                                             float depth, float alpha) {
  if (ax.aux) *reinterpret_cast<float2*>(ax.aux + ((size_t)iy * wp + ix) * 2) = make_float2(depth, alpha);
  const int x = ix - crop.left, y = iy - crop.top;
  if (ax.aux_final && x >= 0 && x < crop.width && y >= 0 && y < crop.height)
    *reinterpret_cast<float2*>(ax.aux_final + ((size_t)y * crop.width + x) * 2) = make_float2(depth, alpha);
}
// (g_D, g_A) of PX pixels ix0 .. ix0 + PX - 1 of row iy (padded grad_aux, or the cropped one when grad_is_final:
// depth / alpha are not clamped, only the crop masks their gradient); R += g_D depth + g_A alpha (forward's aux)
template <int PX>
__device__ __forceinline__ void gs_load_aux_grad(const float* __restrict__ aux, const float* __restrict__ grad_aux,
                                                 int grad_is_final, int ix0, int iy, int wp, const GsCrop& crop,
                                                 float (&gD)[PX], float (&gA)[PX], float (&R)[PX]) {
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    const size_t off = ((size_t)iy * wp + ix0 + p) * 2;
    const float2 da = *reinterpret_cast<const float2*>(aux + off);
    float2 g = make_float2(0.f, 0.f);
    if (!grad_is_final) {
      g = *reinterpret_cast<const float2*>(grad_aux + off);
    } else {
      const int x = ix0 + p - crop.left, y = iy - crop.top;
      if (x >= 0 && x < crop.width && y >= 0 && y < crop.height)
        g = *reinterpret_cast<const float2*>(grad_aux + ((size_t)y * crop.width + x) * 2);
    }
    gD[p] = g.x;
    gA[p] = g.y;
    R[p] = fmaf(g.x, da.x, fmaf(g.y, da.y, R[p]));
  }
}
#endif

// world-space ray setup for per-pixel SH (reference splatter.py:305-321), DEVICE pointers to 3 floats each
struct GsRayPtrs {
  const float *rays_o, *lefttop, *dx, *dy;
};

// Run-time tuning knobs (A/B experiments; the defaults are the configuration measured fastest on the H100).
// Set with gs_tune("name", value) or the environment variable GS_TUNE_<NAME> (read once).
struct GsTuning {
  int fwd_kernel;   // 0 = consumer thread 0 issues the copies, 1 = dedicated producer warp
  int fwd_ch;       // staging chunk of kernel 0: 64 / 128 / 256
  int bwd_kernel;   // 0 = shuffle-network reduction (round 1), 1 = two-phase shared-memory reduction
  int bwd_px;       // pixels per consumer thread: 4 or 8
  int bwd_ws;       // dedicated producer warp
  int bwd_unroll;   // instances per unrolled step: 1, 2, 4
  int bwd_stages;   // staging ring depth: 2 or 3
  int bwd_minb;     // __launch_bounds__ min blocks (register cap); 1 = none
  int bwd_rq;       // reducer threads per instance in the second phase: 4 (16 instances per round) or 8 (8)
  int fwd_px;       // pixels per thread of forward kernel 0: 4 (2 warps per tile) or 8 (1 warp)
  int bwd_ch;       // gather path: instances per staging chunk of the backward (64 or 32)
  int strict;       // 1: an un-instantiated knob combination is an error (sweeps); 0: falls back to the shipped kernel
  int gather;       // fused frame path (RGB and SH): 1 = no pack pass, blend kernels gather records from rec[N]; 0 = packed streams
  int sh_tc;        // SH blend on the tensor cores (blend_sh_tc.cu, gather path only): -1 = by colour width (gs_sh_tc_mode),
                    // else bit 0 = forward, bit 1 = backward, bit 2 = two pixels per thread in the backward
  int blend_repack; // shipped RGB backward blend (plain and aux): 1 = repack live pixels into fewer slots per lane as
                    // pixels saturate, 0 = every lane keeps its 8 pixels until the whole tile is saturated
};
GsTuning& gs_tuning();

// every launch of one of OUR kernels is counted (bench.py reports the count of the timed region)
void gs_count_launch(int n = 1);

// ---- blend_sh.cu -----------------------------------------------------------------------
int gs_sh_basis_count(int d);      // 27 -> 9, 48 -> 16, else 0
int gs_sh_stream_width(int d);     // floats per instance row of the SH stream (coefficients + slot, padded)
int gs_sh_grad_width(int d);       // floats per instance gradient row (6 geometry + d coefficients, padded)
int gs_sh_tc_mode(int d);          // the sh_tc bits in effect for colour width d
// grec != nullptr: gather path (records from rec[N], raw coefficients from the parameter tensor rgb[N, d])
cudaError_t gs_launch_blend_sh_fwd(const float4* pA, const float2* pB, const float* pS, const GsRec* grec,
                                   const float* rgb, const uint32_t* ids, const uint32_t* goff /*offsets_g*/, int d,
                                   const int* tile_accum,
                                   const GsFrameGeom& g, const GsRayPtrs& r, float* image, int* tile_neff,
                                   float* final_img, const GsCrop& crop, cudaStream_t st,
                                   const GsAuxOut* aux = nullptr /*non-null: AUX kernel (gather)*/);
cudaError_t gs_launch_blend_sh_bwd(const float4* pA, const float2* pB, const float* pS, const GsRec* grec,
                                   const float* rgb, const uint32_t* ids, const uint32_t* goff /*offsets_g*/, int d,
                                   const int* tile_accum,
                                   const GsFrameGeom& g, const GsRayPtrs& r, const float* image,
                                   const float* grad_image, float* grad_inst, int grad_is_final, const GsCrop& crop,
                                   uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b, cudaStream_t st,
                                   const float* aux = nullptr, const float* grad_aux = nullptr /*non-null: AUX*/);

// ---- blend_sh_tc.cu (wgmma) ---------------------------------------------------------------
cudaError_t gs_launch_blend_sh_fwd_tc(const GsRec* grec, const float* rgb, const uint32_t* ids, int d,
                                      const int* tile_accum, const GsFrameGeom& g, const GsRayPtrs& r, float* image,
                                      int* tile_neff, float* final_img, const GsCrop& crop, cudaStream_t st,
                                      const GsAuxOut* aux = nullptr);
cudaError_t gs_launch_blend_sh_bwd_tc(const GsRec* grec, const float* rgb, const uint32_t* ids, const uint32_t* goff, int d,
                                      const int* tile_accum, const GsFrameGeom& g, const GsRayPtrs& r, const float* image,
                                      const float* grad_image, float* grad_inst, int grad_is_final, const GsCrop& crop,
                                      uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b, cudaStream_t st,
                                      const float* aux = nullptr, const float* grad_aux = nullptr);

// ---- project.cu ------------------------------------------------------------------------
cudaError_t gs_launch_fused_project(const float* pos, const float* rgb, const float* opa, const float* quat,
                                    const float* scale, int n, int d, int scale_act, const GsCam& cam,
                                    const GsTileGrid& grid, float near_plane, float half_w, float half_h,
                                    GsRec* rec, uint2* rect /*[n]: tile rectangle, zero without instances*/,
                                    uint32_t* count, uint32_t* dkey, int64_t* mask, unsigned int* n_visible, cudaStream_t st,
                                    bool sh_gaussian = false /*d = 27 / 48: SH evaluated per Gaussian into rec's RGB*/,
                                    const GsFilter2d* filt = nullptr /*non-null: 2-D screen-space filter*/,
                                    const float* f3d = nullptr /*non-null: 3-D filter [n] (with filt, or a zero one)*/,
                                    const GsLens* lens = nullptr /*non-null: the lens (with the 2-D and 3-D filter paths)*/);

// One view of a batched frame (gs_render_forward_batch): the per-view constants of the projection, the blend, the
// projection backward and the densification statistics, formed on the host exactly as a single-view frame forms them
// and read by the batched kernels from a device table [n_views].  View v owns tile rows v nty .. (v + 1) nty - 1 of
// the frame's tile grid and rows v Hp .. (v + 1) Hp - 1 of the tall padded image.
struct GsView {
  GsCam cam;
  GsTileGrid grid;     // the view's own grid (nty rows); the projection offsets the rectangle's rows by v nty
  GsFilter2d filt;     // zero when the frame has no 2-D filter
  float half_w, half_h, fx, fy;
};

cudaError_t gs_launch_fused_project_batch(const float* pos, const float* rgb, const float* opa, const float* quat,
                                          const float* scale, int n, int n_views, int d, int scale_act,
                                          const GsView* views, float near_plane, GsRec* rec /*[B n]*/,
                                          uint2* rect /*[B n]*/, uint32_t* count /*[B n]*/, uint32_t* dkey /*[B n]*/,
                                          int64_t* mask /*[B, n], nullable*/, unsigned int* n_visible,
                                          cudaStream_t st, bool sh_gaussian, bool filt,
                                          const float* f3d = nullptr /*non-null: 3-D filter [n]*/,
                                          const GsLens* lenses = nullptr /*non-null: DEVICE [n_views] lenses*/);

// Data-parallel gradient push (device view of gs_grad_push): world == 0 disables it.
struct GsGradPush {
  float* bucket;                  // this rank's flat gradient bucket (the five grad pointers lie inside)
  float* staging[GS_MAX_PEERS];   // staging[p] = rank p's staging buffer [world][per] as mapped here
  uint32_t per;                   // floats per slice (multiple of 4)
  int rank, world;
};

cudaError_t gs_launch_fused_project_bwd(const float* pos, const float* rgb, const float* opa, const float* quat,
                                        const float* scale, int n, int d, int scale_act, const GsCam& cam,
                                        float near_plane, float half_w, float half_h, const uint32_t* offsets_g,
                                        const uint32_t* count, const float* grad_inst, const uint32_t* row_epoch, uint32_t epoch,
                                        float* g_pos, float* g_rgb, float* g_opa,
                                        float* g_quat, float* g_scale, const GsGradPush& push, cudaStream_t st,
                                        bool depth_grad = false /*rows carry dL/d|p_c| in the column after the colour*/,
                                        bool sh_gaussian = false /*d = 27 / 48 coefficients, RGB gradient rows*/,
                                        const GsFilter2d* filt = nullptr /*the forward's 2-D filter*/,
                                        const float* f3d = nullptr /*the forward's 3-D filter [n]*/,
                                        const GsLens* lens = nullptr /*the forward's lens (no push)*/);
// The same without a push, for RGB and per-Gaussian SH, plus the camera gradient: the projection backward leaves one
// 12-float partial sum per CTA in cam_part (gs_cam_grad_workspace_bytes(n)), and a one-CTA kernel sums them in fp64
// into grad_cam[12] = {dL/drot row-major, dL/dtran} (zeros when n == 0).  The five gradient pointers may all be NULL
// (camera only).  Two launches (one when n == 0).
size_t gs_cam_grad_workspace_bytes(int n);
cudaError_t gs_launch_fused_project_bwd_cam(const float* pos, const float* rgb, const float* opa, const float* quat,
                                            const float* scale, int n, int d, int scale_act, const GsCam& cam,
                                            float near_plane, float half_w, float half_h, const uint32_t* offsets_g,
                                            const uint32_t* count, const float* grad_inst, const uint32_t* row_epoch,
                                            uint32_t epoch, float* g_pos, float* g_rgb, float* g_opa, float* g_quat,
                                            float* g_scale, float* cam_part, float* grad_cam, cudaStream_t st,
                                            bool depth_grad, bool sh_gaussian, const GsFilter2d* filt = nullptr,
                                            const float* f3d = nullptr,
                                            const GsLens* lens = nullptr);

// Batched frame: one thread per Gaussian sums, view by view in view order, the rows of pair v n + i exactly as
// gs_launch_fused_project_bwd does for one view, chains them with view v's camera and filter, and writes the sum over
// the views of each parameter gradient once.  No push.  One launch when n > 0.
cudaError_t gs_launch_fused_project_bwd_batch(const float* pos, const float* rgb, const float* opa, const float* quat,
                                              const float* scale, int n, int n_views, int d, int scale_act,
                                              const GsView* views, float near_plane, const uint32_t* offsets_g,
                                              const uint32_t* count, const float* grad_inst, const uint32_t* row_epoch,
                                              uint32_t epoch, float* g_pos, float* g_rgb, float* g_opa, float* g_quat,
                                              float* g_scale, cudaStream_t st, bool depth_grad, bool sh_gaussian,
                                              bool filt, const float* f3d = nullptr,
                                              const GsLens* lenses = nullptr);
// The same plus each view's camera gradient (RGB and per-Gaussian SH): the projection backward leaves view v's per-CTA
// partial sums in cam_part[v][grid][12] (n_views * gs_cam_grad_workspace_bytes(n)), and one CTA per view sums them in
// fp64 into grad_cams[v][12] (zeros when n == 0).  The five gradient pointers may all be NULL (camera only).  Two
// launches (one when n == 0), whatever n_views.
cudaError_t gs_launch_fused_project_bwd_batch_cam(const float* pos, const float* rgb, const float* opa,
                                                  const float* quat, const float* scale, int n, int n_views, int d,
                                                  int scale_act, const GsView* views, float near_plane,
                                                  const uint32_t* offsets_g, const uint32_t* count,
                                                  const float* grad_inst, const uint32_t* row_epoch, uint32_t epoch,
                                                  float* g_pos, float* g_rgb, float* g_opa, float* g_quat,
                                                  float* g_scale, float* cam_part, float* grad_cams, cudaStream_t st,
                                                  bool depth_grad, bool sh_gaussian, bool filt,
                                                  const float* f3d = nullptr,
                                                  const GsLens* lenses = nullptr);

// ---- densify_stats.cu ------------------------------------------------------------------
// Accumulates the screen-space densification statistics of the backward that just wrote grad_inst (rows of gw floats;
// s.absgrad != NULL reads columns 10, 11 written by the ABS blend kernels) into s's buffers.  One launch when n > 0.
cudaError_t gs_launch_densify_stats(const float* pos, const float* quat, const float* scale, int n, int scale_act,
                                    const GsCam& cam, float near_plane, float half_w, float half_h,
                                    const GsFilter2d& filt /*the forward's; zero when it had none*/,
                                    const uint32_t* offsets_g, const uint32_t* count, const float* grad_inst, int gw,
                                    const uint32_t* row_epoch, uint32_t epoch, const GsFrameGeom& g,
                                    const gs_densify_stats& s, cudaStream_t st,
                                    const float* f3d = nullptr /*the forward's 3-D filter [n]*/,
                                    const GsLens* lens = nullptr /*the forward's lens*/);
// The same for a batched frame: each view's statistics are added in view order (g: the per-view width and height)
cudaError_t gs_launch_densify_stats_batch(const float* pos, const float* quat, const float* scale, int n, int n_views,
                                          int scale_act, const GsView* views, float near_plane,
                                          const uint32_t* offsets_g, const uint32_t* count, const float* grad_inst,
                                          int gw, const uint32_t* row_epoch, uint32_t epoch, const GsFrameGeom& g,
                                          const gs_densify_stats& s, cudaStream_t st, const float* f3d = nullptr,
                                          const GsLens* lenses = nullptr);

// ---- filter3d.cu -----------------------------------------------------------------------
// One view of gs_filter3d_compute, formed on the host: the depth and the rate in fp64, the margin test in fp32.
struct GsF3View {
  double rz[3], tz;            // row 2 of R and t_z: z = rz . p + tz
  double fxd;                  // fx: the rate fx / z
  float r[6], t[2];            // rows 0, 1 of R and t_x, t_y
  float fx, fy, cx, cy;        // cx = W / 2, cy = H / 2 (with a lens: its principal point)
  float ulo, uhi, wlo, whi;    // -m W, (1 + m) W, -m H, (1 + m) H
  double near;                 // seen only where z > near
};
// f3d[n] = sqrt(variance) / (the largest fx / z among the views that see Gaussian i), or that of the smallest seen
// rate for a Gaussian no view sees (0 everywhere when none is seen).  min_rate: one u32 set to 0xffffffff by the
// caller.  Two launches when n > 0.
// lenses (DEVICE [n_views], nullable): the lens variant of the rate and the visibility test (gs_ctx_set_lens).
cudaError_t gs_launch_filter3d(const float* pos, int n, const GsF3View* views /*DEVICE [n_views]*/, int n_views,
                               float variance, float* f3d, unsigned int* min_rate, cudaStream_t st,
                               const GsLens* lenses = nullptr);

// ---- optim.cu --------------------------------------------------------------------------
// visible[n] (uint8) = count[v n + i] > 0 in any of the n_views views, OR-ed into visible when accumulate is set
// (gs_frame_visible).  One launch when n > 0.
cudaError_t gs_launch_frame_visible(const uint32_t* count, int n, int n_views, int accumulate, unsigned char* visible,
                                    cudaStream_t st);

// ---- scores.cu -------------------------------------------------------------------------
// gs_frame_scores: the blend-weight rows of the last gather-path forward (views: its DEVICE view table when batched,
// else NULL) to rows[M] / row_epoch[M] tagged with `epoch`, then added into weight_sum / weight_max [n].  Two
// launches when n > 0.
cudaError_t gs_launch_frame_scores(const GsRec* grec, const uint32_t* ids, const uint32_t* offsets_g,
                                   const uint32_t* count, const int* tile_accum, const GsFrameGeom& g,
                                   const GsView* views, int n, int n_views, const GsCrop& crop, float2* rows,
                                   uint32_t* row_epoch, uint32_t epoch, float* weight_sum, float* weight_max,
                                   cudaStream_t st);

// ---- blend_feat.cu ---------------------------------------------------------------------
// Feature maps (gs_render_forward_feat / gs_render_backward_feat), gather path only.  f: 8, 16 or 32.
bool gs_feat_width_ok(int f);
// the RGB forward (+ AUX: background, depth / alpha) that also writes map[Hp,Wp,f] and map_final[h,w,f] (nullable)
cudaError_t gs_launch_blend_feat_fwd(const GsRec* grec, const float* feat, int f, const uint32_t* ids,
                                     const int* tile_accum, const GsFrameGeom& g, float* image, int* tile_neff,
                                     float* final_img, const GsCrop& crop, const GsAuxOut* aux /*nullable*/, float* map,
                                     float* map_final, cudaStream_t st);
// the RGB backward (+ AUX when grad_aux) with the feature terms: GS_GREC rows to grad_inst, f-float rows to
// grad_feat_inst, both at the instance's slot and tagged in row_epoch
cudaError_t gs_launch_blend_feat_bwd(const GsRec* grec, const float* feat, int f, const uint32_t* ids,
                                     const uint32_t* goff, const int* tile_accum, const GsFrameGeom& g,
                                     const float* image, const float* grad_image, const float* map,
                                     const float* grad_map, float* grad_inst, float* grad_feat_inst, int grad_is_final,
                                     const GsCrop& crop, uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b,
                                     const float* aux, const float* grad_aux, cudaStream_t st);
// grad_feat[n, f] = per-Gaussian sums of the epoch-tagged rows of grad_feat_inst (one launch when n > 0)
cudaError_t gs_launch_feat_grad(const uint32_t* offsets_g, const uint32_t* count, const float* grad_feat_inst,
                                const uint32_t* row_epoch, uint32_t epoch, int n, int f, float* grad_feat,
                                cudaStream_t st);

// ---- surfel.cu / blend_surfel.cu (2D Gaussian surfels: gs_render_forward_surfel) ----------------------------------
// One surfel's record (64 bytes), written by the surfel projection and gathered by the surfel blend kernels:
//   M = [s_u R r0 | s_v R r1 | p_c] row-major (rows m_x, m_y, m_z), op = sigmoid(opa), the activated colour, and the
//   camera-frame normal R r2 flipped to face the camera.
struct __align__(16) GsSurfelRec {
  float M[9];
  float op;
  float rgb[3];
  float nrm[3];
};
// Per padded pixel, written by the surfel forward for its backward: ws[p] = {sum w c (3), T_f}; with maps also
// wsm[2p] = {sum w z, sum w, sum w m, sum w m^2} (m relative to the first blended instance) and wsm[2p + 1] = {sum w n (3), median instance (int bits, -1: none)}.
// The map channels of gs_render_surfel: GS_SURFEL_MAP_CH floats per pixel.
struct GsSurfelMaps {
  float* maps;         // [Hp, Wp, 8] or NULL
  float* maps_final;   // [height, width, 8] or NULL
  float dist_near, dist_far;
};
// KG = 0: RGB logits (d = 3); 9 / 16: per-Gaussian SH of degree 2 / 3.  One launch when n > 0.
cudaError_t gs_launch_surfel_project(const float* pos, const float* rgb, const float* opa, const float* quat,
                                     const float* scale, int n, int kg, int scale_act, const GsCam& cam,
                                     const GsTileGrid& grid, float near_plane, float half_w, float half_h, float fx,
                                     float fy, GsSurfelRec* rec, uint2* rect, uint32_t* count, uint32_t* dkey,
                                     int64_t* mask, unsigned int* n_visible, cudaStream_t st);
// Chains the epoch-tagged GS_SURFEL_GREC rows of each surfel to the raw parameters.  One launch when n > 0.
#define GS_SURFEL_GREC 16
cudaError_t gs_launch_surfel_project_bwd(const float* pos, const float* rgb, const float* opa, const float* quat,
                                         const float* scale, int n, int kg, int scale_act, const GsCam& cam,
                                         const uint32_t* offsets_g, const uint32_t* count, const float* grad_inst,
                                         const uint32_t* row_epoch, uint32_t epoch, float* g_pos, float* g_rgb,
                                         float* g_opa, float* g_quat, float* g_scale, cudaStream_t st);
cudaError_t gs_launch_blend_surfel_fwd(const GsSurfelRec* rec, const uint32_t* ids, const int* tile_accum,
                                       const GsFrameGeom& g, const float* bg /*3 floats, by value*/, float* image,
                                       float* final_img, const GsCrop& crop, const GsSurfelMaps* maps /*nullable*/,
                                       float near /*hits at z <= near are skipped*/, float4* ws, float4* wsm, int* tile_neff, cudaStream_t st);
cudaError_t gs_launch_blend_surfel_bwd(const GsSurfelRec* rec, const uint32_t* ids, const uint2* rect,
                                       const uint32_t* goff, const int* tile_accum, const GsFrameGeom& g,
                                       const float* bg, const float* image, const float* grad_image, int grad_is_final,
                                       const GsCrop& crop, const float* grad_maps /*nullable*/, float dist_near,
                                       float dist_far, float near, const float4* ws, const float4* wsm, float* grad_inst,
                                       uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b, cudaStream_t st);

// ---- binning.cu ------------------------------------------------------------------------
cudaError_t gs_launch_emit_keys(const uint2* rect, const uint32_t* perm, const uint32_t* offsets_sorted, int n, int ntx,
                                void* keys, int key_bytes, uint32_t* vals, cudaStream_t st);
cudaError_t gs_launch_tile_ranges(const void* keys, int key_bytes, long long m, int n_tiles, int* tile_accum,
                                  cudaStream_t st);

cudaError_t gs_launch_pack_sorted(const void* keys, int key_bytes, const uint32_t* vals, long long m, int n_tiles,
                                  int ntx, const GsRec* rec, const uint32_t* offsets_g, float4* pA, float2* pB, float4* pC,
                                  int* tile_accum, cudaStream_t st);

cudaError_t gs_launch_pack_sorted_sh(const void* keys, int key_bytes, const uint32_t* vals, long long m, int n_tiles,
                                     int ntx, const GsRec* rec, const uint32_t* offsets_g, const float* rgb, int d, int sw,
                                     float4* pA, float2* pB, float* pS, int* tile_accum, cudaStream_t st);
cudaError_t gs_launch_iota(uint32_t* out, int n, cudaStream_t st);

// ---- blend.cu --------------------------------------------------------------------------
// grec / ids != nullptr: gather path (records pulled straight from rec[N] through the sorted id list; the packed
// stream pointers are ignored); else the packed streams written by the pack pass / the legacy draw API.
cudaError_t gs_launch_blend_fwd(const float4* pA, const float2* pB, const float4* pC, const GsRec* grec,
                                const uint32_t* ids, const int* tile_accum, const GsFrameGeom& g, float* image,
                                int* tile_neff, float* final_img, const GsCrop& crop, cudaStream_t st,
                                const GsAuxOut* aux = nullptr /*non-null: AUX kernel (gather path, shipped knobs)*/);

cudaError_t gs_launch_blend_bwd(const float4* pA, const float2* pB, const float4* pC, const GsRec* grec,
                                const uint32_t* ids, const uint32_t* goff /*offsets_g (gather path)*/,
                                const int* tile_accum, const GsFrameGeom& g, const float* image,
                                const float* grad_image, float* grad_inst /*[M,GS_GREC] rows addressed by slot*/,
                                int grad_is_final, const GsCrop& crop, uint32_t* row_epoch /*nullable (packed only)*/,
                                uint32_t epoch, int* tile_neff_b /*nullable: instances the backward consumed per tile*/,
                                cudaStream_t st, const float* aux = nullptr /*forward's [Hp,Wp,2]*/,
                                const float* grad_aux = nullptr /*non-null: AUX kernel; [Hp,Wp,2] or [h,w,2]*/,
                                bool absgrad = false /*ABS kernel: sum |d/dx|, sum |d/dy| to columns 10, 11*/);
// The ABS blend backward kernels exist only for the shipped RGB backward of the gather path (with and without AUX):
// 0 when a frame of blend colour width d on that path (`gather`) runs one under the current knobs, else
// GS_ERR_UNSUPPORTED with a message.
int gs_blend_absgrad_supported(int d, bool gather);
// The AUX blend kernels exist only for the shipped configurations of the gather path (RGB: the default blend knobs;
// SH: the scalar and one-pixel-per-thread tensor-core kernels): 0 when the current tuning knobs for colour width d
// select one, else GS_ERR_UNSUPPORTED with a message.
int gs_blend_aux_supported(int d, bool forward, bool backward);

// Batched frames (gs_render_forward_batch) run the shipped RGB gather kernels with the batched flag: the view of a tile
// is its tile row / (hp / GS_TILE), pixel coordinates use the view's rows and views[v].fx / fy, and final / aux_final /
// a final upstream gradient are addressed per view ([B, height, width, .]).  g: per-view wp, hp, width, height; the
// frame's ntx and n_tiles = B T.  0 when the current knobs select those kernels (the shipped forward and backward blend
// knobs with the live-pixel repack, gather path), else GS_ERR_UNSUPPORTED with a message.
int gs_blend_batch_supported();
cudaError_t gs_launch_blend_fwd_batch(const GsRec* grec, const uint32_t* ids, const int* tile_accum,
                                      const GsFrameGeom& g, const GsView* views, float* image, int* tile_neff,
                                      float* final_img, const GsCrop& crop, cudaStream_t st,
                                      const GsAuxOut* aux /*nullable*/);
cudaError_t gs_launch_blend_bwd_batch(const GsRec* grec, const uint32_t* ids, const uint32_t* goff,
                                      const int* tile_accum, const GsFrameGeom& g, const GsView* views,
                                      const float* image, const float* grad_image, float* grad_inst, int grad_is_final,
                                      const GsCrop& crop, uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b,
                                      cudaStream_t st, const float* aux, const float* grad_aux /*nullable*/,
                                      bool absgrad);
