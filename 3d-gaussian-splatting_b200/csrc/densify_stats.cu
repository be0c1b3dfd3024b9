// Screen-space densification statistics of the fused frame path (gs_ctx_set_densify_stats): one thread per Gaussian
// after the projection backward, accumulating into the caller's buffers.  A kernel of its own, not a flag on the
// projection backward: that body has more than 100 instantiations (D, GW, W, DT, KG, CG, F), and this one kernel
// follows every one of them, the data-parallel push included.
#include "internal.h"

namespace {

constexpr int kBlock = 256;
constexpr float kInf = __builtin_huge_valf();   // gs_project's frustum half-widths in a lens frame (gs_lens_project)

// Gaussian i with count[i] > 0 (it got at least one tile instance in the forward):
//   grad2d  += |(gx sx, gy sy)|, (gx, gy) = sum of columns 0, 1 over its rows tagged with this backward's epoch
//   absgrad += |(Ax sx, Ay sy)|, (Ax, Ay) = the same sums of columns 10, 11 (ABS: sum_p |g_x,p|, sum_p |g_y,p|)
//   count   += 1
//   max_radius = max(max_radius, ceil(3 sqrt(lambda_max))) of the 2-D covariance the forward binned, in px^2
// (sx, sy) = (W / (2 fx), H / (2 fy)) converts dL/d(x/z, y/z) to the NDC convention of 3DGS's viewspace gradient.
// One thread owns one Gaussian and sums its rows in order: bit-deterministic, no atomics.
// G3: the forward applied the 3-D filter f3d[n]: the covariance is the filtered scale's (gs_filter3d).
// L (only with G3): the forward applied the lens `lens`: the covariance is the lensed one (gs_lens_project); f3d may be
// NULL.  (x, y) stays the stored mean's gradient.
#define GS_STATS_PARAMS                                                                                             \
  const float* __restrict__ pos, const float* __restrict__ quat, const float* __restrict__ scale, int n,            \
      int scale_act, GsCam cam, float near_plane, float half_w, float half_h, GsFilter2d filt,                      \
      const uint32_t* __restrict__ offsets_g, const uint32_t* __restrict__ count,                                  \
      const float* __restrict__ grad_inst, int gw, const uint32_t* __restrict__ row_epoch, uint32_t epoch,         \
      float sx, float sy, float fx, float fy, float* __restrict__ grad2d, float* __restrict__ absgrad,             \
      int* __restrict__ n_views, float* __restrict__ max_radius
#define GS_STATS_ARGS                                                                                             \
  pos, quat, scale, n, scale_act, cam, near_plane, half_w, half_h, filt, offsets_g, count, grad_inst, gw, row_epoch, \
      epoch, sx, sy, fx, fy, grad2d, absgrad, n_views, max_radius
template <bool ABS, bool G3, bool L = false>
__device__ __forceinline__ void densify_stats_body(GS_STATS_PARAMS, const float* __restrict__ f3d,
                                                   GsLens lens = GsLens{}) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const uint32_t cnt = count[i];
  if (cnt == 0) return;
  float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  float q[4], s[3], raw_s[3], qn;
  gs_load_activated(quat, scale, i, scale_act, q, s, raw_s, qn);
  if constexpr (G3) {
    float s0[3], dl2o3;
    gs_filter3d((L && !f3d) ? 0.f : f3d[i], s, s0, dl2o3);
  }
  float gx = 0.f, gy = 0.f, ax = 0.f, ay = 0.f;
  const uint32_t o0 = offsets_g[i], o1 = o0 + cnt;
  for (uint32_t r = o0; r < o1; ++r) {
    if (row_epoch[r] != epoch) continue;   // not reached by its (saturated) tile: zero gradient
    const float* row = grad_inst + (size_t)r * gw;
    const float2 g = *reinterpret_cast<const float2*>(row);
    gx += g.x;
    gy += g.y;
    if constexpr (ABS) {
      const float2 a = *reinterpret_cast<const float2*>(row + 10);
      ax += a.x;
      ay += a.y;
    }
  }
  // the covariance the forward binned: with the filter its dilated one (a zero filter leaves it as it is)
  GsProj o = gs_project(cam, p, q, s, near_plane, L ? kInf : half_w, L ? kInf : half_h);
  if constexpr (L) {
    float J[4];
    gs_lens_project(lens, o, half_w, half_h, J);
  }
  const GsFilter2dOut fo = gs_filter2d(filt, o.a, o.b, o.c, o.d);
  const double A = (double)fo.a * fx * fx, B = (double)o.b * fx * fy, D = (double)fo.d * fy * fy;
  const double h = 0.5 * (A - D);
  const double lmax = 0.5 * (A + D) + sqrt(h * h + B * B);
  const float rad = (float)ceil(3.0 * sqrt(fmax(lmax, 0.0)));
  grad2d[i] += sqrtf((gx * sx) * (gx * sx) + (gy * sy) * (gy * sy));
  if constexpr (ABS) absgrad[i] += sqrtf((ax * sx) * (ax * sx) + (ay * sy) * (ay * sy));
  n_views[i] += 1;
  max_radius[i] = fmaxf(max_radius[i], rad);
}

template <bool ABS>
__global__ void __launch_bounds__(kBlock) densify_stats_kernel(GS_STATS_PARAMS) {
  densify_stats_body<ABS, false>(GS_STATS_ARGS, nullptr);
}

template <bool ABS>
__global__ void __launch_bounds__(kBlock) densify_stats_filt3_kernel(GS_STATS_PARAMS, const float* __restrict__ f3d) {
  densify_stats_body<ABS, true>(GS_STATS_ARGS, f3d);
}

template <bool ABS>
__global__ void __launch_bounds__(kBlock) densify_stats_lens_kernel(GS_STATS_PARAMS, const float* __restrict__ f3d,
                                                                    GsLens lens) {
  densify_stats_body<ABS, true, true>(GS_STATS_ARGS, f3d, lens);
}
#undef GS_STATS_ARGS
#undef GS_STATS_PARAMS

// Batched frame: Gaussian i's views in view order, each one's statistics formed as densify_stats_kernel forms them
// (pair v n + i, view v's camera, filter and (sx, sy) = (W / (2 fx), H / (2 fy))) and added to running values that are
// loaded and stored once: the result of B single-view backwards run in view order.  G3 as above.
#define GS_STATS_BATCH_PARAMS                                                                                        \
  const float* __restrict__ pos, const float* __restrict__ quat, const float* __restrict__ scale, int n, int n_views, \
      int scale_act, const GsView* __restrict__ views, float near_plane, const uint32_t* __restrict__ offsets_g,    \
      const uint32_t* __restrict__ count, const float* __restrict__ grad_inst, int gw,                              \
      const uint32_t* __restrict__ row_epoch, uint32_t epoch, int width, int height, float* __restrict__ grad2d,    \
      float* __restrict__ absgrad, int* __restrict__ n_views_out, float* __restrict__ max_radius
#define GS_STATS_BATCH_ARGS                                                                                       \
  pos, quat, scale, n, n_views, scale_act, views, near_plane, offsets_g, count, grad_inst, gw, row_epoch, epoch,   \
      width, height, grad2d, absgrad, n_views_out, max_radius
template <bool ABS, bool G3, bool L = false>
__device__ __forceinline__ void densify_stats_batch_body(GS_STATS_BATCH_PARAMS, const float* __restrict__ f3d,
                                                         const GsLens* __restrict__ lenses = nullptr) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  float q[4], s[3], raw_s[3], qn;
  gs_load_activated(quat, scale, i, scale_act, q, s, raw_s, qn);
  if constexpr (G3) {
    float s0[3], dl2o3;
    gs_filter3d((L && !f3d) ? 0.f : f3d[i], s, s0, dl2o3);
  }
  float g2 = grad2d[i], ga = ABS ? absgrad[i] : 0.f, mr = max_radius[i];
  int nv = n_views_out[i];
  bool any = false;
  for (int v = 0; v < n_views; ++v) {
    const int j = v * n + i;
    const uint32_t cnt = count[j];
    if (cnt == 0) continue;
    any = true;
    const GsView vw = views[v];
    const float sx = (float)((double)width / (2.0 * (double)vw.fx));
    const float sy = (float)((double)height / (2.0 * (double)vw.fy));
    float gx = 0.f, gy = 0.f, ax = 0.f, ay = 0.f;
    const uint32_t o0 = offsets_g[j], o1 = o0 + cnt;
    for (uint32_t r = o0; r < o1; ++r) {
      if (row_epoch[r] != epoch) continue;
      const float* row = grad_inst + (size_t)r * gw;
      const float2 g = *reinterpret_cast<const float2*>(row);
      gx += g.x;
      gy += g.y;
      if constexpr (ABS) {
        const float2 a = *reinterpret_cast<const float2*>(row + 10);
        ax += a.x;
        ay += a.y;
      }
    }
    GsProj o = gs_project(vw.cam, p, q, s, near_plane, L ? kInf : vw.half_w, L ? kInf : vw.half_h);
    if constexpr (L) {
      float J[4];
      gs_lens_project(lenses[v], o, vw.half_w, vw.half_h, J);
    }
    const GsFilter2dOut fo = gs_filter2d(vw.filt, o.a, o.b, o.c, o.d);
    const float fx = vw.fx, fy = vw.fy;
    const double A = (double)fo.a * fx * fx, B = (double)o.b * fx * fy, D = (double)fo.d * fy * fy;
    const double h = 0.5 * (A - D);
    const double lmax = 0.5 * (A + D) + sqrt(h * h + B * B);
    const float rad = (float)ceil(3.0 * sqrt(fmax(lmax, 0.0)));
    g2 += sqrtf((gx * sx) * (gx * sx) + (gy * sy) * (gy * sy));
    if constexpr (ABS) ga += sqrtf((ax * sx) * (ax * sx) + (ay * sy) * (ay * sy));
    nv += 1;
    mr = fmaxf(mr, rad);
  }
  if (!any) return;
  grad2d[i] = g2;
  if constexpr (ABS) absgrad[i] = ga;
  n_views_out[i] = nv;
  max_radius[i] = mr;
}

template <bool ABS>
__global__ void __launch_bounds__(kBlock) densify_stats_batch_kernel(GS_STATS_BATCH_PARAMS) {
  densify_stats_batch_body<ABS, false>(GS_STATS_BATCH_ARGS, nullptr);
}

template <bool ABS>
__global__ void __launch_bounds__(kBlock) densify_stats_batch_filt3_kernel(GS_STATS_BATCH_PARAMS,
                                                                           const float* __restrict__ f3d) {
  densify_stats_batch_body<ABS, true>(GS_STATS_BATCH_ARGS, f3d);
}

template <bool ABS>
__global__ void __launch_bounds__(kBlock) densify_stats_batch_lens_kernel(GS_STATS_BATCH_PARAMS,
                                                                          const float* __restrict__ f3d,
                                                                          const GsLens* __restrict__ lenses) {
  densify_stats_batch_body<ABS, true, true>(GS_STATS_BATCH_ARGS, f3d, lenses);
}
#undef GS_STATS_BATCH_ARGS
#undef GS_STATS_BATCH_PARAMS

}  // namespace

cudaError_t gs_launch_densify_stats_batch(const float* pos, const float* quat, const float* scale, int n, int n_views,
                                          int scale_act, const GsView* views, float near_plane,
                                          const uint32_t* offsets_g, const uint32_t* count, const float* grad_inst,
                                          int gw, const uint32_t* row_epoch, uint32_t epoch, const GsFrameGeom& g,
                                          const gs_densify_stats& s, cudaStream_t st, const float* f3d,
                                          const GsLens* lenses) {
  if (n == 0) return cudaSuccess;
  const int blocks = (n + kBlock - 1) / kBlock;
  if (lenses) {
#define GS_LAUNCH_STATS_BATCHL(ABS)                                                                                \
  densify_stats_batch_lens_kernel<ABS><<<blocks, kBlock, 0, st>>>(                                                  \
      pos, quat, scale, n, n_views, scale_act, views, near_plane, offsets_g, count, grad_inst, gw, row_epoch, epoch, \
      g.width, g.height, s.grad2d, s.absgrad, s.count, s.max_radius, f3d, lenses)
    if (s.absgrad) GS_LAUNCH_STATS_BATCHL(true);
    else GS_LAUNCH_STATS_BATCHL(false);
#undef GS_LAUNCH_STATS_BATCHL
    return cudaGetLastError();
  }
#define GS_LAUNCH_STATS_BATCH(ABS)                                                                                 \
  densify_stats_batch_kernel<ABS><<<blocks, kBlock, 0, st>>>(pos, quat, scale, n, n_views, scale_act, views,       \
                                                             near_plane, offsets_g, count, grad_inst, gw, row_epoch, \
                                                             epoch, g.width, g.height, s.grad2d, s.absgrad, s.count, \
                                                             s.max_radius)
#define GS_LAUNCH_STATS_BATCH3(ABS)                                                                                \
  densify_stats_batch_filt3_kernel<ABS><<<blocks, kBlock, 0, st>>>(                                                 \
      pos, quat, scale, n, n_views, scale_act, views, near_plane, offsets_g, count, grad_inst, gw, row_epoch, epoch, \
      g.width, g.height, s.grad2d, s.absgrad, s.count, s.max_radius, f3d)
  if (f3d && s.absgrad) GS_LAUNCH_STATS_BATCH3(true);
  else if (f3d) GS_LAUNCH_STATS_BATCH3(false);
  else if (s.absgrad) GS_LAUNCH_STATS_BATCH(true);
  else GS_LAUNCH_STATS_BATCH(false);
#undef GS_LAUNCH_STATS_BATCH3
#undef GS_LAUNCH_STATS_BATCH
  return cudaGetLastError();
}

cudaError_t gs_launch_densify_stats(const float* pos, const float* quat, const float* scale, int n, int scale_act,
                                    const GsCam& cam, float near_plane, float half_w, float half_h,
                                    const GsFilter2d& filt, const uint32_t* offsets_g, const uint32_t* count,
                                    const float* grad_inst, int gw, const uint32_t* row_epoch, uint32_t epoch,
                                    const GsFrameGeom& g, const gs_densify_stats& s, cudaStream_t st,
                                    const float* f3d, const GsLens* lens) {
  if (n == 0) return cudaSuccess;
  const float sx = (float)((double)g.width / (2.0 * (double)g.fx));
  const float sy = (float)((double)g.height / (2.0 * (double)g.fy));
  const int blocks = (n + kBlock - 1) / kBlock;
  if (lens) {
#define GS_LAUNCH_STATSL(ABS)                                                                                      \
  densify_stats_lens_kernel<ABS><<<blocks, kBlock, 0, st>>>(pos, quat, scale, n, scale_act, cam, near_plane,       \
                                                            half_w, half_h, filt, offsets_g, count, grad_inst, gw,  \
                                                            row_epoch, epoch, sx, sy, g.fx, g.fy, s.grad2d,        \
                                                            s.absgrad, s.count, s.max_radius, f3d, *lens)
    if (s.absgrad) GS_LAUNCH_STATSL(true);
    else GS_LAUNCH_STATSL(false);
#undef GS_LAUNCH_STATSL
    return cudaGetLastError();
  }
#define GS_LAUNCH_STATS(ABS)                                                                                       \
  densify_stats_kernel<ABS><<<blocks, kBlock, 0, st>>>(pos, quat, scale, n, scale_act, cam, near_plane, half_w,    \
                                                       half_h, filt, offsets_g, count, grad_inst, gw, row_epoch,   \
                                                       epoch, sx, sy, g.fx, g.fy, s.grad2d, s.absgrad, s.count,    \
                                                       s.max_radius)
#define GS_LAUNCH_STATS3(ABS)                                                                                      \
  densify_stats_filt3_kernel<ABS><<<blocks, kBlock, 0, st>>>(pos, quat, scale, n, scale_act, cam, near_plane,      \
                                                             half_w, half_h, filt, offsets_g, count, grad_inst, gw, \
                                                             row_epoch, epoch, sx, sy, g.fx, g.fy, s.grad2d,       \
                                                             s.absgrad, s.count, s.max_radius, f3d)
  if (f3d && s.absgrad) GS_LAUNCH_STATS3(true);
  else if (f3d) GS_LAUNCH_STATS3(false);
  else if (s.absgrad) GS_LAUNCH_STATS(true);
  else GS_LAUNCH_STATS(false);
#undef GS_LAUNCH_STATS3
#undef GS_LAUNCH_STATS
  return cudaGetLastError();
}
