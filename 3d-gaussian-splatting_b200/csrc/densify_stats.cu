// Screen-space densification statistics of the fused frame path (gs_ctx_set_densify_stats): one thread per Gaussian
// after the projection backward, accumulating into the caller's buffers.  A kernel of its own, not a flag on the
// projection backward: that kernel has more than 100 instantiations (KG, D, GW, W, DT, TIER, CG), and this one kernel
// follows every one of them, the data-parallel push included.
#include "internal.h"

#include <type_traits>

namespace {

constexpr int kBlock = 256;
constexpr float kInf = __builtin_huge_valf();   // gs_project's frustum half-widths in a lens frame (gs_lens_project)

// One view's terms of Gaussian i's statistics (loaded parameters p, q, s, the 3-D filtered scale at
// TIER >= GS_TIER_FILT3D), from its rows o0 .. o1 - 1 in a view where it got at least one tile instance in the forward:
//   grad2d  += |(gx sx, gy sy)|, (gx, gy) = sum of columns 0, 1 over its rows tagged with this backward's epoch
//   absgrad += |(Ax sx, Ay sy)|, (Ax, Ay) = the same sums of columns 10, 11 (ABS: sum_p |g_x,p|, sum_p |g_y,p|)
//   count   += 1
//   max_radius = max(max_radius, ceil(3 sqrt(lambda_max))) of the 2-D covariance the forward binned, in px^2
// (sx, sy) = (W / (2 fx), H / (2 fy)) converts dL/d(x/z, y/z) to the NDC convention of 3DGS's viewspace gradient.
// One thread owns one Gaussian and sums its rows in order: bit-deterministic, no atomics.
// TIER: the forward's, at least GS_TIER_FILT2D (a zero filter leaves the covariance as it is).  GS_TIER_LENS: the
// covariance is the lensed one (gs_lens_project); (x, y) stays the stored mean's gradient.
struct StatsTerms {
  float grad2d, absgrad, radius;
};

template <bool ABS, int TIER>
__device__ __forceinline__ StatsTerms densify_stats_one(const GsCam& cam, float near_plane, float half_w, float half_h,
                                                  const GsFilter2d& filt, const GsLens* __restrict__ lens, float sx, float sy,
                                                  float fx, float fy, const float p[3], const float q[4],
                                                  const float s[3], uint32_t o0, uint32_t o1,
                                                  const float* __restrict__ grad_inst, int gw,
                                                  const uint32_t* __restrict__ row_epoch, uint32_t epoch) {
  constexpr bool L = TIER == GS_TIER_LENS;
  float gx = 0.f, gy = 0.f, ax = 0.f, ay = 0.f;
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
    gs_lens_project(*lens, o, half_w, half_h, J);
  }
  const GsFilter2dOut fo = gs_filter2d(filt, o.a, o.b, o.c, o.d);
  const double A = (double)fo.a * fx * fx, B = (double)o.b * fx * fy, D = (double)fo.d * fy * fy;
  const double h = 0.5 * (A - D);
  const double lmax = 0.5 * (A + D) + sqrt(h * h + B * B);
  const float rad = (float)ceil(3.0 * sqrt(fmax(lmax, 0.0)));
  StatsTerms t;
  t.grad2d = sqrtf((gx * sx) * (gx * sx) + (gy * sy) * (gy * sy));
  t.absgrad = ABS ? sqrtf((ax * sx) * (ax * sx) + (ay * sy) * (ay * sy)) : 0.f;
  t.radius = rad;
  return t;
}

// Gaussian i's parameters, its scale 3-D filtered at TIER >= GS_TIER_FILT3D (f3d NULL in a lens frame without one)
template <int TIER>
__device__ __forceinline__ void densify_stats_load(const float* __restrict__ pos, const float* __restrict__ quat,
                                                   const float* __restrict__ scale, const float* __restrict__ f3d,
                                                   int i, int scale_act, float p[3], float q[4], float s[3]) {
  p[0] = pos[3 * i];
  p[1] = pos[3 * i + 1];
  p[2] = pos[3 * i + 2];
  float raw_s[3], qn;
  gs_load_activated(quat, scale, i, scale_act, q, s, raw_s, qn);
  if constexpr (TIER >= GS_TIER_FILT3D) {
    float s0[3], dl2o3;
    gs_filter3d((TIER == GS_TIER_LENS && !f3d) ? 0.f : f3d[i], s, s0, dl2o3);
  }
}

// Single-view frame: Gaussian i with count[i] > 0 adds its statistics to the caller's buffers.
template <bool ABS, int TIER>
__global__ void __launch_bounds__(kBlock) densify_stats_kernel(
    const float* __restrict__ pos, const float* __restrict__ quat, const float* __restrict__ scale, int n,
    int scale_act, GsCam cam, float near_plane, float half_w, float half_h, GsFilter2d filt,
    const uint32_t* __restrict__ offsets_g, const uint32_t* __restrict__ count, const float* __restrict__ grad_inst,
    int gw, const uint32_t* __restrict__ row_epoch, uint32_t epoch, float sx, float sy, float fx, float fy,
    float* __restrict__ grad2d, float* __restrict__ absgrad, int* __restrict__ n_views, float* __restrict__ max_radius,
    const float* __restrict__ f3d, GsLens lens) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const uint32_t cnt = count[i];
  if (cnt == 0) return;
  float p[3], q[4], s[3];
  densify_stats_load<TIER>(pos, quat, scale, f3d, i, scale_act, p, q, s);
  const uint32_t o0 = offsets_g[i];
  const StatsTerms t = densify_stats_one<ABS, TIER>(cam, near_plane, half_w, half_h, filt, &lens, sx, sy, fx, fy, p,
                                                    q, s, o0, o0 + cnt, grad_inst, gw, row_epoch, epoch);
  grad2d[i] += t.grad2d;
  if constexpr (ABS) absgrad[i] += t.absgrad;
  n_views[i] += 1;
  max_radius[i] = fmaxf(max_radius[i], t.radius);
}

// Batched frame: Gaussian i's views in view order, each one's statistics formed as in a single-view frame (pair v n + i,
// view v's camera, filter, lens lenses[v] and (sx, sy) = (W / (2 fx), H / (2 fy))) and added to running values that are
// loaded and stored once: the result of B single-view backwards run in view order.
template <bool ABS, int TIER>
__global__ void __launch_bounds__(kBlock) densify_stats_batch_kernel(
    const float* __restrict__ pos, const float* __restrict__ quat, const float* __restrict__ scale, int n, int n_views,
    int scale_act, const GsView* __restrict__ views, float near_plane, const uint32_t* __restrict__ offsets_g,
    const uint32_t* __restrict__ count, const float* __restrict__ grad_inst, int gw,
    const uint32_t* __restrict__ row_epoch, uint32_t epoch, int width, int height, float* __restrict__ grad2d,
    float* __restrict__ absgrad, int* __restrict__ n_views_out, float* __restrict__ max_radius,
    const float* __restrict__ f3d, const GsLens* __restrict__ lenses) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float p[3], q[4], s[3];
  densify_stats_load<TIER>(pos, quat, scale, f3d, i, scale_act, p, q, s);
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
    const uint32_t o0 = offsets_g[j];
    const StatsTerms t = densify_stats_one<ABS, TIER>(vw.cam, near_plane, vw.half_w, vw.half_h, vw.filt, lenses + v, sx, sy,
                                                      vw.fx, vw.fy, p, q, s, o0, o0 + cnt, grad_inst, gw, row_epoch,
                                                      epoch);
    g2 += t.grad2d;
    if constexpr (ABS) ga += t.absgrad;
    nv += 1;
    mr = fmaxf(mr, t.radius);
  }
  if (!any) return;
  grad2d[i] = g2;
  if constexpr (ABS) absgrad[i] = ga;
  n_views_out[i] = nv;
  max_radius[i] = mr;
}

// The statistics kernels' one map from a frame's configuration to an instantiation: calls launch(ABS, TIER), each a
// std::integral_constant.  The 2-D filter always runs (a zero filter gives its bits), so a frame without one takes the
// GS_TIER_FILT2D kernels.
template <class Launch>
cudaError_t densify_stats_dispatch(bool abs, const float* f3d, bool lens, Launch&& launch) {
  auto by_tier = [&](auto a) {
    switch (gs_tier(true, f3d, lens)) {
      case GS_TIER_LENS: launch(a, std::integral_constant<int, GS_TIER_LENS>{}); break;
      case GS_TIER_FILT3D: launch(a, std::integral_constant<int, GS_TIER_FILT3D>{}); break;
      default: launch(a, std::integral_constant<int, GS_TIER_FILT2D>{}); break;
    }
    return cudaGetLastError();
  };
  return abs ? by_tier(std::true_type{}) : by_tier(std::false_type{});
}

}  // namespace

cudaError_t gs_launch_densify_stats_batch(const float* pos, const float* quat, const float* scale, int n, int n_views,
                                          int scale_act, const GsView* views, float near_plane,
                                          const uint32_t* offsets_g, const uint32_t* count, const float* grad_inst,
                                          int gw, const uint32_t* row_epoch, uint32_t epoch, const GsFrameGeom& g,
                                          const gs_densify_stats& s, cudaStream_t st, const float* f3d,
                                          const GsLens* lenses) {
  if (n == 0) return cudaSuccess;
  const int blocks = (n + kBlock - 1) / kBlock;
  return densify_stats_dispatch(s.absgrad, f3d, lenses, [&](auto abs, auto t) {
    densify_stats_batch_kernel<abs, t><<<blocks, kBlock, 0, st>>>(
        pos, quat, scale, n, n_views, scale_act, views, near_plane, offsets_g, count, grad_inst, gw, row_epoch, epoch,
        g.width, g.height, s.grad2d, s.absgrad, s.count, s.max_radius, f3d, lenses);
  });
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
  const GsLens ln = lens ? *lens : GsLens{};
  return densify_stats_dispatch(s.absgrad, f3d, lens, [&](auto abs, auto t) {
    densify_stats_kernel<abs, t><<<blocks, kBlock, 0, st>>>(pos, quat, scale, n, scale_act, cam, near_plane, half_w,
                                                            half_h, filt, offsets_g, count, grad_inst, gw, row_epoch,
                                                            epoch, sx, sy, g.fx, g.fy, s.grad2d, s.absgrad, s.count,
                                                            s.max_radius, f3d, ln);
  });
}
