// Mip-Splatting's 3-D smoothing filter: the per-Gaussian maximal sampling rate over a set of views
// (gs_filter3d_compute).  Two launches: one thread per Gaussian takes every view (staged through shared memory in
// chunks) and keeps the largest fx / z among the views that see it, writing f = sqrt(v) / nu for a seen Gaussian and
// block-reducing the smallest seen rate into one u32 (atomicMin over positive float bits); the second launch gives
// every unseen Gaussian the filter of that smallest rate.  Max and min are order-independent and every rate is one
// correctly rounded fp64 division, so the result is the same bits for any order of the views, on every call.
#include "internal.h"

namespace {

constexpr int kBlock = 256;
constexpr int kChunk = 64;   // views staged in shared memory per pass (64 x 112 bytes)

static_assert(sizeof(GsF3View) % 4 == 0 && sizeof(GsLens) % 4 == 0, "views are staged as 4-byte words");

__global__ void __launch_bounds__(kBlock) filter3d_rate_kernel(const float* __restrict__ pos, int n,
                                                                const GsF3View* __restrict__ views, int n_views,
                                                                double sqrt_v, float* __restrict__ f3d,
                                                                unsigned int* __restrict__ min_rate) {
  __shared__ GsF3View sv[kChunk];
  __shared__ unsigned int wmin[kBlock / 32];
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const bool valid = i < n;
  float p[3] = {0.f, 0.f, 0.f};
  if (valid) {
    p[0] = pos[3 * i];
    p[1] = pos[3 * i + 1];
    p[2] = pos[3 * i + 2];
  }
  const double pd[3] = {(double)p[0], (double)p[1], (double)p[2]};
  double best = 0.0;   // the largest seen fx / z (0: not seen)
  float best_f = 0.f;  // (float)best
  for (int v0 = 0; v0 < n_views; v0 += kChunk) {
    const int nc = min(kChunk, n_views - v0);
    __syncthreads();   // the previous chunk's readers are done
    const uint32_t* src = reinterpret_cast<const uint32_t*>(views + v0);
    uint32_t* dst = reinterpret_cast<uint32_t*>(sv);
    for (int w = threadIdx.x; w < nc * (int)(sizeof(GsF3View) / 4); w += kBlock) dst[w] = src[w];
    __syncthreads();
    if (!valid) continue;
    for (int c = 0; c < nc; ++c) {
      const GsF3View& vw = sv[c];
      // depth in fp64 (the sampling rate's), the image-plane position in fp32 (only the margin test reads it)
      const double zd = fma(vw.rz[0], pd[0], fma(vw.rz[1], pd[1], fma(vw.rz[2], pd[2], vw.tz)));
      if (!(zd > vw.near)) continue;
      const float z = (float)zd;
      const float x = fmaf(vw.r[0], p[0], fmaf(vw.r[1], p[1], fmaf(vw.r[2], p[2], vw.t[0])));
      const float y = fmaf(vw.r[3], p[0], fmaf(vw.r[4], p[1], fmaf(vw.r[5], p[2], vw.t[1])));
      const float u = vw.fx * (x / z) + vw.cx;
      const float w = vw.fy * (y / z) + vw.cy;
      if (!(u >= vw.ulo && u <= vw.uhi && w >= vw.wlo && w <= vw.whi)) continue;
      // fx / z in fp32 is within 2e-7 of the fp64 rate: only a view that may beat the best pays the fp64 division
      if (vw.fx / z >= best_f * 0.99999f) {
        const double nu = vw.fxd / zd;
        if (nu > best) {
          best = nu;
          best_f = (float)nu;
        }
      }
    }
  }
  if (valid) f3d[i] = best > 0.0 ? (float)(sqrt_v / best) : -1.f;   // -1: not seen, filled by filter3d_fill_kernel
  // the smallest seen rate, as positive float bits (their order is the floats')
  unsigned int bits = (valid && best > 0.0) ? __float_as_uint(best_f) : 0xffffffffu;
  bits = __reduce_min_sync(0xffffffffu, bits);
  if ((threadIdx.x & 31) == 0) wmin[threadIdx.x >> 5] = bits;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int m = wmin[0];
#pragma unroll
    for (int k = 1; k < kBlock / 32; ++k) m = min(m, wmin[k]);
    if (m != 0xffffffffu) atomicMin(min_rate, m);
  }
}

// With lenses (gs_ctx_set_lens): lenses[v] is view v's (its cx, cy in the view are the lens's principal point).  View v
// sees Gaussian i when z > near, rho^2 < rho2_max and the distorted pixel position fx a_d + cx, fy b_d + cy lies inside
// the widened image.  The rate is fx / z for PINHOLE and OPENCV (Mip-Splatting's, which ignores distortion) and
// fx max(theta_d'(theta), theta_d(theta) / sin theta) / |p_c| for FISHEYE (the larger of its radial and tangential
// magnifications; fx / z on the axis), both in fp64.
__global__ void __launch_bounds__(kBlock) filter3d_rate_lens_kernel(const float* __restrict__ pos, int n,
                                                                     const GsF3View* __restrict__ views,
                                                                     const GsLens* __restrict__ lenses, int n_views,
                                                                     double sqrt_v, float* __restrict__ f3d,
                                                                     unsigned int* __restrict__ min_rate) {
  __shared__ GsF3View sv[kChunk];
  __shared__ GsLens sl[kChunk];
  __shared__ unsigned int wmin[kBlock / 32];
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const bool valid = i < n;
  float p[3] = {0.f, 0.f, 0.f};
  if (valid) {
    p[0] = pos[3 * i];
    p[1] = pos[3 * i + 1];
    p[2] = pos[3 * i + 2];
  }
  const double pd[3] = {(double)p[0], (double)p[1], (double)p[2]};
  double best = 0.0;   // the largest seen rate (0: not seen)
  for (int v0 = 0; v0 < n_views; v0 += kChunk) {
    const int nc = min(kChunk, n_views - v0);
    __syncthreads();   // the previous chunk's readers are done
    const uint32_t* src = reinterpret_cast<const uint32_t*>(views + v0);
    uint32_t* dst = reinterpret_cast<uint32_t*>(sv);
    for (int w = threadIdx.x; w < nc * (int)(sizeof(GsF3View) / 4); w += kBlock) dst[w] = src[w];
    const uint32_t* lsrc = reinterpret_cast<const uint32_t*>(lenses + v0);
    uint32_t* ldst = reinterpret_cast<uint32_t*>(sl);
    for (int w = threadIdx.x; w < nc * (int)(sizeof(GsLens) / 4); w += kBlock) ldst[w] = lsrc[w];
    __syncthreads();
    if (!valid) continue;
    for (int c = 0; c < nc; ++c) {
      const GsF3View& vw = sv[c];
      const GsLens& ln = sl[c];
      const double zd = fma(vw.rz[0], pd[0], fma(vw.rz[1], pd[1], fma(vw.rz[2], pd[2], vw.tz)));
      if (!(zd > vw.near)) continue;
      const float z = (float)zd;
      const float x = fmaf(vw.r[0], p[0], fmaf(vw.r[1], p[1], fmaf(vw.r[2], p[2], vw.t[0])));
      const float y = fmaf(vw.r[3], p[0], fmaf(vw.r[4], p[1], fmaf(vw.r[5], p[2], vw.t[1])));
      const float a = x / z, b = y / z;
      if (!(a * a + b * b < ln.rho2_max)) continue;
      float ad, bd, J[4];
      gs_lens_map(ln, a, b, ad, bd, J);
      const float u = vw.fx * ad + vw.cx;
      const float w = vw.fy * bd + vw.cy;
      if (!(u >= vw.ulo && u <= vw.uhi && w >= vw.wlo && w <= vw.whi)) continue;
      double nu;
      if (ln.model == GS_LENS_FISHEYE) {
        double xy[2];   // x and y in fp64, like z
#pragma unroll
        for (int j = 0; j < 2; ++j)
          xy[j] = fma((double)vw.r[3 * j], pd[0],
                      fma((double)vw.r[3 * j + 1], pd[1], fma((double)vw.r[3 * j + 2], pd[2], (double)vw.t[j])));
        const double xd = xy[0], yd = xy[1];
        const double rr = sqrt(xd * xd + yd * yd);
        const double th = atan2(rr, zd), t2 = th * th;
        const double k1 = ln.k[0], k2 = ln.k[1], k3 = ln.k[2], k4 = ln.k[3];
        const double poly = 1.0 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)));
        const double dpoly = 1.0 + t2 * (3.0 * k1 + t2 * (5.0 * k2 + t2 * (7.0 * k3 + t2 * 9.0 * k4)));
        const double tang = th > 0.0 ? th * poly / sin(th) : 1.0;
        nu = vw.fxd * fmax(dpoly, tang) / sqrt(rr * rr + zd * zd);
      } else {
        nu = vw.fxd / zd;
      }
      best = fmax(best, nu);
    }
  }
  if (valid) f3d[i] = best > 0.0 ? (float)(sqrt_v / best) : -1.f;   // -1: not seen, filled by filter3d_fill_kernel
  unsigned int bits = (valid && best > 0.0) ? __float_as_uint((float)best) : 0xffffffffu;
  bits = __reduce_min_sync(0xffffffffu, bits);
  if ((threadIdx.x & 31) == 0) wmin[threadIdx.x >> 5] = bits;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int m = wmin[0];
#pragma unroll
    for (int k = 1; k < kBlock / 32; ++k) m = min(m, wmin[k]);
    if (m != 0xffffffffu) atomicMin(min_rate, m);
  }
}

// A Gaussian no view sees gets the largest filter, that of the smallest seen rate; none seen at all: 0
__global__ void __launch_bounds__(kBlock) filter3d_fill_kernel(float* __restrict__ f3d, int n,
                                                                const unsigned int* __restrict__ min_rate,
                                                                double sqrt_v) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n || !(f3d[i] < 0.f)) return;
  const unsigned int b = *min_rate;
  f3d[i] = b == 0xffffffffu ? 0.f : (float)(sqrt_v / (double)__uint_as_float(b));
}

}  // namespace

cudaError_t gs_launch_filter3d(const float* pos, int n, const GsF3View* views, int n_views, float variance,
                               float* f3d, unsigned int* min_rate, cudaStream_t st, const GsLens* lenses) {
  if (n == 0) return cudaSuccess;
  const double sqrt_v = sqrt((double)variance);
  const int blocks = (n + kBlock - 1) / kBlock;
  if (lenses)
    filter3d_rate_lens_kernel<<<blocks, kBlock, 0, st>>>(pos, n, views, lenses, n_views, sqrt_v, f3d, min_rate);
  else
    filter3d_rate_kernel<<<blocks, kBlock, 0, st>>>(pos, n, views, n_views, sqrt_v, f3d, min_rate);
  filter3d_fill_kernel<<<blocks, kBlock, 0, st>>>(f3d, n, min_rate, sqrt_v);
  return cudaGetLastError();
}
