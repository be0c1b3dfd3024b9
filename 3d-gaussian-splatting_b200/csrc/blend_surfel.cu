// Blend of 2D Gaussian surfels (gs_render_forward_surfel / gs_render_backward_surfel), gather path: each CTA is one
// 16x16 tile, one pixel per thread; the tile's records are gathered from rec[N] through the sorted id list into shared
// memory chunk by chunk.  Per (pixel q, surfel) with M = [u | v | p_c] (rows m_x, m_y, m_z):
//   k = qx m_z - m_x, l = qy m_z - m_y, h = k x l, (a, b) = (h0, h1) / h2, rho3 = a^2 + b^2 (+inf when h2 == 0),
//   z3 = m_z . (a, b, 1);  low-pass: c = (M02, M12) / M22, rho2 = 2 ((qx - cx)^2 fx^2 + (qy - cy)^2 fy^2);
//   rho2 < rho3: (rho, z) = (rho2, M22), else (rho3, z3) (the choice has no gradient);
//   alpha = min(0.99, op exp(-rho / 2)); alpha < 1/255 is skipped, and so is a hit at z <= near (a disk whose plane
//   crosses the camera plane can be met behind the camera past its 3-sigma edge); the stop T <= 1e-4 is tested before
//   an instance.
// MAPS: also alpha, depth = sum w z, the median depth (z of the last blended instance with T > 0.5 before it), the
// distortion sum_i w_i sum_{j<i} w_j (m_i - m_j)^2 (running sums A, D, D2; m = f / (f - n) (1 - n / z)) and the
// normal sum w n.  The distortion depends only on differences of m, so D and D2 are summed over m - m_0 with m_0 the m
// of the pixel's first blended instance: the fp32 cancellation in m^2 A - 2 m D + D2 then scales with the spread of m,
// not with m itself (the backward re-derives m_0 from the same arithmetic).
#include "internal.h"
#include "sh_common.cuh"

namespace {

using gs_sh::reduce8;

constexpr int kNT = GS_TILE * GS_TILE;
constexpr int kNW = kNT / 32;
constexpr float kAlphaMin = 1.f / 255.f;

// one (pixel, surfel) evaluation; the backward also reads the intermediates
struct SurfelHit {
  float k[3], l[3], h[3], a, b;
  float dx, dy;      // low-pass: pixel offsets from the centre (px)
  float rho, z, g;   // g = exp(-rho / 2), 0 at z <= near
  bool lowpass;
};

__device__ __forceinline__ SurfelHit surfel_hit(const float* M, float qx, float qy, float fx, float fy, float near) {
  SurfelHit s;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    s.k[j] = qx * M[6 + j] - M[j];
    s.l[j] = qy * M[6 + j] - M[3 + j];
  }
  s.h[0] = s.k[1] * s.l[2] - s.k[2] * s.l[1];
  s.h[1] = s.k[2] * s.l[0] - s.k[0] * s.l[2];
  s.h[2] = s.k[0] * s.l[1] - s.k[1] * s.l[0];
  float rho3 = __builtin_huge_valf();
  s.a = 0.f;
  s.b = 0.f;
  if (s.h[2] != 0.f) {
    s.a = s.h[0] / s.h[2];
    s.b = s.h[1] / s.h[2];
    rho3 = s.a * s.a + s.b * s.b;
  }
  const float cx = M[2] / M[8], cy = M[5] / M[8];
  s.dx = (qx - cx) * fx;
  s.dy = (qy - cy) * fy;
  const float rho2 = 2.f * (s.dx * s.dx + s.dy * s.dy);
  s.lowpass = rho2 < rho3;
  if (s.lowpass) {
    s.rho = rho2;
    s.z = M[8];
  } else {
    s.rho = rho3;
    s.z = M[6] * s.a + M[7] * s.b + M[8];
  }
  s.g = s.z > near ? expf(-0.5f * s.rho) : 0.f;   // a hit at z <= near: alpha 0, skipped
  return s;
}

// chunk of CH records of the tile (first = index of the chunk's first instance in the sorted list) into shared memory
template <int CH>
__device__ __forceinline__ void load_chunk(float4* dst, const GsSurfelRec* __restrict__ rec,
                                           const uint32_t* __restrict__ ids, int first, int n, int tid) {
  for (int t = tid; t < n * 4; t += kNT) {
    const uint32_t id = __ldg(ids + first + t / 4);
    dst[t] = __ldg(reinterpret_cast<const float4*>(rec + id) + (t & 3));
  }
}

template <bool MAPS>
__global__ void __launch_bounds__(kNT) blend_surfel_fwd_kernel(
    const GsSurfelRec* __restrict__ rec, const uint32_t* __restrict__ ids, const int* __restrict__ tile_accum, int wp,
    int hp, int ntx, float fx, float fy, float3 bg, float* __restrict__ image, float* __restrict__ final_img,
    GsCrop crop, GsSurfelMaps mp, float dA, float dB, float near, float4* __restrict__ ws, float4* __restrict__ wsm,
    int* __restrict__ tile_neff) {
  constexpr int CH = 64;
  __shared__ __align__(16) GsSurfelRec sr[CH];
  const int tile = blockIdx.x, tid = threadIdx.x;
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix = tx * GS_TILE + (tid % GS_TILE), iy = ty * GS_TILE + tid / GS_TILE;
  const float qx = gs_pixel_coord(ix, wp, fx), qy = gs_pixel_coord(iy, hp, fy);
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  float T = 1.f, C[3] = {0.f, 0.f, 0.f};
  float Z = 0.f, A = 0.f, D = 0.f, D2 = 0.f, dist = 0.f, N[3] = {0.f, 0.f, 0.f}, med = 0.f;
  int med_idx = -1;
  float m0 = __int_as_float(0x7fffffff);   // m of the first blended instance (NaN: none yet)
  bool done = false;
  int consumed = cnt;
  for (int base = 0; base < cnt; base += CH) {
    if (__syncthreads_count(!done) == 0) {   // also: every thread is done with the previous chunk
      consumed = base;
      break;
    }
    const int n = min(CH, cnt - base);
    load_chunk<CH>(reinterpret_cast<float4*>(sr), rec, ids, start + base, n, tid);
    __syncthreads();
    for (int j = 0; j < n && !done; ++j) {
      if (!(T > GS_T_STOP)) {
        done = true;
        break;
      }
      const GsSurfelRec& r = sr[j];
      const SurfelHit s = surfel_hit(r.M, qx, qy, fx, fy, near);
      const float alpha = fminf(0.99f, r.op * s.g);
      if (alpha < kAlphaMin) continue;
      const float w = alpha * T;
#pragma unroll
      for (int c = 0; c < 3; ++c) C[c] = fmaf(w, r.rgb[c], C[c]);
      if constexpr (MAPS) {
        const float mr = dA - dB / s.z;
        if (m0 != m0) m0 = mr;
        const float m = mr - m0;
        dist = fmaf(w, fmaf(m, fmaf(m, A, -2.f * D), D2), dist);
        A += w;
        D = fmaf(w, m, D);
        D2 = fmaf(w * m, m, D2);
        Z = fmaf(w, s.z, Z);
#pragma unroll
        for (int c = 0; c < 3; ++c) N[c] = fmaf(w, r.nrm[c], N[c]);
        if (T > 0.5f) {
          med = s.z;
          med_idx = start + base + j;
        }
      }
      T *= 1.f - alpha;
    }
  }
  const size_t p = (size_t)iy * wp + ix;
  const float o0 = fmaf(T, bg.x, C[0]), o1 = fmaf(T, bg.y, C[1]), o2 = fmaf(T, bg.z, C[2]);
  image[3 * p] = o0;
  image[3 * p + 1] = o1;
  image[3 * p + 2] = o2;
  if (final_img) gs_store_final(final_img, ix, iy, crop.left, crop.top, crop.width, crop.height, o0, o1, o2);
  ws[p] = make_float4(C[0], C[1], C[2], T);
  if constexpr (MAPS) {
    wsm[2 * p] = make_float4(Z, A, D, D2);
    wsm[2 * p + 1] = make_float4(N[0], N[1], N[2], __int_as_float(med_idx));
    const float4 q0 = make_float4(1.f - T, Z, med, dist), q1 = make_float4(N[0], N[1], N[2], 0.f);
    if (mp.maps) {
      reinterpret_cast<float4*>(mp.maps)[2 * p] = q0;
      reinterpret_cast<float4*>(mp.maps)[2 * p + 1] = q1;
    }
    const int x = ix - crop.left, y = iy - crop.top;
    if (mp.maps_final && x >= 0 && x < crop.width && y >= 0 && y < crop.height) {
      const size_t pf = (size_t)y * crop.width + x;
      reinterpret_cast<float4*>(mp.maps_final)[2 * pf] = q0;
      reinterpret_cast<float4*>(mp.maps_final)[2 * pf + 1] = q1;
    }
  }
  if (tile_neff && tid == 0) tile_neff[tile] = consumed;
}

// ---------------------------------------------------------------------------------------
// backward: front to back, T recomputed as the forward computed it.  For F(w) with per-instance values G_i:
//   dL/dalpha_i = T_i G_i - R_i / (1 - alpha_i),  R starts at sum_j w_j G_j + T_f g . bg and loses w_i G_i at i.
//   G_i = g . c_i (+ MAPS: g_D z_i + g_N . n_i + g_A + g_dist (m_i^2 A_f - 2 m_i D_f + D2_f))
// Direct terms: dL/dc_i = g w_i, dL/dn_i = g_N w_i, dL/dz_i = g_D w_i + g_dist 2 w_i (m_i A_f - D_f) dm/dz (+ g_med at
// the median instance).  A clamped alpha passes no gradient through alpha.  Per instance the 16 sums {dL/dM (9),
// dL/dop, dL/dc (3), dL/dn (3)} are reduced over each warp with reduce8 and across the 8 warps through shared memory
// in a fixed order (no atomics: bit-deterministic), and stored at the instance's slot, tagged with the epoch.
// ---------------------------------------------------------------------------------------
template <bool MAPS>
__global__ void __launch_bounds__(kNT) blend_surfel_bwd_kernel(
    const GsSurfelRec* __restrict__ rec, const uint32_t* __restrict__ ids, const uint2* __restrict__ rect,
    const uint32_t* __restrict__ goff, const int* __restrict__ tile_accum, int wp, int hp, int ntx, float fx,
    float fy, float3 bg, const float* __restrict__ image, const float* __restrict__ grad_image, int grad_is_final,
    GsCrop crop, const float* __restrict__ grad_maps, float dA, float dB, float near, const float4* __restrict__ ws,
    const float4* __restrict__ wsm, float* __restrict__ grad_inst, uint32_t* __restrict__ row_epoch, uint32_t epoch,
    int* __restrict__ tile_neff_b) {
  constexpr int CH = 32, NV = GS_SURFEL_GREC;
  __shared__ __align__(16) GsSurfelRec sr[CH];
  __shared__ uint32_t sslot[CH];
  __shared__ float part[kNW][CH][NV];
  const int tile = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = tile % ntx, ty = tile / ntx;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int ix = tx * GS_TILE + (tid % GS_TILE), iy = ty * GS_TILE + tid / GS_TILE;
  const float qx = gs_pixel_coord(ix, wp, fx), qy = gs_pixel_coord(iy, hp, fy);
  const size_t p = (size_t)iy * wp + ix;
  float gc[3];
  if (!grad_is_final) {
#pragma unroll
    for (int c = 0; c < 3; ++c) gc[c] = grad_image[3 * p + c];
  } else {
    gs_load_final_grad(grad_image, image + 3 * p, ix, iy, crop.left, crop.top, crop.width, crop.height, gc[0], gc[1],
                       gc[2]);
  }
  const float4 w0 = ws[p];
  float R = gc[0] * w0.x + gc[1] * w0.y + gc[2] * w0.z + w0.w * (gc[0] * bg.x + gc[1] * bg.y + gc[2] * bg.z);
  float gA = 0.f, gZ = 0.f, gMed = 0.f, gDist = 0.f, gN[3] = {0.f, 0.f, 0.f}, Af = 0.f, Df = 0.f, D2f = 0.f;
  int med_idx = -1;
  if constexpr (MAPS) {
    const float* gm = nullptr;
    if (!grad_is_final) {
      gm = grad_maps + p * GS_SURFEL_MAP_CH;
    } else {
      const int x = ix - crop.left, y = iy - crop.top;
      if (x >= 0 && x < crop.width && y >= 0 && y < crop.height)
        gm = grad_maps + ((size_t)y * crop.width + x) * GS_SURFEL_MAP_CH;
    }
    if (gm) {
      gA = gm[0];
      gZ = gm[1];
      gMed = gm[2];
      gDist = gm[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) gN[c] = gm[4 + c];
    }
    const float4 a = wsm[2 * p], b = wsm[2 * p + 1];
    Af = a.y;
    Df = a.z;
    D2f = a.w;
    med_idx = __float_as_int(b.w);
    R += gZ * a.x + gN[0] * b.x + gN[1] * b.y + gN[2] * b.z + gA * Af + gDist * 2.f * (Af * D2f - Df * Df);
  }
  float T = 1.f, m0 = __int_as_float(0x7fffffff);   // as in the forward
  bool done = false;
  int consumed = cnt;
  for (int base = 0; base < cnt; base += CH) {
    if (__syncthreads_count(!done) == 0) {   // also: every thread is done with the previous chunk and its sums
      consumed = base;
      break;
    }
    const int n = min(CH, cnt - base);
    load_chunk<CH>(reinterpret_cast<float4*>(sr), rec, ids, start + base, n, tid);
    for (int t = tid; t < n; t += kNT) {
      const uint32_t id = __ldg(ids + start + base + t);
      const uint2 rc = __ldg(rect + id);
      sslot[t] = __ldg(goff + id) + ((uint32_t)ty - (rc.x >> 16)) * (rc.y & 0xffffu) + ((uint32_t)tx - (rc.x & 0xffffu));
    }
    __syncthreads();
    for (int j = 0; j < n; ++j) {
      float v[NV];
#pragma unroll
      for (int u = 0; u < NV; ++u) v[u] = 0.f;
      if (!done && !(T > GS_T_STOP)) done = true;
      if (!done) {
        const GsSurfelRec& r = sr[j];
        const SurfelHit s = surfel_hit(r.M, qx, qy, fx, fy, near);
        const float araw = r.op * s.g;
        const float alpha = fminf(0.99f, araw);
        if (alpha >= kAlphaMin) {
          const float w = alpha * T;
          float G = gc[0] * r.rgb[0] + gc[1] * r.rgb[1] + gc[2] * r.rgb[2];
          float gz = 0.f;
          if constexpr (MAPS) {
            const float mr = dA - dB / s.z;
            if (m0 != m0) m0 = mr;
            const float m = mr - m0;
            G += gZ * s.z + gN[0] * r.nrm[0] + gN[1] * r.nrm[1] + gN[2] * r.nrm[2] + gA +
                 gDist * fmaf(m, fmaf(m, Af, -2.f * Df), D2f);
            gz = gZ * w + gDist * 2.f * w * fmaf(m, Af, -Df) * (dB / (s.z * s.z));
            if (start + base + j == med_idx) gz += gMed;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[13 + c] = gN[c] * w;
          }
#pragma unroll
          for (int c = 0; c < 3; ++c) v[10 + c] = gc[c] * w;
          R = fmaf(-w, G, R);
          const float dal = araw > 0.99f ? 0.f : fmaf(T, G, -R / (1.f - alpha));
          v[9] = dal * s.g;                      // dL/dop
          const float grho = -0.5f * dal * alpha;
          const float* M = r.M;
          if (s.lowpass) {
            const float gcx = grho * (-4.f * s.dx * fx), gcy = grho * (-4.f * s.dy * fy);
            const float im = 1.f / M[8];
            v[2] += gcx * im;
            v[5] += gcy * im;
            v[8] += gz - (gcx * M[2] + gcy * M[5]) * im * im;
          } else {
            const float ga = fmaf(grho, 2.f * s.a, gz * M[6]), gb = fmaf(grho, 2.f * s.b, gz * M[7]);
            v[6] += gz * s.a;
            v[7] += gz * s.b;
            v[8] += gz;
            const float ih = 1.f / s.h[2];
            const float gh[3] = {ga * ih, gb * ih, -(ga * s.a + gb * s.b) * ih};
            // dL/dk = l x gh, dL/dl = gh x k
            const float gk[3] = {s.l[1] * gh[2] - s.l[2] * gh[1], s.l[2] * gh[0] - s.l[0] * gh[2],
                                 s.l[0] * gh[1] - s.l[1] * gh[0]};
            const float gl[3] = {gh[1] * s.k[2] - gh[2] * s.k[1], gh[2] * s.k[0] - gh[0] * s.k[2],
                                 gh[0] * s.k[1] - gh[1] * s.k[0]};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              v[c] -= gk[c];
              v[3 + c] -= gl[c];
              v[6 + c] += qx * gk[c] + qy * gl[c];
            }
          }
          T *= 1.f - alpha;
        }
      }
#pragma unroll
      for (int blk = 0; blk < NV / 8; ++blk) {
        const float rsum = reduce8(v + blk * 8, lane);
        if ((lane & 3) == 0) part[warp][j][blk * 8 + ((lane >> 2) & 7)] = rsum;
      }
    }
    __syncthreads();
    for (int t = tid; t < n * NV; t += kNT) {
      const int i = t / NV, u = t % NV;
      float sum = 0.f;
#pragma unroll
      for (int w = 0; w < kNW; ++w) sum += part[w][i][u];
      const uint32_t slot = sslot[i];
      grad_inst[(size_t)slot * NV + u] = sum;
      if (u == 0) row_epoch[slot] = epoch;
    }
  }
  if (tile_neff_b && tid == 0) tile_neff_b[tile] = consumed;
}

}  // namespace

cudaError_t gs_launch_blend_surfel_fwd(const GsSurfelRec* rec, const uint32_t* ids, const int* tile_accum,
                                       const GsFrameGeom& g, const float* bg, float* image, float* final_img,
                                       const GsCrop& crop, const GsSurfelMaps* maps, float near, float4* ws,
                                       float4* wsm, int* tile_neff, cudaStream_t st) {
  const float3 b = make_float3(bg[0], bg[1], bg[2]);
  GsSurfelMaps mp = maps ? *maps : GsSurfelMaps{nullptr, nullptr, 0.2f, 100.f};
  const float dA = (float)((double)mp.dist_far / ((double)mp.dist_far - (double)mp.dist_near));
  const float dB = (float)((double)mp.dist_far * (double)mp.dist_near / ((double)mp.dist_far - (double)mp.dist_near));
  if (maps)
    blend_surfel_fwd_kernel<true><<<g.n_tiles, kNT, 0, st>>>(rec, ids, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, b,
                                                             image, final_img, crop, mp, dA, dB, near, ws, wsm, tile_neff);
  else
    blend_surfel_fwd_kernel<false><<<g.n_tiles, kNT, 0, st>>>(rec, ids, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, b,
                                                              image, final_img, crop, mp, dA, dB, near, ws, wsm, tile_neff);
  return cudaGetLastError();
}

cudaError_t gs_launch_blend_surfel_bwd(const GsSurfelRec* rec, const uint32_t* ids, const uint2* rect,
                                       const uint32_t* goff, const int* tile_accum, const GsFrameGeom& g,
                                       const float* bg, const float* image, const float* grad_image, int grad_is_final,
                                       const GsCrop& crop, const float* grad_maps, float dist_near, float dist_far,
                                       float near, const float4* ws, const float4* wsm, float* grad_inst, uint32_t* row_epoch,
                                       uint32_t epoch, int* tile_neff_b, cudaStream_t st) {
  const float3 b = make_float3(bg[0], bg[1], bg[2]);
  const float dA = (float)((double)dist_far / ((double)dist_far - (double)dist_near));
  const float dB = (float)((double)dist_far * (double)dist_near / ((double)dist_far - (double)dist_near));
  if (grad_maps)
    blend_surfel_bwd_kernel<true><<<g.n_tiles, kNT, 0, st>>>(rec, ids, rect, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx,
                                                             g.fy, b, image, grad_image, grad_is_final, crop, grad_maps,
                                                             dA, dB, near, ws, wsm, grad_inst, row_epoch, epoch, tile_neff_b);
  else
    blend_surfel_bwd_kernel<false><<<g.n_tiles, kNT, 0, st>>>(rec, ids, rect, goff, tile_accum, g.wp, g.hp, g.ntx,
                                                              g.fx, g.fy, b, image, grad_image, grad_is_final, crop,
                                                              nullptr, dA, dB, near, ws, wsm, grad_inst, row_epoch, epoch,
                                                              tile_neff_b);
  return cudaGetLastError();
}
