// 2D Gaussian surfels (Huang et al. 2024) on the fused frame path: the projection forward (activations, culling, the
// 3-sigma disk's tile rectangle, the depth key, one GsSurfelRec per surfel) and its backward (segment sum of the
// epoch-tagged instance rows, chained to the raw parameters).  Binning and ordering are the 3DGS frame's, unchanged:
// they read only count[N], dkey[N] and rect[N].
#include "internal.h"
#include "sh_common.cuh"

namespace {

constexpr int kBlock = 256;

// unit direction from the camera centre C = -R^T t to the mean (world frame) and 1 / |pos - C|: project.cu's view_dir
__device__ __forceinline__ void surfel_view_dir(const GsCam& cam, const float p[3], float dir[3], float& inv_len) {
  float u[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) u[j] = p[j] + (cam.r[j] * cam.t[0] + cam.r[3 + j] * cam.t[1] + cam.r[6 + j] * cam.t[2]);
  inv_len = 1.f / sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
#pragma unroll
  for (int j = 0; j < 3; ++j) dir[j] = u[j] * inv_len;
}

template <int K>
__device__ __forceinline__ void surfel_sh_logits(const float* coef, const float* Y, float l[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) s = fmaf(Y[k], coef[c * K + k], s);
    l[c] = s;
  }
}

// R v for the camera rotation R (row-major) and a world vector v
__device__ __forceinline__ void cam_rot(const GsCam& cam, const float v[3], float o[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r) o[r] = cam.r[3 * r] * v[0] + cam.r[3 * r + 1] * v[1] + cam.r[3 * r + 2] * v[2];
}
// R^T v
__device__ __forceinline__ void cam_rot_t(const GsCam& cam, const float v[3], float o[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = cam.r[k] * v[0] + cam.r[3 + k] * v[1] + cam.r[6 + k] * v[2];
}

// The camera-frame tangent columns u = s_u R r0, v = s_v R r1, the camera normal R r2 and p_c of one surfel
struct SurfelGeom {
  float u[3], v[3], nc[3], pc[3];
  float Rr0[3], Rr1[3];
  GsRot Q;
};
__device__ __forceinline__ SurfelGeom surfel_geom(const GsCam& cam, const float p[3], const float q[4], const float s[3]) {
  SurfelGeom g;
  g.Q = gs_quat_to_rot(q[0], q[1], q[2], q[3]);
  const float r0[3] = {g.Q.m[0], g.Q.m[3], g.Q.m[6]};
  const float r1[3] = {g.Q.m[1], g.Q.m[4], g.Q.m[7]};
  const float r2[3] = {g.Q.m[2], g.Q.m[5], g.Q.m[8]};
  cam_rot(cam, r0, g.Rr0);
  cam_rot(cam, r1, g.Rr1);
  cam_rot(cam, r2, g.nc);
  gs_world_to_cam(cam, p, g.pc);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    g.u[k] = s[0] * g.Rr0[k];
    g.v[k] = s[1] * g.Rr1[k];
  }
  return g;
}

// Tile rectangle of the box [left, right] x [top, bottom] (normalised image plane) with gs_tile_rect's rule
__device__ __forceinline__ bool surfel_tile_rect(const GsTileGrid& g, float left, float right, float top, float bottom,
                                                 uint32_t& tx0, uint32_t& tx1, uint32_t& ty0, uint32_t& ty1) {
  ty0 = (uint32_t)fmaxf((top - g.topmost) / g.ly, 0.f);
  ty1 = (uint32_t)((bottom - g.topmost) / g.ly + 1.f);
  tx0 = (uint32_t)fmaxf((left - g.leftmost) / g.lx, 0.f);
  tx1 = (uint32_t)((right - g.leftmost) / g.lx + 1.f);
  ty1 = min(ty1, (uint32_t)g.nty);
  tx1 = min(tx1, (uint32_t)g.ntx);
  return (ty1 > ty0) && (tx1 > tx0);
}

// ---------------------------------------------------------------------------------------
// forward: one thread per surfel.  Culling on the centre as the 3DGS projection (z > near, the 1.2x frustum); the
// rectangle is the box of the projected 3-sigma disk a^2 + b^2 <= 9 from the dual conic C* = M diag(9, 9, -1) M^T,
// joined with the box of radius sqrt(2)/2 px around the centre; C*22 >= 0 (the disk reaches the camera plane): no
// instances.  Sort key: camera z of the centre.
// ---------------------------------------------------------------------------------------
template <int KG>
__global__ void __launch_bounds__(kBlock) surfel_project_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int scale_act, GsCam cam, GsTileGrid grid,
    float near_plane, float half_w, float half_h, float fx, float fy, GsSurfelRec* __restrict__ rec,
    uint2* __restrict__ rect, uint32_t* __restrict__ count, uint32_t* __restrict__ dkey, int64_t* __restrict__ mask,
    unsigned int* __restrict__ n_visible) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  bool vis = false;
  uint32_t cnt = 0;
  if (i < n) {
    const float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
    float q[4], s[3], raw_s[3], qn;
    gs_load_activated(quat, scale, i, scale_act, q, s, raw_s, qn);
    const SurfelGeom G = surfel_geom(cam, p, q, s);
    float zc = G.pc[2];
    if (zc > near_plane) {
      const float cx = G.pc[0] / zc, cy = G.pc[1] / zc;
      vis = fabsf(cx) < half_w && fabsf(cy) < half_h;
    }
    if (mask) mask[i] = vis ? 1 : 0;
    uint2 rc = make_uint2(0u, 0u);
    if (vis) {
      // C*_jk = 9 (u_j u_k + v_j v_k) - p_j p_k
      const float c22 = 9.f * (G.u[2] * G.u[2] + G.v[2] * G.v[2]) - G.pc[2] * G.pc[2];
      if (c22 < 0.f) {
        const float c00 = 9.f * (G.u[0] * G.u[0] + G.v[0] * G.v[0]) - G.pc[0] * G.pc[0];
        const float c11 = 9.f * (G.u[1] * G.u[1] + G.v[1] * G.v[1]) - G.pc[1] * G.pc[1];
        const float c02 = 9.f * (G.u[0] * G.u[2] + G.v[0] * G.v[2]) - G.pc[0] * G.pc[2];
        const float c12 = 9.f * (G.u[1] * G.u[2] + G.v[1] * G.v[2]) - G.pc[1] * G.pc[2];
        const float ex = c02 / c22, ey = c12 / c22;
        const float hx = sqrtf(fmaxf(ex * ex - c00 / c22, 0.f));
        const float hy = sqrtf(fmaxf(ey * ey - c11 / c22, 0.f));
        const float cx = G.pc[0] / G.pc[2], cy = G.pc[1] / G.pc[2];
        const float rx = 0.70710678f / fx, ry = 0.70710678f / fy;
        const float left = fminf(ex - hx, cx - rx), right = fmaxf(ex + hx, cx + rx);
        const float top = fminf(ey - hy, cy - ry), bottom = fmaxf(ey + hy, cy + ry);
        uint32_t tx0, tx1, ty0, ty1;
        if (surfel_tile_rect(grid, left, right, top, bottom, tx0, tx1, ty0, ty1)) {
          cnt = (tx1 - tx0) * (ty1 - ty0);
          rc = make_uint2(tx0 | (ty0 << 16), (tx1 - tx0) | ((ty1 - ty0) << 16));
          GsSurfelRec r;
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            r.M[3 * k] = G.u[k];
            r.M[3 * k + 1] = G.v[k];
            r.M[3 * k + 2] = G.pc[k];
          }
          r.op = gs_sigmoid(opa[i]);
          if constexpr (KG > 0) {
            float coef[3 * KG], dir[3], il, Y[KG], l[3];
#pragma unroll
            for (int k = 0; k < 3 * KG; ++k) coef[k] = rgb[(size_t)i * (3 * KG) + k];
            surfel_view_dir(cam, p, dir, il);
            gs_sh::sh_basis<KG>(dir[0], dir[1], dir[2], Y);
            surfel_sh_logits<KG>(coef, Y, l);
#pragma unroll
            for (int c = 0; c < 3; ++c) r.rgb[c] = gs_sigmoid(l[c]);
          } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) r.rgb[c] = gs_sigmoid(rgb[3 * i + c]);
          }
          const float sgn = (G.nc[0] * G.pc[0] + G.nc[1] * G.pc[1] + G.nc[2] * G.pc[2]) > 0.f ? -1.f : 1.f;
#pragma unroll
          for (int k = 0; k < 3; ++k) r.nrm[k] = sgn * G.nc[k];
          float4* dst = reinterpret_cast<float4*>(rec + i);
          const float4* src = reinterpret_cast<const float4*>(&r);
#pragma unroll
          for (int k = 0; k < 4; ++k) dst[k] = src[k];
        }
      }
    }
    rect[i] = rc;
    count[i] = cnt;
    dkey[i] = cnt ? __float_as_uint(zc) : 0xffffffffu;
  }
  // 64-bit instance total next to the visible count (counters[2..3]), as the 3DGS projection
  __shared__ unsigned long long wsum[kBlock / 32];
  unsigned long long c64 = cnt;
#pragma unroll
  for (int o = 16; o; o >>= 1) c64 += __shfl_xor_sync(0xffffffffu, c64, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c64;
  const int nv = __syncthreads_count(vis);
  if (threadIdx.x == 0) {
    unsigned long long tot = 0;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) tot += wsum[w];
    if (nv) atomicAdd(n_visible, (unsigned int)nv);
    if (tot) atomicAdd(reinterpret_cast<unsigned long long*>(n_visible + 2), tot);
  }
}

// ---------------------------------------------------------------------------------------
// backward: one thread per surfel sums its epoch-tagged rows {dL/dM (9), dL/dop, dL/dc (3), dL/dn (3)} in row order
// (no atomics: deterministic), then
//   dL/dp_c = column 3 of dL/dM, dL/du = column 1, dL/dv = column 2;  u = s_u R r0, v = s_v R r1, n = +-R r2
//   dL/ds_u = dL/du . R r0,  dL/dr0 = s_u R^T dL/du  (r1, r2 alike),  dL/dpos = R^T dL/dp_c (+ the SH direction term)
// and the activation chains of the 3DGS projection backward (normalised quaternion, abs / exp scale, sigmoid).
// scale[:, 2] gets exactly 0.
// ---------------------------------------------------------------------------------------
template <int KG>
__global__ void __launch_bounds__(kBlock) surfel_project_bwd_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int scale_act, GsCam cam,
    const uint32_t* __restrict__ offsets_g, const uint32_t* __restrict__ count, const float* __restrict__ grad_inst,
    const uint32_t* __restrict__ row_epoch, uint32_t epoch, float* __restrict__ g_pos, float* __restrict__ g_rgb,
    float* __restrict__ g_opa, float* __restrict__ g_quat, float* __restrict__ g_scale) {
  constexpr int D = KG ? 3 * KG : 3;
  constexpr int GW = GS_SURFEL_GREC;
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float acc[GW];
#pragma unroll
  for (int k = 0; k < GW; ++k) acc[k] = 0.f;
  float gp[3] = {0.f, 0.f, 0.f}, gq_raw[4] = {0.f, 0.f, 0.f, 0.f}, gs_raw[3] = {0.f, 0.f, 0.f}, go = 0.f;
  float gcol[D];
#pragma unroll
  for (int k = 0; k < D; ++k) gcol[k] = 0.f;
  const uint32_t cnt = count[i], o0 = offsets_g[i];
  if (cnt > 0) {
    for (uint32_t r = o0; r < o0 + cnt; ++r) {
      if (row_epoch[r] != epoch) continue;   // not reached by its (saturated) tile
      const float4* row = reinterpret_cast<const float4*>(grad_inst + (size_t)r * GW);
#pragma unroll
      for (int qq = 0; qq < GW / 4; ++qq) {
        const float4 v = row[qq];
        acc[4 * qq] += v.x;
        acc[4 * qq + 1] += v.y;
        acc[4 * qq + 2] += v.z;
        acc[4 * qq + 3] += v.w;
      }
    }
    const float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
    float q[4], s[3], raw_s[3], qn;
    gs_load_activated(quat, scale, i, scale_act, q, s, raw_s, qn);
    const SurfelGeom G = surfel_geom(cam, p, q, s);
    float gu[3], gv[3], gpc[3], gn[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      gu[k] = acc[3 * k];
      gv[k] = acc[3 * k + 1];
      gpc[k] = acc[3 * k + 2];
      gn[k] = acc[13 + k];
    }
    const float sgn = (G.nc[0] * G.pc[0] + G.nc[1] * G.pc[1] + G.nc[2] * G.pc[2]) > 0.f ? -1.f : 1.f;
    float gsv[3];
    gsv[0] = gu[0] * G.Rr0[0] + gu[1] * G.Rr0[1] + gu[2] * G.Rr0[2];
    gsv[1] = gv[0] * G.Rr1[0] + gv[1] * G.Rr1[1] + gv[2] * G.Rr1[2];
    gsv[2] = 0.f;
    float gr0[3], gr1[3], gr2[3];
    cam_rot_t(cam, gu, gr0);
    cam_rot_t(cam, gv, gr1);
    cam_rot_t(cam, gn, gr2);
    cam_rot_t(cam, gpc, gp);
    // dL/dQ (row-major, Q = [r0 | r1 | r2])
    float gR[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      gR[3 * k] = s[0] * gr0[k];
      gR[3 * k + 1] = s[1] * gr1[k];
      gR[3 * k + 2] = sgn * gr2[k];
    }
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    float gq[4];
    gq[0] = 2.f * (-z * gR[1] + y * gR[2] + z * gR[3] - x * gR[5] - y * gR[6] + x * gR[7]);
    gq[1] = 2.f * (y * gR[1] + z * gR[2] + y * gR[3] - 2.f * x * gR[4] - w * gR[5] + z * gR[6] + w * gR[7] - 2.f * x * gR[8]);
    gq[2] = 2.f * (-2.f * y * gR[0] + x * gR[1] + w * gR[2] + x * gR[3] + z * gR[5] - w * gR[6] + z * gR[7] - 2.f * y * gR[8]);
    gq[3] = 2.f * (-2.f * z * gR[0] - w * gR[1] + x * gR[2] + w * gR[3] - 2.f * z * gR[4] + y * gR[5] + x * gR[6] + y * gR[7]);
    const float dot = q[0] * gq[0] + q[1] * gq[1] + q[2] * gq[2] + q[3] * gq[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) gq_raw[k] = (gq[k] - q[k] * dot) / qn;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (scale_act == GS_SCALE_ABS)
        gs_raw[k] = gsv[k] * (raw_s[k] > 0.f ? 1.f : (raw_s[k] < 0.f ? -1.f : 0.f));
      else
        gs_raw[k] = gsv[k] * expf(fminf(fmaxf(raw_s[k], -1.f), 1.f));   // as the 3DGS projection backward
    }
    const float op = gs_sigmoid(opa[i]);
    go = acc[9] * op * (1.f - op);
    if constexpr (KG > 0) {
      // c = sigmoid(l), l_c = sum_k Y_k(dir) coef[c K + k]; ddir/dpos = (I - dir dir^T) / |pos - C|
      float coef[D], dir[3], il, Y[KG], l[3], gl[3], wk[KG], gd[3];
#pragma unroll
      for (int k = 0; k < D; ++k) coef[k] = rgb[(size_t)i * D + k];
      surfel_view_dir(cam, p, dir, il);
      gs_sh::sh_basis<KG>(dir[0], dir[1], dir[2], Y);
      surfel_sh_logits<KG>(coef, Y, l);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float sg = gs_sigmoid(l[c]);
        gl[c] = acc[10 + c] * sg * (1.f - sg);
      }
#pragma unroll
      for (int k = 0; k < KG; ++k) {
#pragma unroll
        for (int c = 0; c < 3; ++c) gcol[c * KG + k] = gl[c] * Y[k];
        wk[k] = gl[0] * coef[k] + gl[1] * coef[KG + k] + gl[2] * coef[2 * KG + k];
      }
      gs_sh::sh_basis_grad<KG>(dir[0], dir[1], dir[2], wk, gd);
      const float dd = dir[0] * gd[0] + dir[1] * gd[1] + dir[2] * gd[2];
#pragma unroll
      for (int j = 0; j < 3; ++j) gp[j] += (gd[j] - dir[j] * dd) * il;
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float sg = gs_sigmoid(rgb[3 * i + c]);
        gcol[c] = acc[10 + c] * sg * (1.f - sg);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < D; ++k) g_rgb[(size_t)i * D + k] = gcol[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    g_pos[3 * i + k] = gp[k];
    g_scale[3 * i + k] = gs_raw[k];
  }
  reinterpret_cast<float4*>(g_quat)[i] = make_float4(gq_raw[0], gq_raw[1], gq_raw[2], gq_raw[3]);
  g_opa[i] = go;
}

}  // namespace

cudaError_t gs_launch_surfel_project(const float* pos, const float* rgb, const float* opa, const float* quat,
                                     const float* scale, int n, int kg, int scale_act, const GsCam& cam,
                                     const GsTileGrid& grid, float near_plane, float half_w, float half_h, float fx,
                                     float fy, GsSurfelRec* rec, uint2* rect, uint32_t* count, uint32_t* dkey,
                                     int64_t* mask, unsigned int* n_visible, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const int blocks = (n + kBlock - 1) / kBlock;
#define GS_SURFEL_P(K)                                                                                              \
  surfel_project_kernel<K><<<blocks, kBlock, 0, st>>>(pos, rgb, opa, quat, scale, n, scale_act, cam, grid,         \
                                                      near_plane, half_w, half_h, fx, fy, rec, rect, count, dkey, \
                                                      mask, n_visible)
  switch (kg) {
    case 0: GS_SURFEL_P(0); break;
    case 9: GS_SURFEL_P(9); break;
    case 16: GS_SURFEL_P(16); break;
    default: return cudaErrorInvalidValue;
  }
#undef GS_SURFEL_P
  return cudaGetLastError();
}

cudaError_t gs_launch_surfel_project_bwd(const float* pos, const float* rgb, const float* opa, const float* quat,
                                         const float* scale, int n, int kg, int scale_act, const GsCam& cam,
                                         const uint32_t* offsets_g, const uint32_t* count, const float* grad_inst,
                                         const uint32_t* row_epoch, uint32_t epoch, float* g_pos, float* g_rgb,
                                         float* g_opa, float* g_quat, float* g_scale, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const int blocks = (n + kBlock - 1) / kBlock;
#define GS_SURFEL_PB(K)                                                                                           \
  surfel_project_bwd_kernel<K><<<blocks, kBlock, 0, st>>>(pos, rgb, opa, quat, scale, n, scale_act, cam,         \
                                                          offsets_g, count, grad_inst, row_epoch, epoch, g_pos,  \
                                                          g_rgb, g_opa, g_quat, g_scale)
  switch (kg) {
    case 0: GS_SURFEL_PB(0); break;
    case 9: GS_SURFEL_PB(9); break;
    case 16: GS_SURFEL_PB(16); break;
    default: return cudaErrorInvalidValue;
  }
#undef GS_SURFEL_PB
  return cudaGetLastError();
}
