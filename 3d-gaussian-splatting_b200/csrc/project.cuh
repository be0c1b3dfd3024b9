// Per-Gaussian projection math shared by the legacy (global_culling) and fused kernels.
// Behaviour follows reference gaussian.cu:1131-1336 (forward) and :1371-1576 (backward);
// the arithmetic is re-derived (only the two image-plane rows of J*W are formed and
// cov2d = (J W R S)(J W R S)^T), it is not a transcription.
#pragma once
#include "gs_common.cuh"

struct GsCam {
  float r[9];
  float t[3];
};

struct GsProj {
  float x, y, depth;   // x/z, y/z, |p_c|
  float a, b, c, d;    // 2x2 covariance in normalised image-plane units
  bool visible;
};

struct GsRot {
  float m[9];
};

__device__ __forceinline__ GsRot gs_quat_to_rot(float w, float x, float y, float z) {
  GsRot R;
  R.m[0] = 1.f - 2.f * y * y - 2.f * z * z;
  R.m[1] = 2.f * x * y - 2.f * z * w;
  R.m[2] = 2.f * x * z + 2.f * y * w;
  R.m[3] = 2.f * x * y + 2.f * z * w;
  R.m[4] = 1.f - 2.f * x * x - 2.f * z * z;
  R.m[5] = 2.f * y * z - 2.f * x * w;
  R.m[6] = 2.f * x * z - 2.f * y * w;
  R.m[7] = 2.f * y * z + 2.f * x * w;
  R.m[8] = 1.f - 2.f * x * x - 2.f * y * y;
  return R;
}

__device__ __forceinline__ void gs_world_to_cam(const GsCam& cam, const float p[3], float pc[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
    pc[i] = cam.r[i * 3 + 0] * p[0] + cam.r[i * 3 + 1] * p[1] + cam.r[i * 3 + 2] * p[2] + cam.t[i];
}

// rows 0,1 of J*W with J = d(x/z, y/z)/d p_c evaluated at the un-clamped p_c
__device__ __forceinline__ void gs_jw_rows(const GsCam& cam, const float pc[3], float jw0[3], float jw1[3]) {
  float iz = 1.f / pc[2];
  float jx = -pc[0] / (pc[2] * pc[2]);
  float jy = -pc[1] / (pc[2] * pc[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    jw0[k] = iz * cam.r[0 * 3 + k] + jx * cam.r[2 * 3 + k];
    jw1[k] = iz * cam.r[1 * 3 + k] + jy * cam.r[2 * 3 + k];
  }
}

// Gaussian i's normalised quaternion q (and the norm qnorm of the raw one), activated scale s and raw scale raw_s, as
// the fused frame path applies them (splatter.py:519-524).
__device__ __forceinline__ void gs_load_activated(const float* __restrict__ quat, const float* __restrict__ scale,
                                                  int i, int scale_act, float q[4], float s[3], float raw_s[3],
                                                  float& qnorm) {
  float4 q4 = reinterpret_cast<const float4*>(quat)[i];
  qnorm = sqrtf(q4.x * q4.x + q4.y * q4.y + q4.z * q4.z + q4.w * q4.w);
  q[0] = q4.x / qnorm;
  q[1] = q4.y / qnorm;
  q[2] = q4.z / qnorm;
  q[3] = q4.w / qnorm;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    raw_s[k] = scale[3 * i + k];
    s[k] = (scale_act == GS_SCALE_ABS) ? (fabsf(raw_s[k]) + 1e-4f) : expf(raw_s[k]);
  }
}

// q (w,x,y,z) must be normalised and s activated by the caller.
__device__ __forceinline__ GsProj gs_project(const GsCam& cam, const float p[3], const float q[4],
                                             const float s[3], float near_plane, float half_w, float half_h) {
  GsProj o;
  o.visible = false;
  float pc[3];
  gs_world_to_cam(cam, p, pc);
  if (!(pc[2] > near_plane)) return o;                       // :1208  (z <= near culled)
  o.x = pc[0] / pc[2];
  o.y = pc[1] / pc[2];
  o.depth = sqrtf(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
  // :1220, written so that a NaN x/z or y/z (p_c.x and p_c.z both overflowed to inf) is culled too
  if (!(fabsf(o.x) < half_w) || !(fabsf(o.y) < half_h)) return o;
  o.visible = true;
  float jw0[3], jw1[3];
  gs_jw_rows(cam, pc, jw0, jw1);
  GsRot R = gs_quat_to_rot(q[0], q[1], q[2], q[3]);
  float m0[3], m1[3];                                         // M = (JW)(RS), 2x3
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m0[c] = (jw0[0] * R.m[0 * 3 + c] + jw0[1] * R.m[1 * 3 + c] + jw0[2] * R.m[2 * 3 + c]) * s[c];
    m1[c] = (jw1[0] * R.m[0 * 3 + c] + jw1[1] * R.m[1 * 3 + c] + jw1[2] * R.m[2 * 3 + c]) * s[c];
  }
  o.a = m0[0] * m0[0] + m0[1] * m0[1] + m0[2] * m0[2];
  o.b = m0[0] * m1[0] + m0[1] * m1[1] + m0[2] * m1[2];
  o.c = o.b;
  o.d = m1[0] * m1[0] + m1[1] * m1[1] + m1[2] * m1[2];
  return o;
}

// Backward of gs_project for a visible Gaussian.  g_xyd = dL/d(x/z, y/z, depth),
// g_cov = dL/d(a,b,c,d).  Outputs dL/dp (world), dL/dq (wrt the NORMALISED quaternion
// entries as independent variables, like the reference), dL/ds (activated scale).
__device__ __forceinline__ void gs_project_backward(const GsCam& cam, const float p[3], const float q[4],
                                                    const float s[3], const float g_xyd[3],
                                                    const float g_cov[4], float gp[3], float gq[4],
                                                    float gs[3]) {
  float pc[3];
  gs_world_to_cam(cam, p, pc);
  float r = sqrtf(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
  float iz = 1.f / pc[2];
  float ir = 1.f / r;
  float gc[3];
  gc[0] = g_xyd[0] * iz + g_xyd[2] * pc[0] * ir;                         // :1404-1406
  gc[1] = g_xyd[1] * iz + g_xyd[2] * pc[1] * ir;
  gc[2] = -(g_xyd[0] * pc[0] + g_xyd[1] * pc[1]) * iz * iz + g_xyd[2] * pc[2] * ir;
#pragma unroll
  for (int k = 0; k < 3; ++k) gp[k] = cam.r[0 * 3 + k] * gc[0] + cam.r[1 * 3 + k] * gc[1] + cam.r[2 * 3 + k] * gc[2];

  float jw0[3], jw1[3];
  gs_jw_rows(cam, pc, jw0, jw1);
  GsRot R = gs_quat_to_rot(q[0], q[1], q[2], q[3]);
  float m0[3], m1[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m0[c] = (jw0[0] * R.m[0 * 3 + c] + jw0[1] * R.m[1 * 3 + c] + jw0[2] * R.m[2 * 3 + c]) * s[c];
    m1[c] = (jw1[0] * R.m[0 * 3 + c] + jw1[1] * R.m[1 * 3 + c] + jw1[2] * R.m[2 * 3 + c]) * s[c];
  }
  // cov3 gradient G3 = JW2^T G2 JW2; d(RS) = (G3 + G3^T) RS = JW2^T (G2 + G2^T) M   (:1440-1519)
  float s00 = 2.f * g_cov[0], s01 = g_cov[1] + g_cov[2], s11 = 2.f * g_cov[3];
  float h0[3], h1[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    h0[c] = s00 * m0[c] + s01 * m1[c];
    h1[c] = s01 * m0[c] + s11 * m1[c];
  }
  float grs[9];
#pragma unroll
  for (int rr = 0; rr < 3; ++rr)
#pragma unroll
    for (int c = 0; c < 3; ++c) grs[rr * 3 + c] = jw0[rr] * h0[c] + jw1[rr] * h1[c];
  float gR[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    gs[c] = grs[0 * 3 + c] * R.m[0 * 3 + c] + grs[1 * 3 + c] * R.m[1 * 3 + c] + grs[2 * 3 + c] * R.m[2 * 3 + c];  // :1522-1526
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) gR[rr * 3 + c] = grs[rr * 3 + c] * s[c];
  }
  float w = q[0], x = q[1], y = q[2], z = q[3];
  gq[0] = 2.f * (-z * gR[1] + y * gR[2] + z * gR[3] - x * gR[5] - y * gR[6] + x * gR[7]);
  gq[1] = 2.f * (y * gR[1] + z * gR[2] + y * gR[3] - 2.f * x * gR[4] - w * gR[5] + z * gR[6] + w * gR[7] - 2.f * x * gR[8]);
  gq[2] = 2.f * (-2.f * y * gR[0] + x * gR[1] + w * gR[2] + x * gR[3] + z * gR[5] - w * gR[6] + z * gR[7] - 2.f * y * gR[8]);
  gq[3] = 2.f * (-2.f * z * gR[0] - w * gR[1] + x * gR[2] + w * gR[3] - 2.f * z * gR[4] + y * gR[5] + x * gR[6] + y * gR[7]);
}

// gs_project_backward plus what the camera gradient needs: gc = dL/dp_c and gjw = dL/d(JW) for the two image-plane
// rows of JW (row-major 2x3), h (RS)^T with h = (G2 + G2^T) M.  The parameter gradients are gs_project_backward's own
// (the subexpressions repeated below are shared after inlining).
__device__ __forceinline__ void gs_project_backward_cam(const GsCam& cam, const float p[3], const float q[4],
                                                        const float s[3], const float g_xyd[3], const float g_cov[4],
                                                        float gp[3], float gq[4], float gs[3], float gc[3],
                                                        float gjw[6]) {
  gs_project_backward(cam, p, q, s, g_xyd, g_cov, gp, gq, gs);
  float pc[3];
  gs_world_to_cam(cam, p, pc);
  float r = sqrtf(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
  float iz = 1.f / pc[2];
  float ir = 1.f / r;
  gc[0] = g_xyd[0] * iz + g_xyd[2] * pc[0] * ir;
  gc[1] = g_xyd[1] * iz + g_xyd[2] * pc[1] * ir;
  gc[2] = -(g_xyd[0] * pc[0] + g_xyd[1] * pc[1]) * iz * iz + g_xyd[2] * pc[2] * ir;
  float jw0[3], jw1[3];
  gs_jw_rows(cam, pc, jw0, jw1);
  GsRot R = gs_quat_to_rot(q[0], q[1], q[2], q[3]);
  float m0[3], m1[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m0[c] = (jw0[0] * R.m[0 * 3 + c] + jw0[1] * R.m[1 * 3 + c] + jw0[2] * R.m[2 * 3 + c]) * s[c];
    m1[c] = (jw1[0] * R.m[0 * 3 + c] + jw1[1] * R.m[1 * 3 + c] + jw1[2] * R.m[2 * 3 + c]) * s[c];
  }
  float s00 = 2.f * g_cov[0], s01 = g_cov[1] + g_cov[2], s11 = 2.f * g_cov[3];
  float h0[3], h1[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    h0[c] = s00 * m0[c] + s01 * m1[c];
    h1[c] = s01 * m0[c] + s11 * m1[c];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    gjw[k] = (h0[0] * R.m[k * 3 + 0] * s[0] + h0[1] * R.m[k * 3 + 1] * s[1]) + h0[2] * R.m[k * 3 + 2] * s[2];
    gjw[3 + k] = (h1[0] * R.m[k * 3 + 0] * s[0] + h1[1] * R.m[k * 3 + 1] * s[1]) + h1[2] * R.m[k * 3 + 2] * s[2];
  }
}

// One Gaussian's share of the camera gradient, added to cg[12] = {dL/dR row-major [9], dL/dt [3]} for p_c = R p + t:
// dL/dt += gc, dL/dR += gc p^T + J2^T gjw, with J2 = d(x/z, y/z)/dp_c detached (as for pos) and W = R live in JW.
__device__ __forceinline__ void gs_cam_grad_add(const GsCam& cam, const float p[3], const float gc[3],
                                                const float gjw[6], float cg[12]) {
  float pc[3];
  gs_world_to_cam(cam, p, pc);
  const float iz = 1.f / pc[2];
  const float jx = -pc[0] / (pc[2] * pc[2]);
  const float jy = -pc[1] / (pc[2] * pc[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    cg[k] += gc[0] * p[k] + iz * gjw[k];
    cg[3 + k] += gc[1] * p[k] + iz * gjw[3 + k];
    cg[6 + k] += gc[2] * p[k] + (jx * gjw[k] + jy * gjw[3 + k]);
    cg[9 + k] += gc[k];
  }
}

// Screen-space 2-D filter of the fused frame path (gs_ctx_set_filter2d): Sigma' = Sigma + diag(ex, ey), ex = s / fx^2,
// ey = s / fy^2 for a filter variance of s px^2.  The conic, the det test and the tile rectangle use Sigma'.
// compensate (antialias): l2o gains 0.5 log2(det / det'), which keeps the screen-space integral of alpha unchanged.
struct GsFilter2d {
  float ex, ey;
  int compensate;
};

struct GsFilter2dOut {
  float a, d;       // Sigma' diagonal (b, c unchanged)
  float dl2o;       // added to l2o (0 without compensation)
  float k[4];       // d dl2o / d(a, b, c, d): (d, -c, -b, a) / det - (d', -c, -b, a') / det', over 2 ln 2
  bool keep;        // false: the compensated Gaussian has det <= 0 and gets no instances
};

// Forward and backward of the filter for one projected covariance (a, b, c, d).  The backward chains the conic with
// Sigma' (Sigma' - Sigma is constant) and adds g_l2o * k to dL/dSigma; k is dead code in the forward.
__device__ __forceinline__ GsFilter2dOut gs_filter2d(const GsFilter2d& f, float a, float b, float c, float d) {
  GsFilter2dOut o;
  o.a = a + f.ex;
  o.d = d + f.ey;
  o.dl2o = 0.f;
  o.keep = true;
#pragma unroll
  for (int j = 0; j < 4; ++j) o.k[j] = 0.f;
  if (f.compensate) {
    const float det = a * d - b * c;
    const float detf = o.a * o.d - b * c;
    o.keep = det > 0.f;
    o.dl2o = 0.5f * log2f(det / detf);
    const float s = 0.5f / GS_LN2, id = 1.f / det, idf = 1.f / detf;
    o.k[0] = s * (d * id - o.d * idf);
    o.k[1] = s * (c * idf - c * id);
    o.k[2] = s * (b * idf - b * id);
    o.k[3] = s * (a * id - o.a * idf);
  }
  return o;
}

// 3-D smoothing filter of the fused frame path (gs_ctx_set_filter3d; Mip-Splatting's 3D filter): with Gaussian i's
// filter std f >= 0 (world units), its activated scale s becomes s' = sqrt(s^2 + f^2) and l2o gains
// dl2o = 0.5 sum_k log2(s_k^2 / s'_k^2), i.e. sigma' = sigma prod_k s_k / s'_k, which keeps sigma sqrt(det Sigma3), the
// Gaussian's 3-D integral.  f == 0 keeps s and dl2o = 0 by selection, so a zero filter gives the unfiltered bits.  A
// scale of 0 (exp underflow) gives dl2o = -inf: opacity 0.
// s: the activated scale on entry, s' on return; s0: the activated scale.
__device__ __forceinline__ void gs_filter3d(float f, float s[3], float s0[3], float& dl2o) {
  dl2o = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) s0[k] = s[k];
  if (f != 0.f) {
    const float f2 = f * f;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float s2 = s0[k] * s0[k];
      const float t = s2 + f2;
      s[k] = sqrtf(t);
      acc += log2f(s2 / t);
    }
    dl2o = 0.5f * acc;
  }
}

// Backward of gs_filter3d (f is a constant): gs = dL/ds' on entry, dL/ds on return,
//   dL/ds_k = dL/ds'_k s_k / s'_k + g_l2o f^2 / (ln 2 s_k (s_k^2 + f^2)).
// The second term is taken as 0 where g_l2o == 0 or s_k == 0 (a Gaussian whose opacity underflowed has no blend
// gradient, and 0 * inf must not reach the parameters).
__device__ __forceinline__ void gs_filter3d_backward(float f, const float s0[3], const float sf[3], float g_l2o,
                                                     float gs[3]) {
  if (f == 0.f) return;
  const float f2 = f * f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float s = s0[k];
    const float comp = (g_l2o != 0.f && s > 0.f) ? g_l2o * f2 / (GS_LN2 * s * (s * s + f2)) : 0.f;
    gs[k] = gs[k] * (s / sf[k]) + comp;
  }
}

// Lens of the fused frame path (gs_ctx_set_lens): a 2-D map D of the undistorted image-plane position (a, b) =
// (x/z, y/z), COLMAP's OPENCV or OPENCV_FISHEYE model, applied after the pinhole.  The stored mean is D(a, b) + (ox, oy),
// (ox, oy) = ((cx - W/2) / fx, (cy - H/2) / fy), and the 2-D covariance J_D Sigma J_D^T with J_D the map's Jacobian.
// rho2_max: the squared undistorted radius past which the polynomial folds back (+inf: none); farther Gaussians are
// culled.  model is GS_LENS_PINHOLE (D = identity), GS_LENS_OPENCV (k = k1, k2, p1, p2) or GS_LENS_FISHEYE (k1..k4).
struct GsLens {
  int model;
  float ox, oy, rho2_max;
  float k[4];
};

// The features a fused-frame projection kernel applies, cumulative: each tier also runs every lower one's arithmetic
// (a frame without the lower feature passes a zero 2-D filter or a NULL 3-D filter, which give the bits without it).
enum GsTier { GS_TIER_NONE = 0, GS_TIER_FILT2D, GS_TIER_FILT3D, GS_TIER_LENS };

inline int gs_tier(bool filt2d, const float* f3d, bool lens) {
  return lens ? GS_TIER_LENS : (f3d ? GS_TIER_FILT3D : (filt2d ? GS_TIER_FILT2D : GS_TIER_NONE));
}

// (a, b) -> (ad, bd) = D(a, b) and J = dD/d(a, b) row-major {d ad/da, d ad/db, d bd/da, d bd/db}
__device__ __forceinline__ void gs_lens_map(const GsLens& L, float a, float b, float& ad, float& bd, float J[4]) {
  const float r2 = a * a + b * b;
  if (L.model == GS_LENS_OPENCV) {
    const float k1 = L.k[0], k2 = L.k[1], p1 = L.k[2], p2 = L.k[3];
    const float rad = 1.f + r2 * (k1 + k2 * r2);
    const float drad = 2.f * k1 + 4.f * k2 * r2;   // d rad / d a = drad a
    ad = a * rad + 2.f * p1 * a * b + p2 * (r2 + 2.f * a * a);
    bd = b * rad + p1 * (r2 + 2.f * b * b) + 2.f * p2 * a * b;
    J[0] = rad + drad * a * a + 2.f * p1 * b + 6.f * p2 * a;
    J[1] = drad * a * b + 2.f * p1 * a + 2.f * p2 * b;
    J[2] = J[1];
    J[3] = rad + drad * b * b + 6.f * p1 * b + 2.f * p2 * a;
  } else if (L.model == GS_LENS_FISHEYE) {
    // (ad, bd) = f (a, b), f = theta_d / rho, theta = atan(rho); J = f I + g (a, b)^T (a, b) with g = f'(rho) / rho.
    // Near the axis f and g come from their series in rho^2 (the closed forms are 0 / 0 there).
    const float k1 = L.k[0], k2 = L.k[1], k3 = L.k[2], k4 = L.k[3];
    float f, g;
    if (r2 < 1e-4f) {
      f = 1.f + (k1 - 1.f / 3.f) * r2 + (0.2f - k1 + k2) * r2 * r2;
      g = 2.f * (k1 - 1.f / 3.f) + 4.f * (0.2f - k1 + k2) * r2;
    } else {
      const float rho = sqrtf(r2);
      const float th = atanf(rho), t2 = th * th;
      const float poly = 1.f + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)));
      const float dpoly = 1.f + t2 * (3.f * k1 + t2 * (5.f * k2 + t2 * (7.f * k3 + t2 * 9.f * k4)));   // d theta_d / d theta
      const float thd = th * poly;
      f = thd / rho;
      g = (dpoly * rho / (1.f + r2) - thd) / (r2 * rho);
    }
    ad = f * a;
    bd = f * b;
    J[0] = f + g * a * a;
    J[1] = g * a * b;
    J[2] = J[1];
    J[3] = f + g * b * b;
  } else {
    ad = a;
    bd = b;
    J[0] = 1.f;
    J[1] = 0.f;
    J[2] = 0.f;
    J[3] = 1.f;
  }
}

// The lens on a projection of gs_project taken without its frustum test (half_w = half_h = +inf): o.visible on entry is
// z > near.  It becomes z > near, rho^2 < rho2_max and the stored mean inside the 1.2x frustum (half_w, half_h); a
// visible o gets the stored mean and J_D Sigma J_D^T, and J the Jacobian (the backward's detached J_D).
__device__ __forceinline__ void gs_lens_project(const GsLens& L, GsProj& o, float half_w, float half_h, float J[4]) {
  if (!o.visible) return;
  const float r2 = o.x * o.x + o.y * o.y;
  float ad, bd;
  gs_lens_map(L, o.x, o.y, ad, bd, J);
  o.x = ad + L.ox;
  o.y = bd + L.oy;
  if (!(r2 < L.rho2_max) || !(fabsf(o.x) < half_w) || !(fabsf(o.y) < half_h)) {
    o.visible = false;
    return;
  }
  // Sigma' = J Sigma J^T, Sigma = [[a, b], [c, d]] symmetric
  const float t00 = J[0] * o.a + J[1] * o.c, t01 = J[0] * o.b + J[1] * o.d;
  const float t10 = J[2] * o.a + J[3] * o.c, t11 = J[2] * o.b + J[3] * o.d;
  o.a = t00 * J[0] + t01 * J[1];
  o.b = t00 * J[2] + t01 * J[3];
  o.c = o.b;
  o.d = t10 * J[2] + t11 * J[3];
}

// Backward of gs_lens_project with J_D detached in the covariance: g_xyd[0..1] = dL/d(stored mean) becomes
// J_D^T dL/dmean = dL/d(x/z, y/z), and g_cov = dL/dSigma' becomes J_D^T (dL/dSigma') J_D = dL/dSigma.
__device__ __forceinline__ void gs_lens_backward(const float J[4], float g_xyd[3], float g_cov[4]) {
  const float gx = g_xyd[0], gy = g_xyd[1];
  g_xyd[0] = J[0] * gx + J[2] * gy;
  g_xyd[1] = J[1] * gx + J[3] * gy;
  // G = J^T G' J, G' = [[g0, g1], [g2, g3]]
  const float u00 = g_cov[0] * J[0] + g_cov[1] * J[2], u01 = g_cov[0] * J[1] + g_cov[1] * J[3];
  const float u10 = g_cov[2] * J[0] + g_cov[3] * J[2], u11 = g_cov[2] * J[1] + g_cov[3] * J[3];
  g_cov[0] = J[0] * u00 + J[2] * u10;
  g_cov[1] = J[0] * u01 + J[2] * u11;
  g_cov[2] = J[1] * u00 + J[3] * u10;
  g_cov[3] = J[1] * u01 + J[3] * u11;
}

// Tile rectangle covered by a Gaussian, method 2 "prob2" (gaussian.cu:226-242): axis aligned
// bbox of the `thresh` iso-probability ellipse; float->uint32 casts truncate / saturate.
struct GsTileGrid {
  float lx, ly, leftmost, topmost, t2;   // t2 = -2*logf(thresh)
  int ntx, nty;
};

__device__ __forceinline__ bool gs_tile_rect(const GsTileGrid& g, float cx, float cy, float a, float b, float c,
                                             float d, uint32_t& tx0, uint32_t& tx1, uint32_t& ty0, uint32_t& ty1) {
  float det = a * d - b * c;
  if (det <= 0.f) return false;                                              // :227
  float ai = (float)((double)d / ((double)det + 1e-14));                     // :229
  float di = (float)((double)a / ((double)det + 1e-14));                     // :232
  float shift_x = sqrtf(di * g.t2 * det);
  float shift_y = sqrtf(ai * g.t2 * det);
  float right = cx + shift_x, left = cx - shift_x;
  float top = cy - shift_y, bottom = cy + shift_y;
  ty0 = (uint32_t)fmaxf((top - g.topmost) / g.ly, 0.f);                      // :241
  ty1 = (uint32_t)((bottom - g.topmost) / g.ly + 1.f);
  tx0 = (uint32_t)fmaxf((left - g.leftmost) / g.lx, 0.f);                    // :242
  tx1 = (uint32_t)((right - g.leftmost) / g.lx + 1.f);
  ty1 = min(ty1, (uint32_t)g.nty);
  tx1 = min(tx1, (uint32_t)g.ntx);
  return (ty1 > ty0) && (tx1 > tx0);
}
