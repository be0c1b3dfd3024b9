// Shared by the scalar (blend_sh.cu) and the tensor-core (blend_sh_tc.cu) SH blend kernels: row widths,
// the real SH basis of the reference (gaussian.cu:405-426; degree 3 = svox2's constants, :395-403) and the
// per-pixel ray direction (gaussian.cu:849-860).
#pragma once
#include "internal.h"

namespace gs_sh {

__host__ __device__ constexpr int sh_sw(int K) { return (3 * K + 1 + 3) / 4 * 4; }       // floats per pS row
__host__ __device__ constexpr int sh_nv(int K) { return 6 + 3 * K; }                     // reduced values
__host__ __device__ constexpr int sh_nvp(int K) { return (sh_nv(K) + 7) / 8 * 8; }       // padded to blocks of 8

constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
constexpr float SH_C2_0 = 1.0925484305920792f, SH_C2_1 = -1.0925484305920792f, SH_C2_2 = 0.31539156525252005f,
                SH_C2_3 = -1.0925484305920792f, SH_C2_4 = 0.5462742152960396f;
constexpr float SH_C3_0 = -0.5900435899266435f, SH_C3_1 = 2.890611442640554f, SH_C3_2 = -0.4570457994644658f,
                SH_C3_3 = 0.3731763325901154f, SH_C3_4 = -0.4570457994644658f, SH_C3_5 = 1.445305721320277f,
                SH_C3_6 = -0.5900435899266435f;

template <int K>
__device__ __forceinline__ void sh_basis(float x, float y, float z, float* out) {
  out[0] = SH_C0;
  out[1] = -SH_C1 * y;
  out[2] = SH_C1 * z;
  out[3] = -SH_C1 * x;
  const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
  out[4] = SH_C2_0 * xy;
  out[5] = SH_C2_1 * yz;
  out[6] = SH_C2_2 * (2.0f * zz - xx - yy);
  out[7] = SH_C2_3 * xz;
  out[8] = SH_C2_4 * (xx - yy);
  if (K > 9) {
    out[9] = SH_C3_0 * y * (3.f * xx - yy);
    out[10] = SH_C3_1 * xy * z;
    out[11] = SH_C3_2 * y * (4.f * zz - xx - yy);
    out[12] = SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy);
    out[13] = SH_C3_4 * x * (4.f * zz - xx - yy);
    out[14] = SH_C3_5 * z * (xx - yy);
    out[15] = SH_C3_6 * x * (xx - 3.f * yy);
  }
}

// g = sum_k w[k] dY_k / d(x, y, z): the derivative of sh_basis<K> contracted with weights w[K] (direction treated as
// three free coordinates; the caller projects out the radial part)
template <int K>
__device__ __forceinline__ void sh_basis_grad(float x, float y, float z, const float* w, float g[3]) {
  g[0] = -SH_C1 * w[3] + SH_C2_0 * y * w[4] - 2.f * SH_C2_2 * x * w[6] + SH_C2_3 * z * w[7] + 2.f * SH_C2_4 * x * w[8];
  g[1] = -SH_C1 * w[1] + SH_C2_0 * x * w[4] + SH_C2_1 * z * w[5] - 2.f * SH_C2_2 * y * w[6] - 2.f * SH_C2_4 * y * w[8];
  g[2] = SH_C1 * w[2] + SH_C2_1 * y * w[5] + 4.f * SH_C2_2 * z * w[6] + SH_C2_3 * x * w[7];
  if (K > 9) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    g[0] += SH_C3_0 * 6.f * xy * w[9] + SH_C3_1 * yz * w[10] - SH_C3_2 * 2.f * xy * w[11] - SH_C3_3 * 6.f * xz * w[12] +
            SH_C3_4 * (4.f * zz - 3.f * xx - yy) * w[13] + SH_C3_5 * 2.f * xz * w[14] + SH_C3_6 * 3.f * (xx - yy) * w[15];
    g[1] += SH_C3_0 * 3.f * (xx - yy) * w[9] + SH_C3_1 * xz * w[10] + SH_C3_2 * (4.f * zz - xx - 3.f * yy) * w[11] -
            SH_C3_3 * 6.f * yz * w[12] - SH_C3_4 * 2.f * xy * w[13] - SH_C3_5 * 2.f * yz * w[14] - SH_C3_6 * 6.f * xy * w[15];
    g[2] += SH_C3_1 * xy * w[10] + SH_C3_2 * 8.f * yz * w[11] + SH_C3_3 * (6.f * zz - 3.f * xx - 3.f * yy) * w[12] +
            SH_C3_4 * 8.f * xz * w[13] + SH_C3_5 * (xx - yy) * w[14];
  }
}

// ray direction of padded pixel (ix, iy): gaussian.cu:849-860
template <int K>
__device__ __forceinline__ void pixel_sh(int ix, int iy, const float* __restrict__ rays_o,
                                         const float* __restrict__ lefttop, const float* __restrict__ vdx,
                                         const float* __restrict__ vdy, float* out) {
  float d[3], nn = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    d[i] = __ldg(lefttop + i) + (float)ix * __ldg(vdx + i) + (float)iy * __ldg(vdy + i) - __ldg(rays_o + i);
    nn += d[i] * d[i];
  }
  const float inv = 1.f / (sqrtf(nn) + 1e-7f);
  sh_basis<K>(d[0] * inv, d[1] * inv, d[2] * inv, out);
}

__device__ __forceinline__ float sh_sigmoid(float x) { return gs_rcp(1.f + gs_ex2(-x * GS_LOG2E)); }

// reduce 8 values over the warp: afterwards lane L holds the total of value ((L >> 2) & 7)
// (bit 4 -> +4, bit 3 -> +2, bit 2 -> +1) in v[0]; 9 SHFL instead of 40
__device__ __forceinline__ float reduce8(float* v, int lane) {
  {
    const bool up = (lane & 16) != 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float keep = up ? v[u + 4] : v[u];
      const float send = up ? v[u] : v[u + 4];
      v[u] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  }
  {
    const bool up = (lane & 8) != 0;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const float keep = up ? v[u + 2] : v[u];
      const float send = up ? v[u] : v[u + 2];
      v[u] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
  }
  {
    const bool up = (lane & 4) != 0;
    const float keep = up ? v[1] : v[0];
    const float send = up ? v[0] : v[1];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
  return v[0];
}

}  // namespace gs_sh
