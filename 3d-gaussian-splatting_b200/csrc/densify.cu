// Densification on the device (SURVEY.md §8 f-2): prune / clone / split of reference
// splatter.py:122-228 (`Gaussian3ds.adaptive_control`, called from train.py:156-172) as
//   classify (1 kernel) -> three exclusive scans (CUB) -> apply (1 kernel writing the new arrays),
// instead of ~40 torch ops (boolean-mask gathers, cats, clones) and their host syncs.
// The new arrays have the reference's layout: [kept Gaussians in order (split ones moved to their first
// sample and shrunk)], [clones in order], [second samples of the split ones in order].
#include <cub/device/device_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <cmath>

#include "internal.h"

namespace {

constexpr int kBlock = 256;

struct FlagOf {
  const unsigned char* code;
  int bit;
  __host__ __device__ __forceinline__ int operator()(int i) const { return (code[i] >> bit) & 1; }
};

__device__ __forceinline__ float act_norm(const float* s, int act) {
  float a = s[0], b = s[1], c = s[2];
  if (act == GS_SCALE_EXP) {
    a = expf(a);
    b = expf(b);
    c = expf(c);
  }
  return sqrtf(a * a + b * b + c * c);                       // |scale| (abs) / |exp(scale)| (exp): splatter.py:129-136
}

// code of a kept Gaussian: bit 0, plus clone (bit 1, norm <= tau) or split (bit 2) when it densifies
__device__ __forceinline__ unsigned char densify_code(bool hit, float nrm, float tau, int use_clone, int use_split) {
  unsigned char c = 1;
  if (hit) {
    if (nrm > tau) {
      if (use_split) c |= 4;
    } else if (use_clone) {
      c |= 2;
    }
  }
  return c;
}

__global__ void __launch_bounds__(kBlock) densify_classify_kernel(const float* __restrict__ opa,
                                                                   const float* __restrict__ scale,
                                                                   const float* __restrict__ grad, int n, int act,
                                                                   float opa_logit_min, float delete_thresh,
                                                                   float grad_thresh, int agg_max, float tau,
                                                                   int use_clone, int use_split,
                                                                   unsigned char* __restrict__ code) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const float s[3] = {scale[3 * i], scale[3 * i + 1], scale[3 * i + 2]};
  const float nrm = act_norm(s, act);
  const bool keep = opa[i] > opa_logit_min && nrm < delete_thresh;          // splatter.py:137-139
  unsigned char c = 0;
  if (keep) {
    const float g0 = fabsf(grad[3 * i]), g1 = fabsf(grad[3 * i + 1]), g2 = fabsf(grad[3 * i + 2]);
    const float agg = agg_max ? fmaxf(g0, fmaxf(g1, g2)) : (g0 + g1 + g2) / 3.f;   // :152-157
    c = densify_code(agg > grad_thresh, nrm, tau, use_clone, use_split);
  }
  code[i] = c;
}

// Screen-space statistics (gs_densify_plan_stats): the 3DGS score accum / max(count, 1) >= grad_thresh, and with
// max_radius a prune of Gaussians that grew larger than max_screen_px on screen.
__global__ void __launch_bounds__(kBlock) densify_classify_stats_kernel(
    const float* __restrict__ opa, const float* __restrict__ scale, const float* __restrict__ accum,
    const int* __restrict__ count, const float* __restrict__ max_radius, float max_screen_px, int n, int act,
    float opa_logit_min, float delete_thresh, float grad_thresh, float tau, int use_clone, int use_split,
    unsigned char* __restrict__ code) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const float s[3] = {scale[3 * i], scale[3 * i + 1], scale[3 * i + 2]};
  const float nrm = act_norm(s, act);
  const bool keep = opa[i] > opa_logit_min && nrm < delete_thresh && !(max_radius && max_radius[i] > max_screen_px);
  unsigned char c = 0;
  if (keep) c = densify_code(accum[i] / (float)max(count[i], 1) >= grad_thresh, nrm, tau, use_clone, use_split);
  code[i] = c;
}

// wxyz -> R WITHOUT normalising (the reference builds the split covariance from the raw quaternion,
// splatter.py:100-103 -> utils.py:318-333)
__device__ __forceinline__ void quat_rot(const float4 q, float R[9]) {
  const float w = q.x, x = q.y, y = q.z, z = q.w;
  R[0] = 1 - 2 * y * y - 2 * z * z; R[1] = 2 * x * y - 2 * z * w;     R[2] = 2 * x * z + 2 * y * w;
  R[3] = 2 * x * y + 2 * z * w;     R[4] = 1 - 2 * x * x - 2 * z * z; R[5] = 2 * y * z - 2 * x * w;
  R[6] = 2 * x * z - 2 * y * w;     R[7] = 2 * y * z + 2 * x * w;     R[8] = 1 - 2 * x * x - 2 * y * y;
}

__global__ void __launch_bounds__(kBlock) densify_apply_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int d,
    const unsigned char* __restrict__ code, const int* __restrict__ dst_keep, const int* __restrict__ dst_clone,
    const int* __restrict__ dst_split, const float* __restrict__ grad, float clone_dt, const float* __restrict__ z,
    int n_split, int act, int n_keep, int n_clone, float* __restrict__ o_pos, float* __restrict__ o_rgb,
    float* __restrict__ o_opa, float* __restrict__ o_quat, float* __restrict__ o_scale) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const unsigned char c = code[i];
  if (!(c & 1)) return;                                            // pruned
  const float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  const float s[3] = {scale[3 * i], scale[3 * i + 1], scale[3 * i + 2]};
  const float4 q = reinterpret_cast<const float4*>(quat)[i];
  const float o = opa[i];
  auto put = [&](int row, const float* pp, const float* ss) {
    o_pos[3 * (size_t)row] = pp[0]; o_pos[3 * (size_t)row + 1] = pp[1]; o_pos[3 * (size_t)row + 2] = pp[2];
    o_scale[3 * (size_t)row] = ss[0]; o_scale[3 * (size_t)row + 1] = ss[1]; o_scale[3 * (size_t)row + 2] = ss[2];
    reinterpret_cast<float4*>(o_quat)[row] = q;
    o_opa[row] = o;
    const float* src = rgb + (size_t)i * d;
    float* dstc = o_rgb + (size_t)row * d;
    for (int k = 0; k < d; ++k) dstc[k] = src[k];
  };
  const int kr = dst_keep[i];
  if (c & 4) {
    // two positions drawn from N(pos, R diag(s_act^2) R^T) of the UN-shrunk Gaussian: pos + R (s_act * z)
    float R[9], sa[3], ss[3];
    quat_rot(q, R);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      sa[k] = act == GS_SCALE_ABS ? fabsf(s[k]) + 1e-4f : expf(s[k]);
      ss[k] = act == GS_SCALE_ABS ? s[k] / 1.6f : s[k] - 0.4700036292457356f;     // log(1.6)
    }
    const int j = dst_split[i];
    float p1[3], p2[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float a1 = 0.f, a2 = 0.f;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        a1 = fmaf(R[3 * r + k] * sa[k], z[3 * (size_t)j + k], a1);
        a2 = fmaf(R[3 * r + k] * sa[k], z[3 * ((size_t)n_split + j) + k], a2);
      }
      p1[r] = p[r] + a1;
      p2[r] = p[r] + a2;
    }
    put(kr, p1, ss);
    put(n_keep + n_clone + j, p2, ss);
  } else {
    put(kr, p, s);
    if (c & 2) {
      if (grad) {
        const float pc[3] = {p[0] - grad[3 * i] * clone_dt, p[1] - grad[3 * i + 1] * clone_dt,
                             p[2] - grad[3 * i + 2] * clone_dt};                  // splatter.py:170-171
        put(n_keep + dst_clone[i], pc, s);
      } else {
        put(n_keep + dst_clone[i], p, s);                                       // exact copy (3DGS)
      }
    }
  }
}

// row i of a per-Gaussian [n, w] tensor to the rows densify_apply_kernel gives Gaussian i: kept, clone, second split
// sample; every one an exact copy
__global__ void __launch_bounds__(kBlock) densify_apply_rows_kernel(
    const float* __restrict__ src, int n, int w, const unsigned char* __restrict__ code,
    const int* __restrict__ dst_keep, const int* __restrict__ dst_clone, const int* __restrict__ dst_split, int n_keep,
    int n_clone, float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= (long long)n * w) return;
  const int i = (int)(t / w), k = (int)(t % w);
  const unsigned char c = code[i];
  if (!(c & 1)) return;                                            // pruned
  const float v = src[t];
  out[(size_t)dst_keep[i] * w + k] = v;
  if (c & 4) out[((size_t)n_keep + n_clone + dst_split[i]) * w + k] = v;
  else if (c & 2) out[((size_t)n_keep + dst_clone[i]) * w + k] = v;
}

inline size_t up256(size_t x) { return (x + 255) / 256 * 256; }

size_t scan_tmp_bytes(int n) {
  size_t b = 0;
  FlagOf f{nullptr, 0};
  cub::CountingInputIterator<int> idx(0);
  cub::TransformInputIterator<int, FlagOf, cub::CountingInputIterator<int>> it(idx, f);
  cub::DeviceScan::ExclusiveSum(nullptr, b, it, static_cast<int*>(nullptr), n + 1);
  return b;
}

}  // namespace

extern "C" size_t gs_densify_workspace_bytes(int n) { return n < 0 ? 0 : up256(scan_tmp_bytes(n)) + 256; }

// dst[3][n+1] = exclusive scans of the three flag bits of code[n+1]
static int plan_scans(unsigned char* code, int* dst, int n, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  // code[n] is read by the (n+1)-item scans: the caller provides n+1 bytes, the last one zero
  GS_CUDA_TRY(cudaMemsetAsync(code + n, 0, 1, st));
  size_t tmp = workspace_bytes;
  for (int b = 0; b < 3; ++b) {
    FlagOf f{code, b};
    cub::CountingInputIterator<int> idx(0);
    cub::TransformInputIterator<int, FlagOf, cub::CountingInputIterator<int>> it(idx, f);
    GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(workspace, tmp, it, dst + (size_t)b * (n + 1), n + 1, st));
  }
  return 0;
}

extern "C" int gs_densify_plan(const float* opa, const float* scale, const float* grad, int n, int scale_activation,
                               float opa_logit_min, float delete_thresh, float grad_thresh, int grad_agg_max, float tau,
                               int use_clone, int use_split, unsigned char* code, int* dst, void* workspace,
                               size_t workspace_bytes, gs_stream_t stream) {
  if (n < 0 || (n > 0 && (!opa || !scale || !grad || !code || !dst || !workspace)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_plan: bad arguments");
  if (workspace_bytes < gs_densify_workspace_bytes(n))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_plan: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  densify_classify_kernel<<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(opa, scale, grad, n, scale_activation,
                                                                       opa_logit_min, delete_thresh, grad_thresh,
                                                                       grad_agg_max, tau, use_clone, use_split, code);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return plan_scans(code, dst, n, workspace, workspace_bytes, st);
}

extern "C" int gs_densify_plan_stats(const float* opa, const float* scale, const float* accum, const int* count,
                                     const float* max_radius, float max_screen_px, int n, int scale_activation,
                                     float opa_logit_min, float delete_thresh, float grad_thresh, float tau,
                                     int use_clone, int use_split, unsigned char* code, int* dst, void* workspace,
                                     size_t workspace_bytes, gs_stream_t stream) {
  if (n < 0 || (n > 0 && (!opa || !scale || !accum || !count || !code || !dst || !workspace)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_plan_stats: bad arguments");
  if (max_radius && std::isnan(max_screen_px))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_plan_stats: max_screen_px is NaN");
  if (workspace_bytes < gs_densify_workspace_bytes(n))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_plan_stats: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  densify_classify_stats_kernel<<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(
      opa, scale, accum, count, max_radius, max_screen_px, n, scale_activation, opa_logit_min, delete_thresh,
      grad_thresh, tau, use_clone, use_split, code);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return plan_scans(code, dst, n, workspace, workspace_bytes, st);
}

extern "C" int gs_densify_apply(const float* pos, const float* rgb, const float* opa, const float* quat,
                                const float* scale, int n, int d, const unsigned char* code, const int* dst,
                                const float* grad, float clone_dt, const float* normals, int n_keep, int n_clone,
                                int n_split, int scale_activation, float* out_pos, float* out_rgb, float* out_opa,
                                float* out_quat, float* out_scale, gs_stream_t stream) {
  if (n < 0 || d <= 0 || n_keep < 0 || n_clone < 0 || n_split < 0 || (n_split > 0 && !normals))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_apply: bad arguments");
  if (n == 0) return 0;
  densify_apply_kernel<<<(n + kBlock - 1) / kBlock, kBlock, 0, (cudaStream_t)stream>>>(
      pos, rgb, opa, quat, scale, n, d, code, dst, dst + (n + 1), dst + 2 * (size_t)(n + 1), grad, clone_dt, normals,
      n_split, scale_activation, n_keep, n_clone, out_pos, out_rgb, out_opa, out_quat, out_scale);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_densify_apply_rows(const float* src, int n, int w, const unsigned char* code, const int* dst,
                                     int n_keep, int n_clone, int n_split, float* out, gs_stream_t stream) {
  if (n < 0 || w <= 0 || n_keep < 0 || n_clone < 0 || n_split < 0 ||
      (n > 0 && (!src || !code || !dst || (n_keep + n_clone + n_split > 0 && !out))))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_densify_apply_rows: bad arguments");
  if (n == 0) return 0;
  const long long threads = (long long)n * w;
  densify_apply_rows_kernel<<<(int)((threads + kBlock - 1) / kBlock), kBlock, 0, (cudaStream_t)stream>>>(
      src, n, w, code, dst, dst + (n + 1), dst + 2 * (size_t)(n + 1), n_keep, n_clone, out);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}
