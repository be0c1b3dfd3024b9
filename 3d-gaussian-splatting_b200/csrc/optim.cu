// Fused Adam over the flat parameter / gradient buckets (SURVEY.md §8 f-2).
// The reference steps torch.optim.Adam with 5 parameter groups (train.py:56-64: opa, rgb, pos,
// scale, quat; betas (0.9, 0.99), eps 1e-8, no weight decay) right after the rasterizer backward.
// Here the five gradients already live in ONE flat buffer written by fused_project_bwd_kernel
// (and all-reduced in place), so the optimizer is a single HBM-bound pass: 4 streams read
// (p, g, m, v), 3 written.  Same update as torch's `_single_tensor_adam`:
//   m += (1-b1)(g-m);  v = b2 v + (1-b2) g^2;  p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
#include "internal.h"

#include <cmath>

namespace {

constexpr int kMaxSeg = 8;
struct AdamSegs {
  long long end[kMaxSeg];    // exclusive end (in floats) of each segment of the flat buffer
  float step_size[kMaxSeg];  // lr / bias_correction1 per segment
  int n;
};

__global__ void __launch_bounds__(256) adam_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                    float4* __restrict__ m, float4* __restrict__ v, long long n4,
                                                    AdamSegs segs, float beta1, float beta2, float inv_bc2_sqrt,
                                                    float eps) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n4) return;
  // segments are 16-byte aligned (renderer._flat_grads), so a float4 never straddles two of them
  const long long e0 = i * 4;
  float step = segs.step_size[0];
#pragma unroll
  for (int s = 1; s < kMaxSeg; ++s)
    if (s < segs.n && e0 >= segs.end[s - 1]) step = segs.step_size[s];
  const float4 gg = g[i];
  float4 mm = m[i], vv = v[i], pp = p[i];
  const float om1 = 1.f - beta1, om2 = 1.f - beta2;
#define GS_ADAM(C)                                            \
  mm.C = fmaf(om1, gg.C - mm.C, mm.C);                        \
  vv.C = fmaf(om2 * gg.C, gg.C, beta2 * vv.C);                \
  pp.C -= step * (mm.C / (sqrtf(vv.C) * inv_bc2_sqrt + eps));
  GS_ADAM(x) GS_ADAM(y) GS_ADAM(z) GS_ADAM(w)
#undef GS_ADAM
  m[i] = mm;
  v[i] = vv;
  p[i] = pp;
}

// ---- visible-only Adam (gs_adam_step_visible) ------------------------------------------------
// The rows of the Gaussians the last frames binned, and nothing else: an unseen Gaussian keeps its parameters and
// both moments.  DRAM traffic follows the visible rows: a warp owns 32 consecutive Gaussians, reads their 32 mask
// bytes with one request, and walks, segment by segment, the floats of its visible rows only, consecutive lanes on
// consecutive floats of a row and on through the next visible row, so a run of visible rows is one contiguous run of
// whole sectors.  Segments whose rows are whole float4s (quat; SH degree 3's 48 floats) move as float4.

struct AdamRowSegs {
  long long start[kMaxSeg];  // first float of segment s = row-major [n_rows, width[s]]
  int width[kMaxSeg];
  float step_size[kMaxSeg];  // lr / bias_correction1 per segment
  int n;
};

// adam_kernel's update with every rounding spelled out, so that no other contraction can be chosen here.  In its SASS
// the two moment updates and sqrt(v) * inv_bc2_sqrt + eps are FFMAs and the square root and the quotient are the
// correctly rounded ones; p - step * q is an FMUL followed by an FADD for the x, y and z components of a float4 and
// one FFMA (-step * q + p) for w.  The dense kernel's results are pinned, so `last` (the float is the fourth of its
// aligned group of four in the flat buffer) selects the same rounding here.
__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, bool last, float om1, float om2,
                                            float beta2, float inv_bc2_sqrt, float eps, float step) {
  m = __fmaf_rn(om1, __fsub_rn(g, m), m);
  v = __fmaf_rn(__fmul_rn(om2, g), g, __fmul_rn(beta2, v));
  const float q = __fdiv_rn(m, __fmaf_rn(__fsqrt_rn(v), inv_bc2_sqrt, eps));
  p = last ? __fmaf_rn(-step, q, p) : __fsub_rn(p, __fmul_rn(step, q));
}
__device__ __forceinline__ void adam_update(float4& p, const float4& g, float4& m, float4& v, bool, float om1,
                                            float om2, float beta2, float inv_bc2_sqrt, float eps, float step) {
  adam_update(p.x, g.x, m.x, v.x, false, om1, om2, beta2, inv_bc2_sqrt, eps, step);
  adam_update(p.y, g.y, m.y, v.y, false, om1, om2, beta2, inv_bc2_sqrt, eps, step);
  adam_update(p.z, g.z, m.z, v.z, false, om1, om2, beta2, inv_bc2_sqrt, eps, step);
  adam_update(p.w, g.w, m.w, v.w, true, om1, om2, beta2, inv_bc2_sqrt, eps, step);
}

// The warp's nv visible rows (local indices rows[0 .. nv)) of one segment whose rows are w elements of T (float or
// float4) and whose row 0 of this warp is at p / g / m / v: item t = (visible row t / w, element t % w), lane by lane.
// Scalar items are taken four at a time, all loads before the first update, to keep enough bytes in flight; o4 is
// the position of p in its aligned group of four floats (0 for float4 rows).
template <typename T>
__device__ __forceinline__ void adam_rows(T* __restrict__ p, const T* __restrict__ g, T* __restrict__ m,
                                          T* __restrict__ v, int o4, int w, const unsigned char* rows, int nv,
                                          int lane, float om1, float om2, float beta2, float inv_bc2_sqrt, float eps,
                                          float step) {
  constexpr int U = sizeof(T) == sizeof(float) ? 4 : 1;
  const int total = nv * w;
  const int dr = 32 / w, de = 32 - dr * w;   // 32 items further on: dr rows and de elements
  int r = lane / w, e = lane - r * w;
  for (int t = lane; t < total; t += 32 * U) {
    int idx[U];
    T gg[U], mm[U], vv[U], pp[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      idx[u] = t + 32 * u < total ? (int)rows[r] * w + e : -1;
      r += dr;
      e += de;
      if (e >= w) {
        e -= w;
        ++r;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (idx[u] >= 0) {
        gg[u] = g[idx[u]];
        mm[u] = m[idx[u]];
        vv[u] = v[idx[u]];
        pp[u] = p[idx[u]];
      }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (idx[u] >= 0) {
        adam_update(pp[u], gg[u], mm[u], vv[u], ((o4 + idx[u]) & 3) == 3, om1, om2, beta2, inv_bc2_sqrt, eps,
                    step);
        m[idx[u]] = mm[u];
        v[idx[u]] = vv[u];
        p[idx[u]] = pp[u];
      }
  }
}

constexpr int kRowBlock = 256;

__global__ void __launch_bounds__(kRowBlock) adam_visible_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                                 float* __restrict__ m, float* __restrict__ v,
                                                                 AdamRowSegs segs, int n_rows,
                                                                 const unsigned char* __restrict__ visible, float beta1,
                                                                 float beta2, float inv_bc2_sqrt, float eps) {
  __shared__ unsigned char rows_sh[kRowBlock / 32][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long row0 = ((long long)blockIdx.x * (kRowBlock / 32) + warp) * 32;
  if (row0 >= n_rows) return;
  const bool vis = row0 + lane < n_rows && visible[row0 + lane] != 0;
  const unsigned ballot = __ballot_sync(0xffffffffu, vis);
  if (ballot == 0) return;   // no load of p / g / m / v was issued
  unsigned char* rows = rows_sh[warp];
  if (vis) rows[__popc(ballot & ((1u << lane) - 1u))] = (unsigned char)lane;
  __syncwarp();
  const int nv = __popc(ballot);
  const float om1 = 1.f - beta1, om2 = 1.f - beta2;
  for (int s = 0; s < segs.n; ++s) {
    const int w = segs.width[s];
    const long long o = segs.start[s] + row0 * w;   // a multiple of 4 floats when w % 4 == 0 (start is one, row0 of 32)
    const float step = segs.step_size[s];
    if ((w & 3) == 0)
      adam_rows(reinterpret_cast<float4*>(p + o), reinterpret_cast<const float4*>(g + o),
                reinterpret_cast<float4*>(m + o), reinterpret_cast<float4*>(v + o), 0, w >> 2, rows, nv, lane, om1,
                om2, beta2, inv_bc2_sqrt, eps, step);
    else
      adam_rows(p + o, g + o, m + o, v + o, (int)(o & 3), w, rows, nv, lane, om1, om2, beta2, inv_bc2_sqrt, eps,
                step);
  }
}

// visible[i] = Gaussian i got a tile instance in any of the n_views views of the last forward (count[v n + i] > 0),
// OR what visible[i] held when accumulate is set
__global__ void __launch_bounds__(256) frame_visible_kernel(const uint32_t* __restrict__ count, int n, int n_views,
                                                            int accumulate, unsigned char* __restrict__ visible) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  bool vis = accumulate && visible[i] != 0;
  for (int v = 0; v < n_views && !vis; ++v) vis = count[(size_t)v * n + i] != 0;
  visible[i] = vis ? 1 : 0;
}

}  // namespace

cudaError_t gs_launch_frame_visible(const uint32_t* count, int n, int n_views, int accumulate, unsigned char* visible,
                                    cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  frame_visible_kernel<<<(n + 255) / 256, 256, 0, st>>>(count, n, n_views, accumulate, visible);
  return cudaGetLastError();
}

extern "C" int gs_adam_step_visible(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                    long long n_flat, const long long* seg_start_host, const int* seg_width_host,
                                    const float* lr_host, int n_seg, int n_rows, const unsigned char* visible,
                                    float beta1, float beta2, float eps, int step, gs_stream_t stream) {
  if (n_flat < 0 || n_seg < 1 || n_seg > kMaxSeg || step < 1 || n_rows < 0 || !seg_start_host || !seg_width_host ||
      !lr_host)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step_visible: bad arguments");
  if (n_flat % 4)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step_visible: flat length must be a multiple of 4 floats");
  AdamRowSegs segs{};
  segs.n = n_seg;
  const double bc1 = 1.0 - std::pow((double)beta1, (double)step);
  const double bc2 = 1.0 - std::pow((double)beta2, (double)step);
  long long prev_end = 0;
  for (int s = 0; s < n_seg; ++s) {
    const long long start = seg_start_host[s];
    if (seg_width_host[s] < 1 || seg_width_host[s] > (1 << 24))   // 32 rows of a segment are indexed in an int
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step_visible: segment widths must be in 1 .. 2^24");
    if (start % 4 || start < prev_end)
      return gs_set_error_msg(GS_ERR_INVALID_ARG,
                              "gs_adam_step_visible: segment starts must be ascending multiples of 4 and the segments "
                              "must not overlap");
    prev_end = start + (long long)n_rows * seg_width_host[s];
    if (prev_end > n_flat)
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step_visible: a segment ends beyond the flat buffer");
    segs.start[s] = start;
    segs.width[s] = seg_width_host[s];
    segs.step_size[s] = (float)((double)lr_host[s] / bc1);
  }
  if (n_rows == 0) return 0;
  if (!param || !grad || !exp_avg || !exp_avg_sq || !visible)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step_visible: null buffer");
  const long long warps = ((long long)n_rows + 31) / 32;
  adam_visible_kernel<<<(unsigned)((warps + kRowBlock / 32 - 1) / (kRowBlock / 32)), kRowBlock, 0,
                        (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, segs, n_rows, visible, beta1, beta2,
                                                (float)(1.0 / std::sqrt(bc2)), eps);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                            const long long* seg_end_host, const float* lr_host, int n_seg, float beta1, float beta2,
                            float eps, int step, gs_stream_t stream) {
  if (n < 0 || n_seg < 1 || n_seg > kMaxSeg || step < 1 || !seg_end_host || !lr_host)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step: bad arguments");
  if (n % 4) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step: flat length must be a multiple of 4 floats");
  if (n == 0) return 0;
  AdamSegs segs{};
  segs.n = n_seg;
  const double bc1 = 1.0 - std::pow((double)beta1, (double)step);
  const double bc2 = 1.0 - std::pow((double)beta2, (double)step);
  for (int s = 0; s < n_seg; ++s) {
    if (seg_end_host[s] % 4 || (s && seg_end_host[s] < seg_end_host[s - 1]))
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_adam_step: segment ends must be ascending multiples of 4");
    segs.end[s] = seg_end_host[s];
    segs.step_size[s] = (float)((double)lr_host[s] / bc1);
  }
  const long long n4 = n / 4;
  adam_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<float4*>(param), reinterpret_cast<const float4*>(grad), reinterpret_cast<float4*>(exp_avg),
      reinterpret_cast<float4*>(exp_avg_sq), n4, segs, beta1, beta2, (float)(1.0 / std::sqrt(bc2)), eps);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}
