// MCMC densification on the device (3DGS-MCMC, Kheradmand et al. 2024; gsplat's MCMCStrategy): relocation of dead
// Gaussians onto live ones, growth to a cap, and the position noise added after every optimizer step.
//
//   sampler : weight (o_i in 2^-32 fixed point, dead flags) -> CUB inclusive scan of the uint64 weights -> CUB
//             compaction of the dead indices -> draw (one thread per draw: binary search on the prefix sums, integer
//             atomicAdd into the counts)
// Every sum of the sampler is an integer sum, so the prefix sums, and with them every draw, are the same bits whatever
// order the scan's tiles combine in: same-seed runs and data-parallel replicas draw identical sources.  (A floating-
// point scan would not be: CUB's decoupled look-back adds tile prefixes in a timing-dependent order.)
//   apply A : one thread per draw reads the ORIGINAL source row, evaluates (o', s') in fp64 and writes the whole
//             destination row
//   apply B : one thread per draw copies (opa, scale) of the destination back into the source row and zeroes the
//             moment rows of both
// Destinations are dead rows (relocation) or appended rows (growth), never sources, so A never reads what it writes;
// B runs after A because a source's opacity must not be read after another draw rewrote it.  The number of draws
// stays on the device: the launches cover its upper bound and exit past it, so no entry synchronises.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <curand_kernel.h>

#include <cmath>

#include "internal.h"

namespace {

constexpr int kBlock = 256;
constexpr int kMaxRatio = 51;   // gsplat's n_max: the ratio r is clamped to 1 .. 51
constexpr int kMaxSeg = 8;      // segments of the moment buffers (gs_adam_step_visible's limit)
constexpr double kWeightScale = 4294967296.0;   // 2^32: weights are round(o * 2^32); n < 2^31 keeps the total < 2^63

struct MomentSegs {
  long long start[kMaxSeg];   // first float of segment s = row-major [n, width[s]]
  int width[kMaxSeg];
  int n;
};

__device__ __forceinline__ double sigmoid_d(float x) { return 1.0 / (1.0 + exp(-(double)x)); }

// w_i = round(o_i 2^32) (round half to even; 0 for a dead Gaussian when relocating), dead_i = o_i <= min_opacity
__global__ void __launch_bounds__(kBlock) mcmc_weight_kernel(const float* __restrict__ opa, int n, double min_opacity,
                                                             int zero_dead, unsigned long long* __restrict__ w,
                                                             unsigned char* __restrict__ dead) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const double o = sigmoid_d(opa[i]);
  const bool d = o <= min_opacity;
  w[i] = (zero_dead && d) ? 0ull : (unsigned long long)__double2ll_rn(o * kWeightScale);
  dead[i] = d ? 1 : 0;
}

// Draw j < k (k = *k_dev, or k_host when k_dev is NULL): t_j = min(floor(u_j C_{n-1}), C_{n-1} - 1) (the product in
// fp64), src_j = min{i : C_i > t_j}, count[src_j] += 1; a Gaussian of weight 0 is never drawn.  Thread 0 publishes
// the number of draws that take effect.  A total weight of 0 relocates nothing (k_dev given: nothing is alive); growth
// (k_dev NULL; every opacity below 2^-33) then appends plain copies of row 0 (no count, r = 1).
__global__ void __launch_bounds__(kBlock) mcmc_draw_kernel(const unsigned long long* __restrict__ C, int n,
                                                           const float* __restrict__ u, const int* __restrict__ k_dev,
                                                           int k_host, int* __restrict__ src, int* __restrict__ count,
                                                           int* __restrict__ n_draws) {
  const int j = blockIdx.x * kBlock + threadIdx.x;
  const int k = k_dev ? *k_dev : k_host;
  const unsigned long long total = C[n - 1];
  const bool empty = total == 0ull;
  if (j == 0) *n_draws = (empty && k_dev) ? 0 : k;
  if (j >= k) return;
  if (empty) {
    src[j] = 0;
    return;
  }
  unsigned long long t = __double2ull_rd((double)u[j] * (double)total);
  if (t >= total) t = total - 1;   // the fp64 product may round up to the total
  int lo = 0, hi = n - 1;          // C[n-1] > t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (C[mid] > t) hi = mid;
    else lo = mid + 1;
  }
  src[j] = lo;
  atomicAdd(count + lo, 1);
}

// (o', coefficient s'/s) for a source of activated opacity o drawn r - 1 times (3DGS-MCMC eq. 9, gsplat's
// compute_relocation).  den = sum_{a=1..r} sum_{b=0..a-1} C(a-1, b) (-1)^b o'^(b+1) / sqrt(b+1) is evaluated as
// sum_{b=0..r-1} C(r, b+1) (-1)^b o'^(b+1) / sqrt(b+1) (sum_{a=b+1..r} C(a-1, b) = C(r, b+1)); the binomials are
// exact integers in fp64 (C(51, 26) * 26 < 2^53), the alternating sum is kept in fp64 because it cancels.
__device__ __forceinline__ void mcmc_ratio(double o, int r, double& o_new, double& coef) {
  o_new = 1.0 - pow(1.0 - o, 1.0 / (double)r);
  double den = 0.0, c = 1.0, pw = 1.0;   // c = C(r, b), pw = o'^b
  for (int b = 0; b < r; ++b) {
    c = c * (double)(r - b) / (double)(b + 1);
    pw *= o_new;
    const double term = c * pw / sqrt((double)(b + 1));
    den += (b & 1) ? -term : term;
  }
  coef = den > 0.0 ? o / den : 1.0;
}

__global__ void __launch_bounds__(kBlock) mcmc_apply_rows_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, const float* __restrict__ feat, int d, int f,
    int act, double min_opacity, const int* __restrict__ n_draws, const int* __restrict__ src,
    const int* __restrict__ dst_list, int dst_base, const int* __restrict__ count, float* __restrict__ o_pos,
    float* __restrict__ o_rgb, float* __restrict__ o_opa, float* __restrict__ o_quat, float* __restrict__ o_scale,
    float* __restrict__ o_feat) {
  const int j = blockIdx.x * kBlock + threadIdx.x;
  if (j >= *n_draws) return;
  const int i = src[j];
  const size_t t = dst_list ? (size_t)dst_list[j] : (size_t)dst_base + j;
  const int r = min(1 + count[i], kMaxRatio);
  if (r == 1) {   // an undrawn source (growth with every weight 0): a plain copy
    o_opa[t] = opa[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) o_scale[3 * t + k] = scale[3 * (size_t)i + k];
  } else {
    const double o = sigmoid_d(opa[i]);
    double o_new, coef;
    mcmc_ratio(o, r, o_new, coef);
    o_new = fmin(fmax(o_new, min_opacity), 1.0 - 0x1p-23);
    o_opa[t] = (float)log(o_new / (1.0 - o_new));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float raw = scale[3 * (size_t)i + k];
      const double s = act == GS_SCALE_ABS ? fabs((double)raw) + 1e-4 : exp((double)raw);
      const double s_new = coef * s;
      o_scale[3 * t + k] = act == GS_SCALE_ABS ? (float)copysign(fmax(s_new - 1e-4, 0.0), raw < 0.f ? -1.0 : 1.0)
                                               : (float)log(s_new);
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) o_pos[3 * t + k] = pos[3 * (size_t)i + k];
  reinterpret_cast<float4*>(o_quat)[t] = reinterpret_cast<const float4*>(quat)[i];
  for (int k = 0; k < d; ++k) o_rgb[t * d + k] = rgb[(size_t)i * d + k];
  if (feat)
    for (int k = 0; k < f; ++k) o_feat[t * f + k] = feat[(size_t)i * f + k];
}

// the source takes its destination's new (opa, scale) (every draw of one source writes the same bits); the moment rows
// of source and destination are zeroed in every segment, and both rows flagged in `touched`
__global__ void __launch_bounds__(kBlock) mcmc_apply_sources_kernel(
    const int* __restrict__ n_draws, const int* __restrict__ src, const int* __restrict__ dst_list, int dst_base,
    float* __restrict__ o_opa, float* __restrict__ o_scale, float* __restrict__ m, float* __restrict__ v,
    MomentSegs segs, unsigned char* __restrict__ touched) {
  const int j = blockIdx.x * kBlock + threadIdx.x;
  if (j >= *n_draws) return;
  const size_t i = src[j];
  const size_t t = dst_list ? (size_t)dst_list[j] : (size_t)dst_base + j;
  o_opa[i] = o_opa[t];
#pragma unroll
  for (int k = 0; k < 3; ++k) o_scale[3 * i + k] = o_scale[3 * t + k];
  if (m) {
#pragma unroll
    for (int s = 0; s < kMaxSeg; ++s) {
      if (s >= segs.n) break;
      const int w = segs.width[s];
      for (int k = 0; k < w; ++k) {
        m[segs.start[s] + i * w + k] = 0.f;
        v[segs.start[s] + i * w + k] = 0.f;
        m[segs.start[s] + t * w + k] = 0.f;
        v[segs.start[s] + t * w + k] = 0.f;
      }
    }
  }
  if (touched) {
    touched[i] = 1;
    touched[t] = 1;
  }
}

// pos_i += scaler g(o_i) R diag(s^2) R^T z_i, g(o) = sigmoid(100 ((1 - o) - 0.995)); z_i from z (caller's) or from
// Philox(seed, subsequence i)
__global__ void __launch_bounds__(kBlock) mcmc_noise_kernel(float* __restrict__ pos, const float* __restrict__ quat,
                                                            const float* __restrict__ scale,
                                                            const float* __restrict__ opa, int n, int act, float scaler,
                                                            unsigned long long seed, const float* __restrict__ z) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float zz[3];
  if (z) {
    zz[0] = z[3 * (size_t)i];
    zz[1] = z[3 * (size_t)i + 1];
    zz[2] = z[3 * (size_t)i + 2];
  } else {
    curandStatePhilox4_32_10_t rs;
    curand_init(seed, (unsigned long long)i, 0ull, &rs);
    const float4 g4 = curand_normal4(&rs);
    zz[0] = g4.x;
    zz[1] = g4.y;
    zz[2] = g4.z;
  }
  float q[4], s[3], raw_s[3], qnorm;
  gs_load_activated(quat, scale, i, act, q, s, raw_s, qnorm);
  const GsRot R = gs_quat_to_rot(q[0], q[1], q[2], q[3]);
  // the gate in fp64: (1 - o) - 0.995 cancels and is then scaled by 100
  const double one_minus_o = 1.0 / (1.0 + exp((double)opa[i]));
  const float gate = (float)(1.0 / (1.0 + exp(-100.0 * (one_minus_o - 0.995))));
  float a[3];   // diag(s^2) R^T z
#pragma unroll
  for (int k = 0; k < 3; ++k) a[k] = s[k] * s[k] * (R.m[k] * zz[0] + R.m[3 + k] * zz[1] + R.m[6 + k] * zz[2]);
  const float c = scaler * gate;
#pragma unroll
  for (int r = 0; r < 3; ++r)
    pos[3 * (size_t)i + r] += c * (R.m[3 * r] * a[0] + R.m[3 * r + 1] * a[1] + R.m[3 * r + 2] * a[2]);
}

inline size_t up256(size_t x) { return (x + 255) / 256 * 256; }

size_t cub_tmp_bytes(int n) {
  size_t a = 0, b = 0;
  cub::DeviceScan::InclusiveSum(nullptr, a, static_cast<const unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), n);
  cub::CountingInputIterator<int> idx(0);
  cub::DeviceSelect::Flagged(nullptr, b, idx, static_cast<const unsigned char*>(nullptr), static_cast<int*>(nullptr),
                             static_cast<int*>(nullptr), n);
  return a > b ? a : b;
}

// workspace carve-up for a sampler over n Gaussians with up to n draws
struct Ws {
  unsigned long long *w, *C;
  unsigned char* dead;
  int *dead_idx, *src, *count, *k, *n_draws;
  void* tmp;
  size_t tmp_bytes;
};

Ws carve(void* base, int n) {
  char* p = static_cast<char*>(base);
  Ws ws;
  const size_t nn = n > 0 ? n : 1;
  ws.w = reinterpret_cast<unsigned long long*>(p); p += up256(nn * sizeof(unsigned long long));
  ws.C = reinterpret_cast<unsigned long long*>(p); p += up256(nn * sizeof(unsigned long long));
  ws.dead_idx = reinterpret_cast<int*>(p); p += up256(nn * sizeof(int));
  ws.src = reinterpret_cast<int*>(p); p += up256(nn * sizeof(int));
  ws.count = reinterpret_cast<int*>(p); p += up256(nn * sizeof(int));
  ws.k = reinterpret_cast<int*>(p); p += 256;
  ws.n_draws = reinterpret_cast<int*>(p); p += 256;
  ws.dead = reinterpret_cast<unsigned char*>(p); p += up256(nn);
  ws.tmp = p;
  ws.tmp_bytes = up256(cub_tmp_bytes(n > 0 ? n : 1));
  return ws;
}

inline int grid(long long threads) { return (int)((threads + kBlock - 1) / kBlock); }

bool misaligned(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; }   // quat rows move as float4

bool bad_widths(int d, const float* feat, int f) {
  return !(d == 3 || d == 27 || d == 48) || (feat && !(f == 8 || f == 16 || f == 32));
}

}  // namespace

extern "C" size_t gs_mcmc_workspace_bytes(int n) {
  if (n < 0) return 0;
  const size_t nn = n > 0 ? n : 1;
  return 2 * up256(nn * sizeof(unsigned long long)) + 3 * up256(nn * sizeof(int)) + 512 + up256(nn) +
         up256(cub_tmp_bytes((int)nn));
}

extern "C" int gs_mcmc_relocate(float* pos, float* rgb, float* opa, float* quat, float* scale, float* feat, int f, int n,
                                int d, int scale_activation, float min_opacity, const float* u, float* exp_avg,
                                float* exp_avg_sq, long long n_flat, const long long* seg_start_host,
                                const int* seg_width_host, int n_seg, unsigned char* touched, int* n_relocated,
                                void* workspace, size_t workspace_bytes, gs_stream_t stream) {
  if (n < 0 || (n > 0 && (!pos || !rgb || !opa || !quat || !scale || !u || !n_relocated || !workspace)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: bad arguments");
  if (bad_widths(d, feat, f))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: d must be 3, 27 or 48 and f 8, 16 or 32");
  if (misaligned(quat)) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: quat must be 16-byte aligned");
  if (scale_activation != GS_SCALE_ABS && scale_activation != GS_SCALE_EXP)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: unknown scale activation");
  if (!(min_opacity > 0.f && min_opacity < 1.f))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: min_opacity must be in (0, 1)");
  MomentSegs segs{};
  if (exp_avg || exp_avg_sq) {
    if (!exp_avg || !exp_avg_sq || n_seg < 1 || n_seg > kMaxSeg || !seg_start_host || !seg_width_host || n_flat < 0 ||
        n_flat % 4)
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: bad moment buffers or segment table");
    long long prev_end = 0;
    for (int s = 0; s < n_seg; ++s) {
      const long long start = seg_start_host[s];
      if (seg_width_host[s] < 1 || seg_width_host[s] > (1 << 24))
        return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: segment widths must be in 1 .. 2^24");
      if (start % 4 || start < prev_end)
        return gs_set_error_msg(GS_ERR_INVALID_ARG,
                                "gs_mcmc_relocate: segment starts must be ascending multiples of 4 and the segments "
                                "must not overlap");
      prev_end = start + (long long)n * seg_width_host[s];
      if (prev_end > n_flat)
        return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: a segment ends beyond the flat buffer");
      segs.start[s] = start;
      segs.width[s] = seg_width_host[s];
    }
    segs.n = n_seg;
  }
  if (workspace_bytes < gs_mcmc_workspace_bytes(n))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_relocate: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  Ws ws = carve(workspace, n);
  GS_CUDA_TRY(cudaMemsetAsync(ws.count, 0, (size_t)n * sizeof(int), st));
  mcmc_weight_kernel<<<grid(n), kBlock, 0, st>>>(opa, n, (double)min_opacity, 1, ws.w, ws.dead);
  GS_CUDA_TRY(cudaGetLastError());
  size_t tb = ws.tmp_bytes;
  GS_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws.tmp, tb, ws.w, ws.C, n, st));
  tb = ws.tmp_bytes;
  GS_CUDA_TRY(cub::DeviceSelect::Flagged(ws.tmp, tb, cub::CountingInputIterator<int>(0), ws.dead, ws.dead_idx, ws.k, n,
                                         st));
  mcmc_draw_kernel<<<grid(n), kBlock, 0, st>>>(ws.C, n, u, ws.k, 0, ws.src, ws.count, n_relocated);
  GS_CUDA_TRY(cudaGetLastError());
  mcmc_apply_rows_kernel<<<grid(n), kBlock, 0, st>>>(pos, rgb, opa, quat, scale, feat, d, f, scale_activation,
                                                    (double)min_opacity, n_relocated, ws.src, ws.dead_idx, 0, ws.count,
                                                    pos, rgb, opa, quat, scale, feat);
  GS_CUDA_TRY(cudaGetLastError());
  mcmc_apply_sources_kernel<<<grid(n), kBlock, 0, st>>>(n_relocated, ws.src, ws.dead_idx, 0, opa, scale,
                                                       segs.n ? exp_avg : nullptr, exp_avg_sq, segs, touched);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch(4);
  return 0;
}

extern "C" int gs_mcmc_add(const float* pos, const float* rgb, const float* opa, const float* quat, const float* scale,
                           const float* feat, int f, int n, int d, int scale_activation, float min_opacity, int n_new,
                           const float* u, float* out_pos, float* out_rgb, float* out_opa, float* out_quat,
                           float* out_scale, float* out_feat, void* workspace, size_t workspace_bytes,
                           gs_stream_t stream) {
  if (n < 0 || n_new < 0 || (n_new > 0 && n == 0) ||
      (n > 0 && (!pos || !rgb || !opa || !quat || !scale || !out_pos || !out_rgb || !out_opa || !out_quat ||
                 !out_scale || !workspace || (n_new > 0 && !u) || (feat && !out_feat))))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: bad arguments");
  if ((long long)n + n_new > 0x7fffffffLL)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: n + n_new does not fit an int");
  if (bad_widths(d, feat, f))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: d must be 3, 27 or 48 and f 8, 16 or 32");
  if (misaligned(quat) || misaligned(out_quat))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: quat and out_quat must be 16-byte aligned");
  if (scale_activation != GS_SCALE_ABS && scale_activation != GS_SCALE_EXP)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: unknown scale activation");
  if (!(min_opacity > 0.f && min_opacity < 1.f))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: min_opacity must be in (0, 1)");
  const int m = n > n_new ? n : n_new;
  if (workspace_bytes < gs_mcmc_workspace_bytes(m))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_add: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  const size_t rows = (size_t)n * sizeof(float);
  GS_CUDA_TRY(cudaMemcpyAsync(out_pos, pos, 3 * rows, cudaMemcpyDeviceToDevice, st));
  GS_CUDA_TRY(cudaMemcpyAsync(out_rgb, rgb, (size_t)d * rows, cudaMemcpyDeviceToDevice, st));
  GS_CUDA_TRY(cudaMemcpyAsync(out_opa, opa, rows, cudaMemcpyDeviceToDevice, st));
  GS_CUDA_TRY(cudaMemcpyAsync(out_quat, quat, 4 * rows, cudaMemcpyDeviceToDevice, st));
  GS_CUDA_TRY(cudaMemcpyAsync(out_scale, scale, 3 * rows, cudaMemcpyDeviceToDevice, st));
  if (feat) GS_CUDA_TRY(cudaMemcpyAsync(out_feat, feat, (size_t)f * rows, cudaMemcpyDeviceToDevice, st));
  if (n_new == 0) return 0;
  Ws ws = carve(workspace, m);
  GS_CUDA_TRY(cudaMemsetAsync(ws.count, 0, (size_t)n * sizeof(int), st));
  mcmc_weight_kernel<<<grid(n), kBlock, 0, st>>>(opa, n, (double)min_opacity, 0, ws.w, ws.dead);
  GS_CUDA_TRY(cudaGetLastError());
  size_t tb = ws.tmp_bytes;
  GS_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws.tmp, tb, ws.w, ws.C, n, st));
  mcmc_draw_kernel<<<grid(n_new), kBlock, 0, st>>>(ws.C, n, u, nullptr, n_new, ws.src, ws.count, ws.n_draws);
  GS_CUDA_TRY(cudaGetLastError());
  mcmc_apply_rows_kernel<<<grid(n_new), kBlock, 0, st>>>(pos, rgb, opa, quat, scale, feat, d, f, scale_activation,
                                                        (double)min_opacity, ws.n_draws, ws.src, nullptr, n, ws.count,
                                                        out_pos, out_rgb, out_opa, out_quat, out_scale, out_feat);
  GS_CUDA_TRY(cudaGetLastError());
  mcmc_apply_sources_kernel<<<grid(n_new), kBlock, 0, st>>>(ws.n_draws, ws.src, nullptr, n, out_opa, out_scale, nullptr,
                                                           nullptr, MomentSegs{}, nullptr);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch(4);
  return 0;
}

extern "C" int gs_mcmc_noise(float* pos, const float* quat, const float* scale, const float* opa, int n,
                             int scale_activation, float scaler, unsigned long long seed, const float* z,
                             gs_stream_t stream) {
  if (n < 0 || (n > 0 && (!pos || !quat || !scale || !opa)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_noise: bad arguments");
  if (scale_activation != GS_SCALE_ABS && scale_activation != GS_SCALE_EXP)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_noise: unknown scale activation");
  if (!std::isfinite(scaler)) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_noise: scaler is not finite");
  if (misaligned(quat)) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_mcmc_noise: quat must be 16-byte aligned");
  if (n == 0) return 0;
  mcmc_noise_kernel<<<grid(n), kBlock, 0, (cudaStream_t)stream>>>(pos, quat, scale, opa, n, scale_activation, scaler,
                                                                   seed, z);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}
