// Blend-weight scores of the fused frame path (gs_frame_scores): for every Gaussian, the sum and the largest of its
// blend weights w = alpha T over the pixels of the last forward's image.  Kernels of their own, not a flag on the
// shipped forward: they replay the forward's alpha / T recurrence from the records and the sorted instance list that
// the forward left in the context, and write nothing a backward reads.
//   score_blend_kernel: one CTA per tile; one (sum w, max w) row per instance at its gradient-row slot, tagged with
//                       the pass's own epoch.
//   score_sum_kernel  : one thread per Gaussian; sums its rows tagged with that epoch in row order, view by view.
#include "internal.h"

namespace {

constexpr int kThreads = 64;   // a row of 4 adjacent pixels per thread, as the shipped gather forward
constexpr int kPx = 4;
constexpr int kCh = 32;        // instances per staging chunk: one per thread of warp 0 (21 KB of shared memory)
constexpr int kStages = 2;
constexpr int kRecW = 4;       // {a, b, c, (first gradient row of the Gaussian, -, -, -)}
constexpr int kBlock = 256;

struct ScoreSmem {
  float4 rec[kStages][kCh * kRecW];
  float ps[kThreads][kCh + 1];   // per-thread partial sums of one chunk (+1: the reduction reads a column)
  float pm[kThreads][kCh + 1];   // and partial maxima
};

// instance i = tid of chunk k: the three 16-byte pieces of its record and its Gaussian's first gradient row
__device__ __forceinline__ void score_issue(ScoreSmem& sm, int stage, const GsRec* __restrict__ grec,
                                            const uint32_t* __restrict__ goff, const uint32_t* __restrict__ ids,
                                            int base, int n, int tid) {
  if (tid < n) {
    const uint32_t id = __ldg(ids + base + tid);
    const float4* src = reinterpret_cast<const float4*>(grec + id);
    const uint32_t dst = gs_smem_u32(&sm.rec[stage][tid * kRecW]);
#pragma unroll
    for (int q = 0; q < 3; ++q)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16u * q), "l"(src + q) : "memory");
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst + 48u), "l"(goff + id) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// Per pixel: the forward's alpha = ex2(l2o - (ca dx^2 - cb dx dy + cc dy^2)) and w = alpha T while T > GS_T_STOP, in
// the forward's instance order and arithmetic, so T and the early stop are the forward's.  Per instance: the sum over
// the thread's pixels inside the crop in pixel order, then over the 64 threads in thread order; the max likewise.
// BATCH: the tile's view v = ty / (hp / GS_TILE) gives the pixel rows, views[v].fx / fy and the crop.
template <bool BATCH>
__device__ __forceinline__ void score_blend_body(const GsRec* __restrict__ grec, const uint32_t* __restrict__ ids,
                                                 const uint32_t* __restrict__ goff, const int* __restrict__ tile_accum,
                                                 int wp, int hp, int ntx, float fx, float fy, GsCrop crop,
                                                 const GsView* __restrict__ views, float2* __restrict__ rows,
                                                 uint32_t* __restrict__ row_epoch, uint32_t epoch) {
  __shared__ __align__(16) ScoreSmem sm;
  const int tile = blockIdx.x;
  const int tid = threadIdx.x;
  const int tx = tile % ntx, ty = tile / ntx;
  int lty = ty;
  if constexpr (BATCH) {
    const int v = ty / (hp / GS_TILE);
    lty = ty - v * (hp / GS_TILE);
    fx = views[v].fx;
    fy = views[v].fy;
  }
  constexpr int TPR = GS_TILE / kPx;
  const int ix0 = tx * GS_TILE + (tid % TPR) * kPx;
  const int iyv = lty * GS_TILE + (tid / TPR);
  float px[kPx];
  bool inb[kPx];
  const bool row_in = iyv - crop.top >= 0 && iyv - crop.top < crop.height;
#pragma unroll
  for (int p = 0; p < kPx; ++p) {
    px[p] = gs_pixel_coord(ix0 + p, wp, fx);
    inb[p] = row_in && ix0 + p - crop.left >= 0 && ix0 + p - crop.left < crop.width;
  }
  const float py = gs_pixel_coord(iyv, hp, fy);

  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  const int nchunks = (cnt + kCh - 1) / kCh;
  // one commit group per chunk slot, empty past the end, so that wait_group 1 always means "chunk k has landed"
  for (int k = 0; k < kStages; ++k) score_issue(sm, k, grec, goff, ids, start + k * kCh, min(kCh, cnt - k * kCh), tid);

  float T[kPx];
#pragma unroll
  for (int p = 0; p < kPx; ++p) T[p] = 1.f;
  for (int k = 0; k < nchunks; ++k) {
    const int stage = k % kStages;
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    const int n = min(kCh, cnt - k * kCh);
    const float4* R = sm.rec[stage];
    bool dead = false;
    for (int j = 0; j < n; ++j) {
      float s = 0.f, m = 0.f;
      if (!dead) {
        const float4 a = R[j * kRecW];
        const float4 bb = R[j * kRecW + 1];
        const float2 b = make_float2(bb.x, bb.y);
        const float dy = py - a.y;
        const float m1 = a.w * dy;
        const float ev = fmaf(-b.x * dy, dy, b.y);
        bool all = true;
#pragma unroll
        for (int p = 0; p < kPx; ++p) {
          const float dx = px[p] - a.x;
          const float eu = fmaf(a.z, dx, -m1);
          const float alpha = gs_ex2(fmaf(-dx, eu, ev));   // l2o - (ca dx^2 - cb dx dy + cc dy^2)
          const float w = (T[p] > GS_T_STOP) ? alpha * T[p] : 0.f;
          T[p] -= w;
          const float wc = inb[p] ? w : 0.f;
          s += wc;
          m = fmaxf(m, wc);
          all = all && !(T[p] > GS_T_STOP);
        }
        // a warp whose pixels are all saturated adds exact zeros from here on
        dead = __all_sync(0xffffffffu, all);
      }
      sm.ps[tid][j] = s;
      sm.pm[tid][j] = m;
    }
    __syncthreads();
    if (tid < n) {
      float s = 0.f, m = 0.f;
#pragma unroll 8
      for (int t = 0; t < kThreads; ++t) {
        s += sm.ps[t][tid];
        m = fmaxf(m, sm.pm[t][tid]);
      }
      // the instance's gradient-row slot: first row of the Gaussian + rank of the tile in its rectangle
      const float4 cc = R[tid * kRecW + 2];
      const uint32_t rxy = __float_as_uint(cc.z), rwh = __float_as_uint(cc.w);
      const uint32_t off = __float_as_uint(R[tid * kRecW + 3].x);
      const uint32_t slot = off + ((uint32_t)ty - (rxy >> 16)) * (rwh & 0xffffu) + ((uint32_t)tx - (rxy & 0xffffu));
      rows[slot] = make_float2(s, m);
      row_epoch[slot] = epoch;
    }
    bool sat = true;
#pragma unroll
    for (int p = 0; p < kPx; ++p) sat = sat && !(T[p] > GS_T_STOP);
    // every thread is past the reduction: the stage is free.  A saturated tile adds only zeros from here on, and its
    // rows stay untagged.
    if (__syncthreads_and(sat)) break;
    score_issue(sm, stage, grec, goff, ids, start + (k + kStages) * kCh, min(kCh, cnt - (k + kStages) * kCh), tid);
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
}

__global__ void __launch_bounds__(kThreads) score_blend_kernel(const GsRec* __restrict__ grec,
                                                               const uint32_t* __restrict__ ids,
                                                               const uint32_t* __restrict__ goff,
                                                               const int* __restrict__ tile_accum, int wp, int hp,
                                                               int ntx, float fx, float fy, GsCrop crop,
                                                               float2* __restrict__ rows,
                                                               uint32_t* __restrict__ row_epoch, uint32_t epoch) {
  score_blend_body<false>(grec, ids, goff, tile_accum, wp, hp, ntx, fx, fy, crop, nullptr, rows, row_epoch, epoch);
}

__global__ void __launch_bounds__(kThreads) score_blend_batch_kernel(const GsRec* __restrict__ grec,
                                                                     const uint32_t* __restrict__ ids,
                                                                     const uint32_t* __restrict__ goff,
                                                                     const int* __restrict__ tile_accum, int wp, int hp,
                                                                     int ntx, GsCrop crop,
                                                                     const GsView* __restrict__ views,
                                                                     float2* __restrict__ rows,
                                                                     uint32_t* __restrict__ row_epoch, uint32_t epoch) {
  score_blend_body<true>(grec, ids, goff, tile_accum, wp, hp, ntx, 0.f, 0.f, crop, views, rows, row_epoch, epoch);
}

// Gaussian i, view by view in view order (pair v n + i): the sum and the max of its rows tagged with `epoch`, in row
// order; the view's sum is added to the running sum once, so a B-view frame gives the bits of B one-view calls.
__global__ void __launch_bounds__(kBlock) score_sum_kernel(const uint32_t* __restrict__ offsets_g,
                                                           const uint32_t* __restrict__ count,
                                                           const float2* __restrict__ rows,
                                                           const uint32_t* __restrict__ row_epoch, uint32_t epoch,
                                                           int n, int n_views, float* __restrict__ weight_sum,
                                                           float* __restrict__ weight_max) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float ws = weight_sum[i], wm = weight_max[i];
  bool any = false;
  for (int v = 0; v < n_views; ++v) {
    const int j = v * n + i;
    const uint32_t cnt = count[j];
    if (cnt == 0) continue;
    any = true;
    float s = 0.f, m = 0.f;
    const uint32_t o0 = offsets_g[j], o1 = o0 + cnt;
    for (uint32_t r = o0; r < o1; ++r) {
      if (row_epoch[r] != epoch) continue;   // not reached by its (saturated) tile: zero weight
      const float2 w = rows[r];
      s += w.x;
      m = fmaxf(m, w.y);
    }
    ws += s;
    wm = fmaxf(wm, m);
  }
  if (!any) return;
  weight_sum[i] = ws;
  weight_max[i] = wm;
}

}  // namespace

cudaError_t gs_launch_frame_scores(const GsRec* grec, const uint32_t* ids, const uint32_t* offsets_g,
                                   const uint32_t* count, const int* tile_accum, const GsFrameGeom& g,
                                   const GsView* views, int n, int n_views, const GsCrop& crop, float2* rows,
                                   uint32_t* row_epoch, uint32_t epoch, float* weight_sum, float* weight_max,
                                   cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (views)
    score_blend_batch_kernel<<<g.n_tiles, kThreads, 0, st>>>(grec, ids, offsets_g, tile_accum, g.wp, g.hp, g.ntx, crop,
                                                             views, rows, row_epoch, epoch);
  else
    score_blend_kernel<<<g.n_tiles, kThreads, 0, st>>>(grec, ids, offsets_g, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy,
                                                       crop, rows, row_epoch, epoch);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  score_sum_kernel<<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(offsets_g, count, rows, row_epoch, epoch, n, n_views,
                                                                 weight_sum, weight_max);
  return cudaGetLastError();
}
