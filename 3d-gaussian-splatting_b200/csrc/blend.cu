// Per-tile front-to-back alpha compositing, forward and backward (the hot kernels).
//
// Semantics: reference gaussian.cu:806-970 (draw_kernel) and :440-803 (draw_backward_kernel):
// 16x16 pixel tiles, each tile blends its (depth-sorted) instance range front to back,
// a pixel stops before an instance once its transmittance is < 1e-4, no alpha clamp, no
// 1/255 skip, black background.  Design (not the reference's):
//   * each tile's range is contiguous in three packed record streams (see gs_common.cuh) and is
//     staged into shared memory by 1-D bulk async copies (cp.async.bulk -> UBLKCP, mbarrier
//     complete_tx), double buffered; one elected thread issues, nobody spends LSU slots on it;
//   * per (pixel, instance): one ex2 (opacity folded into the exponent) and ~15 FP32 ops;
//     no FP64, no division in the forward loop;
//   * whole-warp and whole-CTA early exit once every pixel is saturated, so a tile's tail is
//     never read (M_eff accounting);
//   * backward: 64 threads x 4 pixels per tile; 9 moment sums per instance are reduced with a
//     recursive-halving shuffle network (14 SHFL instead of 45), combined across the two warps
//     through shared memory and written as ONE record per instance (no atomics, deterministic).
#include <cstdlib>
#include <type_traits>

#include "internal.h"

namespace {

// =======================================================================================
// forward
// =======================================================================================
constexpr int FWD_THREADS = 64;    // 2 warps per tile; each thread owns a row of 4 adjacent pixels
constexpr int FWD_PX = 4;
constexpr int FWD_STAGES = 2;

template <int FWD_CH>
struct FwdSmem {
  float4 A[FWD_STAGES][FWD_CH];
  float4 C[FWD_STAGES][FWD_CH];
  float2 B[FWD_STAGES][FWD_CH + 2];
  uint64_t full[FWD_STAGES];
};

template <typename SM, int CH>
__device__ __forceinline__ void issue_chunk(SM& sm, int stage, const float4* __restrict__ pA,
                                            const float2* __restrict__ pB, const float4* __restrict__ pC,
                                            int base, int n, int shift) {
  uint32_t bytes_a = (uint32_t)n * 16u;
  uint32_t nb = (uint32_t)(n + shift + 1) & ~1u;
  uint32_t bytes_b = nb * 8u;
  gs_mbar_expect_tx(&sm.full[stage], 2u * bytes_a + bytes_b);
  gs_bulk_g2s(sm.A[stage], pA + base, bytes_a, &sm.full[stage]);
  gs_bulk_g2s(sm.C[stage], pC + base, bytes_a, &sm.full[stage]);
  gs_bulk_g2s(sm.B[stage], pB + (base - shift), bytes_b, &sm.full[stage]);
}

// ---- two ways a tile's sorted range reaches shared memory -------------------------------------------
// packed : three contiguous record streams written by the pack pass (and by the legacy draw API);
//          one thread issues three 1-D bulk copies per chunk.
// gather : NO pack pass - every thread of the CTA issues, for "its" instances of the next chunk, the 16-byte
//          cp.async pieces of the Gaussian's record straight from GsRec rec[N] through the sorted id list and
//          arrives on the stage's mbarrier when they have landed (cp.async.mbarrier.arrive; barrier count = CTA
//          threads).  The per-instance record in shared memory is {a, b, c, d} (gs_common.cuh GsRec).
template <bool GATHER>
struct StageView;
template <>
struct StageView<false> {
  const float4* A;
  const float4* C;
  const float2* B;
  __device__ __forceinline__ float4 a(int j) const { return A[j]; }
  __device__ __forceinline__ float2 b(int j) const { return B[j]; }
  __device__ __forceinline__ float4 c(int j) const { return C[j]; }                   // r, g, b, (slot)
  __device__ __forceinline__ uint32_t slot(int j, int, int) const { return __float_as_uint(C[j].w); }
};
template <>
struct StageView<true> {
  const float4* R;                                                                     // [CH][RECW]
  int recw;
  __device__ __forceinline__ float4 a(int j) const { return R[j * recw]; }
  __device__ __forceinline__ float2 b(int j) const {
    const float4 t = R[j * recw + 1];
    return make_float2(t.x, t.y);
  }
  __device__ __forceinline__ float4 c(int j) const {
    const float4 t = R[j * recw + 1];
    return make_float4(t.z, t.w, R[j * recw + 2].x, 0.f);
  }
  __device__ __forceinline__ float depth(int j) const { return R[j * recw + 2].y; }   // |p_c|
  // gradient row of this (Gaussian, tile) instance: first row of the Gaussian + rank of the tile in its rectangle
  __device__ __forceinline__ uint32_t slot(int j, int tx, int ty) const {
    const float4 cc = R[j * recw + 2];
    const uint32_t rxy = __float_as_uint(cc.z), rwh = __float_as_uint(cc.w);
    const uint32_t off = __float_as_uint(R[j * recw + 3].x);
    return off + ((uint32_t)ty - (rxy >> 16)) * (rwh & 0xffffu) + ((uint32_t)tx - (rxy & 0xffffu));
  }
};

template <int CH, int STAGES, int RECW>
struct GatherRing {
  float4 rec[STAGES][CH * RECW];
  uint64_t full[STAGES];
};

// ids of "this thread's" instances of one chunk, loaded one chunk boundary ahead of their use so that the
// dependent record copies never wait for the id load
template <int NT, int CH>
struct GatherIds {
  uint32_t id[(CH + NT - 1) / NT];
  __device__ __forceinline__ void load(const uint32_t* __restrict__ ids, int base, int n, int tid) {
#pragma unroll
    for (int u = 0; u < (CH + NT - 1) / NT; ++u) {
      const int i = tid + u * NT;
      id[u] = i < n ? __ldg(ids + base + i) : 0u;
    }
  }
};

// RECW = 3: {a, b, c} (forward); RECW = 4: {a, b, c, (first gradient row of the Gaussian, -, -, -)} (backward: the
// 4th piece comes from offsets_g[id], a 4-byte cp.async - patching it into rec[] from another kernel cost more)
template <typename SM, int NT, int CH, int RECW>
__device__ __forceinline__ void gather_issue(SM& sm, int stage, const GsRec* __restrict__ grec,
                                             const uint32_t* __restrict__ goff, const GatherIds<NT, CH>& g, int n,
                                             int tid) {
  // 16-byte cp.async (LDGSTS) pieces: one warp-wide instruction moves a piece of 32 instances.  (Measured: one
  // 1-D bulk copy per instance, i.e. ~6 M tiny TMA requests per frame, made both blend kernels ~15 % slower.)
#pragma unroll
  for (int u = 0; u < (CH + NT - 1) / NT; ++u) {
    const int i = tid + u * NT;
    if (i < n) {
      const float4* src = reinterpret_cast<const float4*>(grec + g.id[u]);
      const uint32_t dst = gs_smem_u32(&sm.rec[stage][i * RECW]);
#pragma unroll
      for (int q = 0; q < 3; ++q)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16u * q), "l"(src + q) : "memory");
      if (RECW == 4)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst + 48u), "l"(goff + g.id[u]) : "memory");
    }
  }
  // this thread's arrival on the stage barrier (count = CTA threads) fires when its copies have landed
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(gs_smem_u32(&sm.full[stage])) : "memory");
}

// Per (thread, instance): 3 broadcast LDS + 4 row-shared FP32 ops (dy, cb*dy, cc*dy, l2o-cc*dy^2)
// + 4 pixels x (dx, u, exponent, MUFU.EX2, setp, mul, sel, 3 FFMA colour, T update) = 12.75
// issue slots per (pixel, instance) instead of 17-18 with one pixel per thread.
// AUX (gather only): one more FFMA per (pixel, instance) accumulates the depth sum w t; at the end the background
// T_f bg is added to the colour and (depth, 1 - T_f) is stored to aux / aux_final.
// BATCH (gather, batched frame): the tile's view v = ty / (hp / GS_TILE) gives the pixel coordinates (its own rows, its
// fx / fy from views[v]) and the final / aux_final crop ([B, height, width, .]); the padded image and aux are the tall
// [B Hp, Wp, .] ones and are addressed as without it.
template <int FWD_CH, int PX, bool GATHER, bool AUX = false, bool BATCH = false>
__device__ __forceinline__ void blend_fwd_body(const float4* __restrict__ pA, const float2* __restrict__ pB,
                                               const float4* __restrict__ pC, const GsRec* __restrict__ grec,
                                               const uint32_t* __restrict__ ids, const int* __restrict__ tile_accum,
                                               int wp, int hp, int ntx, float fx, float fy, float* __restrict__ image,
                                               int* __restrict__ tile_neff, float* __restrict__ final_img, GsCrop crop,
                                               GsAuxOut aux, const GsView* __restrict__ views) {
  static_assert(!AUX || GATHER, "the aux outputs read |p_c| from the gathered records");
  static_assert(!BATCH || GATHER, "batched frames run the gather path");
  using Smem = typename std::conditional<GATHER, GatherRing<FWD_CH, FWD_STAGES, 3>, FwdSmem<FWD_CH>>::type;
  __shared__ __align__(16) Smem sm;
  const int tile = blockIdx.x;
  const int tid = threadIdx.x;
  const int tx = tile % ntx, ty = tile / ntx;
  int lty = ty;   // the tile's row in its view
  if constexpr (BATCH) {
    const int v = ty / (hp / GS_TILE);
    lty = ty - v * (hp / GS_TILE);
    fx = views[v].fx;
    fy = views[v].fy;
    if (final_img) final_img += (size_t)v * crop.width * crop.height * 3;
    if (aux.aux_final) aux.aux_final += (size_t)v * crop.width * crop.height * 2;
  }
  // thread -> a row of PX adjacent pixels (ix0 .. ix0+PX-1, iy); PX = 4: 2 warps per tile, 8: one warp
  constexpr int FWD_PX = PX, TPR = GS_TILE / PX, NTHREADS = 256 / PX;
  const int ix0 = tx * GS_TILE + (tid % TPR) * FWD_PX;
  const int iy = ty * GS_TILE + (tid / TPR);
  const int iyv = lty * GS_TILE + (tid / TPR);   // its row in the view
  float px[FWD_PX];
#pragma unroll
  for (int p = 0; p < FWD_PX; ++p) px[p] = gs_pixel_coord(ix0 + p, wp, fx);
  const float py = gs_pixel_coord(iyv, hp, fy);

  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  const int shift = start & 1;
  const int nchunks = (cnt + FWD_CH - 1) / FWD_CH;

  if (tid == 0) {
    for (int s = 0; s < FWD_STAGES; ++s) gs_mbar_init(&sm.full[s], GATHER ? NTHREADS : 1);
    gs_fence_barrier_init();
  }
  __syncthreads();
  GatherIds<NTHREADS, FWD_CH> gid;
  if constexpr (GATHER) {
    for (int k = 0; k < FWD_STAGES && k < nchunks; ++k) {
      gid.load(ids, start + k * FWD_CH, min(FWD_CH, cnt - k * FWD_CH), tid);
      gather_issue<Smem, NTHREADS, FWD_CH, 3>(sm, k, grec, nullptr, gid, min(FWD_CH, cnt - k * FWD_CH), tid);
    }
    if (FWD_STAGES < nchunks) gid.load(ids, start + FWD_STAGES * FWD_CH, min(FWD_CH, cnt - FWD_STAGES * FWD_CH), tid);
  } else if (tid == 0) {
    for (int k = 0; k < FWD_STAGES && k < nchunks; ++k)
      issue_chunk<Smem, FWD_CH>(sm, k, pA, pB, pC, start + k * FWD_CH, min(FWD_CH, cnt - k * FWD_CH), shift);
  }

  float T[FWD_PX], cr[FWD_PX], cg[FWD_PX], cb[FWD_PX], dep[FWD_PX];
#pragma unroll
  for (int p = 0; p < FWD_PX; ++p) {
    T[p] = 1.f;
    cr[p] = cg[p] = cb[p] = 0.f;
    dep[p] = 0.f;
  }
  int consumed = cnt;
  int k = 0;
  for (; k < nchunks; ++k) {
    const int stage = k % FWD_STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / FWD_STAGES) & 1));
    const int n = min(FWD_CH, cnt - k * FWD_CH);
    StageView<GATHER> sv;
    if constexpr (GATHER) {
      sv.R = sm.rec[stage];
      sv.recw = 3;
    } else {
      sv.A = sm.A[stage];
      sv.C = sm.C[stage];
      sv.B = sm.B[stage] + shift;
    }

#define GS_FWD_BODY(J)                                                                      \
  {                                                                                         \
    const float4 a = sv.a(J);                                                               \
    const float2 b = sv.b(J);                                                               \
    const float4 c = sv.c(J);                                                               \
    const float dy = py - a.y;                                                              \
    const float m1 = a.w * dy;                                                              \
    const float ev = fmaf(-b.x * dy, dy, b.y);                                              \
    float t = 0.f;                                                                          \
    if constexpr (AUX) t = sv.depth(J);                                                     \
    _Pragma("unroll") for (int p = 0; p < FWD_PX; ++p) {                                    \
      const float dx = px[p] - a.x;                                                         \
      const float eu = fmaf(a.z, dx, -m1);                                                  \
      const float alpha = gs_ex2(fmaf(-dx, eu, ev)); /* l2o - (ca dx^2 - cb dx dy + cc dy^2) */ \
      const float w = (T[p] > GS_T_STOP) ? alpha * T[p] : 0.f;                              \
      cr[p] = fmaf(c.x, w, cr[p]);                                                          \
      cg[p] = fmaf(c.y, w, cg[p]);                                                          \
      cb[p] = fmaf(c.z, w, cb[p]);                                                          \
      if constexpr (AUX) dep[p] = fmaf(t, w, dep[p]);                                       \
      T[p] -= w;                                                                            \
    }                                                                                       \
  }
    int j = 0;
    bool warp_dead = false;
    for (; j + 4 <= n; j += 4) {
#pragma unroll
      for (int u = 0; u < 4; ++u) GS_FWD_BODY(j + u)
      bool dead = true;
#pragma unroll
      for (int p = 0; p < FWD_PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
      if (__all_sync(0xffffffffu, dead)) {
        warp_dead = true;
        break;
      }
    }
    if (!warp_dead)
      for (; j < n; ++j) GS_FWD_BODY(j)
#undef GS_FWD_BODY

    bool dead = true;
#pragma unroll
    for (int p = 0; p < FWD_PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
    const int all_dead = NTHREADS == 32 ? __all_sync(0xffffffffu, dead) : __syncthreads_and(dead);
    if (NTHREADS == 32) __syncwarp();
    if (all_dead) {
      consumed = min(cnt, (k + 1) * FWD_CH);
      break;
    }
    if (k + FWD_STAGES < nchunks) {
      const int kn = k + FWD_STAGES;            // every thread is past the barrier above: the stage is free
      if constexpr (GATHER) {
        gather_issue<Smem, NTHREADS, FWD_CH, 3>(sm, stage, grec, nullptr, gid, min(FWD_CH, cnt - kn * FWD_CH), tid);
        if (kn + 1 < nchunks) gid.load(ids, start + (kn + 1) * FWD_CH, min(FWD_CH, cnt - (kn + 1) * FWD_CH), tid);
      } else if (tid == 0)
        issue_chunk<Smem, FWD_CH>(sm, stage, pA, pB, pC, start + kn * FWD_CH, min(FWD_CH, cnt - kn * FWD_CH), shift);
    }
  }
  // drain copies that were issued but never consumed (early exit) before the CTA retires
  if (tid == 0 && k < nchunks) {
    for (int kk = k + 1; kk < nchunks && kk < k + FWD_STAGES; ++kk)
      gs_mbar_wait(&sm.full[kk % FWD_STAGES], (uint32_t)((kk / FWD_STAGES) & 1));
  }
  if constexpr (AUX) {
#pragma unroll
    for (int p = 0; p < FWD_PX; ++p) {
      cr[p] = fmaf(T[p], aux.bg[0], cr[p]);
      cg[p] = fmaf(T[p], aux.bg[1], cg[p]);
      cb[p] = fmaf(T[p], aux.bg[2], cb[p]);
    }
    float ab[FWD_PX * 2];   // (depth, alpha) x PX = PX * 8 contiguous, 16-byte aligned bytes
#pragma unroll
    for (int p = 0; p < FWD_PX; ++p) {
      ab[2 * p] = dep[p];
      ab[2 * p + 1] = 1.f - T[p];
    }
    if (aux.aux) {
      float4* o = reinterpret_cast<float4*>(aux.aux + ((size_t)iy * wp + ix0) * 2);
#pragma unroll
      for (int q = 0; q < FWD_PX / 2; ++q) o[q] = make_float4(ab[4 * q], ab[4 * q + 1], ab[4 * q + 2], ab[4 * q + 3]);
    }
    if (aux.aux_final) {
#pragma unroll
      for (int p = 0; p < FWD_PX; ++p) {
        const int x = ix0 + p - crop.left, y = iyv - crop.top;
        if (x >= 0 && x < crop.width && y >= 0 && y < crop.height)
          *reinterpret_cast<float2*>(aux.aux_final + ((size_t)y * crop.width + x) * 2) = make_float2(ab[2 * p], ab[2 * p + 1]);
      }
    }
  }
  // PX pixels x 3 channels = PX * 12 contiguous, 16-byte aligned bytes
  {
    float ob[FWD_PX * 3];
#pragma unroll
    for (int p = 0; p < FWD_PX; ++p) {
      ob[3 * p] = cr[p];
      ob[3 * p + 1] = cg[p];
      ob[3 * p + 2] = cb[p];
    }
    float4* o = reinterpret_cast<float4*>(image + ((size_t)iy * wp + ix0) * 3);
#pragma unroll
    for (int q = 0; q < FWD_PX * 3 / 4; ++q) o[q] = make_float4(ob[4 * q], ob[4 * q + 1], ob[4 * q + 2], ob[4 * q + 3]);
  }
  if (final_img) {
#pragma unroll
    for (int p = 0; p < FWD_PX; ++p)
      gs_store_final(final_img, ix0 + p, iyv, crop.left, crop.top, crop.width, crop.height, cr[p], cg[p], cb[p]);
  }
  if (tile_neff && tid == 0) tile_neff[tile] = consumed;
}

template <int FWD_CH, int PX, bool GATHER, bool AUX = false>
__global__ void __launch_bounds__(256 / PX) blend_fwd_kernel(const float4* __restrict__ pA,
                                                                 const float2* __restrict__ pB,
                                                                 const float4* __restrict__ pC,
                                                                 const GsRec* __restrict__ grec,
                                                                 const uint32_t* __restrict__ ids,
                                                                 const int* __restrict__ tile_accum, int wp, int hp,
                                                                 int ntx, float fx, float fy,
                                                                 float* __restrict__ image,
                                                                 int* __restrict__ tile_neff,
                                                                 float* __restrict__ final_img, GsCrop crop,
                                                                 GsAuxOut aux) {
  blend_fwd_body<FWD_CH, PX, GATHER, AUX>(pA, pB, pC, grec, ids, tile_accum, wp, hp, ntx, fx, fy, image, tile_neff,
                                          final_img, crop, aux, nullptr);
}

// the shipped gather forward (FWD_CH 128, 4 pixels per thread) of a batched frame
template <bool AUX>
__global__ void __launch_bounds__(64) blend_fwd_batch_kernel(const GsRec* __restrict__ grec,
                                                             const uint32_t* __restrict__ ids,
                                                             const int* __restrict__ tile_accum, int wp, int hp,
                                                             int ntx, const GsView* __restrict__ views,
                                                             float* __restrict__ image, int* __restrict__ tile_neff,
                                                             float* __restrict__ final_img, GsCrop crop, GsAuxOut aux) {
  blend_fwd_body<128, 4, true, AUX, true>(nullptr, nullptr, nullptr, grec, ids, tile_accum, wp, hp, ntx, 0.f, 0.f,
                                          image, tile_neff, final_img, crop, aux, views);
}

// =======================================================================================
// backward
// =======================================================================================
constexpr int BWD_STAGES = 2;
constexpr int BWD_NV = 9;   // Sx Sy Sxx Sxy Syy S0 Cr Cg | Cb

template <int WARPS, int BWD_CH>
struct BwdSmem {
  float4 A[BWD_STAGES][BWD_CH];
  float4 C[BWD_STAGES][BWD_CH];
  float2 B[BWD_STAGES][BWD_CH + 2];
  uint64_t full[BWD_STAGES];
  float partial[WARPS][BWD_CH * BWD_NV];
};

// WARPS warps per tile; every thread owns a row of PX = 8 / WARPS ... i.e. 256 / (32*WARPS)
// horizontally adjacent pixels, so dy and every dy-only factor is shared by its pixels:
// per pixel only S0 += e, Sx += e dx, Sxx += e dx^2 are accumulated and
// Sy = dy S0, Sxy = dy Sx, Syy = dy^2 S0 are formed once per (thread, instance).
template <int WARPS, int BWD_CH>
__global__ void __launch_bounds__(32 * WARPS) blend_bwd_kernel(const float4* __restrict__ pA,
                                                                const float2* __restrict__ pB,
                                                                const float4* __restrict__ pC,
                                                                const int* __restrict__ tile_accum, int wp, int hp,
                                                                int ntx, float fx, float fy,
                                                                const float* __restrict__ image,
                                                                const float* __restrict__ grad_image,
                                                                float* __restrict__ grad_inst, int grad_is_final,
                                                                GsCrop crop, uint32_t* __restrict__ row_epoch,
                                                                uint32_t epoch, int* __restrict__ tile_neff_b) {
  constexpr int THREADS = 32 * WARPS;
  constexpr int PX = 256 / THREADS;          // 8 (1 warp) or 4 (2 warps)
  constexpr int TPR = GS_TILE / PX;          // threads per pixel row
  using Smem = BwdSmem<WARPS, BWD_CH>;
  __shared__ __align__(16) Smem sm;
  const int tile = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = tile % ntx, ty = tile / ntx;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int shift = start & 1;
  const int nchunks = (cnt + BWD_CH - 1) / BWD_CH;

  const int ix0 = tx * GS_TILE + (tid % TPR) * PX;
  const int iy = ty * GS_TILE + (tid / TPR);
  float px[PX];
#pragma unroll
  for (int p = 0; p < PX; ++p) px[p] = gs_pixel_coord(ix0 + p, wp, fx);
  const float py = gs_pixel_coord(iy, hp, fy);

  float T[PX], R[PX], gr[PX], gg[PX], gb[PX];
  {
    const size_t off = ((size_t)iy * wp + ix0) * 3;     // PX*12 contiguous, 16-byte aligned bytes
    const float4* im = reinterpret_cast<const float4*>(image + off);
    float gbuf[PX * 3], ibuf[PX * 3];
#pragma unroll
    for (int q = 0; q < PX * 3 / 4; ++q) {
      const float4 i4 = im[q];
      ibuf[4 * q] = i4.x; ibuf[4 * q + 1] = i4.y; ibuf[4 * q + 2] = i4.z; ibuf[4 * q + 3] = i4.w;
    }
    if (!grad_is_final) {
      const float4* gi = reinterpret_cast<const float4*>(grad_image + off);
#pragma unroll
      for (int q = 0; q < PX * 3 / 4; ++q) {
        const float4 g4 = gi[q];
        gbuf[4 * q] = g4.x; gbuf[4 * q + 1] = g4.y; gbuf[4 * q + 2] = g4.z; gbuf[4 * q + 3] = g4.w;
      }
    } else {
#pragma unroll
      for (int p = 0; p < PX; ++p)
        gs_load_final_grad(grad_image, ibuf + 3 * p, ix0 + p, iy, crop.left, crop.top, crop.width, crop.height,
                           gbuf[3 * p], gbuf[3 * p + 1], gbuf[3 * p + 2]);
    }
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      gr[p] = gbuf[3 * p];
      gg[p] = gbuf[3 * p + 1];
      gb[p] = gbuf[3 * p + 2];
      R[p] = gr[p] * ibuf[3 * p] + gg[p] * ibuf[3 * p + 1] + gb[p] * ibuf[3 * p + 2];
      T[p] = 1.f;
    }
  }

  if (tid == 0) {
    for (int s = 0; s < BWD_STAGES; ++s) gs_mbar_init(&sm.full[s], 1);
    gs_fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    for (int k = 0; k < BWD_STAGES && k < nchunks; ++k)
      issue_chunk<Smem, BWD_CH>(sm, k, pA, pB, pC, start + k * BWD_CH, min(BWD_CH, cnt - k * BWD_CH), shift);
  }

  int consumed = cnt;
  int k = 0;
  for (; k < nchunks; ++k) {
    const int stage = k % BWD_STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / BWD_STAGES) & 1));
    const int n = min(BWD_CH, cnt - k * BWD_CH);
    const float4* __restrict__ sA = sm.A[stage];
    const float4* __restrict__ sC = sm.C[stage];
    const float2* __restrict__ sB = sm.B[stage] + shift;
    float* __restrict__ part = sm.partial[warp];

    int j = 0;
    for (; j < n; ++j) {
      if ((j & 3) == 0) {
        bool dead = true;
#pragma unroll
        for (int p = 0; p < PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
        if (__all_sync(0xffffffffu, dead)) break;
      }
      const float4 a = sA[j];
      const float2 b = sB[j];
      const float4 c = sC[j];
      float s0 = 0.f, sx = 0.f, sxx = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
      const float dy = py - a.y;
      const float m1 = a.w * dy;
      const float ev = fmaf(-b.x * dy, dy, b.y);
#pragma unroll
      for (int p = 0; p < PX; ++p) {
        const float dx = px[p] - a.x;
        const float eu = fmaf(a.z, dx, -m1);
        const float alpha = gs_ex2(fmaf(-dx, eu, ev));   // l2o - (ca dx^2 - cb dx dy + cc dy^2)
        const bool live = T[p] > GS_T_STOP;
        const float w = live ? alpha * T[p] : 0.f;
        const float gc = fmaf(gr[p], c.x, fmaf(gg[p], c.y, gb[p] * c.z));
        R[p] = fmaf(-gc, w, R[p]);                                   // sum_c g_c (out_c - C_c^{<=i})
        const float rc = gs_rcp(1.0000001f - alpha);                 // 1/(1 - alpha + 1e-7)  (:721)
        const float dal = fmaf(T[p], gc, -R[p] * rc);                // d L / d alpha            (:710-722)
        const float e = live ? dal * alpha : 0.f;
        T[p] -= w;
        const float ex = e * dx;
        s0 += e;
        sx += ex;
        sxx = fmaf(ex, dx, sxx);
        c0 = fmaf(gr[p], w, c0);
        c1 = fmaf(gg[p], w, c1);
        c2 = fmaf(gb[p], w, c2);
      }
      float v[8];
      v[0] = sx;
      v[1] = dy * s0;
      v[2] = sxx;
      v[3] = dy * sx;
      v[4] = dy * v[1];
      v[5] = s0;
      v[6] = c0;
      v[7] = c1;
      float v8 = c2;
      // recursive-halving reduction of v[0..7] over the warp, plain butterfly for v8
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
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v8 += __shfl_xor_sync(0xffffffffu, v8, o);
      // lane L now holds the warp total of value index ((L>>4)&1)*4 + ((L>>3)&1)*2 + ((L>>2)&1)
      if ((lane & 3) == 0) part[j * BWD_NV + (((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1))] = v[0];
      if (lane == 0) part[j * BWD_NV + 8] = v8;
    }
    // instances this warp skipped because all of its pixels are saturated
    for (int z = j * BWD_NV + lane; z < n * BWD_NV; z += 32) part[z] = 0.f;
    __syncthreads();

    for (int t = tid; t < n; t += THREADS) {
      float s[BWD_NV];
#pragma unroll
      for (int u = 0; u < BWD_NV; ++u) {
        s[u] = sm.partial[0][t * BWD_NV + u];
#pragma unroll
        for (int w2 = 1; w2 < WARPS; ++w2) s[u] += sm.partial[w2][t * BWD_NV + u];
      }
      const float4 a = sA[t];
      const float2 b = sB[t];
      const uint32_t slot = __float_as_uint(sC[t].w);
      float4* out = reinterpret_cast<float4*>(grad_inst + (size_t)slot * GS_GREC);
      // d/dx, d/dy, d/dca, d/dcb  |  d/dcc, d/dl2o, d/dr, d/dg  |  d/db
      out[0] = make_float4(GS_LN2 * (2.f * a.z * s[0] - a.w * s[1]), GS_LN2 * (2.f * b.x * s[1] - a.w * s[0]),
                           -GS_LN2 * s[2], GS_LN2 * s[3]);
      out[1] = make_float4(-GS_LN2 * s[4], GS_LN2 * s[5], s[6], s[7]);
      out[2] = make_float4(s[8], 0.f, 0.f, 0.f);
      if (row_epoch) row_epoch[slot] = epoch;      // marks the row as written in this frame
    }
    bool dead = true;
#pragma unroll
    for (int p = 0; p < PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
    const int all_dead = __syncthreads_and(dead);
    if (all_dead) {
      consumed = min(cnt, (k + 1) * BWD_CH);
      break;
    }
    if (tid == 0 && k + BWD_STAGES < nchunks) {
      const int kn = k + BWD_STAGES;
      issue_chunk<Smem, BWD_CH>(sm, stage, pA, pB, pC, start + kn * BWD_CH, min(BWD_CH, cnt - kn * BWD_CH), shift);
    }
  }
  if (tid == 0 && k < nchunks) {
    for (int kk = k + 1; kk < nchunks && kk < k + BWD_STAGES; ++kk)
      gs_mbar_wait(&sm.full[kk % BWD_STAGES], (uint32_t)((kk / BWD_STAGES) & 1));
  }
  if (tile_neff_b && tid == 0) tile_neff_b[tile] = consumed;
  // the unread tail of a saturated tile has zero gradient: with an epoch array the rows are simply
  // left stale (the consumer skips rows whose tag is not this frame's); otherwise write zeros
  if (row_epoch) return;
  for (int t = consumed + tid; t < cnt; t += THREADS) {
    const uint32_t slot = __float_as_uint(pC[start + t].w);
    float4* out = reinterpret_cast<float4*>(grad_inst + (size_t)slot * GS_GREC);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    out[0] = z;
    out[1] = z;
    out[2] = z;
  }
}

// =======================================================================================
// warp-specialised kernels (default): one PRODUCER warp issues the bulk-async copies of the tile's
// sorted range, chunk by chunk, into a ring of shared-memory stages guarded by full / empty
// mbarriers; the CONSUMER warps only ever wait on `full`, blend, and release with one arrive on
// `empty`.  Consumers synchronise among themselves on a named barrier the producer never joins.
// =======================================================================================
constexpr int WS_CH = 64;          // instances per staging chunk (40 B each: 2.5 KB per stage)

template <int STAGES>
struct WsRing {
  float4 A[STAGES][WS_CH];
  float4 C[STAGES][WS_CH];
  float2 B[STAGES][WS_CH + 2];
  uint64_t full[STAGES], empty[STAGES], done;
  volatile int stop, consumed_chunks;
};

template <typename SM, int STAGES>
__device__ __forceinline__ void ws_init(SM& sm, int tid) {
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      gs_mbar_init(&sm.full[s], 1);
      gs_mbar_init(&sm.empty[s], 1);
    }
    gs_mbar_init(&sm.done, 1);
    sm.stop = 0;
    sm.consumed_chunks = 0;
    gs_fence_barrier_init();
  }
  __syncthreads();
}

// Producer warp (one elected lane): keeps up to STAGES chunks in flight; stops as soon as the
// consumers report that every pixel of the tile is saturated, and drains copies that were issued
// but never consumed before the CTA may retire (their destination is this CTA's shared memory).
template <typename SM, int STAGES>
__device__ __forceinline__ void ws_producer(SM& sm, const float4* __restrict__ pA, const float2* __restrict__ pB,
                                            const float4* __restrict__ pC, int start, int cnt, int nchunks) {
  const int shift = start & 1;
  int k = 0;
  for (; k < nchunks; ++k) {
    const int s = k % STAGES;
    if (k >= STAGES) gs_mbar_wait(&sm.empty[s], (uint32_t)(((k / STAGES) - 1) & 1));
    if (sm.stop) break;
    issue_chunk<SM, WS_CH>(sm, s, pA, pB, pC, start + k * WS_CH, min(WS_CH, cnt - k * WS_CH), shift);
  }
  gs_mbar_wait(&sm.done, 0u);
  for (int kk = sm.consumed_chunks; kk < k; ++kk) gs_mbar_wait(&sm.full[kk % STAGES], (uint32_t)((kk / STAGES) & 1));
}

// ---- forward ---------------------------------------------------------------------------
constexpr int WSF_STAGES = 4;
constexpr int WSF_CONS = 64;       // consumer threads: 2 warps, each thread a row of 4 adjacent pixels

__global__ void __launch_bounds__(WSF_CONS + 32) blend_fwd_ws_kernel(const float4* __restrict__ pA,
                                                                      const float2* __restrict__ pB,
                                                                      const float4* __restrict__ pC,
                                                                      const int* __restrict__ tile_accum, int wp,
                                                                      int hp, int ntx, float fx, float fy,
                                                                      float* __restrict__ image,
                                                                      int* __restrict__ tile_neff,
                                                                      float* __restrict__ final_img, GsCrop crop) {
  using Smem = WsRing<WSF_STAGES>;
  __shared__ __align__(16) Smem sm;
  const int tile = blockIdx.x;
  const int tid = threadIdx.x;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  const int nchunks = (cnt + WS_CH - 1) / WS_CH;
  ws_init<Smem, WSF_STAGES>(sm, tid);
  if (tid >= WSF_CONS) {
    if (tid == WSF_CONS && nchunks > 0) ws_producer<Smem, WSF_STAGES>(sm, pA, pB, pC, start, cnt, nchunks);
    return;
  }
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix0 = tx * GS_TILE + (tid & 3) * FWD_PX;
  const int iy = ty * GS_TILE + (tid >> 2);
  float px[FWD_PX];
#pragma unroll
  for (int p = 0; p < FWD_PX; ++p) px[p] = gs_pixel_coord(ix0 + p, wp, fx);
  const float py = gs_pixel_coord(iy, hp, fy);
  const int shift = start & 1;

  float T[FWD_PX], cr[FWD_PX], cg[FWD_PX], cb[FWD_PX];
#pragma unroll
  for (int p = 0; p < FWD_PX; ++p) {
    T[p] = 1.f;
    cr[p] = cg[p] = cb[p] = 0.f;
  }
  int consumed = cnt;
  for (int k = 0; k < nchunks; ++k) {
    const int stage = k % WSF_STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / WSF_STAGES) & 1));
    const int n = min(WS_CH, cnt - k * WS_CH);
    const float4* __restrict__ sA = sm.A[stage];
    const float4* __restrict__ sC = sm.C[stage];
    const float2* __restrict__ sB = sm.B[stage] + shift;
#define GS_FWD_BODY(J)                                                                      \
  {                                                                                         \
    const float4 a = sA[J];                                                                 \
    const float2 b = sB[J];                                                                 \
    const float4 c = sC[J];                                                                 \
    const float dy = py - a.y;                                                              \
    const float m1 = a.w * dy;                                                              \
    const float ev = fmaf(-b.x * dy, dy, b.y);                                              \
    _Pragma("unroll") for (int p = 0; p < FWD_PX; ++p) {                                    \
      const float dx = px[p] - a.x;                                                         \
      const float eu = fmaf(a.z, dx, -m1);                                                  \
      const float alpha = gs_ex2(fmaf(-dx, eu, ev));                                        \
      const float w = (T[p] > GS_T_STOP) ? alpha * T[p] : 0.f;                              \
      cr[p] = fmaf(c.x, w, cr[p]);                                                          \
      cg[p] = fmaf(c.y, w, cg[p]);                                                          \
      cb[p] = fmaf(c.z, w, cb[p]);                                                          \
      T[p] -= w;                                                                            \
    }                                                                                       \
  }
    int j = 0;
    bool warp_dead = false;
    for (; j + 4 <= n; j += 4) {
#pragma unroll
      for (int u = 0; u < 4; ++u) GS_FWD_BODY(j + u)
      const bool dead = !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP) && !(T[2] > GS_T_STOP) && !(T[3] > GS_T_STOP);
      if (__all_sync(0xffffffffu, dead)) {
        warp_dead = true;
        break;
      }
    }
    if (!warp_dead)
      for (; j < n; ++j) GS_FWD_BODY(j)
#undef GS_FWD_BODY
    const bool dead = !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP) && !(T[2] > GS_T_STOP) && !(T[3] > GS_T_STOP);
    const int all_dead = gs_bar_red_and(1, WSF_CONS, dead);       // also: both warps are done with the stage
    if (all_dead) {
      consumed = min(cnt, (k + 1) * WS_CH);
      if (tid == 0) {
        sm.consumed_chunks = k + 1;
        sm.stop = 1;
        gs_mbar_arrive(&sm.empty[stage]);
      }
      break;
    }
    if (tid == 0) {
      sm.consumed_chunks = k + 1;
      gs_mbar_arrive(&sm.empty[stage]);
    }
  }
  if (tid == 0 && nchunks > 0) gs_mbar_arrive(&sm.done);
  float4* o = reinterpret_cast<float4*>(image + ((size_t)iy * wp + ix0) * 3);
  o[0] = make_float4(cr[0], cg[0], cb[0], cr[1]);
  o[1] = make_float4(cg[1], cb[1], cr[2], cg[2]);
  o[2] = make_float4(cb[2], cr[3], cg[3], cb[3]);
  if (final_img) {
#pragma unroll
    for (int p = 0; p < FWD_PX; ++p)
      gs_store_final(final_img, ix0 + p, iy, crop.left, crop.top, crop.width, crop.height, cr[p], cg[p], cb[p]);
  }
  if (tile_neff && tid == 0) tile_neff[tile] = consumed;
}

// ---- backward ----------------------------------------------------------------------------
// Cross-thread reduction WITHOUT shuffles: every consumer thread accumulates, over its own row of
// PX pixels, six partial sums per instance (S0, Sx, Sxx, Cr, Cg, Cb; dy is shared by the row) and
// stores them to shared memory ([instance][quarter][thread][6], strides chosen so that both the
// 8-byte stores and the 8-byte loads of the second phase are bank-conflict free).  After R = NT/4
// instances a second phase gives each instance to 4 threads: each sums one quarter of the source
// threads (4 pixel rows: Sy = sum dy S0, Sxy = sum dy Sx, Syy = sum dy^2 S0 are formed per row), two
// xor-shuffles combine the quarters, and each of the 4 lanes stores one 16-byte piece of the
// instance's gradient record.  ~13 instructions per (thread, instance) instead of ~42 for the
// recursive-halving shuffle network; fixed summation order => bit-deterministic.
template <int PX, int STAGES_, int RQ_>
struct Bwd2Cfg {
  static constexpr int NT = 256 / PX;                        // consumer threads (64 or 32)
  static constexpr int TPR = GS_TILE / PX;                   // threads per pixel row
  static constexpr int RQ = RQ_;                             // reducer threads per instance in the second phase
  static constexpr int R = NT / RQ;                          // instances per reduction round
  static constexpr int SQ = NT / RQ;                         // source threads per reducer ("part")
  static constexpr int ROWS = SQ / TPR;                      // pixel rows per reducer
  // strides (floats) of the partial buffer [instance][part][source thread][6]: part stride = 32/RQ and
  // instance stride = 2 (mod 32) make the 8-byte loads of a half-warp (16 / RQ instances x RQ parts) hit
  // 16 distinct bank pairs; the 8-byte stores of 16 consecutive source threads (stride 6) are conflict free
  static constexpr int QS = (SQ * 6 + 31) / 32 * 32 + 32 / RQ;
  static constexpr int IS = RQ * QS + 2 - (RQ * QS) % 32 + ((RQ * QS) % 32 > 2 ? 32 : 0);
  static constexpr int STAGES = STAGES_;
};

template <int PX, int STAGES, int RQ, bool GATHER, int CH>
struct Bwd2Smem : std::conditional<GATHER, GatherRing<CH, STAGES, 4>, WsRing<STAGES>>::type {
  float part[Bwd2Cfg<PX, STAGES, RQ>::R * Bwd2Cfg<PX, STAGES, RQ>::IS];
  float pyt[GS_TILE];
  int valid[2];
};

// AUX backward: the 7th per-(thread, instance) partial sum, d_t = sum g_D w, lives in a plane of its own,
// [instance][part][source thread] with part stride SQ and instance stride NT + 1.  With NT == 32 (one consumer warp)
// a warp's 4-byte stores cover the 32 banks once, and the reducers' loads (32 / RQ instances x RQ parts, all at the
// same source) hit bank ri + (32 / RQ) rq: distinct as well.  The six other sums keep their buffer and strides.
template <int PX, int STAGES, int RQ, bool GATHER, int CH>
struct Bwd2SmemAux : Bwd2Smem<PX, STAGES, RQ, GATHER, CH> {
  static constexpr int TQS = Bwd2Cfg<PX, STAGES, RQ>::SQ, TIS = Bwd2Cfg<PX, STAGES, RQ>::NT + 1;
  static_assert(Bwd2Cfg<PX, STAGES, RQ>::NT == 32 && TQS * RQ == 32 && TIS % 32 == 1,
                "d_t plane strides are conflict free for one consumer warp only");
  float part_t[Bwd2Cfg<PX, STAGES, RQ>::R * TIS];
};

// ABS backward (densification statistics): two more per-(thread, instance) sums, sum_p |g_x,p| and sum_p |g_y,p| of
// the per-pixel contributions to d/dx and d/dy, in two planes laid out like the AUX d_t plane (one consumer warp:
// conflict-free stores and reducer loads).  Base: the plain or the AUX layout.
template <class Base, int R, int NT>
struct Bwd2SmemAbs : Base {
  static constexpr int AIS = NT + 1;
  static_assert(NT == 32, "absolute-gradient planes are conflict free for one consumer warp only");
  float part_ax[R * AIS];
  float part_ay[R * AIS];
};

// one instance x this thread's row of PX pixels: recompute alpha, analytic d/d alpha, six partial sums
// (AUX: gc and R carry the depth / alpha terms, and d_t = sum g_D w goes to *dst_t).  Only the first NP slots are
// evaluated (after a live-pixel repack the others are empty).  ABS: also sum_p |e_p (2 ca dx_p - cb dy)| to *dst_ax and
// sum_p |e_p (2 cc dy - cb dx_p)| to *dst_ay (the per-pixel terms of d/dx and d/dy, before the factor ln 2).
template <int PX, bool AUX = false, int NP = PX, bool ABS = false>
__device__ __forceinline__ void bwd_row(const float4 a, const float2 b, const float4 c, const float (&px)[PX],
                                        const float py, float (&T)[PX], float (&Rr)[PX], const float (&gr)[PX],
                                        const float (&gg)[PX], const float (&gb)[PX], float2* __restrict__ dst,
                                        const float t = 0.f, const float (*gD)[PX] = nullptr,
                                        const float (*gA)[PX] = nullptr, float* __restrict__ dst_t = nullptr,
                                        float* __restrict__ dst_ax = nullptr, float* __restrict__ dst_ay = nullptr) {
  float s0 = 0.f, sx = 0.f, sxx = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, dt = 0.f, ax = 0.f, ay = 0.f;
  const float dy = py - a.y;
  const float m1 = a.w * dy;
  const float ev = fmaf(-b.x * dy, dy, b.y);
  const float ca2 = 2.f * a.z, ccdy2 = 2.f * b.x * dy;   // ABS only
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const float dx = px[p] - a.x;
    const float eu = fmaf(a.z, dx, -m1);
    float alpha = gs_ex2(fmaf(-dx, eu, ev));                     // l2o - (ca dx^2 - cb dx dy + cc dy^2)
    alpha = (T[p] > GS_T_STOP) ? alpha : 0.f;                    // early stop (:578): no weight, no gradient
    const float w = alpha * T[p];
    float gc = fmaf(gr[p], c.x, fmaf(gg[p], c.y, gb[p] * c.z));
    if constexpr (AUX) gc = fmaf((*gD)[p], t, gc + (*gA)[p]);   // + g_D t_i + g_A
    Rr[p] = fmaf(-gc, w, Rr[p]);                                 // sum_c g_c (out_c - C_c^{<=i})
    const float rc = gs_rcp(1.0000001f - alpha);                 // 1/(1 - alpha + 1e-7)  (:721)
    const float dal = fmaf(T[p], gc, -Rr[p] * rc);               // d L / d alpha            (:710-722)
    const float e = dal * alpha;
    T[p] -= w;
    const float ex = e * dx;
    s0 += e;
    sx += ex;
    sxx = fmaf(ex, dx, sxx);
    c0 = fmaf(gr[p], w, c0);
    c1 = fmaf(gg[p], w, c1);
    c2 = fmaf(gb[p], w, c2);
    if constexpr (AUX) dt = fmaf((*gD)[p], w, dt);
    if constexpr (ABS) {
      ax += fabsf(e * fmaf(ca2, dx, -m1));
      ay += fabsf(e * fmaf(-a.w, dx, ccdy2));
    }
  }
  dst[0] = make_float2(s0, sx);
  dst[1] = make_float2(sxx, c0);
  dst[2] = make_float2(c1, c2);
  if constexpr (AUX) *dst_t = dt;
  if constexpr (ABS) {
    *dst_ax = ax;
    *dst_ay = ay;
  }
}

// ---- live-pixel repack (one consumer warp) --------------------------------------------------------------------
// The warp stops only when all 256 pixels of the tile are saturated; until then a saturated pixel still costs a full
// (pixel, instance) evaluation whose result is discarded.  At a reduction-round boundary the warp may therefore move
// the live pixels into fewer slots per lane: it halves the slot count S (8 -> 4 -> 2 -> 1) while the sum over rows of
// ceil(live_r / S) stays <= 32, and deals each row's live pixels to ceil(live_r / S) lanes of their own.  (Only
// halving: the phase-1 loop is compiled once per S, and on the H100 the extra loops for S = 6 and 3 cost more in
// code size than the pairs they save.)  Every lane still holds pixels of ONE row, so dy and its factors stay per lane and bwd_row is unchanged;
// only the pixel-to-lane assignment (the order of the cross-pixel sums) changes.  The rule reads T only, so the plain
// and the AUX kernel repack alike.  Empty slots have T = 0 and zero upstream gradient: they contribute exact zeros.
// The repack adds no shared memory (the kernel's CTAs per SM are limited by it): everything it stages lives in the
// partial buffer, which is free between rounds, and the lanes' row y (read by the reducers) sits in the unused tail
// of each part of instance slot 0: lane l at bwd_lane_y<SQ, QS>(l), never written by phase 1.
template <int SQ, int QS>
__device__ __forceinline__ int bwd_lane_y(int l) {
  static_assert(QS - SQ * 6 >= SQ, "a part has room for its source lanes' row y");
  return (l / SQ) * QS + SQ * 6 + l % SQ;
}

// S: current slot count (warp-uniform, only shrinks); prow / py: this lane's pixel row (GS_TILE: none) and its y.
// Called after phase 2 of a round, when the partial buffer `st` is free.  Layout of st during the call: planes of 256
// floats per pixel state variable at 0 .. 8 * 256, then the transient tables below.
constexpr int RP_ROWLIVE = 2048, RP_SRC = RP_ROWLIVE + GS_TILE, RP_CNT = RP_SRC + 32, RP_ROW = RP_CNT + 32,
              RP_PY = RP_ROW + 32, RP_END = RP_PY + 32;
template <int PX, bool AUX, int SQ, int QS>
__device__ __forceinline__ void bwd_repack(float* __restrict__ st, const float* __restrict__ pyt, int lane, int& S,
                                           int& prow, float& py, float (&px)[PX], float (&T)[PX], float (&Rr)[PX],
                                           float (&gr)[PX], float (&gg)[PX], float (&gb)[PX], float (&gD)[PX],
                                           float (&gA)[PX]) {
  int* const rowlive = reinterpret_cast<int*>(st + RP_ROWLIVE);
  int* const lsrc = reinterpret_cast<int*>(st + RP_SRC);
  int* const lcnt = reinterpret_cast<int*>(st + RP_CNT);
  int* const lrow = reinterpret_cast<int*>(st + RP_ROW);
  float* const lpy = st + RP_PY;
  int c = 0;
#pragma unroll
  for (int p = 0; p < PX; ++p) c += T[p] > GS_T_STOP ? 1 : 0;
  if (__reduce_add_sync(0xffffffffu, c) > 16 * S) return;     // cannot fit into S / 2 slots per lane yet   // cannot fit into fewer slots per lane yet
  if (lane < GS_TILE) rowlive[lane] = 0;
  __syncwarp();
  if (c) atomicAdd(&rowlive[prow], c);
  __syncwarp();
  const int live = lane < GS_TILE ? rowlive[lane] : 0;          // lane r < 16: live pixels of row r
  // lanes needed is non-increasing in S: halve while the rows still fit into 32 lanes
  int ns = S;
  while (ns > 1 && __reduce_add_sync(0xffffffffu, (live + ns / 2 - 1) / (ns / 2)) <= 32) ns /= 2;
  if (ns == S) return;

  // lanes hold their rows in row order, so the exclusive prefix of c over lanes is each lane's first position in the
  // row-major list of live pixels; stage them there, one plane of 256 per state variable
  int incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  int pos = incl - c;
#pragma unroll
  for (int p = 0; p < PX; ++p)
    if (T[p] > GS_T_STOP) {
      st[pos] = px[p];
      st[256 + pos] = T[p];
      st[512 + pos] = Rr[p];
      st[768 + pos] = gr[p];
      st[1024 + pos] = gg[p];
      st[1280 + pos] = gb[p];
      if constexpr (AUX) {
        st[1536 + pos] = gD[p];
        st[1792 + pos] = gA[p];
      }
      ++pos;
    }
  lsrc[lane] = 0;
  lcnt[lane] = 0;
  lrow[lane] = GS_TILE;
  lpy[lane] = 0.f;
  // lane r < 16: row r gets lanes [lane0, lane0 + nl), its pixels start at list position px0 (one packed scan)
  const int nl = (live + ns - 1) / ns;
  int sc = (nl << 16) | live;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, sc, o);
    if (lane >= o) sc += t;
  }
  sc -= (nl << 16) | live;
  __syncwarp();
  for (int q = 0; q < nl; ++q) {
    const int l = (sc >> 16) + q;
    lsrc[l] = (sc & 0xffff) + q * ns;
    lcnt[l] = min(ns, live - q * ns);
    lrow[l] = lane;
    lpy[l] = pyt[lane];
  }
  __syncwarp();
  const int src = lsrc[lane], n = lcnt[lane];
  prow = lrow[lane];
  py = lpy[lane];
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    const bool v = p < n;
    px[p] = v ? st[src + p] : 0.f;
    T[p] = v ? st[256 + src + p] : 0.f;
    Rr[p] = v ? st[512 + src + p] : 0.f;
    gr[p] = v ? st[768 + src + p] : 0.f;
    gg[p] = v ? st[1024 + src + p] : 0.f;
    gb[p] = v ? st[1280 + src + p] : 0.f;
    if constexpr (AUX) {
      gD[p] = v ? st[1536 + src + p] : 0.f;
      gA[p] = v ? st[1792 + src + p] : 0.f;
    }
  }
  __syncwarp();                   // every lane has read the planes: publish the row y over them for the reducers
  st[bwd_lane_y<SQ, QS>(lane)] = py;   // (phase 2 reads it after the warp barrier that ends phase 1)
  S = ns;
}

// WS: dedicated producer warp (full / empty mbarrier ring); !WS: consumer thread 0 issues the copies at the
// chunk boundaries (no extra warp holding registers).  UNR: instances per unrolled step of the first phase.
// AUX (gather only): the upstream gradient also has (g_D, g_A) per pixel (grad_aux, padded or cropped like
// grad_image); gc and R gain g_D t + g_A and g_D depth + g_A alpha (depth / alpha from the forward's aux), and
// the 7th sum d_t = sum g_D w lands in column 6 + 3 of the gradient row.
// REPACK (one consumer warp): live-pixel repack at round boundaries (bwd_repack); until the first repack the kernel
// computes exactly what it computes without it.
// ABS (one consumer warp): also sum_p |g_x,p| and sum_p |g_y,p| per instance (bwd_row), times ln 2, to the free columns
// 10 and 11 of the gradient row; every other column is computed as without it.
// BATCH (gather, batched frame): as in blend_fwd_body, the tile's view gives the pixel coordinates and the crop of a
// final upstream gradient ([B, height, width, .]); slots come from the records' rectangles, whose rows the batched
// projection offset by the view's, so the tile's frame-wide (tx, ty) address them as without it.
template <int PX, bool WS, int UNR, int STAGES, int MINB, int RQ, bool GATHER, int CH, bool AUX = false,
          bool REPACK = false, bool ABS = false, bool BATCH = false>
__device__ __forceinline__ void blend_bwd2_body(
    const float4* __restrict__ pA, const float2* __restrict__ pB, const float4* __restrict__ pC,
    const GsRec* __restrict__ grec, const uint32_t* __restrict__ ids, const uint32_t* __restrict__ goff,
    const int* __restrict__ tile_accum, int wp, int hp, int ntx, float fx, float fy, const float* __restrict__ image,
    const float* __restrict__ grad_image, float* __restrict__ grad_inst, int grad_is_final, GsCrop crop,
    uint32_t* __restrict__ row_epoch, uint32_t epoch, int* __restrict__ tile_neff_b, const float* __restrict__ aux,
    const float* __restrict__ grad_aux, const GsView* __restrict__ views) {
  static_assert(!BATCH || GATHER, "batched frames run the gather path");
  using Cfg = Bwd2Cfg<PX, STAGES, RQ>;
  constexpr int NT = Cfg::NT, TPR = Cfg::TPR, R = Cfg::R, SQ = Cfg::SQ, QS = Cfg::QS, IS = Cfg::IS, ROWS = Cfg::ROWS;
  static_assert(IS % 2 == 0 && QS % 2 == 0 && IS % 32 == 2 && QS % 32 == 32 / RQ, "partial buffer strides");
  static_assert(!(WS && GATHER), "the gather path issues its copies from all consumer threads");
  static_assert(GATHER || CH == WS_CH, "the packed ring is sized for CH instances per stage");
  static_assert(!AUX || GATHER, "the aux terms read |p_c| from the gathered records");
  static_assert(!REPACK || (NT == 32 && PX == 8), "the repack deals one warp's 256 pixels into slots of at most 8");
  static_assert(!REPACK || R * IS >= RP_END, "the partial buffer holds the repack's planes and tables");
  using SmemBase = typename std::conditional<AUX, Bwd2SmemAux<PX, STAGES, RQ, GATHER, CH>,
                                             Bwd2Smem<PX, STAGES, RQ, GATHER, CH>>::type;
  using Smem = typename std::conditional<ABS, Bwd2SmemAbs<SmemBase, R, NT>, SmemBase>::type;
  __shared__ __align__(16) Smem sm;
  const int tile = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int nchunks = (cnt + CH - 1) / CH;
  const int tx = tile % ntx, ty = tile / ntx;
  const int shift = start & 1;
  int lty = ty;   // the tile's row in its view
  if constexpr (BATCH) {
    const int v = ty / (hp / GS_TILE);
    lty = ty - v * (hp / GS_TILE);
    fx = views[v].fx;
    fy = views[v].fy;
    if (grad_is_final) {
      grad_image += (size_t)v * crop.width * crop.height * 3;
      if (grad_aux) grad_aux += (size_t)v * crop.width * crop.height * 2;
    }
  }
  if (tid < GS_TILE) sm.pyt[tid] = gs_pixel_coord(lty * GS_TILE + tid, hp, fy);
  if constexpr (GATHER) {
    if (tid == 0) {
      for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.full[s], NT);
      gs_fence_barrier_init();
    }
    __syncthreads();
  } else {
    ws_init<Smem, STAGES>(sm, tid);
    if (WS) {
      if (tid >= NT) {
        if (tid == NT) ws_producer<Smem, STAGES>(sm, pA, pB, pC, start, cnt, nchunks);
        return;
      }
    } else if (tid == 0) {
      for (int k = 0; k < STAGES && k < nchunks; ++k)
        issue_chunk<Smem, CH>(sm, k, pA, pB, pC, start + k * CH, min(CH, cnt - k * CH), shift);
    }
  }
  GatherIds<NT, CH> gid;
  if constexpr (GATHER) {
    for (int k = 0; k < STAGES && k < nchunks; ++k) {
      gid.load(ids, start + k * CH, min(CH, cnt - k * CH), tid);
      gather_issue<Smem, NT, CH, 4>(sm, k, grec, goff, gid, min(CH, cnt - k * CH), tid);
    }
    if (STAGES < nchunks) gid.load(ids, start + STAGES * CH, min(CH, cnt - STAGES * CH), tid);
  }
  const int ix0 = tx * GS_TILE + (tid % TPR) * PX;
  const int iy = ty * GS_TILE + (tid / TPR);
  const int iyv = lty * GS_TILE + (tid / TPR);   // its row in the view
  float px[PX];
#pragma unroll
  for (int p = 0; p < PX; ++p) px[p] = gs_pixel_coord(ix0 + p, wp, fx);
  float py = sm.pyt[tid / TPR];
  int S = PX, prow = tid / TPR;   // REPACK: slots per lane in use, and this lane's pixel row

  float T[PX], Rr[PX], gr[PX], gg[PX], gb[PX];
  {
    const size_t off = ((size_t)iy * wp + ix0) * 3;     // PX*12 contiguous, 16-byte aligned bytes
    const float4* im = reinterpret_cast<const float4*>(image + off);
    float gbuf[PX * 3], ibuf[PX * 3];
#pragma unroll
    for (int q = 0; q < PX * 3 / 4; ++q) {
      const float4 i4 = im[q];
      ibuf[4 * q] = i4.x; ibuf[4 * q + 1] = i4.y; ibuf[4 * q + 2] = i4.z; ibuf[4 * q + 3] = i4.w;
    }
    if (!grad_is_final) {
      const float4* gi = reinterpret_cast<const float4*>(grad_image + off);
#pragma unroll
      for (int q = 0; q < PX * 3 / 4; ++q) {
        const float4 g4 = gi[q];
        gbuf[4 * q] = g4.x; gbuf[4 * q + 1] = g4.y; gbuf[4 * q + 2] = g4.z; gbuf[4 * q + 3] = g4.w;
      }
    } else {
#pragma unroll
      for (int p = 0; p < PX; ++p)
        gs_load_final_grad(grad_image, ibuf + 3 * p, ix0 + p, iyv, crop.left, crop.top, crop.width, crop.height,
                           gbuf[3 * p], gbuf[3 * p + 1], gbuf[3 * p + 2]);
    }
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      gr[p] = gbuf[3 * p];
      gg[p] = gbuf[3 * p + 1];
      gb[p] = gbuf[3 * p + 2];
      Rr[p] = gr[p] * ibuf[3 * p] + gg[p] * ibuf[3 * p + 1] + gb[p] * ibuf[3 * p + 2];
      T[p] = 1.f;
    }
  }
  float gD[PX], gA[PX];
  if constexpr (AUX) {
    // R = sum_c g_c image_c + g_D depth + g_A alpha (forward outputs); (depth, alpha) x PX = PX * 8 aligned bytes
    const size_t off = ((size_t)iy * wp + ix0) * 2;
    float abuf[PX * 2], gbuf[PX * 2];
#pragma unroll
    for (int q = 0; q < PX / 2; ++q) {
      const float4 v = reinterpret_cast<const float4*>(aux + off)[q];
      abuf[4 * q] = v.x; abuf[4 * q + 1] = v.y; abuf[4 * q + 2] = v.z; abuf[4 * q + 3] = v.w;
    }
    if (!grad_is_final) {
#pragma unroll
      for (int q = 0; q < PX / 2; ++q) {
        const float4 v = reinterpret_cast<const float4*>(grad_aux + off)[q];
        gbuf[4 * q] = v.x; gbuf[4 * q + 1] = v.y; gbuf[4 * q + 2] = v.z; gbuf[4 * q + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int p = 0; p < PX; ++p) {   // depth / alpha are not clamped: only the crop masks their gradient
        const int x = ix0 + p - crop.left, y = iyv - crop.top;
        float2 v = make_float2(0.f, 0.f);
        if (x >= 0 && x < crop.width && y >= 0 && y < crop.height)
          v = *reinterpret_cast<const float2*>(grad_aux + ((size_t)y * crop.width + x) * 2);
        gbuf[2 * p] = v.x;
        gbuf[2 * p + 1] = v.y;
      }
    }
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      gD[p] = gbuf[2 * p];
      gA[p] = gbuf[2 * p + 1];
      Rr[p] = fmaf(gD[p], abuf[2 * p], fmaf(gA[p], abuf[2 * p + 1], Rr[p]));
    }
  }
  // this thread's slot in the partial buffer: quarter tid / SQ, position tid % SQ
  float2* const my_part = reinterpret_cast<float2*>(sm.part + (tid / SQ) * QS + (tid % SQ) * 6);
  float* my_part_t = nullptr;   // AUX: this thread's slot in the d_t plane
  if constexpr (AUX) my_part_t = sm.part_t + (tid / SQ) * Smem::TQS + (tid % SQ);
  float *my_part_ax = nullptr, *my_part_ay = nullptr;   // ABS: this thread's slots in the |g| planes
  if constexpr (ABS) {
    my_part_ax = sm.part_ax + tid;
    my_part_ay = sm.part_ay + tid;
  }
  // second-phase role: instance ri of the round, quarter rq of the source threads
  const int ri = tid / RQ, rq = tid % RQ;
  const float2* const red_src = reinterpret_cast<const float2*>(sm.part + ri * IS + rq * QS);

  int consumed = cnt;
  bool finished = false;
  int k = 0;
  for (; k < nchunks && !finished; ++k) {
    const int stage = k % STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / STAGES) & 1));
    const int n = min(CH, cnt - k * CH);
    StageView<GATHER> sv;
    if constexpr (GATHER) {
      sv.R = sm.rec[stage];
      sv.recw = 4;
    } else {
      sv.A = sm.A[stage];
      sv.C = sm.C[stage];
      sv.B = sm.B[stage] + shift;
    }

    for (int sub = 0; sub < n; sub += R) {
      const int nr = min(R, n - sub);
      // ---- phase 1: per-thread partial sums of up to R instances (NP: slots per lane in use)
      // (the repacked loops are not unrolled over instances: unrolling them grows the kernel's code and was measured
      // slower on the H100 - by ~30 % with 4 instances per step, ~15 % with 2)
      auto phase1 = [&](auto np) -> int {
        constexpr int NP = decltype(np)::value, U = NP == PX ? UNR : 1;
        // instance q of the round: its sums go to slot q of the partial buffer and of the d_t (AUX) / |g| (ABS)
        // planes, whose instance stride is NT + 1 (Bwd2SmemAux::TIS, Bwd2SmemAbs::AIS)
        auto row = [&](int q) {
          float t = 0.f;
          if constexpr (AUX) t = sv.depth(sub + q);
          bwd_row<PX, AUX, NP, ABS>(sv.a(sub + q), sv.b(sub + q), sv.c(sub + q), px, py, T, Rr, gr, gg, gb,
                                    my_part + q * (IS / 2), t, &gD, &gA, AUX ? my_part_t + q * (NT + 1) : nullptr,
                                    ABS ? my_part_ax + q * (NT + 1) : nullptr, ABS ? my_part_ay + q * (NT + 1) : nullptr);
        };
        int j = 0;
        bool wdead = false;
#pragma unroll 1
        for (; j + U <= nr; j += U) {
          if (U >= 4 || (j & 3) == 0) {
            bool dead = true;
#pragma unroll
            for (int p = 0; p < PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
            if (__all_sync(0xffffffffu, dead)) {
              wdead = true;
              break;
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) row(j + u);
        }
        if (U > 1 && !wdead)
          for (; j < nr; ++j) row(j);
        return j;
      };
      int j;
      if constexpr (REPACK) {
        switch (S) {   // warp-uniform
          case 8: j = phase1(std::integral_constant<int, 8>{}); break;
          case 4: j = phase1(std::integral_constant<int, 4>{}); break;
          case 2: j = phase1(std::integral_constant<int, 2>{}); break;
          default: j = phase1(std::integral_constant<int, 1>{}); break;
        }
      } else {
        j = phase1(std::integral_constant<int, PX>{});
      }
      bool dead = true;
#pragma unroll
      for (int p = 0; p < PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
      int all_dead;
      int v0, v1;
      if (NT == 64) {
        if (lane == 0) sm.valid[warp] = j;          // j is warp-uniform (the loop only breaks on a warp vote)
        all_dead = gs_bar_red_and(1, NT, dead);
        v0 = sm.valid[0];
        v1 = sm.valid[1];
      } else {
        __syncwarp();
        all_dead = __all_sync(0xffffffffu, dead);
        v0 = v1 = j;
      }
      // ---- phase 2: 4 threads per instance, one quarter of the source threads (4 pixel rows) each
      {
        float S0 = 0.f, Sx = 0.f, Sxx = 0.f, Sy = 0.f, Sxy = 0.f, Syy = 0.f, C0 = 0.f, C1 = 0.f, C2 = 0.f;
        const bool act = ri < nr;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        float2 b = make_float2(0.f, 0.f);
        if (act) {
          a = sv.a(sub + ri);
          b = sv.b(sub + ri);
        }
        const int vq = (NT == 64 && rq * SQ >= 32) ? v1 : v0;   // instances the part's source warp really processed
        if (REPACK && act && ri < vq && S < PX) {
          // repacked: the source lanes' rows are in the lane table, dy is formed per source lane
#pragma unroll
          for (int s = 0; s < SQ; ++s) {
            const float2 w0 = red_src[s * 3], w1 = red_src[s * 3 + 1], w2 = red_src[s * 3 + 2];
            float dyl = 0.f;
            if constexpr (REPACK) dyl = sm.part[bwd_lane_y<SQ, QS>(rq * SQ + s)] - a.y;
            S0 += w0.x;
            Sx += w0.y;
            Sxx += w1.x;
            C0 += w1.y;
            C1 += w2.x;
            C2 += w2.y;
            Sy = fmaf(dyl, w0.x, Sy);
            Sxy = fmaf(dyl, w0.y, Sxy);
            Syy = fmaf(dyl * dyl, w0.x, Syy);
          }
        } else if (act && ri < vq) {
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            float2 u0 = red_src[(r * TPR) * 3], u1 = red_src[(r * TPR) * 3 + 1], u2 = red_src[(r * TPR) * 3 + 2];
#pragma unroll
            for (int t = 1; t < TPR; ++t) {
              const float2 w0 = red_src[(r * TPR + t) * 3], w1 = red_src[(r * TPR + t) * 3 + 1],
                           w2 = red_src[(r * TPR + t) * 3 + 2];
              u0.x += w0.x; u0.y += w0.y; u1.x += w1.x; u1.y += w1.y; u2.x += w2.x; u2.y += w2.y;
            }
            const float dyr = sm.pyt[ROWS * rq + r] - a.y;
            S0 += u0.x;
            Sx += u0.y;
            Sxx += u1.x;
            C0 += u1.y;
            C1 += u2.x;
            C2 += u2.y;
            Sy = fmaf(dyr, u0.x, Sy);
            Sxy = fmaf(dyr, u0.y, Sxy);
            Syy = fmaf(dyr * dyr, u0.x, Syy);
          }
        }
        float Dt = 0.f;
        if constexpr (AUX) {
          if (act && ri < vq) {
            const float* src = sm.part_t + ri * Smem::TIS + rq * Smem::TQS;
#pragma unroll
            for (int s = 0; s < SQ; ++s) Dt += src[s];
          }
        }
        float Ax = 0.f, Ay = 0.f;
        if constexpr (ABS) {
          if (act && ri < vq) {
            const float* srx = sm.part_ax + ri * Smem::AIS + rq * SQ;
            const float* sry = sm.part_ay + ri * Smem::AIS + rq * SQ;
#pragma unroll
            for (int s = 0; s < SQ; ++s) {
              Ax += srx[s];
              Ay += sry[s];
            }
          }
        }
#define GS_RED4(V)                                   \
  V += __shfl_xor_sync(0xffffffffu, V, 1);           \
  V += __shfl_xor_sync(0xffffffffu, V, 2);           \
  if (RQ == 8) V += __shfl_xor_sync(0xffffffffu, V, 4);
        GS_RED4(S0) GS_RED4(Sx) GS_RED4(Sxx) GS_RED4(Sy) GS_RED4(Sxy) GS_RED4(Syy) GS_RED4(C0) GS_RED4(C1) GS_RED4(C2)
        if constexpr (AUX) { GS_RED4(Dt) }
        if constexpr (ABS) { GS_RED4(Ax) GS_RED4(Ay) }
#undef GS_RED4
        if (act) {
          const uint32_t slot = sv.slot(sub + ri, tx, ty);
          float4* out = reinterpret_cast<float4*>(grad_inst + (size_t)slot * GS_GREC);
          // d/dx, d/dy, d/dca, d/dcb  |  d/dcc, d/dl2o, d/dr, d/dg  |  d/db
          if (rq == 0)
            out[0] = make_float4(GS_LN2 * (2.f * a.z * Sx - a.w * Sy), GS_LN2 * (2.f * b.x * Sy - a.w * Sx),
                                 -GS_LN2 * Sxx, GS_LN2 * Sxy);
          else if (rq == 1)
            out[1] = make_float4(-GS_LN2 * Syy, GS_LN2 * S0, C0, C1);
          else if (rq == 2)
            out[2] = ABS ? make_float4(C2, Dt, GS_LN2 * Ax, GS_LN2 * Ay)   // | d/db, d/dt (AUX; 0 otherwise),
                         : make_float4(C2, Dt, 0.f, 0.f);                  //   sum |d/dx|, sum |d/dy| (ABS)
          else if (rq == 3 && row_epoch)
            row_epoch[slot] = epoch;               // marks the row as written in this frame
        }
      }
      if (NT == 64) gs_bar_sync(1, NT);            // the partial buffer may be overwritten now
      else __syncwarp();
      if (all_dead) {
        consumed = min(cnt, k * CH + sub + nr);
        finished = true;
        break;
      }
      if constexpr (REPACK)
        if (S > 1) bwd_repack<PX, AUX, SQ, QS>(sm.part, sm.pyt, lane, S, prow, py, px, T, Rr, gr, gg, gb, gD, gA);
    }
    if constexpr (GATHER) {
      if (!finished && k + STAGES < nchunks) {   // every consumer is past the barrier: the stage is free
        const int kn = k + STAGES;
        gather_issue<Smem, NT, CH, 4>(sm, stage, grec, goff, gid, min(CH, cnt - kn * CH), tid);
        if (kn + 1 < nchunks) gid.load(ids, start + (kn + 1) * CH, min(CH, cnt - (kn + 1) * CH), tid);
      }
    } else if (tid == 0) {
      if (WS) {
        sm.consumed_chunks = k + 1;
        if (finished) sm.stop = 1;
        gs_mbar_arrive(&sm.empty[stage]);
      } else if (!finished && k + STAGES < nchunks) {
        const int kn = k + STAGES;               // every consumer is past the barrier: the stage is free
        issue_chunk<Smem, CH>(sm, stage, pA, pB, pC, start + kn * CH, min(CH, cnt - kn * CH), shift);
      }
    }
  }
  if (tid == 0) {
    if constexpr (!GATHER && WS) {
      gs_mbar_arrive(&sm.done);
    } else if (finished) {
      // drain copies that were issued but never consumed before the CTA may retire (k was incremented past the
      // chunk that finished): chunks k .. k + STAGES - 2 are in flight
      for (int kk = k; kk < nchunks && kk < k + STAGES - 1; ++kk)
        gs_mbar_wait(&sm.full[kk % STAGES], (uint32_t)((kk / STAGES) & 1));
    }
    if (tile_neff_b) tile_neff_b[tile] = consumed;
  }
  // the unread tail of a saturated tile has zero gradient: with an epoch array the rows are simply
  // left stale (the consumer skips rows whose tag is not this frame's); otherwise write zeros
  if (row_epoch || GATHER) return;              // (the gather path always runs with an epoch array)
  for (int t = consumed + tid; t < cnt; t += NT) {
    const uint32_t slot = __float_as_uint(pC[start + t].w);
    float4* out = reinterpret_cast<float4*>(grad_inst + (size_t)slot * GS_GREC);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    out[0] = z;
    out[1] = z;
    out[2] = z;
  }
}

#define GS_BWD2_PARAMS                                                                                              \
  const float4 *__restrict__ pA, const float2 *__restrict__ pB, const float4 *__restrict__ pC,                      \
      const GsRec *__restrict__ grec, const uint32_t *__restrict__ ids, const uint32_t *__restrict__ goff,          \
      const int *__restrict__ tile_accum, int wp, int hp, int ntx, float fx, float fy,                              \
      const float *__restrict__ image, const float *__restrict__ grad_image, float *__restrict__ grad_inst,         \
      int grad_is_final, GsCrop crop, uint32_t *__restrict__ row_epoch, uint32_t epoch,                             \
      int *__restrict__ tile_neff_b, const float *__restrict__ aux, const float *__restrict__ grad_aux
#define GS_BWD2_ARGS                                                                                              \
  pA, pB, pC, grec, ids, goff, tile_accum, wp, hp, ntx, fx, fy, image, grad_image, grad_inst, grad_is_final, crop, \
      row_epoch, epoch, tile_neff_b, aux, grad_aux

template <int PX, bool WS, int UNR, int STAGES, int MINB, int RQ, bool GATHER, int CH, bool AUX = false,
          bool REPACK = false, bool ABS = false>
__global__ void __launch_bounds__(256 / PX + (WS ? 32 : 0), MINB) blend_bwd2_kernel(GS_BWD2_PARAMS) {
  blend_bwd2_body<PX, WS, UNR, STAGES, MINB, RQ, GATHER, CH, AUX, REPACK, ABS>(GS_BWD2_ARGS, nullptr);
}

// the shipped gather backward with the live-pixel repack (AUX, ABS as in blend_bwd2_kernel) of a batched frame
template <bool AUX, bool ABS>
__global__ void __launch_bounds__(32, 10) blend_bwd2_batch_kernel(GS_BWD2_PARAMS, const GsView* __restrict__ views) {
  blend_bwd2_body<8, false, 4, 3, 10, 4, true, 32, AUX, true, ABS, true>(GS_BWD2_ARGS, views);
}
#undef GS_BWD2_ARGS
#undef GS_BWD2_PARAMS

// =======================================================================================
// legacy boundary helpers: per-instance tensors <-> packed record streams
// =======================================================================================
__global__ void __launch_bounds__(256) legacy_pack_kernel(const float* __restrict__ pos, const float* __restrict__ rgb,
                                                           const float* __restrict__ opa,
                                                           const float* __restrict__ cov, int m,
                                                           float4* __restrict__ pA, float2* __restrict__ pB,
                                                           float4* __restrict__ pC) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= m) return;
  float4 cv = reinterpret_cast<const float4*>(cov)[i];
  GsConic k = gs_make_conic(cv.x, cv.y, cv.z, cv.w);
  pA[i] = make_float4(pos[3 * i], pos[3 * i + 1], k.ca, k.cb);
  pB[i] = make_float2(k.cc, log2f(opa[i]));
  pC[i] = make_float4(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], __uint_as_float((uint32_t)i));
}

__global__ void __launch_bounds__(256) legacy_unpack_grads_kernel(const float* __restrict__ grad_inst,
                                                                   const float* __restrict__ opa,
                                                                   const float* __restrict__ cov, int m,
                                                                   float* __restrict__ g_pos,
                                                                   float* __restrict__ g_rgb,
                                                                   float* __restrict__ g_opa,
                                                                   float* __restrict__ g_cov) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= m) return;
  const float4* row = reinterpret_cast<const float4*>(grad_inst + (size_t)i * GS_GREC);
  float4 v0 = row[0], v1 = row[1], v2 = row[2];
  float4 cv = reinterpret_cast<const float4*>(cov)[i];
  float det = cv.x * cv.w - cv.y * cv.z;
  double pn = 2.0 * (double)det + 1e-14;
  float sc = (float)((double)GS_LOG2E / pn);
  float kk = 2.f * sc * sc / GS_LOG2E;
  float gsc = v0.z * cv.w + v0.w * (cv.y + cv.z) + v1.x * cv.x;
  g_pos[3 * i] = v0.x;
  g_pos[3 * i + 1] = v0.y;                                    // z column untouched (gaussian.cu:785-786)
  reinterpret_cast<float4*>(g_cov)[i] = make_float4(v1.x * sc - gsc * kk * cv.w, v0.w * sc + gsc * kk * cv.z,
                                                    v0.w * sc + gsc * kk * cv.y, v0.z * sc - gsc * kk * cv.x);
  g_opa[i] = opa[i] > 0.f ? v1.y / (opa[i] * GS_LN2) : 0.f;   // opacity exactly 0: alpha == 0 everywhere, log2 undefined
  g_rgb[3 * i] = v1.z;
  g_rgb[3 * i + 1] = v1.w;
  g_rgb[3 * i + 2] = v2.x;
}

// SH variants: third stream row = {coef[0..d), slot, pad}; gradient row = {6 geometry, d coefficient}
__global__ void __launch_bounds__(256) legacy_pack_sh_kernel(const float* __restrict__ pos,
                                                              const float* __restrict__ rgb,
                                                              const float* __restrict__ opa,
                                                              const float* __restrict__ cov, int m, int d, int sw,
                                                              float4* __restrict__ pA, float2* __restrict__ pB,
                                                              float* __restrict__ pS) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= m) return;
  float4 cv = reinterpret_cast<const float4*>(cov)[i];
  GsConic k = gs_make_conic(cv.x, cv.y, cv.z, cv.w);
  pA[i] = make_float4(pos[3 * i], pos[3 * i + 1], k.ca, k.cb);
  pB[i] = make_float2(k.cc, log2f(opa[i]));
  float* row = pS + (size_t)i * sw;
  const float* src = rgb + (size_t)i * d;
  for (int q = 0; q < d; ++q) row[q] = src[q];
  row[d] = __uint_as_float((uint32_t)i);
}

__global__ void __launch_bounds__(256) legacy_unpack_grads_sh_kernel(const float* __restrict__ grad_inst, int gw,
                                                                      const float* __restrict__ opa,
                                                                      const float* __restrict__ cov, int m, int d,
                                                                      float* __restrict__ g_pos,
                                                                      float* __restrict__ g_rgb,
                                                                      float* __restrict__ g_opa,
                                                                      float* __restrict__ g_cov) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= m) return;
  const float* row = grad_inst + (size_t)i * gw;
  float4 cv = reinterpret_cast<const float4*>(cov)[i];
  float det = cv.x * cv.w - cv.y * cv.z;
  double pn = 2.0 * (double)det + 1e-14;
  float sc = (float)((double)GS_LOG2E / pn);
  float kk = 2.f * sc * sc / GS_LOG2E;
  float d_ca = row[2], d_cb = row[3], d_cc = row[4];
  float gsc = d_ca * cv.w + d_cb * (cv.y + cv.z) + d_cc * cv.x;
  g_pos[3 * i] = row[0];
  g_pos[3 * i + 1] = row[1];
  reinterpret_cast<float4*>(g_cov)[i] = make_float4(d_cc * sc - gsc * kk * cv.w, d_cb * sc + gsc * kk * cv.z,
                                                    d_cb * sc + gsc * kk * cv.y, d_ca * sc - gsc * kk * cv.x);
  g_opa[i] = opa[i] > 0.f ? row[5] / (opa[i] * GS_LN2) : 0.f;
  for (int q = 0; q < d; ++q) g_rgb[(size_t)i * d + q] = row[6 + q];
}

struct LegacyWs {
  float4* pA;
  float2* pB;
  float4* pC;
  float* grad_inst;
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// d == 3: pC is the float4 colour stream; d == 27 / 48: pC aliases the SH stream (sw floats / row)
inline size_t legacy_ws_layout(int m, int d, LegacyWs* ws, char* base) {
  size_t off = 0;
  size_t mm = (size_t)(m > 0 ? m : 0);
  size_t crow = d == 3 ? 16 : (size_t)gs_sh_stream_width(d) * 4;
  size_t grow = d == 3 ? (size_t)GS_GREC * 4 : (size_t)gs_sh_grad_width(d) * 4;
  if (ws) ws->pA = reinterpret_cast<float4*>(base + off);
  off += align_up(mm * 16, 256);
  if (ws) ws->pC = reinterpret_cast<float4*>(base + off);
  off += align_up(mm * crow + 16, 256);
  if (ws) ws->pB = reinterpret_cast<float2*>(base + off);
  off += align_up((mm + 2) * 8, 256);
  if (ws) ws->grad_inst = reinterpret_cast<float*>(base + off);
  off += align_up(mm * grow, 256);
  return off;
}

}  // namespace

cudaError_t gs_launch_blend_fwd(const float4* pA, const float2* pB, const float4* pC, const GsRec* grec,
                                const uint32_t* ids, const int* tile_accum, const GsFrameGeom& g, float* image,
                                int* tile_neff, float* final_img, const GsCrop& crop, cudaStream_t st,
                                const GsAuxOut* aux) {
  const GsTuning& tn = gs_tuning();
  const bool gather = grec != nullptr;
  if (aux) {   // the caller has checked gs_blend_aux_supported(true, ...); grec is null only when N == 0 (no instances)
    blend_fwd_kernel<128, 4, true, true><<<g.n_tiles, 64, 0, st>>>(pA, pB, pC, grec, ids, tile_accum, g.wp, g.hp, g.ntx,
                                                                  g.fx, g.fy, image, tile_neff, final_img, crop, *aux);
    return cudaGetLastError();
  }
  if (!gather && tn.fwd_kernel != 0) {
    blend_fwd_ws_kernel<<<g.n_tiles, WSF_CONS + 32, 0, st>>>(pA, pB, pC, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image,
                                                             tile_neff, final_img, crop);
    return cudaGetLastError();
  }
  const int ch = tn.fwd_ch;   // staging chunk
#define GS_FWD_LAUNCH(CH, PX, GA)                                                                                   \
  blend_fwd_kernel<CH, PX, GA><<<g.n_tiles, 256 / PX, 0, st>>>(pA, pB, pC, grec, ids, tile_accum, g.wp, g.hp, g.ntx, \
                                                               g.fx, g.fy, image, tile_neff, final_img, crop, GsAuxOut{})
#define GS_FWD_CH(PX, GA)                     \
  if (ch == 64) GS_FWD_LAUNCH(64, PX, GA);    \
  else if (ch == 256) GS_FWD_LAUNCH(256, PX, GA); \
  else GS_FWD_LAUNCH(128, PX, GA)
  if (gather) {
    if (tn.fwd_px == 8) { GS_FWD_CH(8, true); } else { GS_FWD_CH(4, true); }
  } else {
    if (tn.fwd_px == 8) { GS_FWD_CH(8, false); } else { GS_FWD_CH(4, false); }
  }
#undef GS_FWD_CH
#undef GS_FWD_LAUNCH
  return cudaGetLastError();
}

cudaError_t gs_launch_blend_bwd(const float4* pA, const float2* pB, const float4* pC, const GsRec* grec,
                                const uint32_t* ids, const uint32_t* goff, const int* tile_accum, const GsFrameGeom& g,
                                const float* image,
                                const float* grad_image, float* grad_inst, int grad_is_final, const GsCrop& crop,
                                uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b, cudaStream_t st,
                                const float* aux, const float* grad_aux, bool absgrad) {
  const GsTuning& tn = gs_tuning();
  const bool gather = grec != nullptr;
  if (gather && !row_epoch) return cudaErrorInvalidValue;
  if (absgrad) {   // the caller has checked gs_blend_absgrad_supported (and gs_blend_aux_supported with grad_aux)
    if (!gather || (grad_aux && !aux)) return cudaErrorInvalidValue;
#define GS_BWD2_ABS(AX, RP)                                                                                        \
  blend_bwd2_kernel<8, false, 4, 3, 10, 4, true, 32, AX, RP, true><<<g.n_tiles, 32, 0, st>>>(                       \
      pA, pB, pC, grec, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image, grad_image, grad_inst,         \
      grad_is_final, crop, row_epoch, epoch, tile_neff_b, aux, grad_aux)
    if (grad_aux && tn.blend_repack) GS_BWD2_ABS(true, true);
    else if (grad_aux) GS_BWD2_ABS(true, false);
    else if (tn.blend_repack) GS_BWD2_ABS(false, true);
    else GS_BWD2_ABS(false, false);
#undef GS_BWD2_ABS
    return cudaGetLastError();
  }
  if (grad_aux) {   // the caller has checked gs_blend_aux_supported(..., true)
    if (!gather || !aux) return cudaErrorInvalidValue;
#define GS_BWD2_AUX(RP)                                                                                            \
  blend_bwd2_kernel<8, false, 4, 3, 10, 4, true, 32, true, RP><<<g.n_tiles, 32, 0, st>>>(                           \
      pA, pB, pC, grec, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image, grad_image, grad_inst,         \
      grad_is_final, crop, row_epoch, epoch, tile_neff_b, aux, grad_aux)
    if (tn.blend_repack) GS_BWD2_AUX(true);
    else GS_BWD2_AUX(false);
#undef GS_BWD2_AUX
    return cudaGetLastError();
  }
  if (tn.bwd_kernel != 0 || gather) {
#define GS_BWD2C(PX, WS, UNR, ST, MINB, RQ, GA, CH)                                                                 \
  blend_bwd2_kernel<PX, WS, UNR, ST, MINB, RQ, GA, CH><<<g.n_tiles, 256 / PX + (WS ? 32 : 0), 0, st>>>(              \
      pA, pB, pC, grec, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image, grad_image, grad_inst,          \
      grad_is_final,                                                                                                 \
      crop, row_epoch, epoch, tile_neff_b, nullptr, nullptr)
#define GS_BWD2(PX, WS, UNR, ST, MINB, RQ, GA) GS_BWD2C(PX, WS, UNR, ST, MINB, RQ, GA, 64)
    // key: px | producer warp | unroll | stages | reducers per instance | min blocks (2 digits)
    const int key = ((((tn.bwd_px * 10 + tn.bwd_ws) * 10 + tn.bwd_unroll) * 10 + tn.bwd_stages) * 10 + tn.bwd_rq) * 100 +
                    tn.bwd_minb;
    if (gather && tn.bwd_ch == 32) {
      // the shipped configuration runs with or without the live-pixel repack; the other variants have none
#define GS_BWD2_SHIPPED()                                                                                          \
  if (tn.blend_repack)                                                                                             \
    blend_bwd2_kernel<8, false, 4, 3, 10, 4, true, 32, false, true><<<g.n_tiles, 32, 0, st>>>(                      \
        pA, pB, pC, grec, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image, grad_image, grad_inst,       \
        grad_is_final, crop, row_epoch, epoch, tile_neff_b, nullptr, nullptr);                                     \
  else                                                                                                             \
    GS_BWD2C(8, false, 4, 3, 10, 4, true, 32)
      switch (key) {
        case 8022416: GS_BWD2C(8, false, 2, 2, 16, 4, true, 32); break;
        case 8023416: GS_BWD2C(8, false, 2, 3, 16, 4, true, 32); break;
        case 8042410: GS_BWD2C(8, false, 4, 2, 10, 4, true, 32); break;
        case 8043410: GS_BWD2_SHIPPED(); break;
        default:
          if (gs_tuning().strict) return cudaErrorInvalidValue;
          GS_BWD2_SHIPPED();
          break;
      }
#undef GS_BWD2_SHIPPED
      return cudaGetLastError();
    }
    if (gather) {
      switch (key) {
        case 8012410: GS_BWD2(8, false, 1, 2, 10, 4, true); break;
        case 8022416: GS_BWD2(8, false, 2, 2, 16, 4, true); break;
        case 8022410: GS_BWD2(8, false, 2, 2, 10, 4, true); break;
        case 8042410: GS_BWD2(8, false, 4, 2, 10, 4, true); break;
        case 8023416: GS_BWD2(8, false, 2, 3, 16, 4, true); break;
        case 8012416: GS_BWD2(8, false, 1, 2, 16, 4, true); break;
        case 8012420: GS_BWD2(8, false, 1, 2, 20, 4, true); break;
        case 8012820: GS_BWD2(8, false, 1, 2, 20, 8, true); break;
        case 8013416: GS_BWD2(8, false, 1, 3, 16, 4, true); break;
        case 4012401: GS_BWD2(4, false, 1, 2, 1, 4, true); break;
        case 4042401: GS_BWD2(4, false, 4, 2, 1, 4, true); break;
        default: return gs_tuning().strict ? cudaErrorInvalidValue : (GS_BWD2(8, false, 2, 2, 16, 4, true), cudaGetLastError());
      }
      return cudaGetLastError();
    }
    switch (key) {
      case 4113401: GS_BWD2(4, true, 1, 3, 1, 4, false); break;      // round-2 first version
      case 4143408: GS_BWD2(4, true, 4, 3, 8, 4, false); break;
      case 4012401: GS_BWD2(4, false, 1, 2, 1, 4, false); break;
      case 4042401: GS_BWD2(4, false, 4, 2, 1, 4, false); break;
      case 4042810: GS_BWD2(4, false, 4, 2, 10, 8, false); break;
      case 8012410: GS_BWD2(8, false, 1, 2, 10, 4, false); break;
      case 8012416: GS_BWD2(8, false, 1, 2, 16, 4, false); break;
      case 8012420: GS_BWD2(8, false, 1, 2, 20, 4, false); break;
      case 8013416: GS_BWD2(8, false, 1, 3, 16, 4, false); break;
      case 8022416: GS_BWD2(8, false, 2, 2, 16, 4, false); break;
      case 8022410: GS_BWD2(8, false, 2, 2, 10, 4, false); break;
      case 8042410: GS_BWD2(8, false, 4, 2, 10, 4, false); break;
      case 8012816: GS_BWD2(8, false, 1, 2, 16, 8, false); break;
      case 8012820: GS_BWD2(8, false, 1, 2, 20, 8, false); break;
      case 8112410: GS_BWD2(8, true, 1, 2, 10, 4, false); break;
      case 8012424: GS_BWD2(8, false, 1, 2, 24, 4, false); break;
      case 8012824: GS_BWD2(8, false, 1, 2, 24, 8, false); break;
      // the packed path (legacy draw API, gs_tune("gather", 0)) has fewer instantiated variants than the gather
      // path: any other knob combination runs its shipped configuration (strict mode, used by the sweeps, refuses)
      default: return gs_tuning().strict ? cudaErrorInvalidValue : (GS_BWD2(8, false, 2, 2, 16, 4, false), cudaGetLastError());
    }
#undef GS_BWD2
#undef GS_BWD2C
    return cudaGetLastError();
  }
  const int warps = tn.bwd_px == 8 ? 1 : 2;   // round-1 kernel: 1 warp x 8 px or 2 warps x 4 px
  const int ch = 64;
#define GS_BWD_LAUNCH(W, CH)                                                                                         \
  blend_bwd_kernel<W, CH><<<g.n_tiles, 32 * W, 0, st>>>(pA, pB, pC, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image, \
                                                        grad_image, grad_inst, grad_is_final, crop, row_epoch, epoch, \
                                                        tile_neff_b)
  if (warps == 1) GS_BWD_LAUNCH(1, 64);
  else if (ch == 32) GS_BWD_LAUNCH(2, 32);
  else if (ch == 128) GS_BWD_LAUNCH(2, 128);
  else GS_BWD_LAUNCH(2, 64);
#undef GS_BWD_LAUNCH
  return cudaGetLastError();
}

// the shipped backward knobs of the gather RGB blend, the only configuration with AUX and ABS kernels
static bool shipped_rgb_bwd_knobs(const GsTuning& tn) {
  return tn.bwd_kernel != 0 && tn.bwd_px == 8 && tn.bwd_ws == 0 && tn.bwd_unroll == 4 && tn.bwd_stages == 3 &&
         tn.bwd_rq == 4 && tn.bwd_minb == 10 && tn.bwd_ch == 32;
}

int gs_blend_aux_supported(int d, bool forward, bool backward) {
  const GsTuning& tn = gs_tuning();
  if (!tn.gather)
    return gs_set_error_msg(GS_ERR_UNSUPPORTED, "depth / alpha / background: the packed path (gs_tune(\"gather\", 0)) has no aux kernel");
  if (d != 3) {   // SH: scalar and one-pixel-per-thread tensor-core kernels both have aux variants
    if (backward && (gs_sh_tc_mode(d) & 6) == 6)
      return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                              "depth / alpha gradients: the two-pixel tensor-core SH backward (sh_tc bit 2) has no aux kernel");
    return 0;
  }
  if (forward && (tn.fwd_kernel != 0 || tn.fwd_ch != 128 || tn.fwd_px != 4))
    return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                            "depth / alpha / background: only the shipped forward blend knobs (fwd_kernel 0, fwd_ch 128, fwd_px 4) have an aux kernel");
  if (backward && !shipped_rgb_bwd_knobs(tn))
    return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                            "depth / alpha gradients: only the shipped backward blend knobs have an aux kernel");
  return 0;
}

int gs_blend_absgrad_supported(int d, bool gather) {
  const GsTuning& tn = gs_tuning();
  if (d != 3)
    return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                            "densify statistics: absgrad needs the RGB blend (RGB or per-Gaussian SH colour); SH colour "
                            "evaluated per pixel has only grad2d");
  if (!gather)
    return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                            "densify statistics: absgrad is not available on the packed path (gs_tune(\"gather\", 0))");
  if (!shipped_rgb_bwd_knobs(tn))
    return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                            "densify statistics: absgrad needs the shipped backward blend knobs");
  return 0;
}

int gs_blend_batch_supported() {
  const GsTuning& tn = gs_tuning();
  if (!tn.gather)
    return gs_set_error_msg(GS_ERR_UNSUPPORTED, "batched frame: the packed path (gs_tune(\"gather\", 0)) has no batched kernel");
  if (tn.fwd_kernel != 0 || tn.fwd_ch != 128 || tn.fwd_px != 4 || !shipped_rgb_bwd_knobs(tn) || !tn.blend_repack)
    return gs_set_error_msg(GS_ERR_UNSUPPORTED,
                            "batched frame: only the shipped RGB blend knobs (with the live-pixel repack) have batched kernels");
  return 0;
}

cudaError_t gs_launch_blend_fwd_batch(const GsRec* grec, const uint32_t* ids, const int* tile_accum,
                                      const GsFrameGeom& g, const GsView* views, float* image, int* tile_neff,
                                      float* final_img, const GsCrop& crop, cudaStream_t st, const GsAuxOut* aux) {
  if (aux)
    blend_fwd_batch_kernel<true><<<g.n_tiles, 64, 0, st>>>(grec, ids, tile_accum, g.wp, g.hp, g.ntx, views, image,
                                                           tile_neff, final_img, crop, *aux);
  else
    blend_fwd_batch_kernel<false><<<g.n_tiles, 64, 0, st>>>(grec, ids, tile_accum, g.wp, g.hp, g.ntx, views, image,
                                                            tile_neff, final_img, crop, GsAuxOut{});
  return cudaGetLastError();
}

cudaError_t gs_launch_blend_bwd_batch(const GsRec* grec, const uint32_t* ids, const uint32_t* goff,
                                      const int* tile_accum, const GsFrameGeom& g, const GsView* views,
                                      const float* image, const float* grad_image, float* grad_inst, int grad_is_final,
                                      const GsCrop& crop, uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b,
                                      cudaStream_t st, const float* aux, const float* grad_aux, bool absgrad) {
  if (!row_epoch || (grad_aux && !aux)) return cudaErrorInvalidValue;
#define GS_BWD2_BATCH(AX, AB)                                                                                      \
  blend_bwd2_batch_kernel<AX, AB><<<g.n_tiles, 32, 0, st>>>(nullptr, nullptr, nullptr, grec, ids, goff, tile_accum, \
                                                            g.wp, g.hp, g.ntx, 0.f, 0.f, image, grad_image,         \
                                                            grad_inst, grad_is_final, crop, row_epoch, epoch,       \
                                                            tile_neff_b, aux, grad_aux, views)
  if (grad_aux && absgrad) GS_BWD2_BATCH(true, true);
  else if (grad_aux) GS_BWD2_BATCH(true, false);
  else if (absgrad) GS_BWD2_BATCH(false, true);
  else GS_BWD2_BATCH(false, false);
#undef GS_BWD2_BATCH
  return cudaGetLastError();
}

extern "C" size_t gs_draw_workspace_bytes(int m, int d) {
  if (d != 3 && gs_sh_basis_count(d) == 0) return 0;
  return legacy_ws_layout(m, d, nullptr, nullptr);
}

static int check_draw_args(const char* fn, int m, int d, int wp, int hp, int weight_normalize, int sigmoid,
                           size_t ws_bytes, void* ws) {
  if (m < 0 || wp <= 0 || hp <= 0 || (wp % GS_TILE) || (hp % GS_TILE))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, fn);
  if (weight_normalize || sigmoid || (d != 3 && gs_sh_basis_count(d) == 0)) return gs_set_error_msg(GS_ERR_UNSUPPORTED, fn);
  if (m > 0 && (ws == nullptr || ws_bytes < gs_draw_workspace_bytes(m, d)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, fn);
  return 0;
}

extern "C" int gs_draw_fwd(const float* pos, const float* rgb, const float* opa, const float* cov,
                           const int* tile_n_point_accum, int m, int d, int width_padded, int height_padded,
                           float focal_x, float focal_y, int weight_normalize, int sigmoid, const float* rays_o,
                           const float* lefttop, const float* vec_dx, const float* vec_dy, float* image,
                           void* workspace, size_t workspace_bytes, gs_stream_t stream) {
  int rc = check_draw_args("gs_draw_fwd: bad/unsupported arguments", m, d, width_padded, height_padded,
                           weight_normalize, sigmoid, workspace_bytes, workspace);
  if (rc) return rc;
  if (d != 3 && (!rays_o || !lefttop || !vec_dx || !vec_dy))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_draw_fwd: SH colour needs rays_o / lefttop / vec_dx / vec_dy");
  cudaStream_t st = (cudaStream_t)stream;
  LegacyWs ws{};
  legacy_ws_layout(m, d, &ws, static_cast<char*>(workspace));
  if (m > 0) {
    if (d == 3)
      legacy_pack_kernel<<<(m + 255) / 256, 256, 0, st>>>(pos, rgb, opa, cov, m, ws.pA, ws.pB, ws.pC);
    else
      legacy_pack_sh_kernel<<<(m + 255) / 256, 256, 0, st>>>(pos, rgb, opa, cov, m, d, gs_sh_stream_width(d), ws.pA,
                                                             ws.pB, reinterpret_cast<float*>(ws.pC));
    GS_CUDA_TRY(cudaGetLastError());
    gs_count_launch();
  }
  GsFrameGeom g{};
  g.wp = width_padded;
  g.hp = height_padded;
  g.ntx = width_padded / GS_TILE;
  g.nty = height_padded / GS_TILE;
  g.n_tiles = g.ntx * g.nty;
  g.fx = focal_x;
  g.fy = focal_y;
  if (d == 3) {
    GS_CUDA_TRY(gs_launch_blend_fwd(ws.pA, ws.pB, ws.pC, nullptr, nullptr, tile_n_point_accum, g, image, nullptr, nullptr,
                                    GsCrop{}, st));
  } else {
    GsRayPtrs r{rays_o, lefttop, vec_dx, vec_dy};
    GS_CUDA_TRY(gs_launch_blend_sh_fwd(ws.pA, ws.pB, reinterpret_cast<float*>(ws.pC), nullptr, nullptr, nullptr, nullptr, d,
                                       tile_n_point_accum, g, r,
                                       image, nullptr, nullptr, GsCrop{}, st));
  }
  gs_count_launch();
  return 0;
}

extern "C" int gs_draw_bwd(const float* pos, const float* rgb, const float* opa, const float* cov,
                           const int* tile_n_point_accum, int m, int d, int width_padded, int height_padded,
                           float focal_x, float focal_y, int weight_normalize, int sigmoid, const float* rays_o,
                           const float* lefttop, const float* vec_dx, const float* vec_dy, const float* image,
                           const float* grad_image, float* grad_pos, float* grad_rgb, float* grad_opa,
                           float* grad_cov, void* workspace, size_t workspace_bytes, gs_stream_t stream) {
  int rc = check_draw_args("gs_draw_bwd: bad/unsupported arguments", m, d, width_padded, height_padded,
                           weight_normalize, sigmoid, workspace_bytes, workspace);
  if (rc) return rc;
  if (m == 0) return 0;
  if (d != 3 && (!rays_o || !lefttop || !vec_dx || !vec_dy))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_draw_bwd: SH colour needs rays_o / lefttop / vec_dx / vec_dy");
  cudaStream_t st = (cudaStream_t)stream;
  LegacyWs ws{};
  legacy_ws_layout(m, d, &ws, static_cast<char*>(workspace));
  if (d == 3)
    legacy_pack_kernel<<<(m + 255) / 256, 256, 0, st>>>(pos, rgb, opa, cov, m, ws.pA, ws.pB, ws.pC);
  else
    legacy_pack_sh_kernel<<<(m + 255) / 256, 256, 0, st>>>(pos, rgb, opa, cov, m, d, gs_sh_stream_width(d), ws.pA,
                                                           ws.pB, reinterpret_cast<float*>(ws.pC));
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  GsFrameGeom g{};
  g.wp = width_padded;
  g.hp = height_padded;
  g.ntx = width_padded / GS_TILE;
  g.nty = height_padded / GS_TILE;
  g.n_tiles = g.ntx * g.nty;
  g.fx = focal_x;
  g.fy = focal_y;
  if (d == 3) {
    GS_CUDA_TRY(gs_launch_blend_bwd(ws.pA, ws.pB, ws.pC, nullptr, nullptr, nullptr, tile_n_point_accum, g, image,
                                    grad_image,
                                    ws.grad_inst, 0,
                                    GsCrop{}, nullptr, 0u, nullptr, st));
    legacy_unpack_grads_kernel<<<(m + 255) / 256, 256, 0, st>>>(ws.grad_inst, opa, cov, m, grad_pos, grad_rgb,
                                                              grad_opa, grad_cov);
  } else {
    GsRayPtrs r{rays_o, lefttop, vec_dx, vec_dy};
    GS_CUDA_TRY(gs_launch_blend_sh_bwd(ws.pA, ws.pB, reinterpret_cast<float*>(ws.pC), nullptr, nullptr, nullptr, nullptr, d,
                                       tile_n_point_accum, g, r,
                                       image, grad_image, ws.grad_inst, 0, GsCrop{}, nullptr, 0u, nullptr, st));
    legacy_unpack_grads_sh_kernel<<<(m + 255) / 256, 256, 0, st>>>(ws.grad_inst, gs_sh_grad_width(d), opa, cov, m, d,
                                                                 grad_pos, grad_rgb, grad_opa, grad_cov);
  }
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch(2);   // blend backward + unpack
  return 0;
}
