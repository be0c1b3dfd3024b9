// Feature maps on the fused frame path (gs_render_forward_feat / gs_render_backward_feat): per-Gaussian raw feature
// rows feat[N, F] (F = 8, 16, 32; no activation) blended in the same pass as the RGB image, with the image's weights
//   feature_k(p) = sum_i w_i f_i,k,      w_i = alpha_i T_i      (composited over zero; the background is the image's)
// Gather path only: the records come from rec[N] through the sorted id list (as blend.cu's gather kernels) and the
// F * 4-byte feature rows from feat[N, F] as 16-byte cp.async pieces (rows are 16-byte aligned: F % 4 == 0).
// Every thread owns a row of PX = 32 / F adjacent pixels, so PX * F = 32 feature accumulators per thread at any F.
#include <type_traits>

#include "internal.h"
#include "sh_common.cuh"

namespace {

using gs_sh::reduce8;

template <int F>
struct FeatCfg {
  static_assert(F == 8 || F == 16 || F == 32, "feature width must be 8, 16 or 32");
  static constexpr int PX = 32 / F;              // pixels per thread
  static constexpr int NT = 256 / PX;            // threads per 16x16 tile
  static constexpr int NW = NT / 32;             // warps per tile
  static constexpr int TPR = GS_TILE / PX;       // threads per pixel row
  static constexpr int FQ = F / 4;               // 16-byte pieces per feature row
  static constexpr int NV = 10 + F;              // backward sums: 6 geometry, 3 colour, d_t, F features
  static constexpr int NVP = (NV + 7) / 8 * 8;   // padded to reduce8 blocks
};

template <int F, int CH, int STAGES>
struct FeatStage {
  float4 R[STAGES][CH * 4];                      // {a, b, c, (first gradient row, -, -, -)} per instance
  float4 Fr[STAGES][CH * (F / 4)];               // feature rows
  uint64_t full[STAGES];
};

// every thread issues the copies of "its" instances of the chunk and arrives on the stage's mbarrier (count = NT)
template <int F, int NT, bool GOFF, typename SM>
__device__ __forceinline__ void feat_issue(SM& sm, int stage, const GsRec* __restrict__ grec,
                                           const float* __restrict__ feat, const uint32_t* __restrict__ ids,
                                           const uint32_t* __restrict__ goff, int base, int n, int tid) {
  for (int i = tid; i < n; i += NT) {
    const uint32_t id = __ldg(ids + base + i);
    const float4* src4 = reinterpret_cast<const float4*>(grec + id);
    const uint32_t dr = gs_smem_u32(&sm.R[stage][i * 4]);
#pragma unroll
    for (int q = 0; q < 3; ++q)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dr + 16u * q), "l"(src4 + q) : "memory");
    if (GOFF) asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dr + 48u), "l"(goff + id) : "memory");
    const float4* fs = reinterpret_cast<const float4*>(feat + (size_t)id * F);
    const uint32_t df = gs_smem_u32(&sm.Fr[stage][i * (F / 4)]);
#pragma unroll
    for (int q = 0; q < F / 4; ++q)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(df + 16u * q), "l"(fs + q) : "memory");
  }
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(gs_smem_u32(&sm.full[stage])) : "memory");
}

// one gathered instance: the record fields the blend reads (same layout as blend.cu's StageView<true>)
struct FeatRec {
  const float4* R;
  __device__ __forceinline__ float4 a(int j) const { return R[4 * j]; }
  __device__ __forceinline__ float2 b(int j) const {
    const float4 t = R[4 * j + 1];
    return make_float2(t.x, t.y);
  }
  __device__ __forceinline__ float4 c(int j) const {
    const float4 t = R[4 * j + 1];
    return make_float4(t.z, t.w, R[4 * j + 2].x, 0.f);
  }
  __device__ __forceinline__ float depth(int j) const { return R[4 * j + 2].y; }
  __device__ __forceinline__ uint32_t slot(int j, int tx, int ty) const {
    const float4 cc = R[4 * j + 2];
    const uint32_t rxy = __float_as_uint(cc.z), rwh = __float_as_uint(cc.w);
    return __float_as_uint(R[4 * j + 3].x) + ((uint32_t)ty - (rxy >> 16)) * (rwh & 0xffffu) + ((uint32_t)tx - (rxy & 0xffffu));
  }
};

template <int F>
__device__ __forceinline__ void load_feat_row(const float4* __restrict__ src, float (&f)[F]) {
#pragma unroll
  for (int q = 0; q < F / 4; ++q) {
    const float4 v = src[q];
    f[4 * q] = v.x;
    f[4 * q + 1] = v.y;
    f[4 * q + 2] = v.z;
    f[4 * q + 3] = v.w;
  }
}

// ---------------------------------------------------------------------------------------
// forward.  alpha, T, the early stop and the colour / depth sums use the arithmetic of blend.cu's gather forward
// (blend_fwd_kernel), per pixel and in the same instance order, so image, depth and alpha are bit-identical to
// gs_render_forward_aux's; the stop is a per-pixel test, so the pixel-to-thread layout does not change them.
// AUX: background T_f bg added to the image, (depth, alpha) stored, as blend.cu.
// ---------------------------------------------------------------------------------------
template <int F, bool AUX>
__global__ void __launch_bounds__(FeatCfg<F>::NT) blend_feat_fwd_kernel(
    const GsRec* __restrict__ grec, const float* __restrict__ feat, const uint32_t* __restrict__ ids,
    const int* __restrict__ tile_accum, int wp, int hp, int ntx, float fx, float fy, float* __restrict__ image,
    int* __restrict__ tile_neff, float* __restrict__ final_img, GsCrop crop, GsAuxOut aux, float* __restrict__ fmap,
    float* __restrict__ fmap_final) {
  using Cfg = FeatCfg<F>;
  constexpr int PX = Cfg::PX, NT = Cfg::NT, TPR = Cfg::TPR, CH = 64, STAGES = 2;
  __shared__ __align__(16) FeatStage<F, CH, STAGES> sm;
  const int tile = blockIdx.x, tid = threadIdx.x;
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix0 = tx * GS_TILE + (tid % TPR) * PX;
  const int iy = ty * GS_TILE + tid / TPR;
  float px[PX];
#pragma unroll
  for (int p = 0; p < PX; ++p) px[p] = gs_pixel_coord(ix0 + p, wp, fx);
  const float py = gs_pixel_coord(iy, hp, fy);
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  const int nchunks = (cnt + CH - 1) / CH;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.full[s], NT);
    gs_fence_barrier_init();
  }
  __syncthreads();
  for (int k = 0; k < STAGES && k < nchunks; ++k)
    feat_issue<F, NT, false>(sm, k, grec, feat, ids, nullptr, start + k * CH, min(CH, cnt - k * CH), tid);

  float T[PX], cr[PX], cg[PX], cb[PX], dep[PX], acc[PX][F];
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    T[p] = 1.f;
    cr[p] = cg[p] = cb[p] = 0.f;
    dep[p] = 0.f;
#pragma unroll
    for (int q = 0; q < F; ++q) acc[p][q] = 0.f;
  }
  auto all_dead = [&]() {
    bool dead = true;
#pragma unroll
    for (int p = 0; p < PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
    return dead;
  };
  int consumed = cnt, k = 0;
  for (; k < nchunks; ++k) {
    const int stage = k % STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / STAGES) & 1));
    const int n = min(CH, cnt - k * CH);
    const FeatRec sv{sm.R[stage]};
    for (int j = 0; j < n; ++j) {
      if ((j & 3) == 0 && __all_sync(0xffffffffu, all_dead())) break;
      const float4 a = sv.a(j);
      const float2 b = sv.b(j);
      const float4 c = sv.c(j);
      float f[F];
      load_feat_row<F>(&sm.Fr[stage][j * Cfg::FQ], f);
      const float dy = py - a.y;
      const float m1 = a.w * dy;
      const float ev = fmaf(-b.x * dy, dy, b.y);
      float t = 0.f;
      if constexpr (AUX) t = sv.depth(j);
#pragma unroll
      for (int p = 0; p < PX; ++p) {
        const float dx = px[p] - a.x;
        const float eu = fmaf(a.z, dx, -m1);
        const float alpha = gs_ex2(fmaf(-dx, eu, ev));
        const float w = (T[p] > GS_T_STOP) ? alpha * T[p] : 0.f;
        cr[p] = fmaf(c.x, w, cr[p]);
        cg[p] = fmaf(c.y, w, cg[p]);
        cb[p] = fmaf(c.z, w, cb[p]);
        if constexpr (AUX) dep[p] = fmaf(t, w, dep[p]);
#pragma unroll
        for (int q = 0; q < F; ++q) acc[p][q] = fmaf(f[q], w, acc[p][q]);
        T[p] -= w;
      }
    }
    if (__syncthreads_and(all_dead())) {
      consumed = min(cnt, (k + 1) * CH);
      break;
    }
    if (k + STAGES < nchunks) {   // every thread is past the barrier above: the stage is free
      const int kn = k + STAGES;
      feat_issue<F, NT, false>(sm, stage, grec, feat, ids, nullptr, start + kn * CH, min(CH, cnt - kn * CH), tid);
    }
  }
  // drain copies that were issued but never consumed (early exit) before the CTA retires
  if (tid == 0 && k < nchunks)
    for (int kk = k + 1; kk < nchunks && kk < k + STAGES; ++kk)
      gs_mbar_wait(&sm.full[kk % STAGES], (uint32_t)((kk / STAGES) & 1));
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    const int ix = ix0 + p;
    if constexpr (AUX) {
      cr[p] = fmaf(T[p], aux.bg[0], cr[p]);
      cg[p] = fmaf(T[p], aux.bg[1], cg[p]);
      cb[p] = fmaf(T[p], aux.bg[2], cb[p]);
      gs_store_aux(aux, ix, iy, wp, crop, dep[p], 1.f - T[p]);
    }
    float* o = image + ((size_t)iy * wp + ix) * 3;
    o[0] = cr[p];
    o[1] = cg[p];
    o[2] = cb[p];
    if (final_img) gs_store_final(final_img, ix, iy, crop.left, crop.top, crop.width, crop.height, cr[p], cg[p], cb[p]);
    float4* m = reinterpret_cast<float4*>(fmap + ((size_t)iy * wp + ix) * F);
#pragma unroll
    for (int q = 0; q < F / 4; ++q) m[q] = make_float4(acc[p][4 * q], acc[p][4 * q + 1], acc[p][4 * q + 2], acc[p][4 * q + 3]);
    const int x = ix - crop.left, y = iy - crop.top;
    if (fmap_final && x >= 0 && x < crop.width && y >= 0 && y < crop.height) {
      float4* mf = reinterpret_cast<float4*>(fmap_final + ((size_t)y * crop.width + x) * F);
#pragma unroll
      for (int q = 0; q < F / 4; ++q)
        mf[q] = make_float4(acc[p][4 * q], acc[p][4 * q + 1], acc[p][4 * q + 2], acc[p][4 * q + 3]);
    }
  }
  if (tile_neff && tid == 0) tile_neff[tile] = consumed;
}

// ---------------------------------------------------------------------------------------
// backward.  The RGB backward's maths (blend.cu bwd_row) with the feature terms added:
//   R(p) starts at sum_c g_c image_c (+ g_D depth + g_A alpha under AUX) + sum_k g_F,k feature_k
//   gc(p, i) = sum_c g_c c_i,c (+ g_D t_i + g_A) + sum_k g_F,k f_i,k
//   d/d f_i,k = sum_p w_p,i g_F,k(p)
// Per (thread, instance) the NV sums are reduced over each warp with reduce8 and across the NW warps through shared
// memory in a fixed order (bit-deterministic).  Row `slot` of grad_inst gets the usual GS_GREC columns (geometry,
// colour, d_t in column 9), so the projection backward runs unchanged; the F feature sums go to grad_feat_inst[slot].
// ---------------------------------------------------------------------------------------
template <int F, int CH>
struct FeatBwdSmem {
  FeatStage<F, CH, 2> st;
  float partial[FeatCfg<F>::NW][CH * FeatCfg<F>::NVP];
};

template <int F, bool AUX>
__global__ void __launch_bounds__(FeatCfg<F>::NT) blend_feat_bwd_kernel(
    const GsRec* __restrict__ grec, const float* __restrict__ feat, const uint32_t* __restrict__ ids,
    const uint32_t* __restrict__ goff, const int* __restrict__ tile_accum, int wp, int hp, int ntx, float fx, float fy,
    const float* __restrict__ image, const float* __restrict__ grad_image, const float* __restrict__ fmap,
    const float* __restrict__ grad_map, float* __restrict__ grad_inst, float* __restrict__ grad_feat_inst,
    int grad_is_final, GsCrop crop, uint32_t* __restrict__ row_epoch, uint32_t epoch, int* __restrict__ tile_neff_b,
    const float* __restrict__ aux, const float* __restrict__ grad_aux) {
  using Cfg = FeatCfg<F>;
  constexpr int PX = Cfg::PX, NT = Cfg::NT, NW = Cfg::NW, TPR = Cfg::TPR, NVP = Cfg::NVP, CH = 16, STAGES = 2;
  __shared__ __align__(16) FeatBwdSmem<F, CH> smem;
  auto& sm = smem.st;
  const int tile = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = tile % ntx, ty = tile / ntx;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int nchunks = (cnt + CH - 1) / CH;
  const int ix0 = tx * GS_TILE + (tid % TPR) * PX;
  const int iy = ty * GS_TILE + tid / TPR;
  float px[PX];
#pragma unroll
  for (int p = 0; p < PX; ++p) px[p] = gs_pixel_coord(ix0 + p, wp, fx);
  const float py = gs_pixel_coord(iy, hp, fy);
  float T[PX], R[PX], gr[PX], gg[PX], gb[PX], gF[PX][F];
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    const int ix = ix0 + p;
    const float* im = image + ((size_t)iy * wp + ix) * 3;
    const float i3[3] = {im[0], im[1], im[2]};
    if (!grad_is_final) {
      const float* gi = grad_image + ((size_t)iy * wp + ix) * 3;
      gr[p] = gi[0];
      gg[p] = gi[1];
      gb[p] = gi[2];
    } else {
      gs_load_final_grad(grad_image, i3, ix, iy, crop.left, crop.top, crop.width, crop.height, gr[p], gg[p], gb[p]);
    }
    R[p] = gr[p] * i3[0] + gg[p] * i3[1] + gb[p] * i3[2];
    T[p] = 1.f;
    // feature gradient: padded [Hp,Wp,F], or the crop [h,w,F] (features are not clamped: only the crop masks it)
    const float4* gsrc = nullptr;
    if (!grad_is_final) {
      gsrc = reinterpret_cast<const float4*>(grad_map + ((size_t)iy * wp + ix) * F);
    } else {
      const int x = ix - crop.left, y = iy - crop.top;
      if (x >= 0 && x < crop.width && y >= 0 && y < crop.height)
        gsrc = reinterpret_cast<const float4*>(grad_map + ((size_t)y * crop.width + x) * F);
    }
    const float4* msrc = reinterpret_cast<const float4*>(fmap + ((size_t)iy * wp + ix) * F);
#pragma unroll
    for (int q = 0; q < F / 4; ++q) {
      const float4 g4 = gsrc ? gsrc[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 m4 = msrc[q];
      gF[p][4 * q] = g4.x;
      gF[p][4 * q + 1] = g4.y;
      gF[p][4 * q + 2] = g4.z;
      gF[p][4 * q + 3] = g4.w;
      R[p] = fmaf(g4.x, m4.x, fmaf(g4.y, m4.y, fmaf(g4.z, m4.z, fmaf(g4.w, m4.w, R[p]))));
    }
  }
  float gD[PX], gA[PX];
  if constexpr (AUX) gs_load_aux_grad<PX>(aux, grad_aux, grad_is_final, ix0, iy, wp, crop, gD, gA, R);
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.full[s], NT);
    gs_fence_barrier_init();
  }
  __syncthreads();
  for (int k = 0; k < STAGES && k < nchunks; ++k)
    feat_issue<F, NT, true>(sm, k, grec, feat, ids, goff, start + k * CH, min(CH, cnt - k * CH), tid);
  auto all_dead = [&]() {
    bool dead = true;
#pragma unroll
    for (int p = 0; p < PX; ++p) dead = dead && !(T[p] > GS_T_STOP);
    return dead;
  };

  int consumed = cnt, k = 0;
  for (; k < nchunks; ++k) {
    const int stage = k % STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / STAGES) & 1));
    const int n = min(CH, cnt - k * CH);
    const FeatRec sv{sm.R[stage]};
    float* __restrict__ part = smem.partial[warp];
    int j = 0;
    for (; j < n; ++j) {
      if (__all_sync(0xffffffffu, all_dead())) break;
      const float4 a = sv.a(j);
      const float2 b = sv.b(j);
      const float4 c = sv.c(j);
      float f[F];
      load_feat_row<F>(&sm.Fr[stage][j * Cfg::FQ], f);
      float acc[NVP];
#pragma unroll
      for (int u = 0; u < NVP; ++u) acc[u] = 0.f;
      float s0 = 0.f, sx = 0.f, sxx = 0.f;
      const float dy = py - a.y;
      const float m1 = a.w * dy;
      const float ev = fmaf(-b.x * dy, dy, b.y);
      float t = 0.f;
      if constexpr (AUX) t = sv.depth(j);
#pragma unroll
      for (int p = 0; p < PX; ++p) {
        const float dx = px[p] - a.x;
        const float eu = fmaf(a.z, dx, -m1);
        const float alpha = gs_ex2(fmaf(-dx, eu, ev));
        if (T[p] > GS_T_STOP) {          // saturated pixels contribute exactly nothing
          const float w = alpha * T[p];
          float gc = fmaf(gr[p], c.x, fmaf(gg[p], c.y, gb[p] * c.z));
#pragma unroll
          for (int q = 0; q < F; ++q) gc = fmaf(gF[p][q], f[q], gc);
          if constexpr (AUX) gc = fmaf(gD[p], t, gc + gA[p]);
          R[p] = fmaf(-gc, w, R[p]);
          const float rc = gs_rcp(1.0000001f - alpha);
          const float dal = fmaf(T[p], gc, -R[p] * rc);
          const float e = dal * alpha;
          T[p] -= w;
          const float ex = e * dx;
          s0 += e;
          sx += ex;
          sxx = fmaf(ex, dx, sxx);
          acc[6] = fmaf(gr[p], w, acc[6]);
          acc[7] = fmaf(gg[p], w, acc[7]);
          acc[8] = fmaf(gb[p], w, acc[8]);
          if constexpr (AUX) acc[9] = fmaf(gD[p], w, acc[9]);
#pragma unroll
          for (int q = 0; q < F; ++q) acc[10 + q] = fmaf(gF[p][q], w, acc[10 + q]);
        }
      }
      acc[0] = sx;
      acc[1] = dy * s0;
      acc[2] = sxx;
      acc[3] = dy * sx;
      acc[4] = dy * acc[1];
      acc[5] = s0;
#pragma unroll
      for (int blk = 0; blk < NVP / 8; ++blk) {
        const float r = reduce8(acc + blk * 8, lane);
        if ((lane & 3) == 0) part[j * NVP + blk * 8 + ((lane >> 2) & 7)] = r;
      }
    }
    for (int z = j * NVP + lane; z < n * NVP; z += 32) part[z] = 0.f;   // this warp stopped early: zero sums
    __syncthreads();
    for (int i = tid; i < n; i += NT) {
      float s[10];
#pragma unroll
      for (int u = 0; u < 10; ++u) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) v += smem.partial[w][i * NVP + u];
        s[u] = v;
      }
      const float4 a = sv.a(i);
      const float2 b = sv.b(i);
      const uint32_t slot = sv.slot(i, tx, ty);
      float4* out = reinterpret_cast<float4*>(grad_inst + (size_t)slot * GS_GREC);
      out[0] = make_float4(GS_LN2 * (2.f * a.z * s[0] - a.w * s[1]), GS_LN2 * (2.f * b.x * s[1] - a.w * s[0]),
                           -GS_LN2 * s[2], GS_LN2 * s[3]);
      out[1] = make_float4(-GS_LN2 * s[4], GS_LN2 * s[5], s[6], s[7]);
      out[2] = make_float4(s[8], s[9], 0.f, 0.f);
      row_epoch[slot] = epoch;
    }
    for (int z = tid; z < n * F; z += NT) {
      const int i = z / F, q = z % F;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) v += smem.partial[w][i * NVP + 10 + q];
      grad_feat_inst[(size_t)sv.slot(i, tx, ty) * F + q] = v;
    }
    if (__syncthreads_and(all_dead())) {   // also: every thread is done with the partial buffer and the stage
      consumed = min(cnt, (k + 1) * CH);
      break;
    }
    if (k + STAGES < nchunks) {
      const int kn = k + STAGES;
      feat_issue<F, NT, true>(sm, stage, grec, feat, ids, goff, start + kn * CH, min(CH, cnt - kn * CH), tid);
    }
  }
  if (tid == 0 && k < nchunks)
    for (int kk = k + 1; kk < nchunks && kk < k + STAGES; ++kk)
      gs_mbar_wait(&sm.full[kk % STAGES], (uint32_t)((kk / STAGES) & 1));
  if (tile_neff_b && tid == 0) tile_neff_b[tile] = consumed;
}

// ---------------------------------------------------------------------------------------
// segment sum after the projection backward: grad_feat[i, :] = sum of Gaussian i's rows of grad_feat_inst tagged with
// this backward's epoch, in row order (bit-deterministic, no atomics); zeros for a Gaussian with no consumed row.
// One thread per (Gaussian, 16-byte piece of its row).
// ---------------------------------------------------------------------------------------
constexpr int kSegBlock = 256;

template <int F>
__global__ void __launch_bounds__(kSegBlock) feat_grad_kernel(const uint32_t* __restrict__ offsets_g,
                                                              const uint32_t* __restrict__ count,
                                                              const float* __restrict__ grad_feat_inst,
                                                              const uint32_t* __restrict__ row_epoch, uint32_t epoch,
                                                              int n, float* __restrict__ grad_feat) {
  constexpr int FQ = F / 4;
  const long long t = (long long)blockIdx.x * kSegBlock + threadIdx.x;
  if (t >= (long long)n * FQ) return;
  const int i = (int)(t / FQ), q = (int)(t % FQ);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  const uint32_t o0 = offsets_g[i], o1 = o0 + count[i];
  for (uint32_t r = o0; r < o1; ++r) {
    if (row_epoch[r] != epoch) continue;   // not reached by its (saturated) tile: zero gradient
    const float4 v = reinterpret_cast<const float4*>(grad_feat_inst + (size_t)r * F)[q];
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  float* o = grad_feat + (size_t)i * F + 4 * q;   // grad_feat need not be 16-byte aligned
  o[0] = s.x;
  o[1] = s.y;
  o[2] = s.z;
  o[3] = s.w;
}

}  // namespace

bool gs_feat_width_ok(int f) { return f == 8 || f == 16 || f == 32; }

cudaError_t gs_launch_blend_feat_fwd(const GsRec* grec, const float* feat, int f, const uint32_t* ids,
                                     const int* tile_accum, const GsFrameGeom& g, float* image, int* tile_neff,
                                     float* final_img, const GsCrop& crop, const GsAuxOut* aux, float* map,
                                     float* map_final, cudaStream_t st) {
#define GS_FEATF(F, AX)                                                                                            \
  blend_feat_fwd_kernel<F, AX><<<g.n_tiles, FeatCfg<F>::NT, 0, st>>>(grec, feat, ids, tile_accum, g.wp, g.hp,   \
                                                                      g.ntx, g.fx, g.fy, image, tile_neff,        \
                                                                      final_img, crop, aux ? *aux : GsAuxOut{},   \
                                                                      map, map_final)
#define GS_FEATF_A(F) \
  if (aux) GS_FEATF(F, true); else GS_FEATF(F, false);
  switch (f) {
    case 8: GS_FEATF_A(8) break;
    case 16: GS_FEATF_A(16) break;
    case 32: GS_FEATF_A(32) break;
    default: return cudaErrorInvalidValue;
  }
#undef GS_FEATF_A
#undef GS_FEATF
  return cudaGetLastError();
}

cudaError_t gs_launch_blend_feat_bwd(const GsRec* grec, const float* feat, int f, const uint32_t* ids,
                                     const uint32_t* goff, const int* tile_accum, const GsFrameGeom& g,
                                     const float* image, const float* grad_image, const float* map,
                                     const float* grad_map, float* grad_inst, float* grad_feat_inst, int grad_is_final,
                                     const GsCrop& crop, uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b,
                                     const float* aux, const float* grad_aux, cudaStream_t st) {
  if (grad_aux && !aux) return cudaErrorInvalidValue;
#define GS_FEATB(F, AX)                                                                                            \
  blend_feat_bwd_kernel<F, AX><<<g.n_tiles, FeatCfg<F>::NT, 0, st>>>(                                             \
      grec, feat, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, image, grad_image, map, grad_map,          \
      grad_inst, grad_feat_inst, grad_is_final, crop, row_epoch, epoch, tile_neff_b, aux, grad_aux)
#define GS_FEATB_A(F) \
  if (grad_aux) GS_FEATB(F, true); else GS_FEATB(F, false);
  switch (f) {
    case 8: GS_FEATB_A(8) break;
    case 16: GS_FEATB_A(16) break;
    case 32: GS_FEATB_A(32) break;
    default: return cudaErrorInvalidValue;
  }
#undef GS_FEATB_A
#undef GS_FEATB
  return cudaGetLastError();
}

cudaError_t gs_launch_feat_grad(const uint32_t* offsets_g, const uint32_t* count, const float* grad_feat_inst,
                                const uint32_t* row_epoch, uint32_t epoch, int n, int f, float* grad_feat,
                                cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const long long threads = (long long)n * (f / 4);
  const int blocks = (int)((threads + kSegBlock - 1) / kSegBlock);
#define GS_FEATG(F) \
  feat_grad_kernel<F><<<blocks, kSegBlock, 0, st>>>(offsets_g, count, grad_feat_inst, row_epoch, epoch, n, grad_feat)
  switch (f) {
    case 8: GS_FEATG(8); break;
    case 16: GS_FEATG(16); break;
    case 32: GS_FEATG(32); break;
    default: return cudaErrorInvalidValue;
  }
#undef GS_FEATG
  return cudaGetLastError();
}
