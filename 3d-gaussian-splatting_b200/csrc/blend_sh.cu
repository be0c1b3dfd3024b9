// Tile blend with per-pixel spherical-harmonics colour (reference `use_sh_coeff`,
// gaussian.cu:849-861 ray setup, :405-426 basis, :936-948 forward colour, :665-689 backward).
//
// The reference evaluates SH PER PIXEL RAY inside the blend: colour_c(pixel, instance) =
// sigmoid(sum_k SH_k(dir_pixel) * coef[c*K + k]) with K = 9 (degree 2, D = 27).  K = 16
// (degree 3, D = 48; svox2's C3 constants, defined but unused in the reference :395-403) is the
// extension (bench.py --colour 48).  Same staging / early-exit / reduction design
// as blend.cu; the third stream carries the 3K coefficients + the gradient slot per instance.
#include <type_traits>

#include "internal.h"
#include "sh_common.cuh"

namespace {

using namespace gs_sh;

template <int K, int CH, int STAGES>
struct ShStage {
  float4 A[STAGES][CH];
  float2 B[STAGES][CH + 2];
  float S[STAGES][CH * sh_sw(K)];
  uint64_t full[STAGES];
};

template <int K, typename SM>
__device__ __forceinline__ void issue_sh(SM& sm, int stage, const float4* __restrict__ pA,
                                         const float2* __restrict__ pB, const float* __restrict__ pS, int base,
                                         int n, int shift) {
  const uint32_t bytes_a = (uint32_t)n * 16u;
  const uint32_t bytes_s = (uint32_t)n * (uint32_t)(sh_sw(K) * 4);
  const uint32_t nb = (uint32_t)(n + shift + 1) & ~1u;
  const uint32_t bytes_b = nb * 8u;
  gs_mbar_expect_tx(&sm.full[stage], bytes_a + bytes_s + bytes_b);
  gs_bulk_g2s(sm.A[stage], pA + base, bytes_a, &sm.full[stage]);
  gs_bulk_g2s(sm.S[stage], pS + (size_t)base * sh_sw(K), bytes_s, &sm.full[stage]);
  gs_bulk_g2s(sm.B[stage], pB + (base - shift), bytes_b, &sm.full[stage]);
}

// Gather staging (no pack pass): per instance the Gaussian's 64-byte record (centre, conic, log2 opacity, tile
// rectangle, first gradient row) comes straight from GsRec rec[N] and its 3K raw coefficients straight from the
// parameter tensor rgb[N, 3K], as cp.async pieces (16 B; 4 B for the 108-byte rows of K = 9, which are only
// 4-byte aligned).  Every thread of the CTA issues the copies of "its" instances of the chunk and arrives on the
// stage's mbarrier (count = CTA threads) when they have landed (cp.async.mbarrier.arrive.noinc).
template <int K, int CH, int STAGES>
struct ShGatherStage {
  float4 R[STAGES][CH * 4];
  float S[STAGES][CH * sh_sw(K)];
  uint64_t full[STAGES];
};

template <int K, int NT, typename SM>
__device__ __forceinline__ void issue_sh_gather(SM& sm, int stage, const GsRec* __restrict__ grec,
                                                const float* __restrict__ rgb, const uint32_t* __restrict__ ids,
                                                const uint32_t* __restrict__ goff, int base, int n, int tid) {
  constexpr int SW = sh_sw(K), D = 3 * K;
  for (int i = tid; i < n; i += NT) {
    const uint32_t id = ids[base + i];
    const float4* src4 = reinterpret_cast<const float4*>(grec + id);
    const uint32_t dr = gs_smem_u32(&sm.R[stage][i * 4]);
#pragma unroll
    for (int q = 0; q < 3; ++q)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dr + 16u * q), "l"(src4 + q) : "memory");
    // first gradient row of the Gaussian (offsets_g[id]) into the record's 4th piece
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dr + 48u), "l"(goff + id) : "memory");
    const float* src = rgb + (size_t)id * D;
    const uint32_t ds = gs_smem_u32(&sm.S[stage][i * SW]);
    if ((D * 4) % 16 == 0) {        // K = 16: rows of 192 B are 16-byte aligned
#pragma unroll
      for (int q = 0; q < D / 4; ++q)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ds + 16u * q), "l"(src + 4 * q) : "memory");
    } else {                        // K = 9: rows of 108 B are only 4-byte aligned
#pragma unroll
      for (int q = 0; q < D; ++q)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ds + 4u * q), "l"(src + q) : "memory");
    }
  }
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(gs_smem_u32(&sm.full[stage])) : "memory");
}

// view of one stage: packed streams (pack pass / legacy draw API) or gathered records
template <int K, bool GATHER>
struct ShView;
template <int K>
struct ShView<K, false> {
  const float4* A;
  const float2* B;
  const float* S;
  __device__ __forceinline__ float4 a(int j) const { return A[j]; }
  __device__ __forceinline__ float2 b(int j) const { return B[j]; }
  __device__ __forceinline__ const float* coef(int j) const { return S + j * sh_sw(K); }
  __device__ __forceinline__ uint32_t slot(int j, int, int) const { return __float_as_uint(S[j * sh_sw(K) + 3 * K]); }
};
template <int K>
struct ShView<K, true> {
  const float4* R;
  const float* S;
  __device__ __forceinline__ float4 a(int j) const { return R[4 * j]; }
  __device__ __forceinline__ float2 b(int j) const {
    const float4 t = R[4 * j + 1];
    return make_float2(t.x, t.y);
  }
  __device__ __forceinline__ const float* coef(int j) const { return S + j * sh_sw(K); }
  __device__ __forceinline__ float depth(int j) const { return R[4 * j + 2].y; }   // |p_c|
  __device__ __forceinline__ uint32_t slot(int j, int tx, int ty) const {
    const float4 cc = R[4 * j + 2];
    const uint32_t rxy = __float_as_uint(cc.z), rwh = __float_as_uint(cc.w);
    return __float_as_uint(R[4 * j + 3].x) + ((uint32_t)ty - (rxy >> 16)) * (rwh & 0xffffu) + ((uint32_t)tx - (rxy & 0xffffu));
  }
};

// ---------------------------------------------------------------------------------------
// forward: 64 threads per tile, a row of 4 pixels per thread
// AUX (gather only): depth sum w t per pixel, T_f bg added, (depth, alpha) stored as in blend.cu
// ---------------------------------------------------------------------------------------
template <int K, bool GATHER, bool AUX = false>
__global__ void __launch_bounds__(64) blend_sh_fwd_kernel(const float4* __restrict__ pA, const float2* __restrict__ pB,
                                                           const float* __restrict__ pS,
                                                           const GsRec* __restrict__ grec, const float* __restrict__ rgb,
                                                           const uint32_t* __restrict__ ids,
                                                           const uint32_t* __restrict__ goff,
                                                           const int* __restrict__ tile_accum, int wp, int hp, int ntx,
                                                           float fx, float fy, const float* __restrict__ rays_o,
                                                           const float* __restrict__ lefttop,
                                                           const float* __restrict__ vdx,
                                                           const float* __restrict__ vdy, float* __restrict__ image,
                                                           int* __restrict__ tile_neff,
                                                           float* __restrict__ final_img, GsCrop crop, GsAuxOut aux) {
  constexpr int CH = 64, STAGES = 2, PX = 4, SW = sh_sw(K), NT = 64;
  static_assert(!AUX || GATHER, "the aux outputs read |p_c| from the gathered records");
  using SM = typename std::conditional<GATHER, ShGatherStage<K, CH, STAGES>, ShStage<K, CH, STAGES>>::type;
  __shared__ __align__(16) SM sm;
  const int tile = blockIdx.x, tid = threadIdx.x;
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix0 = tx * GS_TILE + (tid & 3) * PX;
  const int iy = ty * GS_TILE + (tid >> 2);
  float px[PX], sh[PX][K];
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    px[p] = gs_pixel_coord(ix0 + p, wp, fx);
    pixel_sh<K>(ix0 + p, iy, rays_o, lefttop, vdx, vdy, sh[p]);
  }
  const float py = gs_pixel_coord(iy, hp, fy);
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  const int shift = start & 1;
  const int nchunks = (cnt + CH - 1) / CH;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.full[s], GATHER ? NT : 1);
    gs_fence_barrier_init();
  }
  __syncthreads();
  if constexpr (GATHER) {
    for (int k = 0; k < STAGES && k < nchunks; ++k)
      issue_sh_gather<K, NT>(sm, k, grec, rgb, ids, goff, start + k * CH, min(CH, cnt - k * CH), tid);
  } else if (tid == 0) {
    for (int k = 0; k < STAGES && k < nchunks; ++k)
      issue_sh<K>(sm, k, pA, pB, pS, start + k * CH, min(CH, cnt - k * CH), shift);
  }

  float T[PX], cr[PX], cg[PX], cb[PX], dep[PX];
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    T[p] = 1.f;
    cr[p] = cg[p] = cb[p] = 0.f;
    dep[p] = 0.f;
  }
  int consumed = cnt, k = 0;
  for (; k < nchunks; ++k) {
    const int stage = k % STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / STAGES) & 1));
    const int n = min(CH, cnt - k * CH);
    ShView<K, GATHER> sv;
    if constexpr (GATHER) {
      sv.R = sm.R[stage];
    } else {
      sv.A = sm.A[stage];
      sv.B = sm.B[stage] + shift;
    }
    sv.S = sm.S[stage];
    for (int j = 0; j < n; ++j) {
      if ((j & 3) == 0) {
        const bool dead = !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP) && !(T[2] > GS_T_STOP) && !(T[3] > GS_T_STOP);
        if (__all_sync(0xffffffffu, dead)) break;
      }
      const float4 a = sv.a(j);
      const float2 b = sv.b(j);
      float cf[3 * K];
      {
        const float4* c4 = reinterpret_cast<const float4*>(sv.coef(j));
#pragma unroll
        for (int q = 0; q < (3 * K + 3) / 4; ++q) {
          const float4 t4 = c4[q];
          if (4 * q < 3 * K) cf[4 * q] = t4.x;
          if (4 * q + 1 < 3 * K) cf[4 * q + 1] = t4.y;
          if (4 * q + 2 < 3 * K) cf[4 * q + 2] = t4.z;
          if (4 * q + 3 < 3 * K) cf[4 * q + 3] = t4.w;
        }
      }
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
        if (T[p] > GS_T_STOP) {          // a saturated pixel blends nothing: skip its 3K FMAs + 3 sigmoids
          const float w = alpha * T[p];
          float col[3];
          {
            // three sigmoids with ONE reciprocal: the forward is MUFU-bound (7 MUFU per (pixel, instance): ex2 of
            // the blend + 3 x (ex2 + rcp)); 1 / d_c = (prod d) ^-1 * (product of the other two).  d = 1 + 2^(-x log2e)
            // is clamped to <= 2^40 so that the product cannot overflow (sigmoid < 1e-12 there).
            float dsum[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              float acc = 0.f;
#pragma unroll
              for (int q = 0; q < K; ++q) acc = fmaf(sh[p][q], cf[c * K + q], acc);
              dsum[c] = 1.f + gs_ex2(fminf(-acc * GS_LOG2E, 40.f));
            }
            const float d01 = dsum[0] * dsum[1];
            const float r = gs_rcp(d01 * dsum[2]);
            col[2] = r * d01;
            const float r2 = r * dsum[2];
            col[0] = r2 * dsum[1];
            col[1] = r2 * dsum[0];
          }
          cr[p] = fmaf(col[0], w, cr[p]);
          cg[p] = fmaf(col[1], w, cg[p]);
          cb[p] = fmaf(col[2], w, cb[p]);
          if constexpr (AUX) dep[p] = fmaf(t, w, dep[p]);
          T[p] -= w;
        }
      }
    }
    const bool dead = !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP) && !(T[2] > GS_T_STOP) && !(T[3] > GS_T_STOP);
    if (__syncthreads_and(dead)) {
      consumed = min(cnt, (k + 1) * CH);
      break;
    }
    if (k + STAGES < nchunks) {
      const int kn = k + STAGES;
      if constexpr (GATHER)
        issue_sh_gather<K, NT>(sm, stage, grec, rgb, ids, goff, start + kn * CH, min(CH, cnt - kn * CH), tid);
      else if (tid == 0)
        issue_sh<K>(sm, stage, pA, pB, pS, start + kn * CH, min(CH, cnt - kn * CH), shift);
    }
  }
  if (tid == 0 && k < nchunks)
    for (int kk = k + 1; kk < nchunks && kk < k + STAGES; ++kk)
      gs_mbar_wait(&sm.full[kk % STAGES], (uint32_t)((kk / STAGES) & 1));
  if constexpr (AUX) {
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      cr[p] = fmaf(T[p], aux.bg[0], cr[p]);
      cg[p] = fmaf(T[p], aux.bg[1], cg[p]);
      cb[p] = fmaf(T[p], aux.bg[2], cb[p]);
      gs_store_aux(aux, ix0 + p, iy, wp, crop, dep[p], 1.f - T[p]);
    }
  }
  float4* o = reinterpret_cast<float4*>(image + ((size_t)iy * wp + ix0) * 3);
  o[0] = make_float4(cr[0], cg[0], cb[0], cr[1]);
  o[1] = make_float4(cg[1], cb[1], cr[2], cg[2]);
  o[2] = make_float4(cb[2], cr[3], cg[3], cb[3]);
  if (final_img) {
#pragma unroll
    for (int p = 0; p < PX; ++p)
      gs_store_final(final_img, ix0 + p, iy, crop.left, crop.top, crop.width, crop.height, cr[p], cg[p], cb[p]);
  }
  if (tile_neff && tid == 0) tile_neff[tile] = consumed;
}

// ---------------------------------------------------------------------------------------
// backward: 64 threads per tile, a row of 4 pixels per thread
// grad row (GS_SH_GREC(K) floats): d/d{x, y, ca, cb, cc, l2o}, d/d coef[0..3K)
// ---------------------------------------------------------------------------------------
template <int K, bool GATHER>
struct ShBwdSmem {
  typename std::conditional<GATHER, ShGatherStage<K, 32, 2>, ShStage<K, 32, 2>>::type st;
  float partial[2][32 * sh_nvp(K)];
};

// AUX (gather only): gc += g_D t + g_A, R += g_D depth + g_A alpha, and d_t = sum g_D w is reduced in value slot NV
// (the first pad value of the NVP-wide partial row) into column 6 + 3K of the gradient row.
template <int K, bool GATHER, bool AUX = false>
__global__ void __launch_bounds__(64) blend_sh_bwd_kernel(const float4* __restrict__ pA, const float2* __restrict__ pB,
                                                           const float* __restrict__ pS,
                                                           const GsRec* __restrict__ grec, const float* __restrict__ rgb,
                                                           const uint32_t* __restrict__ ids,
                                                           const uint32_t* __restrict__ goff,
                                                           const int* __restrict__ tile_accum, int wp, int hp, int ntx,
                                                           float fx, float fy, const float* __restrict__ rays_o,
                                                           const float* __restrict__ lefttop,
                                                           const float* __restrict__ vdx,
                                                           const float* __restrict__ vdy,
                                                           const float* __restrict__ image,
                                                           const float* __restrict__ grad_image,
                                                           float* __restrict__ grad_inst, int grad_is_final,
                                                           GsCrop crop, uint32_t* __restrict__ row_epoch,
                                                           uint32_t epoch, int* __restrict__ tile_neff_b,
                                                           const float* __restrict__ aux,
                                                           const float* __restrict__ grad_aux) {
  constexpr int CH = 32, STAGES = 2, PX = 4, SW = sh_sw(K), NV = sh_nv(K), NVP = sh_nvp(K), THREADS = 64;
  constexpr int GREC = (NV + 3) / 4 * 4;
  static_assert(!AUX || (GATHER && NV < NVP && NV < GREC), "d_t needs a pad slot in the partial and gradient rows");
  __shared__ __align__(16) ShBwdSmem<K, GATHER> smem;
  auto& sm = smem.st;
  const int tile = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = tile % ntx, ty = tile / ntx;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int shift = start & 1;
  const int nchunks = (cnt + CH - 1) / CH;
  const int ix0 = tx * GS_TILE + (tid & 3) * PX;
  const int iy = ty * GS_TILE + (tid >> 2);
  float px[PX], sh[PX][K];
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    px[p] = gs_pixel_coord(ix0 + p, wp, fx);
    pixel_sh<K>(ix0 + p, iy, rays_o, lefttop, vdx, vdy, sh[p]);
  }
  const float py = gs_pixel_coord(iy, hp, fy);
  float T[PX], R[PX], gr[PX], gg[PX], gb[PX];
  {
    const size_t off = ((size_t)iy * wp + ix0) * 3;
    const float4* im = reinterpret_cast<const float4*>(image + off);
    const float4 i0 = im[0], i1 = im[1], i2 = im[2];
    if (!grad_is_final) {
      const float4* gi = reinterpret_cast<const float4*>(grad_image + off);
      const float4 g0 = gi[0], g1 = gi[1], g2 = gi[2];
      gr[0] = g0.x; gg[0] = g0.y; gb[0] = g0.z; gr[1] = g0.w;
      gg[1] = g1.x; gb[1] = g1.y; gr[2] = g1.z; gg[2] = g1.w;
      gb[2] = g2.x; gr[3] = g2.y; gg[3] = g2.z; gb[3] = g2.w;
    } else {
      const float raw[12] = {i0.x, i0.y, i0.z, i0.w, i1.x, i1.y, i1.z, i1.w, i2.x, i2.y, i2.z, i2.w};
#pragma unroll
      for (int p = 0; p < PX; ++p)
        gs_load_final_grad(grad_image, raw + 3 * p, ix0 + p, iy, crop.left, crop.top, crop.width, crop.height, gr[p],
                           gg[p], gb[p]);
    }
    R[0] = gr[0] * i0.x + gg[0] * i0.y + gb[0] * i0.z;
    R[1] = gr[1] * i0.w + gg[1] * i1.x + gb[1] * i1.y;
    R[2] = gr[2] * i1.z + gg[2] * i1.w + gb[2] * i2.x;
    R[3] = gr[3] * i2.y + gg[3] * i2.z + gb[3] * i2.w;
#pragma unroll
    for (int p = 0; p < PX; ++p) T[p] = 1.f;
  }
  float gD[PX], gA[PX];
  if constexpr (AUX) gs_load_aux_grad<PX>(aux, grad_aux, grad_is_final, ix0, iy, wp, crop, gD, gA, R);
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.full[s], GATHER ? THREADS : 1);
    gs_fence_barrier_init();
  }
  __syncthreads();
  if constexpr (GATHER) {
    for (int k = 0; k < STAGES && k < nchunks; ++k)
      issue_sh_gather<K, THREADS>(sm, k, grec, rgb, ids, goff, start + k * CH, min(CH, cnt - k * CH), tid);
  } else if (tid == 0) {
    for (int k = 0; k < STAGES && k < nchunks; ++k)
      issue_sh<K>(sm, k, pA, pB, pS, start + k * CH, min(CH, cnt - k * CH), shift);
  }

  int consumed = cnt, k = 0;
  for (; k < nchunks; ++k) {
    const int stage = k % STAGES;
    gs_mbar_wait(&sm.full[stage], (uint32_t)((k / STAGES) & 1));
    const int n = min(CH, cnt - k * CH);
    ShView<K, GATHER> sv;
    if constexpr (GATHER) {
      sv.R = sm.R[stage];
    } else {
      sv.A = sm.A[stage];
      sv.B = sm.B[stage] + shift;
    }
    sv.S = sm.S[stage];
    float* __restrict__ part = smem.partial[warp];
    int j = 0;
    for (; j < n; ++j) {
      {
        const bool dead = !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP) && !(T[2] > GS_T_STOP) && !(T[3] > GS_T_STOP);
        if (__all_sync(0xffffffffu, dead)) break;
      }
      const float4 a = sv.a(j);
      const float2 b = sv.b(j);
      float cf[3 * K];
      {
        const float4* c4 = reinterpret_cast<const float4*>(sv.coef(j));
#pragma unroll
        for (int q = 0; q < (3 * K + 3) / 4; ++q) {
          const float4 t4 = c4[q];
          if (4 * q < 3 * K) cf[4 * q] = t4.x;
          if (4 * q + 1 < 3 * K) cf[4 * q + 1] = t4.y;
          if (4 * q + 2 < 3 * K) cf[4 * q + 2] = t4.z;
          if (4 * q + 3 < 3 * K) cf[4 * q + 3] = t4.w;
        }
      }
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
          float col[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            float t = 0.f;
#pragma unroll
            for (int q = 0; q < K; ++q) t = fmaf(sh[p][q], cf[c * K + q], t);
            col[c] = sh_sigmoid(t);
          }
          float gc = fmaf(gr[p], col[0], fmaf(gg[p], col[1], gb[p] * col[2]));
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
          if constexpr (AUX) acc[NV] = fmaf(gD[p], w, acc[NV]);
          // d colour_c / d coef[c*K+q] = sigma'(.) * SH_q      (gaussian.cu:666-674)
          const float d0 = gr[p] * w * col[0] * (1.f - col[0]);
          const float d1 = gg[p] * w * col[1] * (1.f - col[1]);
          const float d2 = gb[p] * w * col[2] * (1.f - col[2]);
#pragma unroll
          for (int q = 0; q < K; ++q) {
            acc[6 + q] = fmaf(d0, sh[p][q], acc[6 + q]);
            acc[6 + K + q] = fmaf(d1, sh[p][q], acc[6 + K + q]);
            acc[6 + 2 * K + q] = fmaf(d2, sh[p][q], acc[6 + 2 * K + q]);
          }
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
    for (int z = j * NVP + lane; z < n * NVP; z += 32) part[z] = 0.f;
    __syncthreads();
    for (int t = tid; t < n; t += THREADS) {
      const float* p0 = smem.partial[0] + t * NVP;
      const float* p1 = smem.partial[1] + t * NVP;
      const float4 a = sv.a(t);
      const float2 b = sv.b(t);
      const uint32_t slot = sv.slot(t, tx, ty);
      float* out = grad_inst + (size_t)slot * GREC;
      float s[6];
#pragma unroll
      for (int u = 0; u < 6; ++u) s[u] = p0[u] + p1[u];
      out[0] = GS_LN2 * (2.f * a.z * s[0] - a.w * s[1]);
      out[1] = GS_LN2 * (2.f * b.x * s[1] - a.w * s[0]);
      out[2] = -GS_LN2 * s[2];
      out[3] = GS_LN2 * s[3];
      out[4] = -GS_LN2 * s[4];
      out[5] = GS_LN2 * s[5];
      for (int u = 6; u < NV; ++u) out[u] = p0[u] + p1[u];
      if constexpr (AUX) out[NV] = p0[NV] + p1[NV];   // d/dt, column 6 + 3K
      if (row_epoch) row_epoch[slot] = epoch;
    }
    const bool dead = !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP) && !(T[2] > GS_T_STOP) && !(T[3] > GS_T_STOP);
    if (__syncthreads_and(dead)) {
      consumed = min(cnt, (k + 1) * CH);
      break;
    }
    if (k + STAGES < nchunks) {
      const int kn = k + STAGES;
      if constexpr (GATHER)
        issue_sh_gather<K, THREADS>(sm, stage, grec, rgb, ids, goff, start + kn * CH, min(CH, cnt - kn * CH), tid);
      else if (tid == 0)
        issue_sh<K>(sm, stage, pA, pB, pS, start + kn * CH, min(CH, cnt - kn * CH), shift);
    }
  }
  if (tid == 0 && k < nchunks)
    for (int kk = k + 1; kk < nchunks && kk < k + STAGES; ++kk)
      gs_mbar_wait(&sm.full[kk % STAGES], (uint32_t)((kk / STAGES) & 1));
  if (tile_neff_b && tid == 0) tile_neff_b[tile] = consumed;
  if (row_epoch || GATHER) return;   // stale rows are skipped by the consumer (see blend.cu)
  for (int t = consumed + tid; t < cnt; t += THREADS) {
    const uint32_t slot = __float_as_uint(pS[(size_t)(start + t) * SW + 3 * K]);
    float* out = grad_inst + (size_t)slot * GREC;
    for (int u = 0; u < NV; ++u) out[u] = 0.f;
  }
}

}  // namespace

int gs_sh_basis_count(int d) { return d == 27 ? 9 : (d == 48 ? 16 : 0); }
int gs_sh_stream_width(int d) { return d == 27 ? sh_sw(9) : sh_sw(16); }
int gs_sh_grad_width(int d) { return d == 27 ? (sh_nv(9) + 3) / 4 * 4 : (sh_nv(16) + 3) / 4 * 4; }
// Default (sh_tc < 0): on the H100 the tensor-core kernels win at degree 3 (K = 16: frame 8.5 vs 11.3 ms at C3) and
// lose at degree 2 (K = 9: 8.3 vs 7.6 ms), where the scalar kernels' FMAs cost less than the hi/lo operand traffic.
int gs_sh_tc_mode(int d) {
  const int t = gs_tuning().sh_tc;
  return t >= 0 ? t : (d == 48 ? 3 : 0);
}

cudaError_t gs_launch_blend_sh_fwd(const float4* pA, const float2* pB, const float* pS, const GsRec* grec,
                                   const float* rgb, const uint32_t* ids, const uint32_t* goff, int d,
                                   const int* tile_accum,
                                   const GsFrameGeom& g, const GsRayPtrs& r, float* image, int* tile_neff,
                                   float* final_img, const GsCrop& crop, cudaStream_t st, const GsAuxOut* aux) {
#define GS_SHF_A(K, GA, AX, AV)                                                                                     \
  blend_sh_fwd_kernel<K, GA, AX><<<g.n_tiles, 64, 0, st>>>(pA, pB, pS, grec, rgb, ids, goff, tile_accum, g.wp, g.hp,   \
                                                           g.ntx, g.fx, g.fy, r.rays_o, r.lefttop, r.dx, r.dy, image,  \
                                                           tile_neff, final_img, crop, AV)
#define GS_SHF(K, GA) GS_SHF_A(K, GA, false, GsAuxOut{})
  // aux: the gather instantiations also serve a frame without instances (grec == nullptr when N == 0)
  if ((grec || aux) && (gs_sh_tc_mode(d) & 1))
    return gs_launch_blend_sh_fwd_tc(grec, rgb, ids, d, tile_accum, g, r, image, tile_neff, final_img, crop, st, aux);
  if (aux) {
    if (d == 27) GS_SHF_A(9, true, true, *aux); else GS_SHF_A(16, true, true, *aux);
  } else if (grec) {
    if (d == 27) GS_SHF(9, true); else GS_SHF(16, true);
  } else {
    if (d == 27) GS_SHF(9, false); else GS_SHF(16, false);
  }
#undef GS_SHF
#undef GS_SHF_A
  return cudaGetLastError();
}

cudaError_t gs_launch_blend_sh_bwd(const float4* pA, const float2* pB, const float* pS, const GsRec* grec,
                                   const float* rgb, const uint32_t* ids, const uint32_t* goff, int d,
                                   const int* tile_accum,
                                   const GsFrameGeom& g, const GsRayPtrs& r, const float* image,
                                   const float* grad_image, float* grad_inst, int grad_is_final, const GsCrop& crop,
                                   uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b, cudaStream_t st,
                                   const float* aux, const float* grad_aux) {
  if (grec && !row_epoch) return cudaErrorInvalidValue;
  if (grad_aux && (!grec || !aux)) return cudaErrorInvalidValue;
  if (grec && (gs_sh_tc_mode(d) & 2))
    return gs_launch_blend_sh_bwd_tc(grec, rgb, ids, goff, d, tile_accum, g, r, image, grad_image, grad_inst, grad_is_final,
                                     crop, row_epoch, epoch, tile_neff_b, st, aux, grad_aux);
#define GS_SHB_A(K, GA, AX)                                                                                         \
  blend_sh_bwd_kernel<K, GA, AX><<<g.n_tiles, 64, 0, st>>>(pA, pB, pS, grec, rgb, ids, goff, tile_accum, g.wp, g.hp,   \
                                                           g.ntx, g.fx, g.fy, r.rays_o, r.lefttop, r.dx, r.dy, image,  \
                                                           grad_image, grad_inst, grad_is_final, crop, row_epoch,      \
                                                           epoch, tile_neff_b, aux, grad_aux)
#define GS_SHB(K, GA) GS_SHB_A(K, GA, false)
  if (grad_aux) {
    if (d == 27) GS_SHB_A(9, true, true); else GS_SHB_A(16, true, true);
  } else if (grec) {
    if (d == 27) GS_SHB(9, true); else GS_SHB(16, true);
  } else {
    if (d == 27) GS_SHB(9, false); else GS_SHB(16, false);
  }
#undef GS_SHB
#undef GS_SHB_A
  return cudaGetLastError();
}
