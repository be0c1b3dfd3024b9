// Tile blend with per-pixel SH colour on the Hopper tensor cores (wgmma, fp32 accumulators in registers).
//
// The two dense contractions of the SH path (reference gaussian.cu:936-948 forward colour, :665-689 backward)
//   logit[pixel, (instance, channel)] = sum_q SH_q(pixel) * coef[instance, channel, q]                  (forward + backward)
//   d coef[(instance, channel), q]    = sum_pixel d logit[pixel, (instance, channel)] * SH_q(pixel)     (backward)
// are the only GEMM-shaped work of the rasterizer: 3K (forward) / 2 * 3K (backward) FMAs per (pixel, instance).
// Here ONE THREAD OWNS ONE PIXEL:
//   * a tile is 256 pixels = four M = 64 accumulator blocks; the SH basis of the tile is written once to shared
//     memory as bf16 hi + lo parts (x = hi + lo to 2^-17) in the no-swizzle canonical layout, whose image is at the
//     same time the K-major A operand of the first and the MN-major B operand of the second contraction;
//   * pixel p sits in accumulator row tc_row(p), chosen so that the fragment rows a warp receives from wgmma are
//     the pixels of that same warp: logits go registers -> shared memory -> registers without a CTA barrier;
//   * per round of 16 instances the raw coefficients (gathered by cp.async, as in blend_sh.cu) are split into
//     bf16 hi / lo K-major B operands [48 x 16] (pre-multiplied by -log2 e); per half round (8 instances x 3
//     channels = N 24) three MMAs per block (hi*hi + hi*lo + lo*hi, fp32 accumulate: logits to ~2e-5 relative);
//   * backward: the per-(pixel, instance) logit gradients are written back to shared memory as the MN-major A
//     operand [96 rows = (hi | lo) x 3 channels x 16 instances, K = 256 pixels] and contracted with the basis
//     image (N = 32 = hi | lo) by 16 K = 16 MMAs per M = 64 block; the six geometry sums per instance keep the
//     warp-shuffle reduction.
// Layouts / descriptor encodings: tc_common.cuh.
#include <cstddef>

#include "internal.h"
#include "sh_common.cuh"
#include "tc_common.cuh"

namespace {

using namespace gs_sh;
using namespace gs_tc;

constexpr int TC_J = 16;     // instances per round
constexpr int TC_NT = 256;   // threads per CTA = pixels per tile
constexpr int TC_LGS = 24;   // floats per row of the logit staging buffer: 3 channels x 8 instances

// float offset of logit column col (c * 8 + jj) of accumulator row `row` in the staging buffer: the six 16-byte
// chunks of a row are swapped in pairs on rows with bit 2 set, so that the eight rows a quarter warp reads (and
// the four a half warp writes) fall into different banks despite the 96-byte row stride
__device__ __forceinline__ int tc_lgs_off(int row, int col) {
  return row * TC_LGS + (((col >> 2) ^ ((row >> 2) & 1)) << 2) + (col & 3);
}

// accumulator row (= K index of the backward contraction) of tile pixel p: warp w of warpgroup g owns pixels
// 128 g + 32 w .. + 31, which are rows 16 w .. 16 w + 15 of blocks 2 g and 2 g + 1 - exactly the fragment rows
// of that warp when warpgroup g issues those two blocks (and of the same warp of a single warpgroup issuing all four)
__device__ __forceinline__ int tc_row(int p) {
  return (p >> 7) * 128 + ((p >> 4) & 1) * 64 + ((p >> 5) & 3) * 16 + (p & 15);
}

template <int K, int STAGES>
struct TcStage {
  float4 R[STAGES][TC_J * 4];
  float S[STAGES][TC_J * sh_sw(K)];
  uint64_t full[STAGES];
};

// NT / 16 threads per instance: record (3 x 16 B), first gradient row (backward), raw coefficients
template <int K, int STAGES, bool BWD, int NT = TC_NT>
__device__ __forceinline__ void tc_gather(TcStage<K, STAGES>& sm, int stage, const GsRec* __restrict__ grec,
                                          const float* __restrict__ rgb, const uint32_t* __restrict__ ids,
                                          const uint32_t* __restrict__ goff, int base, int n, int tid) {
  constexpr int SW = sh_sw(K), D = 3 * K, TPI = NT / TC_J;   // threads per instance
  static_assert(TPI >= 4, "the record pieces and the row offset need four threads");
  const int i = tid / TPI, l = tid % TPI;
  if (i < n) {
    const uint32_t id = ids[base + i];
    const uint32_t dr = gs_smem_u32(&sm.R[stage][i * 4]);
    if (l < 3) {
      const float4* src4 = reinterpret_cast<const float4*>(grec + id) + l;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dr + 16u * l), "l"(src4) : "memory");
    } else if (BWD && l == 3) {
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dr + 48u), "l"(goff + id) : "memory");
    }
    const float* src = rgb + (size_t)id * D;
    const uint32_t ds = gs_smem_u32(&sm.S[stage][i * SW]);
    if ((D * 4) % 16 == 0) {
      for (int q = l; q < D / 4; q += TPI)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ds + 16u * q), "l"(src + 4 * q) : "memory");
    } else {
      for (int q = l; q < D; q += TPI)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ds + 4u * q), "l"(src + q) : "memory");
    }
  }
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(gs_smem_u32(&sm.full[stage])) : "memory");
}

// raw coefficients of one round -> K-major bf16 operands [n = channel * 16 + instance][q], scaled by -log2 e
// (the blend needs 2^(-logit * log2 e)); element (n, q) lives in 16-byte unit (q / 8) * 48 + n.  q >= K stays 0.
template <int K>
__device__ __forceinline__ void tc_split_coefs(const float* __restrict__ S, uint4* __restrict__ bc_hi,
                                               uint4* __restrict__ bc_lo, int tid) {
  constexpr int SW = sh_sw(K);
  if ((unsigned)tid < 96u) {
    const int n = tid % 48, g = tid / 48, c = n >> 4, j = n & 15;
    const float* src = S + j * SW + c * K + g * 8;
    uint32_t h[4], l[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float v0 = (g * 8 + 2 * w < K) ? -GS_LOG2E * src[2 * w] : 0.f;
      const float v1 = (g * 8 + 2 * w + 1 < K) ? -GS_LOG2E * src[2 * w + 1] : 0.f;
      split_bf16x2(v0, v1, h[w], l[w]);
    }
    bc_hi[g * 48 + n] = make_uint4(h[0], h[1], h[2], h[3]);
    bc_lo[g * 48 + n] = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// SH basis of tile pixel p -> bf16 hi / lo operand image: 16-byte unit (q / 8) * 256 + tc_row(p)
template <int K>
__device__ __forceinline__ void tc_store_basis(const float* sh, uint4* __restrict__ img_hi, uint4* __restrict__ img_lo,
                                               int p) {
  const int row = tc_row(p);
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float v0 = (g * 8 + 2 * w < K) ? sh[g * 8 + 2 * w] : 0.f;
      const float v1 = (g * 8 + 2 * w + 1 < K) ? sh[g * 8 + 2 * w + 1] : 0.f;
      split_bf16x2(v0, v1, h[w], l[w]);
    }
    img_hi[g * 256 + row] = make_uint4(h[0], h[1], h[2], h[3]);
    img_lo[g * 256 + row] = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// logits of half round h (instances 8h .. 8h + 7, all three channels) for accumulator blocks b0 .. b0 + NB - 1,
// issued by the calling warpgroup: D[row, c * 8 + jj] = basis[row, :] . coef[c * 16 + 8h + jj, :], left in
// lgs[row * TC_LGS + c * 8 + jj] for the rows of the calling warp (which only that warp reads).
template <int NB>
__device__ __forceinline__ void tc_logits_half(int b0, int h, const uint4* img_hi, const uint4* img_lo, const uint4* bc_hi,
                                               const uint4* bc_lo, float* lgs, int wq, int lane) {
  float acc[NB][12];
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int i = 0; i < 12; ++i) acc[b][i] = 0.f;
  // N = 24 selects the 8-row groups h, h + 2, h + 4 of the [48 x 16] coefficient operand
  const uint64_t b_hi = smem_desc(gs_smem_u32(bc_hi) + h * 128, 768, 256);
  const uint64_t b_lo = smem_desc(gs_smem_u32(bc_lo) + h * 128, 768, 256);
#pragma unroll
  for (int b = 0; b < NB; ++b) acc_fence(acc[b]);
  wg_fence();
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    const uint64_t a_hi = smem_desc(gs_smem_u32(img_hi) + (b0 + b) * 1024, 4096, 128);
    const uint64_t a_lo = smem_desc(gs_smem_u32(img_lo) + (b0 + b) * 1024, 4096, 128);
    mma_n24_kk(acc[b], a_hi, b_hi, 0);
    mma_n24_kk(acc[b], a_hi, b_lo, 1);
    mma_n24_kk(acc[b], a_lo, b_hi, 1);
  }
  wg_commit();
  wg_wait_all();
#pragma unroll
  for (int b = 0; b < NB; ++b) acc_fence(acc[b]);
  __syncwarp();                                             // the warp's reads of the previous half are done
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = (b0 + b) * 64 + wq * 16 + (lane >> 2) + 8 * r;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        *reinterpret_cast<float2*>(lgs + tc_lgs_off(row, c * 8 + 2 * (lane & 3))) =
            make_float2(acc[b][4 * c + 2 * r], acc[b][4 * c + 2 * r + 1]);
    }
  __syncwarp();
}

// the 24 logits of half round of the pixel in accumulator row `row`
__device__ __forceinline__ void tc_read_logits(const float* lgs, int row, float* lr, float* lg, float* lb) {
  float* dst[3] = {lr, lg, lb};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float4 u = *reinterpret_cast<const float4*>(lgs + tc_lgs_off(row, c * 8));
    const float4 v = *reinterpret_cast<const float4*>(lgs + tc_lgs_off(row, c * 8 + 4));
    dst[c][0] = u.x; dst[c][1] = u.y; dst[c][2] = u.z; dst[c][3] = u.w;
    dst[c][4] = v.x; dst[c][5] = v.y; dst[c][6] = v.z; dst[c][7] = v.w;
  }
}

// three sigmoids from v_c = -logit_c * log2 e with ONE reciprocal (see blend_sh.cu)
__device__ __forceinline__ void tc_colours(float v0, float v1, float v2, float* col) {
  const float d0 = 1.f + gs_ex2(fminf(v0, 40.f)), d1 = 1.f + gs_ex2(fminf(v1, 40.f)), d2 = 1.f + gs_ex2(fminf(v2, 40.f));
  const float d01 = d0 * d1;
  const float r = gs_rcp(d01 * d2);
  col[2] = r * d01;
  const float r2 = r * d2;
  col[0] = r2 * d1;
  col[1] = r2 * d0;
}

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
template <int K>
struct TcFwdSmem {
  uint4 img_hi[2 * 256];
  uint4 img_lo[2 * 256];
  // by round parity: with one CTA barrier per round, a warpgroup may split round k + 1 while the other one still
  // runs the logit MMAs of round k
  uint4 bc_hi[2][2 * 48];
  uint4 bc_lo[2][2 * 48];
  float lgs[256 * TC_LGS];
  TcStage<K, 4> st;
};

template <int K>
__global__ void __launch_bounds__(TC_NT) blend_sh_fwd_tc_kernel(const GsRec* __restrict__ grec, const float* __restrict__ rgb,
                                                                const uint32_t* __restrict__ ids,
                                                                const int* __restrict__ tile_accum, int wp, int hp, int ntx,
                                                                float fx, float fy, const float* __restrict__ rays_o,
                                                                const float* __restrict__ lefttop,
                                                                const float* __restrict__ vdx, const float* __restrict__ vdy,
                                                                float* __restrict__ image, int* __restrict__ tile_neff,
                                                                float* __restrict__ final_img, GsCrop crop) {
  constexpr int STAGES = 4;
  extern __shared__ __align__(128) uint8_t tc_smem_raw[];
  TcFwdSmem<K>& sm = *reinterpret_cast<TcFwdSmem<K>*>(tc_smem_raw);
  const int tile = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix = tx * GS_TILE + (tid & 15), iy = ty * GS_TILE + (tid >> 4);
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  float T = 1.f, cr = 0.f, cg = 0.f, cb = 0.f;
  int consumed = cnt;
  if (cnt > 0) {                                              // uniform over the CTA
    const int nchunks = (cnt + TC_J - 1) / TC_J;
    if (tid == 0) {
      for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.st.full[s], TC_NT);
      gs_fence_barrier_init();
    }
    {
      float sh[16];
      pixel_sh<K>(ix, iy, rays_o, lefttop, vdx, vdy, sh);
      tc_store_basis<K>(sh, sm.img_hi, sm.img_lo, tid);
    }
    if (tid < 192) {                                          // q >= K columns of the coefficient operand stay zero
      sm.bc_hi[tid / 96][tid % 96] = make_uint4(0, 0, 0, 0);
      sm.bc_lo[tid / 96][tid % 96] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    const int row = tc_row(tid);
    const float px = gs_pixel_coord(ix, wp, fx), py = gs_pixel_coord(iy, hp, fy);
    for (int k = 0; k < STAGES - 1 && k < nchunks; ++k)
      tc_gather<K, STAGES, false>(sm.st, k, grec, rgb, ids, nullptr, start + k * TC_J, min(TC_J, cnt - k * TC_J), tid);

    for (int k = 0; k < nchunks; ++k) {
      const int stage = k % STAGES;
      gs_mbar_wait(&sm.st.full[stage], (uint32_t)((k / STAGES) & 1));
      const int n = min(TC_J, cnt - k * TC_J);
      uint4* bc_hi = sm.bc_hi[k & 1];
      uint4* bc_lo = sm.bc_lo[k & 1];
      tc_split_coefs<K>(sm.st.S[stage], bc_hi, bc_lo, tid);
      fence_smem_to_async();
      // every thread has finished round k - 1 (its logit MMAs, its staged rows); all pixels saturated -> done
      if (__syncthreads_and(!(T > GS_T_STOP))) {
        consumed = k * TC_J;
        break;
      }
      if (k + STAGES - 1 < nchunks) {
        const int kn = k + STAGES - 1;
        tc_gather<K, STAGES, false>(sm.st, kn % STAGES, grec, rgb, ids, nullptr, start + kn * TC_J,
                                    min(TC_J, cnt - kn * TC_J), tid);
      }
      const float4* R = sm.st.R[stage];
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        if (h * 8 >= n) break;                                // uniform
        tc_logits_half<2>(2 * (warp >> 2), h, sm.img_hi, sm.img_lo, bc_hi, bc_lo, sm.lgs, warp & 3, lane);
        if (__all_sync(0xffffffffu, !(T > GS_T_STOP))) continue;
        float lr[8], lg[8], lb[8];
        tc_read_logits(sm.lgs, row, lr, lg, lb);
        const float4* Rh = R + 32 * h;
        // one (pixel, instance) pair; a saturated pixel blends nothing (w = 0), without a divergent branch
        auto pair = [&](const float4 a, const float4 b4, float l0, float l1, float l2) {
          const float dx = px - a.x, dy = py - a.y;
          const float eu = fmaf(a.z, dx, -a.w * dy);
          const float ev = fmaf(-b4.x * dy, dy, b4.y);
          const float alpha = gs_ex2(fmaf(-dx, eu, ev));
          const float w = (T > GS_T_STOP) ? alpha * T : 0.f;
          float col[3];
          tc_colours(l0, l1, l2, col);
          cr = fmaf(col[0], w, cr);
          cg = fmaf(col[1], w, cg);
          cb = fmaf(col[2], w, cb);
          T -= w;
        };
        if (h * 8 + 8 <= n) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) pair(Rh[4 * jj], Rh[4 * jj + 1], lr[jj], lg[jj], lb[jj]);
        } else {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
            if (h * 8 + jj < n) pair(Rh[4 * jj], Rh[4 * jj + 1], lr[jj], lg[jj], lb[jj]);
        }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  }
  float* o = image + ((size_t)iy * wp + ix) * 3;
  o[0] = cr;
  o[1] = cg;
  o[2] = cb;
  if (final_img) gs_store_final(final_img, ix, iy, crop.left, crop.top, crop.width, crop.height, cr, cg, cb);
  if (tile_neff && tid == 0) tile_neff[tile] = consumed;
}

// ---------------------------------------------------------------------------------------
// backward
// grad row (GS_SH_GREC(K) floats): d/d{x, y, ca, cb, cc, l2o}, d/d coef[0..3K)
// ---------------------------------------------------------------------------------------
template <int K>
struct TcBwdSmem {
  // A operand of the coefficient-gradient contraction, MN-major: 16-byte unit G * 256 + row holds the 8 rows
  // (instances 8h .. 8h+7 of channel c, hi or lo part) G = part * 6 + c * 2 + h of that pixel row.  The second
  // M = 64 block reads 8 groups: the last four fall into img_hi / img_lo, which MUST follow (their rows are unused).
  uint4 dct[12 * 256];
  uint4 img_hi[2 * 256];
  uint4 img_lo[2 * 256];
  uint4 bc_hi[2 * 48];
  uint4 bc_lo[2 * 48];
  float lgs[256 * TC_LGS];
  TcStage<K, 3> st;            // three stages (not four): with them the CTA fits twice into an SM's shared memory
  float part[8][TC_J][8];      // per-warp sums of the six geometry values
  float epi[48][17];           // (lo part) . basis hi, staged for the thread that owns the hi row
};

// Coefficient-gradient contraction of one round, M = 64 blocks mb0 .. mb0 + NB - 1 issued by the calling warpgroup:
// D[row, n] = sum_pixel dct[pixel, row] * basis[pixel, n], rows = part * 48 + channel * 16 + instance,
// n = (hi | lo) x q.  Returns after issuing; tc_contract_finish waits.
template <int NB>
__device__ __forceinline__ void tc_contract_issue(int mb0, const uint4* dct, const uint4* img_hi, float (&acc)[NB][16]) {
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[b][i] = 0.f;
#pragma unroll
  for (int b = 0; b < NB; ++b) acc_fence(acc[b]);
  wg_fence();
  const uint32_t a0 = gs_smem_u32(dct), b0 = gs_smem_u32(img_hi);
#pragma unroll
  for (int s = 0; s < 16; ++s)
#pragma unroll
    for (int b = 0; b < NB; ++b)
      mma_n32_mn(acc[b], smem_desc(a0 + (mb0 + b) * 8 * 4096 + s * 256, 128, 4096), smem_desc(b0 + s * 256, 128, 4096),
                 s > 0);
  wg_commit();
}

// Waits for the contraction, then: rows 48 .. 95 (lo part, basis hi columns) -> epi; rows 0 .. 47 (hi part) keep
// basis hi + basis lo in hs[r][2 i + e] = column q = 8 i + 2 (lane % 4) + e of row 16 wq + lane / 4 + 8 r.
// Only block 0 holds hi rows (warps wq 0 .. 2 of the warpgroup that issued it).
template <int NB>
__device__ __forceinline__ void tc_contract_finish(int mb0, float (&acc)[NB][16], float (*epi)[17], float (&hs)[2][4],
                                                   int wq, int lane) {
  wg_wait_all();
#pragma unroll
  for (int b = 0; b < NB; ++b) acc_fence(acc[b]);
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = (mb0 + b) * 64 + wq * 16 + (lane >> 2) + 8 * r;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float bh = acc[b][4 * i + 2 * r + e], bl = acc[b][4 * (i + 2) + 2 * r + e];   // basis hi | lo columns
          if (row < 48) {
            hs[r][2 * i + e] = bh + bl;
          } else if (row < 96) {
            epi[row - 48][8 * i + 2 * (lane & 3) + e] = bh;
          }
        }
    }
}

// coefficient-gradient rows of the previous round (after a CTA barrier behind tc_contract_finish): threads of
// warps 0 .. 2 of the warpgroup that issued block 0 own rows 16 wq + lane / 4 (+ 8) = channel * 16 + instance.
// (np, Rp: instance count and staged records of THAT round - its stage is not refilled before the next barrier)
template <int K, int GREC>
__device__ __forceinline__ void tc_coef_rows(int np, const float4* Rp, const float (*epi)[17], const float (&hs)[2][4],
                                             int wq, int lane, int tx, int ty, float* __restrict__ grad_inst) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = wq * 16 + (lane >> 2) + 8 * r;
    const int c = row >> 4, j = row & 15;
    if (j < np) {
      const float4 cc = Rp[4 * j + 2];
      const uint32_t rxy = __float_as_uint(cc.z), rwh = __float_as_uint(cc.w);
      const uint32_t slot = __float_as_uint(Rp[4 * j + 3].x) + ((uint32_t)ty - (rxy >> 16)) * (rwh & 0xffffu) +
                            ((uint32_t)tx - (rxy & 0xffffu));
      float* out = grad_inst + (size_t)slot * GREC + 6 + c * K;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int q = 8 * i + 2 * (lane & 3) + e;
          if (q < K) out[q] = hs[r][2 * i + e] + epi[row][q];
        }
    }
  }
}

// geometry row of instance j of a round from the per-warp partial sums (NW warps)
template <int NW, int GREC>
__device__ __forceinline__ void tc_geom_row(int j, const float (*part)[TC_J][8], const float4* Rr, int tx, int ty,
                                            float* __restrict__ grad_inst, uint32_t* __restrict__ row_epoch,
                                            uint32_t epoch) {
  float s[6];
#pragma unroll
  for (int u = 0; u < 6; ++u) {
    float t = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < NW; ++w8) t += part[w8][j][u];
    s[u] = t;
  }
  const float4 a = Rr[4 * j];
  const float4 b4 = Rr[4 * j + 1];
  const float4 cc = Rr[4 * j + 2];
  const uint32_t rxy = __float_as_uint(cc.z), rwh = __float_as_uint(cc.w);
  const uint32_t slot = __float_as_uint(Rr[4 * j + 3].x) + ((uint32_t)ty - (rxy >> 16)) * (rwh & 0xffffu) +
                        ((uint32_t)tx - (rxy & 0xffffu));
  float* out = grad_inst + (size_t)slot * GREC;
  out[0] = GS_LN2 * (2.f * a.z * s[0] - a.w * s[1]);
  out[1] = GS_LN2 * (2.f * b4.x * s[1] - a.w * s[0]);
  out[2] = -GS_LN2 * s[2];
  out[3] = GS_LN2 * s[3];
  out[4] = -GS_LN2 * s[4];
  out[5] = GS_LN2 * s[5];
  row_epoch[slot] = epoch;
}

// Schedule of round k (two CTA-wide barriers per round):
//   wait records(k)  ->  [96 threads: split the coefficients of round k]  ->  B1(k)  ->  [warps 0-2: coefficient rows
//   of round k - 1]  ->  per half: logits (wgmma, waited), blend, store the dct rows  ->  B2(k) + "all pixels saturated"
//   vote  ->  issue contraction(k)  ->  [geometry rows of round k]  ->  gather round k + 2  ->  wait contraction(k),
//   stage its lo rows in epi / keep its hi rows in registers.
// What orders every producer / consumer pair:
//   staged records / coefficients   cp.async -> stage mbarrier (full[s]) -> every reader waits on it; a stage is refilled
//                                   (round k + 2 into the stage of round k - 1) after B2(k), its last readers (blend of
//                                   k - 1, geometry rows of k - 1, coefficient rows of k - 1) all run before B2(k)
//   bc_hi / bc_lo                   written before B1(k); read by the logit MMAs of round k, waited before B2(k)
//   lgs                             rows of a warp are written and read by that warp only (__syncwarp between)
//   sm.dct                          written between B1(k) and B2(k); read by contraction(k), waited before B1(k + 1)
//   sm.part                         written between B1(k) and B2(k); read by the geometry rows before B1(k + 1)
//   sm.epi                          written after contraction(k), before B1(k + 1); read between B1(k + 1) and B2(k + 1)

template <int K>
__global__ void __launch_bounds__(TC_NT, 2) blend_sh_bwd_tc_kernel(const GsRec* __restrict__ grec, const float* __restrict__ rgb,
                                                                const uint32_t* __restrict__ ids,
                                                                const uint32_t* __restrict__ goff,
                                                                const int* __restrict__ tile_accum, int wp, int hp, int ntx,
                                                                float fx, float fy, const float* __restrict__ rays_o,
                                                                const float* __restrict__ lefttop,
                                                                const float* __restrict__ vdx, const float* __restrict__ vdy,
                                                                const float* __restrict__ image,
                                                                const float* __restrict__ grad_image,
                                                                float* __restrict__ grad_inst, int grad_is_final, GsCrop crop,
                                                                uint32_t* __restrict__ row_epoch, uint32_t epoch,
                                                                int* __restrict__ tile_neff_b) {
  constexpr int STAGES = 3, NV = sh_nv(K), GREC = (NV + 3) / 4 * 4;
  static_assert(offsetof(TcBwdSmem<K>, img_hi) == 12 * 256 * 16 && offsetof(TcBwdSmem<K>, img_lo) == 14 * 256 * 16,
                "the basis image must follow the gradient operand: descriptors address both as one region");
  extern __shared__ __align__(128) uint8_t tc_smem_raw[];
  TcBwdSmem<K>& sm = *reinterpret_cast<TcBwdSmem<K>*>(tc_smem_raw);
  const int tile = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3;
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix = tx * GS_TILE + (tid & 15), iy = ty * GS_TILE + (tid >> 4);
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int nchunks = (cnt + TC_J - 1) / TC_J;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.st.full[s], TC_NT);
    gs_fence_barrier_init();
  }
  {
    float sh[16];
    pixel_sh<K>(ix, iy, rays_o, lefttop, vdx, vdy, sh);
    tc_store_basis<K>(sh, sm.img_hi, sm.img_lo, tid);
  }
  if (tid < 96) {
    sm.bc_hi[tid] = make_uint4(0, 0, 0, 0);
    sm.bc_lo[tid] = make_uint4(0, 0, 0, 0);
  }
  float T = 1.f, R, gr, gg, gb;
  {
    const size_t off = ((size_t)iy * wp + ix) * 3;
    const float raw[3] = {image[off], image[off + 1], image[off + 2]};
    if (!grad_is_final) {
      gr = grad_image[off];
      gg = grad_image[off + 1];
      gb = grad_image[off + 2];
    } else {
      gs_load_final_grad(grad_image, raw, ix, iy, crop.left, crop.top, crop.width, crop.height, gr, gg, gb);
    }
    R = gr * raw[0] + gg * raw[1] + gb * raw[2];
  }
  __syncthreads();
  const int row = tc_row(tid);
  const float px = gs_pixel_coord(ix, wp, fx), py = gs_pixel_coord(iy, hp, fy);
  for (int k = 0; k < STAGES - 1 && k < nchunks; ++k)
    tc_gather<K, STAGES, true>(sm.st, k, grec, rgb, ids, goff, start + k * TC_J, min(TC_J, cnt - k * TC_J), tid);

  // one (pixel, instance) pair: blend state update, logit gradients dc[3], geometry values v[0..5]
  auto pair = [&](const float4 a, const float4 b4, float l0, float l1, float l2, float* dc, float* v) {
    const float dx = px - a.x, dy = py - a.y;
    const float eu = fmaf(a.z, dx, -a.w * dy);
    const float ev = fmaf(-b4.x * dy, dy, b4.y);
    const float alpha = gs_ex2(fmaf(-dx, eu, ev));
    const bool live = T > GS_T_STOP;                        // saturated pixels contribute exactly nothing
    const float w = live ? alpha * T : 0.f;
    float col[3];
    tc_colours(l0, l1, l2, col);
    const float gc = fmaf(gr, col[0], fmaf(gg, col[1], gb * col[2]));
    R = fmaf(-gc, w, R);
    const float rc = gs_rcp(1.0000001f - alpha);
    const float dal = fmaf(T, gc, -R * rc);
    const float e = live ? dal * alpha : 0.f;
    T -= w;
    const float ex = e * dx, ey = e * dy;
    v[0] = ex;
    v[1] = ey;
    v[2] = ex * dx;
    v[3] = ex * dy;
    v[4] = ey * dy;
    v[5] = e;
    v[6] = 0.f;
    v[7] = 0.f;
    // d colour_c / d logit_c = sigma'(.)      (gaussian.cu:666-674)
    dc[0] = gr * w * col[0] * (1.f - col[0]);
    dc[1] = gg * w * col[1] * (1.f - col[1]);
    dc[2] = gb * w * col[2] * (1.f - col[2]);
  };

  int consumed = cnt, n_prev = 0, st_prev = 0;
  float hs[2][4];
  for (int k = 0; k < nchunks; ++k) {
    const int stage = k % STAGES;
    const int n = min(TC_J, cnt - k * TC_J);
    gs_mbar_wait(&sm.st.full[stage], (uint32_t)((k / STAGES) & 1));   // records of this round
    tc_split_coefs<K>(sm.st.S[stage], sm.bc_hi, sm.bc_lo, tid);
    fence_smem_to_async();
    __syncthreads();                                        // B1(k)
    if (n_prev > 0 && tid < 96)
      tc_coef_rows<K, GREC>(n_prev, sm.st.R[st_prev], sm.epi, hs, wq, lane, tx, ty, grad_inst);
    const float4* Rr = sm.st.R[stage];
    float(*part)[8] = sm.part[warp];
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      if (h * 8 >= n) break;                                // uniform; rows of a missing half are never read out
      tc_logits_half<2>(2 * wg, h, sm.img_hi, sm.img_lo, sm.bc_hi, sm.bc_lo, sm.lgs, wq, lane);
      uint32_t hw[3][4], lw[3][4];
      if (!__all_sync(0xffffffffu, !(T > GS_T_STOP))) {
        float lr[8], lg[8], lb[8];
        tc_read_logits(sm.lgs, row, lr, lg, lb);
        const float4* Rh = Rr + 32 * h;
        float* ph = &part[h * 8][(lane >> 2) & 7];
        if (h * 8 + 8 <= n) {                               // all eight instances exist: no per-instance tests
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            float dc[2][3];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int jj = 2 * jp + u;
              float v[8];
              pair(Rh[4 * jj], Rh[4 * jj + 1], lr[jj], lg[jj], lb[jj], dc[u], v);
              const float r = reduce8(v, lane);
              if ((lane & 3) == 0) ph[jj * 8] = r;
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) split_bf16x2(dc[0][c], dc[1][c], hw[c][jp], lw[c][jp]);
          }
        } else {
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            float dc[2][3];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int jj = 2 * jp + u;
              dc[u][0] = dc[u][1] = dc[u][2] = 0.f;
              if (h * 8 + jj < n) {
                float v[8];
                pair(Rh[4 * jj], Rh[4 * jj + 1], lr[jj], lg[jj], lb[jj], dc[u], v);
                const float r = reduce8(v, lane);
                if ((lane & 3) == 0) ph[jj * 8] = r;
              }
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) split_bf16x2(dc[0][c], dc[1][c], hw[c][jp], lw[c][jp]);
          }
        }
      } else {
        // nothing left to blend in this warp: the rows of this half round are zeros
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int q = 0; q < 4; ++q) hw[c][q] = lw[c][q] = 0u;
        part[h * 8 + (lane >> 2)][lane & 3] = 0.f;
        part[h * 8 + (lane >> 2)][4 + (lane & 3)] = 0.f;
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        sm.dct[(c * 2 + h) * 256 + row] = make_uint4(hw[c][0], hw[c][1], hw[c][2], hw[c][3]);
        sm.dct[(6 + c * 2 + h) * 256 + row] = make_uint4(lw[c][0], lw[c][1], lw[c][2], lw[c][3]);
      }
    }
    fence_smem_to_async();
    const bool done = __syncthreads_and(!(T > GS_T_STOP)) != 0;   // B2(k): operands of the contraction complete
    float acc[1][16];
    tc_contract_issue<1>(wg, sm.dct, sm.img_hi, acc);
    // geometry rows (while the tensor core contracts): threads 128 .. 143, one instance each
    if (tid >= 128 && tid < 128 + n)
      tc_geom_row<8, GREC>(tid - 128, sm.part, Rr, tx, ty, grad_inst, row_epoch, epoch);
    n_prev = n;
    st_prev = stage;
    // stage (k + 2) % 3 held round k - 1, whose records were last read before this round's B2
    if (!done && k + STAGES - 1 < nchunks) {
      const int kn = k + STAGES - 1;
      tc_gather<K, STAGES, true>(sm.st, kn % STAGES, grec, rgb, ids, goff, start + kn * TC_J, min(TC_J, cnt - kn * TC_J),
                                 tid);
    }
    tc_contract_finish<1>(wg, acc, sm.epi, hs, wq, lane);
    if (done) {
      consumed = min(cnt, (k + 1) * TC_J);
      break;
    }
  }
  __syncthreads();
  if (n_prev > 0 && tid < 96) tc_coef_rows<K, GREC>(n_prev, sm.st.R[st_prev], sm.epi, hs, wq, lane, tx, ty, grad_inst);
  asm volatile("cp.async.wait_all;" ::: "memory");
  if (tile_neff_b && tid == 0) tile_neff_b[tile] = consumed;
}


// ---------------------------------------------------------------------------------------
// backward, TWO pixels per thread: 128 threads (one warpgroup) per tile, thread t owns pixels t and t + 128 (same
// column, 8 rows below) and issues all four accumulator blocks.  The per-instance work that one pixel per thread
// repeats for every 32 pixels (record loads, dx, the shuffle reduction of the six geometry sums) is shared by
// 64 pixels, and every thread carries two independent blend recurrences.  Same operands, schedule and
// result rows as blend_sh_bwd_tc_kernel.
// ---------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(128) blend_sh_bwd_tc2_kernel(const GsRec* __restrict__ grec, const float* __restrict__ rgb,
                                                               const uint32_t* __restrict__ ids,
                                                               const uint32_t* __restrict__ goff,
                                                               const int* __restrict__ tile_accum, int wp, int hp, int ntx,
                                                               float fx, float fy, const float* __restrict__ rays_o,
                                                               const float* __restrict__ lefttop,
                                                               const float* __restrict__ vdx, const float* __restrict__ vdy,
                                                               const float* __restrict__ image,
                                                               const float* __restrict__ grad_image,
                                                               float* __restrict__ grad_inst, int grad_is_final, GsCrop crop,
                                                               uint32_t* __restrict__ row_epoch, uint32_t epoch,
                                                               int* __restrict__ tile_neff_b) {
  constexpr int NT = 128, STAGES = 3, NV = sh_nv(K), GREC = (NV + 3) / 4 * 4;
  extern __shared__ __align__(128) uint8_t tc_smem_raw[];
  TcBwdSmem<K>& sm = *reinterpret_cast<TcBwdSmem<K>*>(tc_smem_raw);
  const int tile = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = tile % ntx, ty = tile / ntx;
  const int ix = tx * GS_TILE + (tid & 15), iy0 = ty * GS_TILE + (tid >> 4), iy1 = iy0 + 8;
  const int start = tile_accum[tile];
  const int cnt = tile_accum[tile + 1] - start;
  if (cnt == 0) return;
  const int nchunks = (cnt + TC_J - 1) / TC_J;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) gs_mbar_init(&sm.st.full[s], NT);
    gs_fence_barrier_init();
  }
  {
    float sh[16];
    pixel_sh<K>(ix, iy0, rays_o, lefttop, vdx, vdy, sh);
    tc_store_basis<K>(sh, sm.img_hi, sm.img_lo, tid);
    pixel_sh<K>(ix, iy1, rays_o, lefttop, vdx, vdy, sh);
    tc_store_basis<K>(sh, sm.img_hi, sm.img_lo, tid + 128);
  }
  if (tid < 96) {
    sm.bc_hi[tid] = make_uint4(0, 0, 0, 0);
    sm.bc_lo[tid] = make_uint4(0, 0, 0, 0);
  }
  float T[2] = {1.f, 1.f}, R[2], gr[2], gg[2], gb[2];
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const int iy = p ? iy1 : iy0;
    const size_t off = ((size_t)iy * wp + ix) * 3;
    const float raw[3] = {image[off], image[off + 1], image[off + 2]};
    if (!grad_is_final) {
      gr[p] = grad_image[off];
      gg[p] = grad_image[off + 1];
      gb[p] = grad_image[off + 2];
    } else {
      gs_load_final_grad(grad_image, raw, ix, iy, crop.left, crop.top, crop.width, crop.height, gr[p], gg[p], gb[p]);
    }
    R[p] = gr[p] * raw[0] + gg[p] * raw[1] + gb[p] * raw[2];
  }
  __syncthreads();
  const int row[2] = {tc_row(tid), tc_row(tid + 128)};
  const float px = gs_pixel_coord(ix, wp, fx);
  const float py[2] = {gs_pixel_coord(iy0, hp, fy), gs_pixel_coord(iy1, hp, fy)};
  for (int k = 0; k < STAGES - 1 && k < nchunks; ++k)
    tc_gather<K, STAGES, true, NT>(sm.st, k, grec, rgb, ids, goff, start + k * TC_J, min(TC_J, cnt - k * TC_J), tid);

  // one instance, both pixels: blend state updates, logit gradients dc[pixel][3], summed geometry values v[0..7]
  auto pair2 = [&](const float4 a, const float4 b4, const float* l0, const float* l1, float (*dc)[3], float* v) {
    const float dx = px - a.x;
    const float adx = a.z * dx;
    float e2[2], ey2[2];
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const float dy = py[p] - a.y;
      const float eu = fmaf(-a.w, dy, adx);
      const float ev = fmaf(-b4.x * dy, dy, b4.y);
      const float alpha = gs_ex2(fmaf(-dx, eu, ev));
      const bool live = T[p] > GS_T_STOP;
      const float w = live ? alpha * T[p] : 0.f;
      float col[3];
      const float* l = p ? l1 : l0;
      tc_colours(l[0], l[1], l[2], col);
      const float gc = fmaf(gr[p], col[0], fmaf(gg[p], col[1], gb[p] * col[2]));
      R[p] = fmaf(-gc, w, R[p]);
      const float rc = gs_rcp(1.0000001f - alpha);
      const float dal = fmaf(T[p], gc, -R[p] * rc);
      const float e = live ? dal * alpha : 0.f;
      T[p] -= w;
      e2[p] = e;
      ey2[p] = e * dy;
      v[4] = p ? fmaf(ey2[1], dy, v[4]) : ey2[0] * dy;
      dc[p][0] = gr[p] * w * col[0] * (1.f - col[0]);
      dc[p][1] = gg[p] * w * col[1] * (1.f - col[1]);
      dc[p][2] = gb[p] * w * col[2] * (1.f - col[2]);
    }
    const float es = e2[0] + e2[1], eys = ey2[0] + ey2[1];
    const float ex = es * dx;
    v[0] = ex;
    v[1] = eys;
    v[2] = ex * dx;
    v[3] = eys * dx;
    v[5] = es;
    v[6] = 0.f;
    v[7] = 0.f;
  };

  int consumed = cnt, n_prev = 0, st_prev = 0;
  float hs[2][4];
  for (int k = 0; k < nchunks; ++k) {
    const int stage = k % STAGES;
    const int n = min(TC_J, cnt - k * TC_J);
    gs_mbar_wait(&sm.st.full[stage], (uint32_t)((k / STAGES) & 1));
    tc_split_coefs<K>(sm.st.S[stage], sm.bc_hi, sm.bc_lo, tid);
    fence_smem_to_async();
    __syncthreads();                                        // B1(k)
    if (n_prev > 0 && tid < 96)
      tc_coef_rows<K, GREC>(n_prev, sm.st.R[st_prev], sm.epi, hs, warp, lane, tx, ty, grad_inst);
    const float4* Rr = sm.st.R[stage];
    float(*part)[8] = sm.part[warp];
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      if (h * 8 >= n) break;
      tc_logits_half<4>(0, h, sm.img_hi, sm.img_lo, sm.bc_hi, sm.bc_lo, sm.lgs, warp, lane);
      uint32_t hw[2][3][4], lw[2][3][4];
      if (!__all_sync(0xffffffffu, !(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP))) {
        float lr[2][8], lg[2][8], lb[2][8];
        tc_read_logits(sm.lgs, row[0], lr[0], lg[0], lb[0]);
        tc_read_logits(sm.lgs, row[1], lr[1], lg[1], lb[1]);
        const float4* Rh = Rr + 32 * h;
        float* ph = &part[h * 8][(lane >> 2) & 7];
        const bool full = h * 8 + 8 <= n;
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          float dc[2][2][3];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int jj = 2 * jp + u;
#pragma unroll
            for (int p = 0; p < 2; ++p) dc[u][p][0] = dc[u][p][1] = dc[u][p][2] = 0.f;
            if (full || h * 8 + jj < n) {
              float v[8];
              const float l0[3] = {lr[0][jj], lg[0][jj], lb[0][jj]}, l1[3] = {lr[1][jj], lg[1][jj], lb[1][jj]};
              pair2(Rh[4 * jj], Rh[4 * jj + 1], l0, l1, dc[u], v);
              const float r = reduce8(v, lane);
              if ((lane & 3) == 0) ph[jj * 8] = r;
            }
          }
#pragma unroll
          for (int p = 0; p < 2; ++p)
#pragma unroll
            for (int c = 0; c < 3; ++c) split_bf16x2(dc[0][p][c], dc[1][p][c], hw[p][c][jp], lw[p][c][jp]);
        }
      } else {
#pragma unroll
        for (int p = 0; p < 2; ++p)
#pragma unroll
          for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int q = 0; q < 4; ++q) hw[p][c][q] = lw[p][c][q] = 0u;
        part[h * 8 + (lane >> 2)][lane & 3] = 0.f;
        part[h * 8 + (lane >> 2)][4 + (lane & 3)] = 0.f;
      }
#pragma unroll
      for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          sm.dct[(c * 2 + h) * 256 + row[p]] = make_uint4(hw[p][c][0], hw[p][c][1], hw[p][c][2], hw[p][c][3]);
          sm.dct[(6 + c * 2 + h) * 256 + row[p]] = make_uint4(lw[p][c][0], lw[p][c][1], lw[p][c][2], lw[p][c][3]);
        }
    }
    fence_smem_to_async();
    const bool done = __syncthreads_and(!(T[0] > GS_T_STOP) && !(T[1] > GS_T_STOP)) != 0;   // B2(k)
    float acc[2][16];
    tc_contract_issue<2>(0, sm.dct, sm.img_hi, acc);
    // geometry rows: threads 96 .. 111 (warp 3), one instance each
    if (tid >= 96 && tid < 96 + n) tc_geom_row<4, GREC>(tid - 96, sm.part, Rr, tx, ty, grad_inst, row_epoch, epoch);
    n_prev = n;
    st_prev = stage;
    if (!done && k + STAGES - 1 < nchunks) {
      const int kn = k + STAGES - 1;
      tc_gather<K, STAGES, true, NT>(sm.st, kn % STAGES, grec, rgb, ids, goff, start + kn * TC_J, min(TC_J, cnt - kn * TC_J),
                                     tid);
    }
    tc_contract_finish<2>(0, acc, sm.epi, hs, warp, lane);
    if (done) {
      consumed = min(cnt, (k + 1) * TC_J);
      break;
    }
  }
  __syncthreads();
  if (n_prev > 0 && tid < 96) tc_coef_rows<K, GREC>(n_prev, sm.st.R[st_prev], sm.epi, hs, warp, lane, tx, ty, grad_inst);
  asm volatile("cp.async.wait_all;" ::: "memory");
  if (tile_neff_b && tid == 0) tile_neff_b[tile] = consumed;
}

}  // namespace

cudaError_t gs_launch_blend_sh_fwd_tc(const GsRec* grec, const float* rgb, const uint32_t* ids, int d,
                                      const int* tile_accum, const GsFrameGeom& g, const GsRayPtrs& r, float* image,
                                      int* tile_neff, float* final_img, const GsCrop& crop, cudaStream_t st) {
#define GS_SHF_TC(K)                                                                                                  \
  do {                                                                                                                \
    /* per device and cheap: set on every launch rather than cached in a process-wide flag */                        \
    cudaError_t e = cudaFuncSetAttribute(blend_sh_fwd_tc_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize,      \
                                         (int)sizeof(TcFwdSmem<K>));                                                  \
    if (e != cudaSuccess) return e;                                                                                   \
    blend_sh_fwd_tc_kernel<K><<<g.n_tiles, TC_NT, sizeof(TcFwdSmem<K>), st>>>(                                         \
        grec, rgb, ids, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, r.rays_o, r.lefttop, r.dx, r.dy, image, tile_neff,  \
        final_img, crop);                                                                                             \
  } while (0)
  if (d == 27) GS_SHF_TC(9); else GS_SHF_TC(16);
#undef GS_SHF_TC
  return cudaGetLastError();
}

cudaError_t gs_launch_blend_sh_bwd_tc(const GsRec* grec, const float* rgb, const uint32_t* ids, const uint32_t* goff, int d,
                                      const int* tile_accum, const GsFrameGeom& g, const GsRayPtrs& r, const float* image,
                                      const float* grad_image, float* grad_inst, int grad_is_final, const GsCrop& crop,
                                      uint32_t* row_epoch, uint32_t epoch, int* tile_neff_b, cudaStream_t st) {
  if (!row_epoch) return cudaErrorInvalidValue;   // unprocessed rows are left stale: the consumer needs the epoch tags
  const bool two_px = (gs_sh_tc_mode(d) & 4) != 0;   // two pixels per thread (128 threads per tile)
#define GS_SHB_TC(K)                                                                                                  \
  do {                                                                                                                \
    cudaError_t e = two_px ? cudaFuncSetAttribute(blend_sh_bwd_tc2_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                                  (int)sizeof(TcBwdSmem<K>))                                          \
                           : cudaFuncSetAttribute(blend_sh_bwd_tc_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                                  (int)sizeof(TcBwdSmem<K>));                                         \
    if (e != cudaSuccess) return e;                                                                                   \
    if (two_px)                                                                                                       \
      blend_sh_bwd_tc2_kernel<K><<<g.n_tiles, 128, sizeof(TcBwdSmem<K>), st>>>(                                        \
          grec, rgb, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, r.rays_o, r.lefttop, r.dx, r.dy, image,     \
          grad_image, grad_inst, grad_is_final, crop, row_epoch, epoch, tile_neff_b);                                 \
    else                                                                                                              \
      blend_sh_bwd_tc_kernel<K><<<g.n_tiles, TC_NT, sizeof(TcBwdSmem<K>), st>>>(                                        \
          grec, rgb, ids, goff, tile_accum, g.wp, g.hp, g.ntx, g.fx, g.fy, r.rays_o, r.lefttop, r.dx, r.dy, image,     \
          grad_image, grad_inst, grad_is_final, crop, row_epoch, epoch, tile_neff_b);                                 \
  } while (0)
  if (d == 27) GS_SHB_TC(9); else GS_SHB_TC(16);
#undef GS_SHB_TC
  return cudaGetLastError();
}
