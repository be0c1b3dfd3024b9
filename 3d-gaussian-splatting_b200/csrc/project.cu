// Per-Gaussian kernels: projection + cull + 2-D covariance (forward / backward), legacy
// helpers (world2camera, jacobian) and the fused frame-path variants that also apply the
// parameter activations and the tile-rectangle rule.  All HBM-bound streaming kernels.
#include "internal.h"
#include "sh_common.cuh"

#include <type_traits>

namespace {

constexpr int kBlock = 256;
// gs_project's frustum half-widths in a lens frame: the lens tests the stored mean itself (gs_lens_project)
constexpr float kInf = __builtin_huge_valf();

__global__ void __launch_bounds__(kBlock) jacobian_kernel(const float* __restrict__ pc, int n,
                                                           float* __restrict__ jac) {
  int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float u0 = pc[3 * i], u1 = pc[3 * i + 1], u2 = pc[3 * i + 2];   // gaussian.cu:10-39
  float rs = rsqrtf(u0 * u0 + u1 * u1 + u2 * u2);
  float* j = jac + 9 * (size_t)i;
  j[0] = 1.f / u2;
  j[1] = 0.f;
  j[2] = -u0 / (u2 * u2);
  j[3] = 0.f;
  j[4] = 1.f / u2;
  j[5] = -u1 / (u2 * u2);
  j[6] = rs * u0;
  j[7] = rs * u1;
  j[8] = rs * u2;
}

// ---------------------------------------------------------------------------------------
// Fused frame path.  Activations (splatter.py:519-524,:539-540) are applied in-register (gs_load_activated).
// ---------------------------------------------------------------------------------------

// Unit direction from the camera centre C = -R^T t to the mean, in the world frame (the frame of the per-pixel rays,
// so that an SH coefficient means the same in both evaluation modes); inv_len = 1 / |pos - C| = 1 / |p_c|.
__device__ __forceinline__ void view_dir(const GsCam& cam, const float p[3], float dir[3], float& inv_len) {
  float u[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) u[j] = p[j] + (cam.r[j] * cam.t[0] + cam.r[3 + j] * cam.t[1] + cam.r[6 + j] * cam.t[2]);
  inv_len = 1.f / sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);   // visible: |u| >= z > near
#pragma unroll
  for (int j = 0; j < 3; ++j) dir[j] = u[j] * inv_len;
}

// logits l_c = sum_k Y_k coef[c*K + k] of the channel-major coefficient row coef[3K]
template <int K>
__device__ __forceinline__ void sh_logits(const float* coef, const float* Y, float l[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) s = fmaf(Y[k], coef[c * K + k], s);
    l[c] = s;
  }
}

// Gaussian i (loaded parameters p, q, s, opa_raw, rgb_raw) seen by one view: its record, rectangle, count and depth key
// go to pair j (j = i in a single-view frame, v n + i for view v of a batched one) with the rectangle's rows offset by
// ty_off (the view's first tile row).  Returns the instance count; vis: in the frustum.
// KG = 0: colour from the rgb[n, 3] logits when d == 3 (per-pixel SH leaves it to the blend).  KG = 9 / 16: SH of
// degree 2 / 3 evaluated once per Gaussian along view_dir (GS_SH_EVAL_GAUSSIAN); the record then carries an RGB colour.
// TIER (GsTier, cumulative):
//   >= GS_TIER_FILT2D: the 2-D screen-space filter `filt` (gs_filter2d) is applied to the covariance before the tile
//     rectangle and the conic, and its compensation to l2o.
//   >= GS_TIER_FILT3D: s is the 3-D filtered scale (gs_filter3d) and dl2o3 its compensation, added to l2o before the
//     2-D filter's when f3 != 0.
//   GS_TIER_LENS: the lens *lens (gs_lens_project) is applied to the projection before the 2-D filter.
template <int KG, int TIER>
__device__ __forceinline__ uint32_t fused_project_one(
    const float* __restrict__ rgb, int i, int d, const GsCam& cam, const GsTileGrid& grid, float near_plane,
    float half_w, float half_h, const GsFilter2d& filt, const float p[3], const float q[4], const float s[3],
    float opa_raw, const float rgb_raw[3], uint32_t ty_off, int j, GsRec* __restrict__ rec, uint2* __restrict__ rect,
    uint32_t* __restrict__ count, uint32_t* __restrict__ dkey, int64_t* __restrict__ mask, bool& vis, float f3,
    float dl2o3, const GsLens* __restrict__ lens) {
  constexpr bool F = TIER >= GS_TIER_FILT2D, G3 = TIER >= GS_TIER_FILT3D, L = TIER == GS_TIER_LENS;
  uint32_t cnt = 0;
  {
    GsProj o = gs_project(cam, p, q, s, near_plane, L ? kInf : half_w, L ? kInf : half_h);
    if constexpr (L) {
      float J[4];
      gs_lens_project(*lens, o, half_w, half_h, J);
    }
    vis = o.visible;
    if (mask) mask[j] = o.visible ? 1 : 0;
    bool keep = o.visible;
    float dl2o = 0.f;
    if constexpr (F) {
      const GsFilter2dOut fo = gs_filter2d(filt, o.a, o.b, o.c, o.d);
      o.a = fo.a;
      o.d = fo.d;
      dl2o = fo.dl2o;
      keep = keep && fo.keep;
    }
    uint2 rc = make_uint2(0u, 0u);
    if (keep) {
      uint32_t tx0, tx1, ty0, ty1;
      if (gs_tile_rect(grid, o.x, o.y, o.a, o.b, o.c, o.d, tx0, tx1, ty0, ty1)) {
        cnt = (tx1 - tx0) * (ty1 - ty0);
        rc = make_uint2(tx0 | ((ty0 + ty_off) << 16), (tx1 - tx0) | ((ty1 - ty0) << 16));
        GsConic k = gs_make_conic(o.a, o.b, o.c, o.d);
        float op = gs_sigmoid(opa_raw);
        GsRec* r = rec + j;
        r->a = make_float4(o.x, o.y, k.ca, k.cb);
        // RGB colour = sigmoid(logit) (splatter.py:539); per-pixel SH coefficients stay raw and are gathered
        // from the parameter tensor by the pack pass
        float cr = 0.f, cg = 0.f, cb = 0.f;
        if constexpr (KG > 0) {
          float coef[3 * KG], dir[3], il, Y[KG], l[3];
#pragma unroll
          for (int k = 0; k < 3 * KG; ++k) coef[k] = rgb[(size_t)i * (3 * KG) + k];
          view_dir(cam, p, dir, il);
          gs_sh::sh_basis<KG>(dir[0], dir[1], dir[2], Y);
          sh_logits<KG>(coef, Y, l);
          cr = gs_sigmoid(l[0]);
          cg = gs_sigmoid(l[1]);
          cb = gs_sigmoid(l[2]);
        } else if (d == 3) {
          cr = gs_sigmoid(rgb_raw[0]);
          cg = gs_sigmoid(rgb_raw[1]);
          cb = gs_sigmoid(rgb_raw[2]);
        }
        float l2o = log2f(op);
        if constexpr (G3) {
          if (f3 != 0.f) l2o += dl2o3;
        }
        r->b = make_float4(k.cc, F ? l2o + dl2o : l2o, cr, cg);
        r->c = make_float4(cb, o.depth, __uint_as_float(rc.x), __uint_as_float(rc.y));
        r->d = make_uint4(0u, 0u, 0u, 0u);   // whole 32-byte sectors: a half-written sector is a DRAM read-modify-write (ECC)
      }
    }
    // the tile rectangle again, densely (zero without instances: whole sectors), for the instance emission: an 8-byte
    // read from a 19 MB array at C3 instead of a 16-byte gather from the 154 MB records
    rect[j] = rc;
    count[j] = cnt;
    // depth sort key: positive float bits order like the floats; Gaussians without instances last
    dkey[j] = cnt ? __float_as_uint(o.depth) : 0xffffffffu;
  }
  return cnt;
}

// Gaussian i's parameters as the projection and its backward load them: position, normalised quaternion (and the raw
// one's norm), activated scale s and raw scale.  TIER >= GS_TIER_FILT3D: s is 3-D filtered (f3, compensation dl2o3)
// and s0 keeps the activated scale.  A lens frame without a 3-D filter passes f3d NULL (the f == 0 bits).
template <int TIER>
__device__ __forceinline__ void fused_project_load(const float* __restrict__ pos, const float* __restrict__ quat,
                                                   const float* __restrict__ scale, const float* __restrict__ f3d,
                                                   int i, int scale_act, float p[3], float q[4], float s[3],
                                                   float raw_s[3], float& qn, float s0[3], float& f3, float& dl2o3) {
  p[0] = pos[3 * i];
  p[1] = pos[3 * i + 1];
  p[2] = pos[3 * i + 2];
  gs_load_activated(quat, scale, i, scale_act, q, s, raw_s, qn);
  f3 = 0.f;
  dl2o3 = 0.f;
  if constexpr (TIER >= GS_TIER_FILT3D) {
    f3 = (TIER == GS_TIER_LENS && !f3d) ? 0.f : f3d[i];
    gs_filter3d(f3, s, s0, dl2o3);
  }
}

// Single-view frame: pair j = i.  The opacity and RGB logits are issued with the geometry, so that the thread makes one
// round trip to HBM, not two (a warp almost always has a binned Gaussian, so their sectors are fetched anyway).
template <int KG, int TIER>
__global__ void __launch_bounds__(kBlock) fused_project_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int d, int scale_act, GsCam cam,
    GsTileGrid grid, float near_plane, float half_w, float half_h, GsRec* __restrict__ rec,
    uint2* __restrict__ rect, uint32_t* __restrict__ count, uint32_t* __restrict__ dkey, int64_t* __restrict__ mask,
    unsigned int* __restrict__ n_visible, GsFilter2d filt, const float* __restrict__ f3d, GsLens lens) {
  int i = blockIdx.x * kBlock + threadIdx.x;
  bool vis = false;
  uint32_t cnt = 0;
  if (i < n) {
    float p[3], q[4], s[3], raw_s[3], qn, s0[3], f3, dl2o3;
    fused_project_load<TIER>(pos, quat, scale, f3d, i, scale_act, p, q, s, raw_s, qn, s0, f3, dl2o3);
    const float opa_raw = opa[i];
    float rgb_raw[3] = {0.f, 0.f, 0.f};
    if (KG == 0 && d == 3) {
      rgb_raw[0] = rgb[3 * i];
      rgb_raw[1] = rgb[3 * i + 1];
      rgb_raw[2] = rgb[3 * i + 2];
    }
    cnt = fused_project_one<KG, TIER>(rgb, i, d, cam, grid, near_plane, half_w, half_h, filt, p, q, s, opa_raw,
                                      rgb_raw, 0u, i, rec, rect, count, dkey, mask, vis, f3, dl2o3, &lens);
  }
  // 64-bit instance total next to the visible count (counters[2..3]): the u32 scans that follow
  // would wrap silently for M >= 2^32 (e.g. diverged scales: every Gaussian on every tile); the
  // host sizes the frame from this total and refuses instead
  __shared__ unsigned long long wsum[kBlock / 32];
  unsigned long long c64 = cnt;
#pragma unroll
  for (int o = 16; o; o >>= 1) c64 += __shfl_xor_sync(0xffffffffu, c64, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c64;
  int nv = __syncthreads_count(vis);
  if (threadIdx.x == 0) {
    unsigned long long tot = 0;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) tot += wsum[w];
    if (nv) atomicAdd(n_visible, (unsigned int)nv);
    if (tot) atomicAdd(reinterpret_cast<unsigned long long*>(n_visible + 2), tot);
  }
}

// Batched frame: one thread per Gaussian loads its parameters once (the 3-D filter applied once, before the views) and
// projects it into each view in turn, writing pair j = v n + i with view v's constants: camera, grid, filter
// views[v].filt and lens lenses[v].  The counters receive the frame's totals over the pairs.
template <int K, int TIER>
__global__ void __launch_bounds__(kBlock) fused_project_batch_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int n_views, int d, int scale_act,
    const GsView* __restrict__ views, float near_plane, GsRec* __restrict__ rec, uint2* __restrict__ rect,
    uint32_t* __restrict__ count, uint32_t* __restrict__ dkey, int64_t* __restrict__ mask,
    unsigned int* __restrict__ n_visible, const float* __restrict__ f3d, const GsLens* __restrict__ lenses) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  unsigned int nv = 0;
  unsigned long long c64 = 0;
  if (i < n) {
    float p[3], q[4], s[3], raw_s[3], qn, s0[3], f3, dl2o3;
    fused_project_load<TIER>(pos, quat, scale, f3d, i, scale_act, p, q, s, raw_s, qn, s0, f3, dl2o3);
    const float opa_raw = opa[i];
    float rgb_raw[3] = {0.f, 0.f, 0.f};
    if (K == 0 && d == 3) {
      rgb_raw[0] = rgb[3 * i];
      rgb_raw[1] = rgb[3 * i + 1];
      rgb_raw[2] = rgb[3 * i + 2];
    }
    for (int v = 0; v < n_views; ++v) {
      const GsView vw = views[v];
      bool vis = false;
      c64 += fused_project_one<K, TIER>(rgb, i, d, vw.cam, vw.grid, near_plane, vw.half_w, vw.half_h, vw.filt, p, q,
                                        s, opa_raw, rgb_raw, (uint32_t)(v * vw.grid.nty), v * n + i, rec, rect, count,
                                        dkey, mask, vis, f3, dl2o3, lenses + v);
      nv += vis ? 1u : 0u;
    }
  }
  __shared__ unsigned long long wsum[kBlock / 32];
  __shared__ unsigned int wvis[kBlock / 32];
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    c64 += __shfl_xor_sync(0xffffffffu, c64, o);
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
  }
  if ((threadIdx.x & 31) == 0) {
    wsum[threadIdx.x >> 5] = c64;
    wvis[threadIdx.x >> 5] = nv;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long tot = 0;
    unsigned int tv = 0;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) {
      tot += wsum[w];
      tv += wvis[w];
    }
    if (tv) atomicAdd(n_visible, tv);
    if (tot) atomicAdd(reinterpret_cast<unsigned long long*>(n_visible + 2), tot);
  }
}

// Segment-sums the per-instance gradient records of each Gaussian (its instances occupy the
// contiguous rows offsets_g[i] .. + count[i]) and chains them to the RAW parameters.  No
// atomics anywhere: the result is deterministic.  Row layout (GW floats): d/d{x, y, ca, cb, cc,
// l2o} then D colour gradients (activated RGB for D == 3, raw SH coefficients otherwise).
// Destination of a run of `cnt` consecutive gradient floats that would land at `local` in this
// rank's flat bucket.  W == 0: the bucket itself.  W > 0 (data-parallel push, SURVEY.md §8e): the
// bucket is cut into W slices of `per` floats owned by rank 0..W-1; floats of another rank's slice
// are stored straight into slot `rank` of that owner's staging buffer over NVLink, so the reduce
// half of the gradient exchange overlaps this kernel.  Returns nullptr when the run straddles two
// slices (the caller then stores element by element).
template <int W>
__device__ __forceinline__ float* push_dst(const GsGradPush& P, float* local, int cnt) {
  if (W == 0) return local;
  const uint32_t idx = (uint32_t)(local - P.bucket);
  const uint32_t owner = idx / P.per;
  if (cnt > 1 && (idx + (uint32_t)cnt - 1) / P.per != owner) return nullptr;
  if (owner == (uint32_t)P.rank) return local;
  float* st = P.staging[0];
#pragma unroll
  for (int p = 1; p < (W > 0 ? W : 1); ++p)
    if (owner == (uint32_t)p) st = P.staging[p];
  return st + (size_t)P.rank * P.per + (idx - owner * P.per);
}

template <int W, int CNT>
__device__ __forceinline__ void push_store(const GsGradPush& P, float* local, const float* v) {
  float* dst = push_dst<W>(P, local, CNT);
  if (dst) {
#pragma unroll
    for (int k = 0; k < CNT; ++k) dst[k] = v[k];
  } else {
#pragma unroll
    for (int k = 0; k < CNT; ++k) *push_dst<W>(P, local + k, 1) = v[k];
  }
}

// One view's share of Gaussian i's parameter gradients over its rows o0 .. o1 - 1 of grad_inst (GW floats each), with
// the loaded parameters p, q, s, raw_s, qn, opa_raw and rgb_raw (D == 3) or coef (KG > 0): acc receives the row sums,
// then gp, gq_raw, gs_raw, go and the colour gradients (acc + 6 for D == 3 and per-pixel SH, gsh for KG > 0) are formed.
// DT: the blend backward stored dL/d|p_c| in the row's pad column 6 + DC (aux depth gradient); it enters as g_xyd[2]
// and reaches pos through p_c / |p_c|.  Without it depth is only a sort key.
// KG = 9 / 16: SH evaluated once per Gaussian (fused_project_one<KG>): the rows carry dL/d(colour) like RGB rows
// (GW = GS_GREC); the D = 3 KG coefficient gradients and the view-direction term are formed here.
// (cam and filt are taken by value, as the kernel parameters they are: by reference, the KG = 0 instantiations would
// no longer compile to the code fused_project_bwd_kernel had before the body was shared.)
// CG (camera gradient): also adds this view's share of dL/d(rot, tran) to cg[12] (gs_cam_grad_add plus the
// view-direction term of per-Gaussian SH); the parameter gradients are the same bits either way.
// TIER, the forward's (fused_project_one):
//   >= GS_TIER_FILT2D: the conic is chained with the filtered covariance, and the compensation's gradient is added to
//     dL/dcov.
//   >= GS_TIER_FILT3D: s is the 3-D filtered scale s', s0 the activated one and f3 the filter: dL/ds' is chained to
//     dL/ds with the compensation's term (gs_filter3d_backward) before the raw-scale chain.
//   GS_TIER_LENS: the conic's gradient is that of the lensed covariance, and gs_lens_backward takes the mean and
//     covariance gradients back through the lens `lens` before the projection backward.
template <int D, int GW, bool DT, int KG, int TIER, bool CG>
__device__ __forceinline__ void fused_project_bwd_one(
    GsCam cam, float near_plane, float half_w, float half_h, GsFilter2d filt, int scale_act, uint32_t o0, uint32_t o1,
    const float* __restrict__ grad_inst, const uint32_t* __restrict__ row_epoch, uint32_t epoch, const float (&p)[3],
    const float (&q)[4], const float (&s)[3], const float (&raw_s)[3], float qn, const float (&s0)[3], float f3,
    float opa_raw, const float (&rgb_raw)[3], const float (&coef)[KG ? D : 1], float (&acc)[GW],
    float (&gsh)[KG ? D : 1], float (&gp)[3], float (&gq_raw)[4], float (&gs_raw)[3], float& go, float* cg,
    const GsLens& lens) {
  static_assert(KG == 0 || (D == 3 * KG && GW == GS_GREC), "per-Gaussian SH: 3K coefficients, RGB gradient rows");
  static_assert(!CG || GW == GS_GREC, "camera gradient: RGB gradient rows");
  constexpr bool F = TIER >= GS_TIER_FILT2D, G3 = TIER >= GS_TIER_FILT3D, L = TIER == GS_TIER_LENS;
  constexpr int DC = KG ? 3 : D;   // colour columns of a gradient row
  {
    // The rows are summed one by one in row order.  For an RGB frame the rows are loaded in groups: the tags of four
    // rows at once, then the live rows among them (48 registers of payload), so that a Gaussian with a few instances
    // waits for two round trips to HBM per group instead of two per row (H100, C3: 0.235 -> 0.230 ms).  Grouping only
    // the tags and loading the rows one at a time was slower (RGB 0.245 ms; per-pixel SH, D = 27: 0.496 -> 0.526 ms),
    // and so was the grouped loop with per-Gaussian SH of degree 2 (80 -> 99 registers, 0.409 -> 0.464 ms): those
    // kernels keep the plain loop.  An instance its (saturated) tile did not reach has a stale tag and contributes
    // nothing.
    if constexpr (GW > GS_GREC || KG > 0) {
      for (uint32_t r = o0; r < o1; ++r) {
        if (row_epoch[r] != epoch) continue;
        const float4* row = reinterpret_cast<const float4*>(grad_inst + (size_t)r * GW);
#pragma unroll
        for (int qq = 0; qq < GW / 4; ++qq) {
          const float4 v = row[qq];
          acc[4 * qq] += v.x;
          acc[4 * qq + 1] += v.y;
          acc[4 * qq + 2] += v.z;
          acc[4 * qq + 3] += v.w;
        }
      }
    } else {
      constexpr int kGroup = 4;
      for (uint32_t r0 = o0; r0 < o1; r0 += kGroup) {
        bool live[kGroup];
#pragma unroll
        for (int j = 0; j < kGroup; ++j) live[j] = r0 + j < o1 && row_epoch[r0 + j] == epoch;
        float4 v[kGroup][GW / 4];
#pragma unroll
        for (int j = 0; j < kGroup; ++j) {
          const float4* row = reinterpret_cast<const float4*>(grad_inst + (size_t)(r0 + j) * GW);
#pragma unroll
          for (int qq = 0; qq < GW / 4; ++qq) v[j][qq] = live[j] ? row[qq] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < kGroup; ++j) {
          if (!live[j]) continue;
#pragma unroll
          for (int qq = 0; qq < GW / 4; ++qq) {
            acc[4 * qq] += v[j][qq].x;
            acc[4 * qq + 1] += v[j][qq].y;
            acc[4 * qq + 2] += v[j][qq].z;
            acc[4 * qq + 3] += v[j][qq].w;
          }
        }
      }
    }
    GsProj o = gs_project(cam, p, q, s, near_plane, L ? kInf : half_w, L ? kInf : half_h);
    float J[4];                                                // L: the lens Jacobian
    if constexpr (L) gs_lens_project(lens, o, half_w, half_h, J);
    float fk[4];                                               // F: d l2o / d cov of the compensation
    if constexpr (F) {
      const GsFilter2dOut fo = gs_filter2d(filt, o.a, o.b, o.c, o.d);
      o.a = fo.a;
      o.d = fo.d;
#pragma unroll
      for (int j = 0; j < 4; ++j) fk[j] = fo.k[j];
    }
    // conic (ca, cb, cc) = (d, b+c, a) * sc,  sc = log2e / (2 det + 1e-14)
    float det = o.a * o.d - o.b * o.c;
    double pn = 2.0 * (double)det + 1e-14;
    float sc = (float)((double)GS_LOG2E / pn);
    float kk = 2.f * sc * sc / GS_LOG2E;                      // d sc / d det = -kk
    float gsc = acc[2] * o.d + acc[3] * (o.b + o.c) + acc[4] * o.a;
    float gcov[4];
    gcov[0] = acc[4] * sc - gsc * kk * o.d;                   // d det/da =  d
    gcov[1] = acc[3] * sc + gsc * kk * o.c;                   // d det/db = -c
    gcov[2] = acc[3] * sc + gsc * kk * o.b;                   // d det/dc = -b
    gcov[3] = acc[2] * sc - gsc * kk * o.a;                   // d det/dd =  a
    if constexpr (F) {
#pragma unroll
      for (int j = 0; j < 4; ++j) gcov[j] += acc[5] * fk[j];
    }
    static_assert(!DT || 6 + DC < GW, "no pad column for the depth gradient");
    float gxyd[3] = {acc[0], acc[1], DT ? acc[6 + DC] : 0.f};   // without DT depth is only a sort key
    if constexpr (L) gs_lens_backward(J, gxyd, gcov);
    float gq[4], gsv[3];
    if constexpr (CG) {
      float gc[3], gjw[6];
      gs_project_backward_cam(cam, p, q, s, gxyd, gcov, gp, gq, gsv, gc, gjw);
      gs_cam_grad_add(cam, p, gc, gjw, cg);
    } else {
      gs_project_backward(cam, p, q, s, gxyd, gcov, gp, gq, gsv);
    }
    if constexpr (G3) gs_filter3d_backward(f3, s0, s, acc[5], gsv);
    if constexpr (KG > 0) {
      // c = sigmoid(l), l_c = sum_k Y_k(dir) coef[c*K + k]: dL/dcoef = g_l,c Y_k; dL/ddir = sum_k w_k dY_k/ddir with
      // w_k = sum_c g_l,c coef[c*K + k]; ddir/dpos = (I - dir dir^T) / |pos - C|
      float dir[3], il, Y[KG], l[3], gl[3], w[KG], gd[3];
      view_dir(cam, p, dir, il);
      gs_sh::sh_basis<KG>(dir[0], dir[1], dir[2], Y);
      sh_logits<KG>(coef, Y, l);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float sg = gs_sigmoid(l[c]);
        gl[c] = acc[6 + c] * sg * (1.f - sg);
      }
#pragma unroll
      for (int k = 0; k < KG; ++k) {
#pragma unroll
        for (int c = 0; c < 3; ++c) gsh[c * KG + k] = gl[c] * Y[k];
        w[k] = gl[0] * coef[k] + gl[1] * coef[KG + k] + gl[2] * coef[2 * KG + k];
      }
      gs_sh::sh_basis_grad<KG>(dir[0], dir[1], dir[2], w, gd);
      const float dd = dir[0] * gd[0] + dir[1] * gd[1] + dir[2] * gd[2];
#pragma unroll
      for (int j = 0; j < 3; ++j) gp[j] += (gd[j] - dir[j] * dd) * il;
      if constexpr (CG) {
        // the direction leaves from u = pos + R^T t: g_u = il v (the term just added to gp) gives dL/dt += R g_u and
        // dL/dR += t g_u^T.  il is applied last, so that no product v * il other than gp's exists: gp keeps the
        // contraction it has in the kernels without CG, bit for bit.
        float v[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) v[j] = gd[j] - dir[j] * dd;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
          for (int j = 0; j < 3; ++j) cg[3 * r + j] += (cam.t[r] * v[j]) * il;
          cg[9 + r] += (cam.r[3 * r] * v[0] + cam.r[3 * r + 1] * v[1] + cam.r[3 * r + 2] * v[2]) * il;
        }
      }
    }
    // quat normalisation backward: q = r/|r|
    float dot = q[0] * gq[0] + q[1] * gq[1] + q[2] * gq[2] + q[3] * gq[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) gq_raw[k] = (gq[k] - q[k] * dot) / qn;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (scale_act == GS_SCALE_ABS)
        gs_raw[k] = gsv[k] * (raw_s[k] > 0.f ? 1.f : (raw_s[k] < 0.f ? -1.f : 0.f));
      else
        gs_raw[k] = gsv[k] * expf(fminf(fmaxf(raw_s[k], -1.f), 1.f));   // renderer.py:98-100
    }
    float op = gs_sigmoid(opa_raw);
    // l2o = log2(op):  d/d logit = d_l2o / (op ln2) * op (1-op) = d_l2o (1-op) / ln2
    go = acc[5] * (1.f - op) / GS_LN2;
    if (D == 3) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float c = gs_sigmoid(rgb_raw[k]);
        acc[6 + k] *= c * (1.f - c);
      }
    }
  }
}

// The parameter gradients of Gaussian i to the caller's tensors (no push).  Per-Gaussian and per-pixel SH colour (D != 3)
// stage the warp's coefficient rows: every thread of the warp takes part, `valid` or not.
template <int D>
__device__ __forceinline__ void fused_project_bwd_store(int i, int n, bool valid, const float* gcol, const float (&gp)[3],
                                                        const float (&gs_raw)[3], const float (&gq_raw)[4], float go,
                                                        float* __restrict__ g_pos, float* __restrict__ g_rgb,
                                                        float* __restrict__ g_opa, float* __restrict__ g_quat,
                                                        float* __restrict__ g_scale) {
  constexpr bool kStagedRgb = D != 3;
  if constexpr (kStagedRgb) {
    // The 32 Gaussians of a warp own 32 * D contiguous floats of g_rgb.  One strided 4-byte store per coefficient
    // makes every store a partial-sector write (read-modify-write under ECC: 8x the bytes): the rows go through
    // shared memory and leave as whole sectors.
    // D = 48: two passes of 24 floats (96-byte, sector-aligned pieces); D = 27: the whole 32 x 108-byte span.
    constexpr int HW = (D % 8 == 0) ? D / 2 : D;
    __shared__ float stage[kBlock / 32][32][HW + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i0 = blockIdx.x * kBlock + warp * 32;
    const int nrow = min(32, n - i0);
#pragma unroll
    for (int pass = 0; pass < D / HW; ++pass) {
      __syncwarp();
#pragma unroll
      for (int k = 0; k < HW; ++k) stage[warp][lane][k] = gcol[pass * HW + k];
      __syncwarp();
      if (HW == D) {
        float* dst = g_rgb + (size_t)i0 * D;
        for (int t = lane; t < nrow * D; t += 32) dst[t] = stage[warp][t / D][t % D];
      } else {
        for (int t = lane; t < nrow * HW; t += 32) {
          const int g = t / HW, c = t % HW;
          g_rgb[(size_t)(i0 + g) * D + pass * HW + c] = stage[warp][g][c];
        }
      }
    }
    if (!valid) return;
  } else {
#pragma unroll
    for (int k = 0; k < D; ++k) g_rgb[(size_t)i * D + k] = gcol[k];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    g_pos[3 * i + k] = gp[k];
    g_scale[3 * i + k] = gs_raw[k];
  }
  reinterpret_cast<float4*>(g_quat)[i] = make_float4(gq_raw[0], gq_raw[1], gq_raw[2], gq_raw[3]);
  g_opa[i] = go;
}

// Camera gradient: the CTA sums its threads' 12-float shares in a fixed order (butterfly shuffles, then the 8 warp sums
// in warp order) into row[12]; cam_grad_finish_kernel adds the rows.  No atomics: the result is bit-deterministic.  Every
// thread of the CTA calls it.
constexpr int kCamGrad = 12;

__device__ __forceinline__ void cam_grad_cta_sum(float (&cg)[kCamGrad], float (&wsum)[kBlock / 32][kCamGrad],
                                                 float* __restrict__ row) {
#pragma unroll
  for (int k = 0; k < kCamGrad; ++k) {
#pragma unroll
    for (int o = 16; o; o >>= 1) cg[k] += __shfl_xor_sync(0xffffffffu, cg[k], o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < kCamGrad; ++k) wsum[threadIdx.x >> 5][k] = cg[k];
  }
  __syncthreads();
  if (threadIdx.x < kCamGrad) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) s += wsum[w][threadIdx.x];
    row[threadIdx.x] = s;
  }
}

// Single-view frame: fused_project_bwd_one over Gaussian i's rows.  (KG, D, GW): RGB (0, 3, 12), per-pixel SH
// (0, 27 / 48, 36 / 56), per-Gaussian SH (9 / 16, 27 / 48, 12).  W == 0: the gradients go to the caller's tensors
// (fused_project_bwd_store); W > 0: through the data-parallel push (push_store).  TIER: the forward's; a lens frame has
// no push.
// CG (camera gradient, gs_render_backward_cam; W = 0, RGB rows): the CTA's sum of its Gaussians' camera terms goes to
// row blockIdx.x of cam_part[gridDim.x][12]; with all five gradient pointers NULL no parameter gradient is stored.
template <int KG, int D, int GW, int W, bool DT, int TIER, bool CG>
__global__ void __launch_bounds__(kBlock) fused_project_bwd_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int scale_act, GsCam cam,
    float near_plane, float half_w, float half_h, const uint32_t* __restrict__ offsets_g,
    const uint32_t* __restrict__ count, const float* __restrict__ grad_inst, const uint32_t* __restrict__ row_epoch,
    uint32_t epoch, float* __restrict__ g_pos, float* __restrict__ g_rgb, float* __restrict__ g_opa,
    float* __restrict__ g_quat, float* __restrict__ g_scale, GsGradPush push, GsFilter2d filt,
    const float* __restrict__ f3d, GsLens lens, float* __restrict__ cam_part) {
  static_assert(TIER != GS_TIER_LENS || W == 0, "the lens runs without a push");
  static_assert(!CG || W == 0, "camera gradient: no push");
  // per-pixel SH takes a principal point only (the host refuses a distortion): the lens map folds to the identity
  if constexpr (KG == 0 && D != 3) lens.model = GS_LENS_PINHOLE;
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const bool valid = i < n;
  float cg[kCamGrad];
#pragma unroll
  for (int k = 0; k < kCamGrad; ++k) cg[k] = 0.f;
  // SH colour on one GPU: the warp writes its coefficient gradients together (fused_project_bwd_store), so threads past
  // n stay
  if (valid || (D != 3 && W == 0)) {
    float gp[3] = {0.f, 0.f, 0.f}, gq_raw[4] = {0.f, 0.f, 0.f, 0.f}, gs_raw[3] = {0.f, 0.f, 0.f};
    float go = 0.f;
    float acc[GW];
#pragma unroll
    for (int k = 0; k < GW; ++k) acc[k] = 0.f;
    float gsh[KG ? D : 1];                    // KG: coefficient gradients
#pragma unroll
    for (int k = 0; k < (KG ? D : 1); ++k) gsh[k] = 0.f;
    const uint32_t cnt = valid ? count[i] : 0u;
    const uint32_t o0 = valid ? offsets_g[i] : 0u;      // loaded with the count: one round trip, not two
    if (cnt > 0) {
      // issue the parameter loads BEFORE the row loop so that both round trips to HBM overlap
      float p[3], q[4], s[3], raw_s[3], qn, s0[3], f3, dl2o3;
      fused_project_load<TIER>(pos, quat, scale, f3d, i, scale_act, p, q, s, raw_s, qn, s0, f3, dl2o3);
      const float opa_raw = opa[i];
      float rgb_raw[3] = {0.f, 0.f, 0.f};
      float coef[KG ? D : 1];
      if constexpr (KG > 0) {
#pragma unroll
        for (int k = 0; k < D; ++k) coef[k] = rgb[(size_t)i * D + k];
      } else if (D == 3) {
        rgb_raw[0] = rgb[3 * i];
        rgb_raw[1] = rgb[3 * i + 1];
        rgb_raw[2] = rgb[3 * i + 2];
      }
      fused_project_bwd_one<D, GW, DT, KG, TIER, CG>(cam, near_plane, half_w, half_h, filt, scale_act, o0, o0 + cnt,
                                                     grad_inst, row_epoch, epoch, p, q, s, raw_s, qn, s0, f3, opa_raw,
                                                     rgb_raw, coef, acc, gsh, gp, gq_raw, gs_raw, go, cg, lens);
    }
    const float* gcol = KG ? gsh : acc + 6;   // the D gradients of this Gaussian's rgb row
    if (!CG || g_pos) {                       // camera only: the pointers are all NULL or all set (uniform)
      if constexpr (W == 0) {
        fused_project_bwd_store<D>(i, n, valid, gcol, gp, gs_raw, gq_raw, go, g_pos, g_rgb, g_opa, g_quat, g_scale);
      } else {
        push_store<W, 3>(push, g_pos + 3 * (size_t)i, gp);
        push_store<W, 3>(push, g_scale + 3 * (size_t)i, gs_raw);
        push_store<W, D>(push, g_rgb + (size_t)i * D, gcol);
        // a quaternion is 4 floats at a 16-byte aligned bucket offset and `per` is a multiple of 4:
        // it never straddles two slices
        *reinterpret_cast<float4*>(push_dst<W>(push, g_quat + 4 * (size_t)i, 1)) =
            make_float4(gq_raw[0], gq_raw[1], gq_raw[2], gq_raw[3]);
        push_store<W, 1>(push, g_opa + i, &go);
      }
    }
  }
  if constexpr (CG) {
    __shared__ float wsum[kBlock / 32][kCamGrad];
    cam_grad_cta_sum(cg, wsum, cam_part + (size_t)blockIdx.x * kCamGrad);
  }
}

// Batched frame: K = 0 RGB, 9 / 16 per-Gaussian SH; DT and TIER as above (views[v].filt, lenses[v]).  Thread i loads
// Gaussian i's parameters once and takes its views in order: view v's share is fused_project_bwd_one over the rows of
// pair v n + i with view v's camera, and the shares are added in view order with no contraction into their last
// products: the sum of B single-view backwards accumulated in view order, to within the FMA contractions the compiler
// chooses differently inside the view loop (measured: 1e-6 relative at most).
// CG (gs_render_backward_batch_cam): also the camera terms of each view, summed per view v by the CTA in
// cam_grad_cta_sum's order into row blockIdx.x of cam_part[v][gridDim.x][12].  The view loop and the sums are then
// uniform across the CTA: threads past n and Gaussians without a row in view v take part with zeros, and a CTA without
// a row in view v stores a zero row (the bits the shuffles would give) without reducing.  With the five gradient
// pointers NULL only cam_part is written.
template <int K, bool DT, int TIER, bool CG>
__global__ void __launch_bounds__(kBlock) fused_project_bwd_batch_kernel(
    const float* __restrict__ pos, const float* __restrict__ rgb, const float* __restrict__ opa,
    const float* __restrict__ quat, const float* __restrict__ scale, int n, int n_views, int scale_act,
    const GsView* __restrict__ views, float near_plane, const uint32_t* __restrict__ offsets_g,
    const uint32_t* __restrict__ count, const float* __restrict__ grad_inst, const uint32_t* __restrict__ row_epoch,
    uint32_t epoch, float* __restrict__ g_pos, float* __restrict__ g_rgb, float* __restrict__ g_opa,
    float* __restrict__ g_quat, float* __restrict__ g_scale, const float* __restrict__ f3d,
    const GsLens* __restrict__ lenses, float* __restrict__ cam_part) {
  constexpr int D = K ? 3 * K : 3, GW = GS_GREC;
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const bool valid = i < n;
  if (!CG && !valid && D == 3) return;   // SH: the whole warp stages its coefficient rows (fused_project_bwd_store)
  float gp[3] = {0.f, 0.f, 0.f}, gq_raw[4] = {0.f, 0.f, 0.f, 0.f}, gs_raw[3] = {0.f, 0.f, 0.f}, go = 0.f;
  float gcol[D];
#pragma unroll
  for (int k = 0; k < D; ++k) gcol[k] = 0.f;
  float p[3] = {0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f}, s[3] = {0.f, 0.f, 0.f}, raw_s[3] = {0.f, 0.f, 0.f};
  float qn = 1.f, s_act[3], f3 = 0.f, dl2o3, opa_raw = 0.f, rgb_raw[3] = {0.f, 0.f, 0.f};
  float coef[K ? D : 1];
#pragma unroll
  for (int k = 0; k < (K ? D : 1); ++k) coef[k] = 0.f;
  if (valid) {
    fused_project_load<TIER>(pos, quat, scale, f3d, i, scale_act, p, q, s, raw_s, qn, s_act, f3, dl2o3);
    opa_raw = opa[i];
    if constexpr (K > 0) {
#pragma unroll
      for (int k = 0; k < D; ++k) coef[k] = rgb[(size_t)i * D + k];
    } else {
      rgb_raw[0] = rgb[3 * i];
      rgb_raw[1] = rgb[3 * i + 1];
      rgb_raw[2] = rgb[3 * i + 2];
    }
  }
  __shared__ float wsum[kBlock / 32][kCamGrad];
  for (int v = 0; v < n_views; ++v) {
    const int j = v * n + i;
    const uint32_t cnt = valid ? count[j] : 0u;
    float cg[kCamGrad];
#pragma unroll
    for (int k = 0; k < kCamGrad; ++k) cg[k] = 0.f;
    if (cnt > 0) {
      const uint32_t o0 = offsets_g[j];
      const GsView vw = views[v];
      const GsLens ln = TIER == GS_TIER_LENS ? lenses[v] : GsLens{};
      // the activated scale, formed again from raw_s in each view (gs_load_activated's expression: the same bits):
      // kept live across the view loop instead, it costs 3-25 registers and a CTA per SM in the RGB kernels
      float s0[3];
      if constexpr (TIER >= GS_TIER_FILT3D) {
#pragma unroll
        for (int k = 0; k < 3; ++k) s0[k] = (scale_act == GS_SCALE_ABS) ? (fabsf(raw_s[k]) + 1e-4f) : expf(raw_s[k]);
      }
      float acc[GW], gsh[K ? D : 1], vp[3], vq[4], vs[3], vo = 0.f;
#pragma unroll
      for (int k = 0; k < GW; ++k) acc[k] = 0.f;
      fused_project_bwd_one<D, GW, DT, K, TIER, CG>(vw.cam, near_plane, vw.half_w, vw.half_h, vw.filt, scale_act, o0,
                                                    o0 + cnt, grad_inst, row_epoch, epoch, p, q, s, raw_s, qn, s0, f3,
                                                    opa_raw, rgb_raw, coef, acc, gsh, vp, vq, vs, vo, cg, ln);
      const float* vc = K ? gsh : acc + 6;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        gp[k] = __fadd_rn(gp[k], vp[k]);
        gs_raw[k] = __fadd_rn(gs_raw[k], vs[k]);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) gq_raw[k] = __fadd_rn(gq_raw[k], vq[k]);
      go = __fadd_rn(go, vo);
#pragma unroll
      for (int k = 0; k < D; ++k) gcol[k] = __fadd_rn(gcol[k], vc[k]);
    }
    if constexpr (CG) {
      float* row = cam_part + ((size_t)v * gridDim.x + blockIdx.x) * kCamGrad;
      // the barrier also keeps the previous view's readers of wsum ahead of this view's writers
      if (__syncthreads_or(cnt > 0)) {
        cam_grad_cta_sum(cg, wsum, row);
      } else if (threadIdx.x < kCamGrad) {
        row[threadIdx.x] = 0.f;
      }
    }
  }
  if (CG && !g_pos) return;              // camera only (the pointers are all NULL or all set: uniform)
  if (!valid && D == 3) return;          // SH: the whole warp stages its coefficient rows (fused_project_bwd_store)
  fused_project_bwd_store<D>(i, n, valid, gcol, gp, gs_raw, gq_raw, go, g_pos, g_rgb, g_opa, g_quat, g_scale);
}

// One CTA: grad_cam[k] = sum over the `rows` rows of cam_part[., k] in fp64, in a fixed order (strided per-thread sums,
// butterfly shuffles, warp sums in warp order).  rows == 0 (no Gaussian) writes zeros.
__device__ __forceinline__ void cam_grad_finish_rows(const float* __restrict__ cam_part, int rows,
                                                     float* __restrict__ grad_cam) {
  double s[kCamGrad];
#pragma unroll
  for (int k = 0; k < kCamGrad; ++k) s[k] = 0.0;
  for (int r = threadIdx.x; r < rows; r += kBlock) {
#pragma unroll
    for (int k = 0; k < kCamGrad; ++k) s[k] += (double)cam_part[(size_t)r * kCamGrad + k];
  }
  __shared__ double wsum[kBlock / 32][kCamGrad];
#pragma unroll
  for (int k = 0; k < kCamGrad; ++k) {
#pragma unroll
    for (int o = 16; o; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < kCamGrad; ++k) wsum[threadIdx.x >> 5][k] = s[k];
  }
  __syncthreads();
  if (threadIdx.x < kCamGrad) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) t += wsum[w][threadIdx.x];
    grad_cam[threadIdx.x] = (float)t;
  }
}

__global__ void __launch_bounds__(kBlock) cam_grad_finish_kernel(const float* __restrict__ cam_part, int rows,
                                                                  float* __restrict__ grad_cam) {
  cam_grad_finish_rows(cam_part, rows, grad_cam);
}

// A batched frame: CTA v sums view v's `rows` rows, cam_part[v][rows][12], into grad_cams[v][12]
__global__ void __launch_bounds__(kBlock) cam_grad_finish_batch_kernel(const float* __restrict__ cam_part, int rows,
                                                                        float* __restrict__ grad_cams) {
  cam_grad_finish_rows(cam_part + (size_t)blockIdx.x * rows * kCamGrad, rows, grad_cams + blockIdx.x * kCamGrad);
}

}  // namespace

// The legacy API passes rot/tran as DEVICE pointers (torch tensors); the kernels read
// them through the read-only path so that no host synchronisation is needed.
namespace {
__global__ void __launch_bounds__(kBlock) project_fwd_kernel_p(const float* pos, const float* quat,
                                                                const float* scale, const float* rot,
                                                                const float* tran, int n, float near_plane,
                                                                float half_w, float half_h, float* res_pos,
                                                                float* res_cov, int64_t* mask) {
  GsCam cam;
#pragma unroll
  for (int k = 0; k < 9; ++k) cam.r[k] = __ldg(rot + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) cam.t[k] = __ldg(tran + k);
  int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  float4 q4 = reinterpret_cast<const float4*>(quat)[i];
  float q[4] = {q4.x, q4.y, q4.z, q4.w};
  float s[3] = {scale[3 * i], scale[3 * i + 1], scale[3 * i + 2]};
  GsProj o = gs_project(cam, p, q, s, near_plane, half_w, half_h);
  if (!o.visible) return;
  mask[i] = 1;
  res_pos[3 * i] = o.x;
  res_pos[3 * i + 1] = o.y;
  res_pos[3 * i + 2] = o.depth;
  reinterpret_cast<float4*>(res_cov)[i] = make_float4(o.a, o.b, o.c, o.d);
}

__global__ void __launch_bounds__(kBlock) project_bwd_kernel_p(const float* pos, const float* quat,
                                                                const float* scale, const float* rot,
                                                                const float* tran, int n, const float* go_pos,
                                                                const float* go_cov, const int64_t* mask,
                                                                float* gi_pos, float* gi_quat, float* gi_scale) {
  GsCam cam;
#pragma unroll
  for (int k = 0; k < 9; ++k) cam.r[k] = __ldg(rot + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) cam.t[k] = __ldg(tran + k);
  int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  if (mask[i] == 0) return;
  float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  float4 q4 = reinterpret_cast<const float4*>(quat)[i];
  float q[4] = {q4.x, q4.y, q4.z, q4.w};
  float s[3] = {scale[3 * i], scale[3 * i + 1], scale[3 * i + 2]};
  float gx[3] = {go_pos[3 * i], go_pos[3 * i + 1], go_pos[3 * i + 2]};
  float4 gc4 = reinterpret_cast<const float4*>(go_cov)[i];
  float gc[4] = {gc4.x, gc4.y, gc4.z, gc4.w};
  float gp[3], gq[4], gs[3];
  gs_project_backward(cam, p, q, s, gx, gc, gp, gq, gs);
  gi_pos[3 * i] = gp[0];
  gi_pos[3 * i + 1] = gp[1];
  gi_pos[3 * i + 2] = gp[2];
  reinterpret_cast<float4*>(gi_quat)[i] = make_float4(gq[0], gq[1], gq[2], gq[3]);
  gi_scale[3 * i] = gs[0];
  gi_scale[3 * i + 1] = gs[1];
  gi_scale[3 * i + 2] = gs[2];
}

__global__ void __launch_bounds__(kBlock) w2c_fwd_kernel_p(const float* pos, const float* rot, const float* tran,
                                                            int n, float* res) {
  GsCam cam;
#pragma unroll
  for (int k = 0; k < 9; ++k) cam.r[k] = __ldg(rot + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) cam.t[k] = __ldg(tran + k);
  int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  float pc[3];
  gs_world_to_cam(cam, p, pc);
  res[3 * i] = pc[0];
  res[3 * i + 1] = pc[1];
  res[3 * i + 2] = pc[2];
}

__global__ void __launch_bounds__(kBlock) w2c_bwd_kernel_p(const float* go, const float* rot, int n, float* gi) {
  float r[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) r[k] = __ldg(rot + k);
  int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  float g[3] = {go[3 * i], go[3 * i + 1], go[3 * i + 2]};
#pragma unroll
  for (int k = 0; k < 3; ++k) gi[3 * i + k] = g[0] * r[k] + g[1] * r[3 + k] + g[2] * r[6 + k];
}
}  // namespace

static inline int grid_for(int n) { return (n + kBlock - 1) / kBlock; }

extern "C" int gs_project_fwd(const float* pos, const float* quat, const float* scale, const float* rot,
                              const float* tran, int n, float near_plane, float half_width, float half_height,
                              float* res_pos, float* res_cov, int64_t* mask, gs_stream_t stream) {
  if (n < 0) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_project_fwd: n < 0");
  if (n == 0) return 0;
  project_fwd_kernel_p<<<grid_for(n), kBlock, 0, (cudaStream_t)stream>>>(pos, quat, scale, rot, tran, n, near_plane,
                                                                        half_width, half_height, res_pos, res_cov,
                                                                        mask);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_project_bwd(const float* pos, const float* quat, const float* scale, const float* rot,
                              const float* tran, const float* gradout_pos, const float* gradout_cov,
                              const int64_t* mask, int n, float* gradin_pos, float* gradin_quat,
                              float* gradin_scale, gs_stream_t stream) {
  if (n < 0) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_project_bwd: n < 0");
  if (n == 0) return 0;
  project_bwd_kernel_p<<<grid_for(n), kBlock, 0, (cudaStream_t)stream>>>(pos, quat, scale, rot, tran, n, gradout_pos,
                                                                        gradout_cov, mask, gradin_pos, gradin_quat,
                                                                        gradin_scale);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_w2c_fwd(const float* pos, const float* rot, const float* tran, int n, float* res,
                          gs_stream_t stream) {
  if (n <= 0) return n == 0 ? 0 : gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_w2c_fwd: n < 0");
  w2c_fwd_kernel_p<<<grid_for(n), kBlock, 0, (cudaStream_t)stream>>>(pos, rot, tran, n, res);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_w2c_bwd(const float* grad_out, const float* rot, int n, float* grad_in, gs_stream_t stream) {
  if (n <= 0) return n == 0 ? 0 : gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_w2c_bwd: n < 0");
  w2c_bwd_kernel_p<<<grid_for(n), kBlock, 0, (cudaStream_t)stream>>>(grad_out, rot, n, grad_in);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_jacobian(const float* pos_cam, int n, float* jac, gs_stream_t stream) {
  if (n <= 0) return n == 0 ? 0 : gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_jacobian: n < 0");
  jacobian_kernel<<<grid_for(n), kBlock, 0, (cudaStream_t)stream>>>(pos_cam, n, jac);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}


namespace {
template <int V>
using Int = std::integral_constant<int, V>;

// The fused projection's one map from a frame's configuration to a kernel instantiation: calls
// launch(KG, D, GW, TIER, DT, W), each a std::integral_constant, and returns cudaGetLastError(), or
// cudaErrorInvalidValue for a configuration no instantiation serves.
//   (d, sh_gaussian) -> (KG, D, GW): per-Gaussian SH d = 27 / 48 -> (9 / 16, d, GS_GREC); otherwise RGB d = 3 ->
//     (0, 3, GS_GREC) and per-pixel SH d = 27 / other -> (0, 27, 36) / (0, 48, 56)
//   tier (GsTier) -> TIER; dt -> DT (kDT families, false otherwise); world 0 / 2 / 4 / 8 -> W (kPush families; a lens
//     frame has no push)
template <bool kDT, bool kPush, class Launch>
cudaError_t fused_project_dispatch(int d, bool sh_gaussian, int tier, bool dt, int world, Launch&& launch) {
  auto by_world = [&](auto kg, auto dd, auto gw, auto t, auto dtc) {
    if (world == 0) {
      launch(kg, dd, gw, t, dtc, Int<0>{});
      return cudaGetLastError();
    }
    if constexpr (kPush && t != GS_TIER_LENS) {
      if (world == 2) launch(kg, dd, gw, t, dtc, Int<2>{});
      else if (world == 4) launch(kg, dd, gw, t, dtc, Int<4>{});
      else if (world == 8) launch(kg, dd, gw, t, dtc, Int<8>{});
      else return cudaErrorInvalidValue;
      return cudaGetLastError();
    }
    return cudaErrorInvalidValue;
  };
  auto by_dt = [&](auto kg, auto dd, auto gw, auto t) {
    if constexpr (kDT) {
      if (dt) return by_world(kg, dd, gw, t, std::true_type{});
    }
    return by_world(kg, dd, gw, t, std::false_type{});
  };
  auto by_tier = [&](auto kg, auto dd, auto gw) {
    switch (tier) {
      case GS_TIER_NONE: return by_dt(kg, dd, gw, Int<GS_TIER_NONE>{});
      case GS_TIER_FILT2D: return by_dt(kg, dd, gw, Int<GS_TIER_FILT2D>{});
      case GS_TIER_FILT3D: return by_dt(kg, dd, gw, Int<GS_TIER_FILT3D>{});
      default: return by_dt(kg, dd, gw, Int<GS_TIER_LENS>{});
    }
  };
  if (sh_gaussian) {
    if (d == 27) return by_tier(Int<9>{}, Int<27>{}, Int<GS_GREC>{});
    if (d == 48) return by_tier(Int<16>{}, Int<48>{}, Int<GS_GREC>{});
    return cudaErrorInvalidValue;
  }
  if (d == 3) return by_tier(Int<0>{}, Int<3>{}, Int<GS_GREC>{});
  if (d == 27) return by_tier(Int<0>{}, Int<27>{}, Int<36>{});
  return by_tier(Int<0>{}, Int<48>{}, Int<56>{});
}
}  // namespace

cudaError_t gs_launch_fused_project(const float* pos, const float* rgb, const float* opa, const float* quat,
                                    const float* scale, int n, int d, int scale_act, const GsCam& cam,
                                    const GsTileGrid& grid, float near_plane, float half_w, float half_h,
                                    GsRec* rec, uint2* rect, uint32_t* count, uint32_t* dkey, int64_t* mask,
                                    unsigned int* n_visible, cudaStream_t st, bool sh_gaussian, const GsFilter2d* filt,
                                    const float* f3d, const GsLens* lens) {
  if (n == 0) return cudaSuccess;
  const GsFilter2d f2 = filt ? *filt : GsFilter2d{};
  const GsLens ln = lens ? *lens : GsLens{};
  return fused_project_dispatch<false, false>(
      d, sh_gaussian, gs_tier(filt, f3d, lens), false, 0, [&](auto kg, auto, auto, auto t, auto, auto) {
        fused_project_kernel<kg, t><<<grid_for(n), kBlock, 0, st>>>(pos, rgb, opa, quat, scale, n, d, scale_act, cam,
                                                                    grid, near_plane, half_w, half_h, rec, rect, count,
                                                                    dkey, mask, n_visible, f2, f3d, ln);
      });
}

cudaError_t gs_launch_fused_project_bwd(const float* pos, const float* rgb, const float* opa, const float* quat,
                                        const float* scale, int n, int d, int scale_act, const GsCam& cam,
                                        float near_plane, float half_w, float half_h, const uint32_t* offsets_g,
                                        const uint32_t* count, const float* grad_inst, const uint32_t* row_epoch, uint32_t epoch,
                                        float* g_pos, float* g_rgb, float* g_opa,
                                        float* g_quat, float* g_scale, const GsGradPush& push, cudaStream_t st,
                                        bool depth_grad, bool sh_gaussian, const GsFilter2d* filt, const float* f3d,
                                        const GsLens* lens) {
  if (n == 0) return cudaSuccess;
  const GsFilter2d f2 = filt ? *filt : GsFilter2d{};
  const GsLens ln = lens ? *lens : GsLens{};
  return fused_project_dispatch<true, true>(
      d, sh_gaussian, gs_tier(filt, f3d, lens), depth_grad, push.world, [&](auto kg, auto dd, auto gw, auto t, auto dt, auto w) {
        fused_project_bwd_kernel<kg, dd, gw, w, dt, t, false><<<grid_for(n), kBlock, 0, st>>>(
            pos, rgb, opa, quat, scale, n, scale_act, cam, near_plane, half_w, half_h, offsets_g, count, grad_inst,
            row_epoch, epoch, g_pos, g_rgb, g_opa, g_quat, g_scale, push, f2, f3d, ln, nullptr);
      });
}

size_t gs_cam_grad_workspace_bytes(int n) { return (size_t)grid_for(n) * kCamGrad * sizeof(float); }

cudaError_t gs_launch_fused_project_bwd_cam(const float* pos, const float* rgb, const float* opa, const float* quat,
                                            const float* scale, int n, int d, int scale_act, const GsCam& cam,
                                            float near_plane, float half_w, float half_h, const uint32_t* offsets_g,
                                            const uint32_t* count, const float* grad_inst, const uint32_t* row_epoch,
                                            uint32_t epoch, float* g_pos, float* g_rgb, float* g_opa, float* g_quat,
                                            float* g_scale, float* cam_part, float* grad_cam, cudaStream_t st,
                                            bool depth_grad, bool sh_gaussian, const GsFilter2d* filt,
                                            const float* f3d, const GsLens* lens) {
  if (d != 3 && !(sh_gaussian && (d == 27 || d == 48))) return cudaErrorInvalidValue;
  const GsFilter2d f2 = filt ? *filt : GsFilter2d{};
  const GsLens ln = lens ? *lens : GsLens{};
  if (n > 0) {
    const cudaError_t e = fused_project_dispatch<true, false>(
        d, d != 3, gs_tier(filt, f3d, lens), depth_grad, 0, [&](auto kg, auto, auto, auto t, auto dt, auto) {
          fused_project_bwd_kernel<kg, kg ? 3 * kg : 3, GS_GREC, 0, dt, t, true><<<grid_for(n), kBlock, 0, st>>>(
              pos, rgb, opa, quat, scale, n, scale_act, cam, near_plane, half_w, half_h, offsets_g, count, grad_inst,
              row_epoch, epoch, g_pos, g_rgb, g_opa, g_quat, g_scale, GsGradPush{}, f2, f3d, ln, cam_part);
        });
    if (e != cudaSuccess) return e;
  }
  cam_grad_finish_kernel<<<1, kBlock, 0, st>>>(cam_part, n > 0 ? grid_for(n) : 0, grad_cam);
  return cudaGetLastError();
}

cudaError_t gs_launch_fused_project_batch(const float* pos, const float* rgb, const float* opa, const float* quat,
                                          const float* scale, int n, int n_views, int d, int scale_act,
                                          const GsView* views, float near_plane, GsRec* rec, uint2* rect,
                                          uint32_t* count, uint32_t* dkey, int64_t* mask, unsigned int* n_visible,
                                          cudaStream_t st, bool sh_gaussian, bool filt, const float* f3d,
                                          const GsLens* lenses) {
  if (n == 0) return cudaSuccess;
  if (d != 3 && !(sh_gaussian && (d == 27 || d == 48))) return cudaErrorInvalidValue;
  return fused_project_dispatch<false, false>(
      d, d != 3, gs_tier(filt, f3d, lenses), false, 0, [&](auto kg, auto, auto, auto t, auto, auto) {
        fused_project_batch_kernel<kg, t><<<grid_for(n), kBlock, 0, st>>>(pos, rgb, opa, quat, scale, n, n_views, d,
                                                                          scale_act, views, near_plane, rec, rect,
                                                                          count, dkey, mask, n_visible, f3d, lenses);
      });
}

cudaError_t gs_launch_fused_project_bwd_batch(const float* pos, const float* rgb, const float* opa, const float* quat,
                                              const float* scale, int n, int n_views, int d, int scale_act,
                                              const GsView* views, float near_plane, const uint32_t* offsets_g,
                                              const uint32_t* count, const float* grad_inst, const uint32_t* row_epoch,
                                              uint32_t epoch, float* g_pos, float* g_rgb, float* g_opa, float* g_quat,
                                              float* g_scale, cudaStream_t st, bool depth_grad, bool sh_gaussian,
                                              bool filt, const float* f3d, const GsLens* lenses) {
  if (n == 0) return cudaSuccess;
  if (d != 3 && !(sh_gaussian && (d == 27 || d == 48))) return cudaErrorInvalidValue;
  return fused_project_dispatch<true, false>(
      d, d != 3, gs_tier(filt, f3d, lenses), depth_grad, 0, [&](auto kg, auto, auto, auto t, auto dt, auto) {
        fused_project_bwd_batch_kernel<kg, dt, t, false><<<grid_for(n), kBlock, 0, st>>>(
            pos, rgb, opa, quat, scale, n, n_views, scale_act, views, near_plane, offsets_g, count, grad_inst,
            row_epoch, epoch, g_pos, g_rgb, g_opa, g_quat, g_scale, f3d, lenses, nullptr);
      });
}

cudaError_t gs_launch_fused_project_bwd_batch_cam(const float* pos, const float* rgb, const float* opa,
                                                  const float* quat, const float* scale, int n, int n_views, int d,
                                                  int scale_act, const GsView* views, float near_plane,
                                                  const uint32_t* offsets_g, const uint32_t* count,
                                                  const float* grad_inst, const uint32_t* row_epoch, uint32_t epoch,
                                                  float* g_pos, float* g_rgb, float* g_opa, float* g_quat,
                                                  float* g_scale, float* cam_part, float* grad_cams, cudaStream_t st,
                                                  bool depth_grad, bool sh_gaussian, bool filt, const float* f3d,
                                                  const GsLens* lenses) {
  if (d != 3 && !(sh_gaussian && (d == 27 || d == 48))) return cudaErrorInvalidValue;
  if (n > 0) {
    const cudaError_t e = fused_project_dispatch<true, false>(
        d, d != 3, gs_tier(filt, f3d, lenses), depth_grad, 0, [&](auto kg, auto, auto, auto t, auto dt, auto) {
          fused_project_bwd_batch_kernel<kg, dt, t, true><<<grid_for(n), kBlock, 0, st>>>(
              pos, rgb, opa, quat, scale, n, n_views, scale_act, views, near_plane, offsets_g, count, grad_inst,
              row_epoch, epoch, g_pos, g_rgb, g_opa, g_quat, g_scale, f3d, lenses, cam_part);
        });
    if (e != cudaSuccess) return e;
  }
  cam_grad_finish_batch_kernel<<<n_views, kBlock, 0, st>>>(cam_part, n > 0 ? grid_for(n) : 0, grad_cams);
  return cudaGetLastError();
}
