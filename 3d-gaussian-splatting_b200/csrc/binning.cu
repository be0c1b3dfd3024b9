// Tile binning.  (1) the reference's legacy dense-list API (calc_tile_list / gather_gaussians);
// (2) the fused path: (tile | depth) key emission, and the post-sort pass that derives the
// per-tile ranges and packs the sorted per-instance record streams the blend kernels stream.
#include "internal.h"

namespace {

constexpr int kBlock = 256;

// ---- legacy: reference gaussian.cu:101-250 ---------------------------------------------
__device__ __forceinline__ void append_to_tile(int* tile_n_point, int* list, int max_per_tile, uint32_t tid,
                                               uint32_t pid) {
  // The reference checks capacity non-atomically and then appends at the atomic's old value
  // (gaussian.cu:244-247), which can overrun a row.  Here the count always increases and only
  // in-capacity slots are written; the caller clamps the count (splatter.py:586).
  int old = atomicAdd(tile_n_point + tid, 1);
  if (old < max_per_tile) list[(size_t)max_per_tile * tid + old] = (int)pid;
}

__global__ void tile_list_dist_kernel(const float* __restrict__ pos, const float* __restrict__ top,
                                      const float* __restrict__ bottom, const float* __restrict__ left,
                                      const float* __restrict__ right, int* tile_n_point, int* list, uint32_t n,
                                      uint32_t n_tiles, int max_per_tile, float thresh) {
  uint32_t pid = blockDim.x * blockIdx.x + threadIdx.x;
  uint32_t tid = blockDim.y * blockIdx.y + threadIdx.y;
  if (pid >= n || tid >= n_tiles) return;
  float cy = (top[tid] + bottom[tid]) / 2;                   // :124-128
  float cx = (left[tid] + right[tid]) / 2;
  float d1 = pos[3 * pid] - cx, d2 = pos[3 * pid + 1] - cy;
  if (d1 * d1 + d2 * d2 < thresh) append_to_tile(tile_n_point, list, max_per_tile, tid, pid);
}

__device__ __forceinline__ bool bbox_of(float cx, float cy, float a, float b, float c, float d, float t2,
                                        float& l, float& r, float& tp, float& bt) {
  float det = a * d - b * c;
  if (det <= 0.f) return false;
  float ai = (float)((double)d / ((double)det + 1e-14));
  float di = (float)((double)a / ((double)det + 1e-14));
  float sx = sqrtf(di * t2 * det), sy = sqrtf(ai * t2 * det);
  r = cx + sx;
  l = cx - sx;
  tp = cy - sy;
  bt = cy + sy;
  return true;
}

__global__ void tile_list_prob_kernel(const float* __restrict__ pos, const float* __restrict__ cov,
                                      const float* __restrict__ top, const float* __restrict__ bottom,
                                      const float* __restrict__ left, const float* __restrict__ right,
                                      int* tile_n_point, int* list, uint32_t n, uint32_t n_tiles, int max_per_tile,
                                      float thresh) {
  uint32_t pid = blockDim.x * blockIdx.x + threadIdx.x;
  uint32_t tid = blockDim.y * blockIdx.y + threadIdx.y;
  if (pid >= n || tid >= n_tiles) return;
  float4 cv = reinterpret_cast<const float4*>(cov)[pid];
  float l, r, tp, bt;
  if (!bbox_of(pos[3 * pid], pos[3 * pid + 1], cv.x, cv.y, cv.z, cv.w, -2.f * logf(thresh), l, r, tp, bt)) return;
  if (!(right[tid] < l || r < left[tid] || bottom[tid] < tp || bt < top[tid]))   // :187
    append_to_tile(tile_n_point, list, max_per_tile, tid, pid);
}

__global__ void __launch_bounds__(kBlock) tile_list_prob2_kernel(const float* __restrict__ pos,
                                                                  const float* __restrict__ cov, GsTileGrid grid,
                                                                  int* tile_n_point, int* list, uint32_t n,
                                                                  int max_per_tile, float thresh) {
  uint32_t pid = blockDim.x * blockIdx.x + threadIdx.x;
  if (pid >= n) return;
  grid.t2 = -2.f * logf(thresh);                              // :233
  float4 cv = reinterpret_cast<const float4*>(cov)[pid];
  uint32_t tx0, tx1, ty0, ty1;
  if (!gs_tile_rect(grid, pos[3 * pid], pos[3 * pid + 1], cv.x, cv.y, cv.z, cv.w, tx0, tx1, ty0, ty1)) return;
  for (uint32_t ty = ty0; ty < ty1; ++ty)
    for (uint32_t tx = tx0; tx < tx1; ++tx) append_to_tile(tile_n_point, list, max_per_tile, tx + ty * grid.ntx, pid);
}

__global__ void gather_kernel(const int* __restrict__ accum, const int* __restrict__ list, int n_tiles,
                              int list_stride, int* __restrict__ gathered, int* __restrict__ tile_ids) {
  // one warp per tile; lanes stride over the tile's entries (coalesced both ways)
  int tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tile >= n_tiles) return;
  int s = accum[tile], e = accum[tile + 1];
  const int* src = list + (size_t)tile * list_stride;
  for (int i = (threadIdx.x & 31); i < e - s; i += 32) {
    gathered[s + i] = src[i];
    tile_ids[s + i] = tile;
  }
}

// ---- fused path ------------------------------------------------------------------------
// Ordering scheme: the (tile, depth, id) order of all M tile-instances is obtained WITHOUT a
// wide M-element sort.  (1) the N Gaussians are stably radix-sorted by depth (32-bit keys, N
// items - cheap); (2) instances are emitted in that order (instance `rank` of the Gaussian at
// sorted position i goes to row offsets_sorted[i] + rank, rank = row-major index inside its
// tile rectangle), so the instance array is already ordered by (depth, id, rank);
// (3) a STABLE radix sort of the M instances on the tile id alone (16-bit key when T <= 65536, else 32-bit;
// only ceil(log2 T) bits are sorted = 2 passes at 1080p, 6 B / item) yields exactly (tile, depth, id).
// The backward writes an instance's gradient record to row ("slot") offsets_g[g] + rank, where
// offsets_g is the exclusive scan of the tile counts in Gaussian-id order: the records of one
// Gaussian are contiguous, and nothing in the pipeline needs a scattered store (scattered
// 4-byte stores are partial-sector read-modify-writes in L2).
// One warp emits the instances of 32 depth-consecutive Gaussians - a CONTIGUOUS range of the key / value arrays -
// cooperatively: lane L writes entries first + L, first + L + 32, ... and finds the owning Gaussian of its entry
// by a 5-step binary search over the warp's offsets (shuffles).  Every store instruction of the warp covers 128
// (values) / 64 (keys) contiguous bytes, i.e. whole 32-byte sectors; the round-1 version (each thread loops over
// its own Gaussian's rectangle) wrote partial sectors, which HBM with ECC turns into read-modify-writes (ncu: 286 MB
// of DRAM traffic for 139 MB of algorithmic bytes).
// The rectangle of the Gaussian comes from the projection's dense rect[N] (8 bytes, 19 MB at C3) rather than from its
// 64-byte record (a 16-byte gather from 154 MB: one DRAM sector per Gaussian), and the sorted id is loaded with the
// offsets, so a thread waits for two round trips before its stores instead of three (H100, C3: 0.104 -> 0.050 ms).
template <typename KeyT>
__global__ void __launch_bounds__(kBlock) emit_keys_kernel(const uint2* __restrict__ rect, const uint32_t* __restrict__ perm,
                                                            const uint32_t* __restrict__ offsets_sorted, int n,
                                                            int ntx, KeyT* __restrict__ keys,
                                                            uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * kBlock + threadIdx.x;      // position in depth order
  const int lane = threadIdx.x & 31;
  const int ic = min(i, n);                              // lanes past the end own an empty range at offsets[n]
  const uint32_t o0 = offsets_sorted[ic], o1 = i < n ? offsets_sorted[i + 1] : o0;
  uint32_t g = i < n ? perm[i] : 0u, rxy = 0, rwh = 1;
  if (o1 > o0) {
    const uint2 rc = rect[g];
    rxy = rc.x;
    rwh = rc.y;
  }
  const uint32_t first = __shfl_sync(0xffffffffu, o0, 0), last = __shfl_sync(0xffffffffu, o1, 31);
  for (uint32_t base = first; base < last; base += 32) {
    const uint32_t e = base + lane;
    int lo = 0, hi = 31;                                 // largest lane whose o0 <= e (ties: the non-empty one is last)
#pragma unroll
    for (int it = 0; it < 5; ++it) {
      const int mid = (lo + hi + 1) >> 1;
      const uint32_t v = __shfl_sync(0xffffffffu, o0, mid);
      if (v <= e) lo = mid; else hi = mid - 1;
    }
    const uint32_t og = __shfl_sync(0xffffffffu, g, lo), oxy = __shfl_sync(0xffffffffu, rxy, lo);
    const uint32_t owh = __shfl_sync(0xffffffffu, rwh, lo), oo = __shfl_sync(0xffffffffu, o0, lo);
    if (e < last) {
      const uint32_t rank = e - oo, w = owh & 0xffffu;
      const uint32_t ty = (oxy >> 16) + rank / w, tx = (oxy & 0xffffu) + rank % w;
      keys[e] = (KeyT)(ty * ntx + tx);
      vals[e] = og;
    }
  }
}

template <typename KeyT>
__global__ void __launch_bounds__(kBlock) pack_sorted_kernel(const KeyT* __restrict__ keys,
                                                              const uint32_t* __restrict__ vals, long long m,
                                                              int n_tiles, int ntx, const GsRec* __restrict__ rec,
                                                              const uint32_t* __restrict__ offsets_g,
                                                              float4* __restrict__ pA, float2* __restrict__ pB,
                                                              float4* __restrict__ pC,
                                                              int* __restrict__ tile_accum) {
  long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= m) return;
  uint32_t tile = keys[i];
  // tile range boundaries (tile_n_point_accum semantics: accum[t] = first sorted index of tile t)
  if (i == 0) {
    for (uint32_t t = 0; t <= tile; ++t) tile_accum[t] = 0;
  } else {
    uint32_t prev = keys[i - 1];
    for (uint32_t t = prev + 1; t <= tile; ++t) tile_accum[t] = (int)i;
  }
  if (i == m - 1)
    for (uint32_t t = tile + 1; t <= (uint32_t)n_tiles; ++t) tile_accum[t] = (int)m;

  const uint32_t g = vals[i];
  const GsRec* r = rec + g;
  float4 a = r->a, b = r->b, c = r->c;
  uint32_t off = offsets_g[g];
  uint32_t rxy = __float_as_uint(c.z), rwh = __float_as_uint(c.w);
  uint32_t tx = tile % ntx, ty = tile / ntx;
  uint32_t slot = off + (ty - (rxy >> 16)) * (rwh & 0xffffu) + (tx - (rxy & 0xffffu));
  pA[i] = a;
  pB[i] = make_float2(b.x, b.y);
  pC[i] = make_float4(b.z, b.w, c.x, __uint_as_float(slot));
}

// SH variant: the third stream row is {raw coefficients rgb[g][0..d), slot, pad}.  8 lanes per
// instance copy the row so that both the gather and the store move 32-byte pieces.
template <typename KeyT>
__global__ void __launch_bounds__(kBlock) pack_sorted_sh_kernel(const KeyT* __restrict__ keys,
                                                                 const uint32_t* __restrict__ vals, long long m,
                                                                 int n_tiles, int ntx, const GsRec* __restrict__ rec,
                                                                 const uint32_t* __restrict__ offsets_g,
                                                                 const float* __restrict__ rgb, int d, int sw,
                                                                 float4* __restrict__ pA, float2* __restrict__ pB,
                                                                 float* __restrict__ pS, int* __restrict__ tile_accum) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  const long long i = t >> 3;
  const int sub = (int)(t & 7);
  if (i >= m) return;
  const uint32_t tile = keys[i];
  const uint32_t g = vals[i];
  if (sub == 0) {
    if (i == 0) {
      for (uint32_t tt = 0; tt <= tile; ++tt) tile_accum[tt] = 0;
    } else {
      uint32_t prev = keys[i - 1];
      for (uint32_t tt = prev + 1; tt <= tile; ++tt) tile_accum[tt] = (int)i;
    }
    if (i == m - 1)
      for (uint32_t tt = tile + 1; tt <= (uint32_t)n_tiles; ++tt) tile_accum[tt] = (int)m;
    const GsRec* r = rec + g;
    float4 a = r->a, b = r->b, c = r->c;
    uint32_t rxy = __float_as_uint(c.z), rwh = __float_as_uint(c.w);
    uint32_t tx = tile % ntx, ty = tile / ntx;
    uint32_t slot = offsets_g[g] + (ty - (rxy >> 16)) * (rwh & 0xffffu) + (tx - (rxy & 0xffffu));
    pA[i] = a;
    pB[i] = make_float2(b.x, b.y);
    pS[(size_t)i * sw + d] = __uint_as_float(slot);
  }
  float* row = pS + (size_t)i * sw;
  const float* src = rgb + (size_t)g * d;
  for (int q = sub; q < d; q += 8) row[q] = src[q];
}

// Tile ranges of the sorted instance list (tile_n_point_accum semantics: accum[t] = first sorted index of
// tile t, accum[T] = M) for the gather path, where no pack pass walks the keys.  8 consecutive keys per thread.
template <typename KeyT>
__global__ void __launch_bounds__(kBlock) tile_ranges_kernel(const KeyT* __restrict__ keys, long long m, int n_tiles,
                                                              int* __restrict__ tile_accum) {
  const long long i0 = ((long long)blockIdx.x * kBlock + threadIdx.x) * 8;
  if (i0 >= m) return;
  uint32_t prev = i0 > 0 ? (uint32_t)keys[i0 - 1] : 0u;
  if (i0 == 0) tile_accum[0] = 0;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const long long i = i0 + u;
    if (i >= m) break;
    const uint32_t tile = keys[i];
    for (uint32_t t = prev + 1; t <= tile; ++t) tile_accum[t] = (int)i;      // (empty for equal neighbours)
    if (i == 0)
      for (uint32_t t = 1; t <= tile; ++t) tile_accum[t] = 0;
    prev = tile;
    if (i == m - 1)
      for (uint32_t t = tile + 1; t <= (uint32_t)n_tiles; ++t) tile_accum[t] = (int)m;
  }
}

__global__ void __launch_bounds__(kBlock) iota_kernel(uint32_t* out, int n) {
  int i = blockIdx.x * kBlock + threadIdx.x;
  if (i < n) out[i] = (uint32_t)i;
}

}  // namespace

cudaError_t gs_launch_pack_sorted_sh(const void* keys, int key_bytes, const uint32_t* vals, long long m, int n_tiles,
                                     int ntx, const GsRec* rec, const uint32_t* offsets_g, const float* rgb, int d,
                                     int sw, float4* pA, float2* pB, float* pS, int* tile_accum, cudaStream_t st) {
  if (m == 0) return cudaMemsetAsync(tile_accum, 0, sizeof(int) * (size_t)(n_tiles + 1), st);
  const unsigned grid = (unsigned)((m * 8 + kBlock - 1) / kBlock);   // 8 lanes per instance
  if (key_bytes == 2)
    pack_sorted_sh_kernel<uint16_t><<<grid, kBlock, 0, st>>>(static_cast<const uint16_t*>(keys), vals, m, n_tiles,
                                                             ntx, rec, offsets_g, rgb, d, sw, pA, pB, pS, tile_accum);
  else
    pack_sorted_sh_kernel<uint32_t><<<grid, kBlock, 0, st>>>(static_cast<const uint32_t*>(keys), vals, m, n_tiles,
                                                             ntx, rec, offsets_g, rgb, d, sw, pA, pB, pS, tile_accum);
  return cudaGetLastError();
}

cudaError_t gs_launch_iota(uint32_t* out, int n, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  iota_kernel<<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(out, n);
  return cudaGetLastError();
}

extern "C" int gs_tile_list(const float* pos, const float* cov, int n, const float* tile_top,
                            const float* tile_bottom, const float* tile_left, const float* tile_right, int n_tiles,
                            int* tile_n_point, int* tile_gaussian_list, int max_per_tile, float thresh, int method,
                            float tile_length_x, float tile_length_y, int n_tiles_x, int n_tiles_y, float leftmost,
                            float topmost, gs_stream_t stream) {
  if (n < 0 || n_tiles < 0 || max_per_tile < 0) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_tile_list: negative size");
  if (n == 0 || n_tiles == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (method == 0 || method == 1) {
    dim3 block(32, 8), grid((n + 31) / 32, (n_tiles + 7) / 8);
    if (grid.y > 65535) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_tile_list: too many tiles for method 0/1");
    if (method == 0)
      tile_list_dist_kernel<<<grid, block, 0, st>>>(pos, tile_top, tile_bottom, tile_left, tile_right, tile_n_point,
                                                    tile_gaussian_list, n, n_tiles, max_per_tile, thresh);
    else
      tile_list_prob_kernel<<<grid, block, 0, st>>>(pos, cov, tile_top, tile_bottom, tile_left, tile_right,
                                                    tile_n_point, tile_gaussian_list, n, n_tiles, max_per_tile,
                                                    thresh);
  } else {
    GsTileGrid g;
    g.lx = tile_length_x;
    g.ly = tile_length_y;
    g.leftmost = leftmost;
    g.topmost = topmost;
    g.t2 = 0.f;
    g.ntx = n_tiles_x;
    g.nty = n_tiles_y;
    tile_list_prob2_kernel<<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(pos, cov, g, tile_n_point,
                                                                        tile_gaussian_list, n, max_per_tile, thresh);
  }
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_gather(const int* tile_n_point_accum, const int* tile_gaussian_list, int n_tiles, int list_stride,
                         int max_points_for_tile, int* gathered_list, int* tile_ids_for_points,
                         gs_stream_t stream) {
  (void)max_points_for_tile;   // only sized the reference's grid (gaussian.cu:367)
  if (n_tiles < 0) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_gather: n_tiles < 0");
  if (n_tiles == 0) return 0;
  int warps = kBlock / 32;
  gather_kernel<<<(n_tiles + warps - 1) / warps, kBlock, 0, (cudaStream_t)stream>>>(
      tile_n_point_accum, tile_gaussian_list, n_tiles, list_stride, gathered_list, tile_ids_for_points);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

cudaError_t gs_launch_emit_keys(const uint2* rect, const uint32_t* perm, const uint32_t* offsets_sorted, int n, int ntx,
                                void* keys, int key_bytes, uint32_t* vals, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (key_bytes == 2)
    emit_keys_kernel<uint16_t><<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(rect, perm, offsets_sorted, n, ntx,
                                                                             static_cast<uint16_t*>(keys), vals);
  else
    emit_keys_kernel<uint32_t><<<(n + kBlock - 1) / kBlock, kBlock, 0, st>>>(rect, perm, offsets_sorted, n, ntx,
                                                                             static_cast<uint32_t*>(keys), vals);
  return cudaGetLastError();
}

cudaError_t gs_launch_tile_ranges(const void* keys, int key_bytes, long long m, int n_tiles, int* tile_accum,
                                  cudaStream_t st) {
  if (m == 0) return cudaMemsetAsync(tile_accum, 0, sizeof(int) * (size_t)(n_tiles + 1), st);
  const unsigned grid = (unsigned)((m + 8LL * kBlock - 1) / (8LL * kBlock));
  if (key_bytes == 2)
    tile_ranges_kernel<uint16_t><<<grid, kBlock, 0, st>>>(static_cast<const uint16_t*>(keys), m, n_tiles, tile_accum);
  else
    tile_ranges_kernel<uint32_t><<<grid, kBlock, 0, st>>>(static_cast<const uint32_t*>(keys), m, n_tiles, tile_accum);
  return cudaGetLastError();
}

cudaError_t gs_launch_pack_sorted(const void* keys, int key_bytes, const uint32_t* vals, long long m, int n_tiles,
                                  int ntx, const GsRec* rec, const uint32_t* offsets_g, float4* pA, float2* pB,
                                  float4* pC, int* tile_accum, cudaStream_t st) {
  if (m == 0) return cudaMemsetAsync(tile_accum, 0, sizeof(int) * (size_t)(n_tiles + 1), st);
  const unsigned grid = (unsigned)((m + kBlock - 1) / kBlock);
  if (key_bytes == 2)
    pack_sorted_kernel<uint16_t><<<grid, kBlock, 0, st>>>(static_cast<const uint16_t*>(keys), vals, m, n_tiles, ntx,
                                                          rec, offsets_g, pA, pB, pC, tile_accum);
  else
    pack_sorted_kernel<uint32_t><<<grid, kBlock, 0, st>>>(static_cast<const uint32_t*>(keys), vals, m, n_tiles, ntx,
                                                          rec, offsets_g, pA, pB, pC, tile_accum);
  return cudaGetLastError();
}
