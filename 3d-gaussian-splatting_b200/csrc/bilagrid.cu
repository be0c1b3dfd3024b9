// Per-view bilateral grids (Wang et al., "Bilateral Guided Radiance Field Processing", SIGGRAPH Asia 2024): slice a
// rendered image through its view's grid of 3x4 affine colour transforms, forward and backward.  Definition and
// layout: include/gs_b200.h, gs_bilagrid_slice_fwd.
//
// Forward: one thread per pixel, 12 B read and 12 B written; the 8 grid nodes of the pixel's cell are three float4
// loads each through the read-only path (a 16x16x8 row is 96 KB and stays in L1 / L2).
//
// Backward, one pass over the pixels: CTA = (image b, spatial cell (cx, cy), row slice s).  Every pixel of a CTA lies
// in one spatial cell, so its grid gradient touches the cell's 4 corner columns only.  The CTA's threads are split
// into roles (corner, coefficient group); a thread accumulates w_xy(corner) * hat_k(gz) * dL/dA over its pixels for
// every knot k with the hat weights fully unrolled, so the accumulators stay in registers.  The roles are reduced in a
// fixed order (xor butterfly, then warps in index order) and the CTA writes its partial rows once.  The image
// gradient of a pixel is computed by one role, chosen round-robin per pixel batch.  bilagrid_reduce_kernel then sums,
// per node of each view in the batch, its partials in index order: images of that view ascending, the up to 4
// adjacent cells, the row slices.  No atomics: the same inputs give the same bits.
#include <algorithm>
#include <cstdio>
#include <vector>

#include "internal.h"

namespace {

constexpr int FWD_THREADS = 256;
constexpr int BWD_THREADS = 256;
constexpr int IDS_PER_LAUNCH = 64;     // forward view ids passed by value
constexpr int BWD_TARGET_CTAS = 1024;  // row slices are added until the backward has about this many CTAs
constexpr int MAX_SLICES = 64;

struct ViewIds {
  int v[IDS_PER_LAUNCH];
};

// the backward's view table reaches the workspace through kernel parameters: no host copy, no synchronisation
constexpr int TABLE_PER_LAUNCH = 960;
struct Table {
  int v[TABLE_PER_LAUNCH];
};

__global__ void bilagrid_table_kernel(Table t, int n, int* __restrict__ dst) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = t.v[i];
}

// spatial lattice coordinate of pixel index i along an axis of n pixels and g nodes, and its cell in [0, g - 2]
__device__ __forceinline__ float lattice_coord(int i, float scale) { return ((float)i + 0.5f) * scale; }
__device__ __forceinline__ int cell_of(float gc, int g) { return min(max((int)floorf(gc), 0), g - 2); }

// luminance guide, in the documented fp32 order
__device__ __forceinline__ float guide(float r, float g, float b) {
  return fmaf(0.114f, b, fmaf(0.587f, g, __fmul_rn(0.299f, r)));
}

// z cell and fraction: gz = clamp(z, 0, 1) * (gl - 1); the cell index is exact (the fma residual decides a product
// that rounds up onto a knot), so an interior knot takes the upper cell as grid_sample does
__device__ __forceinline__ void z_cell(float z, int gl, int& z0, float& fz) {
  const float zc = fminf(fmaxf(z, 0.f), 1.f);
  const float k = (float)(gl - 1);
  const float gz = zc * k;
  float f0 = floorf(gz);
  if (fmaf(zc, k, -f0) < 0.f) f0 -= 1.f;
  z0 = min((int)f0, gl - 2);
  fz = fmaf(zc, k, -(float)z0);
}

__device__ __forceinline__ void load12(const float* p, float a[12]) {
  const float4* q = reinterpret_cast<const float4*>(p);
  const float4 x = __ldg(q), y = __ldg(q + 1), z = __ldg(q + 2);
  a[0] = x.x; a[1] = x.y; a[2] = x.z; a[3] = x.w;
  a[4] = y.x; a[5] = y.y; a[6] = y.z; a[7] = y.w;
  a[8] = z.x; a[9] = z.y; a[10] = z.z; a[11] = z.w;
}

struct PixelCell {
  float fx, fy, fz;
  int x0, y0, z0;
};

// the trilinear affine A (12) of a pixel and, when dA != nullptr, dA / dgz (the upper-cell slope)
__device__ __forceinline__ void interp(const float* grid, int gw, int gl, const PixelCell& c, float A[12], float* dA) {
  const int ld_z = 12, ld_x = gl * 12, ld_y = gw * gl * 12;
#pragma unroll
  for (int j = 0; j < 12; ++j) A[j] = 0.f;
  if (dA) {
#pragma unroll
    for (int j = 0; j < 12; ++j) dA[j] = 0.f;
  }
#pragma unroll
  for (int corner = 0; corner < 4; ++corner) {
    const int a = corner & 1, b = corner >> 1;
    const float w = (a ? c.fx : 1.f - c.fx) * (b ? c.fy : 1.f - c.fy);
    const float* p = grid + (size_t)(c.y0 + b) * ld_y + (size_t)(c.x0 + a) * ld_x + (size_t)c.z0 * ld_z;
    float lo[12], hi[12];
    load12(p, lo);
    load12(p + ld_z, hi);
#pragma unroll
    for (int j = 0; j < 12; ++j) {
      A[j] = fmaf(w, fmaf(c.fz, hi[j] - lo[j], lo[j]), A[j]);
      if (dA) dA[j] = fmaf(w, hi[j] - lo[j], dA[j]);
    }
  }
}

__device__ __forceinline__ PixelCell pixel_cell(int x, int y, float z, float sx, float sy, int gw, int gh, int gl) {
  PixelCell c;
  const float gx = lattice_coord(x, sx), gy = lattice_coord(y, sy);
  c.x0 = cell_of(gx, gw);
  c.y0 = cell_of(gy, gh);
  c.fx = gx - (float)c.x0;
  c.fy = gy - (float)c.y0;
  z_cell(z, gl, c.z0, c.fz);
  return c;
}

__global__ void __launch_bounds__(FWD_THREADS) bilagrid_fwd_kernel(const float* __restrict__ image,
                                                                   const float* __restrict__ grids, ViewIds ids,
                                                                   int b0, int H, int W, int GH, int GW, int GL,
                                                                   float sx, float sy, float* __restrict__ out) {
  const int npx = H * W;
  const int p = blockIdx.x * FWD_THREADS + threadIdx.x;
  if (p >= npx) return;
  const int b = b0 + blockIdx.y;
  const size_t off = ((size_t)b * npx + p) * 3;
  const float r = image[off], g = image[off + 1], bl = image[off + 2];
  const PixelCell c = pixel_cell(p % W, p / W, guide(r, g, bl), sx, sy, GW, GH, GL);
  float A[12];
  interp(grids + (size_t)ids.v[blockIdx.y] * GH * GW * GL * 12, GW, GL, c, A, nullptr);
  out[off] = fmaf(A[0], r, fmaf(A[1], g, fmaf(A[2], bl, A[3])));
  out[off + 1] = fmaf(A[4], r, fmaf(A[5], g, fmaf(A[6], bl, A[7])));
  out[off + 2] = fmaf(A[8], r, fmaf(A[9], g, fmaf(A[10], bl, A[11])));
}

// first pixel index along an axis whose cell is >= c (cells are monotone in the pixel index)
__device__ int first_in_cell(int c, int n, float scale, int g) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cell_of(lattice_coord(mid, scale), g) >= c) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// KMAX: knots unrolled (GL <= KMAX); NC: coefficients per role (12 or 6).  Roles: 4 corners x 12 / NC groups.
template <int KMAX, int NC, bool DO_IMG, bool DO_GRID>
__global__ void __launch_bounds__(BWD_THREADS) bilagrid_bwd_kernel(
    const float* __restrict__ image, const float* __restrict__ grids, const int* __restrict__ ids, int H, int W,
    int GH, int GW, int GL, float sx, float sy, int n_slices, const float* __restrict__ grad_out,
    float* __restrict__ grad_image, float* __restrict__ partial) {
  constexpr int GROUPS = 12 / NC;
  constexpr int ROLES = DO_GRID ? 4 * GROUPS : 1;
  constexpr int PER_ROLE = BWD_THREADS / ROLES;
  constexpr int WARPS_PER_ROLE = PER_ROLE / 32;
  __shared__ float red[DO_GRID ? BWD_THREADS / 32 * KMAX * NC : 1];

  const int ncx = GW - 1, ncy = GH - 1;
  const int slice = blockIdx.x % n_slices;
  const int cell = blockIdx.x / n_slices;
  const int cx = cell % ncx, cy = cell / ncx;
  const int b = blockIdx.y;
  const int xa = first_in_cell(cx, W, sx, GW), xb = cx == ncx - 1 ? W : first_in_cell(cx + 1, W, sx, GW);
  const int ya = first_in_cell(cy, H, sy, GH), yb = cy == ncy - 1 ? H : first_in_cell(cy + 1, H, sy, GH);
  const int nrows = yb - ya, ncols = xb - xa;
  const int r0 = ya + (int)((long long)nrows * slice / n_slices);
  const int r1 = ya + (int)((long long)nrows * (slice + 1) / n_slices);
  const int npx = (r1 - r0) * ncols;

  const int role = threadIdx.x / PER_ROLE, lane = threadIdx.x % PER_ROLE;
  const int corner = role / GROUPS, group = role % GROUPS;
  const float* grid = grids + (size_t)ids[b] * GH * GW * GL * 12;
  const size_t img_off = (size_t)b * H * W;

  float acc[DO_GRID ? KMAX : 1][DO_GRID ? NC : 1];
  if (DO_GRID) {
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
#pragma unroll
      for (int m = 0; m < NC; ++m) acc[k][m] = 0.f;
  }

  for (int base = 0, it = 0; base < npx; base += PER_ROLE, ++it) {
    const int i = base + lane;
    if (i >= npx) continue;
    const int y = r0 + i / ncols, x = xa + i % ncols;
    const size_t off = (img_off + (size_t)y * W + x) * 3;
    const float u0 = image[off], u1 = image[off + 1], u2 = image[off + 2];
    const float g0 = grad_out[off], g1 = grad_out[off + 1], g2 = grad_out[off + 2];
    const float z = guide(u0, u1, u2);
    const PixelCell c = pixel_cell(x, y, z, sx, sy, GW, GH, GL);
    if (DO_GRID) {
      const float w = ((corner & 1) ? c.fx : 1.f - c.fx) * ((corner & 2) ? c.fy : 1.f - c.fy);
      const float u[4] = {u0, u1, u2, 1.f};
      const float gg[3] = {g0 * w, g1 * w, g2 * w};
      float q[12];
#pragma unroll
      for (int j = 0; j < 12; ++j) q[j] = gg[j / 4] * u[j % 4];
      float qs[NC];
#pragma unroll
      for (int m = 0; m < NC; ++m) qs[m] = (GROUPS == 1 || group == 0) ? q[m] : q[(NC * (GROUPS - 1) + m) % 12];
      const float w_lo = 1.f - c.fz, w_hi = c.fz;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        const float h = k == c.z0 ? w_lo : (k == c.z0 + 1 ? w_hi : 0.f);
#pragma unroll
        for (int m = 0; m < NC; ++m) acc[k][m] = fmaf(h, qs[m], acc[k][m]);
      }
    }
    if (DO_IMG && (!DO_GRID || it % ROLES == role)) {
      float A[12], dA[12];
      interp(grid, GW, GL, c, A, dA);
      float gi0 = fmaf(A[0], g0, fmaf(A[4], g1, A[8] * g2));
      float gi1 = fmaf(A[1], g0, fmaf(A[5], g1, A[9] * g2));
      float gi2 = fmaf(A[2], g0, fmaf(A[6], g1, A[10] * g2));
      if (z > 0.f && z < 1.f) {
        const float d0 = fmaf(dA[0], u0, fmaf(dA[1], u1, fmaf(dA[2], u2, dA[3])));
        const float d1 = fmaf(dA[4], u0, fmaf(dA[5], u1, fmaf(dA[6], u2, dA[7])));
        const float d2 = fmaf(dA[8], u0, fmaf(dA[9], u1, fmaf(dA[10], u2, dA[11])));
        const float gz = fmaf(g0, d0, fmaf(g1, d1, g2 * d2)) * (float)(GL - 1);
        gi0 = fmaf(0.299f, gz, gi0);
        gi1 = fmaf(0.587f, gz, gi1);
        gi2 = fmaf(0.114f, gz, gi2);
      }
      grad_image[off] = gi0;
      grad_image[off + 1] = gi1;
      grad_image[off + 2] = gi2;
    }
  }

  if (DO_GRID) {
    const int warp = threadIdx.x / 32, wl = threadIdx.x % 32;
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
#pragma unroll
      for (int m = 0; m < NC; ++m) {
        float v = acc[k][m];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (wl == 0) red[(warp * KMAX + k) * NC + m] = v;
      }
    __syncthreads();
    // partial row of this CTA: [4 corners][GL][12], written once
    float* dst = partial + ((size_t)b * gridDim.x + blockIdx.x) * 4 * GL * 12;
    for (int t = threadIdx.x; t < 4 * GL * 12; t += BWD_THREADS) {
      const int j = t % 12, k = (t / 12) % GL, cn = t / (12 * GL);
      const int rl = cn * GROUPS + j / NC, m = j % NC;
      float s = 0.f;
      for (int wi = 0; wi < WARPS_PER_ROLE; ++wi) s += red[((rl * WARPS_PER_ROLE + wi) * KMAX + k) * NC + m];
      dst[t] = s;
    }
  }
}

// grad_grids row of each view in the batch: node (iy, ix, k), coefficient j = sum over the images of that view
// (ascending), the up to 4 cells around the node, the row slices; one thread per (view slot, node, j)
__global__ void bilagrid_reduce_kernel(const float* __restrict__ partial, const int* __restrict__ ids, int B,
                                       const int* __restrict__ views, int GH, int GW, int GL, int n_slices,
                                       float* __restrict__ grad_grids) {
  const int row = GH * GW * GL * 12;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= row) return;
  const int v = views[blockIdx.y];
  const int j = t % 12, k = (t / 12) % GL, ix = (t / (12 * GL)) % GW, iy = t / (12 * GL * GW);
  const int ncx = GW - 1, ncells = (GH - 1) * ncx;
  float s = 0.f;
  for (int b = 0; b < B; ++b) {
    if (ids[b] != v) continue;
    for (int cy = max(iy - 1, 0); cy <= min(iy, GH - 2); ++cy)
      for (int cx = max(ix - 1, 0); cx <= min(ix, GW - 2); ++cx) {
        const int cn = (iy - cy) * 2 + (ix - cx);
        const float* p = partial + (((size_t)b * ncells + cy * ncx + cx) * n_slices) * 4 * GL * 12 +
                         ((size_t)cn * GL + k) * 12 + j;
        for (int sl = 0; sl < n_slices; ++sl) s += p[(size_t)sl * 4 * GL * 12];
      }
  }
  grad_grids[(size_t)v * row + t] = s;
}

inline size_t up256(size_t x) { return (x + 255) / 256 * 256; }

int n_slices_for(int B, int GH, int GW) {
  const long long cells = (long long)B * (GH - 1) * (GW - 1);
  return (int)std::max(1LL, std::min<long long>(MAX_SLICES, (BWD_TARGET_CTAS + cells - 1) / cells));
}

bool dims_ok(int GH, int GW, int GL) {
  return GH >= 2 && GW >= 2 && GL >= 2 && GH <= GS_BILAGRID_MAX_HW && GW <= GS_BILAGRID_MAX_HW &&
         GL <= GS_BILAGRID_MAX_L;
}

int check_common(const char* fn, const float* image, const float* grids, const int* ids, int B, int H, int W, int V,
                 int GH, int GW, int GL) {
  char msg[160];
  if (!image || !grids || !ids) {
    snprintf(msg, sizeof msg, "%s: null argument", fn);
    return gs_set_error_msg(GS_ERR_INVALID_ARG, msg);
  }
  if (B <= 0 || H <= 0 || W <= 0 || V <= 0 || B > 65535 || (long long)H * W > (1LL << 30)) {
    snprintf(msg, sizeof msg, "%s: B, H, W and V must be positive (B <= 65535, H * W <= 2^30)", fn);
    return gs_set_error_msg(GS_ERR_INVALID_ARG, msg);
  }
  if (!dims_ok(GH, GW, GL)) {
    snprintf(msg, sizeof msg, "%s: grid dimensions must be 2 <= GH, GW <= %d and 2 <= GL <= %d", fn,
             GS_BILAGRID_MAX_HW, GS_BILAGRID_MAX_L);
    return gs_set_error_msg(GS_ERR_INVALID_ARG, msg);
  }
  for (int b = 0; b < B; ++b)
    if (ids[b] < 0 || ids[b] >= V) {
      snprintf(msg, sizeof msg, "%s: view id %d of image %d is outside [0, %d)", fn, ids[b], b, V);
      return gs_set_error_msg(GS_ERR_INVALID_ARG, msg);
    }
  return 0;
}

template <int KMAX, int NC>
cudaError_t launch_bwd(bool img, bool grd, dim3 grid, cudaStream_t st, const float* image, const float* grids,
                       const int* ids, int H, int W, int GH, int GW, int GL, float sx, float sy, int ns,
                       const float* grad_out, float* grad_image, float* partial) {
  if (img && grd)
    bilagrid_bwd_kernel<KMAX, NC, true, true><<<grid, BWD_THREADS, 0, st>>>(image, grids, ids, H, W, GH, GW, GL, sx,
                                                                           sy, ns, grad_out, grad_image, partial);
  else if (grd)
    bilagrid_bwd_kernel<KMAX, NC, false, true><<<grid, BWD_THREADS, 0, st>>>(image, grids, ids, H, W, GH, GW, GL, sx,
                                                                            sy, ns, grad_out, grad_image, partial);
  else
    bilagrid_bwd_kernel<4, 12, true, false><<<grid, BWD_THREADS, 0, st>>>(image, grids, ids, H, W, GH, GW, GL, sx,
                                                                         sy, ns, grad_out, grad_image, partial);
  return cudaGetLastError();
}

}  // namespace

extern "C" size_t gs_bilagrid_workspace_bytes(int B, int H, int W, int V, int GH, int GW, int GL) {
  if (B <= 0 || H <= 0 || W <= 0 || V <= 0 || !dims_ok(GH, GW, GL)) return 0;
  const size_t ns = n_slices_for(B, GH, GW);
  const size_t rows = (size_t)B * (GH - 1) * (GW - 1) * ns;
  return up256((size_t)2 * B * sizeof(int)) + up256(rows * 4 * GL * 12 * sizeof(float));
}

extern "C" int gs_bilagrid_slice_fwd(const float* image, const float* grids, const int* view_ids_host, int B, int H,
                                     int W, int V, int GH, int GW, int GL, float* out, gs_stream_t stream) {
  if (!out) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_bilagrid_slice_fwd: null argument");
  if (int rc = check_common("gs_bilagrid_slice_fwd", image, grids, view_ids_host, B, H, W, V, GH, GW, GL)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float sx = (float)(GW - 1) / (float)W, sy = (float)(GH - 1) / (float)H;
  const int npx = H * W;
  for (int b0 = 0; b0 < B; b0 += IDS_PER_LAUNCH) {
    const int nb = std::min(IDS_PER_LAUNCH, B - b0);
    ViewIds ids{};
    for (int i = 0; i < nb; ++i) ids.v[i] = view_ids_host[b0 + i];
    const dim3 grid((npx + FWD_THREADS - 1) / FWD_THREADS, nb);
    bilagrid_fwd_kernel<<<grid, FWD_THREADS, 0, st>>>(image, grids, ids, b0, H, W, GH, GW, GL, sx, sy, out);
    GS_CUDA_TRY(cudaGetLastError());
    gs_count_launch();
  }
  return 0;
}

extern "C" int gs_bilagrid_slice_bwd(const float* image, const float* grids, const int* view_ids_host, int B, int H,
                                     int W, int V, int GH, int GW, int GL, const float* grad_out, float* grad_image,
                                     float* grad_grids, void* workspace, size_t workspace_bytes, gs_stream_t stream) {
  if (!grad_out || !workspace) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_bilagrid_slice_bwd: null argument");
  if (int rc = check_common("gs_bilagrid_slice_bwd", image, grids, view_ids_host, B, H, W, V, GH, GW, GL)) return rc;
  if (workspace_bytes < gs_bilagrid_workspace_bytes(B, H, W, V, GH, GW, GL))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_bilagrid_slice_bwd: workspace too small");
  if (!grad_image && !grad_grids) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  // ids[B] then the distinct views of the batch, ascending
  std::vector<int> tab(view_ids_host, view_ids_host + B);
  std::vector<int> views(view_ids_host, view_ids_host + B);
  std::sort(views.begin(), views.end());
  views.erase(std::unique(views.begin(), views.end()), views.end());
  tab.insert(tab.end(), views.begin(), views.end());
  int* d_ids = static_cast<int*>(workspace);
  float* partial = reinterpret_cast<float*>(static_cast<char*>(workspace) + up256((size_t)2 * B * sizeof(int)));
  for (size_t i0 = 0; i0 < tab.size(); i0 += TABLE_PER_LAUNCH) {
    const int n = (int)std::min<size_t>(TABLE_PER_LAUNCH, tab.size() - i0);
    Table t;
    std::copy(tab.begin() + i0, tab.begin() + i0 + n, t.v);
    bilagrid_table_kernel<<<1, 256, 0, st>>>(t, n, d_ids + i0);
    GS_CUDA_TRY(cudaGetLastError());
    gs_count_launch();
  }
  const float sx = (float)(GW - 1) / (float)W, sy = (float)(GH - 1) / (float)H;
  const int ns = n_slices_for(B, GH, GW);
  const dim3 grid((unsigned)((GH - 1) * (GW - 1) * ns), (unsigned)B);
  const bool img = grad_image != nullptr, grd = grad_grids != nullptr;
  cudaError_t e;
  if (GL <= 4)
    e = launch_bwd<4, 12>(img, grd, grid, st, image, grids, d_ids, H, W, GH, GW, GL, sx, sy, ns, grad_out,
                          grad_image, partial);
  else if (GL <= 8)
    e = launch_bwd<8, 12>(img, grd, grid, st, image, grids, d_ids, H, W, GH, GW, GL, sx, sy, ns, grad_out,
                          grad_image, partial);
  else
    e = launch_bwd<16, 6>(img, grd, grid, st, image, grids, d_ids, H, W, GH, GW, GL, sx, sy, ns, grad_out,
                          grad_image, partial);
  GS_CUDA_TRY(e);
  gs_count_launch();
  if (grd) {
    const int row = GH * GW * GL * 12;
    const dim3 rgrid((row + 255) / 256, (unsigned)views.size());
    bilagrid_reduce_kernel<<<rgrid, 256, 0, st>>>(partial, d_ids, B, d_ids + B, GH, GW, GL, ns, grad_grids);
    GS_CUDA_TRY(cudaGetLastError());
    gs_count_launch();
  }
  return 0;
}
