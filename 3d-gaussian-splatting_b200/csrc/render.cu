// Frame orchestration for the fused path: owns device workspaces and strings the stages
//   project -> depth sort of the N Gaussians + scan -> emit in depth order -> stable tile-id
//   radix sort of the M instances (CUB onesweep, 2 passes at 1080p) -> range+pack -> blend
// and the backward  blend_bwd -> project_bwd (segment-sum + chain rule).
// Replaces the PyTorch glue of reference splatter.py:513-655 (4 boolean-mask compactions, the
// dense [T, N/20] tile list, cumsum, two 4-tensor gathers, fp32-key torch.sort, >= 7 host
// syncs) with 7 launches and ONE 8-byte readback (the instance count M sizes the sort).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "internal.h"

// count of the Gaussian at depth-sorted position i (0 for the sentinel item i == n)
struct GsCountInSortedOrder {
  const uint32_t* count;
  const uint32_t* perm;
  uint32_t n;
  __host__ __device__ __forceinline__ uint32_t operator()(uint32_t i) const { return i < n ? count[perm[i]] : 0u; }
};

// ---- error plumbing ---------------------------------------------------------------------
static thread_local char g_err[512] = {0};

int gs_set_error(cudaError_t e, const char* what) {
  snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return (int)e;
}
int gs_set_error_msg(int code, const char* what) {
  snprintf(g_err, sizeof(g_err), "%s", what);
  return code;
}
extern "C" const char* gs_last_error(void) { return g_err; }
extern "C" int gs_abi_version(void) { return 2; }

static int tune_env(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}
GsTuning& gs_tuning() {
  // shipped configuration: re-swept on the H100 at C3 (RGB blend knobs: no variant faster beyond run-to-run noise;
  // SH: see gs_sh_tc_mode)
  static GsTuning t = {tune_env("GS_TUNE_FWD_KERNEL", 0),  tune_env("GS_TUNE_FWD_CH", 128),   tune_env("GS_TUNE_BWD_KERNEL", 1),
                       tune_env("GS_TUNE_BWD_PX", 8),      tune_env("GS_TUNE_BWD_WS", 0),     tune_env("GS_TUNE_BWD_UNROLL", 4),
                       tune_env("GS_TUNE_BWD_STAGES", 3),  tune_env("GS_TUNE_BWD_MINB", 10),  tune_env("GS_TUNE_BWD_RQ", 4),
                       tune_env("GS_TUNE_FWD_PX", 4),      tune_env("GS_TUNE_BWD_CH", 32),    tune_env("GS_TUNE_STRICT", 0),
                       tune_env("GS_TUNE_GATHER", 1),      tune_env("GS_TUNE_SH_TC", -1),     tune_env("GS_TUNE_BLEND_REPACK", 1)};
  return t;
}
extern "C" int gs_tune(const char* name, int value) {
  if (!name) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_tune: null name");
  GsTuning& t = gs_tuning();
  struct { const char* k; int* v; } tab[] = {{"fwd_kernel", &t.fwd_kernel}, {"fwd_ch", &t.fwd_ch},
                                             {"bwd_kernel", &t.bwd_kernel}, {"bwd_px", &t.bwd_px},
                                             {"bwd_ws", &t.bwd_ws},         {"bwd_unroll", &t.bwd_unroll},
                                             {"bwd_stages", &t.bwd_stages}, {"bwd_minb", &t.bwd_minb},
                                             {"bwd_rq", &t.bwd_rq},         {"fwd_px", &t.fwd_px},
                                             {"gather", &t.gather},         {"bwd_ch", &t.bwd_ch},
                                             {"strict", &t.strict},         {"sh_tc", &t.sh_tc},
                                             {"blend_repack", &t.blend_repack}};
  for (auto& e : tab)
    if (!strcmp(e.k, name)) {
      *e.v = value;
      return 0;
    }
  return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_tune: unknown knob");
}

#include <atomic>
static std::atomic<unsigned long long> g_launches{0};
void gs_count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
extern "C" unsigned long long gs_kernel_launches(void) { return g_launches.load(std::memory_order_relaxed); }

// ---- growable device buffer -------------------------------------------------------------
// Workspaces come from the caller's allocator when one is installed (gs_ctx_set_allocator: the torch shim
// passes PyTorch's stream-ordered caching allocator, so growth - e.g. after every densification - needs no
// device synchronisation and the memory shows up in torch's accounting); else cudaMalloc / cudaFree with a
// stream synchronisation before a buffer is replaced.
struct GsAllocator {
  gs_alloc_fn alloc = nullptr;
  gs_free_fn free = nullptr;
  void* user = nullptr;
};
static thread_local const GsAllocator* g_cur_alloc = nullptr;   // allocator of the context being served

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  const GsAllocator* owner = nullptr;       // allocator the current block came from (nullptr: cudaMalloc)
  void drop(cudaStream_t st, bool sync) {
    if (!p) return;
    if (owner && owner->free) {
      owner->free(p, owner->user);          // stream-ordered allocator: no synchronisation needed
    } else {
      if (sync) cudaStreamSynchronize(st);
      cudaFree(p);
    }
    p = nullptr;
    cap = 0;
  }
  cudaError_t reserve(size_t bytes, cudaStream_t st) {
    if (bytes <= cap) return cudaSuccess;
    drop(st, true);
    size_t want = bytes + bytes / 8 + 256;   // slack so M jitter between frames does not realloc
    const GsAllocator* a = g_cur_alloc;
    if (a && a->alloc) {
      p = a->alloc(want, a->user, (gs_stream_t)st);
      if (!p) return cudaErrorMemoryAllocation;
      owner = a;
    } else {
      cudaError_t e = cudaMalloc(&p, want);
      if (e != cudaSuccess) return e;
      owner = nullptr;
    }
    cap = want;
    return cudaSuccess;
  }
  void release() { drop(nullptr, false); }
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};

struct gs_ctx {
  int device = 0;
  GsAllocator allocator{};
  // per Gaussian
  DevBuf rec, rect, count, offsets, dkey_in, dkey_out, perm, iota, offsets_g;
  size_t iota_n = 0;
  // per instance
  DevBuf keys_in, keys_out, vals_in, vals_out, pA, pB, pC, grad_inst, row_epoch;
  DevBuf grad_feat_inst;                  // [M][f] per-instance feature gradients (gs_render_backward_feat)
  uint32_t epoch = 0;                      // tag of the current backward in row_epoch[]
  DevBuf score_rows, score_epoch;         // [M] (sum w, max w) rows of gs_frame_scores and their tags
  uint32_t score_ep = 0;                  // tag of the current score pass in score_epoch[]
  // per tile / misc
  DevBuf tile_accum, tile_neff, tile_neff_b, cub_tmp, counters, img_dev, gimg_dev, rays;
  DevBuf cam_part;                        // per-CTA partial sums of the camera gradient (gs_render_backward_cam)
  DevBuf views;                           // GsView[n_views] of the last batched forward (gs_render_forward_batch)
  DevBuf lenses;                          // GsLens[n_views] of the last batched forward with a lens
  float* host_rays = nullptr;             // pinned: rays_o, lefttop, dx, dy (SH colour only)
  GsView* host_views = nullptr;           // pinned: staging of the view table (GS_MAX_VIEWS entries)
  GsLens* host_lenses = nullptr;          // pinned: staging of the lens table (GS_MAX_VIEWS entries, with the views)
  unsigned long long* host_m = nullptr;   // pinned: {M}
  cudaEvent_t ev_m = nullptr;             // marks the completion of the M read-back
  cudaEvent_t ev_views = nullptr;         // marks the completion of the view table's upload from host_views
  // state of the last forward
  bool have_forward = false, have_backward = false, gather = false;
  bool have_aux = false;                  // the last forward wrote (depth, alpha) to a caller's aux buffer
  bool sh_gaussian = false;               // the last forward evaluated its SH colour once per Gaussian
  int feat_f = 0;                         // the last forward blended feat[n, feat_f] (0: no features)
  int n_views = 0;                        // the last forward was batched over n_views views (0: a single-view forward)
  const float* feat = nullptr;
  int n = 0, d = 3, scale_act = 0;
  long long m = 0;
  GsCam cam{};
  GsTileGrid grid{};
  GsFrameGeom geom{};
  float near_plane = 0.f, half_w = 0.f, half_h = 0.f;
  int64_t* mask_ptr = nullptr;
  // optional per-stage timing (CUDA events on the frame's stream)
  bool timing = false;
  cudaEvent_t ev[GS_N_STAGES + 2] = {};
  bool ev_ok = false;
  bool ev_fwd_valid = false, ev_bwd_valid = false;
  // data-parallel gradient push (gs_ctx_set_grad_push); world == 0: off
  GsGradPush push{};
  int sh_eval = GS_SH_EVAL_PIXEL;         // gs_ctx_set_sh_eval: applies to the forwards that follow
  int filter2d = GS_FILTER2D_NONE;        // gs_ctx_set_filter2d: applies to the forwards that follow
  float filter2d_var = 0.3f;              //   its variance in px^2
  bool filt_on = false;                   // the last forward's filter (its backward uses it)
  GsFilter2d filt{};
  bool stats_on = false;                  // gs_ctx_set_densify_stats: accumulated by the backwards that follow
  gs_densify_stats stats{};
  const float* filter3d = nullptr;        // gs_ctx_set_filter3d: applies to the forwards that follow (the caller's [n])
  int filter3d_n = 0;
  const float* f3d = nullptr;             // the last forward's 3-D filter (its backward uses it); NULL: none
  // gs_filter3d_compute: the view table (after a 16-byte slot for the smallest seen rate) and its pinned staging
  DevBuf f3_dev;
  GsF3View* f3_host = nullptr;
  int f3_host_cap = 0;
  cudaEvent_t ev_f3 = nullptr;            // marks the completion of the view table's upload from f3_host
  gs_lens lens_set[GS_MAX_VIEWS] = {};    // gs_ctx_set_lens: applies to the forwards that follow
  int lens_n = 0;                         //   0: off
  bool lens_on = false;                   // the last forward ran the lens kernels (its backward uses them)
  GsLens lens{};                          //   with the lens of its (first) view
  // 2D Gaussian surfels (gs_render_forward_surfel): the last forward's records, per-pixel workspaces and settings
  DevBuf srec, sws, swsm;
  bool surfel = false;                    // the last forward rendered surfels
  bool surfel_maps = false;               //   and wrote maps (swsm holds their sums)
  int surfel_kg = 0;                      //   its colour: 0 RGB, 9 / 16 per-Gaussian SH
  float surfel_bg[3] = {0.f, 0.f, 0.f};
  float dist_near = 0.2f, dist_far = 100.f;
};

// stage boundaries: event i is recorded BEFORE stage i; stage i lasts ev[i+1]-ev[i]
//  forward : 0 project | 1 scan+readback | 2 emit keys | 3 radix sort | 4 pack | 5 blend fwd | (6 end)
//  backward: 7 blend bwd | 8 project bwd | (9 end)
static inline void gs_mark(gs_ctx* c, int i, cudaStream_t st) {
  if (c->timing && c->ev_ok) cudaEventRecord(c->ev[i], st);
}

extern "C" int gs_ctx_create(gs_ctx** out) {
  if (!out) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_create: null out");
  gs_ctx* c = new (std::nothrow) gs_ctx();
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_create: out of host memory");
  GS_CUDA_TRY(cudaGetDevice(&c->device));
  cudaError_t e = cudaMallocHost(reinterpret_cast<void**>(&c->host_m), 64);
  if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&c->host_rays), 64);
  if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&c->host_views), GS_MAX_VIEWS * sizeof(GsView));
  if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&c->host_lenses), GS_MAX_VIEWS * sizeof(GsLens));
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_m, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_views, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    delete c;
    return gs_set_error(e, "cudaMallocHost");
  }
  *out = c;
  return 0;
}

extern "C" void gs_ctx_destroy(gs_ctx* c) {
  if (!c) return;
  // the buffers live on the device that was current at creation, which need not be current now
  int cur = -1;
  const bool switched = cudaGetDevice(&cur) == cudaSuccess && cur != c->device && cudaSetDevice(c->device) == cudaSuccess;
  cudaDeviceSynchronize();
  DevBuf* bufs[] = {&c->rec, &c->rect, &c->count, &c->offsets, &c->dkey_in, &c->dkey_out, &c->perm, &c->iota, &c->offsets_g, &c->keys_in, &c->keys_out,
                    &c->vals_in, &c->vals_out, &c->pA, &c->pB, &c->pC, &c->grad_inst, &c->row_epoch, &c->tile_accum, &c->tile_neff,
                    &c->tile_neff_b, &c->cub_tmp, &c->counters, &c->img_dev, &c->gimg_dev, &c->rays, &c->cam_part,
                    &c->grad_feat_inst, &c->views, &c->f3_dev, &c->lenses, &c->srec, &c->sws, &c->swsm,
                    &c->score_rows, &c->score_epoch};
  for (DevBuf* b : bufs) b->release();
  if (c->host_m) cudaFreeHost(c->host_m);
  if (c->host_rays) cudaFreeHost(c->host_rays);
  if (c->host_views) cudaFreeHost(c->host_views);
  if (c->host_lenses) cudaFreeHost(c->host_lenses);
  if (c->ev_m) cudaEventDestroy(c->ev_m);
  if (c->ev_views) cudaEventDestroy(c->ev_views);
  if (c->f3_host) cudaFreeHost(c->f3_host);
  if (c->ev_f3) cudaEventDestroy(c->ev_f3);
  if (c->ev_ok)
    for (cudaEvent_t e : c->ev) cudaEventDestroy(e);
  if (switched) cudaSetDevice(cur);
  delete c;
}

// a ctx owns buffers on the device that was current at gs_ctx_create; using it under another
// current device would launch on the wrong GPU
static int gs_check_device(int want, const char* who) {
  int dev = -1;
  GS_CUDA_TRY(cudaGetDevice(&dev));
  if (dev != want) {
    char msg[160];
    snprintf(msg, sizeof(msg), "%s: ctx belongs to device %d but device %d is current", who, want, dev);
    return gs_set_error_msg(GS_ERR_INVALID_ARG, msg);
  }
  return 0;
}

static int ceil_log2(unsigned v) {
  int b = 0;
  while ((1u << b) < v) ++b;
  return b;
}

// "who: what" as the last error
static int gs_fail(int code, const char* who, const char* what) {
  char msg[512];
  snprintf(msg, sizeof(msg), "%s: %s", who, what);
  return gs_set_error_msg(code, msg);
}

static int check_camera(const gs_camera& cam, const char* who) {
  if (cam.width <= 0 || cam.height <= 0 || !(cam.focal_x > 0.f) || !(cam.focal_y > 0.f))
    return gs_fail(GS_ERR_INVALID_ARG, who, "bad camera");
  if (!(cam.tile_thresh > 0.f && cam.tile_thresh < 1.f))
    return gs_fail(GS_ERR_INVALID_ARG, who, "tile_thresh must be in (0, 1)");
  return 0;
}

// one view's padded size (splatter.py:259-260); the frame's tile grid stacks the n_views views' grids vertically
static int frame_geom(const gs_camera& cam, int n_views, GsFrameGeom& g, const char* who) {
  g = GsFrameGeom{};
  g.width = cam.width;
  g.height = cam.height;
  g.wp = (cam.width + GS_TILE - 1) / GS_TILE * GS_TILE;
  g.hp = (cam.height + GS_TILE - 1) / GS_TILE * GS_TILE;
  g.ntx = g.wp / GS_TILE;
  const int nty = g.hp / GS_TILE;
  if (g.ntx > 65535 || (long long)nty * n_views > 65535)
    return gs_fail(GS_ERR_INVALID_ARG, who, "image too large (Wp / 16 and B Hp / 16 must not exceed 65535)");
  g.nty = nty * n_views;
  g.n_tiles = g.ntx * g.nty;
  g.fx = cam.focal_x;
  g.fy = cam.focal_y;
  return 0;
}

// the caller's background and depth / alpha outputs; use_aux: the blend runs its aux variant
static int parse_aux(const gs_render_aux* ax, const float* final_img, GsAuxOut& out, bool& use_aux, const char* who) {
  out = GsAuxOut{};
  use_aux = ax && (ax->background || ax->aux || ax->aux_final);
  if (!use_aux) return 0;
  if (ax->aux_final && !final_img) return gs_fail(GS_ERR_INVALID_ARG, who, "aux_final needs image_final");
  if (ax->background) {
    for (int k = 0; k < 3; ++k) {
      if (!std::isfinite(ax->background[k])) return gs_fail(GS_ERR_INVALID_ARG, who, "background must be finite");
      out.bg[k] = ax->background[k];
    }
  }
  out.aux = ax->aux;
  out.aux_final = ax->aux_final;
  return 0;
}

// a forward is about to touch the context: until it completes, the context holds no frame to differentiate
static int begin_forward(gs_ctx* c, const char* who) {
  if (int rc = gs_check_device(c->device, who)) return rc;
  g_cur_alloc = &c->allocator;
  c->have_forward = false;
  c->have_backward = false;
  c->have_aux = false;
  c->n_views = 0;
  c->surfel = false;
  c->ev_fwd_valid = false;
  return 0;
}

// what the backward of a completed forward needs; v: the constants of its (first) view
static void commit_forward(gs_ctx* c, int n, int d, int scale_activation, long long m, const GsFrameGeom& g,
                           const GsView& v, float near_plane, int n_views, bool sh_gaussian, bool gather, bool filt_on,
                           const GsAuxOut& aux_out, const gs_render_feat* ft, const float* f3d, bool lens_on,
                           const GsLens& lens) {
  c->lens_on = lens_on;
  c->lens = lens;
  c->ev_fwd_valid = c->timing && c->ev_ok;
  c->have_forward = true;
  c->have_aux = aux_out.aux != nullptr;
  c->sh_gaussian = sh_gaussian;
  c->feat_f = ft ? ft->f : 0;
  c->feat = ft ? ft->feat : nullptr;
  c->filt_on = filt_on;
  c->filt = v.filt;
  c->f3d = f3d;
  c->gather = gather;
  c->n = n;
  c->d = d;
  c->scale_act = scale_activation;
  c->m = m;
  c->cam = v.cam;
  c->grid = v.grid;
  c->geom = g;
  c->near_plane = near_plane;
  c->half_w = v.half_w;
  c->half_h = v.half_h;
  c->n_views = n_views;
}

// The smallest t in (0, hi] with sum_j c[j] t^j <= 0 (c[0] = 1 > 0), or +inf: a scan to the first sample at or below
// zero, then bisection of that interval (fp64).
static double first_nonpositive(const double* c, int deg, double hi) {
  auto p = [&](double t) {
    double v = 0.0;
    for (int j = deg; j >= 0; --j) v = v * t + c[j];
    return v;
  };
  const int steps = 1 << 14;
  double a = 0.0;
  for (int s = 1; s <= steps; ++s) {
    double b = hi * s / steps;
    if (p(b) > 0.0) {
      a = b;
      continue;
    }
    for (int it = 0; it < 200; ++it) {
      const double m = 0.5 * (a + b);
      if (!(m > a && m < b)) break;
      (p(m) <= 0.0 ? b : a) = m;
    }
    return b;
  }
  return INFINITY;
}

// The squared undistorted radius past which a lens folds back (GS_LENS_* in gs_b200.h), +inf without a limit.
//   OPENCV: the smallest rho^2 > 0 with 1 + 3 k1 rho^2 + 5 k2 rho^4 <= 0 (d(rho rad)/d rho, the radial part only).
//   FISHEYE: tan^2 of the smallest theta in (0, pi/2) with d theta_d / d theta <= 0.
static double lens_rho2_max(const gs_lens& l) {
  if (l.model == GS_LENS_OPENCV) {
    const double b = 3.0 * l.k[0], a = 5.0 * l.k[1];   // the quadratic a u^2 + b u + 1 in u = rho^2
    if (a == 0.0) return b < 0.0 ? -1.0 / b : INFINITY;
    const double disc = b * b - 4.0 * a;
    if (disc < 0.0) return INFINITY;
    const double q = -0.5 * (b + (b >= 0.0 ? 1.0 : -1.0) * sqrt(disc));   // roots q / a and 1 / q
    double best = INFINITY;
    const double r0 = q / a, r1 = q != 0.0 ? 1.0 / q : INFINITY;
    if (r0 > 0.0) best = r0;
    if (r1 > 0.0 && r1 < best) best = r1;
    return best;
  }
  if (l.model == GS_LENS_FISHEYE) {
    const double c[5] = {1.0, 3.0 * l.k[0], 5.0 * l.k[1], 7.0 * l.k[2], 9.0 * l.k[3]};   // in t = theta^2
    const double half_pi = 1.5707963267948966;
    const double t = first_nonpositive(c, 4, half_pi * half_pi);
    if (!(t < half_pi * half_pi)) return INFINITY;
    const double r = tan(sqrt(t));
    return r * r;
  }
  return INFINITY;
}

static bool lens_is_centre_pinhole(const gs_lens& l, const gs_camera& cam) {
  return l.model == GS_LENS_PINHOLE && (double)l.cx == cam.width / 2.0 && (double)l.cy == cam.height / 2.0;
}

// The device constants of lens l on camera cam: (ox, oy) = ((cx - W/2) / fx, (cy - H/2) / fy) and rho2_max, in fp64
// then narrowed.
static GsLens lens_constants(const gs_lens& l, const gs_camera& cam) {
  GsLens L{};
  L.model = l.model;
  L.ox = (float)(((double)l.cx - cam.width / 2.0) / (double)cam.focal_x);
  L.oy = (float)(((double)l.cy - cam.height / 2.0) / (double)cam.focal_y);
  L.rho2_max = (float)lens_rho2_max(l);
  if (l.model != GS_LENS_PINHOLE)
    for (int k = 0; k < 4; ++k) L.k[k] = l.k[k];
  return L;
}

// The lenses of a forward of n_views views: out[v] for view v, and on = false when none is set or every view's is the
// image-centre pinhole (the frame then runs the kernels of a frame without a lens).
static int resolve_lenses(const gs_ctx* c, const gs_camera* cams, int n_views, GsLens* out, bool& on, const char* who) {
  on = false;
  if (c->lens_n == 0) return 0;
  if (c->lens_n != 1 && c->lens_n != n_views)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the context's lenses are set for another number of views (n must be 1 or B)");
  for (int v = 0; v < n_views; ++v) {
    const gs_lens& l = c->lens_set[c->lens_n == 1 ? 0 : v];
    if (!lens_is_centre_pinhole(l, cams[v])) on = true;
    out[v] = lens_constants(l, cams[v]);
  }
  return 0;
}

// The per-camera constants of a frame of padded size g.wp x g.hp, formed from host scalars in double then narrowed, like
// the Python floats that the reference passes through pybind (splatter.py:279-282, :532-533).  The 2-D filter is in
// normalised image-plane units: the variance over the squared pixel pitch 1 / f^2, rounded once (zero without one).
static GsView view_constants(const gs_ctx* c, const gs_camera* cam, const GsFrameGeom& g) {
  GsView v{};
  if (c->filter2d != GS_FILTER2D_NONE) {
    v.filt.ex = (float)((double)c->filter2d_var / ((double)cam->focal_x * (double)cam->focal_x));
    v.filt.ey = (float)((double)c->filter2d_var / ((double)cam->focal_y * (double)cam->focal_y));
    v.filt.compensate = c->filter2d == GS_FILTER2D_ANTIALIAS;
  }
  v.grid.lx = (float)(16.0 / (double)cam->focal_x);
  v.grid.ly = (float)(16.0 / (double)cam->focal_y);
  v.grid.leftmost = (float)(-(double)g.wp / 2.0 / (double)cam->focal_x);
  v.grid.topmost = (float)(-(double)g.hp / 2.0 / (double)cam->focal_y);
  v.grid.t2 = -2.f * logf(cam->tile_thresh);
  v.grid.ntx = g.wp / GS_TILE;
  v.grid.nty = g.hp / GS_TILE;
  memcpy(v.cam.r, cam->rot, sizeof(v.cam.r));
  memcpy(v.cam.t, cam->tran, sizeof(v.cam.t));
  v.half_w = (float)((double)cam->width * 1.2 / 2.0 / (double)cam->focal_x);
  v.half_h = (float)((double)cam->height * 1.2 / 2.0 / (double)cam->focal_y);
  v.fx = cam->focal_x;
  v.fy = cam->focal_y;
  return v;
}

// per-Gaussian (per-pair in a batched frame) and per-tile workspaces of a frame of N items
static int reserve_frame(gs_ctx* c, size_t N, int n_tiles, cudaStream_t st) {
  GS_CUDA_TRY(c->rec.reserve(N * sizeof(GsRec), st));
  GS_CUDA_TRY(c->rect.reserve(N * sizeof(uint2), st));
  GS_CUDA_TRY(c->count.reserve((N + 1) * 4, st));
  GS_CUDA_TRY(c->offsets.reserve((N + 1) * 4, st));
  GS_CUDA_TRY(c->dkey_in.reserve(N * 4 + 4, st));
  GS_CUDA_TRY(c->dkey_out.reserve(N * 4 + 4, st));
  GS_CUDA_TRY(c->perm.reserve(N * 4 + 4, st));
  GS_CUDA_TRY(c->offsets_g.reserve((N + 1) * 4, st));
  GS_CUDA_TRY(c->tile_accum.reserve((size_t)(n_tiles + 1) * 4, st));
  GS_CUDA_TRY(c->tile_neff.reserve((size_t)n_tiles * 4, st));
  GS_CUDA_TRY(c->tile_neff_b.reserve((size_t)n_tiles * 4, st));
  GS_CUDA_TRY(c->counters.reserve(64, st));
  if (c->iota_n < N) {   // 0..N-1 values for the depth sort (kept across frames)
    GS_CUDA_TRY(c->iota.reserve(N * 4 + 4, st));
    GS_CUDA_TRY(gs_launch_iota(c->iota.as<uint32_t>(), (int)N, st));
    gs_count_launch();
    c->iota_n = N;
  }
  return 0;
}

// stages 2-5 of a frame of n items (Gaussians, or (view, Gaussian) pairs): scans and the host read-back of M, the
// depth sort, instance emission, the tile sort and the tile ranges (gather) or the pack pass
static int bin_frame(gs_ctx* c, int n, const GsFrameGeom& g, bool gather, int blend_d, int d, const float* rgb,
                     cudaStream_t st, long long& m_out) {
  // 2. (a) exclusive scan of the tile counts in Gaussian-id order -> gradient-row bases and M;
  //    (b) stable depth sort of the N Gaussians; (c) scan of the counts in depth order (the
  //    count gather is fused into the scan's input iterator) -> instance emission offsets
  gs_mark(c, 1, st);
  size_t tmp_bytes = 0, tmp2 = 0, tmp3 = 0;
  if (n > 0)
    GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, c->dkey_in.as<uint32_t>(),
                                                c->dkey_out.as<uint32_t>(), c->iota.as<uint32_t>(),
                                                c->perm.as<uint32_t>(), n, 0, 32, st));
  GsCountInSortedOrder cnt_it_fn{c->count.as<uint32_t>(), c->perm.as<uint32_t>(), (uint32_t)n};
  cub::CountingInputIterator<uint32_t> idx_it(0);
  cub::TransformInputIterator<uint32_t, GsCountInSortedOrder, cub::CountingInputIterator<uint32_t>> cnt_it(idx_it,
                                                                                                            cnt_it_fn);
  GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp2, cnt_it, c->offsets.as<uint32_t>(), n + 1, st));
  GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp3, c->count.as<uint32_t>(), c->offsets_g.as<uint32_t>(),
                                            n + 1, st));
  if (tmp2 > tmp_bytes) tmp_bytes = tmp2;
  if (tmp3 > tmp_bytes) tmp_bytes = tmp3;
  GS_CUDA_TRY(c->cub_tmp.reserve(tmp_bytes, st));
  GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tmp3, c->count.as<uint32_t>(), c->offsets_g.as<uint32_t>(),
                                            n + 1, st));
  // the one host round trip of the frame: M = offsets_g[N] is known right after the first scan, so
  // its read-back is enqueued BEFORE the depth sort and the host waits on an event recorded there -
  // the GPU keeps sorting while the host wakes up and enqueues the rest of the frame (no bubble)
  *c->host_m = 0;
  GS_CUDA_TRY(cudaMemcpyAsync(c->host_m, c->counters.as<unsigned int>() + 2, 8, cudaMemcpyDeviceToHost, st));
  GS_CUDA_TRY(cudaEventRecord(c->ev_m, st));
  if (n > 0)
    GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tmp_bytes, c->dkey_in.as<uint32_t>(),
                                                c->dkey_out.as<uint32_t>(), c->iota.as<uint32_t>(),
                                                c->perm.as<uint32_t>(), n, 0, 32, st));
  GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tmp2, cnt_it, c->offsets.as<uint32_t>(), n + 1, st));
  GS_CUDA_TRY(cudaEventSynchronize(c->ev_m));
  // 64-bit total accumulated by the projection kernel (== offsets_g[N] whenever the u32 scans did
  // not wrap); instance indices are 32-bit from here on
  if (*c->host_m >= (1ull << 31))
    return gs_set_error_msg(GS_ERR_UNSUPPORTED, "gs_render_forward: more than 2^31 tile instances");
  const long long m = (long long)*c->host_m;
  const size_t M = (size_t)m;
  m_out = m;

  gs_mark(c, 2, st);
  // tile-id sort key width (GS_TILE_KEY_BYTES=4 forces the wide path, for tests)
  static const int forced_key = getenv("GS_TILE_KEY_BYTES") ? atoi(getenv("GS_TILE_KEY_BYTES")) : 0;
  const int key_bytes = (g.n_tiles <= 65536 && forced_key != 4) ? 2 : 4;
  const size_t crow = blend_d == 3 ? 16 : (size_t)gs_sh_stream_width(d) * 4;   // colour / SH stream row bytes
  if (!gather) {
    GS_CUDA_TRY(c->pA.reserve(M * 16 + 16, st));
    GS_CUDA_TRY(c->pC.reserve(M * crow + 16, st));
    GS_CUDA_TRY(c->pB.reserve((M + 2) * 8, st));
  }
  if (m > 0) {
    GS_CUDA_TRY(c->keys_in.reserve(M * 4 + 16, st));
    GS_CUDA_TRY(c->keys_out.reserve(M * 4 + 16, st));
    GS_CUDA_TRY(c->vals_in.reserve(M * 4, st));
    GS_CUDA_TRY(c->vals_out.reserve(M * 4, st));
    // 3. instances in (depth, id) order: tile-id keys + Gaussian-id values
    GS_CUDA_TRY(gs_launch_emit_keys(c->rect.as<uint2>(), c->perm.as<uint32_t>(), c->offsets.as<uint32_t>(), n, g.ntx,
                                    c->keys_in.p, key_bytes, c->vals_in.as<uint32_t>(), st));
    gs_count_launch();
    // 4. stable radix sort on the tile id only -> (tile, depth, id)
    gs_mark(c, 3, st);
    int end_bit = ceil_log2((unsigned)g.n_tiles);
    if (end_bit < 1) end_bit = 1;
    size_t sort_tmp = 0;
    if (key_bytes == 2) {
      GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, c->keys_in.as<uint16_t>(),
                                                  c->keys_out.as<uint16_t>(), c->vals_in.as<uint32_t>(),
                                                  c->vals_out.as<uint32_t>(), (int)m, 0, end_bit, st));
      GS_CUDA_TRY(c->cub_tmp.reserve(sort_tmp, st));
      GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, sort_tmp, c->keys_in.as<uint16_t>(),
                                                  c->keys_out.as<uint16_t>(), c->vals_in.as<uint32_t>(),
                                                  c->vals_out.as<uint32_t>(), (int)m, 0, end_bit, st));
    } else {
      GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, c->keys_in.as<uint32_t>(),
                                                  c->keys_out.as<uint32_t>(), c->vals_in.as<uint32_t>(),
                                                  c->vals_out.as<uint32_t>(), (int)m, 0, end_bit, st));
      GS_CUDA_TRY(c->cub_tmp.reserve(sort_tmp, st));
      GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, sort_tmp, c->keys_in.as<uint32_t>(),
                                                  c->keys_out.as<uint32_t>(), c->vals_in.as<uint32_t>(),
                                                  c->vals_out.as<uint32_t>(), (int)m, 0, end_bit, st));
    }
  }
  // 5. tile ranges + packed sorted record streams
  if (m == 0) gs_mark(c, 3, st);
  gs_mark(c, 4, st);
  if (gather) {
    // no pack pass: only the tile ranges are derived from the sorted keys; the blend kernels pull the records
    // of their tile straight from rec[N] through the sorted id list
    GS_CUDA_TRY(gs_launch_tile_ranges(c->keys_out.p, key_bytes, m, g.n_tiles, c->tile_accum.as<int>(), st));
  } else if (blend_d == 3) {
    GS_CUDA_TRY(gs_launch_pack_sorted(c->keys_out.p, key_bytes, c->vals_out.as<uint32_t>(), m, g.n_tiles, g.ntx,
                                      c->rec.as<GsRec>(), c->offsets_g.as<uint32_t>(), c->pA.as<float4>(),
                                      c->pB.as<float2>(), c->pC.as<float4>(), c->tile_accum.as<int>(), st));
  } else {
    GS_CUDA_TRY(gs_launch_pack_sorted_sh(c->keys_out.p, key_bytes, c->vals_out.as<uint32_t>(), m, g.n_tiles, g.ntx,
                                         c->rec.as<GsRec>(), c->offsets_g.as<uint32_t>(), rgb, d,
                                         gs_sh_stream_width(d), c->pA.as<float4>(), c->pB.as<float2>(),
                                         c->pC.as<float>(), c->tile_accum.as<int>(), st));
  }
  if (m > 0) gs_count_launch();   // pack, or the tile-range pass of the gather path
  return 0;
}

static int render_forward_impl(gs_ctx* c, const char* who, const float* pos, const float* rgb, const float* opa,
                               const float* quat, const float* scale, int n, int d, int scale_activation,
                               const gs_camera* cam, float* image, float* final_img, int64_t* culling_mask,
                               gs_stream_t stream, const gs_render_aux* ax = nullptr,
                               const gs_render_feat* ft = nullptr) {
  if (!c || !cam || n < 0) return gs_fail(GS_ERR_INVALID_ARG, who, "bad arguments");
  if (d != 3 && gs_sh_basis_count(d) == 0)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "colour width must be 3 (RGB), 27 (SH deg 2) or 48 (SH deg 3)");
  if (int rc = check_camera(*cam, who)) return rc;
  if (!image || (n > 0 && (!pos || !rgb || !opa || !quat || !scale)))
    return gs_fail(GS_ERR_INVALID_ARG, who, "null tensor pointer");
  // per-Gaussian SH: the projection writes an RGB colour, and everything that serves the blend runs as for d == 3;
  // only the projection kernels, the push bucket and the caller's tensors keep the parameter width d
  const bool sh_gaussian = d != 3 && c->sh_eval == GS_SH_EVAL_GAUSSIAN;
  const int blend_d = sh_gaussian ? 3 : d;   // colour width of the blend
  const bool filt_on = c->filter2d != GS_FILTER2D_NONE;
  GsAuxOut aux_out;
  bool use_aux;
  if (int rc = parse_aux(ax, final_img, aux_out, use_aux, who)) return rc;
  // a forward that writes aux may be differentiated through it: its backward kernel must exist too
  if (use_aux)
    if (int rc = gs_blend_aux_supported(blend_d, true, ax->aux != nullptr)) return rc;
  const bool gather = gs_tuning().gather != 0;   // RGB and SH: no pack pass
  if (ft) {
    if (!gs_feat_width_ok(ft->f)) return gs_fail(GS_ERR_INVALID_ARG, who, "f must be 8, 16 or 32");
    if (!ft->map || (n > 0 && !ft->feat)) return gs_fail(GS_ERR_INVALID_ARG, who, "null feat or map");
    if ((reinterpret_cast<uintptr_t>(ft->feat) | reinterpret_cast<uintptr_t>(ft->map) |
         reinterpret_cast<uintptr_t>(ft->map_final)) % 16)
      return gs_fail(GS_ERR_INVALID_ARG, who, "feat, map and map_final must be 16-byte aligned");
    if (ft->map_final && !final_img) return gs_fail(GS_ERR_INVALID_ARG, who, "map_final needs image_final");
    if (blend_d != 3)
      return gs_fail(GS_ERR_UNSUPPORTED, who, "SH colour evaluated per pixel has no feature kernel (use GS_SH_EVAL_GAUSSIAN)");
    if (!gather)
      return gs_fail(GS_ERR_UNSUPPORTED, who, "the packed path (gs_tune(\"gather\", 0)) has no feature kernel");
  }
  const float* f3d = c->filter3d;
  if (f3d && c->filter3d_n != n) return gs_fail(GS_ERR_INVALID_ARG, who, "the 3-D filter is sized for another n");
  GsLens lens{};
  bool lens_on;
  if (int rc = resolve_lenses(c, cam, 1, &lens, lens_on, who)) return rc;
  if (lens_on && blend_d != 3 && lens.model != GS_LENS_PINHOLE)
    return gs_fail(GS_ERR_UNSUPPORTED, who,
                   "SH colour evaluated per pixel takes a principal point but no distortion (use GS_SH_EVAL_GAUSSIAN)");
  if (int rc = begin_forward(c, who)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  GsFrameGeom g;
  if (int rc = frame_geom(*cam, 1, g, who)) return rc;

  const GsView vw = view_constants(c, cam, g);
  const GsTileGrid& grid = vw.grid;
  const GsCam& dc = vw.cam;
  const GsFilter2d& filt = vw.filt;
  const float half_w = vw.half_w, half_h = vw.half_h;

  size_t N = (size_t)n;
  if (int rc = reserve_frame(c, N, g.n_tiles, st)) return rc;

  if (blend_d != 3) {
    // world-space ray set-up for per-pixel SH, reference splatter.py:305-321 (RayInfo):
    // c2w = inverse(w2c); rays_o = -c2w t; lefttop = c2w (((-Wp/2+.5)/fx, (-Hp/2+.5)/fy, 1) - t), with a lens's
    // principal point shifting the first two components by -((cx - W/2) / fx, (cy - H/2) / fy)
    GS_CUDA_TRY(c->rays.reserve(64, st));
    double m3[9], inv[9];
    for (int k = 0; k < 9; ++k) m3[k] = cam->rot[k];
    double det3 = m3[0] * (m3[4] * m3[8] - m3[5] * m3[7]) - m3[1] * (m3[3] * m3[8] - m3[5] * m3[6]) +
                  m3[2] * (m3[3] * m3[7] - m3[4] * m3[6]);
    inv[0] = (m3[4] * m3[8] - m3[5] * m3[7]) / det3;
    inv[1] = (m3[2] * m3[7] - m3[1] * m3[8]) / det3;
    inv[2] = (m3[1] * m3[5] - m3[2] * m3[4]) / det3;
    inv[3] = (m3[5] * m3[6] - m3[3] * m3[8]) / det3;
    inv[4] = (m3[0] * m3[8] - m3[2] * m3[6]) / det3;
    inv[5] = (m3[2] * m3[3] - m3[0] * m3[5]) / det3;
    inv[6] = (m3[3] * m3[7] - m3[4] * m3[6]) / det3;
    inv[7] = (m3[1] * m3[6] - m3[0] * m3[7]) / det3;
    inv[8] = (m3[0] * m3[4] - m3[1] * m3[3]) / det3;
    double lt[3] = {(-(double)g.wp / 2 + 0.5) / cam->focal_x - cam->tran[0],
                    (-(double)g.hp / 2 + 0.5) / cam->focal_y - cam->tran[1], 1.0 - cam->tran[2]};
    if (lens_on) {
      const gs_lens& l = c->lens_set[0];
      lt[0] -= ((double)l.cx - cam->width / 2.0) / cam->focal_x;
      lt[1] -= ((double)l.cy - cam->height / 2.0) / cam->focal_y;
    }
    for (int k = 0; k < 3; ++k) {
      c->host_rays[k] = (float)(-(inv[3 * k] * cam->tran[0] + inv[3 * k + 1] * cam->tran[1] + inv[3 * k + 2] * cam->tran[2]));
      c->host_rays[3 + k] = (float)(inv[3 * k] * lt[0] + inv[3 * k + 1] * lt[1] + inv[3 * k + 2] * lt[2]);
      c->host_rays[6 + k] = (float)(inv[3 * k] / cam->focal_x);
      c->host_rays[9 + k] = (float)(inv[3 * k + 1] / cam->focal_y);
    }
    GS_CUDA_TRY(cudaMemcpyAsync(c->rays.p, c->host_rays, 48, cudaMemcpyHostToDevice, st));
  }
  // 1. projection + activations + tile rectangle
  gs_mark(c, 0, st);
  GS_CUDA_TRY(cudaMemsetAsync(c->counters.p, 0, 64, st));
  GS_CUDA_TRY(cudaMemsetAsync(c->count.as<uint32_t>() + N, 0, 4, st));
  GS_CUDA_TRY(gs_launch_fused_project(pos, rgb, opa, quat, scale, n, d, scale_activation, dc, grid, cam->near_plane,
                                      half_w, half_h, c->rec.as<GsRec>(), c->rect.as<uint2>(), c->count.as<uint32_t>(),
                                      c->dkey_in.as<uint32_t>(), culling_mask, c->counters.as<unsigned int>(), st,
                                      sh_gaussian, filt_on ? &filt : nullptr, f3d, lens_on ? &lens : nullptr));
  if (n > 0) gs_count_launch();
  long long m = 0;
  if (int rc = bin_frame(c, n, g, gather, blend_d, d, rgb, st, m)) return rc;
  // 6. blend (+ optional fused clamp & centre crop, splatter.py:652-653 / :267-272)
  GsCrop crop{(g.wp - g.width) / 2, (g.hp - g.height) / 2, g.width, g.height};
  gs_mark(c, 5, st);
  if (ft) {
    GS_CUDA_TRY(gs_launch_blend_feat_fwd(c->rec.as<GsRec>(), ft->feat, ft->f, c->vals_out.as<uint32_t>(),
                                         c->tile_accum.as<int>(), g, image, c->tile_neff.as<int>(), final_img, crop,
                                         use_aux ? &aux_out : nullptr, ft->map, ft->map_final, st));
  } else if (blend_d == 3) {
    GS_CUDA_TRY(gs_launch_blend_fwd(c->pA.as<float4>(), c->pB.as<float2>(), c->pC.as<float4>(),
                                    gather ? c->rec.as<GsRec>() : nullptr, c->vals_out.as<uint32_t>(),
                                    c->tile_accum.as<int>(), g, image, c->tile_neff.as<int>(), final_img, crop, st,
                                    use_aux ? &aux_out : nullptr));
  } else {
    const float* rp = c->rays.as<float>();
    GsRayPtrs rays{rp, rp + 3, rp + 6, rp + 9};
    GS_CUDA_TRY(gs_launch_blend_sh_fwd(c->pA.as<float4>(), c->pB.as<float2>(), c->pC.as<float>(),
                                       gather ? c->rec.as<GsRec>() : nullptr, rgb, c->vals_out.as<uint32_t>(),
                                       c->offsets_g.as<uint32_t>(), d,
                                       c->tile_accum.as<int>(), g, rays, image, c->tile_neff.as<int>(), final_img,
                                       crop, st, use_aux ? &aux_out : nullptr));
  }
  gs_count_launch();   // blend forward
  gs_mark(c, 6, st);
  commit_forward(c, n, d, scale_activation, m, g, vw, cam->near_plane, 0, sh_gaussian, gather, filt_on, aux_out, ft,
                 f3d, lens_on, lens);
  return 0;
}

extern "C" int gs_render_forward(gs_ctx* c, const float* pos, const float* rgb, const float* opa, const float* quat,
                                 const float* scale, int n, int d, int scale_activation, const gs_camera* cam,
                                 float* image, int64_t* culling_mask, gs_stream_t stream) {
  return render_forward_impl(c, "gs_render_forward", pos, rgb, opa, quat, scale, n, d, scale_activation, cam, image,
                             nullptr, culling_mask, stream);
}

extern "C" int gs_render_forward_final(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                       const float* quat, const float* scale, int n, int d, int scale_activation,
                                       const gs_camera* cam, float* image_raw_padded, float* image_final,
                                       int64_t* culling_mask, gs_stream_t stream) {
  if (!image_final) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_forward_final: null image_final");
  return render_forward_impl(c, "gs_render_forward_final", pos, rgb, opa, quat, scale, n, d, scale_activation, cam,
                             image_raw_padded, image_final, culling_mask, stream);
}

// one u32 tag per gradient row: rows written by this backward carry `epoch`; the tails of
// saturated tiles are never written nor read (saves ~0.2 GB of HBM writes + reads at C3)
static int next_row_epoch(gs_ctx* c, size_t M, cudaStream_t st) {
  const size_t before = c->row_epoch.cap;            // (a caching allocator may hand the same address back)
  GS_CUDA_TRY(c->row_epoch.reserve(M * 4 + 16, st));
  if (c->row_epoch.cap != before || c->epoch == 0xffffffffu) {
    GS_CUDA_TRY(cudaMemsetAsync(c->row_epoch.p, 0, c->row_epoch.cap, st));
    c->epoch = 0;
  }
  ++c->epoch;
  return 0;
}

// The backward of the last forward, single-view or batched (batch: the caller is gs_render_backward_batch[_cam], which
// has checked what only a batched frame needs; grad_cam is then [n_views][12]).
static int render_backward_impl(gs_ctx* c, const char* who, bool batch, const float* pos, const float* rgb,
                                const float* opa, const float* quat, const float* scale, const float* image,
                                const float* grad_image, int grad_is_final, float* grad_pos, float* grad_rgb,
                                float* grad_opa, float* grad_quat, float* grad_scale, gs_stream_t stream,
                                const float* aux = nullptr, const float* grad_aux = nullptr,
                                float* grad_cam = nullptr, const float* fmap = nullptr,
                                const float* grad_map = nullptr, float* grad_feat = nullptr) {
  if (!c) return gs_fail(GS_ERR_INVALID_ARG, who, "null ctx");
  if (!c->have_forward) return gs_fail(GS_ERR_NO_FORWARD, who, "no forward on this ctx");
  if (c->n_views && !batch)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward was batched (use gs_render_backward_batch)");
  if (c->surfel)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward rendered surfels (use gs_render_backward_surfel)");
  // camera only (grad_cam, the five parameter gradients all NULL: the caller has checked the set is not mixed)
  const bool cam_only = grad_cam && !grad_pos;
  if (!image || !grad_image || (!cam_only && (!grad_pos || !grad_rgb || !grad_opa || !grad_quat || !grad_scale)) ||
      (c->n > 0 && (!pos || !rgb || !opa || !quat || !scale)))
    return gs_fail(GS_ERR_INVALID_ARG, who, "null tensor pointer");
  if (grad_cam) {
    if (c->d != 3 && !c->sh_gaussian)
      return gs_fail(GS_ERR_UNSUPPORTED, who, "SH colour evaluated per pixel has no camera gradient (use GS_SH_EVAL_GAUSSIAN)");
    if (c->push.world) return gs_fail(GS_ERR_UNSUPPORTED, who, "not available with a gradient push configured");
  }
  if (grad_aux) {
    if (!c->have_aux) return gs_fail(GS_ERR_INVALID_ARG, who, "grad_aux given but the forward wrote no aux");
    if (!aux) return gs_fail(GS_ERR_INVALID_ARG, who, "grad_aux needs the forward's aux");
    if (int rc = gs_blend_aux_supported(c->sh_gaussian ? 3 : c->d, false, true)) return rc;
  }
  const int d = c->d;
  const int blend_d = c->sh_gaussian ? 3 : d;   // colour width of the blend: the forward's SH mode, not the current one
  // densification statistics: every backward that computes parameter gradients, not a camera-only one
  const bool stats = c->stats_on && !cam_only;
  const bool absgrad = stats && c->stats.absgrad;
  if (stats) {
    if (c->stats.n != c->n) return gs_fail(GS_ERR_INVALID_ARG, who, "the densify statistics are sized for another n");
    if (absgrad)
      if (int rc = gs_blend_absgrad_supported(blend_d, c->gather)) return rc;
  }
  if (c->push.world && c->lens_on)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "a frame with a lens has no gradient push (all-reduce the gradients instead)");
  if (c->push.world) {
    // every gradient segment must lie inside the sliced bucket, quaternions on 16-byte offsets
    const float* lo = c->push.bucket;
    const float* hi = lo + (size_t)c->push.world * c->push.per;
    const size_t nn = (size_t)c->n;
    const float* seg[5] = {grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale};
    const size_t len[5] = {3 * nn, (size_t)d * nn, nn, 4 * nn, 3 * nn};
    for (int k = 0; k < 5; ++k)
      if (seg[k] < lo || seg[k] + len[k] > hi)
        return gs_fail(GS_ERR_INVALID_ARG, who, "gradient buffers are not inside the push bucket");
    if ((grad_quat - lo) % 4) return gs_fail(GS_ERR_INVALID_ARG, who, "grad_quat must sit on a 16-byte bucket offset");
  }
  if (int rc = gs_check_device(c->device, who)) return rc;
  g_cur_alloc = &c->allocator;
  cudaStream_t st = (cudaStream_t)stream;
  size_t M = (size_t)c->m;
  const size_t grow = blend_d == 3 ? (size_t)GS_GREC * 4 : (size_t)gs_sh_grad_width(d) * 4;
  GS_CUDA_TRY(c->grad_inst.reserve(M * grow + 16, st));
  if (grad_map) GS_CUDA_TRY(c->grad_feat_inst.reserve(M * (size_t)c->feat_f * 4 + 16, st));
  if (int rc = next_row_epoch(c, M, st)) return rc;
  c->ev_bwd_valid = false;
  GsCrop crop{(c->geom.wp - c->geom.width) / 2, (c->geom.hp - c->geom.height) / 2, c->geom.width, c->geom.height};
  gs_mark(c, 7, st);
  if (c->m > 0) {
    if (c->n_views) {
      GS_CUDA_TRY(gs_launch_blend_bwd_batch(c->rec.as<GsRec>(), c->vals_out.as<uint32_t>(), c->offsets_g.as<uint32_t>(),
                                            c->tile_accum.as<int>(), c->geom, c->views.as<GsView>(), image, grad_image,
                                            c->grad_inst.as<float>(), grad_is_final, crop, c->row_epoch.as<uint32_t>(),
                                            c->epoch, c->tile_neff_b.as<int>(), st, aux, grad_aux, absgrad));
    } else if (grad_map) {
      GS_CUDA_TRY(gs_launch_blend_feat_bwd(c->rec.as<GsRec>(), c->feat, c->feat_f, c->vals_out.as<uint32_t>(),
                                           c->offsets_g.as<uint32_t>(), c->tile_accum.as<int>(), c->geom, image,
                                           grad_image, fmap, grad_map, c->grad_inst.as<float>(),
                                           c->grad_feat_inst.as<float>(), grad_is_final, crop,
                                           c->row_epoch.as<uint32_t>(), c->epoch, c->tile_neff_b.as<int>(), aux,
                                           grad_aux, st));
    } else if (blend_d == 3) {
      GS_CUDA_TRY(gs_launch_blend_bwd(c->pA.as<float4>(), c->pB.as<float2>(), c->pC.as<float4>(),
                                      c->gather ? c->rec.as<GsRec>() : nullptr, c->vals_out.as<uint32_t>(),
                                      c->offsets_g.as<uint32_t>(), c->tile_accum.as<int>(), c->geom, image, grad_image,
                                      c->grad_inst.as<float>(),
                                      grad_is_final, crop, c->row_epoch.as<uint32_t>(), c->epoch,
                                      c->tile_neff_b.as<int>(), st, aux, grad_aux, absgrad));
    } else {
      const float* rp = c->rays.as<float>();
      GsRayPtrs rays{rp, rp + 3, rp + 6, rp + 9};
      GS_CUDA_TRY(gs_launch_blend_sh_bwd(c->pA.as<float4>(), c->pB.as<float2>(), c->pC.as<float>(),
                                         c->gather ? c->rec.as<GsRec>() : nullptr, rgb, c->vals_out.as<uint32_t>(),
                                         c->offsets_g.as<uint32_t>(), d,
                                         c->tile_accum.as<int>(), c->geom, rays, image, grad_image,
                                         c->grad_inst.as<float>(), grad_is_final, crop,
                                         c->row_epoch.as<uint32_t>(), c->epoch, c->tile_neff_b.as<int>(), st, aux,
                                         grad_aux));
    }
    gs_count_launch();
    c->have_backward = true;
  }
  gs_mark(c, 8, st);
  if (grad_cam && c->n_views > 1) {
    // B views: one row of 12 partial sums per CTA and view, one finishing CTA per view (grad_cam is [B][12]).  One
    // view: the single-view kernels below, as for the parameter gradients of a one-view batch
    GS_CUDA_TRY(c->cam_part.reserve((size_t)c->n_views * gs_cam_grad_workspace_bytes(c->n) + 16, st));
    GS_CUDA_TRY(gs_launch_fused_project_bwd_batch_cam(pos, rgb, opa, quat, scale, c->n, c->n_views, d, c->scale_act,
                                                      c->views.as<GsView>(), c->near_plane,
                                                      c->offsets_g.as<uint32_t>(), c->count.as<uint32_t>(),
                                                      c->grad_inst.as<float>(), c->row_epoch.as<uint32_t>(), c->epoch,
                                                      grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale,
                                                      c->cam_part.as<float>(), grad_cam, st, grad_aux != nullptr,
                                                      c->sh_gaussian, c->filt_on, c->f3d,
                                                      c->lens_on ? c->lenses.as<GsLens>() : nullptr));
    gs_count_launch(c->n > 0 ? 2 : 1);   // projection backward + the finishing sums
  } else if (grad_cam) {
    GS_CUDA_TRY(c->cam_part.reserve(gs_cam_grad_workspace_bytes(c->n) + 16, st));
    GS_CUDA_TRY(gs_launch_fused_project_bwd_cam(pos, rgb, opa, quat, scale, c->n, d, c->scale_act, c->cam,
                                                c->near_plane, c->half_w, c->half_h, c->offsets_g.as<uint32_t>(),
                                                c->count.as<uint32_t>(), c->grad_inst.as<float>(),
                                                c->row_epoch.as<uint32_t>(), c->epoch, grad_pos, grad_rgb, grad_opa,
                                                grad_quat, grad_scale, c->cam_part.as<float>(), grad_cam, st,
                                                grad_aux != nullptr, c->sh_gaussian, c->filt_on ? &c->filt : nullptr,
                                                c->f3d, c->lens_on ? &c->lens : nullptr));
    gs_count_launch(c->n > 0 ? 2 : 1);   // projection backward + the finishing sum (always: grad_cam is always written)
  } else if (c->n_views > 1) {
    // B views: the batched kernels, which take each Gaussian's views in order.  One view: the pairs are the Gaussians,
    // so the single-view kernels run (the gradients are theirs bit for bit, and they are the faster kernels for one view)
    GS_CUDA_TRY(gs_launch_fused_project_bwd_batch(pos, rgb, opa, quat, scale, c->n, c->n_views, d, c->scale_act,
                                                  c->views.as<GsView>(), c->near_plane, c->offsets_g.as<uint32_t>(),
                                                  c->count.as<uint32_t>(), c->grad_inst.as<float>(),
                                                  c->row_epoch.as<uint32_t>(), c->epoch, grad_pos, grad_rgb, grad_opa,
                                                  grad_quat, grad_scale, st, grad_aux != nullptr, c->sh_gaussian,
                                                  c->filt_on, c->f3d, c->lens_on ? c->lenses.as<GsLens>() : nullptr));
    if (c->n > 0) gs_count_launch();
  } else {
    GS_CUDA_TRY(gs_launch_fused_project_bwd(pos, rgb, opa, quat, scale, c->n, d, c->scale_act, c->cam, c->near_plane,
                                            c->half_w, c->half_h, c->offsets_g.as<uint32_t>(), c->count.as<uint32_t>(),
                                            c->grad_inst.as<float>(), c->row_epoch.as<uint32_t>(), c->epoch,
                                            grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale, c->push, st,
                                            grad_aux != nullptr, c->sh_gaussian, c->filt_on ? &c->filt : nullptr,
                                            c->f3d, c->lens_on ? &c->lens : nullptr));
    if (c->n > 0) gs_count_launch();
  }
  if (grad_map) {
    GS_CUDA_TRY(gs_launch_feat_grad(c->offsets_g.as<uint32_t>(), c->count.as<uint32_t>(), c->grad_feat_inst.as<float>(),
                                    c->row_epoch.as<uint32_t>(), c->epoch, c->n, c->feat_f, grad_feat, st));
    if (c->n > 0) gs_count_launch();
  }
  if (stats) {
    if (c->n_views > 1)
      GS_CUDA_TRY(gs_launch_densify_stats_batch(pos, quat, scale, c->n, c->n_views, c->scale_act, c->views.as<GsView>(),
                                                c->near_plane, c->offsets_g.as<uint32_t>(), c->count.as<uint32_t>(),
                                                c->grad_inst.as<float>(), (int)(grow / 4), c->row_epoch.as<uint32_t>(),
                                                c->epoch, c->geom, c->stats, st, c->f3d,
                                                c->lens_on ? c->lenses.as<GsLens>() : nullptr));
    else
      GS_CUDA_TRY(gs_launch_densify_stats(pos, quat, scale, c->n, c->scale_act, c->cam, c->near_plane, c->half_w,
                                          c->half_h, c->filt_on ? c->filt : GsFilter2d{}, c->offsets_g.as<uint32_t>(),
                                          c->count.as<uint32_t>(), c->grad_inst.as<float>(), (int)(grow / 4),
                                          c->row_epoch.as<uint32_t>(), c->epoch, c->geom, c->stats, st, c->f3d,
                                          c->lens_on ? &c->lens : nullptr));
    if (c->n > 0) gs_count_launch();
  }
  gs_mark(c, 9, st);
  c->ev_bwd_valid = c->timing && c->ev_ok;
  return 0;
}

extern "C" int gs_render_backward(gs_ctx* c, const float* pos, const float* rgb, const float* opa, const float* quat,
                                  const float* scale, const float* image, const float* grad_image, float* grad_pos,
                                  float* grad_rgb, float* grad_opa, float* grad_quat, float* grad_scale,
                                  gs_stream_t stream) {
  return render_backward_impl(c, "gs_render_backward", false, pos, rgb, opa, quat, scale, image, grad_image, 0,
                              grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale, stream);
}

extern "C" int gs_render_backward_final(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                        const float* quat, const float* scale, const float* image_raw_padded,
                                        const float* grad_final, float* grad_pos, float* grad_rgb, float* grad_opa,
                                        float* grad_quat, float* grad_scale, gs_stream_t stream) {
  return render_backward_impl(c, "gs_render_backward_final", false, pos, rgb, opa, quat, scale, image_raw_padded,
                              grad_final, 1, grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale, stream);
}

extern "C" int gs_render_forward_aux(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                     const float* quat, const float* scale, int n, int d, int scale_activation,
                                     const gs_camera* cam, float* image_raw_padded, float* image_final,
                                     int64_t* culling_mask, const gs_render_aux* aux, gs_stream_t stream) {
  return render_forward_impl(c, "gs_render_forward_aux", pos, rgb, opa, quat, scale, n, d, scale_activation, cam,
                             image_raw_padded, image_final, culling_mask, stream, aux);
}

extern "C" int gs_render_backward_aux(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                      const float* quat, const float* scale, const float* image_raw_padded,
                                      const float* grad_image, int grad_is_final, const float* aux,
                                      const float* grad_aux, float* grad_pos, float* grad_rgb, float* grad_opa,
                                      float* grad_quat, float* grad_scale, gs_stream_t stream) {
  return render_backward_impl(c, "gs_render_backward_aux", false, pos, rgb, opa, quat, scale, image_raw_padded,
                              grad_image, grad_is_final ? 1 : 0, grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale,
                              stream, aux, grad_aux);
}

extern "C" int gs_render_backward_cam(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                      const float* quat, const float* scale, const float* image_raw_padded,
                                      const float* grad_image, int grad_is_final, const float* aux,
                                      const float* grad_aux, float* grad_pos, float* grad_rgb, float* grad_opa,
                                      float* grad_quat, float* grad_scale, float* grad_cam, gs_stream_t stream) {
  if (!grad_cam) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_cam: null grad_cam");
  const int n_null = !grad_pos + !grad_rgb + !grad_opa + !grad_quat + !grad_scale;
  if (n_null != 0 && n_null != 5)
    return gs_set_error_msg(GS_ERR_INVALID_ARG,
                            "gs_render_backward_cam: the five parameter gradients must be all NULL or all non-NULL");
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_cam: null ctx");
  return render_backward_impl(c, "gs_render_backward_cam", false, pos, rgb, opa, quat, scale, image_raw_padded,
                              grad_image, grad_is_final ? 1 : 0, grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale,
                              stream, aux, grad_aux, grad_cam);
}

extern "C" int gs_render_forward_feat(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                      const float* quat, const float* scale, int n, int d, int scale_activation,
                                      const gs_camera* cam, float* image_raw_padded, float* image_final,
                                      int64_t* culling_mask, const gs_render_aux* aux, const gs_render_feat* feat,
                                      gs_stream_t stream) {
  if (!feat) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_forward_feat: null feat");
  return render_forward_impl(c, "gs_render_forward_feat", pos, rgb, opa, quat, scale, n, d, scale_activation, cam,
                             image_raw_padded, image_final, culling_mask, stream, aux, feat);
}

extern "C" int gs_render_backward_feat(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                       const float* quat, const float* scale, const float* image_raw_padded,
                                       const float* grad_image, int grad_is_final, const float* aux,
                                       const float* grad_aux, const float* feat, const float* map,
                                       const float* grad_map, float* grad_pos, float* grad_rgb, float* grad_opa,
                                       float* grad_quat, float* grad_scale, float* grad_feat, gs_stream_t stream) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: null ctx");
  if (!c->have_forward) return gs_set_error_msg(GS_ERR_NO_FORWARD, "gs_render_backward_feat: no forward on this ctx");
  if (c->surfel)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: the last forward rendered surfels (use "
                                                "gs_render_backward_surfel)");
  if (c->n_views)
    return gs_set_error_msg(GS_ERR_INVALID_ARG,
                            "gs_render_backward_feat: the last forward was batched (use gs_render_backward_batch)");
  if (!c->feat_f)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: the forward blended no features");
  if (feat != c->feat)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: feat is not the forward's feature tensor");
  if (c->n > 0 && !grad_feat) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: null grad_feat");
  if (grad_map) {
    if (!map) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: grad_map needs the forward's map");
    if ((reinterpret_cast<uintptr_t>(map) | reinterpret_cast<uintptr_t>(grad_map)) % 16)
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_backward_feat: map and grad_map must be 16-byte aligned");
    if (c->stats_on && c->stats.absgrad)
      return gs_set_error_msg(GS_ERR_UNSUPPORTED, "gs_render_backward_feat: absgrad statistics are not available with a "
                                                  "feature gradient");
    if (c->push.world)
      return gs_set_error_msg(GS_ERR_UNSUPPORTED, "gs_render_backward_feat: a feature gradient is not part of the push "
                                                  "bucket; not available with a gradient push configured");
  }
  const int f = c->feat_f, n = c->n;
  int rc = render_backward_impl(c, "gs_render_backward_feat", false, pos, rgb, opa, quat, scale, image_raw_padded,
                                grad_image, grad_is_final ? 1 : 0, grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale,
                                stream, aux, grad_aux, nullptr, map, grad_map, grad_feat);
  if (rc || grad_map || n == 0) return rc;
  GS_CUDA_TRY(cudaMemsetAsync(grad_feat, 0, (size_t)n * f * sizeof(float), (cudaStream_t)stream));
  return 0;
}

// ---- batched frames ---------------------------------------------------------------------
extern "C" int gs_render_forward_batch(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                       const float* quat, const float* scale, int n, int d, int scale_activation,
                                       int n_views, const gs_camera* cams, float* image, float* final_img,
                                       int64_t* culling_mask, const gs_render_aux* ax, gs_stream_t stream) {
  const char* who = "gs_render_forward_batch";
  if (!c || !cams) return gs_fail(GS_ERR_INVALID_ARG, who, "null ctx or cams");
  if (n_views < 1 || n_views > GS_MAX_VIEWS) return gs_fail(GS_ERR_INVALID_ARG, who, "n_views must be in 1 .. GS_MAX_VIEWS");
  if (n < 0) return gs_fail(GS_ERR_INVALID_ARG, who, "n < 0");
  if (d != 3 && gs_sh_basis_count(d) == 0)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "colour width must be 3 (RGB), 27 (SH deg 2) or 48 (SH deg 3)");
  const gs_camera& c0 = cams[0];
  for (int v = 0; v < n_views; ++v) {
    const gs_camera& cv = cams[v];
    if (int rc = check_camera(cv, who)) return rc;
    if (cv.width != c0.width || cv.height != c0.height || !(cv.near_plane == c0.near_plane) ||
        !(cv.tile_thresh == c0.tile_thresh))
      return gs_fail(GS_ERR_INVALID_ARG, who, "the views must share width, height, near_plane and tile_thresh");
  }
  GsFrameGeom g;
  if (int rc = frame_geom(c0, n_views, g, who)) return rc;
  if ((long long)n * n_views >= (1ll << 31)) return gs_fail(GS_ERR_INVALID_ARG, who, "B n must be < 2^31");
  if (!image || (n > 0 && (!pos || !rgb || !opa || !quat || !scale)))
    return gs_fail(GS_ERR_INVALID_ARG, who, "null tensor pointer");
  const bool sh_gaussian = d != 3 && c->sh_eval == GS_SH_EVAL_GAUSSIAN;
  if (d != 3 && !sh_gaussian)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "SH colour evaluated per pixel has no batched kernel (use GS_SH_EVAL_GAUSSIAN)");
  if (int rc = gs_blend_batch_supported()) return rc;
  if (c->push.world) return gs_fail(GS_ERR_UNSUPPORTED, who, "not available with a gradient push configured");
  const float* f3d = c->filter3d;
  if (f3d && c->filter3d_n != n) return gs_fail(GS_ERR_INVALID_ARG, who, "the 3-D filter is sized for another n");
  GsAuxOut aux_out;
  bool use_aux;
  if (int rc = parse_aux(ax, final_img, aux_out, use_aux, who)) return rc;
  GsLens lenses[GS_MAX_VIEWS] = {};
  bool lens_on;
  if (int rc = resolve_lenses(c, cams, n_views, lenses, lens_on, who)) return rc;
  if (int rc = begin_forward(c, who)) return rc;
  cudaStream_t st = (cudaStream_t)stream;

  const int nb = n * n_views;   // (view, Gaussian) pairs
  if (int rc = reserve_frame(c, (size_t)nb, g.n_tiles, st)) return rc;
  GS_CUDA_TRY(c->views.reserve(sizeof(GsView) * GS_MAX_VIEWS, st));
  // the previous upload from the pinned staging may still be pending when its forward returned early on an error
  GS_CUDA_TRY(cudaEventSynchronize(c->ev_views));
  for (int v = 0; v < n_views; ++v) c->host_views[v] = view_constants(c, &cams[v], g);
  GS_CUDA_TRY(cudaMemcpyAsync(c->views.p, c->host_views, sizeof(GsView) * n_views, cudaMemcpyHostToDevice, st));
  if (lens_on) {
    GS_CUDA_TRY(c->lenses.reserve(sizeof(GsLens) * GS_MAX_VIEWS, st));
    for (int v = 0; v < n_views; ++v) c->host_lenses[v] = lenses[v];
    GS_CUDA_TRY(cudaMemcpyAsync(c->lenses.p, c->host_lenses, sizeof(GsLens) * n_views, cudaMemcpyHostToDevice, st));
  }
  GS_CUDA_TRY(cudaEventRecord(c->ev_views, st));
  const bool filt_on = c->filter2d != GS_FILTER2D_NONE;

  gs_mark(c, 0, st);
  GS_CUDA_TRY(cudaMemsetAsync(c->counters.p, 0, 64, st));
  GS_CUDA_TRY(cudaMemsetAsync(c->count.as<uint32_t>() + nb, 0, 4, st));
  GS_CUDA_TRY(gs_launch_fused_project_batch(pos, rgb, opa, quat, scale, n, n_views, d, scale_activation,
                                            c->views.as<GsView>(), c0.near_plane, c->rec.as<GsRec>(),
                                            c->rect.as<uint2>(), c->count.as<uint32_t>(), c->dkey_in.as<uint32_t>(),
                                            culling_mask, c->counters.as<unsigned int>(), st, sh_gaussian, filt_on,
                                            f3d, lens_on ? c->lenses.as<GsLens>() : nullptr));
  if (n > 0) gs_count_launch();
  long long m = 0;
  if (int rc = bin_frame(c, nb, g, true, 3, d, rgb, st, m)) return rc;
  GsCrop crop{(g.wp - g.width) / 2, (g.hp - g.height) / 2, g.width, g.height};
  gs_mark(c, 5, st);
  GS_CUDA_TRY(gs_launch_blend_fwd_batch(c->rec.as<GsRec>(), c->vals_out.as<uint32_t>(), c->tile_accum.as<int>(), g,
                                        c->views.as<GsView>(), image, c->tile_neff.as<int>(), final_img, crop, st,
                                        use_aux ? &aux_out : nullptr));
  gs_count_launch();   // blend forward
  gs_mark(c, 6, st);
  // view 0's constants: a one-view batch is differentiated by the single-view projection backward
  commit_forward(c, n, d, scale_activation, m, g, c->host_views[0], c0.near_plane, n_views, sh_gaussian, true, filt_on,
                 aux_out, nullptr, f3d, lens_on, lenses[0]);
  return 0;
}

extern "C" int gs_render_backward_batch(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                        const float* quat, const float* scale, const float* image,
                                        const float* grad_image, int grad_is_final, const float* aux,
                                        const float* grad_aux, float* grad_pos, float* grad_rgb, float* grad_opa,
                                        float* grad_quat, float* grad_scale, gs_stream_t stream) {
  const char* who = "gs_render_backward_batch";
  if (!c) return gs_fail(GS_ERR_INVALID_ARG, who, "null ctx");
  if (!c->have_forward) return gs_fail(GS_ERR_NO_FORWARD, who, "no forward on this ctx");
  if (c->surfel)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward rendered surfels (use gs_render_backward_surfel)");
  if (!c->n_views) return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward was not batched");
  if (c->push.world) return gs_fail(GS_ERR_UNSUPPORTED, who, "not available with a gradient push configured");
  if (int rc = gs_blend_batch_supported()) return rc;
  return render_backward_impl(c, who, true, pos, rgb, opa, quat, scale, image, grad_image, grad_is_final ? 1 : 0,
                              grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale, stream, aux, grad_aux);
}

extern "C" int gs_render_backward_batch_cam(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                            const float* quat, const float* scale, const float* image,
                                            const float* grad_image, int grad_is_final, const float* aux,
                                            const float* grad_aux, float* grad_pos, float* grad_rgb, float* grad_opa,
                                            float* grad_quat, float* grad_scale, float* grad_cams,
                                            gs_stream_t stream) {
  const char* who = "gs_render_backward_batch_cam";
  if (!grad_cams) return gs_fail(GS_ERR_INVALID_ARG, who, "null grad_cams");
  const int n_null = !grad_pos + !grad_rgb + !grad_opa + !grad_quat + !grad_scale;
  if (n_null != 0 && n_null != 5)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the five parameter gradients must be all NULL or all non-NULL");
  if (!c) return gs_fail(GS_ERR_INVALID_ARG, who, "null ctx");
  if (!c->have_forward) return gs_fail(GS_ERR_NO_FORWARD, who, "no forward on this ctx");
  if (c->surfel)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward rendered surfels (use gs_render_backward_surfel)");
  if (!c->n_views) return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward was not batched");
  if (c->push.world) return gs_fail(GS_ERR_UNSUPPORTED, who, "not available with a gradient push configured");
  if (int rc = gs_blend_batch_supported()) return rc;
  return render_backward_impl(c, who, true, pos, rgb, opa, quat, scale, image, grad_image, grad_is_final ? 1 : 0,
                              grad_pos, grad_rgb, grad_opa, grad_quat, grad_scale, stream, aux, grad_aux, grad_cams);
}

extern "C" int gs_ctx_set_grad_push(gs_ctx* c, const gs_grad_push* p) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_grad_push: null ctx");
  if (!p) {
    c->push = GsGradPush{};
    return 0;
  }
  if (!(p->world == 2 || p->world == 4 || p->world == 8) || p->rank < 0 || p->rank >= p->world || p->per <= 0 ||
      (p->per % 4) || (unsigned long long)p->per * (unsigned)p->world >= (1ull << 32) || !p->bucket ||
      reinterpret_cast<uintptr_t>(p->bucket) % 16)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_grad_push: bad configuration");
  GsGradPush g{};
  g.bucket = p->bucket;
  g.per = (uint32_t)p->per;
  g.rank = p->rank;
  g.world = p->world;
  for (int k = 0; k < p->world; ++k) {
    if (!p->staging[k] || reinterpret_cast<uintptr_t>(p->staging[k]) % 16)
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_grad_push: staging pointers must be 16-byte aligned");
    g.staging[k] = p->staging[k];
  }
  c->push = g;
  return 0;
}

extern "C" int gs_ctx_set_sh_eval(gs_ctx* c, int mode) {
  if (mode != GS_SH_EVAL_PIXEL && mode != GS_SH_EVAL_GAUSSIAN)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_sh_eval: mode must be GS_SH_EVAL_PIXEL or GS_SH_EVAL_GAUSSIAN");
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_sh_eval: null ctx");
  c->sh_eval = mode;
  return 0;
}

extern "C" int gs_ctx_set_filter2d(gs_ctx* c, int mode, float variance_px2) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_filter2d: null ctx");
  if (mode != GS_FILTER2D_NONE && mode != GS_FILTER2D_DILATE && mode != GS_FILTER2D_ANTIALIAS)
    return gs_set_error_msg(GS_ERR_INVALID_ARG,
                            "gs_ctx_set_filter2d: mode must be GS_FILTER2D_NONE, GS_FILTER2D_DILATE or GS_FILTER2D_ANTIALIAS");
  if (!std::isfinite(variance_px2) || !(variance_px2 > 0.f))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_filter2d: variance must be finite and > 0");
  c->filter2d = mode;
  c->filter2d_var = variance_px2;
  return 0;
}

extern "C" int gs_ctx_set_filter3d(gs_ctx* c, const float* filter3d, int n) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_filter3d: null ctx");
  if (n < 0) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_filter3d: n < 0");
  c->filter3d = filter3d;
  c->filter3d_n = filter3d ? n : 0;
  return 0;
}

extern "C" int gs_ctx_set_lens(gs_ctx* c, const gs_lens* lenses, int n) {
  const char* who = "gs_ctx_set_lens";
  if (!c) return gs_fail(GS_ERR_INVALID_ARG, who, "null ctx");
  if (n < 0 || n > GS_MAX_VIEWS) return gs_fail(GS_ERR_INVALID_ARG, who, "n must be in 0 .. GS_MAX_VIEWS");
  if (!lenses && n > 0) return gs_fail(GS_ERR_INVALID_ARG, who, "NULL lenses with n > 0");
  const int m = lenses ? n : 0;
  for (int v = 0; v < m; ++v) {
    const gs_lens& l = lenses[v];
    if (l.model != GS_LENS_PINHOLE && l.model != GS_LENS_OPENCV && l.model != GS_LENS_FISHEYE)
      return gs_fail(GS_ERR_INVALID_ARG, who, "model must be GS_LENS_PINHOLE, GS_LENS_OPENCV or GS_LENS_FISHEYE");
    bool finite = std::isfinite(l.cx) && std::isfinite(l.cy);
    for (int k = 0; k < 4; ++k) finite = finite && std::isfinite(l.k[k]);
    if (!finite) return gs_fail(GS_ERR_INVALID_ARG, who, "cx, cy and k must be finite");
  }
  for (int v = 0; v < m; ++v) c->lens_set[v] = lenses[v];
  c->lens_n = m;
  return 0;
}

extern "C" int gs_filter3d_compute(gs_ctx* c, const float* pos, int n, const gs_camera* cams_host, int n_cams,
                                   float margin, float variance, float* filter3d, gs_stream_t stream) {
  const char* who = "gs_filter3d_compute";
  if (!c || !cams_host || (n > 0 && (!pos || !filter3d))) return gs_fail(GS_ERR_INVALID_ARG, who, "null argument");
  if (n < 0 || n_cams < 1) return gs_fail(GS_ERR_INVALID_ARG, who, "n must be >= 0 and n_cams >= 1");
  if (!std::isfinite(variance) || !(variance > 0.f))
    return gs_fail(GS_ERR_INVALID_ARG, who, "variance must be finite and > 0");
  if (!std::isfinite(margin) || !(margin >= 0.f)) return gs_fail(GS_ERR_INVALID_ARG, who, "margin must be finite and >= 0");
  for (int v = 0; v < n_cams; ++v) {
    const gs_camera& cm = cams_host[v];
    if (cm.width <= 0 || cm.height <= 0 || !std::isfinite(cm.focal_x) || !(cm.focal_x > 0.f) ||
        !std::isfinite(cm.focal_y) || !(cm.focal_y > 0.f))
      return gs_fail(GS_ERR_INVALID_ARG, who, "bad camera (size and focal lengths must be positive and finite)");
    if (!std::isfinite(cm.near_plane) || cm.near_plane < 0.f)
      return gs_fail(GS_ERR_INVALID_ARG, who, "bad camera (near_plane must be finite and >= 0)");
  }
  if (n == 0) return 0;
  if (c->lens_n && c->lens_n != 1 && c->lens_n != n_cams)
    return gs_fail(GS_ERR_INVALID_ARG, who, "the context's lenses are set for another number of views (n must be 1 or n_cams)");
  // the lens variant unless no lens is set or every view's is the image-centre pinhole (then the rate, the test and
  // the bits are those without a lens)
  bool lens_on = false;
  for (int v = 0; v < n_cams && c->lens_n; ++v)
    if (!lens_is_centre_pinhole(c->lens_set[c->lens_n == 1 ? 0 : v], cams_host[v])) lens_on = true;
  if (int rc = gs_check_device(c->device, who)) return rc;
  g_cur_alloc = &c->allocator;
  cudaStream_t st = (cudaStream_t)stream;
  if (!c->ev_f3) GS_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_f3, cudaEventDisableTiming));
  // the previous upload from the pinned staging may still be pending
  GS_CUDA_TRY(cudaEventSynchronize(c->ev_f3));
  if (c->f3_host_cap < n_cams) {
    if (c->f3_host) cudaFreeHost(c->f3_host);
    c->f3_host = nullptr;
    c->f3_host_cap = 0;
    // the view table, then the lens table (GsLens[cap])
    GS_CUDA_TRY(cudaMallocHost(reinterpret_cast<void**>(&c->f3_host),
                               (sizeof(GsF3View) + sizeof(GsLens)) * (size_t)n_cams));
    c->f3_host_cap = n_cams;
  }
  GsLens* lens_host = reinterpret_cast<GsLens*>(c->f3_host + c->f3_host_cap);
  for (int v = 0; v < n_cams; ++v) {
    const gs_camera& cm = cams_host[v];
    GsF3View& o = c->f3_host[v];
    o = GsF3View{};
    for (int k = 0; k < 3; ++k) o.rz[k] = cm.rot[6 + k];
    o.tz = cm.tran[2];
    o.fxd = cm.focal_x;
    for (int k = 0; k < 6; ++k) o.r[k] = cm.rot[k];
    o.t[0] = cm.tran[0];
    o.t[1] = cm.tran[1];
    o.fx = cm.focal_x;
    o.fy = cm.focal_y;
    o.cx = (float)(cm.width / 2.0);
    o.cy = (float)(cm.height / 2.0);
    o.ulo = (float)(-(double)margin * cm.width);
    o.uhi = (float)((1.0 + (double)margin) * cm.width);
    o.wlo = (float)(-(double)margin * cm.height);
    o.whi = (float)((1.0 + (double)margin) * cm.height);
    o.near = cm.near_plane;
    if (lens_on) {
      const gs_lens& l = c->lens_set[c->lens_n == 1 ? 0 : v];
      o.cx = l.cx;
      o.cy = l.cy;
      lens_host[v] = lens_constants(l, cm);
    }
  }
  const size_t vbytes = sizeof(GsF3View) * (size_t)n_cams, lbytes = lens_on ? sizeof(GsLens) * (size_t)n_cams : 0;
  GS_CUDA_TRY(c->f3_dev.reserve(16 + vbytes + lbytes, st));
  unsigned int* min_rate = c->f3_dev.as<unsigned int>();
  GsF3View* views = reinterpret_cast<GsF3View*>(c->f3_dev.as<char>() + 16);
  GsLens* lenses = lens_on ? reinterpret_cast<GsLens*>(c->f3_dev.as<char>() + 16 + vbytes) : nullptr;
  GS_CUDA_TRY(cudaMemsetAsync(min_rate, 0xff, 4, st));
  GS_CUDA_TRY(cudaMemcpyAsync(views, c->f3_host, vbytes, cudaMemcpyHostToDevice, st));
  if (lens_on) GS_CUDA_TRY(cudaMemcpyAsync(lenses, lens_host, lbytes, cudaMemcpyHostToDevice, st));
  GS_CUDA_TRY(cudaEventRecord(c->ev_f3, st));
  GS_CUDA_TRY(gs_launch_filter3d(pos, n, views, n_cams, variance, filter3d, min_rate, st, lenses));
  gs_count_launch(2);
  return 0;
}

extern "C" int gs_ctx_set_densify_stats(gs_ctx* c, const gs_densify_stats* s) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_densify_stats: null ctx");
  if (!s) {
    c->stats_on = false;
    c->stats = gs_densify_stats{};
    return 0;
  }
  if (s->n < 0 || (s->n > 0 && (!s->grad2d || !s->count || !s->max_radius)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG,
                            "gs_ctx_set_densify_stats: n must be >= 0 and grad2d, count, max_radius non-NULL");
  c->stats = *s;
  c->stats_on = true;
  return 0;
}

extern "C" int gs_ctx_set_allocator(gs_ctx* c, gs_alloc_fn alloc, gs_free_fn free_fn, void* user) {
  if (!c || ((alloc == nullptr) != (free_fn == nullptr)))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_allocator: null ctx, or only one of alloc / free given");
  c->allocator.alloc = alloc;        // blocks already held keep the allocator they came from (DevBuf::owner)
  c->allocator.free = free_fn;
  c->allocator.user = user;
  return 0;
}

extern "C" long long gs_frame_instances(gs_ctx* c) { return (c && c->have_forward) ? c->m : -1; }

extern "C" int gs_frame_stats(gs_ctx* c, gs_frame_info* out, gs_stream_t stream) {
  if (!c || !out) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_stats: null argument");
  if (!c->have_forward) return gs_set_error_msg(GS_ERR_NO_FORWARD, "gs_frame_stats: no forward on this ctx");
  cudaStream_t st = (cudaStream_t)stream;
  int T = c->geom.n_tiles;
  int* h = static_cast<int*>(malloc(sizeof(int) * (size_t)(3 * T + 1)));
  if (!h) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_stats: out of host memory");
  unsigned int nvis = 0;
  cudaError_t e = cudaMemcpyAsync(h, c->tile_accum.p, sizeof(int) * (size_t)(T + 1), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(h + T + 1, c->tile_neff.p, sizeof(int) * (size_t)T, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && c->have_backward)
    e = cudaMemcpyAsync(h + 2 * T + 1, c->tile_neff_b.p, sizeof(int) * (size_t)T, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&nvis, c->counters.p, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    free(h);
    return gs_set_error(e, "gs_frame_stats copy");
  }
  long long meff = 0, meff_b = 0;
  int mx = 0;
  for (int t = 0; t < T; ++t) {
    int cnt = h[t + 1] - h[t];
    if (cnt > mx) mx = cnt;
    meff += h[T + 1 + t];
    if (c->have_backward && cnt > 0) meff_b += h[2 * T + 1 + t];
  }
  free(h);
  out->n_gaussians = c->n;
  out->n_visible = (int)nvis;
  out->n_instances = c->m;
  out->n_instances_eff = meff;
  out->n_instances_eff_bwd = c->have_backward ? meff_b : -1;
  out->width_padded = c->geom.wp;
  out->height_padded = c->geom.hp;
  out->n_tiles = T;
  out->max_tile_count = mx;
  return 0;
}

extern "C" int gs_frame_sorted(gs_ctx* c, int* gauss_idx, long long capacity, int* tile_accum, gs_stream_t stream) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_sorted: null ctx");
  if (!c->have_forward) return gs_set_error_msg(GS_ERR_NO_FORWARD, "gs_frame_sorted: no forward on this ctx");
  cudaStream_t st = (cudaStream_t)stream;
  if (gauss_idx && c->m > 0) {
    long long k = capacity < c->m ? capacity : c->m;
    if (k > 0)
      GS_CUDA_TRY(cudaMemcpyAsync(gauss_idx, c->vals_out.p, sizeof(int) * (size_t)k, cudaMemcpyDeviceToDevice, st));
  }
  if (tile_accum)
    GS_CUDA_TRY(cudaMemcpyAsync(tile_accum, c->tile_accum.p, sizeof(int) * (size_t)(c->geom.n_tiles + 1),
                                cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int gs_frame_tile_consumed(gs_ctx* c, int* tile_consumed, gs_stream_t stream) {
  if (!c || !tile_consumed) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_tile_consumed: null argument");
  if (!c->have_forward) return gs_set_error_msg(GS_ERR_NO_FORWARD, "gs_frame_tile_consumed: no forward on this ctx");
  GS_CUDA_TRY(cudaMemcpyAsync(tile_consumed, c->tile_neff.p, sizeof(int) * (size_t)c->geom.n_tiles,
                              cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int gs_frame_visible(gs_ctx* c, unsigned char* visible, int n, int accumulate, gs_stream_t stream) {
  if (!c || !visible) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_visible: null argument");
  if (!c->have_forward) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_visible: no forward on this ctx");
  if (n != c->n) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_visible: n differs from the last forward's");
  if (int rc = gs_check_device(c->device, "gs_frame_visible")) return rc;
  GS_CUDA_TRY(gs_launch_frame_visible(c->count.as<uint32_t>(), n, c->n_views ? c->n_views : 1, accumulate, visible,
                                      (cudaStream_t)stream));
  if (n > 0) gs_count_launch();
  return 0;
}

extern "C" int gs_frame_scores(gs_ctx* c, const struct gs_frame_scores* s, gs_stream_t stream) {
  const char* who = "gs_frame_scores";
  if (!c || !s || !s->weight_sum || !s->weight_max) return gs_fail(GS_ERR_INVALID_ARG, who, "null argument");
  if (!c->have_forward) return gs_fail(GS_ERR_INVALID_ARG, who, "no forward on this ctx");
  if (c->surfel) return gs_fail(GS_ERR_UNSUPPORTED, who, "the last forward rendered surfels");
  if (!c->gather) return gs_fail(GS_ERR_UNSUPPORTED, who, "the last forward ran the packed path (gs_tune(\"gather\", 0))");
  if (s->n != c->n) return gs_fail(GS_ERR_INVALID_ARG, who, "n differs from the last forward's");
  if (int rc = gs_check_device(c->device, who)) return rc;
  g_cur_alloc = &c->allocator;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t M = (size_t)c->m;
  // the pass's own tags, as next_row_epoch keeps the backward's
  GS_CUDA_TRY(c->score_rows.reserve(M * sizeof(float2) + 16, st));
  const size_t before = c->score_epoch.cap;
  GS_CUDA_TRY(c->score_epoch.reserve(M * 4 + 16, st));
  if (c->score_epoch.cap != before || c->score_ep == 0xffffffffu) {
    GS_CUDA_TRY(cudaMemsetAsync(c->score_epoch.p, 0, c->score_epoch.cap, st));
    c->score_ep = 0;
  }
  ++c->score_ep;
  GsCrop crop{(c->geom.wp - c->geom.width) / 2, (c->geom.hp - c->geom.height) / 2, c->geom.width, c->geom.height};
  GS_CUDA_TRY(gs_launch_frame_scores(c->rec.as<GsRec>(), c->vals_out.as<uint32_t>(), c->offsets_g.as<uint32_t>(),
                                     c->count.as<uint32_t>(), c->tile_accum.as<int>(), c->geom,
                                     c->n_views ? c->views.as<GsView>() : nullptr, c->n, c->n_views ? c->n_views : 1,
                                     crop, c->score_rows.as<float2>(), c->score_epoch.as<uint32_t>(), c->score_ep,
                                     s->weight_sum, s->weight_max, st));
  if (c->n > 0) gs_count_launch(2);
  return 0;
}

extern "C" int gs_render_forward_backward_host(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                               const float* quat, const float* scale, int n, int d,
                                               int scale_activation, const gs_camera* cam,
                                               const float* grad_image_host, float* image_host, float* grad_pos,
                                               float* grad_rgb, float* grad_opa, float* grad_quat, float* grad_scale,
                                               gs_stream_t stream) {
  if (!c || !cam || !grad_image_host || !image_host)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_forward_backward_host: null argument");
  if (cam->width <= 0 || cam->height <= 0)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_render_forward_backward_host: bad camera");
  GsFrameGeom g;
  if (int rc = frame_geom(*cam, 1, g, "gs_render_forward_backward_host")) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  g_cur_alloc = &c->allocator;
  size_t img_bytes = (size_t)g.wp * g.hp * 3 * sizeof(float);
  DevBuf& img_dev = c->img_dev;
  DevBuf& gimg_dev = c->gimg_dev;
  GS_CUDA_TRY(img_dev.reserve(img_bytes, st));
  GS_CUDA_TRY(gimg_dev.reserve(img_bytes, st));
  GS_CUDA_TRY(cudaMemcpyAsync(gimg_dev.p, grad_image_host, img_bytes, cudaMemcpyHostToDevice, st));
  int rc = gs_render_forward(c, pos, rgb, opa, quat, scale, n, d, scale_activation, cam, img_dev.as<float>(), nullptr,
                             stream);
  if (rc) return rc;
  rc = gs_render_backward(c, pos, rgb, opa, quat, scale, img_dev.as<float>(), gimg_dev.as<float>(), grad_pos, grad_rgb,
                          grad_opa, grad_quat, grad_scale, stream);
  if (rc) return rc;
  GS_CUDA_TRY(cudaMemcpyAsync(image_host, img_dev.p, img_bytes, cudaMemcpyDeviceToHost, st));
  GS_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int gs_ctx_set_timing(gs_ctx* c, int enable) {
  if (!c) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_ctx_set_timing: null ctx");
  if (enable && !c->ev_ok) {
    for (cudaEvent_t& e : c->ev) GS_CUDA_TRY(cudaEventCreate(&e));
    c->ev_ok = true;
  }
  c->timing = enable != 0;
  c->ev_fwd_valid = c->ev_bwd_valid = false;
  return 0;
}

extern "C" int gs_frame_stage_ms(gs_ctx* c, float* out, gs_stream_t stream) {
  if (!c || !out) return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_frame_stage_ms: null argument");
  for (int i = 0; i < GS_N_STAGES; ++i) out[i] = -1.f;
  if (!c->ev_ok) return 0;
  GS_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  if (c->ev_fwd_valid)
    for (int i = 0; i < 6; ++i) GS_CUDA_TRY(cudaEventElapsedTime(&out[i], c->ev[i], c->ev[i + 1]));
  if (c->ev_bwd_valid)
    for (int i = 6; i < 8; ++i) GS_CUDA_TRY(cudaEventElapsedTime(&out[i], c->ev[i + 1], c->ev[i + 2]));
  return 0;
}

// ---- 2D Gaussian surfels ----------------------------------------------------------------
// Stage 1 is the surfel projection (surfel.cu), stages 2-5 the 3DGS frame's bin_frame on the gather path, stage 6 the
// surfel blend (blend_surfel.cu); the backward is the surfel blend backward and projection backward.
extern "C" int gs_render_forward_surfel(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                        const float* quat, const float* scale, int n, int d, int scale_activation,
                                        const gs_camera* cam, float* image, float* final_img, int64_t* culling_mask,
                                        const gs_render_surfel* s, gs_stream_t stream) {
  const char* who = "gs_render_forward_surfel";
  if (!c || !cam || n < 0) return gs_fail(GS_ERR_INVALID_ARG, who, "bad arguments");
  if (d != 3 && gs_sh_basis_count(d) == 0)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "colour width must be 3 (RGB), 27 (SH deg 2) or 48 (SH deg 3)");
  if (int rc = check_camera(*cam, who)) return rc;
  if (!image || (n > 0 && (!pos || !rgb || !opa || !quat || !scale)))
    return gs_fail(GS_ERR_INVALID_ARG, who, "null tensor pointer");
  if (scale_activation != GS_SCALE_ABS && scale_activation != GS_SCALE_EXP)
    return gs_fail(GS_ERR_INVALID_ARG, who, "unknown scale activation");
  float bg[3] = {0.f, 0.f, 0.f};
  GsSurfelMaps mp{nullptr, nullptr, 0.2f, 100.f};
  if (s) {
    if (s->background)
      for (int k = 0; k < 3; ++k) {
        if (!std::isfinite(s->background[k])) return gs_fail(GS_ERR_INVALID_ARG, who, "background must be finite");
        bg[k] = s->background[k];
      }
    if (!(std::isfinite(s->dist_near) && std::isfinite(s->dist_far) && s->dist_near > 0.f && s->dist_far > s->dist_near))
      return gs_fail(GS_ERR_INVALID_ARG, who, "dist_near and dist_far must be finite with 0 < dist_near < dist_far");
    if (s->maps_final && (!s->maps || !final_img))
      return gs_fail(GS_ERR_INVALID_ARG, who, "maps_final needs maps and image_final");
    if ((reinterpret_cast<uintptr_t>(s->maps) | reinterpret_cast<uintptr_t>(s->maps_final)) % 16)
      return gs_fail(GS_ERR_INVALID_ARG, who, "maps and maps_final must be 16-byte aligned");
    mp = GsSurfelMaps{s->maps, s->maps_final, s->dist_near, s->dist_far};
  }
  if (d != 3 && c->sh_eval != GS_SH_EVAL_GAUSSIAN)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "SH colour evaluated per pixel has no surfel kernel (use GS_SH_EVAL_GAUSSIAN)");
  if (c->filter2d != GS_FILTER2D_NONE || c->filter3d)
    return gs_fail(GS_ERR_UNSUPPORTED, who, "the 2-D and 3-D filters have no surfel kernel");
  if (c->stats_on) return gs_fail(GS_ERR_UNSUPPORTED, who, "densification statistics have no surfel kernel");
  if (c->push.world) return gs_fail(GS_ERR_UNSUPPORTED, who, "a gradient push has no surfel kernel");
  if (!gs_tuning().gather) return gs_fail(GS_ERR_UNSUPPORTED, who, "the packed path (gs_tune(\"gather\", 0)) has no surfel kernel");
  GsLens lens{};
  bool lens_on;
  if (int rc = resolve_lenses(c, cam, 1, &lens, lens_on, who)) return rc;
  if (lens_on) return gs_fail(GS_ERR_UNSUPPORTED, who, "lenses have no surfel kernel (image-centre pinhole only)");
  if (int rc = begin_forward(c, who)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  GsFrameGeom g;
  if (int rc = frame_geom(*cam, 1, g, who)) return rc;
  const GsView vw = view_constants(c, cam, g);
  const size_t N = (size_t)n, P = (size_t)g.wp * g.hp;
  if (int rc = reserve_frame(c, N, g.n_tiles, st)) return rc;
  GS_CUDA_TRY(c->srec.reserve(N * sizeof(GsSurfelRec) + 64, st));
  GS_CUDA_TRY(c->sws.reserve(P * sizeof(float4), st));
  if (mp.maps) GS_CUDA_TRY(c->swsm.reserve(2 * P * sizeof(float4), st));
  const int kg = d == 3 ? 0 : gs_sh_basis_count(d);

  gs_mark(c, 0, st);
  GS_CUDA_TRY(cudaMemsetAsync(c->counters.p, 0, 64, st));
  GS_CUDA_TRY(cudaMemsetAsync(c->count.as<uint32_t>() + N, 0, 4, st));
  GS_CUDA_TRY(gs_launch_surfel_project(pos, rgb, opa, quat, scale, n, kg, scale_activation, vw.cam, vw.grid,
                                       cam->near_plane, vw.half_w, vw.half_h, cam->focal_x, cam->focal_y,
                                       c->srec.as<GsSurfelRec>(), c->rect.as<uint2>(), c->count.as<uint32_t>(),
                                       c->dkey_in.as<uint32_t>(), culling_mask, c->counters.as<unsigned int>(), st));
  if (n > 0) gs_count_launch();
  long long m = 0;
  if (int rc = bin_frame(c, n, g, true, 3, 3, rgb, st, m)) return rc;
  GsCrop crop{(g.wp - g.width) / 2, (g.hp - g.height) / 2, g.width, g.height};
  gs_mark(c, 5, st);
  GS_CUDA_TRY(gs_launch_blend_surfel_fwd(c->srec.as<GsSurfelRec>(), c->vals_out.as<uint32_t>(), c->tile_accum.as<int>(),
                                         g, bg, image, final_img, crop, mp.maps ? &mp : nullptr, cam->near_plane,
                                         c->sws.as<float4>(),
                                         mp.maps ? c->swsm.as<float4>() : nullptr, c->tile_neff.as<int>(), st));
  gs_count_launch();
  gs_mark(c, 6, st);
  commit_forward(c, n, d, scale_activation, m, g, vw, cam->near_plane, 0, kg > 0, true, false, GsAuxOut{}, nullptr,
                 nullptr, false, lens);
  c->surfel = true;
  c->surfel_maps = mp.maps != nullptr;
  c->surfel_kg = kg;
  memcpy(c->surfel_bg, bg, sizeof(bg));
  c->dist_near = mp.dist_near;
  c->dist_far = mp.dist_far;
  return 0;
}

extern "C" int gs_render_backward_surfel(gs_ctx* c, const float* pos, const float* rgb, const float* opa,
                                         const float* quat, const float* scale, const float* image,
                                         const float* grad_image, int grad_is_final, const float* grad_maps,
                                         float* grad_pos, float* grad_rgb, float* grad_opa, float* grad_quat,
                                         float* grad_scale, gs_stream_t stream) {
  const char* who = "gs_render_backward_surfel";
  if (!c) return gs_fail(GS_ERR_INVALID_ARG, who, "null ctx");
  if (!c->have_forward) return gs_fail(GS_ERR_NO_FORWARD, who, "no forward on this ctx");
  if (!c->surfel) return gs_fail(GS_ERR_INVALID_ARG, who, "the last forward did not render surfels");
  if (!image || !grad_image || !grad_pos || !grad_rgb || !grad_opa || !grad_quat || !grad_scale ||
      (c->n > 0 && (!pos || !rgb || !opa || !quat || !scale)))
    return gs_fail(GS_ERR_INVALID_ARG, who, "null tensor pointer");
  if (grad_maps && !c->surfel_maps) return gs_fail(GS_ERR_INVALID_ARG, who, "grad_maps given but the forward wrote no maps");
  if (reinterpret_cast<uintptr_t>(grad_maps) % 16) return gs_fail(GS_ERR_INVALID_ARG, who, "grad_maps must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(grad_quat) % 16) return gs_fail(GS_ERR_INVALID_ARG, who, "grad_quat must be 16-byte aligned");
  if (c->push.world) return gs_fail(GS_ERR_UNSUPPORTED, who, "a gradient push has no surfel kernel");
  if (c->stats_on) return gs_fail(GS_ERR_UNSUPPORTED, who, "densification statistics have no surfel kernel");
  if (int rc = gs_check_device(c->device, who)) return rc;
  g_cur_alloc = &c->allocator;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t M = (size_t)c->m;
  GS_CUDA_TRY(c->grad_inst.reserve(M * GS_SURFEL_GREC * 4 + 16, st));
  if (int rc = next_row_epoch(c, M, st)) return rc;
  c->ev_bwd_valid = false;
  GsCrop crop{(c->geom.wp - c->geom.width) / 2, (c->geom.hp - c->geom.height) / 2, c->geom.width, c->geom.height};
  gs_mark(c, 7, st);
  if (c->m > 0) {
    GS_CUDA_TRY(gs_launch_blend_surfel_bwd(c->srec.as<GsSurfelRec>(), c->vals_out.as<uint32_t>(), c->rect.as<uint2>(),
                                           c->offsets_g.as<uint32_t>(), c->tile_accum.as<int>(), c->geom, c->surfel_bg,
                                           image, grad_image, grad_is_final, crop, grad_maps, c->dist_near,
                                           c->dist_far, c->near_plane, c->sws.as<float4>(),
                                           c->surfel_maps ? c->swsm.as<float4>() : nullptr, c->grad_inst.as<float>(),
                                           c->row_epoch.as<uint32_t>(), c->epoch, c->tile_neff_b.as<int>(), st));
    gs_count_launch();
    c->have_backward = true;
  }
  gs_mark(c, 8, st);
  GS_CUDA_TRY(gs_launch_surfel_project_bwd(pos, rgb, opa, quat, scale, c->n, c->surfel_kg, c->scale_act, c->cam,
                                           c->offsets_g.as<uint32_t>(), c->count.as<uint32_t>(),
                                           c->grad_inst.as<float>(), c->row_epoch.as<uint32_t>(), c->epoch, grad_pos,
                                           grad_rgb, grad_opa, grad_quat, grad_scale, st));
  if (c->n > 0) gs_count_launch();
  gs_mark(c, 9, st);
  c->ev_bwd_valid = c->timing && c->ev_ok;
  return 0;
}
