// torch / pybind11 shim: the Python module `gaussian` with the exact symbol surface of the
// reference's extension (reference src/bindings.cpp:21-50: 12 functions + classes Tiles and
// Gaussian3ds), so the reference's renderer.py / splatter.py import and run unchanged.
// This is the ONLY libtorch-dependent translation unit; every function validates its tensors
// (the reference does not — SURVEY.md §8b) and forwards raw pointers + the CURRENT CUDA stream
// to the C ABI of libgs_b200.so (include/gs_b200.h).  Additive: class `RenderContext`
// (fused frame path) used by our splatter.py.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDACachingAllocator.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <string>
#include <array>
#include <vector>

#include "../../include/gs_b200.h"

namespace gsb200 {

#define GS_CHECK_F32(x)                                                                         \
  TORCH_CHECK((x).is_cuda(), #x " must be a CUDA tensor");                                      \
  TORCH_CHECK((x).is_contiguous(), #x " must be contiguous");                                   \
  TORCH_CHECK((x).scalar_type() == at::kFloat, #x " must be float32")
#define GS_CHECK_I32(x)                                                                         \
  TORCH_CHECK((x).is_cuda(), #x " must be a CUDA tensor");                                      \
  TORCH_CHECK((x).is_contiguous(), #x " must be contiguous");                                   \
  TORCH_CHECK((x).scalar_type() == at::kInt, #x " must be int32")
#define GS_CHECK_I64(x)                                                                         \
  TORCH_CHECK((x).is_cuda(), #x " must be a CUDA tensor");                                      \
  TORCH_CHECK((x).is_contiguous(), #x " must be contiguous");                                   \
  TORCH_CHECK((x).scalar_type() == at::kLong, #x " must be int64")

static inline void check_rc(int rc, const char* fn) {
  TORCH_CHECK(rc == 0, fn, " failed (", rc, "): ", gs_last_error());
}
static inline gs_stream_t cur_stream() { return (gs_stream_t)at::cuda::getCurrentCUDAStream().stream(); }
static inline const float* fp(const torch::Tensor& t) { return t.data_ptr<float>(); }
static inline float* fpm(const torch::Tensor& t) { return t.data_ptr<float>(); }

// Same attribute names as reference common.hpp:36-74; distinct C++ types so both modules can
// live in one interpreter during parity tests.
struct TilesPy {
  torch::Tensor top, bottom, left, right;
};
struct Gaussian3dsPy {
  torch::Tensor pos, rgb, opa, quat, scale, cov;
};

void culling(torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor) {
  // reference gaussian.cu:6-8 is a stub that prints a string; nothing calls it.
}

void world2camera(torch::Tensor pos, torch::Tensor rot, torch::Tensor trans, torch::Tensor res) {
  GS_CHECK_F32(pos); GS_CHECK_F32(rot); GS_CHECK_F32(trans); GS_CHECK_F32(res);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && res.sizes() == pos.sizes() && rot.numel() == 9 && trans.numel() == 3,
              "world2camera: bad shapes");
  c10::cuda::CUDAGuard guard(pos.device());
  check_rc(gs_w2c_fwd(fp(pos), fp(rot), fp(trans), (int)pos.size(0), fpm(res), cur_stream()), "world2camera");
}

void world2camera_backward(torch::Tensor grad_out, torch::Tensor rot, torch::Tensor grad_inp) {
  GS_CHECK_F32(grad_out); GS_CHECK_F32(rot); GS_CHECK_F32(grad_inp);
  TORCH_CHECK(grad_out.dim() == 2 && grad_out.size(1) == 3 && grad_inp.sizes() == grad_out.sizes() && rot.numel() == 9,
              "world2camera_backward: bad shapes");
  c10::cuda::CUDAGuard guard(grad_out.device());
  check_rc(gs_w2c_bwd(fp(grad_out), fp(rot), (int)grad_out.size(0), fpm(grad_inp), cur_stream()),
           "world2camera_backward");
}

void jacobian(torch::Tensor pos_camera_space, torch::Tensor jac) {
  GS_CHECK_F32(pos_camera_space); GS_CHECK_F32(jac);
  TORCH_CHECK(pos_camera_space.dim() == 2 && pos_camera_space.size(1) == 3 &&
                  jac.numel() == pos_camera_space.size(0) * 9, "jacobian: bad shapes");
  c10::cuda::CUDAGuard guard(jac.device());
  check_rc(gs_jacobian(fp(pos_camera_space), (int)pos_camera_space.size(0), fpm(jac), cur_stream()), "jacobian");
}

void calc_tile_list(Gaussian3dsPy& g, TilesPy& tiles, torch::Tensor tile_n_point, torch::Tensor tile_gaussian_list,
                    float thresh, int method, float tile_length_x, float tile_length_y, int n_tiles_x, int n_tiles_y,
                    float leftmost, float topmost) {
  GS_CHECK_F32(g.pos); GS_CHECK_I32(tile_n_point); GS_CHECK_I32(tile_gaussian_list);
  TORCH_CHECK(g.pos.dim() == 2 && g.pos.size(1) == 3, "calc_tile_list: pos must be [n,3]");
  TORCH_CHECK(tile_gaussian_list.dim() == 2 && tile_gaussian_list.size(0) == tile_n_point.size(0),
              "calc_tile_list: tile_gaussian_list must be [n_tiles, max_points]");
  TORCH_CHECK(method >= 0 && method <= 2, "calc_tile_list: method must be 0, 1 or 2");
  int n = (int)g.pos.size(0);
  int n_tiles = (int)tile_n_point.size(0);
  const float *top = nullptr, *bottom = nullptr, *left = nullptr, *right = nullptr, *cov = nullptr;
  if (method != 0) {
    GS_CHECK_F32(g.cov);
    TORCH_CHECK(g.cov.numel() == (int64_t)n * 4, "calc_tile_list: cov must be [n,2,2]");
    cov = fp(g.cov);
  }
  if (method != 2) {
    GS_CHECK_F32(tiles.top); GS_CHECK_F32(tiles.bottom); GS_CHECK_F32(tiles.left); GS_CHECK_F32(tiles.right);
    TORCH_CHECK(tiles.top.numel() == n_tiles && tiles.bottom.numel() == n_tiles && tiles.left.numel() == n_tiles &&
                    tiles.right.numel() == n_tiles, "calc_tile_list: tile bounds must have n_tiles entries");
    top = fp(tiles.top); bottom = fp(tiles.bottom); left = fp(tiles.left); right = fp(tiles.right);
  } else {
    TORCH_CHECK((int64_t)n_tiles_x * n_tiles_y == n_tiles, "calc_tile_list: n_tiles_x*n_tiles_y != len(tile_n_point)");
  }
  c10::cuda::CUDAGuard guard(g.pos.device());
  check_rc(gs_tile_list(fp(g.pos), cov, n, top, bottom, left, right, n_tiles, tile_n_point.data_ptr<int>(),
                        tile_gaussian_list.data_ptr<int>(), (int)tile_gaussian_list.size(1), thresh, method,
                        tile_length_x, tile_length_y, n_tiles_x, n_tiles_y, leftmost, topmost, cur_stream()),
           "calc_tile_list");
}

void gather_gaussians(torch::Tensor tile_n_point_accum, torch::Tensor tile_gaussian_list, torch::Tensor gathered_list,
                      torch::Tensor tile_ids_for_points, int max_points_for_tile) {
  GS_CHECK_I32(tile_n_point_accum); GS_CHECK_I32(tile_gaussian_list); GS_CHECK_I32(gathered_list);
  GS_CHECK_I32(tile_ids_for_points);
  TORCH_CHECK(tile_gaussian_list.dim() == 2 && tile_n_point_accum.numel() == tile_gaussian_list.size(0) + 1,
              "gather_gaussians: bad shapes");
  TORCH_CHECK(gathered_list.numel() == tile_ids_for_points.numel(), "gather_gaussians: output sizes differ");
  c10::cuda::CUDAGuard guard(gathered_list.device());
  check_rc(gs_gather(tile_n_point_accum.data_ptr<int>(), tile_gaussian_list.data_ptr<int>(),
                     (int)tile_gaussian_list.size(0), (int)tile_gaussian_list.size(1), max_points_for_tile,
                     gathered_list.data_ptr<int>(), tile_ids_for_points.data_ptr<int>(), cur_stream()),
           "gather_gaussians");
}

static void check_draw_inputs(const torch::Tensor& pos, const torch::Tensor& rgb, const torch::Tensor& opa,
                              const torch::Tensor& cov, const torch::Tensor& accum, const torch::Tensor& img,
                              bool use_sh_coeff) {
  GS_CHECK_F32(pos); GS_CHECK_F32(rgb); GS_CHECK_F32(opa); GS_CHECK_F32(cov); GS_CHECK_I32(accum); GS_CHECK_F32(img);
  int64_t m = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3, "draw: pos must be [m,3]");
  if (use_sh_coeff) {   // 27 = degree 2 (the reference's layout [c*9+k]); 48 = degree 3 extension [c*16+k]
    TORCH_CHECK(rgb.dim() == 2 && rgb.size(0) == m && (rgb.size(1) == 27 || rgb.size(1) == 48),
                "draw: SH rgb must be [m,27] or [m,48]");
  } else {
    TORCH_CHECK(rgb.numel() == m * 3, "draw: rgb must be [m,3]");
  }
  TORCH_CHECK(opa.numel() == m && cov.numel() == m * 4, "draw: opa must be [m], cov [m,2,2]");
  TORCH_CHECK(img.dim() == 3 && img.size(2) == 3 && img.size(0) % 16 == 0 && img.size(1) % 16 == 0,
              "draw: image must be [Hp,Wp,3] with Hp,Wp multiples of 16");
  TORCH_CHECK(accum.numel() == (img.size(0) / 16) * (img.size(1) / 16) + 1, "draw: tile_n_point_accum must be [T+1]");
}

void draw(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor cov, torch::Tensor tile_n_point_accum,
          torch::Tensor res, float focal_x, float focal_y, bool weight_normalize, bool sigmoid, bool fast,
          torch::Tensor rays_o, torch::Tensor lefttop_pos, torch::Tensor vec_dx, torch::Tensor vec_dy,
          bool use_sh_coeff) {
  (void)fast;   // both exp flavours of the reference are within 2 ulp of ex2.approx; one code path
  check_draw_inputs(pos, rgb, opa, cov, tile_n_point_accum, res, use_sh_coeff);
  c10::cuda::CUDAGuard guard(pos.device());
  int m = (int)pos.size(0), d = use_sh_coeff ? (int)rgb.size(1) : 3;
  auto ws = torch::empty({(int64_t)gs_draw_workspace_bytes(m, d)}, pos.options().dtype(at::kByte));
  const float *ro = nullptr, *lt = nullptr, *dx = nullptr, *dy = nullptr;
  if (use_sh_coeff) {
    GS_CHECK_F32(rays_o); GS_CHECK_F32(lefttop_pos); GS_CHECK_F32(vec_dx); GS_CHECK_F32(vec_dy);
    ro = fp(rays_o); lt = fp(lefttop_pos); dx = fp(vec_dx); dy = fp(vec_dy);
  }
  check_rc(gs_draw_fwd(fp(pos), fp(rgb), fp(opa), fp(cov), tile_n_point_accum.data_ptr<int>(), m, d, (int)res.size(1),
                       (int)res.size(0), focal_x, focal_y, weight_normalize, sigmoid, ro, lt, dx, dy, fpm(res),
                       ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
           "draw");
}

void draw_backward(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor cov,
                   torch::Tensor tile_n_point_accum, torch::Tensor output, torch::Tensor grad_output,
                   torch::Tensor grad_pos, torch::Tensor grad_rgb, torch::Tensor grad_opa, torch::Tensor grad_cov,
                   float focal_x, float focal_y, bool weight_normalize, bool sigmoid, bool fast, torch::Tensor rays_o,
                   torch::Tensor lefttop_pos, torch::Tensor vec_dx, torch::Tensor vec_dy, bool use_sh_coeff) {
  (void)fast;
  check_draw_inputs(pos, rgb, opa, cov, tile_n_point_accum, output, use_sh_coeff);
  GS_CHECK_F32(grad_pos); GS_CHECK_F32(grad_rgb); GS_CHECK_F32(grad_opa); GS_CHECK_F32(grad_cov);
  TORCH_CHECK(grad_output.is_cuda() && grad_output.scalar_type() == at::kFloat, "grad_output must be a float32 CUDA tensor");
  TORCH_CHECK(grad_output.sizes() == output.sizes(), "draw_backward: grad_output shape != output shape");
  TORCH_CHECK(grad_pos.sizes() == pos.sizes() && grad_rgb.numel() == rgb.numel() && grad_opa.numel() == opa.numel() &&
                  grad_cov.numel() == cov.numel(), "draw_backward: gradient buffers must match their inputs");
  c10::cuda::CUDAGuard guard(pos.device());
  auto go = grad_output.contiguous();   // autograd may hand us a strided view (crop backward)
  int m = (int)pos.size(0), d = use_sh_coeff ? (int)rgb.size(1) : 3;
  auto ws = torch::empty({(int64_t)gs_draw_workspace_bytes(m, d)}, pos.options().dtype(at::kByte));
  const float *ro = nullptr, *lt = nullptr, *dx = nullptr, *dy = nullptr;
  if (use_sh_coeff) {
    GS_CHECK_F32(rays_o); GS_CHECK_F32(lefttop_pos); GS_CHECK_F32(vec_dx); GS_CHECK_F32(vec_dy);
    ro = fp(rays_o); lt = fp(lefttop_pos); dx = fp(vec_dx); dy = fp(vec_dy);
  }
  check_rc(gs_draw_bwd(fp(pos), fp(rgb), fp(opa), fp(cov), tile_n_point_accum.data_ptr<int>(), m, d,
                       (int)output.size(1), (int)output.size(0), focal_x, focal_y, weight_normalize, sigmoid, ro, lt,
                       dx, dy, fp(output), fp(go), fpm(grad_pos), fpm(grad_rgb), fpm(grad_opa), fpm(grad_cov),
                       ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
           "draw_backward");
}

void global_culling(torch::Tensor pos, torch::Tensor quat, torch::Tensor scale, torch::Tensor current_rot,
                    torch::Tensor current_tran, torch::Tensor res_pos, torch::Tensor res_cov,
                    torch::Tensor culling_mask, float near, float half_width, float half_height) {
  GS_CHECK_F32(pos); GS_CHECK_F32(quat); GS_CHECK_F32(scale); GS_CHECK_F32(current_rot); GS_CHECK_F32(current_tran);
  GS_CHECK_F32(res_pos); GS_CHECK_F32(res_cov); GS_CHECK_I64(culling_mask);
  int64_t n = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && quat.numel() == n * 4 && scale.numel() == n * 3 &&
                  current_rot.numel() == 9 && current_tran.numel() == 3 && res_pos.numel() == n * 3 &&
                  res_cov.numel() == n * 4 && culling_mask.numel() == n, "global_culling: bad shapes");
  c10::cuda::CUDAGuard guard(pos.device());
  check_rc(gs_project_fwd(fp(pos), fp(quat), fp(scale), fp(current_rot), fp(current_tran), (int)n, near, half_width,
                          half_height, fpm(res_pos), fpm(res_cov), culling_mask.data_ptr<int64_t>(), cur_stream()),
           "global_culling");
}

void global_culling_backward(torch::Tensor pos, torch::Tensor quat, torch::Tensor scale, torch::Tensor current_rot,
                             torch::Tensor current_tran, torch::Tensor gradout_pos, torch::Tensor gradout_cov,
                             torch::Tensor culling_mask, torch::Tensor gradinput_pos, torch::Tensor gradinput_quat,
                             torch::Tensor gradinput_scale) {
  GS_CHECK_F32(pos); GS_CHECK_F32(quat); GS_CHECK_F32(scale); GS_CHECK_F32(current_rot); GS_CHECK_F32(current_tran);
  GS_CHECK_I64(culling_mask); GS_CHECK_F32(gradinput_pos); GS_CHECK_F32(gradinput_quat); GS_CHECK_F32(gradinput_scale);
  int64_t n = pos.size(0);
  TORCH_CHECK(gradout_pos.is_cuda() && gradout_cov.is_cuda() && gradout_pos.scalar_type() == at::kFloat &&
                  gradout_cov.scalar_type() == at::kFloat, "global_culling_backward: gradients must be float32 CUDA");
  TORCH_CHECK(gradout_pos.numel() == n * 3 && gradout_cov.numel() == n * 4 && culling_mask.numel() == n &&
                  gradinput_pos.numel() == n * 3 && gradinput_quat.numel() == n * 4 && gradinput_scale.numel() == n * 3,
              "global_culling_backward: bad shapes");
  c10::cuda::CUDAGuard guard(pos.device());
  auto gp = gradout_pos.contiguous();
  auto gc = gradout_cov.contiguous();
  check_rc(gs_project_bwd(fp(pos), fp(quat), fp(scale), fp(current_rot), fp(current_tran), fp(gp), fp(gc),
                          culling_mask.data_ptr<int64_t>(), (int)n, fpm(gradinput_pos), fpm(gradinput_quat),
                          fpm(gradinput_scale), cur_stream()),
           "global_culling_backward");
}

// ---- additive: fused frame path ----------------------------------------------------------
struct RenderContext {
  gs_ctx* ctx = nullptr;
  int device = -1;
  // The context holds the intermediate state of ONE forward.  Every forward gets an id; a
  // backward that names another id is refused instead of silently using the wrong frame.
  int64_t frame = 0;
  int64_t frame_id() const { return frame; }
  void check_frame(int64_t expected, const char* fn) const {
    TORCH_CHECK(expected < 0 || expected == frame, fn, ": this RenderContext has rendered another frame (id ", frame,
                ") since the forward being differentiated (id ", expected,
                "); run backward before the next forward, or use one RenderContext / Splatter per in-flight frame");
  }
  static void* torch_alloc(size_t bytes, void*, gs_stream_t stream) {
    try {
      return c10::cuda::CUDACachingAllocator::raw_alloc_with_stream(bytes, (cudaStream_t)stream);
    } catch (...) {
      return nullptr;
    }
  }
  static void torch_free(void* p, void*) { c10::cuda::CUDACachingAllocator::raw_delete(p); }
  RenderContext() {
    check_rc(gs_ctx_create(&ctx), "gs_ctx_create");
    cudaGetDevice(&device);
    // workspaces from PyTorch's stream-ordered caching allocator: growth needs no device synchronisation
    check_rc(gs_ctx_set_allocator(ctx, &torch_alloc, &torch_free, nullptr), "gs_ctx_set_allocator");
  }
  ~RenderContext() { gs_ctx_destroy(ctx); }
  RenderContext(const RenderContext&) = delete;
  RenderContext& operator=(const RenderContext&) = delete;

  static gs_camera make_cam(int width, int height, float fx, float fy, const torch::Tensor& rot,
                            const torch::Tensor& tran, float near, float thresh) {
    TORCH_CHECK(!rot.is_cuda() && !tran.is_cuda(), "RenderContext: rot/tran must be CPU tensors (camera is host data)");
    auto r = rot.to(at::kFloat).contiguous();
    auto t = tran.to(at::kFloat).contiguous();
    TORCH_CHECK(r.numel() == 9 && t.numel() == 3, "RenderContext: rot must be 3x3, tran 3");
    gs_camera cam{};
    cam.width = width;
    cam.height = height;
    cam.focal_x = fx;
    cam.focal_y = fy;
    memcpy(cam.rot, r.data_ptr<float>(), sizeof(cam.rot));
    memcpy(cam.tran, t.data_ptr<float>(), sizeof(cam.tran));
    cam.near_plane = near;
    cam.tile_thresh = thresh;
    return cam;
  }

  // data-parallel gradient push (gs_grad_push): pointers as integers (symmetric-memory mappings)
  void set_grad_push(int64_t bucket_ptr, std::vector<int64_t> staging_ptrs, int64_t per, int rank) {
    gs_grad_push p{};
    p.world = (int)staging_ptrs.size();
    TORCH_CHECK(p.world <= GS_MAX_PEERS, "set_grad_push: at most ", GS_MAX_PEERS, " ranks");
    p.rank = rank;
    p.per = per;
    p.bucket = reinterpret_cast<float*>(static_cast<uintptr_t>(bucket_ptr));
    for (int k = 0; k < p.world; ++k) p.staging[k] = reinterpret_cast<float*>(static_cast<uintptr_t>(staging_ptrs[k]));
    check_rc(gs_ctx_set_grad_push(ctx, &p), "gs_ctx_set_grad_push");
  }
  void clear_grad_push() { check_rc(gs_ctx_set_grad_push(ctx, nullptr), "gs_ctx_set_grad_push"); }

  // where SH colour is evaluated (gs_ctx_set_sh_eval): SH_EVAL_PIXEL (default) or SH_EVAL_GAUSSIAN; applies to the
  // forwards that follow, a backward uses the mode of its forward
  void set_sh_eval(int mode) { check_rc(gs_ctx_set_sh_eval(ctx, mode), "gs_ctx_set_sh_eval"); }

  // screen-space 2-D filter (gs_ctx_set_filter2d): FILTER2D_NONE (default), _DILATE or _ANTIALIAS with a variance in
  // px^2; applies to the forwards that follow, a backward uses the filter of its forward
  void set_filter2d(int mode, double variance) {
    check_rc(gs_ctx_set_filter2d(ctx, mode, (float)variance), "gs_ctx_set_filter2d");
  }

  // 3-D smoothing filter (gs_ctx_set_filter3d): a contiguous float32 CUDA tensor [n] on this context's device, or None
  // (off); applies to the forwards that follow, a backward uses the filter of its forward.  The context keeps the
  // tensor alive while it is set.
  torch::Tensor filter3d_ref;
  void set_filter3d(std::optional<torch::Tensor> f) {
    if (!f) {
      check_rc(gs_ctx_set_filter3d(ctx, nullptr, 0), "gs_ctx_set_filter3d");
      filter3d_ref = torch::Tensor();
      return;
    }
    TORCH_CHECK(f->is_cuda() && f->scalar_type() == at::kFloat && f->is_contiguous() && f->dim() == 1,
                "set_filter3d: filter3d must be a contiguous 1-D float32 CUDA tensor");
    TORCH_CHECK(f->device().index() == device, "set_filter3d: filter3d is on another device than the context");
    TORCH_CHECK(f->numel() < (int64_t(1) << 31), "set_filter3d: n too large");
    check_rc(gs_ctx_set_filter3d(ctx, fp(*f), (int)f->numel()), "gs_ctx_set_filter3d");
    filter3d_ref = *f;
  }

  // camera lenses (gs_ctx_set_lens): models a sequence of n GS_LENS_* codes and params a CPU float32 tensor [n, 6] =
  // (cx, cy, k0, k1, k2, k3) per lens, or None (off); applies to the forwards that follow, a backward uses the lenses
  // of its forward
  void set_lens(std::optional<std::vector<int>> models, std::optional<torch::Tensor> params) {
    if (!models || !params) {
      TORCH_CHECK(!models && !params, "set_lens: give both models and params, or neither");
      check_rc(gs_ctx_set_lens(ctx, nullptr, 0), "gs_ctx_set_lens");
      return;
    }
    const int64_t n = (int64_t)models->size();
    TORCH_CHECK(!params->is_cuda() && params->scalar_type() == at::kFloat && params->dim() == 2 &&
                    params->size(0) == n && params->size(1) == 6,
                "set_lens: params must be a CPU float32 tensor [n, 6] with n = len(models)");
    TORCH_CHECK(n <= GS_MAX_VIEWS, "set_lens: more than GS_MAX_VIEWS lenses");
    const torch::Tensor pc = params->contiguous();
    const float* pp = pc.data_ptr<float>();
    std::vector<gs_lens> lenses((size_t)n);
    for (int64_t v = 0; v < n; ++v) {
      lenses[v].model = (*models)[v];
      lenses[v].cx = pp[6 * v];
      lenses[v].cy = pp[6 * v + 1];
      for (int k = 0; k < 4; ++k) lenses[v].k[k] = pp[6 * v + 2 + k];
    }
    check_rc(gs_ctx_set_lens(ctx, lenses.data(), (int)n), "gs_ctx_set_lens");
  }

  // gs_filter3d_compute over V views: size [V,2] = (width, height), focal [V,2] = (fx, fy), rot [V,3,3], tran [V,3]
  // (CPU tensors), one near plane; writes and returns out [n] (allocated when None)
  torch::Tensor filter3d_compute(torch::Tensor pos, torch::Tensor size, torch::Tensor focal, torch::Tensor rot,
                                 torch::Tensor tran, double near, double margin, double variance,
                                 std::optional<torch::Tensor> out) {
    const char* fn = "filter3d_compute";
    GS_CHECK_F32(pos);
    TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && pos.size(0) < (int64_t(1) << 31), fn, ": pos must be [n,3]");
    TORCH_CHECK(pos.device().index() == device, fn, ": pos is on another device than the context");
    TORCH_CHECK(!size.is_cuda() && !focal.is_cuda() && !rot.is_cuda() && !tran.is_cuda(), fn,
                ": size / focal / rot / tran must be CPU tensors (cameras are host data)");
    const int64_t v = size.dim() == 2 ? size.size(0) : -1;
    TORCH_CHECK(v >= 1 && v < (int64_t(1) << 31) && size.size(1) == 2 && focal.dim() == 2 && focal.size(0) == v &&
                    focal.size(1) == 2 && rot.dim() == 3 && rot.size(0) == v && rot.size(1) == 3 && rot.size(2) == 3 &&
                    tran.dim() == 2 && tran.size(0) == v && tran.size(1) == 3,
                fn, ": size and focal must be [V,2], rot [V,3,3] and tran [V,3] with V >= 1");
    const int64_t n = pos.size(0);
    torch::Tensor f;
    if (out) {
      f = *out;
      TORCH_CHECK(f.is_cuda() && f.scalar_type() == at::kFloat && f.is_contiguous() && f.dim() == 1 && f.numel() == n &&
                      f.device() == pos.device(),
                  fn, ": out must be a contiguous float32 CUDA tensor [n] on pos's device");
    } else {
      f = torch::empty({n}, pos.options());
    }
    auto sz = size.to(at::kLong).contiguous();
    auto fc = focal.to(at::kFloat).contiguous();
    auto r = rot.to(at::kFloat).contiguous();
    auto t = tran.to(at::kFloat).contiguous();
    auto sa = sz.accessor<int64_t, 2>();
    auto fa = fc.accessor<float, 2>();
    std::vector<gs_camera> cams((size_t)v);
    for (int64_t k = 0; k < v; ++k) {
      gs_camera& cm = cams[(size_t)k];
      cm = gs_camera{};
      TORCH_CHECK(sa[k][0] > 0 && sa[k][0] < (int64_t(1) << 31) && sa[k][1] > 0 && sa[k][1] < (int64_t(1) << 31), fn,
                  ": bad view size");
      cm.width = (int)sa[k][0];
      cm.height = (int)sa[k][1];
      cm.focal_x = fa[k][0];
      cm.focal_y = fa[k][1];
      memcpy(cm.rot, r[k].data_ptr<float>(), sizeof(cm.rot));
      memcpy(cm.tran, t[k].data_ptr<float>(), sizeof(cm.tran));
      cm.near_plane = (float)near;
      cm.tile_thresh = 0.05f;
    }
    c10::cuda::CUDAGuard guard(pos.device());
    check_rc(gs_filter3d_compute(ctx, fp(pos), (int)n, cams.data(), (int)v, (float)margin, (float)variance, fpm(f),
                                 cur_stream()),
             "gs_filter3d_compute");
    return f;
  }

  // screen-space densification statistics (gs_ctx_set_densify_stats): accumulated by every backward that computes
  // parameter gradients until cleared.  The context keeps the tensors alive while they are set.
  std::vector<torch::Tensor> densify_stats_refs;
  void set_densify_stats(torch::Tensor grad2d, torch::Tensor count, torch::Tensor max_radius,
                         c10::optional<torch::Tensor> absgrad) {
    const int64_t n = grad2d.numel();
    auto check = [&](const torch::Tensor& t, at::ScalarType dt, const char* name) {
      TORCH_CHECK(t.is_cuda() && t.scalar_type() == dt && t.is_contiguous() && t.dim() == 1 && t.numel() == n,
                  "set_densify_stats: ", name, " must be a contiguous 1-D CUDA ", dt == at::kInt ? "int32" : "float32",
                  " tensor of n = grad2d.numel() elements");
      TORCH_CHECK(t.device().index() == device, "set_densify_stats: ", name, " is on another device than the context");
    };
    check(grad2d, at::kFloat, "grad2d");
    check(count, at::kInt, "count");
    check(max_radius, at::kFloat, "max_radius");
    if (absgrad) check(*absgrad, at::kFloat, "absgrad");
    TORCH_CHECK(n < (int64_t(1) << 31), "set_densify_stats: n too large");
    gs_densify_stats s{};
    s.n = (int)n;
    s.grad2d = fpm(grad2d);
    s.absgrad = absgrad ? fpm(*absgrad) : nullptr;
    s.count = count.data_ptr<int>();
    s.max_radius = fpm(max_radius);
    check_rc(gs_ctx_set_densify_stats(ctx, &s), "gs_ctx_set_densify_stats");
    densify_stats_refs = {grad2d, count, max_radius};
    if (absgrad) densify_stats_refs.push_back(*absgrad);
  }
  void clear_densify_stats() {
    check_rc(gs_ctx_set_densify_stats(ctx, nullptr), "gs_ctx_set_densify_stats");
    densify_stats_refs.clear();
  }

  void set_timing(bool on) { check_rc(gs_ctx_set_timing(ctx, on ? 1 : 0), "gs_ctx_set_timing"); }
  std::vector<float> stage_ms() {
    std::vector<float> v(GS_N_STAGES, -1.f);
    check_rc(gs_frame_stage_ms(ctx, v.data(), cur_stream()), "gs_frame_stage_ms");
    return v;
  }

  static int64_t padded(int64_t size) { return (size + 15) / 16 * 16; }
  static float* fpm_or_null(const torch::Tensor& t) { return t.defined() ? fpm(t) : nullptr; }
  static py::object or_none(const torch::Tensor& t) { return t.defined() ? py::cast(t) : py::none(); }

  // the five parameters (and feat [n, f]) of a frame: contiguous float32 on this context's device; returns n
  int64_t check_params(const char* fn, const torch::Tensor& pos, const torch::Tensor& rgb, const torch::Tensor& opa,
                       const torch::Tensor& quat, const torch::Tensor& scale,
                       const torch::Tensor* feat_or_null = nullptr) const {
    GS_CHECK_F32(pos); GS_CHECK_F32(rgb); GS_CHECK_F32(opa); GS_CHECK_F32(quat); GS_CHECK_F32(scale);
    if (feat_or_null) {
      const torch::Tensor& feat = *feat_or_null;
      GS_CHECK_F32(feat);
    }
    const int64_t n = pos.size(0);
    TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && opa.numel() == n && quat.numel() == n * 4 &&
                    scale.numel() == n * 3 && rgb.dim() == 2 && rgb.size(0) == n && n < (int64_t(1) << 31) &&
                    (!feat_or_null || (feat_or_null->dim() == 2 && feat_or_null->size(0) == n)),
                fn, ": bad shapes");
    TORCH_CHECK(pos.device().index() == device, "RenderContext was created on another device");
    return n;
  }

  // gradient buffers for the parameters, in the same order (pos, rgb, opa, quat, scale[, feat]); the kernels store
  // quaternion gradients as float4
  static void check_grads(const char* fn, const std::vector<torch::Tensor>& params,
                          const std::vector<torch::Tensor>& grads) {
    static const char* names[] = {"g_pos", "g_rgb", "g_opa", "g_quat", "g_scale", "g_feat"};
    bool match = true;
    for (size_t k = 0; k < grads.size(); ++k) {
      const torch::Tensor& g = grads[k];
      TORCH_CHECK(g.is_cuda() && g.is_contiguous() && g.scalar_type() == at::kFloat, fn, ": ", names[k],
                  " must be a contiguous float32 CUDA tensor");
      match = match && g.numel() == params[k].numel();
    }
    TORCH_CHECK(match, fn, ": gradient buffers must match their parameters");
    TORCH_CHECK(reinterpret_cast<uintptr_t>(grads[3].data_ptr()) % 16 == 0, "grad_quat must be 16-byte aligned");
  }

  // a float32 CUDA image of shape pixels + [channels], pixels = [(B,) rows, cols]
  static void check_image(const char* fn, const char* name, const torch::Tensor& t, std::vector<int64_t> pixels,
                          int64_t channels, bool contiguous) {
    pixels.push_back(channels);
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.sizes() == at::IntArrayRef(pixels) &&
                    (!contiguous || t.is_contiguous()),
                fn, ": ", name, " must be a float32", contiguous ? " contiguous" : "", " CUDA tensor of shape ",
                at::IntArrayRef(pixels));
  }

  // The tensors of a backward of the last forward: raw [(B,) Hp, Wp, 3] with aux (2 channels) and map (feat's f
  // channels) like it; the upstream gradients grad_image (3 channels), grad_aux and grad_map over raw's pixels, or
  // (final) over the centre crop's [(B,) H, W].  Batched: B, H, W are those of the last forward_batch.
  void check_backward(const char* fn, int64_t expected_frame, bool batched, bool final, const torch::Tensor& pos,
                      const torch::Tensor& rgb, const torch::Tensor& opa, const torch::Tensor& quat,
                      const torch::Tensor& scale, const torch::Tensor& raw, const torch::Tensor& grad_image,
                      const torch::Tensor* aux, const torch::Tensor* grad_aux, const torch::Tensor* feat = nullptr,
                      const torch::Tensor* map = nullptr, const torch::Tensor* grad_map = nullptr) const {
    check_frame(expected_frame, fn);
    check_params(fn, pos, rgb, opa, quat, scale, feat);
    TORCH_CHECK(raw.dim() == (batched ? 4 : 3), fn, ": raw must be ", batched ? "[B,Hp,Wp,3]" : "[Hp,Wp,3]");
    std::vector<int64_t> pixels = batched ? std::vector<int64_t>{batch[0], padded(batch[1]), padded(batch[2])}
                                          : std::vector<int64_t>{raw.size(0), raw.size(1)};
    check_image(fn, "raw", raw, pixels, 3, true);
    if (aux) check_image(fn, "aux", *aux, pixels, 2, true);
    if (map) check_image(fn, "map", *map, pixels, feat->size(1), true);
    if (final) {
      TORCH_CHECK(grad_image.dim() == raw.dim(), fn, ": grad_image must be ", batched ? "[B,H,W,3]" : "[H,W,3]",
                  " (final) or match raw");
      pixels = batched ? std::vector<int64_t>{batch[0], batch[1], batch[2]}
                       : std::vector<int64_t>{grad_image.size(0), grad_image.size(1)};
    }
    check_image(fn, "grad_image", grad_image, pixels, 3, false);
    if (grad_aux) check_image(fn, "grad_aux", *grad_aux, pixels, 2, false);
    if (grad_map) check_image(fn, "grad_map", *grad_map, pixels, feat->size(1), false);
  }

  // backward of the last single-view (gs_render_backward_aux) or batched (gs_render_backward_batch) forward into the
  // caller's gradient buffers; aux / grad_aux NULL: the plain backward kernels
  void backward_checked(const char* fn, bool batched, const torch::Tensor& pos, const torch::Tensor& rgb,
                        const torch::Tensor& opa, const torch::Tensor& quat, const torch::Tensor& scale,
                        const torch::Tensor& raw, const torch::Tensor& grad_image, bool final,
                        const torch::Tensor* aux, const std::optional<torch::Tensor>& grad_aux,
                        const std::vector<torch::Tensor>& grads, int64_t expected_frame) {
    check_backward(fn, expected_frame, batched, final, pos, rgb, opa, quat, scale, raw, grad_image, aux,
                   grad_aux ? &*grad_aux : nullptr);
    check_grads(fn, {pos, rgb, opa, quat, scale}, grads);
    c10::cuda::CUDAGuard guard(pos.device());
    auto gi = grad_image.contiguous();
    torch::Tensor ga;
    if (grad_aux) ga = grad_aux->contiguous();
    auto entry = batched ? &gs_render_backward_batch : &gs_render_backward_aux;
    check_rc(entry(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), fp(raw), fp(gi), final ? 1 : 0,
                   aux ? fp(*aux) : nullptr, fpm_or_null(ga), fpm(grads[0]), fpm(grads[1]), fpm(grads[2]),
                   fpm(grads[3]), fpm(grads[4]), cur_stream()),
             fn);
  }

  // what a forward renders: raw / aux / map padded [(B,) Hp, Wp, .], fin / aux_fin / map_fin the centre crops
  // [(B,) H, W, .] (final), mask [(B,) n]; tensors a forward does not write stay undefined
  struct Outputs {
    torch::Tensor raw, aux, map, fin, aux_fin, map_fin, mask;
  };
  static Outputs alloc_outputs(const torch::Tensor& pos, int64_t b, int64_t n, int64_t height, int64_t width,
                               bool maps, int64_t f, bool final) {
    auto shape = [b](int64_t rows, int64_t cols, int64_t ch) {
      return b ? std::vector<int64_t>{b, rows, cols, ch} : std::vector<int64_t>{rows, cols, ch};
    };
    const int64_t hp = padded(height), wp = padded(width);
    Outputs o;
    o.raw = torch::empty(shape(hp, wp, 3), pos.options());
    if (maps) o.aux = torch::empty(shape(hp, wp, 2), pos.options());
    if (f) o.map = torch::empty(shape(hp, wp, f), pos.options());
    if (final) {
      o.fin = torch::empty(shape(height, width, 3), pos.options());
      if (maps) o.aux_fin = torch::empty(shape(height, width, 2), pos.options());
      if (f) o.map_fin = torch::empty(shape(height, width, f), pos.options());
    }
    o.mask = torch::empty(b ? std::vector<int64_t>{b, n} : std::vector<int64_t>{n}, pos.options().dtype(at::kLong));
    return o;
  }

  struct Background {
    float rgb[3] = {0.f, 0.f, 0.f};
    bool given = false;
    const float* ptr() const { return given ? rgb : nullptr; }
  };
  static Background background_of(const char* fn, const std::optional<std::vector<double>>& background) {
    TORCH_CHECK(!background || background->size() == 3, fn, ": background must have 3 values");
    Background bg;
    if (background) {
      bg.given = true;
      for (int k = 0; k < 3; ++k) bg.rgb[k] = (float)(*background)[k];
    }
    return bg;
  }

  // the C call of a forward; on success the context holds a new frame
  void rendered(int rc, const char* fn) {
    check_rc(rc, fn);
    ++frame;
  }

  // one view through gs_render_forward_aux: maps = the depth / alpha maps, final = the clamped centre crops
  Outputs render(const char* fn, const torch::Tensor& pos, const torch::Tensor& rgb, const torch::Tensor& opa,
                 const torch::Tensor& quat, const torch::Tensor& scale, int width, int height, float fx, float fy,
                 const torch::Tensor& rot, const torch::Tensor& tran, float near, float thresh, int scale_activation,
                 const std::optional<std::vector<double>>& background, bool maps, bool final) {
    const int64_t n = check_params(fn, pos, rgb, opa, quat, scale);
    const Background bg = background_of(fn, background);
    c10::cuda::CUDAGuard guard(pos.device());
    gs_camera cam = make_cam(width, height, fx, fy, rot, tran, near, thresh);
    Outputs o = alloc_outputs(pos, 0, n, height, width, maps, 0, final);
    gs_render_aux ax{bg.ptr(), fpm_or_null(o.aux), fpm_or_null(o.aux_fin)};
    rendered(gs_render_forward_aux(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), (int)n, (int)rgb.size(1),
                                   scale_activation, &cam, fpm(o.raw), fpm_or_null(o.fin),
                                   o.mask.data_ptr<int64_t>(), &ax, cur_stream()),
             fn);
    return o;
  }

  // returns (image[Hp,Wp,3], culling_mask[n] int64)
  std::tuple<torch::Tensor, torch::Tensor> forward(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa,
                                                   torch::Tensor quat, torch::Tensor scale, int width, int height,
                                                   float fx, float fy, torch::Tensor rot, torch::Tensor tran,
                                                   float near, float thresh, int scale_activation) {
    Outputs o = render("RenderContext.forward", pos, rgb, opa, quat, scale, width, height, fx, fy, rot, tran, near,
                       thresh, scale_activation, std::nullopt, false, false);
    return {o.raw, o.mask};
  }

  std::vector<torch::Tensor> backward(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                                      torch::Tensor scale, torch::Tensor image, torch::Tensor grad_image) {
    std::vector<torch::Tensor> grads = {torch::empty_like(pos), torch::empty_like(rgb), torch::empty_like(opa),
                                        torch::empty_like(quat), torch::empty_like(scale)};
    backward_checked("RenderContext.backward", false, pos, rgb, opa, quat, scale, image, grad_image, false, nullptr,
                     std::nullopt, grads, -1);
    return grads;
  }

  void backward_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat, torch::Tensor scale,
                     torch::Tensor image, torch::Tensor grad_image, torch::Tensor g_pos, torch::Tensor g_rgb,
                     torch::Tensor g_opa, torch::Tensor g_quat, torch::Tensor g_scale, int64_t expected_frame) {
    backward_checked("RenderContext.backward_into", false, pos, rgb, opa, quat, scale, image, grad_image, false,
                     nullptr, std::nullopt, {g_pos, g_rgb, g_opa, g_quat, g_scale}, expected_frame);
  }

  // fused clamp + centre crop: returns (final[H,W,3], raw padded[Hp,Wp,3], mask)
  std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> forward_final(
      torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat, torch::Tensor scale, int width,
      int height, float fx, float fy, torch::Tensor rot, torch::Tensor tran, float near, float thresh,
      int scale_activation) {
    Outputs o = render("RenderContext.forward_final", pos, rgb, opa, quat, scale, width, height, fx, fy, rot, tran,
                       near, thresh, scale_activation, std::nullopt, false, true);
    return {o.fin, o.raw, o.mask};
  }

  void backward_final_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                           torch::Tensor scale, torch::Tensor raw, torch::Tensor grad_final, torch::Tensor g_pos,
                           torch::Tensor g_rgb, torch::Tensor g_opa, torch::Tensor g_quat, torch::Tensor g_scale,
                           int64_t expected_frame) {
    backward_checked("RenderContext.backward_final_into", false, pos, rgb, opa, quat, scale, raw, grad_final, true,
                     nullptr, std::nullopt, {g_pos, g_rgb, g_opa, g_quat, g_scale}, expected_frame);
  }

  // depth / alpha maps and a background colour (gs_render_forward_aux): returns
  // (final[H,W,3] or None, raw padded[Hp,Wp,3], aux padded[Hp,Wp,2], aux_final[H,W,2] or None, mask)
  py::tuple forward_aux(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                        torch::Tensor scale, int width, int height, float fx, float fy, torch::Tensor rot,
                        torch::Tensor tran, float near, float thresh, int scale_activation,
                        std::optional<std::vector<double>> background, bool final) {
    Outputs o = render("RenderContext.forward_aux", pos, rgb, opa, quat, scale, width, height, fx, fy, rot, tran, near,
                       thresh, scale_activation, background, true, final);
    return py::make_tuple(or_none(o.fin), o.raw, o.aux, or_none(o.aux_fin), o.mask);
  }

  // backward of forward_aux; grad_aux = None: the plain backward kernels (zero depth / alpha gradient)
  void backward_aux_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                         torch::Tensor scale, torch::Tensor raw, torch::Tensor grad_image, bool grad_is_final,
                         torch::Tensor aux, std::optional<torch::Tensor> grad_aux, torch::Tensor g_pos,
                         torch::Tensor g_rgb, torch::Tensor g_opa, torch::Tensor g_quat, torch::Tensor g_scale,
                         int64_t expected_frame) {
    backward_checked("RenderContext.backward_aux_into", false, pos, rgb, opa, quat, scale, raw, grad_image,
                     grad_is_final, &aux, grad_aux, {g_pos, g_rgb, g_opa, g_quat, g_scale}, expected_frame);
  }

  // a batch of B views as one frame (gs_render_forward_batch): focal [B,2] = (fx, fy), rot [B,3,3], tran [B,3] are
  // CPU tensors; returns (final[B,H,W,3] or None, raw padded[B,Hp,Wp,3], aux padded[B,Hp,Wp,2],
  // aux_final[B,H,W,2] or None, mask[B,n])
  py::tuple forward_batch(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                          torch::Tensor scale, int width, int height, torch::Tensor focal, torch::Tensor rot,
                          torch::Tensor tran, float near, float thresh, int scale_activation,
                          std::optional<std::vector<double>> background, bool final) {
    const char* fn = "RenderContext.forward_batch";
    const int64_t n = check_params(fn, pos, rgb, opa, quat, scale);
    TORCH_CHECK(!focal.is_cuda() && !rot.is_cuda() && !tran.is_cuda(),
                "RenderContext.forward_batch: focal / rot / tran must be CPU tensors (cameras are host data)");
    const int64_t b = focal.dim() == 2 ? focal.size(0) : -1;
    TORCH_CHECK(b >= 1 && b <= GS_MAX_VIEWS && focal.size(1) == 2 && rot.dim() == 3 && rot.size(0) == b &&
                    rot.size(1) == 3 && rot.size(2) == 3 && tran.dim() == 2 && tran.size(0) == b && tran.size(1) == 3,
                "RenderContext.forward_batch: focal must be [B,2], rot [B,3,3] and tran [B,3] with 1 <= B <= ",
                GS_MAX_VIEWS);
    const Background bg = background_of(fn, background);
    c10::cuda::CUDAGuard guard(pos.device());
    auto f = focal.to(at::kFloat).contiguous();
    std::vector<gs_camera> cams;
    for (int64_t v = 0; v < b; ++v)
      cams.push_back(make_cam(width, height, f[v][0].item<float>(), f[v][1].item<float>(), rot[v], tran[v], near, thresh));
    Outputs o = alloc_outputs(pos, b, n, height, width, true, 0, final);
    gs_render_aux ax{bg.ptr(), fpm(o.aux), fpm_or_null(o.aux_fin)};
    rendered(gs_render_forward_batch(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), (int)n, (int)rgb.size(1),
                                     scale_activation, (int)b, cams.data(), fpm(o.raw), fpm_or_null(o.fin),
                                     o.mask.data_ptr<int64_t>(), &ax, cur_stream()),
             fn);
    batch = {b, height, width};
    return py::make_tuple(or_none(o.fin), o.raw, o.aux, or_none(o.aux_fin), o.mask);
  }

  // (views, height, width) of the last forward_batch: its backward's tensors are checked against them
  std::array<int64_t, 3> batch{0, 0, 0};

  // backward of forward_batch: gradients are the sums over the views; grad_aux = None runs the plain kernels
  void backward_batch_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                           torch::Tensor scale, torch::Tensor raw, torch::Tensor grad_image, bool grad_is_final,
                           torch::Tensor aux, std::optional<torch::Tensor> grad_aux, torch::Tensor g_pos,
                           torch::Tensor g_rgb, torch::Tensor g_opa, torch::Tensor g_quat, torch::Tensor g_scale,
                           int64_t expected_frame) {
    backward_checked("RenderContext.backward_batch_into", true, pos, rgb, opa, quat, scale, raw, grad_image,
                     grad_is_final, &aux, grad_aux, {g_pos, g_rgb, g_opa, g_quat, g_scale}, expected_frame);
  }

  // backward_aux_into plus the camera gradient grad_cam[12] = (dL/drot row-major, dL/dtran) of the forward's camera
  // (gs_render_backward_cam); the five parameter gradients all None: camera only.  aux = None: the forward wrote no
  // maps (forward / forward_final; then grad_aux must be None too)
  void backward_cam_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                         torch::Tensor scale, torch::Tensor raw, torch::Tensor grad_image, bool grad_is_final,
                         std::optional<torch::Tensor> aux, std::optional<torch::Tensor> grad_aux,
                         std::optional<torch::Tensor> g_pos, std::optional<torch::Tensor> g_rgb,
                         std::optional<torch::Tensor> g_opa, std::optional<torch::Tensor> g_quat,
                         std::optional<torch::Tensor> g_scale, torch::Tensor grad_cam, int64_t expected_frame) {
    backward_cam_checked("RenderContext.backward_cam_into", false, pos, rgb, opa, quat, scale, raw, grad_image,
                         grad_is_final, aux ? &*aux : nullptr, grad_aux, {g_pos, g_rgb, g_opa, g_quat, g_scale},
                         grad_cam, expected_frame);
  }

  // backward_batch_into plus each view's camera gradient grad_cams[B,12] (gs_render_backward_batch_cam); the five
  // parameter gradients all None: camera only
  void backward_batch_cam_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                               torch::Tensor scale, torch::Tensor raw, torch::Tensor grad_image, bool grad_is_final,
                               torch::Tensor aux, std::optional<torch::Tensor> grad_aux,
                               std::optional<torch::Tensor> g_pos, std::optional<torch::Tensor> g_rgb,
                               std::optional<torch::Tensor> g_opa, std::optional<torch::Tensor> g_quat,
                               std::optional<torch::Tensor> g_scale, torch::Tensor grad_cams, int64_t expected_frame) {
    backward_cam_checked("RenderContext.backward_batch_cam_into", true, pos, rgb, opa, quat, scale, raw, grad_image,
                         grad_is_final, &aux, grad_aux, {g_pos, g_rgb, g_opa, g_quat, g_scale}, grad_cams,
                         expected_frame);
  }

  // the camera-gradient backward of the last single-view (gs_render_backward_cam: grad_cam [12]) or batched
  // (gs_render_backward_batch_cam: grad_cam [B,12]) forward; the five parameter gradients all given or all None
  void backward_cam_checked(const char* fn, bool batched, const torch::Tensor& pos, const torch::Tensor& rgb,
                            const torch::Tensor& opa, const torch::Tensor& quat, const torch::Tensor& scale,
                            const torch::Tensor& raw, const torch::Tensor& grad_image, bool grad_is_final,
                            const torch::Tensor* aux, const std::optional<torch::Tensor>& grad_aux,
                            const std::array<std::optional<torch::Tensor>, 5>& g, const torch::Tensor& grad_cam,
                            int64_t expected_frame) {
    check_backward(fn, expected_frame, batched, grad_is_final, pos, rgb, opa, quat, scale, raw, grad_image, aux,
                   grad_aux ? &*grad_aux : nullptr);
    GS_CHECK_F32(grad_cam);
    if (batched) {
      TORCH_CHECK(grad_cam.dim() == 2 && grad_cam.size(0) == batch[0] && grad_cam.size(1) == 12 &&
                      grad_cam.device() == pos.device(),
                  fn, ": grad_cams must be [", batch[0], ",12] on the parameters' device");
    } else {
      TORCH_CHECK(grad_cam.numel() == 12 && grad_cam.device() == pos.device(), fn,
                  ": grad_cam must be 12 floats on the parameters' device");
    }
    int n_given = 0;
    for (const auto& t : g) n_given += t.has_value();
    TORCH_CHECK(n_given == 0 || n_given == 5, fn, ": give all five parameter gradients or none (camera only)");
    if (n_given) check_grads(fn, {pos, rgb, opa, quat, scale}, {*g[0], *g[1], *g[2], *g[3], *g[4]});
    auto opt = [](const std::optional<torch::Tensor>& t) { return t ? fpm(*t) : nullptr; };
    c10::cuda::CUDAGuard guard(pos.device());
    auto gi = grad_image.contiguous();
    torch::Tensor ga;
    if (grad_aux) ga = grad_aux->contiguous();
    auto entry = batched ? &gs_render_backward_batch_cam : &gs_render_backward_cam;
    check_rc(entry(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), fp(raw), fp(gi), grad_is_final ? 1 : 0,
                   aux ? fp(*aux) : nullptr, fpm_or_null(ga), opt(g[0]), opt(g[1]), opt(g[2]), opt(g[3]), opt(g[4]),
                   fpm(grad_cam), cur_stream()),
             fn);
  }

  // feature maps (gs_render_forward_feat): forward_aux's outputs plus (map padded [Hp,Wp,f], map_final [H,W,f] or None):
  // (final or None, raw, aux, aux_final or None, map, map_final or None, mask)
  py::tuple forward_feat(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                         torch::Tensor scale, torch::Tensor feat, int width, int height, float fx, float fy,
                         torch::Tensor rot, torch::Tensor tran, float near, float thresh, int scale_activation,
                         std::optional<std::vector<double>> background, bool final) {
    const char* fn = "RenderContext.forward_feat";
    const int64_t n = check_params(fn, pos, rgb, opa, quat, scale, &feat);
    const Background bg = background_of(fn, background);
    c10::cuda::CUDAGuard guard(pos.device());
    gs_camera cam = make_cam(width, height, fx, fy, rot, tran, near, thresh);
    const int64_t f = feat.size(1);
    Outputs o = alloc_outputs(pos, 0, n, height, width, true, f, final);
    gs_render_aux ax{bg.ptr(), fpm(o.aux), fpm_or_null(o.aux_fin)};
    gs_render_feat ft{(int)f, fp(feat), fpm(o.map), fpm_or_null(o.map_fin)};
    rendered(gs_render_forward_feat(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), (int)n, (int)rgb.size(1),
                                    scale_activation, &cam, fpm(o.raw), fpm_or_null(o.fin),
                                    o.mask.data_ptr<int64_t>(), &ax, &ft, cur_stream()),
             fn);
    return py::make_tuple(or_none(o.fin), o.raw, o.aux, or_none(o.aux_fin), o.map, or_none(o.map_fin), o.mask);
  }

  // backward of forward_feat; grad_map = None: the plain / aux backward kernels, g_feat zero-filled
  void backward_feat_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                          torch::Tensor scale, torch::Tensor feat, torch::Tensor raw, torch::Tensor grad_image,
                          bool grad_is_final, torch::Tensor aux, std::optional<torch::Tensor> grad_aux,
                          torch::Tensor map, std::optional<torch::Tensor> grad_map, torch::Tensor g_pos,
                          torch::Tensor g_rgb, torch::Tensor g_opa, torch::Tensor g_quat, torch::Tensor g_scale,
                          torch::Tensor g_feat, int64_t expected_frame) {
    const char* fn = "RenderContext.backward_feat_into";
    check_backward(fn, expected_frame, false, grad_is_final, pos, rgb, opa, quat, scale, raw, grad_image, &aux,
                   grad_aux ? &*grad_aux : nullptr, &feat, &map, grad_map ? &*grad_map : nullptr);
    check_grads(fn, {pos, rgb, opa, quat, scale, feat}, {g_pos, g_rgb, g_opa, g_quat, g_scale, g_feat});
    c10::cuda::CUDAGuard guard(pos.device());
    auto gi = grad_image.contiguous();
    torch::Tensor ga, gm;
    if (grad_aux) ga = grad_aux->contiguous();
    if (grad_map) gm = grad_map->contiguous();
    check_rc(gs_render_backward_feat(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), fp(raw), fp(gi),
                                     grad_is_final ? 1 : 0, fp(aux), fpm_or_null(ga), fp(feat), fp(map),
                                     fpm_or_null(gm), fpm(g_pos), fpm(g_rgb), fpm(g_opa), fpm(g_quat), fpm(g_scale),
                                     fpm(g_feat), cur_stream()),
             fn);
  }

  // 2D Gaussian surfels (gs_render_forward_surfel): maps = the GS_SURFEL_MAP_CH map channels (alpha, depth, median,
  // distortion, normal xyz, 0); returns (final[H,W,3] or None, raw padded[Hp,Wp,3], maps padded[Hp,Wp,8] or None,
  // maps_final[H,W,8] or None, mask)
  py::tuple forward_surfel(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                           torch::Tensor scale, int width, int height, float fx, float fy, torch::Tensor rot,
                           torch::Tensor tran, float near, float thresh, int scale_activation,
                           std::optional<std::vector<double>> background, bool maps, bool final, double dist_near,
                           double dist_far) {
    const char* fn = "RenderContext.forward_surfel";
    const int64_t n = check_params(fn, pos, rgb, opa, quat, scale);
    const Background bg = background_of(fn, background);
    c10::cuda::CUDAGuard guard(pos.device());
    gs_camera cam = make_cam(width, height, fx, fy, rot, tran, near, thresh);
    Outputs o = alloc_outputs(pos, 0, n, height, width, false, maps ? GS_SURFEL_MAP_CH : 0, final);
    gs_render_surfel sf{bg.ptr(), fpm_or_null(o.map), fpm_or_null(o.map_fin), (float)dist_near, (float)dist_far};
    rendered(gs_render_forward_surfel(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), (int)n, (int)rgb.size(1),
                                      scale_activation, &cam, fpm(o.raw), fpm_or_null(o.fin),
                                      o.mask.data_ptr<int64_t>(), &sf, cur_stream()),
             fn);
    return py::make_tuple(or_none(o.fin), o.raw, or_none(o.map), or_none(o.map_fin), o.mask);
  }

  // backward of forward_surfel; grad_maps = None: zero map gradients (the kernels without the map terms)
  void backward_surfel_into(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                            torch::Tensor scale, torch::Tensor raw, torch::Tensor grad_image, bool grad_is_final,
                            std::optional<torch::Tensor> grad_maps, torch::Tensor g_pos, torch::Tensor g_rgb,
                            torch::Tensor g_opa, torch::Tensor g_quat, torch::Tensor g_scale, int64_t expected_frame) {
    const char* fn = "RenderContext.backward_surfel_into";
    check_backward(fn, expected_frame, false, grad_is_final, pos, rgb, opa, quat, scale, raw, grad_image, nullptr,
                   nullptr);
    if (grad_maps) {
      const std::vector<int64_t> pixels = grad_is_final ? std::vector<int64_t>{grad_image.size(0), grad_image.size(1)}
                                                        : std::vector<int64_t>{raw.size(0), raw.size(1)};
      check_image(fn, "grad_maps", *grad_maps, pixels, GS_SURFEL_MAP_CH, false);
    }
    check_grads(fn, {pos, rgb, opa, quat, scale}, {g_pos, g_rgb, g_opa, g_quat, g_scale});
    c10::cuda::CUDAGuard guard(pos.device());
    auto gi = grad_image.contiguous();
    torch::Tensor gm;
    if (grad_maps) gm = grad_maps->contiguous();
    check_rc(gs_render_backward_surfel(ctx, fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), fp(raw), fp(gi),
                                       grad_is_final ? 1 : 0, fpm_or_null(gm), fpm(g_pos), fpm(g_rgb), fpm(g_opa),
                                       fpm(g_quat), fpm(g_scale), cur_stream()),
             fn);
  }

  int64_t last_instances() { return (int64_t)gs_frame_instances(ctx); }

  // weight_sum[n] += sum of the last forward's blend weights per Gaussian, weight_max[n] = max with its largest one
  // (gs_frame_scores)
  void scores_into(torch::Tensor weight_sum, torch::Tensor weight_max) {
    for (auto* t : {&weight_sum, &weight_max}) {
      TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == at::kFloat && t->dim() == 1,
                  "RenderContext.scores_into: weight_sum and weight_max must be contiguous 1-D CUDA float32 tensors");
      TORCH_CHECK(t->device().index() == device,
                  "RenderContext.scores_into: weight_sum / weight_max is on another device than the context");
    }
    TORCH_CHECK(weight_sum.numel() == weight_max.numel(), "RenderContext.scores_into: weight_sum and weight_max differ in size");
    TORCH_CHECK(weight_sum.numel() < (int64_t(1) << 31), "RenderContext.scores_into: too many Gaussians");
    c10::cuda::CUDAGuard guard(weight_sum.device());
    struct gs_frame_scores sc{};
    sc.n = (int)weight_sum.numel();
    sc.weight_sum = weight_sum.data_ptr<float>();
    sc.weight_max = weight_max.data_ptr<float>();
    check_rc(gs_frame_scores(ctx, &sc, cur_stream()), "gs_frame_scores");
  }

  // mask[n] (uint8) = the Gaussians the last forward binned (gs_frame_visible); accumulate: OR into mask
  void visible_into(torch::Tensor mask, bool accumulate) {
    TORCH_CHECK(mask.is_cuda() && mask.is_contiguous() && mask.scalar_type() == at::kByte && mask.dim() == 1,
                "RenderContext.visible_into: mask must be a contiguous 1-D CUDA uint8 tensor");
    TORCH_CHECK(mask.device().index() == device, "RenderContext.visible_into: mask is on another device than the context");
    TORCH_CHECK(mask.numel() < (int64_t(1) << 31), "RenderContext.visible_into: mask too large");
    c10::cuda::CUDAGuard guard(mask.device());
    check_rc(gs_frame_visible(ctx, mask.data_ptr<uint8_t>(), (int)mask.numel(), accumulate ? 1 : 0, cur_stream()),
             "gs_frame_visible");
  }

  py::dict stats() {
    gs_frame_info fi{};
    check_rc(gs_frame_stats(ctx, &fi, cur_stream()), "gs_frame_stats");
    py::dict d;
    d["n_gaussians"] = fi.n_gaussians;
    d["n_visible"] = fi.n_visible;
    d["n_instances"] = fi.n_instances;
    d["n_instances_eff"] = fi.n_instances_eff;
    d["width_padded"] = fi.width_padded;
    d["height_padded"] = fi.height_padded;
    d["n_tiles"] = fi.n_tiles;
    d["max_tile_count"] = fi.max_tile_count;
    d["n_instances_eff_bwd"] = fi.n_instances_eff_bwd;
    return d;
  }

  // (sorted gaussian ids [M] int32, tile_n_point_accum [T+1] int32) of the last forward
  std::tuple<torch::Tensor, torch::Tensor> sorted_instances() {
    gs_frame_info fi{};
    check_rc(gs_frame_stats(ctx, &fi, cur_stream()), "gs_frame_stats");
    auto opts = torch::TensorOptions().device(torch::kCUDA, device).dtype(at::kInt);
    auto idx = torch::empty({(int64_t)fi.n_instances}, opts);
    auto accum = torch::empty({(int64_t)fi.n_tiles + 1}, opts);
    check_rc(gs_frame_sorted(ctx, idx.data_ptr<int>(), fi.n_instances, accum.data_ptr<int>(), cur_stream()),
             "gs_frame_sorted");
    return {idx, accum};
  }

  // consumed instances per tile [T] int32 of the last forward (M_eff = sum)
  torch::Tensor tile_consumed() {
    gs_frame_info fi{};
    check_rc(gs_frame_stats(ctx, &fi, cur_stream()), "gs_frame_stats");
    auto out = torch::empty({(int64_t)fi.n_tiles}, torch::TensorOptions().device(torch::kCUDA, device).dtype(at::kInt));
    check_rc(gs_frame_tile_consumed(ctx, out.data_ptr<int>(), cur_stream()), "gs_frame_tile_consumed");
    return out;
  }
};

// fused Adam over flat buffers (SURVEY.md §8 f-2); seg_ends / lrs are small host lists
void adam_step(torch::Tensor param, torch::Tensor grad, torch::Tensor exp_avg, torch::Tensor exp_avg_sq,
               std::vector<int64_t> seg_ends, std::vector<double> lrs, double beta1, double beta2, double eps,
               int64_t step) {
  GS_CHECK_F32(param); GS_CHECK_F32(grad); GS_CHECK_F32(exp_avg); GS_CHECK_F32(exp_avg_sq);
  int64_t n = param.numel();
  TORCH_CHECK(grad.numel() == n && exp_avg.numel() == n && exp_avg_sq.numel() == n, "adam_step: size mismatch");
  TORCH_CHECK(seg_ends.size() == lrs.size() && !seg_ends.empty() && seg_ends.back() == n,
              "adam_step: segments must cover the flat buffer");
  for (auto* t : {&param, &grad, &exp_avg, &exp_avg_sq})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "adam_step: buffers must be 16-byte aligned");
  std::vector<long long> ends(seg_ends.begin(), seg_ends.end());
  std::vector<float> lr(lrs.begin(), lrs.end());
  c10::cuda::CUDAGuard guard(param.device());
  check_rc(gs_adam_step(fpm(param), fp(grad), fpm(exp_avg), fpm(exp_avg_sq), n, ends.data(), lr.data(), (int)ends.size(),
                        (float)beta1, (float)beta2, (float)eps, (int)step, cur_stream()),
           "gs_adam_step");
}

// Adam on the rows of the visible Gaussians only (gs_adam_step_visible); segment s is [visible.numel(), seg_widths[s]]
// at float seg_starts[s] of the flat buffers
void adam_step_visible(torch::Tensor param, torch::Tensor grad, torch::Tensor exp_avg, torch::Tensor exp_avg_sq,
                       std::vector<int64_t> seg_starts, std::vector<int64_t> seg_widths, std::vector<double> lrs,
                       torch::Tensor visible, double beta1, double beta2, double eps, int64_t step) {
  GS_CHECK_F32(param); GS_CHECK_F32(grad); GS_CHECK_F32(exp_avg); GS_CHECK_F32(exp_avg_sq);
  int64_t n = param.numel();
  TORCH_CHECK(grad.numel() == n && exp_avg.numel() == n && exp_avg_sq.numel() == n, "adam_step_visible: size mismatch");
  TORCH_CHECK(seg_starts.size() == lrs.size() && seg_widths.size() == lrs.size() && !lrs.empty(),
              "adam_step_visible: one start, width and learning rate per segment");
  TORCH_CHECK(visible.is_cuda() && visible.is_contiguous() && visible.scalar_type() == at::kByte &&
                  visible.device() == param.device() && visible.numel() < (int64_t(1) << 31),
              "adam_step_visible: visible must be a contiguous CUDA uint8 tensor on the parameters' device");
  for (auto* t : {&param, &grad, &exp_avg, &exp_avg_sq})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "adam_step_visible: buffers must be 16-byte aligned");
  std::vector<long long> starts(seg_starts.begin(), seg_starts.end());
  std::vector<int> widths;
  for (int64_t w : seg_widths) {
    TORCH_CHECK(w >= 1 && w < (int64_t(1) << 31), "adam_step_visible: bad segment width");
    widths.push_back((int)w);
  }
  std::vector<float> lr(lrs.begin(), lrs.end());
  c10::cuda::CUDAGuard guard(param.device());
  check_rc(gs_adam_step_visible(fpm(param), fp(grad), fpm(exp_avg), fpm(exp_avg_sq), n, starts.data(), widths.data(),
                                lr.data(), (int)lr.size(), (int)visible.numel(), visible.data_ptr<uint8_t>(),
                                (float)beta1, (float)beta2, (float)eps, (int)step, cur_stream()),
           "gs_adam_step_visible");
}

// fused L1 + SSIM loss (SURVEY.md §8 f-3, reference train.py:99-107): returns (out3 = {total, l1, ssim}, grad_image)
std::tuple<torch::Tensor, torch::Tensor> loss_l1_ssim(torch::Tensor image, torch::Tensor target, double w_l1,
                                                      double w_ssim, double bias, bool want_grad) {
  GS_CHECK_F32(image);
  TORCH_CHECK(target.is_cuda() && target.is_contiguous() &&
                  (target.scalar_type() == at::kFloat || target.scalar_type() == at::kHalf),
              "loss_l1_ssim: target must be a contiguous float32 / float16 CUDA tensor");
  TORCH_CHECK(image.dim() == 3 && image.size(2) == 3 && target.sizes() == image.sizes(),
              "loss_l1_ssim: image and target must both be [H, W, 3]");
  TORCH_CHECK(image.size(0) > 10 && image.size(1) > 10, "loss_l1_ssim: the image must be larger than the 11x11 window");
  c10::cuda::CUDAGuard guard(image.device());
  const int h = (int)image.size(0), w = (int)image.size(1);
  auto ws = torch::empty({(int64_t)gs_loss_workspace_bytes(h, w)}, image.options().dtype(at::kByte));
  auto out3 = torch::empty({3}, image.options());
  torch::Tensor grad = want_grad ? torch::empty_like(image) : torch::Tensor();
  check_rc(gs_loss_l1_ssim(fp(image), target.data_ptr(), target.scalar_type() == at::kHalf ? 1 : 0, h, w, (float)w_l1,
                           (float)w_ssim, (float)bias, want_grad ? fpm(grad) : nullptr, fpm(out3), ws.data_ptr(),
                           (size_t)ws.numel(), cur_stream()),
           "gs_loss_l1_ssim");
  return {out3, grad};
}

// the apply half of densify / densify_stats: reads the plan's totals (the one host sync), draws the split samples and
// writes the five new parameter tensors; returns them + (n_deleted, n_clone, n_split)
static std::tuple<std::vector<torch::Tensor>, std::vector<int64_t>> densify_apply(
    const torch::Tensor& pos, const torch::Tensor& rgb, const torch::Tensor& opa, const torch::Tensor& quat,
    const torch::Tensor& scale, const float* grad, int scale_activation, double clone_dt,
    c10::optional<at::Generator> gen, const torch::Tensor& code, const torch::Tensor& dst,
    const c10::optional<torch::Tensor>& feat) {
  const int64_t n = pos.size(0);
  int64_t nk = n, nc = 0, nsp = 0;
  if (n > 0) {
    auto tot = dst.index({torch::indexing::Slice(), n}).cpu();        // the one host sync: sizes of the new arrays
    nk = tot[0].item<int>(); nc = tot[1].item<int>(); nsp = tot[2].item<int>();
  }
  const int64_t m = nk + nc + nsp;
  const int64_t d = rgb.size(1);
  auto z = torch::randn({2, nsp, 3}, gen, pos.options());              // torch's generator: identical on every DP rank
  std::vector<torch::Tensor> out = {torch::empty({m, 3}, pos.options()), torch::empty({m, d}, pos.options()),
                                    torch::empty({m}, pos.options()), torch::empty({m, 4}, pos.options()),
                                    torch::empty({m, 3}, pos.options())};
  check_rc(gs_densify_apply(fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), (int)n, (int)d, code.data_ptr<uint8_t>(),
                            dst.data_ptr<int>(), grad, (float)clone_dt, fp(z), (int)nk, (int)nc, (int)nsp,
                            scale_activation, fpm(out[0]), fpm(out[1]), fpm(out[2]), fpm(out[3]), fpm(out[4]),
                            cur_stream()),
           "gs_densify_apply");
  if (feat) {   // per-Gaussian features follow the same plan (a 6th tensor)
    out.push_back(torch::empty({m, feat->size(1)}, pos.options()));
    check_rc(gs_densify_apply_rows(fp(*feat), (int)n, (int)feat->size(1), code.data_ptr<uint8_t>(), dst.data_ptr<int>(),
                                   (int)nk, (int)nc, (int)nsp, fpm(out[5]), cur_stream()),
             "gs_densify_apply_rows");
  }
  return {out, {n - nk, nc, nsp}};
}

// keep-only densification plan: the rows with keep[i] set, in order (code = keep bit, dst[0] = its exclusive scan, no
// clones or splits); returns the new parameter tensors (+ feat) and the number removed
std::tuple<std::vector<torch::Tensor>, int64_t> prune(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa,
                                                      torch::Tensor quat, torch::Tensor scale, torch::Tensor keep,
                                                      c10::optional<torch::Tensor> feat) {
  GS_CHECK_F32(pos); GS_CHECK_F32(rgb); GS_CHECK_F32(opa); GS_CHECK_F32(quat); GS_CHECK_F32(scale);
  const int64_t n = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && rgb.dim() == 2 && rgb.size(0) == n && opa.numel() == n &&
                  quat.dim() == 2 && quat.size(0) == n && quat.size(1) == 4 && scale.dim() == 2 && scale.size(0) == n &&
                  scale.size(1) == 3,
              "prune: bad shapes");
  TORCH_CHECK(n < (int64_t(1) << 31), "prune: too many Gaussians");
  TORCH_CHECK(keep.is_cuda() && keep.scalar_type() == at::kBool && keep.dim() == 1 && keep.numel() == n &&
                  keep.device() == pos.device(),
              "prune: keep must be a 1-D CUDA bool tensor [n] on the parameters' device");
  if (feat) {
    GS_CHECK_F32(*feat);
    TORCH_CHECK(feat->dim() == 2 && feat->size(0) == n && feat->size(1) > 0, "prune: feat must be [n, f]");
  }
  c10::cuda::CUDAGuard guard(pos.device());
  auto code = torch::zeros({n + 1}, keep.options().dtype(at::kByte));
  code.narrow(0, 0, n).copy_(keep);
  auto dst = torch::zeros({3, n + 1}, keep.options().dtype(at::kInt));
  if (n > 0) dst[0].narrow(0, 1, n).copy_(torch::cumsum(keep, 0, at::kInt));
  auto [out, counts] = densify_apply(pos, rgb, opa, quat, scale, nullptr, 0, 0.0, c10::nullopt, code, dst, feat);
  return {out, counts[0]};
}

// densification (SURVEY.md §8 f-2): returns the five new parameter tensors + (n_deleted, n_clone, n_split)
std::tuple<std::vector<torch::Tensor>, std::vector<int64_t>> densify(
    torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat, torch::Tensor scale, torch::Tensor grad,
    int scale_activation, double opa_logit_min, double delete_thresh, double grad_thresh, bool grad_agg_max, double tau,
    bool use_clone, bool use_split, double clone_dt, c10::optional<at::Generator> gen,
    c10::optional<torch::Tensor> feat) {
  GS_CHECK_F32(pos); GS_CHECK_F32(rgb); GS_CHECK_F32(opa); GS_CHECK_F32(quat); GS_CHECK_F32(scale); GS_CHECK_F32(grad);
  const int64_t n = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && rgb.dim() == 2 && rgb.size(0) == n && opa.numel() == n &&
                  quat.numel() == 4 * n && scale.numel() == 3 * n && grad.numel() == 3 * n && n < (int64_t(1) << 31),
              "densify: bad shapes");
  if (feat) {
    GS_CHECK_F32(*feat);
    TORCH_CHECK(feat->dim() == 2 && feat->size(0) == n && feat->size(1) > 0, "densify: feat must be [n, f]");
  }
  c10::cuda::CUDAGuard guard(pos.device());
  auto bopt = pos.options().dtype(at::kByte);
  auto code = torch::empty({n + 1}, bopt);
  auto dst = torch::empty({3, n + 1}, pos.options().dtype(at::kInt));
  auto ws = torch::empty({(int64_t)gs_densify_workspace_bytes((int)n)}, bopt);
  check_rc(gs_densify_plan(fp(opa), fp(scale), fp(grad), (int)n, scale_activation, (float)opa_logit_min,
                           (float)delete_thresh, (float)grad_thresh, grad_agg_max ? 1 : 0, (float)tau, use_clone ? 1 : 0,
                           use_split ? 1 : 0, code.data_ptr<uint8_t>(), dst.data_ptr<int>(), ws.data_ptr(),
                           (size_t)ws.numel(), cur_stream()),
           "gs_densify_plan");
  return densify_apply(pos, rgb, opa, quat, scale, grad.data_ptr<float>(), scale_activation, clone_dt, gen, code, dst,
                       feat);
}

// densification from the screen-space statistics (gs_densify_plan_stats; clones are exact copies, as in 3DGS)
std::tuple<std::vector<torch::Tensor>, std::vector<int64_t>> densify_stats(
    torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat, torch::Tensor scale,
    torch::Tensor accum, torch::Tensor count, c10::optional<torch::Tensor> max_radius, double max_screen_px,
    int scale_activation, double opa_logit_min, double delete_thresh, double grad_thresh, double tau, bool use_clone,
    bool use_split, c10::optional<at::Generator> gen, c10::optional<torch::Tensor> feat) {
  GS_CHECK_F32(pos); GS_CHECK_F32(rgb); GS_CHECK_F32(opa); GS_CHECK_F32(quat); GS_CHECK_F32(scale); GS_CHECK_F32(accum);
  const int64_t n = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && rgb.dim() == 2 && rgb.size(0) == n && opa.numel() == n &&
                  quat.numel() == 4 * n && scale.numel() == 3 * n && accum.numel() == n && n < (int64_t(1) << 31),
              "densify_stats: bad shapes");
  GS_CHECK_I32(count);
  TORCH_CHECK(count.numel() == n, "densify_stats: count must have n elements");
  if (max_radius) {
    GS_CHECK_F32(*max_radius);
    TORCH_CHECK(max_radius->numel() == n, "densify_stats: max_radius must have n elements");
  }
  if (feat) {
    GS_CHECK_F32(*feat);
    TORCH_CHECK(feat->dim() == 2 && feat->size(0) == n && feat->size(1) > 0, "densify_stats: feat must be [n, f]");
  }
  c10::cuda::CUDAGuard guard(pos.device());
  auto bopt = pos.options().dtype(at::kByte);
  auto code = torch::empty({n + 1}, bopt);
  auto dst = torch::empty({3, n + 1}, pos.options().dtype(at::kInt));
  auto ws = torch::empty({(int64_t)gs_densify_workspace_bytes((int)n)}, bopt);
  check_rc(gs_densify_plan_stats(fp(opa), fp(scale), fp(accum), count.data_ptr<int>(),
                                 max_radius ? fp(*max_radius) : nullptr, (float)max_screen_px, (int)n,
                                 scale_activation, (float)opa_logit_min, (float)delete_thresh, (float)grad_thresh,
                                 (float)tau, use_clone ? 1 : 0, use_split ? 1 : 0, code.data_ptr<uint8_t>(),
                                 dst.data_ptr<int>(), ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
           "gs_densify_plan_stats");
  return densify_apply(pos, rgb, opa, quat, scale, nullptr, scale_activation, 0.0, gen, code, dst, feat);
}

// shapes shared by the MCMC entries: pos [n,3], rgb [n,d], opa [n], quat [n,4], scale [n,3], feat [n,f] or None
static void mcmc_check_params(const char* who, const torch::Tensor& pos, const torch::Tensor& rgb,
                              const torch::Tensor& opa, const torch::Tensor& quat, const torch::Tensor& scale,
                              const c10::optional<torch::Tensor>& feat) {
  GS_CHECK_F32(pos); GS_CHECK_F32(rgb); GS_CHECK_F32(opa); GS_CHECK_F32(quat); GS_CHECK_F32(scale);
  const int64_t n = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && rgb.dim() == 2 && rgb.size(0) == n && opa.numel() == n &&
                  quat.dim() == 2 && quat.size(0) == n && quat.size(1) == 4 && scale.dim() == 2 && scale.size(0) == n &&
                  scale.size(1) == 3 && n < (int64_t(1) << 31),
              who, ": bad shapes");
  for (const torch::Tensor* t : {&rgb, &opa, &quat, &scale})
    TORCH_CHECK(t->device() == pos.device(), who, ": the parameters must be on one device");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(quat.data_ptr()) % 16 == 0, who,
              ": quat must be 16-byte aligned (its rows are read as float4)");
  if (feat) {
    GS_CHECK_F32(*feat);
    TORCH_CHECK(feat->dim() == 2 && feat->size(0) == n && feat->device() == pos.device(), who, ": feat must be [n, f]");
  }
}

// MCMC relocation in place (gs_mcmc_relocate).  u: float32 [n] uniforms; moments: flat Adam buffers + segment table
// (or None); touched: uint8 [n] or None.  Returns the relocated count as a device int32 [1] (no host sync).
torch::Tensor mcmc_relocate(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                            torch::Tensor scale, c10::optional<torch::Tensor> feat, int scale_activation,
                            double min_opacity, torch::Tensor u, c10::optional<torch::Tensor> exp_avg,
                            c10::optional<torch::Tensor> exp_avg_sq, std::vector<int64_t> seg_starts,
                            std::vector<int64_t> seg_widths, c10::optional<torch::Tensor> touched) {
  mcmc_check_params("mcmc_relocate", pos, rgb, opa, quat, scale, feat);
  const int64_t n = pos.size(0);
  GS_CHECK_F32(u);
  TORCH_CHECK(u.numel() == n && u.device() == pos.device(), "mcmc_relocate: u must have n elements");
  TORCH_CHECK(exp_avg.has_value() == exp_avg_sq.has_value(), "mcmc_relocate: give both moment buffers or neither");
  long long n_flat = 0;
  if (exp_avg) {
    GS_CHECK_F32(*exp_avg); GS_CHECK_F32(*exp_avg_sq);
    TORCH_CHECK(exp_avg->numel() == exp_avg_sq->numel() && exp_avg->device() == pos.device() &&
                    exp_avg_sq->device() == pos.device(),
                "mcmc_relocate: the moment buffers must match and be on the parameters' device");
    TORCH_CHECK(seg_starts.size() == seg_widths.size() && !seg_starts.empty(),
                "mcmc_relocate: one start and width per segment");
    n_flat = exp_avg->numel();
  }
  if (touched)
    TORCH_CHECK(touched->is_cuda() && touched->is_contiguous() && touched->scalar_type() == at::kByte &&
                    touched->numel() == n && touched->device() == pos.device(),
                "mcmc_relocate: touched must be a contiguous CUDA uint8 tensor [n]");
  std::vector<long long> starts(seg_starts.begin(), seg_starts.end());
  std::vector<int> widths;
  for (int64_t w : seg_widths) {
    TORCH_CHECK(w >= 1 && w < (int64_t(1) << 31), "mcmc_relocate: bad segment width");
    widths.push_back((int)w);
  }
  c10::cuda::CUDAGuard guard(pos.device());
  auto ws = torch::empty({(int64_t)gs_mcmc_workspace_bytes((int)n)}, pos.options().dtype(at::kByte));
  auto n_rel = torch::zeros({1}, pos.options().dtype(at::kInt));
  check_rc(gs_mcmc_relocate(fpm(pos), fpm(rgb), fpm(opa), fpm(quat), fpm(scale), feat ? fpm(*feat) : nullptr,
                            feat ? (int)feat->size(1) : 0, (int)n, (int)rgb.size(1), scale_activation,
                            (float)min_opacity, fp(u), exp_avg ? fpm(*exp_avg) : nullptr,
                            exp_avg_sq ? fpm(*exp_avg_sq) : nullptr, n_flat, exp_avg ? starts.data() : nullptr,
                            exp_avg ? widths.data() : nullptr, exp_avg ? (int)starts.size() : 0,
                            touched ? touched->data_ptr<uint8_t>() : nullptr, n_rel.data_ptr<int>(), ws.data_ptr(),
                            (size_t)ws.numel(), cur_stream()),
           "gs_mcmc_relocate");
  return n_rel;
}

// MCMC growth (gs_mcmc_add): u.numel() new Gaussians; returns the new [n + n_new] tensors (pos, rgb, opa, quat, scale
// and feat when given)
std::vector<torch::Tensor> mcmc_add(torch::Tensor pos, torch::Tensor rgb, torch::Tensor opa, torch::Tensor quat,
                                    torch::Tensor scale, c10::optional<torch::Tensor> feat, int scale_activation,
                                    double min_opacity, torch::Tensor u) {
  mcmc_check_params("mcmc_add", pos, rgb, opa, quat, scale, feat);
  GS_CHECK_F32(u);
  TORCH_CHECK(u.dim() == 1 && u.device() == pos.device(), "mcmc_add: u must be a 1-D tensor on the parameters' device");
  const int64_t n = pos.size(0), n_new = u.numel(), m = n + n_new, d = rgb.size(1);
  TORCH_CHECK(m < (int64_t(1) << 31), "mcmc_add: n + n_new too large");
  c10::cuda::CUDAGuard guard(pos.device());
  auto ws = torch::empty({(int64_t)gs_mcmc_workspace_bytes((int)std::max(n, n_new))}, pos.options().dtype(at::kByte));
  std::vector<torch::Tensor> out = {torch::empty({m, 3}, pos.options()), torch::empty({m, d}, pos.options()),
                                    torch::empty(opa.dim() == 2 ? std::vector<int64_t>{m, 1} : std::vector<int64_t>{m},
                                                 pos.options()),
                                    torch::empty({m, 4}, pos.options()), torch::empty({m, 3}, pos.options())};
  if (feat) out.push_back(torch::empty({m, feat->size(1)}, pos.options()));
  check_rc(gs_mcmc_add(fp(pos), fp(rgb), fp(opa), fp(quat), fp(scale), feat ? fp(*feat) : nullptr,
                       feat ? (int)feat->size(1) : 0, (int)n, (int)d, scale_activation, (float)min_opacity, (int)n_new,
                       fp(u), fpm(out[0]), fpm(out[1]), fpm(out[2]), fpm(out[3]), fpm(out[4]),
                       feat ? fpm(out[5]) : nullptr, ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
           "gs_mcmc_add");
  return out;
}

// MCMC position noise in place (gs_mcmc_noise); z: float32 [n, 3] or None (Philox stream keyed by seed)
void mcmc_noise(torch::Tensor pos, torch::Tensor quat, torch::Tensor scale, torch::Tensor opa, int scale_activation,
                double scaler, int64_t seed, c10::optional<torch::Tensor> z) {
  GS_CHECK_F32(pos); GS_CHECK_F32(quat); GS_CHECK_F32(scale); GS_CHECK_F32(opa);
  const int64_t n = pos.size(0);
  TORCH_CHECK(pos.dim() == 2 && pos.size(1) == 3 && quat.dim() == 2 && quat.size(0) == n && quat.size(1) == 4 &&
                  scale.dim() == 2 && scale.size(0) == n && scale.size(1) == 3 && opa.numel() == n &&
                  n < (int64_t(1) << 31),
              "mcmc_noise: bad shapes");
  for (const torch::Tensor* t : {&quat, &scale, &opa})
    TORCH_CHECK(t->device() == pos.device(), "mcmc_noise: the parameters must be on one device");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(quat.data_ptr()) % 16 == 0,
              "mcmc_noise: quat must be 16-byte aligned (its rows are read as float4)");
  if (z) {
    GS_CHECK_F32(*z);
    TORCH_CHECK(z->numel() == 3 * n && z->device() == pos.device(), "mcmc_noise: z must be [n, 3]");
  }
  c10::cuda::CUDAGuard guard(pos.device());
  check_rc(gs_mcmc_noise(fpm(pos), fp(quat), fp(scale), fp(opa), (int)n, scale_activation, (float)scaler,
                         (unsigned long long)seed, z ? fp(*z) : nullptr, cur_stream()),
           "gs_mcmc_noise");
}

// NVLS in-place all-reduce of a symmetric flat buffer (multicast address as an integer)
void allreduce_multimem(int64_t multicast_ptr, int64_t n_floats, int rank, int world, int device) {
  c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, (c10::DeviceIndex)device));
  check_rc(gs_allreduce_multimem_f32(reinterpret_cast<void*>(static_cast<uintptr_t>(multicast_ptr)), n_floats, rank,
                                     world, cur_stream()),
           "gs_allreduce_multimem_f32");
}

void allreduce_p2p(std::vector<int64_t> peer_ptrs, int64_t n_floats, int rank, int world, int device) {
  c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, (c10::DeviceIndex)device));
  TORCH_CHECK((int)peer_ptrs.size() == world, "allreduce_p2p: need one pointer per rank");
  std::vector<void*> ptrs;
  for (int64_t p : peer_ptrs) ptrs.push_back(reinterpret_cast<void*>(static_cast<uintptr_t>(p)));
  check_rc(gs_allreduce_p2p_f32(ptrs.data(), n_floats, rank, world, cur_stream()), "gs_allreduce_p2p_f32");
}

void allreduce_push_finish(std::vector<int64_t> bucket_ptrs, int64_t staging_local, int64_t n_floats, int64_t per,
                           int rank, int world, int device) {
  c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, (c10::DeviceIndex)device));
  TORCH_CHECK((int)bucket_ptrs.size() == world, "allreduce_push_finish: need one bucket pointer per rank");
  std::vector<void*> ptrs;
  for (int64_t p : bucket_ptrs) ptrs.push_back(reinterpret_cast<void*>(static_cast<uintptr_t>(p)));
  check_rc(gs_allreduce_push_finish_f32(ptrs.data(), reinterpret_cast<const float*>(static_cast<uintptr_t>(staging_local)),
                                        n_floats, per, rank, world, cur_stream()),
           "gs_allreduce_push_finish_f32");
}

void allreduce_push_finish_mc(int64_t bucket_multicast, int64_t bucket_local, int64_t staging_local, int64_t n_floats,
                              int64_t per, int rank, int world, int device) {
  c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, (c10::DeviceIndex)device));
  check_rc(gs_allreduce_push_finish_mc_f32(reinterpret_cast<void*>(static_cast<uintptr_t>(bucket_multicast)),
                                           reinterpret_cast<const float*>(static_cast<uintptr_t>(bucket_local)),
                                           reinterpret_cast<const float*>(static_cast<uintptr_t>(staging_local)), n_floats,
                                           per, rank, world, cur_stream()),
           "gs_allreduce_push_finish_mc_f32");
}

}  // namespace gsb200

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  using namespace gsb200;
  m.doc() = "H100-native (sm_90a) drop-in for the reference `gaussian` extension (libgs_b200 C ABI underneath)";
  m.def("culling", &culling, "gaussian culling (no-op stub, as in the reference)");
  m.def("world2camera", &world2camera, "world to camera (CUDA)");
  m.def("world2camera_backward", &world2camera_backward, "world to camera backward (CUDA)");
  m.def("jacobian", &jacobian, "jacobian (CUDA)");

  py::class_<TilesPy>(m, "Tiles")
      .def(py::init<>())
      .def_readwrite("top", &TilesPy::top)
      .def_readwrite("bottom", &TilesPy::bottom)
      .def_readwrite("left", &TilesPy::left)
      .def_readwrite("right", &TilesPy::right);

  py::class_<Gaussian3dsPy>(m, "Gaussian3ds")
      .def(py::init<>())
      .def_readwrite("pos", &Gaussian3dsPy::pos)
      .def_readwrite("rgb", &Gaussian3dsPy::rgb)
      .def_readwrite("opa", &Gaussian3dsPy::opa)
      .def_readwrite("quat", &Gaussian3dsPy::quat)
      .def_readwrite("scale", &Gaussian3dsPy::scale)
      .def_readwrite("cov", &Gaussian3dsPy::cov);

  m.def("calc_tile_list", &calc_tile_list, "calc tile list (CUDA)");
  m.def("gather_gaussians", &gather_gaussians, "gather gaussian (CUDA)");
  m.def("draw", &draw, "draw (CUDA)");
  m.def("draw_backward", &draw_backward, "draw backward (CUDA)");
  m.def("global_culling", &global_culling, "global culling (CUDA)");
  m.def("global_culling_backward", &global_culling_backward, "global culling backward (CUDA)");

  py::class_<RenderContext>(m, "RenderContext")
      .def(py::init<>())
      .def("forward", &RenderContext::forward)
      .def("backward", &RenderContext::backward)
      .def("backward_into", &RenderContext::backward_into, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("image"), py::arg("grad_image"), py::arg("g_pos"),
           py::arg("g_rgb"), py::arg("g_opa"), py::arg("g_quat"), py::arg("g_scale"), py::arg("expected_frame") = -1)
      .def("forward_final", &RenderContext::forward_final)
      .def("backward_final_into", &RenderContext::backward_final_into, py::arg("pos"), py::arg("rgb"),
           py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("raw"), py::arg("grad_final"),
           py::arg("g_pos"), py::arg("g_rgb"), py::arg("g_opa"), py::arg("g_quat"), py::arg("g_scale"),
           py::arg("expected_frame") = -1)
      .def("forward_aux", &RenderContext::forward_aux, py::arg("pos"), py::arg("rgb"), py::arg("opa"), py::arg("quat"),
           py::arg("scale"), py::arg("width"), py::arg("height"), py::arg("fx"), py::arg("fy"), py::arg("rot"),
           py::arg("tran"), py::arg("near"), py::arg("thresh"), py::arg("scale_activation"),
           py::arg("background") = py::none(), py::arg("final") = true)
      .def("backward_aux_into", &RenderContext::backward_aux_into, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("raw"), py::arg("grad_image"), py::arg("grad_is_final"),
           py::arg("aux"), py::arg("grad_aux"), py::arg("g_pos"), py::arg("g_rgb"), py::arg("g_opa"),
           py::arg("g_quat"), py::arg("g_scale"), py::arg("expected_frame") = -1)
      .def("forward_batch", &RenderContext::forward_batch, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("width"), py::arg("height"), py::arg("focal"), py::arg("rot"),
           py::arg("tran"), py::arg("near"), py::arg("thresh"), py::arg("scale_activation"),
           py::arg("background") = py::none(), py::arg("final") = true)
      .def("backward_batch_into", &RenderContext::backward_batch_into, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("raw"), py::arg("grad_image"), py::arg("grad_is_final"),
           py::arg("aux"), py::arg("grad_aux"), py::arg("g_pos"), py::arg("g_rgb"), py::arg("g_opa"),
           py::arg("g_quat"), py::arg("g_scale"), py::arg("expected_frame") = -1)
      .def("backward_cam_into", &RenderContext::backward_cam_into, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("raw"), py::arg("grad_image"), py::arg("grad_is_final"),
           py::arg("aux"), py::arg("grad_aux"), py::arg("g_pos"), py::arg("g_rgb"), py::arg("g_opa"),
           py::arg("g_quat"), py::arg("g_scale"), py::arg("grad_cam"), py::arg("expected_frame") = -1)
      .def("backward_batch_cam_into", &RenderContext::backward_batch_cam_into, py::arg("pos"), py::arg("rgb"),
           py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("raw"), py::arg("grad_image"),
           py::arg("grad_is_final"), py::arg("aux"), py::arg("grad_aux"), py::arg("g_pos"), py::arg("g_rgb"),
           py::arg("g_opa"), py::arg("g_quat"), py::arg("g_scale"), py::arg("grad_cams"),
           py::arg("expected_frame") = -1)
      .def("forward_feat", &RenderContext::forward_feat, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("feat"), py::arg("width"), py::arg("height"), py::arg("fx"),
           py::arg("fy"), py::arg("rot"), py::arg("tran"), py::arg("near"), py::arg("thresh"),
           py::arg("scale_activation"), py::arg("background") = py::none(), py::arg("final") = true)
      .def("forward_surfel", &RenderContext::forward_surfel, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("width"), py::arg("height"), py::arg("fx"), py::arg("fy"),
           py::arg("rot"), py::arg("tran"), py::arg("near"), py::arg("thresh"), py::arg("scale_activation"),
           py::arg("background"), py::arg("maps"), py::arg("final"), py::arg("dist_near") = 0.2,
           py::arg("dist_far") = 100.0)
      .def("backward_surfel_into", &RenderContext::backward_surfel_into, py::arg("pos"), py::arg("rgb"),
           py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("raw"), py::arg("grad_image"),
           py::arg("grad_is_final"), py::arg("grad_maps"), py::arg("g_pos"), py::arg("g_rgb"), py::arg("g_opa"),
           py::arg("g_quat"), py::arg("g_scale"), py::arg("expected_frame") = -1)
      .def("backward_feat_into", &RenderContext::backward_feat_into, py::arg("pos"), py::arg("rgb"), py::arg("opa"),
           py::arg("quat"), py::arg("scale"), py::arg("feat"), py::arg("raw"), py::arg("grad_image"),
           py::arg("grad_is_final"), py::arg("aux"), py::arg("grad_aux"), py::arg("map"), py::arg("grad_map"),
           py::arg("g_pos"), py::arg("g_rgb"), py::arg("g_opa"), py::arg("g_quat"), py::arg("g_scale"),
           py::arg("g_feat"), py::arg("expected_frame") = -1)
      .def("frame_id", &RenderContext::frame_id)
      .def("last_instances", &RenderContext::last_instances)
      .def("visible_into", &RenderContext::visible_into, py::arg("mask"), py::arg("accumulate") = false)
      .def("scores_into", &RenderContext::scores_into, py::arg("weight_sum"), py::arg("weight_max"))
      .def("stats", &RenderContext::stats)
      .def("set_sh_eval", &RenderContext::set_sh_eval, py::arg("mode"))
      .def("set_filter2d", &RenderContext::set_filter2d, py::arg("mode"), py::arg("variance") = 0.3)
      .def("set_filter3d", &RenderContext::set_filter3d, py::arg("filter3d"))
      .def("set_lens", &RenderContext::set_lens, py::arg("models"), py::arg("params"))
      .def("set_densify_stats", &RenderContext::set_densify_stats, py::arg("grad2d"), py::arg("count"),
           py::arg("max_radius"), py::arg("absgrad") = py::none())
      .def("clear_densify_stats", &RenderContext::clear_densify_stats)
      .def("set_timing", &RenderContext::set_timing)
      .def("set_grad_push", &RenderContext::set_grad_push)
      .def("clear_grad_push", &RenderContext::clear_grad_push)
      .def("stage_ms", &RenderContext::stage_ms)
      .def("sorted_instances", &RenderContext::sorted_instances)
      .def("tile_consumed", &RenderContext::tile_consumed);
  m.def("allreduce_push_finish", &allreduce_push_finish, "second half of the pushed gradient exchange");
  m.def("allreduce_push_finish_mc", &allreduce_push_finish_mc,
        "second half of the pushed gradient exchange, broadcast through the NVSwitch (multimem.st)");
  m.def("allreduce_p2p", &allreduce_p2p, "peer-to-peer two-shot in-place all-reduce of a symmetric buffer");
  m.def("allreduce_multimem", &allreduce_multimem, "NVLS multimem in-place all-reduce of a symmetric buffer");
  m.def("densify", &densify, "prune / clone / split on the device (reference splatter.py:122-228)", py::arg("pos"),
        py::arg("rgb"), py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("grad"), py::arg("scale_activation"),
        py::arg("opa_logit_min"), py::arg("delete_thresh"), py::arg("grad_thresh"), py::arg("grad_agg_max"), py::arg("tau"),
        py::arg("use_clone"), py::arg("use_split"), py::arg("clone_dt"), py::arg("generator") = py::none(),
        py::arg("feat") = py::none());
  m.def("prune", &prune, "keep the rows with keep[i] set (gs_densify_apply with a keep-only plan)", py::arg("pos"),
        py::arg("rgb"), py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("keep"), py::arg("feat") = py::none());
  m.def("densify_stats", &densify_stats,
        "prune / clone / split on the device from screen-space densification statistics (gs_densify_plan_stats)",
        py::arg("pos"), py::arg("rgb"), py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("accum"),
        py::arg("count"), py::arg("max_radius"), py::arg("max_screen_px"), py::arg("scale_activation"),
        py::arg("opa_logit_min"), py::arg("delete_thresh"), py::arg("grad_thresh"), py::arg("tau"),
        py::arg("use_clone"), py::arg("use_split"), py::arg("generator") = py::none(), py::arg("feat") = py::none());
  m.def("mcmc_relocate", &mcmc_relocate, "MCMC relocation of dead Gaussians, in place (gs_mcmc_relocate)",
        py::arg("pos"), py::arg("rgb"), py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("feat"),
        py::arg("scale_activation"), py::arg("min_opacity"), py::arg("u"), py::arg("exp_avg") = py::none(),
        py::arg("exp_avg_sq") = py::none(), py::arg("seg_starts") = std::vector<int64_t>{},
        py::arg("seg_widths") = std::vector<int64_t>{}, py::arg("touched") = py::none());
  m.def("mcmc_add", &mcmc_add, "MCMC growth: u.numel() Gaussians appended (gs_mcmc_add)", py::arg("pos"),
        py::arg("rgb"), py::arg("opa"), py::arg("quat"), py::arg("scale"), py::arg("feat"),
        py::arg("scale_activation"), py::arg("min_opacity"), py::arg("u"));
  m.def("mcmc_noise", &mcmc_noise, "MCMC position noise, in place (gs_mcmc_noise)", py::arg("pos"), py::arg("quat"),
        py::arg("scale"), py::arg("opa"), py::arg("scale_activation"), py::arg("scaler"), py::arg("seed"),
        py::arg("z") = py::none());
  m.def("filter3d_compute",
        [](RenderContext& rc, torch::Tensor pos, torch::Tensor size, torch::Tensor focal, torch::Tensor rot,
           torch::Tensor tran, double near, double margin, double variance, std::optional<torch::Tensor> out) {
          return rc.filter3d_compute(pos, size, focal, rot, tran, near, margin, variance, out);
        },
        "Mip-Splatting's 3-D filter from the sampling rate over V views (gs_filter3d_compute)", py::arg("ctx"),
        py::arg("pos"), py::arg("size"), py::arg("focal"), py::arg("rot"), py::arg("tran"), py::arg("near"),
        py::arg("margin") = 0.15, py::arg("variance") = 0.2, py::arg("out") = py::none());
  m.def("loss_l1_ssim", &loss_l1_ssim, "fused L1 + SSIM loss, forward + image gradient (CUDA)");
  m.def("adam_step", &adam_step, "fused Adam over flat parameter / gradient buffers (CUDA)");
  m.def("adam_step_visible", &adam_step_visible,
        "Adam over the rows of the visible Gaussians of flat parameter / gradient buffers (CUDA)");
  m.def("tune", [](const std::string& name, int value) { check_rc(gs_tune(name.c_str(), value), "gs_tune"); },
        "set an A/B tuning knob of the blend kernels (see include/gs_b200.h gs_tune)");
  m.def("kernel_launches", []() { return (int64_t)gs_kernel_launches(); },
        "kernels of libgs_b200 launched by this process so far");
  m.attr("abi_version") = gs_abi_version();
  m.attr("SH_EVAL_PIXEL") = GS_SH_EVAL_PIXEL;
  m.attr("SH_EVAL_GAUSSIAN") = GS_SH_EVAL_GAUSSIAN;
  m.attr("SURFEL_MAP_CH") = GS_SURFEL_MAP_CH;
  m.attr("FILTER2D_NONE") = GS_FILTER2D_NONE;
  m.attr("FILTER2D_DILATE") = GS_FILTER2D_DILATE;
  m.attr("FILTER2D_ANTIALIAS") = GS_FILTER2D_ANTIALIAS;
  m.attr("LENS_PINHOLE") = GS_LENS_PINHOLE;
  m.attr("LENS_OPENCV") = GS_LENS_OPENCV;
  m.attr("LENS_FISHEYE") = GS_LENS_FISHEYE;
}
