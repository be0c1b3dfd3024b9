"""Autograd operator boundary — host-side mirror of the reference's renderer.py.

Same public names, positional argument order, return values and zero-fill/ownership
conventions as reference renderer.py (`draw` :89, `trunc_exp` :102,
`world2camera_func` :119, `global_culling` :158), so code written against the
reference keeps working; underneath, every op calls the sm_90a kernels of
libgs_b200 through the `gaussian` extension in this directory.  Additive:
`render_frame`, one autograd node for the whole frame (fused path).

The product path never falls back to PyTorch/CPU math: importing this module
without the built extension raises.
"""
from __future__ import annotations

import torch

try:
    import gaussian
except ImportError as e:  # pragma: no cover - fail loudly, never fall back
    raise ImportError(
        "the `gaussian` CUDA extension is not built; run "
        "`python 3d-gaussian-splatting_b200/build.py` (needs nvcc, sm_90a)") from e


def _f32(t):
    return t.contiguous() if t.dtype == torch.float32 else t.float().contiguous()


class _Drawer(torch.autograd.Function):
    """Tile blend of sorted per-instance tensors (reference renderer.py:6-87)."""

    @staticmethod
    def forward(ctx, gaussians_pos, gaussians_rgb, gaussians_opa, gaussians_cov, tile_n_point_accum,
                padded_height, padded_width, focal_x, focal_y, render_weight_normalize=False,
                sigmoid=False, use_sh_coeff=False, fast=False, rays_o=None, lefttop_pos=None,
                vec_dx=None, vec_dy=None):
        pos, rgb, opa, cov = (_f32(gaussians_pos), _f32(gaussians_rgb), _f32(gaussians_opa), _f32(gaussians_cov))
        accum = tile_n_point_accum.contiguous()
        image = torch.empty(padded_height, padded_width, 3, device=pos.device, dtype=torch.float32)
        dummy = pos.new_zeros(3)
        rays = [dummy if r is None else _f32(r) for r in (rays_o, lefttop_pos, vec_dx, vec_dy)]
        gaussian.draw(pos, rgb, opa, cov, accum, image, focal_x, focal_y, render_weight_normalize, sigmoid,
                      fast, rays[0], rays[1], rays[2], rays[3], use_sh_coeff)
        ctx.save_for_backward(pos, rgb, opa, cov, accum, image, *rays)
        ctx.cfg = (focal_x, focal_y, render_weight_normalize, sigmoid, fast, use_sh_coeff)
        return image

    @staticmethod
    def backward(ctx, grad_output):
        pos, rgb, opa, cov, accum, image, rays_o, lefttop_pos, vec_dx, vec_dy = ctx.saved_tensors
        focal_x, focal_y, weight_normalize, sigmoid, fast, use_sh_coeff = ctx.cfg
        g_pos = torch.zeros_like(pos)          # z column stays 0 (depth is only a sort key)
        g_rgb = torch.empty_like(rgb)
        g_opa = torch.empty_like(opa)
        g_cov = torch.empty_like(cov)
        gaussian.draw_backward(pos, rgb, opa, cov, accum, image, _f32(grad_output), g_pos, g_rgb, g_opa, g_cov,
                               focal_x, focal_y, weight_normalize, sigmoid, fast, rays_o, lefttop_pos, vec_dx,
                               vec_dy, use_sh_coeff)
        return (g_pos, g_rgb, g_opa, g_cov) + (None,) * 13


draw = _Drawer.apply


class _trunc_exp(torch.autograd.Function):
    """exp with a clamped-gradient backward (reference renderer.py:91-100)."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(-1, 1))


trunc_exp = _trunc_exp.apply


class _world2camera(torch.autograd.Function):
    """p @ R^T + t and its adjoint (reference renderer.py:104-117; deprecated path)."""

    @staticmethod
    def forward(ctx, pos, rot, tran):
        pos, rot, tran = _f32(pos), _f32(rot), _f32(tran)
        ctx.save_for_backward(rot)
        res = torch.empty_like(pos)
        gaussian.world2camera(pos, rot, tran, res)
        return res

    @staticmethod
    def backward(ctx, grad_out):
        (rot,) = ctx.saved_tensors
        grad_out = _f32(grad_out)
        grad_inp = torch.empty_like(grad_out)
        gaussian.world2camera_backward(grad_out, rot, grad_inp)
        return grad_inp, None, None


world2camera_func = _world2camera.apply


class _GlobalCulling(torch.autograd.Function):
    """Projection + near/frustum cull + 2-D covariance (reference renderer.py:121-156)."""

    @staticmethod
    def forward(ctx, pos, quat, scale, current_rot, current_tran, near, half_width, half_height):
        pos, quat, scale = _f32(pos), _f32(quat), _f32(scale)
        rot, tran = _f32(current_rot), _f32(current_tran)
        n = pos.shape[0]
        res_pos = torch.zeros_like(pos)                       # culled rows must read 0
        res_cov = torch.zeros((n, 2, 2), device=pos.device, dtype=torch.float32)
        culling_mask = torch.zeros(n, dtype=torch.long, device=pos.device)
        gaussian.global_culling(pos, quat, scale, rot, tran, res_pos, res_cov, culling_mask,
                                near, half_width, half_height)
        ctx.save_for_backward(culling_mask, pos, quat, scale, rot, tran)
        ctx.mark_non_differentiable(culling_mask)
        return res_pos, res_cov, culling_mask

    @staticmethod
    def backward(ctx, gradout_pos, gradout_cov, _grad_mask):
        culling_mask, pos, quat, scale, rot, tran = ctx.saved_tensors
        g_pos = torch.zeros_like(pos)
        g_quat = torch.zeros_like(quat)
        g_scale = torch.zeros_like(scale)
        gaussian.global_culling_backward(pos, quat, scale, rot, tran, _f32(gradout_pos), _f32(gradout_cov),
                                         culling_mask, g_pos, g_quat, g_scale)
        return g_pos, g_quat, g_scale, None, None, None, None, None


global_culling = _GlobalCulling.apply


# ----------------------------------------------------------------------------------------
# additive: the whole frame as one autograd node (fused path)
# ----------------------------------------------------------------------------------------
SCALE_ACTIVATIONS = {"abs": 0, "exp": 1}
# where SH colour is evaluated (RenderContext.set_sh_eval; the mode travels with the context, so the render_frame*
# functions take no argument for it): "pixel" = per pixel ray (the reference), "gaussian" = once per Gaussian along
# the camera-centre -> mean direction, then blended as an RGB colour
SH_EVAL = {"pixel": gaussian.SH_EVAL_PIXEL, "gaussian": gaussian.SH_EVAL_GAUSSIAN}
# screen-space 2-D filter (RenderContext.set_filter2d(mode, variance); a context setting like SH_EVAL): "none" (the
# reference), "dilate" (3DGS: + variance px^2 on the 2-D covariance), "antialias" (dilate + opacity compensation
# sqrt(det / det'), Mip-Splatting's 2-D filter)
FILTER2D = {"none": gaussian.FILTER2D_NONE, "dilate": gaussian.FILTER2D_DILATE,
            "antialias": gaussian.FILTER2D_ANTIALIAS}


_flat_grad_allocator = None


def set_flat_grad_allocator(fn):
    """Install `fn(numel, device) -> 1-D fp32 tensor (16-byte aligned)` (or `(tensor, push)` with
    push = (bucket_ptr, staging_ptrs, per, rank) for `RenderContext.set_grad_push`) as the source of the flat
    gradient bucket the fused backward writes into (None restores torch.empty).  Data-parallel
    runs use it to place the bucket in symmetric memory so the gradient exchange runs in place over
    NVLink (dp.NvlsGradBucket): the backward kernel's stores ARE the collective's send buffer."""
    global _flat_grad_allocator
    _flat_grad_allocator = fn


def _flat_grads(tensors):
    """Five gradient views carved out of ONE flat buffer (order pos, rgb, opa, quat, scale; each
    segment 16-byte aligned for the kernel's float4 stores) so that the data-parallel all-reduce
    runs in place on a single bucket (dp.GradBucket)."""
    sizes = [t.numel() for t in tensors]
    starts, o = [], 0
    for n in sizes:
        starts.append(o)
        o += (n + 3) // 4 * 4
    push = None
    if _flat_grad_allocator is not None:
        flat = _flat_grad_allocator(o, tensors[0].device)
        if isinstance(flat, tuple):                      # (bucket, push configuration) - see dp.py
            flat, push = flat
        assert flat.numel() >= o and flat.dtype == torch.float32 and flat.data_ptr() % 16 == 0
    else:
        flat = torch.empty(o, device=tensors[0].device, dtype=torch.float32)
    outs = []
    for t, n, b in zip(tensors, sizes, starts):
        outs.append(flat[b:b + n].view(t.shape))
        if n % 4:
            flat[b + n:b + (n + 3) // 4 * 4].zero_()     # keep the (<= 3 float) pads finite
    return outs, push


def _apply_push(rctx, push):
    """Route this backward's gradient stores: plain bucket, or (data-parallel push) other ranks'
    slices straight into their owners' staging buffers over NVLink (gs_grad_push)."""
    if push is None:
        rctx.clear_grad_push()
    else:
        rctx.set_grad_push(*push)


def _params(*tensors):
    """The frame's inputs as the contiguous float32 tensors the kernels read."""
    return tuple(_f32(t.detach()) for t in tensors)


def _save_frame(ctx, rctx, mask, saved, final=None, map_shape=None):
    """Keep what the backward of the frame `rctx` has just rendered needs: the context, the frame's id and `saved`.
    Frames with depth / alpha maps also keep `final` and the [(B,) rows, cols] of the maps they return, and let
    autograd pass None for outputs that got no gradient."""
    ctx.rctx = rctx
    ctx.frame = rctx.frame_id()
    ctx.save_for_backward(*saved)
    ctx.mark_non_differentiable(mask)
    if final is not None:
        ctx.final = bool(final)
        ctx.map_shape = tuple(map_shape)
        ctx.set_materialize_grads(False)


def _param_grads(rctx, params):
    """The five parameter gradient buffers of a backward, with its gradient push (or none) set on `rctx`."""
    outs, push = _flat_grads(params)
    _apply_push(rctx, push)
    return outs


def _upstream(raw, shape, grad_image, grad_depth, grad_alpha):
    """(grad_image [*shape, 3], grad_aux [*shape, 2]) from the gradients autograd passed (None: no gradient).  grad_aux
    is None when neither map got one, so the backward runs the plain kernels."""
    if grad_image is None:
        grad_image = raw.new_zeros(*shape, 3)
    grad_aux = None
    if grad_depth is not None or grad_alpha is not None:
        grad_aux = raw.new_zeros(*shape, 2)
        if grad_depth is not None:
            grad_aux[..., 0] = grad_depth
        if grad_alpha is not None:
            grad_aux[..., 1] = grad_alpha
    return _f32(grad_image), grad_aux


class _RenderFrame(torch.autograd.Function):
    """raw parameters -> padded un-clamped image, replacing splatter.py:513-634's glue.

    `rctx` is a `gaussian.RenderContext` (owns device workspaces; holds the state of
    the latest forward, so backward must run before the next forward on the same ctx).
    """

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                near, tile_thresh, scale_activation):
        params = _params(pos, rgb, opa, quat, scale)
        image, mask = rctx.forward(*params, int(width), int(height), float(focal_x), float(focal_y),
                                   rot.detach().cpu(), tran.detach().cpu(), float(near), float(tile_thresh),
                                   SCALE_ACTIVATIONS[scale_activation])
        _save_frame(ctx, rctx, mask, params + (image,))
        return image, mask

    @staticmethod
    def backward(ctx, grad_image, _grad_mask):
        *params, image = ctx.saved_tensors
        outs = _param_grads(ctx.rctx, params)
        ctx.rctx.backward_into(*params, image, _f32(grad_image), *outs, ctx.frame)
        return (None, *outs) + (None,) * 9


render_frame = _RenderFrame.apply


class _RenderFrameFinal(torch.autograd.Function):
    """Like `render_frame`, with reference splatter.py:652-653 (clamp to [0,1] + centre crop)
    fused into the blend kernels: returns the final HxWx3 image; backward consumes its gradient
    directly (no clamp / pad kernels, no padded gradient image)."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                near, tile_thresh, scale_activation):
        params = _params(pos, rgb, opa, quat, scale)
        final, raw, mask = rctx.forward_final(*params, int(width), int(height), float(focal_x), float(focal_y),
                                              rot.detach().cpu(), tran.detach().cpu(), float(near),
                                              float(tile_thresh), SCALE_ACTIVATIONS[scale_activation])
        _save_frame(ctx, rctx, mask, params + (raw,))
        return final, mask

    @staticmethod
    def backward(ctx, grad_final, _grad_mask):
        *params, raw = ctx.saved_tensors
        outs = _param_grads(ctx.rctx, params)
        ctx.rctx.backward_final_into(*params, raw, _f32(grad_final), *outs, ctx.frame)
        return (None, *outs) + (None,) * 9


render_frame_final = _RenderFrameFinal.apply


class _RenderFrameAux(torch.autograd.Function):
    """`render_frame_final` (final=True) or `render_frame` (final=False) over a constant background colour, plus
    the per-pixel depth sum_i w_i |p_c,i| (accumulated, not normalised; Euclidean distance, not camera z) and
    alpha 1 - T_f.  All three outputs are differentiable; a graph that never uses depth or alpha passes no
    gradient for them and runs the plain backward kernels."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                near, tile_thresh, scale_activation, background, final):
        params = _params(pos, rgb, opa, quat, scale)
        bg = None if background is None else [float(v) for v in background]
        fin, raw, aux, aux_fin, mask = rctx.forward_aux(
            *params, int(width), int(height), float(focal_x), float(focal_y), rot.detach().cpu(),
            tran.detach().cpu(), float(near), float(tile_thresh), SCALE_ACTIVATIONS[scale_activation], bg,
            bool(final))
        image, maps = (fin, aux_fin) if final else (raw, aux)
        _save_frame(ctx, rctx, mask, params + (raw, aux), final, maps.shape[:2])
        return image, maps[..., 0].contiguous(), maps[..., 1].contiguous(), mask

    @staticmethod
    def backward(ctx, grad_image, grad_depth, grad_alpha, _grad_mask):
        outs, _ = _RenderFrameAux.backward_with(ctx, grad_image, grad_depth, grad_alpha, cam=False)
        return (None, *outs) + (None,) * 11

    @staticmethod
    def backward_with(ctx, grad_image, grad_depth, grad_alpha, cam):
        """-> (the five parameter gradients, grad_cam[12] or None).  cam: through backward_cam_into, camera only
        (parameter gradients None) when none of the five parameters needs a gradient."""
        *params, raw, aux = ctx.saved_tensors
        grad_image, grad_aux = _upstream(raw, ctx.map_shape, grad_image, grad_depth, grad_alpha)
        if cam and not any(ctx.needs_input_grad[1:6]):          # tracking: the scene is frozen, camera only
            outs = [None] * 5
            _apply_push(ctx.rctx, None)
        else:
            outs = _param_grads(ctx.rctx, params)
        args = (*params, raw, grad_image, ctx.final, aux, grad_aux, *outs)
        if not cam:
            ctx.rctx.backward_aux_into(*args, ctx.frame)
            return outs, None
        grad_cam = raw.new_empty(12)
        ctx.rctx.backward_cam_into(*args, grad_cam, ctx.frame)
        return outs, grad_cam


def render_frame_aux(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran, near,
                     tile_thresh, scale_activation, background=None, final=True):
    """-> (image, depth, alpha, culling_mask).  final=True: image [H,W,3] clamped + cropped as in
    `render_frame_final`, depth / alpha [H,W] (not clamped); final=False: the padded un-clamped image
    [Hp,Wp,3] and [Hp,Wp] maps.  background: 3 floats (None = black, the reference); per pixel
    image = sum_i w_i c_i + T_f background, depth = sum_i w_i |p_c,i|, alpha = 1 - T_f.  RGB and per-pixel SH
    colour on the default kernels."""
    return _RenderFrameAux.apply(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                                 near, tile_thresh, scale_activation, background, final)


SURFEL_MAPS = ("alpha", "depth", "median", "distortion", "normal")


class _RenderFrameSurfel(torch.autograd.Function):
    """2D Gaussian surfels (gs_render_forward_surfel): the five parameters rendered as flat disks evaluated at the
    ray-disk intersection.  Outputs: the image (final: clamped + cropped [H,W,3]; else padded, un-clamped), and with
    maps the alpha, depth (sum w z, camera z), median depth, distortion and camera-frame normal (sum w n) maps, then
    the culling mask.  Every map is differentiable; maps no loss uses pass no gradient."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                near, tile_thresh, scale_activation, background, final, maps, dist_near, dist_far):
        params = _params(pos, rgb, opa, quat, scale)
        bg = None if background is None else [float(v) for v in background]
        fin, raw, m, m_fin, mask = rctx.forward_surfel(
            *params, int(width), int(height), float(focal_x), float(focal_y), rot.detach().cpu(),
            tran.detach().cpu(), float(near), float(tile_thresh), SCALE_ACTIVATIONS[scale_activation], bg,
            bool(maps), bool(final), float(dist_near), float(dist_far))
        image = fin if final else raw
        _save_frame(ctx, rctx, mask, params + (raw,), final, image.shape[:2])
        ctx.maps = bool(maps)
        if not maps:
            return image, mask
        mp = m_fin if final else m
        return (image, mp[..., 0].contiguous(), mp[..., 1].contiguous(), mp[..., 2].contiguous(),
                mp[..., 3].contiguous(), mp[..., 4:7].contiguous(), mask)

    @staticmethod
    def backward(ctx, grad_image, *grads):
        *params, raw = ctx.saved_tensors
        shape = ctx.map_shape
        if grad_image is None:
            grad_image = raw.new_zeros(*shape, 3)
        grad_maps = None
        gm = grads[:-1]                                           # the last is the mask's
        if ctx.maps and any(g is not None for g in gm):
            grad_maps = raw.new_zeros(*shape, 8)
            for k, g in enumerate(gm[:4]):
                if g is not None:
                    grad_maps[..., k] = g
            if gm[4] is not None:
                grad_maps[..., 4:7] = gm[4]
        outs, push = _flat_grads(params)
        if push is not None:
            raise RuntimeError("render_frame_surfel: surfel frames have no data-parallel gradient push; exchange the "
                               "gradients with an all-reduce (dp.py's NCCL bucket) instead")
        _apply_push(ctx.rctx, None)
        ctx.rctx.backward_surfel_into(*params, raw, _f32(grad_image), ctx.final, grad_maps, *outs, ctx.frame)
        return (None, *outs) + (None,) * 14


def render_frame_surfel(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran, near,
                        tile_thresh, scale_activation, background=None, final=True, maps=True, dist_near=0.2,
                        dist_far=100.0):
    """-> (image, maps, culling_mask) of a frame of 2D Gaussian surfels (include/gs_b200.h, gs_render_forward_surfel).
    maps: {} without maps, else {"alpha", "depth", "median", "distortion": [rows, cols], "normal": [rows, cols, 3]}
    over the same pixels as the image (final: the [H,W] crop, not clamped; else [Hp,Wp]).  depth is accumulated
    (expected depth = depth / alpha); the normal is in the camera frame (world: rot^T n).  Only scale[:, :2] is used.
    Per-Gaussian SH colour (d = 27 / 48) needs rctx.set_sh_eval(SH_EVAL_GAUSSIAN)."""
    out = _RenderFrameSurfel.apply(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                                   near, tile_thresh, scale_activation, background, final, maps, dist_near,
                                   dist_far)
    if not maps:
        return out[0], {}, out[1]
    return out[0], dict(zip(SURFEL_MAPS, out[1:6])), out[6]


MAX_VIEWS = 64


class _RenderFrameBatch(torch.autograd.Function):
    """`_RenderFrameAux` over a batch of B views rendered as one frame (gs_render_forward_batch); the backward returns
    the sums over the views of the five parameter gradients."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal, rot, tran, near, tile_thresh,
                scale_activation, background, final):
        params = _params(pos, rgb, opa, quat, scale)
        bg = None if background is None else [float(v) for v in background]
        fin, raw, aux, aux_fin, mask = rctx.forward_batch(
            *params, int(width), int(height), focal, rot, tran, float(near), float(tile_thresh),
            SCALE_ACTIVATIONS[scale_activation], bg, bool(final))
        image, maps = (fin, aux_fin) if final else (raw, aux)
        _save_frame(ctx, rctx, mask, params + (raw, aux), final, maps.shape[:3])
        return image, maps[..., 0].contiguous(), maps[..., 1].contiguous(), mask

    @staticmethod
    def backward(ctx, grad_image, grad_depth, grad_alpha, _grad_mask):
        *params, raw, aux = ctx.saved_tensors
        grad_image, grad_aux = _upstream(raw, ctx.map_shape, grad_image, grad_depth, grad_alpha)
        outs, _ = _flat_grads(params)
        ctx.rctx.backward_batch_into(*params, raw, grad_image, ctx.final, aux, grad_aux, *outs, ctx.frame)
        return (None, *outs) + (None,) * 10


def render_frame_batch(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran, near,
                       tile_thresh, scale_activation, background=None, final=True):
    """B camera views of one scene rendered as one frame: -> (image, depth, alpha, culling_mask) with image
    [B,H,W,3] (final=True, each view clamped and cropped as in `render_frame_aux`) or [B,Hp,Wp,3], depth / alpha
    [B,H,W] or [B,Hp,Wp], culling_mask [B,n].  Per view the outputs are those of `render_frame_aux` with that view's
    camera; the views share width, height, near, tile_thresh and the background.  focal_x / focal_y: B numbers;
    rot [B,3,3], tran [B,3] (any device: they are read on the host).  Differentiable in the five parameters: their
    gradients are the SUMS over the views (divide the loss by B for a mean).  RGB and per-Gaussian SH colour, any 2-D
    filter, densification statistics; per-pixel SH, the packed path, non-default blend knobs and a data-parallel
    gradient push raise RuntimeError.  A graph that never uses depth or alpha runs the plain backward kernels."""
    rot = torch.as_tensor(rot).detach()
    tran = torch.as_tensor(tran).detach()
    if rot.dim() != 3 or tuple(rot.shape[1:]) != (3, 3):
        raise ValueError(f"render_frame_batch: rot must be [B,3,3], got {list(rot.shape)}")
    b = rot.shape[0]
    if not 1 <= b <= MAX_VIEWS:
        raise ValueError(f"render_frame_batch: the batch must have 1 .. {MAX_VIEWS} views, got {b}")
    if tuple(tran.shape) != (b, 3):
        raise ValueError(f"render_frame_batch: tran must be [{b},3], got {list(tran.shape)}")
    fx, fy = (torch.as_tensor(f, dtype=torch.float64).detach().reshape(-1).cpu() for f in (focal_x, focal_y))
    if fx.numel() != b or fy.numel() != b:
        raise ValueError(f"render_frame_batch: focal_x and focal_y must have {b} values each")
    return _RenderFrameBatch.apply(rctx, pos, rgb, opa, quat, scale, width, height, torch.stack([fx, fy], 1),
                                   rot.float().cpu(),
                                   tran.float().cpu(), near, tile_thresh, scale_activation, background, final)


class _RenderFrameCam(_RenderFrameAux):
    """`_RenderFrameAux` whose backward also returns dL/drot and dL/dtran (gs_render_backward_cam)."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                near, tile_thresh, scale_activation, background, final):
        cam = torch.cat([rot.detach().reshape(9), tran.detach().reshape(3)]).cpu()   # one 48-byte host read
        return _RenderFrameAux.forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y,
                                       cam[:9].view(3, 3), cam[9:], near, tile_thresh, scale_activation, background,
                                       final)

    @staticmethod
    def backward(ctx, grad_image, grad_depth, grad_alpha, _grad_mask):
        if not (ctx.needs_input_grad[10] or ctx.needs_input_grad[11]):
            return _RenderFrameAux.backward(ctx, grad_image, grad_depth, grad_alpha, _grad_mask)
        outs, grad_cam = _RenderFrameAux.backward_with(ctx, grad_image, grad_depth, grad_alpha, cam=True)
        return (None, *outs) + (None,) * 4 + (grad_cam[:9].view(3, 3), grad_cam[9:]) + (None,) * 5


def render_frame_cam(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran, near,
                     tile_thresh, scale_activation, background=None, final=True):
    """`render_frame_aux` differentiable with respect to the camera too: -> (image, depth, alpha, culling_mask), and
    the backward returns dL/drot and dL/dtran for p_c = rot p + tran (rot used as given, not re-orthonormalised;
    map them to your own pose parameterisation in torch).  rot [3,3] and tran [3] must be float32 CUDA tensors on the
    parameters' device (ValueError otherwise); reading them for the forward costs one extra host synchronisation
    (12 floats).  When none of the five parameters needs a gradient the backward is camera only (pose tracking
    against a frozen scene).  RGB and per-Gaussian SH colour (RenderContext.set_sh_eval(SH_EVAL["gaussian"]));
    a per-pixel SH frame or a data-parallel gradient push is refused by the backward (RuntimeError)."""
    for name, t, shape in (("rot", rot, (3, 3)), ("tran", tran, (3,))):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or tuple(t.shape) != shape:
            raise ValueError(f"render_frame_cam: {name} must be a float32 CUDA tensor of shape {list(shape)}")
        if t.device != pos.device:
            raise ValueError(f"render_frame_cam: {name} is on {t.device}, the parameters on {pos.device}")
    return _RenderFrameCam.apply(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran,
                                 near, tile_thresh, scale_activation, background, final)


class _RenderFrameBatchCam(_RenderFrameBatch):
    """`_RenderFrameBatch` whose backward also returns each view's dL/drot and dL/dtran
    (gs_render_backward_batch_cam)."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal, rot, tran, near, tile_thresh,
                scale_activation, background, final):
        b = rot.shape[0]
        cams = torch.cat([rot.detach().reshape(b, 9), tran.detach().reshape(b, 3)], 1).cpu()   # one 48 B-byte read
        return _RenderFrameBatch.forward(ctx, rctx, pos, rgb, opa, quat, scale, width, height, focal,
                                         cams[:, :9].reshape(b, 3, 3), cams[:, 9:].contiguous(), near, tile_thresh,
                                         scale_activation, background, final)

    @staticmethod
    def backward(ctx, grad_image, grad_depth, grad_alpha, _grad_mask):
        if not (ctx.needs_input_grad[9] or ctx.needs_input_grad[10]):
            return _RenderFrameBatch.backward(ctx, grad_image, grad_depth, grad_alpha, _grad_mask)
        *params, raw, aux = ctx.saved_tensors
        grad_image, grad_aux = _upstream(raw, ctx.map_shape, grad_image, grad_depth, grad_alpha)
        if not any(ctx.needs_input_grad[1:6]):                  # tracking: the scene is frozen, camera only
            outs = [None] * 5
            _apply_push(ctx.rctx, None)
        else:
            outs = _param_grads(ctx.rctx, params)
        grad_cams = raw.new_empty(ctx.map_shape[0], 12)
        ctx.rctx.backward_batch_cam_into(*params, raw, grad_image, ctx.final, aux, grad_aux, *outs, grad_cams,
                                         ctx.frame)
        return ((None, *outs) + (None,) * 3 + (grad_cams[:, :9].reshape(-1, 3, 3), grad_cams[:, 9:]) +
                (None,) * 5)


def render_frame_batch_cam(rctx, pos, rgb, opa, quat, scale, width, height, focal_x, focal_y, rot, tran, near,
                           tile_thresh, scale_activation, background=None, final=True):
    """`render_frame_batch` differentiable with respect to each view's camera too: -> (image, depth, alpha,
    culling_mask) as `render_frame_batch` returns them, and the backward returns dL/drot [B,3,3] and dL/dtran [B,3],
    per view what `render_frame_cam` returns for that view (p_c = rot[v] p + tran[v], rot used as given).  rot
    [B,3,3] and tran [B,3] (1 <= B <= 64) must be float32 CUDA tensors on the parameters' device (ValueError
    otherwise); reading them for the forward costs one host synchronisation (48 B bytes).  The parameter gradients are
    the sums over the views, as in `render_frame_batch`.  When none of the five parameters needs a gradient the
    backward is camera only (the densification statistics are then left alone); when neither rot nor tran needs one it
    is `render_frame_batch`'s.  RGB and per-Gaussian SH colour; per-pixel SH, the packed path, non-default blend knobs
    and a data-parallel gradient push raise RuntimeError."""
    for name, t, dims in (("rot", rot, 3), ("tran", tran, 2)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != dims:
            raise ValueError(f"render_frame_batch_cam: {name} must be a float32 CUDA tensor of {dims} dimensions")
        if t.device != pos.device:
            raise ValueError(f"render_frame_batch_cam: {name} is on {t.device}, the parameters on {pos.device}")
    b = rot.shape[0]
    if tuple(rot.shape[1:]) != (3, 3) or tuple(tran.shape) != (b, 3):
        raise ValueError(f"render_frame_batch_cam: rot must be [B,3,3] and tran [B,3], got {list(rot.shape)} and "
                         f"{list(tran.shape)}")
    if not 1 <= b <= MAX_VIEWS:
        raise ValueError(f"render_frame_batch_cam: the batch must have 1 .. {MAX_VIEWS} views, got {b}")
    fx, fy = (torch.as_tensor(f, dtype=torch.float64).detach().reshape(-1).cpu() for f in (focal_x, focal_y))
    if fx.numel() != b or fy.numel() != b:
        raise ValueError(f"render_frame_batch_cam: focal_x and focal_y must have {b} values each")
    return _RenderFrameBatchCam.apply(rctx, pos, rgb, opa, quat, scale, width, height, torch.stack([fx, fy], 1), rot,
                                      tran, near, tile_thresh, scale_activation, background, final)


FEATURE_WIDTHS = (8, 16, 32)


class _RenderFrameFeat(torch.autograd.Function):
    """`_RenderFrameAux` that also blends per-Gaussian feature rows feat[n, F] into an [.., .., F] map with the image's
    weights (gs_render_forward_feat / gs_render_backward_feat)."""

    @staticmethod
    def forward(ctx, rctx, pos, rgb, opa, quat, scale, feat, width, height, focal_x, focal_y, rot, tran,
                near, tile_thresh, scale_activation, background, final):
        *params, feat = _params(pos, rgb, opa, quat, scale, feat)
        bg = None if background is None else [float(v) for v in background]
        fin, raw, aux, aux_fin, fmap, fmap_fin, mask = rctx.forward_feat(
            *params, feat, int(width), int(height), float(focal_x), float(focal_y), rot.detach().cpu(),
            tran.detach().cpu(), float(near), float(tile_thresh), SCALE_ACTIVATIONS[scale_activation], bg, bool(final))
        image, maps, feats = (fin, aux_fin, fmap_fin) if final else (raw, aux, fmap)
        _save_frame(ctx, rctx, mask, (*params, feat, raw, aux, fmap), final, maps.shape[:2])
        return image, feats, maps[..., 0].contiguous(), maps[..., 1].contiguous(), mask

    @staticmethod
    def backward(ctx, grad_image, grad_feat, grad_depth, grad_alpha, _grad_mask):
        *params, feat, raw, aux, fmap = ctx.saved_tensors
        grad_image, grad_aux = _upstream(raw, ctx.map_shape, grad_image, grad_depth, grad_alpha)
        outs = _param_grads(ctx.rctx, params)
        g_feat = torch.empty_like(feat)
        if grad_feat is not None:
            grad_feat = _f32(grad_feat)
            if grad_feat.data_ptr() % 16:                      # the kernel reads 16-byte pieces of every pixel's row
                grad_feat = grad_feat.clone()
        ctx.rctx.backward_feat_into(*params, feat, raw, grad_image, ctx.final, aux, grad_aux, fmap, grad_feat, *outs,
                                    g_feat, ctx.frame)
        return (None, *outs, g_feat) + (None,) * 11


def render_frame_feat(rctx, pos, rgb, opa, quat, scale, feat, width, height, focal_x, focal_y, rot, tran, near,
                      tile_thresh, scale_activation, background=None, final=True):
    """`render_frame_aux` plus a feature map: -> (image, features, depth, alpha, culling_mask).  feat [n, F] holds raw
    float32 per-Gaussian features (F = 8, 16 or 32; pad another width with zero channels), blended per pixel as
    features_k = sum_i w_i f_i,k with the image's weights, composited over zero (the background applies to the image
    only; the expected feature is features / alpha) and not clamped: [H,W,F] (final=True, the centre crop) or
    [Hp,Wp,F].  Image, depth and alpha are bit-identical to `render_frame_aux`'s.  Differentiable in the five
    parameters and feat; a graph that never uses `features` runs the plain / aux backward kernels and gets a zero
    feat gradient.  RGB and per-Gaussian SH colour on the default (gather) path, any 2-D filter; per-pixel SH, the
    packed path, and (with a feature gradient) absgrad statistics or a data-parallel gradient push raise RuntimeError."""
    return _RenderFrameFeat.apply(rctx, pos, rgb, opa, quat, scale, feat, width, height, focal_x, focal_y, rot, tran,
                                  near, tile_thresh, scale_activation, background, final)
