"""Scene + per-frame pipeline: host-side mirror of the reference's `Splatter`
(reference splatter.py:323-655) on top of the fused frame path.

Same constructor as the reference (`Splatter(colmap_path, image_path, near=..., ...)`,
splatter.py:324-345) and the surface train.py / visergui.py touch (train.py:57-61,:67,:99,:150,
:161-171,:190,:198-199,:234; visergui.py:137-149): `gaussian_3ds.{pos,rgb,opa,quat,scale}`
(nn.Parameters; opa / rgb logits, wxyz quaternion, raw scale), `gaussian_3ds.adaptive_control`,
`reset_opa`, `forward(camera_id, extrinsics, intrinsics)` -> clamped, centre-cropped HxWx3 image,
`ground_truth`, `imgs`, `culling_mask` (int64), `n_tile_gaussians`, `n_gaussians`, `device`,
`scale_activation`, `set_camera`, `switch_resolution`.  Additionally
`Splatter.from_tensors(gaussians, views, ...)` builds a scene without COLMAP (synthetic
benchmarks / tests).

The per-frame work of reference `project_and_culling` + `render` (:513-634: 4 boolean-mask
compactions, the dense [T, N/20] list, cumsum, two 4-tensor gathers, fp32-key sort, >= 7 host
syncs) and the clamp + crop of `forward` (:652-653) is ONE autograd node here
(`renderer.render_frame_final`).
"""
from __future__ import annotations

import math
import os
import weakref
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

import gaussian
from renderer import (FEATURE_WIDTHS, FILTER2D, SH_EVAL, render_frame, render_frame_aux, render_frame_batch,
                      render_frame_batch_cam, render_frame_cam, render_frame_feat, render_frame_final,
                      render_frame_surfel)

EPS = 1e-4
SH_C0 = 0.28209479177387814


def inverse_sigmoid(y):
    return -math.log(1 / y - 1)


def quat_to_rotmat(q):
    """wxyz -> R (reference utils.py:318-333)."""
    w, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w,
                        2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w,
                        2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y],
                       dim=-1).reshape(q.shape[:-1] + (3, 3))


class Gaussian3ds(nn.Module):
    """Parameter holder + densification (reference splatter.py:39-228, init_values=True branch).  `feat`: optional
    per-Gaussian feature rows [n, F] (`Splatter(..., n_features=F)`), None without features."""

    def __init__(self, pos, rgb, opa, quat, scale, feat=None):
        super().__init__()
        self.pos = nn.Parameter(pos)
        self.rgb = nn.Parameter(rgb)
        self.opa = nn.Parameter(opa)
        self.quat = nn.Parameter(quat)
        self.scale = nn.Parameter(scale)
        self.feat = None if feat is None else nn.Parameter(feat)

    def reset_opa(self):                                        # reference splatter.py:119-120
        with torch.no_grad():
            self.opa.fill_(inverse_sigmoid(0.01))

    def get_gaussian_3d_cov(self, scale_activation="abs"):      # reference splatter.py:100-114
        R = quat_to_rotmat(self.quat)
        s = self.scale.abs() + EPS if scale_activation == "abs" else torch.exp(self.scale)
        RS = R * s.unsqueeze(-2)
        return RS @ RS.transpose(-1, -2)

    @torch.no_grad()
    def adaptive_control(self, grad, taus, delete_thresh, scale_activation="abs", grad_thresh=0.0002,
                         grad_aggregation="max", use_clone=True, use_split=True, clone_dt=0.01, generator=None):
        """Prune / clone / split (reference splatter.py:122-228, same signature as train.py:160-171 calls it):
        delete Gaussians with opacity below sigmoid^-1(0.02) or a scale norm above `delete_thresh`; where the
        accumulated position gradient exceeds `grad_thresh`, clone the small ones (moved against the gradient)
        and split the large ones (scale / 1.6, two positions sampled from the un-shrunk Gaussian itself).
        Runs on the device (`gaussian.densify`: classify -> scans -> one kernel that writes the new arrays);
        the split samples come from torch's CUDA generator, so data-parallel replicas that seed torch
        identically stay identical.  Parameters are re-created: the caller rebuilds its optimizer
        (train.py:173-181)."""
        if scale_activation not in ("abs", "exp"):
            raise ValueError("scale_activation must be 'abs' or 'exp'")
        if grad_aggregation not in ("max", "mean"):
            raise ValueError("grad_aggregation must be 'max' or 'mean'")
        g = grad.detach()
        if g.dtype != torch.float32 or not g.is_contiguous():
            g = g.float().contiguous()
        args = [t.detach().contiguous() for t in (self.pos, self.rgb, self.opa, self.quat, self.scale)]
        new, (n_deleted, n_clone, n_split) = gaussian.densify(
            *args, g, 0 if scale_activation == "abs" else 1, inverse_sigmoid(0.02), float(delete_thresh),
            float(grad_thresh), grad_aggregation == "max", float(taus), bool(use_clone), bool(use_split),
            float(clone_dt), generator, self._feat_arg())
        self._replace(new)
        return dict(deleted=int(n_deleted), cloned=int(n_clone), split=int(n_split), total=self.pos.shape[0])

    def _feat_arg(self):
        return None if self.feat is None else self.feat.detach().contiguous()

    def _replace(self, new):
        """New parameters from a densification: the five, then the feature rows laid out by the same plan."""
        self.pos, self.rgb, self.opa, self.quat, self.scale = (nn.Parameter(t) for t in new[:5])
        if self.feat is not None:
            self.feat = nn.Parameter(new[5])


DENSIFY_STATS = ("none", "grad", "absgrad")


class DensifyStats:
    """Screen-space densification statistics of the Gaussians, accumulated on the device by every backward of the
    fused frame path while they are registered with a `RenderContext` (`gaussian.RenderContext.set_densify_stats`):

    - `grad2d[n]`: sum over views of |dL/d(mean2d)| in the NDC units of 3DGS's `viewspace_points.grad`;
    - `absgrad[n]` (or None): the same with the absolute value of every pixel's contribution taken before summing
      (AbsGS; gsplat's `absgrad=True`);
    - `count[n]` (int32): the views in which the Gaussian was binned into at least one tile;
    - `max_radius[n]`: its largest screen radius in pixels, ceil(3 sqrt(lambda_max)).

    The score 3DGS compares with its threshold (0.0002) is `grad2d / count.clamp(min=1)`."""

    def __init__(self, n, absgrad=False, device=None, rctx=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.with_absgrad = bool(absgrad)
        self._rctx = rctx
        self.grad2d = self.absgrad = self.count = self.max_radius = None
        self.reset(n)

    @property
    def n(self):
        return self.grad2d.numel()

    def reset(self, n):
        """Zero the statistics, sized for n Gaussians (re-registered with the context when n changes)."""
        n = int(n)
        if self.grad2d is not None and self.n == n:
            for t in (self.grad2d, self.absgrad, self.count, self.max_radius):
                if t is not None:
                    t.zero_()
            return
        f = dict(device=self.device, dtype=torch.float32)
        self.grad2d = torch.zeros(n, **f)
        self.absgrad = torch.zeros(n, **f) if self.with_absgrad else None
        self.count = torch.zeros(n, device=self.device, dtype=torch.int32)
        self.max_radius = torch.zeros(n, **f)
        if self._rctx is not None:
            self._rctx.set_densify_stats(self.grad2d, self.count, self.max_radius, self.absgrad)

    def all_reduce(self, group=None):
        """Combine the statistics of all ranks of `group` (sums, and the max of max_radius).  Under data parallel
        every rank renders other views: call this on every rank before densifying."""
        import torch.distributed as dist
        for t in (self.grad2d, self.absgrad, self.count):
            if t is not None:
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.max_radius, op=dist.ReduceOp.MAX, group=group)


class ContributionScores:
    """Per-Gaussian blend-weight scores of the fused frame path, accumulated on the device by
    `Splatter.score_views` / `Splatter.accumulate_scores` (`gaussian.RenderContext.scores_into`, gs_frame_scores):

    - `weight_sum[n]`: the sum over the scored frames' pixels of w = alpha T, the weight each pixel blended the
      Gaussian's colour with (LightGaussian's and Mini-Splatting's importance);
    - `weight_max[n]`: its largest w on any scored pixel (RadSplat's score).

    Only pixels inside the rendered images count.  A Gaussian no scored frame binned keeps 0 in both."""

    def __init__(self, n, device=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.weight_sum = self.weight_max = None
        self.reset(n)

    @property
    def n(self):
        return self.weight_sum.numel()

    def reset(self, n):
        """Zero the scores, sized for n Gaussians."""
        n = int(n)
        if self.weight_sum is not None and self.n == n:
            self.weight_sum.zero_()
            self.weight_max.zero_()
            return
        self.weight_sum = torch.zeros(n, device=self.device, dtype=torch.float32)
        self.weight_max = torch.zeros(n, device=self.device, dtype=torch.float32)

    def all_reduce(self, group=None):
        """Combine the scores of all ranks of `group`: the sum of weight_sum, the max of weight_max.  Under data
        parallel every rank scores other views: call this on every rank before selecting."""
        import torch.distributed as dist
        dist.all_reduce(self.weight_sum, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.weight_max, op=dist.ReduceOp.MAX, group=group)


def _check_features(n_features, use_sh_coeff, sh_eval, densify_stats):
    if n_features != 0 and n_features not in FEATURE_WIDTHS:
        raise ValueError(f"n_features must be 0 or one of {FEATURE_WIDTHS} (pad with zero channels), not {n_features!r}")
    if n_features and use_sh_coeff and sh_eval == "pixel":
        raise ValueError("features need the RGB blend: RGB colour or sh_eval='gaussian', not per-pixel SH")
    if n_features and densify_stats == "absgrad":
        raise ValueError("features are not available with densify_stats='absgrad' (use 'grad')")


def _zero_moment_rows(optimizer, params, rows):
    """Zero the Adam moments of rows `rows` (CUDA bool [n]) of `params`: `torch.optim.Adam`'s per-parameter state, or
    `optim.FlatAdam`'s moments that are not in a live flat buffer (`FlatAdam.zero_moment_rows`).  masked_fill_ writes
    exact zeros and leaves other bits alone."""
    import optim
    if isinstance(optimizer, optim.FlatAdam):
        optimizer.zero_moment_rows(rows)
        return
    for p in params:
        for t in optimizer.state.get(p, {}).values():
            if torch.is_tensor(t) and t.dim() > 0 and t.shape[0] == rows.numel():
                t.masked_fill_(rows.view((-1,) + (1,) * (t.dim() - 1)), 0.0)


def _regrow_optimizer(optimizer, pairs, keep=None):
    """Re-point an optimizer from the old Parameters to the new ones (`pairs` = [(old, new)]): grown ones (the old rows
    first), or with `keep` (bool [n_old]) the old rows keep[i] selects, in order.  `optim.FlatAdam` stages its moments
    (`replace_params`); `torch.optim.Adam`'s per-parameter state is re-keyed and its row tensors padded with zero rows
    or row-selected."""
    import optim
    if isinstance(optimizer, optim.FlatAdam):
        optimizer.replace_params(pairs, keep=keep)
        return
    for old, new in pairs:
        st = optimizer.state.pop(old, None)
        if st is not None:
            for k, t in list(st.items()):
                if torch.is_tensor(t) and t.dim() > 0 and t.shape[0] == old.shape[0]:
                    if keep is not None:
                        st[k] = t[keep]
                    else:
                        st[k] = torch.cat([t, t.new_zeros((new.shape[0] - old.shape[0],) + tuple(t.shape[1:]))])
            optimizer.state[new] = st
    for grp in optimizer.param_groups:
        grp["params"] = [next((nw for od, nw in pairs if od is p), p) for p in grp["params"]]


# what a frame rendered through a Splatter leaves on it (set_camera and the frame entry points)
_FRAME_ATTRS = ("culling_mask", "n_tile_gaussians", "current_view", "current_camera", "current_w2c_rot",
                "current_w2c_tran", "tile_info", "ground_truth")


class Tiles:
    """Padded render-target geometry (reference splatter.py:255-272)."""

    def __init__(self, width, height, focal_x, focal_y):
        self.width, self.height = int(width), int(height)
        self.padded_width = int(math.ceil(self.width / 16)) * 16
        self.padded_height = int(math.ceil(self.height / 16)) * 16
        self.focal_x, self.focal_y = float(focal_x), float(focal_y)
        self.n_tile_x = self.padded_width // 16
        self.n_tile_y = self.padded_height // 16

    def __len__(self):
        return self.n_tile_x * self.n_tile_y

    def crop(self, image):
        top = (self.padded_height - self.height) // 2
        left = (self.padded_width - self.width) // 2
        return image[top:top + self.height, left:left + self.width, :]


CAMERA_MODELS = ("reference", "colmap")
PRIMITIVES = ("gaussian", "surfel")
# COLMAP camera models the fused path renders: name -> (lens model, focal params, cx/cy index, distortion mapping)
_COLMAP_LENSES = {
    "SIMPLE_PINHOLE": ("PINHOLE", 1, 1, ()),
    "PINHOLE": ("PINHOLE", 2, 2, ()),
    "SIMPLE_RADIAL": ("OPENCV", 1, 1, (3,)),            # k -> k1; k2 = p1 = p2 = 0
    "RADIAL": ("OPENCV", 1, 1, (3, 4)),
    "OPENCV": ("OPENCV", 2, 2, (4, 5, 6, 7)),
    "OPENCV_FISHEYE": ("FISHEYE", 2, 2, (4, 5, 6, 7)),
    "SIMPLE_RADIAL_FISHEYE": ("FISHEYE", 1, 1, (3,)),   # the missing k are 0
    "RADIAL_FISHEYE": ("FISHEYE", 1, 1, (3, 4)),
}
LENS_MODELS = {"PINHOLE": gaussian.LENS_PINHOLE, "OPENCV": gaussian.LENS_OPENCV, "FISHEYE": gaussian.LENS_FISHEYE}


def colmap_intrinsics(model, params, downsample=1):
    """(focal_x, focal_y, lens) of a COLMAP camera at 1 / `downsample` resolution, lens = dict(model="PINHOLE" |
    "OPENCV" | "FISHEYE", cx, cy, k=[4]) for `Splatter(camera_model="colmap")`.  Focal lengths and the principal
    point scale with the resolution; the distortion coefficients do not.  ValueError for a model the fused path does
    not render (FULL_OPENCV, FOV, THIN_PRISM_FISHEYE)."""
    if model not in _COLMAP_LENSES:
        raise ValueError(f"COLMAP camera model {model} is not supported (supported: {sorted(_COLMAP_LENSES)})")
    lens_model, nf, ic, ik = _COLMAP_LENSES[model]
    fx = float(params[0]) / downsample
    fy = float(params[nf - 1]) / downsample
    k = [float(params[j]) for j in ik] + [0.0] * (4 - len(ik))
    return fx, fy, dict(model=lens_model, cx=float(params[ic]) / downsample, cy=float(params[ic + 1]) / downsample,
                        k=k)


class Splatter(nn.Module):
    def __init__(self, colmap_path, image_path, near=0.3, jacobian_calc="cuda", render_downsample=1,
                 use_sh_coeff=False, render_weight_normalize=False, opa_init_value=0.1, scale_init_value=0.02,
                 tile_culling_method="prob2", tile_culling_dist_thresh=0.5, tile_culling_prob_thresh=0.1,
                 debug=0, scale_activation="abs", cudaculling=1, load_ckpt=None, debug_align=False,
                 fast_drawing=True, test=False, images: Optional[List[torch.Tensor]] = None, device=None, *,
                 sh_eval="pixel", filter2d="none", filter2d_variance=0.3, densify_stats="none", n_features=0,
                 filter3d=False, filter3d_variance=0.2, camera_model="reference", primitive="gaussian"):
        """Reference signature (splatter.py:324-345).  `colmap_path` may also be a dict of raw
        parameter tensors (pos, rgb, opa, quat, scale) with `image_path` a list of view dicts
        (width, height, focal_x, focal_y, rot[3,3], tran[3]) - see `from_tensors`.

        Options that selected slower variants of the same maths in the reference are accepted and
        ignored (`jacobian_calc`, `cudaculling`, `fast_drawing`, `debug`, `debug_align`); options
        whose result would differ are refused (`render_weight_normalize`, tile culling methods other
        than "prob2", which is train.py's default, train.py:311).

        `sh_eval` (SH colour only): "pixel" evaluates the SH basis per pixel ray, as the reference does;
        "gaussian" evaluates it once per Gaussian along the direction from the camera centre to its mean and
        blends the result as an RGB colour (the usual 3D Gaussian Splatting model, and a much cheaper frame).
        The two modes use the same coefficient tensor but render it differently.

        `filter2d`: screen-space low-pass filter of the projected Gaussians, for scenes rendered at more than one
        resolution.  "none" (default, the reference); "dilate" adds `filter2d_variance` px^2 to every 2-D covariance
        (the original 3D Gaussian Splatting rasterizer, 0.3); "antialias" dilates and scales the opacity by
        sqrt(det / det'), keeping each Gaussian's screen-space integral (Mip-Splatting's 2-D filter, gsplat's
        "antialiased").  Every frame of this Splatter follows it, with gradients.  A scene renders differently under
        another mode: train and render with the same one.

        `filter3d`: Mip-Splatting's 3-D smoothing filter (default off, the reference).  Each Gaussian's scale is
        bounded from below by the finest sampling interval the training views have at it, s' = sqrt(s^2 + f^2) with
        f = sqrt(`filter3d_variance`) z / fx over the view that samples it most finely, and its opacity is scaled by
        prod s / s' (the 3-D integral is kept): no needle-like artefacts when the scene is rendered closer or at a longer
        focal length than it was trained.  The filter lives in `self.filter3d` [n] (a buffer, not a Parameter), is
        computed by `compute_filter3d`, and is recomputed after every densification and whenever the Gaussians were
        replaced; Mip-Splatting also recomputes it every 100 steps (call `compute_filter3d()`).  Densification, MCMC
        noise and regularisers keep using the unfiltered scale and opacity.  Mip-Splatting's configuration:
        filter2d="antialias", filter3d=True, filter3d_variance=0.1 (the default 0.2 is its filter's own default).

        `densify_stats`: "none" (default); "grad" accumulates the screen-space densification statistics of 3D
        Gaussian Splatting in `self.densify_stats` (a `DensifyStats`: view-space gradient norm, view count, largest
        screen radius) during every backward; "absgrad" also the absolute gradient of AbsGS (not available with
        per-pixel SH colour).  `adaptive_control_screen` densifies from them.

        `n_features`: 0 (default) or F = 8, 16, 32 raw per-Gaussian features in `gaussian_3ds.feat` (an nn.Parameter
        [n, F], zero-initialised; `from_tensors` / a checkpoint may provide a "feat" tensor, whose width then sets F),
        blended with the image's weights by `render_features` and carried through densification and checkpoints.
        Not available with per-pixel SH colour, nor with densify_stats="absgrad".

        `camera_model`: "reference" (default) renders every camera as an undistorted pinhole whose principal point is
        the image centre, keeping only the focal lengths of `cameras.bin`, as the reference does.  "colmap" renders
        through each COLMAP camera's own intrinsics (`colmap_intrinsics`): the principal point of PINHOLE and
        SIMPLE_PINHOLE, the radial / tangential distortion of SIMPLE_RADIAL, RADIAL and OPENCV, and the fisheye
        distortion of OPENCV_FISHEYE, SIMPLE_RADIAL_FISHEYE and RADIAL_FISHEYE, with gradients (gs_ctx_set_lens).  The
        view dicts then carry a "lens" (dict(model, cx, cy, k)); view dicts given directly and the free-camera
        `intrinsics` may carry one too (or cx, cy, model, k) under either setting.  FULL_OPENCV, FOV and
        THIN_PRISM_FISHEYE raise a ValueError.  Per-pixel SH colour takes a principal point but no distortion.
        `compute_filter3d` uses the views' lenses (the distorted image for visibility, the fisheye's magnification for
        the rate).

        `primitive`: "gaussian" (default) renders 3-D Gaussians; "surfel" renders each Gaussian as the flat disk of 2D
        Gaussian Splatting (Huang et al. 2024), spanned by its first two scale axes and evaluated where the pixel ray
        meets it (`renderer.render_frame_surfel`).  `forward` then returns the surfel image and `render_surfel_maps`
        the image with alpha, depth, median-depth, distortion and normal maps.  scale[:, 2] is set to the activation's
        floor (raw 0 for "abs", log 1e-4 for "exp") and gets no gradient, so densification and MCMC keep every
        Gaussian flat; checkpoints keep the five-key schema.  Surfels take RGB colour or sh_eval="gaussian", the
        image-centre pinhole ("reference" cameras), and none of the filters, densify_stats or features."""
        super().__init__()
        if camera_model not in CAMERA_MODELS:
            raise ValueError(f"camera_model must be one of {CAMERA_MODELS}, not {camera_model!r}")
        self.camera_model = camera_model
        if primitive not in PRIMITIVES:
            raise ValueError(f"primitive must be one of {PRIMITIVES}, not {primitive!r}")
        if primitive == "surfel":
            if use_sh_coeff and sh_eval != "gaussian":
                raise ValueError("primitive='surfel' with SH colour needs sh_eval='gaussian'")
            for name, value, default in (("filter2d", filter2d, "none"), ("filter3d", bool(filter3d), False),
                                         ("densify_stats", densify_stats, "none"), ("n_features", n_features, 0),
                                         ("camera_model", camera_model, "reference")):
                if value != default:
                    raise ValueError(f"primitive='surfel' does not take {name}={value!r}")
        self.primitive = primitive
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if render_weight_normalize:
            raise NotImplementedError("render_weight_normalize is not supported (the reference never enables it)")
        if tile_culling_method != "prob2":
            raise NotImplementedError("the fused path implements tile_culling_method='prob2' (train.py's default); "
                                      "methods 'dist' / 'prob' are available through gaussian.calc_tile_list")
        if sh_eval not in SH_EVAL:
            raise ValueError(f"sh_eval must be one of {sorted(SH_EVAL)}, not {sh_eval!r}")
        if sh_eval == "gaussian" and not use_sh_coeff:
            raise ValueError("sh_eval='gaussian' needs SH colour (use_sh_coeff=True)")
        if filter2d not in FILTER2D:
            raise ValueError(f"filter2d must be one of {sorted(FILTER2D)}, not {filter2d!r}")
        try:
            filter2d_variance = float(filter2d_variance)
        except (TypeError, ValueError):
            raise ValueError(f"filter2d_variance must be a number, not {filter2d_variance!r}") from None
        if not (math.isfinite(filter2d_variance) and filter2d_variance > 0):
            raise ValueError(f"filter2d_variance must be finite and > 0, not {filter2d_variance!r}")
        try:
            filter3d_variance = float(filter3d_variance)
        except (TypeError, ValueError):
            raise ValueError(f"filter3d_variance must be a number, not {filter3d_variance!r}") from None
        if not (math.isfinite(filter3d_variance) and filter3d_variance > 0):
            raise ValueError(f"filter3d_variance must be finite and > 0, not {filter3d_variance!r}")
        if densify_stats not in DENSIFY_STATS:
            raise ValueError(f"densify_stats must be one of {DENSIFY_STATS}, not {densify_stats!r}")
        if densify_stats == "absgrad" and use_sh_coeff and sh_eval == "pixel":
            raise ValueError("densify_stats='absgrad' needs the RGB blend: RGB colour or sh_eval='gaussian'")
        if isinstance(colmap_path, dict) and colmap_path.get("feat") is not None and not n_features:
            n_features = int(colmap_path["feat"].shape[1])
        _check_features(n_features, use_sh_coeff, sh_eval, densify_stats)
        self.sh_eval = sh_eval
        self.filter2d, self.filter2d_variance = filter2d, filter2d_variance
        self.use_filter3d, self.filter3d_variance = bool(filter3d), filter3d_variance
        self.filter3d = None                                        # [n] once computed (compute_filter3d)
        self._filter3d_of = None                                    # weakref to the pos Parameter it was computed for
        ckpt_filter3d = None
        self.use_sh_coeff = bool(use_sh_coeff)
        self.near = near
        self.render_downsample = render_downsample
        self.tile_culling_method = tile_culling_method
        self.tile_culling_prob_thresh = tile_culling_prob_thresh
        self.scale_activation = scale_activation
        self.debug = debug
        self.test = test
        self.imgs: List[torch.Tensor] = []
        self.views: List[dict] = []
        if isinstance(colmap_path, dict):
            params = {k: colmap_path[k] for k in ("pos", "rgb", "opa", "quat", "scale")}
            self._set_views(image_path)
            self.imgs = [] if images is None else [im.to(self.device) for im in images]
        else:
            params = self._load_colmap(colmap_path, image_path, opa_init_value, scale_init_value)
        if isinstance(colmap_path, dict) and colmap_path.get("feat") is not None:
            params["feat"] = colmap_path["feat"]
        if load_ckpt is not None:                                   # reference splatter.py:417-424
            ckpt = torch.load(load_ckpt, map_location="cpu", weights_only=False)   # nn.Parameters, train.py:284-290
            params = {k: ckpt[k].detach() for k in ("pos", "rgb", "opa", "quat", "scale")}
            ckpt_filter3d = ckpt.get("filter3d")
            if ckpt.get("feat") is not None:                       # a checkpoint with features (checkpoint.py)
                params["feat"] = ckpt["feat"].detach()
                if not n_features:
                    n_features = int(params["feat"].shape[1])
                    _check_features(n_features, use_sh_coeff, sh_eval, densify_stats)
        if self.primitive == "surfel":                             # flat: the third axis at the activation's floor
            params["scale"] = params["scale"].clone()
            params["scale"][:, 2] = 0.0 if scale_activation == "abs" else math.log(EPS)
        if self.use_sh_coeff != (params["rgb"].shape[1] != 3):
            raise ValueError("use_sh_coeff must match the colour width (3 = RGB logits, 27 / 48 = SH)")
        n = params["pos"].shape[0]
        feat = params.get("feat")
        if feat is not None and tuple(feat.shape) != (n, n_features):
            raise ValueError(f"feat must be [n, n_features] = [{n}, {n_features}], not {list(feat.shape)}")
        if feat is None and n_features:
            feat = torch.zeros(n, n_features)
        self.n_features = int(n_features)
        to = dict(device=self.device, dtype=torch.float32)
        self.gaussian_3ds = Gaussian3ds(*(params[k].detach().to(**to).contiguous()
                                         for k in ("pos", "rgb", "opa", "quat", "scale")),
                                        feat=None if feat is None else feat.detach().to(**to).contiguous())
        with torch.cuda.device(self.device):                      # the context lives on self.device, not on the current one
            self._rctx = gaussian.RenderContext()
        self._rctx.set_sh_eval(SH_EVAL[sh_eval])                   # every frame of this Splatter, fused or not
        self._rctx.set_filter2d(FILTER2D[filter2d], filter2d_variance)
        self.densify_stats = None
        if densify_stats != "none":
            self.densify_stats = DensifyStats(self.gaussian_3ds.pos.shape[0], densify_stats == "absgrad", self.device,
                                              self._rctx)
        if self.use_filter3d and ckpt_filter3d is not None and ckpt_filter3d.numel() == self.gaussian_3ds.pos.shape[0]:
            self._set_filter3d(ckpt_filter3d)
        self._visible = None                                        # visible_mask()'s buffer
        self.ground_truth = None
        self.culling_mask = None
        self.n_tile_gaussians = 0
        self.n_gaussians = self.gaussian_3ds.pos.shape[0]
        self.current_view = None
        self.current_camera = None
        self.tile_info = None
        if self.views and not self.test:
            self.set_camera(0)

    @classmethod
    def from_tensors(cls, gaussians, views, images=None, **kw):
        kw.setdefault("tile_culling_prob_thresh", 0.05)            # train.py:310
        return cls(gaussians, views, images=images, **kw)

    # -- scene loading ----------------------------------------------------------------------
    def _set_views(self, views: Sequence[dict]):
        self.views = [dict(v) for v in views]
        for v in self.views:                     # the camera is host data
            v["rot"] = torch.as_tensor(np.asarray(v["rot"]), dtype=torch.float32).cpu().contiguous()
            v["tran"] = torch.as_tensor(np.asarray(v["tran"]), dtype=torch.float32).cpu().contiguous()

    def _load_colmap(self, colmap_path, image_path, opa_init_value, scale_init_value):
        """reference splatter.py:363-412: points -> parameters (colour logits, opacity logit,
        identity rotation, scale = mean distance to the 3 nearest neighbours x scale_init_value)."""
        import colmap_io
        from scipy.spatial import cKDTree
        self.colmap_path, self.image_path = colmap_path, image_path
        self.cameras = colmap_io.read_cameras_binary(os.path.join(colmap_path, "cameras.bin"))
        if self.camera_model == "colmap":
            for cam in self.cameras.values():
                colmap_intrinsics(cam.model, cam.params)        # refuses an unsupported model before any image is read
        self.images_info = colmap_io.read_images_binary(os.path.join(colmap_path, "images.bin"))
        pts = colmap_io.read_points3d_binary(os.path.join(colmap_path, "points3D.bin"))
        if not self.test:
            self.parse_imgs()
        xyz = np.stack([p.xyz for p in pts.values()]).astype(np.float32)
        rgb = np.stack([p.rgb for p in pts.values()]).astype(np.float32) / 255.0
        rgb = np.clip(rgb, 1e-4, 1 - 1e-4)
        logit = torch.from_numpy(-np.log(1 / rgb - 1))
        if self.use_sh_coeff:                                      # utils.py:345-348
            sh = torch.zeros(len(xyz), 3, 9)
            sh[:, :, 0] = logit / SH_C0
            colour = sh.flatten(1)
        else:
            colour = logit
        dist, _ = cKDTree(xyz).query(xyz, k=4)
        s = torch.from_numpy(dist[:, 1:].mean(axis=1).astype(np.float32)) * scale_init_value
        if self.scale_activation == "exp":
            s = s.log()
        n = len(xyz)
        return dict(pos=torch.from_numpy(xyz), rgb=colour.float(),
                    opa=torch.full((n,), inverse_sigmoid(opa_init_value)),
                    quat=torch.tensor([1.0, 0, 0, 0]).repeat(n, 1), scale=s.unsqueeze(1).repeat(1, 3))

    def parse_imgs(self):
        """reference splatter.py:429-452: every registered image that exists on disk becomes a view
        (w2c pose from COLMAP's qvec / tvec) with its uint8 ground truth kept on the GPU."""
        import colmap_io
        import cv2
        self.imgs, views = [], []
        for img_id in sorted(self.images_info):
            info = self.images_info[img_id]
            cam = self.cameras[info.camera_id]
            fn = os.path.join(self.image_path, info.name)
            if not os.path.exists(fn):
                continue
            im = cv2.cvtColor(cv2.imread(fn), cv2.COLOR_BGR2RGB)
            self.imgs.append(torch.from_numpy(im).to(torch.uint8).to(self.device))
            fy = cam.params[1] if cam.model != "SIMPLE_PINHOLE" else cam.params[0]
            v = dict(width=im.shape[1], height=im.shape[0], focal_x=cam.params[0] / self.render_downsample,
                     focal_y=fy / self.render_downsample, rot=colmap_io.qvec_to_rotmat(info.qvec),
                     tran=np.asarray(info.tvec), camera_id=info.camera_id)
            if self.camera_model == "colmap":
                v["focal_x"], v["focal_y"], v["lens"] = colmap_intrinsics(cam.model, cam.params, self.render_downsample)
            views.append(v)
        self._set_views(views)

    def switch_resolution(self, downsample_factor):                 # reference splatter.py:454-463
        if downsample_factor == self.render_downsample:
            return
        self.image_path = self.image_path.replace(f"images_{self.render_downsample}", f"images_{downsample_factor}")
        self.render_downsample = downsample_factor
        self.parse_imgs()
        self.current_camera = None
        self.set_camera(0)

    # -- camera -----------------------------------------------------------------------------
    def set_camera(self, idx, extrinsics=None, intrinsics=None):
        """reference splatter.py:465-511 (idx=None: free camera from the GUI)."""
        if idx is None:
            v = dict(width=int(math.ceil(intrinsics["width"])), height=int(math.ceil(intrinsics["height"])),
                     focal_x=float(intrinsics["focal_x"]), focal_y=float(intrinsics["focal_y"]),
                     rot=torch.as_tensor(np.asarray(extrinsics["rot"]), dtype=torch.float32).cpu().contiguous(),
                     tran=torch.as_tensor(np.asarray(extrinsics["tran"]), dtype=torch.float32).cpu().contiguous())
            if intrinsics.get("lens") is not None:
                v["lens"] = dict(intrinsics["lens"])
            elif any(intrinsics.get(key) is not None for key in ("cx", "cy", "model", "k")):
                v["lens"] = dict(model=intrinsics.get("model", "PINHOLE"),
                                 cx=float(intrinsics.get("cx", v["width"] / 2)),
                                 cy=float(intrinsics.get("cy", v["height"] / 2)), k=list(intrinsics.get("k", [0.0] * 4)))
            self.ground_truth = None
        else:
            v = self.views[idx]
            self.ground_truth = (self.imgs[idx].to(torch.float16) / 255.) if idx < len(self.imgs) else None
        self.current_view = self.current_camera = v
        self.current_w2c_rot = v["rot"]
        self.current_w2c_tran = v["tran"]
        self.tile_info = Tiles(v["width"], v["height"], v["focal_x"], v["focal_y"])

    # -- frame ------------------------------------------------------------------------------
    def _surfel_frame(self, final, maps, background=None, dist_near=0.2, dist_far=100.0):
        g, v = self.gaussian_3ds, self.current_view
        image, mp, mask = render_frame_surfel(self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, v["width"], v["height"],
                                              v["focal_x"], v["focal_y"], v["rot"], v["tran"], self.near,
                                              self.tile_culling_prob_thresh, self.scale_activation,
                                              background=background, final=final, maps=maps, dist_near=dist_near,
                                              dist_far=dist_far)
        self.culling_mask = mask
        self.n_gaussians = g.pos.shape[0]
        self.n_tile_gaussians = self._rctx.last_instances()
        return image, mp

    def _gaussian_only(self, who):
        if self.primitive != "gaussian":
            raise ValueError(f"{who} renders 3-D Gaussians; a Splatter with primitive='surfel' renders with forward, "
                             "render_padded and render_surfel_maps")

    def render_surfel_maps(self, camera_id=None, extrinsics=None, intrinsics=None, background=None, dist_near=0.2,
                           dist_far=100.0):
        """primitive='surfel': dict(image [H,W,3] (clamped, cropped, over `background`), alpha, depth (sum w z, camera
        z: divide by alpha for the expected depth), median, distortion (m(z) = far / (far - near) (1 - near / z) with
        near, far = `dist_near`, `dist_far`) [H,W], normal [H,W,3] (sum w n, camera frame; rot^T n in the world)).  All
        are differentiable (`renderer.render_frame_surfel`)."""
        if self.primitive != "surfel":
            raise ValueError("render_surfel_maps needs primitive='surfel'")
        self.set_camera(camera_id, extrinsics, intrinsics)
        image, mp = self._surfel_frame(True, True, background, dist_near, dist_far)
        return dict(image=image, **mp)

    def render_padded(self):
        """Padded, un-clamped image (what reference `render` returns, splatter.py:563-634)."""
        g, v = self.gaussian_3ds, self.current_view
        if self.primitive == "surfel":
            return self._surfel_frame(False, False)[0]
        self._size_densify_stats()
        self._size_filter3d()
        self._set_lens([v])
        image, mask = render_frame(self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, v["width"], v["height"],
                                   v["focal_x"], v["focal_y"], v["rot"], v["tran"], self.near,
                                   self.tile_culling_prob_thresh, self.scale_activation)
        self.culling_mask = mask
        self.n_gaussians = g.pos.shape[0]
        return image

    def forward(self, camera_id=None, extrinsics=None, intrinsics=None):
        """reference splatter.py:643-655; clamp(0,1) + centre crop (:652-653) run inside the blend
        kernels (`render_frame_final`)."""
        self.set_camera(camera_id, extrinsics, intrinsics)
        if self.primitive == "surfel":
            return self._surfel_frame(True, False)[0]
        g, v = self.gaussian_3ds, self.current_view
        self._size_densify_stats()
        self._size_filter3d()
        self._set_lens([v])
        image, mask = render_frame_final(self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, v["width"], v["height"],
                                         v["focal_x"], v["focal_y"], v["rot"], v["tran"], self.near,
                                         self.tile_culling_prob_thresh, self.scale_activation)
        self.culling_mask = mask
        self.n_gaussians = g.pos.shape[0]
        self.n_tile_gaussians = self._rctx.last_instances()         # train.py:198 reads it every step
        return image

    def render_maps(self, camera_id=None, extrinsics=None, intrinsics=None, background=None):
        """`forward` plus per-pixel maps: dict(image [H,W,3] (clamped, cropped, over `background`, default black),
        depth [H,W] (accumulated sum w |p_c|: divide by alpha for the expected Euclidean distance), alpha [H,W]).
        All three are differentiable (`renderer.render_frame_aux`)."""
        self._gaussian_only("render_maps")
        self.set_camera(camera_id, extrinsics, intrinsics)
        g, v = self.gaussian_3ds, self.current_view
        self._size_densify_stats()
        self._size_filter3d()
        self._set_lens([v])
        image, depth, alpha, mask = render_frame_aux(self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, v["width"],
                                                     v["height"], v["focal_x"], v["focal_y"], v["rot"], v["tran"],
                                                     self.near, self.tile_culling_prob_thresh, self.scale_activation,
                                                     background=background, final=True)
        self.culling_mask = mask
        self.n_gaussians = g.pos.shape[0]
        self.n_tile_gaussians = self._rctx.last_instances()
        return dict(image=image, depth=depth, alpha=alpha)

    def render_batch(self, camera_ids, background=None):
        """The views `camera_ids` rendered as one frame (`renderer.render_frame_batch`): dict(image [B,H,W,3],
        depth [B,H,W], alpha [B,H,W], culling_mask [B,n]), plus `ground_truth` [B,H,W,3] (float16) when the Splatter
        holds images.  Each view is what `render_maps` returns for it; the gradients are SUMS over the views (divide
        the loss by B for a mean).  Sets `culling_mask` to the [n] sum over the views and `n_tile_gaussians` to the
        batch's instance count.  The views must share their size (ValueError otherwise)."""
        self._gaussian_only("render_batch")
        return self._render_batch("render_batch", render_frame_batch, camera_ids, None, None, background)

    def render_batch_at_poses(self, rots, trans, camera_ids, background=None):
        """`render_batch` at caller-supplied poses, differentiable with respect to them: rots [B,3,3] and trans [B,3]
        are float32 CUDA tensors (world -> camera per view), typically a learnable correction per view composed with
        the views' poses in torch (mini-batch pose refinement) or B candidate poses of a frozen scene (localisation).
        The intrinsics and `ground_truth` come from `camera_ids` (B ids).  Returns `render_batch`'s dict and sets the
        same attributes; backward gives rots and trans their gradients (`renderer.render_frame_batch_cam`), and runs
        camera only when no scene parameter needs a gradient.  Costs one host synchronisation (the 12 B pose floats)."""
        self._gaussian_only("render_batch_at_poses")
        return self._render_batch("render_batch_at_poses", render_frame_batch_cam, camera_ids, rots, trans, background)

    def _render_batch(self, who, render, camera_ids, rots, trans, background):
        ids = list(camera_ids)
        if not ids:
            raise ValueError(f"{who}: no camera ids")
        vs = [self.views[i] for i in ids]
        if any(v["width"] != vs[0]["width"] or v["height"] != vs[0]["height"] for v in vs):
            raise ValueError(f"{who}: the views of a batch must have the same width and height")
        if rots is None:
            rots, trans = torch.stack([v["rot"] for v in vs]), torch.stack([v["tran"] for v in vs])
        g = self.gaussian_3ds
        self._size_densify_stats()
        self._size_filter3d()
        self._set_lens(vs)
        image, depth, alpha, mask = render(
            self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, vs[0]["width"], vs[0]["height"],
            [v["focal_x"] for v in vs], [v["focal_y"] for v in vs], rots, trans, self.near,
            self.tile_culling_prob_thresh, self.scale_activation, background=background, final=True)
        self.culling_mask = mask.sum(0)
        self.n_gaussians = g.pos.shape[0]
        self.n_tile_gaussians = self._rctx.last_instances()
        out = dict(image=image, depth=depth, alpha=alpha, culling_mask=mask)
        imgs = getattr(self, "imgs", [])
        if all(i < len(imgs) for i in ids):
            out["ground_truth"] = torch.stack([imgs[i] for i in ids]).to(torch.float16) / 255.
        return out

    def render_features(self, camera_id=None, extrinsics=None, intrinsics=None, background=None):
        """`render_maps` plus the feature map: dict(image, features [H,W,F], depth, alpha).  features_k = sum_i w_i
        f_i,k with the image's weights, composited over zero (the background applies to the image only; divide by
        alpha for the expected feature), not clamped.  All four are differentiable (`renderer.render_frame_feat`);
        the feature loss reaches `gaussian_3ds.feat` and, through alpha, the geometry.  Needs n_features > 0."""
        self._gaussian_only("render_features")
        g = self.gaussian_3ds
        if g.feat is None:
            raise RuntimeError("render_features needs Splatter(..., n_features=8, 16 or 32)")
        self.set_camera(camera_id, extrinsics, intrinsics)
        v = self.current_view
        self._size_densify_stats()
        self._size_filter3d()
        self._set_lens([v])
        image, features, depth, alpha, mask = render_frame_feat(
            self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, g.feat, v["width"], v["height"], v["focal_x"],
            v["focal_y"], v["rot"], v["tran"], self.near, self.tile_culling_prob_thresh, self.scale_activation,
            background=background, final=True)
        self.culling_mask = mask
        self.n_gaussians = g.pos.shape[0]
        self.n_tile_gaussians = self._rctx.last_instances()
        return dict(image=image, features=features, depth=depth, alpha=alpha)

    def render_at_pose(self, rot, tran, camera_id=None, background=None):
        """`render_maps` at a caller-supplied pose, differentiable with respect to it: rot [3,3] and tran [3] are
        float32 CUDA tensors (world -> camera, p_c = rot p + tran), typically a learnable correction composed with a
        view's pose in torch (pose refinement) or a pose being tracked against the frozen scene.  The intrinsics and
        `ground_truth` come from view `camera_id` (default: the current view).  Returns dict(image, depth, alpha) like
        `render_maps`; backward gives rot and tran their gradients (`renderer.render_frame_cam`), and runs camera
        only when no scene parameter needs a gradient.  Costs one extra host synchronisation (the 12 pose floats)."""
        self._gaussian_only("render_at_pose")
        if camera_id is not None:
            self.set_camera(camera_id)
        if self.current_view is None:
            raise ValueError("render_at_pose: no current view; pass camera_id")
        g, v = self.gaussian_3ds, self.current_view
        self._size_densify_stats()
        self._size_filter3d()
        self._set_lens([v])
        image, depth, alpha, mask = render_frame_cam(self._rctx, g.pos, g.rgb, g.opa, g.quat, g.scale, v["width"],
                                                     v["height"], v["focal_x"], v["focal_y"], rot, tran, self.near,
                                                     self.tile_culling_prob_thresh, self.scale_activation,
                                                     background=background, final=True)
        self.culling_mask = mask
        self.n_gaussians = g.pos.shape[0]
        self.n_tile_gaussians = self._rctx.last_instances()
        return dict(image=image, depth=depth, alpha=alpha)

    def forward_unfused_post(self, camera_id=None, extrinsics=None, intrinsics=None):
        """Same image through the padded raw render + torch clamp/crop (kept for cross-checks)."""
        self.set_camera(camera_id, extrinsics, intrinsics)
        padded = self.render_padded()
        return self.tile_info.crop(torch.clamp(padded, 0, 1))

    def _set_lens(self, views):
        """The context's lenses for a frame (or a sampling-rate pass) over `views`: off when no view has a "lens",
        one for every view when they all share one, else one per view (a view without one gets the image-centre
        pinhole; at most 64 distinct per call)."""
        if all(v.get("lens") is None for v in views):
            self._rctx.set_lens(None, None)
            return
        first = views[0].get("lens")
        if first is not None and all(v.get("lens") == first for v in views):
            views = views[:1]
        models, params = [], []
        for v in views:
            ln = v.get("lens") or dict(model="PINHOLE", cx=v["width"] / 2, cy=v["height"] / 2, k=[0.0] * 4)
            if ln["model"] not in LENS_MODELS:
                raise ValueError(f"lens model must be one of {sorted(LENS_MODELS)}, not {ln['model']!r}")
            k = list(ln.get("k", [0.0] * 4))
            if len(k) != 4:
                raise ValueError(f"lens k must have 4 coefficients, not {len(k)}")
            models.append(LENS_MODELS[ln["model"]])
            params.append([float(ln["cx"]), float(ln["cy"])] + [float(x) for x in k])
        self._rctx.set_lens(models, torch.tensor(params, dtype=torch.float32))

    # -- 3-D smoothing filter (Mip-Splatting) ----------------------------------------------------
    @torch.no_grad()
    def compute_filter3d(self, views=None, margin=0.15):
        """(Re)compute `self.filter3d` [n] on the device (`gaussian.filter3d_compute`) from the sampling rate of
        `views` (default: the training views, with their current focal lengths; dicts with width, height, focal_x,
        focal_y, rot, tran) at this Splatter's near plane: f_i = sqrt(filter3d_variance) / max over the views that see
        Gaussian i (in front of the near plane, inside the image widened by `margin` on every side) of fx / z; a
        Gaussian no view sees gets the largest filter.  The same bits for any order of the views, so data-parallel
        replicas that hold the same views agree.  Returns the buffer."""
        if not self.use_filter3d:
            raise RuntimeError("compute_filter3d needs Splatter(..., filter3d=True)")
        vs = list(self.views if views is None else views)
        if not vs:
            raise ValueError("compute_filter3d: no views")
        self._set_lens(vs)                                          # the lens variant of the rate and the test
        g = self.gaussian_3ds
        size = torch.tensor([[int(v["width"]), int(v["height"])] for v in vs], dtype=torch.int64)
        focal = torch.tensor([[float(v["focal_x"]), float(v["focal_y"])] for v in vs], dtype=torch.float32)
        rot = torch.stack([torch.as_tensor(np.asarray(v["rot"]), dtype=torch.float32).reshape(3, 3) for v in vs])
        tran = torch.stack([torch.as_tensor(np.asarray(v["tran"]), dtype=torch.float32).reshape(3) for v in vs])
        n = g.pos.shape[0]
        out = self.filter3d if self.filter3d is not None and self.filter3d.numel() == n else None
        f = gaussian.filter3d_compute(self._rctx, g.pos.detach().contiguous(), size, focal, rot, tran, float(self.near),
                                      float(margin), self.filter3d_variance, out)
        self._set_filter3d(f)
        return f

    def _set_filter3d(self, f):
        self.filter3d = f.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self._filter3d_of = weakref.ref(self.gaussian_3ds.pos)
        self._rctx.set_filter3d(self.filter3d)

    def _size_filter3d(self):
        # the filter follows the scene: recomputed when its Gaussians were replaced (a densification, a checkpoint)
        if not self.use_filter3d:
            return
        if (self.filter3d is None or self.filter3d.numel() != self.gaussian_3ds.pos.shape[0] or
                self._filter3d_of is None or self._filter3d_of() is not self.gaussian_3ds.pos):
            self.compute_filter3d()

    @torch.no_grad()
    def bake_filter3d(self):
        """Raw (opa [n], scale [n, 3]) with the 3-D filter folded in, for renderers without one: the logit of
        sigma prod s / s' formed in fp64, and s' = sqrt(s^2 + f^2) inverted through the scale activation.  Rows with a
        zero filter keep their parameters.  Rendered without a 3-D filter they give the filtered frame."""
        if not self.use_filter3d:
            raise RuntimeError("bake_filter3d needs Splatter(..., filter3d=True)")
        self._size_filter3d()
        g = self.gaussian_3ds
        raw = g.scale.detach().double()
        s = raw.abs() + EPS if self._scale_act() == 0 else torch.exp(raw)
        f = self.filter3d.double().unsqueeze(1)
        sf = torch.sqrt(s * s + f * f)
        sig = torch.sigmoid(g.opa.detach().double()) * torch.prod(s / sf, dim=1)
        opa = torch.log(sig) - torch.log1p(-sig)
        scale = (sf - EPS) if self._scale_act() == 0 else torch.log(sf)
        keep = self.filter3d == 0
        opa = torch.where(keep, g.opa.detach(), opa.float())
        scale = torch.where(keep.unsqueeze(1), g.scale.detach(), scale.float())
        return opa.contiguous(), scale.contiguous()

    # -- densification from screen-space statistics ----------------------------------------------
    def _size_densify_stats(self):
        # the statistics follow the scene: when its Gaussians were replaced by other means (adaptive_control, a
        # checkpoint), they restart from zero at the new count
        if self.densify_stats is not None and self.densify_stats.n != self.gaussian_3ds.pos.shape[0]:
            self.densify_stats.reset(self.gaussian_3ds.pos.shape[0])

    @torch.no_grad()
    def adaptive_control_screen(self, taus, delete_thresh, grad_thresh=0.0002, use_abs=False, max_screen_size=None,
                                use_clone=True, use_split=True, generator=None):
        """Prune / clone / split from the screen-space statistics (`densify_stats`), with 3DGS's rule: a kept Gaussian
        densifies when grad2d / count (absgrad / count with `use_abs`) >= `grad_thresh`; clones are exact copies.
        With `max_screen_size` (pixels), Gaussians whose screen radius exceeded it are pruned too.  Opacity and
        scale-norm pruning and the clone / split choice by `taus` are `Gaussian3ds.adaptive_control`'s.  The
        parameters are re-created like `adaptive_control` (the caller rebuilds its optimizer), and the statistics
        restart from zero.  Under data parallel, call `densify_stats.all_reduce()` first.  Returns the same dict
        as `adaptive_control`."""
        st = self.densify_stats
        if st is None:
            raise RuntimeError("adaptive_control_screen needs Splatter(..., densify_stats='grad' or 'absgrad')")
        if use_abs and st.absgrad is None:
            raise ValueError("use_abs=True needs Splatter(..., densify_stats='absgrad')")
        g = self.gaussian_3ds
        if st.n != g.pos.shape[0]:
            raise RuntimeError("densify_stats are sized for another number of Gaussians than the scene has")
        args = [t.detach().contiguous() for t in (g.pos, g.rgb, g.opa, g.quat, g.scale)]
        new, (n_deleted, n_clone, n_split) = gaussian.densify_stats(
            *args, st.absgrad if use_abs else st.grad2d, st.count,
            st.max_radius if max_screen_size is not None else None,
            float(max_screen_size) if max_screen_size is not None else 0.0,
            0 if self.scale_activation == "abs" else 1, inverse_sigmoid(0.02), float(delete_thresh),
            float(grad_thresh), float(taus), bool(use_clone), bool(use_split), generator, g._feat_arg())
        g._replace(new)
        self.n_gaussians = g.pos.shape[0]
        st.reset(self.n_gaussians)
        self._size_filter3d()
        return dict(deleted=int(n_deleted), cloned=int(n_clone), split=int(n_split), total=self.n_gaussians)

    # -- MCMC densification (3DGS-MCMC; mcmc.MCMC schedules these) -----------------------------------------------------
    def _mcmc_params(self):
        g = self.gaussian_3ds
        return [g.pos, g.rgb, g.opa, g.quat, g.scale] + ([g.feat] if g.feat is not None else [])

    def _scale_act(self):
        if self.scale_activation not in ("abs", "exp"):
            raise ValueError("scale_activation must be 'abs' or 'exp'")
        return 0 if self.scale_activation == "abs" else 1

    @torch.no_grad()
    def mcmc_relocate(self, optimizer=None, min_opacity=0.005, generator=None):
        """Move every dead Gaussian (sigmoid(opa) <= min_opacity) onto a live one drawn with probability proportional
        to its opacity, and split the drawn ones' opacity and scale among their copies (gsplat's `relocate`;
        `gaussian.mcmc_relocate`).  In place: the Parameters keep their identity (and `optim.FlatAdam`'s aliasing).
        The Adam moments of every source and destination row are zeroed (`optim.FlatAdam` or `torch.optim.Adam`; the
        rows of Parameters the optimizer does not hold have no state to zero); nothing before the optimizer's first
        step.  The uniforms come from torch's generator (`generator`, default CUDA), so replicas seeded alike stay
        identical.  Returns the relocated count as a CUDA int32 [1] tensor (no host synchronisation)."""
        import optim
        g = self.gaussian_3ds
        n = g.pos.shape[0]
        u = torch.rand(n, device=self.device, generator=generator)
        mom = optimizer.live_moments(self._mcmc_params()) if isinstance(optimizer, optim.FlatAdam) else None
        touched = None
        if optimizer is not None and mom is None:
            touched = torch.zeros(n, device=self.device, dtype=torch.uint8)
        kw = {}
        if mom is not None:
            kw = dict(exp_avg=mom[0], exp_avg_sq=mom[1], seg_starts=mom[2], seg_widths=mom[3])
        n_rel = gaussian.mcmc_relocate(g.pos.data, g.rgb.data, g.opa.data, g.quat.data, g.scale.data,
                                       None if g.feat is None else g.feat.data, self._scale_act(), float(min_opacity),
                                       u, touched=touched, **kw)
        if touched is not None:
            _zero_moment_rows(optimizer, self._mcmc_params(), touched.bool())
        if self.use_filter3d:                                       # in place: the Parameters kept their identity
            self.compute_filter3d()
        return n_rel

    @torch.no_grad()
    def mcmc_add(self, cap_max, growth=1.05, optimizer=None, generator=None, min_opacity=0.005):
        """Grow to min(cap_max, int(growth n)) Gaussians (gsplat's `sample_add`; `gaussian.mcmc_add`): each new one is
        a copy of a Gaussian drawn with probability proportional to its opacity, and the drawn ones' opacity and scale
        are split as in `mcmc_relocate`.  New Parameters, like `adaptive_control`; the optimizer (`optim.FlatAdam` or
        `torch.optim.Adam`) is re-pointed at them and keeps the moments of the existing rows bit for bit, the new rows
        start at zero.  `densify_stats` and the visible mask re-size from zero.  Returns the number added (host int,
        computed from the sizes: no synchronisation)."""
        g = self.gaussian_3ds
        n = g.pos.shape[0]
        n_new = max(0, min(int(cap_max), int(float(growth) * n)) - n)
        if n_new == 0:
            return 0
        u = torch.rand(n_new, device=self.device, generator=generator)
        old = self._mcmc_params()
        new = gaussian.mcmc_add(g.pos.data, g.rgb.data, g.opa.data, g.quat.data, g.scale.data,
                                None if g.feat is None else g.feat.data, self._scale_act(), float(min_opacity), u)
        g._replace(new)
        if optimizer is not None:
            _regrow_optimizer(optimizer, list(zip(old, self._mcmc_params())))
        self.n_gaussians = g.pos.shape[0]
        self._size_densify_stats()
        self._size_filter3d()
        return n_new

    # -- contribution scores and pruning ---------------------------------------------------------------------------
    def _scores_only(self, who):
        if self.primitive != "gaussian":
            raise ValueError(f"{who} scores 3-D Gaussian frames; a Splatter with primitive='surfel' has no score pass")

    def _check_scores(self, who, scores):
        n = self.gaussian_3ds.pos.shape[0]
        if not isinstance(scores, ContributionScores):
            raise TypeError(f"{who}: scores must be a ContributionScores")
        if scores.n != n:
            raise ValueError(f"{who}: scores are sized for {scores.n} Gaussians, the scene has {n}")

    @torch.no_grad()
    def score_views(self, camera_ids=None, batch_size=8, scores=None):
        """Blend-weight scores (`ContributionScores`) of the views `camera_ids` (default: every training view):
        the views are rendered forward only, in batches of up to `batch_size` views of equal size through the batched
        frame (one view at a time with per-pixel SH colour, which has no batched frame), and each frame is scored on the
        device (gs_frame_scores).  `scores` is zeroed first unless given, in which case the views are added to it.
        Per Gaussian, weight_sum is the sum and weight_max the largest of its weights w = alpha T over the views' pixels.

        The score frames replace the context's last frame: call this between a training frame's backward and the next
        forward, not between a forward and its backward.  A data-parallel gradient push configured by earlier
        backwards is cleared first (batched frames take none; the next backward sets it again).  The Splatter's
        attributes of the last frame (`culling_mask`, `n_tile_gaussians`, the current view and `ground_truth`) are left
        as they were.  Under data parallel, each rank can score its share of the views (`camera_ids=range(rank,
        n_views, world)`) and `scores.all_reduce()` combines them.

        Keeping a budget of the k Gaussians with the largest weight_sum is one line; the stable sort breaks ties by
        index, so data-parallel replicas (after `scores.all_reduce()`) keep the same rows:

            keep = torch.zeros(n, dtype=torch.bool, device=dev).index_fill_(
                0, torch.sort(scores.weight_sum, descending=True, stable=True).indices[:k], True)
            splatter.prune(keep, optimizer)
        """
        self._scores_only("score_views")
        ids = list(range(len(self.views))) if camera_ids is None else [int(i) for i in camera_ids]
        if int(batch_size) < 1:
            raise ValueError(f"score_views: batch_size must be >= 1, not {batch_size!r}")
        if scores is None:
            scores = ContributionScores(self.gaussian_3ds.pos.shape[0], self.device)
        else:
            self._check_scores("score_views", scores)
        saved = {k: getattr(self, k, None) for k in _FRAME_ATTRS}
        self._rctx.clear_grad_push()
        try:
            if self.use_sh_coeff and self.sh_eval == "pixel":
                for i in ids:
                    self.forward(i)
                    self._rctx.scores_into(scores.weight_sum, scores.weight_max)
                return scores
            by_size = {}
            for i in ids:
                by_size.setdefault((self.views[i]["width"], self.views[i]["height"]), []).append(i)
            for group in by_size.values():
                for k in range(0, len(group), int(batch_size)):
                    self._render_batch("score_views", render_frame_batch, group[k:k + int(batch_size)], None, None,
                                       None)
                    self._rctx.scores_into(scores.weight_sum, scores.weight_max)
            return scores
        finally:
            for k, v in saved.items():
                setattr(self, k, v)

    @torch.no_grad()
    def accumulate_scores(self, scores):
        """Add the blend-weight scores of the last frame rendered through this Splatter (`forward`, `render_maps`,
        `render_batch`, `render_features`, `render_at_pose`) to `scores` (a `ContributionScores` sized for the scene):
        a trainer collects them from its training frames without extra forwards.  Returns `scores`."""
        self._scores_only("accumulate_scores")
        self._check_scores("accumulate_scores", scores)
        self._rctx.scores_into(scores.weight_sum, scores.weight_max)
        return scores

    @torch.no_grad()
    def prune(self, keep, optimizer=None):
        """Keep the Gaussians with keep[i] set (CUDA bool [n]), in order, and remove the others (`gaussian.prune`: a
        keep-only `gs_densify_apply` plan; feature rows follow).  New Parameters, like `mcmc_add`; the optimizer
        (`optim.FlatAdam` or `torch.optim.Adam`) is re-pointed at them and keeps the kept rows' moments bit for bit and
        its step count.  `densify_stats` and the visible mask re-size from zero, and the 3-D filter is recomputed.
        Returns the number removed.  ValueError when keep selects nothing."""
        g = self.gaussian_3ds
        n = g.pos.shape[0]
        if not (torch.is_tensor(keep) and keep.is_cuda and keep.dtype == torch.bool and keep.dim() == 1):
            raise TypeError("prune: keep must be a 1-D CUDA bool tensor")
        if keep.numel() != n:
            raise ValueError(f"prune: keep has {keep.numel()} entries, the scene has {n} Gaussians")
        if not bool(keep.any()):
            raise ValueError("prune: keep selects no Gaussian")
        keep = keep.to(self.device).contiguous()
        old = self._mcmc_params()
        new, n_removed = gaussian.prune(*(t.detach().contiguous() for t in (g.pos, g.rgb, g.opa, g.quat, g.scale)),
                                        keep, g._feat_arg())
        g._replace(new)
        if optimizer is not None:
            _regrow_optimizer(optimizer, list(zip(old, self._mcmc_params())), keep)
        self.n_gaussians = g.pos.shape[0]
        self._size_densify_stats()
        self._size_filter3d()
        return int(n_removed)

    @torch.no_grad()
    def mcmc_noise(self, scaler, seed=None):
        """Perturb the positions by scaler g(o) R diag(s^2) R^T z (gsplat's `inject_noise_to_position`;
        `gaussian.mcmc_noise`), z from a Philox stream keyed by (seed, Gaussian index).  `seed` None draws one from
        torch's CPU generator, which checkpoints restore.  Writes `pos` only."""
        g = self.gaussian_3ds
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)))
        gaussian.mcmc_noise(g.pos.data, g.quat.data, g.scale.data, g.opa.data, self._scale_act(), float(scaler),
                            int(seed))

    @torch.no_grad()
    def add_mcmc_regularizer_grads(self, opacity_reg=0.01, scale_reg=0.01):
        """Add the gradients of MCMC's opacity_reg mean(sigmoid(opa)) + scale_reg mean(s) to `opa.grad` and
        `scale.grad`, in place: after the backward (and any gradient exchange), before the step, so that they stay
        views of the flat gradient bucket and every replica adds the same values."""
        g = self.gaussian_3ds
        if g.opa.grad is None or g.scale.grad is None:
            raise RuntimeError("add_mcmc_regularizer_grads: run the backward first (opa.grad / scale.grad are None)")
        n = g.pos.shape[0]
        if opacity_reg and n:
            o = torch.sigmoid(g.opa.detach())
            g.opa.grad.add_(o * (1 - o), alpha=float(opacity_reg) / n)
        if scale_reg and n:
            raw = g.scale.detach()
            ds = torch.exp(raw) if self._scale_act() == 1 else torch.sign(raw)
            g.scale.grad.add_(ds, alpha=float(scale_reg) / (3 * n))

    @torch.no_grad()
    def visible_mask(self, accumulate=False):
        """uint8 [n]: 1 where the last frame rendered through this Splatter (`forward`, `render_maps`, `render_batch`:
        any of its views, `render_features`, `render_at_pose`) binned the Gaussian into at least one tile, the set
        with a gradient and the one `densify_stats.count` counts; every other Gaussian's gradient row is exactly
        zero.  `accumulate=True` ORs into the previous mask (several frames before one optimizer step).  For
        `optim.FlatAdam.step(visible=...)`; under data parallel reduce it with `dp.all_reduce_visible` first.  The
        buffer belongs to the Splatter, is rewritten by the next call and re-sized (from zero) when the number of
        Gaussians changes."""
        n = self.gaussian_3ds.pos.shape[0]
        if self._visible is None or self._visible.numel() != n:
            self._visible = torch.zeros(n, device=self.device, dtype=torch.uint8)
        self._rctx.visible_into(self._visible, bool(accumulate))
        return self._visible

    def save_checkpoint(self, path, optimizer=None, iteration=None, trainer_state=None):
        """reference Trainer.save_checkpoint (train.py:283-291) + resume state; see checkpoint.py."""
        import checkpoint
        return checkpoint.save_checkpoint(self, path, optimizer, iteration, trainer_state)

    def frame_stats(self):
        s = self._rctx.stats()
        self.n_tile_gaussians = int(s["n_instances"])
        return s
