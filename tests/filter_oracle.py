"""CPU oracle of the screen-space 2-D filter of the fused frame path (gs_ctx_set_filter2d, `Splatter(..., filter2d=...)`).

Test infrastructure only, and a composition with no blend code of its own.  It takes oracle/gs_oracle.py's
`global_culling` covariance Sigma = (a, b, c, d) of every visible Gaussian, adds the filter in normalised image-plane
units (ex = s / fx^2, ey = s / fy^2 for a variance of s px^2, rounded to float32 as the host does),

    Sigma' = (a + ex, b, c, d + ey)
    dilate    : opacity unchanged
    antialias : opacity * sqrt(det / det'); a Gaussian with det <= 0 is dropped

bins the instances with Sigma' (gs_oracle.tile_rects / bin_and_sort) and draws them through gs_oracle.draw or
aux_oracle.draw_maps.  Mode "none" leaves Sigma and the opacity untouched: gs_oracle.render's computation.  RGB
logits may come from sh_gaussian_oracle.gaussian_logits (per-Gaussian SH); use_sh_coeff=True blends per-pixel SH as
gs_oracle does.
"""
from __future__ import annotations

import numpy as np
import torch

import aux_oracle as A
import gs_oracle as O

MODES = ("none", "dilate", "antialias")


def filter_eps(cam: O.Camera, variance):
    """(ex, ey) as the host forms them: float32 variance and focal lengths, the quotient in double, rounded once."""
    s = float(np.float32(variance))
    fx, fy = float(np.float32(cam.fx)), float(np.float32(cam.fy))
    return float(np.float32(s / (fx * fx))), float(np.float32(s / (fy * fy)))


def filtered(cov, opa, cam: O.Camera, mode, variance=0.3):
    """(Sigma' [n,2,2], opacity [n], keep [n] bool) of visible rows cov [n,2,2] with activated opacities opa [n]."""
    if mode not in MODES:
        raise ValueError(mode)
    keep = torch.ones(cov.shape[0], dtype=torch.bool)
    if mode == "none":
        return cov, opa, keep
    ex, ey = filter_eps(cam, variance)
    eps = torch.tensor([[ex, 0.0], [0.0, ey]], dtype=cov.dtype)
    covf = cov + eps
    if mode == "antialias":
        c4, f4 = cov.reshape(-1, 4), covf.reshape(-1, 4)
        det = c4[:, 0] * c4[:, 3] - c4[:, 1] * c4[:, 2]
        detf = f4[:, 0] * f4[:, 3] - f4[:, 1] * f4[:, 2]
        c32 = cov.detach().to(torch.float32).reshape(-1, 4)     # the device tests det in float32
        keep = (c32[:, 0] * c32[:, 3] - c32[:, 1] * c32[:, 2]) > 0
        ok = det > 0
        opa = opa * torch.sqrt(torch.where(ok, det, detf) / detf)
    return covf, opa, keep


def _front(pos, rgb, opa, quat, scale, cam, mode, variance, thresh, scale_activation, use_sh_coeff, depth_key):
    dt = pos.dtype
    rot, tran = cam.rot.to(dt), cam.tran.to(dt)
    nq, ns, opa_a, rgb_a = O.preactivate(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
    rp, rc, mask = O.global_culling(pos, nq, ns, rot, tran, cam.near, cam.half_w, cam.half_h)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    c_c, o_c, keep = filtered(rc[idx], opa_a[idx], cam, mode, variance)
    p_c = rp[idx]
    tx0, tx1, ty0, ty1 = O.tile_rects(p_c[:, :2], c_c, thresh, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty,
                                      cam.leftmost, cam.topmost)
    tx1, ty1 = torch.where(keep, tx1, tx0), torch.where(keep, ty1, ty0)
    gi, accum = O.bin_and_sort(p_c, c_c, (tx0, tx1, ty0, ty1), cam.ntx, cam.nty,
                               None if depth_key is None else depth_key[idx])
    rays = O.ray_info(rot, tran, cam.Hp, cam.Wp, cam.fx, cam.fy) if use_sh_coeff else (None,) * 4
    return p_c[gi], rgb_a[idx][gi], o_c[gi], c_c[gi], accum, rays, mask, idx[gi]


def render(pos, rgb, opa, quat, scale, cam: O.Camera, mode="none", variance=0.3, thresh=0.05,
           scale_activation="abs", use_sh_coeff=False, tiles=None, return_aux=False, depth_key=None):
    """gs_oracle.render with the filter (mode "none": the same computation, bit for bit): the clamped + cropped image
    (return_aux: and dict(padded, mask, accum, gauss_idx)); differentiable wrt the five parameter tensors, and rot / tran
    when they are leaves of `cam`."""
    p, c, o, cv, accum, rays, mask, gidx = _front(pos, rgb, opa, quat, scale, cam, mode, variance, thresh,
                                                  scale_activation, use_sh_coeff, depth_key)
    img = O.draw(p, c, o, cv, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, use_sh_coeff, *rays, tiles=tiles)
    out = cam.crop(torch.clamp(img, 0, 1))
    if return_aux:
        return out, dict(padded=img, mask=mask, accum=accum, gauss_idx=gidx)
    return out


def render_maps(pos, rgb, opa, quat, scale, cam: O.Camera, mode="none", variance=0.3, thresh=0.05,
                scale_activation="abs", background=None, use_sh_coeff=False, depth_key=None):
    """aux_oracle.render_maps with the filter (same dict)."""
    p, c, o, cv, accum, rays, mask, _ = _front(pos, rgb, opa, quat, scale, cam, mode, variance, thresh,
                                               scale_activation, use_sh_coeff, depth_key)
    img, dep, alp = A.draw_maps(p, c, o, cv, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, background, use_sh_coeff, rays)

    def crop2(x):
        return cam.crop(x.unsqueeze(-1)).squeeze(-1)

    return dict(image=cam.crop(torch.clamp(img, 0, 1)), depth=crop2(dep), alpha=crop2(alp), padded_image=img,
                padded_depth=dep, padded_alpha=alp, mask=mask)
