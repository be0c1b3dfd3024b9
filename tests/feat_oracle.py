"""CPU oracle of the feature maps (gs_render_forward_feat, renderer.render_frame_feat).

Test infrastructure only, and a composition with no blend code of its own: features are more "colour" channels of
oracle/gs_oracle.py's `draw`, three at a time, as tests/aux_oracle.py does for depth and alpha.  `draw` blends any
per-instance value with the weights w_i = alpha_i T_i live_i of the image, so per pixel

    feature_k = sum_i w_i f_i,k                (composited over zero: the background applies to the image only)

The front end (projection, culling, optional 2-D filter, binning, sort) is tests/filter_oracle.py's (mode "none" is
gs_oracle's computation bit for bit); per-Gaussian SH colour goes through tests/sh_gaussian_oracle.py's logits.
Autograd of the composition gives every gradient, the features' own included.
"""
from __future__ import annotations

import torch

import aux_oracle as A
import filter_oracle as FO
import gs_oracle as O
import sh_gaussian_oracle as SG


def draw_features(pos, feat, opa, cov, tile_n_point_accum, Hp, Wp, fx, fy, tiles=None):
    """[Hp, Wp, F] blend of per-instance rows feat [m, F] (sorted like pos) with gs_oracle.draw's weights (`tiles`:
    only those tiles, as gs_oracle.draw)."""
    F = feat.shape[1]
    pad = (-F) % 3
    f = torch.cat([feat, feat.new_zeros(feat.shape[0], pad)], dim=1) if pad else feat
    maps = [O.draw(pos, f[:, k:k + 3], opa, cov, tile_n_point_accum, Hp, Wp, fx, fy, tiles=tiles)
            for k in range(0, F + pad, 3)]
    return torch.cat(maps, dim=-1)[..., :F]


def render_feat(pos, rgb, opa, quat, scale, feat, cam: O.Camera, mode="none", variance=0.3, thresh=0.05,
                scale_activation="abs", background=None, sh_gaussian=False, depth_key=None):
    """aux_oracle.render_maps plus the feature map: dict(image, depth, alpha, features [H,W,F], padded_image,
    padded_depth, padded_alpha, padded_features [Hp,Wp,F], mask).  rgb: RGB logits [n, 3] or, with sh_gaussian, SH
    coefficients [n, 27 | 48] evaluated once per Gaussian.  Differentiable in the five parameters and feat."""
    if sh_gaussian:
        rgb = SG.gaussian_logits(pos, rgb, cam)
    p, c, o, cv, accum, _, mask, gidx = FO._front(pos, rgb, opa, quat, scale, cam, mode, variance, thresh,
                                                  scale_activation, False, depth_key)
    img, dep, alp = A.draw_maps(p, c, o, cv, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, background)
    fm = draw_features(p, feat[gidx], o, cv, accum, cam.Hp, cam.Wp, cam.fx, cam.fy)

    def crop2(x):
        return cam.crop(x.unsqueeze(-1)).squeeze(-1)

    return dict(image=cam.crop(torch.clamp(img, 0, 1)), depth=crop2(dep), alpha=crop2(alp), features=cam.crop(fm),
                padded_image=img, padded_depth=dep, padded_alpha=alp, padded_features=fm, mask=mask)
