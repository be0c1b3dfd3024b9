"""CPU oracle of the depth / alpha maps and the background colour (gs_render_forward_aux).

Test infrastructure only.  It adds no blend code of its own: the maps are two more "colour" channels of
oracle/gs_oracle.py's `draw`, which blends any per-instance value with the weights w_i = alpha_i T_i live_i
(live_i = T_i >= 1e-4, the early stop).  Blending (t_i, 1) gives (depth, sum w_i), and sum w_i = 1 - T_f exactly
(the product telescopes; a pixel never comes back to life).  So, per pixel:

    image_c = sum_i w_i c_i,c + (1 - alpha) bg_c     (c_i from `draw`'s RGB or per-pixel SH colour)
    depth   = sum_i w_i t_i                          t_i = |p_c,i| = res_pos[:, 2]
    alpha   = sum_i w_i = 1 - T_f

The reference renderer has no such outputs, so nothing pins this oracle externally: tests/test_render_aux_oracle.py
checks it against closed-form identities and finite differences instead.
"""
from __future__ import annotations

import torch

import gs_oracle as O


def draw_maps(pos, rgb, opa, cov, tile_n_point_accum, Hp, Wp, fx, fy, background=None, use_sh_coeff=False,
              rays=(None,) * 4):
    """gs_oracle.draw plus the maps: returns (image[Hp,Wp,3] un-clamped over `background` (None = black),
    depth[Hp,Wp], alpha[Hp,Wp]).  pos[:, 2] is the depth t_i."""
    img = O.draw(pos, rgb, opa, cov, tile_n_point_accum, Hp, Wp, fx, fy, use_sh_coeff, *rays)
    chan = torch.stack([pos[:, 2], torch.ones_like(pos[:, 2]), torch.zeros_like(pos[:, 2])], dim=-1)
    maps = O.draw(pos, chan, opa, cov, tile_n_point_accum, Hp, Wp, fx, fy)
    depth, alpha = maps[..., 0], maps[..., 1]
    if background is not None:
        img = img + (1 - alpha).unsqueeze(-1) * torch.as_tensor(background, dtype=img.dtype)
    return img, depth, alpha


def render_maps(pos, rgb, opa, quat, scale, cam: O.Camera, thresh=0.05, scale_activation="abs", background=None,
                use_sh_coeff=False, depth_key=None):
    """gs_oracle.render with maps: returns dict(image [H,W,3] clamped + cropped, depth [H,W], alpha [H,W],
    padded_image [Hp,Wp,3], padded_depth, padded_alpha [Hp,Wp], mask); differentiable wrt the five parameter
    tensors, depth through res_pos[:, 2] = |p_c|."""
    dt = pos.dtype
    rot, tran = cam.rot.to(dt), cam.tran.to(dt)
    nq, ns, opa_a, rgb_a = O.preactivate(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
    rp, rc, mask = O.global_culling(pos, nq, ns, rot, tran, cam.near, cam.half_w, cam.half_h)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    p_c, c_c, rgb_c, opa_c = rp[idx], rc[idx], rgb_a[idx], opa_a[idx]
    rects = O.tile_rects(p_c[:, :2], c_c, thresh, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                         cam.topmost)
    gi, accum = O.bin_and_sort(p_c, c_c, rects, cam.ntx, cam.nty, None if depth_key is None else depth_key[idx])
    rays = O.ray_info(rot, tran, cam.Hp, cam.Wp, cam.fx, cam.fy) if use_sh_coeff else (None,) * 4
    img, dep, alp = draw_maps(p_c[gi], rgb_c[gi], opa_c[gi], c_c[gi], accum, cam.Hp, cam.Wp, cam.fx, cam.fy,
                              background, use_sh_coeff, rays)

    def crop2(x):
        return cam.crop(x.unsqueeze(-1)).squeeze(-1)

    return dict(image=cam.crop(torch.clamp(img, 0, 1)), depth=crop2(dep), alpha=crop2(alp), padded_image=img,
                padded_depth=dep, padded_alpha=alp, mask=mask)
