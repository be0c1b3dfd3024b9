"""CPU oracle of SH colour evaluated once per Gaussian (gs_ctx_set_sh_eval(ctx, GS_SH_EVAL_GAUSSIAN),
`Splatter(..., sh_eval="gaussian")`).

Test infrastructure only, and a composition with no blend code of its own: the logits of every Gaussian are the SH
basis of oracle/gs_oracle.py evaluated along the world-space direction from the camera centre C = -R^T t to its mean,

    dir = (pos - C) / |pos - C|,        l_c = sum_k Y_k(dir) rgb[c*K + k]        (K = 9 or 16, channel-major)

and those logits go through gs_oracle.render (or aux_oracle.render_maps) as RGB logits, which applies the sigmoid and
blends them.  Autograd of the composition gives every gradient, the direction term dL/dpos through dir included.
"""
from __future__ import annotations

import torch

import aux_oracle as A
import gs_oracle as O


def camera_centre(cam: O.Camera, dtype=torch.float64):
    return -(cam.rot.to(dtype).T @ cam.tran.to(dtype))


def gaussian_logits(pos, rgb, cam: O.Camera, detach_dir=False):
    """[n, 3] logits of the SH coefficients rgb[n, 3K] at each Gaussian's view direction (detach_dir: the direction
    as a constant, to isolate its gradient term in tests)."""
    K = rgb.shape[1] // 3
    u = pos - camera_centre(cam, pos.dtype)
    d = u / u.norm(dim=-1, keepdim=True)
    if detach_dir:
        d = d.detach()
    Y = O.sh_basis9(d) if K == 9 else O.sh_basis16(d)
    return torch.einsum("nk,nck->nc", Y, rgb.reshape(-1, 3, K))


def render(pos, rgb, opa, quat, scale, cam: O.Camera, **kw):
    """gs_oracle.render with per-Gaussian SH colour (same keyword arguments; use_sh_coeff does not apply)."""
    return O.render(pos, gaussian_logits(pos, rgb, cam), opa, quat, scale, cam, use_sh_coeff=False, **kw)


def render_maps(pos, rgb, opa, quat, scale, cam: O.Camera, **kw):
    """aux_oracle.render_maps with per-Gaussian SH colour."""
    return A.render_maps(pos, gaussian_logits(pos, rgb, cam), opa, quat, scale, cam, use_sh_coeff=False, **kw)
