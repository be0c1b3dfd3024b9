"""CPU oracle of the screen-space densification statistics (gs_ctx_set_densify_stats, `Splatter(..., densify_stats=...)`)
and of the plan scored from them (gs_densify_plan_stats).

Test infrastructure only, and a composition: the frame is filter_oracle's (oracle/gs_oracle.py's culling, binning and
`draw`, aux_oracle's maps), with one change of plumbing: the projected means res_pos[:, :2] of the visible Gaussians
are replaced by a leaf, so that autograd yields dL/d(mean2d) of every Gaussian, summed over its instances.

    grad2d  = |(gx W / (2 fx), gy H / (2 fy))|     (gx, gy) = dL/d(mean2d)
    absgrad = |(Ax W / (2 fx), Ay H / (2 fy))|     (Ax, Ay) = sum over pixels of |pixel p's contribution to (gx, gy)|
    count   = 1 for a Gaussian with at least one tile instance
    radius  = 3 sqrt(lambda_max) of the binned (filtered) covariance in px^2 (the device stores its ceil)

The per-pixel contributions come from each tile's blend evaluated with one copy of the instance means per pixel (a
[256, K, 2] leaf): the blend below repeats gs_oracle.draw's RGB arithmetic with those copies, and autograd of
sum(G * tile) then gives every pixel's own share.  Colour channels may carry the aux maps (depth t_i and 1, as
aux_oracle blends them), so their gradients are included.
"""
from __future__ import annotations

import os
import sys

import torch

import filter_oracle as F
import gs_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
import densify_oracle as D  # noqa: E402


def ndc_scale(cam: O.Camera):
    """(W / (2 fx), H / (2 fy)) as the host forms them: float32 focal lengths, the quotient in double, rounded once."""
    import numpy as np
    fx, fy = float(np.float32(cam.fx)), float(np.float32(cam.fy))
    return float(np.float32(cam.width / (2 * fx))), float(np.float32(cam.height / (2 * fy)))


def _front(pos, rgb, opa, quat, scale, cam, mode, variance, thresh, scale_activation, use_sh_coeff, depth_key):
    """filter_oracle._front with the visible means as a leaf: (instances..., mean2d leaf, visible ids)."""
    dt = pos.dtype
    rot, tran = cam.rot.to(dt), cam.tran.to(dt)
    nq, ns, opa_a, rgb_a = O.preactivate(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
    rp, rc, mask = O.global_culling(pos, nq, ns, rot, tran, cam.near, cam.half_w, cam.half_h)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    m2 = rp[idx][:, :2].detach().clone().requires_grad_(True)
    p_c = torch.cat([m2, rp[idx][:, 2:]], dim=1)
    c_c, o_c, keep = F.filtered(rc[idx], opa_a[idx], cam, mode, variance)
    tx0, tx1, ty0, ty1 = O.tile_rects(p_c[:, :2], c_c, thresh, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty,
                                      cam.leftmost, cam.topmost)
    tx1, ty1 = torch.where(keep, tx1, tx0), torch.where(keep, ty1, ty0)
    gi, accum = O.bin_and_sort(p_c, c_c, (tx0, tx1, ty0, ty1), cam.ntx, cam.nty,
                               None if depth_key is None else depth_key[idx])
    rays = O.ray_info(rot, tran, cam.Hp, cam.Wp, cam.fx, cam.fy) if use_sh_coeff else (None,) * 4
    return dict(p=p_c[gi], rgb=rgb_a[idx][gi], opa=o_c[gi], cov=c_c[gi], accum=accum, rays=rays, gi=gi, m2=m2,
                idx=idx, cov_vis=c_c)


def _tile_pixel_grads(fr, t, G, cam):
    """[256, K, 2] per-pixel contributions to dL/d(mean2d) of tile t's K instances, for the upstream gradient
    G[256, C] of its blended channels (RGB, then depth and alpha when C == 5)."""
    s, e = int(fr["accum"][t]), int(fr["accum"][t + 1])
    dt = fr["p"].dtype
    ty, tx = divmod(t, cam.ntx)
    ix = torch.arange(16)
    px = ((tx * 16 + ix).to(dt) + 0.5 - (cam.Wp // 2)) / cam.fx
    py = ((ty * 16 + ix).to(dt) + 0.5 - (cam.Hp // 2)) / cam.fy
    PX = px.reshape(1, 16).expand(16, 16).reshape(-1, 1)
    PY = py.reshape(16, 1).expand(16, 16).reshape(-1, 1)
    means = fr["p"][s:e, :2].detach().unsqueeze(0).expand(256, -1, -1).clone().requires_grad_(True)
    a, b, c, d = fr["cov"][s:e].detach().reshape(-1, 4).unbind(-1)
    X = PX - means[..., 0]
    Y = PY - means[..., 1]
    det = a * d - b * c
    power = -(d * X * X - (b + c) * X * Y + a * Y * Y) / (2 * det + 1e-14)
    alpha = torch.exp(power) * fr["opa"][s:e].detach().reshape(1, -1)
    Tinc = torch.cumprod(1 - alpha, dim=1)
    Texc = torch.cat([torch.ones(256, 1, dtype=dt), Tinc[:, :-1]], dim=1)
    wgt = alpha * Texc * (Texc.detach() >= 0.0001).to(dt)
    col = fr["rgb"][s:e].detach()
    if G.shape[1] == 5:
        t_i = fr["p"][s:e, 2].detach()
        col = torch.cat([col, t_i.unsqueeze(-1), torch.ones_like(t_i).unsqueeze(-1)], dim=-1)
    out = wgt @ col
    (g,) = torch.autograd.grad((out * G).sum(), means)
    return g


def frame_stats(pos, rgb, opa, quat, scale, cam: O.Camera, loss, mode="none", variance=0.3, thresh=0.05,
                scale_activation="abs", use_sh_coeff=False, maps=False, absgrad=True, depth_key=None):
    """Statistics of one frame for the upstream loss `loss(out)`, where out = dict(padded [Hp,Wp,3] and, with maps,
    depth / alpha [Hp,Wp]) of the un-clamped padded frame: dict(grad2d [n], absgrad [n] or None, count [n] int,
    radius [n] (before ceil), vec [n,2] = (gx, gy), pix_sum [n,2] = per-pixel contributions summed without abs,
    loss).  Only parameters' values are used (no parameter gradient)."""
    fr = _front(pos.detach(), rgb.detach(), opa.detach(), quat.detach(), scale.detach(), cam, mode, variance, thresh,
                scale_activation, use_sh_coeff, depth_key)
    return _stats(fr, pos.shape[0], pos.dtype, cam, loss, use_sh_coeff, maps, absgrad)


def tile_stats(pos, rgb, opa, quat, scale, cam: O.Camera, tile_ids, tiles, loss, mode="none", variance=0.3,
               scale_activation="abs"):
    """frame_stats (RGB colour logits, no maps) restricted to the Gaussians a device frame binned into `tiles`, in the
    device's order (tile_ids[k]: its Gaussian ids of tile tiles[k]), so that binning and order parity, checked
    elsewhere, cannot enter.  Returns (U, stats over U): U the sorted ids, the statistics indexed like U."""
    dt = torch.float64
    U = torch.unique(torch.cat(tile_ids))
    p = [t[U].to(dt) for t in (pos, rgb, opa, quat, scale)]
    nq, ns, opa_a, rgb_a = O.preactivate(p[3], p[4], p[2], p[1], scale_activation, False)
    rp, rc, _ = O.global_culling(p[0], nq, ns, cam.rot.to(dt), cam.tran.to(dt), cam.near, cam.half_w, cam.half_h)
    m2 = rp[:, :2].detach().clone().requires_grad_(True)
    p_c = torch.cat([m2, rp[:, 2:]], dim=1)
    c_c, o_c, _ = F.filtered(rc, opa_a, cam, mode, variance)
    loc = torch.cat([torch.searchsorted(U, i) for i in tile_ids])
    counts = torch.zeros(cam.ntx * cam.nty, dtype=torch.int64)
    for t, i in zip(tiles, tile_ids):
        counts[t] = i.numel()
    accum = torch.zeros(cam.ntx * cam.nty + 1, dtype=torch.int64)
    accum[1:] = torch.cumsum(counts, 0)
    fr = dict(p=p_c[loc], rgb=rgb_a[loc], opa=o_c[loc], cov=c_c[loc], accum=accum.to(torch.int32), rays=(None,) * 4,
              gi=loc, m2=m2, idx=torch.arange(U.numel()), cov_vis=c_c)
    return U, _stats(fr, U.numel(), dt, cam, loss, False, False, True)


def _stats(fr, n, dt, cam, loss, use_sh_coeff, maps, absgrad):
    """The statistics of the front-end `fr` (_front's dict) for `loss`, over n Gaussians (fr["idx"] indexes them)."""
    img = O.draw(fr["p"], fr["rgb"], fr["opa"], fr["cov"], fr["accum"], cam.Hp, cam.Wp, cam.fx, cam.fy,
                 use_sh_coeff, *fr["rays"])
    out = dict(padded=img)
    if maps:
        chan = torch.stack([fr["p"][:, 2], torch.ones_like(fr["p"][:, 2]), torch.zeros_like(fr["p"][:, 2])], dim=-1)
        mp = O.draw(fr["p"], chan, fr["opa"], fr["cov"], fr["accum"], cam.Hp, cam.Wp, cam.fx, cam.fy)
        out["depth"], out["alpha"] = mp[..., 0], mp[..., 1]
    L = loss(out)
    keys = ["padded"] + (["depth", "alpha"] if maps else [])
    grads = torch.autograd.grad(L, [out[k] for k in keys] + [fr["m2"]], allow_unused=True)
    gm = grads[-1] if grads[-1] is not None else torch.zeros_like(fr["m2"])
    sx, sy = ndc_scale(cam)
    vec = torch.zeros(n, 2, dtype=dt)
    vec[fr["idx"]] = gm.detach()
    grad2d = torch.sqrt((vec[:, 0] * sx) ** 2 + (vec[:, 1] * sy) ** 2)
    gidx = fr["idx"][fr["gi"]]
    count = torch.zeros(n, dtype=torch.int64)
    count[gidx] = 1
    cv = fr["cov_vis"].detach().reshape(-1, 4)
    A = cv[:, 0] * cam.fx ** 2
    B = cv[:, 1] * cam.fx * cam.fy
    Dd = cv[:, 3] * cam.fy ** 2
    lmax = 0.5 * (A + Dd) + torch.sqrt((0.5 * (A - Dd)) ** 2 + B * B)
    radius = torch.zeros(n, dtype=dt)
    radius[fr["idx"]] = 3 * torch.sqrt(lmax.clamp(min=0))
    radius = torch.where(count > 0, radius, torch.zeros_like(radius))
    res = dict(grad2d=grad2d, count=count, radius=radius, vec=vec, loss=float(L.detach()), absgrad=None, pix_sum=None)
    if absgrad and not use_sh_coeff:
        zeros = (torch.zeros(cam.Hp, cam.Wp, 3, dtype=dt), torch.zeros(cam.Hp, cam.Wp, dtype=dt))
        Gch = [g.detach() if g is not None else zeros[k > 0] for k, g in enumerate(grads[:-1])]
        Gfull = torch.cat([g if g.dim() == 3 else g.unsqueeze(-1) for g in Gch], dim=-1)   # [Hp, Wp, C]
        absum = torch.zeros(n, 2, dtype=dt)
        pix = torch.zeros(n, 2, dtype=dt)
        for t in range(cam.ntx * cam.nty):
            s, e = int(fr["accum"][t]), int(fr["accum"][t + 1])
            if e <= s:
                continue
            ty, tx = divmod(t, cam.ntx)
            Gt = Gfull[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16].reshape(256, -1)
            g = _tile_pixel_grads(fr, t, Gt, cam)
            absum.index_add_(0, gidx[s:e], g.abs().sum(0))
            pix.index_add_(0, gidx[s:e], g.sum(0))
        res["absgrad"] = torch.sqrt((absum[:, 0] * sx) ** 2 + (absum[:, 1] * sy) ** 2)
        res["pix_sum"] = pix
    return res


def adaptive_control_stats(pos, rgb, opa, quat, scale, accum, count, taus, delete_thresh, scale_activation="abs",
                           grad_thresh=0.0002, max_radius=None, max_screen_px=None, use_clone=True, use_split=True,
                           z=None):
    """Densification scored by the statistics (gs_densify_plan_stats + gs_densify_apply with grad NULL), composed from
    oracle/densify_oracle.py's rule: a Gaussian densifies when accum / max(count, 1) >= grad_thresh (float32, as the
    kernel divides), clones are exact copies, and with max_radius a Gaussian larger than max_screen_px on screen is
    pruned like one of too low opacity.  Same outputs as densify_oracle.adaptive_control."""
    hit = accum.float() / count.clamp(min=1).float() >= grad_thresh
    grad = hit.to(pos.dtype).unsqueeze(-1).expand(-1, 3).contiguous()
    if max_radius is not None:
        opa = torch.where(max_radius.float() > max_screen_px, torch.full_like(opa, -float("inf")), opa)
    return D.adaptive_control(pos, rgb, opa, quat, scale, grad, taus, delete_thresh, scale_activation, 0.5, "max",
                              use_clone, use_split, 0.0, z)
