"""CPU restatement of the 2D Gaussian surfel frame (gs_render_forward_surfel, include/gs_b200.h).

Test infrastructure only.  fp64 torch: the surfel's M = [s_u R r0 | s_v R r1 | p_c], the ray-disk intersection and
2DGS's screen filter, alpha, the tile rectangle of the projected 3-sigma disk (evaluated in float32 like the kernel,
then gs_oracle's tile rule and exact (tile, depth, index) ordering), and a vectorised per-tile blend.  Gradients come
from autograd of this forward: the branch choice, the culling, the rectangle and the order are constants.
"""
from __future__ import annotations

import math

import torch

import gs_oracle as O
import sh_gaussian_oracle as SG

ALPHA_MIN = 1.0 / 255.0


def surfel_matrix(pos, quat, scale, cam: O.Camera, scale_activation="abs"):
    """-> (M [n,3,3] rows m_x, m_y, m_z; camera normal R r2 flipped to face the camera [n,3]; p_c [n,3])."""
    dt = pos.dtype
    rot, tran = cam.rot.to(dt), cam.tran.to(dt)
    nq, ns, _, _ = O.preactivate(quat, scale, quat[:, 0], quat[:, :3], scale_activation)
    Q = O.quat_to_rot(nq)                        # columns r0, r1, r2 (world)
    RQ = rot @ Q                                 # columns R r0, R r1, R r2
    pc = pos @ rot.T + tran
    M = torch.stack([RQ[:, :, 0] * ns[:, :1], RQ[:, :, 1] * ns[:, 1:2], pc], dim=-1)
    nc = RQ[:, :, 2]
    sgn = torch.where((nc * pc).sum(-1, keepdim=True).detach() > 0, -1.0, 1.0).to(dt)
    return M, nc * sgn, pc


def ray_hit(M, qx, qy):
    """(a, b) of pixel q = (qx, qy) on every surfel (broadcast over leading dims of qx / qy against M [..., 3, 3]):
    k = qx m_z - m_x, l = qy m_z - m_y, h = k x l; also h2."""
    mx, my, mz = M[..., 0, :], M[..., 1, :], M[..., 2, :]
    k = qx[..., None] * mz - mx
    l = qy[..., None] * mz - my
    h = torch.linalg.cross(k, l, dim=-1)
    return h


def pixel_eval(M, op, qx, qy, fx, fy):
    """Per (pixel, surfel): (alpha, z, lowpass mask, raw alpha).  qx, qy [P, 1]; M [m, 3, 3]."""
    h = ray_hit(M.unsqueeze(0), qx, qy)                       # [P, m, 3]
    h2 = h[..., 2]
    ok = h2 != 0
    h2s = torch.where(ok, h2, torch.ones_like(h2))
    a = h[..., 0] / h2s
    b = h[..., 1] / h2s
    rho3 = torch.where(ok, a * a + b * b, torch.full_like(h2, math.inf))
    z3 = M[None, :, 2, 0] * a + M[None, :, 2, 1] * b + M[None, :, 2, 2]
    cx = M[:, 0, 2] / M[:, 2, 2]
    cy = M[:, 1, 2] / M[:, 2, 2]
    dx = (qx - cx[None]) * fx
    dy = (qy - cy[None]) * fy
    rho2 = 2.0 * (dx * dx + dy * dy)
    low = (rho2 < rho3).detach()
    rho = torch.where(low, rho2, torch.where(ok, rho3, torch.zeros_like(rho3)))
    z = torch.where(low, M[None, :, 2, 2].expand_as(z3), z3)
    araw = op[None] * torch.exp(-0.5 * rho)
    araw = torch.where(low | ok, araw, torch.zeros_like(araw))
    alpha = torch.where(araw.detach() > 0.99, torch.full_like(araw, 0.99), araw)
    alpha = torch.where(alpha.detach() < ALPHA_MIN, torch.zeros_like(alpha), alpha)
    return alpha, z, low, araw


def disk_box(M):
    """Centre (ex, ey) and half extents (hx, hy) of the projected 3-sigma disk a^2 + b^2 <= 9 from the dual conic
    C* = M diag(9, 9, -1) M^T, in M's dtype, and C*22 (the box is meaningful only where C*22 < 0)."""
    u, v, p = M[:, :, 0], M[:, :, 1], M[:, :, 2]
    c = lambda i, j: 9.0 * (u[:, i] * u[:, j] + v[:, i] * v[:, j]) - p[:, i] * p[:, j]
    c22, c00, c11, c02, c12 = c(2, 2), c(0, 0), c(1, 1), c(0, 2), c(1, 2)
    c22s = torch.where(c22 < 0, c22, -torch.ones_like(c22))
    ex, ey = c02 / c22s, c12 / c22s
    hx = torch.sqrt(torch.clamp(ex * ex - c00 / c22s, min=0.0))
    hy = torch.sqrt(torch.clamp(ey * ey - c11 / c22s, min=0.0))
    return ex, ey, hx, hy, c22


def surfel_rects(M, cam: O.Camera, visible):
    """Tile rectangle per surfel (float32 like the kernel): box of the 3-sigma disk from C* = M diag(9,9,-1) M^T joined
    with the sqrt(2)/2 px box around the centre; C*22 >= 0 or invisible: empty.  -> (tx0, tx1, ty0, ty1) int64."""
    f32 = torch.float32
    Mf = M.detach().to(f32)
    p = Mf[:, :, 2]
    ex, ey, hx, hy, c22 = disk_box(Mf)
    ok = (c22 < 0) & visible
    cx, cy = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
    rx = torch.tensor(0.70710678, dtype=f32) / torch.tensor(cam.fx, dtype=f32)
    ry = torch.tensor(0.70710678, dtype=f32) / torch.tensor(cam.fy, dtype=f32)
    left, right = torch.minimum(ex - hx, cx - rx), torch.maximum(ex + hx, cx + rx)
    top, bottom = torch.minimum(ey - hy, cy - ry), torch.maximum(ey + hy, cy + ry)
    lx, ly = torch.tensor(cam.tile_lx, dtype=f32), torch.tensor(cam.tile_ly, dtype=f32)
    lm, tm = torch.tensor(cam.leftmost, dtype=f32), torch.tensor(cam.topmost, dtype=f32)

    def lo(x):
        return torch.nan_to_num(torch.clamp(x, min=0.0), nan=0.0).clamp(max=2.0e9).floor().to(torch.int64)

    def hi(x):
        return torch.nan_to_num(torch.clamp(x + 1.0, min=0.0), nan=0.0).clamp(max=2.0e9).floor().to(torch.int64)

    ty0, tx0 = lo((top - tm) / ly), lo((left - lm) / lx)
    ty1 = torch.minimum(hi((bottom - tm) / ly), torch.tensor(cam.nty))
    tx1 = torch.minimum(hi((right - lm) / lx), torch.tensor(cam.ntx))
    empty = ~ok | (ty1 <= ty0) | (tx1 <= tx0)
    ty1 = torch.where(empty, ty0, ty1)
    tx1 = torch.where(empty, tx0, tx1)
    return tx0, tx1, ty0, ty1


def without_branch_ties(g, cam, tol=1e-5):
    """g without the surfels that have a pixel where the screen filter and the intersection tie (|rho2 - rho3| <
    tol rho3) at an alpha above the skip threshold.  The model's gradient jumps where the branch changes, so at such a
    pixel an fp32 and an fp64 evaluation may take different branches and both be right; a surfel with a projected std
    near sqrt(2)/2 px has them."""
    p = {k: v.double() for k, v in g.items()}
    M, _, _ = surfel_matrix(p["pos"], p["quat"], p["scale"], cam)
    ys, xs = torch.meshgrid(torch.arange(cam.Hp, dtype=torch.float64), torch.arange(cam.Wp, dtype=torch.float64),
                            indexing="ij")
    qx = ((xs + 0.5 - cam.Wp // 2) / cam.fx).reshape(-1, 1)
    qy = ((ys + 0.5 - cam.Hp // 2) / cam.fy).reshape(-1, 1)
    _, _, _, araw = pixel_eval(M, p["opa"].sigmoid(), qx, qy, cam.fx, cam.fy)
    h = ray_hit(M.unsqueeze(0), qx, qy)
    h2 = torch.where(h[..., 2] != 0, h[..., 2], torch.ones_like(h[..., 2]))
    rho3 = (h[..., 0] ** 2 + h[..., 1] ** 2) / h2 ** 2
    cx, cy = M[:, 0, 2] / M[:, 2, 2], M[:, 1, 2] / M[:, 2, 2]
    rho2 = 2.0 * (((qx - cx[None]) * cam.fx) ** 2 + ((qy - cy[None]) * cam.fy) ** 2)
    tie = ((rho2 - rho3).abs() < tol * rho3) & (araw >= ALPHA_MIN) & (h[..., 2] != 0)
    keep = ~tie.any(0)
    return {k: v[keep].contiguous() for k, v in g.items()}


def distortion_m(z, near, far):
    return far / (far - near) * (1.0 - near / z)


def render(pos, rgb, opa, quat, scale, cam: O.Camera, thresh=0.05, scale_activation="abs", background=None,
           dist_near=0.2, dist_far=100.0, tiles=None, depth_key=None):
    """-> (image [Hp,Wp,3] padded, un-clamped; maps dict of [Hp,Wp] / normal [Hp,Wp,3]; info dict).  rgb [n,3]
    logits or [n,27|48] per-Gaussian SH coefficients.  tiles: blend only those tile indices (the others stay 0, with
    no gradient); binning and order are those of the whole frame.  depth_key [n]: the sort key (default: the float32
    camera z of each centre)."""
    dt = pos.dtype
    M, nrm, pc = surfel_matrix(pos, quat, scale, cam, scale_activation)
    op = opa.sigmoid()
    col = (rgb if rgb.shape[1] == 3 else SG.gaussian_logits(pos, rgb, cam)).sigmoid()
    pcd = pc.detach()
    zc = pcd[:, 2]
    zs = torch.where(zc > cam.near, zc, torch.ones_like(zc))
    visible = (zc > cam.near) & ((pcd[:, 0] / zs).abs() < cam.half_w) & ((pcd[:, 1] / zs).abs() < cam.half_h)
    rects = surfel_rects(M, cam, visible)
    key = (pos.detach().float() @ cam.rot.float().T + cam.tran.float())[:, 2] if depth_key is None else depth_key
    gi, accum = O.bin_and_sort(torch.stack([key, key, key], -1), None, rects, cam.ntx, cam.nty, depth_key=key)
    bg = torch.zeros(3, dtype=dt) if background is None else torch.tensor(background, dtype=dt)
    Hp, Wp = cam.Hp, cam.Wp
    img = torch.zeros(cam.nty, cam.ntx, 256, 3, dtype=dt)
    names = ("alpha", "depth", "median", "distortion")
    mp = {k: torch.zeros(cam.nty, cam.ntx, 256, dtype=dt) for k in names}
    mp["normal"] = torch.zeros(cam.nty, cam.ntx, 256, 3, dtype=dt)
    acc = accum.to(torch.int64)
    r16 = torch.arange(16, dtype=dt)
    for t in range(cam.ntx * cam.nty) if tiles is None else tiles:
        s, e = int(acc[t]), int(acc[t + 1])
        ty, tx = divmod(t, cam.ntx)
        ix = (tx * 16 + r16).reshape(1, 16).expand(16, 16).reshape(-1, 1)
        iy = (ty * 16 + r16).reshape(16, 1).expand(16, 16).reshape(-1, 1)
        qx = (ix + 0.5 - (Wp // 2)) / cam.fx
        qy = (iy + 0.5 - (Hp // 2)) / cam.fy
        if e <= s:
            img[ty, tx] = bg.expand(256, 3)
            continue
        g = gi[s:e]
        alpha, z, _, _ = pixel_eval(M[g], op[g], qx, qy, cam.fx, cam.fy)
        alpha = torch.where(z.detach() > cam.near, alpha, torch.zeros_like(alpha))   # no hit behind the near plane
        one_m = 1 - alpha
        Tinc = torch.cumprod(one_m, dim=1)
        Texc = torch.cat([torch.ones(256, 1, dtype=dt), Tinc[:, :-1]], dim=1)
        live = (Texc.detach() > 1e-4).to(dt)
        w = alpha * Texc * live
        Tf = torch.prod(1 - alpha * live, dim=1)
        img[ty, tx] = w @ col[g] + Tf[:, None] * bg
        mp["alpha"][ty, tx] = 1 - Tf
        mp["depth"][ty, tx] = (w * z).sum(1)
        mp["normal"][ty, tx] = w @ nrm[g]
        blended = (live > 0) & (alpha.detach() > 0) & (Texc.detach() > 0.5)
        idx = torch.arange(e - s).expand(256, -1)
        last = torch.where(blended, idx, torch.full_like(idx, -1)).max(dim=1).values
        has = last >= 0
        zmed = torch.gather(z, 1, last.clamp(min=0)[:, None])[:, 0]
        mp["median"][ty, tx] = torch.where(has, zmed, torch.zeros_like(zmed))
        m = distortion_m(z, dist_near, dist_far)
        A = torch.cumsum(w, 1) - w
        D = torch.cumsum(w * m, 1) - w * m
        D2 = torch.cumsum(w * m * m, 1) - w * m * m
        mp["distortion"][ty, tx] = (w * (m * m * A - 2 * m * D + D2)).sum(1)

    def unt(x):
        ch = x.shape[3:] if x.dim() > 3 else ()
        y = x.reshape(cam.nty, cam.ntx, 16, 16, *ch).permute(0, 2, 1, 3, *range(4, 4 + len(ch)))
        return y.reshape(Hp, Wp, *ch)

    info = dict(gauss_idx=gi, accum=accum, visible=visible, rects=rects, M=M, op=op, col=col, nrm=nrm)
    return unt(img), {k: unt(v) for k, v in mp.items()}, info
