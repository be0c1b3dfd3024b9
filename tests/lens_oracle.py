"""CPU fp64 oracle of the fused frame path's camera lenses (gs_ctx_set_lens, `Splatter(camera_model="colmap")`).

Test infrastructure only, with no blend code of its own: the projection is restated here, and the tile rule, binning
and blend are gs_oracle's `tile_rects`, `bin_and_sort` and `draw`.  With (a, b) = (x/z, y/z) and rho = |(a, b)|:

- `lens_map`: COLMAP's OPENCV (k1, k2, p1, p2) and OPENCV_FISHEYE (k1..k4) maps (a, b) -> (a_d, b_d), differentiable;
  the fisheye factor theta_d / rho is taken from its series near the axis.
- `lens_jacobian`: J_D = d(a_d, b_d) / d(a, b) in closed form.
- `rho_max`: where the radial polynomial folds back, from `numpy.roots` of its derivative.
- `global_culling_lens`: the stored mean (a_d + (cx - W/2) / fx, b_d + (cy - H/2) / fy), the depth |p_c| and the 2-D
  covariance J_D J W Sigma W^T J^T J_D^T with J_D J detached (the backward's convention), and the culling mask
  (z > near, rho < rho_max, the stored mean inside the 1.2x frustum).
- `render`: a whole frame (clamped and cropped, or the padded raw image and the culling mask), whose gradients come
  from autograd.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import gs_oracle as O

PINHOLE, OPENCV, FISHEYE = 0, 1, 2
MODELS = {"PINHOLE": PINHOLE, "OPENCV": OPENCV, "FISHEYE": FISHEYE}
SERIES_R2 = 1e-4   # fisheye: below this rho^2 the factor and its derivative come from their series


def _model(m):
    return MODELS[m] if isinstance(m, str) else int(m)


def _fisheye_fg(r2, k):
    """f = theta_d / rho and g = f'(rho) / rho of the fisheye map, as functions of r2 = rho^2 (finite at 0)."""
    k1, k2, k3, k4 = k
    small = r2 < SERIES_R2
    rs = torch.where(small, torch.ones_like(r2), r2)          # keeps the closed form's branch finite (autograd)
    rho = rs.sqrt()
    th = torch.atan(rho)
    t2 = th * th
    poly = 1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))
    dpoly = 1 + t2 * (3 * k1 + t2 * (5 * k2 + t2 * (7 * k3 + t2 * 9 * k4)))
    thd = th * poly
    f_cf = thd / rho
    g_cf = (dpoly * rho / (1 + rs) - thd) / (rs * rho)
    c1, c2 = k1 - 1.0 / 3.0, 0.2 - k1 + k2
    f_s = 1 + c1 * r2 + c2 * r2 * r2
    g_s = 2 * c1 + 4 * c2 * r2
    return torch.where(small, f_s, f_cf), torch.where(small, g_s, g_cf)


def lens_map(a, b, model, k):
    """(a_d, b_d) of COLMAP's model at (a, b) (tensors of one shape), differentiable."""
    m = _model(model)
    k = [float(x) for x in k]
    if m == PINHOLE:
        return a, b
    r2 = a * a + b * b
    if m == OPENCV:
        k1, k2, p1, p2 = k
        rad = 1 + r2 * (k1 + k2 * r2)
        return (a * rad + 2 * p1 * a * b + p2 * (r2 + 2 * a * a),
                b * rad + p1 * (r2 + 2 * b * b) + 2 * p2 * a * b)
    f, _ = _fisheye_fg(r2, k)
    return f * a, f * b


def lens_jacobian(a, b, model, k):
    """J_D [..., 2, 2] = d(a_d, b_d) / d(a, b) in closed form."""
    m = _model(model)
    k = [float(x) for x in k]
    one, zero = torch.ones_like(a), torch.zeros_like(a)
    if m == PINHOLE:
        J = [one, zero, zero, one]
    elif m == OPENCV:
        k1, k2, p1, p2 = k
        r2 = a * a + b * b
        rad = 1 + r2 * (k1 + k2 * r2)
        drad = 2 * k1 + 4 * k2 * r2
        j01 = drad * a * b + 2 * p1 * a + 2 * p2 * b
        J = [rad + drad * a * a + 2 * p1 * b + 6 * p2 * a, j01, j01, rad + drad * b * b + 6 * p1 * b + 2 * p2 * a]
    else:
        f, g = _fisheye_fg(a * a + b * b, k)
        J = [f + g * a * a, g * a * b, g * a * b, f + g * b * b]
    return torch.stack(J, dim=-1).reshape(a.shape + (2, 2))


def rho_max(model, k):
    """The undistorted radius past which the map folds back (math.inf: none).  OPENCV: the smallest rho > 0 with
    1 + 3 k1 rho^2 + 5 k2 rho^4 = 0; FISHEYE: tan of the smallest theta in (0, pi/2) with d theta_d / d theta = 0."""
    m = _model(model)
    k = [float(x) for x in k]
    if m == OPENCV:
        coef = [5 * k[1], 3 * k[0], 1.0]                       # in u = rho^2, highest power first
        lim = math.inf
    elif m == FISHEYE:
        coef = [9 * k[3], 7 * k[2], 5 * k[1], 3 * k[0], 1.0]   # in t = theta^2
        lim = (math.pi / 2) ** 2
    else:
        return math.inf
    while coef and coef[0] == 0.0:
        coef = coef[1:]
    roots = np.roots(coef) if len(coef) > 1 else []
    pos = [r.real for r in roots if abs(r.imag) <= 1e-12 * max(1.0, abs(r)) and r.real > 0 and r.real < lim]
    if not pos:
        return math.inf
    u = min(pos)
    return math.sqrt(u) if m == OPENCV else math.tan(math.sqrt(u))


def offsets(lens, width, height, fx, fy):
    """(ox, oy) = ((cx - W/2) / fx, (cy - H/2) / fy)."""
    return (float(lens["cx"]) - width / 2.0) / fx, (float(lens["cy"]) - height / 2.0) / fy


def global_culling_lens(pos, quat_n, scale_a, rot, tran, near, half_width, half_height, lens, ox, oy):
    """gs_oracle.global_culling through a lens: res_pos [N, 3] = (stored mean, |p_c|), res_cov [N, 2, 2], mask [N]
    int64 (culled rows 0).  J_D J is detached in the covariance; the mean is live through the lens."""
    model, k = lens["model"], lens.get("k", [0.0] * 4)
    pc = pos @ rot.T + tran
    x, y, z = pc.unbind(-1)
    front = z > near
    zs = torch.where(front, z, torch.ones_like(z))
    a, b = x / zs, y / zs
    ad, bd = lens_map(a, b, model, k)
    mx, my = ad + ox, bd + oy
    r = pc.norm(dim=-1)
    rm = rho_max(model, k)
    mask = front & ((a * a + b * b) < rm * rm) & (mx.abs() < half_width) & (my.abs() < half_height)
    R = O.quat_to_rot(quat_n)
    RS = R * scale_a.unsqueeze(-2)
    cov3 = RS @ RS.transpose(-1, -2)
    pcd = pc.detach()
    xd, yd, zd = pcd.unbind(-1)
    zd = torch.where(mask, zd, torch.ones_like(zd))
    zero = torch.zeros_like(xd)
    J = torch.stack([1 / zd, zero, -xd / (zd * zd), zero, 1 / zd, -yd / (zd * zd)], dim=-1).reshape(-1, 2, 3)
    JD = lens_jacobian(xd / zd, yd / zd, model, k)
    M = JD @ J @ rot
    cov2 = M @ cov3 @ M.transpose(-1, -2)
    m = mask.to(pos.dtype)
    res_pos = torch.stack([mx, my, r], dim=-1) * m.unsqueeze(-1)
    return res_pos, cov2 * m.reshape(-1, 1, 1), mask.to(torch.int64)


def render(pos, rgb, opa, quat, scale, cam: O.Camera, lens, thresh=0.05, scale_activation="abs", use_sh_coeff=False,
           depth_key=None):
    """gs_oracle.render through `lens` (dict(model, cx, cy, k)): (clamped cropped image, aux dict(padded, mask))."""
    dt = pos.dtype
    rot, tran = cam.rot.to(dt), cam.tran.to(dt)
    nq, ns, opa_a, rgb_a = O.preactivate(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
    ox, oy = offsets(lens, cam.width, cam.height, cam.fx, cam.fy)
    rp, rc, mask = global_culling_lens(pos, nq, ns, rot, tran, cam.near, cam.half_w, cam.half_h, lens, ox, oy)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    p_c, c_c, rgb_c, opa_c = rp[idx], rc[idx], rgb_a[idx], opa_a[idx]
    rects = O.tile_rects(p_c[:, :2], c_c, thresh, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                         cam.topmost)
    gi, accum = O.bin_and_sort(p_c, c_c, rects, cam.ntx, cam.nty, None if depth_key is None else depth_key[idx])
    rays = (None,) * 4
    if use_sh_coeff:
        rays_o, lefttop, dx, dy = O.ray_info(rot, tran, cam.Hp, cam.Wp, cam.fx, cam.fy)
        lefttop = lefttop - torch.inverse(rot) @ torch.tensor([ox, oy, 0.0], dtype=dt)
        rays = (rays_o, lefttop, dx, dy)
    img = O.draw(p_c[gi], rgb_c[gi], opa_c[gi], c_c[gi], accum, cam.Hp, cam.Wp, cam.fx, cam.fy, use_sh_coeff, *rays)
    return cam.crop(torch.clamp(img, 0, 1)), dict(padded=img, mask=mask, res_pos=rp, rects=rects, idx=idx)


def _view_geometry(p, c):
    R = np.asarray(c["rot"], dtype=np.float32).astype(np.float64).reshape(3, 3)
    t = np.asarray(c["tran"], dtype=np.float32).astype(np.float64).reshape(3)
    pc = p @ R.T + t
    return pc, pc[:, 2]


def sampling_filter_lens(pos, cams, lenses, margin=0.15, variance=0.2):
    """gs_filter3d_compute with lenses, in fp64: (f [n], seen [n] bool).  View c (a dict like filter3d_oracle's, with
    near) and its lens (dict(model, cx, cy, k)) see Gaussian i when z > near, rho < rho_max and the distorted pixel
    position (fx a_d + cx, fy b_d + cy) lies inside the image widened by `margin`.  The rate is fx / z, or for FISHEYE
    fx max(theta_d'(theta), theta_d(theta) / sin theta) / |p_c|."""
    p = np.asarray(pos, dtype=np.float32).astype(np.float64)
    n = p.shape[0]
    m = float(np.float32(margin))
    nu = np.zeros(n)
    for c, ln in zip(cams, lenses):
        pc, z = _view_geometry(p, c)
        W, H = float(c["width"]), float(c["height"])
        fx, fy = float(np.float32(c["focal_x"])), float(np.float32(c["focal_y"]))
        near = float(np.float32(c["near"]))
        k = [float(np.float32(x)) for x in ln["k"]]
        cx, cy = float(np.float32(ln["cx"])), float(np.float32(ln["cy"]))
        front = z > near
        zs = np.where(front, z, 1.0)
        a, b = pc[:, 0] / zs, pc[:, 1] / zs
        ad, bd = lens_map(torch.from_numpy(a), torch.from_numpy(b), ln["model"], k)
        u, w = fx * ad.numpy() + cx, fy * bd.numpy() + cy
        rm = rho_max(ln["model"], k)
        seen = front & (a * a + b * b < rm * rm) & (u >= -m * W) & (u <= (1 + m) * W) & (w >= -m * H) & (w <= (1 + m) * H)
        if _model(ln["model"]) == FISHEYE:
            r = np.hypot(pc[:, 0], pc[:, 1])
            th = np.arctan2(r, z)
            t2 = th * th
            poly = 1 + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3])))
            dpoly = 1 + t2 * (3 * k[0] + t2 * (5 * k[1] + t2 * (7 * k[2] + t2 * 9 * k[3])))
            with np.errstate(divide="ignore", invalid="ignore"):
                tang = np.where(th > 0, th * poly / np.sin(np.where(th > 0, th, 1.0)), 1.0)
            rate = fx * np.maximum(dpoly, tang) / np.linalg.norm(pc, axis=1)
        else:
            rate = fx / zs
        nu = np.maximum(nu, np.where(seen, rate, 0.0))
    seen = nu > 0
    if not seen.any():
        return np.zeros(n), seen
    nu = np.where(seen, nu, nu[seen].min())
    return math.sqrt(float(np.float32(variance))) / nu, seen


def sampling_ties_lens(pos, cams, lenses, margin=0.15, tol=2e-5):
    """[n] bool: Gaussians within a relative `tol` of a view's near plane, rho_max or margin edge (distorted), where the
    device's fp32 test and the fp64 one may disagree."""
    p = np.asarray(pos, dtype=np.float32).astype(np.float64)
    m = float(np.float32(margin))
    tie = np.zeros(p.shape[0], dtype=bool)
    for c, ln in zip(cams, lenses):
        pc, z = _view_geometry(p, c)
        W, H = float(c["width"]), float(c["height"])
        fx, fy = float(np.float32(c["focal_x"])), float(np.float32(c["focal_y"]))
        near = float(np.float32(c["near"]))
        tie |= np.abs(z - near) <= tol * (np.abs(z) + near)
        front = z > near
        zs = np.where(front, z, 1.0)
        a, b = pc[:, 0] / zs, pc[:, 1] / zs
        rho = np.hypot(a, b)
        rm = rho_max(ln["model"], ln["k"])
        if math.isfinite(rm):
            tie |= front & (np.abs(rho - rm) <= tol * rm)
        ad, bd = lens_map(torch.from_numpy(a), torch.from_numpy(b), ln["model"], ln["k"])
        u, w = fx * ad.numpy() + ln["cx"], fy * bd.numpy() + ln["cy"]
        for val, lo, hi, span in ((u, -m * W, (1 + m) * W, W), (w, -m * H, (1 + m) * H, H)):
            tol_px = tol * (np.abs(val) + span)
            tie |= front & ((np.abs(val - lo) <= tol_px) | (np.abs(val - hi) <= tol_px))
    return tie
