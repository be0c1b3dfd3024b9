"""CPU oracle for the differentiable tile rasterizer hot path.

TEST INFRASTRUCTURE ONLY — never imported by the product path
(`3d-gaussian-splatting_b200/`).  Only `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py` may import this module.

It is a plain-PyTorch (CPU, fp32 or fp64) restatement of the algorithm of
WangFeng18/3d-gaussian-splatting's hot path; every function cites the reference
file:line it follows.  It is NOT a port of the CUDA code: per-tile blending is
vectorised as  T = exclusive-cumprod(1 - alpha)  with the early-stop mask
`T >= 1e-4` held constant, and all gradients come from autograd of that forward
(SURVEY.md §8c shows this equals the reference's hand-derived backward).

Parity pinning: the reference ships no tests/golden vectors (SURVEY.md §4), and its
kernels are CUDA-only, so this oracle is pinned against outputs of the reference's
own CUDA build (oracle/_ref, built by oracle/build_ref.py) generated on a GPU by
tests/golden/make_golden.py and committed under tests/golden/*.npz.
Until those fixtures exist the status is "parity unpinned".
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

EPS = 1e-4  # splatter.py:19


# --------------------------------------------------------------------------------------
# a1  pre-activations  (splatter.py:519-524, 539-540; renderer.py:91-100)
# --------------------------------------------------------------------------------------
class _TruncExp(torch.autograd.Function):
    """renderer.py:91-100: fwd exp(x); bwd g*exp(clamp(x,-1,1))."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(-1, 1))


def preactivate(quat, scale, opa, rgb, scale_activation="abs", use_sh_coeff=False):
    """splatter.py:519-524 (quat/scale) and :539-540 (sigmoid on opa, on rgb unless SH)."""
    nq = quat / quat.norm(dim=1, keepdim=True)
    if scale_activation == "abs":
        ns = scale.abs() + EPS
    else:
        ns = _TruncExp.apply(scale)
    return nq, ns, opa.sigmoid(), (rgb if use_sh_coeff else rgb.sigmoid())


# --------------------------------------------------------------------------------------
# a2/a13  projection + culling  (gaussian.cu:1131-1336; backward :1371-1576)
# --------------------------------------------------------------------------------------
def quat_to_rot(q):
    """wxyz -> R, gaussian.cu:1231-1245 (== utils.py:318-333)."""
    w, x, y, z = q.unbind(-1)
    R = torch.stack([
        1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w,
        2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w,
        2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y,
    ], dim=-1)
    return R.reshape(q.shape[:-1] + (3, 3))


def global_culling(pos, quat_n, scale_a, rot, tran, near, half_width, half_height):
    """gaussian.cu:1182-1336.  quat_n / scale_a are the PRE-ACTIVATED tensors.

    Returns res_pos[N,3] (x/z, y/z, |p_c|), res_cov[N,2,2], mask[N] int64; culled rows 0
    (the caller zero-fills, renderer.py:124-126).  The Jacobian is DETACHED: the
    reference's backward does not propagate d cov2d / d pos (gaussian.cu:1397-1421).
    """
    pc = pos @ rot.T + tran                                   # :1131-1154
    x, y, z = pc.unbind(-1)
    zs = torch.where(z > near, z, torch.ones_like(z))         # avoid inf on culled rows
    pix = x / zs
    piy = y / zs
    r = pc.norm(dim=-1)
    mask = (z > near) & (pix.abs() < half_width) & (piy.abs() < half_height)   # :1208,:1220
    R = quat_to_rot(quat_n)
    RS = R * scale_a.unsqueeze(-2)                            # R @ diag(s)  :1259-1270
    cov3 = RS @ RS.transpose(-1, -2)                          # :1272-1283
    pcd = pc.detach()
    xd, yd, zd = pcd.unbind(-1)
    zd = torch.where(mask, zd, torch.ones_like(zd))
    rd = pcd.norm(dim=-1).clamp_min(1e-30)
    zero = torch.zeros_like(xd)
    J = torch.stack([1 / zd, zero, -xd / (zd * zd),
                     zero, 1 / zd, -yd / (zd * zd),
                     xd / rd, yd / rd, zd / rd], dim=-1).reshape(-1, 3, 3)      # :1156-1180
    JW = J @ rot                                              # :1292-1303
    cov2 = (JW @ cov3 @ JW.transpose(-1, -2))[:, :2, :2]      # :1305-1335
    m = mask.to(pos.dtype)
    res_pos = torch.stack([pix, piy, r], dim=-1) * m.unsqueeze(-1)
    res_cov = cov2 * m.reshape(-1, 1, 1)
    return res_pos, res_cov, mask.to(torch.int64)


# --------------------------------------------------------------------------------------
# a5  tile binning rule, method 2 "prob2"  (gaussian.cu:197-250)
# --------------------------------------------------------------------------------------
def tile_rects(pos2d, cov, thresh, tile_length_x, tile_length_y, n_tiles_x, n_tiles_y, leftmost, topmost):
    """Per-Gaussian covered tile rectangle [tx0,tx1) x [ty0,ty1) (empty if det<=0).

    Follows the float32 expression order of gaussian.cu:226-242 (the `1e-14` literal
    makes the two divisions double precision, :229-232); float->uint32 casts truncate
    and saturate at 0 like the CUDA cvt.
    """
    f32 = torch.float32
    pos2d = pos2d.detach().to(f32)
    cov = cov.detach().to(f32).reshape(-1, 4)
    a, b, c, d = cov.unbind(-1)
    cx, cy = pos2d[:, 0], pos2d[:, 1]
    det = a * d - b * c
    ok = det > 0
    detd = det.double() + 1e-14
    _ai = (d.double() / detd).to(f32)
    _di = (a.double() / detd).to(f32)
    t = torch.tensor(-2.0, dtype=f32) * torch.log(torch.tensor(thresh, dtype=f32))   # -2*logf(thr) :233
    shift_x = torch.sqrt(_di * t * det)
    shift_y = torch.sqrt(_ai * t * det)
    right, left = cx + shift_x, cx - shift_x
    top, bottom = cy - shift_y, cy + shift_y
    lx = torch.tensor(tile_length_x, dtype=f32)
    ly = torch.tensor(tile_length_y, dtype=f32)
    lm = torch.tensor(leftmost, dtype=f32)
    tm = torch.tensor(topmost, dtype=f32)

    def lo(v):      # uint32 i = fmaxf(v, 0)
        return torch.nan_to_num(torch.clamp(v, min=0.0), nan=0.0).clamp(max=2.0e9).floor().to(torch.int64)

    def hi(v):      # (uint32)(v + 1)
        return torch.nan_to_num(torch.clamp(v + 1.0, min=0.0), nan=0.0).clamp(max=2.0e9).floor().to(torch.int64)

    ty0 = lo((top - tm) / ly)
    ty1 = torch.minimum(hi((bottom - tm) / ly), torch.tensor(n_tiles_y))
    tx0 = lo((left - lm) / lx)
    tx1 = torch.minimum(hi((right - lm) / lx), torch.tensor(n_tiles_x))
    ty1 = torch.where(ok, ty1, ty0)
    tx1 = torch.where(ok, tx1, tx0)
    ty1 = torch.maximum(ty1, ty0)
    tx1 = torch.maximum(tx1, tx0)
    return tx0, tx1, ty0, ty1


def bin_and_sort(pos_img, cov, rects, n_tiles_x, n_tiles_y, depth_key=None):
    """Exact (tile, depth, index) ordering of all tile-instances.

    The reference appends by atomics (gaussian.cu:244-247) and sorts an fp32 composite
    key (splatter.py:610-613); the exact order here is a valid refinement of it
    (SURVEY.md §8c P3).  Returns (gauss_idx[M] int64, tile_n_point_accum[T+1] int32).
    """
    tx0, tx1, ty0, ty1 = rects
    w = (tx1 - tx0)
    h = (ty1 - ty0)
    cnt = w * h
    M = int(cnt.sum())
    T = n_tiles_x * n_tiles_y
    if M == 0:
        return torch.zeros(0, dtype=torch.int64), torch.zeros(T + 1, dtype=torch.int32)
    g = torch.repeat_interleave(torch.arange(cnt.numel()), cnt)
    start = torch.cumsum(cnt, 0) - cnt
    rank = torch.arange(M) - start[g]
    wg = w[g]
    tile = (ty0[g] + rank // wg) * n_tiles_x + (tx0[g] + rank % wg)
    # The order is defined on float32 depth keys.  Two Gaussians whose depths differ by an ulp can
    # swap between an fp64 and an fp32 evaluation of |p_c|; tests therefore may pass the device's
    # own fp32 depths (`depth_key`, one per row of pos_img) so that both sides sort identical keys.
    dk = pos_img[:, 2].detach().to(torch.float32) if depth_key is None else depth_key.to(torch.float32)
    depth = dk[g]
    # exact lexicographic (tile, depth, index): stable sorts, least-significant first
    order = torch.argsort(g, stable=True)
    order = order[torch.argsort(depth[order], stable=True)]
    order = order[torch.argsort(tile[order], stable=True)]
    counts = torch.bincount(tile, minlength=T)
    accum = torch.zeros(T + 1, dtype=torch.int64)
    accum[1:] = torch.cumsum(counts, 0)
    return g[order], accum.to(torch.int32)


# --------------------------------------------------------------------------------------
# SH basis (gaussian.cu:385-426, svox2 convention) and ray setup (splatter.py:305-321)
# --------------------------------------------------------------------------------------
C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)


def sh_basis9(d):
    x, y, z = d.unbind(-1)
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    return torch.stack([
        torch.full_like(x, C0), -C1 * y, C1 * z, -C1 * x,
        C2[0] * xy, C2[1] * yz, C2[2] * (2.0 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy)], dim=-1)


C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)


def sh_basis16(d):
    """Degree-3 extension (svox2 convention; the reference defines C3 at gaussian.cu:395-403 but
    never evaluates it)."""
    x, y, z = d.unbind(-1)
    xx, yy, zz, xy = x * x, y * y, z * z, x * y
    hi = torch.stack([
        C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy),
        C3[3] * z * (2 * zz - 3 * xx - 3 * yy), C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy),
        C3[6] * x * (xx - 3 * yy)], dim=-1)
    return torch.cat([sh_basis9(d), hi], dim=-1)


def ray_info(rot, tran, Hp, Wp, fx, fy):
    """splatter.py:305-321 -> rays_o, lefttop, dx, dy (world space)."""
    c2w = torch.inverse(rot)
    rays_o = -c2w @ tran
    lefttop_cam = torch.tensor([(-Wp / 2 + 0.5) / fx, (-Hp / 2 + 0.5) / fy, 1.0], dtype=rot.dtype)
    lefttop = c2w @ (lefttop_cam - tran)
    dx = c2w @ torch.tensor([1.0 / fx, 0, 0], dtype=rot.dtype)
    dy = c2w @ torch.tensor([0, 1.0 / fy, 0], dtype=rot.dtype)
    return rays_o, lefttop, dx, dy


# --------------------------------------------------------------------------------------
# a10/a11  per-tile front-to-back alpha blend  (gaussian.cu:806-970; backward :440-803)
# --------------------------------------------------------------------------------------
def draw(pos, rgb, opa, cov, tile_n_point_accum, Hp, Wp, fx, fy,
         use_sh_coeff=False, rays_o=None, lefttop=None, vec_dx=None, vec_dy=None,
         tiles: Optional[torch.Tensor] = None):
    """Blend already sorted per-instance tensors exactly like `draw_kernel`.

    pos[M,3] (x,y used), rgb[M,3|27], opa[M], cov[M,2,2]; returns image[Hp,Wp,3]
    (un-clamped, black background).  Flags weight_normalize/sigmoid are the
    always-False ones (splatter.py:627, train.py:377) and are not modelled.
    `tiles`: optional subset of tile ids to render (others stay 0) — used for the
    bounded CPU-baseline sample.
    """
    dt = pos.dtype
    ntx, nty = Wp // 16, Hp // 16
    accum = tile_n_point_accum.to(torch.int64)
    cov4 = cov.reshape(-1, 4)
    ix = torch.arange(16)
    out_tiles = []
    tile_ids = range(ntx * nty) if tiles is None else [int(t) for t in tiles]
    img = torch.zeros(nty, ntx, 16, 16, 3, dtype=dt)
    for t in tile_ids:
        s, e = int(accum[t]), int(accum[t + 1])
        if e <= s:
            continue
        ty, tx = divmod(t, ntx)
        idx_x = (tx * 16 + ix).to(dt)
        idx_y = (ty * 16 + ix).to(dt)
        px = ((idx_x + 0.5 - (Wp // 2)) / fx)            # :839
        py = ((idx_y + 0.5 - (Hp // 2)) / fy)            # :840
        PX = px.reshape(1, 16).expand(16, 16).reshape(-1, 1)   # pixel p = y*16+x
        PY = py.reshape(16, 1).expand(16, 16).reshape(-1, 1)
        a, b, c, d = cov4[s:e].unbind(-1)
        X = PX - pos[s:e, 0].reshape(1, -1)
        Y = PY - pos[s:e, 1].reshape(1, -1)
        det = a * d - b * c
        power = -(d * X * X - (b + c) * X * Y + a * Y * Y) / (2 * det + 1e-14)    # :920
        alpha = torch.exp(power) * opa[s:e].reshape(1, -1)                        # :926
        one_m = 1 - alpha
        Tinc = torch.cumprod(one_m, dim=1)
        Texc = torch.cat([torch.ones(256, 1, dtype=dt), Tinc[:, :-1]], dim=1)
        live = (Texc.detach() >= 0.0001).to(dt)                                   # :906
        wgt = alpha * Texc * live                                                 # :932
        if use_sh_coeff:
            gx = (tx * 16 + ix).to(dt).reshape(1, 16).expand(16, 16).reshape(-1, 1)
            gy = (ty * 16 + ix).to(dt).reshape(16, 1).expand(16, 16).reshape(-1, 1)
            dirs = lefttop.reshape(1, 3) + gx * vec_dx.reshape(1, 3) + gy * vec_dy.reshape(1, 3) - rays_o.reshape(1, 3)
            dirs = dirs / (dirs.norm(dim=-1, keepdim=True) + 1e-7)                # :852-859
            K = rgb.shape[1] // 3
            SH = sh_basis9(dirs) if K == 9 else sh_basis16(dirs)                  # [256,K]
            coef = rgb[s:e].reshape(-1, 3, K)
            col = torch.sigmoid(torch.einsum("pk,nck->pnc", SH, coef))            # :936-948
            tile_rgb = (wgt.unsqueeze(-1) * col).sum(1)
        else:
            tile_rgb = wgt @ rgb[s:e]                                             # :954-956
        img[ty, tx] = tile_rgb.reshape(16, 16, 3)
    return img.permute(0, 2, 1, 3, 4).reshape(Hp, Wp, 3)


# --------------------------------------------------------------------------------------
# whole frame  (splatter.py:513-655)
# --------------------------------------------------------------------------------------
class Camera:
    """Pinhole, principal point = image centre (splatter.py:499-500,532-533)."""

    def __init__(self, width, height, fx, fy, rot, tran, near=0.3):
        self.width, self.height, self.fx, self.fy = int(width), int(height), float(fx), float(fy)
        self.rot, self.tran, self.near = rot, tran, float(near)
        self.Wp = int(math.ceil(self.width / 16)) * 16          # splatter.py:259-260
        self.Hp = int(math.ceil(self.height / 16)) * 16
        self.ntx, self.nty = self.Wp // 16, self.Hp // 16
        self.half_w = self.width * 1.2 / 2 / self.fx            # splatter.py:532-533
        self.half_h = self.height * 1.2 / 2 / self.fy
        self.tile_lx = 16 / self.fx                             # splatter.py:279-282
        self.tile_ly = 16 / self.fy
        self.leftmost = -self.Wp / 2 / self.fx
        self.topmost = -self.Hp / 2 / self.fy

    def crop(self, image):                                      # splatter.py:267-272
        top = (self.Hp - self.height) // 2
        left = (self.Wp - self.width) // 2
        return image[top:top + self.height, left:left + self.width, :]


def render(pos, rgb, opa, quat, scale, cam: Camera, thresh=0.05, scale_activation="abs",
           use_sh_coeff=False, tiles=None, return_aux=False, depth_key=None):
    """Splatter.forward (splatter.py:643-655) on raw parameters; returns the
    clamped + cropped image (differentiable wrt the five parameter tensors)."""
    dt = pos.dtype
    rot, tran = cam.rot.to(dt), cam.tran.to(dt)
    nq, ns, opa_a, rgb_a = preactivate(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
    rp, rc, mask = global_culling(pos, nq, ns, rot, tran, cam.near, cam.half_w, cam.half_h)
    keep = mask.bool()
    idx = torch.nonzero(keep).squeeze(-1)
    p_c, c_c, rgb_c, opa_c = rp[idx], rc[idx], rgb_a[idx], opa_a[idx]          # a3 :536-542
    rects = tile_rects(p_c[:, :2], c_c, thresh, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty,
                       cam.leftmost, cam.topmost)
    gi, accum = bin_and_sort(p_c, c_c, rects, cam.ntx, cam.nty,
                             None if depth_key is None else depth_key[idx])
    rays = ray_info(rot, tran, cam.Hp, cam.Wp, cam.fx, cam.fy) if use_sh_coeff else (None,) * 4
    img = draw(p_c[gi], rgb_c[gi], opa_c[gi], c_c[gi], accum, cam.Hp, cam.Wp, cam.fx, cam.fy,
               use_sh_coeff, *rays, tiles=tiles)
    out = cam.crop(torch.clamp(img, 0, 1))                                      # :652-653
    if return_aux:
        return out, dict(padded=img, mask=mask, accum=accum, gauss_idx=idx[gi], res_pos=rp, res_cov=rc)
    return out
