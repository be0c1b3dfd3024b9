"""fp64 restatement of the bilateral-grid slice (include/gs_b200.h, gs_bilagrid_slice_fwd): forward, analytic
backward, the grid_sample form it is defined by, and the total-variation term.

The luminance guide z is computed in fp32 exactly as the kernel does, fmaf(0.114f, b, fmaf(0.587f, g, 0.299f * r)),
and everything after it in fp64.  fp32 rounding decides which side of a knot z lies on (a white pixel is z = 1.0
exactly in fp32 but 0.9999999999999999 in fp64), and the z-gradient jumps there.  numpy has no fused multiply-add, so
`fmaf32` forms a * b + c exactly in fp64 with a TwoSum error term, rounds it to odd, and then to fp32: with 53 >= 24 + 2
bits that is the correctly rounded fused result."""
import numpy as np
import torch

LUM = (0.299, 0.587, 0.114)


def fmaf32(a, b, c):
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b                                   # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)               # s + e == p + c exactly
    bits = s.view(np.int64)
    odd = np.where((e != 0) & ((bits & 1) == 0), np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return odd.astype(np.float32)


def guide_f32(rgb):
    """fp32 luminance of [..., 3] (any float dtype), as the kernel computes it; returns float32 numpy."""
    x = np.asarray(rgb.detach().cpu() if torch.is_tensor(rgb) else rgb, dtype=np.float32)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    return fmaf32(np.float32(0.114), b, fmaf32(np.float32(0.587), g, np.float32(0.299) * r))


def _z(image, z_fp32):
    """The guide as a differentiable fp64 tensor: its value is the fp32 guide (or the fp64 one), its gradient the
    linear luminance's."""
    lum = LUM[0] * image[..., 0] + LUM[1] * image[..., 1] + LUM[2] * image[..., 2]
    if not z_fp32:
        return lum
    z32 = torch.from_numpy(guide_f32(image).astype(np.float64))
    return z32 + (lum - lum.detach())


def _cells(n, g):
    c = (torch.arange(n, dtype=torch.float64) + 0.5) / n * (g - 1)
    c0 = c.floor().clamp(0, g - 2)
    return c0.long(), c - c0


def _zcell(z, gl):
    inside = (z > 0) & (z < 1)
    zc = torch.where(inside, z, z.detach().clamp(0, 1))        # grid_sample's border clip: no gradient at 0 and 1
    gz = zc * (gl - 1)
    z0 = gz.detach().floor().clamp(0, gl - 2)
    return z0.long(), gz - z0, inside


def affine_field(image, grids, ids, z_fp32=True):
    """A [B, H, W, 12]: each pixel's trilinearly interpolated affine (differentiable in image and grids)."""
    img = image if image.dim() == 4 else image[None]
    bsz, h, w, _ = img.shape
    _, gh, gw, gl, _ = grids.shape
    y0, fy = _cells(h, gh)
    x0, fx = _cells(w, gw)
    z0, fz, _ = _zcell(_z(img, z_fp32), gl)
    gsel = grids[torch.as_tensor(list(ids), dtype=torch.long)]               # [B, GH, GW, GL, 12]
    bi = torch.arange(bsz)[:, None, None]
    A = 0
    for a in (0, 1):
        wx = fx if a else 1 - fx
        for b in (0, 1):
            wy = fy if b else 1 - fy
            for c in (0, 1):
                wz = fz if c else 1 - fz
                node = gsel[bi, (y0 + b)[None, :, None], (x0 + a)[None, None, :], z0 + c]
                A = A + (wy[None, :, None] * wx[None, None, :] * wz)[..., None] * node
    return A


def apply_affine(A, image):
    img = image if image.dim() == 4 else image[None]
    M = A.reshape(*A.shape[:-1], 3, 4)
    return (M[..., :3] * img[..., None, :]).sum(-1) + M[..., 3]


def slice_forward(image, grids, ids, z_fp32=True):
    """fp64 slice: [B, H, W, 3] (or [H, W, 3]) -> same shape."""
    out = apply_affine(affine_field(image, grids, ids, z_fp32), image)
    return out if image.dim() == 4 else out[0]


def slice_grid_sample(image, grids, ids, z_fp32=True):
    """The definition: grid_sample(grids_ncdhw[ids], coords * 2 - 1, bilinear, align_corners, border) + affine."""
    img = image if image.dim() == 4 else image[None]
    bsz, h, w, _ = img.shape
    ncdhw = grids.permute(0, 4, 3, 1, 2)[torch.as_tensor(list(ids), dtype=torch.long)]
    xs = ((torch.arange(w, dtype=img.dtype) + 0.5) / w).expand(bsz, h, w)
    ys = ((torch.arange(h, dtype=img.dtype) + 0.5) / h)[:, None].expand(bsz, h, w)
    coords = torch.stack([xs, ys, _z(img, z_fp32)], dim=-1)[:, None] * 2 - 1          # [B, 1, H, W, 3]
    A = torch.nn.functional.grid_sample(ncdhw, coords, mode="bilinear", padding_mode="border", align_corners=True)
    out = apply_affine(A[:, :, 0].permute(0, 2, 3, 1), img)
    return out if image.dim() == 4 else out[0]


def slice_backward(image, grids, ids, grad_out):
    """Analytic gradients (fp64, z in fp32): (grad_image, grad_grids), the latter zero outside the batch's rows."""
    img = (image if image.dim() == 4 else image[None]).double().detach()
    go = (grad_out if grad_out.dim() == 4 else grad_out[None]).double()
    grids = grids.double().detach()
    bsz, h, w, _ = img.shape
    nv, gh, gw, gl, _ = grids.shape
    y0, fy = _cells(h, gh)
    x0, fx = _cells(w, gw)
    z = torch.from_numpy(guide_f32(img).astype(np.float64))
    z0, fz, inside = _zcell(z, gl)
    idt = torch.as_tensor(list(ids), dtype=torch.long)
    gsel = grids[idt]
    bi = torch.arange(bsz)[:, None, None]
    u = torch.cat([img, torch.ones_like(img[..., :1])], dim=-1)             # [B, H, W, 4]
    q = (go[..., :, None] * u[..., None, :]).reshape(bsz, h, w, 12)          # dL/dA
    gg = torch.zeros_like(grids)
    A = torch.zeros(bsz, h, w, 12, dtype=torch.float64)
    dA = torch.zeros_like(A)
    for a in (0, 1):
        wx = fx if a else 1 - fx
        for b in (0, 1):
            wy = fy if b else 1 - fy
            wxy = (wy[None, :, None] * wx[None, None, :]).expand(bsz, h, w)
            for c in (0, 1):
                wz = fz if c else 1 - fz
                yy, xx, zz = (y0 + b)[None, :, None].expand(bsz, h, w), (x0 + a)[None, None, :].expand(bsz, h, w), z0 + c
                node = gsel[bi, yy, xx, zz]
                A += (wxy * wz)[..., None] * node
                dA += (wxy * (1.0 if c else -1.0))[..., None] * node
                flat = ((idt[:, None, None].expand(bsz, h, w) * gh + yy) * gw + xx) * gl + zz
                gg.view(-1, 12).index_add_(0, flat.reshape(-1), ((wxy * wz)[..., None] * q).reshape(-1, 12))
    M = A.reshape(bsz, h, w, 3, 4)
    gi = (M[..., :3] * go[..., :, None]).sum(-2)
    dz = (q * dA).sum(-1) * (gl - 1) * inside
    gi = gi + dz[..., None] * torch.tensor(LUM, dtype=torch.float64)
    if image.dim() == 3:
        gi = gi[0]
    return gi, gg


def slice_terms(image, grids, ids, grad_out):
    """Term magnitudes of the slice for per-element error models (fp64, z in fp32 as above), with N the sum of |node|
    over a pixel's 8 nodes [B, H, W, 12] and u = (r, g, b, 1):
      out_mag  [B, H, W, 3]       sum_j N_cj |u_j|
      gi_mag   [B, H, W, 3]       sum_r |go_r| (N_rc + LUM_c (GL - 1) [0 < z < 1] sum_j N_rj |u_j|)
      gg_mag   [V, GH, GW, GL, 12] sum over the pixels reaching the node of |w_xyz dL/dA|
      gg_count [V, GH, GW, GL, 1]  the number of (pixel, corner) terms summed into the node"""
    img = (image if image.dim() == 4 else image[None]).double().detach()
    go = (grad_out if grad_out.dim() == 4 else grad_out[None]).double()
    grids = grids.double().detach()
    bsz, h, w, _ = img.shape
    nv, gh, gw, gl, _ = grids.shape
    y0, fy = _cells(h, gh)
    x0, fx = _cells(w, gw)
    z = torch.from_numpy(guide_f32(img).astype(np.float64))
    z0, fz, inside = _zcell(z, gl)
    idt = torch.as_tensor(list(ids), dtype=torch.long)
    gsel = grids[idt].abs()
    bi = torch.arange(bsz)[:, None, None]
    u = torch.cat([img, torch.ones_like(img[..., :1])], dim=-1).abs()
    q = (go.abs()[..., :, None] * u[..., None, :]).reshape(bsz, h, w, 12)
    N = torch.zeros(bsz, h, w, 12, dtype=torch.float64)
    gg = torch.zeros_like(grids)
    cnt = torch.zeros(nv * gh * gw * gl, 1, dtype=torch.float64)
    for a in (0, 1):
        wx = fx if a else 1 - fx
        for b in (0, 1):
            wy = fy if b else 1 - fy
            wxy = (wy[None, :, None] * wx[None, None, :]).expand(bsz, h, w)
            for c in (0, 1):
                wz = fz if c else 1 - fz
                yy, xx, zz = (y0 + b)[None, :, None].expand(bsz, h, w), (x0 + a)[None, None, :].expand(bsz, h, w), z0 + c
                N += gsel[bi, yy, xx, zz]
                flat = (((idt[:, None, None].expand(bsz, h, w) * gh + yy) * gw + xx) * gl + zz).reshape(-1)
                gg.view(-1, 12).index_add_(0, flat, ((wxy * wz).abs()[..., None] * q).reshape(-1, 12))
                cnt.index_add_(0, flat, torch.ones(flat.numel(), 1, dtype=torch.float64))
    Nm = N.reshape(bsz, h, w, 3, 4)
    out_mag = (Nm * u[..., None, :]).sum(-1)
    zt = out_mag * (gl - 1) * inside[..., None]                                     # [B, H, W, r]
    gi_mag = (go.abs()[..., :, None] * (Nm[..., :3] + zt[..., :, None] * torch.tensor(LUM, dtype=torch.float64))).sum(-2)
    if image.dim() == 3:
        out_mag, gi_mag = out_mag[0], gi_mag[0]
    return dict(out_mag=out_mag, gi_mag=gi_mag, gg_mag=gg, gg_count=cnt.view(nv, gh, gw, gl, 1))


def tv(grids):
    g = grids.double()
    return sum(float(((g.narrow(d, 1, g.shape[d] - 1) - g.narrow(d, 0, g.shape[d] - 1)) ** 2).mean()) for d in (1, 2, 3))


def identity(v, gh, gw, gl, dtype=torch.float64):
    eye = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=dtype)
    return eye.expand(v, gh, gw, gl, 12).clone()


def random_grids(v, gh, gw, gl, seed, scale=0.2):
    g = torch.Generator().manual_seed(seed)
    return (identity(v, gh, gw, gl) + scale * torch.randn(v, gh, gw, gl, 12, generator=g, dtype=torch.float64))


def knot_pixels(gl, n, seed):
    """n grey-ish fp32 pixels whose fp32 guide lands exactly on a lattice knot k / (gl - 1) with a dyadic (gl - 1),
    interior and end knots included; returns float32 [n, 3]."""
    assert (gl - 1) & (gl - 2) == 0, "dyadic knots only"
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        k = int(rng.integers(0, gl))
        t = np.float32(k / (gl - 1))
        rg = np.clip(t + rng.normal(0, 0.05, 2), 0, 1).astype(np.float32)
        # the blue channel that puts z on t: search fp32 neighbours of the real-valued solution
        b0 = (t - 0.299 * rg[0] - 0.587 * rg[1]) / 0.114
        cand = (np.float32(b0) + np.arange(-64, 65, dtype=np.float32) * np.spacing(np.float32(max(abs(b0), 1e-3))))
        cand = cand.astype(np.float32)
        z = guide_f32(np.stack([np.full_like(cand, rg[0]), np.full_like(cand, rg[1]), cand], -1))
        hit = np.nonzero(z == t)[0]
        if hit.size:
            out.append([rg[0], rg[1], cand[hit[0]]])
    return np.asarray(out, dtype=np.float32)
