"""Fixtures and per-element comparators for the two image-space kernels between the rendered image and the blend
backward: the fused L1 + SSIM loss (csrc/loss.cu) and the bilateral-grid slice (csrc/bilagrid.cu).

Test infrastructure only, built on oracle/loss_oracle.py (LO) and tests/bilagrid_oracle.py (BO), both fp64.

Loss.  The kernel works on 16x16 tiles with a 5-pixel halo; a window centre is "inner" when it lies 5 pixels or more
from every border.  LOSS_SHAPES put H mod 16 and W mod 16 at every residue in RESIDUES (the inner band's last row and
column, and the last partial tile, at each position in their tile), every size in (11, 16], and two 11-pixel strips.
The contents are built where SSIM and the L1 sign are worst conditioned: flat blocks at 0, 1, 0.98 +- 1e-3 and
0.999 +- 1e-5; x == y exactly over whole regions; a 0/1 checkerboard; single-pixel impulses at tile corners and on the
inner band's edges.  The comparator (LossRef) is per element, from LO.ssim_terms' term magnitudes:

    |g - g_ref| <= C_GRAD eps (|k_ssim| grad_mag_p + |k_l1|) + 2 |k_l1| [0 < |x_p - y_p| <= ulp]
    |v - v_ref| <= C_VAL eps (|w_l1| mean|x - y| + |w_ssim| mean s_mag + |bias|)

with k_l1 = w_l1 / (3 H W), k_ssim = w_ssim / (3 (H - 10)(W - 10)).  grad_mag carries the fp32 cancellation of
s_xx and s_yy (1 + (E[x^2] + E[y^2]) / d2); the last term is a sign flip of |x - y| where x and y are one rounding
apart (x == y must give sign 0 exactly).  The gradient bound sums term magnitudes and does not follow the
cancellation between A, 2 x B and y C: inside the flat 0.98 and 0.999 blocks it exceeds the gradient itself, so
there it only asserts finiteness and scale; the blocks' edges, the 0 / 1 blocks and the other contents carry the
gradient checks.  loss_fp32 restates the kernel's arithmetic in torch fp32, with the wrong
variants the CPU suite shows the comparator catches.

Bilateral grid.  Round-up knot pixels (roundup_knot_pixels): fp32 guides z just below a knot j / (GL - 1) whose
fp32 product z (GL - 1) rounds up onto j, for every GL <= 16 and knot where such a z exists (ROUNDUP_KNOTS); a plain
floorf puts them in the upper cell, whose z-slope differs.  SliceRef gives per-element bounds from the term
magnitudes in BO.slice_terms; slice_fp32 restates the kernel in fp32, with the plain-floor and missing-row
variants.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

import bilagrid_oracle as BO
import loss_oracle as LO

EPS32 = 2.0 ** -24

# ------------------------------------------------------------------------------------------------------------- loss
TILE, HALF = 16, 5
RESIDUES = (0, 1, 5, 6, 10, 11, 15)
C_GRAD = 64.0
C_VAL = 64.0


def _loss_shapes():
    hs = [32 + r for r in RESIDUES]
    ws = [32 + RESIDUES[(i + 3) % len(RESIDUES)] for i in range(len(RESIDUES))]
    small = [(d, 28 - d) for d in range(12, 17)]
    return list(zip(hs, ws)) + small + [(11, 2000), (2000, 11)]


LOSS_SHAPES = _loss_shapes()
UHD = (2160, 3840)
CONTENTS = ("flat", "equal", "checker", "impulse", "noise")


def impulse_sites(h, w):
    """pixels whose 11x11 footprint straddles a tile corner (the corner's four pixels) or the inner band's edge
    (on the last inner row / column and the first outer one, on all four sides)"""
    sites = {(ty + dy, tx + dx) for ty in range(TILE, h, TILE) for tx in range(TILE, w, TILE)
             for dy in (-1, 0) for dx in (-1, 0)}
    for r in (HALF - 1, HALF, h - HALF - 1, h - HALF):
        sites |= {(r, c) for c in (w // 3, (2 * w) // 3)}
    for c in (HALF - 1, HALF, w - HALF - 1, w - HALF):
        sites |= {(r, c) for r in (h // 3, (2 * h) // 3)}
    return sorted((r, c) for r, c in sites if 0 <= r < h and 0 <= c < w)


def loss_pair(h, w, content, half=False, seed=0):
    """(image float32 [h, w, 3], target float32 or float16 [h, w, 3]) of one content"""
    if content == "mixed":                     # 64x64 blocks, each of one content
        parts = [loss_pair(h, w, c, half, seed + i) for i, c in enumerate(CONTENTS)]
        blk = ((torch.arange(h)[:, None] // 64) * 7 + torch.arange(w)[None, :] // 64) % len(CONTENTS)
        idx = blk[None, :, :, None].expand(1, h, w, 3)
        return tuple(torch.stack([p[k] for p in parts]).gather(0, idx)[0].contiguous() for k in (0, 1))
    g = torch.Generator().manual_seed(seed * 1009 + h * 31 + w)
    u = lambda: torch.rand(h, w, 3, generator=g, dtype=torch.float64)                                   # noqa
    rows, cols = torch.arange(h)[:, None, None], torch.arange(w)[None, :, None]
    same = torch.zeros(h, w, 3, dtype=torch.bool)
    if content == "flat":
        blk = (((rows + 3) // 20 + (cols + 3) // 20) % 4).expand(h, w, 3)
        x, y = torch.empty(h, w, 3, dtype=torch.float64), torch.empty(h, w, 3, dtype=torch.float64)
        ux, uy = u(), u()
        levels = ((0.0, 1e-3), (1.0, 1e-3), (0.98, 1e-3), (0.999, 1e-5))
        for k, (c, a) in enumerate(levels):
            m = blk == k
            if k == 0:      # x exactly 0, y just above
                xk, yk = torch.zeros_like(ux), a * uy
            elif k == 1:    # y exactly 1, x just below
                xk, yk = 1 - a * ux, torch.ones_like(uy)
            else:
                xk, yk = c + a * (2 * ux - 1), c + a * (2 * uy - 1)
            x[m], y[m] = xk[m], yk[m]
    elif content == "equal":
        x, y = u(), u()
        same = (((rows // 9) + (cols // 7)) % 2 == 0).expand(h, w, 3)
    elif content == "checker":
        x = ((rows + cols) % 2).double().expand(h, w, 3).clone()
        y = torch.where(cols < w // 2, x, 1 - x)
        y[::5, ::3] = 0.5
    elif content == "impulse":
        x = torch.full((h, w, 3), 0.5, dtype=torch.float64)
        y = x.clone()
        rc = torch.tensor(impulse_sites(h, w), dtype=torch.long).view(-1, 2)
        amp = torch.where(torch.arange(len(rc)) % 2 == 1, 0.4, -0.45).double()
        x[rc[:, 0], rc[:, 1]] = 0.5 + amp[:, None] * torch.tensor([1.0, 0.6, -0.3], dtype=torch.float64)
        same = x == y
    elif content == "noise":
        y = (0.5 + 0.4 * torch.sin(0.2 * cols + 0.1 * rows + torch.tensor([0.0, 1.0, 2.0])) + 0.05 * u()).clamp(0, 1)
        x = (y + 0.15 * (u() - 0.5)).clamp(0, 1)
    else:
        raise ValueError(content)
    y = y.half() if half else y.float()
    x = torch.where(same, y.float(), x.float())
    return x.contiguous(), y.contiguous()


def loss_weights(mode):
    """(w_l1, w_ssim, bias) of a call: "w=<ssim weight>" -> l1_ssim_loss, "ssim" -> loss.ssim, "l1" -> loss.l1"""
    if mode == "ssim":
        return 0.0, 1.0, 0.0
    if mode == "l1":
        return 1.0, 0.0, 0.0
    w = float(mode[2:])
    return 1.0 - w, -w, w


CALLS = ("w=0", "w=0.1", "w=1", "ssim", "l1")


class LossRef:
    """fp64 oracle of one (image, target) pair, on the inputs' device: every call's value and gradient come from
    the same maps"""

    def __init__(self, x, y):
        xd, yd = x.double(), y.double()
        self.h, self.w = x.shape[:2]
        self.t = LO.ssim_terms(xd, yd)
        self.n_all = 3.0 * self.h * self.w
        self.n_inner = 3.0 * (self.h - 2 * HALF) * (self.w - 2 * HALF)
        self.l1 = float((xd - yd).abs().sum()) / self.n_all
        self.ssim = float(self.t["s"].sum()) / self.n_inner
        self.s_mag = float(self.t["s_mag"].sum()) / self.n_inner
        self.sign = torch.sign(xd - yd)
        diff = (xd - yd).abs()
        ulp = torch.maximum(xd.abs(), yd.abs()).float().double()
        ulp = (torch.nextafter(ulp.float(), torch.tensor(float("inf"), device=x.device)).double() - ulp)
        self.near = (diff > 0) & (diff <= ulp)

    def value(self, mode):
        w_l1, w_ssim, bias = loss_weights(mode)
        v = w_l1 * self.l1 + w_ssim * self.ssim + bias
        bound = C_VAL * EPS32 * (abs(w_l1) * self.l1 + abs(w_ssim) * self.s_mag + abs(bias))
        return v, bound

    def l1_bound(self):
        return C_VAL * EPS32 * self.l1

    def ssim_bound(self):
        return C_VAL * EPS32 * self.s_mag

    def grad(self, mode):
        w_l1, w_ssim, _ = loss_weights(mode)
        k_l1, k_ssim = w_l1 / self.n_all, w_ssim / self.n_inner
        g = k_ssim * self.t["grad"] + k_l1 * self.sign
        bound = C_GRAD * EPS32 * (abs(k_ssim) * self.t["grad_mag"] + abs(k_l1)) + 2 * abs(k_l1) * self.near
        return g, bound


def excess(got, ref, bound):
    """max over elements of |got - ref| / bound (inf where the bound is 0 and they differ; nan fails as inf)"""
    d = (got.double().to(ref.device) - ref).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / bound)
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    return float(r.max()) if r.numel() else 0.0


def _hsum(m, w, drop_halo_tap=False):
    """sum_k w_k m[..., c + k] in fp32, in the kernel's tap order; drop_halo_tap skips tap k = 6, the first column of
    the right halo, for the columns c that are a tile's last column"""
    n = m.shape[-1] - 2 * HALF
    acc = torch.zeros(*m.shape[:-1], n, dtype=torch.float32)
    last = (torch.arange(n) % TILE) == TILE - 1
    for k in range(2 * HALF + 1):
        t = w[k] * m[..., k:k + n]
        if drop_halo_tap and k == HALF + 1:
            t = torch.where(last, torch.zeros_like(t), t)
        acc = acc + t
    return acc


def _vsum(m, w):
    return _hsum(m.transpose(-1, -2), w).transpose(-1, -2)


def loss_fp32(x, y, w_l1, w_ssim, bias, band=0, drop_halo_tap=False, sign0=0.0):
    """The kernel's arithmetic restated in torch fp32 (separable window over clamped halos, per-window A, B, C,
    the transposed window over zero halos): returns ((total, l1, ssim), grad [H, W, 3]).  Wrong variants: `band`
    widens the inner band by that many pixels, `drop_halo_tap` drops the first right-halo tap of the gradient's
    horizontal pass on tiles' last columns (a halo column lost), `sign0` is the L1 sign taken at x == y."""
    h, w = x.shape[:2]
    w1 = LO.gaussian_window(dtype=torch.float64).float()
    X, Y = x.float().permute(2, 0, 1), y.float().permute(2, 0, 1)
    pad = lambda m: F.pad(m[None], (HALF,) * 4, mode="replicate")[0]                                  # noqa
    Xp, Yp = pad(X), pad(Y)
    mx, my, exx, eyy, exy = (_vsum(_hsum(m, w1), w1) for m in (Xp, Yp, Xp * Xp, Yp * Yp, Xp * Yp))
    c1, c2 = np.float32(1e-4), np.float32(9e-4)
    sxx, syy, sxy = exx - mx * mx, eyy - my * my, exy - mx * my
    n1, n2 = 2 * mx * my + c1, 2 * sxy + c2
    d1, d2 = mx * mx + my * my + c1, sxx + syy + c2
    inv = 1 / (d1 * d2)
    s = n1 * n2 * inv
    A = 2 * my * (n2 - n1) * inv - 2 * mx * s * (d2 - d1) * inv
    B = -s / d2
    C = 2 * n1 * inv
    lo = HALF - band
    r, c = torch.arange(h)[:, None], torch.arange(w)[None, :]
    inner = ((r >= lo) & (r < h - lo) & (c >= lo) & (c < w - lo))[None]
    z = torch.zeros_like(s)
    s, A, B, C = (torch.where(inner, m, z) for m in (s, A, B, C))
    n_all, n_inner = 3.0 * h * w, 3.0 * (h - 2 * HALF) * (w - 2 * HALF)
    l1 = np.float32(float((X - Y).abs().sum()) / n_all)
    ss = np.float32(float(s.sum()) / n_inner)
    total = np.float32(w_l1) * l1 + np.float32(w_ssim) * ss + np.float32(bias)
    zpad = lambda m: F.pad(m, (HALF,) * 4)                                                              # noqa
    bA, bB, bC = (_vsum(_hsum(zpad(m), w1, drop_halo_tap), w1) for m in (A, B, C))
    k_l1, k_ssim = np.float32(w_l1 / n_all), np.float32(w_ssim / n_inner)
    sgn = torch.where(X > Y, 1.0, torch.where(X < Y, -1.0, sign0)).float()
    g = k_ssim * (bA + 2 * X * bB + Y * bC) + k_l1 * sgn
    return (float(total), float(l1), float(ss)), g.permute(1, 2, 0).contiguous()


# ------------------------------------------------------------------------------------------------- bilateral grid
# The slice bounds count every term's magnitude and, for a grid node, every summand as a rounding step; the fp32
# restatement uses about 0.003 of them on small grids and 0.3 on the 256 x 256 x 16 grid, while the wrong variants
# exceed them 200-fold or more.
C_SLICE = 32.0
FWD_IDS_PER_LAUNCH = 64        # bilagrid.cu: images per forward launch
TABLE_PER_LAUNCH = 960         # bilagrid.cu: view-table entries per upload launch of the backward
MAX_SLICES = 64                # bilagrid.cu: row slices per cell at most
# knots j (0 < j < GL - 1) with an fp32 z within 6 ulp below j / (GL - 1) whose fp32 product z (GL - 1) rounds up
# onto j; no other GL <= 16 has one
ROUNDUP_KNOTS = {7: (5,), 11: (7, 9), 12: (5, 7, 9, 10), 13: (5, 7, 10, 11), 15: (9, 11, 13)}


def roundup_z(gl, j, span=6):
    """the fp32 z within `span` ulp of fp32(j / (gl - 1)) with fl32(z (gl - 1)) == j but z (gl - 1) < j exactly"""
    t = np.float32(j / (gl - 1))
    cand = [t]
    lo = hi = t
    for _ in range(span):
        lo, hi = np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(2))
        cand += [lo, hi]
    z = np.array(sorted(set(cand)), dtype=np.float32)
    exact = z.astype(np.float64) * (gl - 1)                # exact: 24 + 4 bits
    return z[(exact.astype(np.float32) == np.float32(j)) & (exact < j)]


def roundup_knots(gl):
    return tuple(j for j in range(1, gl - 1) if roundup_z(gl, j).size)


def plain_floor_cell(z, gl):
    """the z cell a plain floorf of the fp32 product gives (the defect the fma residual in z_cell prevents)"""
    zc = np.clip(np.asarray(z, dtype=np.float32), 0, 1)
    gz = (zc.astype(np.float64) * (gl - 1)).astype(np.float32)
    return np.minimum(np.floor(gz), gl - 2).astype(np.int64)


def exact_cell(z, gl):
    zc = np.clip(np.asarray(z, dtype=np.float32), 0, 1).astype(np.float64)
    return np.minimum(np.floor(zc * (gl - 1)), gl - 2).astype(np.int64)


def roundup_knot_pixels(gl, n, seed):
    """n fp32 pixels whose fp32 guide is one of roundup_z(gl, j) for a knot j of ROUNDUP_KNOTS[gl]: the blue channel
    is searched over the fp32 neighbours of the real-valued solution, as BO.knot_pixels does; float32 [n, 3]"""
    rng = np.random.default_rng(seed)
    targets = [(j, roundup_z(gl, j)) for j in ROUNDUP_KNOTS[gl]]
    out = []
    while len(out) < n:
        j, zs = targets[len(out) % len(targets)]
        t = zs[int(rng.integers(0, zs.size))]
        rg = np.clip(np.float32(j / (gl - 1)) + rng.normal(0, 0.05, 2), 0, 1).astype(np.float32)
        b0 = (float(t) - 0.299 * rg[0] - 0.587 * rg[1]) / 0.114
        cand = (np.float32(b0) + np.arange(-256, 257, dtype=np.float32) * np.spacing(np.float32(max(abs(b0), 1e-3))))
        cand = cand.astype(np.float32)
        z = BO.guide_f32(np.stack([np.full_like(cand, rg[0]), np.full_like(cand, rg[1]), cand], -1))
        hit = np.nonzero(z == t)[0]
        if hit.size:
            out.append([rg[0], rg[1], cand[hit[0]]])
    return np.asarray(out, dtype=np.float32)


def _specials(n, seed):
    """black, white and out-of-range pixels"""
    rng = np.random.default_rng(seed)
    px = np.zeros((n, 3), dtype=np.float32)
    px[1::4] = 1.0
    px[2::4] = rng.uniform(-0.6, -0.01, (len(px[2::4]), 3))
    px[3::4] = rng.uniform(1.01, 1.6, (len(px[3::4]), 3))
    return px


class SliceCase:
    def __init__(self, image, grids, ids, seed):
        self.image, self.grids, self.ids = image.contiguous(), grids.float().contiguous(), list(ids)
        g = torch.Generator().manual_seed(seed)
        self.go = torch.randn(image.shape, generator=g).contiguous()

    @property
    def views(self):
        return sorted(set(self.ids))


def _knot_case(gl, roundup, seed):
    b, h, w = 2, 12, 16
    n = b * h * w
    px = roundup_knot_pixels(gl, n // 2, seed) if roundup else BO.knot_pixels(gl, n // 2, seed)
    px = np.concatenate([px, _specials(n - len(px), seed + 1)])
    px = px[np.random.default_rng(seed + 2).permutation(n)]
    img = torch.from_numpy(px).reshape(b, h, w, 3)
    return SliceCase(img, BO.random_grids(3, 4, 5, gl, seed=seed), [2, 0], seed)


def _rand_image(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = -0.1 + 1.2 * torch.rand(b, h, w, 3, generator=g)
    x.view(-1, 3)[::7] = 0.0
    x.view(-1, 3)[3::11] = 1.0
    return x


def _plain(b, h, w, shape, v, ids, seed):
    return SliceCase(_rand_image(b, h, w, seed), BO.random_grids(v, *shape, seed=seed), ids, seed)


def _slice_builders():
    c = {}
    for gl in (2, 3, 5, 9):
        c[f"knots-GL{gl}"] = lambda gl=gl: _knot_case(gl, False, gl)
    for gl in ROUNDUP_KNOTS:
        c[f"roundup-GL{gl}"] = lambda gl=gl: _knot_case(gl, True, 100 + gl)
    c["cells-over-pixels"] = lambda: _plain(1, 45, 67, (256, 256, 16), 2, [1], 3)
    c["one-pixel-cells"] = lambda: _plain(2, 6, 8, (7, 9, 4), 2, [1, 1], 4)
    c["lattice-through-centres"] = lambda: _plain(2, 5, 4, (11, 9, 5), 3, [2, 0], 5)
    c["one-cell-tall"] = lambda: _plain(2, 20, 3, (2, 2, 5), 3, [0, 1], 6)
    for b in (64, 65, 129):
        c[f"fwd-B{b}"] = lambda b=b: _plain(b, 5, 7, (3, 4, 4), 8, [(i * 5 + 3) % 7 for i in range(b)], 7 + b)
    for v in (60, 61):
        c[f"table-{900 + v}"] = lambda v=v: _plain(900, 4, 4, (2, 3, 3), v + 2, [(i * 37) % v + 1 for i in range(900)],
                                                   8 + v)
    c["B65535"] = lambda: _plain(65535, 1, 2, (2, 2, 2), 7, [(i * 3) % 5 + (i % 2) for i in range(65535)], 9)
    return c


SLICE_BUILDERS = _slice_builders()


class SliceRef:
    """fp64 oracle of one case with its per-element bounds"""

    def __init__(self, case):
        im, gr = case.image.double(), case.grids.double()
        self.out = BO.slice_forward(im, gr, case.ids)
        self.gi, self.gg = BO.slice_backward(im, gr, case.ids, case.go.double())
        t = BO.slice_terms(im, gr, case.ids, case.go.double())
        _, gh, gw, _, _ = case.grids.shape
        k = 4 + gh + gw                    # fp32 lattice coordinates: an error of a few ulp of gx < GW, gy < GH
        self.out_bound = C_SLICE * EPS32 * k * t["out_mag"]
        self.gi_bound = C_SLICE * EPS32 * k * t["gi_mag"]
        self.gg_bound = C_SLICE * EPS32 * (k + t["gg_count"]) * t["gg_mag"]     # any order of the node's sum


def _fma_free_cells(n, g):
    s = np.float32(g - 1) / np.float32(n)
    c = (np.arange(n, dtype=np.float32) + np.float32(0.5)) * s
    c0 = np.clip(np.floor(c), 0, g - 2)
    return torch.from_numpy(c0.astype(np.int64)), torch.from_numpy((c - c0.astype(np.float32)).astype(np.float32))


def slice_fp32(case, plain_floor=False, skip_cell_row=False):
    """The kernel's arithmetic restated in torch fp32: fp32 lattice coordinates, the fp32 guide, the exact z cell
    (or, `plain_floor`, floorf of the fp32 product), fp32 interpolation, affine and gradients.  `skip_cell_row`
    drops the first pixel row of every spatial cell after the first from the backward (its grad_image rows stay 0).
    Returns (out, grad_image, grad_grids) float32."""
    img, grids, go = case.image.float(), case.grids.float(), case.go.float()
    bsz, h, w, _ = img.shape
    nv, gh, gw, gl, _ = grids.shape
    y0, fy = _fma_free_cells(h, gh)
    x0, fx = _fma_free_cells(w, gw)
    z = BO.guide_f32(img)
    zc = np.clip(z, 0, 1).astype(np.float32)
    exact = zc.astype(np.float64) * (gl - 1)
    f0 = np.floor(exact.astype(np.float32)).astype(np.float64)
    if not plain_floor:
        f0 = np.where(exact < f0, f0 - 1, f0)
    z0n = np.minimum(f0, gl - 2)
    z0 = torch.from_numpy(z0n.astype(np.int64))
    fz = torch.from_numpy((exact - z0n).astype(np.float32))
    inside = torch.from_numpy((z > 0) & (z < 1))
    idt = torch.as_tensor(case.ids, dtype=torch.long)
    gsel = grids[idt]
    bi = torch.arange(bsz)[:, None, None]
    u = torch.cat([img, torch.ones_like(img[..., :1])], dim=-1)
    q = (go[..., :, None] * u[..., None, :]).reshape(bsz, h, w, 12)
    keep = torch.ones(h, dtype=torch.bool)
    if skip_cell_row:
        keep[1:] = y0[1:] == y0[:-1]
    kq = keep[None, :, None, None].float()
    A = torch.zeros(bsz, h, w, 12)
    dA = torch.zeros(bsz, h, w, 12)
    gg = torch.zeros_like(grids)
    for a in (0, 1):
        wx = fx if a else 1 - fx
        for b in (0, 1):
            wy = fy if b else 1 - fy
            wxy = (wx[None, None, :] * wy[None, :, None]).expand(bsz, h, w)
            yy, xx = (y0 + b)[None, :, None].expand(bsz, h, w), (x0 + a)[None, None, :].expand(bsz, h, w)
            lo, hi = gsel[bi, yy, xx, z0], gsel[bi, yy, xx, z0 + 1]
            A += wxy[..., None] * (lo + fz[..., None] * (hi - lo))
            dA += wxy[..., None] * (hi - lo)
            for c, wz in ((0, 1 - fz), (1, fz)):
                flat = (((idt[:, None, None].expand(bsz, h, w) * gh + yy) * gw + xx) * gl + z0 + c).reshape(-1)
                gg.view(-1, 12).index_add_(0, flat, (wz[..., None] * (wxy[..., None] * q) * kq).reshape(-1, 12))
    M = A.reshape(bsz, h, w, 3, 4)
    out = (M[..., :3] * img[..., None, :]).sum(-1) + M[..., 3]
    gi = (M[..., :3] * go[..., :, None]).sum(-2)
    dz = (q * dA).sum(-1) * np.float32(gl - 1) * inside
    gi = (gi + dz[..., None] * torch.tensor(BO.LUM, dtype=torch.float32)) * kq[..., :1]
    return out, gi, gg


def slice_excess(ref, case, out, gi, gg):
    """(out, grad_image, grad_grids over the batch's views) max |got - ref| / bound"""
    v = case.views
    return (excess(out, ref.out, ref.out_bound), excess(gi, ref.gi, ref.gi_bound),
            excess(gg[v], ref.gg[v], ref.gg_bound[v]))
