"""Scenes that put the fused frame's front end (projection, culling, tile rectangles, instance emission, the tile sort
and the tile ranges) on its edges, and a decision layer that says, for every Gaussian, what the device must do.

Test infrastructure only.  The arithmetic is gs_oracle's (`global_culling`, `tile_rects`, `bin_and_sort`, `draw`);
this module adds two things to it.

1. The host constants as `view_constants` (render.cu) narrows them.  The device culls against float32 `near`,
   `half_w = (float)(W * 1.2 / 2 / fx)`, `half_h`, and bins against float32 `lx`, `ly`, `leftmost`, `topmost` and
   `t2 = -2 logf(thresh)`, all formed in double from the float32 focal lengths.  `gs_oracle.Camera` keeps them as
   Python doubles, so at an exact boundary the unmodified oracle and the device disagree by design.  `View.cam()` is
   an `O.Camera` whose constants are replaced by the narrowed values; nothing in gs_oracle changes.

2. A classification of every placement as *decided* or *ambiguous*.

   Exact-arithmetic placements (identity or axis-permuting camera rotation, dyadic positions, power-of-two depths):
   `p_c = R p + t` and `x / z` are exact in float32, with or without FMA contraction, so the culling decision is
   decided exactly at the boundary: `z > near`, `|x/z| < half_w`, `|y/z| < half_h` on the narrowed constants.
   `exact_culling` verifies the exactness claim for each such placement (float32 replay == float64).

   Every other decision (and every tile rectangle) is a margin decision.  The device's tile edge, in tile units, is
       e = (cx +- sqrt(di * t2 * det) - leftmost) / lx     (gs_tile_rect; +1 before the truncation of tx1 / ty1)
   and E is the same expression in float64 on the float32 inputs and constants.  The bound |e - E| <= delta is
   derived from float32 unit roundoff u = 2^-24 (no -use_fast_math: every operation is correctly rounded, and an FMA
   contraction removes a rounding, never adds one):
     * cx = x / z: exact for the exact-arithmetic positions; otherwise p_c carries <= 3 roundings and the quotient
       one: |dcx| <= 4u |cx|.
     * a, b, d = rows of (J W)(R S): each entry of J W and R is <= 4 roundings deep, times s (1), squared and summed
       (<= 4): <= 16 roundings, so |da| <= 16u' a with u' = 2u (first-order terms doubled for the products of two
       perturbed factors): |da| <= 32u a, |db| <= 32u sqrt(a d).
     * shift^2 = di t2 det with di = a / (det + 1e-14) in double: the computed det multiplies its own reciprocal, so
       its (cancellation-prone) error cancels except through the 1e-14 term; the rest is a (32u), t2 (2u), the
       double quotient rounded to float (u) and two products (2u): |d shift| / shift <= (37u + eps_det 1e-14 / det)
       / 2 + u (sqrtf), with eps_det <= 2 * 34u (ad + |bc|) / det.  That is <= 20u for the scenes here (det >> 1e-14).
     * the edge: one add or subtract for cx +- shift, one for - leftmost, one division, one +1: each rounds
       relative to its own result, so |de| <= (|dcx| + |d shift| + 3u (|cx| + shift + |leftmost|)) / lx
       + 2u (|E| + 1).
   The 2-D filter adds one rounding to a and d (a + ex): 34u.  The OPENCV lens maps the mean (<= 12 roundings: 24u
   on cx) and the covariance (J_D Sigma J_D^T, 8 more levels: 48u on a and d).  `delta` doubles the sum, so that
   no term of the derivation needs to be tight.  An edge at least delta from every integer gives one truncation; a
   placement whose every edge (and culling test) is decided is *decided*, and its rectangle must equal the one
   from E exactly.  Otherwise the candidate rectangles are those of E - delta and E + delta on each undecided edge.

The scenes are built in pixel and depth terms (`Builder`), so each family states what it places where, and the
CPU tests (tests/test_bin_edges_oracle.py) check each scene's claims before any GPU run.
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import torch

import gs_oracle as O

TILE = 16
U = 2.0 ** -24
NAMES = ("pos", "rgb", "opa", "quat", "scale")
WARP, BLOCK = 32, 256                 # emit_keys_kernel: 32 depth-consecutive Gaussians per warp, 256 per block
RANGE_KEYS, RANGE_BLOCK = 8, 2048     # tile_ranges_kernel: 8 keys per thread, 2048 per block
# relative roundoff of the mean and of a, d (see the module docstring), per projection variant
CX_ERR = {"none": 4 * U, "antialias": 4 * U, "opencv": 24 * U}
COV_ERR = {"none": 32 * U, "antialias": 34 * U, "opencv": 48 * U}
CULL_MARGIN = 2.0 ** -12              # margin placements keep |x/z| / half_w and z / near this far from 1


def f32(x):
    return float(np.float32(x))


def next_up(x):
    return float(np.nextafter(np.float32(x), np.float32(np.inf)))


def next_down(x):
    return float(np.nextafter(np.float32(x), np.float32(-np.inf)))


def rot_z(quarter_turns):
    """Camera rotation about the optical axis by 90 degrees times quarter_turns: entries 0 and +-1, so R p is exact."""
    c, s = [(1, 0), (0, 1), (-1, 0), (0, -1)][quarter_turns % 4]
    return torch.tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=torch.float64)


class View:
    """One camera: float32 focal lengths, near and threshold, and the constants the device derives from them."""

    def __init__(self, width, height, fx, fy=None, rot=None, tran=(0.0, 0.0, 0.0), near=0.25, thresh=0.05):
        self.width, self.height = int(width), int(height)
        self.fx, self.fy = f32(fx), f32(fx if fy is None else fy)
        self.rot = torch.eye(3, dtype=torch.float64) if rot is None else rot.double()
        self.tran = torch.tensor(tran, dtype=torch.float64)
        self.near, self.thresh = f32(near), f32(thresh)
        self.Wp, self.Hp = -(-self.width // TILE) * TILE, -(-self.height // TILE) * TILE
        self.ntx, self.nty = self.Wp // TILE, self.Hp // TILE
        # view_constants: double arithmetic on the float inputs, narrowed once
        self.half_w = f32(self.width * 1.2 / 2.0 / self.fx)
        self.half_h = f32(self.height * 1.2 / 2.0 / self.fy)
        self.lx, self.ly = f32(16.0 / self.fx), f32(16.0 / self.fy)
        self.leftmost = f32(-self.Wp / 2.0 / self.fx)
        self.topmost = f32(-self.Hp / 2.0 / self.fy)
        self.t2 = float(np.float32(-2.0) * np.log(np.float32(self.thresh)))

    def cam(self, lens_free=False):
        """gs_oracle.Camera carrying the narrowed constants (lens_free: no frustum test, for the depth keys of a lens
        frame, whose frustum test is on the distorted mean)."""
        c = O.Camera(self.width, self.height, self.fx, self.fy, self.rot, self.tran, self.near)
        c.near, c.tile_lx, c.tile_ly, c.leftmost, c.topmost = self.near, self.lx, self.ly, self.leftmost, self.topmost
        c.half_w, c.half_h = (math.inf, math.inf) if lens_free else (self.half_w, self.half_h)
        return c

    def args(self):
        """Camera arguments of renderer.render_frame after the five parameters."""
        return (self.width, self.height, self.fx, self.fy, self.rot.float(), self.tran.float(), self.near,
                self.thresh, "abs")


def _logit(p):
    return math.log(p) - math.log1p(-p)


class Builder:
    """Gaussians given in normalised image-plane terms on view `view` (identity rotation, tran = 0): centre
    (xn, yn) = (x/z, y/z), camera depth z, footprint half-extents (hx, hy) in normalised units (the bbox half-width
    sqrt(a t2) of a Gaussian with identity quaternion, up to the 1e-4 floor of its third scale)."""

    def __init__(self, view, seed=0):
        self.view = view
        self.gen = torch.Generator().manual_seed(seed)
        self.rows = []      # (pos[3], scale[3], opa logit, exact, tag)

    def raw(self, pos, scale, opa=0.5, exact=False, tag=""):
        self.rows.append((tuple(float(p) for p in pos), tuple(float(s) for s in scale), _logit(opa), exact, tag))

    def at(self, xn, yn, z, hx, hy, opa=0.5, exact=False, tag=""):
        """Centre (xn, yn) at depth z; bbox half-extents hx, hy (normalised)."""
        k = math.sqrt(self.view.t2)
        sx, sy = hx * z / k - 1e-4, hy * z / k - 1e-4
        assert min(sx, sy) > 1e-4, "footprint below the scale floor: place the Gaussian deeper"
        self.raw((xn * z, yn * z, z), (sx, sy, 0.0), opa, exact, tag)

    def tiles(self, tx0, tx1, ty0, ty1, r, inset=0.25, opa=0.5, tag=""):
        """A Gaussian whose bbox covers tiles [tx0, tx1) x [ty0, ty1): its edges `inset` tiles inside the outer
        tiles' far borders, at distance |p_c| = r."""
        v = self.view
        cxt, cyt = (tx0 + tx1) / 2.0, (ty0 + ty1) / 2.0
        xn, yn = v.leftmost + cxt * v.lx, v.topmost + cyt * v.ly
        hx, hy = ((tx1 - tx0) / 2.0 - inset) * v.lx, ((ty1 - ty0) / 2.0 - inset) * v.ly
        z = r / math.sqrt(1.0 + xn * xn + yn * yn)
        self.at(xn, yn, z, hx, hy, opa, tag=tag)

    def edge(self, side, k, off, r, tx=None, ty=None, h=0.3, opa=0.5):
        """A Gaussian with one bbox edge at tile border k + off (in tile units): side 'l' / 'r' (x) or 't' / 'b' (y);
        the other axis is centred in tile column tx / row ty (default: the middle); h: half-extent in tiles."""
        v = self.view
        tx = v.ntx // 2 if tx is None else tx
        ty = v.nty // 2 if ty is None else ty
        cxt, cyt, hxt, hyt = tx + 0.5, ty + 0.5, h, h
        e = k + off
        if side == "l":
            cxt = e + h
        elif side == "r":
            cxt = e - h
        elif side == "t":
            cyt = e + h
        else:
            cyt = e - h
        xn, yn = v.leftmost + cxt * v.lx, v.topmost + cyt * v.ly
        z = r / math.sqrt(1.0 + xn * xn + yn * yn)
        self.at(xn, yn, z, hxt * v.lx, hyt * v.ly, opa, tag=f"edge-{side}")

    def build(self, shuffle=True):
        n = len(self.rows)
        pos = torch.tensor([r[0] for r in self.rows], dtype=torch.float64).reshape(n, 3)
        scale = torch.tensor([r[1] for r in self.rows], dtype=torch.float64).reshape(n, 3)
        opa = torch.tensor([r[2] for r in self.rows], dtype=torch.float64)
        quat = torch.zeros(n, 4, dtype=torch.float64)
        quat[:, 0] = 1.0
        rgb = (torch.rand(n, 3, generator=self.gen, dtype=torch.float64) * 3 - 1.5)
        exact = torch.tensor([r[3] for r in self.rows], dtype=torch.bool)
        tags = [r[4] for r in self.rows]
        perm = torch.randperm(n, generator=self.gen) if shuffle else torch.arange(n)
        g = {"pos": pos, "rgb": rgb, "opa": opa, "quat": quat, "scale": scale}
        g = {q: t[perm].float().contiguous() for q, t in g.items()}
        # the exact placements are given in float32 values: narrowing them changed nothing
        assert torch.equal(g["pos"].double()[exact[perm]], pos[perm][exact[perm]])
        return g, exact[perm].clone(), [tags[i] for i in perm.tolist()]


class Scene:
    """A frame's Gaussians g (float32 CPU tensors), its views (one, or a batch), the projection variant ('none',
    'antialias' or 'opencv'), which placements claim exact arithmetic, and the scene's own claims."""

    def __init__(self, name, family, views, g, exact, tags, mode="none", claims=None, forward_only=False,
                 sample_tiles=None):
        self.name, self.family, self.views, self.g = name, family, list(views), g
        self.exact, self.tags, self.mode = exact, tags, mode
        self.claims = claims or {}
        self.forward_only = forward_only
        self.sample_tiles = sample_tiles
        self.n = g["pos"].shape[0]
        self._dec = {}

    def decide(self, v=0):
        if v not in self._dec:
            self._dec[v] = decide(self.g, self.views[v], self.mode, self.exact)
        return self._dec[v]


OPENCV = dict(model="OPENCV", cx=None, cy=None, k=[0.05, -0.01, 0.002, -0.001])


def lens_of(view):
    return dict(OPENCV, cx=view.width / 2.0 + 1.5, cy=view.height / 2.0 - 0.75)


# --------------------------------------------------------------------------------------------------------------------
# the decision layer
# --------------------------------------------------------------------------------------------------------------------
def _activated(g):
    """(normalised quaternion, activated scale) as float64 copies of the float32 values the device forms."""
    q = g["quat"].double()
    nq = q / q.norm(dim=1, keepdim=True)
    s32 = (g["scale"].abs() + torch.tensor(1e-4, dtype=torch.float32))       # fabsf(raw) + 1e-4f, float32
    return nq, s32.double()


def exact_culling(g, view):
    """[n] bool: p_c = R p + t and (x/z, y/z) evaluate exactly in float32 (every product and partial sum of the
    camera transform, in either FMA contraction, and both quotients)."""
    p = g["pos"].double().numpy()
    R, t = view.rot.numpy(), view.tran.numpy()
    R32, t32 = R.astype(np.float32), t.astype(np.float32)
    ok = np.all(R32.astype(np.float64) == R) and np.all(t32.astype(np.float64) == t)
    pc = p @ R.T + t
    with np.errstate(all="ignore"):
        exact = np.ones(p.shape[0], dtype=bool) & ok
        for i in range(3):
            terms = [R[i, k] * p[:, k] for k in range(3)]
            partial = terms[0]
            for k in range(3):
                exact &= terms[k].astype(np.float32).astype(np.float64) == terms[k]
            for k in (1, 2):
                partial = partial + terms[k]
                exact &= partial.astype(np.float32).astype(np.float64) == partial
            final = partial + t[i]
            exact &= final.astype(np.float32).astype(np.float64) == final
        z = pc[:, 2]
        for i in (0, 1):
            qt = pc[:, i] / np.where(z == 0, 1.0, z)
            exact &= (qt.astype(np.float32).astype(np.float64) == qt) | (z <= view.near)
    return torch.from_numpy(exact)


def _rect(El, Er, Et, Eb, ntx, nty):
    """gs_tile_rect's truncations on edges E (tile units, before the +1 of tx1 / ty1); (0, 0, 0, 0) when empty."""
    def lo(e):
        return int(math.floor(min(max(e, 0.0), 2.0e9)))

    def hi(e):
        return int(math.floor(min(max(e + 1.0, 0.0), 2.0e9)))

    tx0, tx1, ty0, ty1 = lo(El), min(hi(Er), ntx), lo(Et), min(hi(Eb), nty)
    if not (tx1 > tx0 and ty1 > ty0):
        return (0, 0, 0, 0)
    return (tx0, tx1, ty0, ty1)


class Decision:
    """What view `view` must do with each Gaussian of g.

    mask [n] bool           the culling decision (z > near and inside the 1.2x frustum, on the narrowed constants)
    cull_decided [n] bool   the culling decision is exact (exact-arithmetic placement) or has its margin
    rect [n, 4] int64       the tile rectangle (tx0, tx1, ty0, ty1) for decided placements, (0,)*4 when empty
    cands [n] list          candidate rectangles: one for decided placements, two or more for ambiguous ones
    decided [n] bool        culling and rectangle decided
    delta [n] float         the largest edge bound of the placement (tiles); edge_delta [n, 4] per edge
    margin [n] float        the smallest distance of a rectangle edge from an integer, over the edges that matter
    p, cov, opa, rgb        float64 projected mean / depth, covariance (after the filter or lens), opacity, colour
    """


def _project(g, view, mode):
    """float64 projection of the float32 parameters: (res_pos, res_cov, mask, opa, rgb, keep) with the variant's
    filter or lens applied; keep: the antialias filter's det > 0 (float32) test."""
    import filter_oracle as FO
    import lens_oracle as LO
    pos = g["pos"].double()
    nq, ns = _activated(g)
    opa_a = g["opa"].double().sigmoid()
    rgb_a = g["rgb"].double().sigmoid()
    cam = view.cam()
    if mode == "opencv":
        ln = lens_of(view)
        ox, oy = f32((ln["cx"] - view.width / 2.0) / view.fx), f32((ln["cy"] - view.height / 2.0) / view.fy)
        rp, rc, mask = LO.global_culling_lens(pos, nq, ns, view.rot, view.tran, view.near, view.half_w, view.half_h,
                                              ln, ox, oy)
    else:
        rp, rc, mask = O.global_culling(pos, nq, ns, view.rot, view.tran, view.near, view.half_w, view.half_h)
    mask = mask.bool()
    keep = mask.clone()
    if mode == "antialias":
        idx = torch.nonzero(mask).squeeze(-1)
        cf, of, kp = FO.filtered(rc[idx], opa_a[idx], cam, "antialias", 0.3)
        rc = rc.clone()
        rc[idx] = cf
        opa_a = opa_a.clone()
        opa_a[idx] = of
        keep[idx] = kp
    return rp, rc, mask, opa_a, rgb_a, keep


def _cull_margin(g, view, mode):
    """([n], [n]) relative distance of the near-plane test and of the nearer frustum test from their boundaries
    (float64; the frustum margin is +inf behind the near plane)."""
    import lens_oracle as LO
    pc = g["pos"].double() @ view.rot.T + view.tran
    z = pc[:, 2]
    zs = torch.where(z > 0, z, torch.ones_like(z))
    xn, yn = pc[:, 0] / zs, pc[:, 1] / zs
    if mode == "opencv":
        ln = lens_of(view)
        ad, bd = LO.lens_map(xn, yn, "OPENCV", ln["k"])
        xn = ad + (ln["cx"] - view.width / 2.0) / view.fx
        yn = bd + (ln["cy"] - view.height / 2.0) / view.fy
    mz = (z / view.near - 1).abs()
    mx = (xn.abs() / view.half_w - 1).abs()
    my = (yn.abs() / view.half_h - 1).abs()
    return mz, torch.where(z > view.near, torch.minimum(mx, my), torch.full_like(mx, math.inf))


def decide(g, view, mode="none", exact=None):
    n = g["pos"].shape[0]
    rp, rc, mask, opa_a, rgb_a, keep = _project(g, view, mode)
    raw_sign = [det_sign(c) for c in _project(g, view, "none")[1].reshape(n, 4)] if mode == "antialias" else None
    ex = exact_culling(g, view)
    if exact is not None:
        ex = ex & exact
    mz, mxy = _cull_margin(g, view, mode)
    z = (g["pos"].double() @ view.rot.T + view.tran)[:, 2]
    if mode == "opencv":
        # the near-plane test comes before the lens and stays exact; the frustum test is on the distorted mean
        cull_decided = (ex & ((z <= view.near) | (mxy >= CULL_MARGIN))) | (torch.minimum(mz, mxy) >= CULL_MARGIN)
    else:
        cull_decided = ex | (torch.minimum(mz, mxy) >= CULL_MARGIN)
    cx_err, cov_err = CX_ERR[mode], COV_ERR[mode]
    rect = torch.zeros(n, 4, dtype=torch.int64)
    cands, decided = [], torch.zeros(n, dtype=torch.bool)
    delta = torch.zeros(n, dtype=torch.float64)
    edge_delta = torch.zeros(n, 4, dtype=torch.float64)
    margin = torch.full((n,), math.inf, dtype=torch.float64)
    c4 = rc.reshape(n, 4)
    for i in range(n):
        sign = det_sign(c4[i])
        if not bool(mask[i]) or not bool(keep[i]) or sign != 1:
            cands.append([(0, 0, 0, 0)])
            # visible but not kept (antialias: the unfiltered det, det_sign of the filter's input) or det <= 0
            ok = True
            if bool(mask[i]):
                ok = (sign is not None) if bool(keep[i]) else (raw_sign[i] is not None)
            decided[i] = bool(cull_decided[i]) and ok
            continue
        a, b, c, d = (float(t) for t in c4[i])
        det = a * d - b * c
        di, ai = a / (det + 1e-14), d / (det + 1e-14)
        sx, sy = math.sqrt(di * view.t2 * det), math.sqrt(ai * view.t2 * det)
        cx, cy = float(rp[i, 0]), float(rp[i, 1])
        eps_det = 2 * 34 * U * (abs(a * d) + abs(b * c)) / det
        sh_err = (cov_err + 5 * U + eps_det * 1e-14 / det) / 2 + U
        E, D = [], []
        for c0, s, lm, l in ((cx, -sx, view.leftmost, view.lx), (cx, sx, view.leftmost, view.lx),
                             (cy, -sy, view.topmost, view.ly), (cy, sy, view.topmost, view.ly)):
            e = (c0 + s - lm) / l
            err = (abs(c0) * cx_err + abs(s) * sh_err + 3 * U * (abs(c0) + abs(s) + abs(lm))) / l + 2 * U * (abs(e) + 1)
            E.append(e)
            D.append(2 * err)
        delta[i] = max(D)
        edge_delta[i] = torch.tensor(D)
        options = [sorted({e - dd, e, e + dd}) for e, dd in zip(E, D)]
        rs = {_rect(*combo, view.ntx, view.nty) for combo in itertools.product(*options)}
        # the candidate set spans only truncation changes: keep the rectangles of E +- delta
        cands.append(sorted(rs))
        base = _rect(*E, view.ntx, view.nty)
        rect[i] = torch.tensor(base)
        # the distance of the edges that matter (those whose truncation is not clamped away) from an integer
        for e, dd, j in zip(E, D, range(4)):
            lim = view.ntx if j < 2 else view.nty
            if -1.0 < e < lim + 1.0:
                margin[i] = min(float(margin[i]), abs(e - round(e)))
        decided[i] = bool(cull_decided[i]) and len(rs) == 1
    dec = Decision()
    dec.mask, dec.cull_decided, dec.rect, dec.cands, dec.decided = mask, cull_decided, rect, cands, decided
    dec.delta, dec.margin, dec.p, dec.cov, dec.opa, dec.rgb, dec.keep = delta, margin, rp, rc, opa_a, rgb_a, keep
    dec.exact, dec.edge_delta = ex, edge_delta
    return dec


def det_sign(c4):
    """The float32 test det > 0 of gs_tile_rect (and of the antialias filter): 1 when det is far inside the normal
    float32 range and larger than its roundoff bound; 0 when b = c = 0 and a d is so small that it underflows to 0 in
    float32 whatever the last bits of a and d; None (undecided) otherwise."""
    a, b, c, d = (float(t) for t in c4)
    det = a * d - b * c
    if b == 0.0 and c == 0.0 and abs(a * d) * (1 + 64 * U) < 2.0 ** -150:
        return 0
    if det >= 2.0 ** -100 and det > 68 * U * (abs(a * d) + abs(b * c)):
        return 1
    return None


def expected_lists(dec, rects, view, depth_key):
    """(gauss_idx [M] int64, accum [T+1] int32) of the oracle's exact (tile, depth, id) order on rectangles rects
    [n, 4], sorting the device's float32 depth keys depth_key [n]."""
    idx = torch.nonzero(rects[:, 1] > rects[:, 0]).squeeze(-1)
    r = rects[idx]
    gi, accum = O.bin_and_sort(dec.p[idx], dec.cov[idx], (r[:, 0], r[:, 1], r[:, 2], r[:, 3]), view.ntx, view.nty,
                               depth_key[idx])
    return idx[gi], accum


def counts_of(rects):
    return (rects[:, 1] - rects[:, 0]) * (rects[:, 3] - rects[:, 2])


def device_rects(idx, accum, n, ntx, nty_off=0):
    """[n, 4] rectangles read back from a frame's sorted instances (idx, accum), rows made view-relative by nty_off;
    raises when a Gaussian's tiles are not a full rectangle (a lost or duplicated instance)."""
    idx, accum = idx.long().cpu(), accum.long().cpu()
    M = idx.numel()
    tile = torch.repeat_interleave(torch.arange(accum.numel() - 1), accum[1:] - accum[:-1])
    assert tile.numel() == M, "tile ranges do not cover the instances"
    ty, tx = tile // ntx - nty_off, tile % ntx
    out = torch.zeros(n, 4, dtype=torch.int64)
    if M == 0:
        return out
    big = torch.iinfo(torch.int64).max
    tx0 = torch.full((n,), big).scatter_reduce(0, idx, tx, "amin")
    tx1 = torch.full((n,), -1).scatter_reduce(0, idx, tx, "amax") + 1
    ty0 = torch.full((n,), big).scatter_reduce(0, idx, ty, "amin")
    ty1 = torch.full((n,), -1).scatter_reduce(0, idx, ty, "amax") + 1
    cnt = torch.bincount(idx, minlength=n)
    has = cnt > 0
    area = (tx1 - tx0) * (ty1 - ty0)
    assert torch.equal(area[has], cnt[has]), "a Gaussian's instances are not one full rectangle"
    pairs = torch.unique(idx * (accum.numel()) + tile)
    assert pairs.numel() == M, "a (Gaussian, tile) instance is duplicated"
    out[has] = torch.stack([tx0, tx1, ty0, ty1], -1)[has]
    return out


def draw(dec, gi, accum, view, tiles=None):
    """fp64 padded image of the sorted lists (gs_oracle.draw)."""
    return O.draw(dec.p[gi], dec.rgb[gi], dec.opa[gi], dec.cov[gi], accum, view.Hp, view.Wp, view.fx, view.fy,
                  tiles=tiles)


# --------------------------------------------------------------------------------------------------------------------
# families
# --------------------------------------------------------------------------------------------------------------------
def near_plane(mode="none"):
    """Family 1: camera depth z at near, one ulp above and one ulp below, on the axis and off it; footprints from a
    few pixels to one that covers every tile (a Gaussian just past the near plane)."""
    v = View(64, 48, 64.0, near=0.25)
    b = Builder(v, seed=1)
    for z in (v.near, next_up(v.near), next_down(v.near)):
        for xn, yn in ((0.0, 0.0), (0.125, -0.0625), (-0.25, 0.125)):
            for s in (2.0 ** -6, 2.0 ** -3, 4.0):
                b.raw((xn * z, yn * z, z), (s, s, 0.0), opa=0.3, exact=True, tag="near")
    for i in range(12):                                       # ordinary Gaussians behind them
        b.at(-0.4 + 0.07 * i, 0.3 - 0.05 * i, 1.0 + 0.125 * i, 0.04, 0.03, opa=0.4, tag="body")
    g, ex, tags = b.build()
    return Scene(f"near-{mode}", 1, [v], g, ex, tags, mode)


def frustum(mode="none"):
    """Family 2: x/z and y/z at +-half_w / +-half_h, one ulp inside and one outside, alone and in the corners, at
    power-of-two depths.  Small footprints there lie outside the padded grid (visible, unbinned); large ones reach
    back into the border tiles."""
    v = View(96, 64, 128.0, 64.0, near=0.25)
    b = Builder(v, seed=2)
    hw, hh = v.half_w, v.half_h
    xs = [hw, next_down(hw), next_up(hw)]
    ys = [hh, next_down(hh), next_up(hh)]
    for z in (0.5, 1.0, 4.0):
        for sgn in (1.0, -1.0):
            for x in xs:
                for s in (2.0 ** -8, 2.0 ** -3):
                    b.raw((sgn * x * z, 0.0, z), (s * z, s * z, 0.0), opa=0.4, exact=True, tag="fx")
            for y in ys:
                for s in (2.0 ** -8, 2.0 ** -3):
                    b.raw((0.0, sgn * y * z, z), (s * z, s * z, 0.0), opa=0.4, exact=True, tag="fy")
        for x, y in itertools.product(xs, ys):                 # corners
            for sx, sy in ((1, 1), (-1, 1), (1, -1), (-1, -1)):
                b.raw((sx * x * z, sy * y * z, z), (2.0 ** -3 * z,) * 2 + (0.0,), opa=0.4, exact=True, tag="corner")
    for i in range(8):
        b.at(-0.3 + 0.08 * i, -0.4 + 0.1 * i, 1.5 + 0.25 * i, 0.05, 0.05, opa=0.5, tag="body")
    g, ex, tags = b.build()
    return Scene(f"frustum-{mode}", 2, [v], g, ex, tags, mode)


def unbinned(mode="none"):
    """Family 3: visible Gaussians whose footprint lies wholly outside the padded grid on each side and corner (the
    fmaxf(., 0) clamp on the left / top, min(., ntx / nty) on the right / bottom), one whose float32 det underflows
    to 0 (det <= 0; with the antialias filter: keep = false), culled ones behind the camera, and binned ones."""
    v = View(128, 96, 128.0, near=0.25)
    b = Builder(v, seed=3)
    gx, gy = v.Wp / 2.0 / v.fx, v.Hp / 2.0 / v.fy               # the padded grid's half-extent, normalised
    fx_, fy_ = 0.5 * (gx + v.half_w), 0.5 * (gy + v.half_h)      # between the grid edge and the frustum edge
    h = 0.25 * min(v.half_w - gx, v.half_h - gy)
    for xn, yn in ((fx_, 0.0), (-fx_, 0.0), (0.0, fy_), (0.0, -fy_), (fx_, fy_), (-fx_, -fy_), (fx_, -fy_)):
        for z in (0.5, 2.0):
            b.at(xn, yn, z, h, h, tag="outside")
    for xn in (0.0, 0.125):                                      # det underflows: a, d ~ 1e-26 at z = 2^30
        b.raw((xn * 2.0 ** 30, 0.0, 2.0 ** 30), (0.0, 0.0, 0.0), opa=0.5, exact=True, tag="det0")
    for z in (-1.0, 0.0):                                        # behind the camera / at its centre: culled
        b.raw((0.0, 0.0, z), (0.1, 0.1, 0.1), exact=True, tag="behind")
    for i in range(10):
        b.at(-0.35 + 0.07 * i, 0.25 - 0.05 * i, 1.0 + 0.25 * i, 0.06, 0.04, tag="body")
    g, ex, tags = b.build()
    return Scene(f"unbinned-{mode}", 3, [v], g, ex, tags, mode)


OFFSETS = (2.0 ** -10 * 0.9, 2.0 ** -12, 2.0 ** -14, 0.25)     # tile-unit distances of an edge from a border


def tile_borders(width, height, mode="none", fx=None):
    """Family 4: bbox edges at every tile border of the padded grid (both padded-grid edges included) and
    OFFSETS on either side of it, plus a few placed exactly on a border (ambiguous by construction)."""
    v = View(width, height, fx or 4.0 * width, near=0.25)
    b = Builder(v, seed=4 + width + 7 * height)
    r = 1.0
    for k in range(v.ntx + 1):
        for off in OFFSETS:
            for sgn in (1, -1):
                for side in ("l", "r"):
                    b.edge(side, k, sgn * off, r, h=0.3)
                    r += 2.0 ** -7
    for k in range(v.nty + 1):
        for off in OFFSETS:
            for sgn in (1, -1):
                for side in ("t", "b"):
                    b.edge(side, k, sgn * off, r, h=0.3)
                    r += 2.0 ** -7
    for side, k in (("l", 0), ("r", v.ntx), ("t", 1), ("b", v.nty)):     # on the border itself
        b.edge(side, k, 0.0, r, h=0.3)
        r += 2.0 ** -7
    g, ex, tags = b.build()
    return Scene(f"borders-{width}x{height}-{mode}", 4, [v], g, ex, tags, mode)


def emission(pattern):
    """Family 5: Gaussians at designed positions of the depth order with designed tile counts.

    A Gaussian without instances gets the depth key 0xffffffff (project.cu), so the empty ones always sort after
    every non-empty one: in the fused frame empty lanes only trail a warp's non-empty lanes.  The patterns:
      n1       one Gaussian, one instance;  n1-empty  one Gaussian, no instance (M = 0)
      n31      31 one-tile Gaussians: a warp of 31 lanes with 31 instances
      n33      33: warp totals 32 and 1 (lane 0 only)
      n100     63 non-empty (warp 1: lanes 0..30) then 37 empty (n not a multiple of 32)
      n255     warp totals 32, 33, >= 1025 (nine grid-wide-row rectangles), a grid-wide rectangle, exact duplicates,
               193 non-empty (warp 6: lane 0 only) then 62 empty (warp 7: every lane count 0)
      n257     257 non-empty: block 1 holds one Gaussian
    """
    v = View(256, 128, 256.0, near=0.25)
    b = Builder(v, seed=5)
    ntx, nty = v.ntx, v.nty
    r = [1.0]

    def one(k):
        t = k % (ntx * nty)
        ty, tx = divmod(t, ntx)
        b.tiles(tx, tx + 1, ty, ty + 1, r[0], tag="one")
        r[0] += 2.0 ** -7

    def rect(tx0, tx1, ty0, ty1, tag="rect"):
        b.tiles(tx0, tx1, ty0, ty1, r[0], tag=tag)
        r[0] += 2.0 ** -7

    def empty(k):
        for j in range(k):
            b.raw((0.0, 0.0, -1.0 - j), (0.1, 0.1, 0.1), tag="empty")          # culled: no instance

    counts = []
    if pattern == "n1":
        one(37)
    elif pattern == "n1-empty":
        empty(1)
    elif pattern == "n31":
        for k in range(31):
            one(3 * k)
    elif pattern == "n33":
        for k in range(33):
            one(5 * k + 1)
    elif pattern == "n100":
        for k in range(63):
            one(2 * k)
        empty(37)
    elif pattern == "n255":
        for k in range(32):                                   # warp 0: 32
            one(k)
        for k in range(31):                                   # warp 1: 31 + 2 = 33
            one(40 + k)
        rect(3, 5, 6, 7)
        for k in range(9):                                    # warp 2: 9 x 16 x 8... >= 1025
            rect(0, ntx, 0, nty, tag="grid")
        for k in range(23):
            one(90 + k)
        rect(0, ntx, 3, 4, tag="wide")                        # warp 3: one grid-wide row
        for k in range(31):
            one(k * 3)
        for k in range(5):                                    # exact duplicates (equal keys): ordered by id
            b.rows.append(b.rows[-1])
        for k in range(193 - 32 * 4 - 5):
            one(7 * k + 2)
        empty(62)
    elif pattern == "n257":
        for k in range(257):
            one(k)
    else:
        raise ValueError(pattern)
    g, ex, tags = b.build()
    return Scene(f"emit-{pattern}", 5, [v], g, ex, tags, claims=dict(pattern=pattern))


EMISSION = ("n1", "n1-empty", "n31", "n33", "n100", "n255", "n257")


def tile_ranges(case):
    """Family 6: one-tile Gaussians on a 32 x 32 tile grid, placed so that the sorted keys have M instances with
    empty tiles before the first, after the last and in runs that cross tile_ranges_kernel's 8-key and 2048-key
    boundaries; every instance in one tile; exactly one instance per tile."""
    v = View(512, 512, 512.0, near=0.25)
    b = Builder(v, seed=6)
    T = v.ntx * v.nty
    tiles = []
    if case.startswith("m"):                                  # M instances, spread with gaps
        m = int(case[1:])
        gen = torch.Generator().manual_seed(m)
        spread = sorted(torch.randint(1, T - 1, (m,), generator=gen).tolist())
        tiles = spread
        if m == 9:                                            # a run of empty tiles between keys 7 and 8
            tiles = [5, 6, 6, 9, 17, 17, 17, 20, 900]
        if m >= RANGE_BLOCK - 1:                              # the first block's keys in tiles 10..299, then a gap
            low = RANGE_BLOCK if m > RANGE_BLOCK else m - 1
            tiles = sorted(torch.randint(10, 300, (low,), generator=gen).tolist()) + [1000] * (m - low)
    elif case == "one-tile":
        tiles = [517] * 2049
    elif case == "per-tile":
        tiles = list(range(T))
    else:
        raise ValueError(case)
    r = 1.0
    for t in tiles:
        ty, tx = divmod(t, v.ntx)
        b.tiles(tx, tx + 1, ty, ty + 1, r)
        r += 2.0 ** -9
    g, ex, tags = b.build()
    return Scene(f"ranges-{case}", 6, [v], g, ex, tags, claims=dict(tiles=sorted(tiles)))


RANGES = ("m1", "m7", "m8", "m9", "m2047", "m2048", "m2049", "one-tile", "per-tile")


def grid(case):
    """Family 7: tile-sort key widths and the grid limits.  n_tiles 1, 2, 2^8, 2^8 + 1, 65536 (2-byte keys, the
    largest id 65535 used) and 65792 (4-byte keys); ntx = 65535 at H = 16 and 32.  A few hundred Gaussians in the
    first and last tiles and rows and across the grid; forward only, images compared on sampled tiles."""
    sizes = {"t1": (16, 16), "t2": (32, 16), "t256": (256, 256), "t257": (4112, 16), "t65536": (4096, 4096),
             "t65792": (4112, 4096), "w65535h16": (1048560, 16), "w65535h32": (1048560, 32)}
    w, h = sizes[case]
    v = View(w, h, float(max(w, h)) / 2.0, near=0.25)
    b = Builder(v, seed=7)
    ntx, nty = v.ntx, v.nty
    r = 1024.0                                                # deep: a quarter tile is above the scale floor
    spots = {(0, 0), (ntx - 1, nty - 1), (ntx - 1, 0), (0, nty - 1), (ntx // 2, nty // 2)}
    gen = torch.Generator().manual_seed(ntx * 7 + nty)
    for _ in range(200):
        spots.add((int(torch.randint(0, ntx, (1,), generator=gen)), int(torch.randint(0, nty, (1,), generator=gen))))
    for tx, ty in sorted(spots):
        b.tiles(tx, tx + 1, ty, ty + 1, r)
        r += 0.5
    if ntx > 1:
        b.tiles(max(ntx - 3, 0), ntx, nty - 1, nty, r)        # the last tiles of the last row
        r += 0.5
        # one Gaussian as wide as the grid: its bbox overhangs both ends (a one-row footprint is so thin that the
        # 1e-14 added to det shortens its half-width by up to 0.3 %, 100 tiles at ntx = 65535)
        b.tiles(-ntx // 16 - 1, ntx + ntx // 16 + 1, 0, 1, r, tag="grid-wide")
    g, ex, tags = b.build()
    tiles = sorted({ty * ntx + tx for tx, ty in spots})[:24] + [ntx * nty - 1]
    return Scene(f"grid-{case}", 7, [v], g, ex, tags, forward_only=True, sample_tiles=sorted(set(tiles)))


GRID = ("t1", "t2", "t256", "t257", "t65536", "t65792", "w65535h16", "w65535h32")


def batch_rows_limit():
    """Family 7: a batch of B = 15 views of 16 x 69904 px: B Hp / 16 = 65535 tile rows, the largest that fits the
    rectangle's 16-bit row field.  Views differ by a quarter turn about the axis (0 or 180 degrees: the image is
    not square); a few hundred Gaussians, some in the last row of the last view."""
    views = [View(16, 69904, 34952.0, rot=rot_z(2 * (k % 2)), near=0.25) for k in range(15)]
    v = views[0]
    b = Builder(v, seed=8)
    r = 1024.0
    gen = torch.Generator().manual_seed(15)
    rows = sorted({0, v.nty - 1, v.nty - 2, v.nty // 2} | set(torch.randint(0, v.nty, (200,), generator=gen).tolist()))
    for ty in rows:
        b.tiles(0, 1, ty, ty + 1, r)
        r += 0.5
    g, ex, tags = b.build()
    return Scene("grid-batch15", 7, views, g, ex, tags, forward_only=True, sample_tiles=[0, v.nty - 1])


def batched(scene):
    """Family 8: `scene` as a batch of three views: the scene's view, the same view turned half a turn about the
    optical axis (exact: R has entries 0, +-1), and the scene's view again."""
    v = scene.views[0]
    turned = View(v.width, v.height, v.fx, v.fy, rot=rot_z(2), tran=tuple(v.tran.tolist()), near=v.near,
                  thresh=v.thresh)
    return Scene(scene.name + "-batch3", 8, [v, turned, v], scene.g, scene.exact, scene.tags, scene.mode,
                 scene.claims)


BORDER_SIZES = ((16, 16), (16, 80), (80, 16), (17, 16), (31, 31), (96, 48))


def single_view_builders():
    """{name: builder} of the single-view scenes of families 1-6 (projection variant 'none'), plus families 1-4 with
    the antialias filter and the OPENCV lens."""
    out = {}
    for mode in ("none", "antialias", "opencv"):
        out[f"near-{mode}"] = (lambda m=mode: near_plane(m))
        out[f"frustum-{mode}"] = (lambda m=mode: frustum(m))
        out[f"unbinned-{mode}"] = (lambda m=mode: unbinned(m))
        for w, h in BORDER_SIZES:
            out[f"borders-{w}x{h}-{mode}"] = (lambda w=w, h=h, m=mode: tile_borders(w, h, m))
    for p in EMISSION:
        out[f"emit-{p}"] = (lambda p=p: emission(p))
    for c in RANGES:
        out[f"ranges-{c}"] = (lambda c=c: tile_ranges(c))
    return out


BUILDERS = single_view_builders()
GRID_BUILDERS = {f"grid-{c}": (lambda c=c: grid(c)) for c in GRID}
GRID_BUILDERS["grid-batch15"] = batch_rows_limit


def overflow():
    """A diverged Gaussian: coordinates near 3e38 under a rotated camera whose rows 0 and 2 both have a dot product of
    0.707 |p| with p, so p_c.x and p_c.z both overflow float32 to +inf and x/z is NaN.  (In float64 nothing overflows.)
    The device must cull it: |x/z| < half_w is false for NaN."""
    v = View(64, 64, 64.0, near=0.25)
    u = torch.tensor([1.0, 1.0, 1.0], dtype=torch.float64) / math.sqrt(3.0)
    w1 = torch.tensor([1.0, -1.0, 0.0], dtype=torch.float64) / math.sqrt(2.0)
    w2 = torch.linalg.cross(u, w1)
    r0, r2 = (u + w1) / math.sqrt(2.0), (u - w1) / math.sqrt(2.0)
    rot = torch.stack([r0, w2, r2])
    v.rot = rot.float().double()
    b = Builder(v, seed=9)
    b.raw((3e38, 3e38, 3e38), (0.1, 0.1, 0.1), tag="overflow")
    b.raw((-3e38, 2e38, 3e38), (0.1, 0.1, 0.1), tag="overflow")
    for i in range(4):                                        # finite companions, in front of the camera
        p = rot.T @ torch.tensor([0.1 * i - 0.15, 0.05, 2.0 + i], dtype=torch.float64)
        b.raw(p.tolist(), (0.02, 0.02, 0.02), tag="body")
    g, ex, tags = b.build(shuffle=False)
    return Scene("overflow", 2, [v], g, ex, tags)
