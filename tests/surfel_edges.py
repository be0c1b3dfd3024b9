"""Seeded 2D Gaussian surfel scenes whose per-tile instance lists sit on the surfel blend kernels' edges
(blend_surfel.cu: staging chunks of 64 records forward and 32 backward, the early exit, the median-depth index and
the distortion's m0 shift), their per-tile fp64 profile, and a comparator that sees a single lost, duplicated,
swapped or stale instance.

Test infrastructure only, built on tests/surfel_oracle.py (SO).  Every surfel is fronto-parallel (camera rot = I,
scale[:, 2] = 0, quat a rotation about the view axis) and placed in pixel and depth terms:

* confined surfels: sigma 1.3-2 px, centred within 1 px of a tile's centre, so their rectangle (the 3-sigma disk's
  box joined with the sqrt(2)/2 px box) is exactly that tile: each adds one instance to one tile, and its
  per-surfel gradient is its per-instance gradient;
* walls: huge disks (sigma thousands of px along x) spanning every tile, at a fixed depth, that saturate tiles (or
  only their top rows) at the index of the tile's depth order set by the number of confined surfels in front.

Every fixture is checked when it is built: rectangle edges >= 0.01 tile from a tile border (fp64, SO.disk_box), no
live transmittance within a log-margin of 1e-4 of the stop T = 1e-4 or of the median threshold T = 0.5 (so fp32
and fp64 make every stop and median decision alike; in particular no pixel holds two alpha-clamped instances, whose
product is 1e-4 to the last bit), no screen-filter / intersection branch tie (SO.without_branch_ties removes
nothing), camera-z keys >= 1e-3 relative apart within a tile except one group of exact duplicates, and the designed
per-tile counts, last live indices and median indices.
"""
from __future__ import annotations

import math

import torch

import gs_oracle as O
import surfel_oracle as SO
import synthetic as S

TILE = 16
T_STOP = 1e-4
T_MED = 0.5
NAMES = ("pos", "rgb", "opa", "quat", "scale")
BG = (0.2, 0.5, 0.1)
DIST_NEAR, DIST_FAR = 0.2, 100.0
FWD_CH, BWD_CH = 64, 32                    # blend_surfel_fwd_kernel / blend_surfel_bwd_kernel staging chunks

COUNTS = (0, 1, 2, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 191, 192, 193, 300)
# Last live index of the saturating tiles of `stops`.  0 and 1 are out of reach: alpha is clamped at 0.99, and two
# clamped instances leave T = 1e-4 exactly (fp32 9.99998e-5, fp64 1.0000000000000018e-4: a tie), so the earliest
# stop that is not a tie is after three instances, at L = 2.
STOPS = (2, 30, 31, 32, 33, 62, 63, 64, 65, 95, 96, 127, 128, 129)
LONG_TAIL = (64, 600)                      # (L, tail) of the one tile with a long tail; the others have 70, so
TAIL = 70                                  # every STOPS tile exits early in both blend kernels
MEDIANS = (31, 32, 33, 63, 64, 65)


def _logit(p):
    p = torch.as_tensor(p, dtype=torch.float64)
    return torch.log(p) - torch.log1p(-p)


def camera(view):
    return O.Camera(view.width, view.height, view.fx, view.fy, view.rot, view.tran, view.near)


class _Scene:
    """Accumulates fronto-parallel surfels given in pixel / depth terms (centre (u, v) in padded pixels, camera z,
    std (su, sv) in px, in-plane angle, opacity) and converts them to world-space parameters."""

    def __init__(self, width, height, seed):
        self.view = S.make_view(width, height, 0)          # rot = I, tran = (0, 0, 4)
        self.cam = camera(self.view)
        self.Wp, self.Hp = self.cam.Wp, self.cam.Hp
        self.gen = torch.Generator().manual_seed(seed)
        self.rows = []                                     # [u, v, z, su, sv, theta, opa, tile or -1, role]

    def rand(self, lo, hi, n=None):
        t = torch.rand(() if n is None else (n,), generator=self.gen, dtype=torch.float64)
        return lo + (hi - lo) * t

    def add(self, u, v, z, su, sv, theta, opa, tile, role):
        self.rows.append([float(u), float(v), float(z), float(su), float(sv), float(theta), float(opa), int(tile),
                          role])

    def confined(self, tile, z, opa, role="confined"):
        ty, tx = divmod(tile, self.cam.ntx)
        s = float(self.rand(1.3, 2.0))
        self.add(tx * TILE + 8.0 + float(self.rand(-1, 1)), ty * TILE + 8.0 + float(self.rand(-1, 1)), z, s,
                 s * float(self.rand(0.75, 1.0)), float(self.rand(0, math.pi)), opa, tile, role)

    def wall(self, u, v, z, su, sv, opa):
        self.add(u, v, z, su, sv, 0.0, opa, -1, "wall")

    def build(self):
        n = len(self.rows)
        u, v, z, su, sv, th, opa = (torch.tensor([r[k] for r in self.rows], dtype=torch.float64) for k in range(7))
        cam = self.cam
        pos = torch.stack([(u - self.Wp // 2) / cam.fx * z, (v - self.Hp // 2) / cam.fy * z, z - 4.0], -1)
        quat = torch.stack([torch.cos(th / 2), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64),
                            torch.sin(th / 2)], -1)
        rgb = self.rand(-1.5, 1.5, 3 * n).reshape(n, 3)
        shrink = torch.ones(n, dtype=torch.float64)
        for _ in range(50):      # every rectangle edge >= 0.01 tile from a tile border: fp32 cannot move it
            scale = torch.stack([su * shrink * z / cam.fx - O.EPS, sv * shrink * z / cam.fx - O.EPS,
                                 torch.zeros(n, dtype=torch.float64)], -1)
            near = edge_distance(pos, quat, scale, cam) < 0.01
            if not bool(near.any()):
                break
            shrink = torch.where(near, shrink * 0.995, shrink)
        else:
            raise AssertionError("surfel_edges: rectangle edges stay on tile borders")
        g = dict(pos=pos, rgb=rgb, opa=_logit(opa), quat=quat, scale=scale)
        perm = torch.randperm(n, generator=self.gen)       # ids are not in depth order
        g = {q: t[perm].float().contiguous() for q, t in g.items()}
        g["scale"][:, 2] = 0.0
        tile_of = torch.tensor([r[7] for r in self.rows], dtype=torch.int64)[perm]
        role = [self.rows[i][8] for i in perm.tolist()]
        return g, tile_of, role, perm


def edge_distance(pos, quat, scale, cam):
    """[n] distance (in tiles) of each surfel's nearest rectangle edge to a tile border, fp64 (SO.disk_box joined
    with the sqrt(2)/2 px box); edges more than half a tile outside the grid are clamped away and do not count."""
    M, _, pc = SO.surfel_matrix(pos, quat, scale, cam)
    ex, ey, hx, hy, _ = SO.disk_box(M)
    cx, cy = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    rx, ry = 0.70710678 / cam.fx, 0.70710678 / cam.fy
    ex0 = (torch.minimum(ex - hx, cx - rx) - cam.leftmost) / cam.tile_lx
    ex1 = (torch.maximum(ex + hx, cx + rx) - cam.leftmost) / cam.tile_lx
    ey0 = (torch.minimum(ey - hy, cy - ry) - cam.topmost) / cam.tile_ly
    ey1 = (torch.maximum(ey + hy, cy + ry) - cam.topmost) / cam.tile_ly
    d = []
    for e, lim in ((ex0, cam.ntx), (ex1, cam.ntx), (ey0, cam.nty), (ey1, cam.nty)):
        inside = (e > -0.5) & (e < lim + 0.5)
        d.append(torch.where(inside, (e - e.round()).abs(), torch.full_like(e, math.inf)))
    return torch.stack(d, -1).amin(1)


# --------------------------------------------------------------------------------------------------------------
# profile
# --------------------------------------------------------------------------------------------------------------
def _front(g, cam):
    """fp64 matrices, opacities and the oracle's binning of the fp32 parameters g."""
    p = {q: t.double() for q, t in g.items()}
    M, _, pc = SO.surfel_matrix(p["pos"], p["quat"], p["scale"], cam)
    zc = pc[:, 2]
    visible = (zc > cam.near) & ((pc[:, 0] / zc).abs() < cam.half_w) & ((pc[:, 1] / zc).abs() < cam.half_h)
    rects = SO.surfel_rects(M, cam, visible)
    key = (g["pos"].float() @ cam.rot.float().T + cam.tran.float())[:, 2]
    gi, accum = O.bin_and_sort(torch.stack([key] * 3, -1), None, rects, cam.ntx, cam.nty, depth_key=key)
    return dict(M=M, op=p["opa"].sigmoid(), gi=gi, accum=accum.long(), key=key)


def tile_eval(fe, cam, t):
    """(alpha [256, k], z [256, k]) of tile t's k instances in blend order (fp64, the kernel's rule: clamp 0.99,
    skip below 1/255 and at z <= near); pixel p = row * 16 + column."""
    s, e = int(fe["accum"][t]), int(fe["accum"][t + 1])
    ty, tx = divmod(t, cam.ntx)
    r16 = torch.arange(16, dtype=torch.float64)
    ix = (tx * 16 + r16).reshape(1, 16).expand(16, 16).reshape(-1, 1)
    iy = (ty * 16 + r16).reshape(16, 1).expand(16, 16).reshape(-1, 1)
    qx = (ix + 0.5 - cam.Wp // 2) / cam.fx
    qy = (iy + 0.5 - cam.Hp // 2) / cam.fy
    g = fe["gi"][s:e]
    alpha, z, _, _ = SO.pixel_eval(fe["M"][g], fe["op"][g], qx, qy, cam.fx, cam.fy)
    alpha = torch.where(z > cam.near, alpha, torch.zeros_like(alpha))
    return alpha, z


def transmittance(alpha):
    """[256, k + 1] transmittance before each instance and at the end, with the kernel's stop (an instance met at
    T <= 1e-4 is not blended)."""
    T = torch.ones(alpha.shape[0], dtype=torch.float64)
    out = [T]
    for j in range(alpha.shape[1]):
        T = torch.where(T > T_STOP, T * (1 - alpha[:, j]), T)
        out.append(T)
    return torch.stack(out, 1)


def profile(fx):
    """Per tile (fp64 through SO.pixel_eval): count; L, the largest last live index over its pixels (-1: empty; an
    instance is live for a pixel while T > 1e-4 before it); full (every pixel ends with T <= 1e-4); top (rows 0-7
    end below the stop, rows 8-15 do not); med [256] median instance index per pixel (-1: none); stop_margin, the
    smallest |ln(T / 1e-4)| over its pixels' transmittances; med_margin, the smallest |ln(T / 0.5)| before a blended
    live instance; and skip_first: some pixel meets only skipped instances (alpha < 1/255) from its stop to the end
    of that backward chunk, so it is marked done by a skipped instance."""
    cam = fx.cam
    fe = fx.fe
    nt = cam.ntx * cam.nty
    count = fe["accum"][1:] - fe["accum"][:-1]
    out = dict(count=count, L=torch.full((nt,), -1, dtype=torch.int64), full=torch.zeros(nt, dtype=torch.bool),
               top=torch.zeros(nt, dtype=torch.bool), med=torch.full((nt, 256), -1, dtype=torch.int64),
               stop_margin=torch.full((nt,), math.inf, dtype=torch.float64),
               med_margin=torch.full((nt,), math.inf, dtype=torch.float64), skip_first=torch.zeros(nt, dtype=torch.bool))
    for t in range(nt):
        k = int(count[t])
        if k == 0:
            continue
        alpha, _ = tile_eval(fe, cam, t)
        tr = transmittance(alpha)
        live = tr[:, :-1] > T_STOP
        last = torch.where(live, torch.arange(k).expand(256, k), torch.full((256, k), -1)).amax(1)
        out["L"][t] = int(last.max())
        dead = tr[:, -1] <= T_STOP
        out["full"][t] = bool(dead.all())
        out["top"][t] = bool(dead[:128].all()) and not bool(dead[128:].any())
        blended = live & (alpha > 0)
        ismed = blended & (tr[:, :-1] > T_MED)
        out["med"][t] = torch.where(ismed, torch.arange(k).expand(256, k), torch.full((256, k), -1)).amax(1)
        out["stop_margin"][t] = float((tr / T_STOP).log().abs().min())
        if bool(blended.any()):
            out["med_margin"][t] = float((tr[:, :-1][blended] / T_MED).log().abs().min())
        stopped = last < k - 1
        for p in stopped.nonzero().flatten().tolist():
            j0 = int(last[p]) + 1
            j1 = min(k, BWD_CH * (j0 // BWD_CH + 1))
            if not bool((alpha[p, j0:j1] > 0).any()):
                out["skip_first"][t] = True
                break
    return out


def consumed(prof, ch):
    """Instances a blend kernel with staging chunk ch consumes per tile: a pixel whose transmittance falls below the
    stop after instance L is marked done when it meets instance L + 1, and only a whole chunk is ever skipped, so
    min(count, ch (floor((L + 1) / ch) + 1)); count where some pixel never stops (L = count - 1)."""
    L, cnt = prof["L"], prof["count"]
    return torch.minimum(cnt, ch * (torch.div(L + 1, ch, rounding_mode="floor") + 1))


class Fixture:
    """A scene plus what it was built to hit.  g: fp32 CPU parameters; tile_of[n]: tile of a confined surfel, -1 for
    a wall; role[n]; targets {tile: designed value}; prof: profile(); up: upstream weights of the final image."""

    def __init__(self, name, sc, g, tile_of, role, targets=None):
        self.name = name
        self.view = sc.view
        self.cam = sc.cam
        self.g = g
        self.n = g["pos"].shape[0]
        self.tile_of = tile_of
        self.role = role
        self.targets = dict(targets or {})
        self.dist_bound = None                 # per-pixel distortion bound [Hp, Wp] (the `distortion` scene)
        self.fe = _front(g, self.cam)
        self.prof = profile(self)
        gen = torch.Generator().manual_seed(len(name) * 7919 + self.n)
        k = 16
        hi = torch.randn(self.n, 3, k - 1, generator=gen) * 0.1
        self.sh16 = torch.cat([(g["rgb"] / S.SH_C0).unsqueeze(-1), hi], -1).reshape(self.n, 3 * k).contiguous()

    def params(self, kind, dtype=torch.float64):
        """Parameters of output kind `kind` (sh16-*: SH coefficients, exp-*: log scales of the same sizes)."""
        p = {q: t.clone() for q, t in self.g.items()}
        if kind.startswith("sh16"):
            p["rgb"] = self.sh16.clone()
        if kind.startswith("exp"):
            p["scale"] = torch.log(p["scale"].abs().double() + O.EPS).float()
        return {q: t.to(dtype) for q, t in p.items()}

    def weights(self, kind, final=True, seed=0):
        """Upstream weights {output: tensor} of kind: rgb (image), maps / sh16-maps / exp-maps (image and all five
        maps), median-only (the median map alone)."""
        cam = self.cam
        shape = (cam.height, cam.width) if final else (cam.Hp, cam.Wp)
        gen = torch.Generator().manual_seed(seed + 17 * len(kind) + (0 if final else 1))
        which = {"rgb": ("image",), "median-only": ("median",)}.get(kind, ("image",) + SO_MAPS)
        w = {}
        for k in which:
            s = shape + ((3,) if k in ("image", "normal") else ())
            w[k] = torch.randn(s, generator=gen, dtype=torch.float64) * (1.0 if k in ("image", "alpha", "normal")
                                                                        else 0.2)
        return w


SO_MAPS = ("alpha", "depth", "median", "distortion", "normal")


def _check_keys(fx):
    """Within every tile, consecutive camera-z keys differ by >= 1e-3 relative, except exact duplicates of a clone
    group (same position, ordered by id)."""
    fe, cam = fx.fe, fx.cam
    clone = torch.tensor([r == "clone" for r in fx.role])
    for t in range(cam.ntx * cam.nty):
        s, e = int(fe["accum"][t]), int(fe["accum"][t + 1])
        g = fe["gi"][s:e]
        k = fe["key"][g].double()
        for a in range(len(g) - 1):
            if k[a + 1] == k[a]:
                assert bool(clone[g[a]]) and bool(clone[g[a + 1]]) and int(g[a]) < int(g[a + 1]), (fx.name, t)
                assert torch.equal(fx.g["pos"][g[a]], fx.g["pos"][g[a + 1]])
            else:
                assert float(k[a + 1] / k[a]) >= 1 + 1e-3, (fx.name, t, float(k[a]), float(k[a + 1]))


def _check_branch_ties(fx):
    n = fx.n
    for s in range(0, n, 256):
        part = {q: t[s:s + 256] for q, t in fx.g.items()}
        assert SO.without_branch_ties(part, fx.cam)["pos"].shape[0] == part["pos"].shape[0], fx.name


def _settle(name, sc, targets, med_margin=1e-4, tries=40):
    """Build sc, re-drawing the opacities of the confined surfels of every tile whose transmittances come within a
    log-margin of 1e-4 of the stop or of med_margin of the median threshold, until none does."""
    for _ in range(tries):
        g, tile_of, role, perm = sc.build()
        fx = Fixture(name, sc, g, tile_of, role, targets)
        bad = (fx.prof["stop_margin"] < 1e-4) | (fx.prof["med_margin"] < med_margin)
        if not bool(bad.any()):
            _check_keys(fx)
            _check_branch_ties(fx)
            return fx
        for r in sc.rows:
            if r[7] >= 0 and bool(bad[r[7]]):
                r[6] = min(0.9, r[6] * float(sc.rand(0.97, 1.03)))
    raise AssertionError(f"{name}: could not clear the stop and median ties")


def _depths(sc, n, lo, hi):
    """n camera z in [lo, hi], >= 1e-3 relative apart, in random order."""
    z = lo * (hi / lo) ** ((torch.randperm(n, generator=sc.gen).double() + sc.rand(0.4, 0.6, n)) / max(n, 1))
    return z.tolist()


def build_counts(seed=0):
    """Faint confined surfels (optical depth ~2 at the centre: never saturates): tiles holding exactly COUNTS
    instances, 109 x 45 (border tiles cropped).  The tile of 33 holds a group of 4 exact duplicates."""
    ntx, nty = 7, 3
    sc = _Scene(ntx * TILE - 3, nty * TILE - 3, seed)
    order = torch.randperm(ntx * nty, generator=sc.gen).tolist()
    targets = {}
    for t, c in zip(order, COUNTS):
        opa = (sc.rand(0.2, 0.45, max(c, 1)) if c <= 2 else min(0.45, 2.0 / c) * sc.rand(0.8, 1.2, c)).tolist()
        for z, o in zip(_depths(sc, c, 2.0, 2.0 * 1.002 ** (c + 1)), opa):
            sc.confined(t, z, o)
        if c == 33:                               # a clone group: same centre and depth, other shape and colour
            u, v, z = sc.rows[-1][:3]
            for j in range(4):
                r = sc.rows[-1 - j]
                r[0], r[1], r[2], r[8] = u, v, z, "clone"
        targets[t] = c
    fx = _settle("counts", sc, targets)
    for t, c in targets.items():
        assert int(fx.prof["count"][t]) == c and int(fx.prof["L"][t]) == c - 1, ("counts", t)
    assert not bool(fx.prof["full"].any())
    return fx


def _walls_top(sc, ycross, z0, opa=0.97):
    """Three walls over the whole image, uniform along x and fading down from the top: (1 - alpha(y))^3 = 1e-4 at
    pixel row ycross, so every pixel above it stops after the third wall and every pixel below it never stops."""
    a = 1 - T_STOP ** (1 / 3)
    sv = ycross / math.sqrt(-2 * math.log(a / opa))
    for j in range(3):
        sc.wall(sc.Wp / 2, 0.0, z0 + 0.1 * j, 40000.0, sv, opa)


def build_stops(seed=1):
    """107 x 75 (7 x 5 tiles, the border tiles cropped).  Three walls saturate tile rows 0-3 and rows 0-7 of tile
    row 4; in tile row 4 rows 8-15 never stop (one tile there has a tail of 80 as well).  A STOPS tile holds L - 2 faint confined surfels in front of the
    walls (so its last live index is L, the third wall) and a tail of 70 (one: 600) confined surfels behind them;
    the tails are small disks, so a tile corner meets only skipped instances after the stop."""
    ntx, nty = 7, 5
    sc = _Scene(ntx * TILE - 5, nty * TILE - 5, seed)
    _walls_top(sc, 4 * TILE + 8.0, 4.0)
    order = torch.randperm(4 * ntx, generator=sc.gen).tolist()
    targets = {}
    for t, L in zip(order, STOPS):
        nf = L - 2
        for z, o in zip(_depths(sc, nf, 2.0, 3.5), (min(0.3, 1.0 / max(nf, 1)) * sc.rand(0.8, 1.2, nf)).tolist()):
            sc.confined(t, z, o)
        nb = LONG_TAIL[1] if L == LONG_TAIL[0] else TAIL
        for z, o in zip(_depths(sc, nb, 5.0, 15.0 if nb > 100 else 8.0), sc.rand(0.05, 0.3, nb).tolist()):
            sc.confined(t, z, o)
        targets[t] = L
    tailed = 4 * ntx + 3                           # a bottom-row tile with a tail of 80: some pixels never stop
    for z, o in zip(_depths(sc, 80, 5.0, 8.0), sc.rand(0.05, 0.3, 80).tolist()):
        sc.confined(tailed, z, o)
    fx = _settle("stops", sc, targets)
    fx.tailed = tailed
    p = fx.prof
    for t, L in targets.items():
        assert int(p["L"][t]) == L and bool(p["full"][t]) and bool(p["skip_first"][t]), ("stops", t, L)
        assert int(p["count"][t]) >= L + 1 + TAIL
    assert int(p["count"].max()) >= 600
    assert bool(p["full"][:4 * ntx].all())
    bottom = [t for t in range(4 * ntx, 5 * ntx) if t != tailed]
    assert bool(p["top"][bottom].all())                      # rows 0-7 stop at the third wall, rows 8-15 never
    assert int(p["count"][tailed]) == 83 and int(p["L"][tailed]) == 82 and not bool(p["full"][tailed])
    return fx


def build_median(seed=2):
    """64 x 48.  One wall (alpha 0.6) over every tile at z = 4; a MEDIANS tile holds k faint confined surfels in
    front of it (T stays > 0.74), so every pixel's transmittance crosses 0.5 at the wall, instance k; 20 confined
    surfels behind it.  Median margins >= 1e-3."""
    ntx, nty = 4, 3
    sc = _Scene(ntx * TILE, nty * TILE, seed)
    sc.wall(sc.Wp / 2, sc.Hp / 2, 4.0, 40000.0, 40000.0, 0.6)
    order = torch.randperm(ntx * nty, generator=sc.gen).tolist()
    targets = {}
    for t, k in zip(order, MEDIANS):
        for z, o in zip(_depths(sc, k, 2.0, 3.5), (0.3 / k * sc.rand(0.8, 1.2, k)).tolist()):
            sc.confined(t, z, o)
        for z, o in zip(_depths(sc, 20, 5.0, 8.0), sc.rand(0.05, 0.3, 20).tolist()):
            sc.confined(t, z, o)
        targets[t] = k
    fx = _settle("median", sc, targets, med_margin=1e-3)
    for t, k in targets.items():
        assert bool((fx.prof["med"][t] == k).all()), ("median", t, k)
    assert float(fx.prof["med_margin"].min()) >= 1e-3
    return fx


def build_distortion(seed=3):
    """80 x 64: 19 tiles of 10 semi-transparent confined surfels at z = 50 (1 + 1.1e-3 j), a depth spread of 1 %
    (m ~ 1, spread of m ~ 4e-5), and one control tile of 10 spread over z in [2, 50]."""
    ntx, nty = 5, 4
    sc = _Scene(ntx * TILE, nty * TILE, seed)
    control = int(torch.randint(ntx * nty, (1,), generator=sc.gen))
    for t in range(ntx * nty):
        zs = [2.0 * 25.0 ** (j / 9) for j in range(10)] if t == control else [50.0 * (1 + 1.1e-3 * j) for j in range(10)]
        perm = torch.randperm(10, generator=sc.gen).tolist()
        for j in perm:
            sc.confined(t, zs[j], float(sc.rand(0.2, 0.45)))
    fx = _settle("distortion", sc, {control: "control"})
    fx.control = control
    fx.dist_bound = distortion_bound(fx)
    return fx


BUILDERS = {"counts": build_counts, "stops": build_stops, "median": build_median, "distortion": build_distortion}


# --------------------------------------------------------------------------------------------------------------
# distortion
# --------------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24                                   # fp32 unit roundoff


def _dist_terms(fx, t):
    alpha, z = tile_eval(fx.fe, fx.cam, t)
    tr = transmittance(alpha)
    live = (tr[:, :-1] > T_STOP) & (alpha > 0)
    m = SO.distortion_m(z, DIST_NEAR, DIST_FAR)
    return alpha, z, tr, live, m


def _untile(cam, x):
    return x.reshape(cam.nty, cam.ntx, 16, 16).permute(0, 2, 1, 3).reshape(cam.Hp, cam.Wp)


def distortion_bound(fx):
    """[Hp, Wp] bound on |fp32 kernel - fp64| of the distortion map.  The kernel sums over m - m0 (m0: the pixel's
    first blended instance), so a difference m_i - m_j carries only the rounding of the two fp32 values m = dA - dB /
    z (< 1: half an ulp, 2^-25, each; the subtraction m - m0 is exact), 2^-24 in all.  Then
    |d sum_{j<i} w_i w_j (m_i - m_j)^2| <= sum w_i w_j 2 |m_i - m_j| 2^-24 <= 2^-24 spread A^2 with spread the range of
    m over the pixel's blended instances and A its alpha.  Allow 8 x that, plus 1e-4 relative for the fp32 weights
    and sums.  The same sums without the shift cancel terms of size m^2 A ~ 1 to leave the distortion: an error of
    order 2^-24, far above this bound where the spread is small."""
    cam = fx.cam
    out = torch.zeros(cam.nty * cam.ntx, 256, dtype=torch.float64)
    for t in range(cam.ntx * cam.nty):
        if int(fx.prof["count"][t]) == 0:
            continue
        alpha, _, tr, live, m = _dist_terms(fx, t)
        big, small = torch.where(live, m, torch.full_like(m, -math.inf)), torch.where(live, m, torch.full_like(m, math.inf))
        spread = (big.amax(1) - small.amin(1)).clamp(min=0).nan_to_num(0.0, posinf=0.0, neginf=0.0)
        w = alpha * tr[:, :-1] * live
        A = w.sum(1)
        mm = m[..., None] - m[:, None, :]
        ref = (w[..., None] * w[:, None, :] * mm * mm).triu(1).sum((1, 2))
        out[t] = 8 * U32 * spread * A * A + 1e-4 * ref
    return _untile(cam, out.reshape(cam.nty * cam.ntx, 256))


def distortion_fp32(fx, shifted=True):
    """[Hp, Wp] the forward distortion as blend_surfel_fwd_kernel sums it, in fp32 torch from the fp64 alphas and
    depths: running A, D, D2 over m - m0 (shifted) or over m itself (m0 = 0)."""
    cam = fx.cam
    f32 = torch.float32
    dA = torch.tensor(DIST_FAR / (DIST_FAR - DIST_NEAR), dtype=f32)
    dB = torch.tensor(DIST_FAR * DIST_NEAR / (DIST_FAR - DIST_NEAR), dtype=f32)
    out = torch.zeros(cam.nty * cam.ntx, 256, dtype=f32)
    for t in range(cam.ntx * cam.nty):
        k = int(fx.prof["count"][t])
        if k == 0:
            continue
        alpha, z = tile_eval(fx.fe, fx.cam, t)
        alpha, z = alpha.to(f32), z.to(f32)
        T = torch.ones(256, dtype=f32)
        A, D, D2, dist = (torch.zeros(256, dtype=f32) for _ in range(4))
        m0 = torch.full((256,), math.nan, dtype=f32)
        for j in range(k):
            a = alpha[:, j]
            on = (T > T_STOP) & (a > 0)
            mr = dA - dB / z[:, j]
            if shifted:
                m0 = torch.where(on & torch.isnan(m0), mr, m0)
                m = mr - m0
            else:
                m = mr
            w = a * T
            nd = dist + w * (m * (m * A - 2 * D) + D2)
            dist = torch.where(on, nd, dist)
            A = torch.where(on, A + w, A)
            D = torch.where(on, D + w * m, D)
            D2 = torch.where(on, D2 + w * m * m, D2)
            T = torch.where(on, T * (1 - a), T)
        out[t] = dist
    return _untile(cam, out).double()


# --------------------------------------------------------------------------------------------------------------
# oracle and comparator
# --------------------------------------------------------------------------------------------------------------
def oracle(fx, kind, final=True, seed=0, opa=None):
    """fp64 image, maps and parameter gradients of fixture fx for kind's upstream weights (fx.weights)."""
    cam = fx.cam
    p = {q: t.clone().requires_grad_(True) for q, t in fx.params(kind).items()}
    if opa is not None:
        p["opa"] = opa.double().clone().requires_grad_(True)
    act = "exp" if kind.startswith("exp") else "abs"
    img, mp, info = SO.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, background=BG,
                              scale_activation=act, dist_near=DIST_NEAR, dist_far=DIST_FAR)
    if final:
        img = cam.crop(img.clamp(0, 1))
        mp = {k: cam.crop(v[..., None] if v.dim() == 2 else v) for k, v in mp.items()}
        mp = {k: (v[..., 0] if k != "normal" else v) for k, v in mp.items()}
    w = fx.weights(kind, final, seed)
    loss = sum(((img if k == "image" else mp[k]) * wk).sum() for k, wk in w.items())
    grads = torch.autograd.grad(loss, [p[q] for q in NAMES], allow_unused=True)
    grads = {q: (torch.zeros_like(p[q]) if gr is None else gr.detach()) for q, gr in zip(NAMES, grads)}
    return dict(image=img.detach(), maps={k: v.detach() for k, v in mp.items()}, grads=grads, gi=info["gauss_idx"],
                accum=info["accum"].long())


IMG_ATOL = 1e-4
GRAD_RTOL = 1e-3


def compare(fx, got, ref, final=True, maps=True):
    """Failures (empty list: pass).  Image and each map <= 1e-4 absolute (depth and median relative to max(1, their
    largest value); the distortion of a fixture with a dist_bound: that per-pixel bound); every parameter gradient
    <= 1e-3 of its largest reference value (a parameter whose reference is exactly zero: the fp32 noise floor, 1e-6 of
    the frame's largest gradient); and each confined surfel's gradient <= 1e-3 of its own reference magnitude for that
    parameter (floor 1e-6 of the parameter's largest), so that one lost, duplicated, swapped or stale instance shows
    even when it is small."""
    fails = []
    e = float((got["image"].double().cpu() - ref["image"]).abs().max())
    if not e <= IMG_ATOL:
        fails.append(f"image: max|d| {e:.3e}")
    if maps:
        for k in SO_MAPS:
            d = (got["maps"][k].double().cpu() - ref["maps"][k]).abs()
            if k == "distortion" and fx.dist_bound is not None:
                b = fx.dist_bound
                b = fx.cam.crop(b[..., None])[..., 0] if final else b
                if not bool((d <= b).all()):
                    r = torch.where(d > 0, d / b, torch.zeros_like(d))
                    fails.append(f"distortion: max|d| / bound {float(r.max()):.3e}, max|d| {float(d.max()):.3e}")
                continue
            s = max(1.0, float(ref["maps"][k].abs().max())) if k in ("depth", "median") else 1.0
            if not float(d.max()) <= IMG_ATOL * s:
                fails.append(f"{k}: max|d| {float(d.max()):.3e}")
    top = max(float(r.abs().max()) for r in ref["grads"].values())
    conf = fx.tile_of >= 0
    for q in NAMES:
        g = got["grads"][q].double().cpu().reshape(fx.n, -1)
        r = ref["grads"][q].reshape(fx.n, -1)
        if not bool(torch.isfinite(g).all()):
            fails.append(f"{q}: non-finite")
            continue
        glob = float(r.abs().max())
        bound = GRAD_RTOL * glob if glob > 1e-12 * top else 1e-6 * top
        d = (g - r).abs().amax(1)
        if not float(d.max()) <= bound:
            fails.append(f"{q}: max|d| {float(d.max()):.3e} > {bound:.3e}")
        own = torch.maximum(GRAD_RTOL * r.abs().amax(1), torch.full((fx.n,), 1e-6 * max(glob, 1e-12 * top),
                                                                     dtype=torch.float64))
        bad = (conf & (d > own)).nonzero().flatten()
        for i in bad[:4].tolist():
            fails.append(f"{q}: surfel {i} (tile {int(fx.tile_of[i])}, {fx.role[i]}): |d| {float(d[i]):.3e} > "
                         f"{float(own[i]):.3e}")
    return fails
