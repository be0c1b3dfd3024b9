"""Seeded scenes whose per-tile instance lists sit on the blend kernels' edges, their fp64 oracle, and a comparator
that sees a single lost, duplicated, swapped or stale instance.

Test infrastructure only.  The oracle is gs_oracle's front end, binning and `draw` (plus tests/aux_oracle.py,
tests/feat_oracle.py and tests/densify_stats_oracle.py), run in fp64 on the scenes built here; the only blend
arithmetic of this module is `tile_transmittance`, which restates `draw`'s alpha to find where tiles saturate.  The scenes are made of world-space Gaussians, so the fused frame path renders them:

* confined Gaussians: small (sigma 1.3-2 px), anisotropic, centred near a tile's centre, so that their `tile_rects`
  footprint (~2.45 sigma at tile_thresh 0.05) stays inside that tile: each adds exactly one instance to one tile,
  and its per-Gaussian gradient is its per-instance gradient;
* walls: stacks of large (sigma 18 px), nearly opaque Gaussians that saturate whole tiles (or only their top rows)
  at a chosen index of the tile's depth order; they span several tiles.

Every Gaussian's distance |p_c| (the depth sort key) is set directly, at least 1e-3 apart except for one group of
exact duplicates (same position, so the same key; the tie is broken by id, as densify clones produce).  The
Gaussians are shuffled, so ids are not in depth order.
"""
from __future__ import annotations

import math

import torch

import gs_oracle as O
import synthetic as S

TILE = 16
T_STOP = 1e-4                     # a pixel stops before an instance once its transmittance is < 1e-4
NAMES = ("pos", "rgb", "opa", "quat", "scale")
BG = (0.2, 0.5, 0.9)

# Staged kernels: (chunk or round size, pipeline stages).  RGB forward fwd_ch 64 / 128 / 256 (2 stages) and the
# producer-warp forward (64, 4); RGB backward bwd_ch 32 / 64 and the packed WS_CH 64 (2 or 3 stages); round-1
# backward (64, 2); scalar SH (64, 2) forward, (32, 2) backward; tensor-core SH TC_J = 16 (4 stages forward, 3
# backward); features (64, 2) forward, (16, 2) backward.
STAGED = ((64, 2), (128, 2), (256, 2), (64, 4), (32, 2), (32, 3), (64, 3), (16, 4), (16, 3), (16, 2))
CHUNKS = sorted({ch for ch, _ in STAGED})


def target_counts():
    """Per-tile instance counts of the `counts` scene."""
    c = {0, 1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1100}
    for ch in CHUNKS:
        c |= {3 * ch - 1, 3 * ch + 1}
    for ch, st in STAGED:                  # STAGES - 1, STAGES and STAGES + 1 chunks, full and with one more
        for k in (st - 1, st, st + 1):
            c |= {k * ch, k * ch + 1}
    return sorted(c)


# Tile-saturation indices of the `walls` scene: last / first / second instance of a chunk or of a backward round
# (R = (256 / bwd_px) / bwd_rq = 4, 8 or 16 instances; 7, 8, 9 fall on no chunk edge), and exits inside
# chunk >= STAGES (copies of the next chunks still in flight): 50, 70 (TC_J 16), 100 (32 x 3), 200 (64 x 3),
# 300 (64 x 4, 128 x 2), 600 (256 x 2).
STOPS = (7, 8, 9, 31, 32, 33, 50, 63, 64, 65, 70, 100, 127, 128, 129, 200, 255, 256, 257, 300, 600)
IN_FLIGHT = {50: 120, 70: 120, 100: 200, 200: 260, 300: 300, 600: 300}    # tail after the walls (default 40)
# tails behind the single front wall of the `front` scene (every tile stops at instance 0)
FRONT_TAILS = (0, 1, 2, 15, 16, 17, 63, 64, 65, 129, 200, 600)


def _logit(p):
    p = torch.as_tensor(p, dtype=torch.float64)
    return torch.log(p) - torch.log1p(-p)


class _Scene:
    """Accumulates Gaussians given in pixel / depth terms and converts them to world-space parameters."""

    def __init__(self, width, height, seed):
        self.view = S.make_view(width, height, 0)          # rot = I, tran = (0, 0, 4)
        self.Wp, self.Hp = self.view.padded_width, self.view.padded_height
        self.fx = self.view.fx
        self.gen = torch.Generator().manual_seed(seed)
        self.rows = []                                     # (u, v, r, sigma_px, opa, tile or -1, role)

    def rand(self, lo, hi, n=None):
        t = torch.rand(() if n is None else (n,), generator=self.gen, dtype=torch.float64)
        return lo + (hi - lo) * t

    def add(self, u, v, r, sigma, opa, tile, role):
        self.rows.append((float(u), float(v), float(r), float(sigma), float(opa), int(tile), role))

    def confined(self, tile, r, opa, centre=None, sigma=None):
        ntx = self.Wp // TILE
        ty, tx = divmod(tile, ntx)
        cu, cv = centre if centre is not None else (8.0 + float(self.rand(-1, 1)), 8.0 + float(self.rand(-1, 1)))
        s = float(self.rand(1.3, 2.0)) if sigma is None else sigma
        self.add(tx * TILE + cu, ty * TILE + cv, r, s, opa, tile, "confined")

    def build(self):
        n = len(self.rows)
        u, v, r, sig, opa = (torch.tensor([row[k] for row in self.rows], dtype=torch.float64) for k in range(5))
        xn = (u - self.Wp / 2) / self.fx
        yn = (v - self.Hp / 2) / self.fx
        z = r / torch.sqrt(1 + xn * xn + yn * yn)
        pos = torch.stack([xn * z, yn * z, z - 4.0], dim=-1)
        aniso = torch.stack([torch.ones(n, dtype=torch.float64), self.rand(0.75, 1.0, n), self.rand(0.75, 1.0, n)], -1)
        quat = torch.randn(n, 4, generator=self.gen, dtype=torch.float64)
        rgb = self.rand(-1.5, 1.5, 3 * n).reshape(n, 3)
        cam = camera(self.view)
        shrink = torch.ones(n, dtype=torch.float64)
        for _ in range(50):      # keep every footprint edge >= 0.01 tile from a tile border: fp32 rounding cannot move it
            scale = (sig * shrink * z / self.fx).unsqueeze(-1) * aniso - O.EPS
            near = edge_distance(pos, quat, scale, cam) < 0.01
            if not bool(near.any()):
                break
            shrink = torch.where(near, shrink * 0.995, shrink)
        else:
            raise AssertionError("tile_edges: footprint edges stay on tile borders")
        g = dict(pos=pos, rgb=rgb, opa=_logit(opa), quat=quat, scale=scale)
        perm = torch.randperm(n, generator=self.gen)       # ids are not in depth order
        g = {q: t[perm].float().contiguous() for q, t in g.items()}
        tile_of = torch.tensor([row[5] for row in self.rows], dtype=torch.int64)[perm]
        role = [self.rows[i][6] for i in perm.tolist()]
        return g, tile_of, role


def camera(view):
    return O.Camera(view.width, view.height, view.fx, view.fy, view.rot, view.tran, view.near)


def edge_distance(pos, quat, scale, cam, thresh=0.05):
    """[n] distance (in tiles) of the nearest of each Gaussian's four footprint edges (tile_rects' continuous bounds,
    fp64) to an integer: a small one lets fp32 rounding add or drop a tile."""
    nq = quat / quat.norm(dim=1, keepdim=True)               # the footprint depends on shape only, as in preactivate
    ns = scale.abs() + O.EPS
    rp, rc, _ = O.global_culling(pos, nq, ns, cam.rot.double(), cam.tran.double(), cam.near, cam.half_w, cam.half_h)
    t = -2.0 * math.log(thresh)
    a, d = rc[:, 0, 0], rc[:, 1, 1]
    sx, sy = torch.sqrt(a.clamp(min=0) * t), torch.sqrt(d.clamp(min=0) * t)
    edges = torch.stack([(rp[:, 0] - sx - cam.leftmost) / cam.tile_lx, (rp[:, 0] + sx - cam.leftmost) / cam.tile_lx,
                         (rp[:, 1] - sy - cam.topmost) / cam.tile_ly, (rp[:, 1] + sy - cam.topmost) / cam.tile_ly], -1)
    return (edges - edges.round()).abs().amin(1)


def front_end(g, cam, depth_key=None, rgb=None, use_sh=False):
    """gs_oracle's activation, culling, binning and (tile, depth, id) sort of the (fp64 or fp32) parameters g:
    dict(p, c, rgb, opa, gi [M] Gaussian ids in blend order, accum [T+1], rects, idx visible ids)."""
    dt = g["pos"].dtype
    nq, ns, opa_a, rgb_a = O.preactivate(g["quat"], g["scale"], g["opa"], g["rgb"] if rgb is None else rgb, "abs",
                                         use_sh)
    rp, rc, mask = O.global_culling(g["pos"], nq, ns, cam.rot.to(dt), cam.tran.to(dt), cam.near, cam.half_w,
                                    cam.half_h)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    p_c, c_c = rp[idx], rc[idx]
    rects = O.tile_rects(p_c[:, :2], c_c, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                         cam.topmost)
    gi, accum = O.bin_and_sort(p_c, c_c, rects, cam.ntx, cam.nty, None if depth_key is None else depth_key[idx])
    return dict(p=p_c[gi], c=c_c[gi], rgb=rgb_a[idx][gi], opa=opa_a[idx][gi], gi=idx[gi], accum=accum.long(),
                rects=rects, idx=idx, n_vis=int(idx.numel()))


def tile_transmittance(fe, cam, t):
    """[256, k + 1] transmittance in front of each of tile t's k instances and after the last one (fp64, `draw`'s
    alpha), or None for an empty tile.  Pixel p = row * 16 + column."""
    s, e = int(fe["accum"][t]), int(fe["accum"][t + 1])
    if e <= s:
        return None
    ty, tx = divmod(t, cam.ntx)
    ix = torch.arange(16, dtype=torch.float64)
    px = (tx * 16 + ix + 0.5 - cam.Wp // 2) / cam.fx
    py = (ty * 16 + ix + 0.5 - cam.Hp // 2) / cam.fy
    PX = px.reshape(1, 16).expand(16, 16).reshape(-1, 1)
    PY = py.reshape(16, 1).expand(16, 16).reshape(-1, 1)
    p = fe["p"][s:e].detach().double()
    a, b, c, d = fe["c"][s:e].detach().double().reshape(-1, 4).unbind(-1)
    X, Y = PX - p[:, 0], PY - p[:, 1]
    power = -(d * X * X - (b + c) * X * Y + a * Y * Y) / (2 * (a * d - b * c) + 1e-14)
    alpha = torch.exp(power) * fe["opa"][s:e].detach().double()
    return torch.cat([torch.ones(256, 1, dtype=torch.float64), torch.cumprod(1 - alpha, dim=1)], dim=1)


def tile_profile(fe, cam):
    """Per tile: count; last live instance (-1 if empty; instance j is live for a pixel while T_j >= 1e-4); whether
    every pixel ends saturated; whether rows 0-7 end saturated and rows 8-15 do not; and margin, the smallest
    |ln(T / 1e-4)| of any of its (pixel, instance) pairs (inf if empty): how far the tile stays from the early-stop
    threshold.  fp32 evaluates a product of ~1e3 factors to ~6e-5 relative, so a margin >= 1e-4 means fp32 and fp64
    make every early-stop decision of the tile alike."""
    nt = cam.ntx * cam.nty
    count = (fe["accum"][1:] - fe["accum"][:-1]).long()
    last = torch.full((nt,), -1, dtype=torch.int64)
    full = torch.zeros(nt, dtype=torch.bool)
    split = torch.zeros(nt, dtype=torch.bool)
    margin = torch.full((nt,), math.inf, dtype=torch.float64)
    for t in range(nt):
        tr = tile_transmittance(fe, cam, t)
        if tr is None:
            continue
        last[t] = int((tr[:, :-1] >= T_STOP).any(0).nonzero().max())
        dead = tr[:, -1] < T_STOP
        full[t] = bool(dead.all())
        split[t] = bool(dead[:128].all()) and not bool(dead[128:].all())
        margin[t] = float((tr / T_STOP).log().abs().min())
    return dict(count=count, last=last, full=full, split=split, margin=margin)


class Fixture:
    """A scene plus what it was built to hit.  g: fp32 CPU parameters; tile_of[n]: the tile of a confined Gaussian,
    -1 for a wall; targets: {tile: intended last live instance}; profile: tile_profile of the fp64 front end."""

    def __init__(self, name, sc, g, tile_of, role, targets, partial=()):
        self.name = name
        self.view = sc.view
        self.cam = camera(sc.view)
        self.g = g
        self.n = g["pos"].shape[0]
        self.tile_of = tile_of
        self.role = role
        self.targets = dict(targets)
        self.partial = tuple(partial)
        self.wall_rtol = {}                       # per-parameter tolerance of the walls' whole-tensor check
        self.tile_scale = False                   # walls checked against oracle(tile_scale=True)'s summed magnitude
        gen = torch.Generator().manual_seed(len(name) * 7919 + self.n)
        h, w = self.view.height, self.view.width
        self.up = torch.rand(h, w, 3, generator=gen, dtype=torch.float64) + 0.5          # U(0.5, 1.5)
        self.up_depth = (torch.rand(h, w, generator=gen, dtype=torch.float64) + 0.5) * 0.1
        self.up_alpha = torch.rand(h, w, generator=gen, dtype=torch.float64) + 0.5
        self.up_feat = {F: torch.rand(h, w, F, generator=gen, dtype=torch.float64) + 0.5 for F in (8, 16, 32)}
        self.feat = {F: torch.rand(self.n, F, generator=gen) + 0.5 for F in (8, 16, 32)}
        self.sh = {}
        for d in (27, 48):
            k = d // 3
            hi = torch.randn(self.n, 3, k - 1, generator=gen) * 0.1
            self.sh[d] = torch.cat([(g["rgb"] / S.SH_C0).unsqueeze(-1), hi], dim=-1).reshape(self.n, d).contiguous()
        gd = {q: t.double() for q, t in g.items()}
        self.fe = front_end(gd, self.cam)
        self.profile = tile_profile(self.fe, self.cam)

    def params(self, dtype=torch.float64, rgb=None):
        p = {q: t.to(dtype).clone() for q, t in self.g.items()}
        if rgb is not None:
            p["rgb"] = rgb.to(dtype).clone()
        return {q: t.requires_grad_(True) for q, t in p.items()}


def _confined_opacity(sc, count):
    if count <= 5:                                # the ordering regime: alpha 0.2-0.45, adjacent swaps show
        return sc.rand(0.2, 0.45, max(count, 1))
    base = min(0.45, 2.0 / count)                 # optical depth ~2 at the centre: the tile never saturates
    return base * sc.rand(0.8, 1.2, count)


def build_counts(seed=0):
    """Tiles holding exactly target_counts() confined instances; size 3 and 5 px short of a multiple of 16, so the
    border tiles are cropped.  One tile of 33 holds a group of 4 exact duplicates (same depth key)."""
    counts = target_counts()
    ntx = 8
    nty = (len(counts) + ntx - 1) // ntx
    sc = _Scene(ntx * TILE - 3, nty * TILE - 5, seed)
    order = torch.randperm(ntx * nty, generator=sc.gen).tolist()
    targets = {}
    for t, c in zip(order, counts):
        opa = _confined_opacity(sc, c)
        depths = 2.0 + 3.0 * (torch.randperm(c, generator=sc.gen).double() + sc.rand(0.3, 0.7, c)) / max(c, 1)
        for j in range(c):
            sc.confined(t, float(depths[j]), float(opa[j]))
        if c == 33:                               # a clone group: same centre and depth, other shape and colour
            u, v, r = sc.rows[-1][0], sc.rows[-1][1], sc.rows[-1][2]
            for j in range(1, 4):
                sc.rows[-1 - j] = (u, v, r, float(sc.rand(1.3, 2.0)), sc.rows[-1 - j][4], t, "clone")
            sc.rows[-1] = sc.rows[-1][:6] + ("clone",)
        targets[t] = c - 1
    g, tile_of, role = sc.build()
    return Fixture("counts", sc, g, tile_of, role, targets)


def _wall_stack(sc, u, v, k, site):
    # distinct depth keys across sites too: two sites' walls meet in the tiles between them
    for j in range(k):
        sc.add(u, v, 4.0 + 0.1 * j + 0.003 * site, 18.0, 0.9975, -1, "wall")


def build_walls(seed=1):
    """One site per STOPS entry (a stack of 8 walls over its tile, confined instances in front of and behind it,
    the front count tuned so that the tile saturates exactly at the target index) and two partial sites (walls
    centred 2 px above the tile: its top rows saturate, the bottom ones never do).  Sites are 6 tiles apart, so
    their walls (footprint ~44 px) never reach another site's tile."""
    sites = list(STOPS) + ["partial", "partial"]
    cols = 6
    rows = (len(sites) + cols - 1) // cols
    ntx, nty = 6 * cols, 6 * rows
    fronts = {i: max(0, s - 5) for i, s in enumerate(sites) if s != "partial"}
    for _ in range(6):
        sc = _Scene(ntx * TILE, nty * TILE - 8, seed)
        targets, partial, site_tile = {}, [], {}
        for i, s in enumerate(sites):
            cy, cx = divmod(i, cols)
            tx, ty = 6 * cx + 3, 6 * cy + 3
            t = ty * ntx + tx
            if s == "partial":
                _wall_stack(sc, tx * TILE + 8.0, ty * TILE - 2.0, 7, i)
                for j, o in enumerate(sc.rand(0.02, 0.05, 20).tolist()):
                    sc.confined(t, 2.0 + 0.07 * j, o)
                for j, o in enumerate(sc.rand(0.05, 0.2, 20).tolist()):
                    sc.confined(t, 5.0 + 0.04 * j, o, centre=(8.0 + float(sc.rand(-3, 3)), 13.0), sigma=0.8)
                partial.append(t)
                continue
            nf = fronts[i]
            base = min(0.3, 1.0 / max(nf, 1))
            for j, o in enumerate((base * sc.rand(0.8, 1.2, nf)).tolist()):
                sc.confined(t, 2.0 + 2.0 * j / max(nf, 1), o)
            _wall_stack(sc, tx * TILE + 8.0, ty * TILE + 8.0, 8, i)
            nb = IN_FLIGHT.get(s, 40)
            for j, o in enumerate(sc.rand(0.05, 0.3, nb).tolist()):
                sc.confined(t, 5.0 + 1.0 * j / nb, o)
            targets[t] = s
            site_tile[i] = t
        g, tile_of, role = sc.build()
        fx = Fixture("walls", sc, g, tile_of, role, targets, partial)
        off = {i: targets[t] - int(fx.profile["last"][t]) for i, t in site_tile.items()}
        if all(v == 0 for v in off.values()):
            return fx
        for i, d in off.items():               # the walls' own saturation offset barely moves with the front count
            fronts[i] = max(0, fronts[i] + d)
    raise AssertionError("walls: could not place the saturation indices")


def build_front(seed=2):
    """One huge, nearly opaque Gaussian in front of everything: every tile saturates at instance 0, with
    FRONT_TAILS confined instances behind it (copies of later chunks are in flight when the tile exits)."""
    ntx, nty = 4, 3
    sc = _Scene(ntx * TILE, nty * TILE, seed)
    sc.add(ntx * 8.0, nty * 8.0, 1.5, 6000.0, 1 - 6e-5, -1, "wall")
    targets = {}
    for t, c in zip(range(ntx * nty), FRONT_TAILS):
        for j, o in enumerate(sc.rand(0.05, 0.3, c).tolist()):
            sc.confined(t, 2.0 + 3.0 * j / max(c, 1), o)
        targets[t] = 0
    g, tile_of, role = sc.build()
    fx = Fixture("front", sc, g, tile_of, role, targets)
    # Stopping at instance 0 needs 1 - alpha < 1e-4 on every pixel (~8e-5 here).  Two things make the wall's own
    # gradients ill-conditioned, and the wall's whole-tensor check allows for both (its confined instances keep 1e-3):
    # * it is centred on the image, so the tiles' contributions to its mean gradient cancel: their sum is 1/130 to
    #   1/20000 of their summed magnitude (measured on the H100, fp32 kernels: RGB 2e-3 and features F = 32 6.5e-2 of
    #   the pos gradient, 2e-5 and 6e-5 of the summed magnitude), so the wall's error is measured against the sum
    #   over tiles of |each tile's contribution| (oracle's tile_scale);
    # * with the background / depth / alpha outputs, a front-to-back backward recovers the T_f bg term from
    #   1 - alpha = 8e-5 in fp32, ~1e-3 relative: H100 errors up to 2.45e-3 in opa, 2.8e-3 in quat, 2.9e-3 in scale
    #   and absgrad, 2e-3 in grad2d (only the kernels with those outputs), hence 5e-3 for those.
    fx.tile_scale = True
    fx.wall_rtol = {"opa": 5e-3, "quat": 5e-3, "scale": 5e-3, "stats": 5e-3}
    return fx


BUILDERS = {"counts": build_counts, "walls": build_walls, "front": build_front}


# --------------------------------------------------------------------------------------------------------------
# oracle
# --------------------------------------------------------------------------------------------------------------
def _crop2(cam, x):
    return cam.crop(x.unsqueeze(-1)).squeeze(-1)


def oracle(fx, kind="rgb", dtype=torch.float64, depth_key=None, mutate=None, tiles=None, opa=None,
           tile_scale=False):
    """Image and parameter gradients of one frame of fixture fx for its positive upstream gradients.

    kind: "rgb" (image), "aux" (image over BG, depth and alpha), "sh27" / "sh48" (per-pixel SH colour), "sh27-aux" /
    "sh48-aux", "feat8" / "feat16" / "feat32" (image and features).  mutate(gi, accum) -> (gi, accum) edits the
    sorted instance list before blending (fault injection); tiles: blend only those tiles (the loss is a sum over
    tiles, so per-tile pieces add up).  opa: replacement opacity logits.  Returns dict(image, depth, alpha,
    features (final, cropped), grads {name: tensor}, fe and, with tile_scale, tile_scale {name: sum over tiles of
    |that tile's contribution to the gradient|})."""
    cam = fx.cam
    aux = kind.endswith("aux")
    sh = kind.startswith("sh")
    feat = kind.startswith("feat")
    d = int(kind[2:4]) if sh else 3
    p = fx.params(dtype, rgb=fx.sh[d] if sh else None)
    if opa is not None:
        p["opa"] = opa.to(dtype).clone().requires_grad_(True)
    pf = fx.feat[int(kind[4:])].to(dtype).clone().requires_grad_(True) if feat else None
    fe = front_end(p, cam, depth_key, use_sh=sh)
    gi, accum = fe["gi"], fe["accum"]                   # gi: Gaussian ids in blend order
    if mutate is not None:
        gi, accum = mutate(gi.clone(), accum.clone())
    nq, ns, opa_a, rgb_a = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"], "abs", sh)
    rp, rc, _ = O.global_culling(p["pos"], nq, ns, cam.rot.to(dtype), cam.tran.to(dtype), cam.near, cam.half_w,
                                 cam.half_h)
    pos_i, cov_i, opa_i, rgb_i = rp[gi], rc[gi], opa_a[gi], rgb_a[gi]
    rays = O.ray_info(cam.rot.to(dtype), cam.tran.to(dtype), cam.Hp, cam.Wp, cam.fx, cam.fy) if sh else (None,) * 4
    out = dict(fe=fe)
    loss = 0
    if aux:
        import aux_oracle as A
        assert tiles is None, "aux_oracle.draw_maps blends every tile"
        img, dep, alp = A.draw_maps(pos_i, rgb_i, opa_i, cov_i, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, BG, sh, rays)
        dep, alp = _crop2(cam, dep), _crop2(cam, alp)
        out.update(depth=dep.detach(), alpha=alp.detach())
        loss = loss + dep * fx.up_depth.to(dtype) + alp * fx.up_alpha.to(dtype)
    else:
        img = O.draw(pos_i, rgb_i, opa_i, cov_i, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, sh, *rays, tiles=tiles)
    if feat:
        import feat_oracle as FT
        F = pf.shape[1]
        fmc = cam.crop(FT.draw_features(pos_i, pf[gi], opa_i, cov_i, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, tiles))
        out["features"] = fmc.detach()
        loss = loss + (fmc * fx.up_feat[F].to(dtype)).sum(-1)
    final = cam.crop(torch.clamp(img, 0, 1))
    loss = loss + (final * fx.up.to(dtype)).sum(-1)
    leaves = [p[q] for q in NAMES] + ([pf] if feat else [])
    grads = torch.autograd.grad(loss.sum(), leaves, allow_unused=True, retain_graph=tile_scale)
    out["image"] = final.detach()
    out["grads"] = {q: (torch.zeros_like(x) if gr is None else gr).detach()
                    for q, x, gr in zip(NAMES + ("feat",), leaves, grads)}
    if tile_scale:
        # sum over tiles of |each tile's contribution| to every parameter gradient (the loss is a sum over tiles)
        top, left = (cam.Hp - cam.height) // 2, (cam.Wp - cam.width) // 2
        lmap = torch.nn.functional.pad(loss, (left, cam.Wp - cam.width - left, top, cam.Hp - cam.height - top))
        acc = {q: torch.zeros_like(g) for q, g in out["grads"].items()}
        for t in range(cam.ntx * cam.nty):
            ty, tx = divmod(t, cam.ntx)
            part = lmap[ty * TILE:(ty + 1) * TILE, tx * TILE:(tx + 1) * TILE].sum()
            if part.requires_grad:
                gt = torch.autograd.grad(part, leaves, allow_unused=True, retain_graph=True)
                for q, gr in zip(NAMES + ("feat",), gt):
                    if gr is not None:
                        acc[q] += gr.detach().abs()
        out["tile_scale"] = acc
    return out


def stats_oracle(fx, aux=False, depth_key=None):
    """densify_stats_oracle.frame_stats of one frame (absgrad on) for the same loss as oracle(fx, "rgb" / "aux")."""
    import densify_stats_oracle as DS
    cam = fx.cam
    p = {q: t.double() for q, t in fx.g.items()}

    def loss(out):
        lv = (cam.crop(torch.clamp(out["padded"], 0, 1)) * fx.up).sum()
        if aux:
            lv = lv + (_crop2(cam, out["depth"]) * fx.up_depth).sum() + (_crop2(cam, out["alpha"]) * fx.up_alpha).sum()
        return lv
    if aux:       # the image over BG: (image + (1 - alpha) bg) = image - alpha bg + bg
        def loss_aux(out):
            img = out["padded"] + (1 - out["alpha"]).unsqueeze(-1) * torch.tensor(BG, dtype=torch.float64)
            return loss(dict(out, padded=img))
        return DS.frame_stats(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, loss_aux, maps=True,
                              absgrad=True, depth_key=depth_key)
    return DS.frame_stats(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, loss, absgrad=True,
                          depth_key=depth_key)


# --------------------------------------------------------------------------------------------------------------
# comparator
# --------------------------------------------------------------------------------------------------------------
GRAD_RTOL = 1e-3
IMG_ATOL = 1e-4


def compare(fx, got, ref, image=None, ref_image=None, rtol=GRAD_RTOL, atol=IMG_ATOL, extra=(), scale=None):
    """Failures (empty list: pass) of per-tile, per-instance parity.

    For every tile and parameter, max |got - ref| over the tile's confined Gaussians (one instance each) must be
    <= rtol * max |ref| over the same Gaussians; a tile whose Gaussians all have a zero reference (the unread tail
    of a saturated tile) is held to rtol * the largest |ref| of that parameter in the frame, so a stale row shows.
    Walls keep the whole-tensor check over the walls, relative to max |ref| or, given `scale` (oracle's tile_scale),
    to the largest summed magnitude of the tiles' contributions; the image (and `extra` (name, got, ref) maps) 1e-4
    absolute per pixel."""
    fails = []
    conf = fx.tile_of >= 0
    tiles = fx.tile_of[conf]
    nt = fx.cam.ntx * fx.cam.nty
    for q, r in ref.items():
        if q not in got:
            continue
        g = got[q].detach().double().cpu().reshape(fx.n if q != "feat" else r.shape[0], -1)
        r = r.detach().double().cpu().reshape(g.shape)
        if not bool(torch.isfinite(g).all()):
            fails.append(f"{q}: non-finite gradient")
            continue
        dlt = (g - r).abs().amax(1)
        mag = r.abs().amax(1)
        glob = float(mag.max())
        err_t = torch.zeros(nt, dtype=torch.float64).scatter_reduce(0, tiles, dlt[conf], "amax")
        ref_t = torch.zeros(nt, dtype=torch.float64).scatter_reduce(0, tiles, mag[conf], "amax")
        scale_t = torch.where(ref_t > 0, ref_t, torch.full_like(ref_t, glob))
        bad = (err_t > rtol * scale_t).nonzero().flatten().tolist()
        for t in bad[:4]:
            fails.append(f"{q}: tile {t}: max|d| {float(err_t[t]):.3e} > {rtol:g} x {float(scale_t[t]):.3e}")
        if bool((~conf).any()):
            e, s = float(dlt[~conf].max()), float(mag[~conf].max())
            if scale is not None and q in scale:
                s = float(scale[q].double().reshape(g.shape)[~conf].max())
            wr = fx.wall_rtol.get(q, rtol)
            if e > wr * s:
                fails.append(f"{q}: walls: max|d| {e:.3e} > {wr:g} x {s:.3e}")
    pairs = ([("image", image, ref_image)] if image is not None else []) + list(extra)
    for name, a, b in pairs:
        e = float((a.detach().double().cpu() - b.detach().double().cpu()).abs().max())
        if not e <= atol:
            fails.append(f"{name}: max|d| {e:.3e} > {atol:g}")
    return fails


# --------------------------------------------------------------------------------------------------------------
# RGB backward variants: the `case` keys of the three switch tables of gs_launch_blend_bwd (blend.cu), in order.
# key = bwd_px | bwd_ws | bwd_unroll | bwd_stages | bwd_rq | bwd_minb (2 digits)
# --------------------------------------------------------------------------------------------------------------
BWD_GATHER_32 = (8022416, 8023416, 8042410, 8043410)
BWD_GATHER_64 = (8012410, 8022416, 8022410, 8042410, 8023416, 8012416, 8012420, 8012820, 8013416, 4012401, 4042401)
BWD_PACKED = (4113401, 4143408, 4012401, 4042401, 4042810, 8012410, 8012416, 8012420, 8013416, 8022416, 8022410,
              8042410, 8012816, 8012820, 8112410, 8012424, 8012824)
BWD_KNOBS = ("bwd_px", "bwd_ws", "bwd_unroll", "bwd_stages", "bwd_rq", "bwd_minb")


def encode_bwd_key(k):
    return ((((k["bwd_px"] * 10 + k["bwd_ws"]) * 10 + k["bwd_unroll"]) * 10 + k["bwd_stages"]) * 10 +
            k["bwd_rq"]) * 100 + k["bwd_minb"]


def decode_bwd_key(key):
    minb, rest = key % 100, key // 100
    rq, rest = rest % 10, rest // 10
    stages, rest = rest % 10, rest // 10
    unroll, rest = rest % 10, rest // 10
    ws, px = rest % 10, rest // 10
    return dict(bwd_px=px, bwd_ws=ws, bwd_unroll=unroll, bwd_stages=stages, bwd_rq=rq, bwd_minb=minb)
