"""The fused projection's kernel instantiations, scenes that put each one on its edges, the fp64 oracle composed for
them, and a per-Gaussian comparator that sees one lost, duplicated or stale gradient row.

Test infrastructure only.  The projection backward is one template per family (project.cu): single-view and batched,
instantiated over the colour model (KG, D, GW), the feature tier (none < 2-D filter < 3-D filter < lens, cumulative),
the depth gradient DT and the camera gradient CG; the densification statistics (densify_stats.cu) over the tier and
absgrad.  `table()` lists every instantiation the public entry points reach without a gradient push, with the call and
context setters that reach it; `dispatch_literals()` reads the same mappings out of the two sources, so that a colour
family or tier added to a dispatch fails tests/test_project_edges_oracle.py until the table covers it.

Scenes (world-space Gaussians given in pixel and depth terms through bin_edges.Builder, on bin_edges.View cameras
with the host's narrowed constants):

* `frame` (one view, n = 545: the last CTA of 256 holds 33 Gaussians, the last warp one):
  - runs: Gaussians whose tile rectangle has exactly 1, 2, 3, 4, 5, 7, 8, 9, 12 and 13 tiles (the RGB backward
    sums rows in groups of four);
  - wall sites on row 10: stacks of WALL_K = 24 walls (sigma 8 px, opacity 0.86 .. 0.93, drawn again for a stack
    whose tiles miss the early-stop margin) saturate chosen tiles in front of runs of 5, 5, 9 and 2 tiles, whose live
    rows are then {0, 2, 4}, {3}, {1, 2, 3} and {}: live and stale rows mix inside a group of four, and the last
    Gaussian is binned but hidden everywhere (its gradient is exactly zero);
  - visible Gaussians whose footprint lies outside the padded grid (unbinned: exactly zero), and one behind the
    camera;
  - activation edges: raw scale components of exactly 0 (every run, under `abs`), raw scales of +-0.5 and
    +-1.5 (both activations), quaternion norms of 0.25 and 4, opacity logits of +-5.9;
  - fillers with random rotations up to n.
* `batch` (three views with other poses, focal lengths and lenses, n = 545): Gaussians 256..511 (the second CTA)
  lie where only view 0 sees them, so that in views 1 and 2 that CTA has no row while CTAs 0 and 2 do.  Its first B = 1, 2 or 3 views make the batches.

The 3-D filter is 0 for runs and walls (their rectangles keep their design at every tier) and for a third of the
others; the rest get a filter between 0.5 and 1.5 times their smallest activated scale.

Margins.  fp32 and fp64 must bin, cull and stop alike.  Every Gaussian's culling decision and tile rectangle is
unchanged under a relative perturbation STABLE_EPS = 5e-5 of its projected mean and covariance (and of rho against a
lens's fold-back radius), in every configuration: this is test_lens_gpu.py's stability test, and 1e-5 is more than
ten times bin_edges' derived edge bound (<= ~100 u, u = 2^-24, for the lens projections).  Every tile keeps its
early-stop decisions away from the threshold: tile_edges.tile_profile's margin (smallest |ln(T / 1e-4)| over its
(pixel, instance) pairs) is >= 1e-4 in every configuration, and fp32 evaluates those products to ~6e-5.

Tolerances (`compare`): each parameter of each Gaussian within GRAD_RTOL = 1e-3 of that Gaussian's own largest
|reference| component for that parameter (with a floor of 1e-6 of the frame-wide largest), exact zeros where the
oracle's row is exactly zero, the image 1e-4 absolute, each view's camera gradient 1e-3 relative, and the statistics:
count exact, max_radius exact except where the oracle's radius lies within 1e-4 of an integer, grad2d and absgrad
1e-3 per Gaussian.
"""
from __future__ import annotations

import contextlib
import math
import os
import re

import torch

import bin_edges as B
import densify_stats_oracle as DS
import filter3d_oracle as F3
import filter_oracle as FO
import gs_oracle as O
import lens_oracle as LO
import sh_gaussian_oracle as G
import tile_edges as E

NAMES = E.NAMES
TILE = 16
N = 545                                  # n = 17 * 32 + 1: last CTA 33 Gaussians, last warp one
TIERS = ("none", "filt2d", "filt3d", "lens")
TIER_CODE = {"none": "GS_TIER_NONE", "filt2d": "GS_TIER_FILT2D", "filt3d": "GS_TIER_FILT3D", "lens": "GS_TIER_LENS"}
# colour: (KG, D, GW), sh_eval
COLOURS = {"rgb": ((0, 3, "GS_GREC"), "pixel"), "sh27-pixel": ((0, 27, "36"), "pixel"),
           "sh48-pixel": ((0, 48, "56"), "pixel"), "sh27-gauss": ((9, 27, "GS_GREC"), "gaussian"),
           "sh48-gauss": ((16, 48, "GS_GREC"), "gaussian")}
BATCH_COLOURS = ("rgb", "sh27-gauss", "sh48-gauss")
FILTER2D_VAR = 0.3
STABLE_EPS = 5e-5
SAT_MARGIN = 1e-4
GRAD_RTOL = 1e-3
GRAD_FLOOR = 1e-6
IMG_ATOL = 1e-4
CAM_RTOL = 1e-3
STAT_RTOL = 1e-3
LENSES = {
    "pinhole-offset": dict(model="PINHOLE", dcx=5.5, dcy=-3.25, k=[0.0] * 4),
    "opencv": dict(model="OPENCV", dcx=2.0, dcy=1.5, k=[-0.05, 0.01, 0.002, -0.001]),
    "fisheye": dict(model="FISHEYE", dcx=-1.5, dcy=2.5, k=[0.03, -0.01, 0.002, -0.0003]),
}
LENS_ORDER = ("pinhole-offset", "opencv", "fisheye")


def lens_of(name, view):
    d = LENSES[name]
    return dict(model=d["model"], cx=view.width / 2 + d["dcx"], cy=view.height / 2 + d["dcy"], k=list(d["k"]))


# ----------------------------------------------------------------------------------------------------------------------
# the instantiation table
# ----------------------------------------------------------------------------------------------------------------------
def _single_call(dt, cg):
    return "render_frame_cam" if cg else ("render_frame_aux" if dt else "render_frame_final")


def table():
    """Every instantiation the fused projection's four launchers and the statistics kernels reach without a gradient
    push, as dicts: kernel ("bwd", "bwd_batch", "fwd", "fwd_batch", "stats", "stats_batch"), colour, KG / D / GW,
    tier, dt, cg, absgrad, and `call` / `setters`, the public call and context settings that reach it."""
    rows = []
    for col, ((kg, d, gw), sh_eval) in COLOURS.items():
        for tier in TIERS:
            for dt in (False, True):
                for cg in ((False, True) if (kg or d == 3) else (False,)):
                    rows.append(dict(kernel="bwd", colour=col, kg=kg, d=d, gw=gw, tier=tier, dt=dt, cg=cg,
                                     call=_single_call(dt, cg), setters=_setters(col, tier)))
    for col in BATCH_COLOURS:
        (kg, d, gw), _ = COLOURS[col]
        for tier in TIERS:
            for dt in (False, True):
                for cg in (False, True):
                    rows.append(dict(kernel="bwd_batch", colour=col, kg=kg, d=d, gw=gw, tier=tier, dt=dt, cg=cg,
                                     call="render_frame_batch_cam" if cg else "render_frame_batch",
                                     setters=_setters(col, tier)))
    for kernel, cols, call in (("fwd", ("rgb", "sh27-gauss", "sh48-gauss"), "render_frame_final"),
                               ("fwd_batch", BATCH_COLOURS, "render_frame_batch")):
        for col in cols:
            for tier in TIERS:
                rows.append(dict(kernel=kernel, colour=col, kg=COLOURS[col][0][0], tier=tier, call=call,
                                 setters=_setters(col, tier)))
    for kernel, call in (("stats", "render_frame_final"), ("stats_batch", "render_frame_batch")):
        for tier in TIERS[1:]:
            for absgrad in (False, True):
                rows.append(dict(kernel=kernel, colour="rgb", tier=tier, absgrad=absgrad, call=call,
                                 setters=dict(_setters("rgb", tier), densify_stats="absgrad" if absgrad else "grad")))
    return rows


def _setters(colour, tier):
    return dict(sh_eval=COLOURS[colour][1], filter2d="antialias" if tier != "none" else "none",
                filter3d=tier in ("filt3d", "lens"), lens=tier == "lens")


def row_id(r):
    parts = [r["kernel"], r["colour"], r["tier"]]
    if "dt" in r:
        parts += ["dt" if r["dt"] else "nodt", "cg" if r["cg"] else "nocg"]
    if "absgrad" in r:
        parts.append("absgrad" if r["absgrad"] else "grad")
    return "-".join(parts)


def dispatch_literals(root):
    """The literal mappings of the two dispatches: ({(KG, D, GW) of fused_project_dispatch's by_tier calls},
    [tier names of its by_tier switch], [tier names of densify_stats_dispatch's switch])."""
    csrc = os.path.join(root, "3d-gaussian-splatting_b200", "csrc")
    with open(os.path.join(csrc, "project.cu")) as f:
        src = f.read()
    body = src[src.index("cudaError_t fused_project_dispatch("):]
    body = body[:body.index("\n}\n")]
    triples = {(int(a), int(b), c) for a, b, c in
               re.findall(r"by_tier\(Int<(\d+)>\{\}, Int<(\d+)>\{\}, Int<(\w+)>\{\}\)", body)}
    by_tier = body[body.index("auto by_tier"):]
    by_tier = by_tier[:by_tier.index("};")]
    tiers = re.findall(r"Int<(GS_TIER_\w+)>", by_tier)
    with open(os.path.join(csrc, "densify_stats.cu")) as f:
        ds = f.read()
    ds = ds[ds.index("cudaError_t densify_stats_dispatch("):]
    ds = ds[:ds.index("\n}\n")]
    stats_tiers = re.findall(r"integral_constant<int, (GS_TIER_\w+)>", ds)
    return triples, tiers, stats_tiers


# ----------------------------------------------------------------------------------------------------------------------
# scenes
# ----------------------------------------------------------------------------------------------------------------------
RUN_SHAPES = {1: (1, 1), 2: (2, 1), 3: (3, 1), 4: (2, 2), 5: (5, 1), 7: (7, 1), 8: (4, 2), 9: (3, 3), 12: (4, 3),
              13: (13, 1)}
# (name, count, first tile column, wall tiles (run-relative), live rows) on row SITE_ROW.  H lies behind B's walls.
WALL_SITES = (("A", 5, 0, (1, 3), (0, 2, 4)), ("B", 5, 6, (0, 1, 2, 4), (3,)), ("C", 9, 12, (0, 4, 5, 6, 7, 8),
              (1, 2, 3)), ("H", 2, 7, (), ()))
WALL_K, WALL_SIGMA = 24, 8.0
SITE_ROW = 10


class Scene:
    """Gaussians g (float32 CPU), views (bin_edges.View), the scale activation, per-Gaussian roles, the 3-D filter
    f3d [n], SH coefficient tensors sh[27 / 48], the designed runs {name: (id, rect, live rows)} and upstream
    gradients per view."""

    def __init__(self, name, views, g, act, roles, f3d, runs, lenses):
        self.name, self.views, self.g, self.act, self.roles = name, list(views), g, act, roles
        self.f3d, self.runs, self.lenses = f3d, runs, lenses
        self.n = g["pos"].shape[0]
        gen = torch.Generator().manual_seed(len(name) * 104729 + self.n)
        self.sh = {}
        for d in (27, 48):
            k = d // 3
            hi = torch.randn(self.n, 3, k - 1, generator=gen) * 0.15
            self.sh[d] = torch.cat([(g["rgb"] / 0.28209479177387814).unsqueeze(-1), hi], -1).reshape(self.n, d)
            self.sh[d] = self.sh[d].contiguous()
        self.up = []
        for v in self.views:
            h, w = v.height, v.width
            self.up.append(dict(image=torch.rand(h, w, 3, generator=gen, dtype=torch.float64) + 0.5,
                                depth=(torch.rand(h, w, generator=gen, dtype=torch.float64) + 0.5) * 0.1,
                                alpha=torch.rand(h, w, generator=gen, dtype=torch.float64) + 0.5))

    def colour(self, colour):
        return self.g["rgb"] if colour == "rgb" else self.sh[int(colour[2:4])]


def _act_scale(raw_abs, act):
    """The raw scale under `act` with the activated scale of the abs raw value raw_abs (exp: log(|r| + 1e-4))."""
    if act == "abs":
        return raw_abs
    return torch.log(raw_abs.double().abs() + 1e-4).float()


def _rand_quat(gen, n):
    q = torch.randn(n, 4, generator=gen, dtype=torch.float64)
    return q / q.norm(dim=1, keepdim=True)


def _stack(b, view, tx, ty, r0, opa):
    """WALL_K walls of sigma WALL_SIGMA px centred on tile (tx, ty), at distances r0, r0 + 0.004, ..."""
    xn, yn = view.leftmost + (tx + 0.5) * view.lx, view.topmost + (ty + 0.5) * view.ly
    h = math.sqrt(view.t2) * WALL_SIGMA / view.fx
    for j in range(WALL_K):
        z = (r0 + 0.004 * j) / math.sqrt(1 + xn * xn + yn * yn)
        b.at(xn, yn, z, h, h, opa=opa, tag="wall")


def _wall_opacity(gen):
    return 0.86 + 0.07 * float(torch.rand((), generator=gen))


def _redraw_walls(bad, stack_of, stack_opa, gen):
    """Draw a new opacity for every wall stack with a Gaussian in `bad` (its tiles' early stop lies within SAT_MARGIN
    of the threshold in some configuration); returns whether one was redrawn."""
    hit = {int(stack_of[i]) for i in torch.nonzero(bad).flatten().tolist() if stack_of[i] >= 0}
    for k in hit:
        stack_opa[k] = _wall_opacity(gen)
    return bool(hit)


def _fillers(view, n, gen):
    """[x/z, y/z, (distance), sigma px [3], opacity] of n fillers over tile rows 0..7."""
    xs = view.leftmost + view.lx * (0.6 + (view.ntx - 1.2) * torch.rand(n, generator=gen, dtype=torch.float64))
    ys = view.topmost + view.ly * (0.6 + 7.2 * torch.rand(n, generator=gen, dtype=torch.float64))
    sig = 1.5 + 2.0 * torch.rand(n, 3, generator=gen, dtype=torch.float64)
    ops = 0.05 + 0.3 * torch.rand(n, generator=gen, dtype=torch.float64)
    return [xs, ys, None, sig, ops]


def build_frame(act, seed=0, tries=40):
    view = B.View(384, 192, 200.0)
    gen = torch.Generator().manual_seed(1000 + seed)
    stacks = [tx0 + t for _, _, tx0, walls, _ in WALL_SITES for t in walls]
    stack_opa = [_wall_opacity(gen) for _ in stacks]
    acts = []
    vals = (0.5, -0.5, 1.5, -1.5)
    for j in range(16):
        acts.append([vals[(j + k) % 4] * (1 if (j >> k) & 1 else -1) for k in range(3)])
    fill, redraw = None, None
    for attempt in range(tries):
        b = B.Builder(view, seed=seed)
        runs = {}
        # runs in rows 0..7 (no wall reaches them): exactly k tiles each, inset 0.25 tiles
        place = {13: (0, 0), 1: (14, 0), 2: (16, 0), 3: (19, 0), 4: (0, 2), 8: (3, 2), 5: (8, 2), 7: (14, 2),
                 9: (0, 5), 12: (4, 5)}
        for j, (cnt, (tx, ty)) in enumerate(sorted(place.items())):
            w, h = RUN_SHAPES[cnt]
            runs[f"run{cnt}"] = (len(b.rows), (tx, tx + w, ty, ty + h), tuple(range(cnt)))
            b.tiles(tx, tx + w, ty, ty + h, 6.0 + 0.013 * j, opa=0.55, tag="run")
        # wall sites on row SITE_ROW: the runs behind them, then the stacks in front
        for k, (name, cnt, tx0, walls, live) in enumerate(WALL_SITES):
            runs[f"site{name}"] = (len(b.rows), (tx0, tx0 + cnt, SITE_ROW, SITE_ROW + 1), live)
            b.tiles(tx0, tx0 + cnt, SITE_ROW, SITE_ROW + 1, 6.3 + 0.017 * k, opa=0.6, tag="site")
        stack_of = [-1] * len(b.rows)
        for k, tx in enumerate(stacks):
            _stack(b, view, tx, SITE_ROW, 2.0 + 0.11 * k, stack_opa[k])
            stack_of += [k] * WALL_K
        # visible, unbinned (footprint outside the padded grid, inside the 1.2x frustum) and one behind the camera
        gx = view.Wp / 2.0 / view.fx
        xo = 0.5 * (gx + view.half_w)
        hh = 0.25 * (view.half_w - gx)
        for sgn in (1.0, -1.0):
            b.at(sgn * xo, 0.1 * sgn, 3.0 + 0.05 * sgn, hh, hh, tag="unbinned")
        b.raw((0.0, 0.0, -1.0), (0.1, 0.1, 0.1), tag="behind")
        # activation edges: raw scale components +-0.5 / +-1.5, at a depth where they span a few pixels
        for j, raw in enumerate(acts):
            sv = torch.tensor(raw, dtype=torch.float64)
            sa = sv.abs() + 1e-4 if act == "abs" else sv.exp()
            z = float(sa[:2].max()) * view.fx / 3.0 + 0.37 * j
            xn = view.leftmost + (1.5 + 1.4 * (j % 16)) * view.lx
            yn = view.topmost + 7.6 * view.ly
            b.rows.append(((xn * z, yn * z, z), tuple(raw), B._logit(0.5), False, "act"))
        n_fill = N - len(b.rows)
        assert n_fill > 100
        if fill is None:                                # fillers over rows 0..7 (away from the walls of row 10)
            fill = _fillers(view, n_fill, gen)
            fill[2] = 3.5 + 0.004 * torch.randperm(n_fill, generator=gen).double()
        elif redraw is not None:                        # new places and shapes for the fillers on a boundary
            new = _fillers(view, n_fill, gen)
            for k in (0, 1, 3, 4):
                fill[k][redraw] = new[k][redraw]
        xs, ys, rs, sig, ops = fill
        for j in range(n_fill):
            xn, yn, r = float(xs[j]), float(ys[j]), float(rs[j])
            z = r / math.sqrt(1 + xn * xn + yn * yn)
            sj = (sig[j] * z / view.fx).tolist()
            b.rows.append(((xn * z, yn * z, z), tuple(sj), B._logit(float(ops[j])), False, "filler"))
        stack_of = torch.tensor(stack_of + [-1] * (len(b.rows) - len(stack_of)))
        g, _, roles = b.build(shuffle=False)
        n = g["pos"].shape[0]
        agen = torch.Generator().manual_seed(3000 + seed)       # the same rotations and signs on every attempt
        is_fill = torch.tensor([t == "filler" for t in roles])
        is_act = torch.tensor([t == "act" for t in roles])
        free = is_fill | is_act
        # random rotations and raw signs for fillers and act Gaussians; quaternion norms 0.25 and 4 among them
        q = g["quat"].double()
        q[free] = _rand_quat(agen, int(free.sum()))
        norms = torch.ones(n, dtype=torch.float64)
        fid = torch.nonzero(free).squeeze(-1)
        norms[fid[0::4]] = 0.25
        norms[fid[1::4]] = 4.0
        g["quat"] = (q * norms.unsqueeze(1)).float()
        sc = g["scale"].clone()
        sgn = torch.where(torch.rand(n, 3, generator=agen) < 0.5, -1.0, 1.0)
        sc[is_fill] = sc[is_fill] * sgn[is_fill]
        sc[~is_act] = _act_scale(sc[~is_act], act)
        g["scale"] = sc.contiguous()
        opa = g["opa"].clone()
        aid = torch.nonzero(is_act).squeeze(-1)
        opa[aid[0::3]] = 5.9
        opa[aid[1::3]] = -5.9
        g["opa"] = opa
        f3d = _filter3d(g, act, free, agen)
        lens_names = {t: t for t in LENS_ORDER}
        sc_obj = Scene(f"frame-{act}", [view], g, act, roles, f3d, runs, [lens_names])
        sc_obj.stack_of = stack_of
        bad = unstable(sc_obj)
        if not bool(bad.any()):
            return sc_obj
        walls = _redraw_walls(bad, stack_of, stack_opa, gen)
        redraw = bad[is_fill] if bool(bad[is_fill].any()) else None
        design = ~free & (stack_of < 0)
        assert walls or not bool(bad[design].any()), ("a designed Gaussian sits on a decision boundary",
                                                      sorted({roles[i] for i in torch.nonzero(bad).flatten().tolist()}))
    raise AssertionError("frame: could not place the walls and fillers away from every decision boundary")


def _filter3d(g, act, free, gen):
    """f = 0 for the designed Gaussians and every third free one; 0.5 .. 1.5 x the smallest activated scale else."""
    raw = g["scale"].double()
    s = raw.abs() + 1e-4 if act == "abs" else raw.exp()
    c = 0.5 + torch.rand(raw.shape[0], generator=gen, dtype=torch.float64)
    f = c * s.amin(1)
    on = free.clone()
    on[torch.nonzero(free).squeeze(-1)[2::3]] = False
    return torch.where(on, f, torch.zeros_like(f)).float()


def build_batch(act, seed=3, tries=40):
    """n = 545 Gaussians in three views: ids 256..511 in the left part of view 0 only (views 1 and 2 see none of
    them)."""
    W, H = 256, 160
    v0 = B.View(W, H, 180.0)
    v1 = B.View(W, H, 170.0, tran=(-3.0, 0.1, 0.3))
    c, s = math.cos(0.12), math.sin(0.12)
    v2 = B.View(W, H, 210.0, 200.0, rot=torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]]),
                tran=(-3.0, -0.05, 0.0))
    views = [v0, v1, v2]
    gen = torch.Generator().manual_seed(2000 + seed)
    ids = torch.arange(N)
    left = (ids >= 256) & (ids < 512)
    def draw(i):
        lo, hi = (-0.85, -0.45) if bool(left[i]) else (0.1, 0.55)
        xn = lo + (hi - lo) * float(torch.rand((), generator=gen))
        yn = -0.35 + 0.7 * float(torch.rand((), generator=gen))
        dr = 0.0007 * float(torch.rand((), generator=gen))
        sg = 1.2 + 2.0 * torch.rand(3, generator=gen, dtype=torch.float64)
        op = 0.05 + 0.35 * float(torch.rand((), generator=gen))
        return xn, yn, dr, sg, op

    params = [draw(i) for i in range(N)]
    for attempt in range(tries):
        b = B.Builder(v0, seed=seed)
        roles = []
        for i in range(N):
            xn, yn, dr, sg, op = params[i]
            z = (4.5 + 0.003 * i + dr) / math.sqrt(1 + xn * xn + yn * yn)
            if i % 37 == 5 and not bool(left[i]):          # far away: every view sees it
                raw = [0.5, -1.5, 1.5] if i % 2 else [-0.5, 1.5, -1.5]
                z = (1.65 if act == "exp" else 1.5) * v0.fx / 3.0 * 1.5
                b.rows.append(((xn * z, yn * z, z), tuple(raw), B._logit(op), False, "act"))
                roles.append("act")
                continue
            b.rows.append(((xn * z, yn * z, z), tuple((sg * z / v0.fx).tolist()), B._logit(op), False, "filler"))
            roles.append("filler")
        agen = torch.Generator().manual_seed(4000 + seed)       # the same rotations and signs on every attempt
        g, _, _ = b.build(shuffle=False)
        free = torch.tensor([t != "wall" for t in roles])
        is_act = torch.tensor([t == "act" for t in roles])
        q = g["quat"].double()
        q[free] = _rand_quat(agen, int(free.sum()))
        norms = torch.ones(N, dtype=torch.float64)
        fid = torch.nonzero(free).squeeze(-1)
        norms[fid[0::5]] = 0.25
        norms[fid[1::5]] = 4.0
        g["quat"] = (q * norms.unsqueeze(1)).float()
        sc = g["scale"].clone()
        sgn = torch.where(torch.rand(N, 3, generator=agen) < 0.5, -1.0, 1.0)
        fill = free & ~is_act
        sc[fill] = sc[fill] * sgn[fill]
        sc[~is_act] = _act_scale(sc[~is_act], act)
        g["scale"] = sc.contiguous()
        f3d = _filter3d(g, act, free, agen)
        # view v's lens in the lens tier: three lenses, one per view
        lenses = [{t: LENS_ORDER[(k + v) % 3] for k, t in enumerate(LENS_ORDER)} for v in range(3)]
        sc_obj = Scene(f"batch-{act}", views, g, act, roles, f3d, {}, lenses)
        bad = unstable(sc_obj)
        if not bool(bad.any()):
            return sc_obj
        for i in torch.nonzero(bad).flatten().tolist():     # new places and shapes for those on a boundary
            params[i] = draw(i)
    raise AssertionError("batch: could not place the scene away from every decision boundary")


def first_views(sc, nv):
    """Scene sc restricted to its first nv views (a batch of B = nv)."""
    out = Scene.__new__(Scene)
    out.__dict__.update(sc.__dict__)
    out.views, out.lenses, out.up = sc.views[:nv], sc.lenses[:nv], sc.up[:nv]
    out.name = f"{sc.name}-b{nv}"
    return out


BUILDERS = {"frame-abs": lambda: build_frame("abs"), "frame-exp": lambda: build_frame("exp"),
            "batch-abs": lambda: build_batch("abs"), "batch-exp": lambda: build_batch("exp")}


# ----------------------------------------------------------------------------------------------------------------------
# configurations and the composed fp64 oracle
# ----------------------------------------------------------------------------------------------------------------------
def configs(sc):
    """The geometry configurations a scene is rendered in: (tier, lens name or None)."""
    return [("none", None), ("filt2d", None), ("filt3d", None)] + [("lens", ln) for ln in LENS_ORDER]


def view_lens(sc, v, lens):
    """Lens dict of view v for the configuration lens name `lens` (None: no lens)."""
    if lens is None:
        return None
    return lens_of(sc.lenses[v][lens] if v < len(sc.lenses) else lens, sc.views[v])


def _patched_culling(ln, cam):
    """A context in which gs_oracle.global_culling projects through lens `ln` (None: unchanged)."""
    @contextlib.contextmanager
    def ctx():
        if ln is None:
            yield
            return
        orig, orig_rays = O.global_culling, O.ray_info
        ox, oy = LO.offsets(ln, cam.width, cam.height, cam.fx, cam.fy)

        def culled(pos, nq, ns, rot, tran, near, hw, hh):
            return LO.global_culling_lens(pos, nq, ns, rot, tran, near, hw, hh, ln, ox, oy)

        def rays(rot, tran, Hp, Wp, fx, fy):          # per-pixel SH: the rays move with the principal point
            ro, lefttop, dx, dy = orig_rays(rot, tran, Hp, Wp, fx, fy)
            return ro, lefttop - torch.inverse(rot) @ torch.tensor([ox, oy, 0.0], dtype=rot.dtype), dx, dy

        O.global_culling, O.ray_info = culled, rays
        try:
            yield
        finally:
            O.global_culling, O.ray_info = orig, orig_rays
    return ctx()


@contextlib.contextmanager
def _unchained_filter3d(f3d):
    """F3.applied with the filter's backward left out: dL/ds taken as dL/ds' (a fault model for the comparator)."""
    orig = O.preactivate

    def pre(quat, scale, opa, rgb, scale_activation="abs", use_sh_coeff=False):
        nq, ns, o, c = orig(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
        sf, of = F3.filtered(ns, o, f3d)
        return nq, ns + (sf - ns).detach(), o + (of - o).detach(), c
    O.preactivate = pre
    try:
        yield
    finally:
        O.preactivate = orig


@contextlib.contextmanager
def composed(sc, v, tier, lens, cam, unchained=False):
    f3 = tier in ("filt3d", "lens")
    with contextlib.ExitStack() as st:
        st.enter_context(_patched_culling(view_lens(sc, v, lens), cam))
        if f3:
            st.enter_context((_unchained_filter3d if unchained else F3.applied)(sc.f3d.double()))
        yield


def _cam(view, rot=None, tran=None):
    c = view.cam()
    if rot is not None:
        c.rot, c.tran = rot, tran
    return c


def front(sc, v, tier, lens, dtype=torch.float64):
    """The composed front end of view v: dict(p, c, opa, accum, gi, rects, mask, rho) in blend order."""
    view = sc.views[v]
    cam = _cam(view)
    g = {q: t.to(dtype) for q, t in sc.g.items()}
    mode = "antialias" if tier != "none" else "none"
    with composed(sc, v, tier, lens, cam):
        nq, ns, opa_a, _ = O.preactivate(g["quat"], g["scale"], g["opa"], g["rgb"], sc.act)
        rp, rc, mask = O.global_culling(g["pos"], nq, ns, cam.rot.to(dtype), cam.tran.to(dtype), cam.near,
                                        cam.half_w, cam.half_h)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    c_c, o_c, keep = FO.filtered(rc[idx], opa_a[idx], cam, mode, FILTER2D_VAR)
    p_c = rp[idx]
    tx0, tx1, ty0, ty1 = O.tile_rects(p_c[:, :2], c_c, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty,
                                      cam.leftmost, cam.topmost)
    tx1, ty1 = torch.where(keep, tx1, tx0), torch.where(keep, ty1, ty0)
    gi, accum = O.bin_and_sort(p_c, c_c, (tx0, tx1, ty0, ty1), cam.ntx, cam.nty)
    rects = torch.zeros(sc.n, 4, dtype=torch.int64)
    rects[idx] = torch.stack([tx0, tx1, ty0, ty1], -1).long()
    return dict(p=p_c[gi].detach(), c=c_c[gi].detach(), opa=o_c[gi].detach(), accum=accum.long(), gi=idx[gi],
                rects=rects, mask=mask.bool(), idx=idx, pv=p_c.detach(), cv=c_c.detach(), keep=keep)


def unstable(sc):
    """[n] bool: Gaussians whose culling or tile rectangle changes under a relative perturbation STABLE_EPS of the
    projected mean, covariance or (with a lens) the undistorted radius, in any view and configuration; and every
    Gaussian of a tile whose early-stop margin is below SAT_MARGIN."""
    bad = torch.zeros(sc.n, dtype=torch.bool)
    eps = STABLE_EPS
    for v, view in enumerate(sc.views):
        cam = _cam(view)
        for tier, lens in configs(sc):
            fe = front(sc, v, tier, lens)
            idx, pv, cv = fe["idx"], fe["pv"], fe["cv"]
            base = fe["rects"][idx]
            for pos2d, cov in ((pv[:, :2] * (1 - eps), cv), (pv[:, :2] * (1 + eps), cv),
                               (pv[:, :2] + eps * cam.tile_lx, cv * (1 + eps)),
                               (pv[:, :2] - eps * cam.tile_lx, cv * (1 - eps))):
                r = O.tile_rects(pos2d, cov, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                                 cam.topmost)
                r = torch.stack(r, -1).long()
                r[:, 1] = torch.where(fe["keep"], r[:, 1], r[:, 0])
                r[:, 3] = torch.where(fe["keep"], r[:, 3], r[:, 2])
                empty_b, empty_r = base[:, 1] <= base[:, 0], (r[:, 1] <= r[:, 0]) | (r[:, 3] <= r[:, 2])
                diff = ((r != base).any(1) & ~(empty_b & empty_r))
                bad[idx[diff]] = True
            # culling margins: near plane, frustum (on the stored, lensed mean) and the fold-back radius
            pc = sc.g["pos"].double() @ view.rot.T + view.tran
            z = pc[:, 2]
            bad |= (z / view.near - 1).abs() < eps
            front_ = z > view.near
            xz = torch.where(front_, pc[:, 0] / z.clamp(min=1e-30), torch.zeros_like(z))
            yz = torch.where(front_, pc[:, 1] / z.clamp(min=1e-30), torch.zeros_like(z))
            ln = view_lens(sc, v, lens)
            if ln is not None:
                rm = LO.rho_max(ln["model"], ln["k"])
                if math.isfinite(rm):
                    bad |= front_ & (((xz * xz + yz * yz).sqrt() / rm - 1).abs() < 10 * eps)
            allp = torch.zeros(sc.n, 2, dtype=torch.float64)
            with _patched_culling(ln, cam):
                nq = sc.g["quat"].double() / sc.g["quat"].double().norm(dim=1, keepdim=True)
                rp, _, _ = O.global_culling(sc.g["pos"].double(), nq, torch.ones(sc.n, 3, dtype=torch.float64) * 0.01,
                                            view.rot, view.tran, view.near, math.inf, math.inf)
            allp = rp[:, :2]
            bad |= front_ & (((allp[:, 0].abs() / view.half_w - 1).abs() < eps) |
                             ((allp[:, 1].abs() / view.half_h - 1).abs() < eps))
            prof = E.tile_profile(fe, cam)
            low = torch.nonzero(prof["margin"] < SAT_MARGIN).flatten().tolist()
            for t in low:
                s, e = int(fe["accum"][t]), int(fe["accum"][t + 1])
                bad[fe["gi"][s:e]] = True
    return bad


def live_rows(sc, gid, v=0, tier="none", lens=None):
    """Row k of Gaussian gid (its rectangle in raster order) -> live (its tile reaches the instance) in view v."""
    fe = front(sc, v, tier, lens)
    prof = E.tile_profile(fe, _cam(sc.views[v]))
    tx0, tx1, ty0, ty1 = fe["rects"][gid].tolist()
    out = []
    for ty in range(ty0, ty1):
        for tx in range(tx0, tx1):
            t = ty * sc.views[v].ntx + tx
            s, e = int(fe["accum"][t]), int(fe["accum"][t + 1])
            k = (fe["gi"][s:e] == gid).nonzero().flatten()
            assert k.numel() == 1
            out.append(int(k) <= int(prof["last"][t]))
    return out


def oracle(sc, colour, tier, lens, dt, views=None, dtype=torch.float64, unchained=False, tiles=None):
    """Images, parameter gradients and per-view camera gradients of one frame of scene sc (views: the view indices,
    default all; the loss is the sum over them), for its upstream gradients: image, plus depth and alpha with dt.
    Returns dict(images [list], grads {name}, cam [list of (drot, dtran)])."""
    views = range(len(sc.views)) if views is None else views
    p = {q: t.to(dtype).clone().requires_grad_(True) for q, t in sc.g.items()}
    p["rgb"] = sc.colour(colour).to(dtype).clone().requires_grad_(True)
    mode = "antialias" if tier != "none" else "none"
    pix = colour.endswith("pixel") and colour != "rgb"
    gauss = colour.endswith("gauss")
    loss, images, leaves = 0, [], []
    for v in views:
        view = sc.views[v]
        rot = view.rot.to(dtype).clone().requires_grad_(True)
        tran = view.tran.to(dtype).clone().requires_grad_(True)
        leaves += [rot, tran]
        cam = _cam(view, rot, tran)
        up = sc.up[v]
        with composed(sc, v, tier, lens, cam, unchained):
            rgb = G.gaussian_logits(p["pos"], p["rgb"], cam) if gauss else p["rgb"]
            args = (p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, mode, FILTER2D_VAR)
            if dt:
                o = FO.render_maps(*args, scale_activation=sc.act, use_sh_coeff=pix)
                img = o["image"]
                loss = loss + (o["depth"] * up["depth"].to(dtype)).sum() + (o["alpha"] * up["alpha"].to(dtype)).sum()
            else:
                img = FO.render(*args, scale_activation=sc.act, use_sh_coeff=pix, tiles=tiles)
        loss = loss + (img * up["image"].to(dtype)).sum()
        images.append(img.detach())
    gr = torch.autograd.grad(loss, [p[q] for q in NAMES] + leaves, allow_unused=True)
    grads = {q: (torch.zeros_like(p[q]) if x is None else x.detach()) for q, x in zip(NAMES, gr)}
    cams = [(gr[5 + 2 * k].detach(), gr[6 + 2 * k].detach()) for k in range(len(leaves) // 2)]
    return dict(images=images, grads=grads, cam=cams)


def stats_oracle(sc, tier, lens):
    """densify_stats_oracle.frame_stats summed over the views (image-only upstream, RGB)."""
    n = sc.n
    acc = dict(grad2d=torch.zeros(n, dtype=torch.float64), absgrad=torch.zeros(n, dtype=torch.float64),
               count=torch.zeros(n, dtype=torch.int64), radius=torch.zeros(n, dtype=torch.float64))
    p = {q: t.double() for q, t in sc.g.items()}
    for v, view in enumerate(sc.views):
        cam = _cam(view)
        up = sc.up[v]["image"]

        def loss(out, cam=cam, up=up):
            return (cam.crop(torch.clamp(out["padded"], 0, 1)) * up).sum()
        with composed(sc, v, tier, lens, cam):
            r = DS.frame_stats(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, loss, mode="antialias",
                               variance=FILTER2D_VAR, scale_activation=sc.act, absgrad=True)
        acc["grad2d"] += r["grad2d"]
        acc["absgrad"] += r["absgrad"]
        acc["count"] += r["count"]
        acc["radius"] = torch.maximum(acc["radius"], r["radius"])
    return acc


# ----------------------------------------------------------------------------------------------------------------------
# comparator
# ----------------------------------------------------------------------------------------------------------------------
def compare(n, got, ref, images=None, ref_images=None, cams=None, ref_cams=None, rtol=GRAD_RTOL, groups=None):
    """Failures (empty: pass).  Per Gaussian and parameter: max |got - ref| <= rtol * max(its own max |ref|,
    GRAD_FLOOR * the frame's max |ref|); a Gaussian whose reference row is exactly zero must be exactly zero.  groups
    [n] (>= 0: a wall stack): a wall's scale is the largest max |ref| of its stack instead of its own.  Images
    IMG_ATOL absolute; camera gradients CAM_RTOL relative per view.

    Why walls are held per stack: the opacity gradient of a wall deep in a saturating stack is the difference of its
    own colour term and the colour recovered behind it, two nearly equal sums; the fp32 backward forms each to ~1e-6
    relative of the stack's gradient scale, so a deep wall's error is bounded by the stack's scale, not its own (on an
    H100: opacity errors of 2.5e-6 .. 1.2e-5 against own magnitudes of 2e-4 .. 9e-3, at most 1.6e-2 of its own and
    below 1e-4 of the stack's).  tile_edges.compare holds its walls over the walls the same way."""
    fails = []
    for q, r in ref.items():
        if q not in got:
            continue
        g = got[q].detach().double().cpu().reshape(n, -1)
        r = r.detach().double().cpu().reshape(n, -1)
        if not bool(torch.isfinite(g).all()):
            fails.append(f"{q}: non-finite gradient")
            continue
        mag = r.abs().amax(1)
        glob = float(mag.max())
        err = (g - r).abs().amax(1)
        own = mag
        if groups is not None:
            grp = groups.long().cpu()
            wall = grp >= 0
            if bool(wall.any()):
                top = torch.zeros(int(grp.max()) + 1, dtype=torch.float64).scatter_reduce(0, grp[wall], mag[wall],
                                                                                         "amax")
                own = torch.where(wall, top[grp.clamp(min=0)], mag)
        scale = torch.clamp(own, min=GRAD_FLOOR * glob)
        zero = mag == 0
        bad = ((err > rtol * scale) & ~zero) | (zero & (err > 0))
        for i in torch.nonzero(bad).flatten().tolist()[:4]:
            fails.append(f"{q}[{i}]: max|d| {float(err[i]):.3e} vs |ref| {float(mag[i]):.3e}")
        if int(bad.sum()) > 4:
            fails.append(f"{q}: {int(bad.sum())} Gaussians off")
    for k, (a, b) in enumerate(zip(images or [], ref_images or [])):
        e = float((a.detach().double().cpu() - b.detach().double().cpu()).abs().max())
        if not e <= IMG_ATOL:
            fails.append(f"image {k}: max|d| {e:.3e}")
    for k, (a, b) in enumerate(zip(cams or [], ref_cams or [])):
        a = torch.cat([x.detach().double().cpu().reshape(-1) for x in a])
        b = torch.cat([x.detach().double().cpu().reshape(-1) for x in b])
        e, s = float((a - b).abs().max()), float(b.abs().max())
        if not e <= CAM_RTOL * s:
            fails.append(f"camera {k}: max|d| {e:.3e} > {CAM_RTOL:g} x {s:.3e}")
    return fails


def compare_stats(st, ref, absgrad):
    fails = []
    for k in ("grad2d",) + (("absgrad",) if absgrad else ()):
        g = st[k].double().cpu()
        r = ref[k]
        scale = torch.clamp(r.abs(), min=GRAD_FLOOR * float(r.abs().max()))
        bad = (g - r).abs() > STAT_RTOL * scale
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0])
            fails.append(f"{k}: {int(bad.sum())} off, e.g. [{i}] {float(g[i]):.6e} vs {float(r[i]):.6e}")
    if not torch.equal(st["count"].cpu().long(), ref["count"]):
        fails.append("count differs")
    want = torch.ceil(ref["radius"])
    frac = ref["radius"] - torch.floor(ref["radius"])
    tie = (frac < 1e-4) | (frac > 1 - 1e-4)
    bad = (st["max_radius"].double().cpu() != want) & ~tie
    if bool(bad.any()):
        fails.append(f"max_radius: {int(bad.sum())} off")
    return fails
