"""Every fused projection instantiation of the table of tests/project_edges.py (single-view and batched backward and
forward, and the densification statistics), each through its public entry point on the scenes built there, against
the composed fp64 oracle with the per-Gaussian comparator; and stale rows: two frames in one context, the second
with stronger walls.  The oracle is computed once per (scene, colour, tier, lens, upstream kind); the camera
gradient does not change the parameter gradients, so CG and non-CG entries share it."""
import os

import pytest
import torch

import project_edges as P

pytestmark = pytest.mark.gpu

if any(k.startswith("GS_TUNE_") for k in os.environ):
    pytest.skip("GS_TUNE_* is set: the cases need the shipped knob defaults", allow_module_level=True)

TABLE = P.table()
BWD = [r for r in TABLE if r["kernel"] in ("bwd", "bwd_batch")]
FWD = [r for r in TABLE if r["kernel"] in ("fwd", "fwd_batch")]
STATS = [r for r in TABLE if r["kernel"] in ("stats", "stats_batch")]
assert len(BWD) + len(FWD) + len(STATS) == len(TABLE)      # one case per table entry
# batch size per tier: B = 1, 2 and 3 views
BATCH_VIEWS = {"none": 1, "filt2d": 2, "filt3d": 3, "lens": 3}


def _scene_name(r):
    batch = r["kernel"].endswith("batch")
    act = "exp" if r.get("dt") else "abs"
    return f"{'batch' if batch else 'frame'}-{act}"


def _views(r):
    return BATCH_VIEWS[r["tier"]] if r["kernel"].endswith("batch") else 1


def _lens(r):
    """The lens of a lens-tier entry: per-pixel SH takes a principal point only; the others rotate through the three
    lenses with the colour and DT (a batch gives each view a different one)."""
    if r["tier"] != "lens":
        return None
    if r["colour"].endswith("pixel"):
        return "pinhole-offset"
    k = list(P.COLOURS).index(r["colour"]) + int(bool(r.get("dt")))
    return P.LENS_ORDER[k % 3]


class _Cache:
    def __init__(self):
        self.sc, self.ref, self.st = {}, {}, {}

    def scene(self, name, nv=1):
        if name not in self.sc:
            self.sc[name] = P.BUILDERS[name]()
        sc = self.sc[name]
        return P.first_views(sc, nv) if nv < len(sc.views) else sc

    def oracle(self, name, nv, colour, tier, lens, dt):
        key = (name, nv, colour, tier, lens, dt)
        if key not in self.ref:
            self.ref[key] = P.oracle(self.scene(name, nv), colour, tier, lens, dt)
        return self.ref[key]

    def stats(self, name, nv, tier, lens):
        key = (name, nv, tier, lens)
        if key not in self.st:
            self.st[key] = P.stats_oracle(self.scene(name, nv), tier, lens)
        return self.st[key]


@pytest.fixture(scope="module")
def cache(gs, cuda):
    return _Cache()


def _context(gs, sc, r, lens, dev):
    import renderer
    rctx = gs[0].RenderContext()
    s = r["setters"]
    rctx.set_sh_eval(renderer.SH_EVAL[s["sh_eval"]])
    rctx.set_filter2d(renderer.FILTER2D[s["filter2d"]], P.FILTER2D_VAR)
    if s["filter3d"]:
        rctx.set_filter3d(sc.f3d.to(dev).contiguous())
    if s["lens"]:
        import lens_oracle as LO
        lns = [P.view_lens(sc, v, lens) for v in range(len(sc.views))]
        rctx.set_lens([LO.MODELS[ln["model"]] for ln in lns],
                      torch.tensor([[ln["cx"], ln["cy"], *ln["k"]] for ln in lns], dtype=torch.float32))
    return rctx


def _frame(gs, sc, r, lens, dev, stats=None, rctx=None, opa=None, backward=True):
    """One forward + backward of entry r through its public call: (images, parameter grads, per-view camera grads).
    rctx: an existing context (its workspace keeps the previous frame's rows); opa: replacement opacity logits."""
    import renderer
    rctx = _context(gs, sc, r, lens, dev) if rctx is None else rctx
    if stats is not None:
        rctx.set_densify_stats(*stats)
    d = {q: sc.g[q].to(dev).clone().requires_grad_(True) for q in P.NAMES}
    if opa is not None:
        d["opa"] = opa.to(dev).clone().requires_grad_(True)
    d["rgb"] = sc.colour(r["colour"]).to(dev).clone().requires_grad_(True)
    args = [d[q] for q in P.NAMES]
    vs = sc.views
    v = vs[0]
    dt, cg = r.get("dt", False), r.get("cg", False)
    cams = []
    if r["kernel"].endswith("batch"):
        rot = torch.stack([x.rot.float() for x in vs]).to(dev).requires_grad_(cg)
        tran = torch.stack([x.tran.float() for x in vs]).to(dev).requires_grad_(cg)
        fn = renderer.render_frame_batch_cam if cg else renderer.render_frame_batch
        img, dep, alp, _ = fn(rctx, *args, v.width, v.height, [x.fx for x in vs], [x.fy for x in vs], rot, tran,
                              v.near, 0.05, sc.act, final=True)
        up = [torch.stack([u[k] for u in sc.up]).float().to(dev) for k in ("image", "depth", "alpha")]
        outs = [img, dep, alp] if dt else [img]
        if backward:
            torch.autograd.backward(outs, up[:len(outs)])
        images = list(img.detach())
        if cg:
            cams = [(rot.grad[k], tran.grad[k]) for k in range(len(vs))]
    else:
        up = [sc.up[0][k].float().to(dev) for k in ("image", "depth", "alpha")]
        rot, tran = v.rot.float().to(dev).requires_grad_(cg), v.tran.float().to(dev).requires_grad_(cg)
        if cg:
            img, dep, alp, _ = renderer.render_frame_cam(rctx, *args, v.width, v.height, v.fx, v.fy, rot, tran,
                                                         v.near, 0.05, sc.act, final=True)
        elif dt:
            img, dep, alp, _ = renderer.render_frame_aux(rctx, *args, v.width, v.height, v.fx, v.fy, rot, tran,
                                                         v.near, 0.05, sc.act, final=True)
        else:
            img, _ = renderer.render_frame_final(rctx, *args, v.width, v.height, v.fx, v.fy, rot, tran, v.near, 0.05,
                                                 sc.act)
        outs = [img, dep, alp] if dt else [img]
        if backward:
            torch.autograd.backward(outs, up[:len(outs)])
        images = [img.detach()]
        if cg:
            cams = [(rot.grad, tran.grad)]
    torch.cuda.synchronize()
    return images, {q: d[q].grad for q in P.NAMES}, cams


@pytest.mark.parametrize("entry", BWD, ids=[P.row_id(r) for r in BWD])
def test_backward_instantiation_vs_oracle(gs, cuda, cache, entry):
    """Image 1e-4 abs, every Gaussian's five gradients 1e-3 of its own scale (exact zeros where the oracle's row is
    zero), each view's camera gradient 1e-3 relative."""
    name, lens, nv = _scene_name(entry), _lens(entry), _views(entry)
    sc = cache.scene(name, nv)
    ref = cache.oracle(name, nv, entry["colour"], entry["tier"], lens, entry["dt"])
    images, grads, cams = _frame(gs, sc, entry, lens, cuda)
    fails = P.compare(sc.n, grads, ref["grads"], images, ref["images"], cams, ref["cam"] if cams else None,
                      groups=getattr(sc, "stack_of", None))
    assert not fails, fails


@pytest.mark.parametrize("entry", FWD, ids=[P.row_id(r) for r in FWD])
def test_forward_instantiation_vs_oracle(gs, cuda, cache, entry):
    """Each view's image 1e-4 abs (the forward alone, no backward)."""
    name, lens, nv = _scene_name(entry), _lens(entry), _views(entry)
    sc = cache.scene(name, nv)
    ref = cache.oracle(name, nv, entry["colour"], entry["tier"], lens, False)
    images, _, _ = _frame(gs, sc, dict(entry, dt=False, cg=False), lens, cuda, backward=False)
    fails = P.compare(sc.n, {}, {}, images, ref["images"])
    assert not fails, fails


def _weak_walls(sc):
    """The scene's opacity logits with every wall at opacity 0.3: no tile saturates, every row is live."""
    opa = sc.g["opa"].clone()
    opa[torch.tensor([r == "wall" for r in sc.roles])] = float(torch.logit(torch.tensor(0.3)))
    return opa


# (kernel, colour, cg): per-Gaussian SH 48 and per-pixel SH 27 single-view, batched RGB and SH, with and without CG
STALE = [("bwd", "sh48-gauss", False), ("bwd", "sh48-gauss", True), ("bwd", "sh27-pixel", False),
         ("bwd", "rgb", False), ("bwd", "rgb", True), ("bwd_batch", "rgb", False), ("bwd_batch", "rgb", True),
         ("bwd_batch", "sh27-gauss", False), ("bwd_batch", "sh48-gauss", True)]


@pytest.mark.parametrize("kernel,colour,cg", STALE, ids=[f"{k}-{c}-{'cg' if g else 'nocg'}" for k, c, g in STALE])
def test_stale_rows_of_an_earlier_frame_do_not_leak(gs, cuda, cache, kernel, colour, cg):
    """Two frames in one context with the same geometry: the first with weak walls (every row live, written), the
    second with the scene's walls, which stop its saturated tiles earlier, so that the first frame's rows are still in
    the workspace under an older epoch.  The second frame must match its oracle.  Batched with CG: the first frame's
    view 1 is view 0's camera, so the second CTA writes non-zero camera rows for view 1 that the second frame, whose
    view 1 sees none of that CTA's Gaussians, must overwrite with zeros."""
    entry = next(r for r in BWD if (r["kernel"], r["colour"], r["tier"], r["dt"], r["cg"]) ==
                 (kernel, colour, "none", False, cg))
    name, nv = _scene_name(entry), (3 if kernel == "bwd_batch" else 1)
    sc = cache.scene(name, nv)
    ref = cache.oracle(name, nv, colour, "none", None, False)
    rctx = _context(gs, sc, entry, None, cuda)
    first = sc
    if kernel == "bwd_batch":
        first = P.first_views(sc, 3)
        first.views = [sc.views[0], sc.views[0], sc.views[2]]
    _frame(gs, first, entry, None, cuda, rctx=rctx, opa=_weak_walls(sc))
    images, grads, cams = _frame(gs, sc, entry, None, cuda, rctx=rctx)
    fails = P.compare(sc.n, grads, ref["grads"], images, ref["images"], cams, ref["cam"] if cams else None,
                      groups=getattr(sc, "stack_of", None))
    assert not fails, fails


@pytest.mark.parametrize("entry", STATS, ids=[P.row_id(r) for r in STATS])
def test_statistics_instantiation_vs_oracle(gs, cuda, cache, entry):
    """grad2d (and absgrad) 1e-3 per Gaussian, count exact, max_radius exact away from integer ties."""
    name, lens = ("batch-abs" if entry["kernel"] == "stats_batch" else "frame-abs"), None
    nv = _views(entry)
    if entry["tier"] == "lens":
        lens = "opencv"
    sc = cache.scene(name, nv)
    ref = cache.stats(name, nv, entry["tier"], lens)
    n = sc.n
    st = dict(grad2d=torch.zeros(n, device=cuda), count=torch.zeros(n, dtype=torch.int32, device=cuda),
              max_radius=torch.zeros(n, device=cuda))
    args = [st["grad2d"], st["count"], st["max_radius"]]
    if entry["absgrad"]:
        st["absgrad"] = torch.zeros(n, device=cuda)
        args.append(st["absgrad"])
    r = dict(entry, dt=False, cg=False)
    _frame(gs, sc, r, lens, cuda, stats=args)
    fails = P.compare_stats(st, ref, entry["absgrad"])
    assert not fails, fails
