"""Every blend kernel variant on the tile-edge fixtures of tests/tile_edges.py (tile counts at chunk and round
boundaries, tiles that saturate on them or while later chunks are still in flight, partial saturation, cropped
border tiles), through the fused frame with gs_tune("strict", 1), against the fp64 oracle with the per-tile,
per-instance comparator.  Also: the forward's per-tile consumed count, stale gradient rows of a second frame, and
the strict dispatch contract.  The oracle is computed once per fixture and output kind; knobs do not change
binning or order."""
import os

import pytest
import torch

import tile_edges as E
from helpers import device_depth_keys

pytestmark = pytest.mark.gpu

if any(k.startswith("GS_TUNE_") for k in os.environ):
    pytest.skip("GS_TUNE_* is set: the variant matrix needs the shipped knob defaults", allow_module_level=True)

# the shipped knob values (render.cu gs_tuning), restored after every case
SHIPPED = dict(fwd_kernel=0, fwd_ch=128, bwd_kernel=1, bwd_px=8, bwd_ws=0, bwd_unroll=4, bwd_stages=3, bwd_minb=10,
               bwd_rq=4, fwd_px=4, bwd_ch=32, strict=0, gather=1, sh_tc=-1, blend_repack=1)
PACKED_BWD = E.decode_bwd_key(8022416)          # the packed path's own default backward


def _variants():
    v = []
    for ga in (1, 0):
        for px in (4, 8):
            for ch in (64, 128, 256):
                k = dict(gather=ga, fwd_px=px, fwd_ch=ch, **({} if ga else PACKED_BWD))
                v.append((f"fwd-{'gather' if ga else 'packed'}-px{px}-ch{ch}", "rgb", k))
    v.append(("fwd-ws", "rgb", dict(gather=0, fwd_kernel=1, **PACKED_BWD)))
    v.append(("fwd-aux", "aux", {}))
    v += [(f"bwd-gather32-{key}", "rgb", dict(bwd_ch=32, **E.decode_bwd_key(key))) for key in E.BWD_GATHER_32]
    v += [(f"bwd-gather64-{key}", "rgb", dict(bwd_ch=64, **E.decode_bwd_key(key))) for key in E.BWD_GATHER_64]
    v += [(f"bwd-packed-{key}", "rgb", dict(gather=0, **E.decode_bwd_key(key))) for key in E.BWD_PACKED]
    v += [(f"bwd-shipped-repack{r}", "rgb", dict(blend_repack=r)) for r in (0, 1)]
    v += [(f"bwd-round1-px{px}", "rgb", dict(gather=0, bwd_kernel=0, bwd_px=px)) for px in (4, 8)]
    v += [(f"bwd-aux-repack{r}", "aux", dict(blend_repack=r)) for r in (0, 1)]
    v += [(f"abs-{m}-repack{r}", m + "-abs", dict(blend_repack=r)) for m in ("rgb", "aux") for r in (0, 1)]
    for d in (27, 48):
        for tc in (0, 3, 7):
            v.append((f"sh{d}-tc{tc}", f"sh{d}", dict(sh_tc=tc)))
            if tc != 7:                              # the two-pixel tensor-core backward has no aux kernel
                v.append((f"sh{d}-tc{tc}-aux", f"sh{d}-aux", dict(sh_tc=tc)))
    v += [(f"feat{F}", f"feat{F}", {}) for F in (8, 16, 32)]
    return v


VARIANTS = _variants()
CASES = [(fx, name) for name, _, _ in VARIANTS for fx in E.BUILDERS]
KIND = {name: (kind, knobs) for name, kind, knobs in VARIANTS}


def _set(gs, knobs):
    for k, val in knobs.items():
        gs[0].tune(k, val)


def _restore(gs):
    _set(gs, SHIPPED)


class _Cache:
    def __init__(self, cuda):
        self.cuda = cuda
        self.fx, self.keys, self.ref = {}, {}, {}

    def fixture(self, name):
        if name not in self.fx:
            fx = E.BUILDERS[name]()
            self.fx[name] = fx
            self.keys[name] = device_depth_keys(fx.g, fx.cam, self.cuda)
        return self.fx[name]

    def oracle(self, name, kind):
        if (name, kind) not in self.ref:
            fx = self.fixture(name)
            base = kind[:-4] if kind.endswith("-abs") else kind
            r = E.oracle(fx, base, depth_key=self.keys[name], tile_scale=fx.tile_scale)
            if kind.endswith("-abs"):
                r["stats"] = E.stats_oracle(fx, aux=base == "aux", depth_key=self.keys[name])
            self.ref[(name, kind)] = r
        return self.ref[(name, kind)]


@pytest.fixture(scope="module")
def cache(gs, cuda):
    return _Cache(cuda)


def _frame(gs, fx, kind, rctx=None, opa=None):
    """One forward + backward of fixture fx on the fused frame path; returns outputs, gradients and the frame's
    per-tile consumed counts and tile ranges."""
    import renderer
    dev = torch.device("cuda", 0)
    sh = kind.startswith("sh")
    aux = "aux" in kind
    feat = kind.startswith("feat")
    absg = kind.endswith("-abs")
    rctx = rctx if rctx is not None else gs[0].RenderContext()
    g = dict(fx.g)
    if sh:
        g["rgb"] = fx.sh[int(kind[2:4])]
    if opa is not None:
        g["opa"] = opa
    d = {q: g[q].to(dev).clone().requires_grad_(True) for q in E.NAMES}
    v = fx.view
    args = (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")
    stats = None
    if absg:
        stats = dict(grad2d=torch.zeros(fx.n, device=dev), count=torch.zeros(fx.n, dtype=torch.int32, device=dev),
                     max_radius=torch.zeros(fx.n, device=dev), absgrad=torch.zeros(fx.n, device=dev))
        rctx.set_densify_stats(stats["grad2d"], stats["count"], stats["max_radius"], stats["absgrad"])
    up = fx.up.float().to(dev)
    out = {}
    if feat:
        F = int(kind[4:])
        df = fx.feat[F].to(dev).clone().requires_grad_(True)
        img, fm, _, _, _ = renderer.render_frame_feat(rctx, *(d[q] for q in E.NAMES), df, *args, final=True)
        torch.autograd.backward([img, fm], [up, fx.up_feat[F].float().to(dev)])
        out["features"] = fm.detach()
    elif aux:
        img, dep, alp, _ = renderer.render_frame_aux(rctx, *(d[q] for q in E.NAMES), *args, background=E.BG,
                                                     final=True)
        torch.autograd.backward([img, dep, alp], [up, fx.up_depth.float().to(dev), fx.up_alpha.float().to(dev)])
        out.update(depth=dep.detach(), alpha=alp.detach())
    else:
        img, _ = renderer.render_frame_final(rctx, *(d[q] for q in E.NAMES), *args)
        img.backward(up)
    torch.cuda.synchronize()
    out["image"] = img.detach()
    out["grads"] = {q: d[q].grad.detach().cpu() for q in E.NAMES}
    if feat:
        out["grads"]["feat"] = df.grad.detach().cpu()
    out["consumed"] = rctx.tile_consumed().cpu().long()
    out["accum"] = rctx.sorted_instances()[1].cpu().long()
    if absg:
        rctx.clear_densify_stats()
        out["stats"] = {k: t.cpu() for k, t in stats.items()}
    return out


def _check(fx, got, ref):
    extra = []
    if "alpha" in got:
        extra.append(("alpha", got["alpha"], ref["alpha"]))
    fails = E.compare(fx, got["grads"], ref["grads"], got["image"], ref["image"], extra=extra,
                      scale=ref.get("tile_scale"))
    if "features" in got:
        e = float((got["features"].double().cpu() - ref["features"]).abs().max())
        if not e <= 1e-4 * max(1.0, float(fx.feat[got["features"].shape[-1]].abs().max())):
            fails.append(f"features: max|d| {e:.3e}")
    if "depth" in got:
        e = float((got["depth"].double().cpu() - ref["depth"]).abs().max())
        if not e <= 1e-4 * float(ref["depth"].abs().max()):
            fails.append(f"depth: max|d| {e:.3e}")
    assert torch.equal(got["accum"], ref["fe"]["accum"]), "binning differs from the oracle's"
    # the forward's per-tile consumed count, in whole chunks: within [last live + 1, count]; == count if never saturated
    count = ref["fe"]["accum"][1:] - ref["fe"]["accum"][:-1]
    last = fx.profile["last"]
    c = got["consumed"]
    nz = count > 0
    if bool((c > count).any()) or bool((c[nz] < last[nz] + 1).any()):
        bad = ((c > count) | (nz & (c < last + 1))).nonzero().flatten()[:4].tolist()
        fails.append(f"consumed out of range on tiles {bad}: {[(int(c[t]), int(last[t]), int(count[t])) for t in bad]}")
    never = nz & ~fx.profile["full"] & (last == count - 1)
    if not torch.equal(c[never], count[never]):
        fails.append("consumed != count on a tile that never saturates")
    if "stats" in got:
        st, rs = got["stats"], ref["stats"]
        walls = fx.tile_of < 0
        wr = fx.wall_rtol.get("stats", E.GRAD_RTOL)
        for k in ("grad2d", "absgrad"):
            d = (st[k].double() - rs[k]).abs()
            s = float(rs[k].abs().max())
            if not float(d[~walls].max()) <= E.GRAD_RTOL * s:
                fails.append(f"{k}: max|d| {float(d[~walls].max()):.3e} > 1e-3 x {s:.3e}")
            if bool(walls.any()) and not float(d[walls].max()) <= wr * float(rs[k][walls].abs().max()):
                fails.append(f"{k}: walls: max|d| {float(d[walls].max()):.3e}")
        if not torch.equal(st["count"].long(), rs["count"]):
            fails.append("stats count differs")
    return fails


@pytest.mark.parametrize("fixture,variant", CASES)
def test_variant_vs_oracle(gs, cache, fixture, variant):
    kind, knobs = KIND[variant]
    fx = cache.fixture(fixture)
    ref = cache.oracle(fixture, kind)
    try:
        _set(gs, dict(knobs, strict=1))
        got = _frame(gs, fx, kind)
    finally:
        _restore(gs)
    fails = _check(fx, got, ref)
    assert not fails, fails


@pytest.mark.parametrize("path", ["gather", "packed"])
def test_stale_rows_do_not_leak(gs, cache, path):
    """Two frames in one RenderContext, same geometry (same binning, M and gradient rows) but the second with the
    walls' opacities raised: it stops earlier, and the first frame's tail rows, still in the workspace, must not
    reach its gradients."""
    fx = cache.fixture("walls")
    ref = cache.oracle("walls", "rgb")
    weak = torch.where(fx.tile_of < 0, torch.full_like(fx.g["opa"], -0.5), fx.g["opa"])
    knobs = dict(strict=1, **({} if path == "gather" else dict(gather=0, **PACKED_BWD)))
    try:
        _set(gs, knobs)
        rctx = gs[0].RenderContext()
        first = _frame(gs, fx, "rgb", rctx=rctx, opa=weak)
        got = _frame(gs, fx, "rgb", rctx=rctx)
    finally:
        _restore(gs)
    assert torch.equal(first["accum"], got["accum"])
    assert bool((first["consumed"] >= got["consumed"]).all()) and bool((first["consumed"] > got["consumed"]).any())
    fails = _check(fx, got, ref)
    assert not fails, fails


def test_strict_dispatch_contract(gs, cache):
    """strict 1: a backward knob combination with no kernel raises before any launch; strict 0: the same
    combination runs the shipped kernel and matches the oracle."""
    fx = cache.fixture("counts")
    ref = cache.oracle("counts", "rgb")
    off = dict(bwd_minb=11)                         # key 8043411: in no table
    assert E.encode_bwd_key(dict(E.decode_bwd_key(8043410), **off)) not in E.BWD_GATHER_32
    import renderer
    try:
        _set(gs, dict(off, strict=1))
        rctx = gs[0].RenderContext()
        d = {q: fx.g[q].cuda().clone().requires_grad_(True) for q in E.NAMES}
        v = fx.view
        img, _ = renderer.render_frame_final(rctx, *(d[q] for q in E.NAMES), v.width, v.height, v.fx, v.fy, v.rot,
                                             v.tran, v.near, 0.05, "abs")      # the forward has no such knob
        torch.cuda.synchronize()
        n0 = gs[0].kernel_launches()
        with pytest.raises(RuntimeError):
            img.backward(fx.up.float().cuda())
        torch.cuda.synchronize()
        assert gs[0].kernel_launches() == n0
        _set(gs, dict(off, strict=0))
        got = _frame(gs, fx, "rgb")
    finally:
        _restore(gs)
    fails = _check(fx, got, ref)
    assert not fails, fails
