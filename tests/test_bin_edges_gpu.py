"""The fused frame's front end against the decision layer of tests/bin_edges.py: culling mask, per-Gaussian tile
rectangles, the exact (tile, depth, id) instance order and tile ranges, the visible mask, zero gradient rows of
unbinned Gaussians, and the image against gs_oracle.draw on the sorted lists.  Decided placements must match the
oracle exactly; ambiguous ones must pick one of their candidate rectangles and stay consistent.  Every scene also
runs as a three-view batch (rows offset by v * nty, equal to the single-view frames) and, without filter or lens,
through the packed path (gs_tune("gather", 0)), whose tile ranges come from pack_sorted_kernel's own loops."""
import pytest
import torch

import bin_edges as E
from helpers import device_depth_keys

pytestmark = pytest.mark.gpu

IMG_ATOL = 1e-4
_STATS = {}


def _ctx(gs, sc):
    rctx = gs[0].RenderContext()
    if sc.mode == "antialias":
        rctx.set_filter2d(gs[0].FILTER2D_ANTIALIAS, 0.3)
    if sc.mode == "opencv":
        ls = [E.lens_of(v) for v in sc.views]
        rctx.set_lens([gs[0].LENS_OPENCV] * len(ls),
                      torch.tensor([[ln["cx"], ln["cy"], *ln["k"]] for ln in ls], dtype=torch.float32))
    return rctx


def _keys(sc, v, dev):
    return device_depth_keys(sc.g, sc.views[v].cam(lens_free=sc.mode == "opencv"), dev)


def _single(gs, sc, dev, grads=True, views=None):
    """One single-view fused frame per view of sc (forward, and backward with a random upstream gradient)."""
    import renderer
    out = []
    for v in (range(len(sc.views)) if views is None else views):
        one = E.Scene(sc.name, sc.family, [sc.views[v]], sc.g, sc.exact, sc.tags, sc.mode)
        rctx = _ctx(gs, one)
        d = {q: sc.g[q].to(dev).clone().requires_grad_(grads) for q in E.NAMES}
        img, mask = renderer.render_frame(rctx, *(d[q] for q in E.NAMES), *sc.views[v].args())
        idx, accum = rctx.sorted_instances()
        vis = torch.zeros(sc.n, dtype=torch.uint8, device=dev)
        rctx.visible_into(vis, False)
        r = dict(mask=mask.cpu(), idx=idx.cpu().long(), accum=accum.cpu(), stats=rctx.stats(), vis=vis.cpu())
        if grads:
            go = torch.randn(img.shape, generator=torch.Generator().manual_seed(v)).to(dev)
            (img * go).sum().backward()
            r["grads"] = {q: d[q].grad.cpu() for q in E.NAMES}
        r["img"] = img.detach()
        out.append(r)
    return out


def _check_view(sc, v, r, keys, tiles=None):
    """r (one view's frame) against the decision layer; returns (n decided, n ambiguous)."""
    view, dec = sc.views[v], sc.decide(v)
    n = sc.n
    mask = r["mask"].bool()
    cd = dec.cull_decided
    assert torch.equal(mask[cd], dec.mask[cd]), f"culling: {torch.nonzero(mask[cd] != dec.mask[cd]).flatten()}"
    assert r["stats"]["n_visible"] == int(mask.sum())
    rects = E.device_rects(r["idx"], r["accum"], n, view.ntx)
    for i in range(n):
        t = tuple(int(x) for x in rects[i])
        if bool(dec.decided[i]):
            assert t == tuple(int(x) for x in dec.rect[i]), (i, sc.tags[i], t, dec.rect[i].tolist())
        elif bool(mask[i]):
            assert t in dec.cands[i], (i, sc.tags[i], t, dec.cands[i])
        else:
            assert t == (0, 0, 0, 0), (i, "culled with instances")
    cnt = E.counts_of(rects)
    assert not bool(((cnt > 0) & ~mask).any()), "a culled Gaussian has instances"
    # the exact order on the device's own rectangles and float32 depth keys
    gi, acc = E.expected_lists(dec, rects, view, keys)
    assert torch.equal(r["accum"], acc), "tile ranges"
    assert torch.equal(r["idx"], gi), "instance order"
    assert r["stats"]["n_instances"] == int(cnt.sum())
    # the binned set: visible_mask, and exactly zero gradient rows for everything else
    assert torch.equal(r["vis"].bool(), cnt > 0)
    if "grads" in r:
        for q, gq in r["grads"].items():
            rows = gq.reshape(n, -1)
            assert bool((rows[cnt == 0] == 0).all()), f"gradient rows of unbinned Gaussians ({q})"
    # the image on the oracle's lists
    T = view.ntx * view.nty
    if tiles is None:
        tiles = list(range(T)) if T <= 256 else sorted(set(torch.randint(0, T, (64,), generator=torch.Generator()
                                                                            .manual_seed(T)).tolist()) | {0, T - 1})
    ref = E.draw(dec, gi, acc, view, tiles=tiles)
    img = r["img"]
    for t in tiles:
        ty, tx = divmod(int(t), view.ntx)
        a = img[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16].double().cpu()
        b = ref[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16]
        assert float((a - b).abs().max()) < IMG_ATOL, (t, float((a - b).abs().max()))
    nd = int(dec.decided.sum())
    return nd, n - nd


def _record(sc, nd, na):
    key = (sc.family, sc.mode)
    d, a = _STATS.get(key, (0, 0))
    _STATS[key] = (d + nd, a + na)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (fam, mode), (d, a) in sorted(_STATS.items()):
        print(f"family {fam} {mode}: {d} decided, {a} ambiguous placements")


_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        b = E.BUILDERS.get(name) or E.GRID_BUILDERS[name]
        _SCENES[name] = b()
    return _SCENES[name]


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_single_view(gs, cuda, name):
    sc = _scene(name)
    (r,) = _single(gs, sc, cuda)
    nd, na = _check_view(sc, 0, r, _keys(sc, 0, cuda))
    _record(sc, nd, na)
    assert nd >= 0.9 * sc.n


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_batched_equals_single_views(gs, cuda, name):
    """Family 8: fused_project_batch_kernel against fused_project_kernel (single view) and the oracle."""
    import renderer
    sc = E.batched(_scene(name))
    singles = _single(gs, sc, cuda, grads=False)
    rctx = _ctx(gs, sc)
    vs = sc.views
    img, _, _, mask = renderer.render_frame_batch(
        rctx, *(sc.g[q].to(cuda) for q in E.NAMES), vs[0].width, vs[0].height, [v.fx for v in vs],
        [v.fy for v in vs], torch.stack([v.rot.float() for v in vs]), torch.stack([v.tran.float() for v in vs]),
        vs[0].near, vs[0].thresh, "abs", final=False)
    idx, accum = rctx.sorted_instances()
    idx, accum = idx.cpu().long(), accum.cpu()
    n, T = sc.n, vs[0].ntx * vs[0].nty
    exp_idx, exp_acc, base = [], [], 0
    for v, r in enumerate(singles):
        exp_idx.append(r["idx"] + v * n)
        exp_acc.append(r["accum"][:-1] + base)
        base += int(r["accum"][-1])
        assert torch.equal(mask[v].cpu(), r["mask"]), f"view {v} mask"
    exp_acc.append(torch.tensor([base], dtype=torch.int32))
    assert torch.equal(accum, torch.cat(exp_acc).to(torch.int32)), "batched tile ranges"
    assert torch.equal(idx, torch.cat(exp_idx)), "batched instance order"
    for v, r in enumerate(singles):                 # and each view against the oracle, on the batch's image
        s, e = int(accum[v * T]), int(accum[(v + 1) * T])
        r = dict(r, img=img[v].detach(), idx=idx[s:e] - v * n, accum=(accum[v * T:(v + 1) * T + 1] - s).to(torch.int32))
        nd, na = _check_view(sc, v, r, _keys(sc, v, cuda))
        _record(sc, nd, na)


@pytest.mark.parametrize("name", [k for k in E.BUILDERS if k.endswith("-none") or not k.startswith(
    ("near", "frustum", "unbinned", "borders"))])
def test_packed_path_tile_ranges(gs, cuda, name):
    """pack_sorted_kernel derives tile_accum by its own loops: the same bits as tile_ranges_kernel."""
    sc = _scene(name)
    (ref,) = _single(gs, sc, cuda, grads=False)
    gs[0].tune("gather", 0)
    try:
        (r,) = _single(gs, sc, cuda, grads=False)
    finally:
        gs[0].tune("gather", 1)
    assert torch.equal(r["accum"], ref["accum"])
    assert torch.equal(r["idx"], ref["idx"])
    assert torch.equal(r["mask"], ref["mask"])
    assert torch.equal(r["img"], ref["img"])


@pytest.mark.parametrize("name", list(E.GRID_BUILDERS))
def test_grid_limits(gs, cuda, name):
    """Family 7: key widths (2 bytes up to 65536 tiles, 4 above) and the 16-bit rectangle fields at ntx = 65535 and
    B Hp / 16 = 65535; forward only, the image on sampled tiles."""
    import renderer
    sc = _scene(name)
    if len(sc.views) == 1:
        (r,) = _single(gs, sc, cuda, grads=False)
        nd, na = _check_view(sc, 0, r, _keys(sc, 0, cuda), tiles=sc.sample_tiles)
        _record(sc, nd, na)
        return
    vs = sc.views
    rctx = _ctx(gs, sc)
    img, _, _, mask = renderer.render_frame_batch(
        rctx, *(sc.g[q].to(cuda) for q in E.NAMES), vs[0].width, vs[0].height, [v.fx for v in vs],
        [v.fy for v in vs], torch.stack([v.rot.float() for v in vs]), torch.stack([v.tran.float() for v in vs]),
        vs[0].near, vs[0].thresh, "abs", final=False)
    idx, accum = rctx.sorted_instances()
    idx, accum = idx.cpu().long(), accum.cpu()
    n, T = sc.n, vs[0].ntx * vs[0].nty
    assert rctx.stats()["n_tiles"] == len(vs) * T == 65535 * vs[0].ntx
    for v in range(len(vs)):
        s, e = int(accum[v * T]), int(accum[(v + 1) * T])
        r = dict(mask=mask[v].cpu(), idx=idx[s:e] - v * n, accum=(accum[v * T:(v + 1) * T + 1] - s).to(torch.int32),
                 stats=dict(n_visible=int(mask[v].sum()), n_instances=e - s), vis=None, img=img[v].detach())
        dec = sc.decide(v)
        rects = E.device_rects(r["idx"], r["accum"], n, vs[v].ntx)
        r["vis"] = (E.counts_of(rects) > 0).to(torch.uint8)
        nd, na = _check_view(sc, v, r, _keys(sc, v, cuda), tiles=sc.sample_tiles)
        assert nd == n and int(dec.decided.sum()) == n
        _record(sc, nd, na)


def test_overflowed_projection_is_culled(gs, cuda):
    """p_c.x and p_c.z both overflow float32 (x/z = inf/inf = NaN): the Gaussian is culled (mask 0), like the fp64
    oracle and the decision layer's float32 replay, and gets no instances and no gradient."""
    sc = E.overflow()
    (r,) = _single(gs, sc, cuda)
    dec = sc.decide(0)
    assert torch.equal(r["mask"].bool(), dec.mask), r["mask"].tolist()
    assert r["stats"]["n_visible"] == int(dec.mask.sum())
    for q, gq in r["grads"].items():
        assert bool((gq[:2] == 0).all()), q
