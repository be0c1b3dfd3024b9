"""The surfel frame (renderer.render_frame_surfel: surfel.cu, blend_surfel.cu) on the edge fixtures of
tests/surfel_edges.py against the fp64 oracle (tests/surfel_oracle.py) with the per-instance comparator: tile
counts at the 64-record forward and 32-record backward chunk boundaries, tiles that stop on them with long tails,
partial saturation, cropped border tiles, median instances outside the first chunk, and a distortion at m ~ 1 with a
1 % depth spread.  Also the forward's and backward's exact consumed counts, stale gradient rows of a second frame, a
3DGS backward between two surfel frames, and a full-size frame's properties.  The oracle runs once per fixture and
output kind."""
import pytest
import torch

import helpers as H
import surfel_edges as E
import surfel_oracle as SO

pytestmark = pytest.mark.gpu


def _cases():
    c = []
    for fx in E.BUILDERS:
        for kind in ("rgb", "maps", "sh16-maps"):
            c.append((fx, kind, True))
    c += [("stops", "exp-maps", True), ("stops", "rgb", False), ("stops", "maps", False),
          ("median", "median-only", True)]
    return c


CASES = _cases()


class _Cache:
    def __init__(self):
        self.fx, self.ref = {}, {}

    def fixture(self, name):
        if name not in self.fx:
            self.fx[name] = E.BUILDERS[name]()
        return self.fx[name]

    def oracle(self, name, kind, final=True):
        if (name, kind, final) not in self.ref:
            self.ref[(name, kind, final)] = E.oracle(self.fixture(name), kind, final)
        return self.ref[(name, kind, final)]


@pytest.fixture(scope="module")
def cache(gs):
    return _Cache()


def _frame(gs, fx, kind, final=True, rctx=None, opa=None):
    """One surfel frame + backward of fixture fx for kind's upstream weights; outputs, gradients, the sorted
    instances, the forward's per-tile consumed counts and the frame statistics."""
    import renderer
    dev = torch.device("cuda", 0)
    rctx = rctx if rctx is not None else gs[0].RenderContext()
    if kind.startswith("sh16"):
        rctx.set_sh_eval(gs[0].SH_EVAL_GAUSSIAN)
    p = {q: t.to(dev).contiguous().requires_grad_(True) for q, t in fx.params(kind, torch.float32).items()}
    if opa is not None:
        p["opa"] = opa.to(dev).contiguous().requires_grad_(True)
    v = fx.view
    img, mp, _ = renderer.render_frame_surfel(rctx, *(p[q] for q in E.NAMES), v.width, v.height, v.fx, v.fy, v.rot,
                                              v.tran, v.near, 0.05, "exp" if kind.startswith("exp") else "abs", E.BG,
                                              final, kind != "rgb", E.DIST_NEAR, E.DIST_FAR)
    w = fx.weights(kind, final)
    loss = sum(((img if k == "image" else mp[k]) * wk.float().to(dev)).sum() for k, wk in w.items())
    loss.backward()
    torch.cuda.synchronize()
    ids, accum = rctx.sorted_instances()
    return dict(image=img.detach().cpu(), maps={k: t.detach().cpu() for k, t in mp.items()},
                grads={q: p[q].grad.detach().cpu() for q in E.NAMES}, ids=ids.cpu().long(), accum=accum.cpu().long(),
                consumed=rctx.tile_consumed().cpu().long(), stats=rctx.stats(), rctx=rctx)


def _consumed_fails(fx, got):
    fails = []
    cnt = fx.prof["count"]
    want = E.consumed(fx.prof, E.FWD_CH)
    if not torch.equal(got["consumed"], want):
        bad = (got["consumed"] != want).nonzero().flatten()[:4].tolist()
        fails.append(f"forward consumed: tiles {bad}: got {[int(got['consumed'][t]) for t in bad]}, want "
                     f"{[int(want[t]) for t in bad]} (count {[int(cnt[t]) for t in bad]})")
    want_b = int(E.consumed(fx.prof, E.BWD_CH)[cnt > 0].sum())
    if got["stats"]["n_instances_eff_bwd"] != want_b:
        fails.append(f"n_instances_eff_bwd {got['stats']['n_instances_eff_bwd']} != {want_b}")
    return fails


@pytest.mark.parametrize("fixture,kind,final", CASES)
def test_fixture_vs_oracle(gs, cache, fixture, kind, final):
    fx = cache.fixture(fixture)
    ref = cache.oracle(fixture, kind, final)
    got = _frame(gs, fx, kind, final)
    assert torch.equal(got["accum"], ref["accum"]), "tile ranges differ from the oracle's"
    assert torch.equal(got["ids"], ref["gi"]), "instance order differs from the oracle's"
    fails = E.compare(fx, got, ref, final=final, maps=kind != "rgb") + _consumed_fails(fx, got)
    assert not fails, fails


def test_stale_rows_do_not_leak(gs, cache):
    """Two frames in one RenderContext with the same geometry (same binning and gradient rows); the second raises
    the walls' opacities from 0.5 to 0.97, so it stops earlier and the first frame's tail rows stay in the workspace:
    they must not reach its gradients."""
    fx = cache.fixture("stops")
    ref = cache.oracle("stops", "maps")
    weak = torch.where(fx.tile_of < 0, torch.zeros_like(fx.g["opa"]), fx.g["opa"])
    rctx = gs[0].RenderContext()
    first = _frame(gs, fx, "maps", rctx=rctx, opa=weak)
    got = _frame(gs, fx, "maps", rctx=rctx)
    assert torch.equal(first["accum"], got["accum"]) and torch.equal(first["ids"], got["ids"])
    assert bool((first["consumed"] >= got["consumed"]).all()) and bool((first["consumed"] > got["consumed"]).any())
    fails = E.compare(fx, got, ref) + _consumed_fails(fx, got)
    assert not fails, fails


def test_a_3dgs_backward_between_two_surfel_frames(gs, cache):
    """The 3DGS and surfel backwards share the gradient rows and their epoch tags at different row widths: a surfel
    frame after a 3DGS frame and backward in the same context is bit-equal to the one before."""
    import renderer
    fx = cache.fixture("stops")
    rctx = gs[0].RenderContext()
    a = _frame(gs, fx, "maps", rctx=rctx)
    dev = torch.device("cuda", 0)
    p = {q: fx.g[q].to(dev).clone().requires_grad_(True) for q in E.NAMES}
    v = fx.view
    img, _ = renderer.render_frame_final(rctx, *(p[q] for q in E.NAMES), v.width, v.height, v.fx, v.fy, v.rot, v.tran,
                                         v.near, 0.05, "abs")
    img.backward(torch.ones_like(img))
    torch.cuda.synchronize()
    assert rctx.stats()["n_instances_eff_bwd"] > 0
    b = _frame(gs, fx, "maps", rctx=rctx)
    assert torch.equal(a["image"], b["image"])
    for k in E.SO_MAPS:
        assert torch.equal(a["maps"][k], b["maps"][k]), k
    for q in E.NAMES:
        assert torch.equal(a["grads"][q], b["grads"][q]), q


def test_full_size_properties(gs):
    """1920 x 1080, 500k surfels (helpers.scene geometry, scale[:, 2] = 0), maps on: bit-equal reruns, finite
    outputs, monotone tile ranges ending at the instance count, camera z non-decreasing within tiles, a backward
    linear in the upstream gradient, and the image and maps of 6 tiles inside the crop against the oracle."""
    import renderer
    g, v, cam = H.scene(500_000, 1920, 1080, seed=21)
    g = {k: t.clone() for k, t in g.items()}
    g["scale"][:, 2] = 0.0
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(22)
    w1 = {k: torch.randn(cam.height, cam.width, *((3,) if k in ("image", "normal") else ()), generator=gen)
          for k in ("image",) + E.SO_MAPS}
    w2 = {k: torch.randn(t.shape, generator=gen) for k, t in w1.items()}
    rctx = gs[0].RenderContext()

    def run(w):
        p = {q: g[q].to(dev).requires_grad_(True) for q in E.NAMES}
        img, mp, _ = renderer.render_frame_surfel(rctx, *(p[q] for q in E.NAMES), cam.width, cam.height, cam.fx,
                                                  cam.fy, cam.rot, cam.tran, cam.near, 0.05, "abs", E.BG, True, True)
        loss = sum(((img if k == "image" else mp[k]) * wk.to(dev)).sum() for k, wk in w.items())
        loss.backward()
        torch.cuda.synchronize()
        return img.detach().cpu(), {k: t.detach().cpu() for k, t in mp.items()}, [p[q].grad.cpu() for q in E.NAMES]

    a = run(w1)
    ids, accum = (t.cpu().long() for t in rctx.sorted_instances())
    n_inst = rctx.stats()["n_instances"]
    b = run(w1)
    assert torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in E.SO_MAPS)
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    assert bool(torch.isfinite(a[0]).all()) and all(bool(torch.isfinite(t).all()) for t in a[1].values())
    assert all(bool(torch.isfinite(t).all()) for t in a[2])
    assert bool((accum[1:] >= accum[:-1]).all()) and int(accum[0]) == 0 and int(accum[-1]) == n_inst
    key = (g["pos"] @ cam.rot.float().T + cam.tran.float())[:, 2]
    cnt = accum[1:] - accum[:-1]
    top = (cam.Hp - cam.height) // 2
    inside = [t for t in range(cam.ntx * cam.nty) if t // cam.ntx * 16 >= top and t // cam.ntx * 16 + 16 <= top + cam.height]
    heavy = max(inside, key=lambda t: int(cnt[t]))
    sample = [heavy] + [inside[i] for i in torch.randperm(len(inside), generator=gen)[:5].tolist()]
    for t in sample:
        z = key[ids[int(accum[t]):int(accum[t + 1])]]
        assert bool((z[1:] >= z[:-1]).all()), t
    c = run(w2)
    d = run({k: w1[k] + w2[k] for k in w1})
    for x, y, s in zip(a[2], c[2], d[2]):
        assert H.rel_err(x + y, s) < 1e-3
    pd = {q: g[q].double() for q in E.NAMES}
    rimg, rmp, _ = SO.render(*(pd[q] for q in E.NAMES), cam, background=E.BG, tiles=sample)
    for t in sample:
        ty, tx = divmod(t, cam.ntx)
        ys, xs = slice(ty * 16 - top, ty * 16 + 16 - top), slice(tx * 16, tx * 16 + 16)
        pys = slice(ty * 16, ty * 16 + 16)
        assert H.abs_err(a[0][ys, xs], rimg[pys, xs].clamp(0, 1)) <= 1e-4, t
        for k in E.SO_MAPS:
            s = max(1.0, float(rmp[k][pys, xs].abs().max())) if k in ("depth", "median") else 1.0
            assert H.abs_err(a[1][k][ys, xs], rmp[k][pys, xs]) <= 1e-4 * s, (t, k)
