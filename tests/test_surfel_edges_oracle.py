"""CPU checks of the surfel edge fixtures (tests/surfel_edges.py): every builder reaches its designed counts, last
live indices, median indices and margins; the distortion bound separates the kernel's shifted running sums from
unshifted ones; and SO.render(tiles=...) equals the full render on those tiles."""
import pytest
import torch

import helpers as H
import surfel_edges as E
import surfel_oracle as SO

_CACHE = {}


def _fx(name):
    if name not in _CACHE:
        _CACHE[name] = E.BUILDERS[name]()
    return _CACHE[name]


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_builder_reaches_its_design(name):
    fx = _fx(name)                                  # the builders assert their own targets; restate the margins
    p = fx.prof
    assert float(p["stop_margin"].min()) >= 1e-4
    assert float(p["med_margin"].min()) >= (1e-3 if name == "median" else 1e-4)
    assert float(E.edge_distance(*(fx.g[q].double() for q in ("pos", "quat", "scale")), fx.cam).min()) >= 0.01
    assert SO.without_branch_ties(fx.g, fx.cam)["pos"].shape[0] == fx.n
    assert float(fx.g["scale"][:, 2].abs().max()) == 0.0
    # the oracle's binning is the fixture's: confined surfels add one instance to their own tile
    _, _, info = SO.render(*(fx.g[q].double() for q in E.NAMES), fx.cam)
    assert torch.equal(info["accum"].long(), fx.fe["accum"])
    tx0, tx1, ty0, ty1 = info["rects"]
    conf = fx.tile_of >= 0
    assert bool(((tx1 - tx0) * (ty1 - ty0))[conf].eq(1).all())
    assert torch.equal((ty0 * fx.cam.ntx + tx0)[conf], fx.tile_of[conf])
    cnt = p["count"]
    if name == "counts":
        assert sorted(cnt.tolist()) == sorted(list(E.COUNTS) + [0] * (len(cnt) - len(E.COUNTS)))
        assert torch.equal(E.consumed(p, 64), cnt)
    if name == "stops":
        assert sorted(int(p["L"][t]) for t in fx.targets) == sorted(E.STOPS)
        t = list(fx.targets)
        for ch in (E.FWD_CH, E.BWD_CH):                                  # every target tile exits early
            assert bool((E.consumed(p, ch)[t] < cnt[t]).all()), ch
            assert int(E.consumed(p, ch)[fx.tailed]) == int(cnt[fx.tailed])
    if name == "median":
        assert sorted(int(p["med"][t].min()) for t in fx.targets) == sorted(E.MEDIANS)


def test_distortion_bound_sees_the_shift():
    """The kernel's forward distortion restated in fp32 (distortion_fp32): with the m0 shift it stays within
    distortion_bound of the fp64 oracle on every pixel; without it, it exceeds the bound on the narrow-spread tiles."""
    fx = _fx("distortion")
    _, mp, _ = SO.render(*(fx.g[q].double() for q in E.NAMES), fx.cam, dist_near=E.DIST_NEAR, dist_far=E.DIST_FAR)
    ref, bound = mp["distortion"], fx.dist_bound
    shifted = (E.distortion_fp32(fx, shifted=True) - ref).abs()
    unshifted = (E.distortion_fp32(fx, shifted=False) - ref).abs()
    assert bool((shifted <= bound).all()), float((shifted / bound).max())
    ratio = torch.where(unshifted > 0, unshifted / bound, torch.zeros_like(bound))
    narrow = torch.ones(fx.cam.nty, fx.cam.ntx, dtype=torch.bool)
    narrow.view(-1)[fx.control] = False
    narrow = narrow.repeat_interleave(16, 0).repeat_interleave(16, 1)
    # most pixels with a distortion at all fail, by a wide factor
    lit = narrow & (ref > 0)
    assert float((ratio[lit] > 1).double().mean()) > 0.5
    assert float(ratio.max()) > 100


def test_render_tiles_equals_the_full_render_on_those_tiles():
    g, _, cam = H.scene(120, 72, 56, seed=4)
    g = {k: v.clone() for k, v in g.items()}
    g["scale"][:, 2] = 0.0
    g = SO.without_branch_ties(g, cam)
    tiles = [0, 5, 11, 13, 19]
    gen = torch.Generator().manual_seed(1)
    w_img = torch.randn(cam.Hp, cam.Wp, 3, generator=gen, dtype=torch.float64)
    w_map = {k: torch.randn(cam.Hp, cam.Wp, *((3,) if k == "normal" else ()), generator=gen, dtype=torch.float64)
             for k in E.SO_MAPS}
    mask = torch.zeros(cam.nty, cam.ntx, dtype=torch.bool)
    mask.view(-1)[tiles] = True
    mask = mask.repeat_interleave(16, 0).repeat_interleave(16, 1)

    def run(sub):
        p = {k: v.double().clone().requires_grad_(True) for k, v in g.items()}
        img, mp, _ = SO.render(*(p[q] for q in E.NAMES), cam, background=E.BG, tiles=sub)
        m3 = mask[..., None]
        loss = (img * w_img * m3).sum() + sum(((mp[k] * w_map[k]) * (m3 if k == "normal" else mask)).sum()
                                              for k in E.SO_MAPS)
        grads = torch.autograd.grad(loss, [p[q] for q in E.NAMES])
        return img.detach(), {k: v.detach() for k, v in mp.items()}, grads

    full, part = run(None), run(tiles)
    assert torch.equal(full[0][mask], part[0][mask])
    assert float(part[0][~mask].abs().max()) == 0.0
    for k in E.SO_MAPS:
        assert torch.equal(full[1][k][mask], part[1][k][mask]), k
    for a, b in zip(full[2], part[2]):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-14)
    assert float(part[2][0].abs().max()) > 0
