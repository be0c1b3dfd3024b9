"""CPU checks of the front-end edge scenes (tests/bin_edges.py): each scene is what it claims to be.  Exact placements
are exact in float32 and sit on, and one ulp either side of, their boundary; decided placements are at least delta
from every truncation that matters; the float32 replay of gs_oracle.tile_rects gives the decided rectangles; and the
emission, tile-range and grid scenes have the designed count patterns, empty runs and grid sizes."""
import math

import pytest
import torch

import bin_edges as E
import gs_oracle as O

_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        _CACHE[name] = (E.BUILDERS.get(name) or E.GRID_BUILDERS[name])()
    return _CACHE[name]


@pytest.mark.parametrize("name", list(E.BUILDERS) + list(E.GRID_BUILDERS))
def test_decided_placements_keep_their_margin(name):
    sc = _scene(name)
    for v, view in enumerate(sc.views[:2]):
        dec = sc.decide(v)
        assert int(dec.decided.sum()) >= 0.9 * sc.n, (int(dec.decided.sum()), sc.n)
        # the claimed exact placements are exact in float32
        assert bool(E.exact_culling(sc.g, view)[sc.exact].all())
        # every edge of a decided rectangle: delta from an integer, or clamped the same way on [E - delta, E + delta]
        c4 = dec.cov.reshape(-1, 4)
        for i in torch.nonzero(dec.decided & (E.counts_of(dec.rect) > 0)).flatten().tolist():
            a, b, c, d = (float(t) for t in c4[i])
            det = a * d - b * c
            sx = math.sqrt(a / (det + 1e-14) * view.t2 * det)
            sy = math.sqrt(d / (det + 1e-14) * view.t2 * det)
            cx, cy = float(dec.p[i, 0]), float(dec.p[i, 1])
            edges = [(cx - sx - view.leftmost) / view.lx, (cx + sx - view.leftmost) / view.lx,
                     (cy - sy - view.topmost) / view.ly, (cy + sy - view.topmost) / view.ly]
            for j in range(4):
                dl = float(dec.edge_delta[i, j])
                lo, hi = list(edges), list(edges)
                lo[j] -= dl
                hi[j] += dl
                same = E._rect(*lo, view.ntx, view.nty) == E._rect(*hi, view.ntx, view.nty)
                assert same or abs(edges[j] - round(edges[j])) >= dl, (i, j, edges[j], dl)
        # the float32 replay of the oracle's tile rule agrees on every decided placement
        idx = torch.nonzero(dec.mask & dec.keep).flatten()
        rects = O.tile_rects(dec.p[idx, :2], dec.cov[idx], view.thresh, view.lx, view.ly, view.ntx, view.nty,
                             view.leftmost, view.topmost)
        rep = torch.stack(rects, -1)
        rep = torch.where(((rep[:, 1] > rep[:, 0]) & (rep[:, 3] > rep[:, 2])).unsqueeze(-1), rep, 0)
        keep = dec.decided[idx]
        assert torch.equal(rep[keep][:, [0, 1, 2, 3]], dec.rect[idx][keep])


def test_exact_boundaries_are_reached():
    """Family 1 and 2 put exact placements on the boundary and one ulp either side of it, in both directions."""
    near = _scene("near-none")
    v = near.views[0]
    z = near.g["pos"][near.exact, 2].double()
    assert {v.near, E.next_up(v.near), E.next_down(v.near)} <= set(z.tolist())
    dec = near.decide(0)
    assert not bool(dec.mask[near.exact & (near.g["pos"][:, 2].double() <= v.near)].any())
    assert bool(dec.mask[near.exact & (near.g["pos"][:, 2].double() == E.next_up(v.near))].any())
    fr = _scene("frustum-none")
    v = fr.views[0]
    p = fr.g["pos"].double()
    xr, yr = (p[:, 0] / p[:, 2]).abs(), (p[:, 1] / p[:, 2]).abs()
    for r, h in ((xr, v.half_w), (yr, v.half_h)):
        got = set(r[fr.exact].tolist())
        assert {h, E.next_up(h), E.next_down(h)} <= got
    dec = fr.decide(0)
    assert not bool(dec.mask[fr.exact & ((xr == v.half_w) | (yr == v.half_h))].any())
    assert bool(dec.mask[fr.exact & (xr == E.next_down(v.half_w)) & (yr == 0)].all())


def test_unbinned_family():
    """Visible Gaussians with no tile (outside the padded grid, det underflowing to 0) exist in every variant."""
    for mode in ("none", "antialias", "opencv"):
        sc = _scene(f"unbinned-{mode}")
        dec = sc.decide(0)
        vis0 = dec.mask & (E.counts_of(dec.rect) == 0) & dec.decided
        tags = {sc.tags[i] for i in torch.nonzero(vis0).flatten().tolist()}
        assert {"outside", "det0"} <= tags, tags


def _depth_order(sc):
    dec = sc.decide(0)
    cnt = E.counts_of(dec.rect)
    key = torch.where(cnt > 0, dec.p[:, 2].float(), torch.tensor(float("inf")))
    order = torch.argsort(key, stable=True)
    return cnt[order]


def test_emission_patterns():
    warps = {}
    for p in E.EMISSION:
        c = _depth_order(_scene(f"emit-{p}"))
        warps[p] = [c[k:k + E.WARP] for k in range(0, c.numel(), E.WARP)]
    assert [int(w.sum()) for w in warps["n1"]] == [1] and [int(w.sum()) for w in warps["n1-empty"]] == [0]
    assert [int(w.sum()) for w in warps["n31"]] == [31]
    assert [int(w.sum()) for w in warps["n33"]] == [32, 1]
    w = warps["n100"]
    assert len(w) == 4 and int((w[1] > 0).sum()) == 31 and int(w[1][31]) == 0 and int(w[3].sum()) == 0
    w = warps["n255"]
    tot = [int(x.sum()) for x in w]
    assert tot[0] == 32 and tot[1] == 33 and tot[2] >= 1025 and tot[7] == 0
    assert int(w[3].max()) == 16                          # a rectangle as wide as the grid
    assert int((w[6] > 0).sum()) == 1 and int(w[6][0]) > 0   # only lane 0
    sc = _scene("emit-n255")
    dec = sc.decide(0)
    keys = dec.p[:, 2].float()[E.counts_of(dec.rect) > 0]
    assert int(torch.unique(keys, return_counts=True)[1].max()) == 6   # exact duplicates: equal keys
    assert len(warps["n257"]) == 9 and int(warps["n257"][8].sum()) == 1
    assert _scene("emit-n100").n % E.WARP != 0


def test_tile_range_scenes():
    for case in E.RANGES:
        sc = _scene(f"ranges-{case}")
        dec = sc.decide(0)
        v = sc.views[0]
        assert bool(dec.decided.all())
        tiles = (dec.rect[:, 2] * v.ntx + dec.rect[:, 0])[E.counts_of(dec.rect) > 0]
        assert sorted(tiles.tolist()) == sc.claims["tiles"]
        keys = sorted(tiles.tolist())
        M = len(keys)
        if case.startswith("m"):
            assert M == int(case[1:])
            assert keys[0] > 0 and keys[-1] < v.ntx * v.nty - 1          # empty tiles before and after
        if case == "m9":
            assert keys[8] - keys[7] > 1                                 # an empty run across an 8-key group
        if case == "m2049":
            assert keys[2048] - keys[2047] > 1                           # ... and across a 2048-key block
        if case == "one-tile":
            assert len(set(keys)) == 1 and M == 2049
        if case == "per-tile":
            assert keys == list(range(v.ntx * v.nty))


def test_grid_scenes():
    t = {name: (_scene(name).views[0].ntx, _scene(name).views[0].nty) for name in E.GRID_BUILDERS}
    assert t["grid-t1"] == (1, 1) and t["grid-t2"] == (2, 1) and math.prod(t["grid-t256"]) == 256
    assert math.prod(t["grid-t257"]) == 257 and math.prod(t["grid-t65536"]) == 65536
    assert math.prod(t["grid-t65792"]) > 65536
    assert t["grid-w65535h16"] == (65535, 1) and t["grid-w65535h32"] == (65535, 2)
    b = _scene("grid-batch15")
    assert len(b.views) * b.views[0].nty == 65535
    sc = _scene("grid-t65536")
    dec = sc.decide(0)
    last = (dec.rect[:, 3] == 256) & (dec.rect[:, 1] == 256)
    assert bool(last.any())                                              # tile id 65535 is used
    assert bool((E.counts_of(_scene("grid-w65535h16").decide(0).rect) == 65535).any())   # a grid-wide rectangle
