"""CPU checks of the tile-edge fixtures (tests/tile_edges.py): they hit every targeted chunk, round and early-stop
boundary, every live instance's gradient is large enough for a 1e-3 tolerance to see it, the per-tile comparator
fails on single-instance faults injected into the oracle's own sorted lists yet passes the fp32 evaluation, and
the backward variant table equals the dispatch of blend.cu."""
import os
import re

import pytest
import torch

import tile_edges as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLEND_CU = os.path.join(ROOT, "3d-gaussian-splatting_b200", "csrc", "blend.cu")


@pytest.fixture(scope="module")
def fixtures():
    return {name: build() for name, build in E.BUILDERS.items()}


@pytest.fixture(scope="module")
def oracles(fixtures):
    return {name: E.oracle(fx) for name, fx in fixtures.items()}


def _slot(fx):
    """tile and index in the tile's blend order of every Gaussian's first instance (-1 if none)."""
    fe = fx.fe
    tile = torch.full((fx.n,), -1, dtype=torch.int64)
    pos = torch.full((fx.n,), -1, dtype=torch.int64)
    acc = fe["accum"]
    for t in range(len(acc) - 1):
        ids = fe["gi"][int(acc[t]):int(acc[t + 1])]
        first = tile[ids] < 0
        tile[ids[first]] = t
        pos[ids[first]] = torch.arange(ids.numel())[first]
    return tile, pos


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_fixture_hits_targets(fixtures, name):
    fx = fixtures[name]
    pr = fx.profile
    tx0, tx1, ty0, ty1 = fx.fe["rects"]
    assert fx.fe["n_vis"] == fx.n
    conf = fx.tile_of >= 0
    one = ((tx1 - tx0) == 1) & ((ty1 - ty0) == 1) & (ty0 * fx.cam.ntx + tx0 == fx.tile_of)
    assert bool(one[conf].all()), "a confined Gaussian leaves its tile"
    for t, stop in fx.targets.items():
        assert int(pr["last"][t]) == stop, (t, stop, int(pr["last"][t]))
    # fp32 and fp64 make every early-stop decision of the targeted tiles alike (tile_profile's margin)
    aimed = list(fx.targets) + list(fx.partial)
    assert float(pr["margin"][aimed].min()) >= 1e-4, float(pr["margin"][aimed].min())
    if name == "counts":
        got = sorted(int(pr["count"][t]) for t in fx.targets)
        assert got == E.target_counts()
        for ch, st in E.STAGED:                      # STAGES - 1, STAGES, STAGES + 1 chunks of every staged kernel
            for k in (st - 1, st, st + 1):
                assert k * ch in got and k * ch + 1 in got
        assert max(got) >= 1000 and 0 in got
        assert fx.view.width % 16 and fx.view.height % 16          # cropped border tiles
        assert not bool(pr["full"].any())
        tiles, _ = _slot(fx)
        clones = [i for i, r in enumerate(fx.role) if r == "clone"]
        assert len(clones) == 4 and len({tuple(fx.g["pos"][i].tolist()) for i in clones}) == 1
        assert len(set(clones)) == 4 and len({int(tiles[i]) for i in clones}) == 1
    if name == "walls":
        assert sorted(fx.targets.values()) == sorted(E.STOPS)
        for t, stop in fx.targets.items():
            assert bool(pr["full"][t])
            if stop in E.IN_FLIGHT:                  # a long unread tail: copies of later chunks are in flight at the exit
                assert int(pr["count"][t]) - (stop + 1) >= 120
        assert len(fx.partial) == 2 and all(bool(pr["split"][t]) for t in fx.partial)
        assert all(int(pr["last"][t]) == int(pr["count"][t]) - 1 for t in fx.partial)
    if name == "front":
        assert bool(pr["full"].all()) and bool((pr["last"] == 0).all())
        assert sorted(int(c) - 1 for c in pr["count"]) == sorted(E.FRONT_TAILS)


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_live_instances_have_visible_gradients(fixtures, oracles, name):
    """Every live confined instance's colour gradient is >= 1e-2 of its tile's largest (so 1e-3 sees it); every
    instance behind a fully saturated tile's stop has an exactly zero gradient."""
    fx, o = fixtures[name], oracles[name]
    tile, pos = _slot(fx)
    mag = o["grads"]["rgb"].abs().amax(1)
    checked = 0
    for t in fx.targets:
        ids = ((fx.tile_of == t) & (tile == t)).nonzero().flatten()
        if ids.numel() == 0:
            continue
        last = int(fx.profile["last"][t])
        live = ids[pos[ids] <= last]
        dead = ids[pos[ids] > last]
        top = float(mag[ids].max())
        if live.numel():
            assert top > 0
            assert bool((mag[live] >= 1e-2 * top).all()), (t, float(mag[live].min()), top)
        if bool(fx.profile["full"][t]):
            assert bool((o["grads"]["rgb"][dead] == 0).all()) and bool((o["grads"]["pos"][dead] == 0).all())
        checked += live.numel()
    assert checked > 0 or name == "front"       # the front wall leaves nothing live behind it


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_fp32_evaluation_passes(fixtures, oracles, name):
    fx, o = fixtures[name], oracles[name]
    o32 = E.oracle(fx, dtype=torch.float32)
    assert E.compare(fx, o32["grads"], o["grads"], o32["image"], o["image"]) == []


# ---- fault injection: every single-instance fault must fail the comparator ------------------------------------
def _drop(t, k):
    def f(gi, acc):
        p = int(acc[t]) + k
        acc[t + 1:] -= 1
        return torch.cat([gi[:p], gi[p + 1:]]), acc
    return f


def _dup(t, k):
    def f(gi, acc):
        p = int(acc[t]) + k
        acc[t + 1:] += 1
        return torch.cat([gi[:p + 1], gi[p:]]), acc
    return f


def _swap(t, k):
    def f(gi, acc):
        p = int(acc[t]) + k
        gi[p], gi[p + 1] = gi[p + 1].clone(), gi[p].clone()
        return gi, acc
    return f


def _move(t, k):
    """the instance goes to the front of tile t + 1"""
    def f(gi, acc):
        p, e = int(acc[t]) + k, int(acc[t + 1])
        gi[p:e] = torch.roll(gi[p:e], -1)
        acc[t + 1] -= 1
        return gi, acc
    return f


def _faulty(fx, full, mutate, tiles):
    """full-frame gradients with tiles' contributions replaced by the mutated list's (the loss is a sum over tiles)"""
    clean = E.oracle(fx, tiles=tiles)
    bad = E.oracle(fx, mutate=mutate, tiles=tiles)
    return {q: full["grads"][q] - clean["grads"][q] + bad["grads"][q] for q in E.NAMES}


def _tile_with_count(fx, c):
    return next(t for t in fx.targets if int(fx.profile["count"][t]) == c)


def _faults(fx):
    out = []
    if fx.name == "counts":
        t65, t33, t3, t16 = (_tile_with_count(fx, c) for c in (65, 33, 3, 16))
        t1100 = _tile_with_count(fx, 1100)
        for k in (0, 15, 16, 31, 32, 63, 64):
            out.append((f"drop-{k}", _drop(t65, k), [t65]))
        for k in (127, 128, 255, 256, 1099):
            out.append((f"drop-{k}", _drop(t1100, k), [t1100]))
        out.append(("dup-32", _dup(t33, 32), [t33]))
        out.append(("dup-0", _dup(t65, 0), [t65]))
        out.append(("swap-0", _swap(t3, 0), [t3]))
        out.append(("swap-1", _swap(t3, 1), [t3]))
        out.append(("neighbour", _move(t16, 5), [t16, t16 + 1]))
    elif fx.name == "walls":
        # live instances at chunk / round boundaries in front of the walls, the first wall, one duplicated wall
        # (an instance that saturates, or fails to saturate, a tile at its last live index contributes ~1e-4 of it:
        # nothing in fp32 can see it, and nothing needs to)
        for t, stop in fx.targets.items():
            ids = fx.fe["gi"][int(fx.fe["accum"][t]):int(fx.fe["accum"][t + 1])]
            first_wall = int((fx.tile_of[ids] < 0).nonzero().min())
            for k in (0, 7, 8, 15, 16, 31, 32, 63, 64, 127, 128, 255, 256):
                if k < first_wall and k + 8 >= first_wall:
                    out.append((f"drop-{k}-before-stop-{stop}", _drop(t, k), [t]))
            if stop in (32, 64, 128, 256):
                out.append((f"drop-first-wall-{stop}", _drop(t, first_wall), [t]))
                out.append((f"dup-first-wall-{stop}", _dup(t, first_wall), [t]))
    else:
        out.append(("drop-front-wall", _drop(5, 0), [5]))
    return out


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_comparator_sees_faults(fixtures, oracles, name):
    fx, full = fixtures[name], oracles[name]
    faults = _faults(fx)
    assert faults
    for label, mutate, tiles in faults:
        got = _faulty(fx, full, mutate, tiles)
        assert E.compare(fx, got, full["grads"]) != [], label


def test_comparator_sees_stale_row(fixtures, oracles):
    """A gradient row left over from an earlier frame (same scene with weaker walls, so the tail was read then) on
    an instance behind the stop of a saturated tile."""
    fx, full = fixtures["walls"], oracles["walls"]
    walls = fx.tile_of < 0
    weak_opa = torch.where(walls, torch.full_like(fx.g["opa"], -0.5), fx.g["opa"])
    weak = E.oracle(fx, opa=weak_opa)
    tile, pos = _slot(fx)
    stale = [i for i in range(fx.n) if fx.tile_of[i] >= 0 and int(tile[i]) in fx.targets
             and int(pos[i]) > int(fx.profile["last"][int(tile[i])])]
    assert stale
    hit = 0
    for i in stale[::97][:6]:
        if float(weak["grads"]["rgb"][i].abs().max()) == 0:
            continue
        got = {q: g.clone() for q, g in full["grads"].items()}
        for q in E.NAMES:
            got[q][i] = weak["grads"][q][i]
        assert E.compare(fx, got, full["grads"]) != [], i
        hit += 1
    assert hit > 0


# ---- the variant table equals blend.cu's dispatch -----------------------------------------------------------
def _dispatch_keys():
    src = open(BLEND_CU).read()
    body = src[src.index("cudaError_t gs_launch_blend_bwd("):src.index("static bool shipped_rgb_bwd_knobs")]
    blocks = body.split("switch (key) {")[1:]
    return [tuple(int(k) for k in re.findall(r"case (\d+):", b.split("default:")[0])) for b in blocks]


def test_variant_table_matches_dispatch():
    assert _dispatch_keys() == [E.BWD_GATHER_32, E.BWD_GATHER_64, E.BWD_PACKED]
    src = open(BLEND_CU).read()
    enc = re.search(r"const int key = (.*?);", src, re.S).group(1)
    assert re.sub(r"\s+", "", enc) == ("((((tn.bwd_px*10+tn.bwd_ws)*10+tn.bwd_unroll)*10+tn.bwd_stages)*10+tn.bwd_rq)"
                                       "*100+tn.bwd_minb")


@pytest.mark.parametrize("key", sorted(set(E.BWD_GATHER_32 + E.BWD_GATHER_64 + E.BWD_PACKED)))
def test_bwd_key_round_trip(key):
    k = E.decode_bwd_key(key)
    assert E.encode_bwd_key(k) == key
    assert k["bwd_px"] in (4, 8) and k["bwd_ws"] in (0, 1) and k["bwd_unroll"] in (1, 2, 4)
    assert k["bwd_stages"] in (2, 3) and k["bwd_rq"] in (4, 8) and 1 <= k["bwd_minb"] <= 99
